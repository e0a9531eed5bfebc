// lantern_b200 -- the extern "C" layer (include/lantern_b200.h).
//
// Mirrors U/c/lib.cpp (the reference's C shim over index_dense_gt): same argument meaning, same
// error convention (static strings through `lb200_error_t*`, 0/NULL return on failure, no exception
// crosses the ABI).  Every entry point is additionally exported under its reference name
// (`usearch_*`) at the end of the file.
#include <fcntl.h>
#include <stdio.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <mutex>
#include <string>
#include <unordered_set>
#include <vector>

#include "../../include/lantern_b200.h"
#include "distance.cuh"
#include "engine.h"
#include "group.h"

using namespace lb200;

namespace {

// Error strings must outlive the call and never be freed by the caller (usearch.h:35-39): intern them.
const char* intern_error(const std::string& msg) {
    static std::mutex mu;
    static std::unordered_set<std::string> pool;
    std::lock_guard<std::mutex> g(mu);
    return pool.insert(msg).first->c_str();
}

template <typename Fn> void guarded(lb200_error_t* error, Fn&& fn) {
    try {
        fn();
    } catch (const std::exception& e) {
        if (error)
            *error = intern_error(e.what());
    } catch (...) {
        if (error)
            *error = "lantern_b200: unknown failure";
    }
}

Index* as_index(lb200_index_t h) {
    if (!h)
        throw CudaError("null index handle");
    return reinterpret_cast<Index*>(h);
}

struct DeviceTemp { // RAII device scratch for the stateless entry points
    void* p = nullptr;
    explicit DeviceTemp(size_t bytes) { LB_CUDA(cudaMalloc(&p, bytes ? bytes : 1)); }
    ~DeviceTemp() { cudaFree(p); }
    template <typename T> T* as() { return reinterpret_cast<T*>(p); }
};

// host rows (stride) -> device rows in `kind`, 16-byte padded
void upload_rows(const void* host, size_t n, size_t stride, int kind, size_t dims, uint8_t* d_out, size_t row_bytes) {
    const size_t in_bytes = scalar_row_bytes(kind, dims);
    DeviceTemp raw(n * in_bytes);
    LB_CUDA(cudaMemcpy2D(raw.p, in_bytes, host, stride, in_bytes, n, cudaMemcpyHostToDevice));
    launch_cast_rows(raw.p, in_bytes, kind, d_out, row_bytes, kind, dims, n, 0);
    LB_CUDA(cudaDeviceSynchronize());
}

void check_metric_scalar(int metric, int scalar) {
    if (scalar != SK_F32 && scalar != SK_F16 && scalar != SK_I8 && scalar != SK_B1)
        throw CudaError("unsupported scalar kind (f32, f16, i8, b1 are available on the GPU)");
    if (metric != MK_L2SQ && metric != MK_COS && metric != MK_HAMMING)
        throw CudaError("unsupported metric kind (l2sq, cos, hamming are available on the GPU)");
    if (metric == MK_HAMMING && scalar != SK_B1)
        throw CudaError("hamming metric requires b1 scalars (dimensions in bits)");
}

// lb200_init's reading and checking of the options (a group load checks a file against them the same way)
IndexConfig index_config(const lb200_init_options_t* options, const float* codebook) {
    if (!options)
        throw CudaError("null options");
    require_device();
    if (options->metric)
        throw CudaError("custom metric callbacks cannot run on the GPU");
    // options->retriever / retriever_mut / retriever_ctx: Lantern's build.c:512-517 always fills them before usearch_init
    // ("retrievers are not called from here"); they only matter to usearch_view_mem_lazy / usearch_add_external, which
    // refuse on their own.  Accepted and ignored here so that build.c runs unchanged.
    if (options->multi)
        throw CudaError("multi-vector keys are not supported");
    if (options->pq) { // U/c/lib.cpp:135-140, lantern_storage.hpp:90-94
        if (options->num_centroids == 0 || options->num_subvectors == 0)
            throw CudaError("Must provide nonzero values for centroids and subvectors when pq-quantization option is set");
        if (!codebook)
            throw CudaError("pq index needs a codebook");
        if (options->num_centroids > 256)
            throw CudaError("number of centroids must fit in a byte");
        if (options->dimensions % options->num_subvectors != 0)
            throw CudaError("currently vector dimensions must be divisible to num_subvectors");
        if (options->dimensions >= 2000)
            throw CudaError("vectors larger than 2k dimensions not supported");
        if (options->quantization != lb200_scalar_f32_k)
            throw CudaError("pq index stores f32 codebooks only");
    }
    check_metric_scalar(options->metric_kind, options->quantization);
    if (options->dimensions == 0)
        throw CudaError("dimensions must be nonzero");
    IndexConfig cfg;
    cfg.metric_kind = options->metric_kind;
    cfg.scalar_kind = options->quantization;
    cfg.dims = options->dimensions;
    cfg.M = options->connectivity ? options->connectivity : 16; // index.hpp:1249-1250
    cfg.M0 = cfg.M * 2;
    cfg.efc = options->expansion_add ? options->expansion_add : 128;
    cfg.ef = options->expansion_search ? options->expansion_search : 64;
    cfg.pq = options->pq;
    cfg.num_centroids = options->num_centroids;
    cfg.num_subvectors = options->num_subvectors;
    if (cfg.M < 2 || cfg.M > 128)
        throw CudaError("connectivity must be in [2, 128]"); // lantern_hnsw/src/hnsw/options.h:15-27
    if (scalar_row_bytes(cfg.scalar_kind, cfg.dims) > 8192)
        throw CudaError("vectors wider than 8192 bytes are not supported");
    return cfg;
}

} // namespace

extern "C" {

LB200_EXPORT lb200_index_t lb200_init(lb200_init_options_t* options, float* codebook, lb200_error_t* error) {
    lb200_index_t result = nullptr;
    guarded(error, [&] {
        const IndexConfig cfg = index_config(options, codebook);
        result = new Index(cfg, codebook);
    });
    return result;
}

LB200_EXPORT void lb200_free(lb200_index_t h, lb200_error_t* error) {
    guarded(error, [&] { delete reinterpret_cast<Index*>(h); });
}

LB200_EXPORT size_t lb200_size(lb200_index_t h, lb200_error_t* error) {
    size_t r = 0;
    guarded(error, [&] { r = as_index(h)->size(); });
    return r;
}
LB200_EXPORT size_t lb200_capacity(lb200_index_t h, lb200_error_t* error) {
    size_t r = 0;
    guarded(error, [&] { r = as_index(h)->capacity(); });
    return r;
}
LB200_EXPORT size_t lb200_dimensions(lb200_index_t h, lb200_error_t* error) {
    size_t r = 0;
    guarded(error, [&] { r = as_index(h)->config().dims; });
    return r;
}
LB200_EXPORT size_t lb200_connectivity(lb200_index_t h, lb200_error_t* error) {
    size_t r = 0;
    guarded(error, [&] { r = as_index(h)->config().M; });
    return r;
}
LB200_EXPORT size_t lb200_expansion_add(lb200_index_t h, lb200_error_t* error) {
    size_t r = 0;
    guarded(error, [&] { r = as_index(h)->config().efc; });
    return r;
}
LB200_EXPORT size_t lb200_expansion_search(lb200_index_t h, lb200_error_t* error) {
    size_t r = 0;
    guarded(error, [&] { r = as_index(h)->config().ef; });
    return r;
}

LB200_EXPORT lb200_index_metadata_t lb200_index_metadata(lb200_index_t h, lb200_error_t* error) {
    lb200_index_metadata_t m;
    memset(&m, 0, sizeof(m));
    guarded(error, [&] { // U/c/lib.cpp:234-266
        const IndexConfig& c = as_index(h)->config();
        m.init_options.metric_kind = (lb200_metric_kind_t)c.metric_kind;
        m.init_options.quantization = (lb200_scalar_kind_t)c.scalar_kind;
        m.init_options.dimensions = c.dims;
        m.init_options.connectivity = c.M;
        m.init_options.expansion_add = c.efc;
        m.init_options.expansion_search = c.ef;
        m.init_options.pq = c.pq;
        m.init_options.num_centroids = c.pq ? c.num_centroids : 0;
        m.init_options.num_subvectors = c.pq ? c.num_subvectors : 0;
        m.inverse_log_connectivity = 1.0 / log((double)c.M); // index.hpp:1837
        m.neighbors_bytes = c.M * 6 + 4;                      // :1838
        m.neighbors_base_bytes = c.M0 * 6 + 4;                // :1839
        m.dimensions = c.dims;
        m.expansion_search = c.ef;
        m.expansion_add = c.efc;
        m.connectivity = c.M;
        m.metric_kind = (lb200_metric_kind_t)c.metric_kind;
    });
    return m;
}

LB200_EXPORT void lb200_reserve(lb200_index_t h, size_t capacity, lb200_error_t* error) {
    guarded(error, [&] { as_index(h)->reserve(capacity); });
}

LB200_EXPORT void lb200_add(lb200_index_t h, lb200_key_t key, void const* vector, lb200_scalar_kind_t kind, lb200_error_t* error) {
    guarded(error, [&] {
        Index* idx = as_index(h);
        if (idx->size() >= idx->capacity())
            throw CudaError("Reserve capacity ahead of insertions!"); // index.hpp:2514-2517
        idx->add_one_host(key, vector, kind);
    });
}

LB200_EXPORT void lb200_add_batch(lb200_index_t h, lb200_key_t const* keys, void const* vectors, size_t n, size_t stride,
                                  lb200_scalar_kind_t kind, lb200_error_t* error) {
    guarded(error, [&] { as_index(h)->add_host(keys, vectors, n, stride, kind); });
}

LB200_EXPORT void lb200_add_batch_device(lb200_index_t h, lb200_key_t const* host_keys, void const* device_vectors, size_t n,
                                         size_t stride, lb200_scalar_kind_t kind, lb200_error_t* error) {
    guarded(error, [&] { as_index(h)->add_device(host_keys, device_vectors, n, stride, kind); });
}

LB200_EXPORT void lb200_build(lb200_index_t h, lb200_error_t* error) {
    guarded(error, [&] { as_index(h)->build(); });
}

LB200_EXPORT void lb200_last_build_stats(lb200_index_t h, lb200_build_stats_t* stats, lb200_error_t* error) {
    guarded(error, [&] {
        if (!stats)
            throw CudaError("null stats pointer");
        Index* idx = as_index(h);
        std::lock_guard<std::mutex> g(idx->mu_);
        stats->vectors = idx->last_build_n_;
        stats->computed_distances = idx->last_build_dist_;
        stats->algorithmic_bytes = idx->last_build_dist_ * (idx->cfg_.pq ? idx->stored_bytes_ : idx->vec_bytes_);
        stats->device_ms = idx->last_build_ms_;
    });
}

LB200_EXPORT void lb200_set_option(lb200_index_t h, char const* name, size_t value, lb200_error_t* error) {
    guarded(error, [&] {
        Index* idx = as_index(h);
        std::string n(name ? name : "");
        if (n == "build_batch")
            idx->build_batch_ = value;
        else if (n == "build_ratio")
            idx->build_ratio_ = value ? value : 1;
        else if (n == "search_expand")
            idx->search_expand_ = value ? value : 1;
        else if (n == "search_kernel") { // 0 / 1 = one CTA per query, 2 = one warp per query
            if (value > 2)
                throw CudaError("search_kernel: 0, 1 or 2");
            idx->search_kernel_ = value;
        } else if (n == "pq_query_tables") // 1 = precompute a pq search batch's look-up tables when they fit in 1 GB, 0 = never
            idx->pq_query_tables_ = value != 0;
        else if (n == "touched_cap") // testing knob: size of the per-CTA un-visit log
            idx->touched_cap_ = (uint32_t)std::max<size_t>(value, 32);
        else
            throw CudaError("unknown option");
    });
}

LB200_EXPORT size_t lb200_search_ef(lb200_index_t h, void const* query, lb200_scalar_kind_t kind, size_t count, size_t ef,
                                    bool continue_search, lb200_key_t* keys, lb200_distance_t* distances, lb200_error_t* error) {
    size_t found = 0;
    guarded(error, [&] {
        Index* idx = as_index(h);
        std::lock_guard<std::mutex> stream_guard(idx->stream_mu_);
        const size_t qbytes = scalar_row_bytes(kind, idx->config().dims);
        // Streaming (scan.c:240-292 doubles k and passes continue_search=true; index.hpp:3415-3430 then skips what was
        // already returned and resumes from the frontier).  Here the continuation is a fresh search for
        // (already returned + count) neighbours of the same query, of which the new tail is handed out: the caller sees
        // the same contract -- never a result twice, ascending distance -- and, unlike the reference (SURVEY App. A.9),
        // never loses reachable results.
        if (continue_search) {
            if (idx->stream_query_.size() != qbytes || memcmp(idx->stream_query_.data(), query, qbytes) != 0)
                throw CudaError("continue_search: no preceding search of this query on this index");
        } else {
            idx->stream_returned_.clear();
        }
        const size_t skip = idx->stream_returned_.size();
        const size_t want = skip + count;
        if (want > 4096)
            throw CudaError("continue_search: more than 4096 results requested in total");
        std::vector<uint64_t> k(want);
        std::vector<float> d(want);
        size_t c = 0;
        idx->search_host(query, 1, qbytes, kind, want, ef, k.data(), d.data(), &c);
        // hand out the closest `count` results that were not returned before (a wider beam may rank old results
        // differently, so filtering is by key, not by position); dump_to writes only `found` entries (index.hpp:2426-2433)
        std::vector<uint64_t> seen(idx->stream_returned_);
        std::sort(seen.begin(), seen.end());
        for (size_t i = 0; i < c && found < count; ++i) {
            if (std::binary_search(seen.begin(), seen.end(), k[i]))
                continue;
            keys[found] = k[i], distances[found] = d[i];
            idx->stream_returned_.push_back(k[i]);
            ++found;
        }
        idx->stream_query_.assign((const uint8_t*)query, (const uint8_t*)query + qbytes);
    });
    return found;
}

LB200_EXPORT size_t lb200_search(lb200_index_t h, void const* query, lb200_scalar_kind_t kind, size_t count, lb200_key_t* keys,
                                 lb200_distance_t* distances, lb200_error_t* error) {
    return lb200_search_ef(h, query, kind, count, 0, false, keys, distances, error);
}

LB200_EXPORT void lb200_search_batch(lb200_index_t h, void const* queries, size_t nq, size_t stride, lb200_scalar_kind_t kind,
                                     size_t count, size_t ef, lb200_key_t* keys, lb200_distance_t* distances, size_t* counts,
                                     lb200_error_t* error) {
    guarded(error, [&] { as_index(h)->search_host(queries, nq, stride, kind, count, ef, keys, distances, counts); });
}

LB200_EXPORT void lb200_search_batch_device(lb200_index_t h, void const* d_queries, size_t nq, size_t stride,
                                            lb200_scalar_kind_t kind, size_t count, size_t ef, lb200_key_t* d_keys,
                                            lb200_distance_t* d_distances, uint32_t* d_counts, void* cuda_stream,
                                            lb200_error_t* error) {
    guarded(error, [&] {
        as_index(h)->search_device(d_queries, nq, stride, kind, count, ef, d_keys, d_distances, d_counts, (cudaStream_t)cuda_stream);
    });
}

LB200_EXPORT void lb200_last_search_stats(lb200_index_t h, lb200_search_stats_t* stats, lb200_error_t* error) {
    guarded(error, [&] {
        if (!stats)
            throw CudaError("null stats pointer");
        SearchStats s = as_index(h)->last_stats();
        stats->queries = s.queries;
        stats->computed_distances = s.computed_distances;
        stats->base_pops = s.base_pops;
        stats->upper_hops = s.upper_hops;
        stats->algorithmic_bytes = s.algorithmic_bytes;
        stats->kernel_ms = s.kernel_ms;
        stats->limbo_overflows = s.limbo_overflows;
        stats->full_rows_read = s.full_rows_read;
        stats->screen_kind = s.screen_kind;
        stats->screen_dims = s.screen_dims;
        stats->search_kernel = s.search_kernel;
        stats->reserved = 0;
        stats->owner_cycles_produce = s.cycles_produce;
        stats->owner_cycles_screen = s.cycles_screen;
        stats->owner_cycles_evaluate = s.cycles_evaluate;
        stats->owner_cycles_consume = s.cycles_consume;
    });
}

LB200_EXPORT size_t lb200_serialized_length(lb200_index_t h, lb200_error_t* error) {
    size_t r = 0;
    guarded(error, [&] { r = as_index(h)->serialized_length(); });
    return r;
}
LB200_EXPORT void lb200_save_buffer(lb200_index_t h, void* buffer, size_t length, lb200_error_t* error) {
    guarded(error, [&] { as_index(h)->save_buffer(buffer, length); });
}
LB200_EXPORT void lb200_load_buffer(lb200_index_t h, void const* buffer, size_t length, lb200_error_t* error) {
    guarded(error, [&] { as_index(h)->load_buffer(buffer, length); });
}
LB200_EXPORT void lb200_view_buffer(lb200_index_t h, void const* buffer, size_t length, lb200_error_t* error) {
    // a "view" keeps the nodes in the caller's memory in the reference; here the graph must live in HBM
    guarded(error, [&] { as_index(h)->load_buffer(buffer, length); });
}
LB200_EXPORT void lb200_save(lb200_index_t h, char const* path, lb200_error_t* error) {
    guarded(error, [&] {
        Index* idx = as_index(h);
        std::vector<uint8_t> buf(idx->serialized_length());
        size_t n = idx->save_buffer(buf.data(), buf.size());
        FILE* f = fopen(path, "wb");
        if (!f)
            throw CudaError("Can't open file for writing");
        size_t w = fwrite(buf.data(), 1, n, f);
        fclose(f);
        if (w != n)
            throw CudaError("Failed to write the index file");
    });
}
LB200_EXPORT void lb200_load(lb200_index_t h, char const* path, lb200_error_t* error) {
    guarded(error, [&] {
        FILE* f = fopen(path, "rb");
        if (!f)
            throw CudaError("Can't open file for reading");
        fseek(f, 0, SEEK_END);
        long sz = ftell(f);
        fseek(f, 0, SEEK_SET);
        std::vector<uint8_t> buf((size_t)sz);
        size_t r = fread(buf.data(), 1, buf.size(), f);
        fclose(f);
        if (r != buf.size())
            throw CudaError("Failed to read the index file");
        as_index(h)->load_buffer(buf.data(), buf.size());
    });
}
LB200_EXPORT void lb200_view(lb200_index_t h, char const* path, lb200_error_t* error) { lb200_load(h, path, error); }

LB200_EXPORT void lb200_metadata_buffer(void const* buffer, size_t length, lb200_init_options_t* options, lb200_error_t* error) {
    guarded(error, [&] { // U/c/lib.cpp:315-333
        const uint8_t* p = (const uint8_t*)buffer;
        if (length < 80 || memcmp(p, "usearch", 7) != 0)
            throw CudaError("index file: bad magic");
        int metric = 0, scalar = 0;
        switch (p[13]) {
        case 'c': metric = MK_COS; break;
        case 'i': metric = MK_IP; break;
        case 'e': metric = MK_L2SQ; break;
        case 'b': metric = MK_HAMMING; break;
        default: break;
        }
        switch (p[14]) {
        case 1: scalar = SK_B1; break;
        case 4: scalar = SK_F64; break;
        case 5: scalar = SK_F32; break;
        case 6: scalar = SK_F16; break;
        case 15: scalar = SK_I8; break;
        default: break;
        }
        uint64_t dims;
        memcpy(&dims, p + 33, 8);
        options->metric_kind = (lb200_metric_kind_t)metric;
        options->quantization = (lb200_scalar_kind_t)scalar;
        options->dimensions = dims;
        options->multi = p[41] != 0;
        options->connectivity = 0;
        options->expansion_add = 0;
        options->expansion_search = 0;
        options->metric = nullptr;
    });
}

LB200_EXPORT void lb200_metadata(char const* path, lb200_init_options_t* options, lb200_error_t* error) {
    guarded(error, [&] { // U/c/lib.cpp:268-284: only the 80-byte dense head is read
        if (!path || !options)
            throw CudaError("null path or options");
        FILE* f = fopen(path, "rb");
        if (!f)
            throw CudaError("Can't open file for reading");
        uint8_t head[80];
        const size_t r = fread(head, 1, sizeof(head), f);
        fclose(f);
        if (r != sizeof(head))
            throw CudaError("index file: truncated head");
        lb200_error_t inner = nullptr;
        lb200_metadata_buffer(head, sizeof(head), options, &inner);
        if (inner)
            throw CudaError(inner);
    });
}

LB200_EXPORT void lb200_update_header(lb200_index_t h, char* headerp, lb200_error_t* error) {
    guarded(error, [&] {
        if (!headerp)
            throw CudaError("null header buffer");
        as_index(h)->write_header(headerp);
    });
}

LB200_EXPORT size_t lb200_count(lb200_index_t h, lb200_key_t key, lb200_error_t* error) {
    size_t r = 0;
    guarded(error, [&] { r = as_index(h)->count_key(key); });
    return r;
}
LB200_EXPORT bool lb200_contains(lb200_index_t h, lb200_key_t key, lb200_error_t* error) {
    return lb200_count(h, key, error) != 0;
}

LB200_EXPORT uint64_t lb200_header_get_entry_slot(char* headerp) {
    uint64_t res = 0;
    memcpy(&res, headerp + 80 + 32, 6);
    return res;
}
LB200_EXPORT void lb200_header_set_entry_slot(char* headerp, uint64_t entry_slot) { memcpy(headerp + 80 + 32, &entry_slot, 6); }

// i8 distances come from int32 dot products (dp4a): exact up to 131071 dimensions, where 128^2 d still fits
static void check_i8_dims(int scalar_kind, size_t dims) {
    if (scalar_kind == SK_I8 && dims > 131071)
        throw CudaError("i8 rows wider than 131071 dimensions are not supported");
}

LB200_EXPORT void lb200_distance_batch(void const* a, size_t a_stride, void const* b, size_t b_stride, size_t n,
                                       lb200_scalar_kind_t scalar_kind, size_t dimensions, lb200_metric_kind_t metric_kind,
                                       lb200_distance_t* out, lb200_error_t* error) {
    guarded(error, [&] {
        require_device();
        check_metric_scalar(metric_kind, scalar_kind);
        check_i8_dims(scalar_kind, dimensions);
        if (!n)
            return;
        const size_t rb = round_up(scalar_row_bytes(scalar_kind, dimensions), 16);
        DeviceTemp da(n * rb), db(n * rb), dout(n * sizeof(float));
        upload_rows(a, n, a_stride, scalar_kind, dimensions, da.as<uint8_t>(), rb);
        upload_rows(b, n, b_stride, scalar_kind, dimensions, db.as<uint8_t>(), rb);
        launch_pair_distance(distance_mode(metric_kind, scalar_kind), scalar_kind, da.as<uint8_t>(), rb, db.as<uint8_t>(), rb, n,
                             (uint32_t)rb, dout.as<float>(), 0);
        LB_CUDA(cudaMemcpy(out, dout.p, n * sizeof(float), cudaMemcpyDeviceToHost));
    });
}

LB200_EXPORT lb200_distance_t lb200_distance(void const* a, void const* b, lb200_scalar_kind_t scalar_kind, size_t dimensions,
                                             lb200_metric_kind_t metric_kind, lb200_error_t* error) {
    float out = 0.f;
    const size_t bytes = scalar_row_bytes(scalar_kind, dimensions);
    lb200_distance_batch(a, bytes, b, bytes, 1, scalar_kind, dimensions, metric_kind, &out, error);
    return out;
}

LB200_EXPORT void lb200_exact_search_device(void const* d_dataset, size_t dataset_size, size_t dataset_stride,
                                            void const* d_queries, size_t queries_size, size_t queries_stride,
                                            lb200_scalar_kind_t scalar_kind, size_t dimensions, lb200_metric_kind_t metric_kind,
                                            size_t count, lb200_key_t* d_keys, lb200_distance_t* d_distances, void* cuda_stream,
                                            lb200_error_t* error) {
    guarded(error, [&] {
        require_device();
        check_metric_scalar(metric_kind, scalar_kind);
        check_i8_dims(scalar_kind, dimensions);
        cudaStream_t stream = (cudaStream_t)cuda_stream;
        const size_t bytes = scalar_row_bytes(scalar_kind, dimensions);
        const size_t rb = round_up(bytes, 16);
        const uint8_t* data = (const uint8_t*)d_dataset;
        const uint8_t* qs = (const uint8_t*)d_queries;
        size_t dstride = dataset_stride, qstride = queries_stride;
        void *tmp_d = nullptr, *tmp_q = nullptr;
        auto misaligned = [&](const void* p, size_t stride) { return bytes != rb || stride % 16 != 0 || ((uintptr_t)p & 15); };
        if (misaligned(d_dataset, dataset_stride)) {
            LB_CUDA(cudaMallocAsync(&tmp_d, dataset_size * rb, stream));
            launch_cast_rows(d_dataset, dataset_stride, scalar_kind, tmp_d, rb, scalar_kind, dimensions, dataset_size, stream);
            data = (const uint8_t*)tmp_d, dstride = rb;
        }
        if (misaligned(d_queries, queries_stride)) {
            LB_CUDA(cudaMallocAsync(&tmp_q, queries_size * rb, stream));
            launch_cast_rows(d_queries, queries_stride, scalar_kind, tmp_q, rb, scalar_kind, dimensions, queries_size, stream);
            qs = (const uint8_t*)tmp_q, qstride = rb;
        }
        launch_exact(distance_mode(metric_kind, scalar_kind), scalar_kind, data, dataset_size, dstride, qs, queries_size, qstride,
                     (uint32_t)rb, count, d_keys, d_distances, stream);
        if (tmp_d)
            LB_CUDA(cudaFreeAsync(tmp_d, stream));
        if (tmp_q)
            LB_CUDA(cudaFreeAsync(tmp_q, stream));
    });
}

LB200_EXPORT void lb200_exact_search(void const* dataset, size_t dataset_size, size_t dataset_stride, void const* queries,
                                     size_t queries_size, size_t queries_stride, lb200_scalar_kind_t scalar_kind,
                                     size_t dimensions, lb200_metric_kind_t metric_kind, size_t count, size_t threads,
                                     lb200_key_t* keys, size_t keys_stride, lb200_distance_t* distances, size_t distances_stride,
                                     lb200_error_t* error) {
    (void)threads;
    guarded(error, [&] {
        require_device();
        check_metric_scalar(metric_kind, scalar_kind);
        check_i8_dims(scalar_kind, dimensions);
        if (!queries_size || !count)
            return;
        const size_t rb = round_up(scalar_row_bytes(scalar_kind, dimensions), 16);
        DeviceTemp dd(dataset_size * rb), dq(queries_size * rb), dk(queries_size * count * 8), dv(queries_size * count * 4);
        upload_rows(dataset, dataset_size, dataset_stride, scalar_kind, dimensions, dd.as<uint8_t>(), rb);
        upload_rows(queries, queries_size, queries_stride, scalar_kind, dimensions, dq.as<uint8_t>(), rb);
        launch_exact(distance_mode(metric_kind, scalar_kind), scalar_kind, dd.as<uint8_t>(), dataset_size, rb, dq.as<uint8_t>(),
                     queries_size, rb, (uint32_t)rb, count, dk.as<uint64_t>(), dv.as<float>(), 0);
        LB_CUDA(cudaMemcpy2D(keys, keys_stride, dk.p, count * 8, count * 8, queries_size, cudaMemcpyDeviceToHost));
        LB_CUDA(cudaMemcpy2D(distances, distances_stride, dv.p, count * 4, count * 4, queries_size, cudaMemcpyDeviceToHost));
    });
}

LB200_EXPORT void lb200_exact_tc_probe(float const* dataset, size_t dataset_size, float const* queries, size_t queries_size,
                                       size_t dimensions, lb200_metric_kind_t metric_kind, size_t count, uint32_t* plan,
                                       float* eps, float* qn, float* xn, float* cand_d, uint32_t* cand_i, float* dropped_lb,
                                       uint8_t* unsafe, lb200_key_t* keys, lb200_distance_t* distances, lb200_error_t* error) {
    guarded(error, [&] {
        require_device();
        check_metric_scalar(metric_kind, lb200_scalar_f32_k);
        const int dm = distance_mode(metric_kind, SK_F32);
        if (!plan || !eps || !queries_size || !count || (dm != DM_L2SQ && dm != DM_COS) || !dataset_size || count > 192)
            throw CudaError("exact_tc_probe: needs plan, eps, l2sq or cos, queries, rows and 1 <= count <= 192");
        const size_t rb = round_up(dimensions * 4, 16);
        const ExactTcPlan pl = exact_tc_plan(dataset_size, queries_size, count, (uint32_t)rb);
        plan[0] = pl.groups, plan[1] = pl.KP;
        eps[0] = pl.eps.rel, eps[1] = pl.eps.sum, eps[2] = pl.eps.lin, eps[3] = pl.eps.abs;
        if (!cand_d)
            return;
        if (!qn || !xn || !cand_i || !dropped_lb || !unsafe || !keys || !distances)
            throw CudaError("exact_tc_probe: null output buffer");
        DeviceTemp dd(dataset_size * rb), dq(queries_size * rb), dk(queries_size * count * 8), dv(queries_size * count * 4);
        upload_rows(dataset, dataset_size, dimensions * 4, SK_F32, dimensions, dd.as<uint8_t>(), rb);
        upload_rows(queries, queries_size, dimensions * 4, SK_F32, dimensions, dq.as<uint8_t>(), rb);
        const ExactTcProbe probe{qn, xn, cand_d, cand_i, dropped_lb, unsafe};
        launch_exact(dm, SK_F32, dd.as<uint8_t>(), dataset_size, rb, dq.as<uint8_t>(), queries_size, rb, (uint32_t)rb, count,
                     dk.as<uint64_t>(), dv.as<float>(), 0, &probe);
        LB_CUDA(cudaMemcpy(keys, dk.p, queries_size * count * 8, cudaMemcpyDeviceToHost));
        LB_CUDA(cudaMemcpy(distances, dv.p, queries_size * count * 4, cudaMemcpyDeviceToHost));
    });
}

LB200_EXPORT void lb200_search_screen_probe(float const* dataset, size_t dataset_size, float const* queries, size_t queries_size,
                                            size_t dimensions, lb200_metric_kind_t metric_kind, float* lb, float* d,
                                            lb200_error_t* error) {
    guarded(error, [&] {
        require_device();
        check_metric_scalar(metric_kind, lb200_scalar_f32_k);
        const int dm = distance_mode(metric_kind, SK_F32);
        if ((dm != DM_L2SQ && dm != DM_COS) || !dimensions || !lb || !d)
            throw CudaError("search_screen_probe: needs l2sq or cos, dimensions and output buffers");
        if (!dataset_size || !queries_size)
            return;
        const size_t rb = round_up(dimensions * 4, 16);
        DeviceTemp dd(dataset_size * rb), dq(queries_size * rb), dl(queries_size * dataset_size * 4), dv(queries_size * dataset_size * 4);
        upload_rows(dataset, dataset_size, dimensions * 4, SK_F32, dimensions, dd.as<uint8_t>(), rb);
        upload_rows(queries, queries_size, dimensions * 4, SK_F32, dimensions, dq.as<uint8_t>(), rb);
        launch_screen_probe(dm, dd.as<uint8_t>(), dataset_size, dq.as<uint8_t>(), queries_size, (uint32_t)rb, dl.as<float>(), dv.as<float>(), 0);
        LB_CUDA(cudaMemcpy(lb, dl.p, queries_size * dataset_size * 4, cudaMemcpyDeviceToHost));
        LB_CUDA(cudaMemcpy(d, dv.p, queries_size * dataset_size * 4, cudaMemcpyDeviceToHost));
    });
}

LB200_EXPORT void lb200_search_pscreen_probe(float const* dataset, size_t dataset_size, float const* queries, size_t queries_size,
                                             size_t dimensions, lb200_metric_kind_t metric_kind, float const* basis, size_t k, float* lb,
                                             float* d, lb200_error_t* error) {
    guarded(error, [&] {
        require_device();
        check_metric_scalar(metric_kind, lb200_scalar_f32_k);
        const int dm = distance_mode(metric_kind, SK_F32);
        if ((dm != DM_L2SQ && dm != DM_COS) || !dimensions || !lb || !d || k > 112 || (basis && !k))
            throw CudaError("search_pscreen_probe: needs l2sq or cos, dimensions, output buffers and k <= 112 (k >= 1 with a basis)");
        if (!dataset_size || !queries_size)
            return;
        const size_t rb = round_up(dimensions * 4, 16);
        DeviceTemp dd(dataset_size * rb), dq(queries_size * rb), dl(queries_size * dataset_size * 4), dv(queries_size * dataset_size * 4);
        upload_rows(dataset, dataset_size, dimensions * 4, SK_F32, dimensions, dd.as<uint8_t>(), rb);
        upload_rows(queries, queries_size, dimensions * 4, SK_F32, dimensions, dq.as<uint8_t>(), rb);
        std::vector<float> P;
        uint32_t kk = (uint32_t)k;
        if (basis)
            P.assign(basis, basis + k * dimensions);
        else
            kk = ps_choose_basis(dd.as<uint8_t>(), rb, dataset_size, dimensions, true, kk, P);
        float *dP = nullptr, *dPt = nullptr;
        struct FreeBasis {
            float*& a;
            float*& b;
            ~FreeBasis() { cudaFree(a), cudaFree(b); }
        } free_basis{dP, dPt};
        ps_upload_basis(P, dimensions, kk, &dP, &dPt);
        launch_pscreen_probe(dm, dd.as<uint8_t>(), dataset_size, dq.as<uint8_t>(), queries_size, (uint32_t)rb, dimensions, dP, dPt, kk,
                             dl.as<float>(), dv.as<float>(), 0);
        LB_CUDA(cudaMemcpy(lb, dl.p, queries_size * dataset_size * 4, cudaMemcpyDeviceToHost));
        LB_CUDA(cudaMemcpy(d, dv.p, queries_size * dataset_size * 4, cudaMemcpyDeviceToHost));
    });
}

LB200_EXPORT size_t lb200_screen_basis(lb200_index_t h, float* basis, double* seconds, lb200_error_t* error) {
    size_t k = 0;
    guarded(error, [&] {
        Index* idx = as_index(h);
        std::lock_guard<std::mutex> g(idx->mu_);
        k = idx->ps_k_;
        if (basis)
            std::copy(idx->ps_basis_.begin(), idx->ps_basis_.end(), basis);
        if (seconds)
            *seconds = idx->ps_basis_ms_ / 1e3;
    });
    return k;
}

LB200_EXPORT void lb200_pq_probe(lb200_index_t h, int mode, float const* values, uint32_t const* nodes, size_t count, size_t* rows,
                                 size_t* lut_width, float* distances, float* tables, lb200_error_t* error) {
    guarded(error, [&] {
        Index* idx = as_index(h);
        const IndexConfig& c = idx->config();
        if (!c.pq)
            throw CudaError("pq_probe: not a pq index");
        if (mode < 0 || mode > 2)
            throw CudaError("pq_probe: mode 0 (batch tables), 1 (tables built in the kernel) or 2 (node tables)");
        idx->flush_staged();
        std::lock_guard<std::mutex> g(idx->mu_);
        if (idx->pending_n_)
            throw CudaError("pq_probe: the index has vectors that are not built yet");
        GraphView gv = idx->view();
        if (rows)
            *rows = gv.n;
        if (lut_width)
            *lut_width = gv.pq_lut_width;
        if (!distances || !count || !gv.n)
            return;
        if (!tables || (mode == 2 ? !nodes : !values))
            throw CudaError("pq_probe: null input or output buffer");
        if (mode == 2)
            for (size_t i = 0; i < count; ++i)
                if (nodes[i] >= gv.n)
                    throw CudaError("pq_probe: node id out of range");
        const size_t vrow = round_up(c.dims * 4, 16), tf = (size_t)c.num_subvectors * gv.pq_lut_width;
        DeviceTemp dv(mode == 2 ? count * 4 : count * vrow), dd(count * gv.n * 4), dl(count * (tf + 1) * 4),
            dt(mode == 0 ? count * pq_table_floats((uint32_t)c.num_subvectors, gv.pq_lut_width) * 4 : 0);
        if (mode == 2)
            LB_CUDA(cudaMemcpy(dv.p, nodes, count * 4, cudaMemcpyHostToDevice));
        else
            upload_rows(values, count, c.dims * 4, SK_F32, c.dims, dv.as<uint8_t>(), vrow);
        if (mode == 0) {
            launch_pq_query_tables(idx->d_codebook_, c.dims, c.num_subvectors, gv.pq_lut_width, idx->dist_mode_ == DM_COS, dv.as<float>(),
                                   vrow / 4, count, dt.as<float>(), 0);
            gv.pq_query_tables = dt.as<float>();
        }
        // the search kernel's candidate capacity for this index
        const uint32_t cand_cap = (uint32_t)(c.M0 * std::min<size_t>(std::max<size_t>(idx->search_expand_, 1), 8));
        launch_pq_probe(idx->dist_mode_, gv, cand_cap, mode == 2 ? nullptr : dv.as<uint8_t>(), (uint32_t)vrow,
                        mode == 2 ? dv.as<uint32_t>() : nullptr, count, dd.as<float>(), dl.as<float>(), 0);
        LB_CUDA(cudaMemcpy(distances, dd.p, count * gv.n * 4, cudaMemcpyDeviceToHost));
        LB_CUDA(cudaMemcpy(tables, dl.p, count * (tf + 1) * 4, cudaMemcpyDeviceToHost));
    });
}

LB200_EXPORT void lb200_cast_batch(void const* vectors_f32, size_t count, size_t dims, lb200_scalar_kind_t to, void* result,
                                   lb200_error_t* error) {
    guarded(error, [&] {
        require_device();
        if (!count)
            return;
        const size_t out_bytes = scalar_row_bytes(to, dims);
        if (!out_bytes)
            throw CudaError("cast: unsupported target scalar kind");
        DeviceTemp din(count * dims * 4), dout(count * out_bytes);
        LB_CUDA(cudaMemcpy(din.p, vectors_f32, count * dims * 4, cudaMemcpyHostToDevice));
        launch_cast_rows(din.p, dims * 4, SK_F32, dout.p, out_bytes, to, dims, count, 0);
        LB_CUDA(cudaMemcpy(result, dout.p, count * out_bytes, cudaMemcpyDeviceToHost));
    });
}

LB200_EXPORT void lb200_cast(lb200_scalar_kind_t from, void const* vector, lb200_scalar_kind_t to, void* result,
                             size_t result_size, int dims, lb200_error_t* error) {
    guarded(error, [&] {
        if (from != lb200_scalar_f32_k)
            throw CudaError("cast: only f32 sources are supported");
        if (result_size < scalar_row_bytes(to, (size_t)dims))
            throw CudaError("cast: result buffer too small");
    });
    if (error && *error)
        return;
    lb200_cast_batch(vector, 1, (size_t)dims, to, result, error);
}

LB200_EXPORT void lb200_quantize_pq(float const* codebook, size_t dims, size_t num_centroids, size_t num_subvectors,
                                    float const* vectors, size_t count, uint8_t* codes, int compat128, lb200_error_t* error) {
    guarded(error, [&] {
        require_device();
        if (!num_subvectors || !num_centroids || num_centroids > 256 || dims % num_subvectors)
            throw CudaError("pq: bad codebook geometry");
        if (!count)
            return;
        DeviceTemp dcb(num_centroids * dims * 4), dv(count * dims * 4), dc(count * num_subvectors);
        LB_CUDA(cudaMemcpy(dcb.p, codebook, num_centroids * dims * 4, cudaMemcpyHostToDevice));
        LB_CUDA(cudaMemcpy(dv.p, vectors, count * dims * 4, cudaMemcpyHostToDevice));
        launch_pq_encode(dcb.as<float>(), dims, num_centroids, num_subvectors, dv.as<float>(), dims, count, dc.as<uint8_t>(),
                         num_subvectors, compat128 != 0, 0);
        LB_CUDA(cudaMemcpy(codes, dc.p, count * num_subvectors, cudaMemcpyDeviceToHost));
    });
}

LB200_EXPORT void lb200_dequantize_pq(float const* codebook, size_t dims, size_t num_centroids, size_t num_subvectors,
                                      uint8_t const* codes, size_t count, float* vectors, lb200_error_t* error) {
    guarded(error, [&] {
        require_device();
        if (!num_subvectors || !num_centroids || num_centroids > 256 || dims % num_subvectors)
            throw CudaError("pq: bad codebook geometry");
        if (!count)
            return;
        for (size_t i = 0; i < count * num_subvectors; ++i)
            if (codes[i] >= num_centroids)
                throw CudaError("corrupted centroid id"); // lantern_storage.hpp:141
        DeviceTemp dcb(num_centroids * dims * 4), dv(count * dims * 4), dc(count * num_subvectors);
        LB_CUDA(cudaMemcpy(dcb.p, codebook, num_centroids * dims * 4, cudaMemcpyHostToDevice));
        LB_CUDA(cudaMemcpy(dc.p, codes, count * num_subvectors, cudaMemcpyHostToDevice));
        launch_pq_decode(dcb.as<float>(), dims, num_centroids, num_subvectors, dc.as<uint8_t>(), num_subvectors, count, dv.as<float>(), 0);
        LB_CUDA(cudaMemcpy(vectors, dv.p, count * dims * 4, cudaMemcpyDeviceToHost));
    });
}

LB200_EXPORT int lb200_train_pq_device(void const* d_vectors, size_t stride, size_t count, size_t dims, size_t num_subvectors,
                                       size_t num_centroids, lb200_metric_kind_t metric_kind, size_t max_iter, uint64_t seed,
                                       uint32_t const* init_rows, float* codebook, lb200_error_t* error) {
    int rounds = 0;
    guarded(error, [&] {
        require_device();
        if (metric_kind != lb200_metric_l2sq_k && metric_kind != lb200_metric_cos_k)
            throw CudaError("pq training: l2sq or cos");
        if (stride % 4)
            throw CudaError("pq training: stride must be a multiple of 4 bytes");
        if (num_centroids > 256)
            throw CudaError("number of centroids must fit in a byte");
        DeviceTemp dcb(num_centroids * dims * 4);
        rounds = train_pq_codebook((const float*)d_vectors, stride / 4, count, dims, num_subvectors, num_centroids,
                                   metric_kind == lb200_metric_cos_k, max_iter, seed, init_rows, dcb.as<float>(), 0);
        LB_CUDA(cudaMemcpy(codebook, dcb.p, num_centroids * dims * 4, cudaMemcpyDeviceToHost));
    });
    return rounds;
}

LB200_EXPORT int lb200_train_pq(float const* vectors, size_t count, size_t dims, size_t num_subvectors, size_t num_centroids,
                                lb200_metric_kind_t metric_kind, size_t max_iter, uint64_t seed, uint32_t const* init_rows,
                                float* codebook, lb200_error_t* error) {
    int rounds = 0;
    guarded(error, [&] {
        require_device();
        DeviceTemp dv(count * dims * 4);
        LB_CUDA(cudaMemcpy(dv.p, vectors, count * dims * 4, cudaMemcpyHostToDevice));
        lb200_error_t e2 = nullptr;
        rounds = lb200_train_pq_device(dv.p, dims * 4, count, dims, num_subvectors, num_centroids, metric_kind, max_iter, seed,
                                       init_rows, codebook, &e2);
        if (e2)
            throw CudaError(e2);
    });
    return rounds;
}

LB200_EXPORT void lb200_merge_shards_device(lb200_key_t const* d_keys, lb200_distance_t const* d_dists, size_t shards, size_t nq,
                                            size_t count, lb200_key_t* d_out_keys, lb200_distance_t* d_out_dists,
                                            void* cuda_stream, lb200_error_t* error) {
    guarded(error, [&] {
        require_device();
        launch_merge_shards(d_keys, d_dists, shards, nq, count, d_out_keys, d_out_dists, (cudaStream_t)cuda_stream);
    });
}

// ---- row-sharded multi-GPU group (group.cu) ---------------------------------------------------------------------
static Group* as_group(lb200_group_t h) {
    if (!h)
        throw CudaError("null group handle");
    return reinterpret_cast<Group*>(h);
}
LB200_EXPORT lb200_group_t lb200_group_create(int rank, int world, lb200_allgather_fn allgather, void* allgather_ctx,
                                              lb200_error_t* error) {
    lb200_group_t r = nullptr;
    guarded(error, [&] { r = group_create_ipc(rank, world, allgather, allgather_ctx); });
    return r;
}
LB200_EXPORT lb200_group_t lb200_group_create_local(int const* devices, int n_devices, lb200_error_t* error) {
    lb200_group_t r = nullptr;
    guarded(error, [&] { r = group_create_local(devices, n_devices); });
    return r;
}
LB200_EXPORT void lb200_group_free(lb200_group_t h, lb200_error_t* error) {
    guarded(error, [&] { group_free(reinterpret_cast<Group*>(h)); });
}
static size_t group_max_batch(size_t max_batch) { return max_batch ? max_batch : 8192; }
static size_t group_max_results(size_t max_batch, size_t max_results) {
    return max_results ? max_results : group_max_batch(max_batch) * 128;
}
LB200_EXPORT void lb200_group_distribute(lb200_group_t h, lb200_index_t root_index, int root, size_t max_batch, size_t max_results,
                                         lb200_error_t* error) {
    guarded(error, [&] {
        group_distribute(*as_group(h), reinterpret_cast<Index*>(root_index), root, group_max_batch(max_batch),
                         group_max_results(max_batch, max_results));
    });
}
// lb200_init's reading of the options; a group cannot hold PQ codes (distribute refuses PQ indexes the same way)
static IndexConfig group_load_config(const lb200_init_options_t* options) {
    if (options && options->pq)
        throw CudaError("group: pq indexes are not supported");
    return index_config(options, nullptr);
}
LB200_EXPORT void lb200_group_load_buffer(lb200_group_t h, lb200_init_options_t const* options, void const* buffer, size_t length,
                                          int root, size_t max_batch, size_t max_results, lb200_error_t* error) {
    guarded(error, [&] {
        Group& G = *as_group(h);
        const IndexConfig cfg = group_load_config(options);
        if (!buffer && length)
            throw CudaError("null buffer");
        group_load(G, cfg, buffer, length, root, group_max_batch(max_batch), group_max_results(max_batch, max_results));
    });
}
// A read-only mapping of a whole file: the pages are read as the load touches them, and may be dropped again by the kernel
struct MappedFile {
    int fd = -1;
    void* p = MAP_FAILED;
    size_t length = 0;
    explicit MappedFile(const char* path) {
        fd = open(path, O_RDONLY | O_CLOEXEC);
        if (fd < 0)
            throw CudaError("Can't open file for reading");
        struct stat st;
        if (fstat(fd, &st) != 0) {
            close(fd);
            throw CudaError("Failed to read the index file");
        }
        length = (size_t)st.st_size;
        if (length) {
            p = mmap(nullptr, length, PROT_READ, MAP_PRIVATE, fd, 0);
            if (p == MAP_FAILED) {
                close(fd);
                throw CudaError("Failed to map the index file");
            }
            madvise(p, length, MADV_SEQUENTIAL);
        }
    }
    ~MappedFile() {
        if (p != MAP_FAILED)
            munmap(p, length);
        close(fd);
    }
    const void* data() const { return p == MAP_FAILED ? nullptr : p; }
};
LB200_EXPORT void lb200_group_load(lb200_group_t h, lb200_init_options_t const* options, char const* path, int root,
                                   size_t max_batch, size_t max_results, lb200_error_t* error) {
    guarded(error, [&] {
        Group& G = *as_group(h);
        const IndexConfig cfg = group_load_config(options);
        if (!path)
            throw CudaError("null path");
        MappedFile f(path);
        group_load(G, cfg, f.data(), f.length, root, group_max_batch(max_batch), group_max_results(max_batch, max_results));
    });
}
LB200_EXPORT void lb200_group_rank_info(lb200_group_t h, int local_rank, lb200_group_rank_info_t* info, lb200_error_t* error) {
    guarded(error, [&] {
        if (!info)
            throw CudaError("null info pointer");
        group_rank_info(*as_group(h), local_rank, *info);
    });
}
LB200_EXPORT void lb200_group_build(lb200_group_t h, lb200_index_t root_index, int root, lb200_error_t* error) {
    guarded(error, [&] { group_build(*as_group(h), reinterpret_cast<Index*>(root_index), root); });
}
LB200_EXPORT void lb200_group_index_init(lb200_group_t h, lb200_init_options_t const* options, size_t capacity, size_t max_batch,
                                         size_t max_results, lb200_error_t* error) {
    guarded(error, [&] {
        Group& G = *as_group(h);
        const IndexConfig cfg = group_load_config(options);
        group_index_init(G, cfg, capacity, group_max_batch(max_batch), group_max_results(max_batch, max_results));
    });
}
LB200_EXPORT void lb200_group_index_load_buffer(lb200_group_t h, lb200_init_options_t const* options, void const* buffer,
                                                size_t length, size_t capacity, size_t max_batch, size_t max_results,
                                                lb200_error_t* error) {
    guarded(error, [&] {
        Group& G = *as_group(h);
        const IndexConfig cfg = group_load_config(options);
        if (!buffer && length)
            throw CudaError("null buffer");
        group_index_load(G, cfg, buffer, length, capacity, group_max_batch(max_batch), group_max_results(max_batch, max_results));
    });
}
LB200_EXPORT void lb200_group_index_load(lb200_group_t h, lb200_init_options_t const* options, char const* path, size_t capacity,
                                         size_t max_batch, size_t max_results, lb200_error_t* error) {
    guarded(error, [&] {
        Group& G = *as_group(h);
        const IndexConfig cfg = group_load_config(options);
        if (!path)
            throw CudaError("null path");
        MappedFile f(path);
        group_index_load(G, cfg, f.data(), f.length, capacity, group_max_batch(max_batch), group_max_results(max_batch, max_results));
    });
}
LB200_EXPORT void lb200_group_index_reserve(lb200_group_t h, size_t capacity, lb200_error_t* error) {
    guarded(error, [&] { group_index_reserve(*as_group(h), capacity); });
}
LB200_EXPORT void lb200_group_index_add_batch(lb200_group_t h, lb200_key_t const* keys, void const* vectors, size_t n, size_t stride,
                                              lb200_scalar_kind_t kind, lb200_error_t* error) {
    guarded(error, [&] { group_index_add(*as_group(h), keys, vectors, n, stride, kind); });
}
LB200_EXPORT void lb200_group_index_set_option(lb200_group_t h, char const* name, size_t value, lb200_error_t* error) {
    guarded(error, [&] { group_index_set_option(*as_group(h), name ? name : "", value); });
}
LB200_EXPORT void lb200_group_index_build(lb200_group_t h, lb200_error_t* error) {
    guarded(error, [&] { group_index_build(*as_group(h)); });
}
LB200_EXPORT size_t lb200_group_index_size(lb200_group_t h, lb200_error_t* error) {
    size_t r = 0;
    guarded(error, [&] { r = group_index_size(*as_group(h)); });
    return r;
}
LB200_EXPORT void lb200_group_index_last_build_stats(lb200_group_t h, lb200_build_stats_t* stats, lb200_error_t* error) {
    guarded(error, [&] {
        if (!stats)
            throw CudaError("null stats pointer");
        size_t vectors = 0, value_bytes = 0;
        uint64_t dist = 0;
        double ms = 0;
        group_index_build_stats(*as_group(h), vectors, dist, ms, value_bytes);
        stats->vectors = vectors;
        stats->computed_distances = dist;
        stats->algorithmic_bytes = dist * value_bytes;
        stats->device_ms = ms;
    });
}
LB200_EXPORT size_t lb200_group_index_serialized_length(lb200_group_t h, lb200_error_t* error) {
    size_t r = 0;
    guarded(error, [&] { r = group_index_serialized_length(*as_group(h)); });
    return r;
}
LB200_EXPORT void lb200_group_index_save_buffer(lb200_group_t h, void* buffer, size_t length, lb200_error_t* error) {
    guarded(error, [&] {
        Group& G = *as_group(h);
        if (!buffer)
            throw CudaError("null buffer");
        uint8_t* p = (uint8_t*)buffer;
        group_index_save(
            G,
            [&](size_t need) {
                if (length < need)
                    throw CudaError("save_buffer: buffer too small (see lb200_group_index_serialized_length)");
            },
            [&](const void* bytes, size_t n) {
                memcpy(p, bytes, n);
                p += n;
            });
    });
}
LB200_EXPORT void lb200_group_index_save(lb200_group_t h, char const* path, lb200_error_t* error) {
    guarded(error, [&] {
        Group& G = *as_group(h);
        if (!path)
            throw CudaError("null path");
        struct File {
            FILE* f = nullptr;
            ~File() {
                if (f)
                    fclose(f);
            }
        } out;
        bool opened = false;
        group_index_save(
            G,
            [&](size_t) { // (the index is built and its length known before the file is created)
                out.f = fopen(path, "wb");
                if (!out.f)
                    throw CudaError("Can't open file for writing");
                opened = true;
            },
            [&](const void* bytes, size_t n) {
                if (fwrite(bytes, 1, n, out.f) != n)
                    throw CudaError("Failed to write the index file");
            });
        const int rc = opened ? fclose(out.f) : 0;
        out.f = nullptr;
        if (rc != 0)
            throw CudaError("Failed to write the index file");
    });
}
LB200_EXPORT void lb200_group_search_batch(lb200_group_t h, void const* queries, size_t nq, size_t stride,
                                           lb200_scalar_kind_t kind, size_t count, size_t ef, lb200_key_t* keys,
                                           lb200_distance_t* distances, size_t* counts, lb200_error_t* error) {
    guarded(error, [&] { group_search_host(*as_group(h), queries, nq, stride, kind, count, ef, keys, distances, counts); });
}
LB200_EXPORT void lb200_group_search_batch_device(lb200_group_t h, void const* d_queries, size_t nq, size_t stride,
                                                  lb200_scalar_kind_t kind, size_t count, size_t ef, lb200_key_t* d_keys,
                                                  lb200_distance_t* d_distances, uint32_t* d_counts, void* cuda_stream,
                                                  lb200_error_t* error) {
    guarded(error, [&] {
        group_search_device(*as_group(h), d_queries, nq, stride, kind, count, ef, d_keys, d_distances, d_counts,
                            (cudaStream_t)cuda_stream);
    });
}
LB200_EXPORT int lb200_group_plan(int world, size_t nq, uint32_t resident_warps, uint32_t owner_slots_max, uint32_t* owners,
                                  uint32_t* helpers) {
    if (world < 1 || world > 8 || !owners || !helpers)
        return 1;
    uint32_t O = 0, H = 0;
    const bool ok = group_plan(world, nq, resident_warps, owner_slots_max, O, H);
    *owners = O, *helpers = H;
    return ok ? 0 : 1;
}

LB200_EXPORT int lb200_group_selftest_exchange(int rank, int world, lb200_allgather_fn allgather, void* ctx) {
    if (world < 1 || world > 8 || rank < 0 || rank >= world || !allgather)
        return 1;
    for (size_t bytes : {(size_t)4, (size_t)136, (size_t)1000}) { // the sizes group creation / distribution exchange
        std::vector<uint8_t> mine(bytes), all(bytes * (size_t)world, 0xEE);
        for (size_t i = 0; i < bytes; ++i)
            mine[i] = (uint8_t)(rank * 31 + i * 7 + bytes);
        allgather(ctx, mine.data(), all.data(), bytes);
        for (int r = 0; r < world; ++r)
            for (size_t i = 0; i < bytes; ++i)
                if (all[(size_t)r * bytes + i] != (uint8_t)(r * 31 + i * 7 + bytes))
                    return 2;
    }
    return 0;
}

LB200_EXPORT void lb200_group_last_stats(lb200_group_t h, int local_rank, lb200_group_stats_t* stats, lb200_error_t* error) {
    guarded(error, [&] {
        if (!stats)
            throw CudaError("null stats pointer");
        GroupStats s;
        group_stats(*as_group(h), local_rank, s);
        stats->rank = s.rank, stats->world = s.world;
        stats->queries = s.queries;
        stats->owner_computed_distances = s.owner_computed_distances;
        stats->owner_base_pops = s.owner_base_pops, stats->owner_upper_hops = s.owner_upper_hops;
        stats->owner_rounds = s.owner_rounds;
        stats->local_rows_evaluated = s.local_rows_evaluated, stats->local_row_bytes = s.local_row_bytes;
        stats->rows_held = s.rows_held;
        stats->kernel_ms = s.kernel_ms;
        stats->owner_cycles_produce = s.owner_cycles_produce, stats->owner_cycles_local = s.owner_cycles_local;
        stats->owner_cycles_wait = s.owner_cycles_wait, stats->owner_cycles_consume = s.owner_cycles_consume;
    });
}

LB200_EXPORT int lb200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        (void)cudaGetLastError();
        return 0;
    }
    return n;
}
LB200_EXPORT char const* lb200_version(void) { return "lantern_b200 0.1.0 (sm_90a)"; }
LB200_EXPORT uint64_t lb200_kernel_launches(void) { return g_kernel_launches.load(); }

// ---- the reference's own symbol names (U/c/usearch.h), same signatures -------------------------------
#define LB_ALIAS(ret, uname, lname, params, args)                                                                      \
    LB200_EXPORT ret uname params { return lname args; }

LB_ALIAS(lb200_index_t, usearch_init, lb200_init, (lb200_init_options_t * o, float* cb, lb200_error_t* e), (o, cb, e))
LB_ALIAS(void, usearch_free, lb200_free, (lb200_index_t h, lb200_error_t* e), (h, e))
LB_ALIAS(size_t, usearch_serialized_length, lb200_serialized_length, (lb200_index_t h, lb200_error_t* e), (h, e))
LB_ALIAS(void, usearch_save, lb200_save, (lb200_index_t h, char const* p, lb200_error_t* e), (h, p, e))
LB_ALIAS(void, usearch_load, lb200_load, (lb200_index_t h, char const* p, lb200_error_t* e), (h, p, e))
LB_ALIAS(void, usearch_view, lb200_view, (lb200_index_t h, char const* p, lb200_error_t* e), (h, p, e))
LB_ALIAS(void, usearch_save_buffer, lb200_save_buffer, (lb200_index_t h, void* b, size_t l, lb200_error_t* e), (h, b, l, e))
LB_ALIAS(void, usearch_load_buffer, lb200_load_buffer, (lb200_index_t h, void const* b, size_t l, lb200_error_t* e), (h, b, l, e))
LB_ALIAS(void, usearch_view_buffer, lb200_view_buffer, (lb200_index_t h, void const* b, size_t l, lb200_error_t* e), (h, b, l, e))
LB_ALIAS(void, usearch_metadata_buffer, lb200_metadata_buffer,
         (void const* b, size_t l, lb200_init_options_t* o, lb200_error_t* e), (b, l, o, e))
LB_ALIAS(uint64_t, usearch_header_get_entry_slot, lb200_header_get_entry_slot, (char* hp), (hp))
LB_ALIAS(void, usearch_header_set_entry_slot, lb200_header_set_entry_slot, (char* hp, uint64_t s), (hp, s))
LB_ALIAS(lb200_index_metadata_t, usearch_index_metadata, lb200_index_metadata, (lb200_index_t h, lb200_error_t* e), (h, e))
LB_ALIAS(size_t, usearch_size, lb200_size, (lb200_index_t h, lb200_error_t* e), (h, e))
LB_ALIAS(size_t, usearch_capacity, lb200_capacity, (lb200_index_t h, lb200_error_t* e), (h, e))
LB_ALIAS(size_t, usearch_dimensions, lb200_dimensions, (lb200_index_t h, lb200_error_t* e), (h, e))
LB_ALIAS(size_t, usearch_connectivity, lb200_connectivity, (lb200_index_t h, lb200_error_t* e), (h, e))
LB_ALIAS(size_t, usearch_expansion_add, lb200_expansion_add, (lb200_index_t h, lb200_error_t* e), (h, e))
LB_ALIAS(size_t, usearch_expansion_search, lb200_expansion_search, (lb200_index_t h, lb200_error_t* e), (h, e))
LB_ALIAS(void, usearch_reserve, lb200_reserve, (lb200_index_t h, size_t c, lb200_error_t* e), (h, c, e))
LB_ALIAS(void, usearch_add, lb200_add, (lb200_index_t h, lb200_key_t k, void const* v, lb200_scalar_kind_t s, lb200_error_t* e),
         (h, k, v, s, e))
LB_ALIAS(size_t, usearch_search_ef, lb200_search_ef,
         (lb200_index_t h, void const* q, lb200_scalar_kind_t s, size_t c, size_t ef, bool cs, lb200_key_t* k,
          lb200_distance_t* d, lb200_error_t* e),
         (h, q, s, c, ef, cs, k, d, e))
LB_ALIAS(size_t, usearch_search, lb200_search,
         (lb200_index_t h, void const* q, lb200_scalar_kind_t s, size_t c, lb200_key_t* k, lb200_distance_t* d, lb200_error_t* e),
         (h, q, s, c, k, d, e))
LB_ALIAS(lb200_distance_t, usearch_distance, lb200_distance,
         (void const* a, void const* b, lb200_scalar_kind_t s, size_t d, lb200_metric_kind_t m, lb200_error_t* e),
         (a, b, s, d, m, e))
LB_ALIAS(void, usearch_exact_search, lb200_exact_search,
         (void const* ds, size_t dn, size_t dst, void const* q, size_t qn, size_t qst, lb200_scalar_kind_t s, size_t d,
          lb200_metric_kind_t m, size_t c, size_t t, lb200_key_t* k, size_t kst, lb200_distance_t* di, size_t dist,
          lb200_error_t* e),
         (ds, dn, dst, q, qn, qst, s, d, m, c, t, k, kst, di, dist, e))
LB_ALIAS(void, usearch_cast, lb200_cast,
         (lb200_scalar_kind_t f, void const* v, lb200_scalar_kind_t t, void* r, size_t rs, int d, lb200_error_t* e),
         (f, v, t, r, rs, d, e))
LB_ALIAS(void, usearch_metadata, lb200_metadata, (char const* p, lb200_init_options_t* o, lb200_error_t* e), (p, o, e))
LB_ALIAS(void, usearch_update_header, lb200_update_header, (lb200_index_t h, char* hp, lb200_error_t* e), (h, hp, e))
LB_ALIAS(size_t, usearch_count, lb200_count, (lb200_index_t h, lb200_key_t k, lb200_error_t* e), (h, k, e))
LB_ALIAS(bool, usearch_contains, lb200_contains, (lb200_index_t h, lb200_key_t k, lb200_error_t* e), (h, k, e))
#undef LB_ALIAS

// ---- the rest of U/c/usearch.h: entry points of the reference's in-Postgres page storage and of label bookkeeping.  They are
// exported so that a binary built against usearch.h links unchanged; each reports, through the usual error convention, why it
// cannot work on a graph that lives in HBM and what to call instead (INTEGRATION.md). -----------------------------------------
static void unsupported(lb200_error_t* error, const char* msg) {
    if (error)
        *error = msg;
}
LB200_EXPORT void usearch_view_mem_lazy(lb200_index_t, char*, lb200_error_t* error) { // usearch.h:174
    unsupported(error, "usearch_view_mem_lazy: nodes cannot be fetched lazily from caller memory into HBM; pass the whole "
                       "index file to usearch_load_buffer");
}
LB200_EXPORT void usearch_set_node_retriever(lb200_index_t, void*, lb200_node_retriever_t, lb200_node_retriever_t,
                                             lb200_error_t* error) { // usearch.h:352-353
    unsupported(error, "usearch_set_node_retriever: external node retrievers are not supported; load the index with "
                       "usearch_load_buffer");
}
LB200_EXPORT void usearch_add_external(lb200_index_t, lb200_key_t, void const*, void*, lb200_scalar_kind_t, int16_t, uint64_t,
                                       lb200_error_t* error) { // usearch.h:355-357
    unsupported(error, "usearch_add_external: node tapes live in HBM, not in caller pages; use usearch_add / lb200_add_batch");
}
LB200_EXPORT int32_t usearch_newnode_level(lb200_index_t, lb200_error_t* error) { // usearch.h:347
    unsupported(error, "usearch_newnode_level: levels are drawn inside lb200_build (same generator as the reference)");
    return 0;
}
LB200_EXPORT size_t usearch_get(lb200_index_t, lb200_key_t, size_t, void*, lb200_scalar_kind_t, lb200_error_t* error) { // :307
    unsupported(error, "usearch_get: not supported (Lantern never calls it); read vectors back with usearch_save_buffer");
    return 0;
}
LB200_EXPORT size_t usearch_remove(lb200_index_t, lb200_key_t, lb200_error_t* error) { // usearch.h:317
    unsupported(error, "usearch_remove: not supported; Lantern marks deletions with label 0 and filters them in scan.c:294-300");
    return 0;
}
LB200_EXPORT size_t usearch_rename(lb200_index_t, lb200_key_t, lb200_key_t, lb200_error_t* error) { // usearch.h:326
    unsupported(error, "usearch_rename: not supported");
    return 0;
}

} // extern "C"

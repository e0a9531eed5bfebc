// lantern_b200 -- Index: device memory management and the host side of search.
//
// Host-side mirror of what index_dense_gt does around the hot path
// (U/include/usearch/index_dense.hpp:1395-1451: cast the incoming vector to the storage scalar kind,
// pick expansion = max(ef, k), run the search, dump keys+distances), for whole batches.
#include "engine.h"

#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "distance.cuh"
#include "screen.cuh"
#include "walk.cuh"

namespace lb200 {

std::atomic<uint64_t> g_kernel_launches{0};

int device_sm_count() {
    static int sms = -1;
    if (sms < 0) {
        int dev = 0;
        LB_CUDA(cudaGetDevice(&dev));
        LB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    }
    return sms;
}

size_t device_smem_optin() {
    int dev = 0, limit = 0;
    LB_CUDA(cudaGetDevice(&dev));
    LB_CUDA(cudaDeviceGetAttribute(&limit, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    return (size_t)limit;
}

void require_device() {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        (void)cudaGetLastError();
        throw CudaError("CUDA device unavailable: lantern_b200 has no CPU fallback");
    }
}

namespace {

__global__ void fill_results_kernel(uint64_t* keys, float* dists, uint32_t* counts, size_t nq, size_t k) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nq * k)
        keys[i] = ~0ull, dists[i] = INFINITY;
    if (counts && i < nq)
        counts[i] = 0;
}

template <typename T> void grow_device(T*& ptr, size_t old_count, size_t new_count, int fill_byte) {
    T* np = nullptr;
    LB_CUDA(cudaMalloc(&np, std::max<size_t>(new_count, 1) * sizeof(T)));
    if (fill_byte >= 0)
        LB_CUDA(cudaMemset(np, fill_byte, std::max<size_t>(new_count, 1) * sizeof(T)));
    if (ptr && old_count)
        LB_CUDA(cudaMemcpy(np, ptr, old_count * sizeof(T), cudaMemcpyDeviceToDevice));
    if (ptr)
        LB_CUDA(cudaFree(ptr));
    ptr = np;
}

} // namespace

Index::Index(const IndexConfig& cfg, const float* codebook) : cfg_(cfg) {
    dist_mode_ = distance_mode(cfg.metric_kind, cfg.scalar_kind);
    vec_bytes_ = scalar_row_bytes(cfg.scalar_kind, cfg.dims);
    row_bytes_ = stored_row_bytes(cfg);
    if (cfg.pq) {
        stored_bytes_ = cfg.num_subvectors;
        LB_CUDA(cudaMalloc(&d_codebook_, cfg.num_centroids * cfg.dims * sizeof(float)));
        LB_CUDA(cudaMemcpy(d_codebook_, codebook, cfg.num_centroids * cfg.dims * sizeof(float), cudaMemcpyHostToDevice));
        LB_CUDA(cudaMalloc(&d_pq_pair_, cfg.num_subvectors * cfg.num_centroids * cfg.num_centroids * sizeof(float)));
        LB_CUDA(cudaMalloc(&d_pq_norm_, cfg.num_subvectors * cfg.num_centroids * sizeof(float)));
        launch_pq_tables(d_codebook_, cfg.dims, cfg.num_centroids, cfg.num_subvectors, dist_mode_ == DM_COS, d_pq_pair_, d_pq_norm_, 0);
        if ((cfg.num_subvectors * std::min<size_t>(cfg.num_centroids, 128) + cfg.dims + 520) * 4 > 200 * 1024)
            throw CudaError("pq: num_subvectors * num_centroids look-up table does not fit in shared memory");
    } else {
        stored_bytes_ = vec_bytes_;
        if (cfg.scalar_kind == SK_F32 && (dist_mode_ == DM_L2SQ || dist_mode_ == DM_COS))
            sq_bytes_ = screen_code_bytes((uint32_t)row_bytes_);
        sq_on_ = sq_bytes_ != 0;
    }
    LB_CUDA(cudaMalloc(&scratch_.counters, 8 * sizeof(unsigned long long)));
    LB_CUDA(cudaMemset(scratch_.counters, 0, 8 * sizeof(unsigned long long)));
    LB_CUDA(cudaEventCreate(&ev0_));
    LB_CUDA(cudaEventCreate(&ev1_));
}

Index::~Index() {
    cudaFree(d_vectors_), cudaFree(d_adj0_), cudaFree(d_upper_ref_), cudaFree(d_upper_adj_), cudaFree(d_keys_);
    cudaFree(d_codebook_), cudaFree(scratch_.visited), cudaFree(scratch_.touched), cudaFree(scratch_.counters);
    cudaFree(d_query_buf_), cudaFree(d_io_buf_), cudaFree(d_warp_aux_);
    cudaFree(d_pq_pair_), cudaFree(d_pq_norm_), cudaFree(d_pending_raw_), cudaFree(d_pq_tables_);
    cudaFree(d_sq_codes_), cudaFree(d_sq_meta_), cudaFree(d_ps_query_);
    free_pscreen();
    if (ev0_)
        cudaEventDestroy(ev0_);
    if (ev1_)
        cudaEventDestroy(ev1_);
}

void Index::ensure_capacity(size_t cap) {
    if (cap <= capacity_)
        return;
    size_t nc = std::max(cap, capacity_ + capacity_ / 2);
    nc = round_up(nc, 32);
    const size_t used = n_ + pending_n_;
    grow_device(d_vectors_, used * row_bytes_, nc * row_bytes_, 0);
    grow_device(d_adj0_, n_ * cfg_.M0, nc * cfg_.M0, 0xFF);
    grow_device(d_upper_ref_, n_, nc, 0xFF);
    grow_device(d_keys_, n_, nc, 0xFF);
    if (sq_on_) {
        grow_device(d_sq_codes_, used * sq_bytes_, nc * sq_bytes_, 0);
        grow_device(d_sq_meta_, used, nc, 0);
    }
    if (ps_k_)
        grow_device(d_ps_records_, used * ps_record_bytes(ps_k_), nc * ps_record_bytes(ps_k_), 0);
    capacity_ = nc;
}

void Index::init_row_range(size_t capacity, size_t lo, size_t hi) {
    if (capacity_ || n_ || pending_n_ || cfg_.pq || lo > hi || hi > capacity)
        throw CudaError("index: a row range needs an empty, non-pq index and lo <= hi <= capacity");
    sq_bytes_ = 0, sq_on_ = false; // a group's owners do not screen
    grow_device(d_vectors_, 0, std::max<size_t>(hi - lo, 1) * row_bytes_, 0);
    grow_device(d_adj0_, 0, capacity * cfg_.M0, 0xFF);
    grow_device(d_upper_ref_, 0, capacity, 0xFF);
    grow_device(d_keys_, 0, capacity, 0xFF);
    capacity_ = capacity;
    sharded_ = true, row_lo_ = lo, row_hi_ = hi;
}

void Index::replace_row_range(size_t capacity, size_t lo, size_t hi, uint8_t* vectors, uint32_t* adj0, uint32_t* upper_ref,
                              uint64_t* keys) {
    if (!sharded_ || lo > hi || hi > capacity || capacity < n_ + pending_n_)
        throw CudaError("index: a new row range needs a row-sharded index, lo <= hi <= capacity and room for its rows");
    cudaFree(d_vectors_), cudaFree(d_adj0_), cudaFree(d_upper_ref_), cudaFree(d_keys_);
    d_vectors_ = vectors, d_adj0_ = adj0, d_upper_ref_ = upper_ref, d_keys_ = keys;
    free_scratch(); // the build's visited bitmaps are sized for the capacity
    capacity_ = capacity, row_lo_ = lo, row_hi_ = hi;
}

void Index::free_scratch() {
    cudaFree(scratch_.visited), cudaFree(scratch_.touched);
    scratch_.visited = nullptr, scratch_.touched = nullptr;
    scratch_.ctas = 0, scratch_.words_per_cta = 0;
}

void Index::encode_screen(size_t first, size_t count) {
    if (sq_on_)
        launch_sq_encode(d_vectors_ + first * row_bytes_, row_bytes_, count, d_sq_codes_ + first * sq_bytes_, d_sq_meta_ + first, 0);
    if (ps_k_)
        launch_ps_encode(d_vectors_ + first * row_bytes_, row_bytes_, count, cfg_.dims, d_ps_basis_, d_ps_basis_t_, ps_k_,
                         dist_mode_ == DM_COS, d_ps_records_ + first * ps_record_bytes(ps_k_), 0);
}

void Index::reserve(size_t capacity) {
    std::lock_guard<std::mutex> g(mu_);
    ensure_capacity(capacity);
}

void Index::alloc_upper(size_t total_lists) {
    if (total_lists <= upper_lists_cap_)
        return;
    size_t nc = std::max(total_lists, upper_lists_cap_ + upper_lists_cap_ / 2);
    grow_device(d_upper_adj_, upper_lists_ * cfg_.M, nc * cfg_.M, 0xFF);
    upper_lists_cap_ = nc;
}

void* Index::io_buffer(size_t bytes) {
    if (bytes > io_buf_bytes_) {
        if (d_io_buf_)
            LB_CUDA(cudaFree(d_io_buf_));
        d_io_buf_ = nullptr;
        io_buf_bytes_ = round_up(bytes + bytes / 4, 256);
        LB_CUDA(cudaMalloc(&d_io_buf_, io_buf_bytes_));
    }
    return d_io_buf_;
}

uint8_t* Index::query_buffer(size_t bytes) {
    if (bytes > query_buf_bytes_) {
        if (d_query_buf_)
            LB_CUDA(cudaFree(d_query_buf_));
        d_query_buf_ = nullptr;
        query_buf_bytes_ = round_up(bytes + bytes / 4, 256);
        LB_CUDA(cudaMalloc(&d_query_buf_, query_buf_bytes_));
    }
    return d_query_buf_;
}

// ---- staging of new vectors (usearch_add: U/c/lib.cpp:357-365 -> index_dense.hpp:1395-1426) ---------
static void check_input_kind(const IndexConfig& cfg, int kind) {
    if (kind == SK_F32)
        return; // cast to the storage kind on the device (f32 -> sign bits for b1 is what cast_gt does)
    if (kind == SK_B1 && cfg.scalar_kind == SK_B1)
        return;
    throw CudaError("vectors must be passed as f32, or as packed bits (b1) for a b1 index");
}

void Index::add_device(const uint64_t* host_keys, const void* d_vectors, size_t n, size_t stride, int kind) {
    std::lock_guard<std::mutex> g(mu_);
    check_input_kind(cfg_, kind);
    if (!n)
        return;
    for (size_t i = 0; i < n; ++i)
        if (host_keys[i] == ~0ull)
            throw CudaError("key UINT64_MAX is reserved (free key)");
    const size_t used = n_ + pending_n_;
    ensure_capacity(used + n);
    if (cfg_.pq) {
        if (kind != SK_F32)
            throw CudaError("pq index takes f32 vectors");
        if (stride % sizeof(float))
            throw CudaError("pq index: vector stride must be a multiple of 4 bytes");
        // stored side: codes (codebook_t::compress, with the reference's 128-centroid loop quirk, lantern_storage.hpp:123)
        launch_pq_encode(d_codebook_, cfg_.dims, cfg_.num_centroids, cfg_.num_subvectors, (const float*)d_vectors,
                         stride / sizeof(float), n, d_vectors_ + used * row_bytes_, row_bytes_, /*compat128=*/true, 0);
        // value side of the build distances: the raw f32 vector (index_dense.hpp:1423-1425), kept until lb200_build
        const size_t raw_row = round_up(cfg_.dims * 4, 16);
        if ((pending_n_ + n) * raw_row > pending_raw_cap_) {
            size_t nc = std::max((pending_n_ + n) * raw_row, pending_raw_cap_ * 2);
            float* np = nullptr;
            LB_CUDA(cudaMalloc(&np, nc));
            if (d_pending_raw_ && pending_n_)
                LB_CUDA(cudaMemcpy(np, d_pending_raw_, pending_n_ * raw_row, cudaMemcpyDeviceToDevice));
            if (d_pending_raw_)
                LB_CUDA(cudaFree(d_pending_raw_));
            d_pending_raw_ = np, pending_raw_cap_ = nc;
        }
        launch_cast_rows(d_vectors, stride, SK_F32, (uint8_t*)d_pending_raw_ + pending_n_ * raw_row, raw_row, SK_F32, cfg_.dims, n, 0);
    } else {
        launch_cast_rows(d_vectors, stride, kind, d_vectors_ + used * row_bytes_, row_bytes_, cfg_.scalar_kind, cfg_.dims, n, 0);
        encode_screen(used, n);
    }
    h_keys_.insert(h_keys_.end(), host_keys, host_keys + n);
    pending_n_ += n;
}

void Index::add_host(const uint64_t* keys, const void* vectors, size_t n, size_t stride, int kind) {
    if (!n)
        return;
    check_input_kind(cfg_, kind);
    std::lock_guard<std::recursive_mutex> hg(host_mu_);
    const size_t in_bytes = scalar_row_bytes(kind, cfg_.dims);
    void* d_tmp = nullptr;
    {
        std::lock_guard<std::mutex> g(mu_);
        d_tmp = io_buffer(n * in_bytes);
        LB_CUDA(cudaMemcpy2D(d_tmp, in_bytes, vectors, stride, in_bytes, n, cudaMemcpyHostToDevice));
    }
    add_device(keys, d_tmp, n, in_bytes, kind);
    LB_CUDA(cudaDeviceSynchronize());
}

// usearch_add (U/c/lib.cpp:357-365) arrives one row at a time from Lantern's heap scan (build.c:83-140): rows are staged on
// the host and handed to the device 4096 at a time; every consumer of the index flushes first.
void Index::add_one_host(uint64_t key, const void* vector, int kind) {
    check_input_kind(cfg_, kind);
    if (key == ~0ull)
        throw CudaError("key UINT64_MAX is reserved (free key)");
    const size_t in_bytes = scalar_row_bytes(kind, cfg_.dims);
    bool full = false;
    {
        std::lock_guard<std::mutex> g(stage_mu_);
        if (!staged_keys_.empty() && staged_kind_ != kind)
            throw CudaError("vectors of one index must all be passed in the same scalar kind");
        staged_kind_ = kind;
        staged_keys_.push_back(key);
        const uint8_t* p = (const uint8_t*)vector;
        staged_rows_.insert(staged_rows_.end(), p, p + in_bytes);
        full = staged_keys_.size() >= 4096;
    }
    if (full)
        flush_staged();
}

void Index::flush_staged() {
    std::vector<uint8_t> rows;
    std::vector<uint64_t> keys;
    int kind;
    {
        std::lock_guard<std::mutex> g(stage_mu_);
        if (staged_keys_.empty())
            return;
        rows.swap(staged_rows_), keys.swap(staged_keys_);
        kind = staged_kind_;
    }
    add_host(keys.data(), rows.data(), keys.size(), scalar_row_bytes(kind, cfg_.dims), kind);
}

// usearch_count / usearch_contains (U/c/lib.cpp:392-400): keys live in a host mirror, no device work
size_t Index::count_key(uint64_t key) {
    size_t c = 0;
    {
        std::lock_guard<std::mutex> g(stage_mu_);
        c += (size_t)std::count(staged_keys_.begin(), staged_keys_.end(), key);
    }
    std::lock_guard<std::mutex> g(mu_);
    return c + (size_t)std::count(h_keys_.begin(), h_keys_.end(), key);
}

void Index::build() {
    flush_staged();
    std::lock_guard<std::mutex> g(mu_);
    if (pending_n_)
        build_pending(*this);
}

GraphView Index::view() const {
    GraphView g{};
    g.vectors = d_vectors_;
    g.adj0 = d_adj0_;
    g.upper_ref = d_upper_ref_;
    g.upper_adj = d_upper_adj_;
    g.keys = d_keys_;
    g.n = (uint32_t)n_;
    g.row_bytes = (uint32_t)row_bytes_;
    g.M = (uint32_t)cfg_.M, g.M0 = (uint32_t)cfg_.M0;
    g.entry = entry_;
    g.max_level = max_level_;
    g.codebook = d_codebook_;
    g.pq_pair = d_pq_pair_;
    g.pq_norm = d_pq_norm_;
    g.dims = (uint32_t)cfg_.dims;
    g.num_centroids = (uint32_t)cfg_.num_centroids;
    g.num_subvectors = (uint32_t)cfg_.num_subvectors;
    g.pq_lut_width = pq_lut_width(cfg_.num_centroids, pq_max_code_);
    g.sq_codes = d_sq_codes_;
    g.sq_meta = d_sq_meta_;
    g.ps_records = reinterpret_cast<const uint4*>(d_ps_records_);
    g.ps_k = ps_k_;
    g.flags = search_view_flags();
    return g;
}

uint32_t search_view_flags() {
    // L2-prefetch the adjacency line of nodes that enter the top list (2); screened search rounds take both halves of a
    // 64-wide list in one bitmap-atomic round trip (8)
    uint32_t flags = 2u | 8u;
    if (const char* e = getenv("LB200_FLAGS"))
        flags = (uint32_t)atoi(e);
    return flags;
}

// Sized for the walks that stage the value in the CTA and build its table there -- every build kernel, and the search of a
// batch whose tables pass 1 GB -- with a top list of one and the level-0 candidates; larger ef or efc only add to it.  A
// search with precomputed tables needs `dims` floats less, so a table that fits only that way could still answer small
// batches, but could never be built on, inserted into or searched in large batches: such a file is refused too.
void Index::check_pq_table_fits(uint32_t lut_width) const {
    const size_t need = walk_layout_pq((uint32_t)cfg_.num_subvectors, lut_width, (uint32_t)cfg_.dims, 1, (uint32_t)cfg_.M0).total;
    int dev = 0, limit = 0;
    LB_CUDA(cudaGetDevice(&dev));
    LB_CUDA(cudaDeviceGetAttribute(&limit, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    if (need > (size_t)limit)
        throw CudaError("pq: the " + std::to_string(cfg_.num_subvectors) + " x " + std::to_string(lut_width) +
                        " look-up table needs " + std::to_string(need) + " bytes of shared memory per CTA; the device allows " +
                        std::to_string(limit));
}

void Index::ensure_scratch(uint32_t ctas) {
    const size_t words = round_up((capacity_ + 31) / 32, 32);
    if (ctas <= scratch_.ctas && words <= scratch_.words_per_cta && scratch_.touched_cap == touched_cap_)
        return;
    if (scratch_.visited)
        LB_CUDA(cudaFree(scratch_.visited));
    if (scratch_.touched)
        LB_CUDA(cudaFree(scratch_.touched));
    scratch_.visited = nullptr, scratch_.touched = nullptr;
    scratch_.ctas = std::max(ctas, scratch_.ctas);
    scratch_.words_per_cta = words;
    scratch_.touched_cap = touched_cap_;
    LB_CUDA(cudaMalloc(&scratch_.visited, (size_t)scratch_.ctas * words * sizeof(uint32_t)));
    LB_CUDA(cudaMemset(scratch_.visited, 0, (size_t)scratch_.ctas * words * sizeof(uint32_t)));
    LB_CUDA(cudaMalloc(&scratch_.touched, (size_t)scratch_.ctas * scratch_.touched_cap * sizeof(uint32_t)));
}

void Index::search_device(const void* d_queries, size_t nq, size_t stride, int kind, size_t k, size_t ef, uint64_t* d_keys,
                          float* d_dists, uint32_t* d_counts, cudaStream_t stream) {
    flush_staged();
    std::lock_guard<std::mutex> g(mu_);
    check_input_kind(cfg_, kind);
    if (!nq || !k)
        return;
    if (pending_n_)
        build_pending(*this);
    if (n_ == 0) { // index.hpp:2693: empty index -> no results
        size_t total = std::max(nq * k, nq);
        fill_results_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(d_keys, d_dists, d_counts, nq, k);
        LB_CUDA(cudaGetLastError());
        count_launch();
        last_nq_ = 0, last_kernel_ = 0;
        return;
    }
    size_t L = ef ? ef : cfg_.ef; // usearch.h:265-271: 0 = index default
    if (L < k)
        L = k; // index.hpp:2706
    if (L > 4096)
        throw CudaError("search: max(ef, count) > 4096 is not supported");
    // queries -> storage scalar kind, 16-byte padded rows (index_dense.hpp:1435-1441); pq: the raw f32 query is the value
    const size_t qrow = cfg_.pq ? round_up(cfg_.dims * 4, 16) : row_bytes_;
    uint8_t* qbuf = query_buffer(nq * qrow);
    launch_cast_rows(d_queries, stride, kind, qbuf, qrow, cfg_.pq ? (int)SK_F32 : cfg_.scalar_kind, cfg_.dims, nq, stream);

    const uint32_t expand = (uint32_t)std::min<size_t>(std::max<size_t>(search_expand_, 1), 8);
    GraphView gv = view();
    if (cfg_.pq) {
        // the batch's look-up tables in one dense launch (49 KB per query at 96 x 128): the walk kernel then fetches a table with
        // one bulk copy instead of computing nsub * ncent * subdim flops per query at 4 CTAs per SM
        const size_t tbytes = nq * pq_table_floats((uint32_t)cfg_.num_subvectors, gv.pq_lut_width) * sizeof(float);
        if (pq_query_tables_ && tbytes <= ((size_t)1 << 30)) {
            if (tbytes > pq_tables_bytes_) {
                if (d_pq_tables_)
                    LB_CUDA(cudaFree(d_pq_tables_));
                d_pq_tables_ = nullptr;
                pq_tables_bytes_ = round_up(tbytes + tbytes / 4, 256);
                LB_CUDA(cudaMalloc(&d_pq_tables_, pq_tables_bytes_));
            }
            launch_pq_query_tables(d_codebook_, cfg_.dims, cfg_.num_subvectors, gv.pq_lut_width, dist_mode_ == DM_COS, (const float*)qbuf,
                                   qrow / sizeof(float), nq, d_pq_tables_, stream);
            gv.pq_query_tables = d_pq_tables_;
        }
    }
    // screen of the level-0 beam (screen.cuh): the projected one when the index chose a basis, else the int8 one; below 1 KB
    // per row the extra dependent fetch per round is unlikely to pay for the bytes it saves.  LB200_SEARCH_SCREEN overrides
    // the choice for experiments (one graph timed every way): 0 = off, 1 = int8, 2 = projected.  A companion the forced kind
    // needs and the index does not keep is encoded here, before the kernel's events.
    int screen = screen_eligible() ? (ps_auto_ ? 2 : sq_on_ ? 1 : 0) : 0;
    if (const char* e = getenv("LB200_SEARCH_SCREEN")) {
        const int v = atoi(e);
        screen = !sq_bytes_ || v == 0 ? 0 : v == 2 ? 2 : 1;
        if (screen == 1)
            set_int8_companion(true);
        else if (screen == 2)
            force_pscreen();
    }
    gv.sq_codes = d_sq_codes_, gv.sq_meta = d_sq_meta_; // a forced kind may just have been encoded
    gv.ps_records = reinterpret_cast<const uint4*>(d_ps_records_), gv.ps_k = ps_k_;
    if (screen == 2) { // the batch's projections (ps_query_kernel), one dense launch
        const size_t qbytes = nq * ps_query_floats(ps_k_) * sizeof(float);
        if (qbytes > ps_query_bytes_) {
            if (d_ps_query_)
                LB_CUDA(cudaFree(d_ps_query_));
            d_ps_query_ = nullptr;
            ps_query_bytes_ = round_up(qbytes + qbytes / 4, 256);
            LB_CUDA(cudaMalloc(&d_ps_query_, ps_query_bytes_));
        }
        launch_ps_queries(d_ps_basis_, d_ps_basis_t_, cfg_.dims, ps_k_, qbuf, qrow, nq, d_ps_query_, stream);
        gv.ps_query = d_ps_query_;
    }
    // Kernel choice: one CTA per query unless "search_kernel" = 2.  One warp per query walks 24 queries per SM instead of 8 with
    // no CTA barriers, and screens with the projected screen like the CTA kernel, but it measured slower even then (DESIGN.md
    // 6: 0.90x at cfg3), so the automatic choice never takes it.
    const bool warp_kernel = !cfg_.pq && expand == 1 && cfg_.M0 <= 256 && search_kernel_ == 2;
    if (warp_kernel) {
        LB_CUDA(cudaEventRecord(ev0_, stream));
        launch_warp_search(*this, qbuf, qrow, nq, k, (uint32_t)L, screen == 2 ? d_ps_query_ : nullptr, d_keys, d_dists, d_counts,
                           stream);
        LB_CUDA(cudaEventRecord(ev1_, stream));
        last_nq_ = (uint32_t)nq;
        last_screen_ = screen == 2 ? 2 : 0;
        last_kernel_ = 2;
        return;
    }
    const uint32_t max_ctas = search_max_ctas(dist_mode_, cfg_.scalar_kind, gv, (uint32_t)L, cfg_.pq, expand, screen);
    ensure_scratch(max_ctas);
    LB_CUDA(cudaMemsetAsync(scratch_.counters, 0, 8 * sizeof(unsigned long long), stream));

    SearchLaunch p{};
    p.g = gv;
    p.s = scratch_;
    p.s.ctas = max_ctas;
    p.queries = qbuf;
    p.query_stride = (uint32_t)qrow;
    p.nq = (uint32_t)nq, p.k = (uint32_t)k, p.L = (uint32_t)L;
    p.expand = expand;
    p.screen = screen;
    p.out_keys = d_keys, p.out_dists = d_dists, p.out_counts = d_counts;
    LB_CUDA(cudaEventRecord(ev0_, stream));
    launch_search(dist_mode_, cfg_.scalar_kind, cfg_.pq, p, stream);
    LB_CUDA(cudaEventRecord(ev1_, stream));
    last_nq_ = (uint32_t)nq;
    last_screen_ = screen;
    last_kernel_ = 1;
}

void Index::search_host(const void* queries, size_t nq, size_t stride, int kind, size_t k, size_t ef, uint64_t* keys,
                        float* dists, size_t* counts) {
    if (!nq || !k)
        return;
    check_input_kind(cfg_, kind);
    std::lock_guard<std::recursive_mutex> hg(host_mu_); // the staging buffer is shared by every host-buffer call of this index
    flush_staged(); // before the io buffer holds the queries: flushing stages rows through the same buffer
    const size_t in_bytes = scalar_row_bytes(kind, cfg_.dims);
    uint8_t* base = nullptr;
    size_t o_keys, o_dists, o_counts;
    {
        std::lock_guard<std::mutex> g(mu_);
        size_t o = round_up(nq * in_bytes, 256);
        o_keys = o, o += round_up(nq * k * sizeof(uint64_t), 256);
        o_dists = o, o += round_up(nq * k * sizeof(float), 256);
        o_counts = o, o += round_up(nq * sizeof(uint32_t), 256);
        base = (uint8_t*)io_buffer(o);
    }
    cudaStream_t stream = 0;
    LB_CUDA(cudaMemcpy2DAsync(base, in_bytes, queries, stride, in_bytes, nq, cudaMemcpyHostToDevice, stream));
    search_device(base, nq, in_bytes, kind, k, ef, (uint64_t*)(base + o_keys), (float*)(base + o_dists),
                  (uint32_t*)(base + o_counts), stream);
    LB_CUDA(cudaMemcpyAsync(keys, base + o_keys, nq * k * sizeof(uint64_t), cudaMemcpyDeviceToHost, stream));
    LB_CUDA(cudaMemcpyAsync(dists, base + o_dists, nq * k * sizeof(float), cudaMemcpyDeviceToHost, stream));
    std::vector<uint32_t> c32;
    if (counts) {
        c32.resize(nq);
        LB_CUDA(cudaMemcpyAsync(c32.data(), base + o_counts, nq * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
    }
    LB_CUDA(cudaStreamSynchronize(stream));
    if (counts)
        for (size_t i = 0; i < nq; ++i)
            counts[i] = c32[i];
}

SearchStats Index::last_stats() {
    std::lock_guard<std::mutex> g(mu_);
    unsigned long long c[8] = {0};
    LB_CUDA(cudaDeviceSynchronize());
    SearchStats s;
    if (last_kernel_ == 2) { // the warp kernel's counters (GroupLaunch::counters) in the search's order
        unsigned long long w[16] = {0};
        LB_CUDA(cudaMemcpy(w, d_warp_aux_, sizeof(w), cudaMemcpyDeviceToHost));
        c[1] = w[1], c[2] = w[2], c[3] = w[3], c[4] = w[7], c[5] = w[12], c[6] = w[13];
        s.cycles_produce = w[8], s.cycles_screen = w[14], s.cycles_evaluate = w[9] + w[10], s.cycles_consume = w[11];
    } else {
        LB_CUDA(cudaMemcpy(c, scratch_.counters, sizeof(c), cudaMemcpyDeviceToHost));
    }
    s.search_kernel = (uint32_t)last_kernel_;
    s.queries = last_nq_;
    if (last_nq_) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, ev0_, ev1_) == cudaSuccess)
            s.kernel_ms = ms;
        else
            (void)cudaGetLastError();
    }
    s.computed_distances = c[1], s.base_pops = c[2], s.upper_hops = c[3], s.limbo_overflows = c[4];
    const uint64_t screened = last_screen_ ? c[5] : 0, rejected = last_screen_ ? c[6] : 0;
    s.full_rows_read = s.computed_distances - rejected;
    s.screen_kind = (uint32_t)last_screen_;
    s.screen_dims = last_screen_ == 1 ? (uint32_t)cfg_.dims : last_screen_ == 2 ? ps_k_ : 0u;
    // SURVEY.md 8(d): B_alg = n_dist*bytes_per_stored_vector + n_pop*(4 + M_level*4) + query bytes, where a screened search
    // reads a code row + its 16 bytes of metadata (int8) or one record (projected) per screened candidate and a stored row
    // only for the rest
    const uint64_t screen_bytes = last_screen_ == 1 ? sq_bytes_ + 16 : last_screen_ == 2 ? ps_record_bytes(ps_k_) : 0;
    s.algorithmic_bytes = screened * screen_bytes + s.full_rows_read * (cfg_.pq ? stored_bytes_ : vec_bytes_) +
                          s.base_pops * (4 + 4 * cfg_.M0) + s.upper_hops * (4 + 4 * cfg_.M) + s.queries * vec_bytes_;
    return s;
}

} // namespace lb200

// lantern_b200 -- host-side index object behind the C ABI (include/lantern_b200.h).
//
// HBM layout of one index (one shard = one GPU):
//   vectors   [capacity][row_bytes]   stored scalar kind (f32/f16/i8/b1), row_bytes = round_up(bytes,16),
//                                     zero padded; base 256-B aligned -> every row is a whole number of
//                                     16-B chunks and (for d=768 f32) of 128-B lines.   PQ: codes[capacity][nsub_pad]
//   adj0      [capacity][M0] u32      level-0 adjacency, stored order, padded with 0xFFFFFFFF
//   upper_ref [capacity] u32          0xFFFFFFFF for level-0-only nodes, else offset/M into upper_adj of the node's
//                                     level-1 list; level l list at (ref + l-1)*M
//   upper_adj [sum(levels)*M] u32     padded with 0xFFFFFFFF
//   keys      [capacity] u64, levels [capacity] i16
//   sq_codes  [capacity][round_up(dims,16)] i8   f32 l2sq / cos only: the search screen's int8 copy of every row (screen.cuh)
//   sq_meta   [capacity] float4                  {scale, bound on |x - x^|, fp32 |x|^2 as the kernel computes it, |codes|}
//   ps_records [capacity][64 or 128]             instead of sq_*, when the index's rows fit a projected basis (pscreen.cu):
//                                                {s, E, F, b2} then k int8 codes of P x
//   scratch   per resident CTA: visited bitmap (capacity bits) + touched-word list
// The reference keeps the same information in per-node byte tapes with 6-byte slots
// (U/include/usearch/index.hpp:1799-1863); only the (de)serialiser here speaks that format.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <functional>
#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"

namespace lb200 {

struct IndexConfig {
    int metric_kind = MK_L2SQ;
    int scalar_kind = SK_F32;
    size_t dims = 0;
    size_t M = 16, M0 = 32, efc = 128, ef = 64;
    bool pq = false;
    size_t num_centroids = 0, num_subvectors = 0;
};

struct SearchStats {
    uint64_t queries = 0, computed_distances = 0, base_pops = 0, upper_hops = 0, algorithmic_bytes = 0, limbo_overflows = 0;
    uint64_t full_rows_read = 0; // stored rows actually read: computed_distances minus the candidates the screen rejected
    uint32_t screen_kind = 0;    // 0 = no screen, 1 = int8 codes, 2 = projected codes
    uint32_t screen_dims = 0;    // codes per screened candidate: dims (int8) or k (projected)
    double kernel_ms = 0; // device time of the search kernel alone (CUDA events on the launching stream)
    uint32_t search_kernel = 0;  // 1 = one CTA per query (search.cu), 2 = one warp per query (group.cu)
    // one warp per query: SM cycles of the walks' rounds, summed over walks (zero for the CTA kernel)
    uint64_t cycles_produce = 0, cycles_screen = 0, cycles_evaluate = 0, cycles_consume = 0;
};

// Device-side view handed to kernels (plain pointers, trivially copyable).
struct GraphView {
    const uint8_t* vectors;
    const uint32_t* adj0;
    const uint32_t* upper_ref;
    const uint32_t* upper_adj;
    const uint64_t* keys;
    uint32_t n;
    uint32_t row_bytes; // bytes per stored row (multiple of 16)
    uint32_t M, M0;
    uint32_t entry;
    int32_t max_level;
    // PQ (row_bytes then is the padded code width)
    const float* codebook; // [num_centroids][dims]
    const float* pq_pair;  // [nsub][ncent][ncent] centroid-pair table (l2sq: |ca-cb|^2 ; cos: ca.cb)
    const float* pq_norm;  // [nsub][ncent] |centroid slice|^2 (cos)
    const float* pq_query_tables; // search only: per-query look-up tables [nq][pq_table_floats] precomputed for the batch, or NULL
    uint32_t flags;        // tuning: 1 = L2-prefetch the adjacency of every measured node, 2 = of accepted nodes only;
                           // 8 = screened search rounds visit a 64-wide list in one bitmap-atomic round trip
    uint32_t dims, num_centroids, num_subvectors;
    uint32_t pq_lut_width; // centroids the per-value table covers (= num_centroids, or 128 when every stored code is < 128)
    // search screen (f32 l2sq / cos): int8 code rows of screen_code_bytes(row_bytes) and their metadata, or NULL
    const uint8_t* sq_codes;
    const float4* sq_meta;
    // projected screen: records of ps_record_bytes(ps_k), and the search batch's pre-pass (ps_query_floats(ps_k) per query)
    const uint4* ps_records;
    const float* ps_query;
    uint32_t ps_k;
};

// The projected screen's basis (pscreen.cu): chosen from the first build (or load) that leaves kPsMinRows rows, as the smallest
// k of kPsDims whose mean residual energy |x - P^T P x|^2 / |x|^2 over a sample of at most kPsSampleMax rows is <= kPsMaxResidual
constexpr size_t kPsMinRows = 16384;
constexpr size_t kPsSampleMax = 65536;
constexpr double kPsMaxResidual = 0.01;
constexpr uint32_t kPsDims[] = {16, 32, 48, 64, 96, 112};
// above 256 dimensions the top eigenvectors come from subspace iteration with this many vectors and iterations (pscreen.cu)
constexpr size_t kPsSubspace = 128;
constexpr int kPsSubspaceIters = 12;
// rows of at least this many bytes take a screened search path when the index keeps a companion
constexpr size_t kScreenMinRowBytes = 1024;

// Floats of one value's PQ look-up table: [nsub][lut_width] padded to whole 16-byte chunks, then |value|^2 and 3 spare floats.
// Precomputed tables travel to shared memory by bulk copy, whose size and addresses must be multiples of 16 bytes.
LB_HD inline size_t pq_table_floats(uint32_t nsub, uint32_t lut_width) { return (nsub * lut_width + 7u) & ~3u; }

// Centroids a PQ look-up table covers.  The reference's encoder never emits centroid ids >= 128 (signed-char loop,
// lantern_storage.hpp:123) and neither does lb200_add*: then half of a 256-entry table can never be addressed and is not
// built (half the shared memory).  A loaded file whose codes reach 128 needs every centroid.
inline uint32_t pq_lut_width(size_t num_centroids, uint32_t max_code) {
    return (uint32_t)((num_centroids > 128 && max_code < 128) ? 128 : num_centroids);
}

// Bytes of one stored row in HBM: the vector (or PQ code) padded to whole 16-byte chunks
inline size_t stored_row_bytes(const IndexConfig& cfg) {
    return round_up(cfg.pq ? cfg.num_subvectors : scalar_row_bytes(cfg.scalar_kind, cfg.dims), 16);
}
// GraphView::flags of every search (LB200_FLAGS overrides the default; engine.cu)
uint32_t search_view_flags();

// A usearch/lantern index file, parsed and validated on the host against an index configuration (format.cu): the one parser
// behind Index::load_buffer and the group's load.  Every check of the file happens here; the rows stay in the caller's buffer
// (node i's stored bytes start at row_off[i]).
struct ParsedIndexFile {
    size_t n = 0;
    uint32_t entry = 0;
    int32_t max_level = -1;
    std::vector<uint32_t> adj0, upper_ref, upper_adj; // the HBM layout (engine.h top): u32 ids, 0xFFFFFFFF padded
    std::vector<int16_t> levels;
    std::vector<uint64_t> keys;
    std::vector<uint64_t> row_off;
};
// vec_bytes / stored_bytes: those of an index with `cfg` (Index::vec_bytes_, stored_bytes_)
void parse_index_file(const IndexConfig& cfg, size_t vec_bytes, size_t stored_bytes, const void* buffer, size_t length,
                      ParsedIndexFile& out);

struct SearchScratch {
    uint32_t* visited;     // [ctas][words_per_cta]
    uint32_t* touched;     // [ctas][touched_cap]
    unsigned long long* counters; // [0]=next query, [1]=dist evals, [2]=base pops, [3]=upper hops, [4]=limbo overflows,
                                  // [5]=candidates screened, [6]=candidates the screen rejected (8 slots)
    size_t words_per_cta;
    uint32_t touched_cap;
    uint32_t ctas;
};

class Index {
  public:
    explicit Index(const IndexConfig& cfg, const float* codebook);
    ~Index();

    const IndexConfig& config() const { return cfg_; }
    size_t size() const { return n_ + pending_n_ + staged_keys_.size(); }
    size_t capacity() const { return capacity_; }
    size_t row_bytes() const { return row_bytes_; }

    void reserve(size_t capacity);
    // staging (host or device source) of vectors in the *input* kind (f32 or b1)
    void add_host(const uint64_t* keys, const void* vectors, size_t n, size_t stride, int kind);
    void add_device(const uint64_t* host_keys, const void* d_vectors, size_t n, size_t stride, int kind);
    void add_one_host(uint64_t key, const void* vector, int kind); // usearch_add: staged on the host, flushed in blocks
    void flush_staged();                                           // caller holds no lock
    void build(); // insert all pending vectors (build.cu)

    // search: queries in device memory, input kind f32 or b1
    void search_device(const void* d_queries, size_t nq, size_t stride, int kind, size_t k, size_t ef, uint64_t* d_keys,
                       float* d_dists, uint32_t* d_counts, cudaStream_t stream);
    void search_host(const void* queries, size_t nq, size_t stride, int kind, size_t k, size_t ef, uint64_t* keys,
                     float* dists, size_t* counts);
    SearchStats last_stats();

    // usearch/lantern file format (format.cc)
    size_t serialized_length();
    size_t serialized_length_locked(); // caller holds mu_
    size_t save_buffer(void* buffer, size_t length);
    void load_buffer(const void* buffer, size_t length);
    void write_header(void* headerp);      // 136 bytes (usearch_update_header)
    void fill_header(uint8_t* p) const;    // caller holds mu_
    size_t count_key(uint64_t key);        // usearch_count: vectors stored under `key`

    GraphView view() const;

    // --- used by build.cu / format.cc ---
    void ensure_capacity(size_t cap);
    void alloc_upper(size_t total_lists);
    // one rank's part of a group's own index (group.cu): d_vectors_ holds rows [lo, hi) only (row i at (i - lo) * row_bytes_);
    // lists, levels and keys are sized for all `capacity` rows.  No search-screen companion.  Called once, on an empty index.
    void init_row_range(size_t capacity, size_t lo, size_t hi);
    // the same index at a new capacity and row range, contents kept: the caller has copied rows [lo, min(hi, size)) into
    // `vectors` and the lists, upper references and keys of all rows into arrays sized for `capacity` (0xFF beyond them);
    // the old arrays and the build scratch are freed.  Nothing here allocates or throws once the arguments pass.
    void replace_row_range(size_t capacity, size_t lo, size_t hi, uint8_t* vectors, uint32_t* adj0, uint32_t* upper_ref, uint64_t* keys);
    // the graph state of a parsed file (format.cu): lists, upper references and keys on the device (0xFF beyond them), then
    // n, entry, top level and upper-list count; `host_mirrors`: the levels and keys on the host too, moved out of `f`.  The
    // rows are the caller's, and so is a capacity of at least f.n.  The level generator is not touched.
    void commit_file_graph(ParsedIndexFile& f, bool host_mirrors);
    void free_scratch(); // the visited bitmaps and touched lists (they grow with capacity x resident CTAs)

    IndexConfig cfg_;
    int dist_mode_ = 0;
    size_t row_bytes_ = 0;    // stored row (or padded PQ code) bytes
    size_t vec_bytes_ = 0;    // unpadded bytes of a vector in the metric scalar kind (file format)
    size_t stored_bytes_ = 0; // unpadded bytes kept per node in the file (vec_bytes_ or num_subvectors)
    size_t n_ = 0, capacity_ = 0;
    bool sharded_ = false;            // init_row_range: this index holds the rows [row_lo_, row_hi_) of a group's index
    size_t row_lo_ = 0, row_hi_ = 0;
    int32_t max_level_ = -1;
    uint32_t entry_ = 0;
    uint32_t level_rng_ = 1u;   // minstd_rand0 state, default seed (std::default_random_engine, index.hpp:2082)
    size_t build_batch_ = 0;    // max nodes inserted per batch; 0 = one per resident CTA; 1 = the reference's sequential order
    size_t build_ratio_ = 64;   // a batch never exceeds (visible nodes) / build_ratio_
    uint32_t touched_cap_ = 16384; // per-CTA log of bitmap words to un-visit; beyond it the whole bitmap is cleared
    size_t search_expand_ = 1;  // 1 = exact-order search; 2..4 = relaxed order (see walk.cuh)
    size_t search_kernel_ = 0;  // 0 / 1 = one CTA per query (search.cu), 2 = one warp per query (group.cu)
    bool pq_query_tables_ = true; // pq search: precompute the batch's look-up tables when they fit in 1 GB; false = never
    uint8_t* d_warp_aux_ = nullptr; // warp kernel: counters, flags, dummy counts
    size_t warp_aux_bytes_ = 0;
    double last_build_ms_ = 0;
    uint64_t last_build_dist_ = 0;
    size_t last_build_n_ = 0;

    // device arrays
    uint8_t* d_vectors_ = nullptr;
    uint32_t* d_adj0_ = nullptr;
    uint32_t* d_upper_ref_ = nullptr;
    uint32_t* d_upper_adj_ = nullptr;
    size_t upper_lists_ = 0, upper_lists_cap_ = 0; // number of M-wide lists in d_upper_adj_
    uint64_t* d_keys_ = nullptr;
    float* d_codebook_ = nullptr;
    float* d_pq_pair_ = nullptr;
    float* d_pq_norm_ = nullptr;
    float* d_pq_tables_ = nullptr; // per-query look-up tables of the current search batch
    size_t pq_tables_bytes_ = 0;
    uint32_t pq_max_code_ = 0; // largest centroid id present in the stored codes
    float* d_pending_raw_ = nullptr; // pq: raw f32 rows of the pending vectors (the value side of build distances)
    // search screen companion (f32 storage, l2sq / cos, not PQ): written from d_vectors_ by launch_sq_encode
    uint8_t* d_sq_codes_ = nullptr;
    float4* d_sq_meta_ = nullptr;
    size_t sq_bytes_ = 0; // bytes of one code row; 0 = this index cannot keep the int8 companion
    bool sq_on_ = false;  // the int8 companion is allocated and kept up to date
    // projected screen (pscreen.cu): basis [k][dims] (host), device P [slots][dims] and P^T [dims][slots], records [capacity]
    uint32_t ps_k_ = 0; // 0 = no basis
    std::vector<float> ps_basis_;
    float* d_ps_basis_ = nullptr;
    float* d_ps_basis_t_ = nullptr;
    uint8_t* d_ps_records_ = nullptr;
    float* d_ps_query_ = nullptr; // the search batch's pre-pass
    size_t ps_query_bytes_ = 0;
    bool ps_decided_ = false;  // the automatic choice has been made
    bool ps_auto_ = false;     // ... and it is the projected screen (a basis may also exist because LB200_SEARCH_SCREEN=2 forced one)
    double ps_basis_ms_ = 0;   // host time of the last basis choice (moment matrix, eigenvectors, records)
    int last_screen_ = 0;      // screen kind of the last search
    int last_kernel_ = 0;      // search kernel of the last search: 1 = one CTA per query, 2 = one warp per query
    size_t pending_raw_cap_ = 0;
    // host mirrors of the small per-node metadata
    std::vector<int16_t> h_levels_;
    std::vector<uint64_t> h_keys_;

    // pending (not yet inserted) vectors live directly in d_vectors_[n_ ...); only bookkeeping here
    size_t pending_n_ = 0;
    // vectors added one at a time (usearch_add, build.c:128) wait here until a block is worth a host->device copy
    std::vector<uint8_t> staged_rows_;
    std::vector<uint64_t> staged_keys_;
    int staged_kind_ = 0;
    std::mutex stage_mu_;

    // search scratch
    SearchScratch scratch_{};
    uint8_t* d_query_buf_ = nullptr;
    size_t query_buf_bytes_ = 0;
    void* d_io_buf_ = nullptr;
    size_t io_buf_bytes_ = 0;
    cudaEvent_t ev0_ = nullptr, ev1_ = nullptr;
    uint32_t last_nq_ = 0;
    std::mutex mu_;
    std::recursive_mutex host_mu_; // whole host-buffer calls (they share d_io_buf_); always taken before mu_
    // streaming state of the single-query entry point (usearch_search_ef continue_search, scan.c:240-292)
    std::vector<uint8_t> stream_query_;
    std::vector<uint64_t> stream_returned_; // keys handed out so far for stream_query_
    std::mutex stream_mu_;

    void ensure_scratch(uint32_t ctas);
    // throws unless a PQ walk with a look-up table `lut_width` centroids wide fits in one CTA's shared memory
    void check_pq_table_fits(uint32_t lut_width) const;
    void encode_screen(size_t first, size_t count); // companions of rows [first, first + count) from d_vectors_
    // the search screen's choice (pscreen.cu)
    bool screen_eligible() const; // f32 l2sq / cos rows of >= kScreenMinRowBytes
    void decide_screen();         // automatic choice, once rows >= kPsMinRows (after a build, after load_buffer)
    void reset_screen();          // load_buffer: forget the choice, int8 companion back on
    void force_pscreen();         // a basis for LB200_SEARCH_SCREEN=2 when there is none
    void set_pscreen_basis(const std::vector<float>& P, uint32_t k);
    void set_int8_companion(bool on);
    void free_pscreen();
    void* io_buffer(size_t bytes);
    uint8_t* query_buffer(size_t bytes);
};

// ---- kernels' host launchers -----------------------------------------------------------------------
// codec.cu
void launch_cast_rows(const void* d_in, size_t in_stride, int in_kind, void* d_out, size_t out_stride, int out_kind,
                      size_t dims, size_t n, cudaStream_t stream);
void launch_pq_encode(const float* d_codebook, size_t dims, size_t ncent, size_t nsub, const float* d_vecs,
                      size_t vec_stride_floats, size_t n, uint8_t* d_codes, size_t code_stride, bool compat128,
                      cudaStream_t stream);
void launch_pq_tables(const float* d_codebook, size_t dims, size_t ncent, size_t nsub, bool cosine, float* d_pair, float* d_norm,
                      cudaStream_t stream);
// per-query ADC tables of a batch: out[q][s * lut_width + c] (+ |q|^2 at [nsub * lut_width]), row stride pq_table_floats()
void launch_pq_query_tables(const float* d_codebook, size_t dims, size_t nsub, size_t lut_width, bool cosine, const float* d_queries,
                            size_t q_stride_floats, size_t nq, float* d_tables, cudaStream_t stream);
// screen.cuh companion of n stored f32 rows (row_bytes apart): codes[n][screen_code_bytes(row_bytes)], meta[n]
void launch_sq_encode(const uint8_t* d_rows, size_t row_bytes, size_t n, uint8_t* d_codes, float4* d_meta, cudaStream_t stream);
// pscreen.cu: records of n stored f32 rows for the basis (d_P [slots][dims], d_Pt [dims][slots]); the pre-pass of nq queries
// (storage rows q_stride apart) into d_out[nq][ps_query_floats(k)]; device copies of a host basis [k][dims]; the basis choice
void launch_ps_encode(const uint8_t* d_rows, size_t row_bytes, size_t n, size_t dims, const float* d_P, const float* d_Pt, uint32_t k,
                      bool cosine, uint8_t* d_records, cudaStream_t stream);
void launch_ps_queries(const float* d_P, const float* d_Pt, size_t dims, uint32_t k, const uint8_t* d_queries, size_t q_stride, size_t nq,
                       float* d_out, cudaStream_t stream);
void ps_upload_basis(const std::vector<float>& P, size_t dims, uint32_t k, float** d_P, float** d_Pt);
// want_k = 0: the smallest qualifying k (0 = none; `force`: the best one); else the top want_k eigenvectors
uint32_t ps_choose_basis(const uint8_t* d_rows, size_t row_bytes, size_t n, size_t dims, bool force, uint32_t want_k, std::vector<float>& P);
void launch_pq_decode(const float* d_codebook, size_t dims, size_t ncent, size_t nsub, const uint8_t* d_codes,
                      size_t code_stride, size_t n, float* d_vecs, cudaStream_t stream);
// search.cu
struct SearchLaunch {
    GraphView g;
    SearchScratch s;
    const uint8_t* queries; // storage kind, stride = query_stride
    uint32_t query_stride;
    uint32_t nq, k, L;
    uint32_t expand; // candidates expanded per round (1 = the reference's exact order)
    int screen;      // level-0 beam screens candidates before reading their rows (screen.cuh): 1 = g.sq_codes, 2 = g.ps_records
    uint64_t* out_keys;
    float* out_dists;
    uint32_t* out_counts;
};
uint32_t search_max_ctas(int dist_mode, int scalar_kind, const GraphView& g, uint32_t L, bool pq, uint32_t expand, int screen);
// test hook: screen bound and the search kernel's own fp32 distance for every (query, row) pair; device rows / queries
// row_bytes apart, outputs [nq][n]
void launch_screen_probe(int dist_mode, const uint8_t* d_rows, size_t n, const uint8_t* d_queries, size_t nq, uint32_t row_bytes,
                         float* d_lb, float* d_dist, cudaStream_t stream);
// the same for the projected screen with the basis d_P / d_Pt of k rows
void launch_pscreen_probe(int dist_mode, const uint8_t* d_rows, size_t n, const uint8_t* d_queries, size_t nq, uint32_t row_bytes,
                          size_t dims, const float* d_P, const float* d_Pt, uint32_t k, float* d_lb, float* d_dist, cudaStream_t stream);
void launch_search(int dist_mode, int scalar_kind, bool pq, const SearchLaunch& p, cudaStream_t stream);
// test hook: PqEval on the view `g` of a PQ index, for `count` values -- raw f32 rows value_stride bytes apart (tables from
// g.pq_query_tables when set, else built in the kernel), or stored nodes when d_nodes != NULL.  Outputs d_dist[count][g.n]
// (every stored row, measured cand_cap at a time) and d_lut[count][nsub * pq_lut_width + 1] (the table, then |value|^2).
void launch_pq_probe(int dist_mode, const GraphView& g, uint32_t cand_cap, const uint8_t* d_values, uint32_t value_stride,
                     const uint32_t* d_nodes, size_t count, float* d_dist, float* d_lut, cudaStream_t stream);
// group.cu: the warp-per-query kernel as a single-GPU search path; ps_query = the batch's projected-screen pre-pass (the
// level-0 rounds screen their candidates), or NULL (no screen).  Work counters land in idx.d_warp_aux_ (Index::last_stats).
void launch_warp_search(Index& idx, const uint8_t* qbuf, size_t qrow, size_t nq, size_t k, uint32_t L, const float* ps_query,
                        uint64_t* d_keys, float* d_dists, uint32_t* d_counts, cudaStream_t stream);
// exact_tc.cu: launch plan of the tensor-core filter, and a test hook that copies its intermediate buffers to the host
struct ExactTcEps { // |approximate - exact fp32 distance| <= eps(|q|^2, |x|^2): see approx_eps in exact_tc.cu
    float rel;       // 3xTF32 dot product, relative to |q||x|
    float sum;       // fp32 norms, final arithmetic and the exact kernel's own summation, relative to |q|^2 + |x|^2
    float lin, abs;  // dot product with flushed subnormals: lin (|q| + |x|) + abs
};
struct ExactTcPlan {
    uint32_t groups; // row groups per query tile
    uint32_t KP;     // candidates kept per (query, row group)
    ExactTcEps eps;
};
ExactTcPlan exact_tc_plan(size_t n, size_t nq, size_t k, uint32_t row_bytes);
struct ExactTcProbe { // host buffers, sized from exact_tc_plan; filled by launch_exact_tc before it frees its scratch
    float* qn;         // [nq] fp32 |q|^2 as the filter used them
    float* xn;         // [n]  fp32 |x|^2
    float* cand_d;     // [nq][groups][KP] approximate distances, heap order, +inf padded
    uint32_t* cand_i;  // [nq][groups][KP] row offsets, 0xFFFFFFFF padded
    float* dropped_lb; // [nq][groups] smallest lower bound of anything a list dropped
    uint8_t* unsafe;   // [nq] 1 = not certified, answered by the SIMT kernels
};
// exact.cu.  `probe` (tests only) forces the tensor-core path and captures its buffers.
void launch_exact(int dist_mode, int scalar_kind, const uint8_t* d_data, size_t n, size_t data_stride,
                  const uint8_t* d_queries, size_t nq, size_t q_stride, uint32_t row_bytes, size_t k, uint64_t* d_keys,
                  float* d_dists, cudaStream_t stream, const ExactTcProbe* probe = nullptr);
void launch_pair_distance(int dist_mode, int scalar_kind, const uint8_t* d_a, size_t a_stride, const uint8_t* d_b,
                          size_t b_stride, size_t n, uint32_t row_bytes, float* d_out, cudaStream_t stream);
void launch_merge_shards(const uint64_t* d_keys, const float* d_dists, size_t shards, size_t nq, size_t k,
                         uint64_t* d_out_keys, float* d_out_dists, cudaStream_t stream);
// build.cu
void build_pending(Index& idx);
// the same build with every batch shared by the ranks of a single-process group (DESIGN.md 4.2): replicas[r] is rank r's
// index and device, replicas[root].idx == &idx; the others are replicas of idx (group.cu) that receive every list it does
struct BuildReplica {
    Index* idx;
    int device;
};
void build_pending_group(Index& idx, const std::vector<BuildReplica>& replicas, int root);
// format.cu: the file of a row-sharded index, in order, through `write`: header, lists, keys and levels from `graph` (whose
// device is shards[0]'s), row i from the shard whose [row_lo_, row_hi_) holds it, a bounded block at a time
using RowShard = BuildReplica;
void save_row_sharded(Index& graph, const std::vector<RowShard>& shards, const std::function<void(const void*, size_t)>& write);
// kmeans.cu
int train_pq_codebook(const float* d_vectors, size_t stride_floats, size_t n, size_t dims, size_t nsub, size_t ncent, bool cosine,
                      size_t max_iter, uint64_t seed, const uint32_t* init_rows, float* d_codebook, cudaStream_t stream);

int device_sm_count();
void require_device();

} // namespace lb200

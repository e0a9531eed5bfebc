/*
 * lantern_b200 -- C ABI of the H100-native HNSW search/build engine.
 *
 * This is the drop-in boundary (SURVEY.md 8b, "B1"): the entry points Lantern's access method
 * (lantern_hnsw/src/hnsw/{scan,build}.c) and lantern_cli's external indexer bind today through the
 * usearch C API (/root/reference/lantern_hnsw/third_party/usearch/c/usearch.h, "U/c/usearch.h"
 * below), re-exported here with identical argument meaning and error behaviour, plus the batch
 * entry points the reference lacks (it searches one query per call, scan.c:64,220-228).
 *
 * Conventions (all inherited from U/c/usearch.h):
 *   - every call takes `lb200_error_t* error`; on failure the callee stores a pointer to a static,
 *     never-freed C string and returns 0 / NULL (usearch.h:35-39; lib.cpp:183-189 pattern);
 *   - handles are owned by the caller and released with lb200_free (usearch.h:146);
 *   - vectors are copied on add (lib.cpp:89 force_vector_copy=true); result buffers are caller-owned;
 *   - keys are opaque u64 (Lantern: 6-byte heap TID; 0 = deleted, hnsw.h:40); UINT64_MAX is the
 *     reserved "free" key (index_dense.hpp:438) and is rejected by lb200_add*;
 *   - hamming dimensions are given in BITS (scan.c:84-88);
 *   - expansion = max(ef, k) (index.hpp:2706); ef == 0 means "index default" (usearch.h:265-271).
 *     Unlike the vendored shim (lib.cpp:394 drops ef) a non-zero ef IS honoured.
 *
 * Every symbol is also exported under its reference name (`usearch_*`, same signature) so that
 * lantern.so can link this library in place of U/c/lib.cpp; see INTEGRATION.md.
 *
 * There is no CPU fallback: every compute entry point fails with "CUDA device unavailable" when no
 * sm_90 GPU is present.
 */
#ifndef LANTERN_B200_H
#define LANTERN_B200_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LB200_EXPORT __attribute__((visibility("default")))

typedef void* lb200_index_t;       /* U/c/usearch.h:20 usearch_index_t */
typedef uint64_t lb200_key_t;      /* :21 usearch_key_t */
typedef float lb200_distance_t;    /* :25 usearch_distance_t */
typedef char const* lb200_error_t; /* :39 usearch_error_t */
typedef void* (*lb200_node_retriever_t)(void* ctx, unsigned long long index); /* :29 */
typedef lb200_distance_t (*lb200_metric_t)(void const*, void const*);         /* :45 */

/* U/c/usearch.h:51-63 -- numeric values are part of the ABI */
typedef enum lb200_metric_kind_t {
    lb200_metric_unknown_k = 0,
    lb200_metric_cos_k = 1,
    lb200_metric_ip_k = 2,
    lb200_metric_l2sq_k = 3,
    lb200_metric_haversine_k = 4,
    lb200_metric_divergence_k = 5,
    lb200_metric_pearson_k = 6,
    lb200_metric_jaccard_k = 7,
    lb200_metric_hamming_k = 8,
    lb200_metric_tanimoto_k = 9,
    lb200_metric_sorensen_k = 10,
} lb200_metric_kind_t;

/* U/c/usearch.h:65-72 */
typedef enum lb200_scalar_kind_t {
    lb200_scalar_unknown_k = 0,
    lb200_scalar_f32_k = 1,
    lb200_scalar_f64_k = 2,
    lb200_scalar_f16_k = 3,
    lb200_scalar_i8_k = 4,
    lb200_scalar_b1_k = 5,
} lb200_scalar_kind_t;

/* U/c/usearch.h:74-117 -- field-for-field identical layout to usearch_init_options_t */
typedef struct lb200_init_options_t {
    lb200_metric_kind_t metric_kind;
    lb200_metric_t metric; /* custom metrics are not supported on the GPU: must be NULL */
    lb200_scalar_kind_t quantization;
    size_t dimensions;
    size_t connectivity;     /* M; 0 -> 16 */
    size_t expansion_add;    /* ef_construction; 0 -> 128 */
    size_t expansion_search; /* ef; 0 -> 64 */
    bool multi;              /* must be false (Lantern never sets it) */
    void* retriever_ctx;     /* external (Postgres-page) node retrievers have no meaning for HBM-resident */
    lb200_node_retriever_t retriever;     /* graphs: must be NULL; use lb200_load_buffer on the index file */
    lb200_node_retriever_t retriever_mut;
    size_t num_threads; /* ignored: parallelism is the GPU's */
    bool pq;
    size_t num_centroids;
    size_t num_subvectors;
} lb200_init_options_t;

/* U/c/usearch.h:119-131 */
typedef struct lb200_index_metadata_t {
    lb200_init_options_t init_options;
    double inverse_log_connectivity;
    size_t neighbors_bytes;      /* 4 + 6*M   (file-format width, index.hpp:1838) */
    size_t neighbors_base_bytes; /* 4 + 12*M */
    size_t dimensions;
    size_t expansion_search;
    size_t expansion_add;
    size_t connectivity;
    lb200_metric_kind_t metric_kind;
} lb200_index_metadata_t;

/* Work counters of the most recent search batch -- the reference's own definition of work
 * (index.hpp:2370-2374, 2697-2727), used for the roofline's algorithmic bytes (SURVEY.md 8d). */
typedef struct lb200_search_stats_t {
    uint64_t queries;
    uint64_t computed_distances; /* == usearch search_result_t::computed_distances summed over the batch */
    uint64_t base_pops;          /* level-0 candidates expanded */
    uint64_t upper_hops;         /* level>=1 neighbour lists scanned */
    uint64_t algorithmic_bytes;  /* full_rows_read*row_bytes + screened candidates*(code row + 16, or the projected record) +
                                    (base_pops*(4+4*M0) +
                                    upper_hops*(4+4*M)) + queries*row_bytes: the bytes the search needed */
    double kernel_ms;            /* device time of the search kernel alone (CUDA events on the launching stream) */
    uint64_t limbo_overflows;    /* equal-distance candidates beyond the 64 the walker parks at the eviction boundary (only
                                    possible with massive exact ties; each one may be an expansion the reference performs) */
    uint64_t full_rows_read;     /* (appended field) stored rows read in full: computed_distances minus the candidates the
                                    screen of f32 l2sq / cos searches rejected from their codes alone */
    uint32_t screen_kind;        /* (appended field) the search's screen: 0 none, 1 int8 codes of every dimension, 2 projected codes */
    uint32_t screen_dims;        /* (appended field) codes per screened candidate: dimensions (1) or the basis' k (2) */
    uint32_t search_kernel;      /* (appended field) the kernel that ran: 1 one CTA per query, 2 one warp per query */
    uint32_t reserved;           /* (appended field) zero */
    uint64_t owner_cycles_produce;  /* (appended fields) one warp per query: SM cycles of the walks' rounds by phase, summed */
    uint64_t owner_cycles_screen;   /* over walks -- neighbour lists and visited bits, the projected screen, reading the   */
    uint64_t owner_cycles_evaluate; /* surviving rows, the ordered insertions.  Zero for the CTA kernel.                    */
    uint64_t owner_cycles_consume;
} lb200_search_stats_t;

/* Work of the most recent lb200_build (or implicit build): the build metric of SURVEY.md 8d is
 * computed_distances x bytes per stored vector / seconds (counters as index.hpp:2546-2556 accumulates them per add). */
typedef struct lb200_build_stats_t {
    uint64_t vectors;            /* nodes inserted by that build */
    uint64_t computed_distances; /* distance evaluations of the insert + reverse-link kernels */
    uint64_t algorithmic_bytes;  /* computed_distances * bytes per stored vector (PQ: code bytes) */
    double device_ms;            /* CUDA events around the whole build on its stream */
} lb200_build_stats_t;

/* ---- lifecycle: U/c/usearch.h:140-146, lib.cpp:130-176 ---------------------------------------- */
/* `codebook` (float[num_centroids][dimensions]) is copied to the device (the reference borrows it). */
LB200_EXPORT lb200_index_t lb200_init(lb200_init_options_t* options, float* codebook, lb200_error_t* error);
LB200_EXPORT void lb200_free(lb200_index_t, lb200_error_t* error);

/* ---- introspection: usearch.h:224-229, 191 ---------------------------------------------------- */
LB200_EXPORT size_t lb200_size(lb200_index_t, lb200_error_t* error);
LB200_EXPORT size_t lb200_capacity(lb200_index_t, lb200_error_t* error);
LB200_EXPORT size_t lb200_dimensions(lb200_index_t, lb200_error_t* error);
LB200_EXPORT size_t lb200_connectivity(lb200_index_t, lb200_error_t* error);
LB200_EXPORT size_t lb200_expansion_add(lb200_index_t, lb200_error_t* error);
LB200_EXPORT size_t lb200_expansion_search(lb200_index_t, lb200_error_t* error);
LB200_EXPORT lb200_index_metadata_t lb200_index_metadata(lb200_index_t, lb200_error_t* error);
LB200_EXPORT size_t lb200_count(lb200_index_t, lb200_key_t key, lb200_error_t* error);  /* usearch.h:263 */
LB200_EXPORT bool lb200_contains(lb200_index_t, lb200_key_t key, lb200_error_t* error); /* usearch.h:255 */

/* ---- build path: usearch.h:236-247; batch forms are new ---------------------------------------- */
LB200_EXPORT void lb200_reserve(lb200_index_t, size_t capacity, lb200_error_t* error);
/* Stages one vector (host memory, `vector_kind` f32 or b1 as Lantern passes them, build.c:128);
 * the graph is extended on the GPU at the next lb200_build / search / save. */
LB200_EXPORT void lb200_add(lb200_index_t, lb200_key_t key, void const* vector, lb200_scalar_kind_t vector_kind,
                            lb200_error_t* error);
/* n vectors, `stride` bytes apart, host memory. */
LB200_EXPORT void lb200_add_batch(lb200_index_t, lb200_key_t const* keys, void const* vectors, size_t n, size_t stride,
                                  lb200_scalar_kind_t vector_kind, lb200_error_t* error);
/* Same, vectors already resident in device memory (f32 rows, or packed bits for b1). */
LB200_EXPORT void lb200_add_batch_device(lb200_index_t, lb200_key_t const* host_keys, void const* device_vectors,
                                         size_t n, size_t stride, lb200_scalar_kind_t vector_kind, lb200_error_t* error);
/* Inserts every staged vector into the HNSW graph on the GPU (index.hpp:2479-2564 semantics:
 * level draw, efc-wide beam per level, heuristic neighbour selection, reverse links with re-pruning). */
LB200_EXPORT void lb200_build(lb200_index_t, lb200_error_t* error);
LB200_EXPORT void lb200_last_build_stats(lb200_index_t, lb200_build_stats_t* stats, lb200_error_t* error);

/* Engine knobs that have no counterpart in usearch_init_options_t:
 *   "build_batch"  max vectors inserted concurrently per batch (default 0 = one per resident CTA); 1 = strictly sequential insertion,
 *                  i.e. the reference's order of operations (byte-identical graphs on order-independent data);
 *   "build_ratio"  a batch never exceeds (nodes already in the graph) / build_ratio (default 64);
 *   "search_expand" candidates expanded per search round (default 1 = the reference's exact order; 2..8 = relaxed order:
 *                  fewer serial rounds, slightly more distance evaluations, identical results at ef >= N and recall within
 *                  the +-0.5 % window otherwise);
 *   "pq_query_tables" PQ search: 1 (default) = compute the batch's look-up tables in one launch when they take at most 1 GB,
 *                  0 = never (each CTA builds its query's table, as it always does for larger batches; same results). */
LB200_EXPORT void lb200_set_option(lb200_index_t, char const* name, size_t value, lb200_error_t* error);

/* ---- search path: usearch.h:277-296, lib.cpp:389-410 ------------------------------------------ */
/* One query, host buffers.  Returns the number of matches written (ascending distance).
 * continue_search (scan.c:273-281 streaming): returns the NEXT `count` neighbours of the query passed to the preceding
 * call (same bytes required); implemented as a fresh search for (returned so far + count), so results never repeat and,
 * unlike the reference's frontier continuation (index.hpp:3415-3430), reachable neighbours are never lost. */
LB200_EXPORT size_t lb200_search_ef(lb200_index_t, void const* query_vector, lb200_scalar_kind_t query_kind, size_t count,
                                    size_t ef, bool continue_search, lb200_key_t* keys, lb200_distance_t* distances,
                                    lb200_error_t* error);
LB200_EXPORT size_t lb200_search(lb200_index_t, void const* query_vector, lb200_scalar_kind_t query_kind, size_t count,
                                 lb200_key_t* keys, lb200_distance_t* distances, lb200_error_t* error);
/* Batch of nq queries in HOST memory, `stride` bytes apart; outputs keys[nq][count], distances[nq][count]
 * (unused tail: key UINT64_MAX, distance +inf), counts[nq] (may be NULL).  Host<->device copies included. */
LB200_EXPORT void lb200_search_batch(lb200_index_t, void const* queries, size_t nq, size_t stride,
                                     lb200_scalar_kind_t query_kind, size_t count, size_t ef, lb200_key_t* keys,
                                     lb200_distance_t* distances, size_t* counts, lb200_error_t* error);
/* Same with queries and outputs resident in DEVICE memory (counts: uint32_t[nq] or NULL); asynchronous on
 * `cuda_stream` (a cudaStream_t passed as void*; NULL = default stream).  One index owns one set of device scratch (query
 * staging, visited bitmaps, work counters): asynchronous calls on the SAME index must be issued on one stream, or be ordered
 * by the caller; different indexes are independent.  An index belongs to the device that was current in lb200_init. */
LB200_EXPORT void lb200_search_batch_device(lb200_index_t, void const* d_queries, size_t nq, size_t stride,
                                            lb200_scalar_kind_t query_kind, size_t count, size_t ef,
                                            lb200_key_t* d_keys, lb200_distance_t* d_distances, uint32_t* d_counts,
                                            void* cuda_stream, lb200_error_t* error);
LB200_EXPORT void lb200_last_search_stats(lb200_index_t, lb200_search_stats_t* stats, lb200_error_t* error);

/* ---- (de)serialisation in the usearch/lantern file format: usearch.h:152-212, SURVEY App. B ----- */
LB200_EXPORT size_t lb200_serialized_length(lb200_index_t, lb200_error_t* error); /* exact */
LB200_EXPORT void lb200_save_buffer(lb200_index_t, void* buffer, size_t length, lb200_error_t* error);
LB200_EXPORT void lb200_load_buffer(lb200_index_t, void const* buffer, size_t length, lb200_error_t* error);
LB200_EXPORT void lb200_view_buffer(lb200_index_t, void const* buffer, size_t length, lb200_error_t* error);
LB200_EXPORT void lb200_save(lb200_index_t, char const* path, lb200_error_t* error);
LB200_EXPORT void lb200_load(lb200_index_t, char const* path, lb200_error_t* error);
LB200_EXPORT void lb200_view(lb200_index_t, char const* path, lb200_error_t* error);
LB200_EXPORT void lb200_metadata_buffer(void const* buffer, size_t length, lb200_init_options_t* options,
                                        lb200_error_t* error);
LB200_EXPORT void lb200_metadata(char const* path, lb200_init_options_t* options, lb200_error_t* error); /* usearch.h:186 */
/* usearch.h:175 -- writes the first 136 bytes of a save (head, header, vector_size_bytes, node_count) to `headerp` */
LB200_EXPORT void lb200_update_header(lb200_index_t, char* headerp, lb200_error_t* error);
LB200_EXPORT uint64_t lb200_header_get_entry_slot(char* headerp);               /* lib.cpp:219-225 */
LB200_EXPORT void lb200_header_set_entry_slot(char* headerp, uint64_t entry_slot); /* lib.cpp:227-231 */

/* ---- stateless kernels: usearch.h:338-387 ------------------------------------------------------ */
LB200_EXPORT lb200_distance_t lb200_distance(void const* vector_first, void const* vector_second,
                                             lb200_scalar_kind_t scalar_kind, size_t dimensions,
                                             lb200_metric_kind_t metric_kind, lb200_error_t* error);
/* n pairs at once: a[i] vs b[i], host memory, strides in bytes. */
LB200_EXPORT void lb200_distance_batch(void const* a, size_t a_stride, void const* b, size_t b_stride, size_t n,
                                       lb200_scalar_kind_t scalar_kind, size_t dimensions,
                                       lb200_metric_kind_t metric_kind, lb200_distance_t* out, lb200_error_t* error);
/* Brute force (lib.cpp:450-481): keys receive DATASET OFFSETS, ascending distance; host memory. */
LB200_EXPORT void lb200_exact_search(void const* dataset, size_t dataset_size, size_t dataset_stride,
                                     void const* queries, size_t queries_size, size_t queries_stride,
                                     lb200_scalar_kind_t scalar_kind, size_t dimensions, lb200_metric_kind_t metric_kind,
                                     size_t count, size_t threads, lb200_key_t* keys, size_t keys_stride,
                                     lb200_distance_t* distances, size_t distances_stride, lb200_error_t* error);
/* Same, inputs/outputs in device memory (rows densely packed in `scalar_kind`). */
LB200_EXPORT void lb200_exact_search_device(void const* d_dataset, size_t dataset_size, size_t dataset_stride,
                                            void const* d_queries, size_t queries_size, size_t queries_stride,
                                            lb200_scalar_kind_t scalar_kind, size_t dimensions,
                                            lb200_metric_kind_t metric_kind, size_t count, lb200_key_t* d_keys,
                                            lb200_distance_t* d_distances, void* cuda_stream, lb200_error_t* error);
/* Test hook, not a search entry point: lb200_exact_search on dense f32 rows (l2sq or cos, count <= 192) with the
 * tensor-core filter forced on, copying the filter's intermediate buffers out; host memory.  plan[2] receives the row
 * groups G and the candidates per list KP, eps[4] the error-bound constants (relative, summation, linear, absolute).
 * With cand_d == NULL nothing runs: call once that way to size the buffers qn[queries_size], xn[dataset_size],
 * cand_d / cand_i [queries_size][G][KP], dropped_lb [queries_size][G], unsafe [queries_size] (1 = not certified,
 * answered by the SIMT kernels), keys / distances [queries_size][count] (the search's final answer). */
LB200_EXPORT void lb200_exact_tc_probe(float const* dataset, size_t dataset_size, float const* queries, size_t queries_size,
                                       size_t dimensions, lb200_metric_kind_t metric_kind, size_t count, uint32_t* plan,
                                       float* eps, float* qn, float* xn, float* cand_d, uint32_t* cand_i, float* dropped_lb,
                                       uint8_t* unsafe, lb200_key_t* keys, lb200_distance_t* distances,
                                       lb200_error_t* error);
/* Test hook, not a search entry point: for every (query, row) pair of dense f32 rows (l2sq or cos), the search screen's lower
 * bound lb[queries_size][dataset_size] and the search kernel's own fp32 distance d[queries_size][dataset_size], computed
 * by the device functions the search uses (the rows are encoded as an index encodes them); lb <= d must hold. */
LB200_EXPORT void lb200_search_screen_probe(float const* dataset, size_t dataset_size, float const* queries, size_t queries_size,
                                            size_t dimensions, lb200_metric_kind_t metric_kind, float* lb, float* d,
                                            lb200_error_t* error);
/* Test hook, like lb200_search_screen_probe, for the projected screen: `basis` = k x dimensions fp32 (any values), or NULL for
 * the rows' own basis (the top-k eigenvectors of their second moment; k = 0: chosen as an index chooses it, or its best k). */
LB200_EXPORT void lb200_search_pscreen_probe(float const* dataset, size_t dataset_size, float const* queries, size_t queries_size,
                                             size_t dimensions, lb200_metric_kind_t metric_kind, float const* basis, size_t k, float* lb,
                                             float* d, lb200_error_t* error);
/* The projected screen's basis of an index: returns k (0 = the index keeps none) and, when `basis` is not NULL, copies the
 * k x dimensions fp32 basis there; `seconds` (may be NULL) receives the host time its last choice took. */
LB200_EXPORT size_t lb200_screen_basis(lb200_index_t, float* basis, double* seconds, lb200_error_t* error);
/* Test hook, not a search entry point: the asymmetric distances of a built PQ index, computed by the evaluator the search and
 * build kernels use.  mode 0: `count` raw f32 values (values[count][dimensions]) with the look-up tables a search batch
 * precomputes; mode 1: the same values with the tables each CTA builds itself (batches past 1 GB, and the build); mode 2:
 * stored nodes nodes[count] as values, tables from the centroid-pair table (refine and reverse links).  rows / lut_width
 * (may be NULL) receive the stored rows n and the table width W; with distances == NULL nothing runs.  Outputs
 * distances[count][n] (value against every stored row) and tables[count][num_subvectors * W + 1] (the table, then |value|^2,
 * 0 for l2sq values built in the kernel, which do not use it); host memory. */
LB200_EXPORT void lb200_pq_probe(lb200_index_t, int mode, float const* values, uint32_t const* nodes, size_t count, size_t* rows,
                                 size_t* lut_width, float* distances, float* tables, lb200_error_t* error);
/* f32 -> f16 / i8 / b1 (index_plugins.hpp:879-974); host memory; `count` vectors. */
LB200_EXPORT void lb200_cast(lb200_scalar_kind_t from, void const* vectors, lb200_scalar_kind_t to, void* result,
                             size_t result_size, int dims, lb200_error_t* error);
LB200_EXPORT void lb200_cast_batch(void const* vectors_f32, size_t count, size_t dims, lb200_scalar_kind_t to,
                                   void* result, lb200_error_t* error);

/* ---- PQ codec (lantern_storage.hpp:100-149; quantize_vector / dequantize_vector in lantern.sql) -- */
/* codebook float[num_centroids][dims]; codes uint8[count][num_subvectors].
 * compat128 != 0 reproduces the reference index's signed-char loop (only centroids 0..127). */
LB200_EXPORT void lb200_quantize_pq(float const* codebook, size_t dims, size_t num_centroids, size_t num_subvectors,
                                    float const* vectors, size_t count, uint8_t* codes, int compat128,
                                    lb200_error_t* error);
LB200_EXPORT void lb200_dequantize_pq(float const* codebook, size_t dims, size_t num_centroids, size_t num_subvectors,
                                      uint8_t const* codes, size_t count, float* vectors, lb200_error_t* error);

/* PQ codebook training (lantern_hnsw/src/hnsw/product_quantization.c:207-293 semantics: one k-means per subvector,
 * random distinct rows as initial centres, Lloyd rounds until the mean centre shift is <= 0.1 or `max_iter` rounds).
 * vectors: float[count][dims] in host memory; codebook out: float[num_centroids][dims].  init_rows (may be NULL):
 * uint32[num_subvectors][num_centroids] row indices to start from (for reproducible runs).  Returns rounds executed. */
LB200_EXPORT int lb200_train_pq(float const* vectors, size_t count, size_t dims, size_t num_subvectors, size_t num_centroids,
                                lb200_metric_kind_t metric_kind, size_t max_iter, uint64_t seed, uint32_t const* init_rows,
                                float* codebook, lb200_error_t* error);
/* Same with the training vectors resident in device memory (`stride` bytes apart); codebook still returned to the host. */
LB200_EXPORT int lb200_train_pq_device(void const* d_vectors, size_t stride, size_t count, size_t dims, size_t num_subvectors,
                                       size_t num_centroids, lb200_metric_kind_t metric_kind, size_t max_iter, uint64_t seed,
                                       uint32_t const* init_rows, float* codebook, lb200_error_t* error);

/* ---- multi-GPU epilogue: merge G per-shard top-k lists (already all-gathered) per query ---------- */
/* d_keys/d_dists: [G][nq][count] on this device; outputs [nq][count]. */
LB200_EXPORT void lb200_merge_shards_device(lb200_key_t const* d_keys, lb200_distance_t const* d_dists, size_t shards,
                                            size_t nq, size_t count, lb200_key_t* d_out_keys,
                                            lb200_distance_t* d_out_dists, void* cuda_stream, lb200_error_t* error);

/* ---- multi-GPU: one graph searched by G GPUs ("row-sharded group", csrc/group.cu) ------------------------------------
 * The corpus is sharded by contiguous row range (SURVEY.md 8e): GPU r holds the vectors of rows [bounds[r], bounds[r+1])
 * only.  The ranges are balanced by level-0 in-degree (rows that appear in more lists are measured more often), not equal
 * in length; lb200_group_rank_info reports them.  The graph itself (adjacency lists, 4 B per link) is replicated, each query
 * is walked ONCE in the reference's order, and every distance is evaluated on the GPU that holds the row, over NVLink peer
 * memory -- total work equals the 1-GPU search, and so do the results (id for id on the same graph).  Two ways to create a
 * group:
 *   lb200_group_create        one process per GPU (torchrun / MPI style); `allgather` is the caller's bootstrap collective
 *                             (every rank passes `bytes_per_rank` bytes, everybody receives world * bytes_per_rank, rank
 *                             order); it is used at creation/distribution time only, never on the search path;
 *   lb200_group_create_local  one process driving n devices (what a Lantern indexing/search server would do).
 * and four ways to give it its graph (once per group):
 *   lb200_group_distribute    the root rank passes a built (or loaded) index that lives on ITS device; every rank copies its
 *                             row range and the graph from it over NVLink.  The index must fit on one GPU.
 *   lb200_group_load[_buffer] every rank reads its row range and the graph straight from an index file; no GPU ever holds
 *                             all rows, so the group can serve an index larger than one GPU.
 *   lb200_group_index_init    the group gets an empty index of its own, fills it with lb200_group_index_add_batch and builds
 *                             it with all ranks (lb200_group_index_build); no GPU ever holds all rows here either.
 *   lb200_group_index_load    the same index of its own, opened from an index file; it takes more rows, and
 *                             lb200_group_index_reserve grows either kind past its capacity.
 * lb200_group_search_batch*: collective; only the root's queries are read (other ranks may pass NULL); EVERY rank receives
 * the full result (the final all-gather is fused into the kernel's epilogue: owners store their top-k into every rank). */
typedef void* lb200_group_t;
typedef void (*lb200_allgather_fn)(void* ctx, void const* send, void* recv, size_t bytes_per_rank);
typedef struct lb200_group_stats_t {
    int rank, world;
    uint64_t queries;                  /* of the last search batch */
    uint64_t owner_computed_distances; /* distance evaluations REQUESTED by the queries this rank owns (sum over ranks ==
                                          usearch's computed_distances of the same batch on the same graph) */
    uint64_t owner_base_pops, owner_upper_hops, owner_rounds;
    uint64_t local_rows_evaluated; /* rows of THIS rank's slice read and measured (its share of everybody's work) */
    uint64_t local_row_bytes;      /* local_rows_evaluated * bytes per stored vector */
    uint64_t rows_held;
    double kernel_ms; /* device time of this rank's search kernel (CUDA events on its stream) */
    /* where the owner warps of this rank spent their SM cycles (summed over the warps): producing a round's ids (pop, adjacency
     * line, visited bitmap), measuring their local rows, waiting for the other ranks' distances, consuming (ordered insertions) */
    uint64_t owner_cycles_produce, owner_cycles_local, owner_cycles_wait, owner_cycles_consume;
} lb200_group_stats_t;
LB200_EXPORT lb200_group_t lb200_group_create(int rank, int world, lb200_allgather_fn allgather, void* allgather_ctx,
                                              lb200_error_t* error);
LB200_EXPORT lb200_group_t lb200_group_create_local(int const* devices, int n_devices, lb200_error_t* error);
LB200_EXPORT void lb200_group_free(lb200_group_t, lb200_error_t* error);
/* max_batch: largest nq of a search; max_results: largest nq * count (sizes the peer-mapped staging buffers). */
LB200_EXPORT void lb200_group_distribute(lb200_group_t, lb200_index_t root_index, int root, size_t max_batch,
                                         size_t max_results, lb200_error_t* error);
/* Collective.  Forms the group's distribution from a usearch/lantern index file instead of from an index: every rank keeps
 * the rows of its range and a copy of the graph; no rank ever holds all rows.  `options` is checked against the file exactly
 * as lb200_load checks an index's options (metric, scalar kind, dimensions, connectivity; same messages) and supplies
 * expansion_search.  root / max_batch / max_results: as in lb200_group_distribute.  PQ indexes are refused, as distribute
 * refuses them.  The whole file is validated before any rank allocates: after a refusal the group can still take a correct
 * load.  Rows travel through a bounded pinned staging block, so no host copy of the file is made.  Multi-process groups:
 * every rank passes the same bytes (or the same path) and keeps its own range; a rank holding a different file fails the
 * call on every rank.  A group takes one load or one distribute, not both. */
LB200_EXPORT void lb200_group_load_buffer(lb200_group_t, lb200_init_options_t const* options, void const* buffer,
                                          size_t length, int root, size_t max_batch, size_t max_results, lb200_error_t* error);
/* the same from a file, mapped read-only (mmap): a file larger than host memory needs no more than its page cache */
LB200_EXPORT void lb200_group_load(lb200_group_t, lb200_init_options_t const* options, char const* path, int root,
                                   size_t max_batch, size_t max_results, lb200_error_t* error);
/* What a rank keeps on its device, for a group formed either way.  bytes_scratch grows with max_batch * n: one visited
 * bitmap of n bits per owner slot, and a rank has ceil(max_batch / world) slots (at most the resident warps). */
typedef struct lb200_group_rank_info_t {
    int rank, world;
    uint64_t rows_begin, rows_end;         /* this rank's row range */
    uint64_t bytes_rows, bytes_graph;      /* device bytes: its rows; adj0 + upper lists + keys */
    uint64_t bytes_scratch, bytes_mailbox; /* visited bitmaps + touched lists + counters + query staging; the peer-mapped slab */
} lb200_group_rank_info_t;
/* local_rank: as in lb200_group_last_stats.  No device work. */
LB200_EXPORT void lb200_group_rank_info(lb200_group_t, int local_rank, lb200_group_rank_info_t* info, lb200_error_t* error);
/* lb200_group_build: inserts every pending (and staged) vector of `root_index`, which lives on the device of rank `root`,
 * with all ranks of a single-process group.  Every other rank works on a temporary replica of the index (freed when the call
 * returns); each batch's new nodes are split between the ranks, and every list is written into every replica over NVLink.
 * The result is what lb200_build gives on that index with the same batch cap: the same file, lb200_size and
 * lb200_last_build_stats vectors and computed_distances.  `build_batch` still counts the nodes of a batch in total; its
 * default (0) is the one-GPU default times the number of ranks.  The group's distribution is not touched: call
 * lb200_group_distribute afterwards to search the new graph on the group.  Refused for multi-process groups. */
LB200_EXPORT void lb200_group_build(lb200_group_t, lb200_index_t root_index, int root, lb200_error_t* error);
/* ---- the group's own index (single-process groups): built straight into the row-sharded layout, then searched and saved ----
 * lb200_group_index_init: the group gets an empty index with `options` (as lb200_init reads them) and room for `capacity`
 * rows.  Rank r holds rows [capacity r / G, capacity (r+1) / G) until lb200_group_index_reserve changes the capacity; lists and
 * keys of all `capacity`
 * rows are kept on every rank.  max_batch / max_results: as in lb200_group_distribute.  PQ options are refused (a group
 * cannot hold PQ codes), and so are multi-process groups.  A group takes one lb200_group_distribute, lb200_group_load or
 * lb200_group_index_init (or lb200_group_index_load), never two.  lb200_group_search_batch* and lb200_group_rank_info then work
 * on this index; rank_info
 * reports each rank's capacity range and bytes_rows for that range.  Pending rows are built by the next save or search, as
 * with a one-GPU index. */
LB200_EXPORT void lb200_group_index_init(lb200_group_t, lb200_init_options_t const* options, size_t capacity, size_t max_batch,
                                         size_t max_results, lb200_error_t* error);
/* lb200_group_index_load_buffer: the same kind of index as lb200_group_index_init gives, holding the contents of a
 * usearch/lantern index file (written by this library or by usearch).  `options` is read as lb200_init reads it and is checked
 * against the file exactly as lb200_load checks an index (metric, scalar kind, dimensions, connectivity; same messages);
 * expansion_add and expansion_search come from `options`.  capacity 0 means the file's node count n; a capacity below n, or of
 * 2^31 - 1 or more, is refused (an empty file needs a capacity of at least 1).  Rank r receives only the rows of [capacity r /
 * G, capacity (r+1) / G), straight from `buffer` through a bounded pinned block; every rank receives the lists and keys.  The
 * whole file is validated before any rank allocates: after a refusal the group can still take a correct load or an
 * lb200_group_index_init.  The index then holds what lb200_load_buffer gives a one-GPU index (graph, keys, level generator), so
 * the same adds and builds give the same file.  Refusals as in lb200_group_index_init (PQ, multi-process groups, a group that
 * already holds a graph). */
LB200_EXPORT void lb200_group_index_load_buffer(lb200_group_t, lb200_init_options_t const* options, void const* buffer,
                                                size_t length, size_t capacity, size_t max_batch, size_t max_results,
                                                lb200_error_t* error);
/* the same from a file, mapped read-only (mmap): no host buffer and no GPU ever holds all rows */
LB200_EXPORT void lb200_group_index_load(lb200_group_t, lb200_init_options_t const* options, char const* path,
                                         size_t capacity, size_t max_batch, size_t max_results, lb200_error_t* error);
/* As lb200_reserve: room for `capacity` rows; nothing happens at or below the current capacity.  Rank r's range becomes
 * [capacity r / G, capacity (r+1) / G) and every row added so far, built or pending, moves to the rank whose new range holds
 * it (device-to-device copies).  While the call runs, a rank holds its old and new rows and two copies of its level-0 lists,
 * upper references and keys.  Every new array is allocated before any row moves: if one does not fit, the call fails naming
 * the rank, device and what did not fit (rows, graph, scratch), and the index is left exactly as it was. */
LB200_EXPORT void lb200_group_index_reserve(lb200_group_t, size_t capacity, lb200_error_t* error);
/* Host rows, f32 or packed b1, with the input and key checks of lb200_add_batch.  Row i of the index goes only to the rank whose
 * range holds it, cast to the storage kind there, through a bounded pinned block.  Adding past `capacity` is refused and adds
 * nothing (lb200_group_index_reserve raises it). */
LB200_EXPORT void lb200_group_index_add_batch(lb200_group_t, lb200_key_t const* keys, void const* vectors, size_t n, size_t stride,
                                              lb200_scalar_kind_t kind, lb200_error_t* error);
/* "build_batch" and "build_ratio", as lb200_set_option; the default batch cap is the one-GPU default times the ranks. */
LB200_EXPORT void lb200_group_index_set_option(lb200_group_t, char const* name, size_t value, lb200_error_t* error);
/* Inserts every pending row with all ranks: the graph lb200_build makes on one GPU with the same rows and batch cap. */
LB200_EXPORT void lb200_group_index_build(lb200_group_t, lb200_error_t* error);
/* as lb200_size / lb200_last_build_stats of a one-GPU index */
LB200_EXPORT size_t lb200_group_index_size(lb200_group_t, lb200_error_t* error);
LB200_EXPORT void lb200_group_index_last_build_stats(lb200_group_t, lb200_build_stats_t* stats, lb200_error_t* error);
/* The usearch/lantern file, as lb200_serialized_length / lb200_save_buffer / lb200_save.  The graph comes from rank 0 and the
 * rows from each rank in turn through a bounded host block: no host buffer holds all rows, and lb200_group_index_save streams
 * the file to disk. */
LB200_EXPORT size_t lb200_group_index_serialized_length(lb200_group_t, lb200_error_t* error);
LB200_EXPORT void lb200_group_index_save_buffer(lb200_group_t, void* buffer, size_t length, lb200_error_t* error);
LB200_EXPORT void lb200_group_index_save(lb200_group_t, char const* path, lb200_error_t* error);
/* host buffers in and out (host<->device copies included); counts may be NULL */
LB200_EXPORT void lb200_group_search_batch(lb200_group_t, void const* queries, size_t nq, size_t stride,
                                           lb200_scalar_kind_t query_kind, size_t count, size_t ef, lb200_key_t* keys,
                                           lb200_distance_t* distances, size_t* counts, lb200_error_t* error);
/* multi-process groups: device buffers of the calling rank, asynchronous on `cuda_stream`; when the stream reaches the
 * end of this call's work, the results of ALL ranks' queries are in d_keys / d_distances / d_counts of this rank */
LB200_EXPORT void lb200_group_search_batch_device(lb200_group_t, void const* d_queries, size_t nq, size_t stride,
                                                  lb200_scalar_kind_t query_kind, size_t count, size_t ef,
                                                  lb200_key_t* d_keys, lb200_distance_t* d_distances, uint32_t* d_counts,
                                                  void* cuda_stream, lb200_error_t* error);
/* Host-only check of a bootstrap collective (no device needed): every rank sends a rank-stamped blob through `allgather` the
 * way group creation does and verifies what comes back.  Returns 0 when the callback behaves, a non-zero code otherwise. */
LB200_EXPORT int lb200_group_selftest_exchange(int rank, int world, lb200_allgather_fn allgather, void* allgather_ctx);
/* Host-only: how a search of `nq` queries splits the `resident_warps` of each of `world` GPUs into owner warps (one query each)
 * and helper warps (which share the (world-1) * owners inbound mailboxes, at most 32 per helper).  Returns 0 and fills
 * owners / helpers, or 1 when the warps cannot cover the mailboxes.  Every rank computes the same plan. */
LB200_EXPORT int lb200_group_plan(int world, size_t nq, uint32_t resident_warps, uint32_t owner_slots_max, uint32_t* owners,
                                  uint32_t* helpers);
/* local_rank: 0 for a multi-process group; 0..n_devices-1 for a single-process one.  Synchronises that device. */
LB200_EXPORT void lb200_group_last_stats(lb200_group_t, int local_rank, lb200_group_stats_t* stats, lb200_error_t* error);

/* ---- engine info ------------------------------------------------------------------------------- */
LB200_EXPORT int lb200_device_count(void);
LB200_EXPORT char const* lb200_version(void);
/* number of engine kernels launched by this process so far (bench.py's gpu_launches) */
LB200_EXPORT uint64_t lb200_kernel_launches(void);

/* ---- the rest of U/c/usearch.h, exported under the reference names only so that binaries built against usearch.h link:
 * the in-Postgres page storage (nodes fetched from caller memory through retriever callbacks) and label bookkeeping.
 * Each sets *error to a static string that says what to call instead and returns 0; none touches the device. ---------- */
LB200_EXPORT void usearch_view_mem_lazy(lb200_index_t, char* data, lb200_error_t* error);                     /* :174 */
LB200_EXPORT void usearch_set_node_retriever(lb200_index_t, void* retriever_ctx, lb200_node_retriever_t retriever,
                                             lb200_node_retriever_t retriever_mut, lb200_error_t* error);     /* :352 */
LB200_EXPORT void usearch_add_external(lb200_index_t, lb200_key_t key, void const* vector, void* tape,
                                       lb200_scalar_kind_t kind, int16_t level, uint64_t slot, lb200_error_t* error); /* :355 */
LB200_EXPORT int32_t usearch_newnode_level(lb200_index_t, lb200_error_t* error);                              /* :347 */
LB200_EXPORT size_t usearch_get(lb200_index_t, lb200_key_t key, size_t count, void* vector, lb200_scalar_kind_t kind,
                                lb200_error_t* error);                                                        /* :307 */
LB200_EXPORT size_t usearch_remove(lb200_index_t, lb200_key_t key, lb200_error_t* error);                     /* :317 */
LB200_EXPORT size_t usearch_rename(lb200_index_t, lb200_key_t from, lb200_key_t to, lb200_error_t* error);    /* :326 */

#ifdef __cplusplus
}
#endif
#endif /* LANTERN_B200_H */

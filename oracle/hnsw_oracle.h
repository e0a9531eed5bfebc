/* TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's HNSW hot path.
 *
 * This is the parity oracle for the CUDA engine: a plain-C, single-threaded restatement of the
 * algorithm in the usearch fork Lantern vendors (/root/reference/lantern_hnsw/third_party/usearch,
 * "U/" below).  It is NOT part of the product: only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline leg may load it.  Every function cites the reference lines it follows.
 * It is pinned against the unmodified reference (oracle/_ref) and the reference's golden
 * vectors by tests/test_oracle_*.py.
 */
#ifndef HNSW_ORACLE_H
#define HNSW_ORACLE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* numeric values of usearch_metric_kind_t / usearch_scalar_kind_t (U/c/usearch.h:51-72) */
enum { ORA_METRIC_COS = 1, ORA_METRIC_IP = 2, ORA_METRIC_L2SQ = 3, ORA_METRIC_HAMMING = 8 };
enum { ORA_F32 = 1, ORA_F64 = 2, ORA_F16 = 3, ORA_I8 = 4, ORA_B1 = 5 };

typedef struct ora_index ora_index;

typedef struct {
    uint64_t computed_distances; /* U/include/usearch/index.hpp:2726 */
    uint64_t visited_members;    /* "iteration_cycles", index.hpp:2727 */
    uint64_t base_pops;          /* candidates expanded on level 0 (for B_alg, SURVEY 8d) */
    uint64_t upper_hops;         /* neighbour lists scanned on levels >= 1 */
} ora_stats;

/* pq_compat128 != 0 reproduces the signed-char loop quirk of codebook_t::compress
 * (lantern_storage.hpp:123): only centroids 0..127 are ever chosen. */
ora_index* ora_init(int metric, int quant, size_t dims, size_t connectivity, size_t expansion_add,
                    size_t expansion_search, int pq, size_t num_centroids, size_t num_subvectors,
                    const float* codebook, int pq_compat128);
void ora_free(ora_index*);
int ora_reserve(ora_index*, size_t capacity);
size_t ora_size(const ora_index*);
/* 1: the base-layer search and the insertion beams (ora_add, ora_add_batch_engine) pop equal-distance candidates in the CUDA
 * engine's order instead of the reference heap's (results are identical on tie-free data; see beam_engine_order). */
void ora_set_engine_order(ora_index*, int on);
size_t ora_dimensions(const ora_index*);
size_t ora_connectivity(const ora_index*);
int ora_max_level(const ora_index*);
uint64_t ora_entry_slot(const ora_index*);

/* vector: `dims` f32 when kind == ORA_F32, ceil(dims/8) packed bytes when kind == ORA_B1.
 * level < 0 -> drawn from the reference's generator (index.hpp:3208-3212, std::default_random_engine). */
int ora_add(ora_index*, uint64_t key, const void* vector, int kind, int level, ora_stats* stats);

/* Model of the CUDA engine's batched build schedule on top of the reference procedures (NOT a reference function; see
 * the .c file): `n` vectors, `stride` bytes apart, inserted in batches of at most `batch_cap` nodes and at most
 * visible/build_ratio.  batch_cap == 1 is ora_add.  Returns 0, -1 (capacity), -2 (pq not modelled). */
int ora_add_batch_engine(ora_index*, const uint64_t* keys, const void* vectors, size_t n, size_t stride, int kind,
                         size_t batch_cap, size_t build_ratio);

/* ef == 0 -> index default; expansion = max(ef, k) (index.hpp:2706). Returns found count. */
size_t ora_search(ora_index*, const void* query, int kind, size_t k, size_t ef, uint64_t* keys, float* distances,
                  ora_stats* stats);

/* graph inspection */
int ora_node_level(const ora_index*, size_t slot);
uint64_t ora_node_key(const ora_index*, size_t slot);
size_t ora_node_neighbors(const ora_index*, size_t slot, int level, uint32_t* out);
const void* ora_node_vector(const ora_index*, size_t slot); /* storage-domain bytes or PQ codes */

/* usearch/lantern file format (lantern_storage.hpp:471-586, index_dense.hpp:806-842) */
size_t ora_serialized_length(const ora_index*);
size_t ora_save_buffer(const ora_index*, void* buffer, size_t length);
int ora_load_buffer(ora_index*, const void* buffer, size_t length);

/* stateless pieces */
float ora_distance(const void* a, const void* b, int kind, size_t dims, int metric);
void ora_cast_f32(const float* in, size_t dims, int to_kind, void* out);
float ora_f16_to_f32(uint16_t h);
uint16_t ora_f32_to_f16(float f);
void ora_pq_compress(const float* codebook, size_t dims, size_t num_centroids, size_t num_subvectors,
                     const float* vector, uint8_t* codes, int compat128);
void ora_pq_decompress(const float* codebook, size_t dims, size_t num_centroids, size_t num_subvectors,
                       const uint8_t* codes, float* vector);
/* brute force (index_plugins.hpp:1582-1675): offsets + distances, ascending, ties by lower offset */
void ora_exact_search(const void* dataset, size_t n, size_t dataset_stride, const void* queries, size_t nq,
                      size_t queries_stride, int kind, size_t dims, int metric, size_t k, uint64_t* keys,
                      float* distances);
/* PQ codebook training (product_quantization.c restated; initial rows are an input; parity unpinned, see .c) */
int ora_kmeans(const float* data, size_t n, size_t dims, size_t nsub, size_t ncent, int metric, size_t max_iter,
               const uint32_t* init_rows, float* codebook);
/* level generator alone, for tests: returns the i-th (0-based) level of a fresh generator */
int ora_level_sequence(size_t connectivity, size_t count, int16_t* out);

#ifdef __cplusplus
}
#endif
#endif

// lantern_b200 -- row-sharded multi-GPU search group (group.cu): types shared with the C ABI layer.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <functional>
#include <string>

#include "../../include/lantern_b200.h"
#include "engine.h"

namespace lb200 {

constexpr int kGroupMax = 8;

// kernel parameters of group_search_kernel (identical on every rank except `me`, the local pointers and the peer views)
struct GroupLaunch {
    uint32_t G, me, W, cap; // ranks, this rank, query slots (= resident warps) per GPU, ids per message (= M0)
    uint32_t ring_slots;    // rows a warp keeps in flight (its private bulk-copy ring)
    uint32_t O, H;          // owner warps (one query each, slots 0..O) and helper warps (slots O..O+H) per GPU
    uint32_t nq, k, L;
    uint32_t flag_base; // message flags of this launch are flag_base + 1, +2, ...
    uint32_t epoch, root;
    unsigned long long timeout_ns;
    GraphView g; // g.vectors = this rank's row slice (row id - bounds[me]); adjacency, keys: whole graph, local copy
    uint32_t bounds[kGroupMax + 1];
    unsigned long long* req[kGroupMax];  // [G * O][1 + cap] words {payload, flag}: header {count | query << 9, or EXIT}, ids;
                                         // mailbox src * O + oslot belongs to owner slot `oslot` of rank `src`
    uint8_t* reqq[kGroupMax];            // [G * O][row_bytes] the query that owner slot is working on
    unsigned long long* resp[kGroupMax]; // [O][G][cap] words {distance bits, flag}, per OWN owner slot
    uint64_t* res_keys[kGroupMax];       // [nq][k] final results, written by each query's owner into EVERY rank
    float* res_dists[kGroupMax];
    uint32_t* res_counts[kGroupMax];
    unsigned long long* done[kGroupMax];   // [G] epoch of the last launch rank s completed
    unsigned long long* qready[kGroupMax]; // epoch whose queries are staged on the root
    uint32_t* err[kGroupMax];
    const uint8_t* queries; // the root's staging buffer (a peer address on the other ranks)
    uint32_t query_stride;
    uint32_t* vis;     // owner slots: [O][words_per_slot]
    uint32_t* touched; // [O][touched_cap]
    size_t words_per_slot;
    uint32_t touched_cap;
    unsigned long long* counters; // [0] warps finished, [1] owner dist evals, [2] pops, [3] hops, [4] rounds, [5] local rows evaluated,
                                  // [6] next owned query, [7] limbo overflows, [8..11] owner cycles: produce, local, wait, consume
};

struct GroupStats {
    int rank, world;
    uint64_t queries;
    uint64_t owner_computed_distances, owner_base_pops, owner_upper_hops, owner_rounds; // of the queries this rank owns
    uint64_t local_rows_evaluated, local_row_bytes;                                       // rows of this rank's slice read
    uint64_t rows_held;
    uint64_t owner_cycles_produce, owner_cycles_local, owner_cycles_wait, owner_cycles_consume; // SM cycles, summed over owner warps
    double kernel_ms;
};

struct Group;
bool group_plan(int world, size_t nq, uint32_t W, uint32_t Omax, uint32_t& O, uint32_t& H);
Group* group_create_ipc(int rank, int world, lb200_allgather_fn ag, void* ctx);
Group* group_create_local(const int* devices, int ndev);
void group_free(Group* G);
int group_world(const Group& G);
int group_local_ranks(const Group& G);
void group_distribute(Group& G, Index* root_index, int root, size_t max_batch, size_t max_results);
// the same distribution from the bytes of an index file that every rank passes; `cfg` plays the part of the index's options
void group_load(Group& G, const IndexConfig& cfg, const void* buffer, size_t length, int root, size_t max_batch,
                size_t max_results);
void group_rank_info(Group& G, int which, lb200_group_rank_info_t& out);
void group_build(Group& G, Index* root_index, int root);
void group_search_device(Group& G, const void* d_queries, size_t nq, size_t stride, int kind, size_t k, size_t ef,
                         uint64_t* d_keys, float* d_dists, uint32_t* d_counts, cudaStream_t stream);
void group_search_host(Group& G, const void* queries, size_t nq, size_t stride, int kind, size_t k, size_t ef, uint64_t* keys,
                       float* dists, size_t* counts);
void group_stats(Group& G, int which, GroupStats& out);
// the group's own row-sharded index (single-process groups): rank r holds rows [capacity r / G, capacity (r+1) / G)
void group_index_init(Group& G, const IndexConfig& cfg, size_t capacity, size_t max_batch, size_t max_results);
// the same index holding the contents of an index file (capacity 0 = the file's rows); `cfg` is checked against the file as
// Index::load_buffer checks it
void group_index_load(Group& G, const IndexConfig& cfg, const void* buffer, size_t length, size_t capacity, size_t max_batch,
                      size_t max_results);
// raises the capacity (nothing happens at or below it): new ranges [capacity r / G, capacity (r+1) / G), rows moved between ranks
void group_index_reserve(Group& G, size_t capacity);
void group_index_add(Group& G, const uint64_t* keys, const void* vectors, size_t n, size_t stride, int kind);
void group_index_build(Group& G);
void group_index_set_option(Group& G, const std::string& name, size_t value);
size_t group_index_size(Group& G);
void group_index_build_stats(Group& G, size_t& vectors, uint64_t& distances, double& ms, size_t& value_bytes);
size_t group_index_serialized_length(Group& G);
// length_ok(file length) may refuse (throw) before anything is written; write() then receives the whole file, in order
void group_index_save(Group& G, const std::function<void(size_t)>& length_ok, const std::function<void(const void*, size_t)>& write);

} // namespace lb200

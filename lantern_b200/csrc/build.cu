// lantern_b200 -- HNSW construction on the GPU.
//
// Replaces the reference's insertion path
//   index_gt::add                       U/include/usearch/index.hpp:2479-2564
//   connect_node_across_levels_         :3119-3136
//   search_to_insert_                   :3324-3392   (Walker::beam on level l, width = expansion_add)
//   connect_new_node_ / refine_         :3139-3160, :3515-3561   (Walker::refine to `connectivity` on EVERY level)
//   reconnect_neighbor_nodes_           :3163-3206   (reverse links; re-prune to M / M0 when a list is full)
//   choose_random_level_                :3208-3212   (same generator: minstd_rand0 + generate_canonical<double,53>)
// for BATCHES of vectors.  A batch is inserted in two kernels:
//   1. build_insert_kernel : one CTA per new node: greedy descent, efc-wide beam per level, heuristic neighbour
//      selection, writes the node's own lists and emits one reverse-link request per selected neighbour;
//   2. (radix sort of the requests by (level, target), segment heads)
//   3. build_reverse_kernel: one CTA per (level, target) segment applies the requests in insertion order: append
//      while the list has room, otherwise re-prune {new} + list with the same heuristic, distances measured from
//      the target (index.hpp:3194-3198).
// New nodes of one batch do not see each other during step 1 (they are linked to older nodes only).  With batch
// size 1 ("exact-order build") the procedure is the reference's sequential insertion: same levels, same lists,
// byte-identical file on data whose fp32 sums do not depend on summation order.  A node whose level exceeds the
// current top level always forms its own batch so that entry-point updates stay sequential.
//
// Group build (lb200_group_build, DESIGN.md 4.2): G GPUs of one process insert the same batches.  Every rank holds a full
// replica of the graph; rank r runs step 1 on a contiguous slice of the batch, every rank sorts the whole request array, and
// rank r applies the segments seg = r (mod G).  The replicated kernels (REP = true) store every list and every request
// into all replicas over NVLink, so that each phase stays one launch per rank.  The result is the one-GPU graph, byte for
// byte: no step depends on which CTA, or which GPU, does the work.
//
// Row-sharded group build (lb200_group_index_build): the same schedule and phases, but rank r's index holds only the rows of
// its range; the replicated kernels' TABLE instantiation reads every row, the new node's own included, through a per-launch
// table of the ranks' row arrays (RowTable, walk.cuh).
#include <cuda_runtime.h>

#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <type_traits>
#include <vector>

#include "group.h"
#include "walk.cuh"

namespace lb200 {

namespace {

struct BuildLaunch {
    GraphView g;
    SearchScratch s;
    uint32_t* adj0;      // mutable views of g.adj0 / g.upper_adj
    uint32_t* upper_adj;
    uint32_t u0, count;        // batch = nodes [u0, u0 + count)
    const int32_t* new_levels; // [count]
    const uint8_t* values;     // value (query side) of batch item i at values + i * value_stride; NULL = node u's row in `rows`
    size_t value_stride;
    uint32_t efc;
    uint32_t top_cap;
    uint32_t req_stride; // requests per batch item = M * (max_level + 1)
    unsigned long long* req_keys; // (level << 32) | target, ~0 = empty
    unsigned long long* req_vals; // (float bits of d(new, target) << 32) | new
    // reverse phase
    const unsigned long long* sorted_keys;
    const unsigned long long* sorted_vals;
    const uint32_t* seg_start;
    const uint32_t* nseg;
    uint32_t total_reqs;
    // group build: this rank applies segments seg_rank, seg_rank + seg_ranks, ... of the sorted requests (0, 1 on one GPU)
    uint32_t seg_rank, seg_ranks;
    // replicated kernels only: every rank's lists and request arrays (this rank's included), written through by both
    // phases; the request pointers are already offset to this rank's slice of the batch
    uint32_t reps;
    uint32_t* rep_adj0[kGroupMax];
    uint32_t* rep_upper_adj[kGroupMax];
    unsigned long long* rep_req_keys[kGroupMax];
    unsigned long long* rep_req_vals[kGroupMax];
    RowTable rows; // row-sharded group build (TABLE = true): where every row lives (walk.cuh)
};
static_assert(kGroupMax <= (int)kRowRangesMax, "one row range per rank");

template <class W0, bool REP, bool TABLE = false>
__global__ void __launch_bounds__(kWalkThreads) build_insert_kernel(const __grid_constant__ BuildLaunch p, const uint32_t R) {
    static_assert(REP || !TABLE, "the row table serves the replicated kernels only");
    using W = std::conditional_t<TABLE, typename RowTableWalker<W0>::type, W0>;
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const WalkLayout lay = W::layout(p.g, R, p.top_cap, p.g.M0 + 1);
    W w(p.g);
    if constexpr (W::kRowTable)
        w.rows = &p.rows;
    w.init(smem_raw, lay, R, p.s);
    WalkSmem& sm = w.sm;
    const uint32_t M = p.g.M, M0 = p.g.M0;

    for (;;) {
        __syncthreads();
        if (threadIdx.x == 0)
            sm.ctrl->item = (uint32_t)atomicAdd(&p.s.counters[0], 1ull);
        __syncthreads();
        const uint32_t item = sm.ctrl->item;
        if (item >= p.count)
            break;
        const uint32_t u = p.u0 + item;
        const int lu = p.new_levels[item];
        const uint8_t* urow;
        if constexpr (W::kRowTable)
            urow = p.values ? p.values + (size_t)item * p.value_stride : w.row_addr(u);
        else
            urow = p.values + (size_t)item * p.value_stride;
        w.load_value(urow);

        uint32_t cur = p.g.entry;
        float cur_d = w.measure_one(cur);
        w.greedy(cur, cur_d, p.g.max_level, lu); // levels max_level .. lu+1
        for (int level = min(lu, p.g.max_level); level >= 0; --level) {
            const uint32_t size = w.beam(level, cur, cur_d, p.efc, u);
            const uint32_t view = w.refine(size, M); // connect_new_node_: `connectivity` on every level (:3149)
            const uint32_t width = level ? M : M0;
            if constexpr (REP) {
                const size_t off = level ? ((size_t)p.g.upper_ref[u] + (level - 1)) * M : (size_t)u * M0;
                for (uint32_t r = 0; r < p.reps; ++r) {
                    uint32_t* list = (level ? p.rep_upper_adj[r] : p.rep_adj0[r]) + off;
                    for (uint32_t j = threadIdx.x; j < width; j += kWalkThreads)
                        list[j] = j < view ? (sm.top_i[j] & kIdMask) : kNoNeighbor;
                    for (uint32_t j = threadIdx.x; j < view; j += kWalkThreads) {
                        const size_t slot = (size_t)item * p.req_stride + (size_t)level * M + j;
                        const uint32_t v = sm.top_i[j] & kIdMask;
                        p.rep_req_keys[r][slot] = ((unsigned long long)(uint32_t)level << 32) | v;
                        p.rep_req_vals[r][slot] = ((unsigned long long)__float_as_uint(sm.top_d[j]) << 32) | u;
                    }
                }
            } else {
                uint32_t* list = level ? p.upper_adj + ((size_t)p.g.upper_ref[u] + (level - 1)) * M : p.adj0 + (size_t)u * M0;
                for (uint32_t j = threadIdx.x; j < width; j += kWalkThreads)
                    list[j] = j < view ? (sm.top_i[j] & kIdMask) : kNoNeighbor;
                for (uint32_t j = threadIdx.x; j < view; j += kWalkThreads) {
                    const size_t slot = (size_t)item * p.req_stride + (size_t)level * M + j;
                    const uint32_t v = sm.top_i[j] & kIdMask;
                    p.req_keys[slot] = ((unsigned long long)(uint32_t)level << 32) | v;
                    p.req_vals[slot] = ((unsigned long long)__float_as_uint(sm.top_d[j]) << 32) | u;
                }
            }
            cur = sm.top_i[0] & kIdMask, cur_d = sm.top_d[0]; // closest_slot = new_neighbors[0] (:3159)
            __syncthreads();
            if (level > 0)
                w.load_value(urow); // refine() used the value registers for candidate rows
        }
    }
    if (threadIdx.x == 0) {
        atomicAdd(&p.s.counters[1], (unsigned long long)w.st_dist);
        atomicAdd(&p.s.counters[2], (unsigned long long)w.st_pops);
        atomicAdd(&p.s.counters[3], (unsigned long long)w.st_hops);
    }
}

__global__ void segment_heads_kernel(const unsigned long long* __restrict__ keys, uint32_t n, uint32_t* __restrict__ seg_start,
                                     uint32_t* __restrict__ nseg) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    const unsigned long long k = keys[i];
    if (k == ~0ull)
        return;
    if (i == 0 || keys[i - 1] != k)
        seg_start[atomicAdd(nseg, 1u)] = i;
}

// Ordered compaction of the segment heads (group build): seg_start comes out ascending, so that every rank numbers the
// segments alike.  segment_heads_kernel's atomic order differs from run to run, which is harmless only when one rank
// applies every segment.
struct SegmentHead {
    const unsigned long long* keys;
    __device__ bool operator()(uint32_t i) const {
        const unsigned long long k = keys[i];
        return k != ~0ull && (i == 0 || keys[i - 1] != k);
    }
};

template <class W0, bool REP, bool TABLE = false>
__global__ void __launch_bounds__(kWalkThreads) build_reverse_kernel(const __grid_constant__ BuildLaunch p, const uint32_t R) {
    static_assert(REP || !TABLE, "the row table serves the replicated kernels only");
    using W = std::conditional_t<TABLE, typename RowTableWalker<W0>::type, W0>;
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const uint32_t M = p.g.M, M0 = p.g.M0;
    const WalkLayout lay = W::layout(p.g, R, M0 + 2, M0 + 1);
    W w(p.g);
    if constexpr (W::kRowTable)
        w.rows = &p.rows;
    w.init(smem_raw, lay, R, p.s);
    WalkSmem& sm = w.sm;
    uint32_t* lst_i = reinterpret_cast<uint32_t*>(smem_raw + lay.total);
    float* lst_d = reinterpret_cast<float*>(lst_i + M0);
    const uint32_t nseg = *p.nseg;

    for (;;) {
        __syncthreads();
        if (threadIdx.x == 0)
            sm.ctrl->item = (uint32_t)atomicAdd(&p.s.counters[0], 1ull);
        __syncthreads();
        const uint32_t seg = REP ? sm.ctrl->item * p.seg_ranks + p.seg_rank : sm.ctrl->item;
        if (seg >= nseg)
            break;
        const uint32_t s0 = p.seg_start[seg];
        const unsigned long long key = p.sorted_keys[s0];
        const int level = (int)(key >> 32);
        const uint32_t v = (uint32_t)key;
        const uint32_t cmax = level ? M : M0;
        uint32_t* list = level ? p.upper_adj + ((size_t)p.g.upper_ref[v] + (level - 1)) * M : p.adj0 + (size_t)v * M0;

        for (uint32_t j = threadIdx.x; j < cmax; j += kWalkThreads)
            lst_i[j] = list[j];
        __syncthreads();
        uint32_t cnt = 0; // leading valid entries (lists are compact)
        while (cnt < cmax && lst_i[cnt] != kNoNeighbor)
            ++cnt;
        bool have_d = false;

        for (uint32_t r = s0; r < p.total_reqs && p.sorted_keys[r] == key; ++r) {
            const unsigned long long val = p.sorted_vals[r];
            const uint32_t u = (uint32_t)val;
            const float d_uv = __uint_as_float((uint32_t)(val >> 32));
            __syncthreads();
            if (cnt < cmax) { // index.hpp:3186-3189
                if (threadIdx.x == 0)
                    lst_i[cnt] = u, lst_d[cnt] = d_uv;
                cnt++;
                continue;
            }
            if (!have_d) { // distances target -> each current neighbour (index.hpp:3196-3198)
                w.load_node(v);
                for (uint32_t j = threadIdx.x; j < cnt; j += kWalkThreads)
                    sm.cand_id[j] = lst_i[j];
                __syncthreads();
                w.eval(cnt);
                __syncthreads();
                for (uint32_t j = threadIdx.x; j < cnt; j += kWalkThreads)
                    lst_d[j] = sm.cand_d[j];
                w.st_dist += cnt;
                have_d = true;
                __syncthreads();
            }
            if (w.warp == 0) { // top = sorted {new} + successors, inserted in this order (insert_reserved, :3192-3198)
                uint32_t size = 0, cursor = 0;
                top_insert(sm.top_d, sm.top_i, size, cursor, cnt + 2, d_uv, u, w.lane);
                for (uint32_t j = 0; j < cnt; ++j)
                    top_insert(sm.top_d, sm.top_i, size, cursor, cnt + 2, lst_d[j], lst_i[j], w.lane);
            }
            __syncthreads();
            const uint32_t view = w.refine(cnt + 1, cmax);
            for (uint32_t j = threadIdx.x; j < view; j += kWalkThreads)
                lst_i[j] = sm.top_i[j] & kIdMask, lst_d[j] = sm.top_d[j];
            cnt = view;
        }
        __syncthreads();
        if constexpr (REP) {
            const size_t off = list - (level ? p.upper_adj : p.adj0);
            for (uint32_t r = 0; r < p.reps; ++r)
                for (uint32_t j = threadIdx.x; j < cmax; j += kWalkThreads)
                    (level ? p.rep_upper_adj[r] : p.rep_adj0[r])[off + j] = j < cnt ? lst_i[j] : kNoNeighbor;
        } else {
            for (uint32_t j = threadIdx.x; j < cmax; j += kWalkThreads)
                list[j] = j < cnt ? lst_i[j] : kNoNeighbor;
        }
    }
    if (threadIdx.x == 0)
        atomicAdd(&p.s.counters[1], (unsigned long long)w.st_dist);
}

// reference level generator (index.hpp:3208-3212 with libstdc++'s minstd_rand0 / generate_canonical<double,53>)
int draw_level(uint32_t& state, size_t M) {
    auto next = [&]() {
        state = (uint32_t)(((uint64_t)state * 16807ull) % 2147483647ull);
        return state;
    };
    const double Rr = 2147483646.0;
    double sum = (double)(next() - 1u);
    sum += (double)(next() - 1u) * Rr;
    double u = sum / (Rr * Rr);
    if (u >= 1.0)
        u = nextafter(1.0, 0.0);
    return (int)(int16_t)(-log(u) * (1.0 / log((double)M)));
}

template <typename T> struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    void ensure(size_t want) {
        if (want <= n)
            return;
        if (p)
            LB_CUDA(cudaFree(p));
        p = nullptr;
        n = want + want / 2;
        LB_CUDA(cudaMalloc(&p, n * sizeof(T)));
    }
    ~DevBuf() { cudaFree(p); }
};

// The batch schedule of a build: which nodes form each batch, and the graph (visible nodes, top level, entry point) the
// batch searches.  Host arithmetic only; the one-GPU and the group build both run it, so they insert the same batches.
struct BuildBatch {
    size_t pos, bsz;  // pending nodes [pos, pos + bsz)
    size_t visible;   // = n0 + pos
    int32_t max_level;
    uint32_t entry;
};
struct BuildPlan {
    std::vector<BuildBatch> batches;
    int32_t max_level; // after the last batch
    uint32_t entry;
    size_t max_reqs;   // largest request array of a batch
};

BuildPlan plan_batches(const Index& idx, const std::vector<int32_t>& new_levels, size_t batch_cap) {
    BuildPlan plan;
    const size_t P = new_levels.size(), M = idx.cfg_.M;
    size_t n = idx.n_, pos = 0;
    int32_t top = idx.max_level_;
    uint32_t entry = idx.entry_;
    plan.max_reqs = 0;
    if (n == 0) { // first node: entry point, no links (index.hpp:2538-2543)
        entry = 0, top = new_levels[0];
        n = 1, pos = 1;
    }
    while (pos < P) {
        size_t bsz = 1;
        if (new_levels[pos] <= top) {
            const size_t ramp = std::max<size_t>(1, n / idx.build_ratio_);
            bsz = std::min(std::min(P - pos, batch_cap), ramp);
            for (size_t i = 1; i < bsz; ++i)
                if (new_levels[pos + i] > top) {
                    bsz = i;
                    break;
                }
        }
        plan.batches.push_back({pos, bsz, n, top, entry});
        plan.max_reqs = std::max(plan.max_reqs, bsz * M * (size_t)(top + 1));
        if (new_levels[pos] > top) // index.hpp:2558-2562
            entry = (uint32_t)n, top = new_levels[pos];
        n += bsz, pos += bsz;
    }
    plan.max_level = top, plan.entry = entry;
    return plan;
}

// One rank's part of a build: its index (the root's own, or a replica), stream, request buffers, and the events that order
// the phases across ranks.
struct BuildRank {
    Index* idx = nullptr;
    int device = 0;
    cudaStream_t stream = 0; // the legacy stream on one GPU; a stream of its own per rank in a group
    DevBuf<int32_t> levels;
    DevBuf<unsigned long long> req_keys, req_vals, srt_keys, srt_vals;
    DevBuf<uint32_t> seg_start, nseg;
    DevBuf<uint8_t> cub_tmp;
    cudaEvent_t ev_ins = nullptr, ev_rev = nullptr; // end of this rank's phase 1 / phase 3 of the batch last enqueued
    ~BuildRank() {
        cudaSetDevice(device);
        if (stream) { // nothing of this call may still run once it has returned, also when it throws
            cudaStreamSynchronize(stream);
            cudaStreamDestroy(stream);
        }
        if (ev_ins)
            cudaEventDestroy(ev_ins);
        if (ev_rev)
            cudaEventDestroy(ev_rev);
    }
};

} // namespace

static void build_pending_impl(Index& idx, const std::vector<BuildReplica>& replicas, int root);

// Bookkeeping is transactional: if anything below throws (out of memory, launch failure) the level generator, the level /
// list counters and the node count are put back, so that a retry draws the same levels and inserts the same nodes again
// instead of double-inserting (pending_n_ is only cleared on success).
void build_pending_group(Index& idx, const std::vector<BuildReplica>& replicas, int root) {
    if (!idx.pending_n_)
        return;
    const uint32_t rng0 = idx.level_rng_;
    const size_t n0 = idx.n_, lists0 = idx.upper_lists_;
    const int32_t max_level0 = idx.max_level_;
    const uint32_t entry0 = idx.entry_;
    try {
        build_pending_impl(idx, replicas, root);
    } catch (...) {
        idx.level_rng_ = rng0, idx.n_ = n0, idx.upper_lists_ = lists0, idx.max_level_ = max_level0, idx.entry_ = entry0;
        idx.h_levels_.resize(n0);
        (void)cudaGetLastError();
        throw;
    }
    // the search screen's choice, once the index first holds enough rows.  Its basis and records belong on the root's device:
    // the ranks' clean-up above leaves the last rank's device current.
    int cur = 0;
    LB_CUDA(cudaGetDevice(&cur));
    LB_CUDA(cudaSetDevice(replicas[root].device));
    idx.decide_screen();
    LB_CUDA(cudaSetDevice(cur));
}

void build_pending(Index& idx) {
    if (idx.sharded_)
        throw CudaError("build: this index's rows are spread over a group; build it with lb200_group_index_build");
    int dev = 0;
    LB_CUDA(cudaGetDevice(&dev));
    build_pending_group(idx, std::vector<BuildReplica>(1, BuildReplica{&idx, dev}), 0);
}

// replicas[r] = rank r's index and device, replicas[root].idx == &idx.  The other ranks' indexes hold the root's rows
// [0, n0 + P), lists of nodes [0, n0) and level-1+ lists; this function gives them the new nodes' upper lists and keys.
static void build_pending_impl(Index& idx, const std::vector<BuildReplica>& replicas, int root) {
    const size_t P = idx.pending_n_;
    if (!P)
        return;
    const IndexConfig& cfg = idx.cfg_;
    const size_t n0 = idx.n_;
    const uint32_t M = (uint32_t)cfg.M, M0 = (uint32_t)cfg.M0;
    const uint32_t G = (uint32_t)replicas.size();
    const bool group = G > 1;
    if (G < 1 || G > (uint32_t)kGroupMax || root < 0 || (uint32_t)root >= G || replicas[root].idx != &idx)
        throw CudaError("build: bad rank layout");
    // row-sharded (a group's own index, group.cu): rank r's index holds rows [row_lo_, row_hi_) only, the ranks' ranges tile
    // [0, capacity) in rank order, and the replicated kernels read every row through the ranks' table
    const bool sharded = idx.sharded_;
    if (sharded) {
        if (cfg.pq)
            throw CudaError("build: a row-sharded index cannot hold pq codes");
        for (uint32_t r = 0; r < G; ++r)
            if (!replicas[r].idx->sharded_ || replicas[r].idx->row_lo_ != (r ? replicas[r - 1].idx->row_hi_ : 0))
                throw CudaError("build: the ranks' row ranges do not tile the index");
        if (replicas[G - 1].idx->row_hi_ < n0 + P)
            throw CudaError("build: pending rows beyond the ranks' row ranges");
    }

    // ---- levels + upper-list allocation for the new nodes ----
    idx.h_levels_.resize(n0 + P);
    std::vector<int32_t> new_levels(P);
    std::vector<uint32_t> new_upper_ref(P, kNoNeighbor);
    size_t lists = idx.upper_lists_;
    for (size_t i = 0; i < P; ++i) {
        int l = draw_level(idx.level_rng_, cfg.M);
        new_levels[i] = l;
        idx.h_levels_[n0 + i] = (int16_t)l;
        if (l > 0) {
            new_upper_ref[i] = (uint32_t)lists;
            lists += (size_t)l;
        }
    }

    // ---- kernel geometry (the batch cap from the root's device and the one-GPU kernels, so that it is G x the one-GPU
    // default) ----
    const uint32_t row_bytes = (uint32_t)idx.row_bytes_;
    const uint32_t R = pick_ring_slots(row_bytes);
    const int nq = cfg.pq ? 1 : pick_nq(row_bytes);
    if (nq < 0)
        throw CudaError("build: vectors wider than 8192 bytes are not supported");
    const uint32_t top_cap = (uint32_t)std::max<size_t>(cfg.efc, M0 + 2);
    const GraphView gv0 = idx.view();
    const size_t smem_ins = cfg.pq ? walk_layout_pq(gv0.num_subvectors, gv0.pq_lut_width, pq_value_floats(gv0), top_cap, M0 + 1).total
                                   : walk_layout(R, row_bytes, top_cap, M0 + 1).total;
    const size_t smem_rev = (cfg.pq ? walk_layout_pq(gv0.num_subvectors, gv0.pq_lut_width, pq_value_floats(gv0), M0 + 2, M0 + 1).total
                                    : walk_layout(R, row_bytes, M0 + 2, M0 + 1).total) + (size_t)M0 * 8;
    int occ_ins = 0, occ_rev = 0;
    const uint32_t sms = (uint32_t)device_sm_count();
    auto occupancy = [&](auto kernel, size_t smem) {
        int occ = 0;
        LB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        LB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, kWalkThreads, smem));
        if (occ < 1)
            throw CudaError("build: kernel does not fit on an SM (expansion_add too large for shared memory?)");
        return occ;
    };
    std::vector<BuildRank> rk(G);
    std::vector<uint32_t> grid_ins(G), grid_rev(G); // resident CTAs of the kernels each rank launches
    for (uint32_t r = 0; r < G; ++r) {
        BuildRank& b = rk[r];
        b.idx = replicas[r].idx, b.device = replicas[r].device;
        LB_CUDA(cudaSetDevice(b.device));
        dispatch_walker(cfg.pq, idx.dist_mode_, cfg.scalar_kind, nq, [&](auto tag) {
            using W = typename decltype(tag)::type;
            if ((int)r == root) {
                occ_ins = occupancy(build_insert_kernel<W, false>, smem_ins);
                occ_rev = occupancy(build_reverse_kernel<W, false>, smem_rev);
            }
            if (!group) {
                grid_ins[r] = sms * occ_ins, grid_rev[r] = sms * occ_rev;
            } else if (!sharded) {
                grid_ins[r] = sms * occupancy(build_insert_kernel<W, true>, smem_ins);
                grid_rev[r] = sms * occupancy(build_reverse_kernel<W, true>, smem_rev);
            } else if constexpr (W::kTableWalker) {
                grid_ins[r] = sms * occupancy(build_insert_kernel<W, true, true>, smem_ins);
                grid_rev[r] = sms * occupancy(build_reverse_kernel<W, true, true>, smem_rev);
            }
        });
        b.idx->ensure_scratch(std::max(grid_ins[r], grid_rev[r]));
        if (group) {
            LB_CUDA(cudaStreamCreateWithFlags(&b.stream, cudaStreamNonBlocking));
            LB_CUDA(cudaEventCreateWithFlags(&b.ev_ins, cudaEventDisableTiming));
            LB_CUDA(cudaEventCreateWithFlags(&b.ev_rev, cudaEventDisableTiming));
        }
    }
    const size_t batch_cap = idx.build_batch_ ? idx.build_batch_ : (size_t)G * occ_ins * sms;
    const BuildPlan plan = plan_batches(idx, new_levels, batch_cap);
    const std::vector<BuildBatch>& batches = plan.batches;

    // ---- per rank: the new nodes' levels, upper lists and keys; request buffers sized for the largest batch ----
    const size_t max_reqs = std::max<size_t>(plan.max_reqs, 1);
    const int end_bit = 32 + 8; // levels < 256
    size_t sort_bytes = 0, select_bytes = 0;
    LB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                            (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)max_reqs, 0, end_bit));
    if (group)
        LB_CUDA(cub::DeviceSelect::If(nullptr, select_bytes, thrust::counting_iterator<uint32_t>(0), (uint32_t*)nullptr,
                                      (uint32_t*)nullptr, (int)max_reqs, SegmentHead{nullptr}));
    for (uint32_t r = 0; r < G; ++r) {
        BuildRank& b = rk[r];
        Index& x = *b.idx;
        LB_CUDA(cudaSetDevice(b.device));
        x.alloc_upper(lists + 1);
        x.upper_lists_ = lists;
        b.levels.ensure(P);
        b.req_keys.ensure(max_reqs), b.req_vals.ensure(max_reqs), b.srt_keys.ensure(max_reqs), b.srt_vals.ensure(max_reqs);
        b.seg_start.ensure(max_reqs), b.nseg.ensure(1);
        b.cub_tmp.ensure(std::max(sort_bytes, select_bytes));
        LB_CUDA(cudaMemcpyAsync(b.levels.p, new_levels.data(), P * sizeof(int32_t), cudaMemcpyHostToDevice, b.stream));
        LB_CUDA(cudaMemcpyAsync(x.d_upper_ref_ + n0, new_upper_ref.data(), P * sizeof(uint32_t), cudaMemcpyHostToDevice, b.stream));
        LB_CUDA(cudaMemcpyAsync(x.d_keys_ + n0, idx.h_keys_.data() + n0, P * sizeof(uint64_t), cudaMemcpyHostToDevice, b.stream));
        // work counters of this build (SURVEY 8d build metric: sum of computed_distances(add) x row bytes / time)
        LB_CUDA(cudaMemsetAsync(x.scratch_.counters, 0, 8 * sizeof(unsigned long long), b.stream));
        if (!batches.empty())
            LB_CUDA(cudaMemsetAsync(b.req_keys.p, 0xFF, batches[0].bsz * M * (size_t)(batches[0].max_level + 1) * sizeof(unsigned long long),
                                    b.stream));
        if (group) // the rows and lists were written on the legacy stream, which a rank's own stream does not wait for
            LB_CUDA(cudaDeviceSynchronize());
    }
    LB_CUDA(cudaSetDevice(rk[root].device));
    LB_CUDA(cudaEventRecord(idx.ev0_, rk[root].stream));

    // Per batch: phase 1 on every rank, then phases 2 and 3 on every rank.  Across ranks, phase 2 waits for every rank's
    // phase 1 and the next phase 1 waits for every rank's phase 3 (cudaStreamWaitEvent, no host synchronisation).  The
    // peer stores of a kernel are visible to work that waits, through an event, for that kernel's completion: that is the
    // only ordering the replicas rely on.  A rank's request array receives its peers' phase-1 stores, so it is cleared for
    // the next batch right after its own sort, before the event that releases the next phase 1.
    for (size_t bi = 0; bi < batches.size(); ++bi) {
        const BuildBatch& bt = batches[bi];
        const size_t pos = bt.pos, bsz = bt.bsz;
        const uint32_t u0 = (uint32_t)(n0 + pos);
        const uint32_t req_stride = M * ((uint32_t)bt.max_level + 1);
        const size_t nreq = bsz * req_stride;
        for (uint32_t r = 0; r < G; ++r) { // host mirrors: the same graph state on every rank
            rk[r].idx->n_ = bt.visible, rk[r].idx->max_level_ = bt.max_level, rk[r].idx->entry_ = bt.entry;
        }
        std::vector<BuildLaunch> p(G);
        for (uint32_t r = 0; r < G; ++r) {
            BuildRank& b = rk[r];
            Index& x = *b.idx;
            const size_t s0 = bsz * r / G, s1 = bsz * (r + 1) / G; // this rank's slice of the batch
            BuildLaunch& q = p[r];
            q = BuildLaunch{};
            q.g = x.view();
            q.s = x.scratch_;
            q.adj0 = x.d_adj0_, q.upper_adj = x.d_upper_adj_;
            q.u0 = u0 + (uint32_t)s0, q.count = (uint32_t)(s1 - s0);
            q.new_levels = b.levels.p + pos + s0;
            if (cfg.pq) { // value = the raw f32 vector; stored side = codes
                q.value_stride = round_up(cfg.dims * 4, 16);
                q.values = (const uint8_t*)x.d_pending_raw_ + (pos + s0) * q.value_stride;
            } else if (sharded && group) { // the new node's row may live on any rank: read it through the table
                q.value_stride = row_bytes;
                q.values = nullptr;
            } else {
                q.value_stride = row_bytes;
                q.values = x.d_vectors_ + (size_t)q.u0 * row_bytes;
            }
            q.efc = (uint32_t)cfg.efc, q.top_cap = top_cap;
            q.req_stride = req_stride;
            q.req_keys = b.req_keys.p + s0 * req_stride, q.req_vals = b.req_vals.p + s0 * req_stride;
            q.sorted_keys = b.srt_keys.p, q.sorted_vals = b.srt_vals.p;
            q.seg_start = b.seg_start.p, q.nseg = b.nseg.p;
            q.total_reqs = (uint32_t)nreq;
            q.seg_rank = r, q.seg_ranks = G;
            q.reps = G;
            for (uint32_t t = 0; t < G; ++t) {
                q.rep_adj0[t] = rk[t].idx->d_adj0_, q.rep_upper_adj[t] = rk[t].idx->d_upper_adj_;
                q.rep_req_keys[t] = rk[t].req_keys.p + s0 * req_stride, q.rep_req_vals[t] = rk[t].req_vals.p + s0 * req_stride;
            }
            if (sharded) { // every rank's slice: its own, and its peers' through peer mappings (one process, UVA pointers)
                q.rows.count = G, q.rows.own = r;
                for (uint32_t t = 0; t < G; ++t)
                    q.rows.hi[t] = (uint32_t)rk[t].idx->row_hi_, q.rows.base[t] = rk[t].idx->d_vectors_;
            }
        }
        // phase 1: rank r inserts its slice
        for (uint32_t r = 0; r < G; ++r) {
            BuildRank& b = rk[r];
            LB_CUDA(cudaSetDevice(b.device));
            if (group)
                for (uint32_t t = 0; t < G; ++t)
                    if (t != r)
                        LB_CUDA(cudaStreamWaitEvent(b.stream, rk[t].ev_rev, 0));
            LB_CUDA(cudaMemsetAsync(b.idx->scratch_.counters, 0, sizeof(unsigned long long), b.stream));
            LB_CUDA(cudaMemsetAsync(b.nseg.p, 0, sizeof(uint32_t), b.stream));
            const uint32_t grid = (uint32_t)std::min<size_t>(p[r].count, grid_ins[r]);
            if (grid) {
                dispatch_walker(cfg.pq, idx.dist_mode_, cfg.scalar_kind, nq, [&](auto tag) {
                    using W = typename decltype(tag)::type;
                    if (!group)
                        build_insert_kernel<W, false><<<grid, kWalkThreads, smem_ins, b.stream>>>(p[r], R);
                    else if (!sharded)
                        build_insert_kernel<W, true><<<grid, kWalkThreads, smem_ins, b.stream>>>(p[r], R);
                    else if constexpr (W::kTableWalker)
                        build_insert_kernel<W, true, true><<<grid, kWalkThreads, smem_ins, b.stream>>>(p[r], R);
                });
                LB_CUDA(cudaGetLastError());
                count_launch();
            }
            if (group)
                LB_CUDA(cudaEventRecord(b.ev_ins, b.stream));
        }
        // phase 2: every rank sorts the whole request array; phase 3: rank r applies segments r, r + G, ...
        const size_t next_reqs = bi + 1 < batches.size() ? batches[bi + 1].bsz * M * (size_t)(batches[bi + 1].max_level + 1) : 0;
        for (uint32_t r = 0; r < G; ++r) {
            BuildRank& b = rk[r];
            LB_CUDA(cudaSetDevice(b.device));
            if (group)
                for (uint32_t t = 0; t < G; ++t)
                    if (t != r)
                        LB_CUDA(cudaStreamWaitEvent(b.stream, rk[t].ev_ins, 0));
            size_t tmp_bytes = b.cub_tmp.n;
            // keys ~0 (empty) have all bits set and therefore sort last within the examined bits as well
            LB_CUDA(cub::DeviceRadixSort::SortPairs(b.cub_tmp.p, tmp_bytes, b.req_keys.p, b.srt_keys.p, b.req_vals.p, b.srt_vals.p,
                                                    (int)nreq, 0, end_bit, b.stream));
            count_launch(2);
            if (next_reqs)
                LB_CUDA(cudaMemsetAsync(b.req_keys.p, 0xFF, next_reqs * sizeof(unsigned long long), b.stream));
            if (group) {
                tmp_bytes = b.cub_tmp.n;
                LB_CUDA(cub::DeviceSelect::If(b.cub_tmp.p, tmp_bytes, thrust::counting_iterator<uint32_t>(0), b.seg_start.p, b.nseg.p,
                                              (int)nreq, SegmentHead{b.srt_keys.p}, b.stream));
                count_launch(2);
            } else {
                segment_heads_kernel<<<(unsigned)((nreq + 255) / 256), 256, 0, b.stream>>>(b.srt_keys.p, (uint32_t)nreq, b.seg_start.p,
                                                                                          b.nseg.p);
                LB_CUDA(cudaGetLastError());
                count_launch();
            }
            LB_CUDA(cudaMemsetAsync(b.idx->scratch_.counters, 0, sizeof(unsigned long long), b.stream));
            const uint32_t grid = (uint32_t)std::min<size_t>(nreq, grid_rev[r]);
            dispatch_walker(cfg.pq, idx.dist_mode_, cfg.scalar_kind, nq, [&](auto tag) {
                using W = typename decltype(tag)::type;
                if (!group)
                    build_reverse_kernel<W, false><<<grid, kWalkThreads, smem_rev, b.stream>>>(p[r], R);
                else if (!sharded)
                    build_reverse_kernel<W, true><<<grid, kWalkThreads, smem_rev, b.stream>>>(p[r], R);
                else if constexpr (W::kTableWalker)
                    build_reverse_kernel<W, true, true><<<grid, kWalkThreads, smem_rev, b.stream>>>(p[r], R);
            });
            LB_CUDA(cudaGetLastError());
            count_launch();
            if (group)
                LB_CUDA(cudaEventRecord(b.ev_rev, b.stream));
        }
    }
    idx.n_ = n0 + P, idx.max_level_ = plan.max_level, idx.entry_ = plan.entry;

    BuildRank& br = rk[root];
    LB_CUDA(cudaSetDevice(br.device));
    if (group)
        for (uint32_t t = 0; t < G; ++t)
            if (t != (uint32_t)root)
                LB_CUDA(cudaStreamWaitEvent(br.stream, rk[t].ev_rev, 0));
    LB_CUDA(cudaEventRecord(idx.ev1_, br.stream));
    unsigned long long dist = 0;
    for (uint32_t r = 0; r < G; ++r) { // work counters summed over ranks
        LB_CUDA(cudaSetDevice(rk[r].device));
        LB_CUDA(cudaStreamSynchronize(rk[r].stream));
        unsigned long long c[4] = {0, 0, 0, 0};
        LB_CUDA(cudaMemcpy(c, rk[r].idx->scratch_.counters, sizeof(c), cudaMemcpyDeviceToHost));
        dist += c[1];
    }
    LB_CUDA(cudaSetDevice(br.device));
    idx.pending_n_ = 0;
    {
        float ms = 0.f;
        LB_CUDA(cudaEventElapsedTime(&ms, idx.ev0_, idx.ev1_));
        idx.last_build_ms_ = ms, idx.last_build_dist_ = dist, idx.last_build_n_ = P;
        idx.last_nq_ = 0; // the events now bracket a build, not a search
    }
    if (idx.d_pending_raw_) { // raw rows are only needed while inserting
        LB_CUDA(cudaFree(idx.d_pending_raw_));
        idx.d_pending_raw_ = nullptr, idx.pending_raw_cap_ = 0;
    }
}

} // namespace lb200

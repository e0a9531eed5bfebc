// lantern_b200 -- the graph walker shared by the search and build kernels.
//
// One CTA (4 warps) executes, for one "value" (a query or a vector being inserted), the reference's
//   search_for_one_            U/include/usearch/index.hpp:3277-3316   -> Walker::greedy
//   search_to_find_in_base_    :3400-3485                              -> Walker::beam(level 0)
//   search_to_insert_          :3324-3392                              -> Walker::beam(level l)
//   refine_                    :3515-3561                              -> Walker::refine
// with the same decision sequence (stored neighbour order, strict '<', insert-before-equal, evict-last).
// The candidate queue (`next`, a max-heap on -distance in the reference) is represented by "unexpanded"
// flags on the sorted `top` list: an element evicted from `top` has distance >= radius and can never be
// popped before the stop test (:3445 / :3351) fires, so both formulations expand the same nodes; they can
// differ only for exact distance ties.
//
// Data movement: neighbour rows travel HBM -> shared memory as 1-D bulk async copies (TMA engine,
// `cp.async.bulk`, mbarrier complete_tx).  Candidate j of a batch is served by warp j%4, which owns the
// ring slots {warp, warp+4, ...} and refills a slot itself right after reading it, so a warp's pipeline
// needs no cross-warp synchronisation.  Distances are reduced with warp shuffles (distance.cuh).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdlib.h>

#include "distance.cuh"
#include "engine.h"
#include "screen.cuh"

namespace lb200 {

constexpr int kWalkThreads = 128;
constexpr int kWalkWarps = kWalkThreads / 32;
constexpr uint32_t kDone = 0xFFFFFFFFu;
constexpr uint32_t kIdMask = 0x7FFFFFFFu;

struct WalkCtrl {
    uint32_t item;     // current work item (query / node / segment)
    uint32_t n;        // candidates in cand_id[], or kDone
    uint32_t ntouched; // entries in the touched list
    uint32_t top_size; // size of the top list after a beam
    uint32_t m;        // screened walkers: candidates left after the screen
    float radius;      // screened walkers: radius the round's candidates are screened against (NaN = no screen this round)
    uint32_t screened, rejected; // screened walkers: candidates screened / rejected by this CTA (kept here, not in registers)
};

struct WalkSmem {
    uint8_t* ring;
    uint64_t* full;
    float* top_d;
    uint32_t* top_i;
    uint32_t* cand_id;
    float* cand_d;
    uint32_t* limbo; // unexpanded entries evicted from the top list at exactly the current radius (distance ties)
    WalkCtrl* ctrl;
};

struct WalkLayout {
    size_t full, top_d, top_i, cand_id, cand_d, limbo, ctrl, total;
};
constexpr uint32_t kLimboCap = 64;

// `stage_bytes` of value/row staging, `nbar` mbarriers, a top list of `top_cap` entries, candidate arrays of `cand_cap`.
__host__ __device__ inline WalkLayout walk_layout_bytes(size_t stage_bytes, uint32_t nbar, uint32_t top_cap, uint32_t cand_cap) {
    WalkLayout l;
    size_t o = stage_bytes;
    o = (o + 15) & ~(size_t)15;
    l.full = o, o += (size_t)nbar * 8;
    l.top_d = o, o += (size_t)top_cap * 4;
    l.top_i = o, o += (size_t)top_cap * 4;
    l.cand_id = o, o += (size_t)cand_cap * 4;
    l.cand_d = o, o += (size_t)cand_cap * 4;
    l.limbo = o, o += (size_t)kLimboCap * 4;
    o = (o + 15) & ~(size_t)15;
    l.ctrl = o, o += sizeof(WalkCtrl);
    l.total = o;
    return l;
}
// R ring slots of row_bytes (plain rows)
__host__ __device__ inline WalkLayout walk_layout(uint32_t R, uint32_t row_bytes, uint32_t top_cap, uint32_t cand_cap) {
    return walk_layout_bytes((size_t)R * row_bytes, R, top_cap, cand_cap);
}
// PQ: look-up table of pq_table_floats(nsub, lut_width) floats ([nsub][lut_width] padded to whole 16-byte chunks, then the
// value's squared norm, which travels with a precomputed table) + value staging [dims] + per-warp partial sums [warps][2][64];
// one mbarrier (bulk copy of a precomputed table)
constexpr uint32_t kPqPartPerWarp = 64;
// `value_floats` = dims when the kernel builds tables itself from raw vectors (build; search without precomputed tables), else 0
__host__ __device__ inline WalkLayout walk_layout_pq(uint32_t nsub, uint32_t lut_width, uint32_t value_floats, uint32_t top_cap, uint32_t cand_cap) {
    return walk_layout_bytes((pq_table_floats(nsub, lut_width) + value_floats + (size_t)kWalkWarps * 2 * kPqPartPerWarp) * 4, 1, top_cap, cand_cap);
}
__host__ __device__ inline uint32_t pq_value_floats(const GraphView& g) { return g.pq_query_tables ? 0u : g.dims; }

inline uint32_t pick_ring_slots(uint32_t row_bytes) {
    uint32_t budget = 24u * 1024u; // 8 slots of a d=768 f32 row: 8 CTAs/SM
    if (const char* e = getenv("LB200_RING_BYTES")) // tuning knob (bytes of row staging per CTA)
        budget = (uint32_t)atoi(e);
    uint32_t r = (budget / row_bytes) & ~3u;
    if (r < 4)
        r = 4;
    if (r > 16) // narrow rows: more resident CTAs beat deeper rings (768-byte rows: 16 slots beat 32)
        r = 16;
    return r;
}

inline int pick_nq(uint32_t row_bytes) {
    const uint32_t need = (row_bytes / 16 + 31) / 32;
    const int opts[] = {1, 2, 3, 4, 6, 8, 12, 16};
    for (int o : opts)
        if ((uint32_t)o >= need)
            return o;
    return -1;
}

// Warp-cooperative sorted insert == sorted_buffer_gt::insert (index.hpp:752-763): position = lower_bound
// (new element goes BEFORE equal ones), tail evicted when the list is full.
// Precondition (index.hpp:3470): size < L || d < top_d[size-1].
// `ev_d`/`ev_i` receive the evicted tail (ev_i = kNoNeighbor when nothing was evicted).
__device__ __forceinline__ void top_insert(float* td, uint32_t* ti, uint32_t& size, uint32_t& cursor, uint32_t L, float d,
                                           uint32_t id, int lane, float& ev_d, uint32_t& ev_i) {
    ev_i = kNoNeighbor, ev_d = 0.f;
    if (size == L)
        ev_d = td[L - 1], ev_i = ti[L - 1];
    __syncwarp();
    uint32_t pos = 0;
    for (uint32_t b = 0; b < size; b += 32) {
        uint32_t e = b + lane;
        bool less = e < size && td[e] < d;
        pos += __popc(__ballot_sync(0xffffffffu, less));
    }
    const uint32_t last = (size == L) ? L - 1 : size;
    for (int hi = (int)last; hi > (int)pos; hi -= 32) {
        int idx = hi - lane;
        bool act = idx > (int)pos;
        float vd = 0.f;
        uint32_t vi = 0;
        if (act)
            vd = td[idx - 1], vi = ti[idx - 1];
        __syncwarp();
        if (act)
            td[idx] = vd, ti[idx] = vi;
        __syncwarp();
    }
    __syncwarp(); // the position scan's reads are ordered before this write even when nothing was shifted (racecheck)
    if (lane == 0)
        td[pos] = d, ti[pos] = id;
    __syncwarp();
    size = last + 1;
    if (pos <= cursor)
        cursor = pos;
}
__device__ __forceinline__ void top_insert(float* td, uint32_t* ti, uint32_t& size, uint32_t& cursor, uint32_t L, float d,
                                           uint32_t id, int lane) {
    float ev_d;
    uint32_t ev_i;
    top_insert(td, ti, size, cursor, L, d, id, lane, ev_d, ev_i);
}

// ---- the top-`L` list of one walk (warp 0 only) ------------------------------------------------------------------
// sorted_buffer_gt (index.hpp:668-780): ascending by distance, insert at lower_bound (before equal elements), evict the
// tail when full; entries carry an "expanded" flag (kExpandedBit) that replaces the reference's separate candidate heap.
struct TopSmem { // arrays in shared memory
    float* td;
    uint32_t* ti;
    uint32_t size, cursor, L;
    __device__ __forceinline__ void init(const WalkSmem& sm, uint32_t cap, float d, uint32_t id, int lane) {
        td = sm.top_d, ti = sm.top_i, L = cap, size = 1, cursor = 0;
        if (lane == 0)
            td[0] = d, ti[0] = id;
        __syncwarp();
    }
    // closest unexpanded entry -> c (marked expanded); false when none is left
    __device__ __forceinline__ bool pop(uint32_t& c, int lane) {
        if (cursor >= size)
            return false;
        c = ti[cursor];
        __syncwarp();
        if (lane == 0)
            ti[cursor] = c | kExpandedBit;
        __syncwarp();
        uint32_t nxt = size;
        for (uint32_t b = cursor + 1; b < size; b += 32) {
            uint32_t e = b + lane;
            bool un = e < size && !(ti[e] & kExpandedBit);
            uint32_t m = __ballot_sync(0xffffffffu, un);
            if (m) {
                nxt = b + __ffs(m) - 1;
                break;
            }
        }
        cursor = nxt;
        return true;
    }
    __device__ __forceinline__ float radius(int) const { return td[size - 1]; }
    __device__ __forceinline__ void insert(float d, uint32_t id, int lane, float& ev_d, uint32_t& ev_i) {
        top_insert(td, ti, size, cursor, L, d, id, lane, ev_d, ev_i);
    }
    __device__ __forceinline__ void flush(int) {}
};

// value -> registers (lane l holds chunks l, l+32, ...); returns |value|^2 for cos (0 otherwise)
template <int DM, int SK, int NQ>
__device__ __forceinline__ float load_qreg(uint4 (&qreg)[NQ], const uint8_t* row, uint32_t nchunks, int lane) {
    const uint4* qg = reinterpret_cast<const uint4*>(row);
    float part = 0.f;
#pragma unroll
    for (int i = 0; i < NQ; ++i) {
        uint32_t c = lane + 32 * i;
        qreg[i] = c < nchunks ? __ldg(qg + c) : make_uint4(0, 0, 0, 0);
        part = norm_add(part, query_norm_chunk<DM, SK>(qreg[i]));
    }
    if constexpr (DM == DM_COS)
        return warp_sum(part);
    return 0.f;
}

// distance value (registers) -> one stored row (shared or global memory); every lane receives it
template <int DM, int SK, int NQ>
__device__ __forceinline__ float row_distance(const uint4 (&qreg)[NQ], const uint4* row, uint32_t nchunks, float a2, int lane) {
    DistAcc<DM, SK> acc;
    acc.reset();
#pragma unroll
    for (int i = 0; i < NQ; ++i) {
        uint32_t c = lane + 32 * i;
        if (c < nchunks) {
            uint4 r = row[c];
            accum_chunk<DM, SK>(acc, qreg[i], r);
        }
    }
    return finish_distance<DM, SK>(acc, a2);
}

// state shared by every evaluator / walker
struct WalkBase {
    static constexpr bool kScreen = false; // ScreenEval: the level-0 beam screens candidates before measuring them
    static constexpr bool kRowTable = false; // RowEval<..., true>: rows addressed through a RowTable
    static constexpr bool kTableWalker = false; // plain rows: a RowEval<..., true> twin exists (RowTableWalker)
    const GraphView& g; // the kernel's own (__grid_constant__) parameter: fields are read from the constant bank
    WalkSmem sm;
    uint32_t* vis;
    uint32_t* touched;
    uint32_t touched_cap;
    size_t words_per_cta;
    int warp, lane;
    uint32_t st_dist, st_pops, st_hops; // per-launch work counters; thread 0's copy is the one that is reported
    uint32_t st_limbo_drop;             // equal-distance candidates that did not fit in limbo (the walk then expands fewer nodes)

    __device__ __forceinline__ explicit WalkBase(const GraphView& gv) : g(gv) {}
    __device__ __forceinline__ void init_base(uint8_t* smem_raw, const WalkLayout& lay, const SearchScratch& s) {
        sm.ring = smem_raw;
        sm.full = reinterpret_cast<uint64_t*>(smem_raw + lay.full);
        sm.top_d = reinterpret_cast<float*>(smem_raw + lay.top_d);
        sm.top_i = reinterpret_cast<uint32_t*>(smem_raw + lay.top_i);
        sm.cand_id = reinterpret_cast<uint32_t*>(smem_raw + lay.cand_id);
        sm.cand_d = reinterpret_cast<float*>(smem_raw + lay.cand_d);
        sm.limbo = reinterpret_cast<uint32_t*>(smem_raw + lay.limbo);
        sm.ctrl = reinterpret_cast<WalkCtrl*>(smem_raw + lay.ctrl);
        warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        st_dist = st_pops = st_hops = 0;
        st_limbo_drop = 0;
        vis = s.visited + (size_t)blockIdx.x * s.words_per_cta;
        touched = s.touched + (size_t)blockIdx.x * s.touched_cap;
        touched_cap = s.touched_cap;
        words_per_cta = s.words_per_cta;
    }
};

// Where the rows of a replicated build live (build.cu): `count` contiguous ranges, range t = rows [hi[t-1], hi[t]) (hi[-1] = 0)
// starting at base[t].  A full-replica group build passes one range, the rank's own copy; a row-sharded one passes every
// rank's slice, peers' slices as peer-mapped pointers.  Range `own` is in this rank's memory and travels by bulk copy; the
// PTX ISA does not say whether cp.async.bulk may read a peer-mapped address, so rows of the other ranges are read with
// ordinary 16-byte loads (the same bytes land in the same ring slot, so no distance can differ).
constexpr uint32_t kRowRangesMax = 8;
struct RowTable {
    uint32_t count, own;
    uint32_t hi[kRowRangesMax];
    const uint8_t* base[kRowRangesMax];
    __device__ __forceinline__ const uint8_t* row(uint32_t id, uint32_t row_bytes, uint32_t& t) const {
        uint32_t lo = 0;
        t = 0;
        while (t + 1 < count && id >= hi[t])
            lo = hi[t++];
        return base[t] + (size_t)(id - lo) * row_bytes;
    }
};

// ---- evaluator for plain rows (f32 / f16 / i8 / b1): value in registers, rows through the bulk-copy ring --------
// TABLE = rows are addressed through a RowTable (replicated build kernels only); otherwise at g.vectors + id * row_bytes.
template <int DM, int SK, int NQ, bool TABLE = false> struct RowEval : WalkBase {
    static constexpr bool kRowTable = TABLE;
    static constexpr bool kTableWalker = true;
    const RowTable* rows = nullptr; // TABLE: the kernel's own (__grid_constant__) table
    __device__ __forceinline__ const uint8_t* row_addr(uint32_t id) const {
        if constexpr (TABLE) {
            uint32_t t;
            return rows->row(id, g.row_bytes, t);
        }
        return g.vectors + (size_t)id * g.row_bytes;
    }
    static __host__ __device__ WalkLayout layout(const GraphView& g, uint32_t R, uint32_t top_cap, uint32_t cand_cap) {
        return walk_layout(R, g.row_bytes, top_cap, cand_cap);
    }
    uint4 qreg[NQ];
    float a2;
    uint32_t phase_bits;
    uint32_t nchunks, R, SPW, NW;

    __device__ __forceinline__ explicit RowEval(const GraphView& gv) : WalkBase(gv) {}
    __device__ __forceinline__ void init(uint8_t* smem_raw, const WalkLayout& lay, uint32_t ring_slots, const SearchScratch& s) {
        init_base(smem_raw, lay, s);
        nchunks = g.row_bytes / 16;
        NW = blockDim.x >> 5; // 4 warps per query, or 2 for narrow rows (search.cu): uniform across the CTA
        R = ring_slots, SPW = ring_slots / NW;
        phase_bits = 0;
        a2 = 0.f;
        if (threadIdx.x == 0) {
            for (uint32_t i = 0; i < R; ++i)
                mbar_init(&sm.full[i], 1);
            fence_mbar_init();
        }
        __syncthreads();
    }

    // value -> registers; every warp keeps its own copy.  `row` points to a 16-byte padded row in global memory.
    __device__ __forceinline__ void load_value(const uint8_t* row) {
        const float n2 = load_qreg<DM, SK, NQ>(qreg, row, nchunks, lane);
        if constexpr (DM == DM_COS)
            a2 = n2;
    }
    // a stored node becomes the value (refine_: candidate vs accepted; reverse links: target vs its neighbours)
    __device__ __forceinline__ void load_node(uint32_t id) { load_value(row_addr(id)); }
    __device__ __forceinline__ void load_query(uint32_t, const uint8_t* row) { load_value(row); }

    __device__ __forceinline__ void issue(uint32_t slot, uint32_t id) {
        uint64_t* bar = &sm.full[slot];
        if constexpr (TABLE) {
            uint32_t t;
            const uint8_t* src = rows->row(id, g.row_bytes, t);
            if (t != rows->own) { // a peer's row: this thread fills the slot, then arrives (release) without a transaction
                const uint4* s = reinterpret_cast<const uint4*>(src);
                uint4* d = reinterpret_cast<uint4*>(sm.ring + (size_t)slot * g.row_bytes);
#pragma unroll 8
                for (uint32_t c = 0; c < nchunks; ++c)
                    d[c] = __ldg(s + c);
                mbar_arrive(bar);
                return;
            }
            mbar_arrive_expect_tx(bar, g.row_bytes);
            bulk_g2s(sm.ring + (size_t)slot * g.row_bytes, src, g.row_bytes, bar);
        } else {
            mbar_arrive_expect_tx(bar, g.row_bytes);
            bulk_g2s(sm.ring + (size_t)slot * g.row_bytes, g.vectors + (size_t)id * g.row_bytes, g.row_bytes, bar);
        }
    }

    __device__ __forceinline__ float row_distance(const uint4* row) const { return lb200::row_distance<DM, SK, NQ>(qreg, row, nchunks, a2, lane); }

    // distances value -> cand_id[0..n) into cand_d[0..n).  Callers bracket it with __syncthreads().
    __device__ __forceinline__ void eval(uint32_t n) {
        const uint32_t T = n > (uint32_t)warp ? (n - warp + NW - 1) / NW : 0;
        if ((uint32_t)lane < min(T, SPW))
            issue(warp + NW * lane, sm.cand_id[warp + NW * lane]);
        uint32_t si = 0;
        for (uint32_t t = 0; t < T; ++t) {
            const uint32_t slot = warp + NW * si;
            mbar_wait(&sm.full[slot], (phase_bits >> si) & 1u);
            phase_bits ^= 1u << si;
            const float d = row_distance(reinterpret_cast<const uint4*>(sm.ring + (size_t)slot * g.row_bytes));
            if (lane == 0)
                sm.cand_d[warp + NW * t] = d;
            __syncwarp();
            if (t + SPW < T && lane == 0) {
                fence_proxy_async(); // our generic-proxy reads of the slot precede the async refill
                issue(slot, sm.cand_id[warp + NW * (t + SPW)]);
            }
            si = (si + 1 == SPW) ? 0 : si + 1;
        }
    }
};

// Screened walkers: after cand_d[0..n) holds every candidate's lower bound, warp 0 keeps, in stored order, the candidates with
// !(lb >= radius); returns their number (uniform across the CTA)
__device__ __forceinline__ uint32_t screen_compact(WalkSmem& sm, uint32_t n, float radius, int warp, int lane) {
    __syncthreads();
    if (warp == 0) {
        uint32_t m = 0;
        for (uint32_t base = 0; base < n; base += 32) {
            const uint32_t j = base + lane;
            const bool keep = j < n && !(sm.cand_d[j] >= radius);
            const uint32_t id = j < n ? sm.cand_id[j] : 0u;
            const uint32_t mk = __ballot_sync(0xffffffffu, keep);
            __syncwarp();
            if (keep)
                sm.cand_id[m + __popc(mk & ((1u << lane) - 1u))] = id;
            m += __popc(mk);
        }
        if (lane == 0)
            sm.ctrl->m = m, sm.ctrl->screened += n, sm.ctrl->rejected += n - m;
    }
    __syncthreads();
    return sm.ctrl->m;
}

// ---- f32 rows with the int8 screen (screen.cuh, DESIGN.md 4.1): the search kernel's evaluator for l2sq / cos -------------
// screen(n, radius) runs between the compaction of a round's unseen candidates and eval(): every warp fetches the code rows
// of its candidates (j % NW == warp) into its own ring slots with bulk copies, all issued before the first wait, computes
// their bounds, and warp 0 keeps, in stored order, the candidates with !(lb >= radius).  Only those are measured; a rejected
// one has d >= lb >= radius and the replay would have rejected it too, so the walk is unchanged.  eval() itself is untouched.
template <int DM, int NQ> struct ScreenEval : RowEval<DM, SK_F32, NQ> {
    using Base = RowEval<DM, SK_F32, NQ>;
    static constexpr bool kScreen = true;
    // search.cu: hnsw_search_screen_kernel's launch bounds = the CTAs/SM the plain kernel reaches with its own register count
    static constexpr int kMinCtas = NQ <= 6 ? 8 : NQ <= 8 ? 7 : NQ <= 12 ? 5 : 4;

    __device__ __forceinline__ explicit ScreenEval(const GraphView& gv) : Base(gv) {}
    __device__ __forceinline__ void init(uint8_t* smem_raw, const WalkLayout& lay, uint32_t ring_slots, const SearchScratch& s) {
        Base::init(smem_raw, lay, ring_slots, s);
        if (threadIdx.x == 0)
            this->sm.ctrl->screened = this->sm.ctrl->rejected = 0; // read back after the CTA's last barrier
    }

    // cand_id[0..n) -> its survivors, compacted in order; returns their number (uniform across the CTA)
    __device__ __forceinline__ uint32_t screen(uint32_t n, float radius) {
        const GraphView& g = this->g;
        WalkSmem& sm = this->sm;
        const int warp = this->warp, lane = this->lane;
        const uint32_t NW = this->NW, rb = g.row_bytes, cb = screen_code_bytes(rb);
        const uint32_t per_slot = rb / cb; // code rows per ring slot (>= 1; 4 at d = 768)
        const uint32_t cap = min(this->SPW * per_slot, 32u);
        const uint32_t T = n > (uint32_t)warp ? (n - warp + NW - 1) / NW : 0;
        for (uint32_t t0 = 0; t0 < T; t0 += cap) {
            const uint32_t cnt = min(cap, T - t0), nslots = (cnt + per_slot - 1) / per_slot;
            fence_proxy_async(); // our generic-proxy reads of these slots (previous pass or round) precede the async writes
            __syncwarp();
            float4 meta = make_float4(0.f, 0.f, 0.f, 0.f);
            if ((uint32_t)lane < nslots) {
                const uint32_t slot = warp + NW * lane, k = min(per_slot, cnt - lane * per_slot);
                uint64_t* bar = &sm.full[slot];
                mbar_arrive_expect_tx(bar, k * cb);
                for (uint32_t j = 0; j < k; ++j) {
                    const uint32_t id = sm.cand_id[warp + NW * (t0 + lane * per_slot + j)];
                    bulk_g2s(sm.ring + (size_t)slot * rb + j * cb, g.sq_codes + (size_t)id * cb, cb, bar);
                }
            }
            if ((uint32_t)lane < cnt)
                meta = __ldg(g.sq_meta + sm.cand_id[warp + NW * (t0 + lane)]);
            float mine = 0.f;
            for (uint32_t t = 0; t < cnt; ++t) {
                const uint32_t si = t / per_slot, j = t - si * per_slot, slot = warp + NW * si;
                if (j == 0) {
                    mbar_wait(&sm.full[slot], (this->phase_bits >> si) & 1u);
                    this->phase_bits ^= 1u << si;
                }
                const float scale = __shfl_sync(0xffffffffu, meta.x, t);
                const float s = screen_sum<DM, NQ>(this->qreg, reinterpret_cast<const uint32_t*>(sm.ring + (size_t)slot * rb + j * cb),
                                                   scale, this->nchunks, lane);
                if ((uint32_t)lane == t)
                    mine = s;
            }
            if ((uint32_t)lane < cnt)
                sm.cand_d[warp + NW * (t0 + lane)] = screen_bound<DM, NQ>(mine, meta, this->a2);
        }
        fence_proxy_async(); // the code reads precede eval's bulk copies into the same slots
        return screen_compact(sm, n, radius, warp, lane);
    }
};

// ---- f32 rows with the projected screen (screen.cuh, DESIGN.md 4.1): k int8 codes of P x per row ---------------------------
// Same place in the round and the same compaction as ScreenEval, but each lane takes one candidate of its warp (j % NW ==
// warp) and reads its whole record (64 or 128 bytes) with plain 16-byte loads: one round trip for up to 32 candidates, q~
// broadcast from shared memory, no shuffles and no ring slots.  eval() is untouched.
template <int DM, int NQ> struct PScreenEval : RowEval<DM, SK_F32, NQ> {
    using Base = RowEval<DM, SK_F32, NQ>;
    static constexpr bool kScreen = true;
    static constexpr int kMinCtas = ScreenEval<DM, NQ>::kMinCtas;
    // the ring, then the query's q~ and its header (ps_query_floats)
    static __host__ __device__ WalkLayout layout(const GraphView& g, uint32_t R, uint32_t top_cap, uint32_t cand_cap) {
        return walk_layout_bytes((size_t)R * g.row_bytes + (size_t)ps_query_floats(g.ps_k) * 4, R, top_cap, cand_cap);
    }
    float* psq; // shared: q~[ps_code_slots], then {delta, |q~|, G, |q|^2}

    __device__ __forceinline__ explicit PScreenEval(const GraphView& gv) : Base(gv) {}
    __device__ __forceinline__ void init(uint8_t* smem_raw, const WalkLayout& lay, uint32_t ring_slots, const SearchScratch& s) {
        Base::init(smem_raw, lay, ring_slots, s);
        psq = reinterpret_cast<float*>(smem_raw + (size_t)ring_slots * this->g.row_bytes);
        if (threadIdx.x == 0)
            this->sm.ctrl->screened = this->sm.ctrl->rejected = 0; // read back after the CTA's last barrier
    }
    // the query's registers, and its projection from the batch's pre-pass (launch_ps_queries)
    __device__ __forceinline__ void load_query(uint32_t qi, const uint8_t* row) {
        Base::load_value(row);
        const uint32_t nf = ps_query_floats(this->g.ps_k);
        __syncthreads(); // the previous query's screen is done with psq
        for (uint32_t i = threadIdx.x; i < nf; i += blockDim.x)
            psq[i] = __ldg(this->g.ps_query + (size_t)qi * nf + i);
        __syncthreads();
    }

    __device__ __forceinline__ uint32_t screen(uint32_t n, float radius) {
        const GraphView& g = this->g;
        WalkSmem& sm = this->sm;
        const int warp = this->warp, lane = this->lane;
        const uint32_t NW = this->NW, slots = ps_code_slots(g.ps_k), rec = ps_record_bytes(g.ps_k) / 16;
        const uint32_t T = n > (uint32_t)warp ? (n - warp + NW - 1) / NW : 0;
        const float4 qh = *reinterpret_cast<const float4*>(psq + slots);
        for (uint32_t t = lane; t < T; t += 32) {
            const uint32_t j = warp + NW * t;
            const uint4* r = g.ps_records + (size_t)sm.cand_id[j] * rec;
            float sf = 0.f, cc = 0.f;
            const uint4 v0 = __ldg(r), v1 = __ldg(r + 1), v2 = __ldg(r + 2), v3 = __ldg(r + 3);
            ps_accum(psq, v1, sf, cc);
            ps_accum(psq + 16, v2, sf, cc);
            ps_accum(psq + 32, v3, sf, cc);
            if (rec == 8) { // k > 48: the record's second half
                const uint4 v4 = __ldg(r + 4), v5 = __ldg(r + 5), v6 = __ldg(r + 6), v7 = __ldg(r + 7);
                ps_accum(psq + 48, v4, sf, cc);
                ps_accum(psq + 64, v5, sf, cc);
                ps_accum(psq + 80, v6, sf, cc);
                ps_accum(psq + 96, v7, sf, cc);
            }
            const float4 meta = make_float4(__uint_as_float(v0.x), __uint_as_float(v0.y), __uint_as_float(v0.z), __uint_as_float(v0.w));
            sm.cand_d[j] = pscreen_bound<DM, NQ>(sf, cc, meta, qh, this->a2, slots);
        }
        return screen_compact(sm, n, radius, warp, lane);
    }
};

// ---- evaluator for PQ-coded rows: asymmetric distance through a per-value look-up table ----------------------
// Reference semantics (lantern_storage.hpp:137-149,264-267; index_dense.hpp:341-358): every stored operand is
// decompressed (concatenation of centroid slices), the query / new vector never is.  Because a decoded vector is a
// concatenation of centroid slices, d(value, decode(code)) = sum_s lut[s][code_s] with
//   l2sq: lut[s][c] = |value_s - centroid_{c,s}|^2          cos: lut[s][c] = value_s . centroid_{c,s}  (+ norm tables)
// which reproduces the reference up to fp32 summation order (verified 2e-7 relative, SURVEY App. A.10).  When the value
// is itself a stored node (refine_, reverse links) its table rows are copied from the centroid-pair table `pq_pair`
// [nsub][ncent][ncent] precomputed at index creation.  Code rows (nsub bytes) are read straight from HBM/L2.
template <int DM> struct PqEval : WalkBase {
    static __host__ __device__ WalkLayout layout(const GraphView& g, uint32_t, uint32_t top_cap, uint32_t cand_cap) {
        return walk_layout_pq(g.num_subvectors, g.pq_lut_width, pq_value_floats(g), top_cap, cand_cap);
    }
    float* lut;  // shared [nsub][ncent] (+ 4)
    float* qbuf; // shared [dims]
    float* part; // shared [warps][2][64]: per-chunk partial sums of the candidates a warp is measuring
    float a2;
    uint32_t tphase;

    __device__ __forceinline__ explicit PqEval(const GraphView& gv) : WalkBase(gv) {}
    __device__ __forceinline__ void init(uint8_t* smem_raw, const WalkLayout& lay, uint32_t, const SearchScratch& s) {
        init_base(smem_raw, lay, s);
        lut = reinterpret_cast<float*>(smem_raw);
        qbuf = lut + pq_table_floats(g.num_subvectors, g.pq_lut_width);
        part = qbuf + pq_value_floats(g);
        a2 = 0.f;
        tphase = 0;
        if (threadIdx.x == 0) {
            mbar_init(&sm.full[0], 1);
            fence_mbar_init();
        }
        __syncthreads();
    }

    // one table entry: |v_s - c|^2 (l2sq) or v_s . c (cos), dimensions in ascending order (the order pq_query_tables_kernel uses)
    __device__ __forceinline__ static float entry(const float* qs, const float* cen, uint32_t sd) {
        float acc = 0.f;
        if ((sd & 3u) == 0u) {
            for (uint32_t i = 0; i < sd; i += 4) {
                const float4 c4 = __ldg(reinterpret_cast<const float4*>(cen + i));
                if constexpr (DM == DM_COS) {
                    acc = fmaf(qs[i], c4.x, acc), acc = fmaf(qs[i + 1], c4.y, acc);
                    acc = fmaf(qs[i + 2], c4.z, acc), acc = fmaf(qs[i + 3], c4.w, acc);
                } else {
                    float d = qs[i] - c4.x;
                    acc = fmaf(d, d, acc);
                    d = qs[i + 1] - c4.y, acc = fmaf(d, d, acc);
                    d = qs[i + 2] - c4.z, acc = fmaf(d, d, acc);
                    d = qs[i + 3] - c4.w, acc = fmaf(d, d, acc);
                }
            }
        } else {
            for (uint32_t i = 0; i < sd; ++i) {
                const float cv = __ldg(cen + i);
                if constexpr (DM == DM_COS)
                    acc = fmaf(qs[i], cv, acc);
                else {
                    const float d = qs[i] - cv;
                    acc = fmaf(d, d, acc);
                }
            }
        }
        return acc;
    }

    // `row` = raw f32 vector (dims floats) in global memory
    __device__ __forceinline__ void load_value(const uint8_t* row) {
        const float* q = reinterpret_cast<const float*>(row);
        const uint32_t dims = g.dims, ncent = g.pq_lut_width, nsub = g.num_subvectors, sd = dims / nsub;
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < dims; i += kWalkThreads)
            qbuf[i] = __ldg(q + i);
        __syncthreads();
        if constexpr (DM == DM_COS) {
            float p2 = 0.f;
            for (uint32_t i = lane; i < dims; i += 32)
                p2 += qbuf[i] * qbuf[i];
            a2 = warp_sum(p2);
        }
        for (uint32_t e = threadIdx.x; e < nsub * ncent; e += kWalkThreads) {
            const uint32_t s = e / ncent, c = e - s * ncent;
            lut[e] = entry(qbuf + (size_t)s * sd, g.codebook + (size_t)c * dims + (size_t)s * sd, sd);
        }
        __syncthreads();
    }

    // search: query `qi` of the batch.  When the batch's tables were precomputed (pq_query_tables_kernel, one dense launch at
    // full occupancy instead of nsub*ncent*subdim flops per query inside this 4-CTA/SM kernel) the table is one bulk copy away.
    __device__ __forceinline__ void load_query(uint32_t qi, const uint8_t* row) {
        if (!g.pq_query_tables) {
            load_value(row);
            return;
        }
        const uint32_t floats = (uint32_t)pq_table_floats(g.num_subvectors, g.pq_lut_width);
        __syncthreads(); // every look-up of the previous query is done
        if (threadIdx.x == 0) {
            fence_proxy_async();
            mbar_arrive_expect_tx(&sm.full[0], floats * 4);
            bulk_g2s(lut, g.pq_query_tables + (size_t)qi * floats, floats * 4, &sm.full[0]);
        }
        mbar_wait(&sm.full[0], tphase);
        tphase ^= 1u;
        a2 = lut[(size_t)g.num_subvectors * g.pq_lut_width]; // |query|^2 (cos)
    }

    __device__ __forceinline__ void load_node(uint32_t id) {
        const uint32_t ncent = g.pq_lut_width, full = g.num_centroids, nsub = g.num_subvectors;
        const uint8_t* codes = g.vectors + (size_t)id * g.row_bytes;
        __syncthreads();
        for (uint32_t e = threadIdx.x; e < nsub * ncent; e += kWalkThreads) {
            const uint32_t s = e / ncent, c = e - s * ncent;
            lut[e] = __ldg(g.pq_pair + ((size_t)s * full + __ldg(codes + s)) * full + c);
        }
        if constexpr (DM == DM_COS) {
            float p2 = 0.f;
            for (uint32_t s = lane; s < nsub; s += 32)
                p2 += __ldg(g.pq_norm + (size_t)s * full + __ldg(codes + s));
            a2 = warp_sum(p2);
        }
        __syncthreads();
    }

    // 16 codes of one chunk -> partial sums
    __device__ __forceinline__ void chunk_sums(const uint4& v, uint32_t ch, float& acc, float& b2) const {
        const uint32_t ncent = g.pq_lut_width, full = g.num_centroids, nsub = g.num_subvectors;
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        acc = 0.f, b2 = 0.f;
#pragma unroll
        for (int wi = 0; wi < 4; ++wi)
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                const uint32_t s = ch * 16 + wi * 4 + b;
                if (s < nsub) {
                    const uint32_t c = (w[wi] >> (8 * b)) & 255u;
                    acc += lut[s * ncent + c];
                    if constexpr (DM == DM_COS)
                        b2 += __ldg(g.pq_norm + (size_t)s * full + c);
                }
            }
    }

    // distances value -> cand_id[0..n).  Candidate j belongs to warp j % 4.  A warp fetches the code rows of ALL its candidates of
    // a pass at once (16-byte chunks, two per lane, every load issued before the first look-up -- one HBM latency per round
    // instead of one per candidate), each lane sums the 16 look-ups of its chunks, and the chunk sums of a candidate are added
    // in ascending chunk order (a fixed order: the distance does not depend on which lane or pass served the candidate).
    __device__ __forceinline__ void eval(uint32_t n) {
        const uint32_t cpr = g.row_bytes / 16; // chunks per code row (6 at 96 subvectors)
        const uint32_t T = n > (uint32_t)warp ? (n - warp + kWalkWarps - 1) / kWalkWarps : 0;
        float* pa = part + (size_t)warp * 2 * kPqPartPerWarp;
        float* pb = pa + kPqPartPerWarp;
        if (cpr <= kPqPartPerWarp) {
            const uint32_t per_pass = kPqPartPerWarp / cpr; // whole candidates per pass
            for (uint32_t t0 = 0; t0 < T; t0 += per_pass) {
                const uint32_t cnt = min(per_pass, T - t0), chunks = cnt * cpr;
                uint4 v[2];
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const uint32_t idx = lane + 32 * u;
                    if (idx < chunks) {
                        const uint32_t t = idx / cpr, ch = idx - t * cpr;
                        const uint32_t id = sm.cand_id[warp + kWalkWarps * (t0 + t)];
                        v[u] = __ldg(reinterpret_cast<const uint4*>(g.vectors + (size_t)id * g.row_bytes) + ch);
                    }
                }
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const uint32_t idx = lane + 32 * u;
                    if (idx < chunks) {
                        const uint32_t t = idx / cpr, ch = idx - t * cpr;
                        float acc, b2;
                        chunk_sums(v[u], ch, acc, b2);
                        pa[idx] = acc;
                        if constexpr (DM == DM_COS)
                            pb[idx] = b2;
                    }
                }
                __syncwarp();
                if ((uint32_t)lane < cnt) {
                    float acc = 0.f, b2 = 0.f;
                    for (uint32_t ch = 0; ch < cpr; ++ch) {
                        acc += pa[lane * cpr + ch];
                        if constexpr (DM == DM_COS)
                            b2 += pb[lane * cpr + ch];
                    }
                    float d = acc;
                    if constexpr (DM == DM_COS)
                        d = cos_from_parts(acc, a2, b2);
                    sm.cand_d[warp + kWalkWarps * (t0 + lane)] = d;
                }
                __syncwarp();
            }
        } else { // very wide code rows (> 1024 subvectors): one candidate at a time, chunks strided over the lanes
            for (uint32_t t = 0; t < T; ++t) {
                const uint32_t id = sm.cand_id[warp + kWalkWarps * t];
                float acc = 0.f, b2 = 0.f;
                for (uint32_t ch = lane; ch < cpr; ch += 32) {
                    float a1, b1;
                    chunk_sums(__ldg(reinterpret_cast<const uint4*>(g.vectors + (size_t)id * g.row_bytes) + ch), ch, a1, b1);
                    acc += a1, b2 += b1;
                }
                acc = warp_sum(acc);
                float d = acc;
                if constexpr (DM == DM_COS) {
                    b2 = warp_sum(b2);
                    d = cos_from_parts(acc, a2, b2);
                }
                if (lane == 0)
                    sm.cand_d[warp + kWalkWarps * t] = d;
            }
        }
    }
};

template <class E> struct WalkerT : E {
    __device__ __forceinline__ explicit WalkerT(const GraphView& gv) : E(gv) {}
    using E::eval;
    using E::g;
    using E::lane;
    using E::load_node;
    using E::sm;
    using E::st_dist;
    using E::st_hops;
    using E::st_pops;
    using E::st_limbo_drop;
    using E::touched;
    using E::touched_cap;
    using E::vis;
    using E::warp;
    using E::words_per_cta;

    __device__ __forceinline__ const uint32_t* list_of(uint32_t node, int level, uint32_t& width) const {
        if (level == 0) {
            width = g.M0;
            return g.adj0 + (size_t)node * g.M0;
        }
        width = g.M;
        return g.upper_adj + ((size_t)__ldg(g.upper_ref + node) + (level - 1)) * g.M;
    }

    // distance value -> one node (entry point)
    __device__ __forceinline__ float measure_one(uint32_t id) {
        __syncthreads();
        if (threadIdx.x == 0)
            sm.cand_id[0] = id;
        __syncthreads();
        eval(1);
        __syncthreads();
        st_dist += 1;
        return sm.cand_d[0];
    }

    // search_for_one_: levels from_level, from_level-1, ..., stop_level+1
    __device__ __forceinline__ void greedy(uint32_t& cur, float& cur_d, int from_level, int stop_level) {
        for (int level = from_level; level > stop_level; --level) {
            for (;;) {
                __syncthreads(); // everyone is done with cand_* of the previous pass
                if (warp == 0) {
                    uint32_t width;
                    const uint32_t* list = list_of(cur, level, width);
                    uint32_t n = 0;
                    for (uint32_t off = 0; off < width; off += 32) {
                        uint32_t id = (off + lane < width) ? __ldg(list + off + lane) : kNoNeighbor;
                        bool valid = id != kNoNeighbor;
                        uint32_t m = __ballot_sync(0xffffffffu, valid);
                        if (valid)
                            sm.cand_id[n + __popc(m & ((1u << lane) - 1u))] = id;
                        n += __popc(m);
                    }
                    if (lane == 0)
                        sm.ctrl->n = n;
                }
                __syncthreads();
                const uint32_t n_all = sm.ctrl->n;
                uint32_t n = n_all; // candidates measured
                // Screened search walkers: a candidate with lb >= cur_d has d >= cur_d, which the strict '<' below never
                // takes, and the screen keeps stored order, so the first minimum below cur_d is the same node.  cur_d is
                // uniform across the CTA; a NaN cur_d (no candidate can be taken) skips the screen, as the beam's radius does.
                if constexpr (E::kScreen)
                    if (cur_d == cur_d)
                        n = this->screen(n_all, cur_d);
                eval(n);
                __syncthreads();
                // one pass of index.hpp:3304-3311: chain of strict improvements == first minimum below cur_d
                float best = cur_d;
                int bi = -1;
                for (uint32_t j = 0; j < n; ++j) {
                    float d = sm.cand_d[j];
                    if (d < best)
                        best = d, bi = (int)j;
                }
                st_dist += n_all, st_hops += 1; // the screen's rejects count as computed distances: the reference computes them
                if (bi < 0)
                    break;
                cur = sm.cand_id[bi], cur_d = best;
            }
        }
    }

    // Beam search on one level with top list capacity L, starting from `start` (distance start_d already known:
    // the reference re-measures it, so the counter advances).  `skip` = node whose expansion is skipped
    // (index.hpp:3357 new_slot; kNoNeighbor for plain search).  Leaves the ascending top list in shared memory;
    // returns its size (uniform across the CTA).  Visited bits are cleared before returning.
    // (A register-resident top list for L <= 64 needs 72 registers/thread, which costs one resident CTA per SM -- the list
    //  stays in shared memory.)
    // `expand` = candidates expanded per round: 1 reproduces the reference's order exactly; p > 1 ("relaxed order") expands
    // the p closest unexpanded candidates together -- fewer serial rounds, a few per cent more distance evaluations, same
    // result at ef >= N, recall within the +-0.5 % window at finite ef.
    __device__ __forceinline__ uint32_t beam(int level, uint32_t start, float start_d, uint32_t L, uint32_t skip, uint32_t expand = 1) {
        return beam_impl<TopSmem>(level, start, start_d, L, skip, expand);
    }

    template <class Top>
    __device__ __forceinline__ uint32_t beam_impl(int level, uint32_t start, float start_d, uint32_t L, uint32_t skip, uint32_t expand) {
        uint32_t ntouched = 0; // warp-0 uniform
        Top top;
        // Distance ties at the eviction boundary: the reference's queue keeps an element after `top` evicted it, and still
        // expands it while its distance EQUALS the radius (the stop test index.hpp:3445 is a strict '>').  Such elements
        // wait in `limbo`; they all share one distance (the radius at the time) and die as soon as the radius shrinks.
        uint32_t limbo_n = 0;
        float limbo_d = 0.f;
        __syncthreads();
        if (warp == 0) {
            top.init(sm, L, start_d, start, lane);
            if (lane == 0) {
                atomicOr(&vis[start >> 5], 1u << (start & 31));
                touched[0] = start >> 5;
            }
            ntouched = 1;
            st_dist += 1; // index.hpp:3436 / :3343
            __syncwarp();
        }
        for (;;) {
            __syncthreads(); // (A) insertions of the previous round are complete
            if (warp == 0) {
                uint32_t n = 0, popped = 0;
                while (popped < expand) {
                    uint32_t c = kNoNeighbor;
                    if (!top.pop(c, lane) && limbo_n)
                        c = sm.limbo[--limbo_n]; // distance == radius: not beyond it, so the reference expands it too
                    if (c == kNoNeighbor)
                        break;
                    ++popped;
                    if (c == skip)
                        continue;
                    uint32_t width;
                    const uint32_t* list = list_of(c, level, width);
                    bool halves = false; // screened search walkers only: builds and unscreened searches keep the loop below
                    if constexpr (E::kScreen)
                        halves = width == 64 && n == 0 && (g.flags & 8u);
                    if (halves) {
                        // both halves of a 64-wide list at once (flags bit 8): the two bitmap atomics of a lane are in flight
                        // together, one L2 round trip instead of two.  Only the FIRST occurrence of an id in stored order may
                        // count as unseen, so the second half is also checked against the first (through cand_id, free here:
                        // n == 0).  The same selection and order as the loop below (group.cu's owner does the same).
                        const uint32_t id0 = __ldg(list + lane), id1 = __ldg(list + 32 + lane);
                        const bool v0 = id0 != kNoNeighbor, v1 = id1 != kNoNeighbor;
                        sm.cand_id[lane] = id0;
                        __syncwarp();
                        const uint32_t p0 = __match_any_sync(0xffffffffu, id0), p1 = __match_any_sync(0xffffffffu, id1);
                        const bool first0 = v0 && ((uint32_t)(__ffs(p0) - 1) == (uint32_t)lane);
                        bool first1 = v1 && ((uint32_t)(__ffs(p1) - 1) == (uint32_t)lane);
                        if (first1)
                            for (int t = 0; t < 32; ++t)
                                first1 &= sm.cand_id[t] != id1;
                        __syncwarp();
                        const uint32_t bit0 = 1u << (id0 & 31), bit1 = 1u << (id1 & 31);
                        uint32_t old0 = 0, old1 = 0;
                        if (first0)
                            old0 = atomicOr(&vis[id0 >> 5], bit0);
                        if (first1)
                            old1 = atomicOr(&vis[id1 >> 5], bit1);
                        const bool fresh0 = first0 && !(old0 & bit0), fresh1 = first1 && !(old1 & bit1);
                        const uint32_t m0 = __ballot_sync(0xffffffffu, fresh0), m1 = __ballot_sync(0xffffffffu, fresh1);
                        const uint32_t lt = (1u << lane) - 1u, n0 = __popc(m0);
                        if (fresh0) {
                            const uint32_t r = __popc(m0 & lt);
                            sm.cand_id[r] = id0;
                            if (ntouched + r < touched_cap)
                                touched[ntouched + r] = id0 >> 5;
                            if (level == 0 && (g.flags & 1u))
                                prefetch_l2(g.adj0 + (size_t)id0 * g.M0);
                        }
                        __syncwarp(); // the compaction above overwrites entries another lane compared against
                        if (fresh1) {
                            const uint32_t r = n0 + __popc(m1 & lt);
                            sm.cand_id[r] = id1;
                            if (ntouched + r < touched_cap)
                                touched[ntouched + r] = id1 >> 5;
                            if (level == 0 && (g.flags & 1u))
                                prefetch_l2(g.adj0 + (size_t)id1 * g.M0);
                        }
                        n = n0 + __popc(m1);
                        ntouched += n;
                        st_pops += 1;
                        continue;
                    }
                    for (uint32_t off = 0; off < width; off += 32) {
                        uint32_t id = (off + lane < width) ? __ldg(list + off + lane) : kNoNeighbor;
                        bool valid = id != kNoNeighbor;
                        if (!__any_sync(0xffffffffu, valid))
                            break;
                        // duplicate ids inside one list are legal in reference graphs (refine_ padding,
                        // index.hpp:3554-3558): only the first occurrence can be "unseen"
                        uint32_t peers = __match_any_sync(0xffffffffu, id);
                        bool first = valid && ((uint32_t)(__ffs(peers) - 1) == (uint32_t)lane);
                        bool fresh = false;
                        if (first) {
                            uint32_t bit = 1u << (id & 31);
                            fresh = !(atomicOr(&vis[id >> 5], bit) & bit);
                        }
                        uint32_t m = __ballot_sync(0xffffffffu, fresh);
                        uint32_t rank = __popc(m & ((1u << lane) - 1u));
                        if (fresh) {
                            sm.cand_id[n + rank] = id;
                            if (ntouched + rank < touched_cap)
                                touched[ntouched + rank] = id >> 5;
                            if (level == 0 && (g.flags & 1u))
                                prefetch_l2(g.adj0 + (size_t)id * g.M0); // its adjacency line, for when it is popped
                        }
                        n += __popc(m);
                        ntouched += __popc(m);
                    }
                    st_pops += 1;
                }
                if (lane == 0) {
                    sm.ctrl->n = popped ? n : kDone;
                    if constexpr (E::kScreen) // the radius only shrinks within a round: screening against its start is safe
                        sm.ctrl->radius = (level == 0 && top.size == L) ? top.radius(lane) : __int_as_float(0x7fffffff);
                }
            }
            __syncthreads(); // (B)
            const uint32_t n_all = sm.ctrl->n;
            if (n_all == kDone)
                break;
            uint32_t n = n_all; // candidates measured (and replayed) this round
            if constexpr (E::kScreen) {
                const float r = sm.ctrl->radius;
                if (r == r)
                    n = this->screen(n_all, r);
            }
            eval(n);
            __syncthreads(); // (C)
            if (warp == 0) {
                st_dist += n_all; // the screen's rejects count as computed distances: the reference computes them
                // index.hpp:3470 / :3382: accepted iff top.size() < top_limit || successor_dist < radius.  The radius only
                // shrinks once the list is full, so a candidate that fails against the CURRENT radius can never pass
                // later in this round: filter those out in parallel, then replay the survivors in stored order.
                for (uint32_t base = 0; base < n; base += 32) {
                    const uint32_t j = base + lane;
                    const float dj = j < n ? sm.cand_d[j] : INFINITY;
                    float radius = top.radius(lane);
                    uint32_t m = __ballot_sync(0xffffffffu, j < n && (top.size < L || dj < radius));
                    while (m) {
                        const int b = __ffs(m) - 1;
                        m &= m - 1;
                        const float d = __shfl_sync(0xffffffffu, dj, b);
                        if (top.size < L || d < radius) {
                            const uint32_t id = sm.cand_id[base + b];
                            float ev_d;
                            uint32_t ev_i;
                            top.insert(d, id, lane, ev_d, ev_i);
                            if (level == 0 && (g.flags & 2u) && lane == 0)
                                prefetch_l2(g.adj0 + (size_t)id * g.M0);
                            radius = top.radius(lane);
                            if (limbo_n && radius < limbo_d)
                                limbo_n = 0; // the radius shrank below the waiting ties: they can never be expanded
                            if (ev_i != kNoNeighbor && !(ev_i & kExpandedBit) && ev_d == radius) {
                                if (limbo_n < kLimboCap) {
                                    if (lane == 0)
                                        sm.limbo[limbo_n] = ev_i;
                                    limbo_n++, limbo_d = radius;
                                    __syncwarp();
                                } else {
                                    this->st_limbo_drop += 1; // counted and reported (lb200_search_stats_t::limbo_overflows)
                                }
                            }
                        }
                    }
                }
            }
        }
        if (warp == 0) {
            top.flush(lane);
            if (lane == 0)
                sm.ctrl->ntouched = ntouched, sm.ctrl->top_size = top.size;
        }
        __syncthreads();
        { // un-visit only the words this walk touched
            const uint32_t nt = sm.ctrl->ntouched;
            if (nt <= touched_cap) {
                for (uint32_t i = threadIdx.x; i < nt; i += blockDim.x)
                    vis[touched[i]] = 0u;
            } else {
                for (size_t i = threadIdx.x; i < words_per_cta; i += blockDim.x)
                    vis[i] = 0u;
            }
        }
        const uint32_t out = sm.ctrl->top_size;
        __syncthreads(); // bitmap is clean and ctrl may be reused
        return out;
    }

    // refine_ (index.hpp:3515-3561) on the ascending list top_d/top_i[0..count): keeps the closest element, then
    // accepts a candidate only if it is not closer to an accepted element than to the centre; because
    // skip_pruned_connections == false (index.hpp:1245) the accepted prefix is followed by whatever sits at
    // positions [accepted, needed) -- stale entries, possibly duplicates.  Destroys the value registers.
    // Returns the size of the resulting view (uniform across the CTA).
    __device__ __forceinline__ uint32_t refine(uint32_t count, uint32_t needed) {
        if (count < needed)
            return count;
        uint32_t submitted = 1, consumed = 1;
        while (submitted < needed && consumed < count) {
            __syncthreads();
            const uint32_t c_id = sm.top_i[consumed] & kIdMask;
            const float c_d = sm.top_d[consumed];
            load_node(c_id);
            for (uint32_t j = threadIdx.x; j < submitted; j += blockDim.x)
                sm.cand_id[j] = sm.top_i[j] & kIdMask;
            __syncthreads();
            eval(submitted);
            __syncthreads();
            bool good = true;
            for (uint32_t j = 0; j < submitted; ++j)
                if (sm.cand_d[j] < c_d) { // index.hpp:3536
                    good = false;
                    break;
                }
            st_dist += submitted;
            if (good) {
                if (threadIdx.x == 0)
                    sm.top_d[submitted] = c_d, sm.top_i[submitted] = sm.top_i[consumed];
                submitted++;
            }
            consumed++;
        }
        __syncthreads();
        return needed; // count >= needed, so shrink(max(submitted, needed)) == needed
    }
};

template <int DM, int SK, int NQ> using Walker = WalkerT<RowEval<DM, SK, NQ>>;
template <int DM> using PqWalker = WalkerT<PqEval<DM>>;
template <int DM, int NQ> using ScreenWalker = WalkerT<ScreenEval<DM, NQ>>;
template <int DM, int NQ> using PScreenWalker = WalkerT<PScreenEval<DM, NQ>>;
// the row-sharded build kernels' walker: plain-row walkers read through a RowTable; PQ walkers have none (a group index
// cannot hold PQ codes)
template <class W> struct RowTableWalker {
    using type = W;
};
template <int DM, int SK, int NQ> struct RowTableWalker<WalkerT<RowEval<DM, SK, NQ>>> {
    using type = WalkerT<RowEval<DM, SK, NQ, true>>;
};

// ---- (DM, SK, NQ) dispatch shared by the launchers ----------------------------------------------------
// PQ indexes: fn(walker type tag) with PqWalker<DM>
template <typename T> struct TypeTag {
    using type = T;
};
template <typename Fn> void dispatch_walker(bool pq, int dm, int sk, int nq, Fn&& fn);

template <typename Fn> void dispatch_walk(int dm, int sk, int nq, Fn&& fn) {
#define LB_NQ_CASES(DMv, SKv)                                                                                          \
    switch (nq) {                                                                                                      \
    case 1: fn(std::integral_constant<int, DMv>{}, std::integral_constant<int, SKv>{}, std::integral_constant<int, 1>{}); return;   \
    case 2: fn(std::integral_constant<int, DMv>{}, std::integral_constant<int, SKv>{}, std::integral_constant<int, 2>{}); return;   \
    case 3: fn(std::integral_constant<int, DMv>{}, std::integral_constant<int, SKv>{}, std::integral_constant<int, 3>{}); return;   \
    case 4: fn(std::integral_constant<int, DMv>{}, std::integral_constant<int, SKv>{}, std::integral_constant<int, 4>{}); return;   \
    case 6: fn(std::integral_constant<int, DMv>{}, std::integral_constant<int, SKv>{}, std::integral_constant<int, 6>{}); return;   \
    case 8: fn(std::integral_constant<int, DMv>{}, std::integral_constant<int, SKv>{}, std::integral_constant<int, 8>{}); return;   \
    case 12: fn(std::integral_constant<int, DMv>{}, std::integral_constant<int, SKv>{}, std::integral_constant<int, 12>{}); return; \
    case 16: fn(std::integral_constant<int, DMv>{}, std::integral_constant<int, SKv>{}, std::integral_constant<int, 16>{}); return; \
    default: break;                                                                                                    \
    }
    if (dm == DM_L2SQ && sk == SK_F32) {
        LB_NQ_CASES(DM_L2SQ, SK_F32)
    } else if (dm == DM_COS && sk == SK_F32) {
        LB_NQ_CASES(DM_COS, SK_F32)
    } else if (dm == DM_L2SQ && sk == SK_F16) {
        LB_NQ_CASES(DM_L2SQ, SK_F16)
    } else if (dm == DM_COS && sk == SK_F16) {
        LB_NQ_CASES(DM_COS, SK_F16)
    } else if (dm == DM_L2SQ && sk == SK_I8) {
        LB_NQ_CASES(DM_L2SQ, SK_I8)
    } else if (dm == DM_COS && sk == SK_I8) {
        LB_NQ_CASES(DM_COS, SK_I8)
    } else if (dm == DM_HAMMING && sk == SK_B1) {
        LB_NQ_CASES(DM_HAMMING, SK_B1)
    }
#undef LB_NQ_CASES
    throw CudaError("unsupported metric / scalar kind / dimensionality combination");
}

template <typename Fn> void dispatch_walker(bool pq, int dm, int sk, int nq, Fn&& fn) {
    if (pq) {
        if (dm == DM_L2SQ)
            return fn(TypeTag<PqWalker<DM_L2SQ>>{});
        if (dm == DM_COS)
            return fn(TypeTag<PqWalker<DM_COS>>{});
        throw CudaError("pq index: only l2sq and cos metrics are supported");
    }
    dispatch_walk(dm, sk, nq, [&](auto d, auto s, auto n) {
        fn(TypeTag<Walker<decltype(d)::value, decltype(s)::value, decltype(n)::value>>{});
    });
}

} // namespace lb200

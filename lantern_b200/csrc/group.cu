// lantern_b200 -- one HNSW graph searched by G GPUs at once ("row-sharded group").
//
// The multi-GPU form of the hot path (index_gt::search -> search_for_one_ -> search_to_find_in_base_,
// U/include/usearch/index.hpp:2680-2730, 3277-3316, 3400-3485).  SURVEY.md 8(e) shards the corpus by contiguous
// row range with one INDEPENDENT graph per GPU and broadcasts every query to every shard; HNSW's cost barely depends on
// N, so that multiplies the total work by G (measured in round 1: 2.7x at 8 GPUs, recall-matched).  Here the corpus is
// still sharded by row range -- GPU r holds the vectors of rows [bounds[r], bounds[r+1]) and nothing else of the 3 KB/row
// payload -- but there is ONE graph: the adjacency lists (4 B per link, 8 % of the corpus at d=768/M=32) are replicated,
// every query is walked once, by one "owner" warp, in the reference's exact order, and each distance is evaluated on the
// GPU that owns the row.  Total row traffic is that of the 1-GPU search, split G ways; the results are those of the 1-GPU
// search on the same graph, id for id (same decision sequence, same fp32 reduction order).
//
// Mapping to the machine.  Every GPU runs the same persistent kernel of independent warps (no CTA-wide barrier anywhere).
// The first O warps are OWNERS: each takes one of this GPU's queries (q mod G == rank) at a time, keeps the query in
// registers, the top list in shared memory, the visited bitmap in HBM, and makes the reference's decisions.  The other H
// warps are a HELPER POOL that measures local rows for remote owners: the (G-1)*O inbound mailboxes are dealt round-robin
// to the helpers, one lane watching one mailbox.  Per expansion the owner sends each rank the ids of the unseen neighbours
// that live there and receives their distances; messages are 8-byte words {payload, flag} written straight into the peer's
// HBM over NVLink (peer-mapped memory; NCCL's "LL" idea: the flag travels with the data, so no fence is needed and one
// NVLink write latency is the whole cost) and polled locally.  Rows are fetched through a per-warp bulk-copy ring
// (cp.async.bulk + mbarrier) behind an L2 prefetch of the rows to come.  The final top-k of a query is stored into every
// GPU's result buffer by its owner (the all-gather of SURVEY 8e, fused into the search epilogue); a last-warp-out flag
// exchange makes kernel completion imply that all peers' results have landed.  No NCCL, no host synchronisation on the hot
// path.  With G = 1 the same kernel is a one-warp-per-query single-GPU search (launch_warp_search).
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/lantern_b200.h"
#include "group.h"
#include "walk.cuh"

namespace lb200 {

size_t device_smem_optin(); // engine.cu: dynamic shared memory one CTA may opt in to

namespace {

constexpr int kGroupThreads = 128; // 4 independent warps per CTA (no CTA-wide synchronisation anywhere)
constexpr int kGroupWarps = kGroupThreads / 32;

__device__ __forceinline__ unsigned long long ld_sys_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_sys_u64(unsigned long long* p, unsigned long long v) {
    asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_sys_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_sys_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ unsigned long long pack_word(uint32_t payload, uint32_t flag) {
    return ((unsigned long long)flag << 32) | payload;
}
// 16 bytes of a row that nobody caches on our side (queries live in the root's memory: peer addresses bypass our L2 and
// a stale L1 line of the previous batch must not be served)
__device__ __forceinline__ uint4 ld_nocache_u4(const uint4* p) {
    uint4 v;
    asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}

struct GroupWarpLayout {
    uint32_t ring, bars, top_d, top_i, cand_id, cand_d, cand_slot, loc, limbo, psq, total;
};
// per warp: R row slots (the bulk-copy ring), R mbarriers, the top list, the candidate arrays, and for the projected screen
// the query's q~ and its header (psq_floats = ps_query_floats(k); 0 without the screen)
__host__ __device__ inline GroupWarpLayout group_warp_layout(uint32_t row_bytes, uint32_t R, uint32_t L, uint32_t cap,
                                                             uint32_t psq_floats = 0) {
    GroupWarpLayout l;
    uint32_t o = 0;
    l.ring = o, o += R * ((row_bytes + 15u) & ~15u);
    l.bars = o, o += 8 * R;
    l.top_d = o, o += 4 * L;
    l.top_i = o, o += 4 * L;
    l.cand_id = o, o += 4 * cap;
    l.cand_d = o, o += 4 * cap;
    l.cand_slot = o, o += (2 * cap + 3u) & ~3u;
    l.loc = o, o += (cap + 3u) & ~3u;
    l.limbo = o, o += 4 * kLimboCap;
    o = (o + 15u) & ~15u;
    l.psq = o, o += 4 * psq_floats;
    l.total = (o + 15u) & ~15u;
    return l;
}
// rows in flight per warp: 2 for 3 KB rows, more for narrow rows (about 6 KB of staging per warp)
inline uint32_t group_ring_slots(uint32_t row_bytes) {
    uint32_t r = 6144u / row_bytes;
    r = r < 2 ? 2 : (r > 8 ? 8 : r);
    if (const char* e = getenv("LB200_GROUP_RING_SLOTS")) // experiments: deeper rings cost resident warps
        if (atoi(e) >= 1 && atoi(e) <= 8)
            r = (uint32_t)atoi(e);
    return r;
}

// ---- one warp = one query slot -------------------------------------------------------------------------------------
// Header payload of the owner -> helper mailbox: count (bits 0-8, 1..256 ids follow) | query index << 9, or kMsgExit (the
// launch is over for this slot).  The query index travels with EVERY request -- the header is a single word that the next
// message overwrites, so a separate "start of query" message could be lost before the helper had seen it; the helper loads a
// query into shared memory when the index in a request differs from the one it holds.
constexpr uint32_t kMsgExit = 0xFFFFFFFFu;
constexpr uint32_t kMsgCountBits = 9;
constexpr size_t kGroupMaxBatch = (size_t)1 << (32 - kMsgCountBits - 1);

// PS: the level-0 rounds of the owner run the projected screen (screen.cuh) -- one rank only, f32 l2sq / cos
template <int DM, int SK, int NQ, bool PS = false> struct GroupWarp {
    const GroupLaunch& p;
    int lane;
    uint32_t slot, nchunks;
    uint8_t* ws; // this warp's shared memory
    uint4 qreg[NQ]; // the query, in registers (lane l holds chunks l, l+32, ...)
    uint32_t phase_bits; // parity of each ring slot's mbarrier
    float a2;
    uint32_t seq;   // owner: messages sent by this slot in this launch
    uint32_t last;  // helper: flag of the last header seen
    uint32_t cur_q; // the query this slot holds in shared memory (0xFFFFFFFF: none)
    bool dead, waited;
    unsigned long long t0;
    uint32_t st_dist, st_pops, st_hops, st_rounds, st_rows;
    // owner: SM cycles spent producing a round's ids, measuring the local rows, waiting for the helpers, consuming
    uint32_t cy_produce, cy_local, cy_wait, cy_consume; // (32 bits: 2 s of cycles per warp and launch)
    uint32_t cy_screen, st_screened, st_rejected;       // PS only

    __device__ __forceinline__ explicit GroupWarp(const GroupLaunch& gp) : p(gp) {}

    __device__ __forceinline__ uint32_t psq_floats() const { return PS ? ps_query_floats(p.g.ps_k) : 0u; }
    // shared-memory arrays are addressed from one base (fewer live registers than eight pointers)
    __device__ __forceinline__ GroupWarpLayout lay() const {
        return group_warp_layout(p.g.row_bytes, p.ring_slots, p.L, p.cap, psq_floats());
    }
    __device__ __forceinline__ uint8_t* ring() const { return ws; }
    __device__ __forceinline__ uint64_t* bars() const { return reinterpret_cast<uint64_t*>(ws + lay().bars); }
    __device__ __forceinline__ float* top_d() const { return reinterpret_cast<float*>(ws + lay().top_d); }
    __device__ __forceinline__ uint32_t* top_i() const { return reinterpret_cast<uint32_t*>(ws + lay().top_i); }
    __device__ __forceinline__ uint32_t* cand_id() const { return reinterpret_cast<uint32_t*>(ws + lay().cand_id); }
    __device__ __forceinline__ float* cand_d() const { return reinterpret_cast<float*>(ws + lay().cand_d); }
    __device__ __forceinline__ uint16_t* cand_slot() const { return reinterpret_cast<uint16_t*>(ws + lay().cand_slot); }
    __device__ __forceinline__ uint8_t* loc() const { return ws + lay().loc; }
    __device__ __forceinline__ uint32_t* limbo() const { return reinterpret_cast<uint32_t*>(ws + lay().limbo); }
    __device__ __forceinline__ float* psq() const { return reinterpret_cast<float*>(ws + lay().psq); }

    __device__ __noinline__ bool timed_out() {
        if (ld_sys_u32(p.err[p.me]) != 0u)
            return true;
        if (globaltimer_ns() - t0 > p.timeout_ns) {
            for (uint32_t r = 0; r < p.G; ++r)
                st_sys_u32(p.err[r], 1u + p.me);
            return true;
        }
        return false;
    }
    // spin until the word carries `flag`; returns its payload
    __device__ __forceinline__ uint32_t wait_word(const unsigned long long* addr, uint32_t flag) {
        uint32_t spins = 0;
        for (;;) {
            const unsigned long long v = ld_sys_u64(addr);
            if ((uint32_t)(v >> 32) == flag)
                return (uint32_t)v;
            if (dead)
                return 0u;
            if ((++spins & 2047u) == 0u && timed_out()) {
                dead = true;
                return 0u;
            }
        }
    }

    // non-root ranks read the queries from the root's staging buffer once the root's kernel has announced them
    __device__ __forceinline__ void wait_queries() {
        if (waited)
            return;
        if (lane == 0) {
            uint32_t spins = 0;
            while (ld_sys_u64(p.qready[p.me]) != (unsigned long long)p.epoch) {
                if ((++spins & 2047u) == 0u && timed_out()) {
                    dead = true;
                    break;
                }
                __nanosleep(64);
            }
        }
        dead = __any_sync(0xffffffffu, dead);
        waited = true;
    }

    __device__ __forceinline__ void load_query(uint32_t q) {
        wait_queries();
        const uint4* src = reinterpret_cast<const uint4*>(p.queries + (size_t)q * p.query_stride);
        float part = 0.f;
#pragma unroll
        for (int i = 0; i < NQ; ++i) {
            const uint32_t c = lane + 32 * i;
            qreg[i] = c < nchunks ? ld_nocache_u4(src + c) : make_uint4(0, 0, 0, 0);
            part = norm_add(part, query_norm_chunk<DM, SK>(qreg[i]));
        }
        a2 = 0.f;
        if constexpr (DM == DM_COS)
            a2 = warp_sum(part);
    }

    // ---- distances query -> a list of LOCAL rows, through this warp's bulk-copy ring (cp.async.bulk + mbarrier, as
    // RowEval in walk.cuh but private to the warp): ring_slots rows are in flight at once, a slot is refilled as soon as it
    // has been read.  OWNER: entry t of the list is candidate loc[t]; helper: entry t is cand_id[t].  Lane layout and
    // reduction order are RowEval::row_distance's, so every value is bit-identical to the 1-GPU kernel's.
    __device__ __forceinline__ void issue_row(uint32_t s, uint32_t id) {
        uint64_t* bar = bars() + s;
        mbar_arrive_expect_tx(bar, p.g.row_bytes);
        bulk_g2s(ring() + (size_t)s * p.g.row_bytes, p.g.vectors + (size_t)(id - p.bounds[p.me]) * p.g.row_bytes, p.g.row_bytes, bar);
    }
    template <bool OWNER> __device__ __forceinline__ void eval_local(uint32_t n) {
        const uint32_t R = p.ring_slots;
        const uint32_t* ids = cand_id();
        const uint8_t* lj = loc();
        // The ring keeps R rows in flight; the rows behind them are already on their way to L2 (one prefetch per 128-byte line,
        // kPrefetchRows rows ahead), so a slot's refill is an L2 hit instead of a DRAM round trip.  With G GPUs a warp's share of
        // an expansion is a handful of rows: all of them are requested from DRAM at once.
        // Only for SHORT lists (the latency-bound regime of 4+ GPUs): with 24-48 rows per list (1-2 GPUs) the kernel is
        // HBM-bound and 8 rows x 3 KB x 3500 warps of prefetch would not fit in L2 -- measured: 20.9 instead of 15.9 ms at G = 1.
        constexpr uint32_t kPrefetchRows = 8, kPrefetchMaxList = 16;
        const uint32_t pf_off = (uint32_t)lane * 128u;
        const bool pf_lane = pf_off < p.g.row_bytes && n <= kPrefetchMaxList;
        const uint8_t* base = p.g.vectors - (size_t)p.bounds[p.me] * p.g.row_bytes;
        for (uint32_t t = R; t < min(n, R + kPrefetchRows); ++t)
            if (pf_lane)
                prefetch_l2(base + (size_t)ids[OWNER ? lj[t] : t] * p.g.row_bytes + pf_off);
        if ((uint32_t)lane < min(n, R))
            issue_row(lane, ids[OWNER ? lj[lane] : lane]);
        uint32_t s = 0;
#pragma unroll 1
        for (uint32_t t = 0; t < n; ++t) {
            if (t + R + kPrefetchRows < n && pf_lane)
                prefetch_l2(base + (size_t)ids[OWNER ? lj[t + R + kPrefetchRows] : t + R + kPrefetchRows] * p.g.row_bytes + pf_off);
            mbar_wait(bars() + s, (phase_bits >> s) & 1u);
            phase_bits ^= 1u << s;
            const uint4* row = reinterpret_cast<const uint4*>(ring() + (size_t)s * p.g.row_bytes);
            DistAcc<DM, SK> acc;
            acc.reset();
#pragma unroll
            for (int i = 0; i < NQ; ++i) {
                const uint32_t c = lane + 32 * i;
                if (c < nchunks)
                    accum_chunk<DM, SK>(acc, qreg[i], row[c]);
            }
            const float d = finish_distance<DM, SK>(acc, a2);
            if (lane == 0)
                cand_d()[OWNER ? lj[t] : t] = d;
            __syncwarp();
            if (t + R < n && lane == 0) {
                fence_proxy_async(); // our generic-proxy reads of the slot precede the async refill
                issue_row(s, ids[OWNER ? lj[t + R] : t + R]);
            }
            s = (s + 1 == R) ? 0 : s + 1;
        }
        st_rows += n;
    }

    // ---- owner: distances query -> cand_id[0..n) into cand_d[0..n), each evaluated where the row lives -----------
    __device__ __forceinline__ void eval_round(uint32_t n) {
        const uint32_t G = p.G, me = p.me, cap = p.cap;
        const uint32_t flag = p.flag_base + (++seq);
        const uint32_t lt = (1u << lane) - 1u;
        uint32_t cnt = 0; // lane d < G: ids addressed to rank d in this round
#pragma unroll 1
        for (uint32_t base = 0; base < n; base += 32) {
            const uint32_t j = base + lane;
            const bool valid = j < n;
            const uint32_t id = valid ? cand_id()[j] : 0u;
            uint32_t dst = 0xFFu;
            if (valid) {
                dst = 0;
                while (id >= p.bounds[dst + 1])
                    ++dst;
            }
            uint32_t pos = 0;
#pragma unroll 1
            for (uint32_t d = 0; d < G; ++d) {
                const uint32_t m = __ballot_sync(0xffffffffu, dst == d);
                const uint32_t c_d = __shfl_sync(0xffffffffu, cnt, d);
                if (dst == d)
                    pos = c_d + __popc(m & lt);
                if ((uint32_t)lane == d)
                    cnt += __popc(m);
            }
            if (valid) {
                cand_slot()[j] = (uint16_t)((dst << 8) | pos);
                if (dst != me)
                    st_sys_u64(p.req[dst] + ((size_t)me * p.O + slot) * (1 + cap) + 1 + pos, pack_word(id, flag));
                else
                    loc()[pos] = (uint8_t)j;
            }
        }
        if ((uint32_t)lane < G && (uint32_t)lane != me && cnt)
            st_sys_u64(p.req[lane] + ((size_t)me * p.O + slot) * (1 + cap), pack_word(cnt | (cur_q << kMsgCountBits), flag));
        const uint32_t nloc = __shfl_sync(0xffffffffu, cnt, me);
        __syncwarp();
        const uint32_t c0 = (uint32_t)clock64();
        eval_local<true>(nloc);
        const uint32_t c1 = (uint32_t)clock64();
        cy_local += c1 - c0;
        const unsigned long long* inbox = p.resp[me] + (size_t)slot * G * cap;
#pragma unroll 1
        for (uint32_t base = 0; base < n; base += 32) {
            const uint32_t j = base + lane;
            if (j < n) {
                const uint32_t s = cand_slot()[j], dst = s >> 8, pos = s & 255u;
                if (dst != me)
                    cand_d()[j] = __uint_as_float(wait_word(inbox + (size_t)dst * cap + pos, flag));
            }
        }
        dead = __any_sync(0xffffffffu, dead);
        cy_wait += (uint32_t)clock64() - c1;
        st_rounds += 1;
        __syncwarp();
    }

    // ---- helper: one of the H warps of this GPU that measure local rows for REMOTE owners.  The (G-1) * O inbound
    // mailboxes (one per remote owner slot) are dealt round-robin to the helpers; lane i of helper h watches mailbox
    // h + i * H, so one volatile load per lane polls the helper's whole set.  A request names its query; the query vector
    // sits next to the mailbox (the owner stored it there, fence, before its first request) and is loaded into registers
    // whenever the helper switches mailbox or the mailbox switches query. --------------------------------------------------
    __device__ __forceinline__ void load_mailbox_query(const uint8_t* src_bytes) {
        const uint4* src = reinterpret_cast<const uint4*>(src_bytes);
        float part = 0.f;
#pragma unroll
        for (int i = 0; i < NQ; ++i) {
            const uint32_t c = lane + 32 * i;
            qreg[i] = c < nchunks ? ld_nocache_u4(src + c) : make_uint4(0, 0, 0, 0);
            part = norm_add(part, query_norm_chunk<DM, SK>(qreg[i]));
        }
        a2 = 0.f;
        if constexpr (DM == DM_COS)
            a2 = warp_sum(part);
    }

    __device__ __forceinline__ void run_helper(uint32_t h) {
        const uint32_t cap = p.cap, G = p.G, O = p.O, H = p.H, M = (G - 1) * O;
        const uint32_t mp = h + (uint32_t)lane * H; // this lane's mailbox among the M remote ones (if < M)
        bool alive = mp < M;
        uint32_t my_last = p.flag_base;
        uint32_t src = 0, oslot = 0;
        if (alive) {
            src = mp / O, oslot = mp - src * O;
            if (src >= p.me)
                ++src; // own mailboxes are skipped
        }
        const unsigned long long* my_hdr = p.req[p.me] + ((size_t)src * O + oslot) * (1 + cap);
        uint32_t cur_m = 0xFFFFFFFFu;
        uint32_t spins = 0;
#pragma unroll 1
        while (__any_sync(0xffffffffu, alive)) {
            uint32_t pay = 0, flag = 0;
            bool fresh = false;
            if (alive) {
                const unsigned long long v = ld_sys_u64(my_hdr);
                flag = (uint32_t)(v >> 32), pay = (uint32_t)v;
                const uint32_t ahead = flag - my_last;
                fresh = ahead != 0u && ahead < (1u << 20) && flag - p.flag_base < (1u << 20);
            }
            uint32_t ready = __ballot_sync(0xffffffffu, fresh);
            if (!ready) {
                if ((++spins & 1023u) == 0u) {
                    if (lane == 0 && timed_out())
                        dead = true;
                    dead = __any_sync(0xffffffffu, dead);
                    if (dead)
                        return;
                }
                __nanosleep(32);
                continue;
            }
            spins = 0;
            while (ready) {
                const int b = __ffs(ready) - 1;
                ready &= ready - 1;
                const uint32_t r_pay = __shfl_sync(0xffffffffu, pay, b), r_flag = __shfl_sync(0xffffffffu, flag, b);
                const uint32_t r_src = __shfl_sync(0xffffffffu, src, b), r_oslot = __shfl_sync(0xffffffffu, oslot, b);
                if (lane == b)
                    my_last = r_flag;
                if (r_pay == kMsgExit) {
                    if (lane == b)
                        alive = false;
                    continue;
                }
                const uint32_t q = r_pay >> kMsgCountBits, n_d = r_pay & ((1u << kMsgCountBits) - 1u);
                const size_t m = (size_t)r_src * O + r_oslot;
                if ((uint32_t)m != cur_m || q != cur_q) {
                    load_mailbox_query(p.reqq[p.me] + m * p.g.row_bytes);
                    cur_m = (uint32_t)m, cur_q = q;
                }
                const unsigned long long* hdr = p.req[p.me] + m * (1 + cap);
                unsigned long long* outbox = p.resp[r_src] + ((size_t)r_oslot * G + p.me) * cap;
#pragma unroll 1
                for (uint32_t base = 0; base < n_d; base += 32) {
                    const uint32_t cnt = min(32u, n_d - base);
                    const uint32_t my_id = (uint32_t)lane < cnt ? wait_word(hdr + 1 + base + lane, r_flag) : 0u;
                    dead = __any_sync(0xffffffffu, dead);
                    if (dead)
                        return;
                    if ((uint32_t)lane < cnt)
                        cand_id()[lane] = my_id;
                    __syncwarp();
                    eval_local<false>(cnt);
                    __syncwarp();
                    if ((uint32_t)lane < cnt)
                        st_sys_u64(outbox + base + lane, pack_word(__float_as_uint(cand_d()[lane]), r_flag));
                    __syncwarp();
                }
            }
        }
    }

    // ---- owner, PS: the projected screen of a level-0 round (PScreenEval::screen on one warp).  Lane l takes candidates
    // l, l + 32, ...: two 64-byte records per lane travel together (one round trip for a 64-wide list), 128-byte ones one at a
    // time; the bound is pscreen_bound on ps_accum's sums, as in the CTA kernel.  cand_id[0..n) -> the candidates with
    // !(lb >= radius), compacted in stored order; returns their number.  Not inlined: the bound's double arithmetic then
    // lives in its own frame instead of adding to the walk's spills at the 80-register cap of 6 CTAs/SM.
    __device__ __forceinline__ float pscreen_lb(const uint4 (&v)[8], bool wide, float4 qh, uint32_t slots) const {
        const float* qt = psq();
        float sf = 0.f, cc = 0.f;
        ps_accum(qt, v[1], sf, cc);
        ps_accum(qt + 16, v[2], sf, cc);
        ps_accum(qt + 32, v[3], sf, cc);
        if (wide) {
            ps_accum(qt + 48, v[4], sf, cc);
            ps_accum(qt + 64, v[5], sf, cc);
            ps_accum(qt + 80, v[6], sf, cc);
            ps_accum(qt + 96, v[7], sf, cc);
        }
        const float4 meta = make_float4(__uint_as_float(v[0].x), __uint_as_float(v[0].y), __uint_as_float(v[0].z), __uint_as_float(v[0].w));
        return pscreen_bound<DM, NQ>(sf, cc, meta, qh, a2, slots);
    }
    __device__ __noinline__ uint32_t pscreen(uint32_t n, float radius) {
        const uint32_t slots = ps_code_slots(p.g.ps_k), rec = ps_record_bytes(p.g.ps_k) / 16;
        const float4 qh = *reinterpret_cast<const float4*>(psq() + slots);
        uint32_t* ids = cand_id();
        float* lbs = cand_d();
#pragma unroll 1
        for (uint32_t j = lane; j < n; j += 64) {
            uint4 a[8], b[8];
            const uint4* ra = p.g.ps_records + (size_t)ids[j] * rec;
            if (rec == 4) {
                const bool two = j + 32 < n;
                const uint4* rb = p.g.ps_records + (size_t)ids[two ? j + 32 : j] * rec;
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    a[i] = __ldg(ra + i), b[i] = __ldg(rb + i);
                lbs[j] = pscreen_lb(a, false, qh, slots);
                if (two)
                    lbs[j + 32] = pscreen_lb(b, false, qh, slots);
            } else {
#pragma unroll
                for (int i = 0; i < 8; ++i)
                    a[i] = __ldg(ra + i);
                lbs[j] = pscreen_lb(a, true, qh, slots);
                if (j + 32 < n) {
                    const uint4* rb = p.g.ps_records + (size_t)ids[j + 32] * rec;
#pragma unroll
                    for (int i = 0; i < 8; ++i)
                        b[i] = __ldg(rb + i);
                    lbs[j + 32] = pscreen_lb(b, true, qh, slots);
                }
            }
        }
        __syncwarp();
        const uint32_t lt = (1u << lane) - 1u;
        uint32_t m = 0;
        for (uint32_t base = 0; base < n; base += 32) {
            const uint32_t j = base + lane;
            const bool keep = j < n && !(lbs[j] >= radius);
            const uint32_t id = j < n ? ids[j] : 0u;
            const uint32_t mk = __ballot_sync(0xffffffffu, keep);
            __syncwarp();
            if (keep)
                ids[m + __popc(mk & lt)] = id;
            m += __popc(mk);
        }
        __syncwarp();
        st_screened += n, st_rejected += n - m;
        return m;
    }

    __device__ __forceinline__ void tell_helpers(uint32_t payload) {
        const uint32_t flag = p.flag_base + (++seq);
        if ((uint32_t)lane < p.G && (uint32_t)lane != p.me)
            st_sys_u64(p.req[lane] + ((size_t)p.me * p.O + slot) * (1 + p.cap), pack_word(payload, flag));
    }

    // ---- owner: the reference's walk of ONE query by one warp.  A single produce -> evaluate -> consume loop serves the entry
    // point, the greedy descent (search_for_one_, index.hpp:3277-3316) and the base-layer beam (search_to_find_in_base_,
    // :3400-3485), so that eval_round is instantiated once. -------------------------------------------------------------
    __device__ __forceinline__ void run_owner(uint32_t q) {
        const uint32_t M0 = p.g.M0, L = p.L;
        uint32_t* vis = p.vis + (size_t)slot * p.words_per_slot;
        uint32_t* touched = p.touched + (size_t)slot * p.touched_cap;
        load_query(q);
        cur_q = q;
        if constexpr (PS) { // q~ and its header from the batch's pre-pass (launch_ps_queries)
            const uint32_t nf = psq_floats();
            __syncwarp(); // the previous query's screen is done with psq
            for (uint32_t i = lane; i < nf; i += 32)
                psq()[i] = __ldg(p.g.ps_query + (size_t)q * nf + i);
            __syncwarp();
        }
        if (p.G > 1) { // the helpers read the query from the mailbox of this owner slot on THEIR GPU
            for (uint32_t d = 0; d < p.G; ++d) {
                if (d == p.me)
                    continue;
                uint4* dst = reinterpret_cast<uint4*>(p.reqq[d] + ((size_t)p.me * p.O + slot) * p.g.row_bytes);
#pragma unroll
                for (int i = 0; i < NQ; ++i) {
                    const uint32_t c = lane + 32 * i;
                    if (c < nchunks)
                        dst[c] = qreg[i];
                }
            }
            __threadfence_system(); // the vector is in place before the first request that names this query can be seen
        }
        int level = -1; // -1: measuring the entry point; >= 1: greedy on that level; 0: beam on the base layer
        uint32_t cur = p.g.entry;
        float cur_d = 0.f;
        uint32_t size = 0, cursor = 0, ntouched = 0, limbo_n = 0;
        float limbo_d = 0.f;
#pragma unroll 1
        while (!dead) {
            // ---- produce the ids to measure ----
            const uint32_t cp0 = (uint32_t)clock64();
            uint32_t n = 0;
            if (level < 0) {
                if (lane == 0)
                    cand_id()[0] = cur;
                n = 1;
            } else if (level > 0) {
                const uint32_t* list = p.g.upper_adj + ((size_t)__ldg(p.g.upper_ref + cur) + (level - 1)) * p.g.M;
                for (uint32_t off = 0; off < p.g.M; off += 32) {
                    const uint32_t id = (off + lane < p.g.M) ? __ldg(list + off + lane) : kNoNeighbor;
                    const bool valid = id != kNoNeighbor;
                    const uint32_t m = __ballot_sync(0xffffffffu, valid);
                    if (valid)
                        cand_id()[n + __popc(m & ((1u << lane) - 1u))] = id;
                    n += __popc(m);
                }
                st_hops += 1;
            } else {
                // pop the closest unexpanded entry (walk.cuh TopSmem::pop), or a tie waiting in limbo
                uint32_t c = kNoNeighbor;
                uint32_t* ti = top_i();
                if (cursor < size) {
                    c = ti[cursor];
                    __syncwarp();
                    if (lane == 0)
                        ti[cursor] = c | kExpandedBit;
                    __syncwarp();
                    uint32_t nxt = size;
                    for (uint32_t b = cursor + 1; b < size; b += 32) {
                        const uint32_t e = b + lane;
                        const bool un = e < size && !(ti[e] & kExpandedBit);
                        const uint32_t m = __ballot_sync(0xffffffffu, un);
                        if (m) {
                            nxt = b + __ffs(m) - 1;
                            break;
                        }
                    }
                    cursor = nxt;
                } else if (limbo_n) {
                    c = limbo()[--limbo_n];
                }
                if (c == kNoNeighbor)
                    break; // the beam is exhausted: index.hpp:3445 / queue empty
                const uint32_t* list = p.g.adj0 + (size_t)c * M0;
                if (M0 == 64) {
                    // both halves of a 64-wide list at once: the two bitmap atomics of a lane are in flight together (one L2
                    // atomic round trip per expansion instead of two).  Duplicates are legal in reference graphs (refine_
                    // padding, index.hpp:3554-3558): only the FIRST occurrence in stored order may count as unseen, so the
                    // second half is also checked against the first (through the candidate array, free at this point).
                    const uint32_t id0 = __ldg(list + lane), id1 = __ldg(list + 32 + lane);
                    const bool v0 = id0 != kNoNeighbor, v1 = id1 != kNoNeighbor;
                    cand_id()[lane] = id0;
                    __syncwarp();
                    const uint32_t p0 = __match_any_sync(0xffffffffu, id0), p1 = __match_any_sync(0xffffffffu, id1);
                    bool first0 = v0 && ((uint32_t)(__ffs(p0) - 1) == (uint32_t)lane);
                    bool first1 = v1 && ((uint32_t)(__ffs(p1) - 1) == (uint32_t)lane);
                    if (first1)
                        for (int t = 0; t < 32; ++t)
                            first1 &= cand_id()[t] != id1;
                    __syncwarp();
                    bool fresh0 = false, fresh1 = false;
                    uint32_t old0 = 0, old1 = 0;
                    const uint32_t bit0 = 1u << (id0 & 31), bit1 = 1u << (id1 & 31);
                    if (first0)
                        old0 = atomicOr(&vis[id0 >> 5], bit0);
                    if (first1)
                        old1 = atomicOr(&vis[id1 >> 5], bit1);
                    fresh0 = first0 && !(old0 & bit0), fresh1 = first1 && !(old1 & bit1);
                    const uint32_t m0 = __ballot_sync(0xffffffffu, fresh0), m1 = __ballot_sync(0xffffffffu, fresh1);
                    const uint32_t lt = (1u << lane) - 1u, n0 = __popc(m0);
                    if (fresh0) {
                        const uint32_t r = __popc(m0 & lt);
                        cand_id()[r] = id0;
                        if (ntouched + r < p.touched_cap)
                            touched[ntouched + r] = id0 >> 5;
                    }
                    __syncwarp(); // (the compaction above overwrites entries another lane compared against: all compares are done)
                    if (fresh1) {
                        const uint32_t r = n0 + __popc(m1 & lt);
                        cand_id()[r] = id1;
                        if (ntouched + r < p.touched_cap)
                            touched[ntouched + r] = id1 >> 5;
                    }
                    n = n0 + __popc(m1);
                    ntouched += n;
                } else
                    for (uint32_t off = 0; off < M0; off += 32) {
                        const uint32_t id = (off + lane < M0) ? __ldg(list + off + lane) : kNoNeighbor;
                        const bool valid = id != kNoNeighbor;
                        if (!__any_sync(0xffffffffu, valid))
                            break;
                        // duplicate ids inside one list are legal in reference graphs (refine_ padding, index.hpp:3554-3558)
                        const uint32_t peers = __match_any_sync(0xffffffffu, id);
                        const bool first = valid && ((uint32_t)(__ffs(peers) - 1) == (uint32_t)lane);
                        bool fresh = false;
                        if (first) {
                            const uint32_t bit = 1u << (id & 31);
                            fresh = !(atomicOr(&vis[id >> 5], bit) & bit);
                        }
                        const uint32_t m = __ballot_sync(0xffffffffu, fresh);
                        const uint32_t rank = __popc(m & ((1u << lane) - 1u));
                        if (fresh) {
                            cand_id()[n + rank] = id;
                            if (ntouched + rank < p.touched_cap)
                                touched[ntouched + rank] = id >> 5;
                        }
                        n += __popc(m);
                        ntouched += __popc(m);
                    }
                st_pops += 1;
            }
            __syncwarp();
            const uint32_t cp1 = (uint32_t)clock64();
            const uint32_t n_all = n; // the screen's rejects count as computed distances: the reference computes them
            if constexpr (PS) {
                // a level-0 round that starts with a full top list: a candidate can enter only below td[L-1], and the radius
                // only shrinks within the round, so screening against its start is safe (WalkerT::beam_impl's rule, which
                // also skips a NaN radius).  A greedy pass takes only a candidate strictly below cur_d: it is screened against
                // cur_d (WalkerT::greedy's rule).
                const float radius = level > 0 ? cur_d : level == 0 && size == L ? top_d()[size - 1] : __int_as_float(0x7fffffff);
                if (radius == radius && n)
                    n = pscreen(n, radius);
                cy_screen += (uint32_t)clock64() - cp1;
            }
            // ---- evaluate: every id on the GPU that holds its row ----
            if (n)
                eval_round(n);
            if (dead)
                break;
            const uint32_t cp2 = (uint32_t)clock64();
            cy_produce += cp1 - cp0; // classification + sends are counted with the evaluation
            st_dist += n_all;
            // ---- consume ----
            if (level < 0) {
                cur_d = cand_d()[0];
                level = p.g.max_level;
            } else if (level > 0) {
                float best = cur_d; // one pass of index.hpp:3304-3311 == first minimum below cur_d
                int bi = -1;
                for (uint32_t j = 0; j < n; ++j) {
                    const float d = cand_d()[j];
                    if (d < best)
                        best = d, bi = (int)j;
                }
                if (bi >= 0)
                    cur = cand_id()[bi], cur_d = best;
                else
                    --level;
                __syncwarp();
            } else {
                // index.hpp:3470: accepted iff top.size() < L || d < radius; parallel pre-filter, then replay in stored order
                float* td = top_d();
                uint32_t* ti = top_i();
                for (uint32_t base = 0; base < n; base += 32) {
                    const uint32_t j = base + lane;
                    const float dj = j < n ? cand_d()[j] : INFINITY;
                    float radius = td[size - 1];
                    uint32_t m = __ballot_sync(0xffffffffu, j < n && (size < L || dj < radius));
                    while (m) {
                        const int b = __ffs(m) - 1;
                        m &= m - 1;
                        const float d = __shfl_sync(0xffffffffu, dj, b);
                        if (size < L || d < radius) {
                            const uint32_t id = cand_id()[base + b];
                            float ev_d;
                            uint32_t ev_i;
                            top_insert(td, ti, size, cursor, L, d, id, lane, ev_d, ev_i);
                            if ((p.g.flags & 2u) && lane == 0)
                                prefetch_l2(p.g.adj0 + (size_t)id * M0);
                            radius = td[size - 1];
                            if (limbo_n && radius < limbo_d)
                                limbo_n = 0;
                            if (ev_i != kNoNeighbor && !(ev_i & kExpandedBit) && ev_d == radius) {
                                if (limbo_n < kLimboCap) {
                                    if (lane == 0)
                                        limbo()[limbo_n] = ev_i;
                                    limbo_n++, limbo_d = radius;
                                    __syncwarp();
                                } else if (lane == 0) {
                                    atomicAdd(&p.counters[7], 1ull); // rare by construction
                                }
                            }
                        }
                    }
                }
                __syncwarp();
            }
            cy_consume += (uint32_t)clock64() - cp2;
            if (level == 0 && size == 0) { // the descent is over: open the beam at `cur` (its distance is known; the
                if (lane == 0) {           // reference measures it again, index.hpp:3436, so the counter advances)
                    top_d()[0] = cur_d, top_i()[0] = cur;
                    atomicOr(&vis[cur >> 5], 1u << (cur & 31));
                    touched[0] = cur >> 5;
                }
                size = 1, cursor = 0, ntouched = 1;
                st_dist += 1;
                __syncwarp();
            }
        }
        // un-visit only the words this walk touched
        if (ntouched <= p.touched_cap) {
            for (uint32_t i = lane; i < ntouched; i += 32)
                vis[touched[i]] = 0u;
        } else {
            for (size_t i = lane; i < p.words_per_slot; i += 32)
                vis[i] = 0u;
        }
        // results -> every rank (the all-gather of SURVEY 8e, fused); top is ascending, shrink(k), keys
        const uint32_t found = dead ? 0u : min(size, p.k);
        for (uint32_t i = lane; i < p.k; i += 32) {
            unsigned long long key = ~0ull;
            float d = INFINITY;
            if (i < found) {
                key = __ldg(p.g.keys + (top_i()[i] & kIdMask));
                d = top_d()[i];
            }
            for (uint32_t r = 0; r < p.G; ++r) {
                p.res_keys[r][(size_t)q * p.k + i] = key;
                p.res_dists[r][(size_t)q * p.k + i] = d;
            }
        }
        if ((uint32_t)lane < p.G)
            p.res_counts[lane][q] = found;
        __syncwarp();
    }
};

template <int DM, int SK, int NQ, bool PS = false>
__global__ void __launch_bounds__(kGroupThreads, 6) group_search_kernel(const __grid_constant__ GroupLaunch p) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    GroupWarp<DM, SK, NQ, PS> w(p);
    w.lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    w.slot = blockIdx.x * kGroupWarps + warp;
    w.nchunks = p.g.row_bytes / 16;
    w.ws = smem_raw + (size_t)warp * w.lay().total;
    w.phase_bits = 0;
    if (w.lane == 0) {
        for (uint32_t i = 0; i < p.ring_slots; ++i)
            mbar_init(w.bars() + i, 1);
        fence_mbar_init();
    }
    __syncwarp();
    w.seq = 0, w.last = p.flag_base, w.dead = false, w.a2 = 0.f, w.cur_q = 0xFFFFFFFFu;
    w.waited = (p.me == p.root);
    w.st_dist = w.st_pops = w.st_hops = w.st_rounds = w.st_rows = 0;
    w.cy_produce = w.cy_local = w.cy_wait = w.cy_consume = 0;
    w.cy_screen = w.st_screened = w.st_rejected = 0;
    w.t0 = globaltimer_ns();

    // the root's query staging buffer is complete when its kernel starts (stream order): tell everybody
    if (p.me == p.root && w.slot == 0 && (uint32_t)w.lane < p.G)
        st_sys_u64(p.qready[w.lane], (unsigned long long)p.epoch);
    if (w.slot < p.O) {
        // owner warp: this GPU's queries (q mod G == me) are handed to its owner warps as they become free
        for (;;) {
            uint32_t idx = 0;
            if (w.lane == 0)
                idx = (uint32_t)atomicAdd(&p.counters[6], 1ull);
            idx = __shfl_sync(0xffffffffu, idx, 0);
            const unsigned long long q = (unsigned long long)idx * p.G + p.me;
            if (q >= p.nq || w.dead)
                break;
            w.run_owner((uint32_t)q);
        }
        if (p.G > 1)
            w.tell_helpers(kMsgExit);
    } else {
        w.run_helper(w.slot - p.O);
    }
    // completion: results of this GPU's owners are visible system-wide before its done flag is
    __threadfence_system();
    __syncwarp();
    bool last_warp = false;
    if (w.lane == 0) {
        atomicAdd(&p.counters[1], (unsigned long long)w.st_dist);
        atomicAdd(&p.counters[2], (unsigned long long)w.st_pops);
        atomicAdd(&p.counters[3], (unsigned long long)w.st_hops);
        atomicAdd(&p.counters[4], (unsigned long long)w.st_rounds);
        atomicAdd(&p.counters[5], (unsigned long long)w.st_rows);
        if (w.cy_produce | w.cy_wait) {
            atomicAdd(&p.counters[8], (unsigned long long)w.cy_produce), atomicAdd(&p.counters[9], (unsigned long long)w.cy_local);
            atomicAdd(&p.counters[10], (unsigned long long)w.cy_wait), atomicAdd(&p.counters[11], (unsigned long long)w.cy_consume);
        }
        if constexpr (PS) {
            atomicAdd(&p.counters[12], (unsigned long long)w.st_screened), atomicAdd(&p.counters[13], (unsigned long long)w.st_rejected);
            atomicAdd(&p.counters[14], (unsigned long long)w.cy_screen);
        }
        __threadfence();
        last_warp = atomicAdd(&p.counters[0], 1ull) == (unsigned long long)gridDim.x * kGroupWarps - 1ull;
    }
    last_warp = __shfl_sync(0xffffffffu, last_warp, 0);
    if (last_warp) {
        __threadfence_system();
        if ((uint32_t)w.lane < p.G) {
            st_sys_u64(p.done[w.lane] + p.me, (unsigned long long)p.epoch);
            uint32_t spins = 0;
            while (ld_sys_u64(p.done[p.me] + w.lane) != (unsigned long long)p.epoch) {
                if ((++spins & 2047u) == 0u && w.timed_out())
                    break;
                __nanosleep(64);
            }
        }
        __threadfence_system();
    }
}

template <int DM, int SK, int NQ, bool PS = false> void group_launch_one(const GroupLaunch& p, uint32_t grid, size_t smem, cudaStream_t stream) {
    auto kern = group_search_kernel<DM, SK, NQ, PS>;
    LB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, kGroupThreads, smem, stream>>>(p);
    LB_CUDA(cudaGetLastError());
    count_launch();
}
template <int DM, int SK, int NQ, bool PS = false> int group_occupancy_one(size_t smem) {
    auto kern = group_search_kernel<DM, SK, NQ, PS>;
    cudaFuncAttributes fa;
    LB_CUDA(cudaFuncGetAttributes(&fa, kern));
    if (smem + fa.sharedSizeBytes > device_smem_optin()) // deep rings of wide rows (LB200_GROUP_RING_SLOTS): refused by name
        return 0;
    LB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int blocks = 0;
    LB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, kern, kGroupThreads, smem));
    return blocks;
}

// in-degree of the base layer per bucket of consecutive rows: how often the rows of a bucket appear in adjacency lists is
// how often they will be measured.  Row ranges of equal WEIGHT (not equal length) balance the ranks: early rows of an HNSW
// build collect more links than late ones, so equal-length ranges would leave the first rank with ~40 % more work.
constexpr uint32_t kBalanceBuckets = 4096;
__global__ void indegree_hist_kernel(const uint32_t* __restrict__ adj0, size_t total, uint32_t n, unsigned long long* __restrict__ hist) {
    __shared__ uint32_t sh[kBalanceBuckets];
    for (uint32_t i = threadIdx.x; i < kBalanceBuckets; i += blockDim.x)
        sh[i] = 0;
    __syncthreads();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t id = adj0[i];
        if (id < n)
            atomicAdd(&sh[(uint32_t)(((unsigned long long)id * kBalanceBuckets) / n)], 1u);
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < kBalanceBuckets; i += blockDim.x)
        if (sh[i])
            atomicAdd(&hist[i], (unsigned long long)sh[i]);
}

__global__ void group_copy_results_kernel(const uint64_t* __restrict__ rk, const float* __restrict__ rd, const uint32_t* __restrict__ rc,
                                          uint64_t* __restrict__ keys, float* __restrict__ dists, uint32_t* __restrict__ counts,
                                          size_t nq, size_t k) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nq * k) {
        if (keys)
            keys[i] = rk[i];
        if (dists)
            dists[i] = rd[i];
    }
    if (counts && i < nq)
        counts[i] = rc[i];
}

} // namespace

// =====================================================================================================================
// host side
// =====================================================================================================================

// Roles of a launch: O owner warps (one query each at a time; enough for every query this rank owns, but leaving a quarter of
// the resident warps to the helpers) and H helper warps that share the (G-1) * O inbound mailboxes -- no more helpers than
// mailboxes, and no helper watches more than 32 (one per lane).  Deterministic in (world, nq, W, Omax): every rank computes
// the same plan.  Returns false when the resident warps cannot cover the mailboxes.
bool group_plan(int world, size_t nq, uint32_t W, uint32_t Omax, uint32_t& O, uint32_t& H) {
    O = (uint32_t)round_up((nq + world - 1) / world, kGroupWarps), H = 0;
    O = std::min(O, Omax);
    if (world > 1) {
        O = std::min<uint32_t>(O, (W - W / 4) & ~3u);
        if (O == 0)
            return false;
        const uint32_t M = (uint32_t)(world - 1) * O;
        H = std::min<uint32_t>(W - O, (uint32_t)round_up(M, kGroupWarps));
        H = std::max<uint32_t>(H, (uint32_t)round_up((M + 31) / 32, kGroupWarps));
        return O + H <= W;
    }
    O = std::min(O, W & ~3u);
    return O > 0;
}

// every spin in the kernel gives up after this long (LB200_GROUP_TIMEOUT_S, default 20 s; raise it under compute-sanitizer)
static unsigned long long group_timeout_ns() {
    double sec = 20.0;
    if (const char* e = getenv("LB200_GROUP_TIMEOUT_S"))
        sec = atof(e) > 0 ? atof(e) : sec;
    return (unsigned long long)(sec * 1e9);
}

struct DeviceGuard { // the group switches devices; the caller's current device is put back when an entry point returns
    int dev = 0;
    DeviceGuard() { cudaGetDevice(&dev); }
    ~DeviceGuard() { cudaSetDevice(dev); }
};

struct PtrBlob { // how one device allocation is handed to the other ranks
    cudaIpcMemHandle_t ipc;
    void* raw;
};

struct GroupConfigBlob {
    uint32_t valid;
    int32_t metric_kind, scalar_kind;
    uint64_t dims, M, M0, ef, n, upper_lists, row_bytes, vec_bytes;
    uint32_t entry;
    int32_t max_level;
    uint32_t flags;
    uint32_t bounds[kGroupMax + 1]; // row ranges, balanced by base-layer in-degree
    PtrBlob vectors, adj0, upper_ref, upper_adj, keys;
};

struct SlabLayout {
    size_t req, reqq, resp, res_keys, res_dists, res_counts, done, qready, err, qbuf, total;
};

// Omax = owner slots per rank the mailboxes are sized for
static SlabLayout slab_layout(uint32_t Omax, uint32_t G, uint32_t cap, size_t res_cap, size_t max_batch, size_t qrow) {
    SlabLayout s;
    size_t o = 0;
    auto take = [&](size_t bytes) {
        const size_t at = o;
        o += round_up(bytes, 256);
        return at;
    };
    s.req = take((size_t)G * Omax * (1 + cap) * 8);
    s.resp = take((size_t)Omax * G * cap * 8);
    s.reqq = take((size_t)G * Omax * qrow); // (after resp: renew_flags clears [req, reqq) only)
    s.res_keys = take(res_cap * 8);
    s.res_dists = take(res_cap * 4);
    s.res_counts = take(max_batch * 4);
    s.done = take(kGroupMax * 8);
    s.qready = take(8);
    s.err = take(4);
    s.qbuf = take(max_batch * qrow);
    s.total = o;
    return s;
}

// Contiguous row ranges (SURVEY 8e) of equal expected work, from the level-0 in-degree per bucket of kBalanceBuckets
// consecutive rows (indegree_hist_kernel on an index, host_indegree_hist on a parsed file: the same counts).
static void balanced_bounds(const std::vector<unsigned long long>& hist, size_t n_rows, int world, uint32_t* bounds) {
    // weight of a bucket = its in-degree + the mean in-degree: measured on the bench corpus, equal-length ranges leave the
    // first of two ranks 58 % of the evaluations, pure in-degree weighting 45 %; the blend lands near 50 %
    double links = 0;
    for (unsigned long long h : hist)
        links += (double)h;
    const double mean = links / kBalanceBuckets + 1.0;
    double total = 0;
    for (unsigned long long h : hist)
        total += (double)h + mean;
    bounds[0] = 0;
    double acc = 0;
    int r = 1;
    for (uint32_t b = 0; b < kBalanceBuckets && r < world; ++b) {
        acc += (double)hist[b] + mean;
        while (r < world && acc >= total * r / world) {
            bounds[r] = (uint32_t)std::min<size_t>(n_rows, ((size_t)(b + 1) * n_rows + kBalanceBuckets - 1) / kBalanceBuckets);
            ++r;
        }
    }
    for (; r <= world; ++r)
        bounds[r] = (uint32_t)n_rows;
    bounds[world] = (uint32_t)n_rows;
    if (getenv("LB200_GROUP_EQUAL_RANGES")) // experiments: plain n*r/G ranges
        for (int q = 0; q <= world; ++q)
            bounds[q] = (uint32_t)((n_rows * (size_t)q) / (size_t)world);
    for (int q = 1; q <= world; ++q) // monotone, whatever the histogram looked like
        bounds[q] = std::max(bounds[q], bounds[q - 1]);
}

static std::vector<unsigned long long> host_indegree_hist(const std::vector<uint32_t>& adj0, size_t n) {
    std::vector<unsigned long long> hist(kBalanceBuckets, 0);
    for (uint32_t id : adj0)
        if (id < n)
            hist[(uint32_t)(((unsigned long long)id * kBalanceBuckets) / n)] += 1;
    return hist;
}

// Rows [lo, hi) of a file (node i's stored bytes at file + row_off[i]) into d_rows on the current device, row_bytes apart and
// zero padded.  Rows are gathered into one half of a bounded pinned block while the other half is on its way to the device:
// no host copy of a whole slice (or file) is ever made.
static void upload_file_rows(const uint8_t* file, const std::vector<uint64_t>& row_off, size_t stored_bytes, size_t lo, size_t hi,
                             uint8_t* d_rows, size_t row_bytes) {
    if (hi <= lo)
        return;
    struct Staging {
        uint8_t* pinned = nullptr;
        cudaStream_t stream = nullptr;
        cudaEvent_t done[2] = {nullptr, nullptr};
        ~Staging() {
            if (stream)
                cudaStreamSynchronize(stream), cudaStreamDestroy(stream);
            for (cudaEvent_t e : done)
                if (e)
                    cudaEventDestroy(e);
            if (pinned)
                cudaFreeHost(pinned);
        }
    } st;
    const size_t block = std::max<size_t>(1, std::min(hi - lo, ((size_t)32 << 20) / row_bytes)); // rows per half (<= 32 MB)
    LB_CUDA(cudaMallocHost(&st.pinned, 2 * block * row_bytes));
    LB_CUDA(cudaStreamCreateWithFlags(&st.stream, cudaStreamNonBlocking));
    LB_CUDA(cudaEventCreateWithFlags(&st.done[0], cudaEventDisableTiming));
    LB_CUDA(cudaEventCreateWithFlags(&st.done[1], cudaEventDisableTiming));
    bool used[2] = {false, false};
    int h = 0;
    for (size_t b0 = lo; b0 < hi; b0 += block, h ^= 1) {
        const size_t cnt = std::min(block, hi - b0);
        uint8_t* stage = st.pinned + (size_t)h * block * row_bytes;
        if (used[h])
            LB_CUDA(cudaEventSynchronize(st.done[h]));
        for (size_t i = 0; i < cnt; ++i) {
            memcpy(stage + i * row_bytes, file + row_off[b0 + i], stored_bytes);
            memset(stage + i * row_bytes + stored_bytes, 0, row_bytes - stored_bytes);
        }
        LB_CUDA(cudaMemcpyAsync(d_rows + (b0 - lo) * row_bytes, stage, cnt * row_bytes, cudaMemcpyHostToDevice, st.stream));
        LB_CUDA(cudaEventRecord(st.done[h], st.stream));
        used[h] = true;
    }
    LB_CUDA(cudaStreamSynchronize(st.stream));
}

class GroupRank {
  public:
    int rank = 0, world = 1, device = 0;
    bool local = false; // all ranks live in this process (peer pointers are used directly)
    IndexConfig cfg;
    int dist_mode = 0;
    size_t n = 0, row_bytes = 0, vec_bytes = 0, upper_lists = 0;
    uint32_t entry = 0, flags = 2;
    int32_t max_level = -1;
    uint32_t bounds[kGroupMax + 1] = {0};
    // local copies
    uint8_t* d_rows = nullptr;
    uint32_t *d_adj0 = nullptr, *d_upper_ref = nullptr, *d_upper_adj = nullptr;
    uint64_t* d_keys = nullptr;
    // mailboxes
    uint8_t* slab = nullptr;
    uint8_t* peer_slab[kGroupMax] = {nullptr};
    SlabLayout lay{};
    uint32_t Wmax = 0, Omax = 0, cap = 0;
    size_t res_cap = 0, max_batch = 0;
    // owner scratch
    uint32_t *d_vis = nullptr, *d_touched = nullptr;
    size_t words_per_slot = 0;
    uint32_t touched_cap = 16384;
    unsigned long long* d_counters = nullptr;
    uint32_t epoch = 0;
    std::map<uint32_t, uint32_t> W_for_L; // agreed resident warps per GPU for a beam width
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    uint32_t last_nq = 0;
    std::vector<void*> opened; // IPC mappings to close
    void* d_in = nullptr;      // root: staging of the raw input queries of the host-buffer entry point
    size_t in_bytes = 0;
    std::vector<uint32_t> h_counts;
    uint32_t h_err = 0;
    // a group's own index (lb200_group_index_init): rows and graph are those of this rank's Index (borrowed, re-attached after
    // every build); the rank holds the rows [cap_lo, cap_hi) of an index of `capacity` rows
    bool borrowed = false;
    size_t capacity = 0, cap_lo = 0, cap_hi = 0;

    ~GroupRank() {
        cudaSetDevice(device);
        for (void* p : opened)
            cudaIpcCloseMemHandle(p);
        release();
    }

    // what allocate() takes on this rank's device (lb200_group_rank_info_t)
    void footprint(lb200_group_rank_info_t& f) const {
        memset(&f, 0, sizeof(f));
        f.rank = rank, f.world = world;
        f.rows_begin = bounds[rank], f.rows_end = bounds[rank + 1];
        const size_t g = borrowed ? capacity : n; // a group's own index: sized for its capacity
        if (borrowed)
            f.rows_begin = cap_lo, f.rows_end = cap_hi;
        f.bytes_rows = (f.rows_end - f.rows_begin) * row_bytes;
        f.bytes_graph = g * cfg.M0 * 4 + g * 4 + upper_lists * cfg.M * 4 + g * 8;
        f.bytes_scratch = (size_t)Omax * words_per_slot * 4 + (size_t)Omax * touched_cap * 4 + 16 * sizeof(unsigned long long) + in_bytes;
        f.bytes_mailbox = lay.total;
    }

    // frees every device allocation of the rank (its peer mappings stay)
    void release() {
        cudaSetDevice(device);
        if (!borrowed)
            cudaFree(d_rows), cudaFree(d_adj0), cudaFree(d_upper_ref), cudaFree(d_upper_adj), cudaFree(d_keys);
        cudaFree(slab), cudaFree(d_vis), cudaFree(d_touched), cudaFree(d_counters), cudaFree(d_in);
        d_rows = nullptr, d_adj0 = d_upper_ref = d_upper_adj = nullptr, d_keys = nullptr;
        slab = nullptr, d_vis = d_touched = nullptr, d_counters = nullptr, d_in = nullptr;
        if (ev0)
            cudaEventDestroy(ev0);
        if (ev1)
            cudaEventDestroy(ev1);
        ev0 = ev1 = nullptr;
    }

    PtrBlob export_ptr(void* p) const {
        PtrBlob b;
        memset(&b, 0, sizeof(b));
        b.raw = p;
        if (!local && p)
            LB_CUDA(cudaIpcGetMemHandle(&b.ipc, p));
        return b;
    }
    // a pointer of rank `src` usable on this rank's device; `keep` = stays mapped for the life of the group
    void* import_ptr(const PtrBlob& b, int src, bool keep) {
        if (!b.raw)
            return nullptr;
        if (local || src == rank)
            return b.raw;
        void* p = nullptr;
        LB_CUDA(cudaIpcOpenMemHandle(&p, b.ipc, cudaIpcMemLazyEnablePeerAccess));
        if (keep)
            opened.push_back(p);
        return p;
    }
    void release_ptr(void* p, int src) {
        if (!local && src != rank && p)
            LB_CUDA(cudaIpcCloseMemHandle(p));
    }

    // ---- distribute: phase A (root describes its index), B (everybody copies its share), C (map the peers' slabs) ----
    GroupConfigBlob describe(Index* idx) {
        GroupConfigBlob c;
        memset(&c, 0, sizeof(c));
        if (!idx)
            return c;
        idx->flush_staged();
        std::lock_guard<std::mutex> g(idx->mu_);
        if (idx->pending_n_)
            build_pending(*idx);
        if (idx->cfg_.pq)
            throw CudaError("group: pq indexes are not supported");
        if (idx->n_ == 0)
            throw CudaError("group: the index is empty");
        LB_CUDA(cudaDeviceSynchronize());
        c.valid = 1;
        c.metric_kind = idx->cfg_.metric_kind, c.scalar_kind = idx->cfg_.scalar_kind;
        c.dims = idx->cfg_.dims, c.M = idx->cfg_.M, c.M0 = idx->cfg_.M0, c.ef = idx->cfg_.ef;
        c.n = idx->n_, c.upper_lists = idx->upper_lists_, c.row_bytes = idx->row_bytes_, c.vec_bytes = idx->vec_bytes_;
        c.entry = idx->entry_, c.max_level = idx->max_level_;
        c.flags = idx->view().flags;
        { // contiguous row ranges (SURVEY 8e) of equal expected work
            unsigned long long* d_hist = nullptr;
            LB_CUDA(cudaMalloc(&d_hist, kBalanceBuckets * sizeof(unsigned long long)));
            LB_CUDA(cudaMemset(d_hist, 0, kBalanceBuckets * sizeof(unsigned long long)));
            indegree_hist_kernel<<<1024, 256>>>(idx->d_adj0_, (size_t)idx->n_ * idx->cfg_.M0, (uint32_t)idx->n_, d_hist);
            LB_CUDA(cudaGetLastError());
            count_launch();
            std::vector<unsigned long long> hist(kBalanceBuckets);
            LB_CUDA(cudaMemcpy(hist.data(), d_hist, hist.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
            LB_CUDA(cudaFree(d_hist));
            balanced_bounds(hist, idx->n_, world, c.bounds);
        }
        c.vectors = export_ptr(idx->d_vectors_), c.adj0 = export_ptr(idx->d_adj0_);
        c.upper_ref = export_ptr(idx->d_upper_ref_), c.upper_adj = export_ptr(idx->d_upper_adj_);
        c.keys = export_ptr(idx->d_keys_);
        return c;
    }

    // the graph's description, from the root's index (distribute) or from a file (load)
    void configure(const GroupConfigBlob& c) {
        cfg = IndexConfig();
        cfg.metric_kind = c.metric_kind, cfg.scalar_kind = c.scalar_kind;
        cfg.dims = c.dims, cfg.M = c.M, cfg.M0 = c.M0, cfg.ef = c.ef;
        dist_mode = distance_mode(cfg.metric_kind, cfg.scalar_kind);
        n = c.n, row_bytes = c.row_bytes, vec_bytes = c.vec_bytes, upper_lists = c.upper_lists;
        entry = c.entry, max_level = c.max_level, flags = c.flags;
        if (cfg.M0 > 256)
            throw CudaError("group: connectivity above 128 is not supported");
        for (int r = 0; r <= world; ++r)
            bounds[r] = c.bounds[r]; // contiguous row ranges (SURVEY 8e), sized for equal expected work
    }

    template <typename T> void device_alloc(T** p, size_t bytes, const char* what) {
        const cudaError_t e = cudaMalloc((void**)p, bytes);
        if (e == cudaSuccess)
            return;
        (void)cudaGetLastError();
        size_t free_b = 0, total_b = 0;
        if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess)
            (void)cudaGetLastError();
        throw CudaError("group: rank " + std::to_string(rank) + " (device " + std::to_string(device) + "): no room for its " + what +
                        ": " + std::to_string(bytes) + " bytes requested, " + std::to_string(free_b) + " free (" + cudaGetErrorString(e) + ")");
    }

    // Everything the rank keeps on its device, taken at once: no cudaMalloc may happen between the launches of a search (it
    // may wait for kernels already running on this device, and those kernels wait for the rank that is allocating).  On a
    // failure nothing stays allocated and the error names what did not fit: rows, graph, mailbox or scratch
    // (lb200_group_rank_info_t).
    void allocate(size_t max_batch_, size_t max_results, bool graph = true) {
        LB_CUDA(cudaSetDevice(device));
        int sms = 0;
        LB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
        cap = (uint32_t)cfg.M0;
        Wmax = (uint32_t)sms * 8u * kGroupWarps; // upper bound of resident warps (8 CTAs per SM)
        max_batch = max_batch_, res_cap = max_results;
        // owner slots: one per query a rank owns in the largest batch (never more than the resident warps)
        Omax = (uint32_t)std::min<size_t>(Wmax, round_up((max_batch + world - 1) / world, kGroupWarps));
        lay = slab_layout(Omax, (uint32_t)world, cap, res_cap, max_batch, row_bytes);
        words_per_slot = round_up((std::max(n, capacity) + 31) / 32, 32); // owner scratch: one visited bitmap per owned slot
        // staging of raw input queries for the host-buffer entry point
        in_bytes = max_batch * std::max<size_t>(row_bytes, cfg.dims * 4);
        const size_t lo = bounds[rank], hi = bounds[rank + 1], owned = Omax;
        try {
            if (graph) {
                device_alloc(&d_rows, std::max<size_t>((hi - lo) * row_bytes, 16), "rows");
                device_alloc(&d_adj0, n * cfg.M0 * 4, "graph (lists, keys)");
                device_alloc(&d_upper_ref, n * 4, "graph (lists, keys)");
                device_alloc(&d_upper_adj, std::max<size_t>(upper_lists * cfg.M * 4, 16), "graph (lists, keys)");
                device_alloc(&d_keys, n * 8, "graph (lists, keys)");
            }
            device_alloc(&slab, lay.total, "mailbox");
            device_alloc(&d_vis, owned * words_per_slot * 4, "scratch (visited bitmaps)");
            device_alloc(&d_touched, owned * (size_t)touched_cap * 4, "scratch (touched lists)");
            device_alloc(&d_counters, 16 * sizeof(unsigned long long), "scratch (counters)");
            device_alloc(&d_in, in_bytes, "scratch (query staging)");
            LB_CUDA(cudaMemset(slab, 0, lay.total));
            LB_CUDA(cudaMemset(d_vis, 0, owned * words_per_slot * 4));
            LB_CUDA(cudaMemset(d_counters, 0, 16 * sizeof(unsigned long long)));
            LB_CUDA(cudaEventCreate(&ev0));
            LB_CUDA(cudaEventCreate(&ev1));
        } catch (...) {
            release();
            throw;
        }
    }

    PtrBlob adopt(const GroupConfigBlob& c, int root, size_t max_batch_, size_t max_results) {
        if (!c.valid)
            throw CudaError("group: the root rank passed no index");
        LB_CUDA(cudaSetDevice(device));
        configure(c);
        allocate(max_batch_, max_results);
        const size_t lo = bounds[rank], hi = bounds[rank + 1];
        auto fetch = [&](void* dst, const PtrBlob& b, size_t offset, size_t bytes) {
            if (!bytes)
                return;
            uint8_t* src = (uint8_t*)import_ptr(b, root, false);
            LB_CUDA(cudaMemcpy(dst, src + offset, bytes, cudaMemcpyDefault));
            release_ptr(src, root);
        };
        fetch(d_rows, c.vectors, lo * row_bytes, (hi - lo) * row_bytes);
        fetch(d_adj0, c.adj0, 0, n * cfg.M0 * 4);
        fetch(d_upper_ref, c.upper_ref, 0, n * 4);
        fetch(d_upper_adj, c.upper_adj, 0, upper_lists * cfg.M * 4);
        fetch(d_keys, c.keys, 0, n * 8);
        LB_CUDA(cudaDeviceSynchronize());
        return export_ptr(slab);
    }

    // load: this rank's rows from the caller's file bytes, the graph from the parsed lists
    void fill_from_file(const ParsedIndexFile& f, const uint8_t* file, size_t stored_bytes) {
        LB_CUDA(cudaSetDevice(device));
        upload_file_rows(file, f.row_off, stored_bytes, bounds[rank], bounds[rank + 1], d_rows, row_bytes);
        LB_CUDA(cudaMemcpy(d_adj0, f.adj0.data(), f.adj0.size() * 4, cudaMemcpyHostToDevice));
        LB_CUDA(cudaMemcpy(d_upper_ref, f.upper_ref.data(), f.upper_ref.size() * 4, cudaMemcpyHostToDevice));
        if (!f.upper_adj.empty())
            LB_CUDA(cudaMemcpy(d_upper_adj, f.upper_adj.data(), f.upper_adj.size() * 4, cudaMemcpyHostToDevice));
        LB_CUDA(cudaMemcpy(d_keys, f.keys.data(), f.keys.size() * 8, cudaMemcpyHostToDevice));
        LB_CUDA(cudaDeviceSynchronize());
    }

    // a group's own index: search this rank's Index `x` (its row slice) with the graph state of the root's index.  The search
    // bounds are min(capacity split, n): trailing ranks may hold no rows yet.
    void attach(const Index& x, const Index& root) {
        d_rows = x.d_vectors_, d_adj0 = x.d_adj0_, d_upper_ref = x.d_upper_ref_, d_upper_adj = x.d_upper_adj_, d_keys = x.d_keys_;
        n = root.n_, upper_lists = root.upper_lists_, entry = root.entry_, max_level = root.max_level_;
        for (int r = 0; r <= world; ++r)
            bounds[r] = (uint32_t)std::min(capacity * (size_t)r / (size_t)world, n);
    }

    void map_peers(const PtrBlob* slabs) {
        LB_CUDA(cudaSetDevice(device));
        for (int r = 0; r < world; ++r)
            peer_slab[r] = (uint8_t*)import_ptr(slabs[r], r, true);
    }

    int occupancy_for(uint32_t L) {
        LB_CUDA(cudaSetDevice(device));
        const size_t smem = (size_t)group_warp_layout((uint32_t)row_bytes, group_ring_slots((uint32_t)row_bytes), L, cap).total * kGroupWarps;
        const int nq = pick_nq((uint32_t)row_bytes);
        if (nq < 0)
            throw CudaError("group: vectors wider than 8192 bytes are not supported");
        int occ = 0;
        dispatch_walk(dist_mode, cfg.scalar_kind, nq, [&](auto d, auto s, auto q) {
            occ = group_occupancy_one<decltype(d)::value, decltype(s)::value, decltype(q)::value>(smem);
        });
        int sms = 0;
        LB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
        return occ * sms * kGroupWarps;
    }

    uint8_t* qbuf() const { return slab + lay.qbuf; }

    // queries: only the root's are read.  Asynchronous on `stream`.
    void launch(const void* d_queries, size_t nq, size_t stride, int kind, size_t k, uint32_t L, uint32_t W, int root,
                uint64_t* d_out_keys, float* d_out_dists, uint32_t* d_out_counts, cudaStream_t stream) {
        LB_CUDA(cudaSetDevice(device));
        if (nq > max_batch || nq * k > res_cap)
            throw CudaError("group: batch larger than the group was created for (max_batch / max_results)");
        if (nq >= kGroupMaxBatch)
            throw CudaError("group: more than 4 M queries per batch");
        if (rank == root) {
            if (!d_queries)
                throw CudaError("group: the root rank must pass the queries");
            launch_cast_rows(d_queries, stride, kind, qbuf(), row_bytes, cfg.scalar_kind, cfg.dims, nq, stream);
        }
        ++epoch; // callers run renew_flags() first: (epoch & 0xFFF) is never 0 here
        GroupLaunch p;
        memset(&p, 0, sizeof(p));
        p.G = (uint32_t)world, p.me = (uint32_t)rank, p.W = W, p.cap = cap, p.ring_slots = group_ring_slots((uint32_t)row_bytes);
        p.nq = (uint32_t)nq, p.k = (uint32_t)k, p.L = L;
        p.flag_base = (epoch & 0xFFFu) << 20;
        p.epoch = epoch, p.root = (uint32_t)root;
        p.timeout_ns = group_timeout_ns();
        p.g.vectors = d_rows, p.g.adj0 = d_adj0, p.g.upper_ref = d_upper_ref, p.g.upper_adj = d_upper_adj, p.g.keys = d_keys;
        p.g.n = (uint32_t)n, p.g.row_bytes = (uint32_t)row_bytes, p.g.M = (uint32_t)cfg.M, p.g.M0 = (uint32_t)cfg.M0;
        p.g.entry = entry, p.g.max_level = max_level, p.g.flags = flags, p.g.dims = (uint32_t)cfg.dims;
        for (int r = 0; r <= world; ++r)
            p.bounds[r] = bounds[r];
        for (int r = world + 1; r <= kGroupMax; ++r)
            p.bounds[r] = 0xFFFFFFFFu;
        for (int r = 0; r < world; ++r) {
            uint8_t* s = peer_slab[r];
            p.req[r] = (unsigned long long*)(s + lay.req), p.resp[r] = (unsigned long long*)(s + lay.resp);
            p.reqq[r] = s + lay.reqq;
            p.res_keys[r] = (uint64_t*)(s + lay.res_keys), p.res_dists[r] = (float*)(s + lay.res_dists);
            p.res_counts[r] = (uint32_t*)(s + lay.res_counts);
            p.done[r] = (unsigned long long*)(s + lay.done), p.qready[r] = (unsigned long long*)(s + lay.qready);
            p.err[r] = (uint32_t*)(s + lay.err);
        }
        p.queries = peer_slab[root] + lay.qbuf, p.query_stride = (uint32_t)row_bytes;
        p.vis = d_vis, p.touched = d_touched, p.words_per_slot = words_per_slot, p.touched_cap = touched_cap;
        p.counters = d_counters;
        LB_CUDA(cudaMemsetAsync(d_counters, 0, 16 * sizeof(unsigned long long), stream));
        const size_t smem = (size_t)group_warp_layout((uint32_t)row_bytes, group_ring_slots((uint32_t)row_bytes), L, cap).total * kGroupWarps;
        uint32_t O = 0, H = 0;
        if (!group_plan(world, nq, W, Omax, O, H))
            throw CudaError("group: not enough resident warps for this batch's mailboxes");
        p.O = O, p.H = H, p.W = W;
        const uint32_t grid = (O + H) / kGroupWarps;
        const int nqc = pick_nq((uint32_t)row_bytes);
        LB_CUDA(cudaEventRecord(ev0, stream));
        dispatch_walk(dist_mode, cfg.scalar_kind, nqc, [&](auto d, auto s, auto q) {
            group_launch_one<decltype(d)::value, decltype(s)::value, decltype(q)::value>(p, grid, smem, stream);
        });
        LB_CUDA(cudaEventRecord(ev1, stream));
        if (d_out_keys || d_out_dists || d_out_counts) {
            const size_t total = std::max(nq * k, nq);
            group_copy_results_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(
                (const uint64_t*)(slab + lay.res_keys), (const float*)(slab + lay.res_dists), (const uint32_t*)(slab + lay.res_counts),
                d_out_keys, d_out_dists, d_out_counts, nq, k);
            LB_CUDA(cudaGetLastError());
            count_launch();
        }
        last_nq = (uint32_t)nq;
    }

    void check_error() {
        uint32_t e = 0;
        LB_CUDA(cudaMemcpy(&e, slab + lay.err, 4, cudaMemcpyDeviceToHost));
        if (e)
            throw CudaError("group: a rank timed out waiting for a peer (rank " + std::to_string(e - 1) + " gave up first)");
    }
};

// ---- the handle behind lb200_group_t: one rank of a multi-process group, or all ranks of a single-process one --------
struct Group {
    std::vector<GroupRank*> ranks; // 1 entry (multi-process) or `world` entries (single process)
    int world = 1, root = 0;
    lb200_allgather_fn ag = nullptr;
    void* ag_ctx = nullptr;
    bool distributed = false;
    std::mutex mu;
    std::vector<cudaStream_t> streams; // single-process: one per device
    // the group's own index (lb200_group_index_init): rank r's Index holds rows [capacity r / G, capacity (r+1) / G); index[0]
    // also keeps the levels, keys, level generator and batch schedule.  Never handed to the one-GPU entry points.
    std::vector<std::unique_ptr<Index>> index;
    ~Group() {
        drop_index();
        for (GroupRank* r : ranks)
            delete r;
        for (size_t i = 0; i < streams.size(); ++i)
            if (streams[i])
                cudaStreamDestroy(streams[i]);
    }
    bool local() const { return ranks.size() > 1 || world == 1; }
    void drop_index() { // (each on its own device; the ranks' borrowed pointers go with it)
        for (size_t i = 0; i < index.size(); ++i) {
            cudaSetDevice(ranks[i]->device);
            index[i].reset();
        }
        index.clear();
    }

    // every rank contributes `bytes`; everybody receives world * bytes
    void exchange(const std::vector<std::vector<uint8_t>>& mine, std::vector<uint8_t>& all, size_t bytes) {
        all.assign((size_t)world * bytes, 0);
        if (ranks.size() == (size_t)world) {
            for (int r = 0; r < world; ++r)
                memcpy(all.data() + (size_t)r * bytes, mine[r].data(), bytes);
        } else {
            ag(ag_ctx, mine[0].data(), all.data(), bytes);
        }
    }
};

static uint32_t agree_W(Group& G, uint32_t L) {
    GroupRank* r0 = G.ranks[0];
    auto it = r0->W_for_L.find(L);
    if (it != r0->W_for_L.end())
        return it->second;
    // every rank reports how many warps its device keeps resident for this beam width, and which physical device it is:
    // ranks that share a device (a 1-GPU box running the G-rank protocol) must be resident together and split its warps
    struct Offer {
        uint32_t w;
        char uuid[16];
    };
    std::vector<std::vector<uint8_t>> mine(G.ranks.size(), std::vector<uint8_t>(sizeof(Offer)));
    for (size_t i = 0; i < G.ranks.size(); ++i) {
        Offer o;
        o.w = (uint32_t)G.ranks[i]->occupancy_for(L);
        cudaDeviceProp prop;
        LB_CUDA(cudaGetDeviceProperties(&prop, G.ranks[i]->device));
        memcpy(o.uuid, prop.uuid.bytes, 16);
        memcpy(mine[i].data(), &o, sizeof(o));
    }
    std::vector<uint8_t> all;
    G.exchange(mine, all, sizeof(Offer));
    const Offer* offers = (const Offer*)all.data();
    uint32_t W = 0xFFFFFFFFu, share = 1;
    for (int r = 0; r < G.world; ++r) {
        W = std::min(W, offers[r].w);
        uint32_t same = 0;
        for (int t = 0; t < G.world; ++t)
            same += memcmp(offers[r].uuid, offers[t].uuid, 16) == 0;
        share = std::max(share, same);
    }
    W = std::min(W, r0->Wmax);
    W /= share;
    W -= W % (uint32_t)(G.world * kGroupWarps); // whole CTAs, and a slot keeps its owner across waves
    if (W == 0)
        throw CudaError("group: the search kernel does not fit on an SM (ef too large for shared memory)");
    for (GroupRank* r : G.ranks)
        r->W_for_L[L] = W;
    return W;
}

void group_distribute(Group& G, Index* root_index, int root, size_t max_batch, size_t max_results) {
    DeviceGuard dg;
    std::lock_guard<std::mutex> lk(G.mu);
    if (G.distributed)
        throw CudaError("group: already distributed");
    if (root < 0 || root >= G.world)
        throw CudaError("group: bad root rank");
    const size_t nr = G.ranks.size();
    // A: the root describes its index
    std::vector<std::vector<uint8_t>> mine(nr, std::vector<uint8_t>(sizeof(GroupConfigBlob)));
    for (size_t i = 0; i < nr; ++i) {
        GroupRank* r = G.ranks[i];
        LB_CUDA(cudaSetDevice(r->device));
        GroupConfigBlob c = r->describe(r->rank == root ? root_index : nullptr);
        memcpy(mine[i].data(), &c, sizeof(c));
    }
    std::vector<uint8_t> all;
    G.exchange(mine, all, sizeof(GroupConfigBlob));
    GroupConfigBlob cfg;
    memcpy(&cfg, all.data() + (size_t)root * sizeof(GroupConfigBlob), sizeof(cfg));
    // B: every rank copies its row range and the graph from the root, allocates its mailboxes
    std::vector<std::vector<uint8_t>> slabs(nr, std::vector<uint8_t>(sizeof(PtrBlob)));
    try {
        for (size_t i = 0; i < nr; ++i) {
            PtrBlob b = G.ranks[i]->adopt(cfg, root, max_batch, max_results);
            memcpy(slabs[i].data(), &b, sizeof(b));
        }
    } catch (...) {
        for (GroupRank* r : G.ranks)
            r->release();
        throw;
    }
    G.exchange(slabs, all, sizeof(PtrBlob)); // also tells the root that everybody is done reading its index
    // C: map the peers' mailboxes
    for (size_t i = 0; i < nr; ++i)
        G.ranks[i]->map_peers((const PtrBlob*)all.data());
    std::vector<std::vector<uint8_t>> tick(nr, std::vector<uint8_t>(4, 0));
    G.exchange(tick, all, 4); // nobody searches before everybody has mapped everybody
    G.root = root;
    G.distributed = true;
}

// What every rank of a load reports before anything is allocated: whether its file parsed, and what it holds
struct GroupFileBlob {
    uint32_t ok;
    uint8_t header[136];
    uint64_t n, checksum;
    char error[256];
};
// What every rank reports after allocating and filling its share: its mailbox slab, or why it could not
struct GroupSlabBlob {
    PtrBlob slab;
    uint32_t ok;
    char error[256];
};

// keys, levels and lists of a parsed file: two ranks that hold different files with equal headers still disagree here
static uint64_t graph_checksum(const ParsedIndexFile& f) {
    uint64_t h = 1469598103934665603ull;
    auto mix = [&h](uint64_t v) { h = (h ^ v) * 1099511628211ull; };
    for (size_t i = 0; i < f.n; ++i)
        mix(f.keys[i]), mix((uint64_t)(uint16_t)f.levels[i]);
    for (uint32_t v : f.adj0)
        mix(v);
    for (uint32_t v : f.upper_adj)
        mix(v);
    return h;
}

void group_load(Group& G, const IndexConfig& cfg, const void* buffer, size_t length, int root, size_t max_batch,
                size_t max_results) {
    DeviceGuard dg;
    std::lock_guard<std::mutex> lk(G.mu);
    if (G.distributed)
        throw CudaError("group: already distributed");
    if (root < 0 || root >= G.world)
        throw CudaError("group: bad root rank");
    const size_t nr = G.ranks.size();
    const bool one_process = nr == (size_t)G.world;
    const size_t vec_bytes = scalar_row_bytes(cfg.scalar_kind, cfg.dims);
    // A: parse and check the file (once per process) before anything is allocated; then make sure every rank holds the same one
    ParsedIndexFile f;
    GroupFileBlob mine;
    memset(&mine, 0, sizeof(mine));
    try {
        parse_index_file(cfg, vec_bytes, vec_bytes, buffer, length, f);
        if (f.n == 0)
            throw CudaError("group: the index is empty");
        mine.ok = 1;
        memcpy(mine.header, buffer, 136);
        mine.n = f.n, mine.checksum = graph_checksum(f);
    } catch (const std::exception& e) {
        if (one_process)
            throw; // (nobody else to tell)
        snprintf(mine.error, sizeof(mine.error), "%s", e.what());
    }
    std::vector<std::vector<uint8_t>> blobs(nr, std::vector<uint8_t>(sizeof(GroupFileBlob)));
    for (size_t i = 0; i < nr; ++i)
        memcpy(blobs[i].data(), &mine, sizeof(mine));
    std::vector<uint8_t> all;
    G.exchange(blobs, all, sizeof(GroupFileBlob));
    if (!mine.ok)
        throw CudaError(mine.error);
    for (int r = 0; r < G.world; ++r) {
        GroupFileBlob o;
        memcpy(&o, all.data() + (size_t)r * sizeof(GroupFileBlob), sizeof(o));
        if (!o.ok)
            throw CudaError("group: rank " + std::to_string(r) + " could not load its index file: " + o.error);
        if (memcmp(o.header, mine.header, 136) != 0 || o.n != mine.n || o.checksum != mine.checksum)
            throw CudaError("group: the ranks passed different index files (rank " + std::to_string(r) + " differs from rank " +
                            std::to_string(G.ranks[0]->rank) + ")");
    }
    // the description an index with these options would give (GroupRank::describe)
    GroupConfigBlob c;
    memset(&c, 0, sizeof(c));
    c.valid = 1;
    c.metric_kind = cfg.metric_kind, c.scalar_kind = cfg.scalar_kind;
    c.dims = cfg.dims, c.M = cfg.M, c.M0 = cfg.M0, c.ef = cfg.ef;
    c.n = f.n, c.upper_lists = f.upper_adj.size() / cfg.M, c.row_bytes = stored_row_bytes(cfg), c.vec_bytes = vec_bytes;
    c.entry = f.entry, c.max_level = f.max_level;
    c.flags = search_view_flags();
    balanced_bounds(host_indegree_hist(f.adj0, f.n), f.n, G.world, c.bounds);
    // B: every rank allocates and fills its share; the mailbox exchange also carries whether that worked
    std::vector<std::vector<uint8_t>> slabs(nr, std::vector<uint8_t>(sizeof(GroupSlabBlob), 0));
    for (size_t i = 0; i < nr; ++i) {
        GroupRank* r = G.ranks[i];
        GroupSlabBlob b;
        memset(&b, 0, sizeof(b));
        try {
            LB_CUDA(cudaSetDevice(r->device));
            r->configure(c);
            r->allocate(max_batch, max_results);
            r->fill_from_file(f, (const uint8_t*)buffer, vec_bytes);
            b.slab = r->export_ptr(r->slab);
            b.ok = 1;
        } catch (const std::exception& e) {
            snprintf(b.error, sizeof(b.error), "%s", e.what());
        }
        memcpy(slabs[i].data(), &b, sizeof(b));
        if (!b.ok)
            break; // (the ranks after it report neither success nor a reason)
    }
    G.exchange(slabs, all, sizeof(GroupSlabBlob));
    std::vector<PtrBlob> peers(G.world);
    for (int r = 0; r < G.world; ++r) {
        GroupSlabBlob b;
        memcpy(&b, all.data() + (size_t)r * sizeof(GroupSlabBlob), sizeof(b));
        if (!b.ok) {
            for (GroupRank* x : G.ranks)
                x->release();
            throw CudaError(b.error[0] ? std::string(b.error) : "group: rank " + std::to_string(r) + " could not take its share");
        }
        peers[r] = b.slab;
    }
    // C: map the peers' mailboxes
    for (size_t i = 0; i < nr; ++i)
        G.ranks[i]->map_peers(peers.data());
    std::vector<std::vector<uint8_t>> tick(nr, std::vector<uint8_t>(4, 0));
    G.exchange(tick, all, 4); // nobody searches before everybody has mapped everybody
    G.root = root;
    G.distributed = true;
}

void group_rank_info(Group& G, int which, lb200_group_rank_info_t& out) {
    std::lock_guard<std::mutex> lk(G.mu);
    if (which < 0 || (size_t)which >= G.ranks.size())
        throw CudaError("group: no such local rank");
    if (!G.distributed)
        throw CudaError("group: lb200_group_distribute or lb200_group_load has not been called");
    G.ranks[which]->footprint(out);
}

// A temporary copy of `root` on the current device for a group build: the root's config, codebook and PQ tables, its rows
// [0, n0 + P), lists of nodes [0, n0), level-1+ lists and keys.  No search-screen companion: the build never reads it.
static std::unique_ptr<Index> build_replica(Index& root) {
    const IndexConfig& cfg = root.cfg_;
    std::vector<float> codebook;
    if (cfg.pq) {
        codebook.resize(cfg.num_centroids * cfg.dims);
        LB_CUDA(cudaMemcpy(codebook.data(), root.d_codebook_, codebook.size() * sizeof(float), cudaMemcpyDeviceToHost));
    }
    std::unique_ptr<Index> x(new Index(cfg, codebook.data()));
    x->sq_bytes_ = 0, x->sq_on_ = false;
    x->ensure_capacity(root.capacity_);
    x->alloc_upper(root.upper_lists_);
    const size_t n0 = root.n_, P = root.pending_n_;
    auto copy = [](void* dst, const void* src, size_t bytes) {
        if (bytes)
            LB_CUDA(cudaMemcpy(dst, src, bytes, cudaMemcpyDefault));
    };
    copy(x->d_vectors_, root.d_vectors_, (n0 + P) * root.row_bytes_);
    copy(x->d_adj0_, root.d_adj0_, n0 * cfg.M0 * sizeof(uint32_t));
    copy(x->d_upper_ref_, root.d_upper_ref_, n0 * sizeof(uint32_t));
    copy(x->d_upper_adj_, root.d_upper_adj_, root.upper_lists_ * cfg.M * sizeof(uint32_t));
    copy(x->d_keys_, root.d_keys_, n0 * sizeof(uint64_t));
    if (cfg.pq) { // the pair tables as the root computed them, and the raw pending rows (the value side of build distances)
        copy(x->d_pq_pair_, root.d_pq_pair_, cfg.num_subvectors * cfg.num_centroids * cfg.num_centroids * sizeof(float));
        copy(x->d_pq_norm_, root.d_pq_norm_, cfg.num_subvectors * cfg.num_centroids * sizeof(float));
        const size_t raw = P * round_up(cfg.dims * 4, 16);
        LB_CUDA(cudaMalloc(&x->d_pending_raw_, raw));
        x->pending_raw_cap_ = raw;
        copy(x->d_pending_raw_, root.d_pending_raw_, raw);
        x->pq_max_code_ = root.pq_max_code_;
    }
    x->n_ = n0, x->upper_lists_ = root.upper_lists_, x->max_level_ = root.max_level_, x->entry_ = root.entry_;
    LB_CUDA(cudaDeviceSynchronize());
    return x;
}

void group_build(Group& G, Index* root_index, int root) {
    DeviceGuard dg;
    std::lock_guard<std::mutex> lk(G.mu);
    // per-batch barriers between processes are not implemented: a world-1 group of lb200_group_create holds its only rank
    if (G.ranks.size() != (size_t)G.world)
        throw CudaError("group build: a multi-process group cannot build; create the group with lb200_group_create_local");
    if (root < 0 || root >= G.world)
        throw CudaError("group: bad root rank");
    if (!root_index)
        throw CudaError("null index handle");
    Index& idx = *root_index;
    const int dev = G.ranks[root]->device;
    cudaPointerAttributes at;
    LB_CUDA(cudaPointerGetAttributes(&at, idx.scratch_.counters));
    if (at.device != dev)
        throw CudaError("group build: the index does not live on the root rank's device");
    LB_CUDA(cudaSetDevice(dev));
    idx.flush_staged();
    std::lock_guard<std::mutex> g(idx.mu_);
    if (!idx.pending_n_)
        return;
    LB_CUDA(cudaDeviceSynchronize()); // the pending rows are written on the legacy stream
    std::vector<std::unique_ptr<Index>> owned(G.world);
    std::vector<BuildReplica> ranks(G.world);
    try {
        for (int r = 0; r < G.world; ++r) {
            ranks[r].device = G.ranks[r]->device;
            if (r == root) {
                ranks[r].idx = &idx;
                continue;
            }
            LB_CUDA(cudaSetDevice(ranks[r].device));
            owned[r] = build_replica(idx);
            ranks[r].idx = owned[r].get();
        }
        build_pending_group(idx, ranks, root);
    } catch (...) {
        for (int r = 0; r < G.world; ++r) {
            cudaSetDevice(ranks[r].device);
            owned[r].reset();
        }
        throw;
    }
    for (int r = 0; r < G.world; ++r) {
        LB_CUDA(cudaSetDevice(ranks[r].device));
        owned[r].reset();
    }
}

// ---- the group's own index (lb200_group_index_*, DESIGN.md 4.2): built straight into the row-sharded layout ---------------

static void require_own_index(Group& G) {
    if (G.index.empty())
        throw CudaError("group index: lb200_group_index_init (or lb200_group_index_load) has not been called on this group");
}

static std::vector<BuildReplica> index_shards(Group& G) {
    std::vector<BuildReplica> s(G.index.size());
    for (size_t r = 0; r < s.size(); ++r)
        s[r] = BuildReplica{G.index[r].get(), G.ranks[r]->device};
    return s;
}

// the refusals every way of giving a group an index of its own shares; caller holds G.mu
static void check_own_index_formation(Group& G, const IndexConfig& cfg) {
    if (G.ranks.size() != (size_t)G.world)
        throw CudaError("group index: a multi-process group cannot hold an index of its own; create the group with "
                        "lb200_group_create_local");
    if (G.distributed)
        throw CudaError("group index: the group already holds a graph (one lb200_group_distribute, lb200_group_load or "
                        "lb200_group_index_init per group)");
    if (cfg.pq)
        throw CudaError("group index: pq indexes are not supported");
}

// An index of `capacity` rows of the group's own: empty, or holding a parsed file `f` (whose node i's bytes are at
// file + f->row_off[i]).  Rank r's index gets the rows of [capacity r / G, capacity (r+1) / G) only -- copied from the file
// bytes through upload_file_rows' bounded pinned block -- and the lists, upper lists and keys of the whole graph; rank 0 also
// keeps the levels and keys on the host.  On a failure nothing stays allocated.  Caller holds G.mu.
static void form_own_index(Group& G, const IndexConfig& cfg, size_t capacity, size_t max_batch, size_t max_results,
                           ParsedIndexFile* f, const uint8_t* file) {
    const size_t W = (size_t)G.world;
    try {
        for (size_t r = 0; r < W; ++r) {
            LB_CUDA(cudaSetDevice(G.ranks[r]->device));
            G.index.emplace_back(new Index(cfg, nullptr));
            G.index[r]->init_row_range(capacity, capacity * r / W, capacity * (r + 1) / W);
        }
        for (size_t r = W; f && r-- > 0;) { // (rank 0 last: its commit moves the host levels and keys out of `f`)
            Index& x = *G.index[r];
            LB_CUDA(cudaSetDevice(G.ranks[r]->device));
            x.commit_file_graph(*f, r == 0);
            LB_CUDA(cudaDeviceSynchronize()); // (init_row_range's zero fill ran on the legacy stream; the upload has its own)
            upload_file_rows(file, f->row_off, x.stored_bytes_, x.row_lo_, std::min(x.row_hi_, f->n), x.d_vectors_, x.row_bytes_);
            LB_CUDA(cudaDeviceSynchronize());
        }
        for (size_t r = 0; r < W; ++r) {
            GroupRank* gr = G.ranks[r];
            LB_CUDA(cudaSetDevice(gr->device));
            const size_t lo = G.index[r]->row_lo_, hi = G.index[r]->row_hi_;
            gr->cfg = cfg;
            gr->dist_mode = distance_mode(cfg.metric_kind, cfg.scalar_kind);
            gr->row_bytes = G.index[r]->row_bytes_, gr->vec_bytes = G.index[r]->vec_bytes_;
            gr->flags = search_view_flags();
            if (cfg.M0 > 256)
                throw CudaError("group: connectivity above 128 is not supported");
            gr->borrowed = true, gr->capacity = capacity, gr->cap_lo = lo, gr->cap_hi = hi;
            gr->attach(*G.index[r], *G.index[0]);
            gr->allocate(max_batch, max_results, /*graph=*/false); // mailboxes and owner bitmaps sized for `capacity` rows
        }
        std::vector<PtrBlob> slabs(W);
        for (size_t r = 0; r < W; ++r)
            slabs[r] = G.ranks[r]->export_ptr(G.ranks[r]->slab);
        for (size_t r = 0; r < W; ++r)
            G.ranks[r]->map_peers(slabs.data());
    } catch (...) {
        for (GroupRank* r : G.ranks) {
            r->release();
            r->borrowed = false, r->capacity = 0;
            r->d_rows = nullptr, r->d_adj0 = r->d_upper_ref = r->d_upper_adj = nullptr, r->d_keys = nullptr;
        }
        G.drop_index();
        throw;
    }
    G.root = 0;
    G.distributed = true;
}

void group_index_init(Group& G, const IndexConfig& cfg, size_t capacity, size_t max_batch, size_t max_results) {
    DeviceGuard dg;
    std::lock_guard<std::mutex> lk(G.mu);
    check_own_index_formation(G, cfg);
    if (capacity == 0 || capacity >= 0x7FFFFFFFull)
        throw CudaError("group index: capacity must be in [1, 2^31 - 1)");
    form_own_index(G, cfg, capacity, max_batch, max_results, nullptr, nullptr);
}

void group_index_load(Group& G, const IndexConfig& cfg, const void* buffer, size_t length, size_t capacity, size_t max_batch,
                      size_t max_results) {
    DeviceGuard dg;
    std::lock_guard<std::mutex> lk(G.mu);
    check_own_index_formation(G, cfg);
    // the whole file is parsed and checked, as Index::load_buffer checks it, before any rank allocates
    const size_t vec_bytes = scalar_row_bytes(cfg.scalar_kind, cfg.dims);
    ParsedIndexFile f;
    parse_index_file(cfg, vec_bytes, vec_bytes, buffer, length, f);
    if (capacity == 0)
        capacity = f.n;
    if (capacity < std::max<size_t>(f.n, 1) || capacity >= 0x7FFFFFFFull)
        throw CudaError("group index: capacity must be in [max(1, rows in the file), 2^31 - 1); the file holds " +
                        std::to_string(f.n) + " rows");
    form_own_index(G, cfg, capacity, max_batch, max_results, &f, (const uint8_t*)buffer);
}

// Raises the capacity of the group's own index to `capacity`: rank r's range becomes [capacity r / G, capacity (r+1) / G)
// and rows [0, n + pending) move into the new row arrays of the ranks that now hold them, one copy-engine copy per (old rank,
// new rank) overlap.  Every new array of every rank is allocated before any row moves; on a failure they are all freed and
// the index is left as it was.  While the call runs a rank holds its old and new rows and two copies of its level-0 lists,
// upper references and keys.  The mailbox slab does not depend on the capacity (slab_layout takes M0), so the peers' mappings
// stay; the owner bitmaps (words_per_slot) do, and are replaced.
void group_index_reserve(Group& G, size_t capacity) {
    DeviceGuard dg;
    std::lock_guard<std::mutex> lk(G.mu);
    require_own_index(G);
    Index& root = *G.index[0];
    if (capacity <= root.capacity_)
        return; // as lb200_reserve
    if (capacity >= 0x7FFFFFFFull)
        throw CudaError("group index: capacity must be in [1, 2^31 - 1)");
    const size_t W = G.index.size(), n = root.n_, used = root.n_ + root.pending_n_, M0 = root.cfg_.M0, rb = root.row_bytes_;
    struct Fresh { // one rank's new arrays until they are handed over
        int device = 0;
        uint8_t* rows = nullptr;
        uint32_t *adj0 = nullptr, *upper_ref = nullptr, *vis = nullptr;
        uint64_t* keys = nullptr;
        cudaStream_t stream = nullptr;
        size_t lo = 0, hi = 0, words_per_slot = 0;
    };
    struct FreshAll {
        std::vector<Fresh> f;
        bool handed_over = false;
        ~FreshAll() {
            for (Fresh& x : f) {
                cudaSetDevice(x.device);
                if (x.stream)
                    cudaStreamSynchronize(x.stream), cudaStreamDestroy(x.stream);
                if (!handed_over)
                    cudaFree(x.rows), cudaFree(x.adj0), cudaFree(x.upper_ref), cudaFree(x.keys), cudaFree(x.vis);
            }
        }
    } fresh;
    fresh.f.resize(W);
    // every allocation first, named by rank, device and what it holds
    for (size_t r = 0; r < W; ++r) {
        GroupRank& gr = *G.ranks[r];
        Fresh& x = fresh.f[r];
        x.device = gr.device;
        x.lo = capacity * r / W, x.hi = capacity * (r + 1) / W;
        x.words_per_slot = round_up((capacity + 31) / 32, 32);
        LB_CUDA(cudaSetDevice(gr.device));
        gr.device_alloc(&x.rows, std::max<size_t>((x.hi - x.lo) * rb, 16), "rows");
        gr.device_alloc(&x.adj0, capacity * M0 * 4, "graph (lists, keys)");
        gr.device_alloc(&x.upper_ref, capacity * 4, "graph (lists, keys)");
        gr.device_alloc(&x.keys, capacity * 8, "graph (lists, keys)");
        gr.device_alloc(&x.vis, (size_t)gr.Omax * x.words_per_slot * 4, "scratch (visited bitmaps)");
        LB_CUDA(cudaStreamCreateWithFlags(&x.stream, cudaStreamNonBlocking));
    }
    for (size_t r = 0; r < W; ++r) { // (earlier work on the old arrays may still be queued on the legacy stream)
        LB_CUDA(cudaSetDevice(fresh.f[r].device));
        LB_CUDA(cudaDeviceSynchronize());
    }
    // the graph arrays grow as grow_device grows them (0xFF beyond the built nodes); rows beyond n + pending are zero, as
    // init_row_range leaves them
    for (size_t r = 0; r < W; ++r) {
        Index& old = *G.index[r];
        Fresh& x = fresh.f[r];
        LB_CUDA(cudaSetDevice(x.device));
        LB_CUDA(cudaMemsetAsync(x.rows, 0, std::max<size_t>((x.hi - x.lo) * rb, 16), x.stream));
        LB_CUDA(cudaMemsetAsync(x.adj0, 0xFF, capacity * M0 * 4, x.stream));
        LB_CUDA(cudaMemsetAsync(x.upper_ref, 0xFF, capacity * 4, x.stream));
        LB_CUDA(cudaMemsetAsync(x.keys, 0xFF, capacity * 8, x.stream));
        LB_CUDA(cudaMemsetAsync(x.vis, 0, (size_t)G.ranks[r]->Omax * x.words_per_slot * 4, x.stream));
        if (n) {
            LB_CUDA(cudaMemcpyAsync(x.adj0, old.d_adj0_, n * M0 * 4, cudaMemcpyDeviceToDevice, x.stream));
            LB_CUDA(cudaMemcpyAsync(x.upper_ref, old.d_upper_ref_, n * 4, cudaMemcpyDeviceToDevice, x.stream));
            LB_CUDA(cudaMemcpyAsync(x.keys, old.d_keys_, n * 8, cudaMemcpyDeviceToDevice, x.stream));
        }
    }
    // rows [0, used): one peer copy per (old rank s, new rank t) overlap, on the receiving rank's stream (after its memset)
    for (size_t t = 0; t < W; ++t) {
        Fresh& x = fresh.f[t];
        LB_CUDA(cudaSetDevice(x.device));
        for (size_t s = 0; s < W; ++s) {
            const Index& old = *G.index[s];
            const size_t a = std::max(old.row_lo_, x.lo), b = std::min(std::min(old.row_hi_, x.hi), used);
            if (a < b)
                LB_CUDA(cudaMemcpyPeerAsync(x.rows + (a - x.lo) * rb, x.device, old.d_vectors_ + (a - old.row_lo_) * rb,
                                            G.ranks[s]->device, (b - a) * rb, x.stream));
        }
    }
    for (size_t r = 0; r < W; ++r) {
        LB_CUDA(cudaSetDevice(fresh.f[r].device));
        LB_CUDA(cudaStreamSynchronize(fresh.f[r].stream));
    }
    // hand over: nothing below allocates or throws
    fresh.handed_over = true;
    for (size_t r = 0; r < W; ++r) {
        GroupRank& gr = *G.ranks[r];
        Fresh& x = fresh.f[r];
        cudaSetDevice(x.device);
        G.index[r]->replace_row_range(capacity, x.lo, x.hi, x.rows, x.adj0, x.upper_ref, x.keys);
        cudaFree(gr.d_vis);
        gr.d_vis = x.vis, gr.words_per_slot = x.words_per_slot;
        gr.capacity = capacity, gr.cap_lo = x.lo, gr.cap_hi = x.hi;
    }
    for (size_t r = 0; r < W; ++r)
        G.ranks[r]->attach(*G.index[r], root);
}

// Host rows [0, n) (input kind f32 or b1, `stride` apart) -> rows [first, first + n) of the group's index: each row goes only to
// the rank whose range holds it, cast to the storage kind there.  Rows travel through a bounded pinned block (two halves, as in
// upload_file_rows) and a device block of the same size.
static void upload_input_rows(Group& G, const uint8_t* vectors, size_t n, size_t stride, int kind, size_t first) {
    const Index& root = *G.index[0];
    const size_t in_bytes = scalar_row_bytes(kind, root.cfg_.dims), row_bytes = root.row_bytes_;
    for (size_t r = 0; r < G.index.size(); ++r) {
        Index& x = *G.index[r];
        const size_t a = std::max(first, x.row_lo_), b = std::min(first + n, x.row_hi_);
        if (a >= b)
            continue;
        LB_CUDA(cudaSetDevice(G.ranks[r]->device));
        struct Staging {
            uint8_t* pinned = nullptr;
            void* raw = nullptr;
            cudaStream_t stream = nullptr;
            cudaEvent_t done[2] = {nullptr, nullptr};
            ~Staging() {
                if (stream)
                    cudaStreamSynchronize(stream), cudaStreamDestroy(stream);
                for (cudaEvent_t e : done)
                    if (e)
                        cudaEventDestroy(e);
                cudaFreeHost(pinned), cudaFree(raw);
            }
        } st;
        const size_t block = std::max<size_t>(1, std::min(b - a, ((size_t)16 << 20) / in_bytes)); // rows per half (<= 16 MB)
        LB_CUDA(cudaMallocHost(&st.pinned, 2 * block * in_bytes));
        LB_CUDA(cudaMalloc(&st.raw, 2 * block * in_bytes));
        LB_CUDA(cudaStreamCreateWithFlags(&st.stream, cudaStreamNonBlocking));
        LB_CUDA(cudaEventCreateWithFlags(&st.done[0], cudaEventDisableTiming));
        LB_CUDA(cudaEventCreateWithFlags(&st.done[1], cudaEventDisableTiming));
        bool used[2] = {false, false};
        int h = 0;
        for (size_t b0 = a; b0 < b; b0 += block, h ^= 1) {
            const size_t cnt = std::min(block, b - b0);
            uint8_t* stage = st.pinned + (size_t)h * block * in_bytes;
            uint8_t* raw = (uint8_t*)st.raw + (size_t)h * block * in_bytes;
            if (used[h])
                LB_CUDA(cudaEventSynchronize(st.done[h]));
            for (size_t i = 0; i < cnt; ++i)
                memcpy(stage + i * in_bytes, vectors + (b0 - first + i) * stride, in_bytes);
            LB_CUDA(cudaMemcpyAsync(raw, stage, cnt * in_bytes, cudaMemcpyHostToDevice, st.stream));
            launch_cast_rows(raw, in_bytes, kind, x.d_vectors_ + (b0 - x.row_lo_) * row_bytes, row_bytes, root.cfg_.scalar_kind,
                             root.cfg_.dims, cnt, st.stream);
            LB_CUDA(cudaEventRecord(st.done[h], st.stream));
            used[h] = true;
        }
        LB_CUDA(cudaStreamSynchronize(st.stream));
    }
}

void group_index_add(Group& G, const uint64_t* keys, const void* vectors, size_t n, size_t stride, int kind) {
    DeviceGuard dg;
    std::lock_guard<std::mutex> lk(G.mu);
    require_own_index(G);
    Index& root = *G.index[0];
    if (!(kind == SK_F32 || (kind == SK_B1 && root.cfg_.scalar_kind == SK_B1)))
        throw CudaError("vectors must be passed as f32, or as packed bits (b1) for a b1 index");
    if (!n)
        return;
    if (!keys || !vectors)
        throw CudaError("null keys or vectors");
    for (size_t i = 0; i < n; ++i)
        if (keys[i] == ~0ull)
            throw CudaError("key UINT64_MAX is reserved (free key)");
    const size_t used = root.n_ + root.pending_n_;
    if (used + n > root.capacity_)
        throw CudaError("group index: " + std::to_string(n) + " more rows would pass the capacity of " + std::to_string(root.capacity_) +
                        " rows (" + std::to_string(used) + " held; lb200_group_index_reserve raises it); nothing was added");
    upload_input_rows(G, (const uint8_t*)vectors, n, stride, kind, used);
    root.h_keys_.insert(root.h_keys_.end(), keys, keys + n);
    root.pending_n_ += n;
}

// Inserts every pending row with all ranks, then points the search at the new graph.  Caller holds G.mu.
static void group_index_build_locked(Group& G) {
    Index& root = *G.index[0];
    if (!root.pending_n_)
        return;
    std::vector<BuildReplica> shards = index_shards(G);
    auto settle = [&] { // every rank's view of the graph state (the build updates the root's), scratch freed, search re-attached
        for (size_t r = 0; r < shards.size(); ++r) {
            Index& x = *shards[r].idx;
            cudaSetDevice(shards[r].device);
            x.n_ = root.n_, x.max_level_ = root.max_level_, x.entry_ = root.entry_, x.upper_lists_ = root.upper_lists_;
            x.free_scratch();
            G.ranks[r]->attach(x, root);
        }
    };
    try {
        LB_CUDA(cudaSetDevice(shards[0].device));
        build_pending_group(root, shards, 0);
    } catch (...) {
        settle();
        throw;
    }
    settle();
}

void group_index_build(Group& G) {
    DeviceGuard dg;
    std::lock_guard<std::mutex> lk(G.mu);
    require_own_index(G);
    group_index_build_locked(G);
}

void group_index_set_option(Group& G, const std::string& name, size_t value) {
    std::lock_guard<std::mutex> lk(G.mu);
    require_own_index(G);
    Index& root = *G.index[0];
    if (name == "build_batch")
        root.build_batch_ = value;
    else if (name == "build_ratio")
        root.build_ratio_ = value ? value : 1;
    else
        throw CudaError("group index: unknown option (build_batch and build_ratio are available)");
}

size_t group_index_size(Group& G) {
    std::lock_guard<std::mutex> lk(G.mu);
    require_own_index(G);
    return G.index[0]->size();
}

void group_index_build_stats(Group& G, size_t& vectors, uint64_t& distances, double& ms, size_t& value_bytes) {
    std::lock_guard<std::mutex> lk(G.mu);
    require_own_index(G);
    const Index& root = *G.index[0];
    vectors = root.last_build_n_, distances = root.last_build_dist_, ms = root.last_build_ms_, value_bytes = root.vec_bytes_;
}

size_t group_index_serialized_length(Group& G) {
    DeviceGuard dg;
    std::lock_guard<std::mutex> lk(G.mu);
    require_own_index(G);
    group_index_build_locked(G);
    return G.index[0]->serialized_length_locked();
}

void group_index_save(Group& G, const std::function<void(size_t)>& length_ok, const std::function<void(const void*, size_t)>& write) {
    DeviceGuard dg;
    std::lock_guard<std::mutex> lk(G.mu);
    require_own_index(G);
    group_index_build_locked(G);
    length_ok(G.index[0]->serialized_length_locked());
    save_row_sharded(*G.index[0], index_shards(G), write);
}

// Message flags are (epoch mod 4096) << 20 | sequence number.  Before the 12-bit part wraps, every rank waits for its last
// launch (which ends only when all ranks have finished theirs), all ranks meet, clear their mailboxes and meet again:
// a word written 4096 launches ago can then never be mistaken for a fresh one.  Collective; costs two exchanges per 4095
// searches.
static void renew_flags(Group& G, const std::vector<cudaStream_t>& streams) {
    GroupRank* r0 = G.ranks[0];
    if (((r0->epoch + 1) & 0xFFFu) != 0u)
        return;
    std::vector<std::vector<uint8_t>> tick(G.ranks.size(), std::vector<uint8_t>(4, 0));
    std::vector<uint8_t> all;
    for (size_t i = 0; i < G.ranks.size(); ++i) {
        LB_CUDA(cudaSetDevice(G.ranks[i]->device));
        LB_CUDA(cudaStreamSynchronize(streams[i]));
    }
    G.exchange(tick, all, 4);
    for (GroupRank* r : G.ranks) {
        LB_CUDA(cudaSetDevice(r->device));
        LB_CUDA(cudaMemset(r->slab + r->lay.req, 0, r->lay.reqq - r->lay.req)); // request + response mailboxes
        LB_CUDA(cudaDeviceSynchronize());
        r->epoch += 1; // skip the value whose 12-bit part is 0 (flag 0 means "never written")
    }
    G.exchange(tick, all, 4);
}

static uint32_t beam_width(const GroupRank& r, size_t k, size_t ef) {
    size_t L = ef ? ef : r.cfg.ef;
    if (L < k)
        L = k; // index.hpp:2706
    if (L > 4096)
        throw CudaError("search: max(ef, count) > 4096 is not supported");
    return (uint32_t)L;
}

void group_search_device(Group& G, const void* d_queries, size_t nq, size_t stride, int kind, size_t k, size_t ef,
                         uint64_t* d_keys, float* d_dists, uint32_t* d_counts, cudaStream_t stream) {
    DeviceGuard dg;
    std::lock_guard<std::mutex> lk(G.mu);
    if (!G.distributed)
        throw CudaError("group: lb200_group_distribute has not been called");
    if (G.ranks.size() != 1)
        throw CudaError("group: device-buffer search is the multi-process entry point; use lb200_group_search_batch");
    if (!nq || !k)
        return;
    if (!G.index.empty()) // the group's own index: pending rows first, as a one-GPU search does
        group_index_build_locked(G);
    if (G.ranks[0]->n == 0)
        throw CudaError("group: the group's index is empty");
    GroupRank* r = G.ranks[0];
    const uint32_t L = beam_width(*r, k, ef);
    const uint32_t W = agree_W(G, L);
    renew_flags(G, std::vector<cudaStream_t>(1, stream));
    r->launch(d_queries, nq, stride, kind, k, L, W, G.root, d_keys, d_dists, d_counts, stream);
}

// host buffers: queries are read on the root rank only; every rank receives the results
void group_search_host(Group& G, const void* queries, size_t nq, size_t stride, int kind, size_t k, size_t ef, uint64_t* keys,
                       float* dists, size_t* counts) {
    DeviceGuard dg;
    std::lock_guard<std::mutex> lk(G.mu);
    if (!G.distributed)
        throw CudaError("group: lb200_group_distribute has not been called");
    if (!nq || !k)
        return;
    if (!G.index.empty()) { // the group's own index: pending rows first; an empty index finds nothing (index.hpp:2693)
        group_index_build_locked(G);
        if (G.index[0]->n_ == 0) {
            for (size_t i = 0; i < nq * k; ++i) {
                if (keys)
                    keys[i] = ~0ull;
                if (dists)
                    dists[i] = INFINITY;
            }
            for (size_t i = 0; counts && i < nq; ++i)
                counts[i] = 0;
            return;
        }
    }
    const bool trace = getenv("LB200_GROUP_TRACE") != nullptr;
    auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t0 = trace ? now() : 0;
    const size_t nr = G.ranks.size();
    GroupRank* r0 = G.ranks[0];
    const uint32_t L = beam_width(*r0, k, ef);
    const uint32_t W = agree_W(G, L);
    const size_t in_bytes = scalar_row_bytes(kind, r0->cfg.dims);
    if (G.streams.size() != nr) {
        G.streams.assign(nr, nullptr);
        for (size_t i = 0; i < nr; ++i) {
            LB_CUDA(cudaSetDevice(G.ranks[i]->device));
            LB_CUDA(cudaStreamCreateWithFlags(&G.streams[i], cudaStreamNonBlocking));
        }
    }
    renew_flags(G, G.streams);
    size_t first = 0; // the root goes first: its (possibly pageable, hence host-blocking) upload must not sit behind kernels that
    for (size_t i = 0; i < nr; ++i) // already spin on the same device waiting for the root's queries
        if (G.ranks[i]->rank == G.root)
            first = i;
    for (size_t step = 0; step < nr; ++step) {
        const size_t i = (first + step) % nr;
        GroupRank* r = G.ranks[i];
        LB_CUDA(cudaSetDevice(r->device));
        const void* dq = nullptr;
        if (r->rank == G.root) {
            if (!queries)
                throw CudaError("group: the root rank must pass the queries");
            if (nq * in_bytes > r->in_bytes) // (sized for max_batch at distribution time; nothing may be allocated here)
                throw CudaError("group: batch larger than the group was created for (max_batch)");
            LB_CUDA(cudaMemcpy2DAsync(r->d_in, in_bytes, queries, stride, in_bytes, nq, cudaMemcpyHostToDevice, G.streams[i]));
            dq = r->d_in;
        }
        r->launch(dq, nq, in_bytes, kind, k, L, W, G.root, nullptr, nullptr, nullptr, G.streams[i]);
    }
    const double t1 = trace ? now() : 0;
    // results: from the first rank of this process (every rank holds all of them); the error word rides along
    LB_CUDA(cudaSetDevice(r0->device));
    cudaStream_t s0 = G.streams[0];
    if (keys)
        LB_CUDA(cudaMemcpyAsync(keys, r0->slab + r0->lay.res_keys, nq * k * 8, cudaMemcpyDeviceToHost, s0));
    if (dists)
        LB_CUDA(cudaMemcpyAsync(dists, r0->slab + r0->lay.res_dists, nq * k * 4, cudaMemcpyDeviceToHost, s0));
    if (counts) {
        r0->h_counts.resize(nq);
        LB_CUDA(cudaMemcpyAsync(r0->h_counts.data(), r0->slab + r0->lay.res_counts, nq * 4, cudaMemcpyDeviceToHost, s0));
    }
    for (size_t i = 0; i < nr; ++i) {
        GroupRank* r = G.ranks[i];
        LB_CUDA(cudaSetDevice(r->device));
        LB_CUDA(cudaMemcpyAsync(&r->h_err, r->slab + r->lay.err, 4, cudaMemcpyDeviceToHost, G.streams[i]));
    }
    for (size_t i = 0; i < nr; ++i) {
        LB_CUDA(cudaSetDevice(G.ranks[i]->device));
        LB_CUDA(cudaStreamSynchronize(G.streams[i]));
    }
    const double t2 = trace ? now() : 0;
    for (size_t i = 0; i < nr; ++i)
        if (G.ranks[i]->h_err)
            throw CudaError("group: a rank timed out waiting for a peer (rank " + std::to_string(G.ranks[i]->h_err - 1) + " gave up first)");
    if (counts)
        for (size_t i = 0; i < nq; ++i)
            counts[i] = r0->h_counts[i];
    if (trace)
        fprintf(stderr, "lb200 group rank %d: issue %.3f ms, wait %.3f ms\n", r0->rank, t1 - t0, t2 - t1);
}

void group_stats(Group& G, int which, GroupStats& out) {
    DeviceGuard dg;
    std::lock_guard<std::mutex> lk(G.mu);
    if (which < 0 || (size_t)which >= G.ranks.size())
        throw CudaError("group: no such local rank");
    GroupRank* r = G.ranks[which];
    LB_CUDA(cudaSetDevice(r->device));
    LB_CUDA(cudaDeviceSynchronize());
    r->check_error();
    unsigned long long c[16] = {0};
    LB_CUDA(cudaMemcpy(c, r->d_counters, sizeof(c), cudaMemcpyDeviceToHost));
    memset(&out, 0, sizeof(out));
    out.rank = r->rank, out.world = r->world;
    out.queries = r->last_nq;
    out.owner_computed_distances = c[1], out.owner_base_pops = c[2], out.owner_upper_hops = c[3], out.owner_rounds = c[4];
    out.local_rows_evaluated = c[5];
    out.owner_cycles_produce = c[8], out.owner_cycles_local = c[9], out.owner_cycles_wait = c[10], out.owner_cycles_consume = c[11];
    out.local_row_bytes = c[5] * r->vec_bytes;
    out.rows_held = r->bounds[r->rank + 1] - r->bounds[r->rank];
    float ms = 0.f;
    if (r->last_nq && cudaEventElapsedTime(&ms, r->ev0, r->ev1) == cudaSuccess)
        out.kernel_ms = ms;
    else
        (void)cudaGetLastError();
}

Group* group_create_ipc(int rank, int world, lb200_allgather_fn ag, void* ctx) {
    if (world < 1 || world > kGroupMax || rank < 0 || rank >= world)
        throw CudaError("group: world size must be 1..8 and 0 <= rank < world");
    if (world > 1 && !ag)
        throw CudaError("group: an all-gather callback is required to bootstrap a multi-process group");
    require_device();
    Group* G = new Group();
    G->world = world, G->ag = ag, G->ag_ctx = ctx;
    GroupRank* r = new GroupRank();
    r->rank = rank, r->world = world, r->local = (world == 1);
    LB_CUDA(cudaGetDevice(&r->device));
    G->ranks.push_back(r);
    return G;
}

Group* group_create_local(const int* devices, int ndev) {
    if (ndev < 1 || ndev > kGroupMax)
        throw CudaError("group: 1..8 devices");
    require_device();
    DeviceGuard dg;
    int have = 0;
    LB_CUDA(cudaGetDeviceCount(&have));
    Group* G = new Group();
    G->world = ndev;
    try {
        for (int i = 0; i < ndev; ++i) {
            const int dev = devices ? devices[i] : i;
            if (dev < 0 || dev >= have)
                throw CudaError("group: no such CUDA device");
            GroupRank* r = new GroupRank();
            r->rank = i, r->world = ndev, r->local = true, r->device = dev;
            G->ranks.push_back(r);
        }
        for (int i = 0; i < ndev; ++i) {
            LB_CUDA(cudaSetDevice(G->ranks[i]->device));
            for (int j = 0; j < ndev; ++j) {
                if (i == j || G->ranks[i]->device == G->ranks[j]->device)
                    continue;
                int can = 0;
                LB_CUDA(cudaDeviceCanAccessPeer(&can, G->ranks[i]->device, G->ranks[j]->device));
                if (!can)
                    throw CudaError("group: the devices cannot access each other's memory (no NVLink / P2P)");
                cudaError_t e = cudaDeviceEnablePeerAccess(G->ranks[j]->device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled)
                    LB_CUDA(e);
                (void)cudaGetLastError();
            }
        }
    } catch (...) {
        delete G;
        throw;
    }
    return G;
}

// ---- the same kernel as a single-GPU search path: G = 1, every slot is an owner, nothing crosses NVLink ------------------
// One warp per query instead of one CTA per query (search.cu): no CTA-wide barriers, 28 queries in flight per SM instead of
// 8-10.  For narrow rows (binary vectors, short f16/i8 rows) the per-expansion serial chain of the CTA kernel -- warp 0
// working while three warps wait at the barrier -- is what bounds it; here every warp always has its own work.
// fn(dm, sk, nq, ps) tags of the warp kernel: ps = std::true_type for the projected-screen owner (f32 l2sq / cos only)
template <typename Fn> static void dispatch_warp_kernel(int dm, int sk, int nq, bool ps, Fn&& fn) {
    dispatch_walk(dm, sk, nq, [&](auto d, auto s, auto q) {
        if (!ps)
            return fn(d, s, q, std::false_type{});
        if constexpr (decltype(s)::value == SK_F32 && (decltype(d)::value == DM_L2SQ || decltype(d)::value == DM_COS))
            fn(d, s, q, std::true_type{});
        else
            throw CudaError("warp search: the projected screen needs f32 l2sq / cos rows");
    });
}

void launch_warp_search(Index& idx, const uint8_t* qbuf, size_t qrow, size_t nq, size_t k, uint32_t L, const float* ps_query,
                        uint64_t* d_keys, float* d_dists, uint32_t* d_counts, cudaStream_t stream) {
    const IndexConfig& cfg = idx.cfg_;
    if (cfg.pq)
        throw CudaError("warp search: pq indexes use the CTA kernel");
    const uint32_t cap = (uint32_t)cfg.M0;
    if (cap > 256)
        throw CudaError("warp search: connectivity above 128 is not supported");
    const bool ps = ps_query != nullptr;
    const int nqc = pick_nq((uint32_t)idx.row_bytes_);
    const size_t smem = (size_t)group_warp_layout((uint32_t)idx.row_bytes_, group_ring_slots((uint32_t)idx.row_bytes_), L, cap,
                                                  ps ? ps_query_floats(idx.ps_k_) : 0u).total * kGroupWarps;
    int occ = 0;
    dispatch_warp_kernel(idx.dist_mode_, cfg.scalar_kind, nqc, ps, [&](auto d, auto s2, auto q, auto sc) {
        occ = group_occupancy_one<decltype(d)::value, decltype(s2)::value, decltype(q)::value, decltype(sc)::value>(smem);
    });
    if (occ < 1)
        throw CudaError("warp search: kernel does not fit on an SM (ef too large for shared memory)");
    const uint32_t W = (uint32_t)occ * (uint32_t)device_sm_count() * kGroupWarps;
    idx.ensure_scratch(W); // one visited bitmap + touched list per slot
    const size_t aux_need = 256 + round_up(nq * 4, 256);
    if (aux_need > idx.warp_aux_bytes_) {
        if (idx.d_warp_aux_)
            LB_CUDA(cudaFree(idx.d_warp_aux_));
        idx.d_warp_aux_ = nullptr;
        idx.warp_aux_bytes_ = aux_need + aux_need / 2;
        LB_CUDA(cudaMalloc(&idx.d_warp_aux_, idx.warp_aux_bytes_));
    }
    uint8_t* aux = idx.d_warp_aux_;
    LB_CUDA(cudaMemsetAsync(aux, 0, 256, stream)); // [0,128) counters, [128,136) done, [136,144) qready, [144,148) err
    GroupLaunch p;
    memset(&p, 0, sizeof(p));
    p.G = 1, p.me = 0, p.W = W, p.cap = cap, p.ring_slots = group_ring_slots((uint32_t)idx.row_bytes_);
    p.nq = (uint32_t)nq, p.k = (uint32_t)k, p.L = L;
    p.flag_base = 1u << 20, p.epoch = 1, p.root = 0;
    p.timeout_ns = ~0ull;
    p.g = idx.view();
    p.g.ps_query = ps_query;
    p.bounds[0] = 0;
    for (int r = 1; r <= kGroupMax; ++r)
        p.bounds[r] = 0xFFFFFFFFu;
    p.res_keys[0] = d_keys, p.res_dists[0] = d_dists;
    p.res_counts[0] = d_counts ? d_counts : (uint32_t*)(aux + 256);
    p.counters = (unsigned long long*)aux;
    p.done[0] = (unsigned long long*)(aux + 128), p.qready[0] = (unsigned long long*)(aux + 136), p.err[0] = (uint32_t*)(aux + 144);
    p.queries = qbuf, p.query_stride = (uint32_t)qrow;
    p.vis = idx.scratch_.visited, p.touched = idx.scratch_.touched;
    p.words_per_slot = idx.scratch_.words_per_cta, p.touched_cap = idx.scratch_.touched_cap;
    // equal waves: ceil(nq / ceil(nq / W)) owners rather than min(W, nq) -- at 4096 queries and W = 3168, 2048 walks of 2
    // queries each instead of 3168 walks whose second wave is mostly idle (measured 8 % faster at cfg3, DESIGN.md 6)
    const size_t waves = (nq + (W & ~3u) - 1) / (W & ~3u);
    p.O = (uint32_t)std::min<size_t>(W & ~3u, round_up((nq + waves - 1) / waves, kGroupWarps)), p.H = 0;
    const uint32_t grid = p.O / kGroupWarps;
    dispatch_warp_kernel(idx.dist_mode_, cfg.scalar_kind, nqc, ps, [&](auto d, auto s2, auto q, auto sc) {
        group_launch_one<decltype(d)::value, decltype(s2)::value, decltype(q)::value, decltype(sc)::value>(p, grid, smem, stream);
    });
    // Index::last_stats() reads p.counters (d_warp_aux_) after a warp search
}

void group_free(Group* G) {
    DeviceGuard dg;
    delete G;
}
int group_world(const Group& G) { return G.world; }
int group_local_ranks(const Group& G) { return (int)G.ranks.size(); }

} // namespace lb200

// lantern_b200 -- batched multi-query HNSW search (the hot path).
//
// Replaces, for a whole batch of queries at once, the reference's per-query
//   index_gt::search                U/include/usearch/index.hpp:2680-2730
//   search_for_one_  (greedy)       :3277-3316
//   search_to_find_in_base_ (beam)  :3400-3485
//   sorted_buffer_gt / max_heap_gt  :529-780     (top-ef list + candidate queue)
//   growing_hash_set_gt (visited)   :922-1040
//   metric_punned_t                 index_plugins.hpp:1340-1342
// in "exact-order mode": the same decision sequence per query as the reference (see walk.cuh), so on
// tie-free data the returned ids are those of the reference on the same graph, at any ef.
//
// Mapping to the machine: CTAs are persistent and pull queries from an atomic counter; one CTA (4 warps)
// walks one query at a time.  Per expanded node, warp 0 reads the adjacency line (128 B at M=16), filters
// it against the CTA's visited bitmap in HBM and compacts the unseen ids; every warp then streams its share
// of the neighbour rows HBM -> shared memory with bulk async copies and reduces the distances; warp 0
// finally replays the reference's sequential insertions.  No row is read twice; besides rows the only HBM
// traffic is one adjacency line per expansion and the bitmap words.
#include <cuda_runtime.h>
#include <stdlib.h>

#include <algorithm>
#include <type_traits>

#include "walk.cuh"

namespace lb200 {

size_t device_smem_optin(); // engine.cu: dynamic shared memory one CTA may opt in to

namespace {

template <class W> __device__ __forceinline__ void search_body(const SearchLaunch& p, const uint32_t R) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const WalkLayout lay = W::layout(p.g, R, p.L, p.g.M0 * p.expand);
    W w(p.g);
    w.init(smem_raw, lay, R, p.s);
    WalkSmem& sm = w.sm;

    for (;;) {
        __syncthreads();
        if (threadIdx.x == 0)
            sm.ctrl->item = (uint32_t)atomicAdd(&p.s.counters[0], 1ull);
        __syncthreads();
        const uint32_t q = sm.ctrl->item;
        if (q >= p.nq)
            break;
        w.load_query(q, p.queries + (size_t)q * p.query_stride);

        uint32_t cur = p.g.entry;
        float cur_d = w.measure_one(cur);
        w.greedy(cur, cur_d, p.g.max_level, 0);
        const uint32_t size = w.beam(0, cur, cur_d, p.L, kNoNeighbor, p.expand);

        // results: top is ascending; shrink(k); keys (index.hpp:2722-2723, 2426-2433)
        if (w.warp == 0) {
            const uint32_t found = min(size, p.k);
            for (uint32_t i = w.lane; i < p.k; i += 32) {
                uint64_t key = ~0ull;
                float d = INFINITY;
                if (i < found) {
                    key = __ldg(p.g.keys + (sm.top_i[i] & kIdMask));
                    d = sm.top_d[i];
                }
                p.out_keys[(size_t)q * p.k + i] = key;
                p.out_dists[(size_t)q * p.k + i] = d;
            }
            if (w.lane == 0 && p.out_counts)
                p.out_counts[q] = found;
        }
    }
    if (threadIdx.x == 0) {
        atomicAdd(&p.s.counters[1], (unsigned long long)w.st_dist);
        atomicAdd(&p.s.counters[2], (unsigned long long)w.st_pops);
        atomicAdd(&p.s.counters[3], (unsigned long long)w.st_hops);
        if (w.st_limbo_drop)
            atomicAdd(&p.s.counters[4], (unsigned long long)w.st_limbo_drop);
        if constexpr (W::kScreen) {
            atomicAdd(&p.s.counters[5], (unsigned long long)sm.ctrl->screened);
            atomicAdd(&p.s.counters[6], (unsigned long long)sm.ctrl->rejected);
        }
    }
}

template <class W>
__global__ void __launch_bounds__(kWalkThreads) hnsw_search_kernel(const __grid_constant__ SearchLaunch p, const uint32_t R) {
    search_body<W>(p, R);
}
// The screened walker (ScreenEval).  Up to NQ = 6 (d <= 768) it is capped at 64 registers, 8 CTAs/SM like the plain kernel: left to
// itself the compiler takes 72 registers there, which costs the eighth resident CTA; capped, it spills a few words.
template <class W>
__global__ void __launch_bounds__(kWalkThreads, W::kMinCtas) hnsw_search_screen_kernel(const __grid_constant__ SearchLaunch p,
                                                                                    const uint32_t R) {
    search_body<W>(p, R);
}
template <class W> constexpr auto search_kernel_of() {
    if constexpr (W::kScreen)
        return hnsw_search_screen_kernel<W>;
    else
        return hnsw_search_kernel<W>;
}

// test hook (lb200_search_screen_probe): the screen's bound and row_distance() for every (query, row) pair, with the device
// functions the search kernel uses.  One CTA per query, one warp per row.
template <int DM, int NQ>
__global__ void __launch_bounds__(128) screen_probe_kernel(const uint8_t* rows, uint32_t n, const uint8_t* queries, uint32_t row_bytes,
                                                           const uint8_t* codes, const float4* meta, float* out_lb, float* out_d) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t nchunks = row_bytes / 16, cb = screen_code_bytes(row_bytes);
    uint4 qreg[NQ];
    const float a2 = load_qreg<DM, SK_F32, NQ>(qreg, queries + (size_t)blockIdx.x * row_bytes, nchunks, lane);
    for (uint32_t j = warp; j < n; j += blockDim.x / 32) {
        const float4 mt = meta[j];
        const float s = screen_sum<DM, NQ>(qreg, reinterpret_cast<const uint32_t*>(codes + (size_t)j * cb), mt.x, nchunks, lane);
        const float lb = screen_bound<DM, NQ>(s, mt, a2);
        const float d = row_distance<DM, SK_F32, NQ>(qreg, reinterpret_cast<const uint4*>(rows + (size_t)j * row_bytes), nchunks, a2, lane);
        if (lane == 0)
            out_lb[(size_t)blockIdx.x * n + j] = lb, out_d[(size_t)blockIdx.x * n + j] = d;
    }
}

// test hook (lb200_search_pscreen_probe): the projected screen's bound, through PScreenEval's own per-candidate arithmetic
// (records, q~ in shared memory, pscreen_bound), and row_distance() for every (query, row) pair.  One CTA per query, one
// lane per row for the bound, one warp per row for the distance.
template <int DM, int NQ>
__global__ void __launch_bounds__(128) pscreen_probe_kernel(const uint8_t* rows, uint32_t n, const uint8_t* queries, uint32_t row_bytes,
                                                            const uint4* records, const float* qpre, uint32_t k, float* out_lb,
                                                            float* out_d) {
    __shared__ float psq[128];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t nchunks = row_bytes / 16, slots = ps_code_slots(k), rec = ps_record_bytes(k) / 16, nf = ps_query_floats(k);
    for (uint32_t i = threadIdx.x; i < nf; i += blockDim.x)
        psq[i] = qpre[(size_t)blockIdx.x * nf + i];
    __syncthreads();
    uint4 qreg[NQ];
    const float a2 = load_qreg<DM, SK_F32, NQ>(qreg, queries + (size_t)blockIdx.x * row_bytes, nchunks, lane);
    const float4 qh = *reinterpret_cast<const float4*>(psq + slots);
    for (uint32_t j = threadIdx.x; j < n; j += blockDim.x) {
        const uint4* r = records + (size_t)j * rec;
        float sf = 0.f, cc = 0.f;
        for (uint32_t g = 1; g < rec; ++g)
            ps_accum(psq + 16 * (g - 1), __ldg(r + g), sf, cc);
        const uint4 v0 = __ldg(r);
        const float4 meta = make_float4(__uint_as_float(v0.x), __uint_as_float(v0.y), __uint_as_float(v0.z), __uint_as_float(v0.w));
        out_lb[(size_t)blockIdx.x * n + j] = pscreen_bound<DM, NQ>(sf, cc, meta, qh, a2, slots);
    }
    for (uint32_t j = warp; j < n; j += blockDim.x / 32) {
        const float d = row_distance<DM, SK_F32, NQ>(qreg, reinterpret_cast<const uint4*>(rows + (size_t)j * row_bytes), nchunks, a2, lane);
        if (lane == 0)
            out_d[(size_t)blockIdx.x * n + j] = d;
    }
}

// test hook (lb200_pq_probe): the walkers' own PqEval<DM> on the index's view.  CTA v turns value v into its look-up table
// (load_query: the batch's precomputed tables when g.pq_query_tables is set, else load_value; load_node for node values),
// copies the table and |v|^2 out, then measures every stored row through eval(), cand_cap rows per pass, as a walk does.
template <int DM>
__global__ void __launch_bounds__(kWalkThreads) pq_probe_kernel(const __grid_constant__ GraphView g, const uint8_t* values,
                                                                uint32_t value_stride, const uint32_t* nodes, uint32_t cand_cap,
                                                                float* out_d, float* out_lut) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const WalkLayout lay = PqEval<DM>::layout(g, 0, 1, cand_cap);
    PqEval<DM> w(g);
    w.init(smem_raw, lay, 0, SearchScratch{});
    const uint32_t v = blockIdx.x;
    if (nodes)
        w.load_node(nodes[v]);
    else
        w.load_query(v, values + (size_t)v * value_stride);
    const size_t tf = (size_t)g.num_subvectors * g.pq_lut_width;
    for (size_t e = threadIdx.x; e < tf; e += kWalkThreads)
        out_lut[v * (tf + 1) + e] = w.lut[e];
    if (threadIdx.x == 0)
        out_lut[v * (tf + 1) + tf] = w.a2;
    for (uint32_t base = 0; base < g.n; base += cand_cap) {
        const uint32_t cnt = min(cand_cap, g.n - base);
        __syncthreads();
        for (uint32_t j = threadIdx.x; j < cnt; j += kWalkThreads)
            w.sm.cand_id[j] = base + j;
        __syncthreads();
        w.eval(cnt);
        __syncthreads();
        for (uint32_t j = threadIdx.x; j < cnt; j += kWalkThreads)
            out_d[(size_t)v * g.n + base + j] = w.sm.cand_d[j];
    }
}

template <int DM>
void launch_pq_probe_dm(const GraphView& g, uint32_t cand_cap, const uint8_t* d_values, uint32_t value_stride, const uint32_t* d_nodes,
                        size_t count, float* d_dist, float* d_lut, cudaStream_t stream) {
    const size_t smem = PqEval<DM>::layout(g, 0, 1, cand_cap).total;
    LB_CUDA(cudaFuncSetAttribute(pq_probe_kernel<DM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    pq_probe_kernel<DM><<<(unsigned)count, kWalkThreads, smem, stream>>>(g, d_values, value_stride, d_nodes, cand_cap, d_dist, d_lut);
    LB_CUDA(cudaGetLastError());
    count_launch();
}

template <class W> void launch_one(const SearchLaunch& p, uint32_t R, size_t smem, uint32_t grid, int threads, cudaStream_t stream) {
    auto kern = search_kernel_of<W>();
    LB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, threads, smem, stream>>>(p, R);
    LB_CUDA(cudaGetLastError());
    count_launch();
}

template <class W> int occupancy_one(size_t smem, int threads) {
    auto kern = search_kernel_of<W>();
    cudaFuncAttributes fa;
    LB_CUDA(cudaFuncGetAttributes(&fa, kern));
    if (smem + fa.sharedSizeBytes > device_smem_optin()) // a failed cudaFuncSetAttribute would also linger as the next call's last error
        return 0;
    LB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int blocks = 0;
    LB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, kern, threads, smem));
    return blocks;
}

// fn(walker type tag) with the screened walker of an f32 l2sq / cos index: 1 = int8 codes, 2 = projected codes
template <typename Fn> void dispatch_screen(int screen, int dm, int nq, Fn&& fn) {
    dispatch_walk(dm, SK_F32, nq, [&](auto d, auto s, auto n) {
        if constexpr (decltype(s)::value == SK_F32 && (decltype(d)::value == DM_L2SQ || decltype(d)::value == DM_COS)) {
            if (screen == 2)
                fn(TypeTag<PScreenWalker<decltype(d)::value, decltype(n)::value>>{});
            else
                fn(TypeTag<ScreenWalker<decltype(d)::value, decltype(n)::value>>{});
        } else {
            throw CudaError("search screen: f32 l2sq / cos indexes only");
        }
    });
}

} // namespace

// Warps per query: 4.  Two warps per query (twice the CTAs per SM, half the warps waiting at each barrier) was tried for
// 768-byte rows (cfg5t) and did not help: the narrow-row
// bound is the per-expansion latency chain itself, not the idle warps.  LB200_SEARCH_WARPS = 2 keeps the experiment runnable.
static int search_threads(const GraphView& g, bool pq) {
    (void)g;
    int warps = 4;
    if (const char* e = getenv("LB200_SEARCH_WARPS"))
        if (!pq && (atoi(e) == 2 || atoi(e) == 4))
            warps = atoi(e);
    return warps * 32;
}

static size_t search_smem(const GraphView& g, bool pq, int screen, uint32_t R, uint32_t L, uint32_t expand) {
    if (pq)
        return walk_layout_pq(g.num_subvectors, g.pq_lut_width, pq_value_floats(g), L, g.M0 * expand).total;
    if (screen == 2)
        return PScreenEval<DM_L2SQ, 1>::layout(g, R, L, g.M0 * expand).total; // the same for every (DM, NQ)
    return walk_layout(R, g.row_bytes, L, g.M0 * expand).total;
}

uint32_t search_max_ctas(int dist_mode, int scalar_kind, const GraphView& g, uint32_t L, bool pq, uint32_t expand, int screen) {
    const uint32_t R = pick_ring_slots(g.row_bytes);
    const int nq = pq ? 1 : pick_nq(g.row_bytes);
    if (nq < 0)
        throw CudaError("search: vectors wider than 8192 bytes are not supported");
    const size_t smem = search_smem(g, pq, screen, R, L, expand);
    int occ = 0;
    const int threads = search_threads(g, pq);
    auto occ_fn = [&](auto tag) { occ = occupancy_one<typename decltype(tag)::type>(smem, threads); };
    if (screen)
        dispatch_screen(screen, dist_mode, nq, occ_fn);
    else
        dispatch_walker(pq, dist_mode, scalar_kind, nq, occ_fn);
    if (occ < 1)
        throw CudaError("search: kernel does not fit on an SM (ef/k or the pq table too large for shared memory)");
    return (uint32_t)occ * (uint32_t)device_sm_count();
}

void launch_search(int dist_mode, int scalar_kind, bool pq, const SearchLaunch& p, cudaStream_t stream) {
    const uint32_t R = pick_ring_slots(p.g.row_bytes);
    const int nq = pq ? 1 : pick_nq(p.g.row_bytes);
    const size_t smem = search_smem(p.g, pq, p.screen, R, p.L, p.expand);
    const uint32_t grid = p.s.ctas < p.nq ? p.s.ctas : p.nq;
    const int threads = search_threads(p.g, pq);
    auto launch_fn = [&](auto tag) { launch_one<typename decltype(tag)::type>(p, R, smem, grid, threads, stream); };
    if (p.screen)
        dispatch_screen(p.screen, dist_mode, nq, launch_fn);
    else
        dispatch_walker(pq, dist_mode, scalar_kind, nq, launch_fn);
}

void launch_screen_probe(int dist_mode, const uint8_t* d_rows, size_t n, const uint8_t* d_queries, size_t nq, uint32_t row_bytes,
                         float* d_lb, float* d_dist, cudaStream_t stream) {
    const int nqr = pick_nq(row_bytes);
    if (nqr < 0)
        throw CudaError("screen probe: vectors wider than 8192 bytes are not supported");
    const size_t cb = screen_code_bytes(row_bytes);
    uint8_t* codes = nullptr;
    float4* meta = nullptr;
    LB_CUDA(cudaMalloc(&codes, std::max<size_t>(n * cb, 1)));
    cudaError_t e = cudaMalloc(&meta, std::max<size_t>(n, 1) * sizeof(float4));
    if (e != cudaSuccess) {
        cudaFree(codes);
        LB_CUDA(e);
    }
    try {
        launch_sq_encode(d_rows, row_bytes, n, codes, meta, stream);
        dispatch_walk(dist_mode, SK_F32, nqr, [&](auto d, auto s, auto q) {
            constexpr int DM = decltype(d)::value;
            if constexpr (decltype(s)::value == SK_F32 && (DM == DM_L2SQ || DM == DM_COS)) {
                if (n && nq)
                    screen_probe_kernel<DM, decltype(q)::value><<<(unsigned)nq, 128, 0, stream>>>(d_rows, (uint32_t)n, d_queries, row_bytes,
                                                                                              codes, meta, d_lb, d_dist);
                LB_CUDA(cudaGetLastError());
                count_launch();
            } else {
                throw CudaError("screen probe: l2sq or cos only");
            }
        });
        LB_CUDA(cudaStreamSynchronize(stream));
    } catch (...) {
        cudaFree(codes), cudaFree(meta);
        throw;
    }
    cudaFree(codes), cudaFree(meta);
}

void launch_pscreen_probe(int dist_mode, const uint8_t* d_rows, size_t n, const uint8_t* d_queries, size_t nq, uint32_t row_bytes,
                          size_t dims, const float* d_P, const float* d_Pt, uint32_t k, float* d_lb, float* d_dist, cudaStream_t stream) {
    const int nqr = pick_nq(row_bytes);
    if (nqr < 0)
        throw CudaError("pscreen probe: vectors wider than 8192 bytes are not supported");
    if (!n || !nq)
        return;
    uint8_t* records = nullptr;
    float* qpre = nullptr;
    LB_CUDA(cudaMalloc(&records, n * ps_record_bytes(k)));
    cudaError_t e = cudaMalloc(&qpre, nq * ps_query_floats(k) * sizeof(float));
    if (e != cudaSuccess) {
        cudaFree(records);
        LB_CUDA(e);
    }
    try {
        launch_ps_encode(d_rows, row_bytes, n, dims, d_P, d_Pt, k, dist_mode == DM_COS, records, stream);
        launch_ps_queries(d_P, d_Pt, dims, k, d_queries, row_bytes, nq, qpre, stream);
        dispatch_walk(dist_mode, SK_F32, nqr, [&](auto d, auto s, auto q) {
            constexpr int DM = decltype(d)::value;
            if constexpr (decltype(s)::value == SK_F32 && (DM == DM_L2SQ || DM == DM_COS)) {
                pscreen_probe_kernel<DM, decltype(q)::value><<<(unsigned)nq, 128, 0, stream>>>(
                    d_rows, (uint32_t)n, d_queries, row_bytes, reinterpret_cast<const uint4*>(records), qpre, k, d_lb, d_dist);
                LB_CUDA(cudaGetLastError());
                count_launch();
            } else {
                throw CudaError("pscreen probe: l2sq or cos only");
            }
        });
        LB_CUDA(cudaStreamSynchronize(stream));
    } catch (...) {
        cudaFree(records), cudaFree(qpre);
        throw;
    }
    cudaFree(records), cudaFree(qpre);
}

void launch_pq_probe(int dist_mode, const GraphView& g, uint32_t cand_cap, const uint8_t* d_values, uint32_t value_stride,
                     const uint32_t* d_nodes, size_t count, float* d_dist, float* d_lut, cudaStream_t stream) {
    if (!count || !g.n)
        return;
    if (dist_mode == DM_L2SQ)
        launch_pq_probe_dm<DM_L2SQ>(g, cand_cap, d_values, value_stride, d_nodes, count, d_dist, d_lut, stream);
    else if (dist_mode == DM_COS)
        launch_pq_probe_dm<DM_COS>(g, cand_cap, d_values, value_stride, d_nodes, count, d_dist, d_lut, stream);
    else
        throw CudaError("pq probe: l2sq or cos only");
    LB_CUDA(cudaStreamSynchronize(stream));
}

} // namespace lb200

// lantern_b200 -- exhaustive ("ef -> infinity") search, pairwise distances, shard merge.
//
// GPU counterparts of
//   exact_search_t            U/include/usearch/index_plugins.hpp:1582-1675  (all Q x N distances, k smallest)
//   usearch_exact_search      U/c/lib.cpp:450-481   (returns dataset OFFSETS + distances, ascending)
//   usearch_distance          U/c/lib.cpp:440-448
// Distances are computed directly in the metric's own form (sum (a-b)^2, not |a|^2+|b|^2-2ab) in fp32,
// so they agree with the reference to summation-order rounding (1e-5 relative contract) and the
// returned ids are exact on tie-free data.  Ties are ordered by lower dataset offset.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <math.h>

#include <algorithm>
#include <type_traits>

#include "distance.cuh"
#include "engine.h"

namespace lb200 {

namespace {

constexpr int kQT = 8;      // queries per CTA == warps per CTA
constexpr int kExWarps = 8; // 256 threads
constexpr int kSub = 32;    // dataset rows per sub-batch (4 per warp)

__device__ __forceinline__ bool closer(float d, uint64_t id, float od, uint64_t oid) { return closer_total(d, id, od, oid); }

// Sorted (ascending by (dist, id)) insert of one element into a list of capacity k, by a full warp.
__device__ __forceinline__ void list_insert(float* ld, uint64_t* li, uint32_t& size, uint32_t k, float d, uint64_t id, int lane) {
    uint32_t pos = 0;
    for (uint32_t b = 0; b < size; b += 32) {
        uint32_t e = b + lane;
        bool before = e < size && closer(ld[e], li[e], d, id);
        pos += __popc(__ballot_sync(0xffffffffu, before));
    }
    if (pos >= k)
        return;
    uint32_t last = (size == k) ? k - 1 : size;
    for (int hi = (int)last; hi > (int)pos; hi -= 32) {
        int idx = hi - lane;
        bool act = idx > (int)pos;
        float vd = 0.f;
        uint64_t vi = 0;
        if (act)
            vd = ld[idx - 1], vi = li[idx - 1];
        __syncwarp();
        if (act)
            ld[idx] = vd, li[idx] = vi;
        __syncwarp();
    }
    __syncwarp(); // the position scan's reads are ordered before this write even when nothing was shifted (racecheck)
    if (lane == 0)
        ld[pos] = d, li[pos] = id;
    __syncwarp();
    size = last + 1;
}

// grid = (dataset blocks, query tiles), the tiles counted from `tile0`.  Partial results: part_*[block][query][k].
// QG: the kQT query rows are read from global memory (L1 / L2) instead of being staged in shared memory -- for rows so wide
// that kQT of them and the top-k lists exceed the opt-in shared memory of a CTA.  A tile's missing queries (past nq) then
// read the last query; their distances are computed and dropped.
template <int DM, int SK, bool QG>
__global__ void __launch_bounds__(kExWarps * 32) exact_block_kernel(const uint8_t* __restrict__ data, size_t n, size_t data_stride,
                                                                    const uint8_t* __restrict__ queries, uint32_t nq,
                                                                    size_t q_stride, uint32_t row_bytes, uint32_t k,
                                                                    uint32_t rows_per_block, uint32_t tile0,
                                                                    uint64_t* __restrict__ part_keys,
                                                                    float* __restrict__ part_dists,
                                                                    const uint8_t* __restrict__ qmask) {
    extern __shared__ __align__(16) uint8_t sm_raw[];
    const uint32_t q0 = (tile0 + blockIdx.y) * kQT;
    if (qmask) { // second pass behind the tensor-core filter (exact_tc.cu): only the queries it could not certify
        bool any = false;
        for (uint32_t q = 0; q < kQT; ++q)
            any |= q0 + q < nq && qmask[q0 + q];
        if (!any)
            return;
    }
    const uint32_t nchunks = row_bytes / 16;
    const size_t sq_bytes = QG ? 0 : (size_t)kQT * row_bytes;
    uint4* sq = reinterpret_cast<uint4*>(sm_raw);                                // [kQT][nchunks] (not QG)
    float* sdist = reinterpret_cast<float*>(sm_raw + sq_bytes);                    // [kQT][kSub]
    float* ld = sdist + kQT * kSub;                                               // [kQT][k]
    uint64_t* li = reinterpret_cast<uint64_t*>(ld + (((size_t)kQT * k + 1) & ~(size_t)1)); // [kQT][k]
    __shared__ float sa2[kQT];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t row0 = (size_t)blockIdx.x * rows_per_block;
    const size_t row1 = min(n, row0 + rows_per_block);
    // chunk c of query q0 + q
    auto qchunk = [&](int q, uint32_t c) -> uint4 {
        if constexpr (QG)
            return __ldg(reinterpret_cast<const uint4*>(queries + (size_t)min(q0 + q, nq - 1) * q_stride) + c);
        else
            return sq[q * nchunks + c];
    };

    if constexpr (!QG) {
        for (uint32_t i = threadIdx.x; i < kQT * nchunks; i += blockDim.x) {
            uint32_t q = i / nchunks, c = i % nchunks;
            sq[i] = (q0 + q < nq) ? __ldg(reinterpret_cast<const uint4*>(queries + (size_t)(q0 + q) * q_stride) + c)
                                  : make_uint4(0, 0, 0, 0);
        }
        __syncthreads();
    }
    if (DM == DM_COS) { // a2 of query `warp`
        float part = 0.f;
        for (uint32_t c = lane; c < nchunks; c += 32)
            part = norm_add(part, query_norm_chunk<DM, SK>(qchunk(warp, c)));
        part = warp_sum(part);
        if (lane == 0)
            sa2[warp] = part;
    }
    __syncthreads();

    uint32_t size = 0; // list of query `warp`
    float* my_ld = ld + (size_t)warp * k;
    uint64_t* my_li = li + (size_t)warp * k;

    for (size_t base = row0; base < row1; base += kSub) {
        // phase 1: warp w computes rows base + 4w .. +3 against all kQT queries
        for (int r = 0; r < kSub / kExWarps; ++r) {
            const size_t row = base + warp * (kSub / kExWarps) + r;
            DistAcc<DM, SK> acc[kQT];
#pragma unroll
            for (int q = 0; q < kQT; ++q)
                acc[q].reset();
            if (row < row1) {
                const uint4* rp = reinterpret_cast<const uint4*>(data + row * data_stride);
                for (uint32_t c = lane; c < nchunks; c += 32) {
                    const uint4 rv = __ldg(rp + c);
#pragma unroll
                    for (int q = 0; q < kQT; ++q)
                        accum_chunk<DM, SK>(acc[q], qchunk(q, c), rv);
                }
            }
#pragma unroll
            for (int q = 0; q < kQT; ++q) {
                float d = finish_distance<DM, SK>(acc[q], DM == DM_COS ? sa2[q] : 0.f);
                if (lane == 0)
                    sdist[q * kSub + warp * (kSub / kExWarps) + r] = row < row1 ? d : INFINITY;
            }
        }
        __syncthreads();
        // phase 2: warp w owns query w: lane j looks at row base+j
        if (q0 + warp < nq) {
            const size_t row = base + lane;
            const float d = sdist[warp * kSub + lane];
            bool want = row < row1 && (size < k || closer(d, row, my_ld[size - 1], my_li[size - 1]));
            uint32_t m = __ballot_sync(0xffffffffu, want);
            while (m) {
                int j = __ffs(m) - 1;
                m &= m - 1;
                float dj = __shfl_sync(0xffffffffu, d, j);
                uint64_t rj = base + j;
                if (size < k || closer(dj, rj, my_ld[size - 1], my_li[size - 1]))
                    list_insert(my_ld, my_li, size, k, dj, rj, lane);
            }
        }
        __syncthreads();
    }
    if (q0 + warp < nq) {
        uint64_t* ok = part_keys + ((size_t)blockIdx.x * nq + q0 + warp) * k;
        float* od = part_dists + ((size_t)blockIdx.x * nq + q0 + warp) * k;
        for (uint32_t i = lane; i < k; i += 32) {
            ok[i] = i < size ? my_li[i] : ~0ull;
            od[i] = i < size ? my_ld[i] : INFINITY;
        }
    }
}

// One CTA per query: k-way merge of G ascending lists by repeated arg-min over the list heads.
// in_*: [G][nq][k]; ties by lower key.  Also the multi-GPU epilogue after the all-gather.
__global__ void merge_lists_kernel(const uint64_t* __restrict__ in_keys, const float* __restrict__ in_dists, uint32_t G,
                                   uint32_t nq, uint32_t k, uint64_t* __restrict__ out_keys, float* __restrict__ out_dists,
                                   const uint8_t* __restrict__ qmask) {
    extern __shared__ uint32_t heads[]; // [G]
    if (qmask && !qmask[blockIdx.x])
        return;
    __shared__ float red_d[32];
    __shared__ uint64_t red_k[32];
    __shared__ uint32_t red_g[32];
    const uint32_t q = blockIdx.x;
    for (uint32_t g = threadIdx.x; g < G; g += blockDim.x)
        heads[g] = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (uint32_t out = 0; out < k; ++out) {
        float bd = INFINITY;
        uint64_t bk = ~0ull;
        uint32_t bg = 0xFFFFFFFFu;
        for (uint32_t g = threadIdx.x; g < G; g += blockDim.x) {
            uint32_t h = heads[g];
            if (h < k) {
                size_t o = ((size_t)g * nq + q) * k + h;
                float d = in_dists[o];
                uint64_t key = in_keys[o];
                if (key != ~0ull && (bg == 0xFFFFFFFFu || closer(d, key, bd, bk)))
                    bd = d, bk = key, bg = g;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            float od = __shfl_xor_sync(0xffffffffu, bd, o);
            uint64_t ok = __shfl_xor_sync(0xffffffffu, bk, o);
            uint32_t og = __shfl_xor_sync(0xffffffffu, bg, o);
            if (og != 0xFFFFFFFFu && (bg == 0xFFFFFFFFu || closer(od, ok, bd, bk)))
                bd = od, bk = ok, bg = og;
        }
        if (lane == 0)
            red_d[warp] = bd, red_k[warp] = bk, red_g[warp] = bg;
        __syncthreads();
        if (warp == 0) {
            bd = lane < nwarps ? red_d[lane] : INFINITY;
            bk = lane < nwarps ? red_k[lane] : ~0ull;
            bg = lane < nwarps ? red_g[lane] : 0xFFFFFFFFu;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                float od = __shfl_xor_sync(0xffffffffu, bd, o);
                uint64_t ok = __shfl_xor_sync(0xffffffffu, bk, o);
                uint32_t og = __shfl_xor_sync(0xffffffffu, bg, o);
                if (og != 0xFFFFFFFFu && (bg == 0xFFFFFFFFu || closer(od, ok, bd, bk)))
                    bd = od, bk = ok, bg = og;
            }
            if (lane == 0) {
                out_keys[(size_t)q * k + out] = bg == 0xFFFFFFFFu ? ~0ull : bk;
                out_dists[(size_t)q * k + out] = bg == 0xFFFFFFFFu ? INFINITY : bd;
                if (bg != 0xFFFFFFFFu)
                    heads[bg] += 1;
            }
        }
        __syncthreads();
    }
}

template <int DM, int SK>
__global__ void pair_distance_kernel(const uint8_t* __restrict__ a, size_t a_stride, const uint8_t* __restrict__ b,
                                     size_t b_stride, size_t n, uint32_t row_bytes, float* __restrict__ out) {
    const size_t pair = (size_t)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (pair >= n)
        return;
    const uint4* pa = reinterpret_cast<const uint4*>(a + pair * a_stride);
    const uint4* pb = reinterpret_cast<const uint4*>(b + pair * b_stride);
    const uint32_t nchunks = row_bytes / 16;
    DistAcc<DM, SK> acc;
    acc.reset();
    float part = 0.f;
    for (uint32_t c = lane; c < nchunks; c += 32) {
        uint4 qa = __ldg(pa + c), rb = __ldg(pb + c);
        accum_chunk<DM, SK>(acc, qa, rb);
        part = norm_add(part, query_norm_chunk<DM, SK>(qa));
    }
    float a2 = DM == DM_COS ? warp_sum(part) : 0.f;
    float d = finish_distance<DM, SK>(acc, a2);
    if (lane == 0)
        out[pair] = d;
}

template <typename Fn> void dispatch2(int dm, int sk, Fn&& fn) {
#define LB_CASE(DMv, SKv)                                                                                              \
    if (dm == DMv && sk == SKv) {                                                                                      \
        fn(std::integral_constant<int, DMv>{}, std::integral_constant<int, SKv>{});                                    \
        return;                                                                                                        \
    }
    LB_CASE(DM_L2SQ, SK_F32)
    LB_CASE(DM_COS, SK_F32)
    LB_CASE(DM_L2SQ, SK_F16)
    LB_CASE(DM_COS, SK_F16)
    LB_CASE(DM_L2SQ, SK_I8)
    LB_CASE(DM_COS, SK_I8)
    LB_CASE(DM_HAMMING, SK_B1)
#undef LB_CASE
    throw CudaError("unsupported metric / scalar kind combination");
}

} // namespace

static void launch_merge_masked(const uint64_t* d_keys, const float* d_dists, size_t shards, size_t nq, size_t k, uint64_t* d_out_keys,
                                float* d_out_dists, const uint8_t* qmask, cudaStream_t stream) {
    if (!nq || !k)
        return;
    int threads = shards >= 256 ? 256 : (shards >= 64 ? 128 : 32);
    merge_lists_kernel<<<(unsigned)nq, threads, shards * sizeof(uint32_t), stream>>>(
        d_keys, d_dists, (uint32_t)shards, (uint32_t)nq, (uint32_t)k, d_out_keys, d_out_dists, qmask);
    LB_CUDA(cudaGetLastError());
    count_launch();
}

void launch_merge_shards(const uint64_t* d_keys, const float* d_dists, size_t shards, size_t nq, size_t k,
                         uint64_t* d_out_keys, float* d_out_dists, cudaStream_t stream) {
    launch_merge_masked(d_keys, d_dists, shards, nq, k, d_out_keys, d_out_dists, nullptr, stream);
}

size_t device_smem_optin(); // engine.cu

// exact_tc.cu
bool exact_tc_applicable(int dist_mode, int scalar_kind, size_t n, size_t nq, size_t k, uint32_t row_bytes);
bool exact_tc_defined(int dist_mode, int scalar_kind, size_t n, size_t k);
void launch_exact_tc(int dist_mode, const uint8_t* d_data, size_t n, size_t data_stride, const uint8_t* d_queries, size_t nq,
                     size_t q_stride, uint32_t row_bytes, size_t k, uint64_t* d_keys, float* d_dists, uint8_t** d_unsafe,
                     uint32_t** d_unsafe_count, cudaStream_t stream, const ExactTcProbe* probe);

void launch_exact(int dist_mode, int scalar_kind, const uint8_t* d_data, size_t n, size_t data_stride,
                  const uint8_t* d_queries, size_t nq, size_t q_stride, uint32_t row_bytes, size_t k, uint64_t* d_keys,
                  float* d_dists, cudaStream_t stream, const ExactTcProbe* probe) {
    if (!nq || !k)
        return;
    if (k > 1024)
        throw CudaError("exact search: count > 1024 is not supported");
    if (probe && !exact_tc_defined(dist_mode, scalar_kind, n, k))
        throw CudaError("exact search probe: the tensor-core filter takes f32 l2sq / cos, 1 <= n < 2^32 rows and count <= 192");
    // f32 l2sq / cos on a GEMM-sized problem: tensor-core filter + exact re-rank (exact_tc.cu); the SIMT kernels below then
    // run only for the queries the filter could not certify (usually none: every CTA of the second pass exits at once)
    uint8_t* qmask = nullptr;
    uint32_t* unsafe_count = nullptr;
    if (probe || exact_tc_applicable(dist_mode, scalar_kind, n, nq, k, row_bytes))
        launch_exact_tc(dist_mode, d_data, n, data_stride, d_queries, nq, q_stride, row_bytes, k, d_keys, d_dists, &qmask, &unsafe_count,
                        stream, probe);
    size_t rows_per_block = 4096;
    if ((n + rows_per_block - 1) / rows_per_block > 1024)
        rows_per_block = round_up((n + 1023) / 1024, kSub);
    const size_t blocks = n ? (n + rows_per_block - 1) / rows_per_block : 1;
    uint64_t* part_keys = nullptr;
    float* part_dists = nullptr;
    LB_CUDA(cudaMallocAsync(&part_keys, blocks * nq * k * sizeof(uint64_t), stream));
    LB_CUDA(cudaMallocAsync(&part_dists, blocks * nq * k * sizeof(float), stream));
    // shared memory: the kQT staged query rows (unless they do not fit: QG), the sub-batch distances and the top-k lists
    const size_t lists = (size_t)kQT * kSub * 4 + (((size_t)kQT * k + 1) & ~(size_t)1) * 4 + (size_t)kQT * k * 8;
    const size_t optin = device_smem_optin();
    const size_t static_smem = kQT * sizeof(float); // sa2
    const bool qg = (size_t)kQT * row_bytes + lists + static_smem > optin;
    const size_t smem = (qg ? 0 : (size_t)kQT * row_bytes) + lists;
    if (smem + static_smem > optin) // k <= 1024 keeps the lists near 100 KB: never on sm_90
        throw CudaError("exact search: the top-k lists do not fit in shared memory");
    // grid.y is at most 65535: the query tiles go in slices of that many launches
    const size_t tiles = (nq + kQT - 1) / kQT;
    const size_t kMaxTiles = 65535;
    dispatch2(dist_mode, scalar_kind, [&](auto dm, auto sk) {
        auto launch = [&](auto kern) {
            LB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            for (size_t t0 = 0; t0 < tiles; t0 += kMaxTiles) {
                dim3 grid((unsigned)blocks, (unsigned)std::min(kMaxTiles, tiles - t0));
                kern<<<grid, kExWarps * 32, smem, stream>>>(d_data, n, data_stride, d_queries, (uint32_t)nq, q_stride, row_bytes,
                                                            (uint32_t)k, (uint32_t)rows_per_block, (uint32_t)t0, part_keys,
                                                            part_dists, qmask);
                LB_CUDA(cudaGetLastError());
                count_launch();
            }
        };
        if (qg)
            launch(exact_block_kernel<decltype(dm)::value, decltype(sk)::value, true>);
        else
            launch(exact_block_kernel<decltype(dm)::value, decltype(sk)::value, false>);
    });
    launch_merge_masked(part_keys, part_dists, blocks, nq, k, d_keys, d_dists, qmask, stream);
    LB_CUDA(cudaFreeAsync(part_keys, stream));
    LB_CUDA(cudaFreeAsync(part_dists, stream));
    if (qmask) {
        if (getenv("LB200_EXACT_REPORT")) { // diagnostics: how many queries needed the SIMT pass
            uint32_t c = 0;
            LB_CUDA(cudaMemcpyAsync(&c, unsafe_count, 4, cudaMemcpyDeviceToHost, stream));
            LB_CUDA(cudaStreamSynchronize(stream));
            fprintf(stderr, "lb200 exact search: tensor-core filter certified %zu of %zu queries\n", nq - c, nq);
        }
        LB_CUDA(cudaFreeAsync(qmask, stream));
        LB_CUDA(cudaFreeAsync(unsafe_count, stream));
    }
}

void launch_pair_distance(int dist_mode, int scalar_kind, const uint8_t* d_a, size_t a_stride, const uint8_t* d_b,
                          size_t b_stride, size_t n, uint32_t row_bytes, float* d_out, cudaStream_t stream) {
    if (!n)
        return;
    const int warps = 4;
    dispatch2(dist_mode, scalar_kind, [&](auto dm, auto sk) {
        pair_distance_kernel<decltype(dm)::value, decltype(sk)::value>
            <<<(unsigned)((n + warps - 1) / warps), warps * 32, 0, stream>>>(d_a, a_stride, d_b, b_stride, n, row_bytes, d_out);
        LB_CUDA(cudaGetLastError());
        count_launch();
    });
}

} // namespace lb200

// lantern_b200 -- exhaustive search on the Hopper tensor cores (wgmma), f32 l2sq / cos.
//
// The GEMM-shaped piece of the reference path: exact_search_t (U/include/usearch/index_plugins.hpp:1582-1675) behind
// usearch_exact_search (U/c/lib.cpp:450-481) measures every query against every row.  A tensor core cannot reproduce
// the reference's fp32 sum of (a-b)^2 bit for bit, so it is used as a FILTER with an error bound, and the answer is
// produced by the same fp32 arithmetic as before:
//   1. norms_kernel            |x|^2 of every row and query (fp32)
//   2. exact_tc_filter_kernel  D = Q . X^T on wgmma in "3xTF32" (a = hi + lo with hi, lo representable in tf32;
//                              q.x ~ qhi.xhi + qhi.xlo + qlo.xhi, fp32 accumulation in registers), fused epilogue: distance
//                              from norms and dot product, per-query candidate list (a max-heap) of KP > k entries per row
//                              group, plus the smallest lower bound of anything the list had to drop
//   3. exact_tc_rerank_kernel  per query: candidates whose lower bound (approx - eps) does not exceed the k-th smallest
//                              upper bound (approx + eps) are re-measured with the SIMT distance code of exact.cu
//                              (same lane layout, same reduction) and sorted by (distance, offset): ids and distances are
//                              those of exact_block_kernel, ties included.  eps (approx_eps) bounds |approx - exact fp32|:
//                              the split's truncation and the tensor-core accumulation, the fp32 norms and the exact
//                              kernel's own summation (both growing with the chunks per lane), and subnormal products the
//                              tensor cores may flush.  A query whose lists may have dropped a qualifying row, with more
//                              qualifying rows than fit, or with a non-finite approximate distance, is flagged and
//                              answered by the SIMT kernels (exact.cu) -- never silently wrong.
//
// Filter kernel anatomy (one CTA per SM, 4 warpgroups, persistent over its row tiles):
//   warpgroup 0     producers  rows come in as fp32 (LDG.128, 8 consecutive chunks of a row per thread), are split into
//                              hi / lo in registers and stored (STS.128) straight into the K-major no-swizzle core-matrix
//                              layout the wgmma descriptors describe: address(row, chunk) = (row / 8) * 1024 + chunk * 128
//                              + (row % 8) * 16 per 32-float k-block (SBO = 1024 B, LBO = 128 B)
//   warpgroups 1-2  MMA        warpgroup w multiplies queries 64 (w-1) .. 64 w - 1 of the tile: per k-block 4 x 3
//                              wgmma.m64n128k8.tf32 into 64 fp32 registers per thread; per tile the accumulator is stored
//                              to a shared-memory tile (row = query) once the epilogue has drained the previous one
//   warpgroup 3     epilogue   thread t owns query t of the tile and scans its row of the shared-memory tile
// Two shared-memory stages (64 KB each: A hi/lo 2 x 16 KB, B hi/lo 2 x 16 KB) and the 66 KB accumulator tile keep the
// loads of k-block kb+1 under the MMAs of k-block kb, and the epilogue of tile t under the MMAs of tile t+1.
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>
#include <stdlib.h>

#include <type_traits>

#include "distance.cuh"
#include "engine.h"

namespace lb200 {

namespace {

constexpr int kTcThreads = 512;          // 4 producer + 8 MMA + 4 epilogue warps
constexpr uint32_t kTileM = 128;         // queries per tile (two wgmma M = 64 halves)
constexpr uint32_t kTileN = 128;         // rows per tile (wgmma N)
constexpr uint32_t kBlockK = 32;         // floats per k-block (128 B of a row)
constexpr uint32_t kStages = 2;
constexpr uint32_t kABytes = kTileM * kBlockK * 4; // 16 KB
constexpr uint32_t kBBytes = kTileN * kBlockK * 4; // 16 KB
constexpr uint32_t kStageBytes = 2 * kABytes + 2 * kBBytes;
constexpr uint32_t kAccLd = kTileN + 4;  // floats per accumulator-tile row: the epilogue's 16-byte reads are conflict-free
constexpr uint32_t kAccBytes = kTileM * kAccLd * 4;
constexpr uint32_t kTcSmem = kStages * kStageBytes + kAccBytes + 1024;
constexpr uint32_t kMaxKP = 256;

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// K-major, no swizzle: core matrix = 8 rows x 16 bytes, contiguous; LBO = distance between core matrices adjacent in K,
// SBO = distance between 8-row groups (both in 16-byte units in the descriptor); layout_type 0 (no swizzle)
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFFu);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// d (+)= A[smem] * B[smem]^T, M = 64, N = 128, K = 8, tf32 inputs (both K-major), fp32 accumulate in 64 registers
__device__ __forceinline__ void wgmma_tf32_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile("{\n\t"
                 ".reg .pred p;\n\t"
                 "setp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
                 "%64, %65, p, 1, 1;\n\t"
                 "}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(a_desc), "l"(b_desc), "r"(accumulate)
                 : "memory");
}
__device__ __forceinline__ float tf32_round(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
__device__ __forceinline__ void split4(const uint4& v, uint4& hi, uint4& lo) {
    const float x0 = __uint_as_float(v.x), x1 = __uint_as_float(v.y), x2 = __uint_as_float(v.z), x3 = __uint_as_float(v.w);
    const float h0 = tf32_round(x0), h1 = tf32_round(x1), h2 = tf32_round(x2), h3 = tf32_round(x3);
    hi = make_uint4(__float_as_uint(h0), __float_as_uint(h1), __float_as_uint(h2), __float_as_uint(h3));
    lo = make_uint4(__float_as_uint(tf32_round(x0 - h0)), __float_as_uint(tf32_round(x1 - h1)), __float_as_uint(tf32_round(x2 - h2)),
                    __float_as_uint(tf32_round(x3 - h3)));
}

__global__ void norms_kernel(const uint8_t* __restrict__ rows, size_t n, size_t stride, uint32_t nchunks, float* __restrict__ out) {
    const size_t row = (size_t)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= n)
        return;
    const uint4* p = reinterpret_cast<const uint4*>(rows + row * stride);
    float s = 0.f;
    for (uint32_t c = lane; c < nchunks; c += 32) {
        const uint4 v = __ldg(p + c);
        const float a = __uint_as_float(v.x), b = __uint_as_float(v.y), cc = __uint_as_float(v.z), d = __uint_as_float(v.w);
        s += a * a + b * b + cc * cc + d * d;
    }
    s = warp_sum(s);
    if (lane == 0)
        out[row] = s;
}

struct TcParams {
    const uint8_t* data;
    size_t n, data_stride;
    const uint8_t* queries;
    uint32_t nq;
    size_t q_stride;
    uint32_t nchunks; // 16-byte chunks per row (row_bytes / 16)
    const float* xn;
    const float* qn;
    uint32_t groups;  // row groups per query tile: CTA (qt, g) handles row tiles g, g + groups, ...
    uint32_t row_tiles;
    uint32_t KP;
    ExactTcEps eps;
    float* cand_d;    // [nq][groups][KP] approx distances of the kept rows, heap order (+inf padded)
    uint32_t* cand_i; // [nq][groups][KP]
    float* dropped_lb; // [nq][groups] smallest lower bound among entries the list could not keep (+inf if none)
};

template <int DM> __device__ __forceinline__ float approx_distance(float dot, float qn, float xn) {
    if constexpr (DM == DM_COS) {
        if (qn == 0.f && xn == 0.f)
            return 0.f;
        if (qn == 0.f || xn == 0.f)
            return 1.f;
        return 1.f - dot / (sqrtf(qn) * sqrtf(xn));
    } else {
        return qn + xn - 2.f * dot;
    }
}
// Bound on |approx_distance - the exact kernel's fp32 distance| (derivation in exact_tc_plan).  +inf where no bound holds:
// cos with a norm that is non-finite or so small that its fp32 sum is dominated by subnormal rounding.
constexpr float kCosMinNorm = 7.88860905e-31f; // 2^-100
template <int DM> __device__ __forceinline__ float approx_eps(const ExactTcEps& e, float qn, float xn) {
    const float a = sqrtf(qn), b = sqrtf(xn);
    const float dot_err = e.rel * a * b + e.lin * (a + b) + e.abs;
    if constexpr (DM == DM_COS) {
        if (qn == 0.f || xn == 0.f) // both sides take the same zero-norm branch (0 or 1, exactly)
            return e.rel + e.sum;
        if (!(qn >= kCosMinNorm && xn >= kCosMinNorm && qn <= FLT_MAX && xn <= FLT_MAX))
            return INFINITY;
        return dot_err / (a * b) + e.sum; // plus norms, square roots, the division and the exact kernel's own sums
    } else {
        return 2.f * dot_err + e.sum * (qn + xn); // plus norms, the final sum and the exact kernel's own sum
    }
}

template <int DM> __global__ void __launch_bounds__(kTcThreads, 1) exact_tc_filter_kernel(const __grid_constant__ TcParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    __shared__ __align__(8) uint64_t full_bar[kStages], empty_bar[kStages], afull_bar, aempty_bar;
    float* acc_s = reinterpret_cast<float*>(smem + kStages * kStageBytes); // [kTileM][kAccLd]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t qt = blockIdx.x / p.groups, g = blockIdx.x % p.groups;
    const uint32_t q0 = qt * kTileM;
    const uint32_t KB = (p.nchunks * 4 + kBlockK - 1) / kBlockK; // k-blocks per row
    const uint32_t my_tiles = g < p.row_tiles ? (p.row_tiles - g + p.groups - 1) / p.groups : 0;

    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < kStages; ++s) {
            mbar_init(&full_bar[s], 4);  // one arrive per producer warp
            mbar_init(&empty_bar[s], 8); // one arrive per MMA warp
        }
        mbar_init(&afull_bar, 8);  // one arrive per MMA warp: the accumulator tile is stored
        mbar_init(&aempty_bar, 4); // one arrive per epilogue warp: the accumulator tile is drained
        fence_mbar_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ===== producers: global fp32 -> (hi, lo) tf32 pairs in the core-matrix layout =====
        uint32_t it = 0;
        for (uint32_t t = 0; t < my_tiles; ++t) {
            const size_t row0 = (size_t)(g + t * p.groups) * kTileN;
            for (uint32_t kb = 0; kb < KB; ++kb, ++it) {
                const uint32_t s = it % kStages;
                uint8_t* st = smem + (size_t)s * kStageBytes;
                // A: 128 query rows and B: 128 corpus rows = 4 slabs of 32 rows each, one slab per producer warp; lane = row
                // within the slab.  All 16 16-byte loads of the k-block are issued before the first conversion (one memory
                // latency per k-block), and the thread's 128-byte line of the NEXT k-block is requested into L2 meanwhile.
                const uint32_t r = warp * 32 + lane, qa = q0 + r;
                const size_t row_b = row0 + r;
                const uint4* sa = reinterpret_cast<const uint4*>(p.queries + (size_t)qa * p.q_stride) + kb * 8;
                const uint4* sb = reinterpret_cast<const uint4*>(p.data + row_b * p.data_stride) + kb * 8;
                uint4 va[8], vb[8];
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const bool in_k = kb * 8 + c < p.nchunks;
                    va[c] = (qa < p.nq && in_k) ? __ldg(sa + c) : make_uint4(0, 0, 0, 0);
                    vb[c] = (row_b < p.n && in_k) ? __ldg(sb + c) : make_uint4(0, 0, 0, 0);
                }
                if ((kb + 1) * 8 < p.nchunks && row_b < p.n)
                    prefetch_l2(sb + 8);
                mbar_wait(&empty_bar[s], ((it / kStages) & 1u) ^ 1u); // (the loads above are already in flight)
                uint8_t* da = st + (r >> 3) * 1024 + (r & 7) * 16;
                uint8_t* db = st + 2 * kABytes + (r >> 3) * 1024 + (r & 7) * 16;
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    uint4 hi, lo;
                    split4(va[c], hi, lo);
                    *reinterpret_cast<uint4*>(da + c * 128) = hi;
                    *reinterpret_cast<uint4*>(da + kABytes + c * 128) = lo;
                    split4(vb[c], hi, lo);
                    *reinterpret_cast<uint4*>(db + c * 128) = hi;
                    *reinterpret_cast<uint4*>(db + kBBytes + c * 128) = lo;
                }
                fence_proxy_async(); // generic-proxy stores above -> visible to wgmma's async-proxy reads
                __syncwarp();
                if (lane == 0)
                    mbar_arrive(&full_bar[s]);
            }
        }
    } else if (warp < 12) {
        // ===== MMA: warpgroup wg multiplies queries 64 wg .. 64 wg + 63 of the tile by the tile's 128 rows =====
        const uint32_t wg = (uint32_t)(warp - 4) >> 2, wl = (uint32_t)(warp - 4) & 3u;
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i)
            acc[i] = 0.f;
        uint32_t it = 0;
        for (uint32_t t = 0; t < my_tiles; ++t) {
            for (uint32_t kb = 0; kb < KB; ++kb, ++it) {
                const uint32_t s = it % kStages;
                mbar_wait(&full_bar[s], (it / kStages) & 1u);
                const uint32_t a_hi = smem_u32(smem + (size_t)s * kStageBytes) + wg * 8 * 1024, a_lo = a_hi + kABytes;
                const uint32_t b_hi = smem_u32(smem + (size_t)s * kStageBytes) + 2 * kABytes, b_lo = b_hi + kBBytes;
                wgmma_fence();
#pragma unroll
                for (uint32_t kk = 0; kk < kBlockK / 8; ++kk) { // wgmma K = 8 tf32 = two 16-byte core-matrix columns
                    const uint32_t off = kk * 256;
                    const uint64_t dah = gmma_desc(a_hi + off, 128, 1024), dal = gmma_desc(a_lo + off, 128, 1024);
                    const uint64_t dbh = gmma_desc(b_hi + off, 128, 1024), dbl = gmma_desc(b_lo + off, 128, 1024);
                    wgmma_tf32_n128(acc, dah, dbh, (kb | kk) ? 1u : 0u);
                    wgmma_tf32_n128(acc, dah, dbl, 1u);
                    wgmma_tf32_n128(acc, dal, dbh, 1u);
                }
                wgmma_commit();
                wgmma_wait_all();
                __syncwarp();
                if (lane == 0)
                    mbar_arrive(&empty_bar[s]); // the stage may be refilled
            }
            // accumulator fragment -> shared tile: register 4j + {0,1} is (row, 8j + 2 (lane % 4) + {0,1}), 4j + {2,3} row + 8
            mbar_wait(&aempty_bar, (t & 1u) ^ 1u);
            const uint32_t row = wg * 64 + wl * 16 + (lane >> 2), col = 2 * (lane & 3);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                *reinterpret_cast<float2*>(acc_s + row * kAccLd + 8 * j + col) = make_float2(acc[4 * j], acc[4 * j + 1]);
                *reinterpret_cast<float2*>(acc_s + (row + 8) * kAccLd + 8 * j + col) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
            }
            __syncwarp();
            if (lane == 0)
                mbar_arrive(&afull_bar);
        }
    } else {
        // ===== epilogue: thread (warp, lane) owns query q0 + 32 * (warp - 12) + lane = row of the accumulator tile =====
        const uint32_t tq = (uint32_t)(warp - 12) * 32 + lane;
        const uint32_t q = q0 + tq;
        const bool live = q < p.nq;
        const float qn = live ? __ldg(p.qn + q) : 0.f;
        const float* arow = acc_s + tq * kAccLd;
        float ld[kMaxKP];
        uint32_t li[kMaxKP];
        uint32_t size = 0;
        const uint32_t KP = p.KP;
        float thr = INFINITY, dropped = INFINITY;
        for (uint32_t t = 0; t < my_tiles; ++t) {
            const size_t row0 = (size_t)(g + t * p.groups) * kTileN;
            mbar_wait(&afull_bar, t & 1u);
#pragma unroll 1
            for (uint32_t c0 = 0; c0 < kTileN; c0 += 32) {
                float r[32];
#pragma unroll
                for (int j = 0; j < 32; j += 4)
                    *reinterpret_cast<float4*>(r + j) = *reinterpret_cast<const float4*>(arow + c0 + j);
                if (live) {
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
                        const size_t row = row0 + c0 + j;
                        if (row < p.n) {
                            const float xn = __ldg(p.xn + row);
                            const float d = approx_distance<DM>(r[j], qn, xn);
                            if (d < thr && d > -INFINITY) {
                                // max-heap on the distance (root = the list's current worst, = thr once the list is full):
                                // log2(KP) steps per accepted row.  A sorted array costs KP/2 shifts per insert, and every
                                // insert of ANY lane stalls the whole warp.
                                uint32_t pos;
                                if (size < KP) {
                                    pos = size++;
                                    while (pos > 0) {
                                        const uint32_t par = (pos - 1) >> 1;
                                        if (ld[par] >= d)
                                            break;
                                        ld[pos] = ld[par], li[pos] = li[par];
                                        pos = par;
                                    }
                                } else { // replace the root; the evicted row is remembered through its lower bound
                                    dropped = fminf(dropped, ld[0] - approx_eps<DM>(p.eps, qn, __ldg(p.xn + li[0])));
                                    pos = 0;
                                    for (;;) {
                                        uint32_t c = 2 * pos + 1;
                                        if (c >= KP)
                                            break;
                                        if (c + 1 < KP && ld[c + 1] > ld[c])
                                            ++c;
                                        if (ld[c] <= d)
                                            break;
                                        ld[pos] = ld[c], li[pos] = li[c];
                                        pos = c;
                                    }
                                }
                                ld[pos] = d, li[pos] = (uint32_t)row;
                                if (size == KP)
                                    thr = ld[0];
                            } else {
                                // a NaN or infinite approximation bounds nothing (overflowed norms, NaN / inf components):
                                // -inf makes the query unsafe
                                const float lb = d - approx_eps<DM>(p.eps, qn, xn);
                                dropped = lb < INFINITY ? fminf(dropped, lb) : -INFINITY;
                            }
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0)
                mbar_arrive(&aempty_bar);
        }
        if (live) {
            float* od = p.cand_d + ((size_t)q * p.groups + g) * KP;
            uint32_t* oi = p.cand_i + ((size_t)q * p.groups + g) * KP;
            for (uint32_t i = 0; i < KP; ++i) {
                od[i] = i < size ? ld[i] : INFINITY;
                oi[i] = i < size ? li[i] : 0xFFFFFFFFu;
            }
            p.dropped_lb[(size_t)q * p.groups + g] = dropped;
        }
    }
}

// ---- re-rank: exact fp32 distances (exact.cu's arithmetic) of the candidates that can still be in the top k ----------
constexpr uint32_t kRrThreads = 256;
constexpr uint32_t kRrCap = 512; // candidates that survive the bound test, per query

struct RrParams {
    const uint8_t* data;
    size_t n, data_stride;
    const uint8_t* queries;
    uint32_t nq;
    size_t q_stride;
    uint32_t nchunks;
    const float* xn;
    const float* qn;
    uint32_t groups, KP, k;
    ExactTcEps eps;
    const float* cand_d;
    const uint32_t* cand_i;
    const float* dropped_lb;
    uint64_t* out_keys;
    float* out_dists;
    uint8_t* unsafe; // [nq] 1 = answer this query with the SIMT kernels instead
    uint32_t* unsafe_count;
};

__device__ __forceinline__ bool closer_rr(float d, uint32_t id, float od, uint32_t oid) { return closer_total(d, id, od, oid); }

template <int DM> __global__ void __launch_bounds__(kRrThreads) exact_tc_rerank_kernel(const RrParams p) {
    extern __shared__ __align__(16) uint8_t sm_raw[];
    const uint32_t q = blockIdx.x;
    const uint32_t C = p.groups * p.KP;
    uint32_t P2 = 1;
    while (P2 < C)
        P2 <<= 1;
    float* ub = reinterpret_cast<float*>(sm_raw);               // [P2] upper bounds, sorted to find the k-th
    float* sel_d = ub + P2;                                     // [kRrCap]
    uint32_t* sel_i = reinterpret_cast<uint32_t*>(sel_d + kRrCap); // [kRrCap]
    uint4* sq = reinterpret_cast<uint4*>(sel_i + kRrCap);       // [nchunks]
    __shared__ uint32_t nsel;
    __shared__ float kth_ub_s, sa2;
    __shared__ int bad;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float qn = p.qn[q];
    const float* cd = p.cand_d + (size_t)q * C;
    const uint32_t* ci = p.cand_i + (size_t)q * C;
    if (threadIdx.x == 0)
        nsel = 0, bad = 0;
    for (uint32_t i = threadIdx.x; i < P2; i += blockDim.x) {
        float u = INFINITY;
        if (i < C && ci[i] != 0xFFFFFFFFu)
            u = cd[i] + approx_eps<DM>(p.eps, qn, __ldg(p.xn + ci[i]));
        ub[i] = u;
    }
    for (uint32_t c = threadIdx.x; c < p.nchunks; c += blockDim.x)
        sq[c] = __ldg(reinterpret_cast<const uint4*>(p.queries + (size_t)q * p.q_stride) + c);
    __syncthreads();
    // bitonic sort of the upper bounds (ascending)
    for (uint32_t kk = 2; kk <= P2; kk <<= 1)
        for (uint32_t j = kk >> 1; j > 0; j >>= 1) {
            for (uint32_t i = threadIdx.x; i < P2; i += blockDim.x) {
                const uint32_t ixj = i ^ j;
                if (ixj > i) {
                    const float a = ub[i], b = ub[ixj];
                    const bool up = (i & kk) == 0;
                    if ((a > b) == up)
                        ub[i] = b, ub[ixj] = a;
                }
            }
            __syncthreads();
        }
    if (threadIdx.x == 0)
        kth_ub_s = p.k <= P2 ? ub[p.k - 1] : INFINITY; // +inf when fewer than k candidates exist: everything qualifies
    __syncthreads();
    const float kth_ub = kth_ub_s;
    // anything a list dropped that could still qualify makes the query unsafe (+inf: the list dropped nothing, which also
    // holds when fewer than k candidates exist and kth_ub is +inf)
    for (uint32_t gI = threadIdx.x; gI < p.groups; gI += blockDim.x) {
        const float lb = p.dropped_lb[(size_t)q * p.groups + gI];
        if (lb <= kth_ub && lb < INFINITY)
            bad = 1;
    }
    // survivors
    for (uint32_t i = threadIdx.x; i < C; i += blockDim.x) {
        const uint32_t id = ci[i];
        if (id == 0xFFFFFFFFu)
            continue;
        const float lb = cd[i] - approx_eps<DM>(p.eps, qn, __ldg(p.xn + id));
        if (lb <= kth_ub) {
            const uint32_t at = atomicAdd(&nsel, 1u);
            if (at < kRrCap)
                sel_i[at] = id;
            else
                bad = 1;
        }
    }
    __syncthreads();
    const uint32_t ns = min(nsel, kRrCap);
    if (bad || ns < min((size_t)p.k, p.n)) {
        if (threadIdx.x == 0) {
            p.unsafe[q] = 1;
            atomicAdd(p.unsafe_count, 1u);
        }
        return;
    }
    if (threadIdx.x == 0)
        p.unsafe[q] = 0;
    // exact distances: one warp per survivor, exact.cu's lane layout (lane l owns chunks l, l+32, ...)
    if (DM == DM_COS) {
        if (warp == 0) {
            float part = 0.f;
            for (uint32_t c = lane; c < p.nchunks; c += 32)
                part = norm_add(part, query_norm_chunk<DM, SK_F32>(sq[c]));
            part = warp_sum(part);
            if (lane == 0)
                sa2 = part;
        }
        __syncthreads();
    }
    for (uint32_t s = warp; s < ns; s += kRrThreads / 32) {
        const uint4* rp = reinterpret_cast<const uint4*>(p.data + (size_t)sel_i[s] * p.data_stride);
        DistAcc<DM, SK_F32> acc;
        acc.reset();
        for (uint32_t c = lane; c < p.nchunks; c += 32)
            accum_chunk<DM, SK_F32>(acc, sq[c], __ldg(rp + c));
        const float d = finish_distance<DM, SK_F32>(acc, DM == DM_COS ? sa2 : 0.f);
        if (lane == 0)
            sel_d[s] = d;
    }
    __syncthreads();
    // rank by (distance, offset): the survivor at rank r < k is output r.  O(ns^2 / threads), ns is a few dozen.
    for (uint32_t s = threadIdx.x; s < ns; s += blockDim.x) {
        const float d = sel_d[s];
        const uint32_t id = sel_i[s];
        uint32_t rank = 0;
        for (uint32_t t = 0; t < ns; ++t)
            rank += closer_rr(sel_d[t], sel_i[t], d, id) ? 1u : 0u;
        if (rank < p.k) {
            p.out_keys[(size_t)q * p.k + rank] = id;
            p.out_dists[(size_t)q * p.k + rank] = d;
        }
    }
    for (uint32_t r = ns + threadIdx.x; r < p.k; r += blockDim.x) { // fewer rows than k
        p.out_keys[(size_t)q * p.k + r] = ~0ull;
        p.out_dists[(size_t)q * p.k + r] = INFINITY;
    }
}

} // namespace

bool exact_tc_defined(int dist_mode, int scalar_kind, size_t n, size_t k) {
    return scalar_kind == SK_F32 && (dist_mode == DM_L2SQ || dist_mode == DM_COS) && k <= 192 && n && n < 0xFFFFFFFFull;
}

bool exact_tc_applicable(int dist_mode, int scalar_kind, size_t n, size_t nq, size_t k, uint32_t row_bytes) {
    if (const char* e = getenv("LB200_EXACT")) {
        if (e[0] == 's') // "simt"
            return false;
        if (e[0] == 't') // "tc": force (still only where it is defined)
            return exact_tc_defined(dist_mode, scalar_kind, n, k) && nq;
    }
    // the tensor-core pass pays off once the problem is a real GEMM
    return exact_tc_defined(dist_mode, scalar_kind, n, k) && n >= 32768 && nq >= 16 && row_bytes >= 128;
}

ExactTcPlan exact_tc_plan(size_t n, size_t nq, size_t k, uint32_t row_bytes) {
    const uint32_t nchunks = row_bytes / 16, dims = row_bytes / 4;
    const uint32_t q_tiles = (uint32_t)((nq + kTileM - 1) / kTileM);
    const uint32_t row_tiles = (uint32_t)((n + kTileN - 1) / kTileN);
    ExactTcPlan pl{};
    pl.KP = std::min<uint32_t>((uint32_t)round_up(k + std::max<size_t>(32, k / 2), 32), kMaxKP);
    pl.groups = std::min(std::max<uint32_t>(1, (uint32_t)device_sm_count() / q_tiles), row_tiles);
    // The re-rank bitonic-sorts next_pow2(groups * KP) upper bounds in shared memory.  With one query tile on a 132-SM H100
    // SXM and KP = 256 (k >= 150) that is 65536 floats, over the 227 KB opt-in limit; capping groups at 128 (4 SMs idle in
    // that case only) keeps the filter's occupancy and the sort's cost.
    int dev = 0, optin = 0;
    LB_CUDA(cudaGetDevice(&dev));
    LB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    cudaFuncAttributes fa_cos{}, fa_l2{}; // the dynamic request may use what the kernel's static __shared__ leaves
    LB_CUDA(cudaFuncGetAttributes(&fa_cos, exact_tc_rerank_kernel<DM_COS>));
    LB_CUDA(cudaFuncGetAttributes(&fa_l2, exact_tc_rerank_kernel<DM_L2SQ>));
    const size_t rr_static = std::max(fa_cos.sharedSizeBytes, fa_l2.sharedSizeBytes);
    size_t p2max = 1;
    while ((p2max * 2) * 4 + (size_t)kRrCap * 8 + row_bytes + rr_static <= (size_t)optin)
        p2max *= 2;
    pl.groups = std::max<uint32_t>(1, std::min<uint32_t>(pl.groups, (uint32_t)(p2max / pl.KP)));
    // |approx - exact| where u = 2^-24, L = chunks per lane and both sides are fp32:
    //  rel  3xTF32 drops lo*lo and lo's own rounding (3 * 2^-22 |q_i x_i|) and accumulates 3 dims / 8 MMAs into fp32 (about
    //       dims u with truncating adds): (dims + 32) u |q||x|
    //  sum  every fp32 sum here (norms_kernel, exact.cu's sum of (q-x)^2 or of q.x and |x|^2) rounds a term at most L + 9
    //       times (4 inside a chunk, L along the lane, 5 in the butterfly); with the exact distance <= 2 (|q|^2 + |x|^2)
    //       and the final two operations that is (3 L + 29) u (|q|^2 + |x|^2) for l2sq, about (3 L + 33) u for cos.
    //       (3 L + 48) u keeps 3e-6 at L = 1.
    //  lin, abs  the tensor cores may flush subnormal inputs, products and partial sums, each below 2^-126:
    //       2^-126 (sqrt(dims) (|q| + |x|) + 6 dims) with the two sides' subnormal roundings, rounded up to 8 dims
    const uint32_t L = (nchunks + 31) / 32;
    const float u = 5.9604645e-8f, tiny = 1.17549435e-38f; // 2^-24, 2^-126
    pl.eps.rel = (float)(dims + 32) * u;
    pl.eps.sum = (float)(3 * L + 48) * u;
    pl.eps.lin = sqrtf((float)dims) * tiny;
    pl.eps.abs = (float)(8 * dims) * tiny;
    return pl;
}

// Returns the device array of per-query "unsafe" flags (owned by the caller, freed with cudaFreeAsync by the caller) so that
// launch_exact can run the SIMT kernels for exactly those queries.  On an error everything it allocated is freed.
void launch_exact_tc(int dist_mode, const uint8_t* d_data, size_t n, size_t data_stride, const uint8_t* d_queries, size_t nq,
                     size_t q_stride, uint32_t row_bytes, size_t k, uint64_t* d_keys, float* d_dists, uint8_t** d_unsafe,
                     uint32_t** d_unsafe_count, cudaStream_t stream, const ExactTcProbe* probe) {
    const uint32_t nchunks = row_bytes / 16;
    const ExactTcPlan pl = exact_tc_plan(n, nq, k, row_bytes);
    const uint32_t groups = pl.groups, KP = pl.KP;
    const uint32_t q_tiles = (uint32_t)((nq + kTileM - 1) / kTileM);
    const uint32_t row_tiles = (uint32_t)((n + kTileN - 1) / kTileN);

    float *xn = nullptr, *qn = nullptr, *cand_d = nullptr, *dropped = nullptr;
    uint32_t* cand_i = nullptr;
    *d_unsafe = nullptr, *d_unsafe_count = nullptr;
    try {
        LB_CUDA(cudaMallocAsync(&xn, n * sizeof(float), stream));
        LB_CUDA(cudaMallocAsync(&qn, nq * sizeof(float), stream));
        LB_CUDA(cudaMallocAsync(&cand_d, nq * groups * KP * sizeof(float), stream));
        LB_CUDA(cudaMallocAsync(&cand_i, nq * groups * KP * sizeof(uint32_t), stream));
        LB_CUDA(cudaMallocAsync(&dropped, nq * groups * sizeof(float), stream));
        LB_CUDA(cudaMallocAsync(d_unsafe, nq, stream));
        LB_CUDA(cudaMallocAsync(d_unsafe_count, sizeof(uint32_t), stream));
        LB_CUDA(cudaMemsetAsync(*d_unsafe_count, 0, sizeof(uint32_t), stream));
        norms_kernel<<<(unsigned)((n + 7) / 8), 256, 0, stream>>>(d_data, n, data_stride, nchunks, xn);
        norms_kernel<<<(unsigned)((nq + 7) / 8), 256, 0, stream>>>(d_queries, nq, q_stride, nchunks, qn);
        count_launch(2);

        TcParams p{};
        p.data = d_data, p.n = n, p.data_stride = data_stride;
        p.queries = d_queries, p.nq = (uint32_t)nq, p.q_stride = q_stride, p.nchunks = nchunks;
        p.xn = xn, p.qn = qn, p.groups = groups, p.row_tiles = row_tiles, p.KP = KP, p.eps = pl.eps;
        p.cand_d = cand_d, p.cand_i = cand_i, p.dropped_lb = dropped;
        RrParams r{};
        r.data = d_data, r.n = n, r.data_stride = data_stride, r.queries = d_queries, r.nq = (uint32_t)nq, r.q_stride = q_stride;
        r.nchunks = nchunks, r.xn = xn, r.qn = qn, r.groups = groups, r.KP = KP, r.k = (uint32_t)k, r.eps = pl.eps;
        r.cand_d = cand_d, r.cand_i = cand_i, r.dropped_lb = dropped, r.out_keys = d_keys, r.out_dists = d_dists;
        r.unsafe = *d_unsafe, r.unsafe_count = *d_unsafe_count;
        uint32_t P2 = 1;
        while (P2 < groups * KP)
            P2 <<= 1;
        const size_t rr_smem = (size_t)P2 * 4 + (size_t)kRrCap * 8 + row_bytes;
        auto run = [&](auto dm) {
            constexpr int DM = decltype(dm)::value;
            auto fk = exact_tc_filter_kernel<DM>;
            LB_CUDA(cudaFuncSetAttribute(fk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTcSmem));
            fk<<<q_tiles * groups, kTcThreads, kTcSmem, stream>>>(p);
            LB_CUDA(cudaGetLastError());
            auto rk = exact_tc_rerank_kernel<DM>;
            LB_CUDA(cudaFuncSetAttribute(rk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rr_smem));
            rk<<<(unsigned)nq, kRrThreads, rr_smem, stream>>>(r);
            LB_CUDA(cudaGetLastError());
            count_launch(2);
        };
        if (dist_mode == DM_COS)
            run(std::integral_constant<int, DM_COS>{});
        else
            run(std::integral_constant<int, DM_L2SQ>{});
        if (probe) {
            const size_t nc = nq * groups * KP;
            LB_CUDA(cudaMemcpyAsync(probe->qn, qn, nq * sizeof(float), cudaMemcpyDeviceToHost, stream));
            LB_CUDA(cudaMemcpyAsync(probe->xn, xn, n * sizeof(float), cudaMemcpyDeviceToHost, stream));
            LB_CUDA(cudaMemcpyAsync(probe->cand_d, cand_d, nc * sizeof(float), cudaMemcpyDeviceToHost, stream));
            LB_CUDA(cudaMemcpyAsync(probe->cand_i, cand_i, nc * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
            LB_CUDA(cudaMemcpyAsync(probe->dropped_lb, dropped, nq * groups * sizeof(float), cudaMemcpyDeviceToHost, stream));
            LB_CUDA(cudaMemcpyAsync(probe->unsafe, *d_unsafe, nq, cudaMemcpyDeviceToHost, stream));
            LB_CUDA(cudaStreamSynchronize(stream));
        }
    } catch (...) {
        (void)cudaGetLastError(); // a refused launch configuration must not fail the caller's next, unrelated launch
        for (void* b : {(void*)xn, (void*)qn, (void*)cand_d, (void*)cand_i, (void*)dropped, (void*)*d_unsafe, (void*)*d_unsafe_count})
            if (b)
                cudaFreeAsync(b, stream);
        *d_unsafe = nullptr, *d_unsafe_count = nullptr;
        throw;
    }
    LB_CUDA(cudaFreeAsync(xn, stream));
    LB_CUDA(cudaFreeAsync(qn, stream));
    LB_CUDA(cudaFreeAsync(cand_d, stream));
    LB_CUDA(cudaFreeAsync(cand_i, stream));
    LB_CUDA(cudaFreeAsync(dropped, stream));
}

} // namespace lb200

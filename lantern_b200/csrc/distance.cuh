// lantern_b200 -- distance arithmetic shared by the search / exact / build kernels.
//
// GPU counterpart of the reference's scalar metric loops
//   metric_l2sq_gt  U/include/usearch/index_plugins.hpp:1034-1051   sum (a-b)^2, fp32 accumulate
//   metric_cos_gt   :1004-1028   1 - ab/(sqrt(a2) sqrt(b2)), zero-norm table [a2==0][b2==0] -> {.,1;1,0}
//   metric_hamming_gt<b1x8_t> :1058-1081   popcount(a^b) over ceil(bits/8) bytes, returned as float
// for the storage scalar kinds f32 / f16 / i8 / b1 (dispatch :1446-1522; i8 and f16 operands are
// promoted to f32 *values* -- i8 distances therefore live in the x100 integer domain, :938,950).
//
// A vector row is a sequence of 16-byte chunks; lane l of a warp owns chunks l, l+32, l+64, ...
// Each lane accumulates partials over its chunks, then the warp butterfly-reduces.  Rows and
// queries are zero-padded to a multiple of 16 bytes, which contributes 0 to every metric.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace lb200 {

template <int DM, int SK> struct DistAcc {
    float v[4];
    __device__ __forceinline__ void reset() { v[0] = v[1] = v[2] = v[3] = 0.f; }
};
template <int DM> struct DistAcc<DM, SK_I8> { // exact int32 dot products (dp4a)
    int v[4];
    __device__ __forceinline__ void reset() { v[0] = v[1] = v[2] = v[3] = 0; }
};
template <> struct DistAcc<DM_HAMMING, SK_B1> {
    uint32_t v[4];
    __device__ __forceinline__ void reset() { v[0] = v[1] = v[2] = v[3] = 0u; }
};

// ---- accumulate one 16-byte chunk: q = query chunk, r = stored-row chunk ---------------------------
template <int DM, int SK> __device__ __forceinline__ void accum_chunk(DistAcc<DM, SK>& a, const uint4& q, const uint4& r);

template <> __device__ __forceinline__ void accum_chunk<DM_L2SQ, SK_F32>(DistAcc<DM_L2SQ, SK_F32>& a, const uint4& q, const uint4& r) {
    float d0 = __uint_as_float(q.x) - __uint_as_float(r.x);
    float d1 = __uint_as_float(q.y) - __uint_as_float(r.y);
    float d2 = __uint_as_float(q.z) - __uint_as_float(r.z);
    float d3 = __uint_as_float(q.w) - __uint_as_float(r.w);
    a.v[0] = fmaf(d0, d0, a.v[0]);
    a.v[1] = fmaf(d1, d1, a.v[1]);
    a.v[2] = fmaf(d2, d2, a.v[2]);
    a.v[3] = fmaf(d3, d3, a.v[3]);
}
// cos / ip: v[0],v[1] = partial ab ; v[2],v[3] = partial b2 (norm of the STORED row)
template <> __device__ __forceinline__ void accum_chunk<DM_COS, SK_F32>(DistAcc<DM_COS, SK_F32>& a, const uint4& q, const uint4& r) {
    float q0 = __uint_as_float(q.x), q1 = __uint_as_float(q.y), q2 = __uint_as_float(q.z), q3 = __uint_as_float(q.w);
    float r0 = __uint_as_float(r.x), r1 = __uint_as_float(r.y), r2 = __uint_as_float(r.z), r3 = __uint_as_float(r.w);
    a.v[0] = fmaf(q0, r0, a.v[0]);
    a.v[1] = fmaf(q1, r1, a.v[1]);
    a.v[0] = fmaf(q2, r2, a.v[0]);
    a.v[1] = fmaf(q3, r3, a.v[1]);
    a.v[2] = fmaf(r0, r0, a.v[2]);
    a.v[3] = fmaf(r1, r1, a.v[3]);
    a.v[2] = fmaf(r2, r2, a.v[2]);
    a.v[3] = fmaf(r3, r3, a.v[3]);
}

__device__ __forceinline__ float2 h2f(uint32_t w) {
    __half2 h = *reinterpret_cast<const __half2*>(&w);
    return __half22float2(h);
}
template <> __device__ __forceinline__ void accum_chunk<DM_L2SQ, SK_F16>(DistAcc<DM_L2SQ, SK_F16>& a, const uint4& q, const uint4& r) {
    const uint32_t qw[4] = {q.x, q.y, q.z, q.w}, rw[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float2 x = h2f(qw[i]), y = h2f(rw[i]);
        float d0 = x.x - y.x, d1 = x.y - y.y;
        a.v[(2 * i) & 3] = fmaf(d0, d0, a.v[(2 * i) & 3]);
        a.v[(2 * i + 1) & 3] = fmaf(d1, d1, a.v[(2 * i + 1) & 3]);
    }
}
template <> __device__ __forceinline__ void accum_chunk<DM_COS, SK_F16>(DistAcc<DM_COS, SK_F16>& a, const uint4& q, const uint4& r) {
    const uint32_t qw[4] = {q.x, q.y, q.z, q.w}, rw[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float2 x = h2f(qw[i]), y = h2f(rw[i]);
        a.v[0] = fmaf(x.x, y.x, a.v[0]);
        a.v[1] = fmaf(x.y, y.y, a.v[1]);
        a.v[2] = fmaf(y.x, y.x, a.v[2]);
        a.v[3] = fmaf(y.y, y.y, a.v[3]);
    }
}
// i8: exact integer arithmetic; sum (a-b)^2 = a.a - 2 a.b + b.b
template <> __device__ __forceinline__ void accum_chunk<DM_L2SQ, SK_I8>(DistAcc<DM_L2SQ, SK_I8>& a, const uint4& q, const uint4& r) {
    const int qw[4] = {(int)q.x, (int)q.y, (int)q.z, (int)q.w}, rw[4] = {(int)r.x, (int)r.y, (int)r.z, (int)r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        a.v[0] = __dp4a(qw[i], qw[i], a.v[0]);
        a.v[1] = __dp4a(rw[i], rw[i], a.v[1]);
        a.v[2] = __dp4a(qw[i], rw[i], a.v[2]);
    }
}
template <> __device__ __forceinline__ void accum_chunk<DM_COS, SK_I8>(DistAcc<DM_COS, SK_I8>& a, const uint4& q, const uint4& r) {
    const int qw[4] = {(int)q.x, (int)q.y, (int)q.z, (int)q.w}, rw[4] = {(int)r.x, (int)r.y, (int)r.z, (int)r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        a.v[0] = __dp4a(qw[i], rw[i], a.v[0]);
        a.v[2] = __dp4a(rw[i], rw[i], a.v[2]);
    }
}
template <> __device__ __forceinline__ void accum_chunk<DM_HAMMING, SK_B1>(DistAcc<DM_HAMMING, SK_B1>& a, const uint4& q, const uint4& r) {
    a.v[0] += __popc(q.x ^ r.x);
    a.v[1] += __popc(q.y ^ r.y);
    a.v[2] += __popc(q.z ^ r.z);
    a.v[3] += __popc(q.w ^ r.w);
}

// ---- query-side constant (cos: a2 = |q|^2), computed once per query with the same lane layout ------
// Explicitly rounded operations (no fp contraction left to the compiler): every kernel that folds these chunk sums in the
// same order (search.cu, group.cu, exact.cu, exact_tc.cu) then produces the SAME bits for |q|^2, which is what makes the
// multi-GPU group's distances bit-identical to the 1-GPU kernel's.
template <int DM, int SK> __device__ __forceinline__ float query_norm_chunk(const uint4& q) {
    if constexpr (DM != DM_COS)
        return 0.f;
    else if constexpr (SK == SK_F32) {
        float q0 = __uint_as_float(q.x), q1 = __uint_as_float(q.y), q2 = __uint_as_float(q.z), q3 = __uint_as_float(q.w);
        return __fmaf_rn(q3, q3, __fmaf_rn(q2, q2, __fmaf_rn(q1, q1, __fmul_rn(q0, q0))));
    } else if constexpr (SK == SK_F16) {
        const uint32_t qw[4] = {q.x, q.y, q.z, q.w};
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float2 x = h2f(qw[i]);
            s = __fmaf_rn(x.y, x.y, __fmaf_rn(x.x, x.x, s));
        }
        return s;
    } else if constexpr (SK == SK_I8) {
        int s = 0;
        s = __dp4a((int)q.x, (int)q.x, s);
        s = __dp4a((int)q.y, (int)q.y, s);
        s = __dp4a((int)q.z, (int)q.z, s);
        s = __dp4a((int)q.w, (int)q.w, s);
        return (float)s;
    } else
        return 0.f;
}
__device__ __forceinline__ float norm_add(float acc, float chunk) { return __fadd_rn(acc, chunk); }

__device__ __forceinline__ float cos_from_parts(float ab, float a2, float b2) {
    // index_plugins.hpp:1022-1026
    if (a2 == 0.f && b2 == 0.f)
        return 0.f;
    if (a2 == 0.f || b2 == 0.f)
        return 1.f;
    return 1.f - ab / (sqrtf(a2) * sqrtf(b2));
}

// Order of the exhaustive search's results: by distance, ties by lower offset; a NaN distance (a row or query holding NaN
// or opposite infinities) ranks after every number, +inf included, as in numpy's sort.  A plain `<` would let a NaN enter
// a sorted list anywhere and stay there.
template <typename I> __device__ __forceinline__ bool closer_total(float d, I id, float od, I oid) {
    if (d != d || od != od)
        return od != od && (d == d || id < oid);
    return d < od || (d == od && id < oid);
}

// ---- warp-reduce the partials into the final distance (all lanes receive it) ------------------------
template <int DM, int SK> __device__ __forceinline__ float finish_distance(const DistAcc<DM, SK>& a, float a2) {
    if constexpr (DM == DM_HAMMING) {
        return (float)warp_sum_u32(a.v[0] + a.v[1] + a.v[2] + a.v[3]);
    } else if constexpr (SK == SK_I8) {
        if constexpr (DM == DM_L2SQ) {
            // |q|^2 and |r|^2 are below 2^32 and q.r within int32 up to 131071 dimensions (the exhaustive search and the
            // pair distances refuse wider i8 rows); their combination reaches 255^2 d and is formed in 64 bits
            const uint32_t qq = warp_sum_u32((uint32_t)a.v[0]);
            const uint32_t rr = warp_sum_u32((uint32_t)a.v[1]);
            const int qr = (int)warp_sum_u32((uint32_t)a.v[2]);
            return (float)((long long)qq + (long long)rr - 2ll * qr);
        } else {
            float ab = (float)(int)warp_sum_u32((uint32_t)a.v[0]);
            float b2 = (float)(int)warp_sum_u32((uint32_t)a.v[2]);
            return cos_from_parts(ab, a2, b2);
        }
    } else if constexpr (DM == DM_L2SQ) {
        return warp_sum((a.v[0] + a.v[1]) + (a.v[2] + a.v[3]));
    } else { // cos
        float ab = warp_sum(a.v[0] + a.v[1]);
        float b2 = warp_sum(a.v[2] + a.v[3]);
        return cos_from_parts(ab, a2, b2);
    }
}

// Which specialisation serves an index: b1 storage forces hamming whatever the metric
// (index_plugins.hpp:1465,1477); hamming metric always works on bytes.
inline int distance_mode(int metric_kind, int scalar_kind) {
    if (scalar_kind == SK_B1 || metric_kind == MK_HAMMING)
        return DM_HAMMING;
    if (metric_kind == MK_COS)
        return DM_COS;
    return DM_L2SQ;
}

} // namespace lb200

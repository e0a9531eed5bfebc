// lantern_b200 -- int8 screen of the search beam: a cheap, provable lower bound on the fp32 distance the search kernel computes.
//
// f32 l2sq / cos indexes keep a companion copy of every stored row (engine.h): int8 codes c with a per-row scale s
// (x^ = s c) and sq_meta = {s, r >= |x - x^|, b2 = the kernel's own fp32 |x|^2, |c|}.  In the level-0 beam of a search, once
// the top list is full, a candidate can change the walk only if its distance d < radius.  screen_bound() returns lb <= d
// (d = the fp32 number row_distance() would return for that row, rounding included), so a candidate with lb >= radius is
// rejected without reading its fp32 row: the walk takes the same decisions, and results stay bit-identical.  DESIGN.md 4.1
// derives the bound; every term below is named after it.
#pragma once
#include <math.h>

#include "distance.cuh"

namespace lb200 {

// bytes of one code row: one int8 per dimension, words laid out like the 16-byte chunks of the fp32 row (word w = dims
// 4w..4w+3, so lane l owns words l, l+32, ... exactly as it owns fp32 chunks), padded to 16 bytes for the bulk copy
LB_HD inline uint32_t screen_code_bytes(uint32_t row_bytes) { return (row_bytes / 4 + 15u) & ~15u; }

#ifdef __CUDACC__
// unit roundoff of fp32, and gamma(n) >= n u / (1 - n u), the relative error bound of n chained roundings (n u < 2^-10)
constexpr double kU32 = 5.9604644775390625e-08; // 2^-24
__device__ __forceinline__ double gamma32(int n) { return (double)(n + 1) * kU32; }
// absolute error of one fp32 warp sum from roundings in the subnormal range: each rounding is off by <= 2^-150 and no sum here
// has more than 2^13 of them across the warp (2^-137 in all); 2^-120 keeps a wide margin and is still far below any distance
// the screen can reject with
constexpr double kSubAbs = 0x1p-120;

// sum over the row of q_i c_i (cos) or (q_i - s c_i)^2 (l2sq), fp32, lane layout of row_distance(); `words` = the code row
template <int DM, int NQ>
__device__ __forceinline__ float screen_sum(const uint4 (&qreg)[NQ], const uint32_t* words, float scale, uint32_t nchunks, int lane) {
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < NQ; ++i) {
        const uint32_t c = lane + 32 * i;
        if (c < nchunks) {
            const uint32_t w = words[c];
            const float qv[4] = {__uint_as_float(qreg[i].x), __uint_as_float(qreg[i].y), __uint_as_float(qreg[i].z),
                                 __uint_as_float(qreg[i].w)};
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                const float cv = (float)(int8_t)(w >> (8 * b));
                if constexpr (DM == DM_COS) {
                    acc = __fmaf_rn(qv[b], cv, acc);
                } else {
                    const float t = __fmaf_rn(-scale, cv, qv[b]);
                    acc = __fmaf_rn(t, t, acc);
                }
            }
        }
    }
    return warp_sum(acc);
}

// lb <= the distance row_distance<DM, SK_F32, NQ> computes for the same query (registers, a2) and row.  -inf or NaN = "cannot
// tell" (zero norms, non-finite data, overflow): the caller keeps a candidate unless lb >= radius.
template <int DM, int NQ> __device__ __forceinline__ float screen_bound(float s, float4 meta, float a2) {
    const float scale = meta.x, r = meta.y, b2 = meta.z, cnorm = meta.w;
    if (!(r < INFINITY) || !(s < INFINITY) || !(s > -INFINITY))
        return -INFINITY;
    if constexpr (DM == DM_COS) {
        // cos_from_parts' zero-norm branches; non-finite norms; and norms so large that a partial sum of the kernel's dot
        // product could overflow (below 2^126 each, every partial sum stays under |q||x| (1 + gamma) < 2^127)
        if (!(a2 > 0.f) || !(b2 > 0.f) || !(a2 < 0x1p126f) || !(b2 < 0x1p126f))
            return -INFINITY;
        // (a) |q| from the kernel's own fp32 a2: NQ + 9 roundings of non-negative terms
        const double qn = sqrt(((double)a2 + kSubAbs) * (1.0 + gamma32(NQ + 9))) * (1.0 + 0x1p-50);
        // (b) the row: |x^| <= s |c|, |x| <= |x^| + r
        const double xh = (double)scale * (double)cnorm;
        // U >= the kernel's fp32 dot product q.x (a real number):
        //   q.x   <= s sum(q_i c_i) + |q| r                                  (Cauchy-Schwarz on x - x^)
        //   screen: |s_f - sum(q_i c_i)| <= gamma(4 NQ + 5) |q||c| + kSubAbs  (fp32 sum of the screen)
        //   kernel: |ab_k - q.x| <= gamma(2 NQ + 6) |q||x| + kSubAbs         (fp32 sum of accum_chunk + finish_distance)
        const double A = (double)scale * (double)s; // exact: 24 x 24 bits
        const double B = qn * (r + gamma32(4 * NQ + 5) * xh + gamma32(2 * NQ + 6) * (xh + r)) + (double)scale * kSubAbs + kSubAbs;
        const double Bp = B * (1.0 + 0x1p-45); // the double roundings of B
        const float U = __double2float_ru((A + Bp) + (fabs(A) + Bp) * 0x1p-50);
        // (c) the final arithmetic, replayed: cos_from_parts with the same fp32 a2, b2, so the same rounded denominator.  Rounding
        // is monotone, so fl(1 - fl(U / D)) <= fl(1 - fl(ab_k / D)) for every ab_k <= U.
        return __fsub_rn(1.f, __fdiv_rn(U, __fmul_rn(sqrtf(a2), sqrtf(b2))));
    } else {
        // (a) |q - x^| from the screen's fp32 sum of squares (4 NQ + 5 roundings of non-negative terms, plus the rounding of each
        // t_i = fl(q_i - s c_i): relative u, or 2^-150 absolute when subnormal -> Minkowski: 2^-150 sqrt(dims) <= 2^-144)
        const double sum_lo = fmax((double)s - kSubAbs, 0.0) / (1.0 + gamma32(4 * NQ + 5));
        const double e_lo = ((sqrt(sum_lo) * (1.0 - 0x1p-48)) - 0x1p-144) / (1.0 + kU32);
        // (b) |q - x| >= |q - x^| - r
        const double L = fmax(e_lo - (double)r, 0.0);
        // (c) the kernel's sum: fl(q_i - x_i) (relative u; exact when subnormal), squared, NQ fma + 2 adds + 5 shuffles, all
        // non-negative terms: d >= (1 - gamma(NQ + 9)) |q - x|^2 - kSubAbs
        const double lb = L * L * (1.0 - gamma32(NQ + 9)) * (1.0 - 0x1p-46) - kSubAbs;
        return __double2float_rd(lb);
    }
}
#endif

// ---- the projected screen (DESIGN.md 4.1): k int8 codes of y = P x instead of one per dimension -------------------------
// P is a k x dims fp32 basis chosen per index (pscreen.cu); nothing below assumes it is orthonormal, so any P gives a valid
// bound.  One record per row: ps_meta = {s, E >= |e|, F >= |P e|, b2} (e = x - P^T s c), then `ps_code_slots` int8 codes
// (zero beyond k).  b2 is the kernel's own fp32 |x|^2 (cos) or a rounded-down |x|^2 (l2sq).
LB_HD inline uint32_t ps_record_bytes(uint32_t k) { return k <= 48 ? 64u : 128u; }
LB_HD inline uint32_t ps_code_slots(uint32_t k) { return ps_record_bytes(k) - 16u; }
// per query, written once per batch: q~ = fl(P q) in `ps_code_slots` floats (zero beyond k), then
// {delta >= |P q - q~|, >= |q~|, G >= |q - P^T q~|, <= |q|^2}
LB_HD inline uint32_t ps_query_floats(uint32_t k) { return ps_code_slots(k) + 4u; }

#ifdef __CUDACC__
// lb <= the distance row_distance<DM, SK_F32, NQ> computes for the query (registers, a2) and the row, from
//   sf = fl(sum_j q~_j c_j) (`slots` chained fma), cc = sum_j c_j^2 (exact in fp32: < 2^24), the row's meta, the query's header.
// q.x = q~.y^ + (Pq - q~).y^ + q~.(P e) + (q - P^T q~).e  <=  s sf + screen rounding + delta |y^| + |q~| F + G E  (y^ = s c)
template <int DM, int NQ>
__device__ __forceinline__ float pscreen_bound(float sf, float cc, float4 meta, float4 qh, float a2, uint32_t slots) {
    const double s = meta.x, E = meta.y, F = meta.z;
    const float b2 = meta.w;
    const double cn = sqrt((double)cc) * (1.0 + 0x1p-50);    // |c|
    const double qt = qh.y;                                   // >= |q~|
    const double A = s * (double)sf;                          // exact: 24 x 24 bits
    // screen: |sf - q~.c| <= gamma(slots) |q~||c| + kSubAbs; then delta |y^|, |q~| F, G E
    double B = s * (gamma32((int)slots) * qt * cn + kSubAbs) + (double)qh.x * (s * cn) + qt * F + (double)qh.z * E;
    if constexpr (DM == DM_COS) {
        if (!(a2 > 0.f) || !(b2 > 0.f) || !(a2 < 0x1p126f) || !(b2 < 0x1p126f))
            return -INFINITY;
        // the kernel's fp32 dot product: |ab_k - q.x| <= gamma(2 NQ + 6) |q||x| + kSubAbs, |q|, |x| from its own a2, b2
        const double qn = sqrt(((double)a2 + kSubAbs) * (1.0 + gamma32(NQ + 9))) * (1.0 + 0x1p-50);
        const double xn = sqrt(((double)b2 + kSubAbs) * (1.0 + gamma32(NQ + 9))) * (1.0 + 0x1p-50);
        B += gamma32(2 * NQ + 6) * qn * xn + kSubAbs;
    }
    if (!(fabs(A) < INFINITY) || !(B < INFINITY)) // NaN / inf anywhere (non-finite data, overflow): cannot tell
        return -INFINITY;
    const double Bp = B * (1.0 + 0x1p-45); // the double roundings of B
    const double U = (A + Bp) + (fabs(A) + Bp) * 0x1p-50;
    if constexpr (DM == DM_COS) {
        // the final arithmetic replayed, as screen_bound does
        return __fsub_rn(1.f, __fdiv_rn(__double2float_ru(U), __fmul_rn(sqrtf(a2), sqrtf(b2))));
    } else {
        // |q - x|^2 = |q|^2 - 2 q.x + |x|^2 >= qq - 2U + b2 (three double roundings bounded below), then the kernel's sum as in
        // screen_bound: d >= (1 - gamma(NQ + 9)) |q - x|^2 - kSubAbs
        const double qq = qh.w;
        const double D = (qq - 2.0 * U) + (double)b2;
        const double L2 = D - (qq + 2.0 * fabs(U) + (double)b2) * 0x1p-50;
        const double lb = fmax(L2, 0.0) * (1.0 - gamma32(NQ + 9)) * (1.0 - 0x1p-46) - kSubAbs;
        return __double2float_rd(lb);
    }
}

// fl(sum_j q~_j c_j) and sum_j c_j^2 over one 16-byte group of codes, q~ from shared memory
__device__ __forceinline__ void ps_accum(const float* qt, uint4 w, float& sf, float& cc) {
    const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const float c = (float)(int8_t)(ws[i] >> (8 * b));
            sf = __fmaf_rn(qt[4 * i + b], c, sf);
            cc = __fmaf_rn(c, c, cc);
        }
}
#endif

} // namespace lb200

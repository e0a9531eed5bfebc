// lantern_b200 -- scalar-quantisation casts and the PQ codebook codec.
//
// GPU counterparts of
//   cast_gt<f32, f16|i8|b1>   U/include/usearch/index_plugins.hpp:879-974
//       f16: IEEE round-to-nearest-even (fp16 library, :320-334)  -> __float2half_rn
//       i8 : static_cast<int8>(clamp(x*100, -100, 100))  (i8_converted_t :960-961, truncation)
//       b1 : bit (128 >> (i&7)) of byte i/8 set when x > 0  (:909-918)
//   codebook_t::compress / decompress   U/include/usearch/lantern_storage.hpp:112-149
//       per-subvector argmin of squared L2 over the centroids, strict '<' (lowest id wins);
//       compat128 reproduces the reference's signed-char loop counter (:123) which never
//       reaches centroids >= 128.
#include <cuda_fp16.h>

#include "engine.h"
#include "screen.cuh"

namespace lb200 {

namespace {

// One warp per row; output rows are zero-padded up to out_stride.
__global__ void cast_rows_kernel(const uint8_t* __restrict__ in, size_t in_stride, int in_kind, uint8_t* __restrict__ out,
                                 size_t out_stride, int out_kind, uint32_t dims, size_t n) {
    const size_t row = (size_t)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= n)
        return;
    const uint8_t* src = in + row * in_stride;
    uint8_t* dst = out + row * out_stride;
    const size_t out_bytes = scalar_row_bytes(out_kind, dims);
    if (in_kind == out_kind) {
        for (size_t i = lane; i < out_stride; i += 32)
            dst[i] = i < out_bytes ? src[i] : (uint8_t)0;
        return;
    }
    const float* f = reinterpret_cast<const float*>(src); // in_kind == f32
    if (out_kind == SK_F16) {
        __half* h = reinterpret_cast<__half*>(dst);
        for (uint32_t i = lane; i < out_stride / 2; i += 32)
            h[i] = i < dims ? __float2half_rn(f[i]) : __ushort_as_half((unsigned short)0);
    } else if (out_kind == SK_I8) {
        int8_t* o = reinterpret_cast<int8_t*>(dst);
        for (uint32_t i = lane; i < out_stride; i += 32) {
            int8_t v = 0;
            if (i < dims) {
                float s = f[i] * 100.0f;
                s = fminf(fmaxf(s, -100.0f), 100.0f);
                v = (int8_t)(int)s; // truncation toward zero
            }
            o[i] = v;
        }
    } else if (out_kind == SK_B1) {
        for (uint32_t byte = lane; byte < out_stride; byte += 32) {
            uint32_t v = 0;
#pragma unroll
            for (int b = 0; b < 8; ++b) {
                uint32_t i = byte * 8 + b;
                if (i < dims && f[i] > 0.f)
                    v |= 128u >> b;
            }
            dst[byte] = (uint8_t)v;
        }
    }
}

// PQ encode: one warp per (vector, group of subvectors).  Lanes split the centroids; each lane keeps
// its best (dist, id) and the warp reduces with (dist, id) lexicographic min == "first strict minimum".
__global__ void pq_encode_kernel(const float* __restrict__ codebook, uint32_t dims, uint32_t ncent, uint32_t nsub,
                                 const float* __restrict__ vecs, size_t vec_stride, size_t n, uint8_t* __restrict__ codes,
                                 size_t code_stride, uint32_t limit) {
    const size_t gw = (size_t)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (gw >= n * nsub)
        return;
    const size_t v = gw / nsub;
    const uint32_t s = (uint32_t)(gw % nsub);
    const uint32_t subdim = dims / nsub;
    const float* x = vecs + v * vec_stride + (size_t)s * subdim;
    float best = 3.402823466e+38f;
    uint32_t best_c = 0xFFFFFFFFu;
    for (uint32_t c = lane; c < limit; c += 32) {
        const float* cen = codebook + (size_t)c * dims + (size_t)s * subdim;
        float dist = 0.f;
        for (uint32_t i = 0; i < subdim; ++i) { // same accumulation order as codebook_t::distance (:104-110)
            float d = x[i] - __ldg(cen + i);
            dist += d * d;
        }
        if (dist < best)
            best = dist, best_c = c;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        float od = __shfl_xor_sync(0xffffffffu, best, o);
        uint32_t oc = __shfl_xor_sync(0xffffffffu, best_c, o);
        if (od < best || (od == best && oc < best_c))
            best = od, best_c = oc;
    }
    if (lane == 0)
        codes[v * code_stride + s] = (uint8_t)(best_c == 0xFFFFFFFFu ? 0u : best_c);
}

__global__ void pq_decode_kernel(const float* __restrict__ codebook, uint32_t dims, uint32_t nsub,
                                 const uint8_t* __restrict__ codes, size_t code_stride, size_t n, float* __restrict__ vecs) {
    const size_t v = blockIdx.x;
    if (v >= n)
        return;
    const uint32_t subdim = dims / nsub;
    for (uint32_t i = threadIdx.x; i < dims; i += blockDim.x) {
        uint32_t s = i / subdim;
        uint32_t c = codes[v * code_stride + s];
        vecs[v * dims + i] = __ldg(codebook + (size_t)c * dims + i);
    }
}

// pair[s][a][b] = |c_a,s - c_b,s|^2 (l2sq) or c_a,s . c_b,s (cos); norm[s][c] = |c_c,s|^2
__global__ void pq_tables_kernel(const float* __restrict__ codebook, uint32_t dims, uint32_t ncent, uint32_t nsub, int cosine,
                                 float* __restrict__ pair, float* __restrict__ norm) {
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)nsub * ncent * ncent;
    if (e >= total)
        return;
    const uint32_t b = (uint32_t)(e % ncent), a = (uint32_t)((e / ncent) % ncent), s = (uint32_t)(e / ((size_t)ncent * ncent));
    const uint32_t sd = dims / nsub;
    const float* ca = codebook + (size_t)a * dims + (size_t)s * sd;
    const float* cb = codebook + (size_t)b * dims + (size_t)s * sd;
    float acc = 0.f;
    for (uint32_t i = 0; i < sd; ++i) {
        if (cosine)
            acc = fmaf(ca[i], cb[i], acc);
        else {
            const float d = ca[i] - cb[i];
            acc = fmaf(d, d, acc);
        }
    }
    pair[e] = acc;
    if (a == b) {
        float n2 = 0.f;
        for (uint32_t i = 0; i < sd; ++i)
            n2 = fmaf(ca[i], ca[i], n2);
        norm[(size_t)s * ncent + a] = n2;
    }
}

// Per-query ADC tables for a whole batch (the value side of lantern_storage.hpp:249-270 / index_dense.hpp:341-358 is the raw
// query): table[q][s * W + c] = |q_s - c_{c,s}|^2 (l2sq) or q_s . c_{c,s} (cos), dimensions accumulated in ascending order with
// fmaf -- the same arithmetic PqEval::entry performs when a kernel builds the table itself -- and |q|^2 behind the table.
// One CTA per query; the 0.75 MB of centroid slices it touches stay in L2 across the batch.
__global__ void pq_query_tables_kernel(const float* __restrict__ codebook, uint32_t dims, uint32_t nsub, uint32_t W, int cosine,
                                       const float* __restrict__ queries, size_t q_stride, float* __restrict__ tables,
                                       size_t table_floats) {
    extern __shared__ float qs[];
    const uint32_t q = blockIdx.x, sd = dims / nsub;
    const float* src = queries + (size_t)q * q_stride;
    for (uint32_t i = threadIdx.x; i < dims; i += blockDim.x)
        qs[i] = src[i];
    __syncthreads();
    float* out = tables + (size_t)q * table_floats;
    for (uint32_t e = threadIdx.x; e < nsub * W; e += blockDim.x) {
        const uint32_t s = e / W, c = e - s * W;
        const float* cen = codebook + (size_t)c * dims + (size_t)s * sd;
        const float* v = qs + (size_t)s * sd;
        float acc = 0.f;
        if ((sd & 3u) == 0u) {
            for (uint32_t i = 0; i < sd; i += 4) {
                const float4 c4 = __ldg(reinterpret_cast<const float4*>(cen + i));
                if (cosine) {
                    acc = fmaf(v[i], c4.x, acc), acc = fmaf(v[i + 1], c4.y, acc);
                    acc = fmaf(v[i + 2], c4.z, acc), acc = fmaf(v[i + 3], c4.w, acc);
                } else {
                    float d = v[i] - c4.x;
                    acc = fmaf(d, d, acc);
                    d = v[i + 1] - c4.y, acc = fmaf(d, d, acc);
                    d = v[i + 2] - c4.z, acc = fmaf(d, d, acc);
                    d = v[i + 3] - c4.w, acc = fmaf(d, d, acc);
                }
            }
        } else {
            for (uint32_t i = 0; i < sd; ++i) {
                const float cv = __ldg(cen + i);
                if (cosine)
                    acc = fmaf(v[i], cv, acc);
                else {
                    const float d = v[i] - cv;
                    acc = fmaf(d, d, acc);
                }
            }
        }
        out[e] = acc;
    }
    if (threadIdx.x < 32) { // |q|^2 with the lane layout of PqEval::load_value
        float p2 = 0.f;
        for (uint32_t i = threadIdx.x; i < dims; i += 32)
            p2 += qs[i] * qs[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
            p2 += __shfl_xor_sync(0xffffffffu, p2, o);
        if (threadIdx.x < 4)
            out[(size_t)nsub * W + threadIdx.x] = threadIdx.x == 0 ? p2 : 0.f;
    }
}

// Companion int8 copy of stored f32 rows for the search screen (screen.cuh, DESIGN.md 4.1).  One warp per row:
//   codes: c_i = clamp(round(x_i / s), -127, 127), s = max|x_i| / 127 (fp32), word w = dims 4w..4w+3, zero padded;
//   meta:  {s, r >= |x - s c| (double, rounded up), b2 = |x|^2 exactly as the search kernel computes it, |c| rounded up}.
// Rows holding NaN / inf, or whose scale underflows to 0, get r = +inf: their bound is -inf and they always pass.
__global__ void sq_encode_kernel(const uint8_t* __restrict__ rows, uint32_t row_bytes, size_t n, uint8_t* __restrict__ codes,
                                 uint32_t code_bytes, float4* __restrict__ meta) {
    const size_t row = (size_t)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= n)
        return;
    const uint4* x = reinterpret_cast<const uint4*>(rows + row * row_bytes);
    const uint32_t nchunks = row_bytes / 16;
    // |x|^2 with accum_chunk<DM_COS, SK_F32> + finish_distance's fold, chunk for chunk in the kernel's order: the same bits
    DistAcc<DM_COS, SK_F32> acc;
    acc.reset();
    const uint4 zero = make_uint4(0, 0, 0, 0);
    float amax = 0.f;
    bool finite = true;
    for (uint32_t c = lane; c < nchunks; c += 32) {
        const uint4 v = x[c];
        accum_chunk<DM_COS, SK_F32>(acc, zero, v);
        const float f[4] = {__uint_as_float(v.x), __uint_as_float(v.y), __uint_as_float(v.z), __uint_as_float(v.w)};
#pragma unroll
        for (int b = 0; b < 4; ++b)
            finite = finite && isfinite(f[b]), amax = fmaxf(amax, fabsf(f[b]));
    }
    const float b2 = warp_sum(acc.v[2] + acc.v[3]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    finite = __all_sync(0xffffffffu, finite);
    const float scale = (float)((double)amax / 127.0);
    const bool ok = finite && (amax == 0.f || scale > 0.f);
    double e2 = 0.0;
    uint32_t c2 = 0;
    uint32_t* out = reinterpret_cast<uint32_t*>(codes + row * code_bytes);
    for (uint32_t w = lane; w < code_bytes / 4; w += 32) {
        uint32_t word = 0;
        if (w < nchunks && ok && scale > 0.f) {
            const uint4 v = x[w];
            const float f[4] = {__uint_as_float(v.x), __uint_as_float(v.y), __uint_as_float(v.z), __uint_as_float(v.w)};
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                const int ci = (int)fmin(fmax(rint((double)f[b] / (double)scale), -127.0), 127.0);
                const double e = (double)f[b] - (double)scale * (double)ci; // s * c is exact in double
                e2 += e * e, c2 += (uint32_t)(ci * ci);
                word |= (uint32_t)(uint8_t)(int8_t)ci << (8 * b);
            }
        }
        out[w] = word;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        e2 += __shfl_xor_sync(0xffffffffu, e2, o);
        c2 += __shfl_xor_sync(0xffffffffu, c2, o);
    }
    if (lane == 0) {
        // < 80 double roundings of non-negative terms in e2: relative 2^-46; 2^-40 and the final 2^-50 cover them and the sqrt
        const float r = ok ? __double2float_ru(sqrt(e2 * (1.0 + 0x1p-40)) * (1.0 + 0x1p-50)) : INFINITY;
        meta[row] = make_float4(ok ? scale : 0.f, r, b2, __double2float_ru(sqrt((double)c2) * (1.0 + 0x1p-50)));
    }
}

} // namespace

void launch_sq_encode(const uint8_t* d_rows, size_t row_bytes, size_t n, uint8_t* d_codes, float4* d_meta, cudaStream_t stream) {
    if (!n)
        return;
    const int warps = 8;
    sq_encode_kernel<<<(unsigned)((n + warps - 1) / warps), warps * 32, 0, stream>>>(
        d_rows, (uint32_t)row_bytes, n, d_codes, screen_code_bytes((uint32_t)row_bytes), d_meta);
    LB_CUDA(cudaGetLastError());
    count_launch();
}

void launch_pq_query_tables(const float* d_codebook, size_t dims, size_t nsub, size_t lut_width, bool cosine, const float* d_queries,
                            size_t q_stride_floats, size_t nq, float* d_tables, cudaStream_t stream) {
    if (!nq)
        return;
    const size_t table_floats = pq_table_floats((uint32_t)nsub, (uint32_t)lut_width);
    pq_query_tables_kernel<<<(unsigned)nq, 256, dims * sizeof(float), stream>>>(d_codebook, (uint32_t)dims, (uint32_t)nsub,
                                                                                (uint32_t)lut_width, cosine ? 1 : 0, d_queries,
                                                                                q_stride_floats, d_tables, table_floats);
    LB_CUDA(cudaGetLastError());
    count_launch();
}

void launch_pq_tables(const float* d_codebook, size_t dims, size_t ncent, size_t nsub, bool cosine, float* d_pair, float* d_norm,
                      cudaStream_t stream) {
    const size_t total = nsub * ncent * ncent;
    pq_tables_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(d_codebook, (uint32_t)dims, (uint32_t)ncent, (uint32_t)nsub,
                                                                        cosine ? 1 : 0, d_pair, d_norm);
    LB_CUDA(cudaGetLastError());
    count_launch();
}

void launch_cast_rows(const void* d_in, size_t in_stride, int in_kind, void* d_out, size_t out_stride, int out_kind,
                      size_t dims, size_t n, cudaStream_t stream) {
    if (!n)
        return;
    if (in_kind != out_kind && in_kind != SK_F32)
        throw CudaError("cast: only f32 inputs can be converted to another scalar kind");
    const int warps = 8;
    cast_rows_kernel<<<(unsigned)((n + warps - 1) / warps), warps * 32, 0, stream>>>(
        (const uint8_t*)d_in, in_stride, in_kind, (uint8_t*)d_out, out_stride, out_kind, (uint32_t)dims, n);
    LB_CUDA(cudaGetLastError());
    count_launch();
}

void launch_pq_encode(const float* d_codebook, size_t dims, size_t ncent, size_t nsub, const float* d_vecs,
                      size_t vec_stride_floats, size_t n, uint8_t* d_codes, size_t code_stride, bool compat128,
                      cudaStream_t stream) {
    if (!n)
        return;
    const uint32_t limit = (uint32_t)((compat128 && ncent > 128) ? 128 : ncent);
    const int warps = 8;
    const size_t total = n * nsub;
    pq_encode_kernel<<<(unsigned)((total + warps - 1) / warps), warps * 32, 0, stream>>>(
        d_codebook, (uint32_t)dims, (uint32_t)ncent, (uint32_t)nsub, d_vecs, vec_stride_floats, n, d_codes, code_stride, limit);
    LB_CUDA(cudaGetLastError());
    count_launch();
}

void launch_pq_decode(const float* d_codebook, size_t dims, size_t ncent, size_t nsub, const uint8_t* d_codes,
                      size_t code_stride, size_t n, float* d_vecs, cudaStream_t stream) {
    (void)ncent;
    if (!n)
        return;
    pq_decode_kernel<<<(unsigned)n, 128, 0, stream>>>(d_codebook, (uint32_t)dims, (uint32_t)nsub, d_codes, code_stride, n, d_vecs);
    LB_CUDA(cudaGetLastError());
    count_launch();
}

} // namespace lb200

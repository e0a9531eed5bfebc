// lantern_b200 -- the projected screen of the search beam: per-index basis, row records and per-query pre-pass.
//
// The int8 screen (screen.cuh) reads one code per dimension of every screened candidate.  When the stored rows have most of
// their energy in a few directions, k << dims projected coordinates plus two residual norms give a bound of the same
// tightness from a 64- or 128-byte record (DESIGN.md 3, 4.1):
//   basis    P (k x dims, fp32): top-k eigenvectors of the uncentred second moment of up to 65 536 stored rows, the smallest k
//            of kPsDims whose mean residual energy over the sample is <= kPsMaxResidual; chosen once per index
//   records  per row: int8 codes c of y = P x with scale s, E >= |x - P^T s c|, F >= |P (x - P^T s c)|, b2
//   queries  per batch: q~ = fl(P q), delta >= |P q - q~|, |q~|, G >= |q - P^T q~|, |q|^2
// The bound (pscreen_bound) holds for any fp32 P; the basis only decides how tight it is.
#include <math.h>

#include <algorithm>
#include <chrono>
#include <vector>

#include "distance.cuh"
#include "eigsym.h"
#include "engine.h"
#include "screen.cuh"

namespace lb200 {

namespace {

constexpr double kU64 = 0x1p-53; // unit roundoff of double

// M[a][b] = sum over the sample of x_a x_b, in double, samples in ascending order (deterministic).  64 x 64 tiles, 256
// threads of 4 x 4 entries; `rows` = `ns` sampled rows, `stride` bytes apart.
__global__ void __launch_bounds__(256) ps_moment_kernel(const uint8_t* __restrict__ rows, size_t stride, uint32_t ns, uint32_t d,
                                                        double* __restrict__ M) {
    __shared__ float xa[16][64], xb[16][64];
    const uint32_t a0 = blockIdx.y * 64, b0 = blockIdx.x * 64, tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    if (b0 < a0) // the lower triangle is mirrored by the host
        return;
    double acc[4][4] = {};
    for (uint32_t s0 = 0; s0 < ns; s0 += 16) {
        for (uint32_t e = threadIdx.x; e < 16 * 64; e += 256) {
            const uint32_t r = e / 64, c = e % 64, s = s0 + r;
            const float* x = reinterpret_cast<const float*>(rows + (size_t)s * stride);
            const float va = (s < ns && a0 + c < d) ? x[a0 + c] : 0.f, vb = (s < ns && b0 + c < d) ? x[b0 + c] : 0.f;
            xa[r][c] = isfinite(va) ? va : 0.f; // a few non-finite rows must not poison the basis
            xb[r][c] = isfinite(vb) ? vb : 0.f;
        }
        __syncthreads();
        for (uint32_t r = 0; r < 16; ++r)
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    acc[i][j] = fma((double)xa[r][ty + 16 * i], (double)xb[r][tx + 16 * j], acc[i][j]);
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t a = a0 + ty + 16 * i, b = b0 + tx + 16 * j;
            if (a < d && b < d)
                M[(size_t)a * d + b] = acc[i][j];
        }
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// One warp per stored row; P = [slots][d] row-major, Pt = [d][slots], both zero beyond the basis' k rows.  Shared memory per
// warp: x (d floats), e (d doubles), y^ (slots doubles).
__global__ void __launch_bounds__(128) ps_encode_kernel(const uint8_t* __restrict__ rows, uint32_t row_bytes, size_t n, uint32_t d,
                                                        const float* __restrict__ P, const float* __restrict__ Pt, uint32_t slots,
                                                        int cosine, uint8_t* __restrict__ out) {
    extern __shared__ double ps_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t row = (size_t)blockIdx.x * 4 + warp;
    double* e = ps_smem + (size_t)warp * (d + slots + d / 2 + 1);
    double* yh = e + d;
    float* x = reinterpret_cast<float*>(yh + slots);
    if (row >= n)
        return;
    const uint4* xr = reinterpret_cast<const uint4*>(rows + row * row_bytes);
    const uint32_t nchunks = row_bytes / 16;
    // b2: cos -- |x|^2 with accum_chunk<DM_COS, SK_F32> and finish_distance's fold, the kernel's own bits (as sq_encode_kernel);
    // l2sq -- sum x_i^2 in double, rounded down
    DistAcc<DM_COS, SK_F32> acc;
    acc.reset();
    const uint4 zero = make_uint4(0, 0, 0, 0);
    bool finite = true;
    double x2 = 0.0;
    for (uint32_t c = lane; c < nchunks; c += 32) {
        const uint4 v = xr[c];
        accum_chunk<DM_COS, SK_F32>(acc, zero, v);
        const float f[4] = {__uint_as_float(v.x), __uint_as_float(v.y), __uint_as_float(v.z), __uint_as_float(v.w)};
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const uint32_t i = 4 * c + b;
            if (i < d)
                x[i] = f[b];
            finite = finite && isfinite(f[b]);
            x2 = fma((double)f[b], (double)f[b], x2);
        }
    }
    const float b2k = warp_sum(acc.v[2] + acc.v[3]);
    x2 = warp_sum_d(x2);
    finite = __all_sync(0xffffffffu, finite);
    __syncwarp();
    // y = P x (double), its scale and codes; y^ = s c exactly (24 x 8 bits)
    double amax = 0.0;
    for (uint32_t j = lane; j < slots; j += 32) {
        double y = 0.0;
        for (uint32_t i = 0; i < d; ++i)
            y = fma((double)__ldg(Pt + (size_t)i * slots + j), (double)x[i], y);
        yh[j] = y;
        amax = fmax(amax, fabs(y));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        amax = fmax(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    float s = (float)(amax / 127.0);
    if (!(s > 0.f) || !(s < INFINITY) || !finite)
        s = 0.f; // no codes: y^ = 0, e = x (a valid, loose record)
    __syncwarp();
    uint8_t* rec = out + row * (slots + 16);
    for (uint32_t j = lane; j < slots; j += 32) {
        const int c = s > 0.f ? (int)fmin(fmax(rint(yh[j] / (double)s), -127.0), 127.0) : 0;
        yh[j] = (double)s * (double)c;
        rec[16 + j] = (uint8_t)(int8_t)c;
    }
    __syncwarp();
    // e = x - P^T y^ (double): e_i is off by <= err_i = (2 slots + 4) u64 a_i, a_i = |x_i| + sum_j |P_ji y^_j| (slots products
    // and slots + 1 sums); E^2 >= sum_i (|e_i| + err_i)^2
    double E2 = 0.0, A2 = 0.0;
    for (uint32_t i = lane; i < d; i += 32) {
        double t = (double)x[i], a = fabs(t);
        for (uint32_t j = 0; j < slots; ++j) {
            const double p = (double)__ldg(P + (size_t)j * d + i) * yh[j];
            t -= p;
            a += fabs(p);
        }
        const double err = (2.0 * slots + 4.0) * kU64 * a;
        e[i] = t;
        E2 += (fabs(t) + err) * (fabs(t) + err);
        A2 += a * a;
    }
    __syncwarp();
    E2 = warp_sum_d(E2);
    A2 = warp_sum_d(A2);
    // F^2 >= sum_j (|f_j| + slack_j)^2, f = P e in double: (P e_true)_j - f_j is off by the sum's own roundings,
    // <= (2 d + 4) u64 sum_i |P_ji e_i|, plus sum_i |P_ji| err_i <= |P_j| (2 slots + 4) u64 sqrt(A2) (Cauchy-Schwarz)
    double F2 = 0.0;
    for (uint32_t j = lane; j < slots; j += 32) {
        double f = 0.0, pe = 0.0, p2 = 0.0;
        for (uint32_t i = 0; i < d; ++i) {
            const double p = (double)__ldg(Pt + (size_t)i * slots + j);
            f = fma(p, e[i], f);
            pe += fabs(p * e[i]);
            p2 += p * p;
        }
        const double slack = (2.0 * d + 4.0) * kU64 * pe * (1.0 + 0x1p-40) +
                             sqrt(p2 * (1.0 + 0x1p-40)) * (2.0 * slots + 4.0) * kU64 * sqrt(A2 * (1.0 + 0x1p-40)) * (1.0 + 0x1p-40);
        F2 += (fabs(f) + slack) * (fabs(f) + slack);
    }
    F2 = warp_sum_d(F2);
    if (lane == 0) {
        // sums of < 2^12 non-negative double terms: relative 2^-40 covers them and the square roots
        const float E = finite ? __double2float_ru(sqrt(E2 * (1.0 + 0x1p-40)) * (1.0 + 0x1p-50)) : INFINITY;
        const float F = finite ? __double2float_ru(sqrt(F2 * (1.0 + 0x1p-40)) * (1.0 + 0x1p-50)) : INFINITY;
        const float b2 = cosine ? b2k : __double2float_rd(x2 * (1.0 - 0x1p-40));
        *reinterpret_cast<float4*>(rec) = make_float4(s, E, F, b2);
    }
}

// One CTA per query (storage rows, row_bytes apart): out[q] = q~[slots], {delta, |q~|, G, |q|^2 rounded down}.
__global__ void __launch_bounds__(128) ps_query_kernel(const uint8_t* __restrict__ queries, size_t q_stride, uint32_t d,
                                                       const float* __restrict__ P, const float* __restrict__ Pt, uint32_t slots,
                                                       float* __restrict__ out) {
    extern __shared__ float pq_smem[];
    float* q = pq_smem;      // [d]
    float* qt = q + d;       // [slots]
    __shared__ double part[4][128];
    const float* src = reinterpret_cast<const float*>(queries + (size_t)blockIdx.x * q_stride);
    for (uint32_t i = threadIdx.x; i < d; i += blockDim.x)
        q[i] = src[i];
    __syncthreads();
    float* o = out + (size_t)blockIdx.x * (slots + 4);
    double dl2 = 0.0, qt2 = 0.0, g2 = 0.0, q2 = 0.0;
    for (uint32_t j = threadIdx.x; j < slots; j += blockDim.x) {
        // y_j in double: exact products, d roundings -> |y - y_c| <= (d + 1) u64 sum |P_ji q_i|
        double y = 0.0, a = 0.0;
        for (uint32_t i = 0; i < d; ++i) {
            const double p = (double)__ldg(Pt + (size_t)i * slots + j) * (double)q[i];
            y += p;
            a += fabs(p);
        }
        const float t = (float)y;
        const double dj = (fabs(y - (double)t) + (d + 2.0) * kU64 * a) * (1.0 + 0x1p-50);
        qt[j] = t;
        o[j] = t;
        dl2 += dj * dj;
        qt2 += (double)t * (double)t;
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < d; i += blockDim.x) {
        // r_i = q_i - sum_j P_ji q~_j: exact products, slots roundings
        double r = (double)q[i], a = fabs(r);
        for (uint32_t j = 0; j < slots; ++j) {
            const double p = (double)__ldg(P + (size_t)j * d + i) * (double)qt[j];
            r -= p;
            a += fabs(p);
        }
        const double ri = fabs(r) + (slots + 2.0) * kU64 * a;
        g2 += ri * ri;
        q2 += (double)q[i] * (double)q[i];
    }
    part[0][threadIdx.x] = dl2, part[1][threadIdx.x] = qt2, part[2][threadIdx.x] = g2, part[3][threadIdx.x] = q2;
    __syncthreads();
    if (threadIdx.x < 4) {
        double s = 0.0;
        for (int t = 0; t < 128; ++t)
            s += part[threadIdx.x][t];
        // < 2^12 non-negative terms: relative 2^-40 covers the sums and the square roots
        const float v = threadIdx.x == 3 ? __double2float_rd(s * (1.0 - 0x1p-40))
                                         : __double2float_ru(sqrt(s * (1.0 + 0x1p-40)) * (1.0 + 0x1p-50));
        o[slots + threadIdx.x] = v;
    }
}

// Z[j] = M Q[j] for the p rows of Q (each a vector of d doubles): M symmetric, read by columns so that a warp's loads are
// contiguous; sums over b in ascending order (deterministic).  Grid (p, ceil(d / 128)).
__global__ void __launch_bounds__(128) ps_matvecs_kernel(const double* __restrict__ M, const double* __restrict__ Q, uint32_t d,
                                                         double* __restrict__ Z) {
    const uint32_t j = blockIdx.x, a = blockIdx.y * 128 + threadIdx.x;
    if (a >= d)
        return;
    const double* q = Q + (size_t)j * d;
    double acc = 0.0;
    for (uint32_t b = 0; b < d; ++b)
        acc = fma(M[(size_t)b * d + a], q[b], acc);
    Z[(size_t)j * d + a] = acc;
}

} // namespace

// the sample's second-moment matrix (upper triangle), device -> host, mirrored
static std::vector<double> ps_moment(const uint8_t* d_rows, size_t row_bytes, size_t n, size_t d, size_t& ns) {
    const size_t step = std::max<size_t>(1, n / kPsSampleMax);
    ns = std::min(n / step, kPsSampleMax);
    double* dM = nullptr;
    LB_CUDA(cudaMalloc(&dM, d * d * sizeof(double)));
    const dim3 grid((unsigned)((d + 63) / 64), (unsigned)((d + 63) / 64));
    ps_moment_kernel<<<grid, 256>>>(d_rows, step * row_bytes, (uint32_t)ns, (uint32_t)d, dM);
    cudaError_t err = cudaGetLastError();
    count_launch();
    std::vector<double> M(d * d);
    if (err == cudaSuccess)
        err = cudaMemcpy(M.data(), dM, d * d * sizeof(double), cudaMemcpyDeviceToHost);
    cudaFree(dM);
    LB_CUDA(err);
    for (size_t a = 0; a < d; ++a)
        for (size_t b = 0; b < a; ++b)
            M[a * d + b] = M[b * d + a];
    return M;
}

void launch_ps_queries(const float* d_P, const float* d_Pt, size_t dims, uint32_t k, const uint8_t* d_queries, size_t q_stride, size_t nq,
                       float* d_out, cudaStream_t stream) {
    if (!nq)
        return;
    const uint32_t slots = ps_code_slots(k);
    ps_query_kernel<<<(unsigned)nq, 128, (dims + slots) * sizeof(float), stream>>>(d_queries, q_stride, (uint32_t)dims, d_P, d_Pt, slots,
                                                                                 d_out);
    LB_CUDA(cudaGetLastError());
    count_launch();
}

void launch_ps_encode(const uint8_t* d_rows, size_t row_bytes, size_t n, size_t dims, const float* d_P, const float* d_Pt, uint32_t k,
                      bool cosine, uint8_t* d_records, cudaStream_t stream) {
    if (!n)
        return;
    const uint32_t slots = ps_code_slots(k);
    const size_t smem = 4 * (dims + slots + dims / 2 + 1) * sizeof(double);
    LB_CUDA(cudaFuncSetAttribute(ps_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ps_encode_kernel<<<(unsigned)((n + 3) / 4), 128, smem, stream>>>(d_rows, (uint32_t)row_bytes, n, (uint32_t)dims, d_P, d_Pt, slots,
                                                                     cosine ? 1 : 0, d_records);
    LB_CUDA(cudaGetLastError());
    count_launch();
}

// device copies of a basis: P [slots][dims] and P^T [dims][slots], zero rows beyond k.  On failure nothing stays allocated.
void ps_upload_basis(const std::vector<float>& P, size_t dims, uint32_t k, float** d_P, float** d_Pt) {
    const uint32_t slots = ps_code_slots(k);
    std::vector<float> p((size_t)slots * dims, 0.f), pt((size_t)slots * dims, 0.f);
    for (size_t j = 0; j < k; ++j)
        for (size_t i = 0; i < dims; ++i)
            p[j * dims + i] = pt[i * slots + j] = P[j * dims + i];
    float *a = nullptr, *b = nullptr;
    cudaError_t err = cudaMalloc(&a, p.size() * sizeof(float));
    if (err == cudaSuccess)
        err = cudaMalloc(&b, pt.size() * sizeof(float));
    if (err == cudaSuccess)
        err = cudaMemcpy(a, p.data(), p.size() * sizeof(float), cudaMemcpyHostToDevice);
    if (err == cudaSuccess)
        err = cudaMemcpy(b, pt.data(), pt.size() * sizeof(float), cudaMemcpyHostToDevice);
    if (err != cudaSuccess) {
        cudaFree(a), cudaFree(b);
        LB_CUDA(err);
    }
    *d_P = a, *d_Pt = b;
}

// Top `want` unit eigenvectors (rows of `vec`, eigenvalues descending) of the d x d symmetric M.  Up to d = 256 a full
// decomposition (eigsym.h) is cheap; wider, a full one grows as d^3 on one host thread (about 1.5 s at d768 and 90 s at
// d2048), so the top eigenvectors come from subspace iteration instead: kPsSubspace orthonormal vectors (deterministic start),
// kPsSubspaceIters products with M on the device, Gram-Schmidt and a Rayleigh-Ritz step on the host -- O(d^2 p) per
// iteration.  Any basis gives a valid bound; an unconverged one is only less tight, and the residual energy that chooses k is
// measured with the basis actually returned.  The same M always gives the same bits.
static void ps_top_eigvecs(const std::vector<double>& M, size_t d, uint32_t want, std::vector<double>& vec) {
    if (d <= 256) {
        std::vector<double> val;
        eig_symmetric(M, d, val, vec);
        vec.resize(std::min<size_t>(want, d) * d);
        return;
    }
    const size_t p = kPsSubspace;
    std::vector<double> Q(p * d), Z(p * d);
    uint64_t st = 0x9E3779B97F4A7C15ull; // splitmix64: a fixed start
    for (double& v : Q) {
        uint64_t z = (st += 0x9E3779B97F4A7C15ull);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        v = (double)((z ^ (z >> 31)) >> 11) * 0x1p-53 - 0.5;
    }
    // modified Gram-Schmidt on the rows of A -> Q; a row that (numerically) lies in the span of the previous ones is replaced by
    // the next unit coordinate vector not yet in it
    size_t fresh = 0;
    auto orthonormalize = [&](std::vector<double>& A) {
        for (size_t j = 0; j < p; ++j) {
            double* v = &A[j * d];
            for (int attempt = 0;; ++attempt) {
                double n0 = 0.0;
                for (size_t i = 0; i < d; ++i)
                    n0 += v[i] * v[i];
                for (size_t r = 0; r < j; ++r) {
                    const double* u = &A[r * d];
                    double dot = 0.0;
                    for (size_t i = 0; i < d; ++i)
                        dot += u[i] * v[i];
                    for (size_t i = 0; i < d; ++i)
                        v[i] -= dot * u[i];
                }
                double n1 = 0.0;
                for (size_t i = 0; i < d; ++i)
                    n1 += v[i] * v[i];
                if (n1 > 1e-20 * n0 && n1 > 0.0) {
                    const double inv = 1.0 / sqrt(n1);
                    for (size_t i = 0; i < d; ++i)
                        v[i] *= inv;
                    break;
                }
                std::fill(v, v + d, 0.0);
                if (attempt >= (int)d) // cannot happen for p <= d; a zero row is still a valid (useless) direction
                    break;
                v[fresh++ % d] = 1.0;
            }
        }
    };
    orthonormalize(Q);
    double *dM = nullptr, *dQ = nullptr, *dZ = nullptr;
    cudaError_t err = cudaMalloc(&dM, d * d * sizeof(double));
    if (err == cudaSuccess)
        err = cudaMalloc(&dQ, p * d * sizeof(double));
    if (err == cudaSuccess)
        err = cudaMalloc(&dZ, p * d * sizeof(double));
    if (err == cudaSuccess)
        err = cudaMemcpy(dM, M.data(), d * d * sizeof(double), cudaMemcpyHostToDevice);
    for (int it = 0; err == cudaSuccess && it <= kPsSubspaceIters; ++it) {
        err = cudaMemcpy(dQ, Q.data(), p * d * sizeof(double), cudaMemcpyHostToDevice);
        if (err != cudaSuccess)
            break;
        ps_matvecs_kernel<<<dim3((unsigned)p, (unsigned)((d + 127) / 128)), 128>>>(dM, dQ, (uint32_t)d, dZ);
        count_launch();
        err = cudaGetLastError();
        if (err == cudaSuccess)
            err = cudaMemcpy(Z.data(), dZ, p * d * sizeof(double), cudaMemcpyDeviceToHost);
        if (err == cudaSuccess && it < kPsSubspaceIters) {
            orthonormalize(Z);
            Q.swap(Z);
        }
    }
    cudaFree(dM), cudaFree(dQ), cudaFree(dZ);
    LB_CUDA(err);
    // Rayleigh-Ritz: H = Q^T M Q (Z = M Q), its eigenvectors V, then vec = V Q
    std::vector<double> H(p * p), hval, hvec;
    for (size_t a = 0; a < p; ++a)
        for (size_t b = a; b < p; ++b) {
            double h = 0.0, h2 = 0.0;
            for (size_t i = 0; i < d; ++i)
                h += Q[a * d + i] * Z[b * d + i], h2 += Q[b * d + i] * Z[a * d + i];
            H[a * p + b] = H[b * p + a] = 0.5 * (h + h2);
        }
    eig_symmetric(H, p, hval, hvec);
    const size_t m = std::min<size_t>(want, p);
    vec.assign(m * d, 0.0);
    for (size_t r = 0; r < m; ++r)
        for (size_t b = 0; b < p; ++b) {
            const double w = hvec[r * p + b];
            for (size_t i = 0; i < d; ++i)
                vec[r * d + i] += w * Q[b * d + i];
        }
}

// The basis of rows [0, n) (d_rows, row_bytes apart): the smallest k of kPsDims whose mean residual energy |x - P^T P x|^2 / |x|^2
// over the sample is <= kPsMaxResidual (or, `force`d, the best k there is).  Returns k (0 = none qualifies) and P [k][dims].
uint32_t ps_choose_basis(const uint8_t* d_rows, size_t row_bytes, size_t n, size_t dims, bool force, uint32_t want_k, std::vector<float>& P) {
    size_t ns = 0;
    const std::vector<double> M = ps_moment(d_rows, row_bytes, n, dims, ns);
    const uint32_t kmax = kPsDims[sizeof(kPsDims) / sizeof(kPsDims[0]) - 1];
    std::vector<double> vec;
    ps_top_eigvecs(M, dims, kmax, vec);
    std::vector<float> Pmax((size_t)kmax * dims, 0.f);
    for (size_t j = 0; j < std::min<size_t>(kmax, vec.size() / dims); ++j)
        for (size_t i = 0; i < dims; ++i)
            Pmax[j * dims + i] = (float)vec[j * dims + i];
    if (want_k) {
        P.assign(Pmax.begin(), Pmax.begin() + (size_t)std::min(want_k, kmax) * dims);
        return std::min(want_k, kmax);
    }
    // residual energy of every sampled row at every k: |x|^2 - sum_{j<k} (P x)_j^2, from the query pre-pass over the sample
    float *dP = nullptr, *dPt = nullptr, *dout = nullptr;
    ps_upload_basis(Pmax, dims, kmax, &dP, &dPt);
    const uint32_t nf = ps_query_floats(kmax);
    std::vector<float> h(ns * nf);
    const size_t step = std::max<size_t>(1, n / kPsSampleMax);
    cudaError_t err = cudaMalloc(&dout, h.size() * sizeof(float));
    if (err == cudaSuccess) {
        try {
            launch_ps_queries(dP, dPt, dims, kmax, d_rows, step * row_bytes, ns, dout, 0);
            err = cudaMemcpy(h.data(), dout, h.size() * sizeof(float), cudaMemcpyDeviceToHost);
        } catch (...) {
            cudaFree(dP), cudaFree(dPt), cudaFree(dout);
            throw;
        }
    }
    cudaFree(dP), cudaFree(dPt), cudaFree(dout);
    LB_CUDA(err);
    uint32_t best = 0;
    double best_res = INFINITY;
    for (uint32_t k : kPsDims) {
        double sum = 0.0;
        size_t cnt = 0;
        for (size_t s = 0; s < ns; ++s) {
            const float* o = &h[s * nf];
            const double x2 = o[ps_code_slots(kmax) + 3];
            if (!(x2 > 0.0) || !(x2 < INFINITY))
                continue;
            double y2 = 0.0;
            for (uint32_t j = 0; j < k; ++j)
                y2 += (double)o[j] * o[j];
            sum += std::max(0.0, x2 - y2) / x2, ++cnt;
        }
        const double res = cnt ? sum / cnt : INFINITY;
        if (res <= kPsMaxResidual) {
            best = k;
            break;
        }
        if (force && res < best_res - 1e-12)
            best_res = res, best = k;
    }
    if (!best && force)
        best = kPsDims[0];
    P.assign(Pmax.begin(), Pmax.begin() + (size_t)best * dims);
    return best;
}

// ---- Index: the screen's choice and companions -------------------------------------------------------------------

bool Index::screen_eligible() const { return sq_bytes_ && row_bytes_ >= kScreenMinRowBytes; }

void Index::free_pscreen() {
    cudaFree(d_ps_basis_), cudaFree(d_ps_basis_t_), cudaFree(d_ps_records_);
    d_ps_basis_ = d_ps_basis_t_ = nullptr, d_ps_records_ = nullptr;
    ps_k_ = 0;
    ps_basis_.clear();
}

void Index::reset_screen() {
    free_pscreen();
    ps_decided_ = ps_auto_ = false;
    if (sq_bytes_)
        set_int8_companion(true);
}

void Index::set_int8_companion(bool on) {
    if (on == sq_on_)
        return;
    if (on) {
        const size_t used = n_ + pending_n_;
        LB_CUDA(cudaMalloc(&d_sq_codes_, std::max<size_t>(capacity_, 1) * sq_bytes_));
        LB_CUDA(cudaMalloc(&d_sq_meta_, std::max<size_t>(capacity_, 1) * sizeof(float4)));
        LB_CUDA(cudaMemset(d_sq_codes_, 0, std::max<size_t>(capacity_, 1) * sq_bytes_));
        LB_CUDA(cudaMemset(d_sq_meta_, 0, std::max<size_t>(capacity_, 1) * sizeof(float4)));
        sq_on_ = true;
        if (used)
            launch_sq_encode(d_vectors_, row_bytes_, used, d_sq_codes_, d_sq_meta_, 0);
    } else {
        cudaFree(d_sq_codes_), cudaFree(d_sq_meta_);
        d_sq_codes_ = nullptr, d_sq_meta_ = nullptr;
        sq_on_ = false;
    }
}

// Installs a basis and encodes every row; the index takes it only once everything has succeeded (on a throw it keeps no basis)
void Index::set_pscreen_basis(const std::vector<float>& P, uint32_t k) {
    free_pscreen();
    if (!k)
        return;
    float *bp = nullptr, *bt = nullptr;
    uint8_t* rec = nullptr;
    ps_upload_basis(P, cfg_.dims, k, &bp, &bt);
    try {
        const size_t rb = ps_record_bytes(k), used = n_ + pending_n_, cap = std::max<size_t>(capacity_, 1);
        LB_CUDA(cudaMalloc(&rec, cap * rb));
        LB_CUDA(cudaMemset(rec, 0, cap * rb));
        if (used)
            launch_ps_encode(d_vectors_, row_bytes_, used, cfg_.dims, bp, bt, k, dist_mode_ == DM_COS, rec, 0);
        LB_CUDA(cudaDeviceSynchronize());
    } catch (...) {
        cudaFree(bp), cudaFree(bt), cudaFree(rec);
        throw;
    }
    d_ps_basis_ = bp, d_ps_basis_t_ = bt, d_ps_records_ = rec;
    ps_basis_ = P;
    ps_k_ = k;
}

// Automatic choice, once per index (and again after load_buffer): from the first build that leaves >= kPsMinRows rows, the
// projected screen when the rows' spectrum allows a small k, else the int8 screen.  Only the chosen companion is kept.
void Index::decide_screen() {
    if (!screen_eligible() || ps_decided_ || n_ < kPsMinRows)
        return;
    const auto t0 = std::chrono::steady_clock::now();
    ps_decided_ = true;
    // Called after a build has committed: a failure here (out of memory) must not turn that build into an error, and must
    // leave a consistent index, so it falls back to the int8 screen, which is still in place until the very last step.
    try {
        std::vector<float> P;
        const uint32_t k = ps_choose_basis(d_vectors_, row_bytes_, n_, cfg_.dims, false, 0, P);
        set_pscreen_basis(P, k); // k = 0 also drops a basis an experiment forced earlier
        if (k) {
            ps_auto_ = true;
            set_int8_companion(false);
        }
    } catch (const CudaError&) {
        free_pscreen();
        ps_auto_ = false;
        (void)cudaGetLastError();
    }
    ps_basis_ms_ = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

// LB200_SEARCH_SCREEN=2 on an index without a basis: the best one its rows give, whatever the residual or the row count.  The
// automatic mode keeps running what decide_screen chose (ps_auto_).
void Index::force_pscreen() {
    if (ps_k_ || !n_)
        return;
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<float> P;
    const uint32_t k = ps_choose_basis(d_vectors_, row_bytes_, n_, cfg_.dims, true, 0, P);
    set_pscreen_basis(P, k);
    ps_basis_ms_ = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

} // namespace lb200

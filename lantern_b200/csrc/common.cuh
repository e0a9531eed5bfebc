// lantern_b200 -- shared device/host helpers for the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <stdexcept>
#include <string>

namespace lb200 {

// ---- scalar / metric kinds: numeric values of the C ABI (include/lantern_b200.h) --------------------
enum : int { SK_F32 = 1, SK_F64 = 2, SK_F16 = 3, SK_I8 = 4, SK_B1 = 5 };
enum : int { MK_COS = 1, MK_IP = 2, MK_L2SQ = 3, MK_HAMMING = 8 };
// what the distance kernels specialise on
enum : int { DM_L2SQ = 0, DM_COS = 1, DM_HAMMING = 2, DM_IP = 3 };

constexpr uint32_t kNoNeighbor = 0xFFFFFFFFu; // adjacency padding
constexpr uint32_t kExpandedBit = 0x80000000u;

struct CudaError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

#define LB_CUDA(expr)                                                                                                  \
    do {                                                                                                               \
        cudaError_t _e = (expr);                                                                                       \
        if (_e != cudaSuccess)                                                                                         \
            throw ::lb200::CudaError(std::string(#expr) + ": " + cudaGetErrorString(_e));                              \
    } while (0)

extern std::atomic<uint64_t> g_kernel_launches;
inline void count_launch(uint64_t n = 1) { g_kernel_launches.fetch_add(n, std::memory_order_relaxed); }

inline size_t round_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// bytes of one vector in a scalar kind (metric_punned_t::bytes_per_vector, index_plugins.hpp:1397-1399)
#ifdef __CUDACC__
#define LB_HD __host__ __device__
#else
#define LB_HD
#endif
LB_HD inline size_t scalar_row_bytes(int kind, size_t dims) {
    switch (kind) {
    case SK_F32: return dims * 4;
    case SK_F64: return dims * 8;
    case SK_F16: return dims * 2;
    case SK_I8: return dims;
    case SK_B1: return (dims + 7) / 8;
    default: return 0;
    }
}

#ifdef __CUDACC__
// ---- PTX wrappers: mbarrier + 1-D bulk async copy (TMA engine, SASS UBLKCP) ------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// plain arrival (release at CTA scope): the slot was filled by this thread's own stores
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                 "selp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok)
                 : "r"(smem_u32(bar)), "r"(parity)
                 : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// global -> shared::cta bulk copy, completion signalled on `bar` (bytes, src, dst all multiples of 16)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ uint32_t warp_sum_u32(uint32_t v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
#endif

} // namespace lb200

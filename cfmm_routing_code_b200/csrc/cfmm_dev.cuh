// cfmm_dev.cuh -- helpers shared by the kernel translation units (device + launch bookkeeping).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <atomic>

#include "cfmm_b200.h"

namespace cfmm {

extern std::atomic<long long> g_launches;
extern int g_scatter_mode;
extern thread_local cudaError_t g_last_err;

int num_sms();

constexpr double kDtMax = 3.0;      // largest log-price change of one Newton step (solver.py DT_MAX, cfmm_small.cuh DT_MAX)

inline int check_launch() {
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { g_last_err = e; return CFMM_E_CUDA; }
    return CFMM_OK;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ---- mbarrier + 1-D bulk async copy (TMA, cp.async.bulk -> UBLKCP) ---------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
    unsigned ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// LL protocol cell: 8 bytes of payload + 8 bytes of sequence flag, moved by ONE 16-byte store / load
struct __align__(16) LLCell { double val; unsigned long long flag; };
__device__ __forceinline__ void st_ll(LLCell* p, double v, unsigned long long f) {
    asm volatile("st.relaxed.sys.global.v2.b64 [%0], {%1, %2};" ::"l"(p), "l"(__double_as_longlong(v)), "l"(f) : "memory");
}
__device__ __forceinline__ void ld_ll(const LLCell* p, double& v, unsigned long long& f) {
    long long bits;
    asm volatile("ld.relaxed.sys.global.v2.b64 {%0, %1}, [%2];" : "=l"(bits), "=l"(f) : "l"(p) : "memory");
    v = __longlong_as_double(bits);
}

// bulk prefetch of a contiguous global range into L2 (no registers, no shared memory): cp.async.bulk.prefetch.L2
__device__ __forceinline__ void bulk_prefetch_l2(const void* src, unsigned bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}

}  // namespace cfmm

// bf_common.cuh -- shared device/host helpers for the bundlefusion_b200 CUDA library.
//
// Arithmetic contract of the TSDF path (see oracle/tsdf_oracle.c header): every float
// operation is individually rounded (this TU is compiled with -fmad=false, IEEE div/sqrt),
// float->int is cvt.rzi with saturation (CUDA's native behaviour), so results can be
// compared bit-for-bit with the CPU oracle.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define BF_API extern "C" __attribute__((visibility("default")))

namespace bf {

// ---- per-thread last error + global stream --------------------------------------------
void set_last_error(const char* where, cudaError_t e);
cudaStream_t stream();

// returns the error code from the enclosing function (bf* extension API)
#define BF_CHECK(expr)                                                        \
    do {                                                                      \
        cudaError_t _e = (expr);                                              \
        if (_e != cudaSuccess) { ::bf::set_last_error(#expr, _e); return (int)_e; } \
    } while (0)

// cutilSafeCall behaviour for the reference-named stubs: print and exit(-1)
// (FriedLiver/Include/cutil/inc/cutil_inline_runtime.h:277-285, minus the getchar()).
#define BF_SAFE(expr)                                                         \
    do {                                                                      \
        int _rc = (expr);                                                     \
        if (_rc != 0) {                                                       \
            fprintf(stderr, "%s(%i) : bundlefusion_b200 runtime error %d: %s\n", __FILE__, __LINE__, _rc, \
                    cudaGetErrorString((cudaError_t)_rc));                    \
            exit(-1);                                                         \
        }                                                                     \
    } while (0)

static inline int num_sms() {
    static int n = 0;
    if (!n) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    }
    return n;
}

// ---- device helpers ---------------------------------------------------------------------
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ unsigned warp_sum_u(unsigned v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}


// ---- mbarrier + 1-D bulk async copy (TMA engine, SASS: UBLKCP / SYNCS) ---------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// global -> shared bulk copy, completion signalled on an mbarrier (bytes multiple of 16, 16-B aligned)
__device__ __forceinline__ void bulk_g2s(void* dstSmem, const void* srcGlobal, unsigned bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dstSmem)),
                 "l"(srcGlobal), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

}  // namespace bf

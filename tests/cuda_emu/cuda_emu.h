// cuda_emu.h -- TEST INFRASTRUCTURE ONLY.  A minimal host emulation of the CUDA constructs the library's kernels use, so that the very same
// kernel source can be executed on the CPU (tests/test_*_emulated.py, built by tests/cuda_emu/__init__.py): one OS thread per CUDA thread of a
// block, blocks run one after the other, __syncthreads / warp collectives on a block-wide barrier, __shared__ as function-static storage,
// atomics and cache-hint loads / stores under one lock.  With BF_EMU_SEQUENTIAL defined, a launch runs its CUDA threads one after the other
// on the calling thread instead (block after block, thread after thread), for sources that replace their warp collectives under that macro.
// It checks the kernels' LOGIC (tiling, halos, scans, ranks, list layout, hash inserts) against the oracle when no GPU is at hand; it says
// nothing about performance and is never part of the product (the library has no CPU path).
#pragma once
#include <algorithm>
#include <atomic>
#include <cmath>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __grid_constant__
#define __launch_bounds__(...)
#define __shared__ static
#define BF_API extern "C"

struct float2 { float x, y; }; struct float4 { float x, y, z, w; }; struct int2 { int x, y; }; struct uint2 { unsigned x, y; };
struct uchar4 { unsigned char x, y, z, w; };
struct uint4 { unsigned x, y, z, w; }; struct int4 { int x, y, z, w; };
static inline int4 make_int4(int x, int y, int z, int w) { return { x, y, z, w }; }
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return { x, y, z, w }; }
static inline uchar4 make_uchar4(unsigned char x, unsigned char y, unsigned char z, unsigned char w) { return { x, y, z, w }; }
static inline float2 make_float2(float x, float y) { return { x, y }; }
static inline float4 make_float4(float x, float y, float z, float w) { return { x, y, z, w }; }
static inline int2 make_int2(int x, int y) { return { x, y }; }
static inline uint2 make_uint2(unsigned x, unsigned y) { return { x, y }; }
struct dim3 { unsigned x, y, z; dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
struct uint3 { unsigned x, y, z; };

typedef int cudaError_t; typedef void* cudaStream_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
static inline cudaError_t cudaMalloc(void** p, size_t n) { *p = calloc(1, n); return *p ? 0 : 2; }
template <class T> static inline cudaError_t cudaMalloc(T** p, size_t n) { return cudaMalloc(reinterpret_cast<void**>(p), n); }
static inline cudaError_t cudaFree(void* p) { free(p); return 0; }
static inline cudaError_t cudaGetLastError() { return 0; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, int, int) { return 0; }

namespace emu {
struct Barrier {                     // reusable counting barrier
    std::mutex m; std::condition_variable cv; unsigned n = 1, waiting = 0, gen = 0;
    void wait() { std::unique_lock<std::mutex> lk(m); const unsigned g = gen; if (++waiting == n) { waiting = 0; ++gen; cv.notify_all(); } else cv.wait(lk, [&] { return gen != g; }); }
};
inline Barrier g_bar;
inline std::mutex g_atomic;
inline float g_xchg[1024]; inline unsigned g_vote[32];
inline std::vector<float> g_dynSmem;
}  // namespace emu

inline thread_local uint3 threadIdx, blockIdx; inline thread_local dim3 blockDim, gridDim;
alignas(16) inline float sm[64 * 1024];                                       // `extern __shared__ float sm[]`
#define extern_shared_decl

static inline void __syncthreads() { emu::g_bar.wait(); }
static inline unsigned emu_tid() { return threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z); }      // linear id: warps are cut from it
static inline unsigned atomicAdd(unsigned* p, unsigned v) { std::lock_guard<std::mutex> lk(emu::g_atomic); const unsigned o = *p; *p = o + v; return o; }
static inline float atomicAdd(float* p, float v) { std::lock_guard<std::mutex> lk(emu::g_atomic); const float o = *p; *p = o + v; return o; }
static inline unsigned atomicMin(unsigned* p, unsigned v) { std::lock_guard<std::mutex> lk(emu::g_atomic); const unsigned o = *p; if (v < o) *p = v; return o; }
static inline int atomicMax(int* p, int v) { std::lock_guard<std::mutex> lk(emu::g_atomic); const int o = *p; if (v > o) *p = v; return o; }
static inline int atomicAdd(int* p, int v) { std::lock_guard<std::mutex> lk(emu::g_atomic); const int o = *p; *p = o + v; return o; }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { std::lock_guard<std::mutex> lk(emu::g_atomic); const unsigned long long o = *p; *p = o + v; return o; }
static inline unsigned atomicSub(unsigned* p, unsigned v) { std::lock_guard<std::mutex> lk(emu::g_atomic); const unsigned o = *p; *p = o - v; return o; }
static inline unsigned atomicMax(unsigned* p, unsigned v) { std::lock_guard<std::mutex> lk(emu::g_atomic); const unsigned o = *p; if (v > o) *p = v; return o; }
static inline int atomicExch(int* p, int v) { std::lock_guard<std::mutex> lk(emu::g_atomic); const int o = *p; *p = v; return o; }
static inline int atomicCAS(int* p, int cmp, int v) { std::lock_guard<std::mutex> lk(emu::g_atomic); const int o = *p; if (o == cmp) *p = v; return o; }
static inline unsigned long long atomicCAS(unsigned long long* p, unsigned long long cmp, unsigned long long v) {
    std::lock_guard<std::mutex> lk(emu::g_atomic); const unsigned long long o = *p; if (o == cmp) *p = v; return o;
}
template <class T> static inline T __ldcg(const T* p) { std::lock_guard<std::mutex> lk(emu::g_atomic); return *p; }
static inline void __stcg(int* p, int v) { std::lock_guard<std::mutex> lk(emu::g_atomic); *p = v; }
static inline void __threadfence() { std::atomic_thread_fence(std::memory_order_seq_cst); }
static inline void __nanosleep(unsigned) { std::this_thread::yield(); }
static inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(unsigned u) { float f; std::memcpy(&f, &u, 4); return f; }
static inline int __float2int_rz(float v) { if (v != v) return 0; if (v >= 2147483648.0f) return INT32_MAX; if (v <= -2147483648.0f) return INT32_MIN; return (int)v; }     // cvt.rzi.s32.f32
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
static inline unsigned __byte_perm(unsigned x, unsigned y, unsigned s) {
    const unsigned long long v = ((unsigned long long)y << 32) | x; unsigned r = 0;
    for (int i = 0; i < 4; ++i) r |= (unsigned)((v >> (8 * ((s >> (4 * i)) & 7))) & 0xff) << (8 * i);
    return r;
}
static inline unsigned __ballot_sync(unsigned, bool pred) {                   // called by every thread of the block at the same point
    const unsigned t = emu_tid(), w = t >> 5;
    if ((t & 31) == 0) emu::g_vote[w] = 0;
    emu::g_bar.wait();
    if (pred) { std::lock_guard<std::mutex> lk(emu::g_atomic); emu::g_vote[w] |= 1u << (t & 31); }
    emu::g_bar.wait();
    const unsigned r = emu::g_vote[w];
    emu::g_bar.wait();
    return r;
}
static inline float __shfl_xor_sync(unsigned, float v, int mask) {
    const unsigned t = emu_tid();
    emu::g_xchg[t] = v;
    emu::g_bar.wait();
    const float r = emu::g_xchg[(t & ~31u) | ((t ^ (unsigned)mask) & 31u)];
    emu::g_bar.wait();
    return r;
}

static inline float __shfl_down_sync(unsigned, float v, int delta) {         // lanes past the end keep their own value
    const unsigned t = emu_tid(), l = t & 31;
    emu::g_xchg[t] = v;
    emu::g_bar.wait();
    const float r = (l + (unsigned)delta < 32) ? emu::g_xchg[t + delta] : v;
    emu::g_bar.wait();
    return r;
}
static inline float __shfl_sync(unsigned, float v, int src) {
    const unsigned t = emu_tid();
    emu::g_xchg[t] = v;
    emu::g_bar.wait();
    const float r = emu::g_xchg[(t & ~31u) | ((unsigned)src & 31u)];
    emu::g_bar.wait();
    return r;
}
static inline int __shfl_xor_sync(unsigned m, int v, int mask) { float f; std::memcpy(&f, &v, 4); f = __shfl_xor_sync(m, f, mask); std::memcpy(&v, &f, 4); return v; }   // bit pattern through the float path
static inline int __shfl_down_sync(unsigned m, int v, int d) { float f; std::memcpy(&f, &v, 4); f = __shfl_down_sync(m, f, d); std::memcpy(&v, &f, 4); return v; }
static inline int __shfl_sync(unsigned m, int v, int src) { float f; std::memcpy(&f, &v, 4); f = __shfl_sync(m, f, src); std::memcpy(&v, &f, 4); return v; }
static inline unsigned __shfl_sync(unsigned m, unsigned v, int src) { return (unsigned)__shfl_sync(m, (int)v, src); }
static inline void __syncwarp(unsigned = 0xFFFFFFFFu) { emu::g_bar.wait(); }      // the emulated kernels use it only in one-warp blocks, where it is the block barrier
using std::min; using std::max;

// kernel<<<grid, block, smem, stream>>>(args...) is rewritten by the builder into EMU_LAUNCH((kernel), grid, block, args...)
template <class K, class... A>
static inline void emu_launch(K kernel, dim3 grid, dim3 block, A... args) {
    const unsigned nt = block.x * block.y * block.z;
    static const bool trace = getenv("EMU_TRACE") != nullptr;
    static int launchNo = 0;
    if (trace) fprintf(stderr, "[emu] launch %d: grid (%u,%u,%u) block (%u,%u,%u)\n", ++launchNo, grid.x, grid.y, grid.z, block.x, block.y, block.z);
#ifdef BF_EMU_SEQUENTIAL
    emu::g_bar.n = 1;
    blockDim = block; gridDim = grid;
    for (unsigned bz = 0; bz < grid.z; ++bz)
        for (unsigned by = 0; by < grid.y; ++by)
            for (unsigned bx = 0; bx < grid.x; ++bx)
                for (unsigned t = 0; t < nt; ++t) {
                    blockIdx = { bx, by, bz };
                    threadIdx = { t % block.x, (t / block.x) % block.y, t / (block.x * block.y) };
                    kernel(args...);
                }
#else
    emu::g_bar.n = nt;
    std::vector<std::thread> th;
    for (unsigned t = 0; t < nt; ++t)
        th.emplace_back([=]() {
            blockDim = block; gridDim = grid;
            threadIdx = { t % block.x, (t / block.x) % block.y, t / (block.x * block.y) };
            for (unsigned bz = 0; bz < grid.z; ++bz)
                for (unsigned by = 0; by < grid.y; ++by)
                    for (unsigned bx = 0; bx < grid.x; ++bx) {
                        blockIdx = { bx, by, bz };
                        kernel(args...);
                        emu::g_bar.wait();                                    // block boundary: function-static "shared" storage is reused
                    }
        });
    for (auto& x : th) x.join();
#endif
}
#define EMU_LAUNCH(kernel, grid, block, ...) emu_launch(kernel, dim3(grid), dim3(block), ##__VA_ARGS__)

// ref_emu_cuda.h -- TEST INFRASTRUCTURE ONLY.  Lets the REFERENCE's own SiftGPU sources (FL/SiftGPU/ProgramCU.cu and its host classes) be
// compiled by g++ and executed on the CPU: the CUDA execution model comes from tests/cuda_emu/cuda_emu.h (one OS thread per CUDA thread,
// barriers), this header adds what that code needs beyond it -- texture references bound to linear memory (removed from CUDA 12, which is
// why the reference's ProgramCU.cu cannot be rebuilt by nvcc here), the vector types of cutil_math.h, and the handful of runtime calls the
// host classes make.  Approximate device intrinsics are mapped to exact functions (__sincosf -> sinf / cosf, __fdividef -> /, rsqrt ->
// 1 / sqrtf), which is the oracle's stated contract.  This file contains no reference code.
#pragma once
#include "cuda_emu.h"

#include <cassert>
#include <cmath>
#include <math.h>        // libstdc++'s wrapper: float overloads of exp / sqrt / atan2 / ... in the global namespace, as in CUDA device code
#include <string>

#define __constant__
#define __align__(n) __attribute__((aligned(n)))
#define __inline__ inline

// ---- vector types beyond cuda_emu.h ----
struct float3 { float x, y, z; }; struct int3 { int x, y, z; };        // int4 / uint4 and their make_ functions: cuda_emu.h
struct uchar3 { unsigned char x, y, z; }; struct ushort2 { unsigned short x, y; };
static inline float3 make_float3(float x, float y, float z) { return { x, y, z }; }
static inline int3 make_int3(int x, int y, int z) { return { x, y, z }; }
static inline uint3 make_uint3(unsigned x, unsigned y, unsigned z) { return { x, y, z }; }

#define CUDA_VERSION 12090
#define CUDART_VERSION 12090

// ---- intrinsics ----
static inline double min(float a, double b) { return a < b ? (double)a : b; }
static inline double min(double a, float b) { return a < b ? a : (double)b; }
static inline double max(float a, double b) { return a > b ? (double)a : b; }
static inline double max(double a, float b) { return a > b ? a : (double)b; }
static inline unsigned min(unsigned a, int b) { return a < (unsigned)b ? a : (unsigned)b; }
static inline unsigned min(int a, unsigned b) { return (unsigned)a < b ? (unsigned)a : b; }
static inline unsigned max(unsigned a, int b) { return a > (unsigned)b ? a : (unsigned)b; }
static inline unsigned max(int a, unsigned b) { return (unsigned)a > b ? (unsigned)a : b; }
// (unsigned int) of a negative float: 0 on the GPU (cvt.rzi.u32.f32 saturates), undefined in C++ -- the reference relies on the former
static inline unsigned emu_f2u(double x) { if (!(x > 0.0)) return 0u; if (x >= 4294967296.0) return 0xFFFFFFFFu; return (unsigned)x; }
static inline float saturate(float x) { return x < 0.0f ? 0.0f : (x > 1.0f ? 1.0f : x); }
static inline int __mul24(int a, int b) { return a * b; }
static inline float __int_as_float(int v) { float f; std::memcpy(&f, &v, 4); return f; }
static inline int __float_as_int(float f) { int v; std::memcpy(&v, &f, 4); return v; }
static inline void emu_sincosf(float a, float* s, float* c) { *s = sinf(a); *c = cosf(a); }
#define __sincosf emu_sincosf                    /* glibc declares a symbol of that name */
static inline float __fdividef(float a, float b) { return a / b; }
static inline float rsqrt(float x) { return 1.0f / sqrtf(x); }
static inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }
static inline uchar3 make_uchar3(float x, float y, float z) { return { (unsigned char)x, (unsigned char)y, (unsigned char)z }; }     // in-range values: truncation, as cvt.rzi
enum { cudaTextureType1D = 1, cudaTextureType2D = 2 };
static inline float __shfl_down(float v, int d, int = 32) { return __shfl_down_sync(0xFFFFFFFFu, v, d); }
static inline float __shfl_xor(float v, int m, int = 32) { return __shfl_xor_sync(0xFFFFFFFFu, v, m); }
static const int warpSize = 32;
namespace emu { inline Barrier g_barSubset; }
static inline void emu_sync_first(unsigned n) { emu::g_barSubset.n = n; emu::g_barSubset.wait(); }   // a barrier only threads 0..n-1 of the block reach

// ---- runtime API used by the host classes ----
typedef void* cudaEvent_t;
struct cudaArray;
struct cudaChannelFormatDesc { int x, y, z, w, f; };
struct cudaDeviceProp { char name[256]; size_t totalGlobalMem; int major, minor, multiProcessorCount; };
enum { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaChannelFormatKindFloat = 2, cudaEventBlockingSync = 1,
       cudaReadModeElementType = 0, cudaReadModeNormalizedFloat = 1, cudaFilterModePoint = 0 };
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, int) { std::memmove(d, s, n); return 0; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, int, cudaStream_t = nullptr) { std::memmove(d, s, n); return 0; }
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { std::memset(d, v, n); return 0; }
template <class S> static inline cudaError_t cudaMemcpyToSymbol(S& sym, const void* s, size_t n, size_t off = 0, int = 1) { std::memcpy(reinterpret_cast<char*>(&sym) + off, s, n); return 0; }
template <class S> static inline cudaError_t cudaGetSymbolSize(size_t* n, S& sym) { *n = sizeof(S); return 0; }
static inline cudaError_t cudaDeviceSynchronize() { return 0; }
static inline cudaError_t cudaSetDevice(int) { return 0; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return 0; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return 0; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) { std::memset(p, 0, sizeof *p); p->major = 10; return 0; }
static inline const char* cudaGetErrorString(cudaError_t) { return "emulated"; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = nullptr; return 0; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, int) { *e = nullptr; return 0; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return 0; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return 0; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0; return 0; }
static inline cudaError_t cudaMallocArray(cudaArray**, const cudaChannelFormatDesc*, size_t, size_t) { return 1; }
static inline cudaError_t cudaFreeArray(cudaArray*) { return 0; }
static inline cudaError_t cudaMemcpy2DToArray(cudaArray*, size_t, size_t, const void*, size_t, size_t, size_t, int) { return 1; }
static inline cudaError_t cudaMemcpyFromArray(void*, const cudaArray*, size_t, size_t, size_t, int) { return 1; }
static inline cudaError_t cudaGetChannelDesc(cudaChannelFormatDesc*, const cudaArray*) { return 1; }
static inline cudaChannelFormatDesc cudaCreateChannelDesc(int x, int y, int z, int w, int f) { return cudaChannelFormatDesc{ x, y, z, w, f }; }

// ---- texture references over linear memory (point sampling; out-of-range 1-D fetches return zero, 2-D coordinates clamp) ----
struct textureReference { const void* ptr = nullptr; size_t bytes = 0; int width = 0, height = 0; size_t pitch = 0; cudaChannelFormatDesc channelDesc{}; int filterMode = 0; };
template <class T, int Dim = 1, int Mode = 0> struct texture : textureReference {};
static inline cudaError_t cudaBindTexture(size_t* off, textureReference* r, const void* p, const cudaChannelFormatDesc*, size_t bytes) { if (off) *off = 0; r->ptr = p; r->bytes = bytes; return 0; }
static inline cudaError_t cudaBindTexture2D(size_t* off, textureReference* r, const void* p, const cudaChannelFormatDesc*, size_t w, size_t h, size_t pitch) {
    if (off) *off = 0; r->ptr = p; r->width = (int)w; r->height = (int)h; r->pitch = pitch; r->bytes = pitch * h; return 0; }
static inline cudaError_t cudaBindTextureToArray(textureReference*, const cudaArray*, const cudaChannelFormatDesc*) { return 1; }
template <class T> static inline T tex1Dfetch(const texture<T, 1, cudaReadModeElementType>& t, int i) {
    const size_t n = t.bytes / sizeof(T);
    return (i >= 0 && (size_t)i < n) ? static_cast<const T*>(t.ptr)[i] : T();
}
static inline float tex1Dfetch(const texture<unsigned char, 1, cudaReadModeNormalizedFloat>& t, int i) {
    return (i >= 0 && (size_t)i < t.bytes) ? static_cast<const unsigned char*>(t.ptr)[i] / 255.0f : 0.0f;
}
template <class T> static inline T tex2D(const texture<T, 2, cudaReadModeElementType>& t, float x, float y) {
    int ix = (int)floorf(x), iy = (int)floorf(y);
    ix = ix < 0 ? 0 : (ix > t.width - 1 ? t.width - 1 : ix); iy = iy < 0 ? 0 : (iy > t.height - 1 ? t.height - 1 : iy);
    return *reinterpret_cast<const T*>(static_cast<const char*>(t.ptr) + (size_t)iy * t.pitch + (size_t)ix * sizeof(T));
}

// kernel <<< grid, block [, smem, stream] >>> (args) is rewritten into EMU_KERNEL(kernel, grid, block ...)(args); the generic lambda lets the
// call site's argument types pick among overloaded kernels, as the launch syntax does
#define EMU_KERNEL(K, ...) emu::launcher([](auto... a_) { K(a_...); }, __VA_ARGS__)
namespace emu {
template <class K> struct Launcher {
    K k; dim3 g, b;
    template <class... A> void operator()(A... a) const { emu_launch(k, g, b, a...); }
};
template <class K> static inline Launcher<K> launcher(K k, dim3 g, dim3 b, size_t = 0, cudaStream_t = nullptr) { return { k, g, b }; }
}  // namespace emu

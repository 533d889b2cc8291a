// ingest.cu -- per-frame sensor-image preparation for sm_90a.  Implements include/bf_ingest.h (row a21 of SURVEY.md section 8).
//
// Behavioural source (what, not how): FL/CUDAImageManager.cpp:44-61, 88-137 and FL/CUDAImageUtil.cu erodeDepthMapDevice (:701-741),
// gaussFilterDepthMapDevice (:759-794), resampleFloat_Kernel (:93-110), resampleUCHAR4_Kernel (:160-177).
// The reference: erode -> erode -> range-gated Gaussian -> copy/resample, four or five full-image launches through three intermediate
// images.  Here: ONE launch.  A CTA stages a 32x32 tile of the raw depth plus a (2*3 + 4 = 10)-pixel halo in shared memory, erodes it
// twice and filters it there (ping-pong between two tile buffers; pixels outside the image are skipped exactly as the reference's
// bounds tests skip them), then writes the integration-resolution pixels whose nearest source pixel lies in its tile.  The colour
// copy / resample rides along as a grid-stride loop.  One read of the inputs, one write of the outputs.
//
// Arithmetic contract (bit-exact with oracle/ingest_oracle.c): TU built -fmad=false; Gaussian weights from the HOST's expf, once per
// offset; sums in the reference's loop order (x outer, y inner); fmaf only in x * scale + 0.5.
#include <cmath>

#include "../../include/bf_ingest.h"
#include "bf_common.cuh"

namespace bf {

extern unsigned long long g_launchCount;

#define BF_ING_T 32
#define BF_ING_MAX_R 8

struct IngestArgs {
    BFIngestParams p;
    const float* depthRaw; const uchar4* colorRaw; float* depthOut; uchar4* colorOut;
    int iters, s, r, halo;
    float wG[(2 * BF_ING_MAX_R + 1) * (2 * BF_ING_MAX_R + 1)];
};

__device__ __forceinline__ unsigned src_index(unsigned o, float scale) { return (unsigned)__fmaf_rn((float)o, scale, 0.5f); }

// ---- the application's configuration (two 7x7 erosions, 9x9 Gaussian: zParametersDefault.txt) with compile-time extents ----------------------
// Same operations in the same order as the generic loops of ingest_kernel; what changes is what the compiler can do with them: the 49 / 81 taps are
// unrolled (tile addresses become immediate offsets, the Gaussian weights immediate constant-bank operands), the element <-> (tx, ty) maps divide by
// constants, and no tap tests the image bounds: pixels outside the image are staged as NaN, which no tap test accepts (see the staging comment).
#define BF_ING_FS 3
#define BF_ING_FR 4
#define BF_ING_FDIM (BF_ING_T + 2 * (2 * BF_ING_FS + BF_ING_FR))

template <int IT, bool BORDER>
__device__ __forceinline__ void erode_pass_fast(const float* __restrict__ in, float* __restrict__ out, int x0, int y0, int W, int H, float dThresh, float fracReq) {
    constexpr int S = BF_ING_FS, DIM = BF_ING_FDIM, M0 = (IT + 1) * S, WD = DIM - 2 * M0;
    const float sumWin = (float)(unsigned)((2 * S + 1) * (2 * S + 1));
    for (int e = threadIdx.x; e < WD * WD; e += blockDim.x) {
        const int tx = M0 + e % WD, ty = M0 + e / WD, gx = x0 + tx, gy = y0 + ty;
        if (BORDER && (gx < 0 || gx >= W || gy < 0 || gy >= H)) { out[ty * DIM + tx] = nanf(""); continue; }      // stays "outside" for the next pass
        const float* c = in + ty * DIM + tx;
        const float old = c[0];
        unsigned count = 0;
#pragma unroll
        for (int i = -S; i <= S; ++i)
#pragma unroll
            for (int j = -S; j <= S; ++j) {
                const float d = c[i * DIM + j];                              // an out-of-image tap is NaN: none of the three tests holds
                if (d == -INFINITY || d == 0.0f || fabsf(d - old) > dThresh) ++count;
            }
        out[ty * DIM + tx] = ((float)count / sumWin >= fracReq) ? -INFINITY : old;
    }
}

template <bool BORDER>
__device__ __forceinline__ void gauss_pass_fast(const IngestArgs& a, const float* __restrict__ in, float* __restrict__ out, int x0, int y0, int W, int H) {
    constexpr int R = BF_ING_FR, SPAN = 2 * R + 1, DIM = BF_ING_FDIM, HALO = 2 * BF_ING_FS + BF_ING_FR;
    const float sigmaR = a.p.depthSigmaR;
    for (int e = threadIdx.x; e < BF_ING_T * BF_ING_T; e += blockDim.x) {
        const int tx = HALO + e % BF_ING_T, ty = HALO + e / BF_ING_T, gx = x0 + tx, gy = y0 + ty;
        if (gx >= W || gy >= H) continue;
        const float* cp = in + ty * DIM + tx;
        const float c = cp[0];
        float res = -INFINITY;
        if (c != -INFINITY) {
            float sum = 0.0f, sumW = 0.0f;
#pragma unroll
            for (int m = -R; m <= R; ++m)
#pragma unroll
                for (int n = -R; n <= R; ++n) {
                    const float cur = cp[n * DIM + m];                       // out-of-image: NaN, |c - NaN| < sigmaR is false
                    if (cur != -INFINITY && fabsf(c - cur) < sigmaR) { const float wgt = a.wG[(m + R) * SPAN + (n + R)]; sumW += wgt; sum += wgt * cur; }
                }
            if (sumW > 0.0f) res = sum / sumW;
        }
        out[ty * DIM + tx] = res;
    }
}

__global__ void __launch_bounds__(256)
ingest_kernel(const __grid_constant__ IngestArgs a) {
    extern __shared__ float sm[];
    const int W = (int)a.p.depthWidth, H = (int)a.p.depthHeight, w = (int)a.p.widthIntegration, h = (int)a.p.heightIntegration;
    const int halo = a.halo, dim = BF_ING_T + 2 * halo;
    float* bufA = sm; float* bufB = sm + dim * dim;
    const int x0 = (int)blockIdx.x * BF_ING_T - halo, y0 = (int)blockIdx.y * BF_ING_T - halo;      // image coordinates of tile element (0, 0)

    // ---- colour: copy / nearest resample, grid-stride over the integration image (CUDAImageManager.cpp:44-61) ----
    {
        const int CW = (int)a.p.colorWidth, CH = (int)a.p.colorHeight;
        const unsigned nthreads = gridDim.x * gridDim.y * blockDim.x, gtid = (blockIdx.y * gridDim.x + blockIdx.x) * blockDim.x + threadIdx.x;
        const float sw = (float)(CW - 1) / (float)(w - 1), sh = (float)(CH - 1) / (float)(h - 1);
        const bool same = (CW == w && CH == h);
        for (unsigned i = gtid; i < (unsigned)(w * h); i += nthreads) {
            if (same) { a.colorOut[i] = __ldg(&a.colorRaw[i]); continue; }
            const unsigned xi = src_index(i % (unsigned)w, sw), yi = src_index(i / (unsigned)w, sh);
            if (xi < (unsigned)CW && yi < (unsigned)CH) a.colorOut[i] = __ldg(&a.colorRaw[yi * CW + xi]);
        }
    }
    // ---- depth: stage the raw tile + halo.  Elements outside the image hold NaN: the generic passes never read them (they test the bounds), the
    // compile-time passes read them and need no bounds test -- a NaN tap is not -inf, not 0, and no comparison with it holds, so it is skipped exactly as
    // the reference's bounds test skips it (and an in-image NaN behaves as it does in the reference) ----
    for (int e = threadIdx.x; e < dim * dim; e += blockDim.x) {
        const int gx = x0 + e % dim, gy = y0 + e / dim;
        bufA[e] = (gx >= 0 && gx < W && gy >= 0 && gy < H) ? __ldg(&a.depthRaw[gy * W + gx]) : nanf("");     // outside the image: NaN fails every tap test below by itself
    }
    __syncthreads();
    float* out;
    if (a.iters == 2 && a.s == BF_ING_FS && a.r == BF_ING_FR) {
        // the application's configuration, compile-time extents (see erode_pass_fast / gauss_pass_fast); a tile is a border tile if its halo leaves the image
        const bool border = x0 < 0 || y0 < 0 || x0 + dim > W || y0 + dim > H;
        if (border) {
            erode_pass_fast<0, true>(bufA, bufB, x0, y0, W, H, a.p.erodeDThresh, a.p.erodeFracReq); __syncthreads();
            erode_pass_fast<1, true>(bufB, bufA, x0, y0, W, H, a.p.erodeDThresh, a.p.erodeFracReq); __syncthreads();
            gauss_pass_fast<true>(a, bufA, bufB, x0, y0, W, H);
        } else {
            erode_pass_fast<0, false>(bufA, bufB, x0, y0, W, H, a.p.erodeDThresh, a.p.erodeFracReq); __syncthreads();
            erode_pass_fast<1, false>(bufB, bufA, x0, y0, W, H, a.p.erodeDThresh, a.p.erodeFracReq); __syncthreads();
            gauss_pass_fast<false>(a, bufA, bufB, x0, y0, W, H);
        }
        out = bufB;
        __syncthreads();
    } else {
        // ---- erosions (erodeDepthMapDevice, :701-741): pass k is valid on the tile shrunk by (k + 1) * s ----
        float* in = bufA; out = bufB;
        const int s = a.s;
        const float sumWin = (float)(unsigned)((2 * s + 1) * (2 * s + 1));
        for (int it = 0; it < a.iters; ++it) {
            const int m0 = (it + 1) * s, m1 = dim - (it + 1) * s;
            for (int e = threadIdx.x; e < dim * dim; e += blockDim.x) {
                const int tx = e % dim, ty = e / dim, gx = x0 + tx, gy = y0 + ty;
                if (tx < m0 || tx >= m1 || ty < m0 || ty >= m1 || gx < 0 || gx >= W || gy < 0 || gy >= H) continue;
                unsigned count = 0;
                const float old = in[e];
                for (int i = -s; i <= s; ++i)
                    for (int j = -s; j <= s; ++j)
                        if (gx + j >= 0 && gx + j < W && gy + i >= 0 && gy + i < H) {
                            const float d = in[(ty + i) * dim + tx + j];
                            if (d == -INFINITY || d == 0.0f || fabsf(d - old) > a.p.erodeDThresh) ++count;
                        }
                out[e] = ((float)count / sumWin >= a.p.erodeFracReq) ? -INFINITY : old;
            }
            __syncthreads();
            float* t = in; in = out; out = t;
        }
        // ---- range-gated Gaussian (gaussFilterDepthMapDevice, :759-794) on the 32x32 core, result into `out` ----
        {
            const int r = a.r, span = 2 * r + 1;
            for (int e = threadIdx.x; e < BF_ING_T * BF_ING_T; e += blockDim.x) {
                const int tx = halo + e % BF_ING_T, ty = halo + e / BF_ING_T, gx = x0 + tx, gy = y0 + ty;
                if (gx >= W || gy >= H) continue;
                const float c = in[ty * dim + tx];
                float res = c;
                if (r >= 0) {
                    res = -INFINITY;
                    if (c != -INFINITY) {
                        float sum = 0.0f, sumW = 0.0f;
                        for (int m = -r; m <= r; ++m)
                            for (int n = -r; n <= r; ++n)
                                if (gx + m >= 0 && gy + n >= 0 && gx + m < W && gy + n < H) {
                                    const float cur = in[(ty + n) * dim + tx + m];
                                    if (cur != -INFINITY && fabsf(c - cur) < a.p.depthSigmaR) { const float wgt = a.wG[(m + r) * span + (n + r)]; sumW += wgt; sum += wgt * cur; }
                                }
                        if (sumW > 0.0f) res = sum / sumW;
                    }
                }
                out[ty * dim + tx] = res;
            }
        }
        __syncthreads();
    }
    // ---- write: copy, or the integration pixels whose nearest source pixel is in this tile's core (resampleFloat_Kernel, :93-110) ----
    const int cx0 = (int)blockIdx.x * BF_ING_T, cy0 = (int)blockIdx.y * BF_ING_T;
    if (W == w && H == h) {
        for (int e = threadIdx.x; e < BF_ING_T * BF_ING_T; e += blockDim.x) {
            const int gx = cx0 + e % BF_ING_T, gy = cy0 + e / BF_ING_T;
            if (gx < W && gy < H) a.depthOut[gy * W + gx] = out[(halo + e / BF_ING_T) * dim + halo + e % BF_ING_T];
        }
    } else {
        const float sw = (float)(W - 1) / (float)(w - 1), sh = (float)(H - 1) / (float)(h - 1);
        int ox0 = (int)floorf((float)cx0 / sw) - 1, ox1 = (int)ceilf((float)(cx0 + BF_ING_T) / sw) + 2;
        int oy0 = (int)floorf((float)cy0 / sh) - 1, oy1 = (int)ceilf((float)(cy0 + BF_ING_T) / sh) + 2;
        ox0 = ox0 < 0 ? 0 : ox0; oy0 = oy0 < 0 ? 0 : oy0; ox1 = ox1 > w ? w : ox1; oy1 = oy1 > h ? h : oy1;
        const int nx = ox1 - ox0, ny = oy1 - oy0;
        for (int e = threadIdx.x; e < nx * ny; e += blockDim.x) {
            const int ox = ox0 + e % nx, oy = oy0 + e / nx;
            const int xi = (int)src_index((unsigned)ox, sw), yi = (int)src_index((unsigned)oy, sh);
            if (xi >= cx0 && xi < cx0 + BF_ING_T && yi >= cy0 && yi < cy0 + BF_ING_T && xi < W && yi < H)
                a.depthOut[oy * w + ox] = out[(halo + yi - cy0) * dim + halo + xi - cx0];
        }
    }
}

}  // namespace bf

using namespace bf;

BF_API int bfIngestFrame(const BFIngestParams* params, const float* d_depthRaw, const uint8_t* d_colorRaw, float* d_depthIntegration, uint8_t* d_colorIntegration) {
    if (!params || !d_depthRaw || !d_colorRaw || !d_depthIntegration || !d_colorIntegration) return (int)cudaErrorInvalidValue;
    if (params->widthIntegration < 2 || params->heightIntegration < 2 || params->erodeStructureSize < 0) return (int)cudaErrorInvalidValue;
    IngestArgs a;
    a.p = *params;
    a.depthRaw = d_depthRaw; a.colorRaw = reinterpret_cast<const uchar4*>(d_colorRaw);
    a.depthOut = d_depthIntegration; a.colorOut = reinterpret_cast<uchar4*>(d_colorIntegration);
    a.iters = params->erodeIterations > 0 ? 2 * ((params->erodeIterations + 1) / 2) : 0;      // CUDAImageManager.cpp:89-90
    a.s = params->erodeStructureSize;
    a.r = -1;
    if (params->depthSigmaD > 0.0f) {
        a.r = (int)ceil(2.0 * params->depthSigmaD);
        if (a.r > BF_ING_MAX_R) return (int)cudaErrorInvalidValue;
        const float sD = params->depthSigmaD;
        for (int dx = -a.r; dx <= a.r; ++dx) for (int dy = -a.r; dy <= a.r; ++dy)
            a.wG[(dx + a.r) * (2 * a.r + 1) + (dy + a.r)] = expf(-((float)(dx * dx + dy * dy) / (2.0f * sD * sD)));
    }
    a.halo = a.iters * a.s + (a.r > 0 ? a.r : 0);
    const int dim = BF_ING_T + 2 * a.halo;
    const size_t smem = sizeof(float) * 2 * (size_t)dim * dim;
    if (smem > 200 * 1024) return (int)cudaErrorInvalidValue;
    static size_t smemSet = 0;
    if (smem > 48 * 1024 && smem > smemSet) { BF_CHECK(cudaFuncSetAttribute(ingest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); smemSet = smem; }
    dim3 grid((params->depthWidth + BF_ING_T - 1) / BF_ING_T, (params->depthHeight + BF_ING_T - 1) / BF_ING_T);
    ++g_launchCount;
    ingest_kernel<<<grid, 256, smem, stream()>>>(a);
    BF_CHECK(cudaGetLastError());
    return 0;
}

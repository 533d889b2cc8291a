// cache.cu -- dense-cache frame builder for sm_90a.  Implements include/bf_cache.h (row a20 of SURVEY.md section 8).
//
// Behavioural source (what, not how): FL/CUDACache.cpp:45-86 and the eight FL/CUDAImageUtil.cu kernels it calls (listed in the
// header).  The reference filters, back-projects and takes normals of the WHOLE 640x480 image (3 full-resolution float / float4
// intermediates, ~15 MB of traffic, 8 launches) and then keeps 80x60 samples of it.  Here ONE launch evaluates, for each of the
// 4 800 cache pixels, exactly the values the reference would have sampled: the range-gated Gaussian of the depth at the five
// full-resolution pixels the position and its normal need, and -- in 8x8 tiles through shared memory -- the resampled intensity,
// its Gaussian and the Sobel derivatives.  ~100 KB of traffic.
//
// Arithmetic contract (bit-exact with oracle/cache_oracle.c, see its header): this TU is built -fmad=false; fmaf only where written;
// Gaussian weights come from the HOST's expf, once per offset; sums run in the reference's loop order.
#include <cmath>

#include "../../include/bf_cache.h"
#include "bf_common.cuh"

namespace bf {

extern unsigned long long g_launchCount;

#define BF_CACHE_MAX_RD 4          // depth filter radius  (ceil(2 sigmaD)), default 2
#define BF_CACHE_MAX_RI 8          // intensity filter radius (ceil(2 sigma)), default 5

struct CacheArgs {
    BFCacheParams p;
    const float* depth; const uchar4* color;
    float* oDepth; float4* oCampos; float4* oNormals; uchar4* oNormalsU; float* oIntensity; float2* oDerivs;
    int rD, rI;
    float wD[(2 * BF_CACHE_MAX_RD + 1) * (2 * BF_CACHE_MAX_RD + 1)];
    float wI[(2 * BF_CACHE_MAX_RI + 1) * (2 * BF_CACHE_MAX_RI + 1)];
};

__device__ __forceinline__ unsigned src_index(unsigned o, float scale) { return (unsigned)__fmaf_rn((float)o, scale, 0.5f); }

// gaussFilterDepthMapDevice at one full-resolution pixel (CUDAImageUtil.cu:759-794)
__device__ float depth_filtered(const CacheArgs& a, int x, int y) {
    const int W = (int)a.p.inputDepthWidth, H = (int)a.p.inputDepthHeight;
    const float c = __ldg(&a.depth[y * W + x]);
    if (a.rD < 0) return c;                                  // filter off
    if (c == -INFINITY) return -INFINITY;
    const int r = a.rD, span = 2 * r + 1;
    float sum = 0.0f, sumW = 0.0f;
    for (int m = x - r; m <= x + r; ++m)
        for (int n = y - r; n <= y + r; ++n)
            if (m >= 0 && n >= 0 && m < W && n < H) {
                const float cur = __ldg(&a.depth[n * W + m]);
                if (cur != -INFINITY && fabsf(c - cur) < a.p.filterDepthSigmaR) {
                    const float wgt = a.wD[(m - x + r) * span + (n - y + r)];
                    sumW += wgt;
                    sum += wgt * cur;
                }
            }
    return (sumW > 0.0f) ? sum / sumW : -INFINITY;
}
// convertDepthFloatToCameraSpaceFloat4_Kernel at one pixel (:367-386): (x, y, w) of intrinsicsInv * (x d, y d, d, d)
__device__ float4 campos_from(const CacheArgs& a, int x, int y, float d) {
    if (d == -INFINITY) return make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    const float* M = a.p.inputIntrinsicsInv;
    const float v0 = (float)x * d, v1 = (float)y * d;
    const float rx = ((M[0] * v0 + M[1] * v1) + M[2] * d) + M[3] * d;
    const float ry = ((M[4] * v0 + M[5] * v1) + M[6] * d) + M[7] * d;
    const float rw = ((M[12] * v0 + M[13] * v1) + M[14] * d) + M[15] * d;
    return make_float4(rx, ry, rw, 1.0f);
}
__device__ float4 campos_at(const CacheArgs& a, int x, int y) { return campos_from(a, x, y, depth_filtered(a, x, y)); }

#define BF_CACHE_IT 8                                                        // intensity tile edge (cache pixels)
#define BF_CACHE_RDIM (BF_CACHE_IT + 2 + 2 * BF_CACHE_MAX_RI)                // tile + the Sobel ring + the Gaussian halo
#define BF_CACHE_FDIM (BF_CACHE_IT + 2)

__global__ void __launch_bounds__(256)
cache_store_kernel(const __grid_constant__ CacheArgs a, int nIntensityTiles) {
    const int w = (int)a.p.width, h = (int)a.p.height, npx = w * h;
    if ((int)blockIdx.x < nIntensityTiles) {
        // ---- intensity path: resample -> Gaussian -> Sobel / 8 on an 8x8 tile of the cache image.  The CTA recomputes what its tile needs of its
        // neighbours' pixels (resampled intensity on the tile + Sobel ring + Gaussian halo, filtered intensity on the tile + Sobel ring): every value
        // is the same expression of the same inputs whichever CTA evaluates it, so the image is the one a single pass over it produces ----
        __shared__ float sH[BF_CACHE_RDIM * BF_CACHE_RDIM];      // resampled intensity
        __shared__ float sF[BF_CACHE_FDIM * BF_CACHE_FDIM];      // filtered intensity
        const int tilesX = (w + BF_CACHE_IT - 1) / BF_CACHE_IT;
        const int tx0 = ((int)blockIdx.x % tilesX) * BF_CACHE_IT, ty0 = ((int)blockIdx.x / tilesX) * BF_CACHE_IT;
        const int r = a.rI > 0 ? a.rI : 0, dimR = BF_CACHE_IT + 2 + 2 * r, rx0 = tx0 - 1 - r, ry0 = ty0 - 1 - r;
        const int CW = (int)a.p.inputColorWidth, CH = (int)a.p.inputColorHeight;
        const float cw = (float)(CW - 1) / (float)(w - 1), ch = (float)(CH - 1) / (float)(h - 1);
        for (int e = threadIdx.x; e < dimR * dimR; e += blockDim.x) {
            const int x = rx0 + e % dimR, y = ry0 + e / dimR;
            float v = 0.0f;
            if (x >= 0 && x < w && y >= 0 && y < h) {
                const unsigned xi = src_index((unsigned)x, cw), yi = src_index((unsigned)y, ch);
                if (xi < (unsigned)CW && yi < (unsigned)CH) {
                    const uchar4 c = __ldg(&a.color[yi * CW + xi]);
                    v = __fmaf_rn(0.114f, (float)c.z, __fmaf_rn(0.299f, (float)c.x, 0.587f * (float)c.y)) / 255.0f;   // convertToIntensity, :196-199
                }
            }
            sH[e] = v;
        }
        __syncthreads();
        for (int e = threadIdx.x; e < BF_CACHE_FDIM * BF_CACHE_FDIM; e += blockDim.x) {
            const int fx = e % BF_CACHE_FDIM, fy = e / BF_CACHE_FDIM, x = tx0 - 1 + fx, y = ty0 - 1 + fy;
            if (x < 0 || x >= w || y < 0 || y >= h) continue;
            const int cx = fx + r, cy = fy + r;                  // the pixel's position in sH
            float v = sH[cy * dimR + cx];
            if (a.rI >= 0) {                                  // gaussFilterIntensityDevice, :811-848
                const int span = 2 * r + 1;
                float sum = 0.0f, sumW = 0.0f;
                for (int m = -r; m <= r; ++m)
                    for (int n = -r; n <= r; ++n)
                        if (x + m >= 0 && y + n >= 0 && x + m < w && y + n < h) { const float wgt = a.wI[(m + r) * span + (n + r)]; sumW += wgt; sum += wgt * sH[(cy + n) * dimR + cx + m]; }
                v = (sumW > 0.0f) ? sum / sumW : 0.0f;
            }
            sF[e] = v;
            if (fx >= 1 && fx <= BF_CACHE_IT && fy >= 1 && fy <= BF_CACHE_IT) a.oIntensity[y * w + x] = v;
        }
        __syncthreads();
        for (int e = threadIdx.x; e < BF_CACHE_IT * BF_CACHE_IT; e += blockDim.x) {  // computeIntensityDerivatives_Kernel, :260-296
            const int fx = 1 + e % BF_CACHE_IT, fy = 1 + e / BF_CACHE_IT, x = tx0 - 1 + fx, y = ty0 - 1 + fy;
            if (x >= w || y >= h) continue;
            float2 o = make_float2(-INFINITY, -INFINITY);
            if (x > 0 && x < w - 1 && y > 0 && y < h - 1) {
                const float* c = sF + fy * BF_CACHE_FDIM + fx;
                const float p00 = c[-BF_CACHE_FDIM - 1], p01 = c[-1], p02 = c[BF_CACHE_FDIM - 1], p10 = c[-BF_CACHE_FDIM],
                            p12 = c[BF_CACHE_FDIM], p20 = c[-BF_CACHE_FDIM + 1], p21 = c[1], p22 = c[BF_CACHE_FDIM + 1];
                if (!(p00 == -INFINITY || p01 == -INFINITY || p02 == -INFINITY || p10 == -INFINITY || p12 == -INFINITY || p20 == -INFINITY ||
                      p21 == -INFINITY || p22 == -INFINITY)) {
                    const float rU = (-1.0f) * p00 + (1.0f) * p20 + (-2.0f) * p01 + (2.0f) * p21 + (-1.0f) * p02 + (1.0f) * p22;
                    const float rV = (-1.0f) * p00 + (-2.0f) * p10 + (-1.0f) * p20 + (1.0f) * p02 + (2.0f) * p12 + (1.0f) * p22;
                    o = make_float2(rU / 8.0f, rV / 8.0f);
                }
            }
            a.oDerivs[y * w + x] = o;
        }
        return;
    }
    // ---- depth path: one thread per cache pixel ----
    const int i = ((int)blockIdx.x - nIntensityTiles) * (int)blockDim.x + (int)threadIdx.x;
    if (i >= npx) return;
    const int W = (int)a.p.inputDepthWidth, H = (int)a.p.inputDepthHeight;
    const float sw = (float)(W - 1) / (float)(w - 1), sh = (float)(H - 1) / (float)(h - 1);
    const unsigned xi = src_index((unsigned)(i % w), sw), yi = src_index((unsigned)(i / w), sh);
    if (!(xi < (unsigned)W && yi < (unsigned)H)) return;     // resample*_Kernel leave the pixel untouched (:104, :137)
    const int x = (int)xi, y = (int)yi;
    const float d0 = depth_filtered(a, x, y);
    const float4 CC = campos_from(a, x, y, d0);
    a.oDepth[i] = d0;                                        // resampleFloat of the filtered depth (CUDACache.cpp:71)
    a.oCampos[i] = CC;
    float4 nrm = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    if (x > 0 && x < W - 1 && y > 0 && y < H - 1 && CC.x != -INFINITY) {           // computeNormals_Kernel, :404-431
        const float4 PC = campos_at(a, x, y + 1), CP = campos_at(a, x + 1, y), MC = campos_at(a, x, y - 1), CM = campos_at(a, x - 1, y);
        if (PC.x != -INFINITY && CP.x != -INFINITY && MC.x != -INFINITY && CM.x != -INFINITY) {
            const float ax = PC.x - MC.x, ay = PC.y - MC.y, az = PC.z - MC.z, bx = CP.x - CM.x, by = CP.y - CM.y, bz = CP.z - CM.z;
            const float nx = ay * bz - az * by, ny = az * bx - ax * bz, nz = ax * by - ay * bx;
            const float l = sqrtf((nx * nx + ny * ny) + nz * nz);
            if (l > 0.0f) nrm = make_float4(nx / -l, ny / -l, nz / -l, 0.0f);
        }
    }
    a.oNormals[i] = nrm;
    uchar4 u = make_uchar4(0, 0, 0, 0);                      // convertNormalsFloat4ToUCHAR4_Kernel, :497-513
    if (nrm.x != -INFINITY)
        u = make_uchar4((unsigned char)roundf(((nrm.x + 1.0f) / 2.0f) * 255.0f), (unsigned char)roundf(((nrm.y + 1.0f) / 2.0f) * 255.0f),
                        (unsigned char)roundf(((nrm.z + 1.0f) / 2.0f) * 255.0f), 0);
    a.oNormalsU[i] = u;
}

}  // namespace bf

using namespace bf;

BF_API int bfCacheStoreFrame(const BFCacheParams* params, const float* d_depth, const uint8_t* d_color, const BFCUDACachedFrame* frame) {
    if (!params || !d_depth || !d_color || !frame) return (int)cudaErrorInvalidValue;
    if (params->width < 2 || params->height < 2) return (int)cudaErrorInvalidValue;
    CacheArgs a;
    a.p = *params;
    a.depth = d_depth; a.color = reinterpret_cast<const uchar4*>(d_color);
    a.oDepth = frame->d_depthDownsampled; a.oCampos = reinterpret_cast<float4*>(frame->d_cameraposDownsampled);
    a.oNormals = reinterpret_cast<float4*>(frame->d_normalsDownsampled); a.oNormalsU = reinterpret_cast<uchar4*>(frame->d_normalsDownsampledUCHAR4);
    a.oIntensity = frame->d_intensityDownsampled; a.oDerivs = reinterpret_cast<float2*>(frame->d_intensityDerivsDownsampled);
    // gaussD(sigma, dx, dy) = exp(-((dx*dx + dy*dy) / (2 sigma sigma))), :531-534 -- evaluated here, once per offset
    a.rD = -1; a.rI = -1;
    if (params->filterDepthSigmaD > 0.0f) {
        a.rD = (int)ceil(2.0 * params->filterDepthSigmaD);
        if (a.rD > BF_CACHE_MAX_RD) return (int)cudaErrorInvalidValue;
        const float s = params->filterDepthSigmaD;
        for (int dx = -a.rD; dx <= a.rD; ++dx) for (int dy = -a.rD; dy <= a.rD; ++dy)
            a.wD[(dx + a.rD) * (2 * a.rD + 1) + (dy + a.rD)] = expf(-((float)(dx * dx + dy * dy) / (2.0f * s * s)));
    }
    if (params->filterIntensitySigma > 0.0f) {
        a.rI = (int)ceil(2.0 * params->filterIntensitySigma);
        if (a.rI > BF_CACHE_MAX_RI) return (int)cudaErrorInvalidValue;
        const float s = params->filterIntensitySigma;
        for (int dx = -a.rI; dx <= a.rI; ++dx) for (int dy = -a.rI; dy <= a.rI; ++dy)
            a.wI[(dx + a.rI) * (2 * a.rI + 1) + (dy + a.rI)] = expf(-((float)(dx * dx + dy * dy) / (2.0f * s * s)));
    }
    const int npx = (int)(params->width * params->height);
    const int nTiles = (int)((params->width + BF_CACHE_IT - 1) / BF_CACHE_IT) * (int)((params->height + BF_CACHE_IT - 1) / BF_CACHE_IT);
    ++g_launchCount;
    cache_store_kernel<<<nTiles + (npx + 255) / 256, 256, 0, stream()>>>(a, nTiles);
    BF_CHECK(cudaGetLastError());
    return 0;
}

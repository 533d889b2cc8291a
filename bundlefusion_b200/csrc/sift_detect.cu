// sift_detect.cu -- SIFT key-point detection and description for sm_90a (row a17).  Implements bfSiftDetect of include/bf_sift.h.
//
// Written against oracle/sift_detect_oracle.c; tests/test_zz_sift_detect_gpu.py checks it on the GPU.
//
// Behavioural source (what, not how): SiftGPU::RunSIFT + GetKeyPointsAndDescriptorsCUDA as Bundler::detectFeatures configures them
// (FL/Bundler.cpp:55-100; FL/SiftGPU/SiftPyramid.cpp, ProgramCU.cu -- the per-stage citations are in the oracle's header).
// The reference: ~70 launches per frame (FilterH + FilterV per level, DoG per level, key test per level, orientation / reshape /
// descriptor / normalise per level) with a device->host copy of the level counts in the middle and atomically appended, race-ordered
// lists.  Here: 27 launches, no host round trip, deterministic lists:
//   21 x sift_level_kernel      one launch per Gaussian level: separable filter with both passes in shared memory, the DoG against the
//                               input tile's centre and the gradient (magnitude, angle) of the output fused into the same launch;
//                               an octave's first level reads the previous octave through the 2:1 sub-sampling map
//    1 x sift_key_count_kernel  26-neighbour / edge / depth tests, key points counted per image row (all 12 levels in one grid)
//    1 x sift_key_scan_kernel   row offsets per level (one CTA per level)
//    1 x sift_key_emit_kernel   the same tests again, key points written at their raster rank
//    1 x sift_orient_kernel     one CTA per key point: 36-bin histogram, six box-filter passes, up to two peaks
//    1 x sift_reshape_kernel    (x, y, sigma, angle) list per level in raster order, one CTA per level
//    1 x sift_describe_kernel   one CTA per feature: 4x4x8 histogram, normalise / clamp / normalise, bytes and the global key point
// The whole pyramid (10 MB of Gaussians, 8 MB of DoG, 8 MB of gradients at 640x480) lives in L2; the path is launch- and
// latency-bound, not HBM-bound, which is why the work is organised to need few launches rather than tuned tiles.
// Arithmetic: filter taps come from the host (expf once per tap) and are applied with fmaf in tap order -- the pyramid, the DoG, the
// extrema and the gradient magnitudes are bit-identical to the oracle; atan2f / expf / sinf / cosf are CUDA's (a few ulp from glibc's)
// and histogram sums are taken in scheduling order (shared-memory atomics), so orientations and descriptors agree to ~1e-6 relative.
#include <algorithm>
#include <cmath>

#include "../../include/bf_sift.h"
#include "bf_common.cuh"

namespace bf {

extern unsigned long long g_launchCount;

#define SD_OCTAVES 4
#define SD_DOG 3
#define SD_LEVELS 6
#define SD_NLEV (SD_OCTAVES * SD_DOG)
#define SD_MAX_FW 33
#define SD_TILE 32
#define SD_MAX_LEVEL_FEATURES 4096

struct SdPyr {                                  // device pointers of one octave
    int w, h;
    float* gus[SD_LEVELS]; float* dog[SD_LEVELS]; float2* grad[SD_LEVELS];
};
struct SdCommon {
    SdPyr oc[SD_OCTAVES];
    int fmax[SD_OCTAVES];                       // list capacity per level of an octave
    int capBase[SD_NLEV + 1];                   // prefix of capacities over the 12 levels
    int rowBase[SD_NLEV + 1];                   // prefix of image rows over the 12 levels
    BFSiftDetectParams P;
    float sigma0, dogThreshold, edgeT;
    float levelSigma[SD_DOG];          // sigma0 * 2^(j / SD_DOG), host-evaluated
    int* rowCount; int* rowOffset;              // [rowBase[12]]
    int* levelRaw;                              // [12] key points per level after detection (min(count, fmax))
    int2* raw;                                  // [capBase[12]] (col, row)
    unsigned* oriPack;                          // [capBase[12]]
    float4* fin;                                // [capBase[12]] (x, y, sigma, angle)
    int* levelFinal;                            // [12] features per level after reshape
};

// ---- Gaussian level: H + V pass in shared memory, DoG and gradient fused (FilterH / FilterV / ComputeDOG_Kernel) ----
struct LevelArgs {
    const float* src; int srcW, srcH, subsample;        // subsample: 1 = read the previous octave's level through the 2:1 map
    int w, h, fw;
    float taps[SD_MAX_FW];
    float* gus; float* dog; float2* grad;
};

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

__global__ void __launch_bounds__(256)
sift_level_kernel(const __grid_constant__ LevelArgs a) {
    extern __shared__ float sm[];
    const int half = a.fw >> 1;
    const int ow = SD_TILE + 2;                           // outputs incl. the 1-pixel ring the gradient needs
    const int iw = ow + 2 * half;                         // input tile edge
    float* sIn = sm;                                      // [iw][iw]
    float* sH = sm + iw * iw;                             // [iw][ow]   H pass: every input row, output columns
    float* sOut = sH + iw * ow;                           // [ow][ow]
    const int x0 = (int)blockIdx.x * SD_TILE - 1, y0 = (int)blockIdx.y * SD_TILE - 1;      // image coordinates of output (0, 0) of the tile
    // stage the input with clamp-to-edge addressing (fetch_index clamps in FilterH / FilterV).  A warp takes whole tile rows and a lane up to four columns of
    // a row pair: eight independent loads are in flight per thread before the first is stored -- with one CTA per SM (the small octaves) a load's latency
    // is otherwise paid once per element -- and no index is divided
    {
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
        for (int r = 2 * warp; r < iw; r += 2 * nwarp) {
            float v[2][4];
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const int gy = clampi(y0 - half + r + rr, 0, a.h - 1);
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const int c = lane + 32 * k;
                    v[rr][k] = 0.0f;
                    if (c < iw && r + rr < iw) {
                        const int gx = clampi(x0 - half + c, 0, a.w - 1);
                        if (a.subsample) { const int sx = (gx << 1) < a.srcW - 1 ? (gx << 1) : a.srcW - 1; v[rr][k] = __ldg(&a.src[(size_t)(gy << 1) * a.srcW + sx]); }   // DownsampleKernel
                        else v[rr][k] = __ldg(&a.src[(size_t)gy * a.srcW + gx]);
                    }
                }
            }
#pragma unroll
            for (int rr = 0; rr < 2; ++rr)
#pragma unroll
                for (int k = 0; k < 4; ++k) { const int c = lane + 32 * k; if (c < iw && r + rr < iw) sIn[(r + rr) * iw + c] = v[rr][k]; }
        }
    }
    __syncthreads();
    // H pass, then V pass.  An output is a chain of fw dependent fused multiply-adds in tap order (the order is the contract); a thread carries four
    // outputs through the tap loop at once so that four chains overlap.
    // Output column x0 + c clamps its taps in IMAGE coordinates: tap i reads clamp(x0 + c - half + i); the staged tile holds clamp(x0 - half + t) at
    // position t, so for in-image output columns position c + i is exactly that pixel.
    for (int base = threadIdx.x; base < iw * ow; base += 4 * (int)blockDim.x) {
        float acc[4] = { 0.0f, 0.0f, 0.0f, 0.0f };
        int src[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) { const int e = base + u * (int)blockDim.x; src[u] = e < iw * ow ? (e / ow) * iw + e % ow : 0; }
        for (int i = 0; i < a.fw; ++i) {
            const float t = a.taps[i];
#pragma unroll
            for (int u = 0; u < 4; ++u) acc[u] = fmaf(sIn[src[u] + i], t, acc[u]);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) { const int e = base + u * (int)blockDim.x; if (e < iw * ow) sH[e] = acc[u]; }
    }
    __syncthreads();
    for (int base = threadIdx.x; base < ow * ow; base += 4 * (int)blockDim.x) {
        float acc[4] = { 0.0f, 0.0f, 0.0f, 0.0f };
        int src[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) { const int e = base + u * (int)blockDim.x; src[u] = e < ow * ow ? e : 0; }          // sH[(r + i) * ow + c] = sH[e + i * ow]
        for (int i = 0; i < a.fw; ++i) {
            const float t = a.taps[i];
#pragma unroll
            for (int u = 0; u < 4; ++u) acc[u] = fmaf(sH[src[u] + i * ow], t, acc[u]);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) { const int e = base + u * (int)blockDim.x; if (e < ow * ow) sOut[e] = acc[u]; }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < SD_TILE * SD_TILE; e += blockDim.x) {
        const int r = e / SD_TILE + 1, c = e % SD_TILE + 1, gx = x0 + c, gy = y0 + r;
        if (gx >= a.w || gy >= a.h) continue;
        const float v = sOut[r * ow + c];
        const size_t o = (size_t)gy * a.w + gx;
        a.gus[o] = v;
        if (a.dog) a.dog[o] = v - sIn[(r + half) * iw + c + half];
        if (a.grad) {
            float2 g = make_float2(0.0f, 0.0f);
            if (gx >= 1 && gx < a.w - 1 && gy >= 1 && gy < a.h - 1) {
                const float dx = sOut[r * ow + c + 1] - sOut[r * ow + c - 1], dy = sOut[(r + 1) * ow + c] - sOut[(r - 1) * ow + c];
                g.x = 0.5f * sqrtf(fmaf(dx, dx, dy * dy));
                g.y = g.x == 0.0f ? 0.0f : atan2f(dy, dx);
            }
            a.grad[o] = g;
        }
    }
}

// ---- ComputeKEY_Kernel: one test, used by the count and the emit pass ----
__device__ __forceinline__ bool cmp_rows(const float* img, int idx, float v, float& nmax, float& nmin) {      // READ_CMP_DOG_DATA: true = rejected
    const float d0 = __ldg(&img[idx - 1]), d1 = __ldg(&img[idx]), d2 = __ldg(&img[idx + 1]);
    if (v > nmax) { nmax = fmaxf(nmax, d0); nmax = fmaxf(nmax, d1); nmax = fmaxf(nmax, d2); if (v < nmax) return true; }
    else { nmin = fminf(nmin, d0); nmin = fminf(nmin, d1); nmin = fminf(nmin, d2); if (v > nmin) return true; }
    return false;
}

// The test in two parts so that a thread can have the first loads of several pixels in flight: key_where gives the two addresses every pixel's test
// starts with (its depth sample and its own DoG value; false: the pixel is out of range), key_test runs the rejections on the loaded values.  All of them
// are pure rejections, so loading d and v before the range tests changes nothing.
__device__ __forceinline__ bool key_where(const SdCommon& s, int o, int row, int col, int& depthIdx, int& index) {
    const SdPyr& oc = s.oc[o];
    const int w = oc.w;
    if (!(row > 0 && col > 0 && row < oc.h - 2 && col < w - 2)) return false;
    const float keyLocScale = (float)(1 << o);
    const BFSiftDetectParams& P = s.P;
    const int dxp = (int)roundf((keyLocScale * (float)col + 0.5f) * (float)(P.depthWidth - 1) / (float)(P.width - 1));
    const int dyp = (int)roundf((keyLocScale * (float)row + 0.5f) * (float)(P.depthHeight - 1) / (float)(P.height - 1));
    if (dxp < 0 || dxp >= (int)P.depthWidth || dyp < 0 || dyp >= (int)P.depthHeight) return false;
    depthIdx = dyp * (int)P.depthWidth + dxp;
    index = row * w + col;
    return true;
}
__device__ bool key_test(const SdCommon& s, int o, int j, int row, int col, float d, float v) {
    const SdPyr& oc = s.oc[o];
    const int w = oc.w;
    const BFSiftDetectParams& P = s.P;
    if (d == -INFINITY || d < P.depthMin || d > P.depthMax) return false;
    const float* dogP = oc.dog[j + 1]; const float* dogC = oc.dog[j + 2]; const float* dogN = oc.dog[j + 3];
    const int index = row * w + col, up = index - w, dn = index + w;
    if (fabsf(v) <= s.dogThreshold) return false;
    const float l = __ldg(&dogC[index - 1]), r = __ldg(&dogC[index + 1]);
    float nmax = fmaxf(l, r), nmin = fminf(l, r);
    if (v <= nmax && v >= nmin) return false;
    if (cmp_rows(dogC, up, v, nmax, nmin)) return false;
    if (cmp_rows(dogC, dn, v, nmax, nmin)) return false;
    const float vx2 = v * 2.0f;
    const float fxx = l + r - vx2;
    const float fyy = __ldg(&dogC[up]) + __ldg(&dogC[dn]) - vx2;
    const float fxy = 0.25f * (__ldg(&dogC[dn + 1]) + __ldg(&dogC[up - 1]) - __ldg(&dogC[dn - 1]) - __ldg(&dogC[up + 1]));
    const float t1 = fxx * fyy - fxy * fxy, t2 = (fxx + fyy) * (fxx + fyy);
    if (t1 <= 0.0f || t2 > s.edgeT * t1) return false;
    if (cmp_rows(dogP, up, v, nmax, nmin) || cmp_rows(dogP, index, v, nmax, nmin) || cmp_rows(dogP, dn, v, nmax, nmin)) return false;
    if (cmp_rows(dogN, up, v, nmax, nmin) || cmp_rows(dogN, index, v, nmax, nmin) || cmp_rows(dogN, dn, v, nmax, nmin)) return false;
    return true;
}

__device__ __forceinline__ void row_job(const SdCommon& s, int job, int& L, int& row) {      // block -> (level, image row)
    L = 0;
    while (L + 1 < SD_NLEV && job >= s.rowBase[L + 1]) ++L;
    row = job - s.rowBase[L];
}

// count pass and emit pass share the row walk: 128 threads take the row's columns 128 at a time, in order
template <bool kEmit>
__global__ void __launch_bounds__(128)
sift_key_rows_kernel(const __grid_constant__ SdCommon s, const float* __restrict__ depth) {
    __shared__ int sWarp[4];
    __shared__ int sBase;
    int L, row; row_job(s, (int)blockIdx.x, L, row);
    const int o = L / SD_DOG, j = L % SD_DOG, w = s.oc[o].w;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (t == 0) sBase = kEmit ? s.rowOffset[blockIdx.x] : 0;
    __syncthreads();
    // this thread's pixels: columns t, t + 128, ...  First the two loads every test starts with, for all of them (independent, in flight together);
    // then the tests, which go on to further loads only for the few pixels that pass the threshold
    const float* __restrict__ dogC = s.oc[o].dog[j + 2];
    unsigned hitMask = 0;
    for (int c0 = 0; c0 < w; c0 += 128 * 8) {
        float dv[8], vv[8]; bool ok[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int col = c0 + 128 * k + t;
            int di = 0, ix = 0;
            ok[k] = col < w && key_where(s, o, row, col, di, ix);
            dv[k] = ok[k] ? __ldg(&depth[di]) : 0.0f;
            vv[k] = ok[k] ? __ldg(&dogC[ix]) : 0.0f;
        }
#pragma unroll
        for (int k = 0; k < 8; ++k)
            if (ok[k] && key_test(s, o, j, row, c0 + 128 * k + t, dv[k], vv[k])) hitMask |= 1u << ((c0 >> 7) + k);
    }
    for (int c0 = 0; c0 < w; c0 += 128) {
        const int col = c0 + t;
        const bool hit = (hitMask >> (c0 >> 7)) & 1u;
        const unsigned m = __ballot_sync(0xFFFFFFFFu, hit);
        if (lane == 0) sWarp[warp] = __popc(m);
        __syncthreads();
        int before = 0;
        for (int k = 0; k < warp; ++k) before += sWarp[k];
        const int total = sWarp[0] + sWarp[1] + sWarp[2] + sWarp[3];
        if (kEmit && hit) {
            const int at = sBase + before + __popc(m & ((1u << lane) - 1u));
            if (at < s.fmax[o]) s.raw[s.capBase[L] + at] = make_int2(col, row);
        }
        __syncthreads();
        if (t == 0) sBase += total;
        __syncthreads();
    }
    if (!kEmit && t == 0) s.rowCount[blockIdx.x] = sBase;
}

// one CTA per level: exclusive scan of the row counts, level count = min(total, capacity)
__global__ void __launch_bounds__(512)
sift_key_scan_kernel(const __grid_constant__ SdCommon s) {
    __shared__ int sScan[512];
    const int L = blockIdx.x, o = L / SD_DOG, rows = s.oc[o].h, t = threadIdx.x, base = s.rowBase[L];
    int running = 0;
    for (int r0 = 0; r0 < rows; r0 += 512) {
        const int r = r0 + t;
        const int c = r < rows ? s.rowCount[base + r] : 0;
        sScan[t] = c;
        __syncthreads();
        for (int off = 1; off < 512; off <<= 1) { const int v = t >= off ? sScan[t - off] : 0; __syncthreads(); sScan[t] += v; __syncthreads(); }
        if (r < rows) s.rowOffset[base + r] = running + sScan[t] - c;
        running += sScan[511];
        __syncthreads();
    }
    if (t == 0) s.levelRaw[L] = running < s.fmax[o] ? running : s.fmax[o];
}

// SiftPyramid::LimitFeatureCount (_TruncateMethod 0): drops whole levels from the fine end; returns this level's count afterwards
__device__ int limited_count(const int* levelNum, int threshold, int L) {
    int n[SD_NLEV], total = 0;
    for (int i = 0; i < SD_NLEV; ++i) { n[i] = levelNum[i]; total += n[i]; }
    if (threshold > 0) { int i = 0; while (i < SD_NLEV && total - n[i] > threshold) { total -= n[i]; n[i++] = 0; } }
    return n[L];
}

__device__ __forceinline__ unsigned f2u_gpu(float x) { if (!(x > 0.0f)) return 0u; if (x >= 4294967296.0f) return 0xFFFFFFFFu; return (unsigned)x; }

__device__ __forceinline__ void slot_job(const SdCommon& s, int job, int& L, int& k) {       // block -> (level, list slot)
    L = 0;
    while (L + 1 < SD_NLEV && job >= s.capBase[L + 1]) ++L;
    k = job - s.capBase[L];
}

// ---- ComputeOrientation_Kernel: one CTA of 64 threads per key point ----
__global__ void __launch_bounds__(64)
sift_orient_kernel(const __grid_constant__ SdCommon s) {
    __shared__ float vote[36], tmp[36];
    int L, k; slot_job(s, (int)blockIdx.x, L, k);
    if (k >= limited_count(s.levelRaw, s.P.featureCountThreshold, L)) return;
    const int o = L / SD_DOG, j = L % SD_DOG, w = s.oc[o].w, h = s.oc[o].h, t = threadIdx.x;
    const float2* __restrict__ grad = s.oc[o].grad[j + 1];
    const int2 ik = s.raw[s.capBase[L] + k];
    const float kx = ik.x + 0.5f, ky = ik.y + 0.5f;
    const float sigma = s.levelSigma[j];       // GetLevelSigma, evaluated by the host as in the reference (SiftPyramid.h)
    const float tenDegPerRad = 5.7295779513082320876798154814105f;
    const float gsigma = sigma * 1.5f, win = fabsf(sigma) * 1.5f * 2.0f;
    const float distThreshold = (float)(win * win + 0.5);
    const float factor = -0.5f / (gsigma * gsigma);
    const float xmin = fmaxf(1.5f, floorf(kx - win) + 0.5f), ymin = fmaxf(1.5f, floorf(ky - win) + 0.5f);
    const float xmax = fminf(w - 1.5f, floorf(kx + win) + 0.5f), ymax = fminf(h - 1.5f, floorf(ky + win) + 0.5f);
    if (t < 36) vote[t] = 0.0f;
    __syncthreads();
    const unsigned xlen = f2u_gpu(roundf(xmax - xmin + 1)), ylen = f2u_gpu(roundf(ymax - ymin + 1)), num = xlen * ylen;
    for (unsigned i = t; i < num; i += 64) {
        const float x = (float)(i % xlen) + xmin, y = (float)(i / xlen) + ymin;
        const float dx = x - kx, dy = y - ky;
        const float sq = fmaf(dx, dx, dy * dy);
        if (sq < distThreshold) {
            const float2 g = __ldg(&grad[(int)floorf(y) * w + (int)floorf(x)]);
            const float weight = g.x * expf(sq * factor);
            int oidx = (int)floorf(g.y * tenDegPerRad);
            if (oidx < 0) oidx += 36;
            if (oidx > 35) oidx = 35;                    // atan2f == +pi to the last bit: floor(18.0000002) stays 18, but never leave the array
            atomicAdd(&vote[oidx], weight);
        }
    }
    __syncthreads();
    const float oneThird = (float)(1.0 / 3.0);
    float* src = vote; float* dst = tmp;
    for (int it = 0; it < 6; ++it) {
        if (t < 36) dst[t] = (src[(t + 35) % 36] + src[t] + src[(t + 1) % 36]) * oneThird;
        __syncthreads();
        float* q = src; src = dst; dst = q;
    }                                                    // six passes: the result is back in vote[]
    if (t != 0) return;
    float maxVote = 0.0f;
    for (int b = 0; b < 36; ++b) maxVote = fmaxf(maxVote, vote[b]);
    const float thr = maxVote * 0.8f;
    float maxRot[2] = { 0.0f, 0.0f }; int ocount = 0, maxIndex = -1;
    for (int pass = 0; pass < 2; ++pass) {
        float best = -1.0f; int arg = -1;
        for (int c = 0; c < 36; ++c) {
            if (pass == 1 && c == maxIndex) continue;
            const int m = (c + 35) % 36, p = (c + 1) % 36;
            if (vote[c] > thr && vote[c] > vote[m] && vote[c] > vote[p] && vote[c] > best) { best = vote[c]; arg = c; }
        }
        if (arg < 0) { if (pass == 0) break; else continue; }
        const int m = (arg + 35) % 36, p = (arg + 1) % 36;
        const float di = 0.5f * ((vote[p] - vote[m]) / (2.0f * vote[arg] - vote[p] - vote[m]));
        maxRot[pass] = (float)arg + di + 0.5f;
        ++ocount;
        if (pass == 0) maxIndex = arg;
    }
    float fr1 = maxRot[0] / 36.0f; if (fr1 < 0) fr1 += 1.0f;
    const unsigned us1 = ocount == 0 ? 65535u : (unsigned)(unsigned short)floorf(fr1 * 65535.0f);
    unsigned us2 = 65535u;
    if (ocount > 1) { float fr2 = maxRot[1] / 36.0f; if (fr2 < 0) fr2 += 1.0f; us2 = (unsigned)(unsigned short)floorf(fr2 * 65535.0f); }
    s.oriPack[s.capBase[L] + k] = (us2 << 16) | us1;
}

// ---- ReshapeFeatureList_Kernel, in raster order: one CTA per level ----
__global__ void __launch_bounds__(512)
sift_reshape_kernel(const __grid_constant__ SdCommon s) {
    __shared__ int sScan[512];
    const int L = blockIdx.x, o = L / SD_DOG, j = L % SD_DOG, t = threadIdx.x, cap = s.fmax[o];
    const int n = limited_count(s.levelRaw, s.P.featureCountThreshold, L);
    const float sigma = s.levelSigma[j];       // GetLevelSigma, evaluated by the host as in the reference (SiftPyramid.h)
    const float keyLocScale = (float)(1 << o);
    const float factor = (float)(2.0 * 3.14159265358979323846 / 65535.0);
    const bool scaleOk = sigma * keyLocScale >= s.P.minKeyScale;
    int running = 0;
    for (int k0 = 0; k0 < n; k0 += 512) {
        const int k = k0 + t;
        unsigned o0 = 65535u, o1 = 65535u; int2 ik = make_int2(0, 0);
        if (k < n) { const unsigned pack = s.oriPack[s.capBase[L] + k]; o0 = pack & 0xFFFFu; o1 = pack >> 16; ik = s.raw[s.capBase[L] + k]; }
        int c = 0;
        if (k < n && scaleOk && o0 != 65535u) c = (o1 != 65535u && o1 != o0) ? 2 : 1;
        sScan[t] = c;
        __syncthreads();
        for (int off = 1; off < 512; off <<= 1) { const int v = t >= off ? sScan[t - off] : 0; __syncthreads(); sScan[t] += v; __syncthreads(); }
        const int at = running + sScan[t] - c;
        if (c >= 1 && at < cap) s.fin[s.capBase[L] + at] = make_float4(ik.x + 0.5f, ik.y + 0.5f, sigma, factor * (float)o0);
        if (c == 2 && at < cap && at + 1 < cap) s.fin[s.capBase[L] + at + 1] = make_float4(ik.x + 0.5f, ik.y + 0.5f, sigma, factor * (float)o1);
        running += sScan[511];
        __syncthreads();
    }
    if (t == 0) s.levelFinal[L] = running < cap ? running : cap;
}

// ---- ComputeDescriptor_Kernel + NormalizeDescriptor_Kernel + CreateGlobalKeyPointList + ConvertDescriptorToUChar: one CTA per feature ----
// 16 warps, one per cell of the 4x4 grid: a cell's samples vote only into the cell's own 8 bins, so the cells are independent and run side by side
// (the reference walks them one after the other with 128 threads; the sums are order-free there too: shared-memory atomics).  The first 128 threads
// then normalise and convert.
#define SD_DESC_THREADS 512
__global__ void __launch_bounds__(SD_DESC_THREADS)
sift_describe_kernel(const __grid_constant__ SdCommon s, const float* __restrict__ depth, BFSIFTKeyPoint* keyPoints, uint8_t* descriptors, int* numKeyPoints, int* levelCounts) {
    __shared__ float des[128];
    __shared__ float sRed[4];
    const int t = threadIdx.x;
    // LimitFeatureCount(1) and the output position: levels in order, features in list order
    int n[SD_NLEV], total = 0;
    for (int i = 0; i < SD_NLEV; ++i) { n[i] = s.levelFinal[i]; total += n[i]; }
    if (s.P.featureCountThreshold > 0) { int i = 0; while (i < SD_NLEV && total - n[i] > s.P.featureCountThreshold) { total -= n[i]; n[i++] = 0; } }
    if (blockIdx.x == 0 && t == 0) {
        *numKeyPoints = total < (int)s.P.maxKeyPoints ? total : (int)s.P.maxKeyPoints;
        if (levelCounts) for (int i = 0; i < SD_NLEV; ++i) levelCounts[i] = n[i];
    }
    // the grid walks the output positions: nothing is launched for empty list slots
    const int nOut = total < (int)s.P.maxKeyPoints ? total : (int)s.P.maxKeyPoints;
  for (int out = (int)blockIdx.x; out < nOut; out += (int)gridDim.x) {
    int L = 0, k = out;
    while (k >= n[L]) { k -= n[L]; ++L; }
    const int o = L / SD_DOG, j = L % SD_DOG, w = s.oc[o].w, h = s.oc[o].h;
    const float2* __restrict__ grad = s.oc[o].grad[j + 1];
    const float4 key = s.fin[s.capBase[L] + k];
    if (t < 128) des[t] = 0.0f;
    __syncthreads();
    const float rpi = (float)(4.0 / 3.14159265358979323846);
    const float spt = fabsf(key.z * 3.0f);
    const float sn = sinf(key.w), cs = cosf(key.w);
    const float anglef = (double)key.w > 3.14159265358979323846 ? (float)(key.w - (2.0 * 3.14159265358979323846)) : key.w;
    const float cspt = cs * spt, sspt = sn * spt, crspt = cs / spt, srspt = sn / spt;
    const float bsz = fabsf(cspt) + fabsf(sspt);
    {                                                    // cell b = this warp; its 32 lanes share the cell's window
        const int b = t >> 5, lane = t & 31;
        const int ix = b & 3, iy = b >> 2;
        const float ox = ix - 1.5f, oy = iy - 1.5f;
        const float ptx = cspt * ox - sspt * oy + key.x, pty = cspt * oy + sspt * ox + key.y;
        const float xmin = fmaxf(1.5f, floorf(ptx - bsz) + 0.5f), ymin = fmaxf(1.5f, floorf(pty - bsz) + 0.5f);
        const float xmax = fminf(w - 1.5f, floorf(ptx + bsz) + 0.5f), ymax = fminf(h - 1.5f, floorf(pty + bsz) + 0.5f);
        const unsigned xlen = f2u_gpu(roundf(xmax - xmin + 1)), ylen = f2u_gpu(roundf(ymax - ymin + 1)), size = xlen * ylen;
        for (unsigned i = lane; i < size; i += 32) {
            const float x = (float)(i % xlen) + xmin, y = (float)(i / xlen) + ymin;
            const float dx = x - ptx, dy = y - pty;
            const float nx = crspt * dx + srspt * dy, ny = crspt * dy - srspt * dx;
            const float nxn = fabsf(nx), nyn = fabsf(ny);
            if (nxn < 1.0f && nyn < 1.0f) {
                const float2 g = __ldg(&grad[(int)floorf(y) * w + (int)floorf(x)]);
                const float dnx = nx + ox, dny = ny + oy;
                const float ww = expf(-0.125f * (dnx * dnx + dny * dny));
                const float wx = 1.0f - nxn, wy = 1.0f - nyn;
                const float weight = ww * wx * wy * g.x;
                float theta = (anglef - g.y) * rpi;
                if (theta < 0) theta += 8.0f;
                const float fo = floorf(theta);
                const int fidx = (int)fo & 7;
                atomicAdd(&des[8 * b + fidx], (fo + 1.0f - theta) * weight);
                atomicAdd(&des[8 * b + ((fidx + 1) & 7)], (theta - fo) * weight);
            }
        }
    }
    __syncthreads();
    float v = t < 128 ? des[t] : 0.0f;
    for (int pass = 0; pass < 2; ++pass) {               // normalise, clamp at 0.2, normalise (threads 0..127 carry the 128 bins)
        float sq = v * v;
        for (int off = 16; off > 0; off >>= 1) sq += __shfl_xor_sync(0xFFFFFFFFu, sq, off);
        if (t < 128 && (t & 31) == 0) sRed[t >> 5] = sq;
        __syncthreads();
        const float inv = 1.0f / sqrtf(sRed[0] + sRed[1] + sRed[2] + sRed[3]);
        v = pass == 0 ? fminf(0.2f, v * inv) : v * inv;
        __syncthreads();
    }
    if (t < 128) descriptors[(size_t)out * 128 + t] = (uint8_t)(int)(512 * v + 0.5);
    if (t == 0) {                                        // CreateGlobalKeyPointList_Kernel
        const float keyLocScale = (float)(1 << o);
        const float posX = keyLocScale * (key.x - 0.5f) + 0.5f, posY = keyLocScale * (key.y - 0.5f) + 0.5f;
        const int ixd = (int)roundf(posX * (float)(s.P.depthWidth - 1) / (float)(s.P.width - 1)), iyd = (int)roundf(posY * (float)(s.P.depthHeight - 1) / (float)(s.P.height - 1));
        BFSIFTKeyPoint kp;
        kp.pos[0] = posX; kp.pos[1] = posY; kp.scale = keyLocScale * key.z; kp.depth = __ldg(&depth[(size_t)iyd * s.P.depthWidth + ixd]);
        keyPoints[out] = kp;
    }
    __syncthreads();                                     // des / sRed are reused by the CTA's next feature
  }
}

// ---- host side ----
struct SdWorkspace {
    unsigned width = 0, height = 0;
    void* arena = nullptr; size_t bytes = 0;
    SdCommon c;
    float sigmas[SD_LEVELS]; float taps[SD_LEVELS][SD_MAX_FW]; int fw[SD_LEVELS];
};
static SdWorkspace g_sd;

static void sd_filter_kernel(float sigma, float* kernel, int* width) {            // ProgramCU::CreateFilterKernel, ProgramCU.cu:431-462
    int sz = (int)ceil(4.0f * sigma - 0.5);
    *width = 2 * sz + 1;
    if (*width > SD_MAX_FW) { sz = SD_MAX_FW >> 1; *width = SD_MAX_FW; }
    else if (*width < 5) { sz = 2; *width = 5; }
    float rv = 1.0f / (sigma * sigma), ksum = 0.0f;
    for (int i = -sz; i <= sz; ++i) { const float v = expf(-0.5f * i * i * rv); kernel[i + sz] = v; ksum += v; }
    rv = 1.0f / ksum;
    for (int i = 0; i < *width; ++i) kernel[i] *= rv;
}

static void sd_parse_param(SdWorkspace& ws) {                                      // SiftParam::ParseSiftParam, SiftGPU.cpp:127-174
    const float sigma0 = 1.6f * powf(2.0f, 1.0f / SD_DOG), sigmak = powf(2.0f, 1.0f / SD_DOG);
    const float dsigma0 = sigma0 * sqrtf(1.0f - 1.0f / (sigmak * sigmak));
    const float sa = sigma0 * powf(2.0f, -1.0f / (float)SD_DOG), sb = 0.5f / powf(2.0f, 0.0f);
    ws.sigmas[0] = sa > sb + 0.001 ? sqrtf(sa * sa - sb * sb) : 0.0f;
    for (int i = 0; i <= 4; ++i) ws.sigmas[i + 1] = dsigma0 * powf(sigmak, (float)i);
    for (int i = 0; i < SD_LEVELS; ++i) { for (int k = 0; k < SD_MAX_FW; ++k) ws.taps[i][k] = 0.0f; sd_filter_kernel(ws.sigmas[i], ws.taps[i], &ws.fw[i]); }
    ws.c.sigma0 = sigma0;
    for (int j = 0; j < SD_DOG; ++j) ws.c.levelSigma[j] = sigma0 * powf(2.0f, (float)j / (float)SD_DOG);
    ws.c.dogThreshold = 0.02f / SD_DOG;
    const float edge = 10.0f;
    ws.c.edgeT = (edge + 1) * (edge + 1) / edge;
}

static int sd_ensure(const BFSiftDetectParams* P) {
    SdWorkspace& ws = g_sd;
    if (ws.arena && ws.width == P->width && ws.height == P->height) { ws.c.P = *P; return 0; }
    if (ws.arena) { cudaFree(ws.arena); ws.arena = nullptr; }
    sd_parse_param(ws);
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t at = off; off += (bytes + 255) & ~(size_t)255; return at; };
    size_t gusOff[SD_OCTAVES][SD_LEVELS], dogOff[SD_OCTAVES][SD_LEVELS], gradOff[SD_OCTAVES][SD_LEVELS];
    int w = (int)P->width, h = (int)P->height;
    ws.c.capBase[0] = 0; ws.c.rowBase[0] = 0;
    for (int o = 0; o < SD_OCTAVES; ++o, w >>= 1, h >>= 1) {
        ws.c.oc[o].w = w; ws.c.oc[o].h = h;
        int fm = (int)(w * h * 0.005f);
        fm = fm > SD_MAX_LEVEL_FEATURES ? SD_MAX_LEVEL_FEATURES : (fm < 32 ? 32 : fm);
        ws.c.fmax[o] = fm;
        for (int j = 0; j < SD_DOG; ++j) { const int L = o * SD_DOG + j; ws.c.capBase[L + 1] = ws.c.capBase[L] + fm; ws.c.rowBase[L + 1] = ws.c.rowBase[L] + h; }
        for (int l = 0; l < SD_LEVELS; ++l) {
            gusOff[o][l] = take(sizeof(float) * (size_t)w * h);
            dogOff[o][l] = take(sizeof(float) * (size_t)w * h);
            gradOff[o][l] = take(sizeof(float2) * (size_t)w * h);
        }
    }
    const size_t rowCountOff = take(sizeof(int) * ws.c.rowBase[SD_NLEV]), rowOffsetOff = take(sizeof(int) * ws.c.rowBase[SD_NLEV]);
    const size_t levelRawOff = take(sizeof(int) * SD_NLEV), levelFinalOff = take(sizeof(int) * SD_NLEV);
    const size_t rawOff = take(sizeof(int2) * ws.c.capBase[SD_NLEV]), oriOff = take(sizeof(unsigned) * ws.c.capBase[SD_NLEV]), finOff = take(sizeof(float4) * ws.c.capBase[SD_NLEV]);
    BF_CHECK(cudaMalloc(&ws.arena, off));
    ws.bytes = off;
    char* base = static_cast<char*>(ws.arena);
    for (int o = 0; o < SD_OCTAVES; ++o)
        for (int l = 0; l < SD_LEVELS; ++l) {
            ws.c.oc[o].gus[l] = reinterpret_cast<float*>(base + gusOff[o][l]);
            ws.c.oc[o].dog[l] = reinterpret_cast<float*>(base + dogOff[o][l]);
            ws.c.oc[o].grad[l] = reinterpret_cast<float2*>(base + gradOff[o][l]);
        }
    ws.c.rowCount = reinterpret_cast<int*>(base + rowCountOff); ws.c.rowOffset = reinterpret_cast<int*>(base + rowOffsetOff);
    ws.c.levelRaw = reinterpret_cast<int*>(base + levelRawOff); ws.c.levelFinal = reinterpret_cast<int*>(base + levelFinalOff);
    ws.c.raw = reinterpret_cast<int2*>(base + rawOff); ws.c.oriPack = reinterpret_cast<unsigned*>(base + oriOff); ws.c.fin = reinterpret_cast<float4*>(base + finOff);
    ws.width = P->width; ws.height = P->height;
    ws.c.P = *P;
    return 0;
}

}  // namespace bf

using namespace bf;

BF_API int bfSiftDetect(const BFSiftDetectParams* params, const float* d_intensity, const float* d_depth, BFSIFTKeyPoint* d_keyPoints, uint8_t* d_descriptors,
                        int32_t* d_numKeyPoints, int32_t* d_levelCounts) {
    if (!params || !d_intensity || !d_depth || !d_keyPoints || !d_descriptors || !d_numKeyPoints) return (int)cudaErrorInvalidValue;
    if ((params->width & 31u) || params->width < 64 || params->width > 4096 || params->height < 64 || (params->height & 7u) || params->maxKeyPoints == 0) return (int)cudaErrorInvalidValue;   // width <= 4096: a row's hit flags are one 32-bit mask per thread
    const int rc = sd_ensure(params);
    if (rc) return rc;
    SdWorkspace& ws = g_sd;
    cudaStream_t st = stream();
    static bool attrSet = false;
    const int maxHalf = SD_MAX_FW >> 1, maxIw = SD_TILE + 2 + 2 * maxHalf;
    const size_t maxSmem = sizeof(float) * ((size_t)maxIw * maxIw + (size_t)maxIw * (SD_TILE + 2) + (size_t)(SD_TILE + 2) * (SD_TILE + 2));
    if (!attrSet) { BF_CHECK(cudaFuncSetAttribute(sift_level_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)maxSmem)); attrSet = true; }
    // pyramid: octave 0 level 0 from the input; level l from level l - 1; an octave's level 1 from the previous octave's level 3 (2:1)
    for (int o = 0; o < SD_OCTAVES; ++o) {
        const SdPyr& oc = ws.c.oc[o];
        for (int l = (o == 0 ? 0 : 1); l < SD_LEVELS; ++l) {
            LevelArgs a;
            a.w = oc.w; a.h = oc.h; a.fw = ws.fw[l];
            for (int k = 0; k < SD_MAX_FW; ++k) a.taps[k] = ws.taps[l][k];
            a.gus = oc.gus[l]; a.dog = l >= 1 ? oc.dog[l] : nullptr; a.grad = (l >= 1 && l < 1 + SD_DOG) ? oc.grad[l] : nullptr;
            if (o == 0 && l == 0) { a.src = d_intensity; a.srcW = oc.w; a.srcH = oc.h; a.subsample = 0; }
            else if (l == 1 && o > 0) { a.src = ws.c.oc[o - 1].gus[3]; a.srcW = ws.c.oc[o - 1].w; a.srcH = ws.c.oc[o - 1].h; a.subsample = 1; }
            else { a.src = oc.gus[l - 1]; a.srcW = oc.w; a.srcH = oc.h; a.subsample = 0; }
            const int half = a.fw >> 1, iw = SD_TILE + 2 + 2 * half;
            const size_t smem = sizeof(float) * ((size_t)iw * iw + (size_t)iw * (SD_TILE + 2) + (size_t)(SD_TILE + 2) * (SD_TILE + 2));
            dim3 grid((oc.w + SD_TILE - 1) / SD_TILE, (oc.h + SD_TILE - 1) / SD_TILE);
            ++g_launchCount;
            sift_level_kernel<<<grid, 256, smem, st>>>(a);
        }
    }
    BF_CHECK(cudaGetLastError());
    const int rows = ws.c.rowBase[SD_NLEV], slots = ws.c.capBase[SD_NLEV];
    g_launchCount += 6;
    sift_key_rows_kernel<false><<<rows, 128, 0, st>>>(ws.c, d_depth);
    sift_key_scan_kernel<<<SD_NLEV, 512, 0, st>>>(ws.c);
    sift_key_rows_kernel<true><<<rows, 128, 0, st>>>(ws.c, d_depth);
    sift_orient_kernel<<<slots, 64, 0, st>>>(ws.c);
    sift_reshape_kernel<<<SD_NLEV, 512, 0, st>>>(ws.c);
    const int descGrid = std::min(slots, num_sms() * 4);                 // grid-stride over the features that exist: four 512-thread CTAs per SM
    sift_describe_kernel<<<descGrid, SD_DESC_THREADS, 0, st>>>(ws.c, d_depth, d_keyPoints, d_descriptors, d_numKeyPoints, d_levelCounts);
    BF_CHECK(cudaGetLastError());
    return 0;
}

BF_API size_t bfSiftDetectWorkspaceBytes(void) { return g_sd.bytes; }

BF_API int bfSiftDetectReleaseWorkspace(void) {
    if (g_sd.arena) { BF_CHECK(cudaFree(g_sd.arena)); g_sd.arena = nullptr; g_sd.bytes = 0; g_sd.width = g_sd.height = 0; }
    return 0;
}

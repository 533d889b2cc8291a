// sift_verify.cu -- the two match filters that follow the Kabsch filter, for sm_90a (row a19, second and third filter):
// bfSiftFilterMatchesBySurfaceArea and bfSiftFilterMatchesByDenseVerify of include/bf_sift.h.
//
// Behavioural source (what, not how): FL/SiftGPU/SIFTImageManager.cu:318-407 (FilterMatchesBySurfaceAreaCU) with
// FL/SiftGPU/cuda_surfaceArea.h, FL/SiftGPU/cuda_SVD.h:17-214 (eigenSystem / jacobi), FL/SiftGPU/cuda_EigenValue.h:71-105;
// FL/SiftGPU/SIFTImageManager.cu:413-608 (FilterMatchesByDenseVerifyCU / computeProjError, float-normal branch).
// Device functions follow oracle/filter_oracle.c operation for operation (TU built -fmad=false): the shuffle-down trees, the
// rows-of-the-rotation-matrix "eigenvectors", the NaN behaviour (fminf / fmaxf drop NaNs) and the GPU float->int rule are the reference's; normalize() by
// 1 / sqrtf is this implementation's contract; the dense check's block total is the reference's, quirks included (see below).
//
// Surface area: one warp per image pair, every lane carries the pair's small matrices redundantly (no divergence, no shared memory).
// Dense verify: one CTA per image pair in the reference's block shape (width x ceil(height / 32) threads: 160 for the 80x60 cache) walks both
// cached frames (4800 pixels x 2 directions, ~350 KB of gathers out of L2) -- the work is tiny; ALL pairs of a frame go in one launch.
#include <cfloat>

#include "../../include/bf_sift.h"
#include "bf_common.cuh"
#include "mat4.cuh"
#include "sift_pairs.cuh"

namespace bf {

extern unsigned long long g_launchCount;

#define MAX_FILTERED BF_MAX_MATCHES_PER_IMAGE_PAIR_FILTERED

struct KeyPointV { float px, py, scale, depth; };       // SIFTKeyPoint, FL/SiftGPU/SIFTImageManager.h:22-26
struct v3 { float x, y, z; };

// warpReduce{Sum,Min,Max} (FL/SiftGPU/cudaUtil.h:25-43): lane 0's value, handed to every lane
__device__ __forceinline__ float tree_sum(float v) { for (int off = 16; off > 0; off >>= 1) v = v + __shfl_down_sync(0xFFFFFFFFu, v, off); return __shfl_sync(0xFFFFFFFFu, v, 0); }
__device__ __forceinline__ float tree_min(float v) { for (int off = 16; off > 0; off >>= 1) v = fminf(v, __shfl_down_sync(0xFFFFFFFFu, v, off)); return __shfl_sync(0xFFFFFFFFu, v, 0); }
__device__ __forceinline__ float tree_max(float v) { for (int off = 16; off > 0; off >>= 1) v = fmaxf(v, __shfl_down_sync(0xFFFFFFFFu, v, off)); return __shfl_sync(0xFFFFFFFFu, v, 0); }

#define BF_ROT(m, i, j, k, l) { const float g_ = m[i][j], h_ = m[k][l]; m[i][j] = g_ - s * (h_ + g_ * tau); m[k][l] = h_ + s * (g_ - h_ * tau); }
// cuda_SVD.h:112-214 (Numerical-Recipes jacobi, n = 3), zero-based
__device__ bool jacobi3(float a[3][3], float d[3], float v[3][3]) {
    float b[3], z[3];
    for (int p = 0; p < 3; ++p) { for (int q = 0; q < 3; ++q) v[p][q] = 0.0f; v[p][p] = 1.0f; }
    for (int p = 0; p < 3; ++p) { b[p] = d[p] = a[p][p]; z[p] = 0.0f; }
    for (int sweep = 1; sweep <= 50; ++sweep) {
        float sm = 0.0f;
        for (int p = 0; p < 2; ++p) for (int q = p + 1; q < 3; ++q) sm += fabsf(a[p][q]);
        if (sm == 0.0f) return true;
        const float tresh = sweep < 4 ? 0.2f * sm / 9.0f : 0.0f;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                const float g = 100.0f * fabsf(a[p][q]);
                if (sweep > 4 && fabsf(d[p]) + g == fabsf(d[p]) && fabsf(d[q]) + g == fabsf(d[q])) a[p][q] = 0.0f;
                else if (fabsf(a[p][q]) > tresh) {
                    float h = d[q] - d[p], t;
                    if (fabsf(h) + g == fabsf(h)) t = a[p][q] / h;
                    else {
                        const float theta = 0.5f * h / a[p][q];
                        t = 1.0f / (fabsf(theta) + sqrtf(1.0f + theta * theta));
                        if (theta < 0.0f) t = -t;
                    }
                    const float c = 1.0f / sqrtf(1.0f + t * t), s = t * c, tau = s / (1.0f + c);
                    h = t * a[p][q];
                    z[p] -= h; z[q] += h; d[p] -= h; d[q] += h;
                    a[p][q] = 0.0f;
                    for (int j = 0; j < p; ++j) BF_ROT(a, j, p, j, q)
                    for (int j = p + 1; j < q; ++j) BF_ROT(a, p, j, j, q)
                    for (int j = q + 1; j < 3; ++j) BF_ROT(a, p, j, q, j)
                    for (int j = 0; j < 3; ++j) BF_ROT(v, j, p, j, q)
                }
            }
        for (int p = 0; p < 3; ++p) { b[p] += z[p]; d[p] = b[p]; z[p] = 0.0f; }
    }
    return false;
}

// MYEIGEN::eigenSystem (cuda_SVD.h:17-20, 70-110): ev[i] = ROW i of the rotation matrix, rows exchanged by |eigenvalue|
__device__ bool eigen_system3(const float m[9], v3 ev[3]) {
    float a[3][3], d[3], v[3][3];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) a[i][j] = m[i + 3 * j];
    if (!jacobi3(a, d, v)) return false;
    for (int i = 0; i < 3; ++i) {
        float curMax = 0.0f; int arg = -1;
        for (int j = i; j < 3; ++j) if (fabsf(d[j]) > curMax) { curMax = fabsf(d[j]); arg = j; }
        if (arg != i && arg != -1) {
            float t = d[i]; d[i] = d[arg]; d[arg] = t;
            for (int j = 0; j < 3; ++j) { t = v[i][j]; v[i][j] = v[arg][j]; v[arg][j] = t; }
        }
    }
    for (int i = 0; i < 3; ++i) { ev[i].x = v[i][0]; ev[i].y = v[i][1]; ev[i].z = v[i][2]; }
    return true;
}

__device__ __forceinline__ float dot3(v3 a, v3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

struct AreaArgs {
    PairList pl;
    const KeyPointV* kp; int* numFiltered; const uint2* fIdxs; float* areas;
    float Ki[16]; float areaThresh;
};

// one image of one pair; `lane` < n holds key point `lane`
__device__ float surface_area_one(const AreaArgs& a, const uint2* idx, unsigned n, unsigned which, unsigned lane) {
    const bool on = lane < n;
    v3 pt = { 0.0f, 0.0f, 0.0f };
    if (on) {
        const uint2 ij = idx[lane];
        const KeyPointV k = a.kp[which == 0 ? ij.x : ij.y];
        const float v0 = k.depth * k.px, v1 = k.depth * k.py, v2 = k.depth * 1.0f;
        pt.x = a.Ki[0] * v0 + a.Ki[1] * v1 + a.Ki[2] * v2 + a.Ki[3];
        pt.y = a.Ki[4] * v0 + a.Ki[5] * v1 + a.Ki[6] * v2 + a.Ki[7];
        pt.z = a.Ki[8] * v0 + a.Ki[9] * v1 + a.Ki[10] * v2 + a.Ki[11];
    }
    const float nf = (float)n;
    // computeKeyPointMatchesCovariance, cuda_surfaceArea.h:13-53
    float mean[3], V[9];
    mean[0] = tree_sum(pt.x) / nf; mean[1] = tree_sum(pt.y) / nf; mean[2] = tree_sum(pt.z) / nf;
    const float pc[3] = { pt.x, pt.y, pt.z };
    for (int j = 0; j < 9; ++j) {
        const float e = on ? (pc[j / 3] - mean[j / 3]) * (pc[j % 3] - mean[j % 3]) : 0.0f;
        V[j] = tree_sum(e) / nf;
    }
    v3 ev[3];
    if (!eigen_system3(V, ev)) return 0.0f;                      // uniform across the warp: every lane holds the same V
    // projectKeysToPlane, cuda_surfaceArea.h:138-161
    float px = 0.0f, py = 0.0f;
    if (on) {
        const v3 dm = { pt.x - mean[0], pt.y - mean[1], pt.z - mean[2] };
        const float k = dot3(ev[2], dm);
        const v3 s = { (pt.x - k * ev[2].x) - mean[0], (pt.y - k * ev[2].y) - mean[1], (pt.z - k * ev[2].z) - mean[2] };
        px = dot3(s, ev[0]); py = dot3(s, ev[1]);
    }
    // computeCovariance2d, cuda_surfaceArea.h:59-90
    float m2[2], c2[4];
    m2[0] = tree_sum(on ? px : 0.0f) / nf;
    m2[1] = tree_sum(on ? py : 0.0f) / nf;
    const float q[2] = { px - m2[0], py - m2[1] };
    for (int j = 0; j < 4; ++j) c2[j] = tree_sum(on ? q[j / 2] * q[j % 2] : 0.0f) / nf;
    // computeAreaOrientedBoundingBox2, cuda_surfaceArea.h:93-136; cuda_EigenValue.h:71-105
    const float dd = c2[0] - c2[3];
    const float disc = 0.5f * sqrtf(dd * dd + (4.0f * c2[1]) * c2[1]);
    const float ls[2] = { (c2[0] + c2[3]) / 2.0f + disc, (c2[0] + c2[3]) / 2.0f - disc };
    float ax[2][2];
    for (int k = 0; k < 2; ++k) {
        float vx = -c2[1], vy = c2[0] - ls[k];
        const float mag = sqrtf(vx * vx + vy * vy);
        vx /= mag; vy /= mag;
        const float inv = 1.0f / sqrtf(vx * vx + vy * vy);
        ax[k][0] = vx * inv; ax[k][1] = vy * inv;
    }
    float mnx = FLT_MAX, mny = FLT_MAX, mxx = -FLT_MAX, mxy = -FLT_MAX;
    if (on) { const float cx = ax[0][0] * px + ax[0][1] * py, cy = ax[1][0] * px + ax[1][1] * py; mnx = mxx = cx; mny = mxy = cy; }
    const float ex = tree_max(mxx) - tree_min(mnx), ey = tree_max(mxy) - tree_min(mny);
    if (ex < 0.00001f || ey < 0.00001f) return 0.0f;
    return ex * ey;
}

__global__ void __launch_bounds__(32)
sift_surface_area_kernel(const __grid_constant__ AreaArgs a) {
    const PairRef pr = pair_of(a.pl, blockIdx.x);
    const unsigned p = pr.slot, lane = threadIdx.x;
    if (pr.skip) return;
    const int c = a.numFiltered[p];
    if (c <= 0) return;
    const unsigned n = (unsigned)(c < MAX_FILTERED ? c : MAX_FILTERED);
    const uint2* idx = a.fIdxs + (size_t)p * MAX_FILTERED;
    const float a0 = surface_area_one(a, idx, n, 0, lane), a1 = surface_area_one(a, idx, n, 1, lane);
    __syncwarp();                                                // every lane has read numFiltered[p] before lane 0 overwrites it
    if (lane == 0) {
        if (a.areas) { a.areas[2 * p] = a0; a.areas[2 * p + 1] = a1; }
        if (a0 < a.areaThresh && a1 < a.areaThresh) a.numFiltered[p] = 0;
    }
}

// ---- dense verification ----
__device__ __forceinline__ int f2i_gpu(float x) {              // spelled out so that the rule does not depend on the cvt flavour the compiler picks
    if (x != x) return 0;
    if (x >= 2147483648.0f) return 2147483647;
    if (x <= -2147483648.0f) return (-2147483647 - 1);
    return (int)x;
}

struct VerifyArgs {
    PairList pl; unsigned W, H;
    int* numFiltered; const float* fT; const BFCUDACachedFrame* frames; float* stats;
    float K[16];
    float distThresh, normalThresh, errThresh, corrThresh, dMin, dMax;
};

// computeProjError, SIFTImageManager.cu:413-486
__device__ void proj_error(unsigned idx, const VerifyArgs& a, const float* T, const BFCUDACachedFrame& in, const BFCUDACachedFrame& model, float out[3]) {
    out[0] = out[1] = out[2] = 0.0f;
    const float4 p = __ldg(reinterpret_cast<const float4*>(in.d_cameraposDownsampled) + idx);
    const float4 nI = __ldg(reinterpret_cast<const float4*>(in.d_normalsDownsampled) + idx);
    const float d = __ldg(in.d_depthDownsampled + idx);
    if (!(p.x != -INFINITY && nI.x != -INFINITY && d >= a.dMin && d <= a.dMax)) return;
    float pt[4], nt[4];
    for (int r = 0; r < 4; ++r) {
        pt[r] = T[4 * r] * p.x + T[4 * r + 1] * p.y + T[4 * r + 2] * p.z + T[4 * r + 3] * p.w;
        nt[r] = T[4 * r] * nI.x + T[4 * r + 1] * nI.y + T[4 * r + 2] * nI.z + T[4 * r + 3] * 0.0f;
    }
    const float* K = a.K;
    const float tx = K[0] * pt[0] + K[1] * pt[1] + K[2] * pt[2] + K[3], ty = K[4] * pt[0] + K[5] * pt[1] + K[6] * pt[2] + K[7], tz = K[8] * pt[0] + K[9] * pt[1] + K[10] * pt[2] + K[11];
    const int sx = f2i_gpu(roundf(tx / tz)), sy = f2i_gpu(roundf(ty / tz));
    if (!(sx >= 0 && sy >= 0 && sx < (int)a.W && sy < (int)a.H)) return;
    const size_t m = (size_t)sy * a.W + sx;
    const float4 q = __ldg(reinterpret_cast<const float4*>(model.d_cameraposDownsampled) + m);
    const float4 nT = __ldg(reinterpret_cast<const float4*>(model.d_normalsDownsampled) + m);
    if (!(q.x != -INFINITY && nT.x != -INFINITY)) return;
    const float e0 = pt[0] - q.x, e1 = pt[1] - q.y, e2 = pt[2] - q.z, e3 = pt[3] - q.w;
    const float dist = sqrtf(e0 * e0 + e1 * e1 + e2 * e2 + e3 * e3);
    const float dN = nt[0] * nT.x + nt[1] * nT.y + nt[2] * nT.z;
    const float projDepth = pt[2], tgtDepth = __ldg(model.d_depthDownsampled + m);
    if (!(tgtDepth >= a.dMin && tgtDepth <= a.dMax)) return;
    const bool bad = (tgtDepth != -INFINITY && projDepth < tgtDepth) && dist > a.distThresh;
    if ((dN >= a.normalThresh && dist <= a.distThresh) || bad) {
        const float zN = (pt[2] - a.dMin) / (a.dMax - a.dMin);
        const float w = fmaxf(0.0f, 0.5f * ((1.0f - dist / a.distThresh) + (1.0f - zN)));
        out[0] = dist; out[1] = w; out[2] = 1.0f;
    }
}

// The block total is formed exactly as FilterMatchesByDenseVerifyCU_Kernel forms it (SIFTImageManager.cu:520-565) -- which is not the plain sum of the
// per-pixel terms: (W, ceil(H / 32)) threads, thread (x, ty) adds its rows ty * 32 .. in order, warps cut from the linear thread id,
// `val += __shfl_down(val, offset)` (a lane whose source is past the warp's end adds itself), contributions from the lanes with
// threadIdx.x % 32 == 0.  The reference adds those with shared-memory atomics (scheduling order); here they are added in ascending (row, x) order.
// See oracle/filter_oracle.c dense_block_total and tests/test_manager_reference_emulated.py.
// the reference's block total of one image pair (see above); every thread of the (W, ceil(H / 32)) block calls it, thread 0 gets (err, corr)
__device__ __forceinline__ void dense_pair_total(const VerifyArgs& a, const float* sT, const float* sTinv, const BFCUDACachedFrame& in, const BFCUDACachedFrame& model,
                                                 float (*sAdd)[3], float& err, float& corr) {
    const unsigned x = threadIdx.x, ty = threadIdx.y, t = ty * blockDim.x + x;
    float s[3] = { 0.0f, 0.0f, 0.0f };
    for (unsigned i = 0; i < 32; ++i) {
        const unsigned y = ty * 32 + i;
        if (y < a.H) {
            const unsigned idx = y * a.W + x;
            float u[3], v[3];
            proj_error(idx, a, sT, in, model, u);
            proj_error(idx, a, sTinv, model, in, v);
            for (int k = 0; k < 3; ++k) s[k] += u[k] + v[k];
        }
    }
    for (int k = 0; k < 3; ++k)
        for (int off = 16; off > 0; off >>= 1) s[k] = s[k] + __shfl_down_sync(0xFFFFFFFFu, s[k], off);     // past the warp's end the source is the lane itself
    const unsigned perRow = (blockDim.x + 31) / 32;
    if ((x & 31) == 0) for (int k = 0; k < 3; ++k) sAdd[ty * perRow + (x >> 5)][k] = s[k];
    __syncthreads();
    err = 0.0f; corr = 0.0f;
    if (t == 0) {
        float tot[3] = { 0.0f, 0.0f, 0.0f };
        for (unsigned r = 0; r < blockDim.y; ++r) for (unsigned c = 0; c < perRow; ++c) for (int k = 0; k < 3; ++k) tot[k] += sAdd[r * perRow + c][k];
        err = tot[0] / tot[1]; corr = 0.5f * tot[2] / (float)(a.W * a.H);
    }
}

__global__ void __launch_bounds__(1024)
sift_dense_verify_kernel(const __grid_constant__ VerifyArgs a) {
    const PairRef pr = pair_of(a.pl, blockIdx.x);
    const unsigned p = pr.slot;
    if (pr.skip) return;
    if (a.numFiltered[p] == 0) return;
    __shared__ float sT[16], sTinv[16];
    __shared__ float sAdd[64][3];
    const unsigned t = threadIdx.y * blockDim.x + threadIdx.x;
    if (t < 16) sT[t] = a.fT[16 * (size_t)p + t];
    __syncthreads();
    if (t == 0) mat4_inverse_hd(sT, sTinv);
    __syncthreads();
    float err, corr;
    dense_pair_total(a, sT, sTinv, a.frames[pr.i], a.frames[pr.j], sAdd, err, corr);
    if (t == 0) {
        if (a.stats) { a.stats[2 * p] = err; a.stats[2 * p + 1] = corr; }
        if (corr < a.corrThresh || err > a.errThresh || err != err) a.numFiltered[p] = 0;
    }
}

// VerifyTrajectoryCU_Kernel (SIFTImageManager.cu:1036-1130): block b < N (N - 1) / 2 looks at (b / N, b % N) -- the reference's decode, which
// reaches only the pairs whose row-major index is below N (N - 1) / 2 (SURVEY.md Q7); kept, so that the verdict on a chunk is the reference's.
struct TrajVerifyArgs { VerifyArgs v; unsigned numImages; const int* valid; const float* traj; int* validOpt; };
__global__ void __launch_bounds__(1024)
sift_verify_trajectory_kernel(const __grid_constant__ TrajVerifyArgs a) {
    const unsigned img0 = blockIdx.x / a.numImages, img1 = blockIdx.x % a.numImages;
    if (img0 >= img1) return;
    if (a.valid[img0] == 0 || a.valid[img1] == 0) return;
    __shared__ float sT[16], sTinv[16];
    __shared__ float sAdd[64][3];
    const unsigned t = threadIdx.y * blockDim.x + threadIdx.x;
    if (t == 0) {
        float inv1[16];
        mat4_inverse_hd(a.traj + 16 * (size_t)img1, inv1);
        const float* B = a.traj + 16 * (size_t)img0;
        for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) sT[4 * r + c] = inv1[4 * r] * B[c] + inv1[4 * r + 1] * B[4 + c] + inv1[4 * r + 2] * B[8 + c] + inv1[4 * r + 3] * B[12 + c];
        mat4_inverse_hd(sT, sTinv);
    }
    __syncthreads();
    float err, corr;
    dense_pair_total(a.v, sT, sTinv, a.v.frames[img0], a.v.frames[img1], sAdd, err, corr);
    if (t == 0) {
        if (a.v.stats) { a.v.stats[2 * blockIdx.x] = err; a.v.stats[2 * blockIdx.x + 1] = corr; }
        if (corr < a.v.corrThresh || err > a.v.errThresh || err != err) a.validOpt[0] = 0;
    }
}
__global__ void set_int_kernel(int* p, int v) { *p = v; }

}  // namespace bf

using namespace bf;

BF_API int bfSiftFilterMatchesBySurfaceArea(unsigned int curFrame, unsigned int startFrame, unsigned int numFrames, const BFSIFTKeyPoint* d_keyPoints,
                                            int32_t* d_currNumFilteredMatchesPerImagePair, const uint32_t* d_currFilteredMatchKeyPointIndices,
                                            const float* colorIntrinsicsInv, float areaThresh, float* d_areasOut) {
    if (numFrames == 0 || numFrames <= startFrame) return 0;                        // SIFTImageManager.cu:392
    if (!d_keyPoints || !d_currNumFilteredMatchesPerImagePair || !d_currFilteredMatchKeyPointIndices || !colorIntrinsicsInv) return (int)cudaErrorInvalidValue;
    return sift_surface_area_pairs(frame_pairs(curFrame, startFrame), numFrames - startFrame, d_keyPoints, d_currNumFilteredMatchesPerImagePair,
                                   d_currFilteredMatchKeyPointIndices, colorIntrinsicsInv, areaThresh, d_areasOut);
}

int bf::sift_surface_area_pairs(const PairList& L, unsigned nBlocks, const BFSIFTKeyPoint* d_keyPoints, int32_t* d_currNumFilteredMatchesPerImagePair,
                                const uint32_t* d_currFilteredMatchKeyPointIndices, const float* colorIntrinsicsInv, float areaThresh, float* d_areasOut) {
    if (!nBlocks) return 0;
    AreaArgs a;
    a.pl = L;
    a.kp = reinterpret_cast<const KeyPointV*>(d_keyPoints); a.numFiltered = d_currNumFilteredMatchesPerImagePair;
    a.fIdxs = reinterpret_cast<const uint2*>(d_currFilteredMatchKeyPointIndices); a.areas = d_areasOut;
    for (int k = 0; k < 16; ++k) a.Ki[k] = colorIntrinsicsInv[k];
    a.areaThresh = areaThresh;
    ++g_launchCount;
    sift_surface_area_kernel<<<nBlocks, 32, 0, stream()>>>(a);
    BF_CHECK(cudaGetLastError());
    return 0;
}

BF_API int bfSiftFilterMatchesByDenseVerify(unsigned int curFrame, unsigned int startFrame, unsigned int numFrames, unsigned int imageWidth, unsigned int imageHeight,
                                            const float* intrinsics, int32_t* d_currNumFilteredMatchesPerImagePair, const float* d_currFilteredTransforms,
                                            const BFCUDACachedFrame* d_cachedFrames, float distThresh, float normalThresh, float colorThresh, float errThresh,
                                            float corrThresh, float sensorDepthMin, float sensorDepthMax, float* d_statsOut) {
    (void)colorThresh;                                                              // unused by the reference as well (SIFTImageManager.cu:470)
    if (numFrames == 0 || numFrames <= startFrame) return 0;                        // SIFTImageManager.cu:591
    if (!intrinsics || !d_currNumFilteredMatchesPerImagePair || !d_currFilteredTransforms || !d_cachedFrames || imageWidth == 0 || imageHeight == 0)
        return (int)cudaErrorInvalidValue;
    const unsigned by = (imageHeight + 31) / 32, nt = imageWidth * by;
    if (nt % 32 != 0 || nt > 1024) return (int)cudaErrorInvalidValue;             // the reference's block shape; a partial warp in its shuffles is undefined
    return sift_dense_verify_pairs(frame_pairs(curFrame, startFrame), numFrames - startFrame, imageWidth, imageHeight, intrinsics, d_currNumFilteredMatchesPerImagePair,
                                   d_currFilteredTransforms, d_cachedFrames, distThresh, normalThresh, errThresh, corrThresh, sensorDepthMin, sensorDepthMax, d_statsOut);
}

// block shape checked by the caller
int bf::sift_dense_verify_pairs(const PairList& L, unsigned nBlocks, unsigned imageWidth, unsigned imageHeight, const float* intrinsics,
                                int32_t* d_currNumFilteredMatchesPerImagePair, const float* d_currFilteredTransforms, const BFCUDACachedFrame* d_cachedFrames,
                                float distThresh, float normalThresh, float errThresh, float corrThresh, float sensorDepthMin, float sensorDepthMax, float* d_statsOut) {
    if (!nBlocks) return 0;
    VerifyArgs a;
    a.pl = L; a.W = imageWidth; a.H = imageHeight;
    a.numFiltered = d_currNumFilteredMatchesPerImagePair; a.fT = d_currFilteredTransforms; a.frames = d_cachedFrames; a.stats = d_statsOut;
    for (int k = 0; k < 16; ++k) a.K[k] = intrinsics[k];
    a.distThresh = distThresh; a.normalThresh = normalThresh; a.errThresh = errThresh; a.corrThresh = corrThresh;
    a.dMin = sensorDepthMin; a.dMax = sensorDepthMax;
    ++g_launchCount;
    const dim3 block(imageWidth, (imageHeight + 31) / 32);
    sift_dense_verify_kernel<<<nBlocks, block, 0, stream()>>>(a);
    BF_CHECK(cudaGetLastError());
    return 0;
}

BF_API int bfSiftVerifyTrajectory(unsigned int numImages, const int32_t* d_validImages, const float* d_trajectory, unsigned int imageWidth, unsigned int imageHeight,
                                  const float* intrinsics, const BFCUDACachedFrame* d_cachedFrames, float distThresh, float normalThresh, float colorThresh,
                                  float errThresh, float corrThresh, float sensorDepthMin, float sensorDepthMax, int32_t* d_validOpt, float* d_statsOut) {
    (void)colorThresh;
    if (!d_validOpt) return (int)cudaErrorInvalidValue;
    if (numImages < 2) { set_int_kernel<<<1, 1, 0, stream()>>>(d_validOpt, 0); BF_CHECK(cudaGetLastError()); return 0; }      // SIFTImageManager.cu:1138: returns 0
    if (!d_validImages || !d_trajectory || !intrinsics || !d_cachedFrames || imageWidth == 0 || imageHeight == 0) return (int)cudaErrorInvalidValue;
    TrajVerifyArgs a;
    a.v.pl = frame_pairs(0, 0); a.v.W = imageWidth; a.v.H = imageHeight;
    a.v.numFiltered = nullptr; a.v.fT = nullptr; a.v.frames = d_cachedFrames; a.v.stats = d_statsOut;
    for (int k = 0; k < 16; ++k) a.v.K[k] = intrinsics[k];
    a.v.distThresh = distThresh; a.v.normalThresh = normalThresh; a.v.errThresh = errThresh; a.v.corrThresh = corrThresh;
    a.v.dMin = sensorDepthMin; a.v.dMax = sensorDepthMax;
    a.numImages = numImages; a.valid = d_validImages; a.traj = d_trajectory; a.validOpt = d_validOpt;
    const unsigned by = (imageHeight + 31) / 32, nt = imageWidth * by;
    if (nt % 32 != 0 || nt > 1024) return (int)cudaErrorInvalidValue;
    g_launchCount += 2;
    set_int_kernel<<<1, 1, 0, stream()>>>(d_validOpt, 1);
    const dim3 block(imageWidth, by);
    sift_verify_trajectory_kernel<<<numImages * (numImages - 1) / 2, block, 0, stream()>>>(a);
    BF_CHECK(cudaGetLastError());
    return 0;
}

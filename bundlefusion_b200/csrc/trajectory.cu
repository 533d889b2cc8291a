// trajectory.cu -- trajectory glue for sm_90a.  Implements include/bf_bundler.h (row a22 of SURVEY.md section 8).
// Behavioural source (what, not how): FL/OnlineBundler.cu:6-140.  Tiny kernels; what matters is that they exist behind the
// reference's stub names, run on the library stream without a host synchronisation, and agree bit for bit with
// oracle/trajectory_oracle.c (this TU is built -fmad=false; products are fused only as mat4.cuh writes them).
#include "../../include/bf_bundler.h"
#include "bf_common.cuh"
#include "mat4.cuh"
#include "se3.cuh"

namespace bf {

extern unsigned long long g_launchCount;

// getSiftTransformCU_Kernel (OnlineBundler.cu:6-53): one thread, the loop walks back to the most recent matched frame of the chunk
__global__ void sift_transform_kernel(unsigned curFrameIndex, const float* __restrict__ complete, unsigned lastValidComplete, float* siftTraj,
                                      unsigned curFrameIndexAll, const int* __restrict__ numFiltered, const float* __restrict__ filteredInv, float* currIntegrate) {
    for (int i = (int)curFrameIndex - 1; i >= 0; --i) {
        if (numFiltered[i] <= 0) continue;
        const unsigned prev = curFrameIndexAll - (curFrameIndex - (unsigned)i);
        float T[16], R[16];
        mat4_mul_hd(&siftTraj[16 * prev], &filteredInv[16 * i], T);
        for (int k = 0; k < 16; ++k) siftTraj[16 * curFrameIndexAll + k] = T[k];
        if (lastValidComplete == 0) {
            for (int k = 0; k < 16; ++k) R[k] = T[k];
        } else if (prev < lastValidComplete) {
            mat4_mul_hd(&complete[16 * prev], &filteredInv[16 * i], R);
        } else {
            float inv[16], off[16], t2[16];
            mat4_inverse_hd(&siftTraj[16 * lastValidComplete], inv);
            mat4_mul_hd(inv, &siftTraj[16 * prev], off);
            mat4_mul_hd(&complete[16 * lastValidComplete], off, t2);
            mat4_mul_hd(t2, &filteredInv[16 * i], R);
        }
        for (int k = 0; k < 16; ++k) currIntegrate[k] = R[k];
        break;
    }
}

// updateTrajectoryCU_Kernel (OnlineBundler.cu:71-90)
__global__ void update_trajectory_kernel(const float* __restrict__ global, float* complete, unsigned numComplete, const float* __restrict__ local,
                                         unsigned perTraj, const int* __restrict__ invalidate) {
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= numComplete) return;
    const unsigned submap = perTraj - 1, g = idx / submap, l = idx % submap;
    float R[16];
    if (invalidate[idx] == 0) { for (int k = 0; k < 16; ++k) R[k] = -INFINITY; }
    else mat4_mul_hd(&global[16 * g], &local[16 * (g * perTraj + l)], R);
    for (int k = 0; k < 16; ++k) complete[16 * idx + k] = R[k];
}

// initNextGlobalTransformCU_Kernel (OnlineBundler.cu:114-126)
__global__ void init_next_global_kernel(float* global, unsigned numGlobal, unsigned initIdx, const float* __restrict__ local, unsigned lastValidLocal, unsigned perTraj) {
    const float* L = &local[16 * (size_t)(numGlobal * perTraj - (perTraj - lastValidLocal))];
    float R[16];
    mat4_mul_hd(&global[16 * initIdx], L, R);
    for (int k = 0; k < 16; ++k) global[16 * numGlobal + k] = R[k];
}

// dist of TrajectoryManager::generateUpdateLists (TrajectoryManager.cpp:56-75) for every frame, then an iterative arg-max: topN <= a few
// dozen rounds over <= 20 000 frames in ONE CTA -- no trajectory copy to the host, no host sort.
__global__ void __launch_bounds__(1024)
select_reintegration_kernel(const float* __restrict__ opt, const float* __restrict__ integ, const int* __restrict__ state, unsigned n, unsigned topN,
                            float minDist, float scale, float* dist, int* list, int* count) {
    __shared__ float sVal[32];
    __shared__ int sIdx[32];
    __shared__ int sPick;
    __shared__ unsigned sTaken[2048];                                 // one bit per frame (numFrames <= 65 536, checked by the host)
    const unsigned t = threadIdx.x;
    for (unsigned i = t; i < 2048; i += blockDim.x) sTaken[i] = 0u;
    for (unsigned i = t; i < n; i += blockDim.x) {
        float d = -1.0f;                                              // not a candidate
        if (state[i] != 0 && opt[16 * i] != -INFINITY) {
            V3 ro, to, ri, ti;
            matrix_to_pose(&opt[16 * i], ro, to);
            matrix_to_pose(&integ[16 * i], ri, ti);
            // PoseHelper::MatrixToPose packs (translation, rotation) and TrajectoryManager scales components 0..2 (FL/PoseHelper.h:355-358,
            // FL/TrajectoryManager.cpp:66-75): the factor its name gives to the rotation lands on the Lie TRANSLATION
            const V3 dt = ti * scale - to * scale, dr = ri - ro;
            d = dot(dt, dt) + dot(dr, dr);
        }
        dist[i] = d;
    }
    __syncthreads();
    unsigned found = 0;
    for (; found < topN; ++found) {
        float best = -1.0f; int bi = 0x7fffffff;
        for (unsigned i = t; i < n; i += blockDim.x) {
            const float d = dist[i];
            if (d > minDist && d >= 0.0f && !((sTaken[i >> 5] >> (i & 31)) & 1u) && (d > best || (d == best && (int)i < bi))) { best = d; bi = (int)i; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
        }
        if ((t & 31) == 0) { sVal[t >> 5] = best; sIdx[t >> 5] = bi; }
        __syncthreads();
        if (t == 0) {
            float b = -1.0f; int k = 0x7fffffff;
            for (unsigned w = 0; w < blockDim.x / 32; ++w) if (sVal[w] > b || (sVal[w] == b && sIdx[w] < k)) { b = sVal[w]; k = sIdx[w]; }
            sPick = (b >= 0.0f && k != 0x7fffffff) ? k : -1;
            if (sPick >= 0) { list[found] = sPick; sTaken[sPick >> 5] |= 1u << (sPick & 31); }
        }
        __syncthreads();
        if (sPick < 0) break;
    }
    if (t == 0) *count = (int)found;
}

}  // namespace bf

using namespace bf;

BF_API int bfTrajectorySelectReintegration(const float* d_opt, const float* d_integ, const int* d_state, unsigned int numFrames, unsigned int topN,
                                           float minPoseDistSqrt, float rescaleRotToTrans, float* d_dist, int* d_list, int* d_count) {
    if (!d_opt || !d_integ || !d_state || !d_dist || !d_list || !d_count || numFrames > 65536u) return (int)cudaErrorInvalidValue;
    ++g_launchCount;
    select_reintegration_kernel<<<1, 1024, 0, stream()>>>(d_opt, d_integ, d_state, numFrames, topN, minPoseDistSqrt, rescaleRotToTrans, d_dist, d_list, d_count);
    BF_CHECK(cudaGetLastError());
    return 0;
}

BF_API void computeSiftTransformCU(const float* d_currFilteredTransformsInv, const int* d_currNumFilteredMatchesPerImagePair, const float* d_completeTrajectory,
                                   unsigned int lastValidCompleteTransform, float* d_siftTrajectory, unsigned int curFrameIndexAll, unsigned int curFrameIndex,
                                   float* d_currIntegrateTrans) {
    if (curFrameIndex == 0) return;                                              // OnlineBundler.cu:59
    ++g_launchCount;
    sift_transform_kernel<<<1, 1, 0, stream()>>>(curFrameIndex, d_completeTrajectory, lastValidCompleteTransform, d_siftTrajectory, curFrameIndexAll,
                                                 d_currNumFilteredMatchesPerImagePair, d_currFilteredTransformsInv, d_currIntegrateTrans);
    BF_SAFE((int)cudaGetLastError());
}
BF_API void updateTrajectoryCU(const float* d_globalTrajectory, unsigned int numGlobalTransforms, float* d_completeTrajectory, unsigned int numCompleteTransforms,
                               const float* d_localTrajectories, unsigned int numLocalTransformsPerTrajectory, unsigned int numLocalTrajectories, int* d_imageInvalidateList) {
    (void)numGlobalTransforms; (void)numLocalTrajectories;
    if (numCompleteTransforms == 0) return;
    ++g_launchCount;
    update_trajectory_kernel<<<(numCompleteTransforms + 127) / 128, 128, 0, stream()>>>(d_globalTrajectory, d_completeTrajectory, numCompleteTransforms, d_localTrajectories,
                                                                                        numLocalTransformsPerTrajectory, d_imageInvalidateList);
    BF_SAFE((int)cudaGetLastError());
}
BF_API void initNextGlobalTransformCU(float* d_globalTrajectory, unsigned int numGlobalTransforms, unsigned int initGlobalIdx, float* d_localTrajectories,
                                      unsigned int lastValidLocal, unsigned int numLocalTransformsPerTrajectory) {
    ++g_launchCount;
    init_next_global_kernel<<<1, 1, 0, stream()>>>(d_globalTrajectory, numGlobalTransforms, initGlobalIdx, d_localTrajectories, lastValidLocal, numLocalTransformsPerTrajectory);
    BF_SAFE((int)cudaGetLastError());
}

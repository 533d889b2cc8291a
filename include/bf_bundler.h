/*
 * bf_bundler.h -- C-ABI of the trajectory glue between bundling and reconstruction (SURVEY.md section 8, row a22).
 *
 * Re-exports, by NAME and machine-level signature, the `extern "C"` stubs FL/OnlineBundler.cpp:18-27 declares and FL/OnlineBundler.cu
 * defines (float4x4 = 16 row-major floats; C++ references are pointers at the ABI level):
 *   computeSiftTransformCU     FL/OnlineBundler.cu:6-69     pose used to integrate the CURRENT frame: last known pose chained with the
 *                                                            Kabsch transform of the most recent earlier frame of the chunk it matched
 *   updateTrajectoryCU         FL/OnlineBundler.cu:71-110   complete[k] = global[k / submap] * local[k / submap][k % submap], or -inf if invalid
 *   initNextGlobalTransformCU  FL/OnlineBundler.cu:114-140  next keyframe's initial global pose
 * (FL/ = /root/reference/FriedLiver/Source/.)  All three launch asynchronously on the library stream (bfSetStream).
 */
#ifndef BF_BUNDLER_H
#define BF_BUNDLER_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

void computeSiftTransformCU(const float* d_currFilteredTransformsInv, const int* d_currNumFilteredMatchesPerImagePair,
                            const float* d_completeTrajectory, unsigned int lastValidCompleteTransform,
                            float* d_siftTrajectory, unsigned int curFrameIndexAll, unsigned int curFrameIndex, float* d_currIntegrateTrans);
void initNextGlobalTransformCU(float* d_globalTrajectory, unsigned int numGlobalTransforms, unsigned int initGlobalIdx,
                               float* d_localTrajectories, unsigned int lastValidLocal, unsigned int numLocalTransformsPerTrajectory);
void updateTrajectoryCU(const float* d_globalTrajectory, unsigned int numGlobalTransforms, float* d_completeTrajectory, unsigned int numCompleteTransforms,
                        const float* d_localTrajectories, unsigned int numLocalTransformsPerTrajectory, unsigned int numLocalTrajectories,
                        int* d_imageInvalidateList);

/* ---- H100-native extension: the re-integration choice of TrajectoryManager::generateUpdateLists (FL/TrajectoryManager.cpp:45-108) on
 * the device.  The reference copies the whole optimised trajectory to the host every frame, converts every pose with MatrixToPose, and
 * std::sorts all frames to take the top N.  Here one launch computes, per frame, dist = |(s t, w)_integrated - (s t, w)_optimised|^2
 * ((w, t) = the SE(3) logarithm, s = rescaleRotToTrans = 2: despite its name the factor multiplies the TRANSLATION part -- the host's
 * PoseHelper::MatrixToPose packs (translation, rotation) and TrajectoryManager.cpp:67-74 scales components 0..2) and selects the up to topN INTEGRATED frames of largest dist > minPoseDistSqrt, in
 * descending order (ties: lower frame index first; the reference's std::sort leaves ties unspecified).  A frame whose optimised transform
 * is invalid (first entry -inf) is never selected (the reference routes it to the de-integration list).
 * d_frameState[i] != 0 <=> frame i is currently integrated.  Outputs: d_dist[numFrames], d_list[topN] (frame indices), d_count[1].
 * Asynchronous on the library stream; returns 0 or a cudaError_t. */
int bfTrajectorySelectReintegration(const float* d_optimizedTransforms, const float* d_integratedTransforms, const int* d_frameState,
                                    unsigned int numFrames, unsigned int topN, float minPoseDistSqrt, float rescaleRotToTrans,
                                    float* d_dist, int* d_list, int* d_count);

/* ---- TrajectoryManager (FL/TrajectoryManager.{h,cpp}): the host-side state machine that decides which frames are integrated,
 * de-integrated and re-integrated.  Host C++ in the reference and host C++ here (no device work), behind an opaque handle; method for method:
 *   TrajectoryManager(numMaxImage)                      -> bfTrajectoryCreate   (s_topNActive, s_minPoseDistSqrt passed explicitly)
 *   addFrame / updateOptimizedTransform / generateUpdateLists / confirmIntegration / getTopFrom{ReIntegrate,Integrate,DeIntegrate}List /
 *   getNumOptimizedFrames / getNumAddedFrames / getNumActiveOperations / getOptimizedTransforms
 * Differences: updateOptimizedTransform takes a HOST array (the reference cudaMemcpy's from the device itself -- the caller does that, or
 * keeps the trajectory on the device and uses bfTrajectorySelectReintegration); the sort is std::stable_sort (the reference's std::sort
 * leaves the order of equal distances unspecified) and orders NaN distances (a frame integrated with an invalid pose) last, which keeps
 * the comparator a strict weak order.  Kept as in the reference: the refill loop of generateUpdateLists starts at
 * sorted[len(re-integration list)] (cpp:97), so while k frames are still queued the k largest movers are skipped.
 * Frame types: FL/TrajectoryManager.h:8-14. */
enum { BF_TRAJ_INTEGRATED = 0, BF_TRAJ_NOT_INTEGRATED_NO_TRANSFORM = 1, BF_TRAJ_NOT_INTEGRATED_WITH_TRANSFORM = 2, BF_TRAJ_INVALID = 3, BF_TRAJ_REINTEGRATION = 4 };
typedef struct BFTrajectoryManager BFTrajectoryManager;
BFTrajectoryManager* bfTrajectoryCreate(unsigned int numMaxImage, unsigned int topNActive, float minPoseDistSqrt);
void bfTrajectoryDestroy(BFTrajectoryManager* tm);
void bfTrajectoryAddFrame(BFTrajectoryManager* tm, int type, const float* transform, unsigned int idx);
void bfTrajectoryUpdateOptimizedTransform(BFTrajectoryManager* tm, const float* h_trajectory, unsigned int numFrames);
void bfTrajectoryGenerateUpdateLists(BFTrajectoryManager* tm);
void bfTrajectoryConfirmIntegration(BFTrajectoryManager* tm, unsigned int frameIdx);
int  bfTrajectoryGetTopFromReIntegrateList(BFTrajectoryManager* tm, float* oldTransform, float* newTransform, unsigned int* frameIdx);
int  bfTrajectoryGetTopFromIntegrateList(BFTrajectoryManager* tm, float* transform, unsigned int* frameIdx);
int  bfTrajectoryGetTopFromDeIntegrateList(BFTrajectoryManager* tm, float* transform, unsigned int* frameIdx);
unsigned int bfTrajectoryGetNumOptimizedFrames(const BFTrajectoryManager* tm);
unsigned int bfTrajectoryGetNumAddedFrames(const BFTrajectoryManager* tm);
unsigned int bfTrajectoryGetNumActiveOperations(const BFTrajectoryManager* tm);
int  bfTrajectoryGetFrameType(const BFTrajectoryManager* tm, unsigned int frameIdx);
float bfTrajectoryGetFrameDist(const BFTrajectoryManager* tm, unsigned int frameIdx);
/* getOptimizedTransforms: writes min(added, optimized) 4x4s (invalid frames: all -inf); returns that count */
unsigned int bfTrajectoryGetOptimizedTransforms(BFTrajectoryManager* tm, float* h_out);

#ifdef __cplusplus
}
#endif
#endif /* BF_BUNDLER_H */

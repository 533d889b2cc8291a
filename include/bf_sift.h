/*
 * bf_sift.h -- C-ABI of the SIFT descriptor matcher (SURVEY.md section 8, row a18).
 *
 * The reference exposes this path as a C++ class, not as extern "C" stubs:
 *   SiftMatchGPU::SetDescriptors(int index, int num, unsigned char* d_descriptors)     FL/SiftGPU/SiftMatch.cpp:110-131
 *   SiftMatchGPU::GetSiftMatch(int max_match, ImagePairMatch&, uint2 keyPointOffset,
 *                              float distmax, float ratiomax, int mutual_best_match)   FL/SiftGPU/SiftMatch.cpp:160-196
 *   -> ProgramCU::MultiplyDescriptor / GetRowMatch / GetColMatch                        FL/SiftGPU/ProgramCU.cu:1734-1938
 * and calls it once per image pair from Bundler::matchAndFilter (FL/Bundler.cpp:116-137): 2 descriptor copies + 3 launches + a
 * memset per pair, serialised.  (FL/ = /root/reference/FriedLiver/Source/.)
 *
 * This header is the boundary a maintainer binds instead: plain pointers and sizes, one call for ALL pairs of a frame.
 * Descriptors are 128 unsigned bytes per feature, normalised to length 512 (SiftGPU convention), feature-major.
 * Semantics per pair are exactly GetSiftMatch with mutual_best_match = 1 (the only mode the reference's GetBestMatch implements):
 * mutual best matches with dist = acos(dot / 2^18) < distmax and dist < ratiomax * dist_second, including which feature wins a tie;
 * the ORDER in which matches are appended is race-dependent in the reference (atomicAdd) and here -- consumers sort by
 * distance next (SIFTImageManager::SortKeyPointMatchesCU).  Dot products are exact int32.
 * Threading: like the reference's SiftGPU / SIFTImageManager (module-level __constant__ blocks and texture references, FL/Bundler.cpp's
 * mutex_siftMatcher), the entry points of this header share per-process workspaces and one stream (bfSetStream) and are not re-entrant;
 * call them from one thread per process (one process per GPU).
 */
#ifndef BF_SIFT_H
#define BF_SIFT_H

#include <stddef.h>
#include <stdint.h>

#include "bf_solver.h"      /* BFEntryJ */

#ifdef __cplusplus
extern "C" {
#endif

#define BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW 128     /* FL/GlobalDefines.h:8 */
#define BF_MAX_MATCHES_PER_IMAGE_PAIR_FILTERED 25 /* FL/GlobalDefines.h:9 */

/* FL/SiftGPU/SIFTImageManager.h:22-26 */
typedef struct BFSIFTKeyPoint { float pos[2]; float scale; float depth; } BFSIFTKeyPoint;

/* FL/SiftGPU/SIFTImageManager.h:38-42 */
typedef struct BFImagePairMatch {
    int32_t*  d_numMatches;        /* one counter (keeps counting past the cap, as the reference's) */
    float*    d_distances;         /* [BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW] */
    uint32_t* d_keyPointIndices;   /* uint2 [BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW]: (feature of image 1 + offset.x, feature of image 2 + offset.y) */
} BFImagePairMatch;

/* one image pair: what SetDescriptors(0, ..) + SetDescriptors(1, ..) + GetSiftMatch(..) take */
typedef struct BFSiftMatchJob {
    const uint8_t* d_des1; int32_t num1;        /* image 1 ("prev" in Bundler::matchAndFilter) */
    const uint8_t* d_des2; int32_t num2;        /* image 2 (the current frame) */
    BFImagePairMatch out;
    uint32_t keyPointOffset[2];
} BFSiftMatchJob;

/* Matches numJobs image pairs (jobs: HOST array) in two launches, asynchronously on the library stream (bfSetStream).
 * Matches are stored in ascending image-2 feature; when a pair has more than 128 the first 128 in that order are kept and the counter holds the
 * total (the reference appends with an atomicAdd: which 128 survive there depends on the scheduling -- this is one of its outcomes, always the same).
 * A job with num1 <= 0 or num2 <= 0 only zeroes its counter (SiftMatch.cpp:162-165); its descriptor pointers are not read and may be NULL.
 * Alignment contract: d_des1 and d_des2 of every other job must be 16-byte aligned (cudaMalloc'd arrays of 128-byte rows are; a uint8 view that
 * starts at an odd byte is not) -- the reference copies descriptors into its own buffers, this call reads the caller's in 16-byte units.  A batch
 * that breaks it, or has num1 or num2 >= 2^24, returns cudaErrorInvalidValue before any CUDA call: nothing is enqueued, no counter is touched.
 * Returns 0 or a cudaError_t. */
int bfSiftMatchBatch(const BFSiftMatchJob* jobs, int numJobs, float distmax, float ratiomax);

/* Sweep of bfSiftMatchBatch, process-wide.  AUTO (the default; BF_SIFT_MATCH=mma in the environment makes MMA the initial setting): the wgmma +
 * TMA sweep, or the warp-level mma.sync sweep when the driver offers no tensor-map encoder.  WGMMA forces the first: a batch it cannot map
 * returns cudaErrorNotSupported before anything is enqueued, it never falls back.  MMA forces the second.  Both give the same bytes (counter,
 * stored indices in storage order, distances); forcing one lets a test compare them.  Returns the previous setting, or cudaErrorInvalidValue
 * for an unknown one. */
#define BF_SIFT_SWEEP_AUTO 0
#define BF_SIFT_SWEEP_WGMMA 1
#define BF_SIFT_SWEEP_MMA 2
int bfSiftSetMatchSweep(int sweep);
/* The last bfSiftMatchBatch that enqueued work, recorded on the host (does not synchronise): out[0] = the sweep that ran (BF_SIFT_SWEEP_WGMMA or
 * BF_SIFT_SWEEP_MMA; 0 before the first batch), out[1] = its number of jobs. */
int bfSiftGetMatchInfo(int out[2]);

/* SIFTImageManager::SortKeyPointMatchesCU(curFrame, startFrame, numFrames) (FL/SiftGPU/SIFTImageManager.cu:59-177): sorts the raw matches
 * of every image pair p in [startFrame, numFrames), p != curFrame, by ascending distance, in place.  Arrays are the manager's:
 * d_numMatchesPerImagePair[p], d_matchDistances[p * 128 + k], d_matchKeyPointIndices (uint2) [p * 128 + k].
 * The reference's odd-even transposition sort is stable with respect to a race-dependent append order; here equal distances are
 * ordered by (image-2 feature, image-1 feature), so the result does not depend on the append order.  Asynchronous. */
int bfSiftSortKeyPointMatches(unsigned int curFrame, unsigned int startFrame, unsigned int numFrames, const int32_t* d_numMatchesPerImagePair,
                              float* d_matchDistances, uint32_t* d_matchKeyPointIndices);

/* SIFTImageManager::FilterKeyPointMatchesCU(curFrame, startFrame, numFrames, siftIntrinsicsInv, minNumMatches, maxKabschRes2)
 * (FL/SiftGPU/SIFTImageManager.cu:186-316; filterKeyPointMatches FL/SiftGPU/cuda_kabsch.h:417-502): for every image pair p in
 * [startFrame, numFrames), p != curFrame, walks the distance-sorted raw matches, greedily grows a geometrically consistent subset
 * (<= 25 matches: Kabsch re-fit after every insertion, 5-pixel proximity rule, worst residuals dropped until max residual^2 <
 * maxKabschRes2, three condition numbers <= 100) and writes the filtered matches (ascending residual), their count, the rigid transform
 * image p -> current image and its inverse.  Arrays are the manager's (raw: [p * 128 + k], filtered: [p * 25 + k], transforms [p][16]);
 * key-point indices are global indices into d_keyPoints; siftIntrinsicsInv is a HOST 4x4.  The 3x3 SVD inside the Kabsch fit is the
 * reference's own (the fast approximate SVD of FL/SiftGPU/cuda_svd3.h, reflection fixed on the third column), operation for operation,
 * with rsqrt taken as 1 / sqrtf (the reference's device build: CUDA's rsqrtf).  Asynchronous. */
int bfSiftFilterKeyPointMatches(unsigned int curFrame, unsigned int startFrame, unsigned int numFrames, const BFSIFTKeyPoint* d_keyPoints,
                                const int32_t* d_numMatchesPerImagePair, const float* d_matchDistances, const uint32_t* d_matchKeyPointIndices,
                                int32_t* d_numFilteredMatchesPerImagePair, float* d_filteredMatchDistances, uint32_t* d_filteredMatchKeyPointIndices,
                                float* d_filteredTransforms, float* d_filteredTransformsInv, const float* siftIntrinsicsInv,
                                unsigned int minNumMatches, float maxKabschRes2);

/* SIFTImageManager::FilterMatchesBySurfaceAreaCU(curFrame, startFrame, numFrames, colorIntrinsicsInv, areaThresh)
 * (FL/SiftGPU/SIFTImageManager.cu:318-407; FL/SiftGPU/cuda_surfaceArea.h): for every pair p in [startFrame, numFrames), p != curFrame, with
 * filtered matches, projects the matched key points of each image into the plane spanned by the first two vectors of the frame
 * MYEIGEN::eigenSystem returns for their covariance (FL/SiftGPU/cuda_SVD.h:70-110 -- rows of the Jacobi rotation matrix, kept as is),
 * measures the area of the 2-D oriented bounding box there, and sets d_currNumFilteredMatchesPerImagePair[p] = 0 when BOTH areas are
 * below areaThresh (an exactly axis-aligned 2-D covariance yields a 0/0 axis and, through the min / max reductions, area 0 -- as in
 * the reference).
 * colorIntrinsicsInv: HOST 4x4.  d_areasOut: optional [numFrames][2] (area in image p, area in the current image), else NULL.
 * Difference: normalize() multiplies by 1 / sqrtf where the reference multiplies by rsqrtf.  Asynchronous. */
int bfSiftFilterMatchesBySurfaceArea(unsigned int curFrame, unsigned int startFrame, unsigned int numFrames, const BFSIFTKeyPoint* d_keyPoints,
                                     int32_t* d_currNumFilteredMatchesPerImagePair, const uint32_t* d_currFilteredMatchKeyPointIndices,
                                     const float* colorIntrinsicsInv, float areaThresh, float* d_areasOut);

/* SIFTImageManager::FilterMatchesByDenseVerifyCU(curFrame, startFrame, numFrames, imageWidth, imageHeight, intrinsics, d_cachedFrames,
 * distThresh, normalThresh, colorThresh, errThresh, corrThresh, sensorDepthMin, sensorDepthMax) (FL/SiftGPU/SIFTImageManager.cu:413-608):
 * for every pair p with filtered matches, warps cached frame p into the current one with d_currFilteredTransforms[p] and back with its
 * inverse (projective association at the cache resolution, float normals), accumulates residual / weight / count over the pixels
 * whose position and normal agree or that are known to be in front of the target surface, and zeroes the pair's filtered-match count
 * when corr = count / (2 W H) < corrThresh, err = residual / weight > errThresh, or err is NaN.  intrinsics: HOST 4x4 (cache
 * resolution).  colorThresh is accepted and unused, as in the reference.  d_statsOut: optional [numFrames][2] (err, corr), else NULL.
 * The block total is formed as the reference's kernel forms it (SIFTImageManager.cu:520-565), which is NOT the plain sum over the pixels:
 * (width, ceil(height / 32)) threads, `val += __shfl_down(val, offset)` over warps cut from the linear thread id (a lane whose source is past
 * the warp's end adds itself), contributions from the lanes with threadIdx.x % 32 == 0 -- for the 80 x 60 cache some pixels count twice or more
 * and some not at all, and err / corr come out a few percent off the plain ones.  Kept for identical decisions
 * (tests/test_manager_reference_emulated.py); the only difference left is that those contributions are added in a fixed order instead of
 * through shared-memory atomics.  width * ceil(height / 32) must be a multiple of 32 and at most 1024 (else cudaErrorInvalidValue).  Asynchronous. */
int bfSiftFilterMatchesByDenseVerify(unsigned int curFrame, unsigned int startFrame, unsigned int numFrames, unsigned int imageWidth, unsigned int imageHeight,
                                     const float* intrinsics, int32_t* d_currNumFilteredMatchesPerImagePair, const float* d_currFilteredTransforms,
                                     const BFCUDACachedFrame* d_cachedFrames, float distThresh, float normalThresh, float colorThresh, float errThresh,
                                     float corrThresh, float sensorDepthMin, float sensorDepthMax, float* d_statsOut);

/* SIFTImageManager::VerifyTrajectoryCU(numImages, d_trajectory, imageWidth, imageHeight, intrinsics, d_cachedFrames, distThresh, normalThresh,
 * colorThresh, errThresh, corrThresh, sensorDepthMin, sensorDepthMax) (FL/SiftGPU/SIFTImageManager.cu:1036-1150), the check Bundler::optimize runs
 * on a chunk after its local solve (FL/Bundler.cpp:259-275): image pairs of the solved trajectory are warped into each other at the cache
 * resolution (the same projective association and block total as bfSiftFilterMatchesByDenseVerify) and *d_validOpt becomes 0 when a pair has
 * corr < corrThresh, err > errThresh or err NaN, else 1.  The reference launches N (N - 1) / 2 blocks and decodes block b as (b / N, b % N), so only
 * the pairs whose row-major index is below N (N - 1) / 2 are examined (SURVEY.md Q7) -- kept.  numImages < 2: *d_validOpt = 0 (the
 * reference returns 0).  d_trajectory: [numImages][16]; intrinsics: HOST 4x4 (cache resolution); d_statsOut: optional [N (N-1) / 2][2] (err, corr)
 * by block index.  The verdict stays on the device (the reference copies it to the host at once).  Asynchronous. */
int bfSiftVerifyTrajectory(unsigned int numImages, const int32_t* d_validImages, const float* d_trajectory, unsigned int imageWidth, unsigned int imageHeight,
                           const float* intrinsics, const BFCUDACachedFrame* d_cachedFrames, float distThresh, float normalThresh, float colorThresh,
                           float errThresh, float corrThresh, float sensorDepthMin, float sensorDepthMax, int32_t* d_validOpt, float* d_statsOut);

/* SIFTImageManager::AddCurrToResidualsCU(curFrame, startFrame, numFrames, colorIntrinsicsInv) (FL/SiftGPU/SIFTImageManager.cu:610-685):
 * appends the filtered matches of every pair p in [startFrame, numFrames), p != curFrame, to the global correspondence list as
 * EntryJ { p, curFrame, Kinv (d_i (x_i, y_i, 1)), Kinv (d_j (x_j, y_j, 1)) } (+ their key-point index pairs) and advances
 * *d_globNumResiduals -- the solver's input.  The reference reserves each pair's slots with an atomicAdd (pair order race-dependent)
 * and copies the counter to the host; here pairs are appended in ascending pair order and the counter stays on the device.
 * colorIntrinsicsInv: HOST 4x4.  Asynchronous. */
int bfSiftAddCurrToResiduals(unsigned int curFrame, unsigned int startFrame, unsigned int numFrames, BFEntryJ* d_globMatches,
                             uint32_t* d_globMatchesKeyPointIndices, int32_t* d_globNumResiduals, const int32_t* d_currNumFilteredMatchesPerImagePair,
                             const uint32_t* d_currFilteredMatchKeyPointIndices, const BFSIFTKeyPoint* d_keyPoints, const float* colorIntrinsicsInv);

/* SIFTImageManager::InvalidateImageToImageCU(imageToImageIdx) (FL/SiftGPU/SIFTImageManager.cu:692-720): every correspondence of the global list
 * between images (imgIdx_i, imgIdx_j) -- in that order -- is marked invalid (both indices 0xFFFFFFFF).  This is what SBA::removeMaxResidualCUDA
 * (FL/SBA.cpp:165-203) does with the pair the solver's max-residual search returns.  Asynchronous. */
int bfSiftInvalidateImageToImage(BFEntryJ* d_globMatches, unsigned int globNumResiduals, unsigned int imgIdx_i, unsigned int imgIdx_j);

/* SIFTImageManager::CheckForInvalidFramesSimpleCU / CheckForInvalidFramesCU(d_varToCorrNumEntriesPerRow, numVars) (:724-790): images whose row of
 * the solver's variable-to-correspondence table is empty lose their flag in d_validImages (the reference round-trips that array through the host
 * around the kernel; here it stays on the device).  comprehensive != 0 (s_useComprehensiveFrameInvalidation) additionally invalidates every
 * still-valid correspondence touching such an image -- for EVERY (image, correspondence) combination, which is what the reference's kernel is
 * written to do; its grid arithmetic (resIdx = blockDim.x * blockIdx.x + blockIdx.y) reaches only part of them.  Asynchronous. */
int bfSiftCheckForInvalidFrames(const int32_t* d_varToCorrNumEntriesPerRow, int32_t* d_validImages, unsigned int numVars, BFEntryJ* d_globMatches,
                                unsigned int globNumResiduals, int comprehensive);

/* ---- row a17: SIFT detection and description ----
 * SiftGPU::SetParams(width, height, timing, featureCountThreshold, depthMin, depthMax) (FL/SiftGPU/SiftGPU.cpp:224-254) +
 * SiftGPU::RunSIFT(d_intensity, d_depth) (:86-103) + SiftGPU::GetKeyPointsAndDescriptorsCUDA(siftImage, d_depth, maxNumKeyPoints) (:267-272), as
 * Bundler::detectFeatures calls them (FL/Bundler.cpp:55-100): four octaves from octave 0, three DoG levels each, no sub-pixel step, key
 * points only where the depth map holds a value in [depthMin, depthMax], up to two orientations per key point, 128-byte descriptors
 * (unit vector x 512), whole levels dropped from the fine end while more than featureCountThreshold features would remain without them,
 * scale >= minKeyScale (c_siftCameraParams.m_minKeyScale).  d_intensity: [height][width] floats in 0..1; d_depth: [depthHeight][depthWidth]
 * floats, -inf = invalid.  Outputs: d_keyPoints[maxKeyPoints] (x, y, scale, depth -- SIFTKeyPoint), d_descriptors[maxKeyPoints][128],
 * *d_numKeyPoints (DEVICE counter: the reference copies its level counts to the host mid-way, this path never leaves the device),
 * d_levelCounts: optional device int[12], features per (octave, level).  width must be a multiple of 32, height of 8, both >= 64.
 * Differences from the reference (its lists are appended with atomicAdd): key points of a level come in raster order, an orientation
 * pair as (first, second); histogram sums are taken in scheduling order here as there.  Asynchronous on the library stream. */
typedef struct BFSiftDetectParams {
    uint32_t width, height;              /* SIFT (intensity) image */
    uint32_t depthWidth, depthHeight;
    float depthMin, depthMax;
    float minKeyScale;
    int32_t featureCountThreshold;       /* 150 in FL/Bundler.cpp:61; <= 0: no limit */
    uint32_t maxKeyPoints;               /* capacity of the two output arrays (s_maxNumKeysPerImage) */
} BFSiftDetectParams;
int bfSiftDetect(const BFSiftDetectParams* params, const float* d_intensity, const float* d_depth, BFSIFTKeyPoint* d_keyPoints, uint8_t* d_descriptors,
                 int32_t* d_numKeyPoints, int32_t* d_levelCounts);
size_t bfSiftDetectWorkspaceBytes(void);
int bfSiftDetectReleaseWorkspace(void);

/* SIFTImageManager::filterFrames(curFrame, startFrame, numFrames) (FL/SiftGPU/SIFTImageManager.cpp:551-575) without its host round trip (the
 * reference copies the filtered-match counts to the host, searches there and copies one flag back): *d_lastMatchedFrame = the LAST frame i in
 * [startFrame, numFrames), i != curFrame, with d_validImages[i] != 0 and filtered matches, or -1; d_validImages[curFrame] = 1 if there is one,
 * else 0.  One CTA.  Asynchronous. */
int bfSiftFilterFrames(unsigned int curFrame, unsigned int startFrame, unsigned int numFrames, const int32_t* d_currNumFilteredMatchesPerImagePair,
                       int32_t* d_validImages, int32_t* d_lastMatchedFrame);

/* bfSiftAddCurrToResiduals under the condition Bundler::matchAndFilter puts on it (FL/Bundler.cpp:218-219: only when filterFrames found a
 * matched frame), evaluated on the device: nothing is appended when *d_lastMatchedFrame < 0.  With bfSiftFilterFrames this makes the whole
 * match -> sort -> filter -> verify -> residuals chain of a frame free of host synchronisation. */
int bfSiftAddCurrToResidualsIfMatched(unsigned int curFrame, unsigned int startFrame, unsigned int numFrames, BFEntryJ* d_globMatches,
                                      uint32_t* d_globMatchesKeyPointIndices, int32_t* d_globNumResiduals, const int32_t* d_currNumFilteredMatchesPerImagePair,
                                      const uint32_t* d_currFilteredMatchKeyPointIndices, const BFSIFTKeyPoint* d_keyPoints, const float* colorIntrinsicsInv,
                                      const int32_t* d_lastMatchedFrame);

/* SIFTImageManager::fuseToGlobal (FL/SiftGPU/SIFTImageManager.cpp:413-476; computeTracks / findTrack :366-411), the chunk -> keyframe fusion
 * of the sparse features Bundler::fuseToGlobal runs after a chunk's local solve (FL/Bundler.cpp:384-390) -- in the reference on the HOST
 * (device -> host copies of every key, descriptor, correspondence and pose of the chunk, a recursive walk, an upload).  Here: one launch,
 * nothing leaves the device.  Correspondences of the chunk (EntryJ + their global key-point index pairs, count on the device) are grouped
 * into tracks exactly as the reference's recursion visits them; each track with at least one member whose correspondence agrees within 3 cm
 * under the solved poses yields one key point of the new keyframe: position = mean world position projected by colorIntrinsics into the
 * chunk's first frame, depth = its z, scale and descriptor = those of the track's first-visited key.  Key k of image i has the global
 * index i * keyStride + k (d_keyPoints / d_descriptors are indexed by it; d_numKeysPerImage[i] keys of image i are walked).
 * d_transforms: [numImages][16] solved chunk poses; colorIntrinsics: HOST 4x4; maxCorr: capacity bound of the list (<= 4096), numImages *
 * keyStride <= 16384.  Outputs: d_outKeyPoints / d_outDescriptors [maxKeys], *d_outNumKeys; d_status (optional): 1 if the explicit recursion
 * stack overflowed (tracks deeper than 4096 keys).  More than maxKeys tracks: the first maxKeys in track order are kept (the reference sorts
 * the keys -- not the descriptors -- by depth with an unstable sort; unreachable with <= 11 images x ~150 features).  Asynchronous. */
int bfSiftFuseToGlobal(const BFEntryJ* d_corr, const uint32_t* d_corrKeyIndices, const int32_t* d_numCorr, const float* d_transforms, unsigned int numImages,
                       const BFSIFTKeyPoint* d_keyPoints, const uint8_t* d_descriptors, const int32_t* d_numKeysPerImage, unsigned int keyStride,
                       const float* colorIntrinsics, unsigned int maxCorr, BFSIFTKeyPoint* d_outKeyPoints, uint8_t* d_outDescriptors, int32_t* d_outNumKeys,
                       unsigned int maxKeys, int32_t* d_status);

/* device scratch the matcher holds (rowResult / rowDist per job); released by bfSiftReleaseWorkspace */
size_t bfSiftWorkspaceBytes(void);
int bfSiftReleaseWorkspace(void);
/* sizes that scratch for batches of up to maxJobs image pairs of up to maxKeysPerImage features each, so that no later bfSiftMatchBatch has to grow it
 * (growing frees and re-allocates device and pinned host memory: device-wide synchronisation in the middle of a frame) */
int bfSiftReserveWorkspace(unsigned int maxJobs, unsigned int maxKeysPerImage);

#ifdef __cplusplus
}
#endif
#endif /* BF_SIFT_H */

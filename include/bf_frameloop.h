/*
 * bf_frameloop.h -- C-ABI of the per-frame sequencing object: ONE call per sensor frame runs what FriedLiver's frame callback runs.
 *
 * The reference's frame loop (single-threaded build, no RUN_MULTITHREADED) is
 *   OnD3D11FrameRender                       FL/DepthSensing/DepthSensing.cpp:966-1129
 *     CUDAImageManager::process              FL/CUDAImageManager.cpp:22-158      frame ingest (erode, filter, resample), frame store
 *     OnlineBundler::processInput            FL/OnlineBundler.cpp:167-227        SIFT detect, dense cache, match + filters vs the chunk, SIFT pose
 *       Bundler::detectFeatures / storeCachedFrame / matchAndFilter              FL/Bundler.cpp:91-249
 *       OnlineBundler::computeCurrentSiftTransform / prepareLocalSolve           FL/OnlineBundler.cpp:118-165
 *     reintegrate()                          FL/DepthSensing/DepthSensing.cpp:854-902   <= s_maxFrameFixes re-integrations + GC
 *     integrate(current frame, SIFT pose) + TrajectoryManager::addFrame          :1033-1061
 *     OnlineBundler::process                 FL/OnlineBundler.cpp:410-416
 *       optimizeLocal  -> Bundler::optimize -> SBA::align -> CUDASolverBundling::solve (+ VerifyTrajectoryCU)   :229-262, FL/Bundler.cpp:251-283
 *       processGlobal  -> SIFTImageManager::fuseToGlobal, global matchAndFilter, re-validation                  :271-358
 *       optimizeGlobal -> global solve (+ max-residual removal), updateTrajectoryCU, TrajectoryManager update   :369-408
 * (FL/ = /root/reference/FriedLiver/Source/).  bfFrameLoopStep is that sequence behind one call: every stage is a kernel sequence of this
 * library (bf_ingest.h, bf_sift.h, bf_cache.h, bf_solver.h, bf_bundler.h, bf_tsdf.h / bf_host.h); the host state machines (Bundler /
 * OnlineBundler / SIFTImageManager bookkeeping, TrajectoryManager) are C++ inside the library (csrc/frame_loop.cu, csrc/trajectory_host.cu).
 * The host looks at the device three times per frame (key-point count after detection; match verdict + correspondence count; and, on chunk
 * boundaries, the solve verdicts) -- the reference does so dozens of times (every filter stage copies counts back).
 *
 * The end of a recording (the dense global solve of USE_GLOBAL_DENSE_AT_END, the solve stop, the re-integration drain and the validity
 * verdict of StopScanningAndExit) is bfFrameLoopFinish; the mesh is extracted by bf_marchingcubes.h.
 *
 * What is NOT here: sensors / .sens decoding, rendering (ray cast, D3D11), the multi-threaded hand-over between the reconstruction and
 * bundling threads (the call runs the reference's single-threaded order), writing the optimised poses back into the recording.
 * Threading: one BFFrameLoop per process / device, calls from one thread (the stages share the library's stream and workspaces).
 */
#ifndef BF_FRAMELOOP_H
#define BF_FRAMELOOP_H

#include <stddef.h>
#include <stdint.h>

#include "bf_host.h"
#include "bf_keyframe_search.h"
#include "bf_solver.h"
#include "bf_tsdf.h"

#ifdef __cplusplus
extern "C" {
#endif

/* GlobalAppState / GlobalBundlingState values the loop uses (FriedLiver/zParametersDefault.txt, zParametersBundlingDefault.txt) */
typedef struct BFFrameLoopParams {
    uint32_t depthWidth, depthHeight, colorWidth, colorHeight;          /* sensor images */
    uint32_t integrationWidth, integrationHeight;                      /* s_integrationWidth / Height */
    uint32_t siftWidth, siftHeight;                                     /* s_widthSIFT / s_heightSIFT */
    float    depthIntrinsics[16], colorIntrinsics[16];                  /* sensor calibration, 4x4 row-major */
    uint32_t submapSize;                                                /* s_submapSize (10) */
    uint32_t maxNumImages;                                              /* s_maxNumImages: keyframes (1200) */
    uint32_t maxNumKeysPerImage;                                        /* s_maxNumKeysPerImage (1024) */
    uint32_t maxNumFrames;                                              /* frames the device frame store / trajectories hold (<= maxNumImages * submapSize) */
    uint32_t maxGlobalResiduals;                                        /* capacity of the keyframe correspondence list; 0: 25 N (N - 1) / 2 as the reference, capped at 16 M */
    uint32_t numLocalNonLinIterations, numLocalLinIterations;           /* 2, 100 */
    uint32_t numGlobalNonLinIterations, numGlobalLinIterations;         /* 3, 150 */
    uint32_t numOptPerResidualRemoval;                                  /* 1 */
    float    sensorDepthMin, sensorDepthMax;                            /* 0.1, 4.0 */
    float    minKeyScale;                                               /* 3.0 */
    int32_t  featureCountThreshold;                                     /* 150 (FL/Bundler.cpp:61) */
    float    siftMatchThresh, siftMatchRatioMaxLocal, siftMatchRatioMaxGlobal;   /* 0.7, 0.8, 0.8 */
    uint32_t minNumMatchesLocal, minNumMatchesGlobal;                   /* 5, 5 */
    float    maxKabschResidual2;                                        /* 0.0004 */
    float    surfAreaPcaThresh;                                         /* 0.032 */
    float    projCorrDistThres, projCorrNormalThres, projCorrColorThresh;        /* 0.15, 0.97, 0.1 */
    float    verifySiftErrThresh, verifySiftCorrThresh;                 /* 0.075, 0.02 */
    float    verifyOptErrThresh, verifyOptCorrThresh;                   /* 0.05, 0.001 */
    float    optMaxResThresh;                                           /* 0.08 */
    int32_t  useLocalVerify, useLocalDense, useComprehensiveFrameInvalidation;   /* 1, 1, 1 */
    uint32_t downsampledWidth, downsampledHeight;                       /* 80, 60 */
    float    colorDownSigma, depthDownSigmaD, depthDownSigmaR;          /* 2.5, 1.0, 0.05 */
    int32_t  erodeSIFTdepth, depthFilter; float depthSigmaD, depthSigmaR;        /* 1, 1, 2.0, 0.05 */
    uint32_t maxFrameFixes, topNActive; float minPoseDistSqrt;          /* 10, 30, 0.0 */
    int32_t  reconstructionEnabled;                                     /* s_reconstructionEnabled (1) */
    BFHashParams hash;                                                  /* voxel hash parameters (poses are set per operation) */
    float    renderDepthMin, renderDepthMax;                            /* frustum test range (0.1, 4.0; SURVEY.md Q4) */
    uint32_t hashMaxSDFBlocks;                                          /* growth ceiling of the voxel heap (0: a fixed table; see bfFrameLoopGetHashGrowth) */
    uint32_t deviceFrameSlots;                                          /* device frame slots over a pinned host frame store (0: every frame on the device; see bfFrameLoopGetFrameStore) */
} BFFrameLoopParams;

/* fills *p with the defaults of zParametersDefault.txt / zParametersBundlingDefault.txt for a width x height sensor with the synthetic pinhole
 * of SURVEY.md section 8d (fx = fy = 525 * width / 640, principal point at the image centre); integration at sensor resolution */
void bfFrameLoopDefaultParams(BFFrameLoopParams* p, uint32_t width, uint32_t height);

typedef struct BFFrameLoopStatus {
    uint32_t frame;                  /* index of the frame just processed */
    int32_t  validTransform;         /* OnlineBundler::getCurrentIntegrationFrame: the frame got a SIFT pose and was integrated */
    int32_t  globalTrackingLost;
    float    transform[16];          /* the pose it was integrated with (all -inf when invalid) */
    uint32_t numKeyPoints;           /* features detected in the frame */
    int32_t  lastMatchedFrame;       /* chunk-local index of the last frame it matched, -1 if none */
    uint32_t numLocalCorrespondences;
    uint32_t numReintegrated;        /* re-integration operations executed this frame */
    int32_t  localSolved;            /* chunk index solved this frame, -1 if none;  localValid: the solve + verification accepted it */
    int32_t  localValid;
    uint32_t numKeyframes;           /* keyframes in the global manager */
    uint32_t numGlobalCorrespondences;
    int32_t  globalSolved;           /* a global solve ran */
    int32_t  globalRemoved;          /* it removed a max-residual image pair */
    uint32_t numOptimizedFrames;     /* frames the optimised trajectory covers */
} BFFrameLoopStatus;

typedef struct BFFrameLoop BFFrameLoop;

/* allocates every device buffer of the loop (frame store, SIFT managers, caches, solvers, trajectories, voxel hash) and, with deviceFrameSlots > 0,
 * the pinned host frame store (bfFrameLoopFetchFrames); returns 0 or a cudaError_t */
int bfFrameLoopCreate(const BFFrameLoopParams* params, BFFrameLoop** out);
void bfFrameLoopDestroy(BFFrameLoop* loop);

/* One sensor frame through the whole loop.  depth: float [depthHeight][depthWidth], -inf = invalid (FL/SensorDataReader.cpp:104-106); color:
 * uchar4 [colorHeight][colorWidth].  onHost != 0: the pointers are (pinned) host memory and are copied to the device inside the call, as
 * CUDAImageManager::process uploads on arrival; else they are device pointers.  Returns 0 or a cudaError_t; *status (optional) is filled. */
int bfFrameLoopStep(BFFrameLoop* loop, const float* depth, const uint8_t* color, int onHost, BFFrameLoopStatus* status);

/* The same step with look-ahead: (nextDepth, nextColor) is the frame the NEXT call will pass as (depth, color) -- a recorded stream knows it, a live sensor
 * driver knows it once the following frame has arrived.  While this frame is matched, filtered, solved and fused, the work of the next frame that depends
 * on nothing but the frame itself (upload, CUDAImageManager::process, SIFT detection, dense cache: FL/CUDAImageManager.cpp:22-158, FL/Bundler.cpp:91-101,
 * FL/CUDACache.cpp:45-86) is queued on a third stream of the loop -- the overlap the reference gets from its reconstruction and bundling threads
 * (RUN_MULTITHREADED: the image manager processes frame f + 1 while the bundler works on frame f).  Results are identical to bfFrameLoopStep: the same kernels
 * on the same inputs, their destinations (frame-store slot, key / descriptor slot and cache slot of the chunk the frame will belong to) being fixed by
 * host state one frame early.  The next call MUST pass the announced pointers (else cudaErrorInvalidValue); the buffers must stay valid and unchanged until
 * that call returns.  nextDepth == NULL: plain bfFrameLoopStep.  Look-ahead is suspended while the stage profile is on. */
int bfFrameLoopStepAhead(BFFrameLoop* loop, const float* depth, const uint8_t* color, const float* nextDepth, const uint8_t* nextColor, int onHost, BFFrameLoopStatus* status);

/* After the last frame: the reference keeps calling processInput / process with no new frame (FL/OnlineBundler.cpp:170-197) so that the last,
 * partial chunk is solved and re-integration drains.  One such turn per call. */
int bfFrameLoopStepPastEnd(BFFrameLoop* loop, BFFrameLoopStatus* status);

typedef struct BFFrameLoopFinishInfo {
    uint32_t turns;                  /* past-end turns run by this call */
    uint32_t numFramesPastEnd;       /* past-end turns run in total (bfFrameLoopStepPastEnd's included) */
    int32_t  denseTurn;              /* the past-end turn the dense global solve ran at, -1 if it has not run */
    uint32_t denseKeyframes;         /* keyframes N of that solve */
    uint32_t densePairs;             /* its dense image pairs with non-zero weight (bfSolverGetStats out[7]) */
    uint32_t globalSolves;           /* global solves run by this call */
    uint32_t reintegrations;         /* re-integration operations run by this call */
    uint32_t numTransforms;          /* frames of the optimised trajectory */
    uint32_t numValidTransforms;     /* of them with a valid pose */
    uint32_t heapFreeCount;          /* free voxel blocks */
    int32_t  valid;                  /* StopScanningAndExit's verdict: >= 800 free blocks and >= half the transforms valid */
    int32_t  done;                   /* the exit condition held: no re-integration operation is left */
} BFFrameLoopFinishInfo;

/* The end of a recording as the reference runs it with s_numSolveFramesBeforeExit = numSolveFramesBeforeExit (K; the shipped value is 30):
 * past-end turns, each exactly one bfFrameLoopStepPastEnd turn, numbered on from the turns already run, until the exit condition holds or
 * maxTurns turns have run.  Turns before K solve as bfFrameLoopStepPastEnd does.  Turn K is USE_GLOBAL_DENSE_AT_END (FL/OnlineBundler.cpp:174-189):
 * its global solve runs 3 Gauss-Newton iterations with weights sparse 1, dense depth 15, dense colour 0 over the keyframes and their cache
 * (pairwise, the local solve's dense thresholds), unless the last frame index is 10 000 or more.  From turn K + 1 on nothing is solved
 * (:190-193) and a turn only re-integrates; at the end of each such turn the TrajectoryManager's update lists are regenerated and the run is
 * done when no operation is left (FL/DepthSensing/DepthSensing.cpp:1114-1126): every frame is then fused at its final pose.
 * Returns 0 when done (a further call runs nothing), cudaErrorNotReady when maxTurns ran out first (a later call with the same K continues),
 * cudaErrorInvalidValue without running anything when no frame has been stepped, an announced look-ahead frame is pending, more than K
 * past-end turns ran before the first call, or K differs from the first call's.  *info (optional) is filled on 0 and cudaErrorNotReady;
 * the reconstruction stream is joined into the library stream before the call returns. */
int bfFrameLoopFinish(BFFrameLoop* loop, uint32_t numSolveFramesBeforeExit, uint32_t maxTurns, BFFrameLoopFinishInfo* info);

/* Fusion along a fixed trajectory: frames [0, numFrames) of the loop's frame store, frame f at the camera-to-world pose h_poses[f] (host,
 * [numFrames][16], row-major; NULL: the loop's optimised trajectory, bfFrameLoopGetTrajectory), integrated with the loop's integration camera
 * into a caller's voxel hash of any voxel size / truncation (bfTsdfReset it first; it must not be the loop's own).  Frames whose pose is not
 * finite (the trajectory's invalid frames are all -inf) are skipped.  The others go in order, in batches of <= 16 frames with a garbage
 * collection after each: one bfTsdfIntegrateBatch + bfTsdfGarbageCollect per batch when batching is usable (fast arithmetic and batching on,
 * the rule bfTsdfRunOps applies), else the same op list [INTEGRATE x <= 16, GARBAGE_COLLECT] through bfTsdfRunOps.  The reconstruction stream
 * is joined first; the work is queued on the library stream, and the call synchronises it to fill *info.  Nothing in the loop's own model or
 * state changes.  On return hashParams holds the last fused pose.  cudaErrorInvalidValue without running anything: NULL loop / hash / params,
 * an announced look-ahead frame pending (as bfFrameLoopFinish), numFrames beyond the frames stepped, or the loop's own hash. */
typedef struct BFFrameLoopFuseInfo {
    uint32_t framesFused;            /* frames integrated */
    uint32_t framesSkipped;          /* frames whose pose is not finite */
    uint32_t batches;                /* batches of <= 16 frames, one garbage collection each */
    uint32_t heapFreeCount;          /* free voxel blocks of the caller's hash at the end */
    unsigned long long insertsDropped;   /* block inserts dropped since the hash's reset (bfTsdfGetLastFrameStats out[3]): non-zero = heap or table too small */
} BFFrameLoopFuseInfo;
int bfFrameLoopFuse(BFFrameLoop* loop, BFHashDataStruct* hashData, BFHashParams* hashParams, const float* h_poses, uint32_t numFrames, BFFrameLoopFuseInfo* info);

/* Test accessor: the global (keyframe) bundle-adjustment problem as the loop holds it -- its own device pointers, valid until the next loop call.
 * The next global solve of the loop runs on exactly these inputs. */
typedef struct BFFrameLoopGlobalProblem {
    const BFEntryJ* d_correspondences;           /* keyframe correspondences */
    uint32_t numCorrespondences;
    uint32_t numKeyframes;
    const int32_t* d_validImages;                /* [numKeyframes] */
    const float* d_trajectory;                   /* [numKeyframes][16], camera-to-world, row-major */
    const BFCUDACachedFrame* d_cacheFrames;      /* [numKeyframes] keyframe cache frames */
    uint32_t cacheWidth, cacheHeight;
    float    intrinsics[4];                      /* cache-resolution fx, fy, mx, my */
    uint32_t maxNumImages;                       /* the global solver's capacity (maxNumberOfImages) */
    uint32_t maxCorrPerImage;
} BFFrameLoopGlobalProblem;
int bfFrameLoopGetGlobalProblem(const BFFrameLoop* loop, BFFrameLoopGlobalProblem* out);
/* The global (keyframe) SIFT manager's keyframe set -- keys, descriptors, key counts, cache frames, cache size and intrinsics, the inverse SIFT
 * intrinsics -- as bfKeyframeSearch reads it: the loop's own device pointers, valid until the next loop call.  Nothing in the loop changes. */
int bfFrameLoopGetKeyframes(const BFFrameLoop* loop, BFKeyframeSet* out);

/* optimised camera-to-world poses of the first n frames (host, [n][16]; invalid frames all -inf); returns the number written */
unsigned int bfFrameLoopGetTrajectory(BFFrameLoop* loop, float* h_out, unsigned int maxFrames);
/* the voxel hash the loop integrates into (caller may read it; bf_tsdf.h).  With hash growth on, both pointers, and the buffers they name, may
 * change at a growth: fetch them again after any call that runs a turn (step, past-end turn, bfFrameLoopFinish). */
const BFHashDataStruct* bfFrameLoopGetHashData(const BFFrameLoop* loop);
const BFHashParams* bfFrameLoopGetHashParams(const BFFrameLoop* loop);

/* Hash growth.  With hashMaxSDFBlocks > hash.m_numSDFBlocks the loop starts with the table of hash (its bucket and heap sizes) and may move its
 * model into larger ones, up to hashMaxSDFBlocks voxel blocks; 0 or a value <= hash.m_numSDFBlocks keeps the table fixed (the default).
 * When: at the start of a turn's reconstruction (steps, past-end turns and bfFrameLoopFinish's turns alike), before its op list runs, decided
 *   from the free-heap and dropped-insert counters of earlier turns' reconstruction work, which are read back asynchronously (a copy into pinned
 *   memory and an event, consumed when the event has completed; never waited for).  The loop grows when the free blocks of the last read-back
 *   fall below a reserve = 2 x the largest one-turn block increase seen so far x the turns since that read-back (>= 1), or when the dropped
 *   count rose (those inserts are lost: insertsDropped reports them).
 * Size: new heap = min(hashMaxSDFBlocks, max(2 x old, live + 2 x reserve)); buckets = the initial bucket-to-block ratio (doubled by every
 *   discarded attempt, below) times the new heap, odd, at most (2^32 - 1) / BF_HASH_BUCKET_SIZE (32-bit entry indices).
 * How: the reconstruction stream is joined; new buffers are allocated stream-ordered (cudaMallocAsync), bfTsdfReset + bfTsdfRehash move the
 *   model, the loop switches to the new table and frees the old one stream-ordered (cudaFreeAsync) after releasing its library scratch
 *   (bfTsdfReleaseAux).  During a growth the old and the new table are both allocated: the peak is their sum.
 * A new table whose probe windows cannot take every live block (bfTsdfRehash out[1] > 0: the bucket function put too many of them near one
 *   another) is discarded before the switch: the loop keeps the old table, which the rehash only reads, and tries again with twice the buckets
 *   per block, at most three attempts per growth; the raised ratio is kept for later growths.  No live block is lost to a growth.
 * Cost in host synchronisations: a turn that does not grow adds none; each attempt adds BF_FRAMELOOP_GROWTH_SYNCS to bfFrameLoopGetCounters
 *   out[6] (bfTsdfRehash's read of the source and its completion), so out[6] grows by (growths + discarded) x BF_FRAMELOOP_GROWTH_SYNCS.
 * The model equals, block for block and word for word keyed by position, the one a fixed table large enough never to drop would hold, as long
 *   as no insert was dropped (insertsDropped == 0; inserts are dropped when the heap or a probe window of the CURRENT table is full before the
 *   loop sees it -- the first turn, which runs before any read-back, must fit the initial table).
 * bfFrameLoopGetHashGrowth joins the reconstruction stream and synchronises (to read the dropped count). */
#define BF_FRAMELOOP_GROWTH_SYNCS 2
typedef struct BFFrameLoopHashGrowth {
    uint32_t growths;                /* tables the model moved into */
    uint32_t discarded;              /* new tables discarded because they could not take every live block (the old one was kept) */
    uint32_t sdfBlocks;              /* current heap size (voxel blocks) */
    uint32_t buckets;                /* current bucket count */
    uint32_t maxSDFBlocks;           /* the ceiling (hash.m_numSDFBlocks when growth is off) */
    unsigned long long insertsDropped;   /* block inserts dropped since bfFrameLoopCreate */
    int32_t  ceilingReached;         /* 1 once a growth was wanted and the ceiling stopped it */
} BFFrameLoopHashGrowth;
int bfFrameLoopGetHashGrowth(BFFrameLoop* loop, BFFrameLoopHashGrowth* out);
/* The growth-size rule alone (no loop): *newBlocks = min(ceiling, max(2 x blocks, live + 2 x reserve)) and *newBuckets = initBuckets x
 * *newBlocks / initBlocks, made odd, at most (2^32 - 1) / BF_HASH_BUCKET_SIZE.  The loop grows only when *newBlocks > blocks (and never
 * shrinks the bucket count). */
void bfFrameLoopHashGrowthSize(uint32_t blocks, uint32_t live, unsigned long long reserve, uint32_t ceiling, uint32_t initBlocks, uint32_t initBuckets,
                               uint32_t* newBlocks, uint32_t* newBuckets);
/* Op log (off by default; when off it costs one branch per turn): every BFTsdfOp the loop hands to bfTsdfRunOps -- re-integration items, the
 * GARBAGE_COLLECT, the INTEGRATE of the current frame -- in order, with the turn that issued it (steps and past-end turns, bfFrameLoopFinish's
 * included, counted from 0 since bfFrameLoopCreate).  Enabling it from off starts an empty log; returns the previous setting.
 * bfFrameLoopGetOpLog copies the first min(n, maxOps) ops and turns (either pointer may be NULL) and returns n, the number recorded. */
int bfFrameLoopSetOpLog(BFFrameLoop* loop, int enable);
uint32_t bfFrameLoopGetOpLog(const BFFrameLoop* loop, BFTsdfOp* out, uint32_t* turnOfOp, uint32_t maxOps);
/* Device pointers into the loop's frame store: the integration-resolution depth (float [integrationHeight][integrationWidth]) and colour
 * (uchar4) of frame f, the images every TSDF op of frame f reads.  Written on the library stream; cudaErrorInvalidValue for a frame not yet stepped.
 * With deviceFrameSlots = 0 the pointers stay valid while the loop lives.  With deviceFrameSlots > 0 this is bfFrameLoopFetchFrames(loop, &f, 1, ...)
 * and its lifetime applies. */
int bfFrameLoopGetFrame(const BFFrameLoop* loop, uint32_t f, const float** depth, const uint8_t** color);

/* The frame store.
 * deviceFrameSlots = 0 (the default): every frame has its own device slot, allocated at bfFrameLoopCreate (maxNumFrames x integrationWidth x
 *   integrationHeight x 8 bytes).
 * deviceFrameSlots = N > 0: the device holds N slots (N x W x H x 8 bytes); every frame also lives in a pinned host store of maxNumFrames frames,
 *   pinned at create in chunks of 256 frames (a chunk that cannot be pinned fails the create with cudaErrorMemoryAllocation).  N must be at
 *   least max(maxFrameFixes + 2, 16) -- one turn's re-integration frames, the current frame, the frame announced by bfFrameLoopStepAhead, and
 *   one fusion batch of 16 -- else the create returns cudaErrorInvalidValue.
 *   - After a frame's ingest writes its slot, the loop's copy stream copies the slot to the host store (write-back).
 *   - Before a turn's op list, a fusion batch of bfFrameLoopFuse or a bfFrameLoopFetchFrames call, each of its frames without a slot takes one
 *     and is copied in from the host store (fetch).  The victim is the least recently used slot that is not pinned; the frames of the current
 *     turn or batch, the current frame and the announced frame are pinned.  bfFrameLoopFuse with N >= 32 fetches batch b + 1 while batch b
 *     integrates; below 32 fetch and integrate alternate.
 *   - Ordering is by events between streams only, never a host wait: a copy into a slot waits for the slot's last reader (an event on the
 *     stream that read it), and the stream that reads a fetched frame waits for its copy.
 * Results do not depend on N: the same ops run in the same order on the same bytes, only the addresses differ.  Statuses, trajectory, op log,
 * model, bfFrameLoopFinish / bfFrameLoopFuse results and bfFrameLoopGetCounters (host synchronisations included) equal those of
 * deviceFrameSlots = 0.
 *
 * bfFrameLoopFetchFrames makes frames[0, n) resident and writes their slots' device pointers to depth[k] / color[k]; the library stream is ordered
 * after the copies (no host wait).  n <= slots - 2, every frame stepped, else cudaErrorInvalidValue with nothing enqueued.  The pointers are
 * valid until the next bfFrameLoop* call on the loop: work that reads them must be queued on the library stream before that call. */
int bfFrameLoopFetchFrames(BFFrameLoop* loop, const uint32_t* frames, uint32_t n, const float** depth, const uint8_t** color);
typedef struct BFFrameLoopFrameStore {
    uint32_t slots;                      /* device frame slots (maxNumFrames when deviceFrameSlots = 0) */
    int32_t  hostStore;                  /* 1: a pinned host store backs the slots */
    uint32_t residentFrames;             /* frames in a slot now */
    unsigned long long deviceBytes;      /* slots x W x H x 8 */
    unsigned long long hostBytes;        /* pinned host store */
    unsigned long long writeBacks;       /* frames copied to the host store */
    unsigned long long fetches;          /* frames copied into a slot from the host store */
    unsigned long long hits;             /* frames of an op list, fusion batch or fetch call that were already in a slot */
    unsigned long long evictions;        /* frames whose slot was given to another frame */
    unsigned long long h2dBytes, d2hBytes;
    double   pinMs;                      /* host time bfFrameLoopCreate spent pinning the host store */
} BFFrameLoopFrameStore;
int bfFrameLoopGetFrameStore(const BFFrameLoop* loop, BFFrameLoopFrameStore* out);
/* counters for measurement: out[0] frames, out[1] integrations, out[2] re-integrations, out[3] local solves, out[4] global solves,
 * out[5] PCG iterations (global, last solve), out[6] host synchronisations, out[7] keyframes */
void bfFrameLoopGetCounters(const BFFrameLoop* loop, unsigned long long out[8]);

/* Two streams: with overlap on, the re-integration + integration of frame f are queued on a second, lower-priority stream of the loop and run beside
 * the solves of frame f and the feature work of frame f + 1 -- what the reference's reconstruction and bundling threads do -- with the data
 * dependencies of the single-threaded order kept by events (same results).  Off by default (everything on the library stream).
 * bfFrameLoopJoin makes the library stream wait (asynchronously) for the reconstruction stream: call it before recording an event that should
 * cover the fused model, or before reading the voxel hash on the library stream (bfFrameLoopGetHashData does it itself).  Returns the previous setting. */
int bfFrameLoopSetOverlap(BFFrameLoop* loop, int enable);
int bfFrameLoopJoin(BFFrameLoop* loop);

/* Stage profile (measurement only; adds one host synchronisation per step while on).  Stages of a step, in order:
 *   0 upload + ingest      1 SIFT detection      2 dense cache (+ wait for the key-point count)      3 match + filters + SIFT pose
 *   4 re-integration + GC + integration      5 local solve (+ verification)      6 fuse to keyframe + keyframe matching      7 global solve + trajectory update
 * bfFrameLoopGetStageTimes: milliseconds on the device time line summed per stage since bfFrameLoopSetProfiling(loop, 1); returns the steps covered. */
#define BF_FRAMELOOP_STAGES 8
int bfFrameLoopSetProfiling(BFFrameLoop* loop, int enable);
unsigned long long bfFrameLoopGetStageTimes(const BFFrameLoop* loop, double outMs[BF_FRAMELOOP_STAGES]);

#ifdef __cplusplus
}
#endif
#endif /* BF_FRAMELOOP_H */

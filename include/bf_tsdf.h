/*
 * bf_tsdf.h -- C-ABI of the hashed-voxel TSDF path (SURVEY.md section 8, rows a1-a9).
 *
 * Every entry point in the first half of this header carries the NAME and the
 * machine-level signature of an `extern "C"` launch stub of the reference, so a
 * FriedLiver build can link this library in place of its own
 * CUDASceneRepHashSDF.cu / CUDAConstant.cu objects:
 *
 *   reference declaration (C++ reference parameter)         here (pointer; same ABI)
 *   FL/DepthSensing/CUDASceneRepHashSDF.h:15-27             resetCUDA ... garbageCollectFreeCUDA
 *   FL/DepthSensing/VoxelUtilHashSDF.h:101                  updateConstantHashParams
 *   FL/DepthSensing/DepthCameraUtil.h:13                    updateConstantDepthCameraParams
 *
 * (FL/ = /root/reference/FriedLiver/Source/).  A C++ reference parameter and a
 * pointer parameter are the same thing at the x86-64 SysV ABI level, which is
 * why these prototypes can be plain C.
 *
 * The POD structs are layout-identical to the reference's (sizes/offsets probed
 * with nvcc 12.9 + g++ 13 against the reference headers, with the `__align__(16)` of
 * HashEntry / HashParams / DepthCameraParams honoured as MSVC does: HashEntry is 32 bytes,
 * see below and SURVEY.md quirk Q1).  Types carry a BF prefix so that both headers can be
 * visible in one translation unit.
 *
 * The second half (bfTsdf*) is the H100-native, sync-free extension the host
 * mirror class (bundlefusion_b200/host/SceneRepHashSDF.h) drives: one call per
 * integrate / de-integrate, no device->host copy, no constant upload.
 *
 * Ownership: the caller allocates every buffer named in BFHashDataStruct
 * (FL/DepthSensing/VoxelUtilHashSDF.h:124-149) and passes raw DEVICE pointers.
 * Depth / colour images are borrowed for the duration of the call.
 */
#ifndef BF_TSDF_H
#define BF_TSDF_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BF_SDF_BLOCK_SIZE 8          /* FL/DepthSensing/VoxelUtilHashSDF.h:40 */
#define BF_SDF_BLOCK_VOXELS 512
#define BF_HASH_BUCKET_SIZE 4        /* :41 */
#define BF_LOCK_ENTRY (-1)           /* :52 */
#define BF_FREE_ENTRY (-2)           /* :53 */
#define BF_NO_OFFSET 0               /* :54 */

/* row-major 4x4, m[r*4+c]  (FL/SiftGPU/cuda_SimpleMatrixUtil.h:855; mLib mat4f) */
typedef struct BFFloat4x4 { float m[16]; } BFFloat4x4;

/* FL/DepthSensing/VoxelUtilHashSDF.h:56-74 : 5 x int32 declared `__align__(16) struct HashEntry`.
 * In the build the reference actually ships (MSVC host + nvcc, FriedLiver.vcxproj) that is __declspec(align(16)):
 * sizeof == 32, 16-byte aligned -- the layout used here.  (gcc / nvcc-on-Linux ignore an attribute placed BEFORE `struct`,
 * giving 20 bytes; the reference then faults on its own 8-byte entry copies, VoxelUtilHashSDF.h:70-72 -- observed when
 * building oracle/_ref, which therefore moves the attribute.)  Define BF_HASH_ENTRY_PACKED20 to get the 20-byte variant. */
#ifdef BF_HASH_ENTRY_PACKED20
typedef struct BFHashEntry {
    int32_t  pos[3];   /* SDF-block coordinate (block = 8^3 voxels)            */
    int32_t  ptr;      /* heapSlot*512 (index of first voxel) or FREE/LOCK     */
    uint32_t offset;   /* linked-list offset relative to bucket's last slot    */
} BFHashEntry;
#else
typedef struct
#if defined(__GNUC__) || defined(__CUDACC__)
    __attribute__((aligned(16)))
#else
    __declspec(align(16))
#endif
BFHashEntry {
    int32_t  pos[3];   /* SDF-block coordinate (block = 8^3 voxels)            */
    int32_t  ptr;      /* heapSlot*512 (index of first voxel) or FREE/LOCK     */
    uint32_t offset;   /* linked-list offset relative to bucket's last slot    */
    uint32_t _pad[3];  /* tail padding of the 16-byte aligned struct           */
} BFHashEntry;
#endif

/* FL/DepthSensing/VoxelUtilHashSDF.h:77-98 : 12 bytes */
typedef struct BFVoxel {
    float   sdf;
    float   weight;
    uint8_t color[4];
} BFVoxel;

/* FL/DepthSensing/CUDAHashParams.h:10-38 : 224 bytes, 8-byte aligned */
typedef struct BFHashParams {
    BFFloat4x4 m_rigidTransform;            /*   0 */
    BFFloat4x4 m_rigidTransformInverse;     /*  64 */
    uint32_t m_hashNumBuckets;              /* 128 */
    uint32_t m_hashBucketSize;
    uint32_t m_hashMaxCollisionLinkedListSize;
    uint32_t m_numSDFBlocks;
    int32_t  m_SDFBlockSize;                /* 144 */
    float    m_virtualVoxelSize;
    uint32_t m_numOccupiedBlocks;
    float    m_maxIntegrationDistance;      /* 156 */
    float    m_truncScale;
    float    m_truncation;
    uint32_t m_integrationWeightSample;
    uint32_t m_integrationWeightMax;
    float    m_streamingVoxelExtents[3];    /* 176 */
    int32_t  m_streamingGridDimensions[3];
    int32_t  m_streamingMinGridPos[3];
    uint32_t m_streamingInitialChunkListSize;
#if defined(__GNUC__) || defined(__CUDACC__)
    uint32_t m_dummy[2] __attribute__((aligned(8)));   /* 216 (uint2) */
#else
    __declspec(align(8)) uint32_t m_dummy[2];
#endif
} BFHashParams;

/* FL/DepthSensing/CUDADepthCameraParams.h:7-19 : 32 bytes */
typedef struct BFDepthCameraParams {
    float fx, fy, mx, my;
    uint32_t m_imageWidth, m_imageHeight;
    float m_sensorDepthWorldMin;   /* "render depth" min, used by the frustum test */
    float m_sensorDepthWorldMax;
} BFDepthCameraParams;

/* FL/DepthSensing/DepthCameraUtil.h:17-154 : two device pointers */
typedef struct BFDepthCameraData {
    const float*   d_depthData;    /* W*H float, metres, invalid = -inf          */
    const uint8_t* d_colorData;    /* W*H uchar4 RGBA (may be NULL)              */
} BFDepthCameraData;

/* FL/DepthSensing/VoxelUtilHashSDF.h:830-840 : 80 bytes */
typedef struct BFHashDataStruct {
    uint32_t*    d_heap;                    /* free-slot stack                   */
    uint32_t*    d_heapCounter;             /* index of the top element          */
    int32_t*     d_hashDecision;            /* per compactified entry: GC flag   */
    int32_t*     d_hashDecisionPrefix;      /* scratch (4*buckets ints)          */
    BFHashEntry* d_hash;                    /* numBuckets*4 entries              */
    BFHashEntry* d_hashCompactified;        /* in-frustum entries                */
    int32_t*     d_hashCompactifiedCounter;
    BFVoxel*     d_SDFBlocks;               /* numSDFBlocks*512 voxels           */
    int32_t*     d_hashBucketMutex;         /* one int per bucket                */
    uint8_t      m_bIsOnGPU;                /* bool                              */
} BFHashDataStruct;

/* ------------------------------------------------------------------------ *
 *  Part 1: the reference's own launch stubs (drop-in names).               *
 *  Error behaviour follows cutilSafeCall (cutil_inline_runtime.h:277-285): *
 *  a CUDA error prints file/line to stderr and terminates with exit(-1).   *
 * ------------------------------------------------------------------------ */

/* FL/DepthSensing/CUDAConstant.cu:10-20 -- latches the params every later stub uses */
void updateConstantHashParams(const BFHashParams* hashParams);
/* FL/DepthSensing/CUDAConstant.cu:23-33 */
void updateConstantDepthCameraParams(const BFDepthCameraParams* params);
/* FL/DepthSensing/CUDASceneRepHashSDF.cu:15-25 -- latches depth/colour pointers */
void bindInputDepthColorTextures(const BFDepthCameraData* depthCameraData,
                                 unsigned int width, unsigned int height);

/* FL/DepthSensing/CUDASceneRepHashSDF.cu:67-111 */
void resetCUDA(BFHashDataStruct* hashData, const BFHashParams* hashParams);
/* :113-124 */
void resetHashBucketMutexCUDA(BFHashDataStruct* hashData, const BFHashParams* hashParams);
/* :253-264 -- one call allocates EVERY block the frame needs (no host retry loop needed;
 * calling it repeatedly as the reference's host loop does is harmless and idempotent). */
void allocCUDA(BFHashDataStruct* hashData, const BFHashParams* hashParams,
               const BFDepthCameraData* depthCameraData,
               const BFDepthCameraParams* depthCameraParams,
               const unsigned int* d_bitMask);
/* :284-296, :309-320 -- the (unused by the reference's live path) 3-step compactify */
void fillDecisionArrayCUDA(BFHashDataStruct* hashData, const BFHashParams* hashParams);
void compactifyHashCUDA(BFHashDataStruct* hashData, const BFHashParams* hashParams);
/* :368-384 -- returns the in-frustum block count (device->host sync, as the reference) */
unsigned int compactifyHashAllInOneCUDA(BFHashDataStruct* hashData, const BFHashParams* hashParams);
/* :524-536, :538-550 -- grid = hashParams->m_numOccupiedBlocks entries of d_hashCompactified */
void integrateDepthMapCUDA(BFHashDataStruct* hashData, const BFHashParams* hashParams,
                           const BFDepthCameraData* depthCameraData,
                           const BFDepthCameraParams* depthCameraParams);
void deIntegrateDepthMapCUDA(BFHashDataStruct* hashData, const BFHashParams* hashParams,
                             const BFDepthCameraData* depthCameraData,
                             const BFDepthCameraParams* depthCameraParams);
/* :565-577 */
void starveVoxelsKernelCUDA(BFHashDataStruct* hashData, const BFHashParams* hashParams);
/* :633-645, :671-683 */
void garbageCollectIdentifyCUDA(BFHashDataStruct* hashData, const BFHashParams* hashParams);
void garbageCollectFreeCUDA(BFHashDataStruct* hashData, const BFHashParams* hashParams);

/* ------------------------------------------------------------------------ *
 *  Part 2: H100-native extension (what the host mirror class calls).       *
 *  All calls are asynchronous on the stream set by bfSetStream(); they      *
 *  return 0 or a cudaError_t value and never terminate the process.         *
 * ------------------------------------------------------------------------ */

/* stream every entry point of this library launches on (default: legacy stream 0) */
void  bfSetStream(void* cudaStream);
void* bfGetStream(void);
/* last error string recorded by a bf* call on this thread ("" if none) */
const char* bfGetLastErrorString(void);

/* bytes of library-private device scratch bfTsdf* keeps per hash (reported for DESIGN.md) */
size_t bfTsdfAuxBytes(const BFHashParams* hashParams);

/* FL/DepthSensing/CUDASceneRepHashSDF.h:147-155 (reset) */
int bfTsdfReset(BFHashDataStruct* hashData, const BFHashParams* hashParams);

/* Arithmetic of the integrate / de-integrate / re-integration stencil (process-wide; returns the previous setting).
 *   BF_TSDF_ARITH_FAST  (default, also BF_TSDF_ARITH=fast): tolerance contract -- allocated block set and weights identical, |d sdf| <= 1e-5 m,
 *     colour +-1, except for a <= 1e-4 fraction of voxels on a pixel / truncation decision boundary; this is what the reference's shipped
 *     --use_fast_math build is to its IEEE build (FriedLiver.vcxproj; FL/DepthSensing/CUDASceneRepHashSDF.cu:420-521).
 *   BF_TSDF_ARITH_EXACT (BF_TSDF_ARITH=exact): every sdf / weight / colour word bit-identical to the reference's IEEE build and to
 *     oracle/tsdf_oracle.c (~3x the instructions per voxel probe: two IEEE divides, individually rounded operations). */
#define BF_TSDF_ARITH_EXACT 0
#define BF_TSDF_ARITH_FAST 1
int bfTsdfSetArithmetic(int mode);

/* Two-lane replay inside bfTsdfRunOps (default on): the stencil of operation k runs on a library-owned stream while alloc +
 * compactify of operation k+1 run on the caller's stream; the caller's stream is ordered after all of it on return.  Results are
 * identical either way.  Returns the previous setting. */
int bfTsdfSetLanes(int enable);

/* One whole CUDASceneRepHashSDF::integrate (h:65-83) or ::deIntegrate (h:85-108):
 * [alloc] -> compactify -> (de)integrate, three launches, zero host syncs.
 * hashParams carries the pose (m_rigidTransform AND its inverse, as the reference's
 * setLastRigidTransform computes them on the host, h:128-134).  The in-frustum block
 * count stays on the device (d_hashCompactifiedCounter); fetch it with
 * bfTsdfGetNumOccupiedBlocks() only when the host needs it. */
int bfTsdfIntegrateFrame(BFHashDataStruct* hashData, const BFHashParams* hashParams,
                         const BFDepthCameraData* depthCameraData,
                         const BFDepthCameraParams* depthCameraParams,
                         int deIntegrate);

/* deIntegrate(old pose) + integrate(new pose) of the SAME frame -- the body of the reference's re-integration loop
 * (FL/DepthSensing/DepthSensing.cpp:867-895) -- as ONE fused pass: alloc(new) -> compactify over the union of both frusta ->
 * per voxel de-integrate then integrate in registers.  Voxels, block set and heap are bit-identical to the two-call sequence;
 * one voxel read + write instead of two.  d_hashCompactified then holds the union list. */
int bfTsdfReintegrateFrame(BFHashDataStruct* hashData, const BFHashParams* hashParamsOldPose, const BFHashParams* hashParamsNewPose,
                           const BFDepthCameraData* depthCameraData, const BFDepthCameraParams* depthCameraParams);

/* A batch of re-integrations -- numPairs (<= 16) x { deIntegrate(frame, oldPose); integrate(frame, newPose) }, the loop of
 * FL/DepthSensing/DepthSensing.cpp:867-895 -- as numPairs alloc launches, ONE union list and ONE stencil pass: every voxel of the list is
 * read once, taken through the pairs in order in registers, written once.  Blocks inserted by pair k's alloc are invisible to the pairs before
 * k, as in the reference's order.  Fast arithmetic only (bfTsdfSetArithmetic); results are bit-identical to replaying the pairs one by one
 * through bfTsdfReintegrateFrame in fast arithmetic.  hashParams carries the pose-independent parameters and returns holding the last new
 * pose.  d_hashCompactified then holds the union list (its GC flags mark the last pair's new-pose frustum, the list the reference's GC walks).
 * bfTsdfRunOps routes runs of >= 2 pairs here when batching is on (default; BF_TSDF_BATCH=0 / bfTsdfSetBatching(0) replays pair by pair).
 * Batch cull: while building the union list, a (block, pair, pose) whose voxels provably all fail the truncation test against the pair's frame
 * (16x16-pixel depth min / max under the block's screen footprint, left behind by the pair's alloc launch; conservative margins) is not handed
 * to the stencil.  Results are unchanged; E (in-frustum blocks) still counts the culled entries, bfTsdfGetProfileEx out[15] how many were removed. */
typedef struct BFTsdfReintegration { int32_t frame; float oldPose[16]; float newPose[16]; } BFTsdfReintegration;
int bfTsdfReintegrateBatch(BFHashDataStruct* hashData, BFHashParams* hashParams, const BFDepthCameraParams* depthCameraParams,
                           const BFTsdfReintegration* pairs, int numPairs, const float* const* d_depthFrames, const uint8_t* const* d_colorFrames);
int bfTsdfSetBatching(int enable);

/* n (1..16) integrations of frames[k] at poses[k] (camera-to-world, row-major [n][16]) -- n calls of CUDASceneRepHashSDF::integrate --
 * as n alloc launches, ONE union list and ONE stencil pass.  Fast arithmetic; bit-identical to n bfTsdfIntegrateFrame calls in the same order
 * (block set, heap and free list, every voxel word, the live-voxel counters and so what a following bfTsdfGarbageCollect frees), including
 * frames whose blocks a later frame of the batch inserts (they stay invisible to the earlier frames), frames with no valid pixel and a heap
 * that runs out inside the batch.  The machinery is bfTsdfReintegrateBatch's (op-tagged allocs, union list, cost buckets, depth-tile cull)
 * compiled with no old pose: no old frustum is tested and nothing is de-integrated.  On return hashParams holds the last pose and
 * d_hashCompactified the union list (its GC flags mark the last frame's frustum).  Returns cudaErrorInvalidValue with nothing enqueued for
 * n < 1 or n > 16, NULL frames / poses / frame arrays, a negative frame index or one whose depth or colour pointer is NULL.  In exact
 * arithmetic (bfTsdfSetArithmetic) it runs the fast pass, as bfTsdfReintegrateBatch does. */
int bfTsdfIntegrateBatch(BFHashDataStruct* hashData, BFHashParams* hashParams, const BFDepthCameraParams* depthCameraParams,
                         const int32_t* frames, const float* poses, int n, const float* const* d_depthFrames, const uint8_t* const* d_colorFrames);

/* Sizing a hash from the blocks a fusion will allocate.
 *
 * BFBlockKeySet: a caller-owned device set of SDF-block positions.  d_keys holds `capacity` (a power of two, <= 2^31) 64-bit slots, 0 = empty;
 * a stored key is bit 63 | (x + 2^20) << 42 | (y + 2^20) << 21 | (z + 2^20).  d_counters[0] = distinct keys stored, [1] = keys refused because
 * every slot held another key (nothing is written for them: grow the set -- bfTsdfBlockKeyMerge into a larger one -- and count those frames
 * again), [2] = blocks with a coordinate outside [-2^20, 2^20) that no key can hold.  Zero d_keys and d_counters before the first call; calls
 * accumulate, so a recording can be counted 16 frames at a time from a ring of device slots.
 *
 * bfTsdfCountBlocks adds to the set every block that bfTsdfIntegrateBatch's alloc launches would insert for frames[k] at poses[k] (same
 * arguments, hashParams the pose-independent parameters): the same walk compiled with another sink, the pose and its inverse formed on the
 * host as bfTsdfIntegrateBatch forms them, the same frustum test, depth validity and m_maxIntegrationDistance, and the same shard ownership
 * under m_dummy = {rank, world}.  The hash's sizes are not read.
 *
 * bfTsdfBlockKeyLoad writes d_out[0] = keys in the set, d_out[1] = the largest load of any of numBuckets buckets under the hash's own bucket
 * function, d_out[2] = over = sum over buckets of max(0, load - BF_HASH_BUCKET_SIZE); d_bucketLoad (numBuckets words) receives the loads.
 *
 * The guarantee: the blocks live in a hash fused from an empty state by bfTsdfIntegrateBatch / bfFrameLoopFuse over the counted frames and
 * poses are always a subset of the counted union, garbage collection included (GC only removes blocks).  With numBuckets such that over == 0
 * and m_numSDFBlocks >= d_counters[0], every insert therefore finds a free slot in its home bucket: no overflow list, no probe, no drop, and
 * the heap cannot run out.  When over > 0 nothing is claimed beyond what bfTsdfGetLastFrameStats reports after the fusion.
 *
 * All three return cudaErrorInvalidValue with nothing enqueued for: n < 1 or n > 16, NULL set / keys / counters / hashParams / camera / frames /
 * poses / depth array, a negative frame index or NULL depth pointer, a capacity that is 0, not a power of two or above 2^31, numBuckets == 0,
 * NULL d_bucketLoad / d_out, and merging a set into itself.  Asynchronous on the library stream. */
typedef struct BFBlockKeySet {
    uint64_t* d_keys;
    uint32_t* d_counters;     /* [3] */
    uint32_t  capacity;
} BFBlockKeySet;
int bfTsdfCountBlocks(BFBlockKeySet* set, const BFHashParams* hashParams, const BFDepthCameraParams* depthCameraParams, const int32_t* frames,
                      const float* poses, int n, const float* const* d_depthFrames);
int bfTsdfBlockKeyLoad(const BFBlockKeySet* set, uint32_t numBuckets, uint32_t* d_bucketLoad, uint32_t* d_out);
/* every key of src into dst (growing a set); src's counters are not read */
int bfTsdfBlockKeyMerge(BFBlockKeySet* dst, const BFBlockKeySet* src);

/* CUDASceneRepHashSDF::garbageCollect (h:110-126) over the last compactified list */
int bfTsdfGarbageCollect(BFHashDataStruct* hashData, const BFHashParams* hashParams);

/* Move every live block of src into dst, a hash reset by bfTsdfReset with the same voxel size, truncation, truncation scale, maximum
 * integration distance, block / bucket size, linked-list limit and m_dummy shard setting, and any bucket count and heap size.  Synchronises;
 * out[0] = blocks moved, out[1] = blocks dst could not take (0 unless dst is too small: its probe window or heap ran out).
 *
 * Each live block goes into dst through the insertion rule of every alloc launch (home bucket, else the bucket's overflow list, heap pop, the
 * slot table), with its voxel words and its live-voxel counter.  The state later calls read moves with it: the live-voxel validity, the dropped-
 * insert counters (added to dst's, so bfTsdfGetLastFrameStats out[3] still counts every drop since src's reset), the stencil statistics, and
 * the last compactified list -- same order, same count, its GC flags, each entry's ptr translated to its block's new slot -- so that a
 * bfTsdfGarbageCollect issued next frees on dst exactly the blocks it would have freed on src.
 *
 * The guarantee: two hashes that differ only by a rehash hold the same block set and the same voxel words, keyed by block position, and every
 * later operation keeps them so.  Heap slots and entry positions may differ, as they already do between two runs of an alloc launch.
 *
 * Returns cudaErrorInvalidValue with nothing written to dst for: a NULL argument or buffer, src == dst, any buffer the two share, a differing
 * parameter of the list above, a bucket count of 0 or above 2^32 / BF_HASH_BUCKET_SIZE, a hash this library does not maintain (not reset by
 * bfTsdfReset with these sizes), and -- after one synchronising read of src -- a dst heap smaller than src's live blocks or its last list.
 * Work runs on the library stream; its temporaries are stream-ordered allocations (cudaMallocAsync). */
int bfTsdfRehash(const BFHashDataStruct* src, const BFHashParams* srcParams, BFHashDataStruct* dst, const BFHashParams* dstParams,
                 unsigned long long out[2]);

/* synchronising getters (h:168-172 getHeapFreeCount; m_numOccupiedBlocks) */
int bfTsdfGetHeapFreeCount(const BFHashDataStruct* hashData, unsigned int* outCount);
int bfTsdfGetNumOccupiedBlocks(const BFHashDataStruct* hashData, unsigned int* outCount);

/* counters of the last bfTsdfIntegrateFrame, for the roofline arithmetic
 * (SURVEY.md section 8d: U = voxels passing the truncation test, E = in-frustum blocks).
 * out[0]=E, out[1]=0 (reserved), out[2]=U, out[3]=block inserts dropped since reset
 * (heap exhausted or no free entry inside the probe window; 0 in a sanely sized table).  Synchronises. */
int bfTsdfGetLastFrameStats(const BFHashDataStruct* hashData, unsigned long long out[4]);

/* measurement hooks used by bench.py (never needed for correctness):
 * bfGetLaunchCount   -- kernels this library has launched since load (all paths);
 * bfTsdfSetProfiling -- when enabled every integrate / de-integrate stencil launch is bracketed by CUDA events on the library stream;
 * bfTsdfGetProfile   -- out[0] stencil launches, out[1] launches timed, out[2] their summed duration (ns), out[3] sum of U,
 *                       out[4] sum of E over those launches, out[5] frame images those launches read (one per launch, one per pair for a
 *                       batch launch); synchronises and restarts the accumulation. */
unsigned long long bfGetLaunchCount(void);
/* bfTsdfGetProfile plus the batch launches alone: out[8] batch launches, out[9] timed, out[10] their duration (ns), out[11] their U, out[12] their E,
 * out[13] frame images they read, out[14] their duration by in-kernel %globaltimer brackets (first CTA start to last CTA end, ns),
 * out[15] (block, pair, pose) entries the batch cull removed (32-bit running sum); out[6..7] = 0 */
int bfTsdfGetProfileEx(const BFHashDataStruct* hashData, unsigned long long out[16]);
int bfTsdfSetProfiling(int enable);
int bfTsdfGetProfile(const BFHashDataStruct* hashData, unsigned long long out[8]);

/* release the library-private scratch attached to this hash (call before freeing d_hash) */
int bfTsdfReleaseAux(const BFHashDataStruct* hashData);

#ifdef __cplusplus
}
#endif
#endif /* BF_TSDF_H */

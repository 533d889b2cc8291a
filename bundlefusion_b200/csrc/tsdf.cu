// tsdf.cu -- hashed-voxel TSDF: reset / alloc / compactify / integrate / de-integrate / GC
// for sm_90a.  Implements include/bf_tsdf.h (rows a1-a9 of SURVEY.md section 8).
//
// Behavioural source (what, not how): FL/DepthSensing/CUDASceneRepHashSDF.cu:27-684,
// FL/DepthSensing/VoxelUtilHashSDF.h:226-826, FL/DepthSensing/DepthCameraUtil.h:71-144.
//
// Design (see DESIGN.md section "TSDF"):
//  * no __constant__ uploads, no texture binds: parameters travel as __grid_constant__
//    kernel arguments, images are read through the read-only path;
//  * allocation is ONE kernel (in-kernel bucket spin locks), not a host retry loop with a
//    device->host copy per round (reference: CUDASceneRepHashSDF.h:335-348);
//  * compactify walks a dense slot-indexed side table (16 B per EVER-allocated block) instead
//    of the whole 4*numBuckets entry table (reference: .cu:324-384), and leaves its count on
//    the device; the integrate kernel is a persistent grid that reads that count itself;
//  * the integrate stencil owns 4 consecutive voxels (48 B = three 16-byte vector accesses)
//    per thread, touches voxel memory only for threads that pass the truncation test, and
//    can be preceded by a conservative per-block depth-range cull (off by default, measured);
//  * garbage collection is a single fused kernel (identify + unlink + heap push + clear).
//
// Compiled with -fmad=false so that float results are bit-identical to oracle/tsdf_oracle.c.
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/bf_tsdf.h"
#include "bf_common.cuh"
#include "tsdf_shared.cuh"
#include "mat4.cuh"

namespace bf {

// ------------------------------------------------------------------------------------------
// global (per-process) latched state -- the reference keeps the same things in __constant__
// memory and texture references, which makes its entry points non-re-entrant per device too.
// ------------------------------------------------------------------------------------------
static thread_local std::string t_lastError;
static cudaStream_t g_stream = 0;
void set_last_error(const char* where, cudaError_t e) {
    t_lastError = std::string(where) + ": " + cudaGetErrorString(e);
}
cudaStream_t stream() { return g_stream; }

static BFHashParams g_hashParams;           // updateConstantHashParams
static BFDepthCameraParams g_camParams;     // updateConstantDepthCameraParams
static BFDepthCameraData g_bound = {nullptr, nullptr};   // bindInputDepthColorTextures
const BFHashParams* bound_hash_params() { return &g_hashParams; }                  // for the reference-named stubs of other translation units (raycast.cu)
const BFDepthCameraParams* bound_camera_params() { return &g_camParams; }

// library-private per-hash scratch ("aux"), keyed by the d_hash pointer
struct TsdfAux {
    int4* slotInfo = nullptr;        // [numSDFBlocks] {bx,by,bz, entryIdx} ; entryIdx < 0: slot free
    unsigned* ctrs = nullptr;        // see CTR_* below
    int* live = nullptr;             // [numSDFBlocks] number of voxels with weight > 0 in the slot's block
    unsigned char* listFlags = nullptr;   // [numSDFBlocks] per compactified entry: bit0 in old frustum, bit1 in new (fused re-integration)
    int4* work = nullptr;            // [numSDFBlocks] stencil work list {bx,by,bz, slot | pose bits << 28}: list entries that survive the depth-range cull
    float2* tiles = nullptr;         // [tilesCap] per 16x16-pixel tile {min, max} of the depths the stencil would accept
    unsigned tilesCap = 0;
    float2* tilesMulti = nullptr;    // [BF_MULTI_MAX_OPS][tilesMultiPer]: depth tiles of the frames of a re-integration batch
    unsigned tilesMultiPer = 0;
    bool liveValid = false;          // false once something outside integrate/de-integrate changed weights
    unsigned numSlots = 0;
    unsigned parity = 0;             // which of the two compactify counters is live
    bool lastListDual = false;       // the live list is a union list of a fused re-integration (GC then visits only its new-pose part)
    // two-lane replay (bfTsdfRunOps): alloc + compactify of op k+1 on the caller's stream while the stencil of op k runs on `lane`
    int4* work2[2] = { nullptr, nullptr };   // work list per counter set (work2[0] aliases `work`)
    cudaStream_t lane = nullptr;
    cudaEvent_t evFork = nullptr, evList[2] = { nullptr, nullptr }, evStencil[2] = { nullptr, nullptr };
    bool stencilPending[2] = { false, false };
    bool pipeOpen = false;
    // batch re-integration (tsdf_reintegrate_batch): per slot the (batch id << 8 | op index) of the alloc launch that inserted the block,
    // per work item the 2-bit-per-op frustum mask
    unsigned* slotEpoch = nullptr; unsigned* workMask = nullptr; unsigned* workMask2 = nullptr; unsigned batchId = 0;
    const void* owner[3] = { nullptr, nullptr, nullptr };   // the caller's d_SDFBlocks / d_heap / d_hashCompactified: the key (d_hash) can be
                                                            // recycled by an allocator for another table; all four together identify one
};
// launch accounting + optional CUDA-event timing of the integrate / de-integrate stencil (bench.py's roofline line)
unsigned long long g_launchCount = 0;
static bool g_profile = false;
static std::vector<cudaEvent_t> g_evStart, g_evStop;
static size_t g_evUsed = 0;
static unsigned long long g_profLaunches = 0;
static unsigned long long g_profFrames = 0;
static unsigned long long g_profBatchLaunches = 0, g_profBatchFrames = 0;
static std::vector<unsigned char> g_evIsBatch;
static unsigned long long* g_ktime = nullptr;        // [kMaxProfiledLaunches][2] in-kernel %globaltimer brackets of the profiled batch launches      // frame images the profiled stencil launches read (a batch launch reads one per pair)
static const size_t kMaxProfiledLaunches = 16384;

static std::mutex g_auxMutex;
static std::map<const void*, TsdfAux> g_aux;

static int get_aux(const BFHashDataStruct* hd, const BFHashParams* hp, TsdfAux** out, bool create, bool adopt = true);

// ------------------------------------------------------------------------------------------
// device math shared by every kernel (bit-exact mirror of oracle/tsdf_oracle.c)
// ------------------------------------------------------------------------------------------
struct F3 { float x, y, z; };
struct I3 { int x, y, z; };

__device__ __forceinline__ int isign(float v) { return (0.0f < v) - (v < 0.0f); }

// cuda_SimpleMatrixUtil.h:937-944 (affine, implicit w = 1), fused exactly as nvcc fuses the reference's expression
// (oracle/tsdf_oracle.c header: the arithmetic contract); the TU is built -fmad=false so only these explicit FMAs fuse
__device__ __forceinline__ F3 xform(const BFFloat4x4& M, F3 v) {
    F3 r;
    r.x = __fmaf_rn(v.z, M.m[2], __fmaf_rn(v.x, M.m[0], v.y * M.m[1])) + M.m[3];
    r.y = __fmaf_rn(v.z, M.m[6], __fmaf_rn(v.x, M.m[4], v.y * M.m[5])) + M.m[7];
    r.z = __fmaf_rn(v.z, M.m[10], __fmaf_rn(v.x, M.m[8], v.y * M.m[9])) + M.m[11];
    return r;
}
// VoxelUtilHashSDF.h:226-234 (unsigned modulo, see oracle note)
__device__ __forceinline__ unsigned hash_pos(unsigned numBuckets, I3 p) {
    unsigned v = ((unsigned)p.x * 73856093u) ^ ((unsigned)p.y * 19349669u) ^ ((unsigned)p.z * 83492791u);
    return v % numBuckets;
}
__device__ __forceinline__ float truncation(const BFHashParams& hp, float z) { return __fmaf_rn(hp.m_truncScale, z, hp.m_truncation); }
__device__ __forceinline__ I3 world_to_voxel(const BFHashParams& hp, F3 pos) {
    F3 p = { pos.x / hp.m_virtualVoxelSize, pos.y / hp.m_virtualVoxelSize, pos.z / hp.m_virtualVoxelSize };
    I3 r = { (int)(p.x + (float)isign(p.x) * 0.5f), (int)(p.y + (float)isign(p.y) * 0.5f), (int)(p.z + (float)isign(p.z) * 0.5f) };
    return r;
}
__device__ __forceinline__ I3 voxel_to_block(I3 v) {
    if (v.x < 0) v.x -= BF_SDF_BLOCK_SIZE - 1;
    if (v.y < 0) v.y -= BF_SDF_BLOCK_SIZE - 1;
    if (v.z < 0) v.z -= BF_SDF_BLOCK_SIZE - 1;
    I3 r = { v.x / BF_SDF_BLOCK_SIZE, v.y / BF_SDF_BLOCK_SIZE, v.z / BF_SDF_BLOCK_SIZE };
    return r;
}
__device__ __forceinline__ F3 voxel_to_world(const BFHashParams& hp, I3 v) {
    F3 r = { (float)v.x * hp.m_virtualVoxelSize, (float)v.y * hp.m_virtualVoxelSize, (float)v.z * hp.m_virtualVoxelSize };
    return r;
}
__device__ __forceinline__ F3 block_to_world(const BFHashParams& hp, I3 b) {
    I3 v = { b.x * BF_SDF_BLOCK_SIZE, b.y * BF_SDF_BLOCK_SIZE, b.z * BF_SDF_BLOCK_SIZE };
    return voxel_to_world(hp, v);
}
__device__ __forceinline__ I3 world_to_block(const BFHashParams& hp, F3 w) { return voxel_to_block(world_to_voxel(hp, w)); }

__device__ __forceinline__ float proj_z(const BFDepthCameraParams& cp, float z) {
    return (z - cp.m_sensorDepthWorldMin) / (cp.m_sensorDepthWorldMax - cp.m_sensorDepthWorldMin);
}
__device__ __forceinline__ F3 depth_to_skeleton(const BFDepthCameraParams& cp, unsigned ux, unsigned uy, float depth) {
    const float x = ((float)ux - cp.mx) / cp.fx;
    const float y = ((float)uy - cp.my) / cp.fy;
    F3 r = { depth * x, depth * y, depth };
    return r;
}
// DepthCameraUtil.h:95-107,137-144 + VoxelUtilHashSDF.h:322-326
__device__ __forceinline__ bool block_in_frustum_m(float vs, const BFFloat4x4& Minv, const BFDepthCameraParams& cp, I3 b);
__device__ __forceinline__ bool block_in_frustum(const BFHashParams& hp, const BFDepthCameraParams& cp, I3 b) {
    return block_in_frustum_m(hp.m_virtualVoxelSize, hp.m_rigidTransformInverse, cp, b);
}
__device__ __forceinline__ bool block_in_frustum_m(float vs, const BFFloat4x4& Minv, const BFDepthCameraParams& cp, I3 b) {
    const float off = vs * 0.5f * ((float)BF_SDF_BLOCK_SIZE - 1.0f);
    const F3 w = { __fmaf_rn((float)(b.x * BF_SDF_BLOCK_SIZE), vs, off), __fmaf_rn((float)(b.y * BF_SDF_BLOCK_SIZE), vs, off),
                   __fmaf_rn((float)(b.z * BF_SDF_BLOCK_SIZE), vs, off) };
    F3 pc = xform(Minv, w);
    const float px = pc.x * cp.fx / pc.z + cp.mx;
    const float py = pc.y * cp.fy / pc.z + cp.my;
    const float w1 = (float)cp.m_imageWidth - 1.0f, h1 = (float)cp.m_imageHeight - 1.0f;
    float ix = (2.0f * px - w1) / w1;
    float iy = (h1 - 2.0f * py) / h1;
    float iz = proj_z(cp, pc.z);
    ix *= 0.95f; iy *= 0.95f; iz *= 0.95f;
    return !(ix < -1.0f || ix > 1.0f || iy < -1.0f || iy > 1.0f || iz < 0.0f || iz > 1.0f);
}

// ------------------------------------------------------------------------------------------
// hash table primitives.  Entry = 5 ints (20 B).  Loads on the lock-free fast path may come
// from L1 (possibly stale => at worst a spurious miss that is re-checked under the lock);
// loads under a bucket lock use ld.global.cg (L2), stores are followed by __threadfence().
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ bool entry_matches(const BFHashEntry* e, I3 p) {
    return e->pos[0] == p.x && e->pos[1] == p.y && e->pos[2] == p.z && e->ptr != BF_FREE_ENTRY;
}
__device__ __forceinline__ BFHashEntry load_entry_cg(const BFHashEntry* e) {
    BFHashEntry r;
    const int* s = reinterpret_cast<const int*>(e);
    r.pos[0] = __ldcg(s + 0); r.pos[1] = __ldcg(s + 1); r.pos[2] = __ldcg(s + 2); r.ptr = __ldcg(s + 3);
    r.offset = (unsigned)__ldcg(s + 4);
    return r;
}
__device__ __forceinline__ bool entry_matches_v(const BFHashEntry& e, I3 p) {
    return e.pos[0] == p.x && e.pos[1] == p.y && e.pos[2] == p.z && e.ptr != BF_FREE_ENTRY;
}

// VoxelUtilHashSDF.h:440-485 ; returns entry index or -1.  kCoherent: read through L2.
template <bool kCoherent>
__device__ int find_entry(const BFHashEntry* __restrict__ hash, const BFHashParams& hp, I3 p, unsigned h) {
    const unsigned hpz = h * BF_HASH_BUCKET_SIZE;
    const unsigned total = BF_HASH_BUCKET_SIZE * hp.m_hashNumBuckets;
#pragma unroll
    for (unsigned j = 0; j < BF_HASH_BUCKET_SIZE; ++j) {
        if (kCoherent) { if (entry_matches_v(load_entry_cg(&hash[hpz + j]), p)) return (int)(hpz + j); }
        else           { if (entry_matches(&hash[hpz + j], p)) return (int)(hpz + j); }
    }
    const unsigned last = hpz + BF_HASH_BUCKET_SIZE - 1;
    unsigned i = last;
    for (unsigned it = 0; it < hp.m_hashMaxCollisionLinkedListSize; ++it) {
        BFHashEntry c = kCoherent ? load_entry_cg(&hash[i]) : hash[i];
        if (entry_matches_v(c, p)) return (int)i;
        if (c.offset == 0) break;
        i = (last + c.offset) % total;
    }
    return -1;
}

__device__ __forceinline__ bool try_lock(int* mutex) { return atomicCAS(mutex, BF_FREE_ENTRY, BF_LOCK_ENTRY) == BF_FREE_ENTRY; }
__device__ __forceinline__ void unlock(int* mutex) { __threadfence(); atomicExch(mutex, BF_FREE_ENTRY); }

// VoxelUtilHashSDF.h:535-540 consumeHeap, plus an exhaustion guard (the reference has none)
__device__ __forceinline__ bool heap_pop(unsigned* heap, unsigned* heapCounter, unsigned* slot) {
    unsigned addr = atomicSub(heapCounter, 1u);
    if (addr == 0xFFFFFFFFu || addr >= 0x80000000u) { atomicAdd(heapCounter, 1u); return false; }
    *slot = __ldcg(&heap[addr]);
    return true;
}

__device__ __forceinline__ void write_entry(BFHashEntry* e, I3 p, unsigned offset, int ptr) {
    int* d = reinterpret_cast<int*>(e);
    __stcg(d + 0, p.x); __stcg(d + 1, p.y); __stcg(d + 2, p.z); __stcg(d + 4, (int)offset);
    __threadfence();
    __stcg(d + 3, ptr);       // ptr last: a reader that sees a valid ptr sees a valid pos
}

// Insert `pos` (VoxelUtilHashSDF.h:549-655 semantics: bucket slot first, else splice into the
// bucket's overflow list).  Unlike the reference (try-lock, give up, host retries) this spins
// until the block is present, so one launch reaches the reference's fixed point.
// slotEpoch / tag (optional): batch re-integration -- a block inserted by THIS launch is tagged with (batch id << 8 | op index), so that the
// multi-op stencil can tell which operations of the batch saw the block exist (tsdf_reintegrate_batch)
struct AllocEpoch { unsigned* slotEpoch; unsigned tag; };
__device__ void alloc_block(const BFHashDataStruct& hd, const BFHashParams& hp, int4* slotInfo, unsigned* ctrs, I3 pos, AllocEpoch ep = AllocEpoch{nullptr, 0u}) {
    const unsigned h = hash_pos(hp.m_hashNumBuckets, pos);
    if (find_entry<false>(hd.d_hash, hp, pos, h) >= 0) return;      // fast path, no lock

    const unsigned hpz = h * BF_HASH_BUCKET_SIZE;
    const unsigned last = hpz + BF_HASH_BUCKET_SIZE - 1;
    const unsigned total = BF_HASH_BUCKET_SIZE * hp.m_hashNumBuckets;
    const unsigned maxLoop = hp.m_hashMaxCollisionLinkedListSize;
    int* mutexH = &hd.d_hashBucketMutex[h];

    bool done = false;
    unsigned backoff = 32;
    while (!done) {
        if (try_lock(mutexH)) {
            __threadfence();
            if (find_entry<true>(hd.d_hash, hp, pos, h) >= 0) { unlock(mutexH); return; }
            // first free slot of the home bucket
            int firstEmpty = -1;
#pragma unroll
            for (unsigned j = 0; j < BF_HASH_BUCKET_SIZE; ++j) {
                int p = __ldcg(&hd.d_hash[hpz + j].ptr);
                if (firstEmpty == -1 && p == BF_FREE_ENTRY) firstEmpty = (int)(hpz + j);
            }
            if (firstEmpty != -1) {
                unsigned slot;
                if (heap_pop(hd.d_heap, hd.d_heapCounter, &slot)) {
                    slotInfo[slot] = make_int4(pos.x, pos.y, pos.z, firstEmpty);
                    if (ep.slotEpoch) ep.slotEpoch[slot] = ep.tag;
                    atomicMax(&ctrs[CTR_HIGH_WATER], slot + 1u);
                    write_entry(&hd.d_hash[firstEmpty], pos, BF_NO_OFFSET, (int)(slot * BF_SDF_BLOCK_VOXELS));
                } else {
                    atomicAdd(&ctrs[CTR_HEAP_FAIL], 1u);
                }
                unlock(mutexH);
                return;
            }
            // overflow: probe forward for a free non-bucket-last slot (:614-654)
            unsigned offset = 0, it = 0;
            bool retry = false;
            while (it < maxLoop) {
                offset++;
                const unsigned i = (last + offset) % total;
                if ((offset % BF_HASH_BUCKET_SIZE) == 0) continue;
                if (__ldcg(&hd.d_hash[i].ptr) == BF_FREE_ENTRY) {
                    const unsigned h2 = i / BF_HASH_BUCKET_SIZE;
                    int* mutex2 = &hd.d_hashBucketMutex[h2];
                    const bool same = (h2 == h);
                    if (!same && !try_lock(mutex2)) { retry = true; break; }   // avoid lock-order deadlock
                    __threadfence();
                    if (__ldcg(&hd.d_hash[i].ptr) == BF_FREE_ENTRY) {
                        unsigned slot;
                        if (heap_pop(hd.d_heap, hd.d_heapCounter, &slot)) {
                            const unsigned lastOffset = (unsigned)__ldcg(reinterpret_cast<const int*>(&hd.d_hash[last]) + 4);
                            slotInfo[slot] = make_int4(pos.x, pos.y, pos.z, (int)i);
                            if (ep.slotEpoch) ep.slotEpoch[slot] = ep.tag;
                            atomicMax(&ctrs[CTR_HIGH_WATER], slot + 1u);
                            write_entry(&hd.d_hash[i], pos, lastOffset, (int)(slot * BF_SDF_BLOCK_VOXELS));
                            __threadfence();
                            __stcg(reinterpret_cast<int*>(&hd.d_hash[last]) + 4, (int)offset);   // publish: head -> new
                        } else {
                            atomicAdd(&ctrs[CTR_HEAP_FAIL], 1u);
                        }
                        if (!same) unlock(mutex2);
                        unlock(mutexH);
                        return;
                    }
                    if (!same) unlock(mutex2);
                    // slot was taken meanwhile: keep probing (does not count as an iteration)
                    continue;
                }
                it++;
            }
            unlock(mutexH);
            if (!retry) { atomicAdd(&ctrs[CTR_DROPPED], 1u); return; }   // no room within the probe window: dropped (as the reference)
        }
        __nanosleep(backoff + ((threadIdx.x * 7u) & 63u));     // jitter: break lock-step livelock inside a warp
        if (backoff < 1024) backoff <<= 1;
    }
}

// ------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------

// reset (CUDASceneRepHashSDF.cu:27-65): heap = identity stack, voxels = 0, entries = FREE.
__global__ void reset_kernel(BFHashDataStruct hd, unsigned numSDFBlocks, unsigned numBuckets, int4* slotInfo, unsigned* ctrs, int* live) {
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    if (tid == 0) hd.d_heapCounter[0] = numSDFBlocks - 1;
    if (tid < CTR_NUM) ctrs[tid] = 0;
    for (size_t i = tid; i < numSDFBlocks; i += stride) {
        hd.d_heap[i] = numSDFBlocks - (unsigned)i - 1;
        slotInfo[i] = make_int4(0, 0, 0, -1);
        live[i] = 0;
    }
    // voxels: 12 B each -> clear as 16-byte vectors (the heap is 16-byte aligned, 6144 B per block)
    uint4* vox = reinterpret_cast<uint4*>(hd.d_SDFBlocks);
    const size_t nVec = (size_t)numSDFBlocks * (BF_SDF_BLOCK_VOXELS * sizeof(BFVoxel) / 16);
    for (size_t i = tid; i < nVec; i += stride) vox[i] = make_uint4(0, 0, 0, 0);
    const size_t nEntries = (size_t)numBuckets * BF_HASH_BUCKET_SIZE;
    for (size_t i = tid; i < nEntries; i += stride) {
        BFHashEntry e; e.pos[0] = e.pos[1] = e.pos[2] = 0; e.ptr = BF_FREE_ENTRY; e.offset = 0;
        hd.d_hash[i] = e;
        hd.d_hashCompactified[i] = e;
    }
    for (size_t i = tid; i < numBuckets; i += stride) hd.d_hashBucketMutex[i] = BF_FREE_ENTRY;
}

__global__ void reset_mutex_kernel(int* mutex, unsigned numBuckets) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < numBuckets) mutex[i] = BF_FREE_ENTRY;
}

// allocKernel (CUDASceneRepHashSDF.cu:165-251): one thread per depth pixel, DDA over SDF blocks
// along the ray segment [d-t, d+t].
//
// Two phases per 16x16-pixel CTA.  Phase 1 walks every pixel's DDA with NO global-memory access and
// collects the distinct blocks the tile touches in a shared-memory hash set (a tile touches a few dozen
// blocks, each 8^3 block spans ~20 px at 2 m, while its 256 pixels take ~3 000 DDA steps).  Phase 2
// resolves the distinct blocks in parallel, one thread per block: frustum test, table lookup, insert.
// The dependent chain of table lookups a pixel would otherwise pay once per new block (5 L2 round trips
// each) collapses to a single round.  The union over pixels -- the set the reference allocates -- is
// unchanged.
#define BF_ALLOC_SET 1024      // slots of the per-CTA set (power of two); overflow falls back to direct handling

// ---- depth tiles + conservative per-block cull ----------------------------------------------------------------------
// tiles[ty * tilesX + tx] = {min, max} over the 16x16-pixel tile of the depths the stencil accepts (`depth != -inf &&
// depth < maxIntegrationDistance`, .cu:441); {+inf, -inf} when the tile holds none.  Written by alloc_kernel (its CTAs are
// exactly these tiles) or by depth_tiles_kernel when no allocation precedes the stencil (de-integration).
#define BF_TILE 16
__device__ __forceinline__ void tile_minmax(const BFHashParams& hp, float d, bool inImage, unsigned tid, float2* sRed /*[8]*/) {
    const bool ok = inImage && d != -INFINITY && d < hp.m_maxIntegrationDistance;
    float mn = ok ? d : INFINITY, mx = ok ? d : -INFINITY;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o)); mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); }
    if ((tid & 31) == 0) sRed[tid >> 5] = make_float2(mn, mx);
}
__device__ __forceinline__ float2 tile_minmax_finish(const float2* sRed) {
    float2 r = sRed[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) { r.x = fminf(r.x, sRed[w].x); r.y = fmaxf(r.y, sRed[w].y); }
    return r;
}
__global__ void __launch_bounds__(256)
depth_tiles_kernel(const __grid_constant__ BFHashParams hp, const __grid_constant__ BFDepthCameraParams cp, const float* __restrict__ depth, float2* tiles) {
    __shared__ float2 sRed[8];
    const unsigned tid = threadIdx.y * blockDim.x + threadIdx.x;
    const unsigned x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    const bool in = x < cp.m_imageWidth && y < cp.m_imageHeight;
    tile_minmax(hp, in ? __ldg(&depth[y * cp.m_imageWidth + x]) : 0.0f, in, tid, sRed);
    __syncthreads();
    if (tid == 0) tiles[blockIdx.y * gridDim.x + blockIdx.x] = tile_minmax_finish(sRed);
}

// Can ANY voxel of block b pass the stencil's test `on screen && depth valid && |depth - z| < truncation(depth)` for the pose in
// hp?  Conservative (never false when a voxel passes): the cube of voxel centres is bounded by a camera-space AABB, its
// projection by a pixel rectangle with a pixel of slack, the depths under it by the tile min/max, all with a 1 mm (+ relative)
// margin that dwarfs the fp32 rounding of the per-voxel projection.  Results are therefore unchanged; ~35 % of the in-frustum
// blocks of a scan (looking past / short of the surface, or at invalid depth) never reach the stencil.
__device__ __forceinline__ bool block_can_pass_m(float s, float T, float vs, const BFFloat4x4& Minv, const BFDepthCameraParams& cp, const float2* __restrict__ tiles, int tilesX, I3 b) {
    if (!(s >= 0.0f && s < 1.0f && T >= 0.0f && cp.fx > 0.0f && cp.fy > 0.0f && vs > 0.0f)) return true;
    const float* M = Minv.m;
    const float h = 0.5f * ((float)BF_SDF_BLOCK_SIZE - 1.0f) * vs;
    const F3 c = { (float)(b.x * BF_SDF_BLOCK_SIZE) * vs + h, (float)(b.y * BF_SDF_BLOCK_SIZE) * vs + h, (float)(b.z * BF_SDF_BLOCK_SIZE) * vs + h };
    const F3 pc = xform(Minv, c);
    const float eps = 1e-3f + 1e-5f * (fabsf(c.x) + fabsf(c.y) + fabsf(c.z) + fabsf(M[3]) + fabsf(M[7]) + fabsf(M[11]));
    const float ex = (fabsf(M[0]) + fabsf(M[1]) + fabsf(M[2])) * h + eps;
    const float ey = (fabsf(M[4]) + fabsf(M[5]) + fabsf(M[6])) * h + eps;
    const float ez = (fabsf(M[8]) + fabsf(M[9]) + fabsf(M[10])) * h + eps;
    const float zmin = pc.z - ez, zmax = pc.z + ez;
    if (!(zmin > 0.05f)) return true;                       // too close to the camera plane for a projection bound (or NaN)
    const float xlo = pc.x - ex, xhi = pc.x + ex, ylo = pc.y - ey, yhi = pc.y + ey;
    const float ulo = cp.fx * (xlo >= 0.0f ? xlo / zmax : xlo / zmin) + cp.mx, uhi = cp.fx * (xhi >= 0.0f ? xhi / zmin : xhi / zmax) + cp.mx;
    const float vlo = cp.fy * (ylo >= 0.0f ? ylo / zmax : ylo / zmin) + cp.my, vhi = cp.fy * (yhi >= 0.0f ? yhi / zmin : yhi / zmax) + cp.my;
    // the stencil's pixel is trunc(u + 0.5): bound it by floor(u + 0.5) -+ 1, clamped to the image
    const float W1 = (float)cp.m_imageWidth - 1.0f, H1 = (float)cp.m_imageHeight - 1.0f;
    const int x0 = (int)fmaxf(floorf(ulo + 0.5f) - 1.0f, 0.0f), x1 = (int)fminf(floorf(uhi + 0.5f) + 1.0f, W1);
    const int y0 = (int)fmaxf(floorf(vlo + 0.5f) - 1.0f, 0.0f), y1 = (int)fminf(floorf(vhi + 0.5f) + 1.0f, H1);
    if (x1 < x0 || y1 < y0) return false;                   // wholly off screen
    const int tx0 = x0 / BF_TILE, tx1 = x1 / BF_TILE, ty0 = y0 / BF_TILE, ty1 = y1 / BF_TILE;
    if ((tx1 - tx0 + 1) * (ty1 - ty0 + 1) > 64) return true;
    float dmin = INFINITY, dmax = -INFINITY;
    for (int ty = ty0; ty <= ty1; ++ty)
        for (int tx = tx0; tx <= tx1; ++tx) { const float2 t = __ldg(&tiles[ty * tilesX + tx]); dmin = fminf(dmin, t.x); dmax = fmaxf(dmax, t.y); }
    if (!(dmax >= dmin)) return false;                      // no acceptable depth under the footprint
    return !(zmin >= dmax * (1.0f + s) + T + eps || zmax <= dmin * (1.0f - s) - T - eps);
}
__device__ __forceinline__ bool block_can_pass(const BFHashParams& hp, const BFDepthCameraParams& cp, const float2* __restrict__ tiles, int tilesX, I3 b) {
    return block_can_pass_m(hp.m_truncScale, hp.m_truncation, hp.m_virtualVoxelSize, hp.m_rigidTransformInverse, cp, tiles, tilesX, b);
}
__device__ __forceinline__ I3 unpack_block_key(unsigned long long key) {
    const int lim = 1 << 20;
    I3 b = { (int)((key >> 42) & 0x1FFFFF) - lim, (int)((key >> 21) & 0x1FFFFF) - lim, (int)(key & 0x1FFFFF) - lim };
    return b;
}

// Multi-GPU spatial shard (SURVEY.md section 8e): when hp.m_dummy = {rank, world} with world > 1, this device allocates
// (and therefore integrates) only the blocks it owns.  Ownership is a 3-D checkerboard of cubes of BF_SHARD_CUBE^3 blocks
// (64 cm at 1 cm voxels): owner = (cx + cy + cz) mod world.  Cubes, not a per-block hash, so that ownership is coherent along
// a ray: a pixel whose 20-odd-cm ray segment only crosses cubes of other ranks is dropped before its DDA walk (dda_setup).
#define BF_SHARD_CUBE 8
__device__ __forceinline__ int floor_div_cube(int v) { return (v >= 0) ? v / BF_SHARD_CUBE : -((-v + BF_SHARD_CUBE - 1) / BF_SHARD_CUBE); }
__device__ __forceinline__ unsigned cube_owner(int cx, int cy, int cz, unsigned world) {
    const int m = (cx + cy + cz) % (int)world;
    return (unsigned)(m < 0 ? m + (int)world : m);
}
__device__ __forceinline__ bool owns_block(const BFHashParams& hp, I3 b) {
    const unsigned world = hp.m_dummy[1];
    if (world <= 1) return true;
    return cube_owner(floor_div_cube(b.x), floor_div_cube(b.y), floor_div_cube(b.z), world) == hp.m_dummy[0];
}
// does the block-coordinate box [lo, hi] (the DDA of a ray never leaves the box spanned by its first and last block) touch a cube
// this rank owns?
__device__ __forceinline__ bool box_touches_owned(const BFHashParams& hp, I3 a, I3 b) {
    const unsigned world = hp.m_dummy[1];
    if (world <= 1) return true;
    const int x0 = floor_div_cube(min(a.x, b.x)), x1 = floor_div_cube(max(a.x, b.x));
    const int y0 = floor_div_cube(min(a.y, b.y)), y1 = floor_div_cube(max(a.y, b.y));
    const int z0 = floor_div_cube(min(a.z, b.z)), z1 = floor_div_cube(max(a.z, b.z));
    if ((long long)(x1 - x0 + 1) * (y1 - y0 + 1) * (z1 - z0 + 1) > 64) return true;      // a very long segment: just walk it
    for (int z = z0; z <= z1; ++z)
        for (int y = y0; y <= y1; ++y)
            for (int x = x0; x <= x1; ++x)
                if (cube_owner(x, y, z, world) == hp.m_dummy[0]) return true;
    return false;
}

struct DDA {                    // state of one pixel's block walk (.cu:189-219)
    I3 cur, bound;
    F3 step, tMax, tDelta;
};
// returns false when the pixel contributes nothing (.cu:176-187)
__device__ __forceinline__ bool dda_setup(const BFHashParams& hp, const BFDepthCameraParams& cp, const float* __restrict__ depth,
                                          unsigned x, unsigned y, DDA& s) {
    if (!(x < cp.m_imageWidth && y < cp.m_imageHeight)) return false;
    const float d = __ldg(&depth[y * cp.m_imageWidth + x]);
    if (d == -INFINITY || d == 0.0f) return false;
    if (d >= hp.m_maxIntegrationDistance) return false;
    const float t = truncation(hp, d);
    const float minDepth = fminf(hp.m_maxIntegrationDistance, d - t);
    const float maxDepth = fminf(hp.m_maxIntegrationDistance, d + t);
    if (minDepth >= maxDepth) return false;

    const F3 rayMin = xform(hp.m_rigidTransform, depth_to_skeleton(cp, x, y, minDepth));
    const F3 rayMax = xform(hp.m_rigidTransform, depth_to_skeleton(cp, x, y, maxDepth));
    const F3 dv = { rayMax.x - rayMin.x, rayMax.y - rayMin.y, rayMax.z - rayMin.z };
    const float inv = 1.0f / sqrtf(dv.x * dv.x + dv.y * dv.y + dv.z * dv.z);
    const F3 dir = { dv.x * inv, dv.y * inv, dv.z * inv };

    s.cur = world_to_block(hp, rayMin);
    const I3 end = world_to_block(hp, rayMax);
    if (!box_touches_owned(hp, s.cur, end)) return false;      // multi-GPU: nothing on this ray is ours
    s.step.x = (float)isign(dir.x); s.step.y = (float)isign(dir.y); s.step.z = (float)isign(dir.z);
    const I3 nb = { s.cur.x + (int)fminf(fmaxf(s.step.x, 0.0f), 1.0f), s.cur.y + (int)fminf(fmaxf(s.step.y, 0.0f), 1.0f),
                    s.cur.z + (int)fminf(fmaxf(s.step.z, 0.0f), 1.0f) };
    const F3 bw = block_to_world(hp, nb);
    const float vs = hp.m_virtualVoxelSize;
    const float half = 0.5f * vs;
    const F3 boundary = { bw.x - half, bw.y - half, bw.z - half };
    s.tMax.x = (boundary.x - rayMin.x) / dir.x; s.tMax.y = (boundary.y - rayMin.y) / dir.y; s.tMax.z = (boundary.z - rayMin.z) / dir.z;
    s.tDelta.x = (s.step.x * (float)BF_SDF_BLOCK_SIZE * vs) / dir.x;
    s.tDelta.y = (s.step.y * (float)BF_SDF_BLOCK_SIZE * vs) / dir.y;
    s.tDelta.z = (s.step.z * (float)BF_SDF_BLOCK_SIZE * vs) / dir.z;
    s.bound.x = (int)((float)end.x + s.step.x); s.bound.y = (int)((float)end.y + s.step.y); s.bound.z = (int)((float)end.z + s.step.z);
    if (dir.x == 0.0f) { s.tMax.x = INFINITY; s.tDelta.x = INFINITY; }
    if (boundary.x - rayMin.x == 0.0f) { s.tMax.x = INFINITY; s.tDelta.x = INFINITY; }
    if (dir.y == 0.0f) { s.tMax.y = INFINITY; s.tDelta.y = INFINITY; }
    if (boundary.y - rayMin.y == 0.0f) { s.tMax.y = INFINITY; s.tDelta.y = INFINITY; }
    if (dir.z == 0.0f) { s.tMax.z = INFINITY; s.tDelta.z = INFINITY; }
    if (boundary.z - rayMin.z == 0.0f) { s.tMax.z = INFINITY; s.tDelta.z = INFINITY; }
    return true;
}
// advance along the axis with the smallest tMax (same tie-breaking as .cu:232-246); returns false at the end of the walk
__device__ __forceinline__ bool dda_step(DDA& s, int& axis) {
    const bool sx = (s.tMax.x < s.tMax.y) && (s.tMax.x < s.tMax.z);
    const bool sz = !sx && (s.tMax.z < s.tMax.y);
    int v = sx ? s.cur.x : (sz ? s.cur.z : s.cur.y);
    const float st = sx ? s.step.x : (sz ? s.step.z : s.step.y);
    const int bd = sx ? s.bound.x : (sz ? s.bound.z : s.bound.y);
    v = (int)((float)v + st);
    if (v == bd) return false;
    if (sx)      { s.cur.x = v; s.tMax.x += s.tDelta.x; axis = 0; }
    else if (sz) { s.cur.z = v; s.tMax.z += s.tDelta.z; axis = 2; }
    else         { s.cur.y = v; s.tMax.y += s.tDelta.y; axis = 1; }
    return true;
}
// the reference's single-phase walk: every visited in-frustum block goes straight to the table (rare fallback)
__device__ __noinline__ void alloc_pixel_direct(const BFHashDataStruct& hd, const BFHashParams& hp, const BFDepthCameraParams& cp,
                                                const float* __restrict__ depth, unsigned x, unsigned y, int4* slotInfo, unsigned* ctrs, AllocEpoch ep) {
    DDA s;
    if (!dda_setup(hp, cp, depth, x, y, s)) return;
#pragma unroll 1
    for (unsigned iter = 0; iter < 1024; ++iter) {
        if (block_in_frustum(hp, cp, s.cur) && owns_block(hp, s.cur)) alloc_block(hd, hp, slotInfo, ctrs, s.cur, ep);
        int axis;
        if (!dda_step(s, axis)) return;
    }
}

__global__ void __launch_bounds__(256, 8)    // 32 regs: the whole 640x480 frame is resident in one wave
alloc_kernel(BFHashDataStruct hd, const __grid_constant__ BFHashParams hp, const __grid_constant__ BFDepthCameraParams cp,
             const float* __restrict__ depth, int4* slotInfo, unsigned* ctrs, float2* tiles, int zeroSet, AllocEpoch ep) {
    __shared__ unsigned long long sSet[BF_ALLOC_SET];
    __shared__ float2 sRed[8];
    const unsigned tid = threadIdx.y * blockDim.x + threadIdx.x;
    if (zeroSet >= 0 && blockIdx.x == 0 && blockIdx.y == 0 && tid < SET_WORDS) ctrs[zeroSet + tid] = 0;   // nothing in this kernel reads the set
    for (unsigned i = tid; i < BF_ALLOC_SET; i += 256) sSet[i] = 0ull;
    const unsigned x = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned y = blockIdx.y * blockDim.y + threadIdx.y;
    if (tiles) {           // this CTA is one 16x16 depth tile: leave its min / max for the per-block cull of the stencil
        const bool in = x < cp.m_imageWidth && y < cp.m_imageHeight;
        tile_minmax(hp, in ? __ldg(&depth[y * cp.m_imageWidth + x]) : 0.0f, in, tid, sRed);
    }
    __syncthreads();
    if (tiles && tid == 0) tiles[blockIdx.y * gridDim.x + blockIdx.x] = tile_minmax_finish(sRed);

    DDA s;
    bool needDirect = false;
    if (dda_setup(hp, cp, depth, x, y, s)) {
        // Set bookkeeping maintained incrementally along the walk: a 64-bit key with three biased 21-bit fields
        // and an additive hash (both change by a per-axis constant when the walk steps along that axis).
        const int lim = 1 << 20;
        const bool packable = s.cur.x > -lim && s.cur.x < lim && s.cur.y > -lim && s.cur.y < lim && s.cur.z > -lim && s.cur.z < lim &&
                              s.bound.x > -lim && s.bound.x < lim && s.bound.y > -lim && s.bound.y < lim && s.bound.z > -lim && s.bound.z < lim;
        if (!packable) {
            needDirect = true;
        } else {
            const unsigned HA = 0x9E3779B1u, HB = 0x85EBCA77u, HC = 0xC2B2AE3Du;
            unsigned long long key = (1ull << 63) | ((unsigned long long)(unsigned)(s.cur.x + lim) << 42) |
                                     ((unsigned long long)(unsigned)(s.cur.y + lim) << 21) | (unsigned long long)(unsigned)(s.cur.z + lim);
            unsigned h = (unsigned)s.cur.x * HA + (unsigned)s.cur.y * HB + (unsigned)s.cur.z * HC;
            const int isx = (int)s.step.x, isy = (int)s.step.y, isz = (int)s.step.z;
            const long long dk[3] = { (long long)isx * (1ll << 42), (long long)isy * (1ll << 21), (long long)isz };
            const unsigned dh[3] = { (unsigned)isx * HA, (unsigned)isy * HB, (unsigned)isz * HC };
#pragma unroll 1
            for (unsigned iter = 0; iter < 1024; ++iter) {
                // record the block in the CTA's set (linear probing, <= 8 probes)
                bool recorded = false;
                unsigned slot = h >> 22;                                    // BF_ALLOC_SET == 1024 slots
#pragma unroll 1
                for (int probe = 0; probe < 8; ++probe) {
                    const unsigned long long seen = sSet[slot];
                    if (seen == key) { recorded = true; break; }
                    if (seen == 0ull) {
                        const unsigned long long prev = atomicCAS(&sSet[slot], 0ull, key);
                        if (prev == 0ull || prev == key) { recorded = true; break; }
                    }
                    slot = (slot + 1) & (BF_ALLOC_SET - 1);
                }
                if (!recorded) { needDirect = true; break; }
                int axis;
                if (!dda_step(s, axis)) break;
                key += (unsigned long long)(axis == 0 ? dk[0] : (axis == 2 ? dk[2] : dk[1]));
                h += (axis == 0 ? dh[0] : (axis == 2 ? dh[2] : dh[1]));
            }
        }
    }
    __syncthreads();
    // phase 2: one thread per distinct block
    for (unsigned i = tid; i < BF_ALLOC_SET; i += 256) {
        const unsigned long long key = sSet[i];
        if (key == 0ull) continue;
        const I3 b = unpack_block_key(key);
        if (block_in_frustum(hp, cp, b) && owns_block(hp, b)) alloc_block(hd, hp, slotInfo, ctrs, b, ep);
    }
    if (needDirect) alloc_pixel_direct(hd, hp, cp, depth, x, y, slotInfo, ctrs, ep);   // set overflow / coordinates out of key range
}

// compactify: list of allocated AND in-frustum blocks (CUDASceneRepHashSDF.cu:324-366),
// produced from the dense slot table [0, highWater) instead of the 4*numBuckets entry table.
// Warp-aggregated append; counts accumulate in the counter set `set` (zeroed by the preceding launch).
__global__ void __launch_bounds__(256)
compactify_kernel(BFHashDataStruct hd, const __grid_constant__ BFHashParams hp, const __grid_constant__ BFDepthCameraParams cp,
                  const int4* __restrict__ slotInfo, unsigned* ctrs, int set,
                  int4* __restrict__ work, const float2* __restrict__ tiles, int tilesX) {
    const unsigned highWater = ctrs[CTR_HIGH_WATER];
    const unsigned tid = blockIdx.x * blockDim.x + threadIdx.x;
    const int countIdx = set + SET_COUNT, workIdx = set + SET_WORK;       // zeroed by the launch before this one
    const unsigned stride = gridDim.x * blockDim.x;
    const unsigned lane = threadIdx.x & 31;
    for (unsigned base = tid - lane; base < highWater; base += stride) {
        const unsigned slot = base + lane;
        bool keep = false, probe = false;
        int4 info = make_int4(0, 0, 0, -1);
        if (slot < highWater) {
            info = __ldcg(&slotInfo[slot]);
            if (info.w >= 0) {
                I3 b = { info.x, info.y, info.z };
                keep = block_in_frustum(hp, cp, b);
                probe = keep && (tiles == nullptr || block_can_pass(hp, cp, tiles, tilesX, b));
            }
        }
        const unsigned ballot = __ballot_sync(0xffffffffu, keep);
        if (ballot) {
            const unsigned ballotW = __ballot_sync(0xffffffffu, probe);
            unsigned warpBase = 0, workBase = 0;
            if (lane == 0) {
                warpBase = atomicAdd(&ctrs[countIdx], __popc(ballot));
                if (work) {
                    if (ballotW) workBase = atomicAdd(&ctrs[workIdx], __popc(ballotW));
                    if (ballot != ballotW) atomicAdd(&ctrs[set + SET_CULLED], __popc(ballot) - __popc(ballotW));
                    atomicAdd(reinterpret_cast<unsigned long long*>(&ctrs[CTR_E_TOT_LO]), (unsigned long long)__popc(ballot));
                }
            }
            warpBase = __shfl_sync(0xffffffffu, warpBase, 0);
            workBase = __shfl_sync(0xffffffffu, workBase, 0);
            if (keep) {
                BFHashEntry e;
                e.pos[0] = info.x; e.pos[1] = info.y; e.pos[2] = info.z;
                e.ptr = (int)(slot * BF_SDF_BLOCK_VOXELS);
                e.offset = hd.d_hash[info.w].offset;
                hd.d_hashCompactified[warpBase + __popc(ballot & ((1u << lane) - 1u))] = e;
            }
            if (work && probe) work[workBase + __popc(ballotW & ((1u << lane) - 1u))] = make_int4(info.x, info.y, info.z, (int)(slot | (1u << 28)));
        }
    }
}

// legacy full-table variants (fillDecisionArrayKernel / compactifyHashKernel, .cu:268-320, and a
// table-scan rebuild of the slot table for hashes populated outside this library)
__global__ void fill_decision_kernel(BFHashDataStruct hd, const __grid_constant__ BFHashParams hp, const __grid_constant__ BFDepthCameraParams cp) {
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= hp.m_hashNumBuckets * BF_HASH_BUCKET_SIZE) return;
    int dec = 0;
    const BFHashEntry e = hd.d_hash[idx];
    if (e.ptr != BF_FREE_ENTRY) { I3 b = { e.pos[0], e.pos[1], e.pos[2] }; if (block_in_frustum(hp, cp, b)) dec = 1; }
    hd.d_hashDecision[idx] = dec;
}
__global__ void compactify_prefix_kernel(BFHashDataStruct hd, unsigned numEntries) {
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= numEntries) return;
    if (hd.d_hashDecision[idx] == 1) hd.d_hashCompactified[hd.d_hashDecisionPrefix[idx] - 1] = hd.d_hash[idx];
}
__global__ void rebuild_aux_kernel(BFHashDataStruct hd, unsigned numEntries, unsigned numSlots, int4* slotInfo, unsigned* ctrs) {
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= numEntries) return;
    const BFHashEntry e = hd.d_hash[idx];
    if (e.ptr == BF_FREE_ENTRY || e.ptr == BF_LOCK_ENTRY) return;
    const unsigned slot = (unsigned)e.ptr / BF_SDF_BLOCK_VOXELS;
    if (e.ptr < 0 || slot >= numSlots) return;
    slotInfo[slot] = make_int4(e.pos[0], e.pos[1], e.pos[2], (int)idx);
    atomicMax(&ctrs[CTR_HIGH_WATER], slot + 1u);
}

// ---- the integrate / de-integrate stencil (CUDASceneRepHashSDF.cu:420-521) --------------
// 128 threads per SDF block, 4 consecutive voxels (48 B) per thread.  Persistent grid: each CTA
// walks the compactified list with stride gridDim.x; the list length is read from device memory.
struct VoxelQuad { uint4 a, b, c; };
#ifndef BF_SPEC_BLOCKS
#define BF_SPEC_BLOCKS 24576u
#endif   // 4 voxels = 12 words: v0{a.x,a.y,a.z} v1{a.w,b.x,b.y} v2{b.z,b.w,c.x} v3{c.y,c.z,c.w}

__device__ __forceinline__ float clamp_color(float v) { return fmaxf(0.0f, fminf(v, 254.5f)); }

// The stencil is bound by the XU pipe (conversions, roundf and MUFU run at 1/8 rate), not by FMA/ALU issue, so the
// byte <-> float traffic of the colour update and the float -> pixel conversions are done with exact integer/FMA-pipe
// identities instead of cvt / frnd.  Each is value-identical to the plain expression in its comment for EVERY input.
// (float)b for b in [0, 255]
__device__ __forceinline__ float u8_to_float(unsigned b) { return __uint_as_float(0x4B000000u | b) - 8388608.0f; }
// (unsigned)clamp_color(roundf(r))   [roundf: half away from zero; cvt.rzi of a value in [0, 254.5]]
__device__ __forceinline__ unsigned round_clamp_u8(float r) {
    const float rc = fmaxf(-1.0f, fminf(r, 256.0f));           // roundf is monotone, so pre-clamping cannot change the clamped result; NaN -> 256 -> 254
    float t = (rc + 12582912.0f) - 12582912.0f;                // nearest integer, ties to even (|rc| <= 2^22)
    if (rc - t == 0.5f) t += 1.0f;                             // the ties roundf sends away from zero (the negative one, -0.5, clamps to 0 either way)
    const float v = clamp_color(t);                            // an integer in [0, 254] or 254.5
    return __float_as_uint(v + 8388608.0f) & 0xffu;            // 254.5 + 2^23 rounds to the even 254 = trunc
}
// idx = (unsigned)(int)t and the test idx < limit, t = screen coordinate + 0.5   [cvt.rzi.s32.f32: NaN -> 0, (-1, 0) -> 0]
#ifndef BF_PIXEL_F2I
#define BF_PIXEL_F2I 1      // 1: one cvt.rzi per coordinate (XU pipe); 0: the ~10-instruction FMA/ALU-pipe identity below
#endif
__device__ __forceinline__ bool pixel_index(float t, unsigned limit, float limitF, unsigned& idx) {
    if (BF_PIXEL_F2I || limit > (1u << 22)) { idx = (unsigned)(int)t; return idx < limit; }
    if (t <= -1.0f || t >= limitF) return false;               // NaN passes both tests, as the conversion gives 0
    const float c = fmaxf(t, 0.0f);                            // fmaxf(NaN, 0) = 0
    const float n = c + 8388608.0f;                            // 2^23 + rne(c)
    idx = (__float_as_uint(n) & 0x7FFFFFu) - ((n - 8388608.0f) > c ? 1u : 0u);   // floor(c)
    return true;
}

template <bool kDeIntegrate>
__device__ __forceinline__ void update_voxel(const BFHashParams& hp, float sdf, uchar4 cur, unsigned& wSdf, unsigned& wWeight, unsigned& wColor, int& liveDelta) {
    const float oldSdf = __uint_as_float(wSdf), oldW = __uint_as_float(wWeight);
    const float oc[3] = { u8_to_float(wColor & 0xff), u8_to_float((wColor >> 8) & 0xff), u8_to_float((wColor >> 16) & 0xff) };
    const float cc[3] = { u8_to_float(cur.x), u8_to_float(cur.y), u8_to_float(cur.z) };
    float nSdf, nW;
    unsigned nColor = 0;
    if (!kDeIntegrate) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float r = (oldW == 0) ? cc[k] : __fmaf_rn(cc[k], 0.2f, 0.8f * oc[k]);
            nColor |= round_clamp_u8(r) << (8 * k);
        }
        nColor |= 255u << 24;
        nSdf = __fmaf_rn(oldSdf, oldW, sdf) / (1.0f + oldW);
        nW = fminf((float)hp.m_integrationWeightMax, 1.0f + oldW);
    } else {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float r = __fmaf_rn(oc[k], oldW, -cc[k]) / (oldW - 1.0f);
            nColor |= round_clamp_u8(r) << (8 * k);
        }
        nColor |= 255u << 24;
        nSdf = __fmaf_rn(oldSdf, oldW, -sdf) / (oldW - 1.0f);
        nW = fmaxf(0.0f, oldW - 1.0f);
        if (nW <= 0.001f) { nSdf = 0.0f; nW = 0.0f; nColor = 0; }
    }
    liveDelta += (int)(nW > 0.0f) - (int)(oldW > 0.0f);
    wSdf = __float_as_uint(nSdf); wWeight = __float_as_uint(nW); wColor = nColor;
}

template <bool kDeIntegrate>
__global__ void __launch_bounds__(128)
integrate_kernel(BFHashDataStruct hd, const __grid_constant__ BFHashParams hp, const __grid_constant__ BFDepthCameraParams cp,
                 const float* __restrict__ depthImg, const uchar4* __restrict__ colorImg,
                 int useListCount, unsigned countOverride, unsigned* ctrs, int* __restrict__ live,
                 const int4* __restrict__ work, int set) {
    const unsigned* countPtr = useListCount ? ctrs + set + SET_COUNT : nullptr;
    const unsigned* workCountPtr = ctrs + set + SET_WORK;
    // `work` (from the library's own compactify): the list entries that survive the depth-range cull, 16 B each; without it
    // (reference-named stubs, whose list may come from anywhere) the kernel walks d_hashCompactified itself.
    const unsigned listCount = countPtr ? *countPtr : countOverride;
    const unsigned count = work ? *workCountPtr : listCount;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        if (countPtr) { hd.d_hashCompactifiedCounter[0] = (int)listCount; ctrs[CTR_E] = listCount; }
        if (!work) atomicAdd(reinterpret_cast<unsigned long long*>(&ctrs[CTR_E_TOT_LO]), (unsigned long long)listCount);
    }
    const unsigned t = threadIdx.x;
    const unsigned W = cp.m_imageWidth, H = cp.m_imageHeight;
    const float Wf = (float)W, Hf = (float)H;
    // local voxel coordinates of this thread's first voxel: i = 4t -> x = (4t)%8, y = (4t%64)/8, z = 4t/64
    const int lx = (int)((4 * t) & 7), ly = (int)(((4 * t) & 63) >> 3), lz = (int)((4 * t) >> 6);
    unsigned passed = 0;
    // Latency, not bandwidth, bounds this kernel while the list is short (a few thousand blocks: each warp walks a dependent
    // chain work item -> projection -> depth gather -> voxel load -> store).  Below BF_SPEC_BLOCKS list entries the voxel quad is
    // loaded up front, in the shadow of the projection arithmetic, whether or not one of its voxels will pass (<= 2x the voxel
    // read bytes, still far from the HBM roof at that size); above it only passing threads touch voxel memory, which is what
    // keeps the long-list regime at ~80 % of the roof.  The next work item is prefetched either way.
    const bool spec = count < BF_SPEC_BLOCKS;
    int4 wNext = make_int4(0, 0, 0, 0);
    if (work && blockIdx.x < count) wNext = __ldg(&work[blockIdx.x]);

    for (unsigned b = blockIdx.x; b < count; b += gridDim.x) {
        int bx, by, bz;
        unsigned ptr;
        if (work) {
            const int4 w = wNext;
            if (b + gridDim.x < count) wNext = __ldg(&work[b + gridDim.x]);
            bx = w.x; by = w.y; bz = w.z; ptr = ((unsigned)w.w & 0x0FFFFFFFu) * BF_SDF_BLOCK_VOXELS;
        } else {
            const BFHashEntry* ep = &hd.d_hashCompactified[b];
            bx = __ldg(&ep->pos[0]); by = __ldg(&ep->pos[1]); bz = __ldg(&ep->pos[2]);
            ptr = (unsigned)__ldg(&ep->ptr);
        }

        uint4* const vp = reinterpret_cast<uint4*>(hd.d_SDFBlocks + (size_t)ptr) + 3 * t;   // 48 B per thread, 16-B aligned
        VoxelQuad q;
        if (spec) { q.a = vp[0]; q.b = vp[1]; q.c = vp[2]; }
        float sdfv[4];
        uchar4 colv[4];
        unsigned mask = 0;
        int liveDelta = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const I3 pi = { bx * BF_SDF_BLOCK_SIZE + lx + k, by * BF_SDF_BLOCK_SIZE + ly, bz * BF_SDF_BLOCK_SIZE + lz };
            const F3 pf = xform(hp.m_rigidTransformInverse, voxel_to_world(hp, pi));
            const float sx = pf.x * cp.fx / pf.z + cp.mx;
            const float sy = pf.y * cp.fy / pf.z + cp.my;
            unsigned px, py;
            if (pixel_index(sx + 0.5f, W, Wf, px) && pixel_index(sy + 0.5f, H, Hf, py) && colorImg != nullptr) {
                const float depth = __ldg(&depthImg[py * W + px]);
                if (depth != -INFINITY && depth < hp.m_maxIntegrationDistance) {
                    float sdf = depth - pf.z;
                    const float trunc = truncation(hp, depth);
                    if (fabsf(sdf) < trunc) {
                        sdf = (sdf >= 0.0f) ? fminf(trunc, sdf) : fmaxf(-trunc, sdf);
                        sdfv[k] = sdf;
                        colv[k] = __ldg(&colorImg[py * W + px]);
                        mask |= 1u << k;
                    }
                }
            }
        }
        if (mask) {
            if (!spec) { q.a = vp[0]; q.b = vp[1]; q.c = vp[2]; }
            if (mask & 1u) update_voxel<kDeIntegrate>(hp, sdfv[0], colv[0], q.a.x, q.a.y, q.a.z, liveDelta);
            if (mask & 2u) update_voxel<kDeIntegrate>(hp, sdfv[1], colv[1], q.a.w, q.b.x, q.b.y, liveDelta);
            if (mask & 4u) update_voxel<kDeIntegrate>(hp, sdfv[2], colv[2], q.b.z, q.b.w, q.c.x, liveDelta);
            if (mask & 8u) update_voxel<kDeIntegrate>(hp, sdfv[3], colv[3], q.c.y, q.c.z, q.c.w, liveDelta);
            // write back only the 16-byte pieces that contain an updated voxel
            // words: v0 = a.xyz | v1 = a.w b.xy | v2 = b.zw c.x | v3 = c.yzw
            if (mask & 0x3u) vp[0] = q.a;
            if (mask & 0x6u) vp[1] = q.b;
            if (mask & 0xCu) vp[2] = q.c;
            passed += __popc(mask);
        }
        // live-voxel bookkeeping for O(E) garbage collection: one RED per warp, only when a weight crossed zero
        if (__any_sync(0xffffffffu, liveDelta != 0)) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) liveDelta += __shfl_xor_sync(0xffffffffu, liveDelta, o);
            if ((t & 31) == 0 && liveDelta != 0) atomicAdd(&live[ptr / BF_SDF_BLOCK_VOXELS], liveDelta);
        }
    }
    // U statistics: one 64-bit atomic per CTA
    passed = warp_sum_u(passed);
    __shared__ unsigned sPassed[4];
    if ((t & 31) == 0) sPassed[t >> 5] = passed;
    __syncthreads();
    if (t == 0) {
        const unsigned long long tot = (unsigned long long)sPassed[0] + sPassed[1] + sPassed[2] + sPassed[3];
        if (tot) { atomicAdd(reinterpret_cast<unsigned long long*>(&ctrs[set + SET_U_LO]), tot); atomicAdd(reinterpret_cast<unsigned long long*>(&ctrs[CTR_U_TOT_LO]), tot); }
    }
}

// ---- TMA-staged variant of the same stencil -------------------------------------------------------
// One producer warp streams whole 6144-byte voxel tiles into a 4-deep shared-memory ring with the bulk
// async-copy engine (cp.async.bulk, mbarrier completion); four consumer warps (128 threads, 4 voxels
// each) project / gather depth for block k+1 while tile k is in flight, read their 48 bytes from shared
// memory, and write only the dirty 16-byte pieces back to HBM.  Latency of the entry -> tile dependency
// is carried by the copy engine instead of by resident warps.
#define BF_TMA_STAGES 4
#define BF_TILE_BYTES (BF_SDF_BLOCK_VOXELS * 12)

struct GatherSet {           // what consumer thread t needs to update its 4 voxels of one block
    float pz[4];             // camera-space z of the voxel centres
    float depth[4];          // depth at the projected pixel (or -inf)
    uchar4 col[4];
    unsigned onscreen;       // bit k: voxel k projects inside the image
};

__device__ __forceinline__ void gather_block(const BFHashParams& hp, const BFDepthCameraParams& cp, const float* __restrict__ depthImg,
                                             const uchar4* __restrict__ colorImg, int bx, int by, int bz, int lx, int ly, int lz, GatherSet& g) {
    const unsigned W = cp.m_imageWidth, H = cp.m_imageHeight;
    g.onscreen = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const I3 pi = { bx * BF_SDF_BLOCK_SIZE + lx + k, by * BF_SDF_BLOCK_SIZE + ly, bz * BF_SDF_BLOCK_SIZE + lz };
        const F3 pf = xform(hp.m_rigidTransformInverse, voxel_to_world(hp, pi));
        const float sx = pf.x * cp.fx / pf.z + cp.mx;
        const float sy = pf.y * cp.fy / pf.z + cp.my;
        const unsigned px = (unsigned)(int)(sx + 0.5f), py = (unsigned)(int)(sy + 0.5f);
        g.pz[k] = pf.z;
        g.depth[k] = -INFINITY;
        g.col[k] = make_uchar4(0, 0, 0, 0);
        if (px < W && py < H) {
            g.onscreen |= 1u << k;
            g.depth[k] = __ldg(&depthImg[py * W + px]);
            g.col[k] = __ldg(&colorImg[py * W + px]);
        }
    }
}

template <bool kDeIntegrate>
__global__ void __launch_bounds__(160)
integrate_tma_kernel(BFHashDataStruct hd, const __grid_constant__ BFHashParams hp, const __grid_constant__ BFDepthCameraParams cp,
                     const float* __restrict__ depthImg, const uchar4* __restrict__ colorImg,
                     const unsigned* __restrict__ countPtr, unsigned countOverride, unsigned* ctrs, int* __restrict__ live, int set) {
    __shared__ __align__(128) uint4 sTile[BF_TMA_STAGES][BF_TILE_BYTES / 16];
    __shared__ __align__(8) unsigned long long sFull[BF_TMA_STAGES], sEmpty[BF_TMA_STAGES];
    __shared__ unsigned sPassed[4];

    const unsigned count = countPtr ? *countPtr : countOverride;
    if (blockIdx.x == 0 && threadIdx.x == 0 && countPtr) { hd.d_hashCompactifiedCounter[0] = (int)count; ctrs[CTR_E] = count; }
    const unsigned t = threadIdx.x;
    const unsigned nLocal = (count > blockIdx.x) ? (count - blockIdx.x - 1) / gridDim.x + 1 : 0;   // blocks this CTA owns
    if (nLocal == 0 || colorImg == nullptr) return;        // without colour nothing passes (.cu:441-448)

    if (t == 0) {
#pragma unroll
        for (int s = 0; s < BF_TMA_STAGES; ++s) { mbar_init(&sFull[s], 1); mbar_init(&sEmpty[s], 4); }
        mbar_fence_init();
    }
    __syncthreads();

    const BFHashEntry* __restrict__ list = hd.d_hashCompactified;
    if (t >= 128) {
        // ---------------- producer warp ----------------
        const unsigned lane = t - 128;
        unsigned ptrBatch = 0;
        for (unsigned k = 0; k < nLocal; ++k) {
            if ((k & 31) == 0) {                                // prefetch the next 32 block pointers, one per lane
                const unsigned kk = k + lane;
                ptrBatch = (kk < nLocal) ? (unsigned)__ldg(&list[blockIdx.x + (size_t)kk * gridDim.x].ptr) : 0u;
            }
            const unsigned ptr = __shfl_sync(0xffffffffu, ptrBatch, k & 31);
            const unsigned s = k % BF_TMA_STAGES, use = k / BF_TMA_STAGES;
            if (lane == 0) {
                if (use > 0) mbar_wait(&sEmpty[s], (use - 1) & 1);
                mbar_arrive_expect_tx(&sFull[s], BF_TILE_BYTES);
                bulk_g2s(&sTile[s][0], hd.d_SDFBlocks + (size_t)ptr, BF_TILE_BYTES, &sFull[s]);
            }
            __syncwarp();
        }
        return;
    }

    // ---------------- consumer warps ----------------
    const int lx = (int)((4 * t) & 7), ly = (int)(((4 * t) & 63) >> 3), lz = (int)((4 * t) >> 6);
    unsigned passed = 0;
    auto loadPos = [&](unsigned k, int& x, int& y, int& z, unsigned& p) {
        const BFHashEntry* e = &list[blockIdx.x + (size_t)k * gridDim.x];
        x = __ldg(&e->pos[0]); y = __ldg(&e->pos[1]); z = __ldg(&e->pos[2]); p = (unsigned)__ldg(&e->ptr);
    };
    int nx = 0, ny = 0, nz = 0; unsigned nptr = 0;              // entry of block k+1
    unsigned curPtr;
    GatherSet cur, nxt;
    {
        int x0, y0, z0;
        loadPos(0, x0, y0, z0, curPtr);
        if (nLocal > 1) loadPos(1, nx, ny, nz, nptr);
        gather_block(hp, cp, depthImg, colorImg, x0, y0, z0, lx, ly, lz, cur);
    }
    for (unsigned k = 0; k < nLocal; ++k) {
        // (1) start the gathers of block k+1 and the entry load of block k+2
        int fx = 0, fy = 0, fz = 0; unsigned fptr = 0;
        const bool haveNext = (k + 1 < nLocal);
        if (haveNext) gather_block(hp, cp, depthImg, colorImg, nx, ny, nz, lx, ly, lz, nxt);
        if (k + 2 < nLocal) loadPos(k + 2, fx, fy, fz, fptr);

        // (2) truncation test of block k (gathers issued one iteration ago)
        float sdfv[4];
        unsigned mask = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float depth = cur.depth[j];
            sdfv[j] = 0.0f;
            if (((cur.onscreen >> j) & 1u) && depth != -INFINITY && depth < hp.m_maxIntegrationDistance) {
                float sdf = depth - cur.pz[j];
                const float trunc = truncation(hp, depth);
                if (fabsf(sdf) < trunc) { sdfv[j] = (sdf >= 0.0f) ? fminf(trunc, sdf) : fmaxf(-trunc, sdf); mask |= 1u << j; }
            }
        }
        // (3) tile k: wait for the bulk copy, pull this thread's 48 bytes, release the stage
        const unsigned s = k % BF_TMA_STAGES;
        mbar_wait(&sFull[s], (k / BF_TMA_STAGES) & 1);
        VoxelQuad q;
        q.a = sTile[s][3 * t]; q.b = sTile[s][3 * t + 1]; q.c = sTile[s][3 * t + 2];
        __syncwarp();
        if ((t & 31) == 0) mbar_arrive(&sEmpty[s]);
        // (4) update + write back dirty 16-byte pieces
        int liveDelta = 0;
        if (mask) {
            uint4* vp = reinterpret_cast<uint4*>(hd.d_SDFBlocks + (size_t)curPtr) + 3 * t;
            if (mask & 1u) update_voxel<kDeIntegrate>(hp, sdfv[0], cur.col[0], q.a.x, q.a.y, q.a.z, liveDelta);
            if (mask & 2u) update_voxel<kDeIntegrate>(hp, sdfv[1], cur.col[1], q.a.w, q.b.x, q.b.y, liveDelta);
            if (mask & 4u) update_voxel<kDeIntegrate>(hp, sdfv[2], cur.col[2], q.b.z, q.b.w, q.c.x, liveDelta);
            if (mask & 8u) update_voxel<kDeIntegrate>(hp, sdfv[3], cur.col[3], q.c.y, q.c.z, q.c.w, liveDelta);
            if (mask & 0x3u) vp[0] = q.a;
            if (mask & 0x6u) vp[1] = q.b;
            if (mask & 0xCu) vp[2] = q.c;
            passed += __popc(mask);
        }
        if (__any_sync(0xffffffffu, liveDelta != 0)) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) liveDelta += __shfl_xor_sync(0xffffffffu, liveDelta, o);
            if ((t & 31) == 0 && liveDelta != 0) atomicAdd(&live[curPtr / BF_SDF_BLOCK_VOXELS], liveDelta);
        }
        cur = nxt; curPtr = nptr;
        nx = fx; ny = fy; nz = fz; nptr = fptr;
    }
    passed = warp_sum_u(passed);
    if ((t & 31) == 0) sPassed[t >> 5] = passed;
    asm volatile("bar.sync 1, 128;" ::: "memory");          // consumers only (the producer warp has left)
    if (t == 0) {
        const unsigned long long tot = (unsigned long long)sPassed[0] + sPassed[1] + sPassed[2] + sPassed[3];
        if (tot) { atomicAdd(reinterpret_cast<unsigned long long*>(&ctrs[set + SET_U_LO]), tot); atomicAdd(reinterpret_cast<unsigned long long*>(&ctrs[CTR_U_TOT_LO]), tot); }
    }
}

// ---- fused re-integration: deIntegrate(old pose) + integrate(new pose) of ONE frame in one pass -------------------
// The reference re-integrates a frame as two full passes (DepthSensing.cpp:867-895): compactify + stencil for the old pose,
// alloc + compactify + stencil for the new one.  Each voxel's result depends only on its own state, so running "alloc(new),
// then per voxel: de-integrate with the old pose, integrate with the new pose" in registers gives bit-identical voxels with one
// voxel read + one write instead of two of each, and 3 launches instead of 5.
__global__ void __launch_bounds__(256)
compactify_dual_kernel(BFHashDataStruct hd, const __grid_constant__ BFHashParams hpOld, const __grid_constant__ BFHashParams hpNew,
                       const __grid_constant__ BFDepthCameraParams cp, const int4* __restrict__ slotInfo, unsigned* ctrs, int set,
                       unsigned char* __restrict__ listFlags, int4* __restrict__ work, const float2* __restrict__ tiles, int tilesX) {
    const unsigned highWater = ctrs[CTR_HIGH_WATER];
    const unsigned tid = blockIdx.x * blockDim.x + threadIdx.x;
    const int countIdx = set + SET_COUNT, workIdx = set + SET_WORK;
    const unsigned stride = gridDim.x * blockDim.x;
    const unsigned lane = threadIdx.x & 31;
    for (unsigned base = tid - lane; base < highWater; base += stride) {
        const unsigned slot = base + lane;
        unsigned fl = 0, pr = 0;          // fl: in the old / new frustum (list membership); pr: poses whose stencil can touch the block
        int4 info = make_int4(0, 0, 0, -1);
        if (slot < highWater) {
            info = __ldcg(&slotInfo[slot]);
            if (info.w >= 0) {
                I3 b = { info.x, info.y, info.z };
                fl = (block_in_frustum(hpOld, cp, b) ? 1u : 0u) | (block_in_frustum(hpNew, cp, b) ? 2u : 0u);
                pr = fl;
                if (tiles) {
                    if ((pr & 1u) && !block_can_pass(hpOld, cp, tiles, tilesX, b)) pr &= ~1u;
                    if ((pr & 2u) && !block_can_pass(hpNew, cp, tiles, tilesX, b)) pr &= ~2u;
                }
            }
        }
        const unsigned ballot = __ballot_sync(0xffffffffu, fl != 0);
        if (ballot) {
            const unsigned ballotW = __ballot_sync(0xffffffffu, pr != 0);
            const unsigned nE = __popc(__ballot_sync(0xffffffffu, fl & 1u)) + __popc(__ballot_sync(0xffffffffu, fl & 2u));   // E of both passes
            const unsigned nP = __popc(__ballot_sync(0xffffffffu, pr & 1u)) + __popc(__ballot_sync(0xffffffffu, pr & 2u));
            unsigned warpBase = 0, workBase = 0;
            if (lane == 0) {
                warpBase = atomicAdd(&ctrs[countIdx], __popc(ballot));
                if (ballotW) workBase = atomicAdd(&ctrs[workIdx], __popc(ballotW));
                if (nE != nP) atomicAdd(&ctrs[set + SET_CULLED], nE - nP);
                atomicAdd(reinterpret_cast<unsigned long long*>(&ctrs[CTR_E_TOT_LO]), (unsigned long long)nE);
            }
            warpBase = __shfl_sync(0xffffffffu, warpBase, 0);
            workBase = __shfl_sync(0xffffffffu, workBase, 0);
            if (fl) {
                const unsigned k = warpBase + __popc(ballot & ((1u << lane) - 1u));
                BFHashEntry e;
                e.pos[0] = info.x; e.pos[1] = info.y; e.pos[2] = info.z;
                e.ptr = (int)(slot * BF_SDF_BLOCK_VOXELS);
                e.offset = hd.d_hash[info.w].offset;
                hd.d_hashCompactified[k] = e;
                listFlags[k] = (unsigned char)fl;
            }
            if (pr) work[workBase + __popc(ballotW & ((1u << lane) - 1u))] = make_int4(info.x, info.y, info.z, (int)(slot | (pr << 28)));
        }
    }
}

// ---- batch re-integration: ONE list for up to BF_MULTI_MAX_OPS (de-integrate old pose, integrate new pose) pairs ---------------------------
// The reference replays the pairs one after the other (FL/DepthSensing/DepthSensing.cpp:867-895), each with its own alloc / compactify /
// kernel launches.  Here the allocs of all pairs run first (each tags the blocks IT inserts with its op index), then this kernel builds
// one union list: per allocated block the 2-bit-per-op mask {in the old pose's frustum, in the new pose's frustum} for the ops that saw
// the block exist (op index >= the block's tag; a block inserted by op j's alloc does not exist for ops < j in the reference's order),
// and the multi-op stencil (tsdf_fast.cu) applies the ops to each voxel in order, in registers: one voxel read and write for the batch.
struct MultiFrusta { int nOps; float voxelSize; float truncScale, truncation; int tilesX; unsigned tilesPerOp; BFFloat4x4 inv[2 * BF_MULTI_MAX_OPS]; };     // inv[2k] = old pose of op k (inverse), inv[2k+1] = new
__global__ void __launch_bounds__(256)
compactify_multi_kernel(BFHashDataStruct hd, const __grid_constant__ MultiFrusta fr, const __grid_constant__ BFDepthCameraParams cp,
                        const int4* __restrict__ slotInfo, const unsigned* __restrict__ slotEpoch, unsigned batchId, unsigned* ctrs, int set,
                        unsigned char* __restrict__ listFlags, int4* __restrict__ workA, int4* __restrict__ workB, unsigned* __restrict__ maskA,
                        unsigned* __restrict__ maskB, unsigned workCap, const float2* __restrict__ tiles) {
    // tiles (optional): per op the 16x16-pixel {min, max} of the depths its frame offers (depth tiles, above).  A (block, op, pose) whose voxels provably
    // all fail the truncation test is dropped from the WORK mask -- its probes would all fail, the voxels stay as they are -- while list membership, the
    // GC flags and the E statistics keep the frustum mask: same results, fewer probes (in a scanned room more than half of the in-frustum blocks of an
    // old frame are beyond its integration distance, hidden behind nearer surfaces or at invalid depth).
    const unsigned highWater = ctrs[CTR_HIGH_WATER];
    const unsigned tid = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned stride = gridDim.x * blockDim.x;
    const unsigned lane = threadIdx.x & 31;
    for (unsigned base = tid - lane; base < highWater; base += stride) {
        const unsigned slot = base + lane;
        unsigned mask = 0, wmask = 0;
        int4 info = make_int4(0, 0, 0, -1);
        if (slot < highWater) {
            info = __ldcg(&slotInfo[slot]);
            if (info.w >= 0) {
                const I3 b = { info.x, info.y, info.z };
                const unsigned e = __ldcg(&slotEpoch[slot]);
                const int first = ((e >> 8) == batchId) ? (int)(e & 0xffu) : 0;
                for (int k = first; k < fr.nOps; ++k) {
                    const float2* const tk = tiles ? tiles + (size_t)k * fr.tilesPerOp : nullptr;
                    if (block_in_frustum_m(fr.voxelSize, fr.inv[2 * k], cp, b)) {
                        mask |= 1u << (2 * k);
                        if (!tk || block_can_pass_m(fr.truncScale, fr.truncation, fr.voxelSize, fr.inv[2 * k], cp, tk, fr.tilesX, b)) wmask |= 1u << (2 * k);
                    }
                    if (block_in_frustum_m(fr.voxelSize, fr.inv[2 * k + 1], cp, b)) {
                        mask |= 2u << (2 * k);
                        if (!tk || block_can_pass_m(fr.truncScale, fr.truncation, fr.voxelSize, fr.inv[2 * k + 1], cp, tk, fr.tilesX, b)) wmask |= 2u << (2 * k);
                    }
                }
            }
        }
        const unsigned ballot = __ballot_sync(0xffffffffu, mask != 0);
        if (ballot) {
            // E of the batch = sum over ops of the blocks in either frustum = what the per-op lists would have held
            const unsigned bits = (unsigned)__popc(wmask);
            unsigned nE = (unsigned)__popc(mask), nW = bits;
            for (int o = 16; o > 0; o >>= 1) { nE += __shfl_xor_sync(0xffffffffu, nE, o); nW += __shfl_xor_sync(0xffffffffu, nW, o); }
            // Work order: a block's cost grows with the number of (op, pose) probes it takes -- up to 2 nOps of them, ~60 k cycles for a CTA at
            // 20.  Items go to four buckets by cost quartile and the stencil deals the costliest bucket first (longest-processing-time-first), so
            // the kernel ends on cheap blocks and its tail is a quartile-0 block, not a 20-probe one.
            const unsigned n2 = 2u * (unsigned)fr.nOps;
            const int q = (wmask == 0) ? -1 : (4u * bits > 3u * n2 ? 3 : (2u * bits > n2 ? 2 : (4u * bits > n2 ? 1 : 0)));
            const unsigned b3 = __ballot_sync(0xffffffffu, q == 3), b2 = __ballot_sync(0xffffffffu, q == 2), b1 = __ballot_sync(0xffffffffu, q == 1), b0 = __ballot_sync(0xffffffffu, q == 0);
            unsigned warpBase = 0, base3 = 0, base2 = 0, base1 = 0, base0 = 0;
            if (lane == 0) {
                warpBase = atomicAdd(&ctrs[set + SET_COUNT], __popc(ballot));
                if (b3) base3 = atomicAdd(&ctrs[set + SET_WORK], __popc(b3));
                if (b2) base2 = atomicAdd(&ctrs[set + SET_CULLED], __popc(b2));      // the batch has no cull: the slot counts quartile-2 items
                if (b1) base1 = atomicAdd(&ctrs[set + SET_Q1], __popc(b1));
                if (b0) base0 = atomicAdd(&ctrs[set + SET_Q0], __popc(b0));
                atomicAdd(reinterpret_cast<unsigned long long*>(&ctrs[CTR_E_TOT_LO]), (unsigned long long)nE);
                atomicAdd(reinterpret_cast<unsigned long long*>(&ctrs[CTR_EB_TOT_LO]), (unsigned long long)nE);
                if (nE != nW) atomicAdd(&ctrs[CTR_CULLB], nE - nW);
            }
            warpBase = __shfl_sync(0xffffffffu, warpBase, 0);
            base3 = __shfl_sync(0xffffffffu, base3, 0); base2 = __shfl_sync(0xffffffffu, base2, 0);
            base1 = __shfl_sync(0xffffffffu, base1, 0); base0 = __shfl_sync(0xffffffffu, base0, 0);
            if (mask) {
                const unsigned below = (1u << lane) - 1u;
                const unsigned k = warpBase + __popc(ballot & below);
                BFHashEntry en;
                en.pos[0] = info.x; en.pos[1] = info.y; en.pos[2] = info.z;
                en.ptr = (int)(slot * BF_SDF_BLOCK_VOXELS);
                en.offset = hd.d_hash[info.w].offset;
                hd.d_hashCompactified[k] = en;
                // the reference's GC walks the list of the LAST integrate (DepthSensing.cpp:901): bit 1 = in the last op's new-pose frustum
                listFlags[k] = (unsigned char)(((mask >> (2 * (fr.nOps - 1))) & 2u) | 1u);
                if (q >= 0) {
                    int4* const wArr = (q >= 2) ? workA : workB;
                    unsigned* const mArr = (q >= 2) ? maskA : maskB;
                    const unsigned w = (q == 3) ? base3 + __popc(b3 & below) : (q == 2) ? (workCap - 1u) - (base2 + __popc(b2 & below))
                                     : (q == 1) ? base1 + __popc(b1 & below) : (workCap - 1u) - (base0 + __popc(b0 & below));
                    wArr[w] = make_int4(info.x, info.y, info.z, (int)slot);
                    mArr[w] = wmask;
                }
            }
        }
    }
}

// truncation test of one voxel against one pose; returns true and the clamped sdf / colour when it passes (.cu:433-463)
__device__ __forceinline__ bool probe_voxel(const BFHashParams& hp, const BFDepthCameraParams& cp, const float* __restrict__ depthImg,
                                            const uchar4* __restrict__ colorImg, F3 world, float Wf, float Hf, float& sdfOut, uchar4& colOut) {
    const F3 pf = xform(hp.m_rigidTransformInverse, world);
    const float sx = pf.x * cp.fx / pf.z + cp.mx;
    const float sy = pf.y * cp.fy / pf.z + cp.my;
    unsigned px, py;
    if (!(pixel_index(sx + 0.5f, cp.m_imageWidth, Wf, px) && pixel_index(sy + 0.5f, cp.m_imageHeight, Hf, py))) return false;
    const float depth = __ldg(&depthImg[py * cp.m_imageWidth + px]);
    if (!(depth != -INFINITY && depth < hp.m_maxIntegrationDistance)) return false;
    float sdf = depth - pf.z;
    const float trunc = truncation(hp, depth);
    if (!(fabsf(sdf) < trunc)) return false;
    sdfOut = (sdf >= 0.0f) ? fminf(trunc, sdf) : fmaxf(-trunc, sdf);
    colOut = __ldg(&colorImg[py * cp.m_imageWidth + px]);
    return true;
}

#ifndef BF_REINT_MINBLOCKS
#define BF_REINT_MINBLOCKS 8
#endif
__global__ void __launch_bounds__(128, BF_REINT_MINBLOCKS)
reintegrate_kernel(BFHashDataStruct hd, const __grid_constant__ BFHashParams hpOld, const __grid_constant__ BFHashParams hpNew,
                   const __grid_constant__ BFDepthCameraParams cp, const float* __restrict__ depthImg, const uchar4* __restrict__ colorImg,
                   const int4* __restrict__ work, int set, unsigned* ctrs, int* __restrict__ live) {
    const unsigned* countPtr = ctrs + set + SET_COUNT;
    const unsigned count = ctrs[set + SET_WORK];
    const unsigned t = threadIdx.x;
    const int lx = (int)((4 * t) & 7), ly = (int)(((4 * t) & 63) >> 3), lz = (int)((4 * t) >> 6);
    unsigned passed = 0;
    const bool spec = count < BF_SPEC_BLOCKS;           // see integrate_kernel
    const float Wf = (float)cp.m_imageWidth, Hf = (float)cp.m_imageHeight;
    int4 wNext = make_int4(0, 0, 0, 0);
    if (blockIdx.x < count) wNext = __ldg(&work[blockIdx.x]);
    for (unsigned b = blockIdx.x; b < count; b += gridDim.x) {
        const int4 w = wNext;
        if (b + gridDim.x < count) wNext = __ldg(&work[b + gridDim.x]);
        const int bx = w.x, by = w.y, bz = w.z;
        const unsigned ptr = ((unsigned)w.w & 0x0FFFFFFFu) * BF_SDF_BLOCK_VOXELS;
        const unsigned fl = (unsigned)w.w >> 28;        // bit0: the old pose can touch this block, bit1: the new pose can
        uint4* const vp = reinterpret_cast<uint4*>(hd.d_SDFBlocks + (size_t)ptr) + 3 * t;
        VoxelQuad q;
        if (spec) { q.a = vp[0]; q.b = vp[1]; q.c = vp[2]; }
        float sdfD[4], sdfI[4];
        uchar4 colD[4], colI[4];
        unsigned maskD = 0, maskI = 0;
        int liveDelta = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const I3 pi = { bx * BF_SDF_BLOCK_SIZE + lx + k, by * BF_SDF_BLOCK_SIZE + ly, bz * BF_SDF_BLOCK_SIZE + lz };
            const F3 world = voxel_to_world(hpNew, pi);       // both poses of one scene share the voxel size (checked by the host)
            if ((fl & 1u) && probe_voxel(hpOld, cp, depthImg, colorImg, world, Wf, Hf, sdfD[k], colD[k])) maskD |= 1u << k;
            if ((fl & 2u) && probe_voxel(hpNew, cp, depthImg, colorImg, world, Wf, Hf, sdfI[k], colI[k])) maskI |= 1u << k;
        }
        const unsigned mask = maskD | maskI;
        if (mask) {
            if (!spec) { q.a = vp[0]; q.b = vp[1]; q.c = vp[2]; }
            if (maskD & 1u) update_voxel<true>(hpOld, sdfD[0], colD[0], q.a.x, q.a.y, q.a.z, liveDelta);
            if (maskI & 1u) update_voxel<false>(hpNew, sdfI[0], colI[0], q.a.x, q.a.y, q.a.z, liveDelta);
            if (maskD & 2u) update_voxel<true>(hpOld, sdfD[1], colD[1], q.a.w, q.b.x, q.b.y, liveDelta);
            if (maskI & 2u) update_voxel<false>(hpNew, sdfI[1], colI[1], q.a.w, q.b.x, q.b.y, liveDelta);
            if (maskD & 4u) update_voxel<true>(hpOld, sdfD[2], colD[2], q.b.z, q.b.w, q.c.x, liveDelta);
            if (maskI & 4u) update_voxel<false>(hpNew, sdfI[2], colI[2], q.b.z, q.b.w, q.c.x, liveDelta);
            if (maskD & 8u) update_voxel<true>(hpOld, sdfD[3], colD[3], q.c.y, q.c.z, q.c.w, liveDelta);
            if (maskI & 8u) update_voxel<false>(hpNew, sdfI[3], colI[3], q.c.y, q.c.z, q.c.w, liveDelta);
            if (mask & 0x3u) vp[0] = q.a;
            if (mask & 0x6u) vp[1] = q.b;
            if (mask & 0xCu) vp[2] = q.c;
            passed += __popc(maskD) + __popc(maskI);
        }
        if (__any_sync(0xffffffffu, liveDelta != 0)) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) liveDelta += __shfl_xor_sync(0xffffffffu, liveDelta, o);
            if ((t & 31) == 0 && liveDelta != 0) atomicAdd(&live[ptr / BF_SDF_BLOCK_VOXELS], liveDelta);
        }
    }
    passed = warp_sum_u(passed);
    __shared__ unsigned sPassed[4];
    if ((t & 31) == 0) sPassed[t >> 5] = passed;
    __syncthreads();
    if (t == 0) {
        const unsigned long long tot = (unsigned long long)sPassed[0] + sPassed[1] + sPassed[2] + sPassed[3];
        if (tot) { atomicAdd(reinterpret_cast<unsigned long long*>(&ctrs[set + SET_U_LO]), tot); atomicAdd(reinterpret_cast<unsigned long long*>(&ctrs[CTR_U_TOT_LO]), tot); }
        if (blockIdx.x == 0) { const unsigned listCount = *countPtr; hd.d_hashCompactifiedCounter[0] = (int)listCount; ctrs[CTR_E] = listCount; }
    }
}

// starveVoxelsKernel (.cu:554-563)
__global__ void starve_kernel(BFHashDataStruct hd) {
    const BFHashEntry& e = hd.d_hashCompactified[blockIdx.x];
    BFVoxel* v = &hd.d_SDFBlocks[(size_t)(unsigned)e.ptr + threadIdx.x];
    int w = (int)v->weight;
    w = max(0, w - 1);
    v->weight = (float)w;
}

// ---- garbage collection ------------------------------------------------------------------
// identify (.cu:584-631): d_hashDecision[i] = (uint(max weight of block i) == 0)
__device__ __forceinline__ unsigned block_max_weight_u(const BFVoxel* base, unsigned t, float* sWarp) {
    const uint4* vp = reinterpret_cast<const uint4*>(base) + 3 * t;
    const uint4 a = vp[0], b = vp[1], c = vp[2];
    float m = fmaxf(fmaxf(__uint_as_float(a.y), __uint_as_float(b.x)), fmaxf(__uint_as_float(b.w), __uint_as_float(c.z)));
    m = warp_max(m);
    if ((t & 31) == 0) sWarp[t >> 5] = m;
    __syncthreads();
    const float bm = fmaxf(fmaxf(sWarp[0], sWarp[1]), fmaxf(sWarp[2], sWarp[3]));
    __syncthreads();
    return (unsigned)bm;        // cvt.rzi.u32.f32: the reference reduces through a uint array (Q13)
}

__global__ void __launch_bounds__(128)
gc_identify_kernel(BFHashDataStruct hd, unsigned count) {
    __shared__ float sWarp[4];
    for (unsigned b = blockIdx.x; b < count; b += gridDim.x) {
        const unsigned ptr = (unsigned)hd.d_hashCompactified[b].ptr;
        const unsigned mw = block_max_weight_u(hd.d_SDFBlocks + (size_t)ptr, threadIdx.x, sWarp);
        if (threadIdx.x == 0) hd.d_hashDecision[b] = (mw == 0) ? 1 : 0;
    }
}

// deleteHashEntryElement (VoxelUtilHashSDF.h:739-826) under the home bucket's spin lock.
__device__ bool delete_entry(const BFHashDataStruct& hd, const BFHashParams& hp, int4* slotInfo, I3 p) {
    const unsigned h = hash_pos(hp.m_hashNumBuckets, p);
    const unsigned hpz = h * BF_HASH_BUCKET_SIZE;
    const unsigned last = hpz + BF_HASH_BUCKET_SIZE - 1;
    const unsigned total = BF_HASH_BUCKET_SIZE * hp.m_hashNumBuckets;
    int* mutexH = &hd.d_hashBucketMutex[h];
    unsigned backoff = 32;
    while (!try_lock(mutexH)) { __nanosleep(backoff); if (backoff < 1024) backoff <<= 1; }
    __threadfence();
    bool ok = false;
    BFHashEntry freeE; freeE.pos[0] = freeE.pos[1] = freeE.pos[2] = 0; freeE.ptr = BF_FREE_ENTRY; freeE.offset = 0;
    for (unsigned j = 0; j < BF_HASH_BUCKET_SIZE && !ok; ++j) {
        const unsigned i = hpz + j;
        const BFHashEntry c = load_entry_cg(&hd.d_hash[i]);
        if (entry_matches_v(c, p)) {
            const unsigned slot = (unsigned)c.ptr / BF_SDF_BLOCK_VOXELS;
            const unsigned addr = atomicAdd(hd.d_heapCounter, 1u);            // appendHeap :541-546
            hd.d_heap[addr + 1] = slot;
            slotInfo[slot] = make_int4(0, 0, 0, -1);
            if (c.offset != 0) {
                const unsigned next = (i + c.offset) % total;
                const BFHashEntry n = load_entry_cg(&hd.d_hash[next]);
                hd.d_hash[i] = n;
                if (n.ptr >= 0) slotInfo[(unsigned)n.ptr / BF_SDF_BLOCK_VOXELS].w = (int)i;   // the moved entry changed index
                hd.d_hash[next] = freeE;
            } else {
                hd.d_hash[i] = freeE;
            }
            ok = true;
        }
    }
    if (!ok) {
        BFHashEntry c = load_entry_cg(&hd.d_hash[last]);
        unsigned prev = last;
        unsigned i = (last + c.offset) % total;
        for (unsigned it = 0; it < hp.m_hashMaxCollisionLinkedListSize; ++it) {
            c = load_entry_cg(&hd.d_hash[i]);
            if (entry_matches_v(c, p)) {
                const unsigned slot = (unsigned)c.ptr / BF_SDF_BLOCK_VOXELS;
                const unsigned addr = atomicAdd(hd.d_heapCounter, 1u);
                hd.d_heap[addr + 1] = slot;
                slotInfo[slot] = make_int4(0, 0, 0, -1);
                hd.d_hash[i] = freeE;
                hd.d_hash[prev].offset = c.offset;
                ok = true;
                break;
            }
            if (c.offset == 0) break;
            prev = i;
            i = (last + c.offset) % total;
        }
    }
    unlock(mutexH);
    return ok;
}

// free (.cu:648-668) given d_hashDecision
__global__ void __launch_bounds__(128)
gc_free_kernel(BFHashDataStruct hd, const __grid_constant__ BFHashParams hp, unsigned count, int4* slotInfo, unsigned* ctrs) {
    __shared__ int sOk;
    for (unsigned b = blockIdx.x; b < count; b += gridDim.x) {
        if (hd.d_hashDecision[b] == 0) continue;           // uniform per CTA
        const BFHashEntry e = hd.d_hashCompactified[b];
        if (threadIdx.x == 0) {
            I3 p = { e.pos[0], e.pos[1], e.pos[2] };
            sOk = delete_entry(hd, hp, slotInfo, p) ? 1 : 0;
            if (sOk) atomicAdd(&ctrs[CTR_FREED], 1u);
        }
        __syncthreads();
        if (sOk) {
            uint4* vp = reinterpret_cast<uint4*>(hd.d_SDFBlocks + (size_t)(unsigned)e.ptr) + 3 * threadIdx.x;
            const uint4 z = make_uint4(0, 0, 0, 0);
            vp[0] = z; vp[1] = z; vp[2] = z;
        }
        __syncthreads();
    }
}

// fused identify + free: what bfTsdfGarbageCollect launches (one pass over the voxels)
__global__ void __launch_bounds__(128)
gc_fused_kernel(BFHashDataStruct hd, const __grid_constant__ BFHashParams hp, const unsigned* __restrict__ countPtr, int4* slotInfo, unsigned* ctrs) {
    __shared__ float sWarp[4];
    __shared__ int sOk;
    const unsigned count = *countPtr;
    for (unsigned b = blockIdx.x; b < count; b += gridDim.x) {
        const BFHashEntry e = hd.d_hashCompactified[b];
        const unsigned mw = block_max_weight_u(hd.d_SDFBlocks + (size_t)(unsigned)e.ptr, threadIdx.x, sWarp);
        if (threadIdx.x == 0) hd.d_hashDecision[b] = (mw == 0) ? 1 : 0;
        if (mw != 0) continue;                               // uniform per CTA
        if (threadIdx.x == 0) {
            I3 p = { e.pos[0], e.pos[1], e.pos[2] };
            sOk = delete_entry(hd, hp, slotInfo, p) ? 1 : 0;
            if (sOk) atomicAdd(&ctrs[CTR_FREED], 1u);
        }
        __syncthreads();
        if (sOk) {
            uint4* vp = reinterpret_cast<uint4*>(hd.d_SDFBlocks + (size_t)(unsigned)e.ptr) + 3 * threadIdx.x;
            const uint4 z = make_uint4(0, 0, 0, 0);
            vp[0] = z; vp[1] = z; vp[2] = z;
        }
        __syncthreads();
    }
}

// O(E) garbage collection from the live-voxel counters the integrate kernels maintain: a block is garbage iff
// no voxel has weight > 0 (weights are whole numbers, so this equals the reference's uint(max weight) == 0).
// Freed blocks are already all-zero (de-integration clears a voxel when its weight reaches 0, .cu:509-513).
__global__ void __launch_bounds__(256)
gc_live_kernel(BFHashDataStruct hd, const __grid_constant__ BFHashParams hp, const unsigned* __restrict__ countPtr,
               int4* slotInfo, unsigned* ctrs, const int* __restrict__ live, const unsigned char* __restrict__ listFlags) {
    const unsigned count = *countPtr;
    for (unsigned b = blockIdx.x * blockDim.x + threadIdx.x; b < count; b += gridDim.x * blockDim.x) {
        // after a fused re-integration the list is the union of two frusta; the reference's GC walks the list of the LAST
        // integrate only (DepthSensing.cpp:901), i.e. the entries inside the new pose's frustum
        if (listFlags && !(listFlags[b] & 2u)) { hd.d_hashDecision[b] = 0; continue; }
        const BFHashEntry e = hd.d_hashCompactified[b];
        const int dead = (__ldcg(&live[(unsigned)e.ptr / BF_SDF_BLOCK_VOXELS]) <= 0) ? 1 : 0;
        hd.d_hashDecision[b] = dead;
        if (dead) {
            I3 p = { e.pos[0], e.pos[1], e.pos[2] };
            if (delete_entry(hd, hp, slotInfo, p)) atomicAdd(&ctrs[CTR_FREED], 1u);
        }
    }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
static void free_aux(TsdfAux& a) {
    cudaFree(a.slotInfo); cudaFree(a.ctrs); cudaFree(a.live); cudaFree(a.listFlags); cudaFree(a.work2[0]); cudaFree(a.work2[1]); cudaFree(a.tiles); cudaFree(a.tilesMulti);
    cudaFree(a.slotEpoch); cudaFree(a.workMask); cudaFree(a.workMask2);
    if (a.lane) cudaStreamDestroy(a.lane);
    if (a.evFork) cudaEventDestroy(a.evFork);
    for (int k = 0; k < 2; ++k) { if (a.evList[k]) cudaEventDestroy(a.evList[k]); if (a.evStencil[k]) cudaEventDestroy(a.evStencil[k]); }
}

static int get_aux(const BFHashDataStruct* hd, const BFHashParams* hp, TsdfAux** out, bool create, bool adopt) {
    std::lock_guard<std::mutex> lk(g_auxMutex);
    auto it = g_aux.find(hd->d_hash);
    const void* owner[3] = { hd->d_SDFBlocks, hd->d_heap, hd->d_hashCompactified };
    const bool same = it != g_aux.end() && memcmp(it->second.owner, owner, sizeof(owner)) == 0;
    if (same && (hp == nullptr || it->second.numSlots == hp->m_numSDFBlocks)) { *out = &it->second; return 0; }
    if (!create || hp == nullptr) { *out = nullptr; return (int)cudaErrorInvalidValue; }
    if (it != g_aux.end()) { free_aux(it->second); g_aux.erase(it); }
    TsdfAux a;
    a.numSlots = hp->m_numSDFBlocks;
    memcpy(a.owner, owner, sizeof(owner));
    BF_CHECK(cudaMalloc(&a.slotInfo, sizeof(int4) * (size_t)a.numSlots));
    BF_CHECK(cudaMalloc(&a.ctrs, sizeof(unsigned) * CTR_NUM));
    BF_CHECK(cudaMalloc(&a.live, sizeof(int) * (size_t)a.numSlots));
    BF_CHECK(cudaMalloc(&a.listFlags, (size_t)a.numSlots));
    if (a.numSlots < (1u << 28)) {                                   // slot index shares a word with 4 flag bits
        BF_CHECK(cudaMalloc(&a.work2[0], sizeof(int4) * (size_t)a.numSlots));
        BF_CHECK(cudaMalloc(&a.work2[1], sizeof(int4) * (size_t)a.numSlots));
        a.work = a.work2[0];
    }
    BF_CHECK(cudaMemsetAsync(a.live, 0, sizeof(int) * (size_t)a.numSlots, g_stream));
    a.liveValid = !adopt;           // an adopted table has unknown weights: fall back to the scanning GC
    BF_CHECK(cudaMemsetAsync(a.ctrs, 0, sizeof(unsigned) * CTR_NUM, g_stream));
    BF_CHECK(cudaMemsetAsync(a.slotInfo, 0xff, sizeof(int4) * (size_t)a.numSlots, g_stream));
    // adopt whatever the table already holds (a hash populated elsewhere, or a fresh reset)
    const unsigned numEntries = hp->m_hashNumBuckets * BF_HASH_BUCKET_SIZE;
    if (adopt) {
        rebuild_aux_kernel<<<(numEntries + 255) / 256, 256, 0, g_stream>>>(*hd, numEntries, a.numSlots, a.slotInfo, a.ctrs);
        BF_CHECK(cudaGetLastError());
    }
    auto res = g_aux.emplace(hd->d_hash, a);
    *out = &res.first->second;
    return 0;
}

static inline int grid_for(unsigned work, int perSm) {
    int g = num_sms() * perSm;
    if (work > 0 && (unsigned)g > work) g = (int)work;
    return g < 1 ? 1 : g;
}

static int do_reset(BFHashDataStruct* hd, const BFHashParams* hp) {
    TsdfAux* aux;
    { // (re)create aux without the table-adopting scan mattering: reset overwrites everything
        int rc = get_aux(hd, hp, &aux, true, /*adopt=*/false);
        if (rc) return rc;
    }
    aux->parity = 0;
    aux->liveValid = true;
    reset_kernel<<<num_sms() * 8, 256, 0, g_stream>>>(*hd, hp->m_numSDFBlocks, hp->m_hashNumBuckets, aux->slotInfo, aux->ctrs, aux->live);
    BF_CHECK(cudaGetLastError());
    return 0;
}

static inline int tiles_x(const BFDepthCameraParams* cp) { return (int)((cp->m_imageWidth + BF_TILE - 1) / BF_TILE); }
static inline int tiles_y(const BFDepthCameraParams* cp) { return (int)((cp->m_imageHeight + BF_TILE - 1) / BF_TILE); }
static int ensure_tiles(TsdfAux* aux, const BFDepthCameraParams* cp) {
    const unsigned need = (unsigned)(tiles_x(cp) * tiles_y(cp));
    if (need <= aux->tilesCap) return 0;
    if (aux->tiles) { BF_CHECK(cudaStreamSynchronize(g_stream)); BF_CHECK(cudaFree(aux->tiles)); aux->tiles = nullptr; aux->tilesCap = 0; }
    BF_CHECK(cudaMalloc(&aux->tiles, sizeof(float2) * need));
    aux->tilesCap = need;
    return 0;
}
// Per-block depth-range cull: OFF by default.  The cull test lengthens the compactify kernels' critical path on every call while the
// blocks it can prove dead (mostly: looking at
// depths beyond the integration distance) were cheap for the stencil anyway (their probes exit at the depth test).
// bfTsdfSetBlockCull(1) or BF_TSDF_CULL=1 switches it on; results are identical either way (tests/test_tsdf_gpu.py).
static int g_lanes = -1;             // two-lane op replay (bfTsdfRunOps), see "two lanes" below
// Stencil arithmetic: BF_TSDF_ARITH_FAST (default; tsdf_fast.cu: tolerance contract, what the reference's --use_fast_math build is to
// its IEEE build) or BF_TSDF_ARITH_EXACT (this file's kernels: bit-identical to the reference's IEEE build and to oracle/tsdf_oracle.c).
static int g_arith = -1;
static bool arith_fast() {
    if (g_arith < 0) { const char* e = getenv("BF_TSDF_ARITH"); g_arith = (e && (e[0] == 'e' || e[0] == '0')) ? BF_TSDF_ARITH_EXACT : BF_TSDF_ARITH_FAST; }
    return g_arith == BF_TSDF_ARITH_FAST;
}
static int g_cull = -1;
static bool cull_enabled() {
    if (g_cull < 0) { const char* e = getenv("BF_TSDF_CULL"); g_cull = (e && e[0] == '1') ? 1 : 0; }
    return g_cull == 1;
}

// ---- two lanes ---------------------------------------------------------------------------------------------------
// Front lane = the caller's stream (g_stream): alloc, depth tiles, compactify, GC.  Back lane = aux->lane: the stencils.
// Inside a bfTsdfRunOps bracket the stencil of op k runs on the back lane while alloc + compactify of op k+1 run on the
// front lane: they touch disjoint state (hash / heap / slot table / list k+1  vs  work list k / voxels), both are
// issue-bound at roughly half an SM's capacity, and the stencil is launched with a grid that leaves room for the other.
// Ordering: stencil k waits for list k (evList); the first front-lane launch of op k+2 waits for stencil k (evStencil),
// because it recycles stencil k's counter set and work list; stencils are serial on the back lane (consecutive stencils
// may touch the same voxels); GC and the end of the bracket join both lanes.  Outside a bracket everything is launched on
// the caller's stream, as before.
static inline int set_of(unsigned parity) { return parity ? CTR_SET1 : CTR_SET0; }
static inline cudaStream_t back_lane(const TsdfAux* aux) { return aux->pipeOpen ? aux->lane : g_stream; }
// called before the first front-lane launch of an op whose list will use `parity`
static int front_acquire_set(TsdfAux* aux, unsigned parity) {
    if (aux->pipeOpen && aux->stencilPending[parity]) { BF_CHECK(cudaStreamWaitEvent(g_stream, aux->evStencil[parity], 0)); aux->stencilPending[parity] = false; }
    return 0;
}
static int join_lanes(TsdfAux* aux) {
    if (!aux->pipeOpen) return 0;
    for (unsigned p = 0; p < 2; ++p)
        if (aux->stencilPending[p]) { BF_CHECK(cudaStreamWaitEvent(g_stream, aux->evStencil[p], 0)); aux->stencilPending[p] = false; }
    return 0;
}

// withTiles: also leave the depth-tile min/max for the stencil's block cull (library sequences only; the reference-named
// allocCUDA stub has no say over what is integrated afterwards).  zeroParity >= 0: the launch also zeroes that counter set
// (the one the following compactify fills).
static int do_alloc(BFHashDataStruct* hd, const BFHashParams* hp, const float* depth, const BFDepthCameraParams* cp, TsdfAux* aux, bool withTiles, int zeroParity,
                    AllocEpoch ep = AllocEpoch{nullptr, 0u}, float2* tilesOut = nullptr) {
    dim3 block(BF_TILE, BF_TILE);
    dim3 grid((cp->m_imageWidth + block.x - 1) / block.x, (cp->m_imageHeight + block.y - 1) / block.y);
    if (withTiles) { int rc = ensure_tiles(aux, cp); if (rc) return rc; }
    if (zeroParity >= 0) { int rc = front_acquire_set(aux, (unsigned)zeroParity); if (rc) return rc; }
    ++g_launchCount;
    alloc_kernel<<<grid, block, 0, g_stream>>>(*hd, *hp, *cp, depth, aux->slotInfo, aux->ctrs, tilesOut ? tilesOut : (withTiles ? aux->tiles : nullptr),
                                               zeroParity >= 0 ? set_of((unsigned)zeroParity) : -1, ep);
    BF_CHECK(cudaGetLastError());
    return 0;
}
static int do_depth_tiles(const BFHashParams* hp, const float* depth, const BFDepthCameraParams* cp, TsdfAux* aux) {
    int rc = ensure_tiles(aux, cp); if (rc) return rc;
    dim3 block(BF_TILE, BF_TILE);
    dim3 grid((cp->m_imageWidth + block.x - 1) / block.x, (cp->m_imageHeight + block.y - 1) / block.y);
    ++g_launchCount;
    depth_tiles_kernel<<<grid, block, 0, g_stream>>>(*hp, *cp, depth, aux->tiles);
    BF_CHECK(cudaGetLastError());
    return 0;
}

// useWork: also emit the stencil work list (library sequences); useTiles: aux->tiles describe the depth image the following
// stencil will read -> entries no voxel of which can pass are left out of the work list.  setZeroed: the preceding launch
// (alloc_kernel) already zeroed the counter set of the new parity.
static int do_compactify(BFHashDataStruct* hd, const BFHashParams* hp, const BFDepthCameraParams* cp, TsdfAux* aux, bool useWork, bool useTiles, bool setZeroed) {
    aux->parity ^= 1u;
    aux->lastListDual = false;
    const int set = set_of(aux->parity);
    if (!setZeroed) {
        int rc = front_acquire_set(aux, aux->parity); if (rc) return rc;
        BF_CHECK(cudaMemsetAsync(aux->ctrs + set, 0, SET_WORDS * sizeof(unsigned), g_stream));
    }
    ++g_launchCount;
    compactify_kernel<<<grid_for((hp->m_numSDFBlocks + 255) / 256, 4), 256, 0, g_stream>>>(*hd, *hp, *cp, aux->slotInfo, aux->ctrs, set,
                                                                                            useWork ? aux->work2[aux->parity] : nullptr, (useWork && useTiles) ? aux->tiles : nullptr, tiles_x(cp));
    BF_CHECK(cudaGetLastError());
    if (aux->pipeOpen) BF_CHECK(cudaEventRecord(aux->evList[aux->parity], g_stream));
    return 0;
}

static inline const unsigned* live_count_ptr(const TsdfAux* aux) { return aux->ctrs + set_of(aux->parity) + SET_COUNT; }

// before / after a stencil launch on the back lane
static int stencil_begin(TsdfAux* aux) {
    if (aux->pipeOpen) BF_CHECK(cudaStreamWaitEvent(aux->lane, aux->evList[aux->parity], 0));
    return 0;
}
static int stencil_end(TsdfAux* aux) {
    if (aux->pipeOpen) { BF_CHECK(cudaEventRecord(aux->evStencil[aux->parity], aux->lane)); aux->stencilPending[aux->parity] = true; }
    return 0;
}
// Stencil CTAs per SM inside a two-lane bracket.  Capping the stencil at 4-6 CTAs per SM so that alloc CTAs can co-reside slows the
// stencil by more than the overlap returns; uncapped, the front lane fills the SMs the stencil's last wave frees.
static int stencil_per_sm() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("BF_TSDF_LANE_STENCIL_PER_SM"); v = e ? atoi(e) : 16; if (v < 1) v = 1; if (v > 16) v = 16; }
    return v;
}

static int do_integrate(BFHashDataStruct* hd, const BFHashParams* hp, const BFDepthCameraData* dd, const BFDepthCameraParams* cp,
                        TsdfAux* aux, bool deIntegrate, bool useListCount, unsigned countOverride) {
    const unsigned upper = useListCount ? hp->m_numSDFBlocks : countOverride;
    if (upper == 0) return 0;
    const uchar4* color = reinterpret_cast<const uchar4*>(dd->d_colorData);
    static int variant = -1;        // BF_TSDF_INTEGRATE=tma selects the TMA-staged variant (measured slower, see DESIGN.md)
    if (variant < 0) { const char* e = getenv("BF_TSDF_INTEGRATE"); variant = (e && e[0] == 't') ? 1 : 0; }
    const cudaStream_t sb = back_lane(aux);
    int rc = stencil_begin(aux); if (rc) return rc;
    const bool timeIt = g_profile && g_evUsed < kMaxProfiledLaunches;
    if (g_profile) { ++g_profLaunches; ++g_profFrames; }
    if (timeIt) {
        if (g_evStart.size() <= g_evUsed) { cudaEvent_t a, b; BF_CHECK(cudaEventCreate(&a)); BF_CHECK(cudaEventCreate(&b)); g_evStart.push_back(a); g_evStop.push_back(b); }
        if (g_evIsBatch.size() > g_evUsed) g_evIsBatch[g_evUsed] = 0;
        BF_CHECK(cudaEventRecord(g_evStart[g_evUsed], sb));
    }
    ++g_launchCount;
    const int set = set_of(aux->parity);
    if (arith_fast() && variant == 0) {
        const int4* work = useListCount ? aux->work2[aux->parity] : nullptr;
        rc = launch_integrate_fast(hd, hp, cp, dd->d_depthData, dd->d_colorData, deIntegrate, useListCount, countOverride, aux->ctrs, aux->live, work, set,
                                   grid_for(upper, fast_stencil_ctas_per_sm(false)), sb);
        if (rc) return rc;
    } else if (variant == 0) {
        const int grid = grid_for(upper, aux->pipeOpen ? stencil_per_sm() : 16);
        const int4* work = useListCount ? aux->work2[aux->parity] : nullptr;        // the stubs' list (countOverride) has no work list
        if (deIntegrate) integrate_kernel<true><<<grid, 128, 0, sb>>>(*hd, *hp, *cp, dd->d_depthData, color, useListCount ? 1 : 0, countOverride, aux->ctrs, aux->live, work, set);
        else             integrate_kernel<false><<<grid, 128, 0, sb>>>(*hd, *hp, *cp, dd->d_depthData, color, useListCount ? 1 : 0, countOverride, aux->ctrs, aux->live, work, set);
    } else {
        const int grid = grid_for(upper, 6);
        const unsigned* countPtr = useListCount ? live_count_ptr(aux) : nullptr;
        if (deIntegrate) integrate_tma_kernel<true><<<grid, 160, 0, sb>>>(*hd, *hp, *cp, dd->d_depthData, color, countPtr, countOverride, aux->ctrs, aux->live, set);
        else             integrate_tma_kernel<false><<<grid, 160, 0, sb>>>(*hd, *hp, *cp, dd->d_depthData, color, countPtr, countOverride, aux->ctrs, aux->live, set);
    }
    BF_CHECK(cudaGetLastError());
    if (timeIt) { BF_CHECK(cudaEventRecord(g_evStop[g_evUsed], sb)); ++g_evUsed; }
    return stencil_end(aux);
}

// bracket of a two-lane replay (used by bfTsdfRunOps, host_api.cu)
int tsdf_lanes_begin(const BFHashDataStruct* hd, const BFHashParams* hp) {
    if (g_lanes < 0) {               // BF_TSDF_LANES=0 / bfTsdfSetLanes(0): everything on the caller's stream
        const char* e = getenv("BF_TSDF_LANES"); g_lanes = (e && e[0] == '0') ? 0 : 1;
    }
    const char* v = getenv("BF_TSDF_INTEGRATE");
    if (!g_lanes || (v && v[0] == 't')) return 0;      // the TMA variant walks d_hashCompactified, which the front lane rewrites
    TsdfAux* aux;
    int rc = get_aux(hd, hp, &aux, true);
    if (rc) return rc;
    if (aux->pipeOpen) return 0;
    if (!aux->lane) {
        int lo = 0, hi = 0;
        BF_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        BF_CHECK(cudaStreamCreateWithPriority(&aux->lane, cudaStreamNonBlocking, hi));     // the stencil is the critical path
        BF_CHECK(cudaEventCreateWithFlags(&aux->evFork, cudaEventDisableTiming));
        for (int k = 0; k < 2; ++k) {
            BF_CHECK(cudaEventCreateWithFlags(&aux->evList[k], cudaEventDisableTiming));
            BF_CHECK(cudaEventCreateWithFlags(&aux->evStencil[k], cudaEventDisableTiming));
        }
    }
    BF_CHECK(cudaEventRecord(aux->evFork, g_stream));          // the back lane starts after everything already queued by the caller
    BF_CHECK(cudaStreamWaitEvent(aux->lane, aux->evFork, 0));
    aux->stencilPending[0] = aux->stencilPending[1] = false;
    aux->pipeOpen = true;
    return 0;
}
int tsdf_lanes_end(const BFHashDataStruct* hd) {
    TsdfAux* aux;
    if (get_aux(hd, nullptr, &aux, false) != 0 || !aux->pipeOpen) return 0;
    int rc = join_lanes(aux);          // the caller's stream continues after the last stencil
    aux->pipeOpen = false;
    return rc;
}

}  // namespace bf

using namespace bf;

// ==========================================================================================
// extension API
// ==========================================================================================
BF_API void bfSetStream(void* s) { g_stream = (cudaStream_t)s; }
BF_API void* bfGetStream(void) { return (void*)g_stream; }
BF_API const char* bfGetLastErrorString(void) { return t_lastError.c_str(); }

BF_API size_t bfTsdfAuxBytes(const BFHashParams* hp) { return (3 * sizeof(int4) + sizeof(int) + 1) * (size_t)hp->m_numSDFBlocks + sizeof(unsigned) * CTR_NUM; }

BF_API int bfTsdfReset(BFHashDataStruct* hd, const BFHashParams* hp) { return do_reset(hd, hp); }

BF_API int bfTsdfSetLanes(int enable) { const int prev = g_lanes; g_lanes = enable ? 1 : 0; return prev < 0 ? 1 : prev; }
BF_API int bfTsdfSetArithmetic(int mode) { const int prev = arith_fast() ? BF_TSDF_ARITH_FAST : BF_TSDF_ARITH_EXACT; g_arith = (mode == BF_TSDF_ARITH_EXACT) ? BF_TSDF_ARITH_EXACT : BF_TSDF_ARITH_FAST; return prev; }
BF_API int bfTsdfSetBlockCull(int enable) { const int prev = cull_enabled() ? 1 : 0; g_cull = enable ? 1 : 0; return prev; }

BF_API int bfTsdfIntegrateFrame(BFHashDataStruct* hd, const BFHashParams* hp, const BFDepthCameraData* dd,
                                const BFDepthCameraParams* cp, int deIntegrate) {
    TsdfAux* aux;
    int rc = get_aux(hd, hp, &aux, true);
    if (rc) return rc;
    const bool cull = cull_enabled() && dd->d_colorData != nullptr;
    if (!deIntegrate) { rc = do_alloc(hd, hp, dd->d_depthData, cp, aux, cull, (int)(aux->parity ^ 1u)); if (rc) return rc; }
    else if (cull)    { rc = front_acquire_set(aux, aux->parity ^ 1u); if (rc) return rc; rc = do_depth_tiles(hp, dd->d_depthData, cp, aux); if (rc) return rc; }
    rc = do_compactify(hd, hp, cp, aux, true, cull, /*setZeroed=*/!deIntegrate); if (rc) return rc;
    return do_integrate(hd, hp, dd, cp, aux, deIntegrate != 0, true, 0);
}

// CUDASceneRepHashSDF::deIntegrate(old pose) immediately followed by ::integrate(new pose) of the SAME frame
// (the body of the reference's re-integration loop, DepthSensing.cpp:867-895) as one fused pass; voxels bit-identical.
BF_API int bfTsdfReintegrateFrame(BFHashDataStruct* hd, const BFHashParams* hpOld, const BFHashParams* hpNew,
                                  const BFDepthCameraData* dd, const BFDepthCameraParams* cp) {
    TsdfAux* aux;
    int rc = get_aux(hd, hpNew, &aux, true);
    if (rc) return rc;
    if (dd->d_colorData == nullptr) return do_alloc(hd, hpNew, dd->d_depthData, cp, aux, false, -1);     // no colour: neither pass updates a voxel
    if (aux->work == nullptr || hpOld->m_virtualVoxelSize != hpNew->m_virtualVoxelSize) return (int)cudaErrorNotSupported;
    // the tiles are built with the new pose's parameters; both passes may use them only if they accept the same depths
    const bool cull = cull_enabled() && hpOld->m_maxIntegrationDistance == hpNew->m_maxIntegrationDistance;
    rc = do_alloc(hd, hpNew, dd->d_depthData, cp, aux, cull, (int)(aux->parity ^ 1u)); if (rc) return rc;
    aux->parity ^= 1u;
    aux->lastListDual = true;
    const int set = set_of(aux->parity);
    ++g_launchCount;
    compactify_dual_kernel<<<grid_for((hpNew->m_numSDFBlocks + 255) / 256, 4), 256, 0, g_stream>>>(*hd, *hpOld, *hpNew, *cp, aux->slotInfo, aux->ctrs, set, aux->listFlags,
                                                                                                    aux->work2[aux->parity], cull ? aux->tiles : nullptr, tiles_x(cp));
    BF_CHECK(cudaGetLastError());
    if (aux->pipeOpen) BF_CHECK(cudaEventRecord(aux->evList[aux->parity], g_stream));
    const cudaStream_t sb = back_lane(aux);
    rc = stencil_begin(aux); if (rc) return rc;
    const bool timeIt = g_profile && g_evUsed < kMaxProfiledLaunches;
    if (g_profile) { ++g_profLaunches; ++g_profFrames; }
    if (timeIt) {
        if (g_evStart.size() <= g_evUsed) { cudaEvent_t a, b; BF_CHECK(cudaEventCreate(&a)); BF_CHECK(cudaEventCreate(&b)); g_evStart.push_back(a); g_evStop.push_back(b); }
        if (g_evIsBatch.size() > g_evUsed) g_evIsBatch[g_evUsed] = 0;
        BF_CHECK(cudaEventRecord(g_evStart[g_evUsed], sb));
    }
    ++g_launchCount;
    if (arith_fast()) {
        rc = launch_reintegrate_fast(hd, hpOld, hpNew, cp, dd->d_depthData, dd->d_colorData, aux->work2[aux->parity], set, aux->ctrs, aux->live,
                                     grid_for(hpNew->m_numSDFBlocks, fast_stencil_ctas_per_sm(true)), sb);
        if (rc) return rc;
    } else {
        reintegrate_kernel<<<grid_for(hpNew->m_numSDFBlocks, aux->pipeOpen ? stencil_per_sm() : 16), 128, 0, sb>>>(
            *hd, *hpOld, *hpNew, *cp, dd->d_depthData, reinterpret_cast<const uchar4*>(dd->d_colorData), aux->work2[aux->parity], set, aux->ctrs, aux->live);
    }
    BF_CHECK(cudaGetLastError());
    if (timeIt) { BF_CHECK(cudaEventRecord(g_evStop[g_evUsed], sb)); ++g_evUsed; }
    return stencil_end(aux);
}

// Up to BF_MULTI_MAX_OPS re-integration pairs {deIntegrate(frame f, old pose); integrate(frame f, new pose)} -- the loop body of
// FL/DepthSensing/DepthSensing.cpp:867-895, replayed as: n alloc launches (op-tagged inserts), ONE union list, ONE stencil pass in which
// every voxel of the list is read once, taken through the n pairs in order in registers, and written once.  Fast arithmetic only (the
// bit-exact kernels keep the one-pair-per-pass path); voxels are bit-identical to the one-pair-per-pass fast path (same probe expression,
// same per-voxel op order, blocks invisible to the ops that precede their insertion).  hp: pose-independent parameters; on return it holds
// the last new pose, as after the reference's last integrate.
static int g_batching = -1;
static bool batching_on() {
    if (g_batching < 0) { const char* e = getenv("BF_TSDF_BATCH"); g_batching = (e && e[0] == '0') ? 0 : 1; }
    return g_batching == 1;
}
BF_API int bfTsdfSetBatching(int enable) { const int prev = batching_on() ? 1 : 0; g_batching = enable ? 1 : 0; return prev; }
// Batch cull (compactify_multi_kernel): on by default; BF_TSDF_BATCH_CULL=0 or bfTsdfSetBatchCull(0) switches it off.  Results are identical either way.
static int g_batchCull = -1;
static bool batch_cull_on() {
    if (g_batchCull < 0) { const char* e = getenv("BF_TSDF_BATCH_CULL"); g_batchCull = (e && e[0] == '0') ? 0 : 1; }
    return g_batchCull == 1;
}
BF_API int bfTsdfSetBatchCull(int enable) { const int prev = batch_cull_on() ? 1 : 0; g_batchCull = enable ? 1 : 0; return prev; }

BF_API int bfTsdfReintegrateBatch(BFHashDataStruct* hd, BFHashParams* hp, const BFDepthCameraParams* cp, const BFTsdfReintegration* pairs, int numPairs,
                                  const float* const* d_depthFrames, const uint8_t* const* d_colorFrames) {
    if (numPairs < 1 || numPairs > BF_MULTI_MAX_OPS || !d_colorFrames) return (int)cudaErrorInvalidValue;
    TsdfAux* aux;
    int rc = get_aux(hd, hp, &aux, true);
    if (rc) return rc;
    if (aux->work == nullptr) return (int)cudaErrorNotSupported;
    if (!aux->slotEpoch) {
        BF_CHECK(cudaMalloc(&aux->slotEpoch, sizeof(unsigned) * (size_t)aux->numSlots));
        BF_CHECK(cudaMalloc(&aux->workMask, sizeof(unsigned) * (size_t)aux->numSlots));
        BF_CHECK(cudaMalloc(&aux->workMask2, sizeof(unsigned) * (size_t)aux->numSlots));
        BF_CHECK(cudaMemsetAsync(aux->slotEpoch, 0, sizeof(unsigned) * (size_t)aux->numSlots, g_stream));
        aux->batchId = 0;
    }
    rc = join_lanes(aux); if (rc) return rc;            // the batch runs on the caller's stream, after every stencil in flight
    aux->batchId = (aux->batchId + 1u) & 0x00FFFFFFu;
    if (aux->batchId == 0) { BF_CHECK(cudaMemsetAsync(aux->slotEpoch, 0, sizeof(unsigned) * (size_t)aux->numSlots, g_stream)); aux->batchId = 1; }
    static BFHashParams hpOld[BF_MULTI_MAX_OPS], hpNew[BF_MULTI_MAX_OPS];
    static MultiFrusta fr;
    BFMultiOpDesc desc[BF_MULTI_MAX_OPS];
    fr.nOps = numPairs; fr.voxelSize = hp->m_virtualVoxelSize; fr.truncScale = hp->m_truncScale; fr.truncation = hp->m_truncation;
    fr.tilesX = tiles_x(cp); fr.tilesPerOp = (unsigned)(tiles_x(cp) * tiles_y(cp));
    const bool cull = batch_cull_on();
    if (cull && aux->tilesMultiPer < fr.tilesPerOp) {
        if (aux->tilesMulti) { BF_CHECK(cudaStreamSynchronize(g_stream)); BF_CHECK(cudaFree(aux->tilesMulti)); aux->tilesMulti = nullptr; aux->tilesMultiPer = 0; }
        BF_CHECK(cudaMalloc(&aux->tilesMulti, sizeof(float2) * (size_t)fr.tilesPerOp * BF_MULTI_MAX_OPS));
        aux->tilesMultiPer = fr.tilesPerOp;
    }
    const unsigned newParity = aux->parity ^ 1u;
    for (int k = 0; k < numPairs; ++k) {
        hpOld[k] = *hp; hpNew[k] = *hp;
        for (int e = 0; e < 16; ++e) { hpOld[k].m_rigidTransform.m[e] = pairs[k].oldPose[e]; hpNew[k].m_rigidTransform.m[e] = pairs[k].newPose[e]; }
        mat4_inverse_ref(pairs[k].oldPose, hpOld[k].m_rigidTransformInverse.m);          // as setLastRigidTransform forms it on the reference's host
        mat4_inverse_ref(pairs[k].newPose, hpNew[k].m_rigidTransformInverse.m);
        fr.inv[2 * k] = hpOld[k].m_rigidTransformInverse; fr.inv[2 * k + 1] = hpNew[k].m_rigidTransformInverse;
        desc[k].hpOld = &hpOld[k]; desc[k].hpNew = &hpNew[k];
        desc[k].depth = d_depthFrames[pairs[k].frame]; desc[k].color = d_colorFrames[pairs[k].frame];
        if (!desc[k].color || !desc[k].depth) return (int)cudaErrorInvalidValue;
        // the first alloc launch also zeroes the counter set the list is about to use
        rc = do_alloc(hd, &hpNew[k], desc[k].depth, cp, aux, false, k == 0 ? (int)newParity : -1, AllocEpoch{aux->slotEpoch, (aux->batchId << 8) | (unsigned)k},
                      cull ? aux->tilesMulti + (size_t)k * fr.tilesPerOp : nullptr);
        if (rc) return rc;
    }
    aux->parity = newParity;
    aux->lastListDual = true;
    const int set = set_of(aux->parity);
    ++g_launchCount;
    compactify_multi_kernel<<<grid_for((hp->m_numSDFBlocks + 255) / 256, 4), 256, 0, g_stream>>>(*hd, fr, *cp, aux->slotInfo, aux->slotEpoch, aux->batchId, aux->ctrs, set,
                                                                                                 aux->listFlags, aux->work2[aux->parity], aux->work2[aux->parity ^ 1u], aux->workMask, aux->workMask2, aux->numSlots,
                                                                                                 cull ? aux->tilesMulti : nullptr);
    BF_CHECK(cudaGetLastError());
    const bool timeIt = g_profile && g_evUsed < kMaxProfiledLaunches;
    if (g_profile) { ++g_profLaunches; g_profFrames += (unsigned long long)numPairs; ++g_profBatchLaunches; g_profBatchFrames += (unsigned long long)numPairs; }
    if (timeIt) {
        if (g_evStart.size() <= g_evUsed) { cudaEvent_t a, b; BF_CHECK(cudaEventCreate(&a)); BF_CHECK(cudaEventCreate(&b)); g_evStart.push_back(a); g_evStop.push_back(b); }
        if (g_evIsBatch.size() <= g_evUsed) g_evIsBatch.resize(g_evUsed + 1, 0);
        g_evIsBatch[g_evUsed] = 1;
        if (!g_ktime) BF_CHECK(cudaMalloc(&g_ktime, sizeof(unsigned long long) * 2 * kMaxProfiledLaunches));
        BF_CHECK(cudaMemsetAsync(g_ktime + 2 * g_evUsed, 0xff, sizeof(unsigned long long), g_stream));
        BF_CHECK(cudaMemsetAsync(g_ktime + 2 * g_evUsed + 1, 0, sizeof(unsigned long long), g_stream));
        BF_CHECK(cudaEventRecord(g_evStart[g_evUsed], g_stream));
    }
    ++g_launchCount;
    rc = launch_reintegrate_multi_fast(hd, desc, numPairs, cp, aux->work2[aux->parity], aux->work2[aux->parity ^ 1u], aux->workMask, aux->workMask2, aux->numSlots, set, aux->ctrs, aux->live,
                                       grid_for(hp->m_numSDFBlocks, fast_stencil_ctas_per_sm(true)), g_stream, timeIt ? g_ktime + 2 * g_evUsed : nullptr);
    if (rc) return rc;
    if (timeIt) { BF_CHECK(cudaEventRecord(g_evStop[g_evUsed], g_stream)); ++g_evUsed; }
    *hp = hpNew[numPairs - 1];
    return 0;
}
namespace bf { int tsdf_batching_usable() { return (batching_on() && arith_fast()) ? 1 : 0; } }

BF_API int bfTsdfGarbageCollect(BFHashDataStruct* hd, const BFHashParams* hp) {
    TsdfAux* aux;
    int rc = get_aux(hd, hp, &aux, true);
    if (rc) return rc;
    rc = join_lanes(aux); if (rc) return rc;          // GC edits the hash, the heap and the slot table: no stencil may be in flight
    ++g_launchCount;
    if (aux->liveValid) gc_live_kernel<<<grid_for((hp->m_numSDFBlocks + 255) / 256, 2), 256, 0, g_stream>>>(*hd, *hp, live_count_ptr(aux), aux->slotInfo, aux->ctrs, aux->live, aux->lastListDual ? aux->listFlags : nullptr);
    else                gc_fused_kernel<<<grid_for(hp->m_numSDFBlocks, 16), 128, 0, g_stream>>>(*hd, *hp, live_count_ptr(aux), aux->slotInfo, aux->ctrs);
    BF_CHECK(cudaGetLastError());
    return 0;
}

BF_API int bfTsdfGetHeapFreeCount(const BFHashDataStruct* hd, unsigned int* out) {
    unsigned c = 0;
    BF_CHECK(cudaMemcpyAsync(&c, hd->d_heapCounter, sizeof(unsigned), cudaMemcpyDeviceToHost, g_stream));
    BF_CHECK(cudaStreamSynchronize(g_stream));
    *out = c + 1;     // CUDASceneRepHashSDF.h:168-172
    return 0;
}

BF_API int bfTsdfGetNumOccupiedBlocks(const BFHashDataStruct* hd, unsigned int* out) {
    int c = 0;
    BF_CHECK(cudaMemcpyAsync(&c, hd->d_hashCompactifiedCounter, sizeof(int), cudaMemcpyDeviceToHost, g_stream));
    BF_CHECK(cudaStreamSynchronize(g_stream));
    *out = (unsigned)c;
    return 0;
}

BF_API int bfTsdfGetLastFrameStats(const BFHashDataStruct* hd, unsigned long long out[4]) {
    TsdfAux* aux;
    int rc = get_aux(hd, nullptr, &aux, false);
    if (rc) return rc;
    unsigned c[CTR_NUM];
    BF_CHECK(cudaMemcpyAsync(c, aux->ctrs, sizeof(c), cudaMemcpyDeviceToHost, g_stream));
    BF_CHECK(cudaStreamSynchronize(g_stream));
    out[0] = c[CTR_E];
    const int set = set_of(aux->parity);
    out[1] = c[set + SET_CULLED];
    out[2] = ((unsigned long long)c[set + SET_U_HI] << 32) | c[set + SET_U_LO];
    out[3] = (unsigned long long)c[CTR_HEAP_FAIL] + c[CTR_DROPPED];
    return 0;
}

BF_API unsigned long long bfGetLaunchCount(void) { return g_launchCount; }

BF_API int bfTsdfSetProfiling(int enable) {
    g_profile = enable != 0;
    g_evUsed = 0; g_profLaunches = 0; g_profFrames = 0; g_profBatchLaunches = 0; g_profBatchFrames = 0;
    std::fill(g_evIsBatch.begin(), g_evIsBatch.end(), 0);
    std::lock_guard<std::mutex> lk(g_auxMutex);
    for (auto& kv : g_aux) {                    // restart the U / E sums
        BF_CHECK(cudaMemsetAsync(kv.second.ctrs + CTR_U_TOT_LO, 0, 4 * sizeof(unsigned), g_stream));
        BF_CHECK(cudaMemsetAsync(kv.second.ctrs + CTR_UB_TOT_LO, 0, 4 * sizeof(unsigned), g_stream));
        BF_CHECK(cudaMemsetAsync(kv.second.ctrs + CTR_CULLB, 0, sizeof(unsigned), g_stream));
    }
    return 0;
}

// out[0] = stencil launches since bfTsdfSetProfiling(1), out[1] = launches that were timed, out[2] = their summed duration in ns,
// out[3] = sum of U (voxels rewritten) over ALL launches since the last reset, out[4] = sum of E (blocks visited).  Synchronises.
// out[0..5] as bfTsdfGetProfile (all stencil launches); out[8] batch launches, out[9] of them timed, out[10] their summed duration (ns),
// out[11] U of the batch launches, out[12] their E, out[13] frame images they read
BF_API int bfTsdfGetProfileEx(const BFHashDataStruct* hd, unsigned long long out[16]) {
    TsdfAux* aux;
    int rc = get_aux(hd, nullptr, &aux, false);
    if (rc) return rc;
    BF_CHECK(cudaStreamSynchronize(g_stream));
    double ms = 0.0, msB = 0.0; unsigned long long nB = 0;
    for (size_t i = 0; i < g_evUsed; ++i) {
        float t = 0.0f; BF_CHECK(cudaEventElapsedTime(&t, g_evStart[i], g_evStop[i])); ms += t;
        if (i < g_evIsBatch.size() && g_evIsBatch[i]) { msB += t; ++nB; }
    }
    unsigned c[CTR_NUM];
    BF_CHECK(cudaMemcpy(c, aux->ctrs, sizeof(c), cudaMemcpyDeviceToHost));
    for (int k = 0; k < 16; ++k) out[k] = 0;
    out[0] = g_profLaunches; out[1] = g_evUsed; out[2] = (unsigned long long)(ms * 1e6);
    out[3] = ((unsigned long long)c[CTR_U_TOT_HI] << 32) | c[CTR_U_TOT_LO];
    out[4] = ((unsigned long long)c[CTR_E_TOT_HI] << 32) | c[CTR_E_TOT_LO];
    out[5] = g_profFrames;          // frame images read by those launches (a batch launch reads one per re-integration pair)
    out[8] = g_profBatchLaunches; out[9] = nB; out[10] = (unsigned long long)(msB * 1e6);
    out[11] = ((unsigned long long)c[CTR_UB_TOT_HI] << 32) | c[CTR_UB_TOT_LO];
    out[12] = ((unsigned long long)c[CTR_EB_TOT_HI] << 32) | c[CTR_EB_TOT_LO];
    out[13] = g_profBatchFrames;
    out[15] = c[CTR_CULLB];         // (block, op, pose) probes the batch cull removed (E counts them: they are in-frustum)
    if (g_ktime && g_evUsed) {          // out[14]: the batch launches' duration by the in-kernel %globaltimer brackets (first CTA start -> last CTA end), ns
        std::vector<unsigned long long> kt(2 * g_evUsed);
        BF_CHECK(cudaMemcpy(kt.data(), g_ktime, sizeof(unsigned long long) * 2 * g_evUsed, cudaMemcpyDeviceToHost));
        unsigned long long sum = 0;
        for (size_t i = 0; i < g_evUsed; ++i) if (i < g_evIsBatch.size() && g_evIsBatch[i] && kt[2 * i + 1] > kt[2 * i]) sum += kt[2 * i + 1] - kt[2 * i];
        out[14] = sum;
    }
    // restart accumulation
    BF_CHECK(cudaMemsetAsync(aux->ctrs + CTR_U_TOT_LO, 0, 4 * sizeof(unsigned), g_stream));
    BF_CHECK(cudaMemsetAsync(aux->ctrs + CTR_UB_TOT_LO, 0, 4 * sizeof(unsigned), g_stream));
    BF_CHECK(cudaMemsetAsync(aux->ctrs + CTR_CULLB, 0, sizeof(unsigned), g_stream));
    g_evUsed = 0; g_profLaunches = 0; g_profFrames = 0; g_profBatchLaunches = 0; g_profBatchFrames = 0;
    std::fill(g_evIsBatch.begin(), g_evIsBatch.end(), 0);
    return 0;
}
BF_API int bfTsdfGetProfile(const BFHashDataStruct* hd, unsigned long long out[8]) {
    unsigned long long o[16];
    const int rc = bfTsdfGetProfileEx(hd, o);
    if (rc) return rc;
    for (int k = 0; k < 8; ++k) out[k] = o[k];
    return 0;
}

BF_API int bfTsdfReleaseAux(const BFHashDataStruct* hd) {
    std::lock_guard<std::mutex> lk(g_auxMutex);
    auto it = g_aux.find(hd->d_hash);
    if (it == g_aux.end()) return 0;
    free_aux(it->second);
    g_aux.erase(it);
    return 0;
}

// ==========================================================================================
// reference-named stubs
// ==========================================================================================
BF_API void updateConstantHashParams(const BFHashParams* hp) { g_hashParams = *hp; }
BF_API void updateConstantDepthCameraParams(const BFDepthCameraParams* p) { g_camParams = *p; }
BF_API void bindInputDepthColorTextures(const BFDepthCameraData* dd, unsigned int width, unsigned int height) {
    g_bound = *dd; (void)width; (void)height;      // the image size travels in DepthCameraParams (the reference only needs it for its texture binding)
}

BF_API void resetCUDA(BFHashDataStruct* hd, const BFHashParams* hp) { BF_SAFE(do_reset(hd, hp)); }

BF_API void resetHashBucketMutexCUDA(BFHashDataStruct* hd, const BFHashParams* hp) {
    reset_mutex_kernel<<<(hp->m_hashNumBuckets + 255) / 256, 256, 0, g_stream>>>(hd->d_hashBucketMutex, hp->m_hashNumBuckets);
    BF_SAFE((int)cudaGetLastError());
}

// The reference's kernels read c_hashParams / c_depthCameraParams and the bound textures, not the
// stub arguments (which only size the grid): the stubs below do the same with the latched copies.
BF_API void allocCUDA(BFHashDataStruct* hd, const BFHashParams* hp, const BFDepthCameraData* dd, const BFDepthCameraParams* cp, const unsigned int* d_bitMask) {
    (void)hp; (void)dd;
    if (d_bitMask != nullptr) { fprintf(stderr, "bundlefusion_b200: allocCUDA: chunk streaming (d_bitMask) is out of scope (disabled in BundleFusion)\n"); exit(-1); }
    TsdfAux* aux;
    BF_SAFE(get_aux(hd, &g_hashParams, &aux, true));
    BFDepthCameraParams cam = g_camParams;
    cam.m_imageWidth = cp->m_imageWidth; cam.m_imageHeight = cp->m_imageHeight;   // grid follows the argument (.cu:255)
    BF_SAFE(do_alloc(hd, &g_hashParams, g_bound.d_depthData, &cam, aux, false, -1));
}

BF_API void fillDecisionArrayCUDA(BFHashDataStruct* hd, const BFHashParams* hp) {
    const unsigned n = hp->m_hashNumBuckets * BF_HASH_BUCKET_SIZE;
    fill_decision_kernel<<<(n + 255) / 256, 256, 0, g_stream>>>(*hd, g_hashParams, g_camParams);
    BF_SAFE((int)cudaGetLastError());
}
BF_API void compactifyHashCUDA(BFHashDataStruct* hd, const BFHashParams* hp) {
    const unsigned n = hp->m_hashNumBuckets * BF_HASH_BUCKET_SIZE;
    compactify_prefix_kernel<<<(n + 255) / 256, 256, 0, g_stream>>>(*hd, n);
    BF_SAFE((int)cudaGetLastError());
}

BF_API unsigned int compactifyHashAllInOneCUDA(BFHashDataStruct* hd, const BFHashParams* hp) {
    (void)hp;
    TsdfAux* aux;
    BF_SAFE(get_aux(hd, &g_hashParams, &aux, true));
    BF_SAFE(do_compactify(hd, &g_hashParams, &g_camParams, aux, false, false, false));
    unsigned res = 0;
    BF_SAFE((int)cudaMemcpyAsync(&res, live_count_ptr(aux), sizeof(unsigned), cudaMemcpyDeviceToHost, g_stream));
    BF_SAFE((int)cudaStreamSynchronize(g_stream));
    BF_SAFE((int)cudaMemcpyAsync(hd->d_hashCompactifiedCounter, &res, sizeof(unsigned), cudaMemcpyHostToDevice, g_stream));
    return res;
}

static void integrate_stub(BFHashDataStruct* hd, const BFHashParams* hp, bool de) {
    TsdfAux* aux;
    BF_SAFE(get_aux(hd, &g_hashParams, &aux, true));
    BF_SAFE(do_integrate(hd, &g_hashParams, &g_bound, &g_camParams, aux, de, false, hp->m_numOccupiedBlocks));
}
BF_API void integrateDepthMapCUDA(BFHashDataStruct* hd, const BFHashParams* hp, const BFDepthCameraData*, const BFDepthCameraParams*) { integrate_stub(hd, hp, false); }
BF_API void deIntegrateDepthMapCUDA(BFHashDataStruct* hd, const BFHashParams* hp, const BFDepthCameraData*, const BFDepthCameraParams*) { integrate_stub(hd, hp, true); }

BF_API void starveVoxelsKernelCUDA(BFHashDataStruct* hd, const BFHashParams* hp) {
    if (hp->m_numOccupiedBlocks == 0) return;
    { TsdfAux* aux; if (get_aux(hd, nullptr, &aux, false) == 0) aux->liveValid = false; }
    starve_kernel<<<hp->m_numOccupiedBlocks, BF_SDF_BLOCK_VOXELS, 0, g_stream>>>(*hd);
    BF_SAFE((int)cudaGetLastError());
}

BF_API void garbageCollectIdentifyCUDA(BFHashDataStruct* hd, const BFHashParams* hp) {
    if (hp->m_numOccupiedBlocks == 0) return;
    gc_identify_kernel<<<grid_for(hp->m_numOccupiedBlocks, 16), 128, 0, g_stream>>>(*hd, hp->m_numOccupiedBlocks);
    BF_SAFE((int)cudaGetLastError());
}
BF_API void garbageCollectFreeCUDA(BFHashDataStruct* hd, const BFHashParams* hp) {
    if (hp->m_numOccupiedBlocks == 0) return;
    TsdfAux* aux;
    BF_SAFE(get_aux(hd, &g_hashParams, &aux, true));
    gc_free_kernel<<<grid_for(hp->m_numOccupiedBlocks, 16), 128, 0, g_stream>>>(*hd, g_hashParams, hp->m_numOccupiedBlocks, aux->slotInfo, aux->ctrs);
    BF_SAFE((int)cudaGetLastError());
}

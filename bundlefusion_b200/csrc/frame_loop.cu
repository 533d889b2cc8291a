// frame_loop.cu -- the per-frame sequencing object behind include/bf_frameloop.h: host C++ that drives this library's kernels in the order
// FriedLiver's frame callback drives the reference's.
//
// Behavioural sources (FL/ = /root/reference/FriedLiver/Source/):
//   frame callback, reintegrate()                      FL/DepthSensing/DepthSensing.cpp:854-902, 966-1129
//   OnlineBundler (state machine, trajectories)        FL/OnlineBundler.cpp:28-416, FL/OnlineBundlerHelper.h:74-110
//   Bundler (detect, cache, matchAndFilter, optimize)  FL/Bundler.cpp:18-390
//   SIFTImageManager bookkeeping                       FL/SiftGPU/SIFTImageManager.cpp:44-84, 551-575; SIFTImageManager.h:112-124, 158-163, 263-273
//   SBA::align / removeMaxResidualCUDA                 FL/SBA.cpp:19-203
//   CUDASolverBundling (buffers, solve, max residual)  FL/Solver/CUDASolverBundling.cpp:19-86, 187-298, 313-329, 429-476
//   CUDACache (frames, intrinsics, copy / increment)   FL/CUDACache.cpp:14-86, FL/CUDACache.h
// Differences, all on the host side of the boundary: one thread runs the reference's single-threaded order; counts that the reference copies
// to the host after every stage stay on the device until a decision needs them (3 small reads per frame); key points live at image * maxKeys
// + key (the reference packs them by a prefix sum -- which needs each count on the host before the next image can be placed); the chunk ->
// keyframe fusion and the verification run on the device (csrc/sift_fuse.cu, csrc/sift_verify.cu).
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <list>
#include <vector>

#include "../../include/bf_bundler.h"
#include "../../include/bf_cache.h"
#include "../../include/bf_frameloop.h"
#include "../../include/bf_host.h"
#include "../../include/bf_ingest.h"
#include "../../include/bf_keyframe_search.h"
#include "../../include/bf_sift.h"
#include "../../include/bf_solver.h"
#include "bf_common.cuh"
#include "mat4.cuh"

namespace bf {
int tsdf_batching_usable();          // tsdf.cu: batching on and fast arithmetic selected (bfTsdfRunOps' rule)
int tsdf_stats_async(const BFHashDataStruct* hd, unsigned* h_out);     // tsdf.cu: heap counter + drop counters into pinned memory, no host wait

extern unsigned long long g_launchCount;

#define FL_OK(expr) do { int _rc = (int)(expr); if (_rc) return _rc; } while (0)
static const float kNegInf = -INFINITY;

// ---- tiny kernels ---------------------------------------------------------------------------------------------------------------
// CUDAImageUtil::resampleToIntensity (FL/CUDAImageUtil.cu:224-241): nearest resample + 0.299 r + 0.587 g + 0.114 b, / 255
__global__ void fl_resample_intensity_kernel(float* out, unsigned ow, unsigned oh, const uchar4* in, unsigned iw, unsigned ih) {
    const unsigned x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= ow || y >= oh) return;
    const float sw = (float)(iw - 1) / (float)(ow - 1), sh = (float)(ih - 1) / (float)(oh - 1);
    const unsigned xi = (unsigned)((float)x * sw + 0.5f), yi = (unsigned)((float)y * sh + 0.5f);
    if (xi < iw && yi < ih) { const uchar4 c = in[yi * iw + xi]; out[y * ow + x] = (0.299f * c.x + 0.587f * c.y + 0.114f * c.z) / 255.0f; }
}
__global__ void fl_set_identity_kernel(float* T, unsigned n) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n * 16) T[i] = ((i % 16) % 5 == 0) ? 1.0f : 0.0f;
}
__global__ void fl_set_int_kernel(int* p, int v, unsigned n) { const unsigned i = blockIdx.x * blockDim.x + threadIdx.x; if (i < n) p[i] = v; }

// ---- device memory owner ----------------------------------------------------------------------------------------------------------
struct Arena {
    std::vector<void*> ptrs;
    int err = 0;
    template <class T> T* get(size_t n, bool zero = true) {
        void* p = nullptr;
        const size_t bytes = std::max<size_t>(n, 1) * sizeof(T);
        cudaError_t e = cudaMalloc(&p, bytes);
        if (e != cudaSuccess) { set_last_error("frame loop: cudaMalloc", e); err = (int)e; return nullptr; }
        if (zero) cudaMemsetAsync(p, 0, bytes, stream());
        ptrs.push_back(p);
        return reinterpret_cast<T*>(p);
    }
    ~Arena() { for (void* p : ptrs) cudaFree(p); }
};

static void mat_identity(float* m) { for (int i = 0; i < 16; ++i) m[i] = (i % 5 == 0) ? 1.0f : 0.0f; }
// mat4f::getInverse of an intrinsics matrix (FL/CUDACache.cpp:25, 38; FL/Bundler.cpp:25): the general inverse in the reference's operation order -- the closed form
// 1 / fx, -mx / fx rounds differently for some calibrations
static void intrinsics_inverse(const float* K, float* Ki) { mat4_inverse_ref(K, Ki); }

// ---- CUDACache ------------------------------------------------------------------------------------------------------------------------
struct Cache {
    unsigned maxImages = 0, w = 0, h = 0, cur = 0;
    BFCacheParams p;
    float K[16];                                   // cache-resolution intrinsics (FL/CUDACache.cpp:20-24)
    std::vector<BFCUDACachedFrame> frames;         // host copy of the pointer records
    BFCUDACachedFrame* d_frames = nullptr;
    size_t planeBytes[6];
    int init(Arena& A, const BFFrameLoopParams& P, unsigned maxImg) {
        maxImages = maxImg; w = P.downsampledWidth; h = P.downsampledHeight;
        memset(&p, 0, sizeof(p));
        p.inputDepthWidth = P.depthWidth; p.inputDepthHeight = P.depthHeight; p.inputColorWidth = P.colorWidth; p.inputColorHeight = P.colorHeight;
        p.width = w; p.height = h;
        intrinsics_inverse(P.depthIntrinsics, p.inputIntrinsicsInv);
        p.filterIntensitySigma = P.colorDownSigma; p.filterDepthSigmaD = P.depthDownSigmaD; p.filterDepthSigmaR = P.depthDownSigmaR;
        memcpy(K, P.depthIntrinsics, sizeof(K));
        K[0] *= (float)w / (float)P.depthWidth; K[5] *= (float)h / (float)P.depthHeight;
        K[2] *= (float)(w - 1) / (float)(P.depthWidth - 1); K[6] *= (float)(h - 1) / (float)(P.depthHeight - 1);
        const size_t n = (size_t)w * h;
        const size_t bytes[6] = { n * 4, n * 16, n * 4, n * 8, n * 4, n * 16 };
        memcpy(planeBytes, bytes, sizeof(bytes));
        frames.resize(maxImages);
        for (unsigned k = 0; k < maxImages; ++k) {
            frames[k].d_depthDownsampled = A.get<float>(n); frames[k].d_cameraposDownsampled = A.get<float>(4 * n);
            frames[k].d_intensityDownsampled = A.get<float>(n); frames[k].d_intensityDerivsDownsampled = A.get<float>(2 * n);
            frames[k].d_normalsDownsampledUCHAR4 = A.get<uint8_t>(4 * n); frames[k].d_normalsDownsampled = A.get<float>(4 * n);
        }
        d_frames = A.get<BFCUDACachedFrame>(maxImages);
        if (A.err) return A.err;
        BF_CHECK(cudaMemcpyAsync(d_frames, frames.data(), sizeof(BFCUDACachedFrame) * maxImages, cudaMemcpyHostToDevice, stream()));
        BF_CHECK(cudaStreamSynchronize(stream()));            // `frames` is pageable host memory
        return 0;
    }
    int storeFrame(const float* d_depthRaw, const uint8_t* d_color) {        // CUDACache::storeFrame (cpp:45-86)
        if (cur >= maxImages) return (int)cudaErrorMemoryAllocation;
        FL_OK(bfCacheStoreFrame(&p, d_depthRaw, d_color, &frames[cur]));
        ++cur;
        return 0;
    }
    int copyFrom(const Cache& o, unsigned frame) {                            // copyCacheFrameFrom (CUDACache.h): appends o's frame
        if (cur >= maxImages) return (int)cudaErrorMemoryAllocation;
        const void* src[6] = { o.frames[frame].d_depthDownsampled, o.frames[frame].d_cameraposDownsampled, o.frames[frame].d_intensityDownsampled,
                               o.frames[frame].d_intensityDerivsDownsampled, o.frames[frame].d_normalsDownsampledUCHAR4, o.frames[frame].d_normalsDownsampled };
        void* dst[6] = { frames[cur].d_depthDownsampled, frames[cur].d_cameraposDownsampled, frames[cur].d_intensityDownsampled,
                         frames[cur].d_intensityDerivsDownsampled, frames[cur].d_normalsDownsampledUCHAR4, frames[cur].d_normalsDownsampled };
        for (int k = 0; k < 6; ++k) BF_CHECK(cudaMemcpyAsync(dst[k], src[k], planeBytes[k], cudaMemcpyDeviceToDevice, stream()));
        ++cur;
        return 0;
    }
    void incrementCache() { ++cur; }
    void reset() { cur = 0; }
};

// ---- SIFTImageManager ---------------------------------------------------------------------------------------------------------------
struct SiftManager {
    unsigned maxImages = 0, maxKeys = 0, maxResiduals = 0;
    BFSIFTKeyPoint* d_keys = nullptr; uint8_t* d_descs = nullptr; int* d_numKeys = nullptr;        // key k of image i at i * maxKeys + k
    std::vector<int> numKeys;                                                                       // host mirror
    int* d_numMatches = nullptr; float* d_matchDist = nullptr; uint32_t* d_matchIdx = nullptr;     // raw matches per previous image
    int* d_numFilt = nullptr; float* d_filtDist = nullptr; uint32_t* d_filtIdx = nullptr; float* d_filtT = nullptr; float* d_filtTinv = nullptr;
    int* d_valid = nullptr; std::vector<int> valid;
    BFEntryJ* d_glob = nullptr; uint32_t* d_globIdx = nullptr; int* d_globNum = nullptr; int globNum = 0;
    int* d_lastMatched = nullptr; int* d_validOpt = nullptr;
    unsigned numImages = 0, curFrame = 0;
    std::list<unsigned> retry;
    int init(Arena& A, unsigned maxImg, unsigned maxK, unsigned maxRes) {
        maxImages = maxImg; maxKeys = maxK; maxResiduals = maxRes;
        d_keys = A.get<BFSIFTKeyPoint>((size_t)maxImg * maxK); d_descs = A.get<uint8_t>((size_t)maxImg * maxK * 128, false); d_numKeys = A.get<int>(maxImg);
        d_numMatches = A.get<int>(maxImg); d_matchDist = A.get<float>((size_t)maxImg * BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW);
        d_matchIdx = A.get<uint32_t>((size_t)maxImg * BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW * 2);
        d_numFilt = A.get<int>(maxImg); d_filtDist = A.get<float>((size_t)maxImg * BF_MAX_MATCHES_PER_IMAGE_PAIR_FILTERED);
        d_filtIdx = A.get<uint32_t>((size_t)maxImg * BF_MAX_MATCHES_PER_IMAGE_PAIR_FILTERED * 2);
        d_filtT = A.get<float>((size_t)maxImg * 16); d_filtTinv = A.get<float>((size_t)maxImg * 16);
        d_valid = A.get<int>(maxImg);
        d_glob = A.get<BFEntryJ>(maxRes, false); d_globIdx = A.get<uint32_t>((size_t)maxRes * 2, false); d_globNum = A.get<int>(1);
        d_lastMatched = A.get<int>(1); d_validOpt = A.get<int>(1);
        numKeys.assign(maxImg, 0);
        reset();
        return A.err;
    }
    void reset() {                                  // SIFTImageManager::reset (h:112-124)
        numImages = 0; curFrame = 0; globNum = 0;
        cudaMemsetAsync(d_globNum, 0, sizeof(int), stream());
        valid.assign(maxImages, 0); valid[0] = 1;
        std::fill(numKeys.begin(), numKeys.end(), 0);
    }
    int pushValid(unsigned n) { if (!n) return 0; BF_CHECK(cudaMemcpyAsync(d_valid, valid.data(), sizeof(int) * n, cudaMemcpyHostToDevice, stream())); return 0; }
    BFSIFTKeyPoint* keysOf(unsigned i) const { return d_keys + (size_t)i * maxKeys; }
    uint8_t* descsOf(unsigned i) const { return d_descs + (size_t)i * maxKeys * 128; }
    // createSIFTImageGPU + finalizeSIFTImageGPU (cpp:44-75): the new image is the current one
    unsigned addImage(int nKeys) { const unsigned i = numImages++; numKeys[i] = nKeys; curFrame = i; return i; }
};

// ---- CUDASolverBundling + SBA ---------------------------------------------------------------------------------------------------------------
struct Solver {
    unsigned maxImages = 0, maxCorrPerImage = 0, maxResiduals = 0;
    BFSolverState st;
    int* d_varToCorr = nullptr; int* d_numEntriesPerRow = nullptr;
    float* d_xRot = nullptr; float* d_xTrans = nullptr; float* d_maxOut = nullptr;
    float maxResidualThresh = 0.08f, verifyOptDistThresh = 0.02f, verifyOptPercentThresh = 0.05f;      // cpp:35-36, s_optMaxResThresh
    float maxRes = -1.0f; int maxResIdx = 0;
    BFSolverInput lastInput; BFSolverParameters lastPar;
    std::vector<float> wS, wD, wC;
    int init(Arena& A, unsigned maxImg, unsigned maxRes_) {       // CUDASolverBundling ctor (cpp:19-86)
        maxImages = maxImg; maxResiduals = maxRes_;
        maxCorrPerImage = std::max(1000u, std::min(4000u, maxRes_ / std::max(1u, maxImg)));           // cpp:39
        memset(&st, 0, sizeof(st));
        const size_t N = maxImg;
        st.d_deltaRot = A.get<float>(3 * N); st.d_deltaTrans = A.get<float>(3 * N); st.d_rRot = A.get<float>(3 * N); st.d_rTrans = A.get<float>(3 * N);
        st.d_zRot = A.get<float>(3 * N); st.d_zTrans = A.get<float>(3 * N); st.d_pRot = A.get<float>(3 * N); st.d_pTrans = A.get<float>(3 * N);
        st.d_Jp = A.get<float>(8); st.d_Ap_XRot = A.get<float>(3 * N); st.d_Ap_XTrans = A.get<float>(3 * N); st.d_scanAlpha = A.get<float>(2);
        st.d_rDotzOld = A.get<float>(N); st.d_precondionerRot = A.get<float>(3 * N); st.d_precondionerTrans = A.get<float>(3 * N);
        st.d_sumResidual = A.get<float>(1); st.d_countHighResidual = A.get<int>(1);
        st.d_denseJtJ = A.get<float>(8); st.d_denseJtr = A.get<float>(6 * N); st.d_denseCorrCounts = A.get<float>(8);
        st.d_xTransforms = A.get<float>(16 * N); st.d_xTransformInverses = A.get<float>(16 * N);
        st.d_denseOverlappingImages = A.get<uint32_t>(8); st.d_numDenseOverlappingImages = A.get<int>(1);
        st.d_corrCount = A.get<int>(1); st.d_corrCountColor = A.get<int>(1); st.d_sumResidualColor = A.get<float>(1);
        d_varToCorr = A.get<int>(N * maxCorrPerImage); d_numEntriesPerRow = A.get<int>(N);
        d_xRot = A.get<float>(3 * N); d_xTrans = A.get<float>(3 * N); d_maxOut = A.get<float>(2);
        return A.err;
    }
};

// ---- Bundler ------------------------------------------------------------------------------------------------------------------------
struct Bundler {
    bool isLocal = true;
    SiftManager sm; Cache cache; Solver solver;
    float* d_trajectory = nullptr;
    int continueRetry = 0; unsigned revalidatedIdx = 0xFFFFFFFFu;
    bool verifyFlag = false;      // SBA::m_bVerify
};

// ---- the frame store: integration-resolution depth + colour of every frame (CUDAImageManager's frames) -----------------------------------
// `slots` device slots; frame f's images are in slot slotOf[f] while it is resident.  deviceFrameSlots = 0: one slot per frame, every frame
// stays where its ingest wrote it.  deviceFrameSlots = N: N slots over a pinned host store of every frame; each ingest is written back to
// the host on the copy stream, and a frame an op reads is fetched back into a slot (the least recently used one that is not pinned) first.
// Ordering, never a host wait: a slot is overwritten only after its last reader (evRead, recorded on the stream that read it) and its last
// copy (evCopy, on the copy stream); a reader waits for the copy that filled the slot.
struct FrameStore {
    static const unsigned kChunk = 256;           // frames per pinned host allocation
    unsigned slots = 0, used = 0;                 // slots are handed out in order until all are used, then reused
    size_t px = 0;
    float* d_depth = nullptr; uint8_t* d_color = nullptr;
    bool spill = false;                           // deviceFrameSlots > 0: the pinned host store exists
    std::vector<uint8_t*> chunks;                 // host frame f: chunks[f / kChunk] + (f % kChunk) * 8 px, depth then colour
    cudaStream_t copy = nullptr; cudaEvent_t evIngest = nullptr;
    std::vector<int> slotOf, frameIn;             // frame -> slot, slot -> frame (-1: none)
    std::vector<unsigned long long> lastUse;      // slot -> use tick of its last use (LRU victim: the smallest, unpinned)
    std::vector<char> pin;
    std::vector<cudaEvent_t> evRead, evCopy;
    std::vector<int> lent;                        // slots bfFrameLoopFetchFrames handed out: read on the library stream until the next call
    unsigned long long tick = 0, writeBacks = 0, fetches = 0, hits = 0, evictions = 0, h2d = 0, d2h = 0, hostBytes = 0;
    double pinMs = 0.0;
    float* depthOf(int s) const { return d_depth + px * (size_t)s; }
    uint8_t* colorOf(int s) const { return d_color + px * 4 * (size_t)s; }
    uint8_t* hostOf(unsigned f) const { return chunks[f / kChunk] + (size_t)(f % kChunk) * px * 8; }
};

struct Loop {
    BFFrameLoopParams P;
    Arena A;
    // frame input / store
    float* d_depthRaw = nullptr; uint8_t* d_colorRaw = nullptr; float* d_depthFilt = nullptr; float* d_intensity = nullptr;
    FrameStore fs;
    std::vector<const float*> depthPtrs; std::vector<const uint8_t*> colorPtrs;    // per frame: its slot's images while resident, else NULL
    BFIngestParams ingest, ingestSensorRes; bool needSensorResFilter = false;
    BFSiftDetectParams detect;
    float siftK[16], siftKinv[16];
    Bundler local, optLocal, global;
    Bundler* pLocal = nullptr; Bundler* pOptLocal = nullptr;
    // OnlineBundler
    float* d_completeTrajectory = nullptr; float* d_localTrajectories = nullptr; float* d_siftTrajectory = nullptr; float* d_currIntegrateTransform = nullptr;
    int* d_imageInvalidateList = nullptr;
    std::vector<int> invalidImagesList; std::vector<std::vector<int>> localTrajectoriesValid;
    float* h_complete = nullptr;                  // pinned: the complete trajectory as the TrajectoryManager reads it (maxNumFrames poses)
    // BundlerState (OnlineBundlerHelper.h:74-110)
    enum { DO_NOTHING = 0, PROCESS = 1, INVALIDATE = 2 };
    int lastFrameProcessed = -1; bool lastFrameValid = false; int localToSolve = -1; int lastLocalSolved = -1; unsigned numFramesPastEnd = 0;
    unsigned numCompleteTransforms = 0, lastValidCompleteTransform = 0; bool globalTrackingLost = false; int processState = DO_NOTHING; bool useSolve = true;
    unsigned totalNumOptLocalFrames = 0;
    // end of the recording (bfFrameLoopFinish): K of its first call, the dense end solve of turn K (SBA's global weights switched by
    // OnlineBundler::processInput, FL/OnlineBundler.cpp:174-189), where it ran and what it covered
    int finishK = -1; bool finished = false, denseEndSolve = false;
    int denseTurn = -1; unsigned denseKeyframes = 0, densePairs = 0;
    unsigned numFrames = 0;                      // frames received (CUDAImageManager::getCurrFrameNumber() + 1)
    float currIntegrate[16];
    BFTrajectoryManager* tm = nullptr;
    // scene: the table's buffers are stream-ordered allocations the loop owns (hash_alloc), not the arena's, so that growth can replace them
    BFHashDataStruct hd; BFHashParams hp; BFDepthCameraParams cam;
    // pinned status block
    int* h_pin = nullptr;
    unsigned long long counters[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
    BFFrameLoopStatus status;
    // reconstruction stream: the TSDF work of frame f runs beside process() of frame f and processInput() of frame f + 1, as the reference's
    // reconstruction and bundling threads do; the data dependencies of the single-threaded order are kept by events
    cudaStream_t tsdfStream = nullptr; cudaEvent_t evMain = nullptr, evTsdf = nullptr; bool overlap = false, tsdfPending = false;
    // feature stream (bfFrameLoopStepAhead): upload, ingest, SIFT detection and dense cache of frame f + 1 are queued on a third stream while frame f is
    // matched, solved and fused -- the hand-over the reference makes between CUDAImageManager::process on the reconstruction thread and the bundling
    // thread (RUN_MULTITHREADED).  Destinations of that work (frame store slot, key / descriptor slot, cache slot of the chunk the frame will belong
    // to) are fixed by host state alone, so they are known one frame early; nothing frame f still reads is written.
    cudaStream_t featStream = nullptr; cudaEvent_t evStepStart = nullptr, evFeat = nullptr; bool featUsed = false;
    struct Ahead { bool valid = false; unsigned frame = 0; const float* depth = nullptr; const uint8_t* color = nullptr; Bundler* b = nullptr; unsigned li = 0; } ahead;
    bool aheadWanted = false, aheadArmed = false; const float* nextDepth = nullptr; const uint8_t* nextColor = nullptr; int nextOnHost = 0;
    Bundler* aheadTarget = nullptr; unsigned aheadLi = 0;
    // stage profile (bfFrameLoopSetProfiling): events at the stage boundaries of a step, elapsed times summed per stage
    bool profile = false; cudaEvent_t stageEv[BF_FRAMELOOP_STAGES + 1] = {}; bool stageHit[BF_FRAMELOOP_STAGES + 1] = {}; double stageMs[BF_FRAMELOOP_STAGES] = {}; unsigned long long profiledSteps = 0;
    // op log (bfFrameLoopSetOpLog): every TSDF op reconstruct() hands to bfTsdfRunOps, with the turn (step or past-end turn, counted from 0) that issued it
    bool opLogOn = false; unsigned turn = 0; std::vector<BFTsdfOp> opLog; std::vector<uint32_t> opLogTurn;
    // hash growth (bfFrameLoopGetHashGrowth): h_stat receives {heap counter, heap failures, drops} of the turn statTurn, ev marks its arrival
    struct Growth {
        bool on = false, ceilingReached = false, pending = false, sampled = false;
        unsigned growths = 0, discarded = 0, initBlocks = 0, initBuckets = 0, bucketScale = 1;
        unsigned* h_stat = nullptr; cudaEvent_t ev = nullptr; unsigned statTurn = 0, statBlocks = 0;
        unsigned live = 0, sampleTurn = 0, maxInc = 0; unsigned long long dropped = 0; bool dropRose = false;
    } grow;
};
// boundary k = end of stage k - 1 / start of stage k
static void mark(Loop& L, int k) { if (L.profile && L.stageEv[k]) { cudaEventRecord(L.stageEv[k], stream()); L.stageHit[k] = true; } }
static void stage_collect(Loop& L) {
    if (!L.profile) return;
    cudaStreamSynchronize(stream());
    int prev = -1;
    for (int k = 0; k <= BF_FRAMELOOP_STAGES; ++k) {
        if (!L.stageHit[k]) continue;
        if (prev >= 0) { float ms = 0.0f; if (cudaEventElapsedTime(&ms, L.stageEv[prev], L.stageEv[k]) == cudaSuccess) L.stageMs[k - 1] += ms; }   // a skipped stage's time belongs to the one that ran
        prev = k;
    }
    for (int k = 0; k <= BF_FRAMELOOP_STAGES; ++k) L.stageHit[k] = false;
    ++L.profiledSteps;
}

static const int PIN_FEAT = 3072;            // h_pin slot the feature stream's key-point count lands in (h_pin: 4096 ints; 16 .. 2016 carry valid flags)
static int launch_ahead(Loop& L);
// every host wait on the library stream: if the next frame's feature work is armed, it is queued first, so that it runs while the host waits
static int sync_stream(Loop& L) { if (L.aheadArmed) FL_OK(launch_ahead(L)); ++L.counters[6]; BF_CHECK(cudaStreamSynchronize(stream())); return 0; }

// ---- frame store slots ----------------------------------------------------------------------------------------------------------------
// a slot for frame f (not resident): a never-used one while there are any, else the least recently used unpinned one, whose frame is
// evicted.  The caller orders the overwrite after the slot's last reader and copy.  Returns -1 when every slot is pinned.
static int take_slot(Loop& L, unsigned f) {
    FrameStore& S = L.fs;
    int s = -1;
    if (S.used < S.slots) s = (int)S.used++;
    else
        for (unsigned k = 0; k < S.slots; ++k)
            if (!S.pin[k] && (s < 0 || S.lastUse[k] < S.lastUse[s])) s = (int)k;
    if (s < 0) return -1;
    const int g = S.frameIn[s];
    if (g >= 0) { S.slotOf[g] = -1; L.depthPtrs[g] = nullptr; L.colorPtrs[g] = nullptr; ++S.evictions; }
    S.frameIn[s] = (int)f; S.slotOf[f] = s;
    L.depthPtrs[f] = S.depthOf(s); L.colorPtrs[f] = S.colorOf(s);
    return s;
}

// the slot frame f's ingest writes, on the current stream, pinned until the turn that integrates the frame has fetched its frames
static int ingest_slot(Loop& L, unsigned f, int* slot) {
    FrameStore& S = L.fs;
    const int s = take_slot(L, f);
    if (s < 0) { set_last_error("frame loop: every frame slot is pinned", cudaErrorInvalidValue); return (int)cudaErrorInvalidValue; }
    if (S.spill) { BF_CHECK(cudaStreamWaitEvent(stream(), S.evRead[s], 0)); BF_CHECK(cudaStreamWaitEvent(stream(), S.evCopy[s], 0)); }
    S.pin[s] = 1; S.lastUse[s] = ++S.tick;
    *slot = s;
    return 0;
}

// after the ingest work of frame f on the current stream (its SIFT detection reads the slot too): the copy stream writes the slot back to the host
static int write_back(Loop& L, unsigned f) {
    FrameStore& S = L.fs;
    if (!S.spill) return 0;
    const int s = S.slotOf[f];
    uint8_t* h = S.hostOf(f);
    BF_CHECK(cudaEventRecord(S.evIngest, stream()));
    BF_CHECK(cudaStreamWaitEvent(S.copy, S.evIngest, 0));
    BF_CHECK(cudaMemcpyAsync(h, S.depthOf(s), S.px * 4, cudaMemcpyDeviceToHost, S.copy));
    BF_CHECK(cudaMemcpyAsync(h + S.px * 4, S.colorOf(s), S.px * 4, cudaMemcpyDeviceToHost, S.copy));
    BF_CHECK(cudaEventRecord(S.evCopy[s], S.copy));
    ++S.writeBacks; S.d2h += S.px * 8;
    return 0;
}

// Make frames[0, n) resident and pin their slots (one use tick for the group).  A frame without a slot takes one: the copy stream waits for
// the slot's last reader, copies the frame from the host store and records the slot's copy event; the slot goes into *fetched.  The write-back
// of the frame was queued on the same copy stream earlier, so the fetch follows it.
static int fetch_frames(Loop& L, const uint32_t* frames, unsigned n, std::vector<int>* fetched) {
    FrameStore& S = L.fs;
    const unsigned long long t = ++S.tick;
    for (unsigned k = 0; k < n; ++k) {
        const unsigned f = frames[k];
        int s = S.slotOf[f];
        if (s >= 0) { if (S.lastUse[s] != t) ++S.hits; }
        else {
            s = take_slot(L, f);
            if (s < 0) { set_last_error("frame loop: every frame slot is pinned", cudaErrorInvalidValue); return (int)cudaErrorInvalidValue; }
            const uint8_t* h = S.hostOf(f);
            BF_CHECK(cudaStreamWaitEvent(S.copy, S.evRead[s], 0));
            BF_CHECK(cudaMemcpyAsync(S.depthOf(s), h, S.px * 4, cudaMemcpyHostToDevice, S.copy));
            BF_CHECK(cudaMemcpyAsync(S.colorOf(s), h + S.px * 4, S.px * 4, cudaMemcpyHostToDevice, S.copy));
            BF_CHECK(cudaEventRecord(S.evCopy[s], S.copy));
            ++S.fetches; S.h2d += S.px * 8;
            fetched->push_back(s);
        }
        S.pin[s] = 1; S.lastUse[s] = t;
    }
    return 0;
}

// the current stream waits for the copies that filled the fetched slots
static int wait_fetched(Loop& L, const std::vector<int>& fetched) {
    for (int s : fetched) BF_CHECK(cudaStreamWaitEvent(stream(), L.fs.evCopy[s], 0));
    return 0;
}

// frames[0, n) were read by work queued on the current stream: that is their slots' last reader; unpin them
static int release_frames(Loop& L, const uint32_t* frames, unsigned n) {
    FrameStore& S = L.fs;
    for (unsigned k = 0; k < n; ++k) {
        const int s = S.slotOf[frames[k]];
        if (s < 0 || !S.pin[s]) continue;
        if (S.spill) BF_CHECK(cudaEventRecord(S.evRead[s], stream()));
        S.pin[s] = 0;
    }
    return 0;
}

// at the entry of a call that may reuse slots: the slots the last bfFrameLoopFetchFrames handed out were read on the library stream up to now
static int settle_lent(Loop& L) {
    FrameStore& S = L.fs;
    if (S.spill) for (int s : S.lent) BF_CHECK(cudaEventRecord(S.evRead[s], stream()));
    S.lent.clear();
    return 0;
}

// ---- Bundler::matchAndFilter (FL/Bundler.cpp:103-249) ----------------------------------------------------------------------------------------
// returns lastMatchedFrame (or -1) in *lastMatched; one host synchronisation at the end (verdict + correspondence count)
static int match_and_filter(Loop& L, Bundler& b, int* lastMatched) {
    SiftManager& sm = b.sm;
    const BFFrameLoopParams& P = L.P;
    const unsigned numFrames = sm.numImages, cur = sm.curFrame;
    *lastMatched = -1;
    const unsigned start = (numFrames == cur + 1) ? 0 : cur + 1;
    const int num2 = sm.numKeys[cur];
    if (num2 == 0) return 0;
    std::vector<BFSiftMatchJob> jobs;
    jobs.reserve(numFrames);
    for (unsigned prev = start; prev < numFrames; ++prev) {
        if (prev == cur) continue;
        BFSiftMatchJob j;
        j.d_des1 = sm.descsOf(prev); j.num1 = (sm.valid[prev] == 0) ? 0 : sm.numKeys[prev];          // invalid image / no keys: the pair only gets its counter zeroed (:127-130)
        j.d_des2 = sm.descsOf(cur); j.num2 = num2;
        j.out.d_numMatches = sm.d_numMatches + prev;
        j.out.d_distances = sm.d_matchDist + (size_t)prev * BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW;
        j.out.d_keyPointIndices = sm.d_matchIdx + (size_t)prev * BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW * 2;
        j.keyPointOffset[0] = prev * sm.maxKeys; j.keyPointOffset[1] = cur * sm.maxKeys;
        jobs.push_back(j);
    }
    if (!jobs.empty())
        FL_OK(bfSiftMatchBatch(jobs.data(), (int)jobs.size(), P.siftMatchThresh, b.isLocal ? P.siftMatchRatioMaxLocal : P.siftMatchRatioMaxGlobal));
    if (cur == 0) return 0;
    FL_OK(bfSiftSortKeyPointMatches(cur, start, numFrames, sm.d_numMatches, sm.d_matchDist, sm.d_matchIdx));
    FL_OK(bfSiftFilterKeyPointMatches(cur, start, numFrames, sm.d_keys, sm.d_numMatches, sm.d_matchDist, sm.d_matchIdx, sm.d_numFilt, sm.d_filtDist, sm.d_filtIdx,
                                      sm.d_filtT, sm.d_filtTinv, L.siftKinv, b.isLocal ? P.minNumMatchesLocal : P.minNumMatchesGlobal, P.maxKabschResidual2));
    FL_OK(bfSiftFilterMatchesBySurfaceArea(cur, start, numFrames, sm.d_keys, sm.d_numFilt, sm.d_filtIdx, L.siftKinv, P.surfAreaPcaThresh, nullptr));
    FL_OK(bfSiftFilterMatchesByDenseVerify(cur, start, numFrames, b.cache.w, b.cache.h, b.cache.K, sm.d_numFilt, sm.d_filtT, b.cache.d_frames, P.projCorrDistThres,
                                           P.projCorrNormalThres, P.projCorrColorThresh, P.verifySiftErrThresh, P.verifySiftCorrThresh, P.sensorDepthMin, P.sensorDepthMax, nullptr));
    // filterFrames + AddCurrToResiduals, decided on the device (:215-219); the verdict and the correspondence count come back in one read
    FL_OK(sm.pushValid(numFrames));
    FL_OK(bfSiftFilterFrames(cur, start, numFrames, sm.d_numFilt, sm.d_valid, sm.d_lastMatched));
    FL_OK(bfSiftAddCurrToResidualsIfMatched(cur, start, numFrames, sm.d_glob, sm.d_globIdx, sm.d_globNum, sm.d_numFilt, sm.d_filtIdx, sm.d_keys, L.siftKinv, sm.d_lastMatched));
    BF_CHECK(cudaMemcpyAsync(L.h_pin, sm.d_lastMatched, sizeof(int), cudaMemcpyDeviceToHost, stream()));
    BF_CHECK(cudaMemcpyAsync(L.h_pin + 1, sm.d_globNum, sizeof(int), cudaMemcpyDeviceToHost, stream()));
    FL_OK(sync_stream(L));
    *lastMatched = L.h_pin[0];
    sm.globNum = L.h_pin[1];
    sm.valid[cur] = (*lastMatched >= 0) ? 1 : 0;
    return 0;
}

// Bundler::tryRevalidation (FL/Bundler.cpp:306-352, USE_RETRY)
static int global_match_and_filter(Loop& L, int* lastMatched);
static int try_revalidation(Loop& L, unsigned curGlobalFrame, bool isScanDone, unsigned* out) {
    Bundler& g = L.global;
    g.revalidatedIdx = 0xFFFFFFFFu;
    *out = g.revalidatedIdx;
    if (g.continueRetry < 0) { *out = 0; return 0; }        // "return false" through an unsigned return type: 0
    if (!g.sm.retry.empty()) {
        const unsigned idx = g.sm.retry.front(); g.sm.retry.pop_front();
        if (isScanDone) {
            if (g.continueRetry == 0) g.continueRetry = (int)idx;
            else if (g.continueRetry == (int)idx) { g.continueRetry = -1; return 0; }
        }
        g.sm.curFrame = idx;
        int lm = -1;
        FL_OK(global_match_and_filter(L, &lm));
        if (g.sm.valid[idx] != 0) {
            BF_CHECK(cudaMemcpyAsync(g.d_trajectory + 16 * (size_t)idx, g.d_trajectory + 16 * (size_t)lm, 64, cudaMemcpyDeviceToDevice, stream()));
            g.revalidatedIdx = idx;
        } else g.sm.retry.push_front(idx);
        g.sm.curFrame = curGlobalFrame;
    }
    *out = g.revalidatedIdx;
    return 0;
}
// matchAndFilter of the global bundler with its extras (:222-236)
static int global_match_and_filter(Loop& L, int* lastMatched) {
    Bundler& g = L.global;
    const unsigned numFrames = g.sm.numImages, cur = g.sm.curFrame;
    FL_OK(match_and_filter(L, g, lastMatched));
    if (cur == 0 || g.sm.numKeys[cur] == 0) return 0;
    const int lm = *lastMatched;
    if (lm >= 0 && (unsigned)lm + 1 != cur) {           // re-initialise to a better location based off of the last match
        BF_CHECK(cudaMemcpyAsync(g.d_trajectory + 16 * (size_t)cur, g.d_trajectory + 16 * (size_t)lm, 64, cudaMemcpyDeviceToDevice, stream()));
        BF_CHECK(cudaMemcpyAsync(g.d_trajectory + 16 * (size_t)(cur + 1), g.d_trajectory + 16 * (size_t)lm, 64, cudaMemcpyDeviceToDevice, stream()));
    }
    if (cur + 1 == numFrames) {                          // a current frame, not a retry frame
        if (lm >= 0) { unsigned r; FL_OK(try_revalidation(L, cur, false, &r)); }
        else g.sm.retry.push_front(cur);
    }
    return 0;
}

// ---- SBA::align + CUDASolverBundling::solve + removeMaxResidualCUDA (FL/SBA.cpp:53-203) ---------------------------------------------------------
static int sba_align(Loop& L, Bundler& b, unsigned maxNumIters, unsigned numPCGits, bool useVerify, bool isEnd, bool isScanDone, unsigned revalidateIdx, bool* removed) {
    (void)isScanDone;
    const BFFrameLoopParams& P = L.P;
    SiftManager& sm = b.sm; Solver& sv = b.solver;
    *removed = false; b.verifyFlag = false; sv.maxRes = -1.0f;
    const unsigned maxIts = std::max(P.numGlobalNonLinIterations, P.numLocalNonLinIterations);
    sv.wS.assign(maxIts, 1.0f); sv.wD.assign(maxIts, 0.0f); sv.wC.assign(maxIts, 0.0f);
    bool useCache = false;
    if (b.isLocal && P.useLocalDense) { for (unsigned i = 0; i < maxIts; ++i) sv.wD[i] = (float)(i + 1); useCache = true; }       // SBA.cpp:28-31
    if (!b.isLocal && L.denseEndSolve) {                  // Bundler::setSolveWeights at the end of the recording (FL/OnlineBundler.cpp:180-186, SBA.cpp:70-79)
        sv.wS.assign(3, 1.0f); sv.wD.assign(3, 15.0f); sv.wC.assign(3, 0.0f); useCache = true;
    }
    const unsigned numImages = sm.numImages;
    FL_OK(sm.pushValid(numImages));                       // valid flags are host-authoritative between stages
    convertMatricesToPosesCU(b.d_trajectory, numImages, sv.d_xRot, sv.d_xTrans, sm.d_valid);
    const unsigned nNonLin = std::min<unsigned>(maxNumIters, (unsigned)sv.wS.size());
    BFSolverInput in; memset(&in, 0, sizeof(in));
    in.d_correspondences = sm.d_glob; in.d_variablesToCorrespondences = sv.d_varToCorr; in.d_numEntriesPerRow = sv.d_numEntriesPerRow;
    in.numberOfCorrespondences = (unsigned)sm.globNum; in.numberOfImages = numImages; in.maxNumberOfImages = sv.maxImages; in.maxCorrPerImage = sv.maxCorrPerImage;
    in.d_validImages = sm.d_valid;
    if (useCache) {
        in.d_cacheFrames = b.cache.d_frames; in.denseDepthWidth = b.cache.w; in.denseDepthHeight = b.cache.h;
        in.intrinsics[0] = b.cache.K[0]; in.intrinsics[1] = b.cache.K[5]; in.intrinsics[2] = b.cache.K[2]; in.intrinsics[3] = b.cache.K[6];
    } else { in.d_cacheFrames = nullptr; for (int k = 0; k < 4; ++k) in.intrinsics[k] = kNegInf; }
    in.maxNumDenseImPairs = sv.maxImages * (sv.maxImages - 1) / 2;
    in.weightsSparse = sv.wS.data(); in.weightsDenseDepth = sv.wD.data(); in.weightsDenseColor = sv.wC.data();
    BFSolverParameters par; memset(&par, 0, sizeof(par));
    par.nNonLinearIterations = nNonLin; par.nLinIterations = numPCGits;
    par.verifyOptDistThresh = sv.verifyOptDistThresh; par.verifyOptPercentThresh = sv.verifyOptPercentThresh; par.highResidualThresh = INFINITY;
    par.denseDistThresh = 0.15f; par.denseNormalThresh = 0.97f; par.denseColorThresh = 0.1f; par.denseColorGradientMin = 0.005f;      // zParametersBundlingDefault.txt:22-28
    par.denseDepthMin = 0.5f; par.denseDepthMax = 4.0f; par.denseOverlapCheckSubsampleFactor = 4;
    par.weightSparse = sv.wS[0]; par.weightDenseDepth = sv.wD[0]; par.weightDenseColor = sv.wC[0];
    par.useDense = (par.weightDenseDepth > 0 || par.weightDenseColor > 0) ? 1 : 0; par.useDenseDepthAllPairwise = 1;
    sv.st.d_xRot = sv.d_xRot; sv.st.d_xTrans = sv.d_xTrans;
    FL_OK(bfSolverSolve(&in, &sv.st, &par));
    sv.lastInput = in; sv.lastPar = par;
    bool needSync = false;
    if (isEnd && sv.wS[0] > 0) {                          // findMaxResidual (cpp:281-283) -> removeMaxResidualCUDA (SBA.cpp:131-135)
        FL_OK(bfSolverMaxResidual(&in, &sv.st, &par, sv.d_maxOut));
        BF_CHECK(cudaMemcpyAsync(L.h_pin + 4, sv.d_maxOut, 8, cudaMemcpyDeviceToHost, stream()));
        needSync = true;
    }
    if (useVerify && sv.wS[0] > 0) {                      // CUDASolverBundling::useVerification (cpp:454-476): device count, host ratio
        BF_CHECK(cudaMemsetAsync(sv.st.d_countHighResidual, 0, sizeof(int), stream()));
        // countHighResiduals is a synchronising stub in the reference's surface; use it as such (one read)
        const int n = countHighResiduals(&in, &sv.st, &par, nullptr);
        ++L.counters[6];
        b.verifyFlag = ((float)n / (float)std::max(1u, in.numberOfCorrespondences)) >= sv.verifyOptPercentThresh;
        needSync = false;                                  // countHighResiduals synchronised the stream: the max-residual read has landed too
        if (isEnd && sv.wS[0] > 0) { memcpy(&sv.maxRes, L.h_pin + 4, 4); memcpy(&sv.maxResIdx, L.h_pin + 5, 4); }
    } else if (useVerify) b.verifyFlag = true;
    if (needSync) { FL_OK(sync_stream(L)); memcpy(&sv.maxRes, L.h_pin + 4, 4); memcpy(&sv.maxResIdx, L.h_pin + 5, 4); }
    convertPosesToMatricesCU(sv.d_xRot, sv.d_xTrans, numImages, b.d_trajectory, sm.d_valid);
    if (isEnd && sv.wS[0] > 0 && in.numberOfCorrespondences > 0) {
        // getMaxResidual (cpp:429-452): image pair of the worst correspondence; never the pair (0, < 10)
        BFEntryJ worst;
        BF_CHECK(cudaMemcpyAsync(L.h_pin + 8, sm.d_glob + sv.maxResIdx, sizeof(BFEntryJ), cudaMemcpyDeviceToHost, stream()));
        FL_OK(sync_stream(L));
        memcpy(&worst, L.h_pin + 8, sizeof(worst));
        const bool rem = !(worst.imgIdx_i == 0 && worst.imgIdx_j < 10) && sv.maxRes > sv.maxResidualThresh;
        (void)revalidateIdx;
        if (rem) {
            FL_OK(bfSiftInvalidateImageToImage(sm.d_glob, (unsigned)sm.globNum, worst.imgIdx_i, worst.imgIdx_j));
            FL_OK(bfSiftCheckForInvalidFrames(sv.d_numEntriesPerRow, sm.d_valid, numImages, sm.d_glob, (unsigned)sm.globNum, P.useComprehensiveFrameInvalidation ? 1 : 0));
            // the reference round-trips the flags through the host around the kernel (SIFTImageManager.cu:724-790): bring them back
            BF_CHECK(cudaMemcpyAsync(L.h_pin + 16, sm.d_valid, sizeof(int) * std::min(numImages, 2000u), cudaMemcpyDeviceToHost, stream()));
            FL_OK(sync_stream(L));
            for (unsigned i = 0; i < std::min(numImages, 2000u); ++i) sm.valid[i] = L.h_pin[16 + i];
            *removed = true;
        }
    }
    return 0;
}

// Bundler::optimize (FL/Bundler.cpp:251-283)
static int bundler_optimize(Loop& L, Bundler& b, unsigned nNonLin, unsigned nLin, bool useVerify, bool removeMaxResidual, bool isScanDone, bool* removed, bool* valid) {
    const BFFrameLoopParams& P = L.P;
    FL_OK(sba_align(L, b, nNonLin, nLin, useVerify, removeMaxResidual, isScanDone, b.revalidatedIdx, removed));
    *valid = true;
    if (b.verifyFlag) {
        FL_OK(b.sm.pushValid(b.sm.numImages));
        FL_OK(bfSiftVerifyTrajectory(b.sm.numImages, b.sm.d_valid, b.d_trajectory, b.cache.w, b.cache.h, b.cache.K, b.cache.d_frames, P.projCorrDistThres, P.projCorrNormalThres,
                                     P.projCorrColorThresh, P.verifyOptErrThresh, P.verifyOptCorrThresh, 0.1f, 3.0f, b.sm.d_validOpt, nullptr));
        BF_CHECK(cudaMemcpyAsync(L.h_pin, b.sm.d_validOpt, sizeof(int), cudaMemcpyDeviceToHost, stream()));
        FL_OK(sync_stream(L));
        *valid = L.h_pin[0] > 0;
    }
    return 0;
}

// ---- OnlineBundler ------------------------------------------------------------------------------------------------------------------------
static void invalidate_images(Loop& L, unsigned s, unsigned e = 0xFFFFFFFFu) {
    if (e == 0xFFFFFFFFu) { if (s < L.invalidImagesList.size()) L.invalidImagesList[s] = 0; }
    else for (unsigned i = s; i < e && i < L.invalidImagesList.size(); ++i) L.invalidImagesList[i] = 0;
}
static void validate_images(Loop& L, unsigned s) { if (s < L.invalidImagesList.size()) L.invalidImagesList[s] = 1; }
static bool is_last_local_frame(const Loop& L, unsigned curFrame) { return curFrame >= L.P.submapSize && (curFrame % L.P.submapSize) == 0; }
static bool bundler_is_valid(const Bundler& b) { for (unsigned i = 1; i < b.sm.numImages; ++i) if (b.sm.valid[i] != 0) return true; return false; }
static int bundler_reset(Bundler& b) {                 // Bundler::reset (FL/Bundler.cpp:354-360)
    if (b.sm.numImages) { fl_set_identity_kernel<<<(b.sm.numImages * 16 + 255) / 256, 256, 0, stream()>>>(b.d_trajectory, b.sm.numImages); BF_CHECK(cudaGetLastError()); ++g_launchCount; }
    b.sm.reset(); b.cache.reset();
    return 0;
}

static void prepare_local_solve(Loop& L, unsigned curFrame, bool isSequenceEnd) {          // FL/OnlineBundler.cpp:134-165
    L.processState = Loop::DO_NOTHING;
    unsigned curLocalIdx = (std::max(curFrame, 1u) - 1) / L.P.submapSize;
    if (isSequenceEnd && (curFrame % L.P.submapSize) == 0) {
        ++curLocalIdx;
        L.localToSolve = -((int)curLocalIdx + 2); L.processState = Loop::INVALIDATE;
    } else if (bundler_is_valid(*L.pLocal)) { L.localToSolve = (int)curLocalIdx; L.processState = Loop::PROCESS; }
    else { L.localToSolve = -((int)curLocalIdx + 2); L.processState = Loop::INVALIDATE; }
    std::swap(L.pLocal, L.pOptLocal);
}

// The device work of a new frame that depends on nothing but the frame itself -- CUDAImageManager::process (FL/CUDAImageManager.cpp:22-158: upload,
// erode + filter + resample into the frame store), getCurrentFrame's intensity image, Bundler::detectFeatures (FL/Bundler.cpp:91-101) into key slot
// `li` of bundler `b`, Bundler::storeCachedFrame -- queued on the CURRENT library stream; the key-point count is copied to *h_count (pinned).
static int front_half(Loop& L, unsigned frame, const float* depth, const uint8_t* color, int onHost, Bundler& b, unsigned li, int* h_count) {
    const BFFrameLoopParams& P = L.P;
    const size_t dB = sizeof(float) * (size_t)P.depthWidth * P.depthHeight, cB = (size_t)4 * P.colorWidth * P.colorHeight;
    BF_CHECK(cudaMemcpyAsync(L.d_depthRaw, depth, dB, onHost ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, stream()));
    BF_CHECK(cudaMemcpyAsync(L.d_colorRaw, color, cB, onHost ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, stream()));
    int slot = -1;
    FL_OK(ingest_slot(L, frame, &slot));
    FL_OK(bfIngestFrame(&L.ingest, L.d_depthRaw, L.d_colorRaw, L.fs.depthOf(slot), L.fs.colorOf(slot)));
    float* depthFilt = L.fs.depthOf(slot);
    if (L.needSensorResFilter) { FL_OK(bfIngestFrame(&L.ingestSensorRes, L.d_depthRaw, L.d_colorRaw, L.d_depthFilt, L.d_colorRaw)); depthFilt = L.d_depthFilt; }
    // getCurrentFrame: intensity at SIFT resolution
    {
        dim3 blk(16, 16), grd((P.siftWidth + 15) / 16, (P.siftHeight + 15) / 16);
        fl_resample_intensity_kernel<<<grd, blk, 0, stream()>>>(L.d_intensity, P.siftWidth, P.siftHeight, reinterpret_cast<const uchar4*>(L.d_colorRaw), P.colorWidth, P.colorHeight);
        BF_CHECK(cudaGetLastError()); ++g_launchCount;
    }
    mark(L, 1);
    FL_OK(bfSiftDetect(&L.detect, L.d_intensity, depthFilt, b.sm.keysOf(li), b.sm.descsOf(li), b.sm.d_numKeys + li, nullptr));
    BF_CHECK(cudaMemcpyAsync(h_count, b.sm.d_numKeys + li, sizeof(int), cudaMemcpyDeviceToHost, stream()));
    mark(L, 2);
    FL_OK(b.cache.storeFrame(L.d_depthRaw, L.d_colorRaw));
    return write_back(L, frame);
}

// the front half of the NEXT frame on the feature stream (armed by bfFrameLoopStepAhead once this frame's bookkeeping has fixed the destinations)
static int launch_ahead(Loop& L) {
    L.aheadArmed = false;
    cudaStream_t mainStream = stream();
    BF_CHECK(cudaStreamWaitEvent(L.featStream, L.evStepStart, 0));      // after everything the library stream held when this step began (earlier users of the slots)
    bfSetStream(L.featStream);
    int rc = front_half(L, L.numFrames, L.nextDepth, L.nextColor, L.nextOnHost, *L.aheadTarget, L.aheadLi, L.h_pin + PIN_FEAT);
    if (!rc) { const cudaError_t e = cudaEventRecord(L.evFeat, L.featStream); if (e != cudaSuccess) { set_last_error("frame loop: cudaEventRecord(evFeat)", e); rc = (int)e; } }
    bfSetStream(mainStream);
    if (rc) return rc;
    L.ahead.valid = true; L.ahead.frame = L.numFrames; L.ahead.depth = L.nextDepth; L.ahead.color = L.nextColor; L.ahead.b = L.aheadTarget; L.ahead.li = L.aheadLi;
    L.featUsed = true;
    return 0;
}

// OnlineBundler::processInput (FL/OnlineBundler.cpp:167-227) for a NEW frame whose features (key slot of the current chunk, `nk` of them) and cache frame are in place
static int process_input(Loop& L, unsigned curFrame, int nkDetected) {
    const BFFrameLoopParams& P = L.P;
    const bool isLastLocal = is_last_local_frame(L, curFrame);
    Bundler& loc = *L.pLocal;
    const int nk = std::min(nkDetected, (int)P.maxNumKeysPerImage);
    loc.sm.addImage(nk);
    L.status.numKeyPoints = (unsigned)nk;
    const unsigned curLocalFrame = loc.sm.curFrame;
    if (isLastLocal) {                                   // the overlap frame opens the next chunk (Bundler::copyFrame, FL/Bundler.cpp:290-299)
        Bundler& o = *L.pOptLocal;
        const unsigned oi = o.sm.numImages;
        BF_CHECK(cudaMemcpyAsync(o.sm.keysOf(oi), loc.sm.keysOf(curLocalFrame), sizeof(BFSIFTKeyPoint) * (size_t)nk, cudaMemcpyDeviceToDevice, stream()));
        BF_CHECK(cudaMemcpyAsync(o.sm.descsOf(oi), loc.sm.descsOf(curLocalFrame), (size_t)128 * nk, cudaMemcpyDeviceToDevice, stream()));
        BF_CHECK(cudaMemcpyAsync(o.sm.d_numKeys + oi, loc.sm.d_numKeys + curLocalFrame, sizeof(int), cudaMemcpyDeviceToDevice, stream()));
        o.sm.addImage(nk);
        FL_OK(o.cache.copyFrom(loc.cache, curLocalFrame));
    }
    if (L.aheadWanted) {                                  // where the next frame's features go is settled: the chunk that will be current, its next slot
        L.aheadWanted = false;
        L.aheadTarget = isLastLocal ? L.pOptLocal : L.pLocal;           // prepare_local_solve (below) swaps the two on a chunk's last frame
        L.aheadLi = L.aheadTarget->sm.numImages;
        L.aheadArmed = true;                               // queued at the first host wait of this step (sync_stream), or at the end of this function
    }
    L.lastFrameValid = true;
    L.status.lastMatchedFrame = -1;
    if (curLocalFrame > 0) {
        int lm = -1;
        FL_OK(match_and_filter(L, loc, &lm));
        L.lastFrameValid = lm >= 0;
        L.status.lastMatchedFrame = lm;
        L.status.numLocalCorrespondences = (unsigned)loc.sm.globNum;
        // computeCurrentSiftTransform (:118-132)
        if (!L.lastFrameValid) {
            for (int k = 0; k < 16; ++k) L.currIntegrate[k] = kNegInf;
            BF_CHECK(cudaMemcpyAsync(L.d_siftTrajectory + 16 * (size_t)curFrame, L.d_siftTrajectory + 16 * (size_t)(curFrame - 1), 64, cudaMemcpyDeviceToDevice, stream()));
        } else if (curFrame > 0) {
            computeSiftTransformCU(loc.sm.d_filtTinv, loc.sm.d_numFilt, L.d_completeTrajectory, L.lastValidCompleteTransform, L.d_siftTrajectory, curFrame, curLocalFrame,
                                   L.d_currIntegrateTransform + 16 * (size_t)curFrame);
            BF_CHECK(cudaMemcpyAsync(L.h_pin + 32, L.d_currIntegrateTransform + 16 * (size_t)curFrame, 64, cudaMemcpyDeviceToHost, stream()));
            FL_OK(sync_stream(L));
            memcpy(L.currIntegrate, L.h_pin + 32, 64);
        }
    } else if (curFrame == 0) mat_identity(L.currIntegrate);
    if (L.aheadArmed) FL_OK(launch_ahead(L));
    if (isLastLocal) prepare_local_solve(L, curFrame, false);
    L.lastFrameProcessed = (int)curFrame;
    mark(L, 4);
    return 0;
}

// processInput when no new frame arrives (:171-197)
static void process_input_past_end(Loop& L) {
    const unsigned curFrame = L.numFrames - 1;
    if (L.numFramesPastEnd == 0 && L.localToSolve == -1 && !is_last_local_frame(L, curFrame)) prepare_local_solve(L, curFrame, true);
    ++L.numFramesPastEnd;
}

// OnlineBundler::optimizeLocal (:229-262)
static int optimize_local(Loop& L) {
    if (L.processState == Loop::DO_NOTHING) return 0;
    const int optState = L.processState;
    L.processState = Loop::DO_NOTHING;
    Bundler& o = *L.pOptLocal;
    unsigned curLocalIdx = 0xFFFFFFFFu;
    const unsigned numLocalFrames = std::min(L.P.submapSize, o.sm.numImages);
    if (optState == Loop::PROCESS) {
        curLocalIdx = (unsigned)L.localToSolve;
        bool removed = false, valid = false;
        FL_OK(bundler_optimize(L, o, L.P.numLocalNonLinIterations, L.P.numLocalLinIterations, L.P.useLocalVerify != 0, false, L.numFramesPastEnd != 0, &removed, &valid));
        ++L.counters[3];
        L.status.localSolved = (int)curLocalIdx; L.status.localValid = valid ? 1 : 0;
        if (valid) {
            BF_CHECK(cudaMemcpyAsync(L.d_localTrajectories + 16 * (size_t)(L.P.submapSize + 1) * curLocalIdx, o.d_trajectory, 64 * (size_t)(L.P.submapSize + 1), cudaMemcpyDeviceToDevice, stream()));
            L.processState = Loop::PROCESS;
        } else L.processState = Loop::INVALIDATE;
    } else if (optState == Loop::INVALIDATE) {
        curLocalIdx = (unsigned)(-L.localToSolve - 2);
        L.processState = Loop::INVALIDATE;
    }
    L.localToSolve = -1;
    L.lastLocalSolved = (int)curLocalIdx;
    L.totalNumOptLocalFrames = L.P.submapSize * (unsigned)L.lastLocalSolved + numLocalFrames;
    return 0;
}

// OnlineBundler::processGlobal (:271-358)
static int process_global(Loop& L) {
    const BFFrameLoopParams& P = L.P;
    Bundler& g = L.global; Bundler& o = *L.pOptLocal;
    const int ps = L.processState;
    if (ps == Loop::DO_NOTHING) {
        if (L.numFramesPastEnd != 0 && g.sm.numImages > 0) {        // sequence is over: still try re-validation
            unsigned idx; FL_OK(try_revalidation(L, (unsigned)L.lastLocalSolved, true, &idx));
            if (idx != 0xFFFFFFFFu && idx < L.localTrajectoriesValid.size()) {
                const std::vector<int>& v = L.localTrajectoriesValid[idx];
                for (unsigned i = 0; i < v.size(); ++i) if (v[i] == 1) validate_images(L, idx * P.submapSize + i);
                L.processState = Loop::PROCESS;
            }
        }
        return 0;
    }
    L.processState = Loop::DO_NOTHING;
    if (ps == Loop::PROCESS) {
        // fuse the solved chunk into the next keyframe (Bundler::fuseToGlobal, FL/Bundler.cpp:384-390)
        if (g.sm.numImages >= g.sm.maxImages) return (int)cudaErrorMemoryAllocation;
        const unsigned gi = g.sm.numImages;
        FL_OK(bfSiftFuseToGlobal(o.sm.d_glob, o.sm.d_globIdx, o.sm.d_globNum, o.d_trajectory, o.sm.numImages, o.sm.d_keys, o.sm.d_descs, o.sm.d_numKeys, o.sm.maxKeys, L.siftK,
                                 std::min(o.sm.maxResiduals, 4096u), g.sm.keysOf(gi), g.sm.descsOf(gi), g.sm.d_numKeys + gi, g.sm.maxKeys, nullptr));
        BF_CHECK(cudaMemcpyAsync(L.h_pin, g.sm.d_numKeys + gi, sizeof(int), cudaMemcpyDeviceToHost, stream()));
        FL_OK(g.cache.copyFrom(o.cache, 0));
        FL_OK(sync_stream(L));
        g.sm.addImage(L.h_pin[0]);
        const unsigned curGlobalFrame = g.sm.curFrame;
        const std::vector<int> validLocal(o.sm.valid.begin(), o.sm.valid.begin() + o.sm.numImages);
        const unsigned numLocalFrames = std::min(P.submapSize, o.sm.numImages);
        unsigned lastValidLocal = 0;
        for (int i = (int)o.sm.numImages - 1; i >= 0; --i) if (validLocal[i]) { lastValidLocal = (unsigned)i; break; }
        for (unsigned i = 0; i < numLocalFrames; ++i) if (validLocal[i] == 0) invalidate_images(L, curGlobalFrame * P.submapSize + i);
        if (curGlobalFrame < L.localTrajectoriesValid.size()) { L.localTrajectoriesValid[curGlobalFrame] = validLocal; L.localTrajectoriesValid[curGlobalFrame].resize(numLocalFrames); }
        // initializeNextGlobalTransform (:264-269)
        initNextGlobalTransformCU(g.d_trajectory, g.sm.numImages, curGlobalFrame, L.d_localTrajectories, lastValidLocal, P.submapSize + 1);
        FL_OK(bundler_reset(o));
        if (g.sm.numImages > 1) {
            int lm = -1;
            FL_OK(global_match_and_filter(L, &lm));
            if (lm < 0) { L.globalTrackingLost = true; L.processState = Loop::INVALIDATE; }
            else {
                L.globalTrackingLost = false;
                const unsigned rv = g.revalidatedIdx;
                if (rv != 0xFFFFFFFFu && rv < L.localTrajectoriesValid.size()) {
                    const std::vector<int>& v = L.localTrajectoriesValid[rv];
                    for (unsigned i = 0; i < v.size(); ++i) if (v[i] == 1) validate_images(L, rv * P.submapSize + i);
                }
                L.processState = Loop::PROCESS;
            }
        }
    } else if (ps == Loop::INVALIDATE) {
        L.processState = Loop::INVALIDATE;
        // Bundler::addInvalidFrame (FL/Bundler.cpp:362-368)
        if (g.sm.numImages >= g.sm.maxImages) return (int)cudaErrorMemoryAllocation;
        g.cache.incrementCache();
        const unsigned gi = g.sm.numImages;
        BF_CHECK(cudaMemsetAsync(g.sm.d_numKeys + gi, 0, sizeof(int), stream()));
        g.sm.addImage(0);
        BF_CHECK(cudaMemcpyAsync(g.d_trajectory + 16 * (size_t)g.sm.numImages, g.d_trajectory + 16 * (size_t)(g.sm.numImages - 1), 64, cudaMemcpyDeviceToDevice, stream()));   // initializeNextTransformUnknown
        FL_OK(bundler_reset(o));
        invalidate_images(L, P.submapSize * (unsigned)L.lastLocalSolved, L.totalNumOptLocalFrames);
    }
    L.status.numKeyframes = g.sm.numImages;
    L.status.numGlobalCorrespondences = (unsigned)g.sm.globNum;
    return 0;
}

// OnlineBundler::updateTrajectory + TrajectoryManager::updateOptimizedTransform (:360-368, 393-395)
static int update_trajectory(Loop& L, unsigned curFrame) {
    if (curFrame == 0) return 0;
    Bundler& g = L.global;
    BF_CHECK(cudaMemcpyAsync(L.d_imageInvalidateList, L.invalidImagesList.data(), sizeof(int) * curFrame, cudaMemcpyHostToDevice, stream()));
    updateTrajectoryCU(g.d_trajectory, g.sm.numImages, L.d_completeTrajectory, curFrame, L.d_localTrajectories, L.P.submapSize + 1, g.sm.numImages, L.d_imageInvalidateList);
    BF_CHECK(cudaMemcpyAsync(L.h_complete, L.d_completeTrajectory, 64 * (size_t)curFrame, cudaMemcpyDeviceToHost, stream()));
    FL_OK(sync_stream(L));
    bfTrajectoryUpdateOptimizedTransform(L.tm, L.h_complete, curFrame);
    L.numCompleteTransforms = curFrame;
    return 0;
}

// OnlineBundler::optimizeGlobal (:369-408)
static int optimize_global(Loop& L) {
    const BFFrameLoopParams& P = L.P;
    Bundler& g = L.global;
    const bool isSequenceDone = L.numFramesPastEnd > 0;
    if (!isSequenceDone && L.processState == Loop::DO_NOTHING) return 0;
    if (L.lastLocalSolved < 0) return 0;
    const int state = isSequenceDone ? (int)Loop::PROCESS : L.processState;
    const unsigned numTotalFrames = L.totalNumOptLocalFrames;
    if (state == Loop::PROCESS) {
        if (g.sm.numImages > 1) {
            const unsigned countNumFrames = (L.numFramesPastEnd > 0) ? L.numFramesPastEnd : numTotalFrames / P.submapSize;
            const bool removeMax = (countNumFrames % P.numOptPerResidualRemoval) == (P.numOptPerResidualRemoval - 1);
            bool removed = false, valid = false;
            const unsigned nNonLin = L.denseEndSolve ? 3u : P.numGlobalNonLinIterations;        // s_numGlobalNonLinIterations = 3 with the end weights (:181)
            FL_OK(bundler_optimize(L, g, nNonLin, P.numGlobalLinIterations, false, removeMax, L.numFramesPastEnd > 0, &removed, &valid));
            ++L.counters[4];
            if (L.denseEndSolve) {
                unsigned long long st[8];
                FL_OK(bfSolverGetStats(&g.solver.st, st));
                L.denseTurn = (int)L.numFramesPastEnd - 1; L.denseKeyframes = g.sm.numImages; L.densePairs = (unsigned)st[7];
            }
            L.status.globalSolved = 1; L.status.globalRemoved = removed ? 1 : 0;
            if (removed)
                for (unsigned i = 0; i < g.sm.numImages; ++i)
                    if (g.sm.valid[i] == 0) invalidate_images(L, i * P.submapSize, std::min((i + 1) * P.submapSize, numTotalFrames));
            FL_OK(update_trajectory(L, numTotalFrames));
            if (valid) L.lastValidCompleteTransform = P.submapSize * (unsigned)L.lastLocalSolved;
        } else FL_OK(update_trajectory(L, numTotalFrames));
    } else if (state == Loop::INVALIDATE) {
        if (g.sm.numImages > 1) g.sm.valid[g.sm.numImages - 1] = 0;                   // Bundler::invalidateLastFrame (the first chunk cannot be invalidated)
        invalidate_images(L, P.submapSize * (unsigned)L.lastLocalSolved, L.totalNumOptLocalFrames);
        FL_OK(update_trajectory(L, numTotalFrames));
    }
    L.processState = Loop::DO_NOTHING;
    return 0;
}

// ---- the voxel hash's buffers, and its growth (bf_frameloop.h, bfFrameLoopGetHashGrowth) ----------------------------------------------
// the buffers of a voxel hash of hp's sizes, as stream-ordered allocations on the library stream (bfTsdfReset initialises them); the heap
// counter, the d_hashDecision arrays and the list counter start zeroed
static void hash_free(BFHashDataStruct& hd) {
    void* p[9] = { hd.d_heap, hd.d_heapCounter, hd.d_hashDecision, hd.d_hashDecisionPrefix, hd.d_hash, hd.d_hashCompactified, hd.d_hashCompactifiedCounter,
                   hd.d_SDFBlocks, hd.d_hashBucketMutex };
    for (void* q : p) if (q) cudaFreeAsync(q, stream());
    memset(&hd, 0, sizeof(hd));
}
static int hash_alloc(BFHashDataStruct& hd, const BFHashParams& hp) {
    memset(&hd, 0, sizeof(hd));
    const size_t nE = (size_t)hp.m_hashNumBuckets * BF_HASH_BUCKET_SIZE;
    struct { void** p; size_t bytes; bool zero; } b[9] = {
        { (void**)&hd.d_heap, sizeof(uint32_t) * (size_t)hp.m_numSDFBlocks, false }, { (void**)&hd.d_heapCounter, sizeof(uint32_t), true },
        { (void**)&hd.d_hashDecision, sizeof(int32_t) * nE, true }, { (void**)&hd.d_hashDecisionPrefix, sizeof(int32_t) * nE, true },
        { (void**)&hd.d_hash, sizeof(BFHashEntry) * nE, false }, { (void**)&hd.d_hashCompactified, sizeof(BFHashEntry) * nE, false },
        { (void**)&hd.d_hashCompactifiedCounter, sizeof(int32_t), true }, { (void**)&hd.d_SDFBlocks, sizeof(BFVoxel) * BF_SDF_BLOCK_VOXELS * (size_t)hp.m_numSDFBlocks, false },
        { (void**)&hd.d_hashBucketMutex, sizeof(int32_t) * (size_t)hp.m_hashNumBuckets, false } };
    for (auto& x : b) {
        cudaError_t e = cudaMallocAsync(x.p, x.bytes, stream());
        if (e == cudaSuccess && x.zero) e = cudaMemsetAsync(*x.p, 0, x.bytes, stream());
        if (e != cudaSuccess) { set_last_error("frame loop: hash allocation", e); hash_free(hd); return (int)e; }
    }
    hd.m_bIsOnGPU = 1;
    return 0;
}

// the growth-size rule (bfFrameLoopHashGrowthSize): heap = min(ceiling, max(2 x old, live + 2 x reserve)); buckets at the initial ratio, odd,
// within the 32-bit entry-index limit
static unsigned grown_blocks(unsigned blocks, unsigned live, unsigned long long reserve, unsigned ceiling) {
    return (unsigned)std::min<unsigned long long>(std::max<unsigned long long>(2ull * blocks, live + 2ull * reserve), ceiling);
}
static unsigned grown_buckets(unsigned initBlocks, unsigned initBuckets, unsigned blocks) {
    const unsigned long long nb = (unsigned long long)initBuckets * blocks / std::max(initBlocks, 1u);
    return (unsigned)std::min<unsigned long long>(nb | 1ull, 0xFFFFFFFFull / BF_HASH_BUCKET_SIZE);
}

static int join_tsdf(Loop& L);
// Move the model into a table of `blocks` voxel blocks (buckets at the initial bucket-to-block ratio), before turn `turn`'s op list runs.
static int grow_hash(Loop& L, unsigned blocks, unsigned turn) {
    Loop::Growth& G = L.grow;
    FL_OK(join_tsdf(L));                                        // the old table's last work, queued on the reconstruction stream, comes first
    const unsigned long long cap = 0xFFFFFFFFull / BF_HASH_BUCKET_SIZE;
    for (int attempt = 0; attempt < 3; ++attempt) {
        BFHashParams hp = L.hp;
        const unsigned initBuckets = (unsigned)std::min<unsigned long long>((unsigned long long)G.initBuckets * G.bucketScale, cap);
        hp.m_numSDFBlocks = blocks; hp.m_hashNumBuckets = std::max(grown_buckets(G.initBlocks, initBuckets, blocks), L.hp.m_hashNumBuckets);
        BFHashDataStruct hd;
        FL_OK(hash_alloc(hd, hp));
        unsigned long long moved[2] = { 0, 0 };
        int rc = bfTsdfReset(&hd, &hp);
        if (!rc) rc = bfTsdfRehash(&L.hd, &L.hp, &hd, &hp, moved);
        L.counters[6] += BF_FRAMELOOP_GROWTH_SYNCS;
        if (rc) { bfTsdfReleaseAux(&hd); hash_free(hd); return rc; }
        if (moved[1] == 0) {
            bfTsdfReleaseAux(&L.hd);
            hash_free(L.hd);
            L.hd = hd; L.hp = hp;
            ++G.growths;
            // bfTsdfRehash synchronised: an exact sample of the state after the previous turn; a read-back still in flight is older
            G.pending = false; G.live = (unsigned)moved[0]; G.sampleTurn = turn - 1; G.dropRose = false;
            return 0;
        }
        // the new table's probe windows could not take every live block: discard it and keep the old one, which the rehash only read, and
        // try again with twice the buckets per block (kept for later growths)
        bfTsdfReleaseAux(&hd); hash_free(hd);
        ++G.discarded;
        if (hp.m_hashNumBuckets >= cap) break;
        G.bucketScale *= 2;
    }
    G.dropRose = false;                                         // no table took the model: the loop goes on with the old one
    return 0;
}

// At the start of turn `turn`'s reconstruction: take the last read-back if it has arrived (never waiting for it), then grow if the free
// blocks it saw are below the reserve or the dropped count rose.
static int maybe_grow(Loop& L, unsigned turn) {
    Loop::Growth& G = L.grow;
    if (G.pending) {
        const cudaError_t q = cudaEventQuery(G.ev);
        if (q == cudaErrorNotReady) cudaGetLastError();        // not an error: the read-back is still in flight
        else {
            BF_CHECK(q);
            G.pending = false;
            const unsigned c = G.h_stat[0];
            const unsigned freeBlocks = c >= 0x80000000u ? 0u : std::min(c + 1u, G.statBlocks);
            const unsigned live = G.statBlocks - freeBlocks;
            const unsigned long long dropped = (unsigned long long)G.h_stat[1] + G.h_stat[2];
            const unsigned before = G.sampled ? G.live : 0u;
            if (live > before) G.maxInc = std::max(G.maxInc, live - before);
            if (dropped > G.dropped) G.dropRose = true;
            G.live = live; G.dropped = dropped; G.sampleTurn = G.statTurn; G.sampled = true;
        }
    }
    if (!G.sampled) return 0;
    const unsigned blocks = L.hp.m_numSDFBlocks;
    const unsigned long long reserve = 2ull * G.maxInc * std::max(1u, turn - G.sampleTurn);
    if (!((unsigned long long)(blocks - std::min(G.live, blocks)) < reserve || G.dropRose)) return 0;
    const unsigned want = grown_blocks(blocks, G.live, reserve, L.P.hashMaxSDFBlocks);
    if (want <= blocks) { G.ceilingReached = true; G.dropRose = false; return 0; }
    return grow_hash(L, want, turn);
}

// reintegrate() (FL/DepthSensing/DepthSensing.cpp:854-902) + the integration of the current frame (:1033-1061): one op list, one bfTsdfRunOps
static int reconstruct(Loop& L, bool gotFrame, unsigned curFrame) {
    const BFFrameLoopParams& P = L.P;
    std::vector<BFTsdfOp> ops;
    if (bfTrajectoryGetNumActiveOperations(L.tm) < P.maxFrameFixes) bfTrajectoryGenerateUpdateLists(L.tm);
    unsigned nRe = 0;
    for (unsigned fixes = 0; fixes < P.maxFrameFixes; ++fixes) {
        float oldT[16], newT[16]; unsigned f = 0xFFFFFFFFu;
        BFTsdfOp op; memset(&op, 0, sizeof(op));
        if (bfTrajectoryGetTopFromDeIntegrateList(L.tm, oldT, &f)) { op.kind = BF_TSDF_OP_DEINTEGRATE; op.frame = (int)f; memcpy(op.pose, oldT, 64); ops.push_back(op); ++nRe; continue; }
        if (bfTrajectoryGetTopFromIntegrateList(L.tm, newT, &f)) { op.kind = BF_TSDF_OP_INTEGRATE; op.frame = (int)f; memcpy(op.pose, newT, 64); ops.push_back(op); bfTrajectoryConfirmIntegration(L.tm, f); ++nRe; continue; }
        if (bfTrajectoryGetTopFromReIntegrateList(L.tm, oldT, newT, &f)) {
            op.kind = BF_TSDF_OP_DEINTEGRATE; op.frame = (int)f; memcpy(op.pose, oldT, 64); ops.push_back(op);
            op.kind = BF_TSDF_OP_INTEGRATE; memcpy(op.pose, newT, 64); ops.push_back(op);
            bfTrajectoryConfirmIntegration(L.tm, f); ++nRe; continue;
        }
        break;
    }
    { BFTsdfOp gc; memset(&gc, 0, sizeof(gc)); gc.kind = BF_TSDF_OP_GARBAGE_COLLECT; ops.push_back(gc); }
    L.status.numReintegrated = nRe; L.counters[2] += nRe;
    if (gotFrame) {
        const bool validTransform = L.lastFrameValid;                       // getCurrentIntegrationFrame (:228-240)
        L.status.validTransform = validTransform ? 1 : 0; L.status.globalTrackingLost = L.globalTrackingLost ? 1 : 0;
        if (validTransform && P.reconstructionEnabled) {
            BFTsdfOp op; memset(&op, 0, sizeof(op)); op.kind = BF_TSDF_OP_INTEGRATE; op.frame = (int)curFrame; memcpy(op.pose, L.currIntegrate, 64); ops.push_back(op);
            bfTrajectoryAddFrame(L.tm, BF_TRAJ_INTEGRATED, L.currIntegrate, curFrame);
            memcpy(L.status.transform, L.currIntegrate, 64);
            ++L.counters[1];
        } else {
            float ninf[16]; for (int k = 0; k < 16; ++k) ninf[k] = kNegInf;
            bfTrajectoryAddFrame(L.tm, BF_TRAJ_NOT_INTEGRATED_NO_TRANSFORM, ninf, curFrame);
            memcpy(L.status.transform, ninf, 64);
        }
    }
    const unsigned turn = L.turn++;
    if (P.reconstructionEnabled) {
        if (L.opLogOn) { L.opLog.insert(L.opLog.end(), ops.begin(), ops.end()); L.opLogTurn.insert(L.opLogTurn.end(), ops.size(), turn); }
        if (L.grow.on) FL_OK(maybe_grow(L, turn));
        // the turn's frames into slots (bfTsdfRunOps reads depthPtrs / colorPtrs of these frames only, and not after it returns)
        std::vector<uint32_t> opFrames; std::vector<int> fetched;
        for (const BFTsdfOp& op : ops) if (op.kind != BF_TSDF_OP_GARBAGE_COLLECT) opFrames.push_back((uint32_t)op.frame);
        FL_OK(fetch_frames(L, opFrames.data(), (unsigned)opFrames.size(), &fetched));
        // inputs of this call that live on the main stream: the frame store (ingest of this frame) -- the poses and the op list are host data
        const bool side = L.overlap && !L.profile && L.tsdfStream;
        cudaStream_t mainStream = stream();
        if (side) { BF_CHECK(cudaEventRecord(L.evMain, mainStream)); BF_CHECK(cudaStreamWaitEvent(L.tsdfStream, L.evMain, 0)); bfSetStream(L.tsdfStream); }
        int rc = wait_fetched(L, fetched);
        if (!rc) rc = bfTsdfRunOps(&L.hd, &L.hp, &L.cam, ops.data(), (int)ops.size(), L.depthPtrs.data(), L.colorPtrs.data());
        if (!rc) rc = release_frames(L, opFrames.data(), (unsigned)opFrames.size());
        if (!rc && L.grow.on && !L.grow.pending) {              // read back this turn's heap and drop counters behind its work
            rc = tsdf_stats_async(&L.hd, L.grow.h_stat);
            if (!rc) rc = (int)cudaEventRecord(L.grow.ev, stream());
            L.grow.pending = rc == 0; L.grow.statTurn = turn; L.grow.statBlocks = L.hp.m_numSDFBlocks;
        }
        if (side) { cudaEventRecord(L.evTsdf, L.tsdfStream); L.tsdfPending = true; bfSetStream(mainStream); }
        if (rc) return rc;
    }
    if (gotFrame) { const int s = L.fs.slotOf[curFrame]; if (s >= 0) L.fs.pin[s] = 0; }     // the current frame's pin from its ingest
    return 0;
}
// the main stream waits for the reconstruction stream (asynchronously): before anything on it reads the voxel hash, and at the end of a timed region
static int join_tsdf(Loop& L) {
    if (L.tsdfPending) { BF_CHECK(cudaStreamWaitEvent(stream(), L.evTsdf, 0)); L.tsdfPending = false; }
    if (L.ahead.valid) BF_CHECK(cudaStreamWaitEvent(stream(), L.evFeat, 0));       // an announced frame's feature work, if any, is covered too
    return 0;
}

static int bundler_init(Loop& L, Bundler& b, bool isLocal, unsigned maxImages) {
    const BFFrameLoopParams& P = L.P;
    b.isLocal = isLocal;
    unsigned long long maxRes = (unsigned long long)BF_MAX_MATCHES_PER_IMAGE_PAIR_FILTERED * maxImages * (maxImages - 1) / 2;          // FL/Bundler.cpp:29
    if (!isLocal) { const unsigned long long cap = P.maxGlobalResiduals ? P.maxGlobalResiduals : (16ull << 20); if (maxRes > cap) maxRes = cap; }
    FL_OK(b.sm.init(L.A, maxImages, P.maxNumKeysPerImage, (unsigned)maxRes));
    FL_OK(b.cache.init(L.A, P, maxImages));
    FL_OK(b.solver.init(L.A, maxImages, (unsigned)maxRes));
    b.solver.maxResidualThresh = P.optMaxResThresh;
    b.d_trajectory = L.A.get<float>((size_t)(maxImages + 1) * 16);
    if (L.A.err) return L.A.err;
    fl_set_identity_kernel<<<((maxImages + 1) * 16 + 255) / 256, 256, 0, stream()>>>(b.d_trajectory, maxImages + 1);
    BF_CHECK(cudaGetLastError());
    return 0;
}

// the loop's table, and a growing loop's read-back slot and event (bfFrameLoopDestroy, or a failed bfFrameLoopCreate); the table's memory
// is back with the device when this returns
static void release_hash(Loop& L) {
    bfTsdfReleaseAux(&L.hd);
    hash_free(L.hd);
    cudaStreamSynchronize(stream());
    if (L.grow.h_stat) cudaFreeHost(L.grow.h_stat);
    if (L.grow.ev) cudaEventDestroy(L.grow.ev);
}

// the smallest non-zero deviceFrameSlots: one turn's re-integration frames, the current frame, the announced one, and one fusion batch
static unsigned min_frame_slots(const BFFrameLoopParams& P) { return std::max(P.maxFrameFixes + 2u, 16u); }

static int frame_store_init(Loop& L) {
    const BFFrameLoopParams& P = L.P;
    FrameStore& S = L.fs;
    S.px = (size_t)P.integrationWidth * P.integrationHeight;
    S.spill = P.deviceFrameSlots > 0;
    S.slots = S.spill ? P.deviceFrameSlots : P.maxNumFrames;
    S.d_depth = L.A.get<float>(S.px * S.slots, false); S.d_color = L.A.get<uint8_t>(S.px * 4 * S.slots, false);
    if (L.A.err) return L.A.err;
    S.slotOf.assign(P.maxNumFrames, -1); S.frameIn.assign(S.slots, -1); S.lastUse.assign(S.slots, 0); S.pin.assign(S.slots, 0);
    L.depthPtrs.assign(P.maxNumFrames, nullptr); L.colorPtrs.assign(P.maxNumFrames, nullptr);
    if (!S.spill) return 0;
    BF_CHECK(cudaStreamCreateWithFlags(&S.copy, cudaStreamNonBlocking));
    BF_CHECK(cudaEventCreateWithFlags(&S.evIngest, cudaEventDisableTiming));
    S.evRead.assign(S.slots, nullptr); S.evCopy.assign(S.slots, nullptr);
    for (unsigned s = 0; s < S.slots; ++s) {
        BF_CHECK(cudaEventCreateWithFlags(&S.evRead[s], cudaEventDisableTiming));
        BF_CHECK(cudaEventCreateWithFlags(&S.evCopy[s], cudaEventDisableTiming));
    }
    // the host store, pinned now: pinning inside a step would stall it
    const auto t0 = std::chrono::steady_clock::now();
    for (unsigned f = 0; f < P.maxNumFrames; f += FrameStore::kChunk) {
        const size_t bytes = (size_t)std::min(FrameStore::kChunk, P.maxNumFrames - f) * S.px * 8;
        void* p = nullptr;
        const cudaError_t e = cudaHostAlloc(&p, bytes, cudaHostAllocDefault);
        if (e != cudaSuccess) { set_last_error("bfFrameLoopCreate: the pinned host frame store", e); cudaGetLastError(); return (int)cudaErrorMemoryAllocation; }
        S.chunks.push_back(static_cast<uint8_t*>(p)); S.hostBytes += bytes;
    }
    S.pinMs = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}

static void frame_store_release(Loop& L) {
    FrameStore& S = L.fs;
    if (S.copy) cudaStreamSynchronize(S.copy);
    for (uint8_t* p : S.chunks) cudaFreeHost(p);
    for (cudaEvent_t e : S.evRead) if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : S.evCopy) if (e) cudaEventDestroy(e);
    if (S.evIngest) cudaEventDestroy(S.evIngest);
    if (S.copy) cudaStreamDestroy(S.copy);
    S.chunks.clear(); S.evRead.clear(); S.evCopy.clear(); S.evIngest = nullptr; S.copy = nullptr;
}

static void fill_status_tail(Loop& L) {
    L.status.numKeyframes = L.global.sm.numImages;
    L.status.numGlobalCorrespondences = (unsigned)L.global.sm.globNum;
    L.status.numOptimizedFrames = bfTrajectoryGetNumOptimizedFrames(L.tm);
    L.counters[7] = L.global.sm.numImages;
    if (L.status.globalSolved) {
        unsigned long long st[8];
        if (bfSolverGetStats(&L.global.solver.st, st) == 0) L.counters[5] = st[1];
    }
}

}  // namespace bf

using namespace bf;

BF_API void bfFrameLoopDefaultParams(BFFrameLoopParams* p, uint32_t width, uint32_t height) {
    memset(p, 0, sizeof(*p));
    p->depthWidth = p->colorWidth = p->integrationWidth = p->siftWidth = width;
    p->depthHeight = p->colorHeight = p->integrationHeight = p->siftHeight = height;
    float K[16]; mat_identity(K);
    K[0] = K[5] = 525.0f * (float)width / 640.0f; K[2] = ((float)width - 1.0f) / 2.0f; K[6] = ((float)height - 1.0f) / 2.0f;
    memcpy(p->depthIntrinsics, K, sizeof(K)); memcpy(p->colorIntrinsics, K, sizeof(K));
    p->submapSize = 10; p->maxNumImages = 1200; p->maxNumKeysPerImage = 1024; p->maxNumFrames = 12000; p->maxGlobalResiduals = 0;
    p->numLocalNonLinIterations = 2; p->numLocalLinIterations = 100; p->numGlobalNonLinIterations = 3; p->numGlobalLinIterations = 150; p->numOptPerResidualRemoval = 1;
    p->sensorDepthMin = 0.1f; p->sensorDepthMax = 4.0f; p->minKeyScale = 3.0f; p->featureCountThreshold = 150;
    p->siftMatchThresh = 0.7f; p->siftMatchRatioMaxLocal = 0.8f; p->siftMatchRatioMaxGlobal = 0.8f; p->minNumMatchesLocal = 5; p->minNumMatchesGlobal = 5;
    p->maxKabschResidual2 = 0.0004f; p->surfAreaPcaThresh = 0.032f;
    p->projCorrDistThres = 0.15f; p->projCorrNormalThres = 0.97f; p->projCorrColorThresh = 0.1f;
    p->verifySiftErrThresh = 0.075f; p->verifySiftCorrThresh = 0.02f; p->verifyOptErrThresh = 0.05f; p->verifyOptCorrThresh = 0.001f; p->optMaxResThresh = 0.08f;
    p->useLocalVerify = 1; p->useLocalDense = 1; p->useComprehensiveFrameInvalidation = 1;
    p->downsampledWidth = 80; p->downsampledHeight = 60; p->colorDownSigma = 2.5f; p->depthDownSigmaD = 1.0f; p->depthDownSigmaR = 0.05f;
    p->erodeSIFTdepth = 1; p->depthFilter = 1; p->depthSigmaD = 2.0f; p->depthSigmaR = 0.05f;
    p->maxFrameFixes = 10; p->topNActive = 30; p->minPoseDistSqrt = 0.0f; p->reconstructionEnabled = 1;
    BFHashParams& h = p->hash;
    h.m_hashNumBuckets = 800000; h.m_hashBucketSize = BF_HASH_BUCKET_SIZE; h.m_hashMaxCollisionLinkedListSize = 7; h.m_numSDFBlocks = 200000;
    h.m_SDFBlockSize = BF_SDF_BLOCK_SIZE; h.m_virtualVoxelSize = 0.010f; h.m_maxIntegrationDistance = 3.0f; h.m_truncScale = 0.02f; h.m_truncation = 0.06f;
    h.m_integrationWeightSample = 1; h.m_integrationWeightMax = 99999999;
    mat_identity(h.m_rigidTransform.m); mat_identity(h.m_rigidTransformInverse.m);
    p->renderDepthMin = 0.1f; p->renderDepthMax = 4.0f;
}

BF_API int bfFrameLoopCreate(const BFFrameLoopParams* params, BFFrameLoop** out) {
    if (!params || !out) return (int)cudaErrorInvalidValue;
    Loop* Lp = new Loop();
    Loop& L = *Lp;
    L.P = *params;
    const BFFrameLoopParams& P = L.P;
    if (P.maxNumFrames == 0 || P.submapSize == 0 || P.maxNumImages < 2) { delete Lp; return (int)cudaErrorInvalidValue; }
    if (P.deviceFrameSlots > 0 && P.deviceFrameSlots < min_frame_slots(P)) {
        set_last_error("bfFrameLoopCreate: deviceFrameSlots below max(maxFrameFixes + 2, 16)", cudaErrorInvalidValue);
        delete Lp; return (int)cudaErrorInvalidValue;
    }
    int rc = 0;
    do {
        L.d_depthRaw = L.A.get<float>((size_t)P.depthWidth * P.depthHeight); L.d_colorRaw = L.A.get<uint8_t>((size_t)P.colorWidth * P.colorHeight * 4);
        L.d_intensity = L.A.get<float>((size_t)P.siftWidth * P.siftHeight);
        L.needSensorResFilter = (P.integrationWidth != P.depthWidth || P.integrationHeight != P.depthHeight);
        if (L.needSensorResFilter) L.d_depthFilt = L.A.get<float>((size_t)P.depthWidth * P.depthHeight);
        // the device frame store: one slot per frame (deviceFrameSlots = 0), or deviceFrameSlots slots over a pinned host store of every frame
        if ((rc = frame_store_init(L))) break;
        memset(&L.ingest, 0, sizeof(L.ingest));
        L.ingest.depthWidth = P.depthWidth; L.ingest.depthHeight = P.depthHeight; L.ingest.colorWidth = P.colorWidth; L.ingest.colorHeight = P.colorHeight;
        L.ingest.widthIntegration = P.integrationWidth; L.ingest.heightIntegration = P.integrationHeight;
        L.ingest.erodeIterations = P.erodeSIFTdepth ? 2 : 0; L.ingest.erodeStructureSize = 3; L.ingest.erodeDThresh = 0.05f; L.ingest.erodeFracReq = 0.3f;
        L.ingest.depthSigmaD = P.depthFilter ? P.depthSigmaD : 0.0f; L.ingest.depthSigmaR = P.depthSigmaR;
        L.ingestSensorRes = L.ingest; L.ingestSensorRes.widthIntegration = P.depthWidth; L.ingestSensorRes.heightIntegration = P.depthHeight;
        // SIFT intrinsics: colour intrinsics scaled to the SIFT resolution (OnlineBundlerHelper.h:50-56)
        memcpy(L.siftK, P.colorIntrinsics, sizeof(L.siftK));
        L.siftK[0] *= (float)P.siftWidth / (float)P.colorWidth; L.siftK[5] *= (float)P.siftHeight / (float)P.colorHeight;
        L.siftK[2] *= (float)(P.siftWidth - 1) / (float)(P.colorWidth - 1); L.siftK[6] *= (float)(P.siftHeight - 1) / (float)(P.colorHeight - 1);
        intrinsics_inverse(L.siftK, L.siftKinv);
        memset(&L.detect, 0, sizeof(L.detect));
        L.detect.width = P.siftWidth; L.detect.height = P.siftHeight; L.detect.depthWidth = P.depthWidth; L.detect.depthHeight = P.depthHeight;
        L.detect.depthMin = P.sensorDepthMin; L.detect.depthMax = P.sensorDepthMax; L.detect.minKeyScale = P.minKeyScale;
        L.detect.featureCountThreshold = P.featureCountThreshold; L.detect.maxKeyPoints = P.maxNumKeysPerImage;
        if ((rc = bundler_init(L, L.local, true, P.submapSize + 1))) break;
        if ((rc = bundler_init(L, L.optLocal, true, P.submapSize + 1))) break;
        if ((rc = bundler_init(L, L.global, false, P.maxNumImages))) break;
        L.pLocal = &L.local; L.pOptLocal = &L.optLocal;
        const size_t nF = P.maxNumFrames;
        L.d_completeTrajectory = L.A.get<float>(nF * 16); L.d_siftTrajectory = L.A.get<float>(nF * 16); L.d_currIntegrateTransform = L.A.get<float>(nF * 16);
        L.d_localTrajectories = L.A.get<float>((size_t)P.maxNumImages * (P.submapSize + 1) * 16);
        L.d_imageInvalidateList = L.A.get<int>(nF);
        if (L.A.err) { rc = L.A.err; break; }
        fl_set_identity_kernel<<<((unsigned)(P.maxNumImages * (P.submapSize + 1)) * 16 + 255) / 256, 256, 0, stream()>>>(L.d_localTrajectories, P.maxNumImages * (P.submapSize + 1));
        fl_set_identity_kernel<<<1, 16, 0, stream()>>>(L.d_siftTrajectory, 1);
        fl_set_identity_kernel<<<1, 16, 0, stream()>>>(L.d_currIntegrateTransform, 1);
        L.invalidImagesList.assign(nF, 1); L.localTrajectoriesValid.resize(P.maxNumImages);
        mat_identity(L.currIntegrate);
        L.tm = bfTrajectoryCreate(P.maxNumFrames, P.topNActive, P.minPoseDistSqrt);
        // scene representation
        L.hp = P.hash; L.hp.m_hashBucketSize = BF_HASH_BUCKET_SIZE; L.hp.m_SDFBlockSize = BF_SDF_BLOCK_SIZE;
        if ((rc = hash_alloc(L.hd, L.hp))) break;
        L.grow.on = P.hashMaxSDFBlocks > L.hp.m_numSDFBlocks && L.hp.m_numSDFBlocks > 0;
        if (L.grow.on) {                 // a table the loop may replace: a pinned read-back slot and its event
            L.grow.initBlocks = L.hp.m_numSDFBlocks; L.grow.initBuckets = L.hp.m_hashNumBuckets;
            cudaError_t e = cudaMallocHost(&L.grow.h_stat, 4 * sizeof(unsigned));
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&L.grow.ev, cudaEventDisableTiming);
            if (e != cudaSuccess) { rc = (int)e; break; }
        }
        memset(&L.cam, 0, sizeof(L.cam));
        // integration camera: depth intrinsics scaled to the integration resolution (CUDAImageManager: m_depthIntrinsics adapted, cpp:60-70)
        L.cam.fx = P.depthIntrinsics[0] * (float)P.integrationWidth / (float)P.depthWidth; L.cam.fy = P.depthIntrinsics[5] * (float)P.integrationHeight / (float)P.depthHeight;
        L.cam.mx = P.depthIntrinsics[2] * (float)(P.integrationWidth - 1) / (float)(P.depthWidth - 1); L.cam.my = P.depthIntrinsics[6] * (float)(P.integrationHeight - 1) / (float)(P.depthHeight - 1);
        L.cam.m_imageWidth = P.integrationWidth; L.cam.m_imageHeight = P.integrationHeight; L.cam.m_sensorDepthWorldMin = P.renderDepthMin; L.cam.m_sensorDepthWorldMax = P.renderDepthMax;
        if ((rc = bfTsdfReset(&L.hd, &L.hp))) break;
        cudaError_t e = cudaMallocHost(&L.h_pin, sizeof(int) * 4096);
        if (e != cudaSuccess) { rc = (int)e; break; }
        e = cudaMallocHost(&L.h_complete, sizeof(float) * 16 * (size_t)P.maxNumFrames);
        if (e != cudaSuccess) { rc = (int)e; break; }
        // Library-private workspaces at their final size NOW: growing one later means cudaFree + cudaMalloc in the middle of a frame, and with the loop's other
        // streams busy that shows up as a single long stall.  Matcher: one job per keyframe at most;
        // solvers: the chunk's and the keyframe set's residual capacities (the keyframe solver's capped at 1 M entries up front, it doubles beyond)
        if ((rc = bfSiftReserveWorkspace(std::max(P.maxNumImages, P.submapSize + 1), P.maxNumKeysPerImage))) break;
        if ((rc = bfSolverReserveWorkspace(&L.local.solver.st, L.local.solver.maxImages, L.local.solver.maxResiduals, P.useLocalDense ? 1 : 0))) break;
        if ((rc = bfSolverReserveWorkspace(&L.optLocal.solver.st, L.optLocal.solver.maxImages, L.optLocal.solver.maxResiduals, P.useLocalDense ? 1 : 0))) break;
        if ((rc = bfSolverReserveWorkspace(&L.global.solver.st, L.global.solver.maxImages, std::min(L.global.solver.maxResiduals, 1u << 20), 0))) break;
        e = cudaStreamSynchronize(stream());
        if (e != cudaSuccess) { rc = (int)e; break; }
    } while (0);
    if (rc) {
        if (L.tm) bfTrajectoryDestroy(L.tm);
        if (L.h_pin) cudaFreeHost(L.h_pin);
        if (L.h_complete) cudaFreeHost(L.h_complete);
        release_hash(L);
        frame_store_release(L);
        delete Lp; return rc;
    }
    *out = reinterpret_cast<BFFrameLoop*>(Lp);
    return 0;
}

BF_API void bfFrameLoopDestroy(BFFrameLoop* loop) {
    if (!loop) return;
    Loop* L = reinterpret_cast<Loop*>(loop);
    if (L->tsdfStream) cudaStreamSynchronize(L->tsdfStream);
    if (L->featStream) cudaStreamSynchronize(L->featStream);
    cudaStreamSynchronize(stream());
    release_hash(*L);
    frame_store_release(*L);
    if (L->tsdfStream) cudaStreamDestroy(L->tsdfStream);
    if (L->featStream) cudaStreamDestroy(L->featStream);
    if (L->evStepStart) cudaEventDestroy(L->evStepStart);
    if (L->evFeat) cudaEventDestroy(L->evFeat);
    if (L->evMain) cudaEventDestroy(L->evMain);
    if (L->evTsdf) cudaEventDestroy(L->evTsdf);
    bfSolverReleaseWorkspace(&L->local.solver.st); bfSolverReleaseWorkspace(&L->optLocal.solver.st); bfSolverReleaseWorkspace(&L->global.solver.st);
    if (L->tm) bfTrajectoryDestroy(L->tm);
    if (L->h_pin) cudaFreeHost(L->h_pin);
    if (L->h_complete) cudaFreeHost(L->h_complete);
    delete L;
}

static int step_common(Loop& L, bool gotFrame, unsigned curFrame, BFFrameLoopStatus* status) {
    mark(L, 4);
    FL_OK(reconstruct(L, gotFrame, curFrame));
    mark(L, 5);
    if (L.useSolve) {                                   // OnlineBundler::process (:410-416)
        FL_OK(optimize_local(L));
        mark(L, 6);
        FL_OK(process_global(L));
        mark(L, 7);
        FL_OK(optimize_global(L));
    }
    mark(L, 8);
    stage_collect(L);
    fill_status_tail(L);
    if (status) *status = L.status;
    return 0;
}

static int ensure_feature_stream(Loop& L) {
    if (L.featStream) return 0;
    int lo = 0, hi = 0;
    BF_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    BF_CHECK(cudaStreamCreateWithPriority(&L.featStream, cudaStreamNonBlocking, lo));              // below the bundling chain, which stays the latency-critical one
    BF_CHECK(cudaEventCreateWithFlags(&L.evStepStart, cudaEventDisableTiming));
    BF_CHECK(cudaEventCreateWithFlags(&L.evFeat, cudaEventDisableTiming));
    return 0;
}

static int step_frame(Loop& L, const float* depth, const uint8_t* color, const float* nextDepth, const uint8_t* nextColor, int onHost, BFFrameLoopStatus* status) {
    const BFFrameLoopParams& P = L.P;
    if (L.numFrames >= P.maxNumFrames) return (int)cudaErrorMemoryAllocation;
    FL_OK(settle_lent(L));
    const unsigned curFrame = L.numFrames;
    memset(&L.status, 0, sizeof(L.status));
    L.status.frame = curFrame; L.status.localSolved = -1; L.status.lastMatchedFrame = -1;
    Bundler& loc = *L.pLocal;
    const unsigned li = loc.sm.numImages;
    int nk = 0;
    if (L.ahead.valid) {
        // this frame's front half was queued on the feature stream during the previous step: it must be the frame announced there
        if (L.ahead.frame != curFrame || L.ahead.depth != depth || L.ahead.color != color || L.ahead.b != &loc || L.ahead.li != li) {
            set_last_error("bfFrameLoopStep: the frame differs from the one announced as `next` by the previous bfFrameLoopStepAhead", cudaErrorInvalidValue);
            return (int)cudaErrorInvalidValue;
        }
        L.ahead.valid = false;
        ++L.counters[6];
        BF_CHECK(cudaEventSynchronize(L.evFeat));                       // the key-point count is on the host, keys / descriptors / cache frame / frame store slot are written
        nk = L.h_pin[PIN_FEAT];
    } else {
        if (L.featUsed) BF_CHECK(cudaStreamWaitEvent(stream(), L.evFeat, 0));          // raw-image buffers and the detector workspace were last used on the feature stream
        mark(L, 0);
        FL_OK(front_half(L, curFrame, depth, color, onHost, loc, li, L.h_pin));
        FL_OK(sync_stream(L));
        nk = L.h_pin[0];
    }
    mark(L, 3);
    ++L.numFrames; ++L.counters[0];
    L.aheadWanted = false; L.aheadArmed = false;
    if (nextDepth && nextColor && !L.profile && L.numFrames < P.maxNumFrames) {
        FL_OK(ensure_feature_stream(L));
        BF_CHECK(cudaEventRecord(L.evStepStart, stream()));
        L.nextDepth = nextDepth; L.nextColor = nextColor; L.nextOnHost = onHost; L.aheadWanted = true;
    }
    FL_OK(process_input(L, curFrame, nk));
    return step_common(L, true, curFrame, status);
}

BF_API int bfFrameLoopStep(BFFrameLoop* loop, const float* depth, const uint8_t* color, int onHost, BFFrameLoopStatus* status) {
    if (!loop || !depth || !color) return (int)cudaErrorInvalidValue;
    return step_frame(*reinterpret_cast<Loop*>(loop), depth, color, nullptr, nullptr, onHost, status);
}

BF_API int bfFrameLoopStepAhead(BFFrameLoop* loop, const float* depth, const uint8_t* color, const float* nextDepth, const uint8_t* nextColor, int onHost, BFFrameLoopStatus* status) {
    if (!loop || !depth || !color) return (int)cudaErrorInvalidValue;
    return step_frame(*reinterpret_cast<Loop*>(loop), depth, color, nextDepth, nextColor, onHost, status);
}

static int past_end_turn(Loop& L, BFFrameLoopStatus* status) {
    FL_OK(settle_lent(L));
    memset(&L.status, 0, sizeof(L.status));
    L.status.frame = L.numFrames - 1; L.status.localSolved = -1; L.status.lastMatchedFrame = -1;
    process_input_past_end(L);
    return step_common(L, false, L.numFrames - 1, status);
}

BF_API int bfFrameLoopStepPastEnd(BFFrameLoop* loop, BFFrameLoopStatus* status) {
    if (!loop) return (int)cudaErrorInvalidValue;
    Loop& L = *reinterpret_cast<Loop*>(loop);
    if (L.numFrames == 0) return (int)cudaErrorInvalidValue;
    if (L.ahead.valid) { set_last_error("bfFrameLoopStepPastEnd: a frame announced by bfFrameLoopStepAhead is still pending", cudaErrorInvalidValue); return (int)cudaErrorInvalidValue; }
    return past_end_turn(L, status);
}

BF_API int bfFrameLoopFinish(BFFrameLoop* loop, uint32_t numSolveFramesBeforeExit, uint32_t maxTurns, BFFrameLoopFinishInfo* info) {
    if (!loop) return (int)cudaErrorInvalidValue;
    Loop& L = *reinterpret_cast<Loop*>(loop);
    const unsigned K = numSolveFramesBeforeExit;
    if (L.numFrames == 0) { set_last_error("bfFrameLoopFinish: no frame has been stepped", cudaErrorInvalidValue); return (int)cudaErrorInvalidValue; }
    if (L.ahead.valid) { set_last_error("bfFrameLoopFinish: a frame announced by bfFrameLoopStepAhead is still pending", cudaErrorInvalidValue); return (int)cudaErrorInvalidValue; }
    if (L.finishK < 0 && L.numFramesPastEnd > K) {
        set_last_error("bfFrameLoopFinish: more past-end turns than numSolveFramesBeforeExit have run: the dense end solve's turn has passed", cudaErrorInvalidValue);
        return (int)cudaErrorInvalidValue;
    }
    if (L.finishK >= 0 && (unsigned)L.finishK != K) {
        set_last_error("bfFrameLoopFinish: numSolveFramesBeforeExit differs from the first call's", cudaErrorInvalidValue);
        return (int)cudaErrorInvalidValue;
    }
    L.finishK = (int)K;
    const unsigned long long solves0 = L.counters[4], reint0 = L.counters[2];
    unsigned turns = 0;
    while (!L.finished && turns < maxTurns) {
        // OnlineBundler::processInput past the end (FL/OnlineBundler.cpp:171-194): the turn's number is m_numFramesPastEnd before its increment
        const unsigned t = L.numFramesPastEnd;
        L.denseEndSolve = t == K && L.lastFrameProcessed < 10000;
        if (t == K + 1) L.useSolve = false;
        const int rc = past_end_turn(L, nullptr);
        L.denseEndSolve = false;
        if (rc) return rc;
        ++turns;
        // DepthSensing.cpp:1114-1126: from turn K + 1 on, regenerate the update lists; none left ends the run (StopScanningAndExit)
        if (t >= K + 1) {
            bfTrajectoryGenerateUpdateLists(L.tm);
            if (bfTrajectoryGetNumActiveOperations(L.tm) == 0) L.finished = true;
        }
    }
    FL_OK(join_tsdf(L));
    if (info) {
        memset(info, 0, sizeof(*info));
        info->turns = turns; info->numFramesPastEnd = L.numFramesPastEnd;
        info->denseTurn = L.denseTurn; info->denseKeyframes = L.denseKeyframes; info->densePairs = L.densePairs;
        info->globalSolves = (uint32_t)(L.counters[4] - solves0); info->reintegrations = (uint32_t)(L.counters[2] - reint0);
        // StopScanningAndExit (DepthSensing.cpp:922-932)
        std::vector<float> all((size_t)L.P.maxNumFrames * 16);
        const unsigned n = bfTrajectoryGetOptimizedTransforms(L.tm, all.data());
        unsigned nValid = 0;
        for (unsigned f = 0; f < n; ++f) if (all[16 * (size_t)f] != kNegInf) ++nValid;          // PoseHelper::countNumValidTransforms
        unsigned heapFree = 0;
        FL_OK(bfTsdfGetHeapFreeCount(&L.hd, &heapFree));
        info->numTransforms = n; info->numValidTransforms = nValid; info->heapFreeCount = heapFree;
        info->valid = (heapFree >= 800 && nValid >= (unsigned)std::round(0.5f * (float)n)) ? 1 : 0;
        info->done = L.finished ? 1 : 0;
    }
    return L.finished ? 0 : (int)cudaErrorNotReady;
}

BF_API int bfFrameLoopFuse(BFFrameLoop* loop, BFHashDataStruct* hd, BFHashParams* hp, const float* h_poses, uint32_t numFrames, BFFrameLoopFuseInfo* info) {
    if (!loop || !hd || !hp) return (int)cudaErrorInvalidValue;
    Loop& L = *reinterpret_cast<Loop*>(loop);
    if (L.ahead.valid) { set_last_error("bfFrameLoopFuse: a frame announced by bfFrameLoopStepAhead is still pending", cudaErrorInvalidValue); return (int)cudaErrorInvalidValue; }
    if (numFrames > L.numFrames) { set_last_error("bfFrameLoopFuse: numFrames exceeds the frames stepped", cudaErrorInvalidValue); return (int)cudaErrorInvalidValue; }
    if (hd->d_hash == L.hd.d_hash) { set_last_error("bfFrameLoopFuse: the target is the loop's own voxel hash", cudaErrorInvalidValue); return (int)cudaErrorInvalidValue; }
    std::vector<float> traj;
    if (!h_poses) {
        traj.assign((size_t)std::max(L.P.maxNumFrames, numFrames) * 16, kNegInf);
        bfTrajectoryGetOptimizedTransforms(L.tm, traj.data());          // frames it has no pose for stay -inf: skipped
        h_poses = traj.data();
    }
    FL_OK(settle_lent(L));
    FL_OK(join_tsdf(L));
    const bool batch = tsdf_batching_usable() != 0;
    BFFrameLoopFuseInfo fi; memset(&fi, 0, sizeof(fi));
    // the batches: the finite-pose frames in order, <= 16 per batch
    std::vector<std::vector<uint32_t>> bFrames; std::vector<std::vector<float>> bPoses;
    for (uint32_t f = 0; f < numFrames; ++f) {
        const float* T = h_poses + 16 * (size_t)f;
        bool finite = true;
        for (int e = 0; e < 16; ++e) finite = finite && std::isfinite(T[e]);
        if (!finite) { ++fi.framesSkipped; continue; }
        if (bFrames.empty() || bFrames.back().size() == 16) { bFrames.emplace_back(); bPoses.emplace_back(); }
        bFrames.back().push_back(f); bPoses.back().insert(bPoses.back().end(), T, T + 16);
    }
    // each batch is staged through slots; with room for two batches the next one is fetched while this one integrates
    const bool prefetch = L.fs.slots >= 32;
    std::vector<int> fetched[2];
    std::vector<BFTsdfOp> ops;
    for (size_t b = 0; b < bFrames.size(); ++b) {
        const std::vector<uint32_t>& fr = bFrames[b];
        const unsigned n = (unsigned)fr.size();
        if (b == 0 || !prefetch) FL_OK(fetch_frames(L, fr.data(), n, &fetched[b & 1]));
        if (prefetch && b + 1 < bFrames.size()) FL_OK(fetch_frames(L, bFrames[b + 1].data(), (unsigned)bFrames[b + 1].size(), &fetched[(b + 1) & 1]));
        FL_OK(wait_fetched(L, fetched[b & 1]));
        fetched[b & 1].clear();
        if (batch) {
            const std::vector<int32_t> frames(fr.begin(), fr.end());
            FL_OK(bfTsdfIntegrateBatch(hd, hp, &L.cam, frames.data(), bPoses[b].data(), (int)n, L.depthPtrs.data(), L.colorPtrs.data()));
            FL_OK(bfTsdfGarbageCollect(hd, hp));
        } else {
            ops.assign(n + 1, BFTsdfOp{});
            for (unsigned k = 0; k < n; ++k) { ops[k].kind = BF_TSDF_OP_INTEGRATE; ops[k].frame = (int32_t)fr[k]; memcpy(ops[k].pose, bPoses[b].data() + 16 * k, 64); }
            ops[n].kind = BF_TSDF_OP_GARBAGE_COLLECT;
            FL_OK(bfTsdfRunOps(hd, hp, &L.cam, ops.data(), (int)ops.size(), L.depthPtrs.data(), L.colorPtrs.data()));
        }
        FL_OK(release_frames(L, fr.data(), n));
        fi.framesFused += n; ++fi.batches;
    }
    unsigned long long st[4] = { 0, 0, 0, 0 };
    if (fi.batches) FL_OK(bfTsdfGetLastFrameStats(hd, st));
    fi.insertsDropped = st[3];
    FL_OK(bfTsdfGetHeapFreeCount(hd, &fi.heapFreeCount));
    if (info) *info = fi;
    return 0;
}

BF_API int bfFrameLoopGetGlobalProblem(const BFFrameLoop* loop, BFFrameLoopGlobalProblem* out) {
    if (!loop || !out) return (int)cudaErrorInvalidValue;
    const Loop& L = *reinterpret_cast<const Loop*>(loop);
    const Bundler& g = L.global;
    memset(out, 0, sizeof(*out));
    out->d_correspondences = g.sm.d_glob; out->numCorrespondences = (uint32_t)g.sm.globNum;
    out->numKeyframes = g.sm.numImages; out->d_validImages = g.sm.d_valid; out->d_trajectory = g.d_trajectory;
    out->d_cacheFrames = g.cache.d_frames; out->cacheWidth = g.cache.w; out->cacheHeight = g.cache.h;
    out->intrinsics[0] = g.cache.K[0]; out->intrinsics[1] = g.cache.K[5]; out->intrinsics[2] = g.cache.K[2]; out->intrinsics[3] = g.cache.K[6];
    out->maxNumImages = g.solver.maxImages; out->maxCorrPerImage = g.solver.maxCorrPerImage;
    return 0;
}

BF_API int bfFrameLoopGetKeyframes(const BFFrameLoop* loop, BFKeyframeSet* out) {
    if (!loop || !out) return (int)cudaErrorInvalidValue;
    const Loop& L = *reinterpret_cast<const Loop*>(loop);
    const Bundler& g = L.global;
    memset(out, 0, sizeof(*out));
    out->numImages = g.sm.numImages; out->maxKeys = g.sm.maxKeys;
    out->d_keyPoints = g.sm.d_keys; out->d_descriptors = g.sm.d_descs; out->d_numKeys = g.sm.d_numKeys;
    out->d_cacheFrames = g.cache.d_frames; out->cacheWidth = g.cache.w; out->cacheHeight = g.cache.h;
    memcpy(out->cacheIntrinsics, g.cache.K, sizeof(out->cacheIntrinsics));
    memcpy(out->siftIntrinsicsInv, L.siftKinv, sizeof(out->siftIntrinsicsInv));
    return 0;
}

BF_API unsigned int bfFrameLoopGetTrajectory(BFFrameLoop* loop, float* h_out, unsigned int maxFrames) {
    if (!loop || !h_out) return 0;
    Loop& L = *reinterpret_cast<Loop*>(loop);
    std::vector<float> all((size_t)L.P.maxNumFrames * 16);
    const unsigned n = bfTrajectoryGetOptimizedTransforms(L.tm, all.data());
    const unsigned m = std::min(n, maxFrames);
    memcpy(h_out, all.data(), (size_t)m * 64);
    return m;
}
BF_API const BFHashDataStruct* bfFrameLoopGetHashData(const BFFrameLoop* loop) {
    if (!loop) return nullptr;
    join_tsdf(*const_cast<Loop*>(reinterpret_cast<const Loop*>(loop)));          // work the caller queues on the library stream after this call sees the fused model
    return &reinterpret_cast<const Loop*>(loop)->hd;
}
BF_API int bfFrameLoopSetOpLog(BFFrameLoop* loop, int enable) {
    if (!loop) return (int)cudaErrorInvalidValue;
    Loop& L = *reinterpret_cast<Loop*>(loop);
    const int prev = L.opLogOn ? 1 : 0;
    if (enable && !L.opLogOn) { L.opLog.clear(); L.opLogTurn.clear(); }
    L.opLogOn = enable != 0;
    return prev;
}
BF_API uint32_t bfFrameLoopGetOpLog(const BFFrameLoop* loop, BFTsdfOp* out, uint32_t* turnOfOp, uint32_t maxOps) {
    if (!loop) return 0;
    const Loop& L = *reinterpret_cast<const Loop*>(loop);
    const size_t m = std::min<size_t>(L.opLog.size(), maxOps);
    if (out) std::copy(L.opLog.begin(), L.opLog.begin() + m, out);
    if (turnOfOp) std::copy(L.opLogTurn.begin(), L.opLogTurn.begin() + m, turnOfOp);
    return (uint32_t)L.opLog.size();
}
BF_API int bfFrameLoopFetchFrames(BFFrameLoop* loop, const uint32_t* frames, uint32_t n, const float** depth, const uint8_t** color) {
    if (!loop || !frames || !depth || !color) return (int)cudaErrorInvalidValue;
    Loop& L = *reinterpret_cast<Loop*>(loop);
    if ((unsigned long long)n + 2 > L.fs.slots) { set_last_error("bfFrameLoopFetchFrames: more than deviceFrameSlots - 2 frames", cudaErrorInvalidValue); return (int)cudaErrorInvalidValue; }
    for (uint32_t k = 0; k < n; ++k)
        if (frames[k] >= L.numFrames) { set_last_error("bfFrameLoopFetchFrames: a frame has not been stepped", cudaErrorInvalidValue); return (int)cudaErrorInvalidValue; }
    FL_OK(settle_lent(L));
    FL_OK(join_tsdf(L));                    // every earlier reader of a slot is on the library stream: its next read event covers them all
    std::vector<int> fetched;
    FL_OK(fetch_frames(L, frames, n, &fetched));
    FL_OK(wait_fetched(L, fetched));
    for (uint32_t k = 0; k < n; ++k) {
        depth[k] = L.depthPtrs[frames[k]]; color[k] = L.colorPtrs[frames[k]];
        const int s = L.fs.slotOf[frames[k]];
        if (L.fs.pin[s]) { L.fs.pin[s] = 0; L.fs.lent.push_back(s); }
    }
    return 0;
}
BF_API int bfFrameLoopGetFrame(const BFFrameLoop* loop, uint32_t f, const float** depth, const uint8_t** color) {
    if (!loop || !depth || !color) return (int)cudaErrorInvalidValue;
    const Loop& L = *reinterpret_cast<const Loop*>(loop);
    if (f >= L.numFrames) { set_last_error("bfFrameLoopGetFrame: the frame has not been stepped", cudaErrorInvalidValue); return (int)cudaErrorInvalidValue; }
    if (L.fs.spill) return bfFrameLoopFetchFrames(const_cast<BFFrameLoop*>(loop), &f, 1, depth, color);
    *depth = L.depthPtrs[f]; *color = L.colorPtrs[f];
    return 0;
}
BF_API int bfFrameLoopGetFrameStore(const BFFrameLoop* loop, BFFrameLoopFrameStore* out) {
    if (!loop || !out) return (int)cudaErrorInvalidValue;
    const FrameStore& S = reinterpret_cast<const Loop*>(loop)->fs;
    memset(out, 0, sizeof(*out));
    out->slots = S.slots; out->hostStore = S.spill ? 1 : 0;
    unsigned resident = 0;
    for (int f : S.frameIn) resident += f >= 0 ? 1u : 0u;
    out->residentFrames = resident;
    out->deviceBytes = (unsigned long long)S.slots * S.px * 8; out->hostBytes = S.hostBytes;
    out->writeBacks = S.writeBacks; out->fetches = S.fetches; out->hits = S.hits; out->evictions = S.evictions;
    out->h2dBytes = S.h2d; out->d2hBytes = S.d2h; out->pinMs = S.pinMs;
    return 0;
}
BF_API int bfFrameLoopJoin(BFFrameLoop* loop) { return loop ? join_tsdf(*reinterpret_cast<Loop*>(loop)) : (int)cudaErrorInvalidValue; }
BF_API int bfFrameLoopSetOverlap(BFFrameLoop* loop, int enable) {
    if (!loop) return (int)cudaErrorInvalidValue;
    Loop& L = *reinterpret_cast<Loop*>(loop);
    const int prev = L.overlap ? 1 : 0;
    if (enable && !L.tsdfStream) {
        int lo = 0, hi = 0;
        BF_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        BF_CHECK(cudaStreamCreateWithPriority(&L.tsdfStream, cudaStreamNonBlocking, lo));          // lowest priority: the bundling chain is the latency-critical one
        BF_CHECK(cudaEventCreateWithFlags(&L.evMain, cudaEventDisableTiming));
        BF_CHECK(cudaEventCreateWithFlags(&L.evTsdf, cudaEventDisableTiming));
    }
    if (!enable) { const int rc = join_tsdf(L); if (rc) return rc; }
    L.overlap = enable != 0;
    return prev;
}
BF_API const BFHashParams* bfFrameLoopGetHashParams(const BFFrameLoop* loop) { return loop ? &reinterpret_cast<const Loop*>(loop)->hp : nullptr; }
BF_API void bfFrameLoopHashGrowthSize(uint32_t blocks, uint32_t live, unsigned long long reserve, uint32_t ceiling, uint32_t initBlocks, uint32_t initBuckets,
                                      uint32_t* newBlocks, uint32_t* newBuckets) {
    const unsigned b = grown_blocks(blocks, live, reserve, ceiling);
    if (newBlocks) *newBlocks = b;
    if (newBuckets) *newBuckets = grown_buckets(initBlocks, initBuckets, b);
}
BF_API int bfFrameLoopGetHashGrowth(BFFrameLoop* loop, BFFrameLoopHashGrowth* out) {
    if (!loop || !out) return (int)cudaErrorInvalidValue;
    Loop& L = *reinterpret_cast<Loop*>(loop);
    FL_OK(join_tsdf(L));
    unsigned long long st[4] = { 0, 0, 0, 0 };
    FL_OK(bfTsdfGetLastFrameStats(&L.hd, st));          // out[3]: drops since the reset, carried across every rehash
    memset(out, 0, sizeof(*out));
    out->growths = L.grow.growths; out->discarded = L.grow.discarded; out->sdfBlocks = L.hp.m_numSDFBlocks; out->buckets = L.hp.m_hashNumBuckets;
    out->maxSDFBlocks = L.grow.on ? L.P.hashMaxSDFBlocks : L.hp.m_numSDFBlocks;
    out->insertsDropped = st[3]; out->ceilingReached = L.grow.ceilingReached ? 1 : 0;
    return 0;
}
BF_API int bfFrameLoopSetProfiling(BFFrameLoop* loop, int enable) {
    if (!loop) return (int)cudaErrorInvalidValue;
    Loop& L = *reinterpret_cast<Loop*>(loop);
    if (enable) for (int k = 0; k <= BF_FRAMELOOP_STAGES; ++k) if (!L.stageEv[k]) BF_CHECK(cudaEventCreate(&L.stageEv[k]));
    L.profile = enable != 0;
    for (int k = 0; k < BF_FRAMELOOP_STAGES; ++k) L.stageMs[k] = 0.0;
    for (int k = 0; k <= BF_FRAMELOOP_STAGES; ++k) L.stageHit[k] = false;
    L.profiledSteps = 0;
    return 0;
}
BF_API unsigned long long bfFrameLoopGetStageTimes(const BFFrameLoop* loop, double outMs[BF_FRAMELOOP_STAGES]) {
    if (!loop) return 0;
    const Loop& L = *reinterpret_cast<const Loop*>(loop);
    for (int k = 0; k < BF_FRAMELOOP_STAGES; ++k) outMs[k] = L.stageMs[k];
    return L.profiledSteps;
}
BF_API void bfFrameLoopGetCounters(const BFFrameLoop* loop, unsigned long long out[8]) {
    if (!loop) return;
    memcpy(out, reinterpret_cast<const Loop*>(loop)->counters, sizeof(unsigned long long) * 8);
}

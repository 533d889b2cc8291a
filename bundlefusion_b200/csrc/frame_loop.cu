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
#include <cmath>
#include <cstring>
#include <list>
#include <vector>

#include "../../include/bf_bundler.h"
#include "../../include/bf_cache.h"
#include "../../include/bf_frameloop.h"
#include "../../include/bf_host.h"
#include "../../include/bf_ingest.h"
#include "../../include/bf_sift.h"
#include "../../include/bf_solver.h"
#include "bf_common.cuh"
#include "mat4.cuh"

namespace bf {

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

struct Loop {
    BFFrameLoopParams P;
    Arena A;
    // frame input / store
    float* d_depthRaw = nullptr; uint8_t* d_colorRaw = nullptr; float* d_depthFilt = nullptr; float* d_intensity = nullptr;
    std::vector<float*> d_frameDepth; std::vector<uint8_t*> d_frameColor;      // integration-resolution frame store (CUDAImageManager's frames, kept on the device)
    std::vector<const float*> depthPtrs; std::vector<const uint8_t*> colorPtrs;
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
    unsigned numFrames = 0;                      // frames received (CUDAImageManager::getCurrFrameNumber() + 1)
    float currIntegrate[16];
    BFTrajectoryManager* tm = nullptr;
    // scene
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
    FL_OK(bfIngestFrame(&L.ingest, L.d_depthRaw, L.d_colorRaw, L.d_frameDepth[frame], L.d_frameColor[frame]));
    float* depthFilt = L.d_frameDepth[frame];
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
    return 0;
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
            FL_OK(bundler_optimize(L, g, P.numGlobalNonLinIterations, P.numGlobalLinIterations, false, removeMax, L.numFramesPastEnd > 0, &removed, &valid));
            ++L.counters[4];
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
    if (P.reconstructionEnabled) {
        // inputs of this call that live on the main stream: the frame store (ingest of this frame) -- the poses and the op list are host data
        const bool side = L.overlap && !L.profile && L.tsdfStream;
        cudaStream_t mainStream = stream();
        if (side) { BF_CHECK(cudaEventRecord(L.evMain, mainStream)); BF_CHECK(cudaStreamWaitEvent(L.tsdfStream, L.evMain, 0)); bfSetStream(L.tsdfStream); }
        const int rc = bfTsdfRunOps(&L.hd, &L.hp, &L.cam, ops.data(), (int)ops.size(), L.depthPtrs.data(), L.colorPtrs.data());
        if (side) { cudaEventRecord(L.evTsdf, L.tsdfStream); L.tsdfPending = true; bfSetStream(mainStream); }
        if (rc) return rc;
    }
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
    int rc = 0;
    do {
        L.d_depthRaw = L.A.get<float>((size_t)P.depthWidth * P.depthHeight); L.d_colorRaw = L.A.get<uint8_t>((size_t)P.colorWidth * P.colorHeight * 4);
        L.d_intensity = L.A.get<float>((size_t)P.siftWidth * P.siftHeight);
        L.needSensorResFilter = (P.integrationWidth != P.depthWidth || P.integrationHeight != P.depthHeight);
        if (L.needSensorResFilter) L.d_depthFilt = L.A.get<float>((size_t)P.depthWidth * P.depthHeight);
        // the device frame store: every frame's integration-resolution depth + colour stays resident for re-integration
        {
            const size_t px = (size_t)P.integrationWidth * P.integrationHeight;
            float* allD = L.A.get<float>(px * P.maxNumFrames, false); uint8_t* allC = L.A.get<uint8_t>(px * 4 * P.maxNumFrames, false);
            if (L.A.err) { rc = L.A.err; break; }
            L.d_frameDepth.resize(P.maxNumFrames); L.d_frameColor.resize(P.maxNumFrames); L.depthPtrs.resize(P.maxNumFrames); L.colorPtrs.resize(P.maxNumFrames);
            for (unsigned f = 0; f < P.maxNumFrames; ++f) { L.d_frameDepth[f] = allD + px * f; L.d_frameColor[f] = allC + px * 4 * f; L.depthPtrs[f] = L.d_frameDepth[f]; L.colorPtrs[f] = L.d_frameColor[f]; }
        }
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
        const size_t nEntries = (size_t)L.hp.m_hashNumBuckets * BF_HASH_BUCKET_SIZE;
        memset(&L.hd, 0, sizeof(L.hd));
        L.hd.d_heap = L.A.get<uint32_t>(L.hp.m_numSDFBlocks, false); L.hd.d_heapCounter = L.A.get<uint32_t>(1);
        L.hd.d_hashDecision = L.A.get<int32_t>(nEntries); L.hd.d_hashDecisionPrefix = L.A.get<int32_t>(nEntries);
        L.hd.d_hash = L.A.get<BFHashEntry>(nEntries, false); L.hd.d_hashCompactified = L.A.get<BFHashEntry>(nEntries, false);
        L.hd.d_hashCompactifiedCounter = L.A.get<int32_t>(1);
        L.hd.d_SDFBlocks = L.A.get<BFVoxel>((size_t)L.hp.m_numSDFBlocks * BF_SDF_BLOCK_VOXELS, false);
        L.hd.d_hashBucketMutex = L.A.get<int32_t>(L.hp.m_hashNumBuckets, false);
        L.hd.m_bIsOnGPU = 1;
        if (L.A.err) { rc = L.A.err; break; }
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
    if (rc) { if (L.tm) bfTrajectoryDestroy(L.tm); if (L.h_pin) cudaFreeHost(L.h_pin); if (L.h_complete) cudaFreeHost(L.h_complete); delete Lp; return rc; }
    *out = reinterpret_cast<BFFrameLoop*>(Lp);
    return 0;
}

BF_API void bfFrameLoopDestroy(BFFrameLoop* loop) {
    if (!loop) return;
    Loop* L = reinterpret_cast<Loop*>(loop);
    if (L->tsdfStream) cudaStreamSynchronize(L->tsdfStream);
    if (L->featStream) cudaStreamSynchronize(L->featStream);
    cudaStreamSynchronize(stream());
    bfTsdfReleaseAux(&L->hd);
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

BF_API int bfFrameLoopStepPastEnd(BFFrameLoop* loop, BFFrameLoopStatus* status) {
    if (!loop) return (int)cudaErrorInvalidValue;
    Loop& L = *reinterpret_cast<Loop*>(loop);
    if (L.numFrames == 0) return (int)cudaErrorInvalidValue;
    if (L.ahead.valid) { set_last_error("bfFrameLoopStepPastEnd: a frame announced by bfFrameLoopStepAhead is still pending", cudaErrorInvalidValue); return (int)cudaErrorInvalidValue; }
    memset(&L.status, 0, sizeof(L.status));
    L.status.frame = L.numFrames - 1; L.status.localSolved = -1; L.status.lastMatchedFrame = -1;
    process_input_past_end(L);
    return step_common(L, false, L.numFrames - 1, status);
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

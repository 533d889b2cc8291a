// keyframe_search.cu -- the all-pairs correspondence search of include/bf_keyframe_search.h for sm_90a.
//
// A call walks its pair range in waves of BF_KEYFRAME_SEARCH_WAVE pairs of the canonical order p(i, j) = j (j - 1) / 2 + i.  Per wave:
//   1. kf_build_jobs: the wave's match jobs, built on the device from p alone (image i against image j, offsets (i maxKeys, j maxKeys)) --
//      no host job table, and the scratch of job b sits at b * maxKeys;
//   2. the wgmma + TMA sweep of bfSiftMatchBatch (sift_best_wgmma_kernel, row pass then column pass, unchanged) over that table, with one
//      tensor map per image encoded once per call: the raw matches are bfSiftMatchBatch's bytes by construction;
//   3. sort, Kabsch filter, surface-area filter and dense verify: the frame loop's kernels, each launched once for the whole wave with a
//      canonical PairList (sift_pairs.cuh);
//   4. kf_wave_stats (pairs with raw matches, pairs surviving, the optional per-pair filtered count), then the residual append of
//      bfSiftAddCurrToResiduals with the running total carried on the device: a scan of the wave's counts, entries written in canonical order.
// Nine launches per wave, whatever N is.  The workspace holds one wave (plus one tensor map per image), never the N^2 pair set.
//
// Bound: the sweep forms each dot product twice (row pass and column pass, as bfSiftMatchBatch does) and its cost is the per-product best /
// second-best bookkeeping on the integer pipe, not the tensor-core contraction (sift_match.cu); the filters are a fixed cost per pair.
#include <cuda.h>

#include <algorithm>
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/bf_keyframe_search.h"
#include "bf_common.cuh"
#include "sift_pairs.cuh"
#include "sift_sweep.cuh"

namespace bf {

extern unsigned long long g_launchCount;

#define KF_RAW BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW
#define KF_FILT BF_MAX_MATCHES_PER_IMAGE_PAIR_FILTERED
#define KF_OK(expr) do { const int _rc = (int)(expr); if (_rc) return _rc; } while (0)

struct KfBufs {
    unsigned keyCap = 0, imgCap = 0;
    SiftJobDev* jobs = nullptr;                              // [2 W]
    int* rowResult = nullptr; float* rowDist = nullptr; int* colResult = nullptr;      // [W * keyCap]
    int* done = nullptr;                                     // [W], each job's last column CTA leaves it at 0
    int* rawNum = nullptr; float* rawDist = nullptr; uint2* rawIdx = nullptr;
    int* numFilt = nullptr; float* fDist = nullptr; uint2* fIdx = nullptr; float* fT = nullptr; float* fTinv = nullptr;
    unsigned long long* counters = nullptr;                  // [2]: pairs with raw matches, pairs surviving
    CUtensorMap* maps = nullptr;                             // [imgCap]
};
struct KfWs : KfBufs {
    std::vector<CUtensorMap> hMaps;
    std::vector<int> hKeys;
    cudaEvent_t evDone = nullptr;
};
static KfWs g_kf;
static std::mutex g_kfMutex;

static void kf_free() {
    cudaFree(g_kf.jobs); cudaFree(g_kf.rowResult); cudaFree(g_kf.rowDist); cudaFree(g_kf.colResult); cudaFree(g_kf.done);
    cudaFree(g_kf.rawNum); cudaFree(g_kf.rawDist); cudaFree(g_kf.rawIdx); cudaFree(g_kf.numFilt); cudaFree(g_kf.fDist); cudaFree(g_kf.fIdx);
    cudaFree(g_kf.fT); cudaFree(g_kf.fTinv); cudaFree(g_kf.counters); cudaFree(g_kf.maps);
}
static int kf_reserve(cudaStream_t s, unsigned numImages, unsigned maxKeys) {
    if (!g_kf.evDone) BF_CHECK(cudaEventCreateWithFlags(&g_kf.evDone, cudaEventDisableTiming));
    if (maxKeys <= g_kf.keyCap && numImages <= g_kf.imgCap) return 0;
    BF_CHECK(cudaStreamWaitEvent(s, g_kf.evDone, 0));
    BF_CHECK(cudaStreamSynchronize(s));
    const unsigned keyCap = std::max(maxKeys, g_kf.keyCap), imgCap = std::max(numImages, g_kf.imgCap);
    kf_free();
    static_cast<KfBufs&>(g_kf) = KfBufs();
    const size_t W = BF_KEYFRAME_SEARCH_WAVE, F = W * keyCap;
    BF_CHECK(cudaMalloc(&g_kf.jobs, sizeof(SiftJobDev) * 2 * W));
    BF_CHECK(cudaMalloc(&g_kf.rowResult, sizeof(int) * F)); BF_CHECK(cudaMalloc(&g_kf.rowDist, sizeof(float) * F)); BF_CHECK(cudaMalloc(&g_kf.colResult, sizeof(int) * F));
    BF_CHECK(cudaMalloc(&g_kf.done, sizeof(int) * W));
    BF_CHECK(cudaMemsetAsync(g_kf.done, 0, sizeof(int) * W, s));
    BF_CHECK(cudaMalloc(&g_kf.rawNum, sizeof(int) * W)); BF_CHECK(cudaMalloc(&g_kf.rawDist, sizeof(float) * W * KF_RAW)); BF_CHECK(cudaMalloc(&g_kf.rawIdx, sizeof(uint2) * W * KF_RAW));
    BF_CHECK(cudaMalloc(&g_kf.numFilt, sizeof(int) * W)); BF_CHECK(cudaMalloc(&g_kf.fDist, sizeof(float) * W * KF_FILT)); BF_CHECK(cudaMalloc(&g_kf.fIdx, sizeof(uint2) * W * KF_FILT));
    BF_CHECK(cudaMalloc(&g_kf.fT, sizeof(float) * 16 * W)); BF_CHECK(cudaMalloc(&g_kf.fTinv, sizeof(float) * 16 * W));
    BF_CHECK(cudaMalloc(&g_kf.counters, sizeof(unsigned long long) * 2));
    BF_CHECK(cudaMalloc(&g_kf.maps, sizeof(CUtensorMap) * imgCap));
    g_kf.keyCap = keyCap; g_kf.imgCap = imgCap;
    return 0;
}
static size_t kf_bytes() {
    const size_t W = BF_KEYFRAME_SEARCH_WAVE;
    if (!g_kf.keyCap) return 0;
    return sizeof(SiftJobDev) * 2 * W + (2 * sizeof(int) + sizeof(float)) * W * g_kf.keyCap + sizeof(int) * 3 * W + (sizeof(float) + sizeof(uint2)) * W * (KF_RAW + KF_FILT)
           + sizeof(float) * 32 * W + 2 * sizeof(unsigned long long) + sizeof(CUtensorMap) * g_kf.imgCap;
}

// the wave's jobs, laid out as bfSiftMatchBatch lays out a batch: [row-pass jobs | column-pass jobs]
__global__ void kf_build_jobs(unsigned long long pBase, unsigned nW, const uint8_t* __restrict__ des, unsigned maxKeys, const int* __restrict__ numKeys,
                              const CUtensorMap* maps, const KfBufs ws) {
    const unsigned b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nW) return;
    const PairRef pr = pair_of(canonical_pairs(pBase), b);
    const int n1 = numKeys[pr.i], n2 = numKeys[pr.j];
    const bool live = n1 > 0 && n2 > 0;
    SiftJobDev r;
    r.desA = des + (size_t)pr.i * maxKeys * 128; r.nA = live ? n1 : 0;
    r.desB = des + (size_t)pr.j * maxKeys * 128; r.nB = live ? n2 : 0;
    r.rowResult = ws.rowResult + (size_t)b * ws.keyCap; r.rowDist = ws.rowDist + (size_t)b * ws.keyCap;
    r.numMatches = ws.rawNum + b; r.outDist = ws.rawDist + (size_t)b * KF_RAW; r.outIdx = ws.rawIdx + (size_t)b * KF_RAW;
    r.offset = make_uint2(pr.i * maxKeys, pr.j * maxKeys);
    r.colResult = ws.colResult + (size_t)b * ws.keyCap; r.done = ws.done + b;
    r.mapA = live ? maps + pr.i : nullptr; r.mapB = live ? maps + pr.j : nullptr;
    SiftJobDev c = r;                                       // column pass: image j owns the sweep, image i is swept
    c.desA = r.desB; c.nA = r.nB; c.desB = r.desA; c.nB = r.nA; c.mapA = r.mapB; c.mapB = r.mapA;
    ws.jobs[b] = r; ws.jobs[nW + b] = c;
}

// pairs with raw matches / surviving the filters (info), and the optional per-pair filtered count
__global__ void kf_wave_stats(unsigned nW, const int* __restrict__ rawNum, const int* __restrict__ numFilt, int* numFiltOut, unsigned long long* counters) {
    const unsigned b = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = b < nW;
    const int f = in ? numFilt[b] : 0;
    if (in && numFiltOut) numFiltOut[b] = f;
    const unsigned r = __ballot_sync(0xffffffffu, in && rawNum[b] > 0), s = __ballot_sync(0xffffffffu, f > 0);
    if ((threadIdx.x & 31) == 0 && (r | s)) { atomicAdd(&counters[0], (unsigned long long)__popc(r)); atomicAdd(&counters[1], (unsigned long long)__popc(s)); }
}

static int refuse(const char* what) { set_last_error(what, cudaErrorInvalidValue); return (int)cudaErrorInvalidValue; }

}  // namespace bf

using namespace bf;

BF_API void bfKeyframeSearchDefaultParams(BFKeyframeSearchParams* p) {
    if (!p) return;
    p->siftMatchThresh = 0.7f; p->siftMatchRatioMax = 0.8f; p->minNumMatches = 5;
    p->maxKabschResidual2 = 0.0004f; p->surfAreaPcaThresh = 0.032f;
    p->projCorrDistThres = 0.15f; p->projCorrNormalThres = 0.97f; p->projCorrColorThresh = 0.1f;
    p->verifySiftErrThresh = 0.075f; p->verifySiftCorrThresh = 0.02f;
    p->sensorDepthMin = 0.1f; p->sensorDepthMax = 4.0f;
}

BF_API int bfKeyframePairRanges(const int32_t* numKeys, uint32_t numImages, uint32_t parts, uint64_t* bounds) {
    if (!numKeys || !bounds || numImages < 2 || numImages > BF_KEYFRAME_SEARCH_MAX_IMAGES || parts < 1 || parts > 65536)
        return refuse("bfKeyframePairRanges: arguments");
    for (uint32_t i = 0; i < numImages; ++i) if (numKeys[i] < 0) return refuse("bfKeyframePairRanges: negative key count");
    auto cost = [&](uint32_t i, uint32_t j) { return (uint64_t)numKeys[i] * (uint64_t)numKeys[j] + BF_KEYFRAME_PAIR_COST; };
    uint64_t total = 0;
    for (uint32_t j = 1; j < numImages; ++j) for (uint32_t i = 0; i < j; ++i) total += cost(i, j);
    // bounds[k] = the first p whose preceding pairs cost prefix(p) >= k total / parts (compared as prefix * parts >= k * total: exact)
    uint64_t prefix = 0, p = 0;
    uint32_t k = 1;
    bounds[0] = 0;
    for (uint32_t j = 1; j < numImages; ++j)
        for (uint32_t i = 0; i < j; ++i, ++p) {
            while (k < parts && prefix * parts >= (uint64_t)k * total) bounds[k++] = p;
            prefix += cost(i, j);
        }
    while (k <= parts) bounds[k++] = p;
    return 0;
}

BF_API int bfKeyframeSearch(const BFKeyframeSet* kf, const BFKeyframeSearchParams* P, uint64_t pBegin, uint64_t pEnd, BFEntryJ* d_entries,
                            uint32_t* d_entryKeyIndices, int32_t* d_numEntries, uint32_t capacity, int32_t* d_numFilteredOut, const BFKeyframeRawMatches* raw,
                            BFKeyframeSearchInfo* info) {
    // ---- refusals: before anything is enqueued ----
    if (!kf || !P || !d_entries || !d_entryKeyIndices || !d_numEntries) return refuse("bfKeyframeSearch: NULL argument");
    if (!kf->d_keyPoints || !kf->d_descriptors || !kf->d_numKeys || !kf->d_cacheFrames) return refuse("bfKeyframeSearch: NULL keyframe-set pointer");
    if (raw && (!raw->d_numMatches || !raw->d_distances || !raw->d_keyPointIndices)) return refuse("bfKeyframeSearch: NULL raw-match pointer");
    const uint32_t N = kf->numImages, maxKeys = kf->maxKeys;
    if (N < 2 || N > BF_KEYFRAME_SEARCH_MAX_IMAGES) return refuse("bfKeyframeSearch: numImages outside [2, BF_KEYFRAME_SEARCH_MAX_IMAGES]");
    const uint64_t numPairs = (uint64_t)N * (N - 1) / 2;
    if (pBegin > pEnd || pEnd > numPairs) return refuse("bfKeyframeSearch: pair range outside [0, N (N - 1) / 2)");
    if (maxKeys == 0 || maxKeys > BF_KEYFRAME_SEARCH_MAX_KEYS) return refuse("bfKeyframeSearch: maxKeys outside [1, BF_KEYFRAME_SEARCH_MAX_KEYS]");
    if ((reinterpret_cast<uintptr_t>(kf->d_keyPoints) | reinterpret_cast<uintptr_t>(kf->d_descriptors)) & 15u)
        return refuse("bfKeyframeSearch: key-point or descriptor array not 16-byte aligned");
    const unsigned by = (kf->cacheHeight + 31) / 32, nt = kf->cacheWidth * by;
    if (kf->cacheWidth == 0 || kf->cacheHeight == 0 || nt % 32 != 0 || nt > 1024) return refuse("bfKeyframeSearch: cache size (verification block shape)");

    std::lock_guard<std::mutex> lk(g_kfMutex);
    cudaStream_t s = stream();
    const unsigned long long launch0 = g_launchCount;
    // ---- key counts (host) and one tensor map per image ----
    g_kf.hKeys.resize(N);
    BF_CHECK(cudaMemcpyAsync(g_kf.hKeys.data(), kf->d_numKeys, sizeof(int) * N, cudaMemcpyDeviceToHost, s));
    BF_CHECK(cudaStreamSynchronize(s));
    int maxN = 0;
    for (uint32_t i = 0; i < N; ++i) {
        if (g_kf.hKeys[i] < 0 || g_kf.hKeys[i] > (int)maxKeys) return refuse("bfKeyframeSearch: key count outside [0, maxKeys]");
        maxN = std::max(maxN, g_kf.hKeys[i]);
    }
    g_kf.hMaps.assign(N, CUtensorMap());
    for (uint32_t i = 0; i < N; ++i)
        if (g_kf.hKeys[i] > 0 && !sift_encode_descriptor_map(kf->d_descriptors + (size_t)i * maxKeys * 128, g_kf.hKeys[i], &g_kf.hMaps[i])) {
            set_last_error("bfKeyframeSearch: no tensor map for the descriptors (the wgmma sweep cannot run)", cudaErrorNotSupported);
            return (int)cudaErrorNotSupported;
        }
    { const int rc = kf_reserve(s, N, maxKeys); if (rc) return rc; }
    BF_CHECK(cudaStreamWaitEvent(s, g_kf.evDone, 0));         // a previous call (possibly on another stream) still reads the maps / wave buffers
    BF_CHECK(cudaMemcpyAsync(g_kf.maps, g_kf.hMaps.data(), sizeof(CUtensorMap) * N, cudaMemcpyHostToDevice, s));       // pageable: staged before return
    BF_CHECK(cudaMemsetAsync(d_numEntries, 0, sizeof(int32_t), s));
    BF_CHECK(cudaMemsetAsync(g_kf.counters, 0, 2 * sizeof(unsigned long long), s));

    const BFKeyframeSearchParams& p = *P;
    const int gx = maxN > 0 ? (maxN + 127) / 128 : 1;
    uint32_t waves = 0;
    for (uint64_t w0 = pBegin; w0 < pEnd; w0 += BF_KEYFRAME_SEARCH_WAVE, ++waves) {
        const unsigned nW = (unsigned)std::min<uint64_t>(BF_KEYFRAME_SEARCH_WAVE, pEnd - w0);
        const PairList pl = canonical_pairs(w0);
        ++g_launchCount;
        kf_build_jobs<<<(nW + 127) / 128, 128, 0, s>>>(w0, nW, kf->d_descriptors, maxKeys, kf->d_numKeys, g_kf.maps, static_cast<const KfBufs&>(g_kf));
        BF_CHECK(cudaGetLastError());
        { const int rc = sift_wgmma_sweep(g_kf.jobs, (int)nW, gx, gx, p.siftMatchThresh, p.siftMatchRatioMax, s); if (rc) return rc; }
        if (raw) {
            const uint64_t o = w0 - pBegin;
            BF_CHECK(cudaMemcpyAsync(raw->d_numMatches + o, g_kf.rawNum, sizeof(int) * nW, cudaMemcpyDeviceToDevice, s));
            BF_CHECK(cudaMemcpyAsync(raw->d_distances + o * KF_RAW, g_kf.rawDist, sizeof(float) * KF_RAW * nW, cudaMemcpyDeviceToDevice, s));
            BF_CHECK(cudaMemcpyAsync(raw->d_keyPointIndices + o * KF_RAW * 2, g_kf.rawIdx, sizeof(uint2) * KF_RAW * nW, cudaMemcpyDeviceToDevice, s));
        }
        uint32_t* rawIdx = reinterpret_cast<uint32_t*>(g_kf.rawIdx);
        uint32_t* fIdx = reinterpret_cast<uint32_t*>(g_kf.fIdx);
        KF_OK(sift_sort_pairs(pl, nW, g_kf.rawNum, g_kf.rawDist, rawIdx));
        KF_OK(sift_filter_pairs(pl, nW, kf->d_keyPoints, g_kf.rawNum, g_kf.rawDist, rawIdx, g_kf.numFilt, g_kf.fDist, fIdx, g_kf.fT, g_kf.fTinv,
                                   kf->siftIntrinsicsInv, p.minNumMatches, p.maxKabschResidual2));
        KF_OK(sift_surface_area_pairs(pl, nW, kf->d_keyPoints, g_kf.numFilt, fIdx, kf->siftIntrinsicsInv, p.surfAreaPcaThresh, nullptr));
        KF_OK(sift_dense_verify_pairs(pl, nW, kf->cacheWidth, kf->cacheHeight, kf->cacheIntrinsics, g_kf.numFilt, g_kf.fT, kf->d_cacheFrames, p.projCorrDistThres,
                                         p.projCorrNormalThres, p.verifySiftErrThresh, p.verifySiftCorrThresh, p.sensorDepthMin, p.sensorDepthMax, nullptr));
        ++g_launchCount;
        kf_wave_stats<<<(nW + 255) / 256, 256, 0, s>>>(nW, g_kf.rawNum, g_kf.numFilt, d_numFilteredOut ? d_numFilteredOut + (w0 - pBegin) : nullptr, g_kf.counters);
        BF_CHECK(cudaGetLastError());
        KF_OK(sift_add_pairs(pl, nW, d_entries, d_entryKeyIndices, d_numEntries, capacity, g_kf.numFilt, fIdx, kf->d_keyPoints, kf->siftIntrinsicsInv, nullptr));
    }
    BF_CHECK(cudaEventRecord(g_kf.evDone, s));
    if (info) {
        unsigned long long c[2] = { 0, 0 }; int entries = 0;
        BF_CHECK(cudaMemcpyAsync(c, g_kf.counters, sizeof(c), cudaMemcpyDeviceToHost, s));
        BF_CHECK(cudaMemcpyAsync(&entries, d_numEntries, sizeof(int), cudaMemcpyDeviceToHost, s));
        BF_CHECK(cudaStreamSynchronize(s));
        info->pairs = pEnd - pBegin; info->waves = waves; info->launches = (uint32_t)(g_launchCount - launch0);
        info->pairsWithRawMatches = c[0]; info->pairsSurviving = c[1]; info->entries = (uint64_t)entries;
    }
    return 0;
}

BF_API int bfKeyframeSearchReserveWorkspace(uint32_t numImages, uint32_t maxKeys) {
    if (numImages < 2 || numImages > BF_KEYFRAME_SEARCH_MAX_IMAGES || maxKeys == 0 || maxKeys > BF_KEYFRAME_SEARCH_MAX_KEYS) return refuse("bfKeyframeSearchReserveWorkspace: arguments");
    std::lock_guard<std::mutex> lk(g_kfMutex);
    return kf_reserve(stream(), numImages, maxKeys);
}
BF_API size_t bfKeyframeSearchWorkspaceBytes(void) {
    std::lock_guard<std::mutex> lk(g_kfMutex);
    return kf_bytes();
}
BF_API int bfKeyframeSearchReleaseWorkspace(void) {
    std::lock_guard<std::mutex> lk(g_kfMutex);
    if (g_kf.evDone) { cudaEventSynchronize(g_kf.evDone); cudaEventDestroy(g_kf.evDone); }
    kf_free();
    g_kf = KfWs();
    return 0;
}

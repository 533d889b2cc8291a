// sift_fuse.cu -- chunk -> keyframe fusion of the sparse features on the device (SURVEY.md section 8f, row N2).
//
// Behavioural source: SIFTImageManager::computeTracks / findTrack / fuseToGlobal,
// /root/reference/FriedLiver/Source/SiftGPU/SIFTImageManager.cpp:366-476 -- HOST code in the reference: after a chunk's local solve it copies
// all keys (16 B), descriptors (128 B), correspondences and poses of the chunk to the CPU, builds per-key correspondence lists, walks them
// recursively into tracks, averages each track's world position, projects it into the chunk's first frame and uploads the fused key points
// with one representative descriptor each as the next keyframe of the global manager.
//
// Here the whole thing is one launch of one CTA and nothing leaves the device, and every phase runs on all threads.  The lists are filled in
// shared memory and sorted into push order; connected components of the key / correspondence graph are labelled; the reference's serial walk
// over all roots equals one walk per component that holds a root, in the order of its first root, so each such component's walk is replayed
// by one thread with an explicit stack, into its own slot of the track list (the visiting order decides which key represents a track and which
// correspondence supplies a member's position, so it is reproduced exactly).  A walk's stack is sized by its component, so d_status (stack
// overflow) cannot be raised.  Then the tracks are reduced, compacted and their descriptors gathered.  Output and count stay on the device.
// Arithmetic as the reference's host code: individually rounded IEEE operations (this TU is built -fmad=false -prec-div=true -prec-sqrt=true),
// float4x4 * float3 as ((m0 x + m1 y) + m2 z) + m3.  Bit-identical to oracle/fuse_oracle.c.
#include "../../include/bf_sift.h"
#include "bf_common.cuh"

namespace bf {

extern unsigned long long g_launchCount;

#define FUSE_MAX_KEYS 16384u       // numImages * keyStride
#define FUSE_MAX_CORR 4096u
#define FUSE_THREADS 1024

struct FuseArgs {
    const BFEntryJ* corr; const uint2* keyIdx; const int* numCorr; const float* T; unsigned numImages;
    const BFSIFTKeyPoint* keys; const uint8_t* descs; const int* numKeys; unsigned keyStride;
    float K[16];
    BFSIFTKeyPoint* outKeys; uint8_t* outDescs; int* outNum; unsigned maxKeys; int* status;
};

__device__ __forceinline__ void xform3(const float* M, const float* p, float* o) {
#pragma unroll
    for (int r = 0; r < 3; ++r) o[r] = ((M[4 * r] * p[0] + M[4 * r + 1] * p[1]) + M[4 * r + 2] * p[2]) + M[4 * r + 3];
}

__global__ void __launch_bounds__(FUSE_THREADS)
sift_fuse_kernel(const __grid_constant__ FuseArgs a) {
    extern __shared__ unsigned smem[];
    const unsigned M = a.numImages * a.keyStride, t = threadIdx.x;
    const unsigned C = min((unsigned)max(*a.numCorr, 0), FUSE_MAX_CORR);
    unsigned* start = smem;                       // [M + 1]   first list entry of each key (corrPerKey)
    unsigned* adjKey = start + (M + 1);           // [2C]      target key of a list entry
    unsigned* adjCE = adjKey + 2 * C;             // [2C]      correspondence * 2 + side (0: target is the j side, 1: the i side)
    unsigned* trackItem = adjCE + 2 * C;          // [2C]      list entries in visiting order
    unsigned* trackStart = trackItem + 2 * C;     // [C + 1]
    unsigned* label = trackStart + (C + 1);       // [2C]      component label of a key's list-begin node
    unsigned* comp = label + 2 * C;               // [C]       root of each track
    unsigned* scan = comp + C;                    // [FUSE_THREADS]
    unsigned* rootList = scan + FUSE_THREADS;     // [2C]      keys with a non-empty list, in (image, key) order: the only roots that can start a track
    unsigned* ckx = rootList + 2 * C;             // [C]       key of the correspondence in image i (0xFFFFFFFF: invalid correspondence) ...
    unsigned* cky = ckx + C;                      // [C]       ... and in image j
    unsigned char* marker = reinterpret_cast<unsigned char*>(cky + C);                   // [M]
    unsigned char* errOk = marker + ((M + 3) & ~3u);                                      // [C]
    __shared__ unsigned sNumTracks, sOverflow, sNumRoots, sTotal, sChanged;

    for (unsigned k = t; k <= M; k += FUSE_THREADS) start[k] = 0;
    for (unsigned k = t; k < M; k += FUSE_THREADS) marker[k] = 0;
    if (t == 0) { sNumTracks = 0; sOverflow = 0; }
    __syncthreads();
    // per-correspondence: list lengths, and the track error test (computeTracks :389-399)
    for (unsigned c = t; c < C; c += FUSE_THREADS) {
        const BFEntryJ e = a.corr[c];
        unsigned char ok = 0;
        ckx[c] = 0xFFFFFFFFu; cky[c] = 0xFFFFFFFFu;
        if (e.imgIdx_i != 0xFFFFFFFFu) {
            const uint2 k = a.keyIdx[c];
            ckx[c] = k.x; cky[c] = k.y;
            atomicAdd(&start[k.x + 1], 1u); atomicAdd(&start[k.y + 1], 1u);
            float pa[3], pb[3];
            xform3(a.T + 16 * (size_t)e.imgIdx_i, e.pos_i, pa); xform3(a.T + 16 * (size_t)e.imgIdx_j, e.pos_j, pb);
            const float d0 = pa[0] - pb[0], d1 = pa[1] - pb[1], d2 = pa[2] - pb[2];
            ok = sqrtf((d0 * d0 + d1 * d1) + d2 * d2) < 0.03f ? 1 : 0;                   // MAX_TRACK_CORR_ERROR
        }
        errOk[c] = ok;
    }
    __syncthreads();
    // exclusive scan of the list lengths (start[k + 1] holds the length of key k)
    {
        const unsigned per = (M + FUSE_THREADS) / FUSE_THREADS;      // elements of start[1..M] per thread
        unsigned local = 0;
        for (unsigned q = 0; q < per; ++q) { const unsigned k = 1 + t * per + q; if (k <= M) local += start[k]; }
        scan[t] = local;
        __syncthreads();
        for (unsigned off = 1; off < FUSE_THREADS; off <<= 1) {
            const unsigned v = (t >= off) ? scan[t - off] : 0u;
            __syncthreads();
            scan[t] += v;
            __syncthreads();
        }
        unsigned run = scan[t] - local;
        for (unsigned q = 0; q < per; ++q) { const unsigned k = 1 + t * per + q; if (k <= M) { const unsigned len = start[k]; start[k] = run + len; run += len; } }
        __syncthreads();           // now start[k + 1] = end of key k's list, start[0] = 0  => start[k] = begin of key k
    }
    // After the scan start[k] = begin of key k's list (= end of key k - 1's), start[M] = total.  Pre-decrementing the END pointer of
    // a key (start[key + 1]) for each of its entries turns it into the BEGIN of key's list; its end is then the begin of the next
    // key's list, start[key + 2] (the total for the last key).  The lists must be in push order = ascending correspondence index,
    // the i side before the j side (:389-399): entries land in any order, then every list is sorted by adjCE.
    if (t == 0) sTotal = start[M];                   // start[M] is about to become the begin of the last key's list
    __syncthreads();
    for (unsigned c = t; c < C; c += FUSE_THREADS) {
        const unsigned kx = ckx[c], ky = cky[c];
        if (kx == 0xFFFFFFFFu) continue;
        adjCE[atomicAdd(&start[ky + 1], 0xFFFFFFFFu) - 1u] = 2u * c + 1u;
        adjCE[atomicAdd(&start[kx + 1], 0xFFFFFFFFu) - 1u] = 2u * c;
    }
    __syncthreads();
    const unsigned total = sTotal;
    for (unsigned k = t; k < M; k += FUSE_THREADS) {
        const unsigned b = start[k + 1], e = (k + 1 < M) ? start[k + 2] : total;
        for (unsigned i = b + 1; i < e; ++i) {                    // insertion sort: a list holds a few entries
            const unsigned v = adjCE[i];
            unsigned j = i;
            for (; j > b && adjCE[j - 1] > v; --j) adjCE[j] = adjCE[j - 1];
            adjCE[j] = v;
        }
        for (unsigned i = b; i < e; ++i) { const unsigned ce = adjCE[i]; adjKey[i] = (ce & 1u) ? ckx[ce >> 1] : cky[ce >> 1]; }
    }
    // Connected components of the key / correspondence graph.  A key with a non-empty list is named by its list's begin (node
    // start[k + 1] < total, increasing with k); label[node] converges to the smallest node of its component by min-hooking and
    // pointer jumping (label[x] <= x and in x's component throughout).
    volatile unsigned* vlabel = label;                 // read while other threads lower it
    for (unsigned i = t; i < total; i += FUSE_THREADS) label[i] = i;
    for (;;) {
        if (t == 0) sChanged = 0;
        __syncthreads();
        for (unsigned c = t; c < C; c += FUSE_THREADS) {
            const unsigned kx = ckx[c], ky = cky[c];
            if (kx == 0xFFFFFFFFu) continue;
            const unsigned la = vlabel[start[kx + 1]], lb = vlabel[start[ky + 1]];
            if (la != lb) { const unsigned m = min(la, lb); atomicMin(&label[la], m); atomicMin(&label[lb], m); sChanged = 1; }
        }
        __syncthreads();
        for (unsigned i = t; i < total; i += FUSE_THREADS) {
            unsigned p = vlabel[i];
            for (unsigned pp = vlabel[p]; pp != p; pp = vlabel[p]) p = pp;
            vlabel[i] = p;
        }
        const unsigned changed = sChanged;
        __syncthreads();
        if (!changed) break;
    }
    // findTrack is called for every key in (image, key) order (:401-410), but a key without correspondences starts and joins nothing: all threads pick
    // out, in that order, the keys whose list is not empty (of ~2 000 keys of a chunk a few hundred), so that the serial walk below touches only those
    {
        const unsigned total = sTotal;
        const unsigned per = (M + FUSE_THREADS - 1) / FUSE_THREADS;
        unsigned local = 0;
        for (unsigned q = 0; q < per; ++q) {
            const unsigned k = t * per + q;
            if (k < M) {
                const unsigned img = k / a.keyStride, kk = k % a.keyStride;
                const bool live = kk < (unsigned)max(a.numKeys[img], 0) && start[k + 1] < ((k + 1 < M) ? start[k + 2] : total);
                local += live ? 1u : 0u;
            }
        }
        scan[t] = local;
        __syncthreads();
        for (unsigned off = 1; off < FUSE_THREADS; off <<= 1) {
            const unsigned v = (t >= off) ? scan[t - off] : 0u;
            __syncthreads();
            scan[t] += v;
            __syncthreads();
        }
        unsigned o = scan[t] - local;
        for (unsigned q = 0; q < per; ++q) {
            const unsigned k = t * per + q;
            if (k < M) {
                const unsigned img = k / a.keyStride, kk = k % a.keyStride;
                if (kk < (unsigned)max(a.numKeys[img], 0) && start[k + 1] < ((k + 1 < M) ? start[k + 2] : total)) rootList[o++] = k;
            }
        }
        if (t == FUSE_THREADS - 1) sNumRoots = scan[t];
        __syncthreads();
    }
    // The serial reference walks findTrack from every root in rootList order.  A walk from root r marks exactly r's component, so
    // only the first root of each component opens a track, and that track is the component's walk, independent of the others.
    // Tracks are therefore the components that hold a root, in the order of their first root, walked in parallel below.
    {
        unsigned* firstRoot = trackItem;                 // [total] per component label: smallest rootList index (trackItem is written by the walks only)
        unsigned* compSize = ckx;                        // [total] (ckx, cky: 2C words, no longer needed) per component label: keys
        const unsigned nRoots = sNumRoots;
        for (unsigned i = t; i < total; i += FUSE_THREADS) { firstRoot[i] = 0xFFFFFFFFu; compSize[i] = 0; }
        __syncthreads();
        for (unsigned r = t; r < nRoots; r += FUSE_THREADS) atomicMin(&firstRoot[label[start[rootList[r] + 1]]], r);
        for (unsigned k = t; k < M; k += FUSE_THREADS)
            if (start[k + 1] < ((k + 1 < M) ? start[k + 2] : total)) atomicAdd(&compSize[label[start[k + 1]]], 1u);
        __syncthreads();
        // compaction of the first roots in rootList order: comp[track] = root, trackStart[track] = its component's size
        const unsigned per = (nRoots + FUSE_THREADS - 1) / FUSE_THREADS;
        unsigned local = 0;
        for (unsigned q = 0; q < per; ++q) { const unsigned r = t * per + q; if (r < nRoots && firstRoot[label[start[rootList[r] + 1]]] == r) ++local; }
        scan[t] = local;
        __syncthreads();
        for (unsigned off = 1; off < FUSE_THREADS; off <<= 1) {
            const unsigned v = (t >= off) ? scan[t - off] : 0u;
            __syncthreads();
            scan[t] += v;
            __syncthreads();
        }
        unsigned o = scan[t] - local;
        for (unsigned q = 0; q < per; ++q) {
            const unsigned r = t * per + q;
            if (r < nRoots) {
                const unsigned lab = label[start[rootList[r] + 1]];
                if (firstRoot[lab] == r) { comp[o] = rootList[r]; trackStart[o] = compSize[lab]; ++o; }
            }
        }
        if (t == FUSE_THREADS - 1) sNumTracks = scan[t];
        __syncthreads();
        // exclusive scan of the component sizes: trackStart[track] = first item of the track, trackStart[nTracks] = items
        const unsigned nT = sNumTracks, perT = (nT + FUSE_THREADS) / FUSE_THREADS;
        local = 0;
        for (unsigned q = 0; q < perT; ++q) { const unsigned i = t * perT + q; if (i < nT) local += trackStart[i]; }
        scan[t] = local;
        __syncthreads();
        for (unsigned off = 1; off < FUSE_THREADS; off <<= 1) {
            const unsigned v = (t >= off) ? scan[t - off] : 0u;
            __syncthreads();
            scan[t] += v;
            __syncthreads();
        }
        unsigned run = scan[t] - local;
        for (unsigned q = 0; q < perT; ++q) { const unsigned i = t * perT + q; if (i < nT) { const unsigned len = trackStart[i]; trackStart[i] = run; run += len; } }
        if (t == FUSE_THREADS - 1) trackStart[nT] = scan[t];
        __syncthreads();
    }
    // One thread per track: the recursion of findTrack replaced by an explicit stack of list positions.  Every push marks a key of
    // the component, so a track of n keys is at most n + 1 deep: its stack lives at trackStart[track] + track of the pool
    // (rootList, ckx, cky: 4C words >= items + tracks) and cannot overflow into the next one.
    for (unsigned tr = t; tr < sNumTracks; tr += FUSE_THREADS) {
        const unsigned root = comp[tr], first = trackStart[tr], depth = trackStart[tr + 1] - first + 1;
        unsigned* stack = rootList + first + tr;
        unsigned nItems = first, sp = 1;
        stack[0] = start[root + 1];
        while (sp) {
            const unsigned cur = (sp == 1) ? root : adjKey[stack[sp - 2] - 1];      // the entry that descended to this level
            const unsigned end = (cur + 1 < M) ? start[cur + 2] : total;
            unsigned pos = stack[sp - 1];
            bool descended = false;
            while (pos < end) {
                const unsigned tgt = adjKey[pos];
                if (!marker[tgt]) {
                    trackItem[nItems++] = pos;
                    marker[tgt] = 1;
                    stack[sp - 1] = pos + 1;
                    if (sp >= depth) { sOverflow = 1; break; }
                    stack[sp] = start[tgt + 1]; ++sp;
                    descended = true;
                    break;
                }
                ++pos;
            }
            if (!descended) --sp;
        }
    }
    __syncthreads();
    const unsigned nTracks = sNumTracks;
    // one thread per track: average of the usable members' world positions, projection into the first frame (fuseToGlobal :432-456)
    unsigned outBase = 0;
    for (unsigned t0 = 0; t0 < nTracks; t0 += FUSE_THREADS) {
        const unsigned tr = t0 + t;
        bool has = false;
        BFSIFTKeyPoint key; key.pos[0] = key.pos[1] = key.scale = key.depth = 0.0f;
        unsigned rep = 0;
        if (tr < nTracks) {
            float pos[3] = { 0.0f, 0.0f, 0.0f }; unsigned num = 0;
            for (unsigned q = trackStart[tr]; q < trackStart[tr + 1]; ++q) {
                const unsigned ce = adjCE[trackItem[q]], c = ce >> 1;
                if (!errOk[c]) continue;
                const BFEntryJ e = a.corr[c];
                float w[3];
                if (ce & 1u) xform3(a.T + 16 * (size_t)e.imgIdx_i, e.pos_i, w); else xform3(a.T + 16 * (size_t)e.imgIdx_j, e.pos_j, w);
                pos[0] += w[0]; pos[1] += w[1]; pos[2] += w[2]; ++num;
            }
            if (num > 0) {
                pos[0] /= (float)num; pos[1] /= (float)num; pos[2] /= (float)num;
                float p[3]; xform3(a.K, pos, p);
                rep = adjKey[trackItem[trackStart[tr]]];
                key.pos[0] = p[0] / p[2]; key.pos[1] = p[1] / p[2]; key.scale = a.keys[rep].scale; key.depth = p[2];
                has = true;
            }
        }
        // compaction in track order
        scan[t] = has ? 1u : 0u;
        __syncthreads();
        for (unsigned off = 1; off < FUSE_THREADS; off <<= 1) {
            const unsigned v = (t >= off) ? scan[t - off] : 0u;
            __syncthreads();
            scan[t] += v;
            __syncthreads();
        }
        const unsigned o = outBase + scan[t] - (has ? 1u : 0u);
        if (has && o < a.maxKeys) {
            a.outKeys[o] = key;
            const uint4* src = reinterpret_cast<const uint4*>(a.descs + 128 * (size_t)rep);
            uint4* dst = reinterpret_cast<uint4*>(a.outDescs + 128 * (size_t)o);
#pragma unroll
            for (int w = 0; w < 8; ++w) dst[w] = src[w];
        }
        outBase += scan[FUSE_THREADS - 1];
        __syncthreads();
    }
    if (t == 0) { *a.outNum = (int)min(outBase, a.maxKeys); if (a.status) *a.status = (int)sOverflow; }
}

}  // namespace bf

using namespace bf;

BF_API int bfSiftFuseToGlobal(const BFEntryJ* d_corr, const uint32_t* d_corrKeyIndices, const int32_t* d_numCorr, const float* d_transforms, unsigned int numImages,
                              const BFSIFTKeyPoint* d_keyPoints, const uint8_t* d_descriptors, const int32_t* d_numKeysPerImage, unsigned int keyStride,
                              const float* colorIntrinsics, unsigned int maxCorr, BFSIFTKeyPoint* d_outKeyPoints, uint8_t* d_outDescriptors, int32_t* d_outNumKeys,
                              unsigned int maxKeys, int32_t* d_status) {
    if (!d_corr || !d_corrKeyIndices || !d_numCorr || !d_transforms || !d_keyPoints || !d_descriptors || !d_numKeysPerImage || !colorIntrinsics || !d_outKeyPoints ||
        !d_outDescriptors || !d_outNumKeys || numImages == 0 || keyStride == 0) return (int)cudaErrorInvalidValue;
    const unsigned M = numImages * keyStride;
    if (M > FUSE_MAX_KEYS || maxCorr > FUSE_MAX_CORR) return (int)cudaErrorInvalidValue;
    FuseArgs a;
    a.corr = d_corr; a.keyIdx = reinterpret_cast<const uint2*>(d_corrKeyIndices); a.numCorr = d_numCorr; a.T = d_transforms; a.numImages = numImages;
    a.keys = d_keyPoints; a.descs = d_descriptors; a.numKeys = d_numKeysPerImage; a.keyStride = keyStride;
    for (int k = 0; k < 16; ++k) a.K[k] = colorIntrinsics[k];
    a.outKeys = d_outKeyPoints; a.outDescs = d_outDescriptors; a.outNum = d_outNumKeys; a.maxKeys = maxKeys; a.status = d_status;
    const size_t words = (size_t)(M + 1) + 13 * (size_t)maxCorr + (maxCorr + 1) + FUSE_THREADS;
    const size_t bytes = words * 4 + ((M + 3) & ~3u) + ((maxCorr + 3) & ~3u);
    static size_t attr = 0;
    if (bytes > attr) { BF_CHECK(cudaFuncSetAttribute(sift_fuse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes)); attr = bytes; }
    ++g_launchCount;
    sift_fuse_kernel<<<1, FUSE_THREADS, bytes, stream()>>>(a);
    BF_CHECK(cudaGetLastError());
    return 0;
}

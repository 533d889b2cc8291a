/*
 * bf_keyframe_search.h -- the all-pairs correspondence search over a keyframe set (SURVEY.md section 8e: "SIFT all-pairs").
 *
 * Given N keyframes, one call returns the global correspondence graph of every pair (i, j), i < j: raw SIFT matches exactly as
 * bfSiftMatchBatch gives them for (image 1 = i, image 2 = j), then the distance sort, the Kabsch filter, the surface-area filter and the dense
 * verification with the frame loop's global thresholds, then the surviving matches as the EntryJ list bfSiftAddCurrToResiduals writes --
 * what the frame loop's global matchAndFilter computes for cur = j, prev = i with every image valid.
 *
 * Pairs are numbered p(i, j) = j (j - 1) / 2 + i (j ascending, then i ascending: the order the frame loop appends its global list in).  A call
 * covers a pair range [pBegin, pEnd); the lists of consecutive ranges, concatenated, are the list of their union byte for byte, so a caller can
 * split the pairs over GPUs (bfKeyframePairRanges) and concatenate the parts in range order.
 *
 * Threading: as bf_sift.h (per-process workspace, the library stream; one thread per process).
 */
#ifndef BF_KEYFRAME_SEARCH_H
#define BF_KEYFRAME_SEARCH_H

#include <stddef.h>
#include <stdint.h>

#include "bf_sift.h"

#ifdef __cplusplus
extern "C" {
#endif

#define BF_KEYFRAME_SEARCH_MAX_IMAGES 4096        /* the global solver's image limit */
#define BF_KEYFRAME_SEARCH_MAX_KEYS 1024          /* key stride limit (the frame loop's s_maxNumKeysPerImage) */
#define BF_KEYFRAME_SEARCH_WAVE 4096              /* pairs per wave: the workspace holds one wave */
#define BF_KEYFRAME_PAIR_COST 16384               /* bfKeyframePairRanges: cost of a pair = n_i n_j + this (its filters) */

/* A keyframe set as the frame loop's global SIFT manager holds it.  Key k of image i is at i * maxKeys + k. */
typedef struct BFKeyframeSet {
    uint32_t numImages;
    uint32_t maxKeys;                             /* key stride */
    const BFSIFTKeyPoint* d_keyPoints;            /* [numImages][maxKeys], 16-byte aligned */
    const uint8_t* d_descriptors;                 /* [numImages][maxKeys][128], 16-byte aligned */
    const int32_t* d_numKeys;                     /* [numImages] (device) */
    const BFCUDACachedFrame* d_cacheFrames;       /* [numImages] dense-cache frames */
    uint32_t cacheWidth, cacheHeight;
    float cacheIntrinsics[16];                    /* 4x4, cache resolution */
    float siftIntrinsicsInv[16];                  /* 4x4, inverse of the SIFT / colour intrinsics */
} BFKeyframeSet;

/* Thresholds; bfKeyframeSearchDefaultParams gives the frame loop's global values. */
typedef struct BFKeyframeSearchParams {
    float siftMatchThresh, siftMatchRatioMax;     /* 0.7, 0.8 (global) */
    uint32_t minNumMatches;                       /* 5 (global) */
    float maxKabschResidual2, surfAreaPcaThresh;  /* 0.0004, 0.032 */
    float projCorrDistThres, projCorrNormalThres, projCorrColorThresh, verifySiftErrThresh, verifySiftCorrThresh;
    float sensorDepthMin, sensorDepthMax;
} BFKeyframeSearchParams;
void bfKeyframeSearchDefaultParams(BFKeyframeSearchParams* out);

/* Optional raw-match output, per pair of the range (index p - pBegin), in bfSiftMatchBatch's layout. */
typedef struct BFKeyframeRawMatches {
    int32_t* d_numMatches;                        /* [pEnd - pBegin] */
    float* d_distances;                           /* [pEnd - pBegin][128] */
    uint32_t* d_keyPointIndices;                  /* [pEnd - pBegin][128][2] */
} BFKeyframeRawMatches;

typedef struct BFKeyframeSearchInfo {
    uint64_t pairs;                               /* pEnd - pBegin */
    uint32_t waves, launches;
    uint64_t pairsWithRawMatches, pairsSurviving, entries;
} BFKeyframeSearchInfo;

/* Searches pairs [pBegin, pEnd) of kf.  Writes the range's correspondences from index 0: d_entries[k] / d_entryKeyIndices[k] (uint2: global key
 * indices) for k < capacity; *d_numEntries (device) is set to the number of entries of the range, which may exceed capacity (the entries past
 * it are not written: an undersized list holds the prefix of the full one).  d_numFilteredOut (optional, [pEnd - pBegin]): the filtered-match
 * count of each pair after the last filter.  raw (optional, NULL in normal use): the raw matches.  info (optional): when given, the call
 * synchronises the library stream at the end and fills it.
 * Reads the key counts to the host once (a synchronisation) before anything is enqueued.  Returns cudaErrorInvalidValue, with nothing
 * enqueued, for numImages < 2 or > BF_KEYFRAME_SEARCH_MAX_IMAGES, pBegin > pEnd or pEnd > N (N - 1) / 2, maxKeys 0 or >
 * BF_KEYFRAME_SEARCH_MAX_KEYS, key-point or descriptor arrays not 16-byte aligned, a NULL required pointer, or a cache size whose verification
 * block is not a whole number of warps <= 1024 threads; a key count outside [0, maxKeys] is refused after the count read.  No other path
 * is taken when the wgmma sweep cannot run (cudaErrorNotSupported). */
int bfKeyframeSearch(const BFKeyframeSet* kf, const BFKeyframeSearchParams* params, uint64_t pBegin, uint64_t pEnd, BFEntryJ* d_entries,
                     uint32_t* d_entryKeyIndices, int32_t* d_numEntries, uint32_t capacity, int32_t* d_numFilteredOut, const BFKeyframeRawMatches* raw,
                     BFKeyframeSearchInfo* info);

/* The balanced split of the canonical pair order of N images into `parts` contiguous ranges: bounds[0] = 0 <= bounds[1] <= ... <= bounds[parts] =
 * N (N - 1) / 2, range k = [bounds[k], bounds[k + 1]).  Cost of a pair: numKeys[i] numKeys[j] + BF_KEYFRAME_PAIR_COST; bounds[k] is the first pair
 * whose preceding pairs cost at least k / parts of the total, so each range's cost is within one pair's cost of the share.  numKeys: HOST [N].
 * Returns cudaErrorInvalidValue for N < 2 or > BF_KEYFRAME_SEARCH_MAX_IMAGES, parts < 1, a NULL pointer or a negative count. */
int bfKeyframePairRanges(const int32_t* numKeys, uint32_t numImages, uint32_t parts, uint64_t* bounds);

/* Sizes the search's workspace for key stride maxKeys and numImages images so that no later call with at most these grows it. */
int bfKeyframeSearchReserveWorkspace(uint32_t numImages, uint32_t maxKeys);
size_t bfKeyframeSearchWorkspaceBytes(void);
int bfKeyframeSearchReleaseWorkspace(void);

#ifdef __cplusplus
}
#endif
#endif /* BF_KEYFRAME_SEARCH_H */

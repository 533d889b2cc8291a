// sift_pairs.cuh -- which image pair a block of the match-filter kernels works on, and the internal launchers that take it.
//
// The filter chain (sort -> Kabsch -> surface area -> dense verify -> residual append) was written for one current image against a range of
// earlier ones: block b works on pair (startFrame + b, curFrame) and indexes its arrays by the earlier image.  The keyframe search
// (keyframe_search.cu) runs the same kernels over a wave of pairs of the canonical all-pairs order p(i, j) = j (j - 1) / 2 + i, i < j: block b
// works on pair p = pBase + b and indexes its arrays by b.  A PairList says which of the two a launch is; the pair is arithmetic, not a table.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/bf_sift.h"

namespace bf {

struct PairList {
    unsigned curFrame, startFrame;       // per-frame form
    unsigned long long pBase;            // canonical form: pair of block 0
    int canonical;
};
struct PairRef { unsigned i, j, slot; bool skip; };

// the image j of canonical pair p: the largest j with j (j - 1) / 2 <= p
__host__ __device__ inline unsigned pair_image_j(unsigned long long p) {
    unsigned long long j = (unsigned long long)((1.0 + sqrt(1.0 + 8.0 * (double)p)) * 0.5);
    while (j > 1 && j * (j - 1) / 2 > p) --j;
    while ((j + 1) * j / 2 <= p) ++j;
    return (unsigned)j;
}
__host__ __device__ inline unsigned long long pair_index(unsigned i, unsigned j) { return (unsigned long long)j * (j - 1) / 2 + i; }

__host__ __device__ inline PairRef pair_of(const PairList& L, unsigned b) {
    PairRef r;
    if (!L.canonical) { r.i = L.startFrame + b; r.j = L.curFrame; r.slot = r.i; r.skip = r.i == L.curFrame; return r; }
    const unsigned long long p = L.pBase + b;
    r.j = pair_image_j(p); r.i = (unsigned)(p - pair_index(0, r.j)); r.slot = b; r.skip = false;
    return r;
}
__host__ __device__ inline PairList frame_pairs(unsigned curFrame, unsigned startFrame) { PairList L; L.curFrame = curFrame; L.startFrame = startFrame; L.pBase = 0; L.canonical = 0; return L; }
__host__ __device__ inline PairList canonical_pairs(unsigned long long pBase) { PairList L; L.curFrame = 0; L.startFrame = 0; L.pBase = pBase; L.canonical = 1; return L; }

// ---- internal launchers (nBlocks blocks, one per pair of L; asynchronous on the library stream) ----
// sift_match.cu
int sift_sort_pairs(const PairList& L, unsigned nBlocks, const int32_t* numMatches, float* dists, uint32_t* idxs);
// sift_filter.cu
int sift_filter_pairs(const PairList& L, unsigned nBlocks, const BFSIFTKeyPoint* kp, const int32_t* numMatches, const float* dists, const uint32_t* idxs,
                      int32_t* numFiltered, float* fDists, uint32_t* fIdxs, float* fT, float* fTinv, const float* siftKinv, unsigned minNum, float maxRes2);
// entries past `cap` are not written; *globNum still advances by every entry
int sift_add_pairs(const PairList& L, unsigned nBlocks, BFEntryJ* glob, uint32_t* globIdx, int32_t* globNum, unsigned cap, const int32_t* numFiltered,
                   const uint32_t* fIdxs, const BFSIFTKeyPoint* kp, const float* Kinv, const int32_t* lastMatched);
// sift_verify.cu
int sift_surface_area_pairs(const PairList& L, unsigned nBlocks, const BFSIFTKeyPoint* kp, int32_t* numFiltered, const uint32_t* fIdxs, const float* Kinv,
                            float areaThresh, float* areas);
int sift_dense_verify_pairs(const PairList& L, unsigned nBlocks, unsigned W, unsigned H, const float* K, int32_t* numFiltered, const float* fT,
                            const BFCUDACachedFrame* frames, float distThresh, float normalThresh, float errThresh, float corrThresh, float dMin, float dMax,
                            float* stats);

}  // namespace bf

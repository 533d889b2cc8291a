// tsdf_shared.cuh -- what tsdf.cu (bit-exact arithmetic contract, built -fmad=false -prec-div=true) and tsdf_fast.cu (the
// tolerance-mode stencil, built with FMA contraction and approximate reciprocals) share: the private counter layout and the
// launchers of the fast stencil.
#pragma once
#include <cuda_runtime.h>

#include "../../include/bf_tsdf.h"

namespace bf {

enum { CTR_HIGH_WATER = 0, CTR_E = 3, CTR_UB_TOT_LO = 4, CTR_UB_TOT_HI = 5, CTR_EB_TOT_LO = 6, CTR_EB_TOT_HI = 7 /* U / E of the batch launches alone */, CTR_FREED = 8, CTR_HEAP_FAIL = 9, CTR_DROPPED = 10, CTR_CULLB = 11 /* (block, op, pose) probes the batch cull removed, 32-bit running sum */, CTR_U_TOT_LO = 12, CTR_U_TOT_HI = 13, CTR_E_TOT_LO = 14, CTR_E_TOT_HI = 15,
       // two per-list counter sets (the list / work list of op k and of op k+1 are alive at the same time when alloc + compactify of
       // op k+1 run on the front lane while the stencil of op k runs on the back lane); a set is zeroed by the op that is about to fill it
       CTR_SET0 = 16, CTR_SET1 = 24, CTR_NUM = 32,
       SET_COUNT = 0, SET_WORK = 1, SET_Q2 = 2, SET_TICKET = 3 /* dynamic block deal of the fast stencil */, SET_U_LO = 4, SET_U_HI = 5, SET_Q1 = 6, SET_Q0 = 7 /* batch: items of cost quartile 2 / 1 / 0 (quartile 3: SET_WORK) */, SET_WORDS = 8 };

// tolerance-mode stencils (tsdf_fast.cu).  `work` may be NULL (the list is then d_hashCompactified[0..count)); useListCount /
// countOverride as in tsdf.cu's integrate_kernel<MODE>.
int launch_integrate_fast(const BFHashDataStruct* hd, const BFHashParams* hp, const BFDepthCameraParams* cp, const float* depth, const void* color,
                          bool deIntegrate, bool useListCount, unsigned countOverride, unsigned* ctrs, int* live, const int4* work, int set,
                          int grid, cudaStream_t s);
int launch_reintegrate_fast(const BFHashDataStruct* hd, const BFHashParams* hpOld, const BFHashParams* hpNew, const BFDepthCameraParams* cp,
                            const float* depth, const void* color, const int4* work, int set, unsigned* ctrs, int* live, int grid, cudaStream_t s);
int fast_stencil_ctas_per_sm(bool fused);

// batch re-integration: up to BF_MULTI_MAX_OPS (old pose, new pose, frame) triples applied to every voxel of the union list in one pass; batch
// integration: (pose, frame) pairs, hpOld NULL in every op (the stencil's kOldPose = false instantiation).
// work item = {block x, y, z, slot}, its mask = 2 bits per op {old pose may touch the block, new pose may}.  Items are bucketed by cost (number of
// set bits, quartiles of 2 nOps): quartile 3 at workA[0 ..), quartile 2 at workA[cap - 1 ..] downwards, quartile 1 at workB[0 ..), quartile 0 at
// workB[cap - 1 ..] downwards (counts in ctrs[set + SET_WORK / SET_Q2 / SET_Q1 / SET_Q0]); the stencil deals them in that order, costliest first.
#define BF_MULTI_MAX_OPS 16
struct BFMultiOpDesc { const BFHashParams* hpOld; const BFHashParams* hpNew; const float* depth; const void* color; };
int launch_reintegrate_multi_fast(const BFHashDataStruct* hd, const BFMultiOpDesc* ops, int nOps, const BFDepthCameraParams* cp, const int4* workA, const int4* workB,
                                  const unsigned* maskA, const unsigned* maskB, unsigned workCap, int set, unsigned* ctrs, int* live, int grid, cudaStream_t s,
                                  unsigned long long* ktime = nullptr);

}  // namespace bf

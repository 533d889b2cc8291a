// sift_sweep.cuh -- the wgmma + TMA match sweep of sift_match.cu as the keyframe search (keyframe_search.cu) drives it: a device-resident job table
// and the tensor maps of the descriptor arrays.  Kept apart from sift_pairs.cuh because it needs the driver API's types.
#pragma once
#include <cuda.h>
#include <stdint.h>

namespace bf {

// ---- the wgmma + TMA match sweep over a device-resident job table (sift_match.cu) ----
struct SiftJobDev {
    const uint8_t* desA; int nA;       // the features this pass owns ("rows" of the pass)
    const uint8_t* desB; int nB;       // the features they are compared with
    int* rowResult; float* rowDist;    // row pass: outputs; column pass: inputs (indexed by image-1 feature)
    int* numMatches; float* outDist; uint2* outIdx;
    uint2 offset;
    int* colResult; int* done;         // column pass: match of each image-2 feature (-1 none), CTAs of the job that have finished
    const CUtensorMap* mapA; const CUtensorMap* mapB;      // TMA sweep: [n][128 B] tensor maps of the two descriptor arrays (box 128 x 128, 128-byte swizzle, zero fill past n)
};
// dJobs: [numJobs row-pass jobs | numJobs column-pass jobs]; gx1 / gx2: CTAs per job of each pass (ceil(max rows / 128))
int sift_wgmma_sweep(const SiftJobDev* dJobs, int numJobs, int gx1, int gx2, float distmax, float ratiomax, cudaStream_t s);
// [rows][128] bytes, box 128 x 128, 128-byte swizzle, rows past the end read as zeros; false when the driver has no encoder or the array is unusable
bool sift_encode_descriptor_map(const uint8_t* base, int rows, CUtensorMap* out);

}  // namespace bf

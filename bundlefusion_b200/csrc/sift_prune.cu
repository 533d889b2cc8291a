// sift_prune.cu -- correspondence / frame invalidation after a solve, for sm_90a (the device half of SBA::removeMaxResidualCUDA,
// FL/SBA.cpp:165-203; rows a16 / a19).  Implements bfSiftInvalidateImageToImage and bfSiftCheckForInvalidFrames of include/bf_sift.h.
//
// Behavioural source (what, not how): InvalidateImageToImageCU_Kernel / CheckForInvalidFramesSimpleCU_Kernel /
// CheckForInvalidFramesCU_Kernel, FL/SiftGPU/SIFTImageManager.cu:692-790.  Integer work, bit-exact.
// Verified under the CPU emulation of tests/cuda_emu (tests/test_sift_prune_emulated.py) and on the GPU (tests/test_zz_sift_prune_gpu.py).
#include "../../include/bf_sift.h"
#include "bf_common.cuh"

namespace bf {

extern unsigned long long g_launchCount;

// EntryJ::setInvalid / isValid, FL/SiftGPU/SIFTImageManager.h:51-59
__device__ __forceinline__ void set_invalid(BFEntryJ* e) { e->imgIdx_i = 0xFFFFFFFFu; e->imgIdx_j = 0xFFFFFFFFu; }

__global__ void __launch_bounds__(128)
sift_invalidate_pair_kernel(BFEntryJ* glob, unsigned numResiduals, unsigned imgI, unsigned imgJ) {
    const unsigned idx = blockDim.x * blockIdx.x + threadIdx.x;
    if (idx < numResiduals && glob[idx].imgIdx_i == imgI && glob[idx].imgIdx_j == imgJ) set_invalid(&glob[idx]);
}

// frames without any correspondence left in the solver's table lose their valid flag (Simple); the comprehensive variant first
// invalidates every still-valid correspondence that touches such a frame
__global__ void __launch_bounds__(128)
sift_invalid_frames_kernel(const int* __restrict__ numEntriesPerRow, int* validImages, unsigned numVars, BFEntryJ* glob, unsigned numResiduals, int comprehensive) {
    const unsigned idx = blockDim.x * blockIdx.x + threadIdx.x;
    if (comprehensive && idx < numResiduals) {
        const unsigned i = glob[idx].imgIdx_i, j = glob[idx].imgIdx_j;
        if (i != 0xFFFFFFFFu && ((i < numVars && numEntriesPerRow[i] == 0) || (j < numVars && numEntriesPerRow[j] == 0))) set_invalid(&glob[idx]);
    }
    if (idx < numVars && numEntriesPerRow[idx] == 0) validImages[idx] = 0;
}

}  // namespace bf

using namespace bf;

BF_API int bfSiftInvalidateImageToImage(BFEntryJ* d_globMatches, unsigned int globNumResiduals, unsigned int imgIdx_i, unsigned int imgIdx_j) {
    if (globNumResiduals == 0) return 0;
    if (!d_globMatches) return (int)cudaErrorInvalidValue;
    ++g_launchCount;
    sift_invalidate_pair_kernel<<<(globNumResiduals + 127) / 128, 128, 0, stream()>>>(d_globMatches, globNumResiduals, imgIdx_i, imgIdx_j);
    BF_CHECK(cudaGetLastError());
    return 0;
}

BF_API int bfSiftCheckForInvalidFrames(const int32_t* d_varToCorrNumEntriesPerRow, int32_t* d_validImages, unsigned int numVars, BFEntryJ* d_globMatches,
                                       unsigned int globNumResiduals, int comprehensive) {
    if (numVars == 0) return 0;
    if (!d_varToCorrNumEntriesPerRow || !d_validImages || (comprehensive && globNumResiduals > 0 && !d_globMatches)) return (int)cudaErrorInvalidValue;
    const unsigned n = comprehensive && globNumResiduals > numVars ? globNumResiduals : numVars;
    ++g_launchCount;
    sift_invalid_frames_kernel<<<(n + 127) / 128, 128, 0, stream()>>>(d_varToCorrNumEntriesPerRow, d_validImages, numVars, d_globMatches, globNumResiduals, comprehensive);
    BF_CHECK(cudaGetLastError());
    return 0;
}

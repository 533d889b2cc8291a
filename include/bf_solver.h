/*
 * bf_solver.h -- C-ABI of the bundle-adjustment solver path (SURVEY.md section 8, rows a10-a16).
 *
 * Part 1 re-exports, by NAME and machine-level signature, the `extern "C"` stubs FriedLiver's host code binds:
 *
 *   FL/Solver/CUDASolverBundling.cpp:8-16   evalMaxResidual, buildVariablesToCorrespondencesTableCUDA,
 *                                           solveBundlingStub, countHighResiduals,
 *                                           convertLiePosesToMatricesCU, collectHighResiduals
 *   FL/SBA.cpp:12-15                        convertMatricesToPosesCU, convertPosesToMatricesCU
 *
 * (FL/ = /root/reference/FriedLiver/Source/; C++ reference parameters are pointers at the ABI level.)
 * The POD structs mirror FL/Solver/SolverBundlingState.h:10-103, SolverBundlingParameters.h:6-31,
 * FL/SiftGPU/SIFTImageManager.h:45-60 (EntryJ) and FL/CUDACacheUtil.h:10-53 field for field; float3 arrays
 * are 12-byte packed triples, float4x4 is 16 row-major floats.
 *
 * Ownership follows the reference: the CALLER allocates every buffer in BFSolverState / BFSolverInput
 * (FL/Solver/CUDASolverBundling.cpp:42-86) and passes device pointers.  The library additionally keeps a
 * private block-sparse workspace per BFSolverState (keyed by d_deltaRot), created on first use; d_denseJtJ
 * (the reference's dense (6N)^2 matrix), d_Jp, d_zRot/d_zTrans and d_Ap_* are accepted but not needed.
 *
 * Part 2 (bfSolver*) is the sync-free entry: one call = one whole CUDASolverBundling::solve, all GN
 * iterations and PCG iterations on the device, early-outs evaluated on the device, no device->host copy.
 */
#ifndef BF_SOLVER_H
#define BF_SOLVER_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* FL/SiftGPU/SIFTImageManager.h:45-60 : 32 bytes; invalid <=> imgIdx_i == 0xFFFFFFFF */
typedef struct BFEntryJ {
    uint32_t imgIdx_i;
    uint32_t imgIdx_j;
    float    pos_i[3];   /* camera-space point in image i */
    float    pos_j[3];   /* camera-space point in image j */
} BFEntryJ;

/* FL/CUDACacheUtil.h:41-53 : six device pointers, one 80x60 (default) cache frame */
typedef struct BFCUDACachedFrame {
    float*   d_depthDownsampled;            /* W*H float                       */
    float*   d_cameraposDownsampled;        /* W*H float4                      */
    float*   d_intensityDownsampled;        /* W*H float                       */
    float*   d_intensityDerivsDownsampled;  /* W*H float2                      */
    uint8_t* d_normalsDownsampledUCHAR4;    /* W*H uchar4                      */
    float*   d_normalsDownsampled;          /* W*H float4                      */
} BFCUDACachedFrame;

/* FL/Solver/SolverBundlingState.h:10-34 : 128 bytes, 16-byte aligned (float4 member) */
typedef struct BFSolverInput {
    BFEntryJ* d_correspondences;                 /*   0 */
    int32_t*  d_variablesToCorrespondences;      /*   8 */
    int32_t*  d_numEntriesPerRow;                /*  16 */
    uint32_t  numberOfCorrespondences;           /*  24 */
    uint32_t  numberOfImages;                    /*  28 */
    uint32_t  maxNumberOfImages;                 /*  32 */
    uint32_t  maxCorrPerImage;                   /*  36 */
    const int32_t* d_validImages;                /*  40 */
    const BFCUDACachedFrame* d_cacheFrames;      /*  48 */
    uint32_t  denseDepthWidth;                   /*  56 */
    uint32_t  denseDepthHeight;                  /*  60 */
#if defined(__GNUC__) || defined(__CUDACC__)
    float     intrinsics[4] __attribute__((aligned(16)));   /* 64: fx, fy, mx, my */
#else
    __declspec(align(16)) float intrinsics[4];
#endif
    uint32_t  maxNumDenseImPairs;                /*  80 */
    uint32_t  _pad0;
    float     colorFocalLength[2];               /*  88 */
    const float* weightsSparse;                  /*  96  HOST arrays, one weight per GN iteration */
    const float* weightsDenseDepth;              /* 104 */
    const float* weightsDenseColor;              /* 112 */
} BFSolverInput;

/* FL/Solver/SolverBundlingState.h:37-92 : 29 device pointers (float3 = 3 packed floats) */
typedef struct BFSolverState {
    float* d_deltaRot;  float* d_deltaTrans;
    float* d_xRot;      float* d_xTrans;         /* the unknowns (in/out), [N][3] each */
    float* d_rRot;      float* d_rTrans;
    float* d_zRot;      float* d_zTrans;
    float* d_pRot;      float* d_pTrans;
    float* d_Jp;
    float* d_Ap_XRot;   float* d_Ap_XTrans;
    float* d_scanAlpha;
    float* d_rDotzOld;
    float* d_precondionerRot; float* d_precondionerTrans;
    float* d_sumResidual;
    int32_t* d_countHighResidual;
    float* d_denseJtJ;  float* d_denseJtr;  float* d_denseCorrCounts;
    float* d_xTransforms;        /* [N][16] */
    float* d_xTransformInverses; /* [N][16] */
    uint32_t* d_denseOverlappingImages;   /* uint2 per pair */
    int32_t*  d_numDenseOverlappingImages;
    int32_t*  d_corrCount;  int32_t* d_corrCountColor;  float* d_sumResidualColor;
} BFSolverState;

/* FL/Solver/SolverBundlingParameters.h:6-31 : 68 bytes */
typedef struct BFSolverParameters {
    uint32_t nNonLinearIterations;
    uint32_t nLinIterations;
    float verifyOptDistThresh;
    float verifyOptPercentThresh;
    float highResidualThresh;
    float denseDistThresh;
    float denseNormalThresh;
    float denseColorThresh;
    float denseColorGradientMin;
    float denseDepthMin;
    float denseDepthMax;
    uint8_t useDenseDepthAllPairwise;  /* bool */
    uint8_t _pad0[3];
    uint32_t denseOverlapCheckSubsampleFactor;
    float weightSparse;
    float weightDenseDepth;
    float weightDenseColor;
    uint8_t useDense;                  /* bool */
    uint8_t _pad1[3];
} BFSolverParameters;

/* FL/Solver/SolverBundlingState.h:94-103 */
typedef struct BFSolverStateAnalysis {
    int32_t* d_maxResidualIndex;
    float*   d_maxResidual;
    int32_t* h_maxResidualIndex;
    float*   h_maxResidual;
} BFSolverStateAnalysis;

/* ---------------- Part 1: reference-named stubs ---------------- */

/* FL/Solver/SolverBundling.cu:1137-1220.  `timer` (CUDATimer*) is ignored (the reference passes NULL,
 * CUDASolverBundling.cpp:28).  convergenceAnalysis (may be NULL) receives nNonLinearIterations+1 energies. */
void solveBundlingStub(BFSolverInput* input, BFSolverState* state, BFSolverParameters* parameters,
                       BFSolverStateAnalysis* analysis, float* convergenceAnalysis, void* timer);
/* :1250-1264 -- fills the reference-format [image][slot] table (slot order: ascending correspondence index,
 * i.e. deterministic, where the reference's atomic append is not); correspondences beyond maxCorrPerImage
 * of either image are invalidated exactly as :1241-1245 does. */
void buildVariablesToCorrespondencesTableCUDA(BFEntryJ* d_correspondences, unsigned int numberOfCorrespondences,
                                              unsigned int maxNumCorrespondencesPerImage,
                                              int* d_variablesToCorrespondences, int* d_numEntriesPerRow, void* timer);
/* :552-564 -- per-512-correspondence block maxima into analysis->d_maxResidual / d_maxResidualIndex */
void evalMaxResidual(BFSolverInput* input, BFSolverState* state, BFSolverStateAnalysis* analysis,
                     BFSolverParameters* parameters, void* timer);
/* :670-687 (synchronises, returns the count) */
int countHighResiduals(BFSolverInput* input, BFSolverState* state, BFSolverParameters* parameters, void* timer);
/* :491-505 */
void collectHighResiduals(BFSolverInput* input, BFSolverState* state, BFSolverStateAnalysis* analysis,
                          BFSolverParameters* parameters, void* timer);
/* :1122-1130 */
void convertLiePosesToMatricesCU(const float* d_rot, const float* d_trans, unsigned int numTransforms,
                                 float* d_transforms, float* d_transformInvs);
/* FL/SBA.cu:86-98 and :111-119 (only entries with d_validImages[i] != 0 are written) */
void convertMatricesToPosesCU(const float* d_transforms, unsigned int numTransforms, float* d_rot, float* d_trans,
                              const int* d_validImages);
void convertPosesToMatricesCU(const float* d_rot, const float* d_trans, unsigned int numImages, float* d_transforms,
                              const int* d_validImages);

/* ---------------- Part 2: H100-native extension ---------------- */

/* One whole solve, asynchronous on the library stream.  weights*: HOST arrays of nNonLinearIterations entries
 * (copied into the launch).  Returns 0 or a cudaError_t. */
int bfSolverSolve(const BFSolverInput* input, const BFSolverState* state, const BFSolverParameters* parameters);

/* statistics of the last bfSolverSolve on this state (synchronises):
 * out[0] = GN iterations run, out[1] = PCG iterations run (all GN iterations), out[2] = image pairs (6x6 blocks),
 * out[3] = overlapping dense image pairs (last GN iteration), out[4] = last max|delta| * 1e6 (fixed point), out[5] = error flag,
 * out[6] = converged early, out[7] = dense pairs with non-zero weight */
int bfSolverGetStats(const BFSolverState* state, unsigned long long out[8]);

/* CUDASolverBundling::getMaxResidual's device part (FL/Solver/CUDASolverBundling.cpp:313-329) without the host
 * reduction: writes {max residual, index as float bits} to d_out[0..1].  Asynchronous. */
int bfSolverMaxResidual(const BFSolverInput* input, const BFSolverState* state, const BFSolverParameters* parameters,
                        float* d_out2);

/* bytes of private workspace the library holds for a solver of this size */
size_t bfSolverWorkspaceBytes(unsigned int maxNumberOfImages, unsigned int maxNumResiduals);
int bfSolverReleaseWorkspace(const BFSolverState* state);
/* Creates (or grows) the library-private workspace of `state` for up to maxNumberOfImages images and maxNumResiduals correspondences now, so that no
 * later bfSolverSolve has to: a solve whose correspondence count crosses the workspace's capacity frees and re-allocates it (cudaFree / cudaMalloc:
 * device-wide synchronisation, measured at hundreds of milliseconds when other streams are busy).  withDenseTerm != 0 also creates the pair tables of
 * the dense depth / colour term.  A caller with a steady-state loop (csrc/frame_loop.cu) reserves at start-up. */
int bfSolverReserveWorkspace(const BFSolverState* state, unsigned int maxNumberOfImages, unsigned int maxNumResiduals, int withDenseTerm);

/* Test / diagnosis accessor: the dense depth/colour normal equations of the last Gauss-Newton iteration that built them, in the
 * reference's layout -- what it keeps in SolverState::d_denseJtJ [(6N)^2, row-major, translation first per image] and d_denseJtr [6N]
 * (FL/Solver/SolverBundling.cu:308-471).  Either output may be NULL.  Asynchronous device-to-device copies. */
int bfSolverDebugDenseSystem(const BFSolverState* state, unsigned int numberOfImages, float* d_JtJ, float* d_Jtr);

/* ---- one solve sharded over the GPUs of a box (one process per GPU) ----
 * The rows of the block-sparse J^T J are dealt to the ranks (row v to rank v mod world).  Inside the persistent PCG kernel a rank computes (J^T J p)(v)
 * for its rows only and stores each 6-vector straight into every rank's exchange buffer over NVLink (peer stores), with its partial p.Ap sums; one
 * barrier across the GPUs per iteration (release / acquire flags in peer memory), after which every rank holds the whole vector and forms the same
 * dot products in the same order -- the replicated state (poses, residuals, directions) stays bit-identical on all ranks, no further exchange, and the
 * 6N pose update is everywhere when the kernel ends.  What is replicated: the per-iteration vector updates (6N) and the per-GN-iteration block build.
 * Set-up, once per solver object (all ranks, same sizes): bfSolverPeerCreate -> all-gather the 64-byte handles (e.g. torch.distributed) ->
 * bfSolverPeerConnect(rank, world, handles[world][64]).  Every rank then calls bfSolverSolve with IDENTICAL inputs.  Requires peer access between the
 * devices (NVLink / NVSwitch) and world <= 8.  The sparse term only is sharded (the dense term's rows follow the same ownership). */
int bfSolverPeerCreate(const BFSolverState* state, unsigned int maxImages, unsigned int maxCorrespondences, void* ipcHandleOut64);
int bfSolverPeerConnect(const BFSolverState* state, int rank, int world, const void* ipcHandles);
int bfSolverPeerDisconnect(const BFSolverState* state);

#ifdef __cplusplus
}
#endif
#endif /* BF_SOLVER_H */

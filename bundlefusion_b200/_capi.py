"""ctypes view of the C-ABI declared in include/*.h.

The shared library is built in-tree by ``__graft_entry__.build()`` (``make -C
bundlefusion_b200/csrc``).  There is NO CPU fallback: ``lib()`` raises if the library is
missing, and every compute entry point needs a CUDA device.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libbundlefusion_b200.so")

BF_SDF_BLOCK_SIZE = 8
BF_SDF_BLOCK_VOXELS = 512
BF_HASH_BUCKET_SIZE = 4
BF_LOCK_ENTRY = -1
BF_FREE_ENTRY = -2


class BFFloat4x4(C.Structure):
    _fields_ = [("m", C.c_float * 16)]


class BFHashEntry(C.Structure):
    _fields_ = [("pos", C.c_int32 * 3), ("ptr", C.c_int32), ("offset", C.c_uint32), ("_pad", C.c_uint32 * 3)]


HASH_ENTRY_INTS = 8        # sizeof(BFHashEntry) / 4: the MSVC layout of `__align__(16) struct HashEntry` (32 bytes)


class BFVoxel(C.Structure):
    _fields_ = [("sdf", C.c_float), ("weight", C.c_float), ("color", C.c_uint8 * 4)]


class _Dummy2(C.Structure):
    _pack_ = 8
    _fields_ = [("v", C.c_uint32 * 2)]


class BFHashParams(C.Structure):
    _fields_ = [
        ("m_rigidTransform", BFFloat4x4),
        ("m_rigidTransformInverse", BFFloat4x4),
        ("m_hashNumBuckets", C.c_uint32),
        ("m_hashBucketSize", C.c_uint32),
        ("m_hashMaxCollisionLinkedListSize", C.c_uint32),
        ("m_numSDFBlocks", C.c_uint32),
        ("m_SDFBlockSize", C.c_int32),
        ("m_virtualVoxelSize", C.c_float),
        ("m_numOccupiedBlocks", C.c_uint32),
        ("m_maxIntegrationDistance", C.c_float),
        ("m_truncScale", C.c_float),
        ("m_truncation", C.c_float),
        ("m_integrationWeightSample", C.c_uint32),
        ("m_integrationWeightMax", C.c_uint32),
        ("m_streamingVoxelExtents", C.c_float * 3),
        ("m_streamingGridDimensions", C.c_int32 * 3),
        ("m_streamingMinGridPos", C.c_int32 * 3),
        ("m_streamingInitialChunkListSize", C.c_uint32),
        ("m_dummy", C.c_uint64),  # uint2, 8-byte aligned
    ]


class BFDepthCameraParams(C.Structure):
    _fields_ = [
        ("fx", C.c_float), ("fy", C.c_float), ("mx", C.c_float), ("my", C.c_float),
        ("m_imageWidth", C.c_uint32), ("m_imageHeight", C.c_uint32),
        ("m_sensorDepthWorldMin", C.c_float), ("m_sensorDepthWorldMax", C.c_float),
    ]


class BFDepthCameraData(C.Structure):
    _fields_ = [("d_depthData", C.c_void_p), ("d_colorData", C.c_void_p)]


class BFHashDataStruct(C.Structure):
    _fields_ = [
        ("d_heap", C.c_void_p),
        ("d_heapCounter", C.c_void_p),
        ("d_hashDecision", C.c_void_p),
        ("d_hashDecisionPrefix", C.c_void_p),
        ("d_hash", C.c_void_p),
        ("d_hashCompactified", C.c_void_p),
        ("d_hashCompactifiedCounter", C.c_void_p),
        ("d_SDFBlocks", C.c_void_p),
        ("d_hashBucketMutex", C.c_void_p),
        ("m_bIsOnGPU", C.c_uint8),
    ]


class BFBlockKeySet(C.Structure):
    _fields_ = [("d_keys", C.c_void_p), ("d_counters", C.c_void_p), ("capacity", C.c_uint32)]


assert C.sizeof(BFHashParams) == 224, C.sizeof(BFHashParams)
assert BFHashParams.m_dummy.offset == 216
assert C.sizeof(BFHashEntry) == 32 and C.sizeof(BFVoxel) == 12
assert C.sizeof(BFDepthCameraParams) == 32 and C.sizeof(BFHashDataStruct) == 80

# every symbol include/bf_tsdf.h declares (the "library exports what the header says" test walks this)
TSDF_SYMBOLS = [
    "updateConstantHashParams", "updateConstantDepthCameraParams", "bindInputDepthColorTextures",
    "resetCUDA", "resetHashBucketMutexCUDA", "allocCUDA", "fillDecisionArrayCUDA", "compactifyHashCUDA",
    "compactifyHashAllInOneCUDA", "integrateDepthMapCUDA", "deIntegrateDepthMapCUDA", "starveVoxelsKernelCUDA",
    "garbageCollectIdentifyCUDA", "garbageCollectFreeCUDA",
    "bfSetStream", "bfGetStream", "bfGetLastErrorString", "bfTsdfAuxBytes", "bfTsdfReset", "bfTsdfIntegrateFrame",
    "bfTsdfGarbageCollect", "bfTsdfGetHeapFreeCount", "bfTsdfGetNumOccupiedBlocks", "bfTsdfGetLastFrameStats",
    "bfTsdfReleaseAux", "bfTsdfReintegrateFrame", "bfGetLaunchCount", "bfTsdfSetProfiling", "bfTsdfGetProfile", "bfTsdfGetProfileEx", "bfTsdfSetLanes", "bfTsdfSetArithmetic", "bfTsdfReintegrateBatch", "bfTsdfSetBatching",
    "bfTsdfIntegrateBatch", "bfTsdfCountBlocks", "bfTsdfBlockKeyLoad", "bfTsdfBlockKeyMerge", "bfTsdfRehash",
]

HOST_SYMBOLS = ["bfMat4Inverse", "bfTsdfRunOps"]

SENS_SYMBOLS = ["bfSensOpen", "bfSensReadFrame", "bfSensReadFrameRaw", "bfSensClose", "bfSensCreate", "bfSensAppendFrame", "bfSensFinish",
                "bfSensDecodeJpeg", "bfSensDecodePng", "bfSensErrorString"]

RAYCAST_SYMBOLS = ["updateConstantRayCastParams", "rayIntervalSplatCUDA", "resetRayIntervalSplatCUDA", "renderCS",
                   "bfRayCastSplat", "bfRayCastRender", "bfRayCastComputeNormals", "bfRayCastRenderPose"]


class BFRayCastParams(C.Structure):
    """include/bf_raycast.h (FL/DepthSensing/CUDARayCastParams.h:8-27), 192 bytes"""
    _fields_ = [("m_viewMatrix", BFFloat4x4), ("m_viewMatrixInverse", BFFloat4x4),
                ("mx", C.c_float), ("my", C.c_float), ("fx", C.c_float), ("fy", C.c_float),
                ("m_width", C.c_uint32), ("m_height", C.c_uint32), ("m_numOccupiedSDFBlocks", C.c_uint32), ("m_maxNumVertices", C.c_uint32),
                ("m_splatMinimum", C.c_int32), ("m_minDepth", C.c_float), ("m_maxDepth", C.c_float), ("m_rayIncrement", C.c_float),
                ("m_thresSampleDist", C.c_float), ("m_thresDist", C.c_float), ("m_useGradients", C.c_uint8), ("m_pad", C.c_uint8 * 3), ("dummy0", C.c_uint32)]


class BFRayCastData(C.Structure):
    """include/bf_raycast.h (FL/DepthSensing/RayCastSDFUtil.h:296-302): seven device pointers"""
    _fields_ = [("d_depth", C.c_void_p), ("d_depth4", C.c_void_p), ("d_normals", C.c_void_p), ("d_colors", C.c_void_p), ("d_vertexBuffer", C.c_void_p),
                ("d_rayIntervalSplatMin", C.c_void_p), ("d_rayIntervalSplatMax", C.c_void_p)]

MARCHINGCUBES_SYMBOLS = ["resetMarchingCubesCUDA", "extractIsoSurfaceCUDA", "bfMarchingCubesExtract", "bfMarchingCubesCreate", "bfMarchingCubesDestroy",
                         "bfMarchingCubesExtractIsoSurface", "bfMarchingCubesClearMeshBuffer", "bfMarchingCubesGetSoup", "bfMarchingCubesSaveMesh",
                         "bfMeshMergeCloseVertices", "bfMeshRemoveDuplicateFaces", "bfMeshSavePly", "bfMarchingCubesCount", "bfMarchingCubesExtractRange",
                         "bfMarchingCubesExtractIsoSurfaceWhole", "bfMarchingCubesGetLastExtraction", "bfMeshApplyTransform", "bfMeshWeldWorkspaceBytes",
                         "bfMeshWeld"]
BF_MC_CHUNK_SLOTS = 512                  # hash slots per chunk of the count pass and of bfMarchingCubesExtractRange


class BFMarchingCubesParams(C.Structure):
    """include/bf_marchingcubes.h (FL/DepthSensing/MarchingCubesSDFUtil.h:9-23), 64 bytes"""
    _fields_ = [("m_boxEnabled", C.c_uint8), ("m_pad", C.c_uint8 * 3), ("m_minCorner", C.c_float * 3), ("m_maxNumTriangles", C.c_uint32), ("m_maxCorner", C.c_float * 3),
                ("m_sdfBlockSize", C.c_uint32), ("m_hashNumBuckets", C.c_uint32), ("m_hashBucketSize", C.c_uint32),
                ("m_threshMarchingCubes", C.c_float), ("m_threshMarchingCubes2", C.c_float), ("dummy", C.c_float * 3)]


class BFMarchingCubesData(C.Structure):
    """include/bf_marchingcubes.h (FL/DepthSensing/MarchingCubesSDFUtil.h:281-286)"""
    _fields_ = [("d_params", C.c_void_p), ("d_numTriangles", C.c_void_p), ("d_triangles", C.c_void_p), ("m_bIsOnGPU", C.c_uint8)]


class BFMarchingCubesWholeInfo(C.Structure):
    """include/bf_marchingcubes.h: what bfMarchingCubesExtractIsoSurfaceWhole did, 40 bytes"""
    _fields_ = [("trianglesCounted", C.c_uint64), ("trianglesExtracted", C.c_uint64), ("chunks", C.c_uint32), ("parts", C.c_uint32),
                ("largestPart", C.c_uint32), ("bufferTriangles", C.c_uint32), ("bufferEnlarged", C.c_uint32), ("hostSyncs", C.c_uint32)]


class BFMeshWeldInfo(C.Structure):
    """include/bf_marchingcubes.h: what bfMeshWeld did, 56 bytes"""
    _fields_ = [("trianglesIn", C.c_uint64), ("verticesOut", C.c_uint64), ("degenerateFaces", C.c_uint64), ("duplicateFaces", C.c_uint64),
                ("facesOut", C.c_uint64), ("cells", C.c_uint32), ("rounds", C.c_uint32), ("hostSyncs", C.c_uint32)]


CACHE_SYMBOLS = ["bfCacheStoreFrame"]
INGEST_SYMBOLS = ["bfIngestFrame"]
BUNDLER_SYMBOLS = ["computeSiftTransformCU", "initNextGlobalTransformCU", "updateTrajectoryCU", "bfTrajectorySelectReintegration",
                   "bfTrajectoryCreate", "bfTrajectoryDestroy", "bfTrajectoryAddFrame", "bfTrajectoryUpdateOptimizedTransform",
                   "bfTrajectoryGenerateUpdateLists", "bfTrajectoryConfirmIntegration", "bfTrajectoryGetTopFromReIntegrateList",
                   "bfTrajectoryGetTopFromIntegrateList", "bfTrajectoryGetTopFromDeIntegrateList", "bfTrajectoryGetNumOptimizedFrames",
                   "bfTrajectoryGetNumAddedFrames", "bfTrajectoryGetNumActiveOperations", "bfTrajectoryGetFrameType", "bfTrajectoryGetFrameDist",
                   "bfTrajectoryGetOptimizedTransforms"]

SIFT_SYMBOLS = ["bfSiftMatchBatch", "bfSiftSortKeyPointMatches", "bfSiftFilterKeyPointMatches", "bfSiftFilterMatchesBySurfaceArea", "bfSiftFilterMatchesByDenseVerify",
                "bfSiftAddCurrToResiduals", "bfSiftWorkspaceBytes", "bfSiftReleaseWorkspace", "bfSiftReserveWorkspace", "bfSiftDetect", "bfSiftDetectWorkspaceBytes",
                "bfSiftDetectReleaseWorkspace", "bfSiftInvalidateImageToImage", "bfSiftCheckForInvalidFrames", "bfSiftFilterFrames",
                "bfSiftAddCurrToResidualsIfMatched", "bfSiftVerifyTrajectory", "bfSiftFuseToGlobal", "bfSiftSetMatchSweep", "bfSiftGetMatchInfo"]

SOLVER_SYMBOLS = [
    "solveBundlingStub", "buildVariablesToCorrespondencesTableCUDA", "evalMaxResidual", "countHighResiduals", "collectHighResiduals",
    "convertLiePosesToMatricesCU", "convertMatricesToPosesCU", "convertPosesToMatricesCU",
    "bfSolverSolve", "bfSolverGetStats", "bfSolverMaxResidual", "bfSolverWorkspaceBytes", "bfSolverReleaseWorkspace", "bfSolverReserveWorkspace",
    "bfSolverDebugDenseSystem", "bfSolverPeerCreate", "bfSolverPeerConnect", "bfSolverPeerDisconnect",
    "bfSolverSetGridPolicy", "bfSolverGetLaunchInfo",
]


class BFSiftDetectParams(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("depthWidth", C.c_uint32), ("depthHeight", C.c_uint32), ("depthMin", C.c_float),
                ("depthMax", C.c_float), ("minKeyScale", C.c_float), ("featureCountThreshold", C.c_int32), ("maxKeyPoints", C.c_uint32)]


class BFImagePairMatch(C.Structure):      # FL/SiftGPU/SIFTImageManager.h:38-42
    _fields_ = [("d_numMatches", C.c_void_p), ("d_distances", C.c_void_p), ("d_keyPointIndices", C.c_void_p)]


class BFSiftMatchJob(C.Structure):
    _fields_ = [("d_des1", C.c_void_p), ("num1", C.c_int32), ("d_des2", C.c_void_p), ("num2", C.c_int32),
                ("out", BFImagePairMatch), ("keyPointOffset", C.c_uint32 * 2)]


class BFEntryJ(C.Structure):
    _fields_ = [("imgIdx_i", C.c_uint32), ("imgIdx_j", C.c_uint32), ("pos_i", C.c_float * 3), ("pos_j", C.c_float * 3)]


class BFCUDACachedFrame(C.Structure):
    _fields_ = [("d_depthDownsampled", C.c_void_p), ("d_cameraposDownsampled", C.c_void_p), ("d_intensityDownsampled", C.c_void_p),
                ("d_intensityDerivsDownsampled", C.c_void_p), ("d_normalsDownsampledUCHAR4", C.c_void_p), ("d_normalsDownsampled", C.c_void_p)]


class _F4(C.Structure):
    _pack_ = 16
    _fields_ = [("v", C.c_float * 4)]


class BFIngestParams(C.Structure):         # FL/CUDAImageManager.cpp:88-137 settings
    _fields_ = [("depthWidth", C.c_uint32), ("depthHeight", C.c_uint32), ("colorWidth", C.c_uint32), ("colorHeight", C.c_uint32),
                ("widthIntegration", C.c_uint32), ("heightIntegration", C.c_uint32), ("erodeIterations", C.c_int32), ("erodeStructureSize", C.c_int32),
                ("erodeDThresh", C.c_float), ("erodeFracReq", C.c_float), ("depthSigmaD", C.c_float), ("depthSigmaR", C.c_float)]


class BFCacheParams(C.Structure):          # what CUDACache's constructor latches, FL/CUDACache.cpp:14-40
    _fields_ = [("inputDepthWidth", C.c_uint32), ("inputDepthHeight", C.c_uint32), ("inputColorWidth", C.c_uint32), ("inputColorHeight", C.c_uint32),
                ("width", C.c_uint32), ("height", C.c_uint32), ("inputIntrinsicsInv", C.c_float * 16),
                ("filterIntensitySigma", C.c_float), ("filterDepthSigmaD", C.c_float), ("filterDepthSigmaR", C.c_float)]


class BFSolverInput(C.Structure):
    _fields_ = [
        ("d_correspondences", C.c_void_p), ("d_variablesToCorrespondences", C.c_void_p), ("d_numEntriesPerRow", C.c_void_p),
        ("numberOfCorrespondences", C.c_uint32), ("numberOfImages", C.c_uint32), ("maxNumberOfImages", C.c_uint32), ("maxCorrPerImage", C.c_uint32),
        ("d_validImages", C.c_void_p), ("d_cacheFrames", C.c_void_p), ("denseDepthWidth", C.c_uint32), ("denseDepthHeight", C.c_uint32),
        ("intrinsics", C.c_float * 4), ("maxNumDenseImPairs", C.c_uint32), ("_pad0", C.c_uint32), ("colorFocalLength", C.c_float * 2),
        ("weightsSparse", C.POINTER(C.c_float)), ("weightsDenseDepth", C.POINTER(C.c_float)), ("weightsDenseColor", C.POINTER(C.c_float)),
        ("_tail", C.c_uint64),
    ]


_STATE_FIELDS = ["d_deltaRot", "d_deltaTrans", "d_xRot", "d_xTrans", "d_rRot", "d_rTrans", "d_zRot", "d_zTrans", "d_pRot", "d_pTrans", "d_Jp",
                 "d_Ap_XRot", "d_Ap_XTrans", "d_scanAlpha", "d_rDotzOld", "d_precondionerRot", "d_precondionerTrans", "d_sumResidual",
                 "d_countHighResidual", "d_denseJtJ", "d_denseJtr", "d_denseCorrCounts", "d_xTransforms", "d_xTransformInverses",
                 "d_denseOverlappingImages", "d_numDenseOverlappingImages", "d_corrCount", "d_corrCountColor", "d_sumResidualColor"]


class BFSolverState(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in _STATE_FIELDS]


class BFSolverParameters(C.Structure):
    _fields_ = [
        ("nNonLinearIterations", C.c_uint32), ("nLinIterations", C.c_uint32), ("verifyOptDistThresh", C.c_float), ("verifyOptPercentThresh", C.c_float),
        ("highResidualThresh", C.c_float), ("denseDistThresh", C.c_float), ("denseNormalThresh", C.c_float), ("denseColorThresh", C.c_float),
        ("denseColorGradientMin", C.c_float), ("denseDepthMin", C.c_float), ("denseDepthMax", C.c_float),
        ("useDenseDepthAllPairwise", C.c_uint8), ("_pad0", C.c_uint8 * 3), ("denseOverlapCheckSubsampleFactor", C.c_uint32),
        ("weightSparse", C.c_float), ("weightDenseDepth", C.c_float), ("weightDenseColor", C.c_float), ("useDense", C.c_uint8), ("_pad1", C.c_uint8 * 3),
    ]


class BFSolverStateAnalysis(C.Structure):
    _fields_ = [("d_maxResidualIndex", C.c_void_p), ("d_maxResidual", C.c_void_p), ("h_maxResidualIndex", C.c_void_p), ("h_maxResidual", C.c_void_p)]


assert C.sizeof(BFEntryJ) == 32 and C.sizeof(BFCUDACachedFrame) == 48
assert BFSolverInput.intrinsics.offset == 64 and BFSolverInput.colorFocalLength.offset == 88 and BFSolverInput.weightsSparse.offset == 96
assert C.sizeof(BFSolverInput) == 128 and C.sizeof(BFSolverState) == 232 and C.sizeof(BFSolverParameters) == 68


class BFTsdfOp(C.Structure):
    _fields_ = [("kind", C.c_int32), ("frame", C.c_int32), ("pose", C.c_float * 16)]


BF_TSDF_OP_INTEGRATE, BF_TSDF_OP_DEINTEGRATE, BF_TSDF_OP_GARBAGE_COLLECT = 0, 1, 2

_lib = None


def lib() -> C.CDLL:
    """Load libbundlefusion_b200.so (raises RuntimeError if it has not been built)."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("BF_B200_LIB", LIB_PATH)        # development: A/B a differently compiled build of the same sources
    if not os.path.exists(path):
        raise RuntimeError(
            f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C bundlefusion_b200/csrc`). There is no CPU fallback.")
    L = C.CDLL(path)
    P = C.POINTER
    vp = C.c_void_p
    # reference-named stubs
    L.updateConstantHashParams.argtypes = [P(BFHashParams)]
    L.updateConstantDepthCameraParams.argtypes = [P(BFDepthCameraParams)]
    L.bindInputDepthColorTextures.argtypes = [P(BFDepthCameraData), C.c_uint, C.c_uint]
    for name in ("resetCUDA", "resetHashBucketMutexCUDA", "fillDecisionArrayCUDA", "compactifyHashCUDA",
                 "starveVoxelsKernelCUDA", "garbageCollectIdentifyCUDA", "garbageCollectFreeCUDA"):
        getattr(L, name).argtypes = [P(BFHashDataStruct), P(BFHashParams)]
        getattr(L, name).restype = None
    L.allocCUDA.argtypes = [P(BFHashDataStruct), P(BFHashParams), P(BFDepthCameraData), P(BFDepthCameraParams), vp]
    L.allocCUDA.restype = None
    L.compactifyHashAllInOneCUDA.argtypes = [P(BFHashDataStruct), P(BFHashParams)]
    L.compactifyHashAllInOneCUDA.restype = C.c_uint
    for name in ("integrateDepthMapCUDA", "deIntegrateDepthMapCUDA"):
        getattr(L, name).argtypes = [P(BFHashDataStruct), P(BFHashParams), P(BFDepthCameraData), P(BFDepthCameraParams)]
        getattr(L, name).restype = None
    # extension
    L.bfSetStream.argtypes = [vp]
    L.bfSetStream.restype = None
    L.bfGetStream.restype = vp
    L.bfGetLastErrorString.restype = C.c_char_p
    L.bfTsdfAuxBytes.argtypes = [P(BFHashParams)]
    L.bfTsdfAuxBytes.restype = C.c_size_t
    L.bfTsdfReset.argtypes = [P(BFHashDataStruct), P(BFHashParams)]
    L.bfTsdfSetBatching.argtypes = [C.c_int]
    L.bfTsdfSetBatching.restype = C.c_int
    L.bfTsdfSetArithmetic.argtypes = [C.c_int]
    L.bfTsdfSetArithmetic.restype = C.c_int
    L.bfTsdfSetLanes.argtypes = [C.c_int]
    L.bfTsdfSetLanes.restype = C.c_int
    L.bfTsdfIntegrateFrame.argtypes = [P(BFHashDataStruct), P(BFHashParams), P(BFDepthCameraData), P(BFDepthCameraParams), C.c_int]
    L.bfTsdfGarbageCollect.argtypes = [P(BFHashDataStruct), P(BFHashParams)]
    L.bfTsdfGetHeapFreeCount.argtypes = [P(BFHashDataStruct), P(C.c_uint)]
    L.bfTsdfGetNumOccupiedBlocks.argtypes = [P(BFHashDataStruct), P(C.c_uint)]
    L.bfTsdfGetLastFrameStats.argtypes = [P(BFHashDataStruct), C.c_ulonglong * 4]
    L.bfTsdfReleaseAux.argtypes = [P(BFHashDataStruct)]
    L.bfTsdfReintegrateFrame.argtypes = [P(BFHashDataStruct), P(BFHashParams), P(BFHashParams), P(BFDepthCameraData), P(BFDepthCameraParams)]
    L.bfGetLaunchCount.restype = C.c_ulonglong
    L.bfTsdfSetProfiling.argtypes = [C.c_int]
    L.bfTsdfGetProfile.argtypes = [P(BFHashDataStruct), C.c_ulonglong * 8]
    L.bfTsdfGetProfileEx.argtypes = [P(BFHashDataStruct), C.c_ulonglong * 16]
    L.bfMat4Inverse.argtypes = [P(C.c_float), P(C.c_float)]
    L.bfMat4Inverse.restype = None
    L.bfTsdfRunOps.argtypes = [P(BFHashDataStruct), P(BFHashParams), P(BFDepthCameraParams), P(BFTsdfOp), C.c_int, P(vp), P(vp)]
    L.bfTsdfIntegrateBatch.argtypes = [P(BFHashDataStruct), P(BFHashParams), P(BFDepthCameraParams), vp, vp, C.c_int, vp, vp]
    L.bfTsdfCountBlocks.argtypes = [P(BFBlockKeySet), P(BFHashParams), P(BFDepthCameraParams), vp, vp, C.c_int, vp]
    L.bfTsdfBlockKeyLoad.argtypes = [P(BFBlockKeySet), C.c_uint32, vp, vp]
    L.bfTsdfBlockKeyMerge.argtypes = [P(BFBlockKeySet), P(BFBlockKeySet)]
    L.bfTsdfRehash.argtypes = [P(BFHashDataStruct), P(BFHashParams), P(BFHashDataStruct), P(BFHashParams), P(C.c_ulonglong)]
    # solver
    L.solveBundlingStub.argtypes = [P(BFSolverInput), P(BFSolverState), P(BFSolverParameters), P(BFSolverStateAnalysis), P(C.c_float), vp]
    L.solveBundlingStub.restype = None
    L.buildVariablesToCorrespondencesTableCUDA.argtypes = [vp, C.c_uint, C.c_uint, vp, vp, vp]
    L.buildVariablesToCorrespondencesTableCUDA.restype = None
    L.evalMaxResidual.argtypes = [P(BFSolverInput), P(BFSolverState), P(BFSolverStateAnalysis), P(BFSolverParameters), vp]
    L.evalMaxResidual.restype = None
    L.countHighResiduals.argtypes = [P(BFSolverInput), P(BFSolverState), P(BFSolverParameters), vp]
    L.countHighResiduals.restype = C.c_int
    L.collectHighResiduals.argtypes = [P(BFSolverInput), P(BFSolverState), P(BFSolverStateAnalysis), P(BFSolverParameters), vp]
    L.collectHighResiduals.restype = None
    L.convertLiePosesToMatricesCU.argtypes = [vp, vp, C.c_uint, vp, vp]
    L.convertLiePosesToMatricesCU.restype = None
    L.convertMatricesToPosesCU.argtypes = [vp, C.c_uint, vp, vp, vp]
    L.convertMatricesToPosesCU.restype = None
    L.convertPosesToMatricesCU.argtypes = [vp, vp, C.c_uint, vp, vp]
    L.convertPosesToMatricesCU.restype = None
    L.bfSolverSolve.argtypes = [P(BFSolverInput), P(BFSolverState), P(BFSolverParameters)]
    L.bfSolverGetStats.argtypes = [P(BFSolverState), C.c_ulonglong * 8]
    L.bfSolverSetGridPolicy.argtypes = [C.c_int]
    L.bfSolverSetGridPolicy.restype = C.c_int
    L.bfSolverGetLaunchInfo.argtypes = [P(BFSolverState), C.c_int * 4]
    L.bfSolverMaxResidual.argtypes = [P(BFSolverInput), P(BFSolverState), P(BFSolverParameters), vp]
    L.bfSolverWorkspaceBytes.argtypes = [C.c_uint, C.c_uint]
    L.bfSolverWorkspaceBytes.restype = C.c_size_t
    L.bfSolverReleaseWorkspace.argtypes = [P(BFSolverState)]
    L.bfSiftVerifyTrajectory.argtypes = [C.c_uint, vp, vp, C.c_uint, C.c_uint, P(C.c_float), vp] + [C.c_float] * 7 + [vp, vp]
    L.bfSiftFuseToGlobal.argtypes = [vp, vp, vp, vp, C.c_uint, vp, vp, vp, C.c_uint, P(C.c_float), C.c_uint, vp, vp, vp, C.c_uint, vp]
    L.bfSolverDebugDenseSystem.argtypes = [P(BFSolverState), C.c_uint, vp, vp]
    L.bfSolverPeerCreate.argtypes = [P(BFSolverState), C.c_uint, C.c_uint, vp]
    L.bfSolverPeerConnect.argtypes = [P(BFSolverState), C.c_int, C.c_int, C.c_char_p]
    L.bfSolverPeerDisconnect.argtypes = [P(BFSolverState)]
    L.bfCacheStoreFrame.argtypes = [P(BFCacheParams), vp, vp, P(BFCUDACachedFrame)]
    L.bfIngestFrame.argtypes = [P(BFIngestParams), vp, vp, vp, vp]
    L.computeSiftTransformCU.argtypes = [vp, vp, vp, C.c_uint, vp, C.c_uint, C.c_uint, vp]
    L.computeSiftTransformCU.restype = None
    L.initNextGlobalTransformCU.argtypes = [vp, C.c_uint, C.c_uint, vp, C.c_uint, C.c_uint]
    L.initNextGlobalTransformCU.restype = None
    L.updateTrajectoryCU.argtypes = [vp, C.c_uint, vp, C.c_uint, vp, C.c_uint, C.c_uint, vp]
    L.updateTrajectoryCU.restype = None
    L.bfTrajectorySelectReintegration.argtypes = [vp, vp, vp, C.c_uint, C.c_uint, C.c_float, C.c_float, vp, vp, vp]
    # SIFT descriptor matcher
    L.bfSiftMatchBatch.argtypes = [P(BFSiftMatchJob), C.c_int, C.c_float, C.c_float]
    L.bfSiftSetMatchSweep.argtypes = [C.c_int]
    L.bfSiftSetMatchSweep.restype = C.c_int
    L.bfSiftGetMatchInfo.argtypes = [C.c_int * 2]
    L.bfSiftSortKeyPointMatches.argtypes = [C.c_uint, C.c_uint, C.c_uint, vp, vp, vp]
    L.bfSiftFilterKeyPointMatches.argtypes = [C.c_uint, C.c_uint, C.c_uint] + [vp] * 9 + [P(C.c_float), C.c_uint, C.c_float]
    L.bfSiftAddCurrToResiduals.argtypes = [C.c_uint, C.c_uint, C.c_uint] + [vp] * 6 + [P(C.c_float)]
    L.bfSiftFilterMatchesBySurfaceArea.argtypes = [C.c_uint, C.c_uint, C.c_uint, vp, vp, vp, P(C.c_float), C.c_float, vp]
    L.bfSiftFilterMatchesByDenseVerify.argtypes = [C.c_uint] * 5 + [P(C.c_float), vp, vp, vp] + [C.c_float] * 7 + [vp]
    L.bfSiftWorkspaceBytes.restype = C.c_size_t
    L.bfSiftDetect.argtypes = [P(BFSiftDetectParams), vp, vp, vp, vp, vp, vp]
    L.bfSiftInvalidateImageToImage.argtypes = [vp, C.c_uint, C.c_uint, C.c_uint]
    L.bfSiftFilterFrames.argtypes = [C.c_uint, C.c_uint, C.c_uint, vp, vp, vp]
    L.bfSiftAddCurrToResidualsIfMatched.argtypes = [C.c_uint, C.c_uint, C.c_uint] + [vp] * 6 + [P(C.c_float), vp]
    L.bfSiftCheckForInvalidFrames.argtypes = [vp, vp, C.c_uint, vp, C.c_uint, C.c_int]
    L.bfSiftDetectWorkspaceBytes.restype = C.c_size_t
    _lib = L
    return L


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().bfGetLastErrorString().decode()
        raise RuntimeError(f"bundlefusion_b200: {what} failed with CUDA error {rc}: {msg}")

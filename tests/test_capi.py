"""CPU-side checks of the drop-in boundary: the shared library loads and exports every symbol the
headers declare, and the POD layouts match the reference's (sizes probed from the reference headers,
SURVEY.md section 8a / appendix Q1)."""
import ctypes as C
import os
import re

from bundlefusion_b200 import _capi as capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_pod_layouts():
    assert C.sizeof(capi.BFHashEntry) == 32          # `__align__(16) struct HashEntry` as MSVC lays it out (Q1); 5 ints + tail padding
    assert C.sizeof(capi.BFVoxel) == 12
    assert C.sizeof(capi.BFHashParams) == 224
    assert capi.BFHashParams.m_hashNumBuckets.offset == 128
    assert capi.BFHashParams.m_SDFBlockSize.offset == 144
    assert capi.BFHashParams.m_maxIntegrationDistance.offset == 156
    assert capi.BFHashParams.m_streamingVoxelExtents.offset == 176
    assert capi.BFHashParams.m_dummy.offset == 216
    assert C.sizeof(capi.BFDepthCameraParams) == 32
    assert C.sizeof(capi.BFDepthCameraData) == 16
    assert C.sizeof(capi.BFHashDataStruct) == 80
    assert capi.BFHashDataStruct.d_hash.offset == 32
    assert capi.BFHashDataStruct.d_hashBucketMutex.offset == 64
    assert capi.BFHashDataStruct.m_bIsOnGPU.offset == 72


def _declared_symbols(header):
    src = open(os.path.join(ROOT, "include", header)).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = re.findall(r"^[A-Za-z_][A-Za-z0-9_ \*]*?\b([A-Za-z_][A-Za-z0-9_]*)\s*\([^;{]*\)\s*;", src, flags=re.M)
    return [n for n in names if n not in ("aligned", "__attribute__", "align")]


def test_library_exports_every_declared_symbol():
    L = capi.lib()
    for header in sorted(os.listdir(os.path.join(ROOT, "include"))):
        if not header.endswith(".h"):
            continue
        names = _declared_symbols(header)
        assert names, header
        for n in names:
            assert hasattr(L, n), f"{header}: {n} not exported"


def test_symbol_list_matches_header():
    assert sorted(set(_declared_symbols("bf_tsdf.h"))) == sorted(set(capi.TSDF_SYMBOLS))
    assert sorted(set(_declared_symbols("bf_host.h"))) == sorted(set(capi.HOST_SYMBOLS))
    assert sorted(set(_declared_symbols("bf_solver.h"))) == sorted(set(capi.SOLVER_SYMBOLS))
    assert sorted(set(_declared_symbols("bf_sift.h"))) == sorted(set(capi.SIFT_SYMBOLS))
    assert sorted(set(_declared_symbols("bf_cache.h"))) == sorted(set(capi.CACHE_SYMBOLS))
    assert sorted(set(_declared_symbols("bf_ingest.h"))) == sorted(set(capi.INGEST_SYMBOLS))
    assert sorted(set(_declared_symbols("bf_bundler.h"))) == sorted(set(capi.BUNDLER_SYMBOLS))
    assert sorted(set(_declared_symbols("bf_raycast.h"))) == sorted(set(capi.RAYCAST_SYMBOLS))
    assert sorted(set(_declared_symbols("bf_sens.h"))) == sorted(set(capi.SENS_SYMBOLS))
    assert sorted(set(_declared_symbols("bf_marchingcubes.h"))) == sorted(set(capi.MARCHINGCUBES_SYMBOLS))


def test_frame_loop_op_log_and_frame_store_accessors():
    """bfFrameLoopSetOpLog / bfFrameLoopGetOpLog / bfFrameLoopGetFrame are declared, exported and refuse a null loop without a device"""
    from bundlefusion_b200 import frame_loop
    names = set(_declared_symbols("bf_frameloop.h"))
    L = frame_loop._bind(capi.lib())
    for n in ("bfFrameLoopSetOpLog", "bfFrameLoopGetOpLog", "bfFrameLoopGetFrame"):
        assert n in names and hasattr(L, n), n
    assert C.sizeof(capi.BFTsdfOp) == 72
    assert L.bfFrameLoopSetOpLog(None, 1) == 1                           # cudaErrorInvalidValue
    assert L.bfFrameLoopGetOpLog(None, None, None, 0) == 0
    d, c = C.c_void_p(), C.c_void_p()
    assert L.bfFrameLoopGetFrame(None, 0, C.byref(d), C.byref(c)) == 1


def test_solver_grid_policy_override_is_checked_on_the_host():
    """bfSolverSetGridPolicy / bfSolverGetLaunchInfo are exported; an unknown policy is refused without a device and leaves the policy as it was"""
    L = capi.lib()
    assert hasattr(L, "bfSolverSetGridPolicy") and hasattr(L, "bfSolverGetLaunchInfo")
    assert L.bfSolverSetGridPolicy(99) == 1                              # cudaErrorInvalidValue
    assert L.bfSolverSetGridPolicy(-1) == 1
    assert L.bfSolverSetGridPolicy(3) == 0                               # previous: auto
    assert L.bfSolverSetGridPolicy(0) == 3
    assert L.bfSolverGetLaunchInfo(C.byref(capi.BFSolverState()), (C.c_int * 4)()) == 1      # no solve on this state


def test_sift_match_sweep_switch_is_checked_on_the_host():
    """bfSiftSetMatchSweep / bfSiftGetMatchInfo are exported; an unknown sweep is refused without a device and leaves the setting as it was"""
    from bundlefusion_b200 import sift
    L = capi.lib()
    assert hasattr(L, "bfSiftSetMatchSweep") and hasattr(L, "bfSiftGetMatchInfo")
    assert (sift.SIFT_SWEEP_AUTO, sift.SIFT_SWEEP_WGMMA, sift.SIFT_SWEEP_MMA) == (0, 1, 2)
    prev = L.bfSiftSetMatchSweep(2)
    assert prev in (0, 2)                                                # auto, or mma when BF_SIFT_MATCH=mma
    assert L.bfSiftSetMatchSweep(3) == 1 and L.bfSiftSetMatchSweep(-1) == 1      # cudaErrorInvalidValue
    assert L.bfSiftSetMatchSweep(1) == 2
    assert L.bfSiftSetMatchSweep(prev) == 1
    out = (C.c_int * 2)()
    assert L.bfSiftGetMatchInfo(out) == 0 and out[0] in (0, 1, 2)


def test_raycast_pod_layouts():
    assert C.sizeof(capi.BFRayCastParams) == 192 and capi.BFRayCastParams.mx.offset == 128 and capi.BFRayCastParams.m_splatMinimum.offset == 160
    assert capi.BFRayCastParams.m_useGradients.offset == 184 and capi.BFRayCastParams.dummy0.offset == 188       # FL/DepthSensing/CUDARayCastParams.h:8-27
    assert C.sizeof(capi.BFRayCastData) == 56


def test_marchingcubes_pod_layouts():
    P = capi.BFMarchingCubesParams                                       # FL/DepthSensing/MarchingCubesSDFUtil.h:9-23
    assert C.sizeof(P) == 64 and P.m_minCorner.offset == 4 and P.m_maxNumTriangles.offset == 16 and P.m_maxCorner.offset == 20 and P.m_sdfBlockSize.offset == 32
    assert P.m_threshMarchingCubes.offset == 44 and P.m_threshMarchingCubes2.offset == 48
    assert C.sizeof(capi.BFMarchingCubesData) == 32


def test_marchingcubes_refuses_other_geometries_before_any_cuda_call():
    """argument checks run on the host: no GPU needed to see them"""
    L = capi.lib()
    L.bfMarchingCubesExtract.argtypes = [C.c_void_p] * 5
    hd, hp, p = capi.BFHashDataStruct(), capi.BFHashParams(), capi.BFMarchingCubesParams()
    hp.m_hashNumBuckets = 1009; hp.m_virtualVoxelSize = 0.01
    p.m_maxNumTriangles = 10; p.m_sdfBlockSize = 8; p.m_hashBucketSize = 4; p.m_hashNumBuckets = 1009
    buf = (C.c_float * 18)(); n = C.c_uint32(0)
    ok = lambda: L.bfMarchingCubesExtract(C.byref(hd), C.byref(hp), C.byref(p), buf, C.byref(n))
    assert L.bfMarchingCubesExtract(None, C.byref(hp), C.byref(p), buf, C.byref(n)) == 1                      # cudaErrorInvalidValue
    p.m_sdfBlockSize = 16
    assert ok() == 1
    p.m_sdfBlockSize = 8; p.m_hashBucketSize = 10
    assert ok() == 1
    p.m_hashBucketSize = 4; p.m_hashNumBuckets = 2003
    assert ok() == 1
    p.m_hashNumBuckets = 1009; hp.m_virtualVoxelSize = 0.0
    assert ok() == 1


def test_sift_pod_layouts():
    assert C.sizeof(capi.BFImagePairMatch) == 24                      # three device pointers, SIFTImageManager.h:38-42
    assert C.sizeof(capi.BFSiftMatchJob) == 64 and capi.BFSiftMatchJob.out.offset == 32 and capi.BFSiftMatchJob.keyPointOffset.offset == 56


def test_solver_pod_layouts():
    assert C.sizeof(capi.BFEntryJ) == 32
    assert C.sizeof(capi.BFSolverInput) == 128 and capi.BFSolverInput.intrinsics.offset == 64
    assert capi.BFSolverInput.d_validImages.offset == 40 and capi.BFSolverInput.weightsDenseColor.offset == 112
    assert C.sizeof(capi.BFSolverState) == 29 * 8
    assert C.sizeof(capi.BFSolverParameters) == 68 and capi.BFSolverParameters.denseOverlapCheckSubsampleFactor.offset == 48
    assert capi.BFSolverParameters.useDense.offset == 64
    assert C.sizeof(capi.BFCUDACachedFrame) == 48

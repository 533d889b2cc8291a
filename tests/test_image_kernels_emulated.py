"""The dense-cache, frame-ingest and trajectory kernels (csrc/cache.cu, csrc/ingest.cu, csrc/trajectory.cu) under the CPU emulation of
tests/cuda_emu, against the oracle, bit for bit.  These kernels are verified on the GPU (tests/test_cache_gpu.py, test_ingest_gpu.py,
test_trajectory_gpu.py); the emulated runs keep them covered when no GPU is at hand and qualify the emulation a second time."""
import ctypes as C

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from bundlefusion_b200 import synth
from oracle import oracle as orc
from tests.cuda_emu import build_emulated

F = np.float32


def bits(a):
    return np.ascontiguousarray(a, F).view(np.uint32)


@pytest.fixture(scope="module")
def libs():
    return build_emulated("cache.cu", 1), build_emulated("ingest.cu", 1), build_emulated("trajectory.cu", 4)


@pytest.mark.parametrize("frame,W,H", [(100, 160, 120), (40, 320, 240)])
def test_cache_store_frame_emulated(libs, frame, W, H):
    Lc = libs[0]
    depth, color, _ = synth.make_frame(frame, W, H)
    depth, color = np.ascontiguousarray(depth, F), np.ascontiguousarray(color, np.uint8)
    fx = 525.0 * W / 640.0
    K = np.array([[fx, 0, (W - 1) / 2.0, 0], [0, fx, (H - 1) / 2.0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    o = orc.cache_store_frame(depth, color, K, 80, 60, 2.5, 1.0, 0.05)
    Kinv = np.linalg.inv(K).astype(F)
    from bundlefusion_b200.cache import intrinsics_inverse
    P = capi.BFCacheParams(W, H, W, H, 80, 60, (C.c_float * 16)(*np.asarray(intrinsics_inverse(K), F).reshape(16).tolist()), 2.5, 1.0, 0.05)
    b = {"depth": np.zeros((60, 80), F), "campos": np.zeros((60, 80, 4), F), "intensity": np.zeros((60, 80), F), "derivs": np.zeros((60, 80, 2), F),
         "normalsU": np.zeros((60, 80, 4), np.uint8), "normals": np.zeros((60, 80, 4), F)}
    fr = capi.BFCUDACachedFrame(b["depth"].ctypes.data, b["campos"].ctypes.data, b["intensity"].ctypes.data, b["derivs"].ctypes.data, b["normalsU"].ctypes.data, b["normals"].ctypes.data)
    Lc.bfCacheStoreFrame.argtypes = [C.c_void_p] * 4
    assert Lc.bfCacheStoreFrame(C.addressof(P), depth.ctypes.data, color.ctypes.data, C.addressof(fr)) == 0
    for name, mine in (("depth", "depth"), ("campos", "campos"), ("normals", "normals"), ("intensity", "intensity"), ("derivs", "intensityDerivs")):
        assert np.array_equal(bits(b[name]).reshape(-1), bits(o[mine]).reshape(-1)), name
    assert np.array_equal(b["normalsU"].reshape(-1), np.asarray(o["normalsU"]).reshape(-1))


@pytest.mark.parametrize("wi,hi,erode,filt", [(160, 120, True, True), (80, 60, True, True), (160, 120, False, False), (80, 60, False, True)])
def test_ingest_frame_emulated(libs, wi, hi, erode, filt):
    Li = libs[1]
    depth, color, _ = synth.make_frame(250, 160, 120)
    depth, color = np.ascontiguousarray(depth, F), np.ascontiguousarray(color, np.uint8)
    d, c = orc.ingest_frame(depth, color, wi, hi, erode=erode, depth_filter=filt)
    p = orc.ingest_params(depth.shape, color.shape, wi, hi, erode=erode, depth_filter=filt)
    od, oc = np.full((hi, wi), 7.0, F), np.zeros((hi, wi, 4), np.uint8)
    Li.bfIngestFrame.argtypes = [C.c_void_p] * 5
    assert Li.bfIngestFrame(C.addressof(p), depth.ctypes.data, color.ctypes.data, od.ctypes.data, oc.ctypes.data) == 0
    assert np.array_equal(bits(od), bits(d)) and np.array_equal(oc, c)


def test_trajectory_kernels_emulated(libs):
    Lt = libs[2]
    from tests.test_manager_reference_emulated import trajectory_case
    tc = trajectory_case()
    vp, u = C.c_void_p, C.c_uint
    Lt.updateTrajectoryCU.argtypes = [vp, u, vp, u, vp, u, u, vp]; Lt.updateTrajectoryCU.restype = None
    Lt.initNextGlobalTransformCU.argtypes = [vp, u, u, vp, u, u]; Lt.initNextGlobalTransformCU.restype = None
    Lt.computeSiftTransformCU.argtypes = [vp, vp, vp, u, vp, u, u, vp]; Lt.computeSiftTransformCU.restype = None
    n = len(tc["inval"])
    comp = np.zeros((n, 4, 4), F); inval = tc["inval"].copy()
    Lt.updateTrajectoryCU(tc["glob"].ctypes.data, tc["G"], comp.ctypes.data, n, tc["loc"].ctypes.data, tc["per"], tc["G"], inval.ctypes.data)
    assert np.array_equal(bits(comp), bits(orc.update_trajectory(tc["glob"], tc["loc"], tc["per"], tc["inval"])))
    g2 = tc["glob"].copy()
    Lt.initNextGlobalTransformCU(g2.ctypes.data, 3, 2, tc["loc"].ctypes.data, 9, tc["per"])
    assert np.array_equal(bits(g2), bits(orc.init_next_global(tc["glob"], 3, 2, tc["loc"], 9, tc["per"])))
    for lv in tc["last_valids"]:
        sift = tc["sift"].copy(); cur = np.zeros((4, 4), F)
        Lt.computeSiftTransformCU(tc["finv"].ctypes.data, tc["nf"].ctypes.data, tc["comp"].ctypes.data, lv, sift.ctypes.data, tc["cur_all"], tc["cur"], cur.ctypes.data)
        t2, c2 = orc.compute_sift_transform(tc["finv"], tc["nf"], tc["comp"], lv, tc["sift"], tc["cur_all"], tc["cur"])
        # the integration transform goes through a 4x4 inverse: sub-determinant adjugate in the kernel (mat4.cuh), triple products in the oracle
        assert np.array_equal(bits(sift), bits(t2)) and np.abs(cur - c2).max() <= 2e-6 * max(1.0, float(np.abs(c2).max()))


def test_select_reintegration_emulated(libs):
    """bfTrajectorySelectReintegration (verified on the GPU before the scaled component of the pose distance was corrected to the translation
    part, FL/TrajectoryManager.cpp:67-74): the kernel against the oracle under the emulation."""
    Lt = libs[2]
    from tests.test_manager_reference_emulated import poses
    n = 300
    integ = poses(n, 7)
    rng = np.random.default_rng(8)
    opt = integ.copy()
    for k in rng.choice(n, 60, replace=False):
        opt[k] = (synth.se3_exp(rng.standard_normal(3) * 0.02, rng.standard_normal(3) * 0.05) @ integ[k].astype(np.float64)).astype(F)
    state = (rng.random(n) < 0.85).astype(np.int32)
    opt[[5, 50, 200], 0, 0] = -np.inf
    Lt.bfTrajectorySelectReintegration.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    for topN, minDist in ((10, 0.0004), (30, 0.0), (5, 0.01)):
        od, ol = orc.select_reintegration(opt, integ, state, topN, minDist)
        dist = np.zeros(n, F); lst = np.full(topN, -1, np.int32); cnt = np.zeros(1, np.int32)
        assert Lt.bfTrajectorySelectReintegration(opt.ctypes.data, integ.ctypes.data, state.ctypes.data, n, topN, minDist, 2.0, dist.ctypes.data, lst.ctypes.data, cnt.ctypes.data) == 0
        assert cnt[0] == len(ol) and np.array_equal(lst[:cnt[0]], ol)
        assert np.array_equal(bits(dist), bits(od))

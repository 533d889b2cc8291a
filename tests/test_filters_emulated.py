"""The match-filter kernels (csrc/sift_filter.cu, csrc/sift_verify.cu) under the CPU emulation of tests/cuda_emu, against the oracle.
These kernels ARE verified on the GPU (tests/test_filter_gpu.py, tests/test_verify_filters_gpu.py: bit-identical to the oracle); running
the same sources through the emulation and getting the same bits is what qualifies the emulation as a checker for the kernels that
have not been on hardware yet (tests/test_sift_detect_emulated.py, tests/test_sift_prune_emulated.py)."""
import ctypes as C

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from bundlefusion_b200 import synth
from oracle import oracle as orc
from tests.cuda_emu import build_emulated
from tests.test_verify_filters_oracle import VERIFY


def f16(m):
    return np.ascontiguousarray(m, np.float32).reshape(16).ctypes.data_as(C.POINTER(C.c_float))


def same(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a.view(np.uint32)[~na], b.view(np.uint32)[~nb])


@pytest.fixture(scope="module")
def verify_emu():
    L = build_emulated("sift_verify.cu", 5)
    vp, u, f = C.c_void_p, C.c_uint, C.c_float
    L.bfSiftVerifyTrajectory.argtypes = [u, vp, vp, u, u, C.POINTER(f), vp] + [f] * 7 + [vp, vp]
    L.bfSiftFilterMatchesBySurfaceArea.argtypes = [u, u, u, vp, vp, vp, C.POINTER(f), f, vp]
    L.bfSiftFilterMatchesByDenseVerify.argtypes = [u] * 5 + [C.POINTER(f), vp, vp, vp] + [f] * 7 + [vp]
    return L


@pytest.fixture(scope="module")
def filter_emu():
    L = build_emulated("sift_filter.cu", 3)
    vp, u, f = C.c_void_p, C.c_uint, C.c_float
    L.bfSiftFilterKeyPointMatches.argtypes = [u, u, u] + [vp] * 9 + [C.POINTER(f), u, f]
    L.bfSiftAddCurrToResiduals.argtypes = [u, u, u] + [vp] * 6 + [C.POINTER(f)]
    return L


def test_surface_area_emulated(verify_emu):
    pb = synth.make_area_problem(2)
    for start, thresh in ((0, 0.032), (2, 1e9)):
        nf_o, ar_o = orc.sift_filter_surface_area(pb["cur"], start, pb["P"], pb["keys"], pb["num"], pb["fidx"], pb["Kinv"], thresh)
        num = pb["num"].copy(); areas = np.full((pb["P"], 2), -1.0, np.float32)
        keys = np.ascontiguousarray(pb["keys"], np.float32); fidx = np.ascontiguousarray(pb["fidx"], np.uint32)
        assert verify_emu.bfSiftFilterMatchesBySurfaceArea(pb["cur"], start, pb["P"], keys.ctypes.data, num.ctypes.data, fidx.ctypes.data, f16(pb["Kinv"]), thresh, areas.ctypes.data) == 0
        assert np.array_equal(num, nf_o) and same(areas, ar_o)


def test_dense_verify_emulated(verify_emu):
    pb = synth.make_dense_verify_problem(n_prev=3)
    P, cur = pb["P"], pb["cur"]
    num = np.array([5, 5, 0, 5], np.int32)
    nf_o, st_o = orc.sift_filter_dense_verify(cur, 0, P, pb["W"], pb["H"], pb["K"], num, pb["T"], pb["caches"], **VERIFY)
    keep = [{k: np.ascontiguousarray(f[k], np.float32) for k in ("depth", "campos", "normals")} for f in pb["caches"]]
    recs = (capi.BFCUDACachedFrame * P)()
    for r, f in zip(recs, keep):
        r.d_depthDownsampled, r.d_cameraposDownsampled, r.d_normalsDownsampled = f["depth"].ctypes.data, f["campos"].ctypes.data, f["normals"].ctypes.data
    n = num.copy(); T = np.ascontiguousarray(pb["T"], np.float32); stats = np.full((P, 2), -1.0, np.float32)
    o = VERIFY
    assert verify_emu.bfSiftFilterMatchesByDenseVerify(cur, 0, P, pb["W"], pb["H"], f16(pb["K"]), n.ctypes.data, T.ctypes.data, C.addressof(recs), o["distThresh"], o["normalThresh"],
                                                       o["colorThresh"], o["errThresh"], o["corrThresh"], o["dMin"], o["dMax"], stats.ctypes.data) == 0
    assert np.array_equal(n, nf_o) and same(stats, st_o)


def test_kabsch_filter_and_residuals_emulated(filter_emu):
    pb = synth.make_filter_problem(n_pairs=4, n_inliers=30, n_outliers=10, noise=0.002, seed=5)
    P, cur = pb["P"], pb["cur"]
    o = orc.sift_filter_matches(cur, 0, P, pb["keys"], pb["num"], pb["dists"], pb["idxs"], pb["Kinv"])
    keys = np.ascontiguousarray(pb["keys"], np.float32); num = np.ascontiguousarray(pb["num"], np.int32)
    d = np.ascontiguousarray(pb["dists"], np.float32); ix = np.ascontiguousarray(pb["idxs"], np.uint32)
    nf = np.full(P, -7, np.int32); fd = np.zeros((P, 25), np.float32); fi = np.zeros((P, 25, 2), np.uint32); T = np.zeros((P, 16), np.float32); Ti = np.zeros((P, 16), np.float32)
    assert filter_emu.bfSiftFilterKeyPointMatches(cur, 0, P, keys.ctypes.data, num.ctypes.data, d.ctypes.data, ix.ctypes.data, nf.ctypes.data, fd.ctypes.data, fi.ctypes.data,
                                                  T.ctypes.data, Ti.ctypes.data, f16(pb["Kinv"]), 5, 0.0004) == 0
    for p in range(P - 1):
        assert nf[p] == o[0][p] and np.array_equal(fi[p], o[2][p]) and np.array_equal(fd[p], o[1][p])
        assert np.array_equal(T[p].reshape(4, 4), o[3][p])                   # the same operations in the same order: identical bits
    ent_o, idx_o = orc.sift_add_residuals(cur, 0, P, o[0], o[2], pb["keys"], pb["Kinv"])
    cap = len(ent_o) + 4
    ent = np.zeros(32 * cap, np.uint8); eidx = np.zeros((cap, 2), np.uint32); cnt = np.zeros(1, np.int32)
    nfc = np.where(np.arange(P) == cur, 0, nf).astype(np.int32)
    assert filter_emu.bfSiftAddCurrToResiduals(cur, 0, P, ent.ctypes.data, eidx.ctypes.data, cnt.ctypes.data, nfc.ctypes.data, fi.ctypes.data, keys.ctypes.data, f16(pb["Kinv"])) == 0
    assert cnt[0] == len(ent_o) and ent[:32 * len(ent_o)].tobytes() == ent_o.tobytes() and np.array_equal(eidx[:len(ent_o)], idx_o)


@pytest.mark.parametrize("break_pair", [False, True])
def test_verify_trajectory_emulated(verify_emu, break_pair):
    """bfSiftVerifyTrajectory (VerifyTrajectoryCU) under the emulation against the oracle; on a consistent trajectory whose last pose is the
    identity, the pair (p, last) sees exactly what the dense-verification filter sees for pair p."""
    from tests.test_verify_filters_gpu import trajectory_verify_case
    pb, N, valid, traj = trajectory_verify_case(3, break_pair, None)
    opt = dict(VERIFY, errThresh=0.05, corrThresh=0.001, dMin=0.1, dMax=3.0)
    ok_o, st_o = orc.sift_verify_trajectory(N, valid, traj, pb["W"], pb["H"], pb["K"], pb["caches"], **opt)
    keep = [{k: np.ascontiguousarray(f[k], np.float32) for k in ("depth", "campos", "normals")} for f in pb["caches"]]
    recs = (capi.BFCUDACachedFrame * N)()
    for r, f in zip(recs, keep):
        r.d_depthDownsampled, r.d_cameraposDownsampled, r.d_normalsDownsampled = f["depth"].ctypes.data, f["campos"].ctypes.data, f["normals"].ctypes.data
    ok = np.full(1, 9, np.int32); stats = np.full((N * (N - 1) // 2, 2), -1.0, np.float32); T = np.ascontiguousarray(traj, np.float32)
    assert verify_emu.bfSiftVerifyTrajectory(N, valid.ctypes.data, T.ctypes.data, pb["W"], pb["H"], f16(pb["K"]), C.addressof(recs), opt["distThresh"], opt["normalThresh"],
                                             opt["colorThresh"], opt["errThresh"], opt["corrThresh"], opt["dMin"], opt["dMax"], ok.ctypes.data, stats.ctypes.data) == 0
    assert ok[0] == ok_o == (0 if break_pair else 1) and same(stats, st_o)
    # pair (0, N - 1) = block N - 1: the filter's view of pair 0 with the transform trajectory[0]
    num = np.full(N, 5, np.int32)
    _, st_f = orc.sift_filter_dense_verify(N - 1, 0, N, pb["W"], pb["H"], pb["K"], num, traj, pb["caches"], **opt)
    assert same(st_o[N - 1], st_f[0])


@pytest.mark.parametrize("seed,numFrames", [(0, 1), (1, 7), (2, 300), (3, 1000)])
def test_filter_frames_and_conditional_residuals_emulated(filter_emu, seed, numFrames):
    """bfSiftFilterFrames (not yet on hardware) against the oracle, and the device-side condition on the residual assembly."""
    filter_emu.bfSiftFilterFrames.argtypes = [C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p]
    filter_emu.bfSiftAddCurrToResidualsIfMatched.argtypes = [C.c_uint, C.c_uint, C.c_uint] + [C.c_void_p] * 6 + [C.POINTER(C.c_float), C.c_void_p]
    rng = np.random.default_rng(seed)
    for trial in range(4):
        cur = int(rng.integers(0, numFrames)); start = int(rng.integers(0, cur + 1)) if trial % 2 else 0
        nf = (rng.integers(0, 12, numFrames) * (rng.random(numFrames) < (0.02 if trial == 3 else 0.4))).astype(np.int32)
        valid = (rng.random(numFrames) < 0.8).astype(np.int32)
        if trial == 2:
            nf[:] = 0                                   # nothing matched: the current frame becomes invalid
        want_last, want_valid = orc.sift_filter_frames(cur, start, numFrames, nf, valid)
        got_valid = valid.copy(); last = np.full(1, 12345, np.int32)
        assert filter_emu.bfSiftFilterFrames(cur, start, numFrames, nf.ctypes.data, got_valid.ctypes.data, last.ctypes.data) == 0
        assert last[0] == want_last and np.array_equal(got_valid, want_valid)
        assert got_valid[cur] == (1 if want_last >= 0 else 0)
    # the condition on the residual assembly
    pb = synth.make_filter_problem(n_pairs=3, n_inliers=20, n_outliers=5, noise=0.002, seed=9)
    P, cur = pb["P"], pb["cur"]
    o = orc.sift_filter_matches(cur, 0, P, pb["keys"], pb["num"], pb["dists"], pb["idxs"], pb["Kinv"])
    ent_o, idx_o = orc.sift_add_residuals(cur, 0, P, o[0], o[2], pb["keys"], pb["Kinv"])
    keys = np.ascontiguousarray(pb["keys"], np.float32); nfc = np.where(np.arange(P) == cur, 0, o[0]).astype(np.int32); fi = np.ascontiguousarray(o[2], np.uint32)
    for lastMatched, expect in ((-1, 0), (0, len(ent_o)), (2, len(ent_o))):
        cap = len(ent_o) + 4
        ent = np.zeros(32 * cap, np.uint8); eidx = np.zeros((cap, 2), np.uint32); cnt = np.zeros(1, np.int32); lm = np.array([lastMatched], np.int32)
        assert filter_emu.bfSiftAddCurrToResidualsIfMatched(cur, 0, P, ent.ctypes.data, eidx.ctypes.data, cnt.ctypes.data, nfc.ctypes.data, fi.ctypes.data, keys.ctypes.data,
                                                            f16(pb["Kinv"]), lm.ctypes.data) == 0
        assert cnt[0] == expect and ent[:32 * expect].tobytes() == ent_o[:expect].tobytes() and not ent[32 * expect:].any()


def _filter_emulated_equals_oracle(filter_emu, pb):
    P, cur = pb["P"], pb["cur"]
    o = orc.sift_filter_matches(cur, 0, P, pb["keys"], pb["num"], pb["dists"], pb["idxs"], pb["Kinv"])
    keys = np.ascontiguousarray(pb["keys"], np.float32); num = np.ascontiguousarray(pb["num"], np.int32)
    d = np.ascontiguousarray(pb["dists"], np.float32); ix = np.ascontiguousarray(pb["idxs"], np.uint32)
    nf = np.full(P, -7, np.int32); fd = np.zeros((P, 25), np.float32); fi = np.zeros((P, 25, 2), np.uint32); T = np.zeros((P, 16), np.float32); Ti = np.zeros((P, 16), np.float32)
    assert filter_emu.bfSiftFilterKeyPointMatches(cur, 0, P, keys.ctypes.data, num.ctypes.data, d.ctypes.data, ix.ctypes.data, nf.ctypes.data, fd.ctypes.data, fi.ctypes.data,
                                                  T.ctypes.data, Ti.ctypes.data, f16(pb["Kinv"]), 5, 0.0004) == 0
    for p in range(P - 1):
        assert nf[p] == o[0][p] and np.array_equal(fi[p], o[2][p]) and np.array_equal(fd[p], o[1][p]) and same(T[p].reshape(4, 4), o[3][p]), p
    return [int(x) for x in nf[:P - 1]]


@pytest.mark.parametrize("case", ["outliers", "invalid-depth", "quantised", "zero-residuals"])
def test_kabsch_filter_warp_cooperative_paths_emulated(filter_emu, case):
    """The Kabsch filter spreads the sums of a fit over the lanes of the pair's warp (csrc/sift_filter.cu).  Cases that steer it through every branch:
    many outliers (removal loop, rejected pairs), invalid depths (NaN residuals: the reference's exchange sort is replayed), exact geometry on a coarse
    grid and identical frames (equal / zero residuals: replay as well) -- each bit-identical to the serial oracle."""
    if case == "outliers":
        pb = synth.make_filter_problem(n_pairs=5, n_inliers=25, n_outliers=40, noise=0.006, seed=21)
    elif case == "invalid-depth":
        pb = synth.make_filter_problem(n_pairs=4, n_inliers=40, n_outliers=10, noise=0.002, seed=31)
        bad = np.random.default_rng(31).random(len(pb["keys"])) < 0.08
        pb["keys"][bad, 3] = -np.inf
    else:
        pb = synth.make_filter_problem(n_pairs=4, n_inliers=30, n_outliers=6, noise=0.0, seed=41 if case == "quantised" else 43)
        k = pb["keys"]; k[:, 0] = np.round(k[:, 0]); k[:, 1] = np.round(k[:, 1]); k[:, 3] = np.round(k[:, 3] * 4) / 4
        if case == "zero-residuals":
            n = pb["n"]
            for p in range(pb["P"] - 1):
                k[p * n:(p + 1) * n] = k[pb["cur"] * n:(pb["cur"] + 1) * n]
    counts = _filter_emulated_equals_oracle(filter_emu, pb)
    if case == "zero-residuals":
        assert all(c == 25 for c in counts)
    if case == "invalid-depth":
        assert all(c == 0 for c in counts)

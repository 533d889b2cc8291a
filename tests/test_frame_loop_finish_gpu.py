"""bfFrameLoopFinish (FrameLoop.finish, scan.reconstruct(..., solve_frames_before_exit=K)): the end of a recording as the reference runs it --
sparse global solves on past-end turns 0 .. K - 1, the dense global solve (weights 1 / 15 / 0, 3 Gauss-Newton iterations, keyframe cache) on turn K,
then re-integration only until the TrajectoryManager has no operation left.  On the synthetic stream of test_frame_loop_gpu.py: 43 frames (5 keyframes:
the one-CTA Gauss-Newton policy) and 200 frames (about 20 keyframes: the resident-cluster policy).

What is checked: the turns before K are bit for bit bfFrameLoopStepPastEnd's; the end solve is bfSolverSolve on the loop's own keyframe problem with the
reference's end weights, bit for bit; the finished model is the fusion of the returned trajectory: a fresh hash fed every frame at its final pose holds
the same voxels with the same weights and sdf but for a small, measured fraction that allocation history explains (assert_model_is_fusion_of
states it).  Colour is not compared: the reference's colour de-integration is not an inverse."""
import ctypes as C
import math

import numpy as np
import pytest

from bundlefusion_b200 import synth
from bundlefusion_b200.frame_loop import FrameLoop, default_params

pytestmark = pytest.mark.gpu
W, H = 320, 240
K_TEST = 3
SDF_TOL = 1e-3                    # metres; a tenth of a voxel


def rel_pose(T0, T):
    return np.linalg.inv(T0.astype(np.float64)) @ T.astype(np.float64)


_STREAMS = {}


def stream(n, dev):
    """n raw frames (device tensors) and their true poses: synth.make_frame every second pose of the Lissajous path (the frame-loop test's stream)"""
    import torch
    if n not in _STREAMS:
        fr = [synth.make_frame(2 * i, W, H, texture="rich") for i in range(n)]
        _STREAMS[n] = ([(torch.from_numpy(d).to(dev), torch.from_numpy(c).to(dev)) for d, c, _ in fr], [T for _, _, T in fr])
    return _STREAMS[n]


def make_loop(n, dev, steps=None):
    """a loop that has stepped the first `steps` (default all n) frames of the n-frame stream"""
    p = default_params(W, H)
    p.maxNumImages = max(16, n // 10 + 8); p.maxNumFrames = n + 16
    p.hash.m_hashNumBuckets = 100003 if n <= 64 else 200003
    p.hash.m_numSDFBlocks = 90000 if n <= 64 else 200000
    loop = FrameLoop(p, dev)
    frames, _ = stream(n, dev)
    for d, c in frames[:n if steps is None else steps]:
        loop.step(d, c)
    return loop


def state(loop, n):
    c = loop.counters()
    c.pop("host_syncs")
    return c, loop.trajectory(n), loop.heap_free()


def assert_same_state(a, b, what):
    (ca, ta, fa), (cb, tb, fb) = a, b
    assert ca == cb, (what, ca, cb)
    assert np.array_equal(ta, tb, equal_nan=True), what
    assert fa == fb, (what, fa, fb)


def device_bytes(ptr, nbytes, dev):
    """a uint8 torch view of device memory the library owns (no copy)"""
    import torch

    class _View:
        pass
    v = _View()
    v.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False), "version": 3, "strides": None}
    return torch.as_tensor(v, device=dev)


def voxels(hash_ptr, sdf_ptr, hp, dev):
    """every voxel with weight > 0: keys (block x, y, z, voxel index) sorted, their sdf and weight"""
    import torch
    torch.cuda.synchronize(dev)
    n_entries = int(hp.m_hashNumBuckets) * 4
    h = device_bytes(hash_ptr, n_entries * 32, dev).view(torch.int32).view(n_entries, 8)
    ent = h[h[:, 3] != -2]
    blocks = device_bytes(sdf_ptr, int(hp.m_numSDFBlocks) * 512 * 12, dev).view(torch.int32).view(-1, 512, 3)
    vox = blocks[(ent[:, 3] // 512).long()].cpu().numpy()
    ent = ent.cpu().numpy()
    sdf, w = vox[..., 0].view(np.float32), vox[..., 1].view(np.float32)
    bi, vi = np.nonzero(w > 0)
    keys = np.stack([ent[bi, 0], ent[bi, 1], ent[bi, 2], vi], 1).astype(np.int64)
    order = np.lexsort(keys.T[::-1])
    return keys[order], sdf[bi, vi][order], w[bi, vi][order]


def loop_voxels(loop, dev):
    hd = loop.lib.bfFrameLoopGetHashData(loop._h).contents
    return voxels(hd.d_hash, hd.d_SDFBlocks, loop.lib.bfFrameLoopGetHashParams(loop._h).contents, dev)


def fused_voxels(hash_params, raw_frames, trajectory, dev):
    """a fresh hash with the loop's parameters, every frame with a finite pose integrated at that pose from the library's ingest of its raw frame"""
    from bundlefusion_b200 import _capi as capi
    from bundlefusion_b200.image_manager import CUDAImageManager
    from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF, camera_params
    hp = capi.BFHashParams()
    C.memmove(C.byref(hp), C.byref(hash_params), C.sizeof(capi.BFHashParams))
    im = CUDAImageManager(W, H, dev)
    ingested = [im.process(d, c) for d, c in raw_frames]
    ops = [(capi.BF_TSDF_OP_INTEGRATE, f, trajectory[f]) for f in range(len(trajectory)) if np.isfinite(trajectory[f]).all()]
    scene = CUDASceneRepHashSDF(hp, dev, arithmetic="fast")
    scene.runOps(ops, [d for d, _ in ingested], [c for _, c in ingested], camera_params(W, H))
    out = voxels(scene.d_hash.data_ptr(), scene.d_SDFBlocks.data_ptr(), hp, dev)
    scene.close()
    return out, len(ops)


def assert_model_is_fusion_of(got, want, what):
    """the loop's model against the fresh fusion of its trajectory.  It is not that fusion bit for bit, and the cause is allocation history:
    the model is the exact replay of the TSDF ops the loop ran (tests/test_frame_loop_model_gpu.py, bit for bit), no contribution is stranded
    on these streams, and integration fills every allocated block in the frustum -- so a frame adds weight to blocks that earlier poses,
    or later frames, allocated in one model and not (yet) in the other.  The fresh fusion itself moves by the same kind of amount when every
    block is allocated before the first integration that counts (200 frames: 131 voxels in one model only, 8703 with another weight).
    Measured on an H100, as fractions of the voxels with weight > 0: in one model only 1e-5 (43 frames), 1.0e-4 (200 frames), 5e-6 (14-frame
    scan); another weight 7e-5, 2.5e-3, 5e-5; where the weights agree the sdf agrees to 8e-4 m at 43 frames and in the scan, while 1.7e-4 of
    the 200-frame model's voxels differ by more than 1e-3 m (none against the fusion with every block allocated first).  The bounds are
    those figures with a factor 2 of headroom."""
    (kg, sg, wg), (kw, sw, ww) = got, want
    assert len(kg) > 10000, (what, len(kg))
    pack = lambda k: (((k[:, 0] + 32768) * 65536 + (k[:, 1] + 32768)) * 65536 + (k[:, 2] + 32768)) * 512 + k[:, 3]
    common, ig, iw = np.intersect1d(pack(kg), pack(kw), assume_unique=True, return_indices=True)
    one_side = len(kg) + len(kw) - 2 * len(common)
    same_w = wg[ig] == ww[iw]
    dsdf = np.abs(sg[ig][same_w] - sw[iw][same_w])
    far = int((dsdf > SDF_TOL).sum())
    print("%s: %d / %d voxels with weight > 0 (loop / fusion of the trajectory), %d in one model only, %d with another weight, max |delta sdf| %.3g m "
          "where the weights agree (%d above %g m)" % (what, len(kg), len(kw), one_side, int((~same_w).sum()), float(dsdf.max()), far, SDF_TOL))
    assert one_side <= 2.5e-4 * len(kw), (what, one_side)
    assert (~same_w).sum() <= 5e-3 * len(kw), (what, int((~same_w).sum()))
    assert far <= 4e-4 * len(kw), (what, far)


class LoopCache:
    """the loop's keyframe cache as solver.CUDASolverBundling takes a CUDACache"""

    def __init__(self, prob, dev):
        self.width, self.height = prob.cacheWidth, prob.cacheHeight
        self.intrinsics = tuple(float(x) for x in prob.intrinsics)
        self._frames = device_bytes(prob.d_cacheFrames, 48 * prob.numKeyframes, dev)

    def getCacheFramesGPU(self):
        return self._frames


def solve_end_problem(loop, dev):
    """the loop's keyframe problem (copied), solved as the reference's end solve: weights (1, 15, 0), 3 GN x numGlobalLinIterations, pairwise dense"""
    import torch
    from bundlefusion_b200.solver import CUDASolverBundling
    prob = loop.global_problem()
    N = prob.numKeyframes
    copy = lambda ptr, nbytes: device_bytes(ptr, nbytes, dev).clone()
    corr = copy(prob.d_correspondences, 32 * max(1, prob.numCorrespondences))
    valid = copy(prob.d_validImages, 4 * N).view(torch.int32)
    traj = copy(prob.d_trajectory, 64 * N).view(torch.float32)
    sol = CUDASolverBundling(prob.maxNumImages, prob.maxCorrPerImage * prob.maxNumImages, dev)
    assert sol.m_maxCorrPerImage == prob.maxCorrPerImage
    rot = torch.zeros(3 * N, dtype=torch.float32, device=dev); trans = torch.zeros_like(rot)
    cache = LoopCache(prob, dev)
    loop._bind_stream()
    sol.lib.convertMatricesToPosesCU(traj.data_ptr(), N, rot.data_ptr(), trans.data_ptr(), valid.data_ptr())
    sol.solve(corr, prob.numCorrespondences, valid, N, 3, int(loop.params.numGlobalLinIterations), [1.0] * 3, [15.0] * 3, [0.0] * 3, rot, trans, cudaCache=cache)
    sol.lib.convertPosesToMatricesCU(rot.data_ptr(), trans.data_ptr(), N, traj.data_ptr(), valid.data_ptr())
    out = traj.view(N, 4, 4).cpu().numpy()
    stats, launch = sol.getStats(), sol.getLaunchInfo()
    sol.close()
    return N, out, stats, launch


def loop_keyframe_poses(loop, dev):
    import torch
    prob = loop.global_problem()
    torch.cuda.synchronize(dev)
    return device_bytes(prob.d_trajectory, 64 * prob.numKeyframes, dev).view(torch.float32).view(-1, 4, 4).cpu().numpy()


def turn_bound(K, n_frames, max_frame_fixes=10):
    return K + 2 + math.ceil(n_frames / max_frame_fixes)


def test_finish_equals_past_end_turns_before_K_then_solves_densely_once_and_drains(cuda_device):
    n, K = 43, K_TEST
    _, truth = stream(n, cuda_device)
    A, B = make_loop(n, cuda_device), make_loop(n, cuda_device)
    assert_same_state(state(A, n), state(B, n), "after the last frame")
    for t in range(K):
        info = A.finish(K, max_turns=1)
        st = B.step_past_end().as_dict()
        assert info["turns"] == 1 and info["frames_past_end"] == t + 1 and not info["done"] and info["dense_turn"] == -1, (t, info)
        assert info["global_solves"] == st["globalSolved"] and info["reintegrations"] == st["numReintegrated"], (t, info, st)
        assert_same_state(state(A, n), state(B, n), "past-end turn %d" % t)
    c0 = A.counters()
    info = A.finish(K, max_turns=1)                                       # turn K: the dense end solve
    assert info["dense_turn"] == K and info["dense_keyframes"] == 5 and info["dense_pairs"] > 0 and info["global_solves"] == 1, info
    assert A.counters()["global_solves"] == c0["global_solves"] + 1 and A.counters()["local_solves"] == c0["local_solves"]
    c1 = A.counters()
    info = A.finish(K)
    assert info["done"] and info["global_solves"] == 0, info
    assert A.counters()["global_solves"] == c1["global_solves"] and A.counters()["local_solves"] == c1["local_solves"]
    assert info["frames_past_end"] <= turn_bound(K, n), info
    assert info["valid"] and info["transforms"] == n and info["valid_transforms"] >= n - 2, info
    traj = A.trajectory(n)
    err = [np.abs(traj[f] - rel_pose(truth[0], truth[f]))[:3, 3].max() for f in range(len(traj)) if np.isfinite(traj[f]).all()]
    assert len(err) >= 38 and max(err) < 0.05, (len(err), max(err))
    print("finish(%d) on %d frames: %s; max translation error %.4f m" % (K, n, info, max(err)))
    A.close(); B.close()


@pytest.mark.parametrize("n, policy", [(43, 2), (200, 3)])
def test_end_solve_is_the_dense_global_solve_and_the_model_is_the_fusion_of_the_trajectory(cuda_device, n, policy):
    """the keyframe problem after turn K - 1 solved through solver.py with the end weights gives the loop's keyframe poses after turn K bit for bit
    (policy: the Gauss-Newton launch policy that size takes, 2 = one CTA, 3 = resident cluster); after the drain the model is the fusion of the trajectory"""
    from bundlefusion_b200 import _capi as capi
    K = K_TEST
    prev_arith = capi.lib().bfTsdfSetArithmetic(1)                       # the default tolerance arithmetic, for the loop and the fresh hash alike
    try:
        loop = make_loop(n, cuda_device)
        info = loop.finish(K, max_turns=K)
        assert info["frames_past_end"] == K and info["dense_turn"] == -1 and not info["done"], info
        N, want, stats, launch = solve_end_problem(loop, cuda_device)
        info = loop.finish(K, max_turns=1)
        assert info["dense_turn"] == K and info["dense_keyframes"] == N and info["dense_pairs"] == stats["dense_weighted_pairs"] > 0, (info, stats)
        assert stats["error"] == 0 and launch["policy"] == policy, (stats, launch)
        got = loop_keyframe_poses(loop, cuda_device)
        assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.abs(got - want).max()
        if n >= 200:
            assert N >= 15, N
        info = loop.finish(K)
        assert info["done"] and info["frames_past_end"] <= turn_bound(K, n) and info["valid"], info
        traj = loop.trajectory(n)
        assert len(traj) == n
        frames, _ = stream(n, cuda_device)
        want_model, n_fused = fused_voxels(loop.lib.bfFrameLoopGetHashParams(loop._h).contents, frames, traj, cuda_device)
        assert n_fused == info["valid_transforms"] and n_fused >= n - 4, (n_fused, info)
        assert_model_is_fusion_of(loop_voxels(loop, cuda_device), want_model, "%d frames" % n)
        loop.close()
    finally:
        capi.lib().bfTsdfSetArithmetic(prev_arith)


def test_finish_edge_cases(cuda_device):
    import torch
    n, K = 23, K_TEST
    # reference: one call
    ref = make_loop(n, cuda_device)
    r = ref.finish(K)
    assert r["done"] and r["dense_turn"] == K and r["dense_keyframes"] == 3, r
    ref_state = state(ref, n)
    again = ref.finish(K)                                                  # done: a further call runs nothing
    assert again["done"] and again["turns"] == 0 and again["global_solves"] == 0 and again["reintegrations"] == 0, again
    assert_same_state(state(ref, n), ref_state, "after a call on a finished loop")
    ref.close()
    # turns run by bfFrameLoopStepPastEnd count: 2 of them, then finish
    a = make_loop(n, cuda_device)
    a.step_past_end(); a.step_past_end()
    i = a.finish(K)
    assert i["done"] and i["dense_turn"] == K and i["turns"] == r["frames_past_end"] - 2 and i["frames_past_end"] == r["frames_past_end"], (i, r)
    assert_same_state(state(a, n), ref_state, "finish after 2 step_past_end turns")
    # max_turns too small: not ready, a second call finishes with the one-call result; a continuation must keep K
    a.close()
    a = make_loop(n, cuda_device)
    i = a.finish(K, max_turns=2)
    assert not i["done"] and i["turns"] == 2 and i["dense_turn"] == -1, i
    with pytest.raises(RuntimeError, match="error 1:"):
        a.finish(K + 1)
    i = a.finish(K)
    assert i["done"] and i["turns"] == r["frames_past_end"] - 2 and i["dense_turn"] == K, i
    assert_same_state(state(a, n), ref_state, "finish in two calls")
    a.close()
    # more than K turns already: refused, nothing changes
    a = make_loop(n, cuda_device)
    for _ in range(K + 1):
        a.step_past_end()
    before = state(a, n)
    with pytest.raises(RuntimeError, match="error 1:"):
        a.finish(K)
    assert_same_state(state(a, n), before, "refused finish")
    assert a.finish(K + 1)["done"]                                       # the dense turn is still ahead for a larger K
    a.close()
    # K = 0: the dense solve on the turn that solves the last, partial chunk
    a = make_loop(n, cuda_device)
    i = a.finish(0)
    assert i["done"] and i["dense_turn"] == 0 and i["dense_keyframes"] == 3 and i["dense_pairs"] > 0 and i["frames_past_end"] <= turn_bound(0, n), i
    a.close()
    # a pending look-ahead frame: refused
    frames, _ = stream(n, cuda_device)
    a = make_loop(n, cuda_device, steps=n - 2)
    a.step(frames[n - 2][0], frames[n - 2][1], frames[n - 1][0], frames[n - 1][1])
    with pytest.raises(RuntimeError, match="error 1:"):
        a.finish(K)
    a.step(frames[n - 1][0], frames[n - 1][1])
    assert a.finish(K)["done"]
    a.close()
    # no frame stepped: refused
    a = make_loop(n, cuda_device, steps=0)
    with pytest.raises(RuntimeError, match="error 1:"):
        a.finish(K)
    a.close()
    # one keyframe: finishes without a dense solve (nor any global solve)
    a = make_loop(8, cuda_device)
    i = a.finish(K)
    assert i["done"] and i["dense_turn"] == -1 and i["global_solves"] == 0 and a.counters()["keyframes"] == 1 and i["valid"], i
    a.close()
    torch.cuda.synchronize()


def test_scan_finish_writes_the_fusion_of_its_trajectory(cuda_device, tmp_path, monkeypatch):
    """scan.reconstruct(..., solve_frames_before_exit=3): valid verdict, a mesh on the recorded surfaces, and the model the mesh was extracted from is the
    fusion of the trajectory the call returns"""
    import torch
    from bundlefusion_b200 import _capi as capi
    from bundlefusion_b200 import frame_loop, scan, sens
    n = 14
    Kint = np.array(list(default_params(W, H).depthIntrinsics), np.float32).reshape(4, 4)
    path = str(tmp_path / "seq.sens")
    w = sens.SensorDataWriter(path, W, H, Kint, depth_shift=1000.0, zlib_depth=True)
    truth, depths = [], []
    for i in range(n):
        d, c, T = synth.make_frame(2 * i, W, H, texture="rich")
        w.append(np.where(np.isfinite(d), np.clip(np.round(d * 1000.0), 1, 65535), 0).astype(np.uint16), c[..., :3], T)
        truth.append(T); depths.append(d)
    w.finish()
    snap = {}

    class SnapshotLoop(frame_loop.FrameLoop):                              # the model as the loop leaves it, read just before the loop is closed
        def close(self):
            if getattr(self, "_h", None) and "voxels" not in snap:
                snap["voxels"] = loop_voxels(self, cuda_device)
                hp = capi.BFHashParams()
                C.memmove(C.byref(hp), C.byref(self.lib.bfFrameLoopGetHashParams(self._h).contents), C.sizeof(capi.BFHashParams))
                snap["hp"] = hp
            super().close()
    monkeypatch.setattr(scan, "FrameLoop", SnapshotLoop)
    prev_arith = capi.lib().bfTsdfSetArithmetic(1)
    try:
        ply = str(tmp_path / "out" / "scan.ply")
        o = scan.reconstruct(path, ply, cuda_device, hash_buckets=100003, sdf_blocks=90000, max_num_triangles=2_000_000, solve_frames_before_exit=3)
        f = o["finish"]
        assert f["valid"] and f["done"] and f["dense_turn"] == 3 and f["frames_past_end"] <= turn_bound(3, n), f
        assert o["frames"] == n and o["mesh_path"] == ply and o["triangles"] > 20000
        traj = o["trajectory"]
        T0inv = np.linalg.inv(truth[0].astype(np.float64))
        err = [np.abs((T0inv @ truth[i].astype(np.float64))[:3, 3] - traj[i][:3, 3].astype(np.float64)).max() for i in range(len(traj)) if np.isfinite(traj[i]).all()]
        assert len(err) >= n - 4 and max(err) < 0.05
        # the mesh: its vertices lie on the depth some recorded frame saw along its ray (the scan test's check)
        head, body = open(ply, "rb").read().split(b"end_header\n", 1)
        nv = int([l for l in head.decode().splitlines() if l.startswith("element vertex")][0].split()[-1])
        v = np.frombuffer(body[:16 * nv], np.dtype([("p", "<f4", 3), ("c", "u1", 4)]))["p"].astype(np.float64)
        assert nv > 10000
        fx, fy, mx, my = Kint[0, 0], Kint[1, 1], Kint[0, 2], Kint[1, 2]
        sample = v[:: max(1, nv // 4000)]
        best = np.full(len(sample), np.inf)
        for i in (0, n // 2, n - 1):
            cam = (np.linalg.inv(T0inv @ truth[i].astype(np.float64)) @ np.c_[sample, np.ones(len(sample))].T).T[:, :3]
            z = cam[:, 2]
            u = np.round(cam[:, 0] / np.maximum(z, 1e-6) * fx + mx).astype(int); vv = np.round(cam[:, 1] / np.maximum(z, 1e-6) * fy + my).astype(int)
            ok = (z > 0.1) & (u >= 0) & (u < W) & (vv >= 0) & (vv < H)
            dd = np.full(len(sample), np.inf); dd[ok] = depths[i][vv[ok], u[ok]]
            best = np.minimum(best, np.where(np.isfinite(dd), np.abs(dd - z), np.inf))
        seen = np.isfinite(best)
        assert seen.mean() > 0.9 and np.percentile(best[seen], 90) < 0.06
        # the model is the fusion of the returned trajectory, from the raw frames the reader decodes
        r = sens.SensorDataReader(path)
        raw = [tuple(torch.from_numpy(x).to(cuda_device) for x in r.frame(i)[:2]) for i in range(n)]
        r.close()
        want, n_fused = fused_voxels(snap["hp"], raw, traj, cuda_device)
        assert n_fused == f["valid_transforms"]
        assert_model_is_fusion_of(snap["voxels"], want, "scan")
    finally:
        capi.lib().bfTsdfSetArithmetic(prev_arith)
    torch.cuda.synchronize()

"""Fusion along a fixed trajectory on the GPU: bfTsdfIntegrateBatch against bfTsdfIntegrateFrame one frame at a time (bit for bit, at 1 cm and
4 mm, batch sizes 1 / 7 / 16, a heap that runs out inside a batch); FrameLoop.fuse against the one-op-per-call replay of its op list
[INTEGRATE x <= 16, GARBAGE_COLLECT] through bfTsdfRunOps and, in the exact arithmetic, against the CPU oracle's replay and the reference's own
CUDA (oracle/_ref); fuse_recording on a synthetic .sens file and the two scan.py options that run through it."""
import ctypes as C
import json

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from bundlefusion_b200 import synth
from tests.test_frame_loop_model_gpu import DeviceReplay, W, H, hash_params_of, loop_model, run_loop

pytestmark = pytest.mark.gpu
INT, GC = capi.BF_TSDF_OP_INTEGRATE, capi.BF_TSDF_OP_GARBAGE_COLLECT


def _model(scene):
    from oracle import oracle as orc
    return orc.canonical_blocks(scene.download()), scene.getHeapFreeCount()


def _assert_same(a, b, what):
    ((ba, va), fa), ((bb, vb), fb) = a, b
    assert ba.shape == bb.shape and np.array_equal(ba, bb), (what, "block set", len(ba), len(bb))
    diff = np.nonzero((va != vb).any(axis=-1))[0]
    assert len(diff) == 0, (what, "voxel words differ in %d voxels" % len(diff))
    assert fa == fb, (what, "heap free", fa, fb)


def _frames(dev, n=40):
    """n synthetic frames 12 path steps apart (overlapping frustums); frame 5 has no valid depth"""
    from bundlefusion_b200 import synth_gpu
    d, c, T = synth_gpu.make_frames(list(range(0, 12 * n, 12)), W, H, device=dev)
    d[5].fill_(float("-inf"))
    return [d[i] for i in range(n)], [c[i] for i in range(n)], T


def _hash(voxel, blocks=None):
    from bundlefusion_b200.scene_rep import default_hash_params
    s = (0.01 / voxel) ** 2
    return default_hash_params(num_buckets=int(100003 * s) | 1, num_sdf_blocks=blocks or int(60000 * s), voxel_size=voxel)


def _one_by_one_and_batched(dev, hp, depth, color, T, batch):
    """the same frames into two fresh hashes: bfTsdfIntegrateFrame per frame vs bfTsdfIntegrateBatch per `batch` frames, GC after each batch"""
    from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF, camera_params
    cam = camera_params(W, H)
    one, bat = CUDASceneRepHashSDF(hp, dev), CUDASceneRepHashSDF(hp, dev)
    n = len(depth)
    for s in range(0, n, batch):
        idx = list(range(s, min(n, s + batch)))
        for i in idx:
            one.integrate(T[i], depth[i], color[i], cam)
        one.garbageCollect()
        bat.integrateBatch(idx, T[idx], depth, color, cam)
        bat.garbageCollect()
    return one, bat


@pytest.mark.parametrize("voxel,batch", [(0.01, 16), (0.004, 16), (0.01, 1), (0.01, 7)])
def test_integrate_batch_equals_frame_by_frame(cuda_device, voxel, batch):
    depth, color, T = _frames(cuda_device)
    one, bat = _one_by_one_and_batched(cuda_device, _hash(voxel), depth, color, T, batch)
    a, b = _model(one), _model(bat)
    _assert_same(b, a, "voxel %g, batch %d" % (voxel, batch))
    assert one.getLastFrameStats()["dropped"] == bat.getLastFrameStats()["dropped"] == 0
    assert np.allclose(np.array(list(bat.m_hashParams.m_rigidTransform.m)).reshape(4, 4), T[-1])       # hashParams holds the last pose
    print("voxel %g, batch %d: %d blocks, heap free %d" % (voxel, batch, len(a[0][0]), a[1]))
    one.close(); bat.close()


def test_integrate_batch_heap_runs_out_inside_a_batch(cuda_device):
    """a heap exactly as large as the blocks frames 0..6 insert: frames 7..15 of the 16-frame batch find it empty, and the batch drops the same
    inserts as the frames one by one"""
    from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF, camera_params
    depth, color, T = _frames(cuda_device, 16)
    probe = CUDASceneRepHashSDF(_hash(0.01), cuda_device)
    for i in range(7):
        probe.integrate(T[i], depth[i], color[i], camera_params(W, H))
    used = probe.m_hashParams.m_numSDFBlocks - probe.getHeapFreeCount()
    probe.close()
    one, bat = _one_by_one_and_batched(cuda_device, _hash(0.01, blocks=used), depth, color, T, 16)
    a, b = _model(one), _model(bat)
    _assert_same(b, a, "heap of %d blocks" % used)
    d1, d2 = one.getLastFrameStats()["dropped"], bat.getLastFrameStats()["dropped"]
    assert d1 == d2 and d1 > 0, (d1, d2)
    print("heap of %d blocks: %d inserts dropped, %d blocks kept" % (used, d1, len(a[0][0])))
    one.close(); bat.close()


@pytest.fixture(scope="module")
def finished_loop(cuda_device):
    r = run_loop(43, cuda_device)
    yield r
    r.loop.close()


def _fuse_ops(r):
    fin = [f for f in range(len(r.final)) if np.isfinite(r.final[f]).all()]
    ops = []
    for s in range(0, len(fin), 16):
        ops += [(INT, f, r.final[f]) for f in fin[s:s + 16]] + [(GC, 0, np.zeros((4, 4), np.float32))]
    return fin, ops


def test_frame_loop_fuse_equals_its_op_list_one_op_per_call(cuda_device, finished_loop):
    from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF
    r = finished_loop
    before = loop_model(r.loop, cuda_device)
    scene = CUDASceneRepHashSDF(hash_params_of(r.loop), cuda_device)
    info = r.loop.fuse(scene)
    fin, ops = _fuse_ops(r)
    assert info["frames_fused"] == len(fin) and info["frames_skipped"] == len(r.final) - len(fin) and info["batches"] == (len(fin) + 15) // 16
    assert info["inserts_dropped"] == 0 and info["heap_free"] == scene.getHeapFreeCount()
    rep = DeviceReplay(r, cuda_device)
    rep.run(ops)
    _assert_same(_model(scene), rep.model(), "FrameLoop.fuse vs its op list through bfTsdfRunOps, one op per call")
    _assert_same(loop_model(r.loop, cuda_device), before, "the loop's own model")
    rep.close(); scene.close()


def test_frame_loop_fuse_exact_equals_the_oracle_replay(cuda_device, finished_loop):
    from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF, camera_params
    from oracle import oracle as orc
    r = finished_loop
    scene = CUDASceneRepHashSDF(hash_params_of(r.loop), cuda_device, arithmetic="exact")
    r.loop.fuse(scene)
    _, ops = _fuse_ops(r)
    o = orc.OracleSceneRepHashSDF(hash_params_of(r.loop))
    cam = camera_params(W, H)
    for kind, f, T in ops:
        if kind == GC:
            o.garbageCollect(); continue
        d, c = r.loop.frame(f)
        o.integrate(T, d.cpu().numpy(), np.ascontiguousarray(c.cpu().numpy()), cam)
    _assert_same(_model(scene), (orc.canonical_blocks(o.download()), o.getHeapFreeCount()), "exact FrameLoop.fuse vs the oracle's replay")
    scene.close()


def test_exact_fusion_at_4mm_matches_reference_cuda(cuda_device, finished_loop):
    """the fusion at 4 mm in the exact arithmetic against the reference's own kernels (IEEE build) driven frame by frame along the same poses,
    with the same garbage collections: same block set, every voxel word identical"""
    from oracle import ref_tsdf
    if not ref_tsdf.available(fast=False):
        pytest.skip("oracle/_ref not built")
    from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF, camera_params
    from oracle import oracle as orc
    r = finished_loop
    n = 24
    hp = hash_params_of(r.loop)
    hp.m_virtualVoxelSize = 0.004; hp.m_hashNumBuckets = 600011; hp.m_numSDFBlocks = 400000
    scene = CUDASceneRepHashSDF(hp, cuda_device, arithmetic="exact")
    r.loop.fuse(scene, n=n)
    ref = ref_tsdf.ReferenceSceneRepHashSDF(hp, cuda_device, fast_math=False)
    cam = camera_params(W, H)
    fin = [f for f in range(n) if np.isfinite(r.final[f]).all()]
    for s in range(0, len(fin), 16):
        for f in fin[s:s + 16]:
            d, c = r.loop.frame(f)
            ref.integrate(r.final[f], d, c, cam)
        ref.garbageCollect()
    _assert_same(_model(scene), (orc.canonical_blocks(ref.download()), ref.getHeapFreeCount()), "exact fusion at 4 mm vs the reference's IEEE build")
    scene.close()


# ---- the application path ----------------------------------------------------------------------------------------------------------------
N_SENS, SKIP = 20, (3, 11)


@pytest.fixture(scope="module")
def recording(tmp_path_factory):
    from bundlefusion_b200 import sens
    from bundlefusion_b200.frame_loop import default_params
    K = np.array(list(default_params(W, H).depthIntrinsics), np.float32).reshape(4, 4)
    path = str(tmp_path_factory.mktemp("fuse") / "seq.sens")
    w = sens.SensorDataWriter(path, W, H, K, depth_shift=1000.0, zlib_depth=True)
    truth = []
    for i in range(N_SENS):
        d, c, T = synth.make_frame(2 * i, W, H, texture="rich")
        if i in SKIP:
            T = np.full((4, 4), -np.inf, np.float32)
        w.append(np.where(np.isfinite(d), np.clip(np.round(d * 1000.0), 1, 65535), 0).astype(np.uint16), c[..., :3], T)
        truth.append(T)
    w.finish()
    return path, np.stack(truth)


def _ply_triangles(path):
    head, body = open(path, "rb").read().split(b"end_header\n", 1)
    lines = head.decode().splitlines()
    nv = int([l for l in lines if l.startswith("element vertex")][0].split()[-1])
    nf = int([l for l in lines if l.startswith("element face")][0].split()[-1])
    v = np.frombuffer(body[:16 * nv], np.dtype([("p", "<f4", 3), ("c", "u1", 4)]))["p"]
    f = np.frombuffer(body[16 * nv:16 * nv + 13 * nf], np.dtype([("n", "u1"), ("i", "<u4", 3)]))["i"]
    return v[f].reshape(nf, 9).astype(np.float64)


def test_fuse_recording_equals_the_loops_fusion_of_the_same_file(cuda_device, recording, tmp_path):
    import torch
    from scipy.spatial import cKDTree

    from bundlefusion_b200 import fuse
    from bundlefusion_b200.frame_loop import FrameLoop
    from bundlefusion_b200.marching_cubes import CUDAMarchingCubesHashSDF, marching_cubes_params, merge_close_vertices, remove_duplicate_faces
    from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF
    from bundlefusion_b200.sens import SensorDataReader
    path, truth = recording
    rd = SensorDataReader(path)
    P = fuse.recording_params(rd.header, N_SENS)
    P.hash.m_hashNumBuckets, P.hash.m_numSDFBlocks = 100003, 90000
    loop = FrameLoop(P, cuda_device)
    ip = fuse.ingest_params(P)
    for i in range(N_SENS):
        d, c, _, _ = rd.frame(i, pinned=True)
        loop.step(d, c)
        # the ingest fuse_recording runs, on the same decoded frame: the loop's frame store bit for bit
        dd, dc = d.to(cuda_device), c.to(cuda_device)
        od = torch.empty((H, W), dtype=torch.float32, device=cuda_device); oc = torch.empty((H, W, 4), dtype=torch.uint8, device=cuda_device)
        capi.check(capi.lib().bfIngestFrame(C.byref(ip), dd.data_ptr(), dc.data_ptr(), od.data_ptr(), oc.data_ptr()), "bfIngestFrame")
        ld, lc = loop.frame(i)
        torch.cuda.synchronize(cuda_device)
        assert torch.equal(od.view(torch.int32), ld.view(torch.int32)) and torch.equal(oc, lc), "frame %d: ingest differs from the loop's frame store" % i
    loop.join()
    rd.close()
    hp = fuse.fine_hash_params(P, 0.005)
    ply = str(tmp_path / "fused.ply")
    o = fuse.fuse_recording(path, ply, 0.005, "recorded", hp.m_hashNumBuckets, hp.m_numSDFBlocks, cuda_device)
    assert o["frames"] == N_SENS and o["skipped"] == len(SKIP) and o["fused"] == N_SENS - len(SKIP) and o["batches"] == 2
    assert o["inserts_dropped"] == 0 and o["mesh_path"] == ply and o["triangles"] > 20000
    ref = CUDASceneRepHashSDF(hp, cuda_device)
    info = loop.fuse(ref, poses=truth)
    assert info["frames_skipped"] == len(SKIP) and info["frames_fused"] == N_SENS - len(SKIP)
    _assert_same(_model(o["scene"]), _model(ref), "fuse_recording vs FrameLoop.fuse along the recorded poses")
    # the mesh written = extractIsoSurface of that model, as a triangle multiset, after the clean-up saveMesh applies (vertices merged within
    # 1e-5 m -- which of two merged vertices stays depends on the extraction order -- degenerate and duplicate faces removed)
    mc = CUDAMarchingCubesHashSDF(marching_cubes_params(int(hp.m_hashNumBuckets), 0.005, 6_000_000), cuda_device)
    mc.extractIsoSurface(o["scene"])
    pos, col = mc.soup()
    mc.close()
    p2, _, f2 = merge_close_vertices(pos, col, np.arange(len(pos), dtype=np.uint32).reshape(-1, 3))
    want = p2[remove_duplicate_faces(f2)].reshape(-1, 9).astype(np.float64)
    got = _ply_triangles(ply)
    assert len(got) == len(want), (len(got), len(want))
    for a, b in ((got, want), (want, got)):
        dist, _ = cKDTree(b).query(a)
        assert dist.max() < 1e-4, dist.max()
    o["scene"].close(); ref.close(); loop.close()


def _face_count(path):
    head = open(path, "rb").read().split(b"end_header\n", 1)[0].decode()
    return int([l for l in head.splitlines() if l.startswith("element face")][0].split()[-1])


def test_scan_poses_recorded_and_mesh_voxel_size(cuda_device, recording, tmp_path, capsys):
    from bundlefusion_b200 import scan
    path, _ = recording
    sizes = ["--hash-buckets", "100003", "--sdf-blocks", "90000", "--device", str(cuda_device)]
    rec = str(tmp_path / "recorded.ply")
    assert scan.main([path, rec, "--poses", "recorded"] + sizes) == 0
    s = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert s["fuse"]["skipped"] == len(SKIP) and s["fuse"]["fused"] == N_SENS - len(SKIP) and s["mesh_path"] == rec and _face_count(rec) > 10000
    coarse, fine = str(tmp_path / "coarse.ply"), str(tmp_path / "fine.ply")
    assert scan.main([path, coarse, "--solve-frames-before-exit", "3"] + sizes) == 0
    capsys.readouterr()
    assert scan.main([path, fine, "--solve-frames-before-exit", "3", "--mesh-voxel-size", "0.005"] + sizes) == 0
    s = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert s["fuse"]["frames_fused"] >= N_SENS - 4 and s["fuse"]["inserts_dropped"] == 0 and s["mesh_path"] == fine
    print("triangles: recorded poses %d, 1 cm %d, 5 mm %d" % (_face_count(rec), _face_count(coarse), _face_count(fine)))
    assert _face_count(fine) > _face_count(coarse)

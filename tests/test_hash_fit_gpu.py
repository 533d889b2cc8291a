"""Sizing a fusion's voxel hash from a device count of the blocks it will allocate, on the GPU: the counted keys against the blocks
bfTsdfIntegrateBatch actually inserts into an ample hash (1 cm and 4 mm, one call and 16-frame chunks, a frame with no valid depth, a 2-rank
shard setting) and against the CPU oracle's allocs; a fusion into the fitted hash against the same fusion into a much larger one (no drop, the
same model); fuse_recording(fit_hash=True), FrameLoop.fit_hash_params, the table cap and both scan.py paths with --fit-hash."""
import ctypes as C
import json

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from tests.test_frame_loop_model_gpu import W, H, run_loop
from tests.test_trajectory_fusion_gpu import N_SENS, SKIP, _frames, _hash, recording  # noqa: F401  (recording: a fixture)

pytestmark = pytest.mark.gpu


def _blocks(scene):
    """the occupied block positions of a scene's hash, int32 [n, 3] in lexicographic order"""
    h = scene.download()["hash"]
    p = h[h[:, 3] != capi.BF_FREE_ENTRY, :3]
    return p[np.lexsort((p[:, 2], p[:, 1], p[:, 0]))]


def _with_shard(hp, rank, world):
    q = capi.BFHashParams()
    C.memmove(C.byref(q), C.byref(hp), C.sizeof(capi.BFHashParams))
    q.m_dummy = rank | (world << 32)
    return q


def _ample(voxel):
    hp = _hash(voxel)
    hp.m_hashNumBuckets = (4 * hp.m_hashNumBuckets) | 1
    hp.m_numSDFBlocks = 3 * hp.m_numSDFBlocks
    return hp


@pytest.mark.parametrize("voxel,chunked,shard", [(0.01, False, None), (0.01, True, None), (0.004, False, None), (0.004, True, None),
                                                 (0.01, True, (0, 2)), (0.004, False, (1, 2))])
def test_counted_union_equals_the_blocks_the_batch_inserts(cuda_device, voxel, chunked, shard):
    from bundlefusion_b200.fuse import BlockCounter
    from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF, camera_params
    depth, color, T = _frames(cuda_device)                    # 40 frames; frame 5 has no valid depth
    hp = _ample(voxel) if shard is None else _with_shard(_ample(voxel), *shard)
    cam = camera_params(W, H)
    scene = CUDASceneRepHashSDF(hp, cuda_device)
    for s in range(0, len(depth), 16):                         # never garbage-collected: the hash keeps every block it ever inserted
        idx = list(range(s, min(len(depth), s + 16)))
        scene.integrateBatch(idx, T[idx], depth, color, cam)
    assert scene.getLastFrameStats()["dropped"] == 0
    counter = BlockCounter(hp, cuda_device, capacity=1024)     # small on purpose: it has to grow, and recount, on the way
    if chunked:
        for s in range(0, len(depth), 16):
            counter.add(depth[s:s + 16], T[s:s + 16], cam)
    else:
        counter.add(depth, T, cam)
    want = _blocks(scene)
    got = counter.keys()
    assert counter.count == len(want) == len(got) > 0
    np.testing.assert_array_equal(got, want)
    assert counter.capacity > 1024
    print("voxel %g shard %s: %d blocks, key set of %d" % (voxel, shard, len(want), counter.capacity))
    scene.close()


def test_counted_union_equals_the_oracle_allocs(cuda_device):
    from bundlefusion_b200.fuse import BlockCounter
    from bundlefusion_b200.scene_rep import camera_params, default_hash_params
    from oracle import oracle as orc
    depth, color, T = _frames(cuda_device, 8)                 # frame 5 has no valid depth
    hp, cam = default_hash_params(num_buckets=200003, num_sdf_blocks=40000), camera_params(W, H)
    o = orc.OracleSceneRepHashSDF(hp)
    for i in range(8):                                         # the union of the per-frame alloc sets: one hash, no GC
        o._set_pose(T[i])
        assert o.L.orc_tsdf_alloc(C.byref(o.hd), C.byref(o.hp), np.ascontiguousarray(depth[i].cpu().numpy(), np.float32), C.byref(cam)) == 0
    h = o.download()["hash"]
    want = h[h[:, 3] != capi.BF_FREE_ENTRY, :3]
    want = want[np.lexsort((want[:, 2], want[:, 1], want[:, 0]))]
    counter = BlockCounter(hp, cuda_device)
    counter.add(depth, T, cam)
    np.testing.assert_array_equal(counter.keys(), want)


@pytest.fixture(scope="module")
def finished_loop(cuda_device):
    r = run_loop(43, cuda_device)
    yield r
    r.loop.close()


def _model(scene):
    from oracle import oracle as orc
    return orc.canonical_blocks(scene.download())


def test_fitted_fusion_at_4mm_drops_nothing_and_equals_an_ample_one(cuda_device, finished_loop):
    from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF
    r = finished_loop
    hp, rep = r.loop.fit_hash_params(0.004)
    assert rep["predicted_overflow"] == 0 and rep["max_load"] <= capi.BF_HASH_BUCKET_SIZE
    assert hp.m_numSDFBlocks == rep["blocks_counted"] and hp.m_hashNumBuckets == rep["buckets"] and hp.m_hashNumBuckets & 1
    fit = CUDASceneRepHashSDF(hp, cuda_device)
    info = r.loop.fuse(fit)                                    # a GC after every batch, as bfFrameLoopFuse runs it
    assert info["inserts_dropped"] == 0                        # neither a heap failure nor an insert without room
    big_hp = capi.BFHashParams()
    C.memmove(C.byref(big_hp), C.byref(hp), C.sizeof(capi.BFHashParams))
    big_hp.m_hashNumBuckets = (6 * hp.m_hashNumBuckets) | 1
    big_hp.m_numSDFBlocks = 4 * hp.m_numSDFBlocks
    big = CUDASceneRepHashSDF(big_hp, cuda_device)
    assert r.loop.fuse(big)["inserts_dropped"] == 0
    (ba, va), (bb, vb) = _model(fit), _model(big)
    np.testing.assert_array_equal(ba, bb)
    assert np.array_equal(va, vb), "voxel words differ"
    assert fit.getHeapFreeCount() == hp.m_numSDFBlocks - len(ba)
    print("4 mm: %d blocks counted, %d live after the last GC, %d buckets (%d candidates), %.1f MB table" %
          (rep["blocks_counted"], len(ba), rep["buckets"], rep["candidates_tried"], rep["table_bytes"] / 1e6))
    fit.close(); big.close()


def test_frame_loop_fit_then_fuse_meshes_as_an_ample_hash(cuda_device, finished_loop, tmp_path):
    from bundlefusion_b200 import fuse
    from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF
    r = finished_loop
    hp, rep = r.loop.fit_hash_params(0.005)
    fit = CUDASceneRepHashSDF(hp, cuda_device)
    assert r.loop.fuse(fit)["inserts_dropped"] == 0
    big = CUDASceneRepHashSDF(fuse.fine_hash_params(r.loop.params, 0.005, (8 * hp.m_hashNumBuckets) | 1, 4 * hp.m_numSDFBlocks), cuda_device)
    assert r.loop.fuse(big)["inserts_dropped"] == 0
    a = fuse.mesh_scene(fit, str(tmp_path / "fit.ply"), cuda_device)["triangles"]
    b = fuse.mesh_scene(big, str(tmp_path / "big.ply"), cuda_device)["triangles"]
    assert a == b > 0
    # the loop's state is untouched: counting again gives the same report
    assert r.loop.fit_hash_params(0.005)[1] == rep
    fit.close(); big.close()


def test_fuse_recording_fit_hash(cuda_device, recording, tmp_path):
    from bundlefusion_b200 import fuse
    path, _ = recording
    o = fuse.fuse_recording(path, str(tmp_path / "fit.ply"), 0.005, device=cuda_device, fit_hash=True)
    assert o["inserts_dropped"] == 0 and o["predicted_overflow"] == 0 and o["fused"] == N_SENS - len(SKIP)
    assert o["blocks_counted"] == o["scene"].m_hashParams.m_numSDFBlocks and o["buckets"] == o["scene"].m_hashParams.m_hashNumBuckets
    ample = fuse.fuse_recording(path, str(tmp_path / "ample.ply"), 0.005, hash_buckets=(8 * o["buckets"]) | 1, sdf_blocks=4 * o["blocks_counted"],
                                device=cuda_device)
    assert ample["inserts_dropped"] == 0
    assert o["triangles"] == ample["triangles"] > 0
    np.testing.assert_array_equal(_model(o["scene"])[0], _model(ample["scene"])[0])
    o["scene"].close(); ample["scene"].close()


def test_table_cap_predicts_overflow_and_the_fusion_still_runs(cuda_device, recording):
    from bundlefusion_b200 import fuse
    path, _ = recording
    free = fuse.fuse_recording(path, None, 0.005, device=cuda_device, fit_hash=True)
    cap = fuse.table_bytes(free["blocks_counted"] // 16)
    o = fuse.fuse_recording(path, None, 0.005, device=cuda_device, fit_hash=True, max_table_bytes=cap)
    assert o["predicted_overflow"] > 0 and o["fit"]["table_bytes"] <= cap and o["blocks_counted"] == free["blocks_counted"]
    assert o["batches"] == free["batches"] and isinstance(o["inserts_dropped"], int)
    print("cap %d B: %d buckets for %d blocks, predicted overflow %d, inserts dropped %d" %
          (cap, o["buckets"], o["blocks_counted"], o["predicted_overflow"], o["inserts_dropped"]))
    free["scene"].close(); o["scene"].close()


def test_scan_fit_hash_end_to_end(cuda_device, recording, tmp_path, capsys):
    from bundlefusion_b200 import scan
    path, _ = recording
    rec = str(tmp_path / "recorded.ply")
    assert scan.main([path, rec, "--poses", "recorded", "--mesh-voxel-size", "0.005", "--fit-hash", "--device", str(cuda_device)]) == 0
    s = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert s["fit"]["predicted_overflow"] == 0 and s["fuse"]["inserts_dropped"] == 0 and s["fuse"]["fused"] == N_SENS - len(SKIP)
    assert s["mesh_path"] == rec and s["triangles"] > 0
    fine = str(tmp_path / "fine.ply")
    assert scan.main([path, fine, "--solve-frames-before-exit", "3", "--mesh-voxel-size", "0.005", "--fit-hash", "--hash-buckets", "100003",
                      "--sdf-blocks", "90000", "--device", str(cuda_device)]) == 0
    s = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert s["fit"]["predicted_overflow"] == 0 and s["fuse"]["inserts_dropped"] == 0 and s["mesh_path"] == fine and s["triangles"] > 0
    assert s["fit"]["blocks_counted"] > 0

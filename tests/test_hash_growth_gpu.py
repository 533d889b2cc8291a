"""Growing the voxel hash, on the GPU.  bfTsdfRehash (CUDASceneRepHashSDF.rehash): after a rehash into a larger, a same-size and a smaller
table the model equals the source's keyed by block position, a garbage collection issued next frees the same blocks -- for each kind of last
list: a single integrate, a GC's stale list, a fused re-integration, a re-integration batch, an integrate batch and a bfTsdfRunOps replay -- and a
further op list keeps the two equal; in fast and exact arithmetic and under a 2-rank shard setting.  The frame loop with growth on against a
fixed table large enough never to drop: statuses, trajectory, op log and model bit for bit, after the steps and after finish(30), and the host
synchronisation rule.  A fixed table's loop hands the table's memory back when it is destroyed.  scan.py --grow-hash against a fixed large hash,
and with a ceiling too small to hold the scan."""
import ctypes as C
import json

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from bundlefusion_b200 import fuse, synth
from bundlefusion_b200.frame_loop import FrameLoop
from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF, camera_params, default_hash_params
from oracle import oracle as orc
from tests.test_frame_loop_model_gpu import loop_model, loop_params, stream
from tests.test_trajectory_fusion_gpu import recording  # noqa: F401  (a fixture)

pytestmark = pytest.mark.gpu
INT, DEINT, GC = capi.BF_TSDF_OP_INTEGRATE, capi.BF_TSDF_OP_DEINTEGRATE, capi.BF_TSDF_OP_GARBAGE_COLLECT
W, H = 160, 120
BLOCKS, BUCKETS = 30000, 20011


def _frames(dev):
    import torch
    fr = [synth.make_frame(3 * i, W, H) for i in range(8)]
    return ([torch.from_numpy(d).to(dev) for d, _, _ in fr], [torch.from_numpy(c).to(dev) for _, c, _ in fr], [T for _, _, T in fr])


def _moved(T, dx):
    U = np.array(T, np.float32).copy()
    U[0, 3] += dx
    return U


def _build(kind, dev, arith, shard, fr):
    """a model with integrations, a de-integration and GCs, ending on the kind of last list given"""
    D, Cc, T = fr
    hp = default_hash_params(num_buckets=BUCKETS, num_sdf_blocks=BLOCKS)
    if shard:
        hp.m_dummy = shard[0] | (shard[1] << 32)
    s = CUDASceneRepHashSDF(hp, dev, arithmetic=arith)
    cam = camera_params(W, H)
    for i in range(4):
        s.integrate(T[i], D[i], Cc[i], cam)
    s.garbageCollect()
    s.deIntegrate(T[3], D[3], Cc[3], cam)              # the blocks only frame 3 reached are now empty: garbage for the next GC of a list that holds them
    if kind == "single":
        s.integrate(T[2], D[2], Cc[2], cam)
    elif kind == "stale":                              # a turn without re-integration: its GC walks the list the previous GC walked
        s.integrate(T[2], D[2], Cc[2], cam)
        s.garbageCollect()
    elif kind == "dual":                               # the last list (bit 1: the new pose's frustum) is where frame 3's emptied blocks lie
        s.runOps([(DEINT, 2, T[2]), (INT, 2, _moved(T[2], 0.01))], D, Cc, cam)
    elif kind == "batch":
        s.runOps([op for k in (0, 1, 2) for op in ((DEINT, k, T[k]), (INT, k, _moved(T[k], 0.01)))], D, Cc, cam)
    elif kind == "integrate_batch":                    # frames that never reached frame 3's emptied blocks; GC flags: the last frame's frustum, as in "single"
        s.integrateBatch([1, 2], np.stack([T[1], T[2]]), D, Cc, cam)
    elif kind == "run_ops":                            # a replay with a GC inside, ending on a de-integration that leaves frame 2's own blocks empty
        s.runOps([(DEINT, 0, T[0]), (INT, 0, _moved(T[0], -0.01)), (GC, 0, None), (INT, 5, T[5]), (DEINT, 2, T[2])], D, Cc, cam)
    return s, cam


def _model(s):
    b, v = orc.canonical_blocks(s.download())
    return b, v


def _same(a, b, what):
    (ba, va), (bb, vb) = a, b
    assert ba.shape == bb.shape and np.array_equal(ba, bb), (what, "block set", len(ba), len(bb))
    assert np.array_equal(va, vb), (what, "voxel words differ in %d voxels" % int((va != vb).any(-1).sum()))


def _live(s):
    return s.m_hashParams.m_numSDFBlocks - s.getHeapFreeCount()


@pytest.mark.parametrize("arith,shard", [("fast", None), ("exact", None), ("fast", (1, 2))])
@pytest.mark.parametrize("kind", ["single", "stale", "dual", "batch", "integrate_batch", "run_ops"])
def test_rehash_keeps_the_model_and_what_the_next_gc_frees(cuda_device, kind, arith, shard):
    fr = _frames(cuda_device)
    D, Cc, T = fr
    ref, cam = _build(kind, cuda_device, arith, shard, fr)
    live = _live(ref)
    assert live > 0
    sizes = [(2 * BLOCKS, 2 * BUCKETS + 1), (BLOCKS, BUCKETS), (min(BLOCKS - 1, live + 4000), 10007)]
    freed_any = False
    for blocks, buckets in sizes:
        s, _ = _build(kind, cuda_device, arith, shard, fr)
        _same(_model(s), _model(ref), "%s: two builds" % kind)
        before = s.getLastFrameStats()
        got = s.rehash(blocks, buckets)
        assert got == {"moved": live, "refused": 0}, got
        assert s.m_hashParams.m_numSDFBlocks == blocks and s.m_hashParams.m_hashNumBuckets == buckets
        assert s.getLastFrameStats()["dropped"] == before["dropped"] == 0
        _same(_model(s), _model(ref), "%s -> %d blocks: after the rehash" % (kind, blocks))
        orc.check_hash_invariants(s.download(), s.m_hashParams)
        # GC right after the rehash, on a fresh twin of the source and on the rehashed copy
        twin, _ = _build(kind, cuda_device, arith, shard, fr)
        twin.garbageCollect(); s.garbageCollect()
        _same(_model(s), _model(twin), "%s -> %d blocks: after the GC" % (kind, blocks))
        freed_any |= _live(twin) < live
        assert _live(s) == _live(twin)
        # a further op list on both
        more = [(DEINT, 2, T[2]), (INT, 2, _moved(T[2], 0.02)), (INT, 6, T[6]), (GC, 0, None), (INT, 7, T[7]), (DEINT, 6, T[6]), (GC, 0, None)]
        twin.runOps(more, D, Cc, cam); s.runOps(more, D, Cc, cam)
        _same(_model(s), _model(twin), "%s -> %d blocks: after further ops" % (kind, blocks))
        s.close(); twin.close()
    # every last list no GC has walked holds emptied blocks ("stale": a GC walked it before the rehash; under the shard setting this rank may own
    # none of them), so its GC must free some: a list whose flags or parity did not move would free none
    if kind != "stale" and shard is None:
        assert freed_any, "%s: the GC after the rehash freed nothing: the case does not test the list" % kind
    ref.close()


def _snapshot(s):
    d = s.download()
    return {k: d[k].copy() if hasattr(d[k], "copy") else d[k] for k in ("hash", "compactified", "compactified_count", "heap", "heap_counter", "voxels")}, \
        s.getLastFrameStats()


def _unchanged(a, b, what):
    (da, sa), (db, sb) = a, b
    assert sa == sb, (what, "counters", sa, sb)
    for k in da:
        assert np.array_equal(da[k], db[k]), (what, k)


def test_rehash_refusals_write_nothing_to_dst(cuda_device):
    """every refusal on real tables: rc 1 (cudaErrorInvalidValue), the reason the check names, and dst -- its entries, list, heap, voxels and
    counters -- as it was; src keeps its model"""
    fr = _frames(cuda_device)
    src, _ = _build("single", cuda_device, "fast", None, fr)
    live, model = _live(src), _model(src)
    dst = CUDASceneRepHashSDF(default_hash_params(num_buckets=BUCKETS, num_sdf_blocks=BLOCKS), cuda_device)
    small = CUDASceneRepHashSDF(default_hash_params(num_buckets=BUCKETS, num_sdf_blocks=live - 1), cuda_device)
    lib = capi.lib()
    out = (C.c_ulonglong * 2)()

    def params(**kw):
        hp = capi.BFHashParams()
        C.memmove(C.byref(hp), C.byref(dst.m_hashParams), C.sizeof(capi.BFHashParams))
        for k, v in kw.items():
            setattr(hp, k, v)
        return hp
    shared = capi.BFHashDataStruct()
    C.memmove(C.byref(shared), C.byref(dst.m_hashData), C.sizeof(capi.BFHashDataStruct))
    shared.d_SDFBlocks = src.m_hashData.d_SDFBlocks
    cases = {
        "voxel size differs": params(m_virtualVoxelSize=0.005), "truncation differs": params(m_truncation=0.05),
        "truncation scale differs": params(m_truncScale=0.03), "max integration distance differs": params(m_maxIntegrationDistance=2.0),
        "block size differs": params(m_SDFBlockSize=4), "bucket size differs": params(m_hashBucketSize=2),
        "linked-list limit differs": params(m_hashMaxCollisionLinkedListSize=9), "shard setting (m_dummy) differs": params(m_dummy=1 | (2 << 32)),
    }
    before, before_small = _snapshot(dst), _snapshot(small)
    for why, hp in cases.items():
        assert lib.bfTsdfRehash(C.byref(src.m_hashData), C.byref(src.m_hashParams), C.byref(dst.m_hashData), C.byref(hp), out) == 1, why
        assert lib.bfGetLastErrorString().decode() == "bfTsdfRehash: " + why
        _unchanged(_snapshot(dst), before, why)
    assert lib.bfTsdfRehash(C.byref(src.m_hashData), C.byref(src.m_hashParams), C.byref(src.m_hashData), C.byref(src.m_hashParams), out) == 1
    assert lib.bfGetLastErrorString().decode() == "bfTsdfRehash: src == dst"
    assert lib.bfTsdfRehash(C.byref(src.m_hashData), C.byref(src.m_hashParams), C.byref(shared), C.byref(dst.m_hashParams), out) == 1
    assert lib.bfGetLastErrorString().decode() == "bfTsdfRehash: src and dst share a buffer"
    _unchanged(_snapshot(dst), before, "shared buffer")
    # a heap one block short of the live blocks: refused after one read of src
    assert lib.bfTsdfRehash(C.byref(src.m_hashData), C.byref(src.m_hashParams), C.byref(small.m_hashData), C.byref(small.m_hashParams), out) == 1
    assert lib.bfGetLastErrorString().decode() == "bfTsdfRehash: dst heap smaller than src's live blocks or its last list"
    _unchanged(_snapshot(small), before_small, "heap too small")
    with pytest.raises(RuntimeError, match="error 1"):
        src.rehash(live - 1, BUCKETS)
    assert src.m_hashParams.m_numSDFBlocks == BLOCKS
    _same(_model(src), model, "src after the refusals")
    # and the same tables rehash once the arguments are right
    assert src.rehash(BLOCKS, BUCKETS) == {"moved": live, "refused": 0}
    _same(_model(src), model, "src rehashed after the refusals")
    src.close(); dst.close(); small.close()


# ---- the frame loop ------------------------------------------------------------------------------------------------------------------------
N_LOOP, K_FINISH = 43, 30


def _run(p, dev):
    loop = FrameLoop(p, dev)
    loop.set_op_log(True)
    status = [loop.step(d, c).as_dict() for d, c in stream(N_LOOP, dev)]
    loop.join()
    r = {"status": status, "traj": loop.trajectory(N_LOOP), "model": loop_model(loop, dev)[0], "growth": loop.hash_growth(),
         "syncs": loop.counters()["host_syncs"]}
    r["finish"] = loop.finish(K_FINISH)
    loop.join()
    r.update({"traj_end": loop.trajectory(N_LOOP), "model_end": loop_model(loop, dev)[0], "growth_end": loop.hash_growth(),
              "syncs_end": loop.counters()["host_syncs"], "log": loop.op_log()})
    loop.close()
    return r


def _first_turn_blocks(dev):
    """blocks the loop's first turn allocates (the table must hold them before any read-back exists)"""
    p = loop_params(N_LOOP)
    loop = FrameLoop(p, dev)
    d, c = stream(N_LOOP, dev)[0]
    loop.step(d, c)
    used = p.hash.m_numSDFBlocks - loop.heap_free()
    loop.close()
    return used


@pytest.fixture(scope="module")
def loop_runs(cuda_device):
    fixed = _run(loop_params(N_LOOP), cuda_device)
    final = len(fixed["model_end"][0])
    start = max(final // 8, _first_turn_blocks(cuda_device) * 5 // 4)
    p = loop_params(N_LOOP)
    p.hashMaxSDFBlocks = p.hash.m_numSDFBlocks
    p.hash.m_hashNumBuckets = (4 * start) | 1                  # the reference's 4 buckets per block: the XOR bucket function fills probe windows at 1
    p.hash.m_numSDFBlocks = start
    grown = _run(p, cuda_device)
    print("fixed: %d blocks at the end; growing from %d blocks: %s, after finish %s" % (final, start, grown["growth"], grown["growth_end"]))
    return fixed, grown, start


def test_growing_loop_equals_a_fixed_ample_table(cuda_device, loop_runs):
    fixed, grown, start = loop_runs
    assert fixed["growth"]["growths"] == 0 and fixed["growth_end"]["inserts_dropped"] == 0
    assert grown["growth"]["growths"] >= 1 and grown["growth_end"]["growths"] >= 2, (grown["growth"], grown["growth_end"])
    assert grown["growth_end"]["inserts_dropped"] == 0 and not grown["growth_end"]["ceiling_reached"]
    assert grown["growth_end"]["sdf_blocks"] > start
    assert len(fixed["status"]) == len(grown["status"])
    for a, b in zip(fixed["status"], grown["status"]):
        assert a.keys() == b.keys() and all((a[k].tobytes() == b[k].tobytes()) if k == "transform" else a[k] == b[k] for k in a), (a, b)
    assert fixed["traj"].tobytes() == grown["traj"].tobytes() and fixed["traj_end"].tobytes() == grown["traj_end"].tobytes()
    for x, y in zip(fixed["log"], grown["log"]):
        assert x.tobytes() == y.tobytes()
    same_heap = ("heap_free", "valid")                              # the heaps differ in size: the free count and the verdict that reads it
    assert {k: v for k, v in fixed["finish"].items() if k not in same_heap} == {k: v for k, v in grown["finish"].items() if k not in same_heap}
    _same(grown["model"], fixed["model"], "after the steps")
    _same(grown["model_end"], fixed["model_end"], "after finish(%d)" % K_FINISH)


def test_growth_adds_host_synchronisations_only_when_it_grows(cuda_device, loop_runs):
    fixed, grown, _ = loop_runs
    per = 2                                                     # BF_FRAMELOOP_GROWTH_SYNCS, per attempt
    attempts = lambda g: g["growths"] + g["discarded"]
    assert grown["syncs"] - fixed["syncs"] == per * attempts(grown["growth"])
    assert grown["syncs_end"] - fixed["syncs_end"] == per * attempts(grown["growth_end"])


def test_fixed_table_loop_hands_its_table_back(cuda_device):
    """a fixed table comes from the same stream-ordered allocator as a growing one; destroying the loop returns it to the device"""
    import torch
    p = loop_params(N_LOOP)
    assert p.hashMaxSDFBlocks == 0
    table = fuse.table_bytes(p.hash.m_hashNumBuckets) + (4 + C.sizeof(capi.BFVoxel) * capi.BF_SDF_BLOCK_VOXELS) * p.hash.m_numSDFBlocks
    FrameLoop(p, cuda_device).close()                           # the library's process-wide workspaces outlive the first loop
    torch.cuda.synchronize(cuda_device)
    before = torch.cuda.mem_get_info(cuda_device)[0]
    loop = FrameLoop(p, cuda_device)
    during = torch.cuda.mem_get_info(cuda_device)[0]
    loop.close()
    torch.cuda.synchronize(cuda_device)
    after = torch.cuda.mem_get_info(cuda_device)[0]
    print("free bytes: before %d, with the loop %d, after %d; table %d" % (before, during, after, table))
    assert before - during >= table
    assert abs(after - before) < table // 16, (before, after)


def test_scan_grow_hash(cuda_device, recording, tmp_path, capsys):  # noqa: F811
    from bundlefusion_b200 import scan
    path, _ = recording
    dev = str(cuda_device)
    assert scan.main([path, str(tmp_path / "fixed.ply"), "--solve-frames-before-exit", "3", "--hash-buckets", "100003", "--sdf-blocks", "90000",
                      "--device", dev]) == 0
    fixed = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert "hash" not in fixed and fixed["triangles"] > 0
    start = _first_turn_blocks(cuda_device) * 3 // 2 + 256
    assert scan.main([path, str(tmp_path / "grown.ply"), "--solve-frames-before-exit", "3", "--hash-buckets", str((4 * start) | 1),
                      "--sdf-blocks", str(start), "--grow-hash", "90000", "--device", dev]) == 0
    grown = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert grown["hash"]["growths"] >= 1 and grown["hash"]["inserts_dropped"] == 0 and grown["hash"]["sdf_blocks"] > start, grown["hash"]
    assert grown["triangles"] == fixed["triangles"]
    # a ceiling too small to hold the scan: drops are reported and the scan ends normally
    assert scan.main([path, str(tmp_path / "small.ply"), "--solve-frames-before-exit", "3", "--hash-buckets", "1009", "--sdf-blocks", "600",
                      "--grow-hash", "1200", "--device", dev]) == 0
    small = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert small["hash"]["inserts_dropped"] > 0 and small["hash"]["sdf_blocks"] <= 1200 and small["mesh_path"] is not None

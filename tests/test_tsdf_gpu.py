"""GPU parity tests of the TSDF path: CUDA library (through the C-ABI) vs the CPU oracle on the same
seeded inputs.  Parity key (SURVEY.md section 7): the sorted SET of block coordinates must be bit-exact and
the voxel words keyed by world block position must be bit-exact (both sides use individually rounded fp32
operations, see oracle/tsdf_oracle.c header); slot / table-index assignment is race-dependent in the
reference and is not compared.
"""
import ctypes as C

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from bundlefusion_b200 import synth
from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF, camera_params, default_hash_params, set_pose
from oracle import oracle as orc

pytestmark = pytest.mark.gpu
F = np.float32


def to_dev(torch, dev, depth, color):
    return torch.from_numpy(depth).to(dev), torch.from_numpy(color).to(dev)


def assert_same_state(gpu: CUDASceneRepHashSDF, cpu: orc.OracleSceneRepHashSDF, hp, check_list=True):
    gs, cs = gpu.download(), cpu.download()
    orc.check_hash_invariants(gs, hp)
    gb, gv = orc.canonical_blocks(gs)
    cb, cv = orc.canonical_blocks(cs)
    np.testing.assert_array_equal(gb, cb)                       # block set: bit-exact
    np.testing.assert_array_equal(gv, cv)                       # sdf / weight / colour words: bit-exact
    assert gpu.getHeapFreeCount() == cpu.getHeapFreeCount()
    if check_list:
        n = gpu.getNumOccupiedBlocks()
        assert n == cpu.num_occupied
        gl = gs["compactified"][:n]
        cl = cs["compactified"][:n]
        key = lambda a: a[np.lexsort((a[:, 2], a[:, 1], a[:, 0]))][:, :3]
        np.testing.assert_array_equal(key(gl), key(cl))
        # every compactified entry points at the voxels of the block it names
        lut = {tuple(e[:3]): e[3] for e in gs["hash"][gs["hash"][:, 3] != -2]}
        for e in gl[:: max(1, n // 500)]:
            assert lut[tuple(e[:3])] == e[3]


def small_params(**kw):
    kw.setdefault("num_buckets", 20011)
    kw.setdefault("num_sdf_blocks", 30000)
    return default_hash_params(**kw)


def test_single_frame_parity(cuda_device):
    import torch
    W, H = 160, 120
    cam, hp = camera_params(W, H), small_params()
    depth, color, T = synth.make_frame(3, W, H)
    gpu, cpu = CUDASceneRepHashSDF(hp, cuda_device, arithmetic="exact"), orc.OracleSceneRepHashSDF(hp)
    d, c = to_dev(torch, cuda_device, depth, color)
    gpu.integrate(T, d, c, cam)
    cpu.integrate(T, depth, color, cam)
    assert_same_state(gpu, cpu, hp)
    st = gpu.getLastFrameStats()
    assert st["E"] == cpu.num_occupied and st["U"] == cpu.last_U and st["U"] > 0


def test_sequence_reintegration_gc_parity(cuda_device):
    """The per-frame loop of DepthSensing.cpp:854-902,1049: integrate a stream, then de-integrate two frames at their
    old pose, re-integrate them at an updated pose, garbage-collect; compare after every step."""
    import torch
    W, H = 160, 120
    cam, hp = camera_params(W, H), small_params()
    gpu, cpu = CUDASceneRepHashSDF(hp, cuda_device, arithmetic="exact"), orc.OracleSceneRepHashSDF(hp)
    frames = [synth.make_frame(40 * i, W, H) for i in range(5)]
    dev = [to_dev(torch, cuda_device, f[0], f[1]) for f in frames]
    for (depth, color, T), (d, c) in zip(frames, dev):
        gpu.integrate(T, d, c, cam)
        cpu.integrate(T, depth, color, cam)
        assert_same_state(gpu, cpu, hp)
    for k in (1, 3):
        depth, color, T = frames[k]
        d, c = dev[k]
        gpu.deIntegrate(T, d, c, cam)
        cpu.deIntegrate(T, depth, color, cam)
        assert_same_state(gpu, cpu, hp)
        T2 = T.copy()
        T2[:3, 3] += np.array([0.013, -0.007, 0.004], F)
        gpu.integrate(T2, d, c, cam)
        cpu.integrate(T2, depth, color, cam)
        assert_same_state(gpu, cpu, hp)
    # remove frame 0 entirely, then collect garbage
    depth, color, T = frames[0]
    gpu.deIntegrate(T, dev[0][0], dev[0][1], cam)
    cpu.deIntegrate(T, depth, color, cam)
    gpu.garbageCollect()
    freed = cpu.garbageCollect()
    assert_same_state(gpu, cpu, hp, check_list=False)
    assert freed >= 0


def test_full_resolution_frame_parity(cuda_device):
    """BASELINE.json frame size (640x480) with the reference's default table sizes (zParametersDefault.txt:48-50)."""
    import torch
    W, H = 640, 480
    cam, hp = camera_params(W, H), default_hash_params()
    gpu, cpu = CUDASceneRepHashSDF(hp, cuda_device, arithmetic="exact"), orc.OracleSceneRepHashSDF(hp)
    for idx in (0, 25):
        depth, color, T = synth.make_frame(idx, W, H)
        d, c = to_dev(torch, cuda_device, depth, color)
        gpu.integrate(T, d, c, cam)
        cpu.integrate(T, depth, color, cam)
    assert_same_state(gpu, cpu, hp)


def test_roundtrip_and_idempotence_properties(cuda_device):
    """Size-independent properties at full frame size: (1) integrate then de-integrate of the same frame/pose leaves
    every voxel zero; (2) garbage collection then returns every in-frustum block; (3) a second alloc of the same
    frame allocates nothing (the fixed point the reference's host loop iterates to)."""
    import torch
    W, H = 640, 480
    cam, hp = camera_params(W, H), default_hash_params()
    gpu = CUDASceneRepHashSDF(hp, cuda_device, arithmetic="exact")
    depth, color, T = synth.make_frame(100, W, H)
    d, c = to_dev(torch, cuda_device, depth, color)
    free0 = gpu.getHeapFreeCount()
    gpu.integrate(T, d, c, cam)
    free1 = gpu.getHeapFreeCount()
    assert free1 < free0
    # idempotent alloc through the reference-named stub (same latched params)
    L = gpu.lib
    L.updateConstantHashParams(C.byref(gpu.m_hashParams))
    L.updateConstantDepthCameraParams(C.byref(cam))
    dd = capi.BFDepthCameraData(); dd.d_depthData = d.data_ptr(); dd.d_colorData = c.data_ptr()
    L.bindInputDepthColorTextures(C.byref(dd), W, H)
    L.allocCUDA(C.byref(gpu.m_hashData), C.byref(gpu.m_hashParams), C.byref(dd), C.byref(cam), None)
    assert gpu.getHeapFreeCount() == free1
    gpu.deIntegrate(T, d, c, cam)
    snap = gpu.download()
    assert not snap["voxels"].any()
    n = gpu.getNumOccupiedBlocks()
    gpu.garbageCollect()
    assert gpu.getHeapFreeCount() == free1 + n
    orc.check_hash_invariants(gpu.download(), hp)


def test_overflow_chains_parity(cuda_device):
    """Tiny table: most blocks live in overflow lists (VoxelUtilHashSDF.h:614-654) and inserts contend for the
    same buckets.  No duplicates, all reachable, same block set and voxels as the sequential oracle."""
    import torch
    W, H = 160, 120
    cam = camera_params(W, H)
    hp = small_params(num_buckets=2053, num_sdf_blocks=6000)
    T = np.eye(4, dtype=F)
    T[:3, :3] = np.array([[-1, 0, 0], [0, 1, 0], [0, 0, -1]], F)
    T[:3, 3] = [-0.33, -0.21, -0.17]
    depth, color, _ = synth.make_frame(7, W, H)
    gpu, cpu = CUDASceneRepHashSDF(hp, cuda_device, arithmetic="exact"), orc.OracleSceneRepHashSDF(hp)
    d, c = to_dev(torch, cuda_device, depth, color)
    gpu.integrate(T, d, c, cam)
    cpu.integrate(T, depth, color, cam)
    gs = gpu.download()
    used = gs["hash"][:, 3] != -2
    assert np.any(gs["hash"][used, 4] != 0)
    # which blocks get DROPPED when a probe window is full depends on insertion order (a race in the reference too);
    # set equality is only defined when nothing was dropped on either side
    assert cpu.dropped == 0 and gpu.getLastFrameStats()["dropped"] == 0
    assert_same_state(gpu, cpu, hp)
    gpu.deIntegrate(T, d, c, cam)
    cpu.deIntegrate(T, depth, color, cam)
    gpu.garbageCollect()
    cpu.garbageCollect()
    assert_same_state(gpu, cpu, hp, check_list=False)


def test_reference_named_stubs_sequence(cuda_device):
    """Drive the library exactly as CUDASceneRepHashSDF::integrate does in the reference (h:65-83, 328-384): latch
    constants, bind images, host alloc loop on the heap count, compactifyHashAllInOneCUDA, integrateDepthMapCUDA,
    then garbageCollectIdentify/Free.  Result must equal the oracle's."""
    import torch
    W, H = 160, 120
    cam, hp = camera_params(W, H), small_params()
    depth, color, T = synth.make_frame(9, W, H)
    gpu, cpu = CUDASceneRepHashSDF(hp, cuda_device, arithmetic="exact"), orc.OracleSceneRepHashSDF(hp)
    d, c = to_dev(torch, cuda_device, depth, color)
    L, hd, p = gpu.lib, gpu.m_hashData, gpu.m_hashParams
    L.bfSetStream(None)
    torch.cuda.synchronize()
    dd = capi.BFDepthCameraData(); dd.d_depthData = d.data_ptr(); dd.d_colorData = c.data_ptr()
    L.resetCUDA(C.byref(hd), C.byref(p))
    L.updateConstantDepthCameraParams(C.byref(cam))
    L.bindInputDepthColorTextures(C.byref(dd), W, H)
    set_pose(p, T)
    L.updateConstantHashParams(C.byref(p))
    prev, rounds = gpu.getHeapFreeCount(), 0
    while True:
        L.resetHashBucketMutexCUDA(C.byref(hd), C.byref(p))
        L.allocCUDA(C.byref(hd), C.byref(p), C.byref(dd), C.byref(cam), None)
        cur = gpu.getHeapFreeCount()
        rounds += 1
        if cur == prev:
            break
        prev = cur
    assert rounds == 2                                # one productive round, one confirming round
    p.m_numOccupiedBlocks = L.compactifyHashAllInOneCUDA(C.byref(hd), C.byref(p))
    L.updateConstantHashParams(C.byref(p))
    L.integrateDepthMapCUDA(C.byref(hd), C.byref(p), C.byref(dd), C.byref(cam))
    torch.cuda.synchronize()
    cpu.integrate(T, depth, color, cam)
    assert p.m_numOccupiedBlocks == cpu.num_occupied
    assert_same_state(gpu, cpu, hp)
    # de-integrate + GC through the stubs
    L.deIntegrateDepthMapCUDA(C.byref(hd), C.byref(p), C.byref(dd), C.byref(cam))
    L.garbageCollectIdentifyCUDA(C.byref(hd), C.byref(p))
    L.resetHashBucketMutexCUDA(C.byref(hd), C.byref(p))
    L.garbageCollectFreeCUDA(C.byref(hd), C.byref(p))
    torch.cuda.synchronize()
    cpu.deIntegrate(T, depth, color, cam)
    cpu.garbageCollect()
    assert_same_state(gpu, cpu, hp, check_list=False)


def test_depth_only_frame_is_a_noop(cuda_device):
    """Reference behaviour: without colour data no voxel passes `color.x != MINF` (.cu:441-448), blocks are still allocated."""
    import torch
    W, H = 80, 60
    cam, hp = camera_params(W, H), small_params()
    depth, _ = synth.plane_frame(W, H, 1.0)
    gpu = CUDASceneRepHashSDF(hp, cuda_device, arithmetic="exact")
    gpu.integrate(np.eye(4, dtype=F), torch.from_numpy(depth).to(cuda_device), None, cam)
    snap = gpu.download()
    assert not snap["voxels"].any()
    assert gpu.getHeapFreeCount() < hp.m_numSDFBlocks


def test_overfull_table_keeps_invariants(cuda_device):
    """Over-full table (drops happen): the structure must stay consistent -- no duplicates, no leaked slots, all locks
    released, every entry reachable -- even though WHICH blocks are dropped is order-dependent."""
    import torch
    W, H = 160, 120
    cam = camera_params(W, H)
    hp = small_params(num_buckets=509, num_sdf_blocks=1500)
    gpu = CUDASceneRepHashSDF(hp, cuda_device, arithmetic="exact")
    for idx in (7, 300, 600):
        depth, color, T = synth.make_frame(idx, W, H)
        d, c = to_dev(torch, cuda_device, depth, color)
        gpu.integrate(T, d, c, cam)
        orc.check_hash_invariants(gpu.download(), hp)
    assert gpu.getLastFrameStats()["dropped"] > 0
    assert gpu.getHeapFreeCount() >= 0


def test_fused_reintegration_matches_two_pass_oracle(cuda_device):
    """bfTsdfRunOps fuses every (de-integrate f @ old pose, integrate f @ new pose) pair into one pass
    (bfTsdfReintegrateFrame); voxels, block set and heap must equal the oracle's two separate passes bit for bit."""
    import torch
    W, H = 160, 120
    cam, hp = camera_params(W, H), small_params()
    gpu, cpu = CUDASceneRepHashSDF(hp, cuda_device, arithmetic="exact"), orc.OracleSceneRepHashSDF(hp)
    frames = [synth.make_frame(35 * i, W, H) for i in range(6)]
    dl = [torch.from_numpy(f[0]).to(cuda_device) for f in frames]
    cl = [torch.from_numpy(f[1]).to(cuda_device) for f in frames]
    gpu.runOps([(capi.BF_TSDF_OP_INTEGRATE, i, frames[i][2]) for i in range(6)], dl, cl, cam)
    for d, c, T in frames:
        cpu.integrate(T, d, c, cam)
    assert_same_state(gpu, cpu, hp)
    rng = np.random.default_rng(4)
    ops = []
    for k in (4, 2, 0, 5):
        T = frames[k][2]
        T2 = (synth.se3_exp(rng.standard_normal(3) * 0.01, rng.standard_normal(3) * 0.02) @ T.astype(np.float64)).astype(F)
        ops += [(capi.BF_TSDF_OP_DEINTEGRATE, k, T), (capi.BF_TSDF_OP_INTEGRATE, k, T2)]
        cpu.deIntegrate(T, frames[k][0], frames[k][1], cam)
        cpu.integrate(T2, frames[k][0], frames[k][1], cam)
    ops.append((capi.BF_TSDF_OP_GARBAGE_COLLECT, 0, None))
    gpu.runOps(ops, dl, cl, cam)
    cpu.garbageCollect()
    assert_same_state(gpu, cpu, hp, check_list=False)
    # a lone de-integration (no partner) still takes the single-pass route
    gpu.runOps([(capi.BF_TSDF_OP_DEINTEGRATE, 1, frames[1][2]), (capi.BF_TSDF_OP_GARBAGE_COLLECT, 0, None)], dl, cl, cam)
    cpu.deIntegrate(frames[1][2], frames[1][0], frames[1][1], cam)
    cpu.garbageCollect()
    assert_same_state(gpu, cpu, hp, check_list=False)


def degrade_depth(frames, seed=7):
    """In place, on 320x240 depth maps: a hole, a band beyond an integration distance of 2.5 m and salt noise of invalid pixels -- what
    the batch re-integration's depth-range cull keys on (blocks in front of / behind the surface, depths beyond the integration distance,
    invalid pixels, depth discontinuities)."""
    rng = np.random.default_rng(seed)
    for d, c, T in frames:
        H, W = d.shape
        d[60:90, 100:180] = -np.inf
        d[150:170, 20:300] = 3.4
        d[rng.integers(0, H, 300), rng.integers(0, W, 300)] = -np.inf


def test_degraded_depth_matches_oracle(cuda_device):
    """Integrations, two fused re-integrations and a lone de-integration of degraded depth maps (degrade_depth) are bit-identical to the
    oracle."""
    import torch
    W, H = 320, 240
    cam = camera_params(W, H)
    hp = small_params(num_buckets=100003, num_sdf_blocks=60000, max_integration_distance=2.5)
    frames = [list(synth.make_frame(40 * i, W, H)) for i in range(7)]
    degrade_depth(frames)
    gpu = CUDASceneRepHashSDF(hp, cuda_device, arithmetic="exact")
    for d, c, T in frames:
        dd, dc = to_dev(torch, cuda_device, d, c)
        gpu.integrate(T, dd, dc, cam)
    dl = [torch.from_numpy(f[0]).to(cuda_device) for f in frames]
    cl = [torch.from_numpy(f[1]).to(cuda_device) for f in frames]
    ops = []
    for k in (1, 5):
        T = frames[k][2]
        T2 = T.copy(); T2[:3, 3] += np.array([0.02, -0.01, 0.015], F)
        ops += [(capi.BF_TSDF_OP_DEINTEGRATE, k, T), (capi.BF_TSDF_OP_INTEGRATE, k, T2)]
    gpu.runOps(ops, dl, cl, cam)
    gpu.deIntegrate(frames[3][2], dl[3], cl[3], cam)
    b1, v1 = orc.canonical_blocks(gpu.download())
    cpu = orc.OracleSceneRepHashSDF(hp)
    for d, c, T in frames:
        cpu.integrate(T, d, c, cam)
    for k in (1, 5):
        T = frames[k][2]
        T2 = T.copy(); T2[:3, 3] += np.array([0.02, -0.01, 0.015], F)
        cpu.deIntegrate(T, frames[k][0], frames[k][1], cam); cpu.integrate(T2, frames[k][0], frames[k][1], cam)
    cpu.deIntegrate(frames[3][2], frames[3][0], frames[3][1], cam)
    cb, cv = orc.canonical_blocks(cpu.download())
    np.testing.assert_array_equal(b1, cb)
    np.testing.assert_array_equal(v1, cv)


def test_spatial_shard_matches_oracle_and_unsharded(cuda_device):
    """Multi-GPU shard (hp.m_dummy = {rank, world}), both ranks run one after the other on this GPU: each shard is bit-identical to
    the oracle's shard, the shards are disjoint and their union is the unsharded state (SURVEY.md section 8e; the world-size-2
    process-level version with the frame broadcast runs on CPU/gloo in tests/test_shard_gloo_cpu.py)."""
    import torch
    W, H = 160, 120
    cam = camera_params(W, H)
    frames = [synth.make_frame(35 * i, W, H) for i in range(4)]
    whole = orc.OracleSceneRepHashSDF(small_params())
    for d, c, T in frames:
        whole.integrate(T, d, c, cam)
    wb, wv = orc.canonical_blocks(whole.download())
    got_b, got_v = [], []
    for rank in range(2):
        hp = small_params(); hp.m_dummy = (2 << 32) | rank
        gpu, cpu = CUDASceneRepHashSDF(hp, cuda_device, arithmetic="exact"), orc.OracleSceneRepHashSDF(hp)
        for d, c, T in frames:
            dd, dc = to_dev(torch, cuda_device, d, c)
            gpu.integrate(T, dd, dc, cam); cpu.integrate(T, d, c, cam)
        assert_same_state(gpu, cpu, hp)
        b, v = orc.canonical_blocks(gpu.download())
        got_b.append(b); got_v.append(v)
    assert not (set(map(tuple, got_b[0])) & set(map(tuple, got_b[1])))
    mb, mv = np.concatenate(got_b), np.concatenate(got_v)
    order = np.lexsort((mb[:, 2], mb[:, 1], mb[:, 0]))
    np.testing.assert_array_equal(mb[order], wb)
    np.testing.assert_array_equal(mv[order], wv)

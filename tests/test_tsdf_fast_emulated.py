"""The tolerance-arithmetic TSDF stencil (bundlefusion_b200/csrc/tsdf_fast.cu) executed on the CPU -- the very same source, compiled by g++
against the shim of tests/cuda_emu with one CUDA thread run after the other (BF_EMU_SEQUENTIAL replaces the two warp reductions by plain
atomics and the approximate reciprocal by a division) -- on the oracle's own host-side voxel hash, against the oracle's stencil.  Checks the
kernel's LOGIC without a GPU: affine voxel -> camera chain, pixel / truncation decisions, word layout of the 4-voxel quads, integer colour
blend, de-integration rounding, the fused old-pose / new-pose pass, live-voxel and U counters.  TEST INFRASTRUCTURE around a product source;
the GPU statement is tests/test_tsdf_fast_gpu.py."""
import ctypes as C

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from bundlefusion_b200 import synth
from bundlefusion_b200.scene_rep import camera_params, default_hash_params, set_pose
from oracle import oracle as orc
from tests.cuda_emu import build_emulated

F = np.float32

# the glue of both stencil test files (this one and tests/test_tsdf_integrate_batch_emulated.py); emu_reintegrate_multi with hpOld NULL is
# the integration batch
_GLUE = r'''
extern "C" int emu_integrate_fast(const BFHashDataStruct* hd, const BFHashParams* hp, const BFDepthCameraParams* cp, const float* depth, const void* color,
                                  int deIntegrate, unsigned count, unsigned* ctrs, int* live, int grid) {
    return bf::launch_integrate_fast(hd, hp, cp, depth, color, deIntegrate != 0, false, count, ctrs, live, nullptr, bf::CTR_SET0, grid, nullptr);
}
extern "C" int emu_reintegrate_fast(const BFHashDataStruct* hd, const BFHashParams* hpOld, const BFHashParams* hpNew, const BFDepthCameraParams* cp, const float* depth,
                                    const void* color, const void* work, unsigned* ctrs, int* live, int grid) {
    return bf::launch_reintegrate_fast(hd, hpOld, hpNew, cp, depth, color, (const int4*)work, bf::CTR_SET0, ctrs, live, grid, nullptr);
}
extern "C" int emu_reintegrate_multi(const BFHashDataStruct* hd, const BFHashParams* hpOld, const BFHashParams* hpNew, int nOps, const BFDepthCameraParams* cp,
                                     const float* const* depth, const void* const* color, const void* workA, const void* workB, const unsigned* maskA, const unsigned* maskB, unsigned workCap, unsigned* ctrs, int* live, int grid) {
    bf::BFMultiOpDesc d[BF_MULTI_MAX_OPS];
    for (int k = 0; k < nOps; ++k) { d[k].hpOld = hpOld ? hpOld + k : nullptr; d[k].hpNew = hpNew + k; d[k].depth = depth[k]; d[k].color = color[k]; }
    return bf::launch_reintegrate_multi_fast(hd, d, nOps, cp, (const int4*)workA, (const int4*)workB, maskA, maskB, workCap, bf::CTR_SET0, ctrs, live, grid, nullptr);
}
'''


def fast_stencil():
    L = build_emulated("tsdf_fast.cu", 6, glue=_GLUE, sequential=True)
    vp = C.c_void_p
    L.emu_integrate_fast.argtypes = [vp, vp, vp, vp, vp, C.c_int, C.c_uint, vp, vp, C.c_int]
    L.emu_reintegrate_fast.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int]
    L.emu_reintegrate_multi.argtypes = [vp, vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, C.c_uint, vp, vp, C.c_int]
    return L


@pytest.fixture(scope="module")
def emu():
    return fast_stencil()


def _compare(a, b, sdf_tol):
    """the tolerance contract of tests/test_tsdf_vs_reference_gpu.compare_states, on two oracle-format snapshots"""
    ab, av = orc.canonical_blocks(a); bb, bv = orc.canonical_blocks(b)
    np.testing.assert_array_equal(ab, bb)
    aw, bw = av[..., 1].view(F), bv[..., 1].view(F)
    n = aw.size
    assert np.count_nonzero(aw != bw) <= max(2, 2e-5 * n)
    same = (aw == bw) & (bw > 0)
    dsdf = np.abs(av[..., 0].view(F)[same] - bv[..., 0].view(F)[same])
    flips = np.count_nonzero(dsdf > sdf_tol)
    assert flips <= max(3, 1e-4 * dsdf.size), (flips, dsdf.size, float(dsdf.max()))
    ac = av[..., 2].copy().view(np.uint8).reshape(av.shape[:-1] + (4,))[same].astype(np.int32)
    bc = bv[..., 2].copy().view(np.uint8).reshape(bv.shape[:-1] + (4,))[same].astype(np.int32)
    dc = np.abs(ac - bc).max(axis=-1)
    assert np.count_nonzero(dc > 1) <= max(3, 1e-4 * dsdf.size) + flips
    return {"touched": int(dsdf.size), "weight_mismatch": int(np.count_nonzero(aw != bw)), "flips": int(flips), "max_dsdf_nonflip": float(dsdf[dsdf <= sdf_tol].max(initial=0)),
            "colour_differs": int(np.count_nonzero(dc > 0))}


class _FastOnOracle:
    """oracle hash (alloc, compactify, GC on the host) with the emulated fast stencil doing the voxel updates"""

    def __init__(self, L, hp):
        self.L, self.o = L, orc.OracleSceneRepHashSDF(hp)
        self.ctrs = np.zeros(64, np.uint32)
        self.live = np.zeros(hp.m_numSDFBlocks, np.int32)

    def _stencil(self, T, depth, color, cam, de):
        o = self.o
        o._set_pose(T)
        depth = np.ascontiguousarray(depth, F)
        if not de:
            o.L.orc_tsdf_alloc(C.byref(o.hd), C.byref(o.hp), depth, C.byref(cam))
        o.num_occupied = o.L.orc_tsdf_compactify(C.byref(o.hd), C.byref(o.hp), C.byref(cam))
        self.ctrs[16:24] = 0
        rc = self.L.emu_integrate_fast(C.byref(o.hd), C.byref(o.hp), C.byref(cam), depth.ctypes.data, color.ctypes.data, 1 if de else 0, o.num_occupied,
                                       self.ctrs.ctypes.data, self.live.ctypes.data, 3)
        assert rc == 0
        return int(self.ctrs[20]) | (int(self.ctrs[21]) << 32)

    def integrate(self, T, d, c, cam): return self._stencil(T, d, c, cam, False)
    def deIntegrate(self, T, d, c, cam): return self._stencil(T, d, c, cam, True)


def test_fast_stencil_emulated_stream_matches_oracle(emu):
    W, H = 160, 120
    cam = camera_params(W, H)
    hp = default_hash_params(num_buckets=20011, num_sdf_blocks=30000)
    ref = orc.OracleSceneRepHashSDF(hp)
    fast = _FastOnOracle(emu, hp)
    frames = [synth.make_frame(35 * i, W, H) for i in range(4)]
    for d, c, T in frames:
        ref.integrate(T, d, c, cam)
        U = fast.integrate(T, d, np.ascontiguousarray(c), cam)
        assert abs(U - ref.last_U) <= max(4, 1e-4 * ref.last_U)
    s1 = _compare(fast.o.download(), ref.download(), 1e-5)
    # live-voxel counters = voxels with weight > 0 per slot
    v = fast.o.download()["voxels"]
    np.testing.assert_array_equal(fast.live, (v[..., 1].view(F) > 0).sum(axis=1).astype(np.int32))
    for k in (1, 3):
        d, c, T = frames[k]
        T2 = T.copy(); T2[:3, 3] += np.array([0.011, -0.006, 0.004], F)
        ref.deIntegrate(T, d, c, cam); ref.integrate(T2, d, c, cam)
        fast.deIntegrate(T, d, np.ascontiguousarray(c), cam); fast.integrate(T2, d, np.ascontiguousarray(c), cam)
    d, c, T = frames[0]
    ref.deIntegrate(T, d, c, cam); fast.deIntegrate(T, d, np.ascontiguousarray(c), cam)
    s2 = _compare(fast.o.download(), ref.download(), 1e-4)
    v = fast.o.download()["voxels"]
    np.testing.assert_array_equal(fast.live, (v[..., 1].view(F) > 0).sum(axis=1).astype(np.int32))
    ref.garbageCollect(); fast.o.garbageCollect()
    assert fast.o.getHeapFreeCount() == ref.getHeapFreeCount()
    print(s1, s2)


def test_fast_fused_reintegration_emulated_equals_its_two_passes(emu):
    """MODE 2 (old pose de-integrated, new pose integrated, one read-modify-write) against MODE 1 followed by MODE 0 of the same source: same
    probes, same decisions, so weights and colours are identical word for word; the sdf of a voxel both poses touch comes from the composed
    update (s w - sD + sI) / w instead of two divisions and may differ in the last bits."""
    W, H = 160, 120
    cam = camera_params(W, H)
    hp = default_hash_params(num_buckets=20011, num_sdf_blocks=30000)
    two, one = _FastOnOracle(emu, hp), _FastOnOracle(emu, hp)
    frames = [synth.make_frame(35 * i, W, H) for i in range(3)]
    for d, c, T in frames:
        two.integrate(T, d, np.ascontiguousarray(c), cam); one.integrate(T, d, np.ascontiguousarray(c), cam)
    d, c, T = frames[1]
    c = np.ascontiguousarray(c)
    T2 = (synth.se3_exp(np.array([0.004, -0.003, 0.002]), np.array([0.012, -0.007, 0.005])) @ T.astype(np.float64)).astype(F)
    two.deIntegrate(T, d, c, cam); U2 = two.integrate(T2, d, c, cam)
    # fused: alloc at the new pose, then a union work list {block, slot | flags} (bit 0: in the old pose's frustum list, bit 1: in the new one's)
    o = one.o
    hpOld = capi.BFHashParams(); C.memmove(C.byref(hpOld), C.byref(o.hp), C.sizeof(capi.BFHashParams)); set_pose(hpOld, T)
    o._set_pose(T2)
    depth = np.ascontiguousarray(d, F)
    o.L.orc_tsdf_alloc(C.byref(o.hd), C.byref(o.hp), depth, C.byref(cam))
    nOld = o.L.orc_tsdf_compactify(C.byref(o.hd), C.byref(hpOld), C.byref(cam)); inOld = {int(p) for p in o.compactified.reshape(-1, 8)[:nOld, 3]}
    nNew = o.L.orc_tsdf_compactify(C.byref(o.hd), C.byref(o.hp), C.byref(cam)); inNew = {int(p) for p in o.compactified.reshape(-1, 8)[:nNew, 3]}
    h = o.hash
    used = np.array([i for i in np.nonzero(h[:, 3] != -2)[0] if int(h[i, 3]) in inOld or int(h[i, 3]) in inNew])
    work = np.zeros((len(used), 4), np.int32)
    work[:, :3] = h[used, :3]
    work[:, 3] = [(int(h[i, 3]) // 512) | ((1 if int(h[i, 3]) in inOld else 0) << 28) | ((2 if int(h[i, 3]) in inNew else 0) << 28) for i in used]
    one.ctrs[16:24] = 0; one.ctrs[16] = len(used); one.ctrs[17] = len(used)
    rc = emu.emu_reintegrate_fast(C.byref(o.hd), C.byref(hpOld), C.byref(o.hp), C.byref(cam), depth.ctypes.data, c.ctypes.data, work.ctypes.data,
                                  one.ctrs.ctypes.data, one.live.ctypes.data, 5)
    assert rc == 0
    ab, av = orc.canonical_blocks(one.o.download()); bb, bv = orc.canonical_blocks(two.o.download())
    np.testing.assert_array_equal(ab, bb)
    np.testing.assert_array_equal(av[..., 1], bv[..., 1])                     # weights
    np.testing.assert_array_equal(av[..., 2], bv[..., 2])                     # colours
    assert np.abs(av[..., 0].view(F) - bv[..., 0].view(F)).max() < 2e-7
    np.testing.assert_array_equal(one.live, two.live)


def _frustum_slots(o, hp_pose, cam):
    """hash-entry ptr values of the blocks in the frustum list of a pose (the oracle's compactify)"""
    n = o.L.orc_tsdf_compactify(C.byref(o.hd), C.byref(hp_pose), C.byref(cam))
    return {int(p) for p in o.compactified.reshape(-1, 8)[:n, 3]}


def test_batch_stencil_emulated_equals_pair_by_pair(emu):
    """stencil_multi_kernel (all pairs of a batch applied per voxel in registers, one read / write) against the pair-by-pair fused passes of
    the same source, word for word -- including the rule that a block inserted by pair k's alloc is invisible to the pairs before k."""
    W, H = 160, 120
    cam = camera_params(W, H)
    hp = default_hash_params(num_buckets=20011, num_sdf_blocks=30000)
    seq, bat = _FastOnOracle(emu, hp), _FastOnOracle(emu, hp)
    frames = [synth.make_frame(35 * i, W, H) for i in range(4)]
    for d, c, T in frames[:3]:
        seq.integrate(T, d, np.ascontiguousarray(c), cam); bat.integrate(T, d, np.ascontiguousarray(c), cam)
    # three pairs; the third re-integrates a frame towards a region nobody has looked at yet (frame 3's pose), so that its alloc inserts new blocks
    moves = [(1, synth.se3_exp(np.array([0.004, -0.003, 0.002]), np.array([0.012, -0.007, 0.005]))),
             (0, synth.se3_exp(np.array([-0.002, 0.005, 0.001]), np.array([-0.01, 0.004, 0.008]))),
             (2, None)]
    pairs = []
    for f, M in moves:
        d, c, T = frames[f]
        T2 = frames[3][2] if M is None else (M @ T.astype(np.float64)).astype(F)
        pairs.append((np.ascontiguousarray(d, F), np.ascontiguousarray(c), T, T2))

    def hp_at(o, T):
        q = capi.BFHashParams(); C.memmove(C.byref(q), C.byref(o.hp), C.sizeof(capi.BFHashParams)); set_pose(q, T); return q

    def used_slots(o):
        h = o.hash
        return {int(p) for p in h[h[:, 3] != -2, 3]}

    def work_list(o, masks):                      # masks: {ptr: mask}
        h = o.hash
        rows = [i for i in np.nonzero(h[:, 3] != -2)[0] if masks.get(int(h[i, 3]), 0)]
        work = np.zeros((len(rows), 4), np.int32); wm = np.zeros(len(rows), np.uint32)
        for n, i in enumerate(rows):
            work[n, :3] = h[i, :3]; work[n, 3] = int(h[i, 3]) // 512; wm[n] = masks[int(h[i, 3])]
        return work, wm

    # pair by pair (what bfTsdfReintegrateFrame does): alloc(new), union list with per-pose flags, fused pass
    u_seq = 0
    for d, c, T, T2 in pairs:
        o = seq.o
        hpO, hpN = hp_at(o, T), hp_at(o, T2)
        o._set_pose(T2); o.L.orc_tsdf_alloc(C.byref(o.hd), C.byref(o.hp), d, C.byref(cam))
        inO, inN = _frustum_slots(o, hpO, cam), _frustum_slots(o, hpN, cam)
        work, wm = work_list(o, {p: (1 if p in inO else 0) | (2 if p in inN else 0) for p in inO | inN})
        work[:, 3] |= (wm.astype(np.int32) << 28)
        seq.ctrs[16:24] = 0; seq.ctrs[16] = seq.ctrs[17] = len(work)
        assert emu.emu_reintegrate_fast(C.byref(o.hd), C.byref(hpO), C.byref(hpN), C.byref(cam), d.ctypes.data, c.ctypes.data, work.ctypes.data, seq.ctrs.ctypes.data, seq.live.ctypes.data, 4) == 0
        u_seq += int(seq.ctrs[20])
    # batch: all allocs first (remember which alloc inserted which block), one union list with 2 bits per pair, one pass
    o = bat.o
    epoch = {}
    for k, (d, c, T, T2) in enumerate(pairs):
        before = used_slots(o)
        o._set_pose(T2); o.L.orc_tsdf_alloc(C.byref(o.hd), C.byref(o.hp), d, C.byref(cam))
        for p in used_slots(o) - before:
            epoch[p] = k
    assert any(v == 2 for v in epoch.values()), "the third pair is meant to insert new blocks"
    masks = {}
    hpOs = (capi.BFHashParams * 3)(); hpNs = (capi.BFHashParams * 3)()
    for k, (d, c, T, T2) in enumerate(pairs):
        hpOs[k], hpNs[k] = hp_at(o, T), hp_at(o, T2)
        inO, inN = _frustum_slots(o, hpOs[k], cam), _frustum_slots(o, hpNs[k], cam)
        for p in inO | inN:
            if epoch.get(p, 0) <= k:
                masks[p] = masks.get(p, 0) | ((1 if p in inO else 0) | (2 if p in inN else 0)) << (2 * k)
    work, wm = work_list(o, masks)
    # the layout compactify_multi_kernel produces: four cost buckets (quartiles of the 2 x 3 = 6 possible probes) in two capacity-sized arrays
    cap = len(work) + 7
    bits = np.array([bin(int(m)).count("1") for m in wm])
    q = np.where(4 * bits > 3 * 6, 3, np.where(2 * bits > 6, 2, np.where(4 * bits > 6, 1, 0)))
    WA, WB, MA, MB = np.zeros((cap, 4), np.int32), np.zeros((cap, 4), np.int32), np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
    n = [int((q == k).sum()) for k in range(4)]
    WA[:n[3]], MA[:n[3]] = work[q == 3], wm[q == 3]
    if n[2]: WA[cap - n[2]:], MA[cap - n[2]:] = work[q == 2][::-1], wm[q == 2][::-1]
    WB[:n[1]], MB[:n[1]] = work[q == 1], wm[q == 1]
    if n[0]: WB[cap - n[0]:], MB[cap - n[0]:] = work[q == 0][::-1], wm[q == 0][::-1]
    assert sum(1 for k in n if k > 0) >= 3, n
    dptr = (C.c_void_p * 3)(*[p[0].ctypes.data for p in pairs]); cptr = (C.c_void_p * 3)(*[p[1].ctypes.data for p in pairs])
    bat.ctrs[16:24] = 0; bat.ctrs[16] = len(work); bat.ctrs[17] = n[3]; bat.ctrs[18] = n[2]; bat.ctrs[22] = n[1]; bat.ctrs[23] = n[0]
    assert emu.emu_reintegrate_multi(C.byref(o.hd), C.addressof(hpOs), C.addressof(hpNs), 3, C.byref(cam), C.addressof(dptr), C.addressof(cptr), WA.ctypes.data, WB.ctypes.data,
                                     MA.ctypes.data, MB.ctypes.data, cap, bat.ctrs.ctypes.data, bat.live.ctypes.data, 5) == 0
    ab, av = orc.canonical_blocks(bat.o.download()); bb, bv = orc.canonical_blocks(seq.o.download())
    np.testing.assert_array_equal(ab, bb)
    np.testing.assert_array_equal(av, bv)
    np.testing.assert_array_equal(bat.live, seq.live)
    assert int(bat.ctrs[20]) == u_seq                            # U of the batch = sum of the pairs' U

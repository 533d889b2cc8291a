"""The integration-only batch pass (bfTsdfIntegrateBatch: stencil_multi_kernel<false> of bundlefusion_b200/csrc/tsdf_fast.cu) executed on the
CPU -- the same source compiled by g++ against tests/cuda_emu, one CUDA thread after the other, as tests/test_tsdf_fast_emulated.py runs it --
on the oracle's host-side voxel hash, against the one-frame fast stencil applied frame by frame: every voxel word, the live-voxel counters and
U must be identical.  Also the refusals of bfTsdfIntegrateBatch / bfFrameLoopFuse, which return before any CUDA call."""
import ctypes as C

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from bundlefusion_b200 import synth
from bundlefusion_b200.scene_rep import camera_params, default_hash_params, set_pose
from oracle import oracle as orc
from tests.cuda_emu import run_without_device
from tests.test_tsdf_fast_emulated import fast_stencil

F = np.float32
W, H = 160, 120


@pytest.fixture(scope="module")
def emu():
    return fast_stencil()


class _Scene:
    """oracle hash (alloc, compactify on the host) with the emulated fast stencils doing the voxel updates"""

    def __init__(self, L, hp, cam):
        self.L, self.o, self.cam = L, orc.OracleSceneRepHashSDF(hp), cam
        self.ctrs = np.zeros(64, np.uint32)
        self.live = np.zeros(hp.m_numSDFBlocks, np.int32)

    def hp_at(self, T):
        q = capi.BFHashParams(); C.memmove(C.byref(q), C.byref(self.o.hp), C.sizeof(capi.BFHashParams)); set_pose(q, T); return q

    def used_slots(self):
        h = self.o.hash
        return {int(p) for p in h[h[:, 3] != -2, 3]}

    def frustum_slots(self, hp):
        o = self.o
        n = o.L.orc_tsdf_compactify(C.byref(o.hd), C.byref(hp), C.byref(self.cam))
        return {int(p) for p in o.compactified.reshape(-1, 8)[:n, 3]}

    def integrate(self, d, c, T):
        """bfTsdfIntegrateFrame in fast arithmetic: alloc, compactify, the one-frame stencil (MODE 0)"""
        o = self.o
        o._set_pose(T)
        o.L.orc_tsdf_alloc(C.byref(o.hd), C.byref(o.hp), d, C.byref(self.cam))
        n = o.L.orc_tsdf_compactify(C.byref(o.hd), C.byref(o.hp), C.byref(self.cam))
        self.ctrs[16:24] = 0
        assert self.L.emu_integrate_fast(C.byref(o.hd), C.byref(o.hp), C.byref(self.cam), d.ctypes.data, c.ctypes.data, 0, n, self.ctrs.ctypes.data,
                                         self.live.ctypes.data, 3) == 0
        return int(self.ctrs[20]) | (int(self.ctrs[21]) << 32)

    def integrate_batch(self, frames):
        """bfTsdfIntegrateBatch: every alloc first (each remembers the blocks it inserted), one union list with mask bit 1 of op k set where
        frame k's frustum holds a block that existed for it, the multi-op stencil with no old pose"""
        o, n = self.o, len(frames)
        epoch = {}
        for k, (d, c, T) in enumerate(frames):
            before = self.used_slots()
            o._set_pose(T); o.L.orc_tsdf_alloc(C.byref(o.hd), C.byref(o.hp), d, C.byref(self.cam))
            for p in self.used_slots() - before:
                epoch[p] = k
        hps = (capi.BFHashParams * n)()
        masks = {}
        for k, (d, c, T) in enumerate(frames):
            hps[k] = self.hp_at(T)
            for p in self.frustum_slots(hps[k]):
                if epoch.get(p, 0) <= k:
                    masks[p] = masks.get(p, 0) | (2 << (2 * k))
        h = o.hash
        rows = [i for i in np.nonzero(h[:, 3] != -2)[0] if masks.get(int(h[i, 3]), 0)]
        cap = len(rows) + 5
        WA, WB, MA, MB = np.zeros((cap, 4), np.int32), np.zeros((cap, 4), np.int32), np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
        # one item in each of the lower three cost buckets (see compactify_multi_kernel), the rest in the costliest: the stencil deals all four
        lay = {3: [], 2: [], 1: [], 0: []}
        for j, i in enumerate(rows):
            lay[j if j < 3 else 3].append(i)
        def put(arr, marr, idx, i):
            arr[idx, :3] = h[i, :3]; arr[idx, 3] = int(h[i, 3]) // 512; marr[idx] = masks[int(h[i, 3])]
        for j, i in enumerate(lay[3]): put(WA, MA, j, i)
        for j, i in enumerate(lay[2]): put(WA, MA, cap - 1 - j, i)
        for j, i in enumerate(lay[1]): put(WB, MB, j, i)
        for j, i in enumerate(lay[0]): put(WB, MB, cap - 1 - j, i)
        dptr = (C.c_void_p * n)(*[f[0].ctypes.data for f in frames]); cptr = (C.c_void_p * n)(*[f[1].ctypes.data for f in frames])
        self.ctrs[16:24] = 0
        self.ctrs[16] = len(rows); self.ctrs[17] = len(lay[3]); self.ctrs[18] = len(lay[2]); self.ctrs[22] = len(lay[1]); self.ctrs[23] = len(lay[0])
        assert self.L.emu_reintegrate_multi(C.byref(o.hd), None, C.addressof(hps), n, C.byref(self.cam), C.addressof(dptr), C.addressof(cptr), WA.ctypes.data,
                                            WB.ctypes.data, MA.ctypes.data, MB.ctypes.data, cap, self.ctrs.ctypes.data, self.live.ctypes.data, 5) == 0
        return int(self.ctrs[20]) | (int(self.ctrs[21]) << 32), epoch


def _frame(i):
    d, c, T = synth.make_frame(i, W, H)
    return np.ascontiguousarray(d, F), np.ascontiguousarray(c), T


@pytest.mark.parametrize("n", [1, 2, 5, 16])
def test_integration_batch_emulated_equals_frame_by_frame(emu, n):
    cam = camera_params(W, H)
    hp = default_hash_params(num_buckets=20011, num_sdf_blocks=30000)
    seq, bat = _Scene(emu, hp, cam), _Scene(emu, hp, cam)
    for i in (0, 40):                                              # the seeded scene both start from
        d, c, T = _frame(i)
        seq.integrate(d, c, T); bat.integrate(d, c, T)
    # overlapping frustums 9 frames apart; the last frame looks at a region nobody has seen (its blocks are first inserted by it); with
    # n >= 5 one frame has no valid depth at all
    frames = [_frame(60 + 9 * k) for k in range(n - 1)] + [_frame(400)]
    if n >= 5:
        d, c, T = frames[2]
        frames[2] = (np.full_like(d, -np.inf), c, T)
    u_seq = sum(seq.integrate(d, c, T) for d, c, T in frames)
    u_bat, epoch = bat.integrate_batch(frames)
    assert any(v == n - 1 for v in epoch.values()), "the last frame is meant to insert blocks of its own"
    ab, av = orc.canonical_blocks(bat.o.download()); bb, bv = orc.canonical_blocks(seq.o.download())
    np.testing.assert_array_equal(ab, bb)
    np.testing.assert_array_equal(av, bv)                          # every sdf, weight and colour word
    np.testing.assert_array_equal(bat.live, seq.live)
    assert u_bat == u_seq
    assert bat.o.getHeapFreeCount() == seq.o.getHeapFreeCount()


_REFUSALS = r'''
import ctypes as C, json, sys
sys.path.insert(0, sys.argv[1])
from bundlefusion_b200 import _capi as capi
from bundlefusion_b200.scene_rep import camera_params, default_hash_params
L = capi.lib()
hd, hp, cam = capi.BFHashDataStruct(), default_hash_params(num_buckets=101, num_sdf_blocks=64), camera_params(64, 48)
fake = (C.c_void_p * 4)(0x1000, 0x2000, None, 0x4000)          # never dereferenced on the device: every case is refused first
frames = (C.c_int32 * 17)(*([0, 1] + [3] * 15))
poses = (C.c_float * (17 * 16))()
B = lambda fr, po, n, d, c: L.bfTsdfIntegrateBatch(C.byref(hd), C.byref(hp), C.byref(cam), fr, po, n, d, c)
vp = lambda x: C.cast(x, C.c_void_p)
bad_frame = (C.c_int32 * 3)(0, 2, 1)
neg_frame = (C.c_int32 * 2)(0, -1)
out = {
    "n0": B(vp(frames), vp(poses), 0, vp(fake), vp(fake)),
    "n17": B(vp(frames), vp(poses), 17, vp(fake), vp(fake)),
    "null_frames": B(None, vp(poses), 2, vp(fake), vp(fake)),
    "null_poses": B(vp(frames), None, 2, vp(fake), vp(fake)),
    "null_depth_array": B(vp(frames), vp(poses), 2, None, vp(fake)),
    "null_color_array": B(vp(frames), vp(poses), 2, vp(fake), None),
    "frame_ptr_null": B(vp(bad_frame), vp(poses), 3, vp(fake), vp(fake)),
    "negative_frame": B(vp(neg_frame), vp(poses), 2, vp(fake), vp(fake)),
    "fuse_null_loop": L.bfFrameLoopFuse(None, C.byref(hd), C.byref(hp), None, 0, None),
}
print(json.dumps(out))
'''


def test_integration_batch_refusals_enqueue_nothing():
    """each malformed call returns cudaErrorInvalidValue (1) before any CUDA call: run in a child process that sees no CUDA device, where a call
    that went on to the runtime would fail with another code (or touch the fake pointers)"""
    out = run_without_device(_REFUSALS)
    assert out == {k: 1 for k in out}, out

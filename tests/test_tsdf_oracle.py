"""Known-answer tests that pin oracle/tsdf_oracle.c (CPU only).

The reference ships no golden vectors for this path ("parity unpinned", SURVEY.md section 4), so
the oracle is pinned by (1) closed-form cases whose answer follows from the reference's formulae
(CUDASceneRepHashSDF.cu:420-521, VoxelUtilHashSDF.h:226-299) and (2) an independent vectorised
numpy float32 restatement of the per-voxel rule that must agree bit-for-bit.
"""
import ctypes as C

import numpy as np
import pytest

from bundlefusion_b200 import synth
from bundlefusion_b200._capi import BF_SDF_BLOCK_VOXELS
from bundlefusion_b200.scene_rep import camera_params, default_hash_params, mat4_inverse_f32
from oracle import oracle as orc

F = np.float32


def small_params(**kw):
    kw.setdefault("num_buckets", 20011)
    kw.setdefault("num_sdf_blocks", 30000)
    return default_hash_params(**kw)


def fma32(a, b, c):
    """fmaf(a, b, c) on float32 arrays: the product of two binary32 values is exact in binary64; the one binary64 addition is
    then rounded to binary32 (double rounding can differ from a true FMA only when the binary64 sum lands within 2^-29 relative
    of a binary32 rounding boundary -- not on these seeds)."""
    D = np.float64
    return (np.asarray(a, F).astype(D) * np.asarray(b, F).astype(D) + np.asarray(c, F).astype(D)).astype(F)


def numpy_expected_voxels(blocks, T, depth, color, cam, hp, old=None, deintegrate=False):
    """Vectorised float32 restatement of integrateDepthMapKernel for a list of block coords.
    Returns (sdf, weight, rgba, passed-mask) arrays of shape (N,512[,4])."""
    N = len(blocks)
    i = np.arange(BF_SDF_BLOCK_VOXELS)
    lx, ly, lz = i % 8, (i % 64) // 8, i // 64
    vx = (blocks[:, 0:1] * 8 + lx[None, :]).astype(F) * F(hp.m_virtualVoxelSize)
    vy = (blocks[:, 1:2] * 8 + ly[None, :]).astype(F) * F(hp.m_virtualVoxelSize)
    vz = (blocks[:, 2:3] * 8 + lz[None, :]).astype(F) * F(hp.m_virtualVoxelSize)
    M = mat4_inverse_f32(T)

    def row(r):       # the contract's fused form of m0*x + m1*y + m2*z + m3 (oracle/tsdf_oracle.c header)
        return fma32(vz, M[r, 2], fma32(vx, M[r, 0], vy * M[r, 1])) + M[r, 3]
    px, py, pz = row(0), row(1), row(2)
    with np.errstate(all="ignore"):
        sx = px * F(cam.fx) / pz + F(cam.mx)
        sy = py * F(cam.fy) / pz + F(cam.my)
        ix = np.trunc(sx + F(0.5)).astype(np.int64)
        iy = np.trunc(sy + F(0.5)).astype(np.int64)
    W, H = cam.m_imageWidth, cam.m_imageHeight
    on = (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
    ixc, iyc = np.clip(ix, 0, W - 1), np.clip(iy, 0, H - 1)
    d = depth[iyc, ixc]
    c = color[iyc, ixc].astype(F)
    with np.errstate(all="ignore"):
        ok = on & (d != -np.inf) & (d < F(hp.m_maxIntegrationDistance))
        sdf = d - pz
        trunc = fma32(F(hp.m_truncScale), d, F(hp.m_truncation))
        ok &= np.abs(sdf) < trunc
        sdf = np.where(sdf >= 0, np.minimum(trunc, sdf), np.maximum(-trunc, sdf)).astype(F)
    if old is None:
        old_sdf = np.zeros((N, 512), F); old_w = np.zeros((N, 512), F); old_c = np.zeros((N, 512, 4), F)
    else:
        old_sdf, old_w, old_c = old
    with np.errstate(all="ignore"):
        if not deintegrate:
            n_sdf = fma32(old_sdf, old_w, sdf) / (F(1) + old_w)
            n_w = np.minimum(F(hp.m_integrationWeightMax), F(1) + old_w)
            blend = fma32(c[..., :3], F(0.2), F(0.8) * old_c[..., :3])
            res = np.where((old_w == 0)[..., None], c[..., :3], blend)
        else:
            n_sdf = fma32(old_sdf, old_w, -sdf) / (old_w - F(1))
            n_w = np.maximum(F(0), old_w - F(1))
            res = fma32(old_c[..., :3], old_w[..., None], -c[..., :3]) / (old_w - F(1))[..., None]
        r = np.where(res >= 0, np.floor(res + F(0.5)), np.ceil(res - F(0.5)))        # roundf: half away from zero
        r = np.maximum(F(0), np.fmin(r, F(254.5)))
        rgba = np.concatenate([np.trunc(np.nan_to_num(r)).astype(np.uint8), np.full((N, 512, 1), 255, np.uint8)], -1)
    if deintegrate:
        dead = n_w <= F(0.001)
        n_sdf = np.where(dead, F(0), n_sdf); n_w = np.where(dead, F(0), n_w); rgba = np.where(dead[..., None], 0, rgba)
    return n_sdf.astype(F), n_w.astype(F), rgba.astype(np.uint8), ok


def unpack(vox_words):
    sdf = vox_words[..., 0].view(F)
    w = vox_words[..., 1].view(F)
    rgba = vox_words[..., 2].copy().view(np.uint8).reshape(vox_words.shape[:-1] + (4,))
    return sdf, w, rgba


def test_hash_function_known_values(oracle_lib):
    # ((x*73856093) ^ (y*19349669) ^ (z*83492791)) mod numBuckets with 32-bit wraparound and an UNSIGNED modulo
    hp = small_params(num_buckets=800000, num_sdf_blocks=64)
    o = orc.OracleSceneRepHashSDF(hp)
    cases = [(0, 0, 0), (1, 2, 3), (-1, -2, -3), (100, -50, 25), (-12345, 6789, -1011)]
    for (x, y, z) in cases:
        v = ((x * 73856093) & 0xFFFFFFFF) ^ ((y * 19349669) & 0xFFFFFFFF) ^ ((z * 83492791) & 0xFFFFFFFF)
        expect_bucket = v % 800000
        # insert by faking a depth pixel is heavy; instead place the entry by hand and let find() hash to it
        idx = expect_bucket * 4
        o.hash[idx, :5] = (x, y, z, 512 * 7, 0)
        assert oracle_lib.orc_tsdf_find(C.byref(o.hd), C.byref(o.hp), x, y, z) == idx
        o.hash[idx, :5] = (0, 0, 0, -2, 0)
        assert oracle_lib.orc_tsdf_find(C.byref(o.hd), C.byref(o.hp), x, y, z) == -1


def test_plane_wall_closed_form(oracle_lib):
    """Fronto-parallel wall at z0, identity pose: every voxel whose centre projects on screen and lies
    within trunc(z0) = 0.06 + 0.02*z0 of the wall gets sdf = clamp(z0 - z), weight 1, the wall colour."""
    W, H, z0 = 160, 120, 1.0
    cam = camera_params(W, H)
    hp = small_params()
    depth, color = synth.plane_frame(W, H, z0, (128, 64, 32))
    o = orc.OracleSceneRepHashSDF(hp)
    o.integrate(np.eye(4, dtype=F), depth, color, cam)
    assert o.num_occupied > 0 and o.last_U > 0
    orc.check_hash_invariants(o.download(), hp)
    blocks, vox = orc.canonical_blocks(o.download())
    sdf, w, rgba = unpack(vox)
    i = np.arange(512)
    zc = (blocks[:, 2:3] * 8 + (i // 64)[None, :]).astype(F) * F(0.01)
    trunc = F(0.06) + F(0.02) * F(z0)
    touched = w > 0
    assert touched.sum() == o.last_U
    np.testing.assert_array_equal(w[touched], 1.0)
    np.testing.assert_array_equal(sdf[touched], (F(z0) - zc)[touched])
    assert np.all(np.abs(sdf[touched]) < trunc)
    assert np.all(rgba[touched] == np.array([128, 64, 32, 255], np.uint8))
    # untouched voxels are exactly zero
    assert np.all(vox[~touched] == 0)
    # the band is complete along z for a voxel column through the image centre
    centre = touched & (np.abs((blocks[:, 0:1] * 8 + (i % 8)[None, :])) <= 1) & (np.abs((blocks[:, 1:2] * 8 + ((i % 64) // 8)[None, :])) <= 1)
    zs = np.unique(zc[centre])
    # strict interior of the band must be complete; the two voxels AT |sdf| == trunc fall either way in float32
    got = set(np.round(zs * 100).astype(int).tolist())
    lo, hi = int(round((z0 - float(trunc)) * 100)), int(round((z0 + float(trunc)) * 100))
    assert set(range(lo + 1, hi)) <= got <= set(range(lo, hi + 1))


@pytest.mark.parametrize("frame_idx", [0, 37])
def test_room_frame_matches_numpy_restatement(oracle_lib, frame_idx):
    W, H = 160, 120
    cam = camera_params(W, H)
    hp = small_params()
    depth, color, T = synth.make_frame(frame_idx, W, H)
    o = orc.OracleSceneRepHashSDF(hp)
    o.integrate(T, depth, color, cam)
    snap = o.download()
    orc.check_hash_invariants(snap, hp)
    blocks, vox = orc.canonical_blocks(snap)
    assert len(blocks) > 100
    # all blocks were allocated by this one frame and are in the frustum list or not; compute expectation for all,
    # apply it only where the block is in the compactified (in-frustum) list
    comp = snap["compactified"][: snap["compactified_count"], :3]
    in_list = np.array([tuple(b) in set(map(tuple, comp)) for b in blocks])
    e_sdf, e_w, e_rgba, ok = numpy_expected_voxels(blocks, T, depth, color, cam, hp)
    ok &= in_list[:, None]
    sdf, w, rgba = unpack(vox)
    np.testing.assert_array_equal(w > 0, ok)
    np.testing.assert_array_equal(sdf[ok].view(np.uint32), e_sdf[ok].view(np.uint32))   # bit-exact
    np.testing.assert_array_equal(rgba[ok], e_rgba[ok])
    assert int(ok.sum()) == o.last_U


def test_integrate_deintegrate_roundtrip_and_gc(oracle_lib):
    """integrate -> de-integrate with the same frame and pose returns every voxel to zero (weight 1 -> 0 clears the
    voxel, .cu:509-513); garbage collection then frees every in-frustum block and the heap is full again."""
    W, H = 160, 120
    cam = camera_params(W, H)
    hp = small_params()
    depth, color, T = synth.make_frame(11, W, H)
    o = orc.OracleSceneRepHashSDF(hp)
    free0 = o.getHeapFreeCount()
    assert free0 == hp.m_numSDFBlocks
    o.integrate(T, depth, color, cam)
    n_alloc = free0 - o.getHeapFreeCount()
    assert n_alloc > 0
    o.deIntegrate(T, depth, color, cam)
    assert np.all(o.voxels == 0)
    freed = o.garbageCollect()
    assert freed == o.num_occupied
    orc.check_hash_invariants(o.download(), hp)
    # blocks allocated outside the 0.95-shrunk frustum list are not visited by GC; the rest are gone
    assert o.getHeapFreeCount() == free0 - (n_alloc - freed)


def test_two_frames_running_average(oracle_lib):
    """Second observation of the same wall from the same pose: sdf stays, weight 2, colour blends 0.2/0.8 and rounds."""
    W, H = 80, 60
    cam = camera_params(W, H)
    hp = small_params()
    o = orc.OracleSceneRepHashSDF(hp)
    d1, c1 = synth.plane_frame(W, H, 1.5, (200, 100, 50))
    d2, c2 = synth.plane_frame(W, H, 1.5, (100, 200, 251))
    I = np.eye(4, dtype=F)
    o.integrate(I, d1, c1, cam)
    _, vox1 = orc.canonical_blocks(o.download())
    o.integrate(I, d2, c2, cam)
    blocks, vox2 = orc.canonical_blocks(o.download())
    s1, w1, _ = unpack(vox1)
    s2, w2, rgba2 = unpack(vox2)
    t = w2 > 0
    np.testing.assert_array_equal(w2[t], 2.0)
    np.testing.assert_allclose(s2[t], s1[t], rtol=0, atol=1e-7)
    # 0.2*cur + 0.8*old, rounded, clamped to 254.5 then truncated
    exp = np.array([round(0.2 * 100 + 0.8 * 200), round(0.2 * 200 + 0.8 * 100), min(254, round(0.2 * 251 + 0.8 * 50)), 255], np.uint8)
    assert np.all(rgba2[t] == exp)


def test_overflow_lists_and_negative_coordinates(oracle_lib):
    """Tiny bucket count forces the linked-list path (VoxelUtilHashSDF.h:614-654); the camera looks down -z so block
    coordinates are negative (floor division, :290-299).  Invariants must hold and every block stay findable."""
    W, H = 80, 60
    cam = camera_params(W, H)
    hp = small_params(num_buckets=257, num_sdf_blocks=4000)
    T = np.eye(4, dtype=F)
    T[:3, :3] = np.array([[-1, 0, 0], [0, 1, 0], [0, 0, -1]], F)     # rotate pi about y
    T[:3, 3] = [-0.33, -0.21, -0.17]
    depth, color = synth.plane_frame(W, H, 1.2)
    o = orc.OracleSceneRepHashSDF(hp)
    o.integrate(T, depth, color, cam)
    snap = o.download()
    orc.check_hash_invariants(snap, hp)
    blocks, _ = orc.canonical_blocks(snap)
    assert blocks[:, 2].max() < 0
    used = snap["hash"][:, 3] != -2
    assert np.any(snap["hash"][used, 4] != 0), "expected at least one overflow chain"
    for b in blocks[:: max(1, len(blocks) // 200)]:
        assert oracle_lib.orc_tsdf_find(C.byref(o.hd), C.byref(o.hp), int(b[0]), int(b[1]), int(b[2])) >= 0


def test_dense_grid_config0(oracle_lib):
    """BASELINE.json configs[0]: one 640x480 depth frame into a dense 64^3 grid (4 cm voxels, centred 2 m ahead)."""
    W, H = 640, 480
    cam = camera_params(W, H)
    hp = small_params(voxel_size=0.04)
    depth, color = synth.plane_frame(W, H, 2.0)
    grid = np.zeros((64, 64, 64, 3), np.int32)
    origin = (C.c_float * 3)(-1.28, -1.28, 2.0 - 1.28)
    U = oracle_lib.orc_tsdf_integrate_dense(grid.ctypes.data, 64, 0.04, origin, C.byref(hp), depth, color.ctypes.data, C.byref(cam), 0)
    sdf, w, _ = unpack(grid.reshape(-1, 3))
    assert U == int((w > 0).sum()) and U > 0
    z = (np.arange(64 ** 3) // (64 * 64)).astype(F) * F(0.04) + F(2.0 - 1.28)
    t = w > 0
    np.testing.assert_allclose(sdf[t], 2.0 - z[t], atol=2e-6)
    assert np.all(np.abs(sdf[t]) < 0.06 + 0.02 * 2.0)


@pytest.mark.parametrize("frame_idx", [100, 200])
def test_allocation_history_widens_the_integrated_voxel_set(oracle_lib, frame_idx):
    """integrate(P1), deIntegrate(P1), integrate(P2) is not integrate(P2) on a fresh hash: de-integration clears P1's voxels but not its blocks
    (GC frees a block only once it is visited with no weight left), and integration fills every allocated block in the frustum, not only the
    blocks P2's rays allocate.  So the history holds weight in voxels the fresh hash does not have -- every one of them in a block the fresh
    hash never allocated -- while every block both allocated holds the same voxel words.  This is why a re-integrated model differs from a
    fresh fusion of its final poses."""
    W, H = 160, 120
    cam = camera_params(W, H)
    hp = small_params()
    depth, color, P1 = synth.make_frame(frame_idx, W, H)
    P2 = (synth.se3_exp(np.array([0.01, -0.02, 0.015]), np.array([0.03, -0.02, 0.04])) @ P1.astype(np.float64)).astype(F)
    P2[3] = [0, 0, 0, 1]
    hist, fresh = orc.OracleSceneRepHashSDF(hp), orc.OracleSceneRepHashSDF(hp)
    hist.integrate(P1, depth, color, cam)
    hist.deIntegrate(P1, depth, color, cam)
    assert np.all(hist.voxels == 0)
    hist.integrate(P2, depth, color, cam)
    fresh.integrate(P2, depth, color, cam)
    hb, hv = orc.canonical_blocks(hist.download())
    fb, fv = orc.canonical_blocks(fresh.download())
    key = lambda b: [tuple(x) for x in b]
    fset = set(key(fb))
    in_fresh = np.array([k in fset for k in key(hb)])
    assert in_fresh.sum() == len(fb)                                     # the history allocated every block the fresh hash did ...
    np.testing.assert_array_equal(hv[in_fresh], fv)                       # ... and those hold the same voxel words
    hw = hv[..., 1].view(F)
    extra = (hw > 0) & ~in_fresh[:, None]
    assert extra.sum() > 0                                                # weight the fresh hash does not have, all in blocks it never allocated
    assert int((hw > 0).sum()) == int((fv[..., 1].view(F) > 0).sum()) + int(extra.sum())


def test_integrate_at_a_non_finite_pose_changes_no_voxel_and_gc_returns_what_it_allocated(oracle_lib):
    """the frame loop can issue an INTEGRATE at newT = -inf (every frame left in the re-integration list lost its pose): the inverse pose is NaN,
    the ray walk inserts a few blocks at meaningless positions, the NaN frustum test passes every block, no voxel passes the truncation test, and
    the garbage collection of the same turn -- over that all-blocks list -- frees exactly the blocks the call inserted"""
    W, H = 160, 120
    cam = camera_params(W, H)
    hp = small_params()
    depth, color, T = synth.make_frame(5, W, H)
    o = orc.OracleSceneRepHashSDF(hp)
    o.integrate(T, depth, color, cam)
    before = orc.canonical_blocks(o.download())
    before = (before[0].copy(), before[1].copy())
    free0 = o.getHeapFreeCount()
    o.integrate(np.full((4, 4), -np.inf, F), depth, color, cam)
    assert o.last_U == 0 and o.getHeapFreeCount() < free0
    o.garbageCollect()
    after = orc.canonical_blocks(o.download())
    assert o.getHeapFreeCount() == free0
    np.testing.assert_array_equal(after[0], before[0])
    np.testing.assert_array_equal(after[1], before[1])
    orc.check_hash_invariants(o.download(), hp)

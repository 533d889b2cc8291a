"""Parity of this implementation against the REFERENCE'S OWN CUDA kernels (oracle/_ref: FL/DepthSensing/CUDASceneRepHashSDF.cu built
for sm_90a with the compatibility patch of oracle/build_ref.py), on identical frames and poses, on the GPU.  The reference's states are
recorded on an H100 in tests/golden/tsdf_reference_cuda.npz (block set and per-block CRCs of the voxel words whole, voxel words sampled:
tests/reference_cuda.py).

* block coordinates (the allocated set, and the in-frustum list): bit-exact, both builds;
* IEEE build of the reference (no --use_fast_math): EVERY voxel word -- sdf, weight, colour -- bit-identical, also after
  re-integration, de-integration and GC (the library's arithmetic contract places its FMAs where nvcc places them in the
  reference's expressions, oracle/tsdf_oracle.c header);
* --use_fast_math build (the configuration the reference ships): weights exact, sdf within 1e-4, colours +-1 at rounding ties,
  for all but a vanishing fraction (~1e-5) of voxels whose projected pixel or truncation test sits on a decision boundary
  (approximate division rounds differently there)."""
import numpy as np
import pytest

from bundlefusion_b200 import synth
from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF, camera_params, default_hash_params
from oracle import oracle as orc
from tests.reference_cuda import Recorded, block_crcs, sample_state, saving_fixture

pytestmark = pytest.mark.gpu
F = np.float32
REF = Recorded("tsdf_reference_cuda.npz")
_save_recorded = saving_fixture(REF)


def compare_states(ours, ref, sdf_tol, exact=False):
    """ours: a download(); ref: another download(), or a sampled state of the reference (tests/reference_cuda.py)"""
    ob, ov = orc.canonical_blocks(ours)
    sampled = "idx" in ref
    rb, rv = (ref["blocks"], ref["vox"]) if sampled else orc.canonical_blocks(ref)
    np.testing.assert_array_equal(ob, rb)                                  # block set bit-exact
    if sampled:
        if exact:                                                          # every voxel word, through the per-block CRCs of the whole state
            np.testing.assert_array_equal(block_crcs(ov), ref["crc"])
        ov = ov.reshape(-1, ov.shape[-1])[ref["idx"]]
    if exact:                                                              # IEEE build: every sdf / weight / colour word bit-identical
        np.testing.assert_array_equal(ov, rv)
    o_sdf, o_w, o_c = ov[..., 0].view(F), ov[..., 1].view(F), ov[..., 2].copy().view(np.uint8).reshape(ov.shape[:-1] + (4,))
    r_sdf, r_w, r_c = rv[..., 0].view(F), rv[..., 1].view(F), rv[..., 2].copy().view(np.uint8).reshape(rv.shape[:-1] + (4,))
    n = o_w.size
    w_mismatch = np.count_nonzero(o_w != r_w)
    assert w_mismatch <= max(2, 2e-5 * n), f"{w_mismatch} of {n} voxel weights differ"      # decision-boundary voxels only
    same = o_w == r_w
    touched = same & (o_w > 0)
    dsdf = np.abs(o_sdf[touched] - r_sdf[touched])
    # A voxel whose projection lands within rounding distance of a pixel boundary reads the neighbouring depth pixel in one
    # implementation and not the other (IEEE vs FMA-contracted / fast-math projection): same weight, different sample.  Those
    # are counted, not tolerated silently: they must stay below 1e-4 of the touched voxels; everything else is within sdf_tol.
    flips = np.count_nonzero(dsdf > sdf_tol)
    assert flips <= max(3, 1e-4 * dsdf.size), f"{flips} of {dsdf.size} touched voxels differ by more than {sdf_tol}"
    dc = np.abs(o_c[touched].astype(np.int32) - r_c[touched].astype(np.int32)).max(axis=-1)
    assert np.count_nonzero(dc > 1) <= max(3, 1e-4 * dsdf.size) + flips
    return {"weight_mismatch_frac": w_mismatch / n, "pixel_flip_frac": flips / max(1, dsdf.size), "median_dsdf": float(np.median(dsdf)),
            "p999_dsdf": float(np.quantile(dsdf, 0.999)), "colour_differs_frac": float((dc > 0).mean()), "touched": int(dsdf.size)}


def reintegration_pose(T):
    T2 = T.copy(); T2[:3, 3] += np.array([0.011, -0.006, 0.004], F)
    return T2


def reference_stream(dev, hp, cam, frames, fast_math):
    """the reference's states along the stream both tests here and tests/test_tsdf_fast_gpu.py run: integrate x 6 (state 1); de-integrate /
    integrate frames 1 and 4 at updated poses, de-integrate frame 0, GC (state 2)"""
    def live():
        import torch
        from oracle import ref_tsdf
        ref = ref_tsdf.ReferenceSceneRepHashSDF(hp, dev, fast_math=fast_math)
        dl = [(torch.from_numpy(f[0]).to(dev), torch.from_numpy(f[1]).to(dev)) for f in frames]
        for (d, c, T), (dd, dc) in zip(frames, dl):
            ref.integrate(T, dd, dc, cam)
        out = {"s1_" + k: v for k, v in sample_state(ref.download()).items()}
        out.update(occupied1=ref.hp.m_numOccupiedBlocks, free1=ref.getHeapFreeCount(), alloc_rounds=ref.alloc_rounds)
        for k in (1, 4):
            T = frames[k][2]
            ref.deIntegrate(T, dl[k][0], dl[k][1], cam); ref.integrate(reintegration_pose(T), dl[k][0], dl[k][1], cam)
        ref.deIntegrate(frames[0][2], dl[0][0], dl[0][1], cam)
        ref.garbageCollect()
        out.update({"s2_" + k: v for k, v in sample_state(ref.download()).items()})
        out.update(free2=ref.getHeapFreeCount())
        return out
    r = REF.get(f"stream/fast_math={int(fast_math)}", live)
    return ({k[3:]: r[k] for k in ("s1_blocks", "s1_idx", "s1_vox", "s1_crc")}, {k[3:]: r[k] for k in ("s2_blocks", "s2_idx", "s2_vox", "s2_crc")},
            {k: int(r[k]) for k in ("occupied1", "free1", "alloc_rounds", "free2")})


@pytest.mark.parametrize("fast_math", [False, True])
def test_stream_with_reintegration_matches_reference_cuda(cuda_device, fast_math):
    import torch
    W, H = 320, 240
    cam = camera_params(W, H)
    hp = default_hash_params(num_buckets=100003, num_sdf_blocks=60000)
    ours = CUDASceneRepHashSDF(hp, cuda_device, arithmetic="exact")
    frames = [synth.make_frame(30 * i, W, H) for i in range(6)]
    ref1, ref2, n = reference_stream(cuda_device, hp, cam, frames, fast_math)
    dev = [(torch.from_numpy(f[0]).to(cuda_device), torch.from_numpy(f[1]).to(cuda_device)) for f in frames]
    tol = 1e-4 if fast_math else 1e-5
    for (d, c, T), (dd, dc) in zip(frames, dev):
        ours.integrate(T, dd, dc, cam)
    stats = compare_states(ours.download(), ref1, tol, exact=not fast_math)
    assert ours.getNumOccupiedBlocks() == n["occupied1"]
    assert ours.getHeapFreeCount() == n["free1"]
    assert n["alloc_rounds"] >= 2 * len(frames)             # the reference needs >= 2 alloc launches (+ D2H) per frame; we need 1
    # re-integration of two frames at updated poses + GC, as DepthSensing.cpp:854-902
    for k in (1, 4):
        d, c, T = frames[k]
        ours.deIntegrate(T, dev[k][0], dev[k][1], cam); ours.integrate(reintegration_pose(T), dev[k][0], dev[k][1], cam)
    ours.deIntegrate(frames[0][2], dev[0][0], dev[0][1], cam)
    ours.garbageCollect()
    stats2 = compare_states(ours.download(), ref2, 10 * tol, exact=not fast_math)     # fast-math: de-integration divides by (w - 1), errors grow a little
    assert ours.getHeapFreeCount() == n["free2"]
    print("weight-mismatch fraction, max |dsdf|, colour-differs fraction:", stats, stats2)

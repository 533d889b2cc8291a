"""The CPU oracle against committed outputs of the REFERENCE'S OWN CUDA (tests/golden/*.npz, produced on a GPU by
scripts/make_golden_from_reference.py from oracle/_ref's IEEE build of CUDASceneRepHashSDF.cu / SolverBundling.cu): the same seeded inputs
are regenerated here and replayed through oracle/*.c.  This is the pin of the oracle that runs without a GPU.
TSDF: allocated block set, heap count and every voxel word (CRC per block) bit-identical to the reference's kernels.
Solver: poses within 1e-4 relative L2 (BASELINE north_star), dense overlap count equal."""
import os
import zlib

import numpy as np
import pytest

from bundlefusion_b200 import synth
from bundlefusion_b200.scene_rep import camera_params, default_hash_params
from oracle import oracle as orc

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
F = np.float32


def _load(name):
    p = os.path.join(GOLD, name)
    if not os.path.exists(p):
        pytest.skip(f"{name} not generated yet (scripts/make_golden_from_reference.py on a GPU box)")
    return np.load(p)


def _inverse_subdeterminants(T):
    """The 4x4 inverse through 2x2 sub-determinants, float32, each operation rounded: how the pose inverses handed to the reference's kernels were formed when
    tsdf_reference_ieee.npz was generated on a GPU (round 1).  The library now forms them as the reference's host does (tests/test_mat4_inverse_reference.py); the
    kernels' parity does not depend on which inverse they are handed, the stored voxel words do -- so this test hands the oracle the inverses the generator used."""
    f = np.float32
    a = [f(x) for x in np.asarray(T, F).reshape(16)]
    a00, a01, a02, a03, a10, a11, a12, a13, a20, a21, a22, a23, a30, a31, a32, a33 = a
    s0, s1, s2 = a00 * a11 - a10 * a01, a00 * a12 - a10 * a02, a00 * a13 - a10 * a03
    s3, s4, s5 = a01 * a12 - a11 * a02, a01 * a13 - a11 * a03, a02 * a13 - a12 * a03
    c5, c4, c3 = a22 * a33 - a32 * a23, a21 * a33 - a31 * a23, a21 * a32 - a31 * a22
    c2, c1, c0 = a20 * a33 - a30 * a23, a20 * a32 - a30 * a22, a20 * a31 - a30 * a21
    det = s0 * c5 - s1 * c4 + s2 * c3 + s3 * c2 - s4 * c1 + s5 * c0
    r = f(1.0) / det
    out = [(a11 * c5 - a12 * c4 + a13 * c3) * r, (-a01 * c5 + a02 * c4 - a03 * c3) * r, (a31 * s5 - a32 * s4 + a33 * s3) * r, (-a21 * s5 + a22 * s4 - a23 * s3) * r,
           (-a10 * c5 + a12 * c2 - a13 * c1) * r, (a00 * c5 - a02 * c2 + a03 * c1) * r, (-a30 * s5 + a32 * s2 - a33 * s1) * r, (a20 * s5 - a22 * s2 + a23 * s1) * r,
           (a10 * c4 - a11 * c2 + a13 * c0) * r, (-a00 * c4 + a01 * c2 - a03 * c0) * r, (a30 * s4 - a31 * s2 + a33 * s0) * r, (-a20 * s4 + a21 * s2 - a23 * s0) * r,
           (-a10 * c3 + a11 * c1 - a12 * c0) * r, (a00 * c3 - a01 * c1 + a02 * c0) * r, (-a30 * s3 + a31 * s1 - a32 * s0) * r, (a20 * s3 - a21 * s1 + a22 * s0) * r]
    return np.array(out, F).reshape(4, 4)


def test_tsdf_oracle_equals_reference_kernels():
    g = _load("tsdf_reference_ieee.npz")
    c = eval(bytes(g["case"]).decode())
    cam = camera_params(c["W"], c["H"])
    hp = default_hash_params(num_buckets=c["num_buckets"], num_sdf_blocks=c["num_sdf_blocks"])
    o = orc.OracleSceneRepHashSDF(hp)
    if "pose_inverse" not in g.files:                       # generated before the library's host inverse followed the reference's formula

        def set_pose(T, hp=o.hp):
            T = np.ascontiguousarray(T, F).reshape(4, 4); inv = _inverse_subdeterminants(T)
            for k in range(16):
                hp.m_rigidTransform.m[k] = float(T.reshape(16)[k]); hp.m_rigidTransformInverse.m[k] = float(inv.reshape(16)[k])
        o._set_pose = set_pose
    frames = [synth.make_frame(i, c["W"], c["H"]) for i in c["frames"]]
    for d, col, T in frames:
        o.integrate(T, d, col, cam)
    k = c["reint"]
    d, col, T = frames[k]
    T2 = T.copy(); T2[:3, 3] += np.array(c["shift"], F)
    o.deIntegrate(T, d, col, cam); o.integrate(T2, d, col, cam)
    o.garbageCollect()
    b, v = orc.canonical_blocks(o.download())
    np.testing.assert_array_equal(b, g["blocks"])
    crcs = np.array([zlib.crc32(np.ascontiguousarray(x).tobytes()) for x in v], np.uint32)
    np.testing.assert_array_equal(crcs, g["crcs"])
    np.testing.assert_array_equal(v[:4], g["first_voxels"])
    assert o.getHeapFreeCount() == int(g["heap_free"])


def test_solver_oracle_matches_reference_kernels():
    g = _load("solver_reference_ieee.npz")
    s = eval(bytes(g["sparse_case"]).decode())
    prob = synth.make_ba_problem(s["n_images"], degree=s["degree"], corr_per_pair=s["corr_per_pair"], noise=s["noise"], seed=s["seed"])
    o = orc.solve_sparse(prob["corr"], prob["init_rot"], prob["init_trans"], s["n_gn"], s["n_pcg"])
    x_o, x_r = np.c_[o["rot"], o["trans"]], np.c_[g["sparse_rot"], g["sparse_trans"]]
    assert np.linalg.norm(x_o - x_r) / np.linalg.norm(x_r) < 1e-4
    e = orc.energy(prob["corr"], o["rot"], o["trans"])
    assert abs(e - float(g["sparse_energy"][-1])) <= 0.02 * float(g["sparse_energy"][-1]) + 1e-7
    dc = eval(bytes(g["dense_case"]).decode())
    dp = synth.make_dense_ba_problem(dc["n_images"], stride=dc["stride"], W=dc["W"], H=dc["H"])
    o = orc.solve(dp["corr"], dp["init_rot"], dp["init_trans"], dc["n_gn"], dc["n_pcg"], [1.0] * dc["n_gn"], [1.0, 2.0], [0.0, 0.0], dp["caches"], dp["intrinsics"])
    x_o, x_r = np.c_[o["rot"], o["trans"]], np.c_[g["dense_rot"], g["dense_trans"]]
    assert np.linalg.norm(x_o - x_r) / np.linalg.norm(x_r) < 1e-4
    assert o["overlap_pairs"] == int(g["dense_overlap"])

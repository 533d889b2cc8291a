"""The Gauss-Newton kernel's three grid policies (solver.cu: CoopGrid, OneCtaGrid, ResidentCluster) give bit-identical results.

Each problem is solved under the automatic choice and under every policy forced with bfSolverSetGridPolicy that can run it; the poses
must be equal bit for bit and the solver statistics equal, a forced policy that cannot run must be refused without touching the poses,
and the automatic choice must be the documented rule.  The cases sit where the policies go wrong: the size boundaries (16 / 17, 64 / 65,
128 / 129, the shared-memory fit of the dense term at 89 / 90), a partial last CTA, clusters of 1 and 16 CTAs, the one-CTA kernel with
3 and 4 virtual CTAs, rows that fill every shared-memory slot, PCG exits at both mbarrier parities and at iteration 0, a Gauss-Newton
early stop, invalid images, one workspace reused across sizes and policies, and the frame loop.  Accuracy against the CPU oracle and a
float64 Gauss-Newton is checked alongside (tolerances as tests/test_solver_gpu.py)."""
import ctypes as C
import functools
import math

import numpy as np
import pytest

from bundlefusion_b200 import synth
from bundlefusion_b200.solver import (GRID_POLICY_AUTO, GRID_POLICY_CLUSTER, GRID_POLICY_GRID, GRID_POLICY_ONE_CTA, CUDASolverBundling,
                                      DeviceCache, set_grid_policy)
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

FORCED = {"grid": GRID_POLICY_GRID, "one_cta": GRID_POLICY_ONE_CTA, "cluster": GRID_POLICY_CLUSTER}
NOT_SUPPORTED = 801                                  # cudaErrorNotSupported
STATS_EQUAL = ("gn", "pcg", "pairs", "max_delta", "converged", "dense_overlap_pairs", "dense_weighted_pairs")
DENSE_W = {"wS": [1.0, 1.0], "wD": [1.0, 2.0], "wC": [0.1, 0.1]}      # as test_solver_gpu.py::test_dense_term_beyond_64_images_matches_oracle


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-12)


@pytest.fixture(autouse=True)
def _auto_policy_after_each_test():
    yield
    set_grid_policy(GRID_POLICY_AUTO)


# ---- the documented rule (solver.cu pick_policy, include/bf_solver.h) ------------------------------------------------------------
def grid_ctas(N):
    return math.ceil(N / 8)


def resident_bytes(N, dense):
    """dynamic shared memory of pcg_resident (solver.cu resident_smem_words): per-row blocks, diagonals, eight 6N vectors, partials, slots"""
    k = 2 if dense else 1
    return 4 * (8 * N * 36 * k + 8 * 72 + 48 * N + 64 + 8 * N * k)


def can_run(policy, N, dense, lim):
    G = grid_ctas(N)
    if policy == GRID_POLICY_ONE_CTA:
        return G <= 4
    if policy == GRID_POLICY_CLUSTER:
        return G <= lim["cluster_cap"] and resident_bytes(N, dense) <= lim["dyn_smem"]
    return True


def auto_policy(N, dense, lim):
    if N <= 16 and can_run(GRID_POLICY_ONE_CTA, N, dense, lim):
        return GRID_POLICY_ONE_CTA
    if can_run(GRID_POLICY_CLUSTER, N, dense, lim):
        return GRID_POLICY_CLUSTER
    return GRID_POLICY_GRID


@pytest.fixture(scope="module")
def lim(cuda_device):
    """the cluster cap and the resident kernel's shared memory limit, as the library probed them"""
    prob = synth.make_ba_problem(2, degree=1, corr_per_pair=25, seed=1)
    info = solve(cuda_device, prob, GRID_POLICY_AUTO, 1, 2)["info"]
    assert info["cluster_cap"] in (8, 16) and info["dyn_smem"] > 0
    print(f"cluster cap {info['cluster_cap']}, resident dynamic shared memory limit {info['dyn_smem']} bytes")
    return info


def skip_if_cap_limits(N, lim):
    if grid_ctas(N) > lim["cluster_cap"] and grid_ctas(N) <= 16:
        pytest.skip(f"the cluster cap probed on this device is {lim['cluster_cap']}: no cluster of {grid_ctas(N)} CTAs to compare at N = {N}")


# ---- solving ----------------------------------------------------------------------------------------------------------------------
def solve(dev, prob, policy, n_gn, n_pcg, *, weights=None, dense=None, valid=None, solver=None, refused=False):
    """one solve of `prob` with the grid policy forced (GRID_POLICY_AUTO: the default), restored to auto before returning.
    dense: {"cache": DeviceCache, "wD": [...], "wC": [...]}.  refused: the solve must fail with cudaErrorNotSupported and leave the poses alone."""
    import torch
    N = len(prob["init_rot"])
    corr = torch.from_numpy(np.ascontiguousarray(prob["corr"]).view(np.uint8).reshape(-1).copy()).to(dev)
    rot = torch.from_numpy(prob["init_rot"].copy()).to(dev)
    trans = torch.from_numpy(prob["init_trans"].copy()).to(dev)
    v = torch.from_numpy(np.ones(N, np.int32) if valid is None else np.ascontiguousarray(valid, np.int32)).to(dev)
    sol = solver if solver is not None else CUDASolverBundling(N, max(len(prob["corr"]), 1000 * N), dev)
    kw = {} if dense is None else {"weightsDenseDepth": dense["wD"], "weightsDenseColor": dense["wC"], "cudaCache": dense["cache"]}
    w = weights if weights is not None else [1.0] * n_gn
    set_grid_policy(policy)
    try:
        if refused:
            with pytest.raises(RuntimeError, match=f"CUDA error {NOT_SUPPORTED}"):
                sol.solve(corr, len(prob["corr"]), v, N, n_gn, n_pcg, w, d_rotationAnglesUnknowns=rot, d_translationUnknowns=trans, **kw)
            torch.cuda.synchronize()
            np.testing.assert_array_equal(rot.cpu().numpy(), prob["init_rot"])
            np.testing.assert_array_equal(trans.cpu().numpy(), prob["init_trans"])
            return None
        sol.solve(corr, len(prob["corr"]), v, N, n_gn, n_pcg, w, d_rotationAnglesUnknowns=rot, d_translationUnknowns=trans, **kw)
        info = sol.getLaunchInfo()
        torch.cuda.synchronize()
    finally:
        set_grid_policy(GRID_POLICY_AUTO)
    return {"rot": rot.cpu().numpy(), "trans": trans.cpu().numpy(), "stats": sol.getStats(), "info": info, "solver": sol}


def assert_same(runs):
    """every run bit-equal to the first, statistics equal, no error flag"""
    (name0, r0), *rest = runs.items()
    assert r0["stats"]["error"] == 0, name0
    for name, r in rest:
        assert r["stats"]["error"] == 0, name
        np.testing.assert_array_equal(r["rot"], r0["rot"], err_msg=f"rot: {name} vs {name0}")
        np.testing.assert_array_equal(r["trans"], r0["trans"], err_msg=f"trans: {name} vs {name0}")
        for k in STATS_EQUAL:
            assert r["stats"][k] == r0["stats"][k], (k, name, r["stats"][k], name0, r0["stats"][k])


def solve_all(dev, prob, n_gn, n_pcg, lim, *, dense=None, **kw):
    """`prob` under auto and every forced policy: the runnable ones must agree bit for bit, the others must be refused.  Returns the runs."""
    N = len(prob["init_rot"])
    dense_on = dense is not None
    runs = {"auto": solve(dev, prob, GRID_POLICY_AUTO, n_gn, n_pcg, dense=dense, **kw)}
    info = runs["auto"]["info"]
    assert info["policy"] == auto_policy(N, dense_on, lim), (N, info)
    assert info["ctas"] == grid_ctas(N)
    for name, pol in FORCED.items():
        if can_run(pol, N, dense_on, lim):
            runs[name] = solve(dev, prob, pol, n_gn, n_pcg, dense=dense, **kw)
            assert runs[name]["info"]["policy"] == pol
        else:
            solve(dev, prob, pol, n_gn, n_pcg, dense=dense, refused=True, **kw)
    assert_same(runs)
    return runs


@functools.lru_cache(maxsize=None)
def sparse_problem(N, degree=6, corr_per_pair=25, seed=None, **kw):
    return synth.make_ba_problem(N, degree=min(degree, N - 1), corr_per_pair=corr_per_pair, noise=kw.pop("noise", 0.002), seed=N if seed is None else seed, **kw)


# ---- sparse -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [2, 3, 9, 11, 16, 17, 24, 25, 32, 33, 63, 64, 65, 100, 127, 128, 129])
def test_sparse_size_sweep(cuda_device, lim, N):
    """policy boundaries, a partial last CTA, clusters of 1 .. 16 CTAs, the one-CTA kernel with G = 1 .. 4 virtual CTAs"""
    skip_if_cap_limits(N, lim)
    prob = sparse_problem(N)
    runs = solve_all(cuda_device, prob, 2, 20, lim)
    r = runs["auto"]
    assert r["stats"]["pairs"] == len(prob["pairs"])
    np.testing.assert_array_equal(r["rot"][0], prob["init_rot"][0])       # variable 0 is fixed
    assert ("cluster" in runs) == (grid_ctas(N) <= lim["cluster_cap"])
    assert ("one_cta" in runs) == (N <= 32)


@pytest.mark.parametrize("N", [17, 64, 65, 128])
def test_full_rows(cuda_device, lim, N):
    """every image paired with every other: a row's N - 1 segments fill its shared-memory slots"""
    skip_if_cap_limits(N, lim)
    prob = sparse_problem(N, degree=N - 1, corr_per_pair=6)
    runs = solve_all(cuda_device, prob, 1, 10, lim)
    assert runs["auto"]["solver"].m_maxCorrPerImage >= 6 * (N - 1)        # no row is cut
    assert runs["auto"]["stats"]["pairs"] == N * (N - 1) // 2


@pytest.mark.parametrize("n_pcg", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("N", [11, 40, 100])
def test_pcg_exit_parity(cuda_device, lim, N, n_pcg):
    """the PCG leaves at an odd and an even iteration count (both mbarrier parities, both p buffers), the Lie update on the last one"""
    runs = solve_all(cuda_device, sparse_problem(N), 1, n_pcg, lim)
    assert runs["auto"]["stats"]["pcg"] == n_pcg                           # by count, not by the early-out


@pytest.mark.parametrize("N", [11, 40])
def test_exit_at_iteration_zero(cuda_device, lim, N):
    """exact correspondences at the true poses: p.Ap ~ 0 at iteration 0, a zero step, convergence after one GN iteration"""
    prob = sparse_problem(N, noise=0.0, perturb_rot=0.0, perturb_trans=0.0)
    runs = solve_all(cuda_device, prob, 2, 10, lim)
    s = runs["auto"]["stats"]
    assert s["gn"] == 1 and s["pcg"] == 1 and s["max_delta"] == 0 and s["converged"] == 1, s
    # the zero update still maps each pose through its matrix and back: equal to the input to float32 rounding
    np.testing.assert_allclose(runs["auto"]["rot"], prob["init_rot"], rtol=0, atol=2e-6)
    np.testing.assert_allclose(runs["auto"]["trans"], prob["init_trans"], rtol=0, atol=2e-6)


@pytest.mark.parametrize("N", [11, 40])
def test_gn_early_stop(cuda_device, lim, N):
    """a small perturbation converges (max|delta| < 0.005) before the last of 5 GN iterations: the later launches return at once"""
    prob = sparse_problem(N, noise=0.0005, perturb_rot=0.002, perturb_trans=0.003)
    runs = solve_all(cuda_device, prob, 5, 30, lim)
    o = orc.solve_sparse(prob["corr"], prob["init_rot"], prob["init_trans"], 5, 30)
    s = runs["auto"]["stats"]
    assert s["gn"] == o["gn"] < 5 and s["converged"] == 1, (s, o["gn"])
    assert rel_l2(np.c_[runs["auto"]["rot"], runs["auto"]["trans"]], np.c_[o["rot"], o["trans"]]) < 1e-4


def test_invalid_images(cuda_device, lim):
    """the convergence maximum is over valid images only"""
    prob = sparse_problem(40)
    valid = np.ones(40, np.int32)
    valid[3] = valid[7] = 0
    runs = solve_all(cuda_device, prob, 3, 60, lim, valid=valid)
    o = orc.solve(prob["corr"], prob["init_rot"], prob["init_trans"], 3, 60, [1.0] * 3, valid=valid)
    assert runs["auto"]["stats"]["gn"] == o["gn"]
    assert rel_l2(np.c_[runs["auto"]["rot"], runs["auto"]["trans"]], np.c_[o["rot"], o["trans"]]) < 1e-4


@pytest.mark.parametrize("N", [17, 65, 128])
def test_accuracy_vs_oracle_and_float64(cuda_device, lim, N):
    """each policy's poses against the CPU oracle (1e-4 relative L2) and an independent float64 Gauss-Newton"""
    skip_if_cap_limits(N, lim)
    prob = sparse_problem(N, seed=11)
    runs = solve_all(cuda_device, prob, 3, 150, lim)
    o = orc.solve_sparse(prob["corr"], prob["init_rot"], prob["init_trans"], 3, 150)
    for name, r in runs.items():
        assert rel_l2(np.c_[r["rot"], r["trans"]], np.c_[o["rot"], o["trans"]]) < 1e-4, name
    runs = solve_all(cuda_device, prob, 6, 150, lim)
    ref_rot, ref_trans = synth.ba_reference_f64(prob["corr"], prob["init_rot"], prob["init_trans"], n_gn=8)
    e_ref = orc.energy(prob["corr"], ref_rot.astype(np.float32), ref_trans.astype(np.float32))
    for name, r in runs.items():
        assert orc.energy(prob["corr"], r["rot"], r["trans"]) <= e_ref * 1.01 + 1e-7, name
        assert rel_l2(np.c_[r["rot"], r["trans"]], np.c_[ref_rot, ref_trans]) < 2e-3, name


# ---- dense ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dense90():
    """90 consecutive frames (stride 1: most pairs overlap), every pair with 8 sparse correspondences; smaller cases take its first N frames"""
    return synth.make_dense_ba_problem(90, stride=1, start=60, corr_per_pair=8, W=320, H=240)


def dense_subset(P, N):
    c = P["corr"]
    keep = (c["i"] < N) & (c["j"] < N)
    return {"corr": np.ascontiguousarray(c[keep]), "init_rot": P["init_rot"][:N].copy(), "init_trans": P["init_trans"][:N].copy(),
            "caches": P["caches"][:N], "intrinsics": P["intrinsics"], "pairs": [p for p in P["pairs"] if p[1] < N]}


def densest_row(sol, N, dev):
    """most dense pairs of one image in the last dense system the solver built"""
    import torch
    jtj = torch.zeros(36 * N * N, dtype=torch.float32, device=dev)
    assert sol.lib.bfSolverDebugDenseSystem(C.byref(sol.m_solverState), N, C.c_void_p(jtj.data_ptr()), None) == 0
    torch.cuda.synchronize()
    nz = np.abs(jtj.cpu().numpy().reshape(N, 6, N, 6)).sum(axis=(1, 3)) != 0
    np.fill_diagonal(nz, False)
    return int(nz.sum(axis=1).max())


@pytest.mark.parametrize("N", [11, 17, 40, 89, 90])
def test_dense(cuda_device, lim, dense90, N):
    """sparse + dense depth + colour: the transposed dense block of the hi image in residency, and the shared-memory fit of the dense
    system, 2560 (N + 1) bytes: 89 images are the most that fit, 90 fall back to the grid"""
    skip_if_cap_limits(N, lim)
    prob = dense_subset(dense90, N)
    dense = {"cache": DeviceCache(prob["caches"], prob["intrinsics"], cuda_device), "wD": DENSE_W["wD"], "wC": DENSE_W["wC"]}
    if N in (89, 90):
        assert resident_bytes(N, True) == 2560 * (N + 1)
        assert (resident_bytes(N, True) <= lim["dyn_smem"]) == (N == 89), lim
    runs = solve_all(cuda_device, prob, 2, 15, lim, dense=dense, weights=DENSE_W["wS"])
    assert runs["auto"]["info"]["policy"] == {11: GRID_POLICY_ONE_CTA, 90: GRID_POLICY_GRID}.get(N, GRID_POLICY_CLUSTER)
    # at 89 and 90 images the strict oracle build takes ~40 s a solve; its optimised OpenMP build runs the same source
    o = orc.solve(prob["corr"], prob["init_rot"], prob["init_trans"], 2, 15, DENSE_W["wS"], DENSE_W["wD"], DENSE_W["wC"], prob["caches"], prob["intrinsics"],
                  fast=N >= 89)
    s = runs["auto"]["stats"]
    assert s["dense_overlap_pairs"] == o["overlap_pairs"] and s["dense_weighted_pairs"] == o["weighted_pairs"] > 0
    for name, r in runs.items():
        assert rel_l2(np.c_[r["rot"], r["trans"]], np.c_[o["rot"], o["trans"]]) < 1e-4, name
    print(f"dense N = {N}: {s['dense_weighted_pairs']} weighted pairs, densest row {densest_row(runs['auto']['solver'], N, cuda_device)} dense pairs")


# ---- one workspace across sizes and policies --------------------------------------------------------------------------------------
def test_workspace_reuse(cuda_device, lim, dense90):
    """one solver (130 images) solving N = 100, 11, 129, 40 (dense), 17 (dense) in turn under each policy: every result equals a fresh
    solver's under the same policy, and all policies agree"""
    cases = [(sparse_problem(100), None), (sparse_problem(11), None), (sparse_problem(129), None),
             (dense_subset(dense90, 40), True), (dense_subset(dense90, 17), True)]
    caches = {}
    results = {}
    for pname, pol in [("auto", GRID_POLICY_AUTO)] + list(FORCED.items()):
        shared = CUDASolverBundling(130, 130 * 1000, cuda_device)
        for prob, is_dense in cases:
            N = len(prob["init_rot"])
            if pol != GRID_POLICY_AUTO and not can_run(pol, N, bool(is_dense), lim):
                continue
            dense, w = None, None
            if is_dense:
                if N not in caches:
                    caches[N] = DeviceCache(prob["caches"], prob["intrinsics"], cuda_device)
                dense, w = {"cache": caches[N], "wD": DENSE_W["wD"], "wC": DENSE_W["wC"]}, DENSE_W["wS"]
            a = solve(cuda_device, prob, pol, 2, 15, weights=w, dense=dense, solver=shared)
            b = solve(cuda_device, prob, pol, 2, 15, weights=w, dense=dense)
            assert_same({f"{pname} shared N={N}": a, f"{pname} fresh N={N}": b})
            results.setdefault(N, {})[pname] = a
        shared.close()
    for N, runs in results.items():
        assert_same(runs)


# ---- the frame loop ---------------------------------------------------------------------------------------------------------------
def test_frame_loop_under_every_policy(cuda_device):
    """the 43-frame stream of test_frame_loop_gpu.py::test_frame_loop_tracks_solves_and_reintegrates (local solves at N = 11 with the dense
    term, global solves of up to 5 keyframes) with the policy left automatic and forced to one CTA, the cluster and the grid: every status
    field, the counters and the optimised trajectory are identical"""
    import torch
    from bundlefusion_b200.frame_loop import FrameLoop, default_params
    W, H = 320, 240
    frames = [synth.make_frame(2 * i, W, H, texture="rich") for i in range(43)]
    dev_frames = [(torch.from_numpy(d).to(cuda_device), torch.from_numpy(c).to(cuda_device)) for d, c, T in frames]
    out = {}
    for pname, pol in [("auto", GRID_POLICY_AUTO)] + list(FORCED.items()):
        p = default_params(W, H)
        p.maxNumImages = 16; p.maxNumFrames = 64
        p.hash.m_hashNumBuckets = 100003; p.hash.m_numSDFBlocks = 90000
        set_grid_policy(pol)
        try:
            loop = FrameLoop(p, cuda_device)
            sts = [loop.step(d, c).as_dict() for d, c in dev_frames]
            sts += [loop.step_past_end().as_dict() for _ in range(12)]
            torch.cuda.synchronize()
            out[pname] = (sts, loop.trajectory(43), loop.counters())
            loop.close()
        finally:
            set_grid_policy(GRID_POLICY_AUTO)
    s0, t0, c0 = out["auto"]
    assert c0["local_solves"] >= 4 and c0["global_solves"] >= 3
    for pname, (s1, t1, c1) in out.items():
        assert c1 == c0, pname
        for a, b in zip(s0, s1):
            for k in a:
                if k == "transform":
                    assert np.array_equal(a[k], b[k], equal_nan=True), (pname, a["frame"])
                else:
                    assert a[k] == b[k], (pname, a["frame"], k, a[k], b[k])
        assert np.array_equal(t0, t1, equal_nan=True), pname

"""Both sweeps of the SIFT descriptor matcher (row a18) -- wgmma + TMA (sift_best_wgmma_kernel) and warp-level mma.sync (sift_best_kernel),
forced with bfSiftSetMatchSweep -- at every slice, tile, CTA and ring boundary, on tie lattices and extreme values, across batches, streams and
the frame loop.  Every case asserts three things: the counter and the stored matches equal the oracle's (the oracle stores the first 128 in
ascending image-2 feature, as the library does, so the order is compared too; distances within 2e-7: acosf of CUDA and glibc may differ in
the last bit), the two sweeps store the same bytes (counter, indices in storage order, distance bits), and the sweep that ran
(bfSiftGetMatchInfo) is the one forced.  The descriptor sets and the closed-form statement of the rule are in tests/_sift_cases.py;
test_sift_match_boundaries_oracle.py holds the oracle to that statement on the same sets."""
import ctypes as C

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from bundlefusion_b200 import synth
from bundlefusion_b200.sift import (SIFT_SWEEP_AUTO, SIFT_SWEEP_MMA, SIFT_SWEEP_WGMMA, ImagePairMatch, SiftMatchGPU, match_info,
                                    set_match_sweep)
from oracle import oracle as orc
from tests import _sift_cases as sc

pytestmark = pytest.mark.gpu

SWEEPS = (SIFT_SWEEP_WGMMA, SIFT_SWEEP_MMA)
GARBAGE = 0x5A5A5A5A


@pytest.fixture
def dev(cuda_device):
    yield cuda_device
    set_match_sweep(SIFT_SWEEP_AUTO)


def upload(dev, d):
    import torch
    return torch.from_numpy(np.ascontiguousarray(d, np.uint8)).to(dev) if len(d) else None


def run_batch(dev, jobs, sweep, distmax=0.7, ratiomax=0.8):
    """jobs: [(t1, n1, t2, n2, offset)] (t = uint8 cuda tensor or None) as ONE bfSiftMatchBatch under `sweep`; counters pre-filled with
    garbage.  Returns [(indices [n, 2] uint32, distances [n] float32, counter)] in storage order."""
    import torch
    set_match_sweep(sweep)
    ipms = []
    for _ in jobs:
        ipm = ImagePairMatch(dev)
        ipm.d_numMatches.fill_(GARBAGE); ipm.d_distances.fill_(-1.0); ipm.d_keyPointIndices.fill_(-1)
        ipms.append(ipm)
    SiftMatchGPU(device=dev).matchBatch([(t1, n1, t2, n2, ipm, off) for (t1, n1, t2, n2, off), ipm in zip(jobs, ipms)], distmax, ratiomax)
    assert match_info() == (sweep, len(jobs)), "the sweep that ran is not the one forced"
    torch.cuda.synchronize()
    return [ipm.download() for ipm in ipms]


def assert_oracle(g, d1, d2, distmax, ratiomax, offset, what=""):
    gi, gd, gc = g
    oi, od, oc = orc.sift_match(d1, d2, distmax, ratiomax, offset)
    assert gc == oc, what
    np.testing.assert_array_equal(gi, oi, err_msg=what)
    np.testing.assert_allclose(gd, od, rtol=0, atol=2e-7, err_msg=what)


def assert_same_bytes(a, b, what=""):
    assert a[2] == b[2], what
    np.testing.assert_array_equal(a[0], b[0], err_msg=what)
    np.testing.assert_array_equal(a[1].view(np.uint32), b[1].view(np.uint32), err_msg=what)


def check_cases(dev, cases, distmax=0.7, ratiomax=0.8, offset=(7, 11)):
    """cases: [(name, d1, d2)] as one batch under both sweeps, each job against the oracle, the sweeps against each other"""
    jobs = [(upload(dev, d1), len(d1), upload(dev, d2), len(d2), offset) for _, d1, d2 in cases]
    res = {sw: run_batch(dev, jobs, sw, distmax, ratiomax) for sw in SWEEPS}
    for k, (name, d1, d2) in enumerate(cases):
        what = f"{name} distmax={distmax} ratiomax={ratiomax}"
        assert_oracle(res[SIFT_SWEEP_WGMMA][k], d1, d2, distmax, ratiomax, offset, what)
        assert_same_bytes(res[SIFT_SWEEP_WGMMA][k], res[SIFT_SWEEP_MMA][k], what)
    return res[SIFT_SWEEP_WGMMA]


# ---- 1. sizes --------------------------------------------------------------------------------------------------------------------------------
# the 32-column slice, the mma.sync step (64) and CTA (64), the wgmma tile (128) and CTA (128), the ring fill (512), its first refill (513), the
# third phase of stage 0 (1025, 1152) and many phases (2049, 4096); one side small when the other is large
SIZES = (1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512, 513, 639, 640, 1023, 1024, 1025, 1152, 2049, 4096)
SHAPES = sorted({(s, 16) for s in SIZES} | {(16, s) for s in SIZES} | {(s, s) for s in SIZES if s <= 640}
                | {(1024, 1024), (1025, 1025), (4096, 1), (1, 2049), (513, 1152), (1152, 639), (129, 1025)})


@pytest.mark.parametrize("n1,n2", SHAPES)
def test_sizes(dev, n1, n2):
    d1, d2, _ = synth.make_sift_pair(n1, n2, min(n1, n2, 100), noise=0.05, seed=7 * n1 + n2)
    (g,) = check_cases(dev, [(f"{n1}x{n2}", d1, d2)])
    if min(n1, n2) >= 16:
        assert g[2] > 0


# ---- 2. tie lattices -------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lattices():
    return sc.lattice_jobs()


@pytest.mark.parametrize("ratiomax", [1.5, 0.8])
def test_tie_lattices(dev, lattices, ratiomax):
    """a few hundred lattices in one batch: at ratiomax 1.5 the stored pair reveals the row and the column winner of each tie, at 0.8 a pure
    tie is never accepted"""
    got = check_cases(dev, [(lat.name, lat.d1, lat.d2) for lat in lattices], 0.7, ratiomax, offset=(0, 0))
    for lat, (gi, _, _) in zip(lattices, got):
        pairs = set(map(tuple, gi.tolist()))
        if ratiomax > 1 and lat.reveal is not None:
            assert lat.reveal in pairs, lat.name
        if ratiomax < 1 and lat.pure_tie:
            assert lat.reveal not in pairs, lat.name


# ---- 3. extreme values -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("distmax", sc.DISTMAX)
@pytest.mark.parametrize("ratiomax", sc.RATIOMAX)
def test_extreme_values(dev, distmax, ratiomax):
    check_cases(dev, sc.extreme_cases(), distmax, ratiomax)


# ---- 4. batches and the shared workspace -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("release", [False, True])
def test_workspace_across_growing_and_shrinking_batches(dev, release):
    """batches of 1, 7, 300 and 3 jobs through one workspace (release: released and re-reserved between batches), empty jobs with NULL
    pointers among them, counters pre-filled with garbage"""
    L = capi.lib()
    rng = np.random.default_rng(31 + release)
    for k, nj in enumerate((1, 7, 300, 3)):
        cases = []
        for i in range(nj):
            n1, n2 = (int(x) for x in rng.integers(0, 200, 2))
            if i % 5 == 2:
                n1 = 0                                             # empty, NULL pointers
            if i % 7 == 3:
                n2 = 0
            d1, d2, _ = synth.make_sift_pair(max(n1, 1), max(n2, 1), 60, noise=0.05, seed=1000 * k + i)
            cases.append((f"batch {nj} job {i}", d1[:n1], d2[:n2]))
        got = check_cases(dev, cases, offset=(3, 5))
        for (_, d1, d2), g in zip(cases, got):
            if len(d1) == 0 or len(d2) == 0:
                assert g[2] == 0
        if release:
            assert L.bfSiftReleaseWorkspace() == 0 and L.bfSiftWorkspaceBytes() == 0
            capi.check(L.bfSiftReserveWorkspace(8 + 100 * k, 256), "bfSiftReserveWorkspace")


def test_cap_with_several_column_ctas(dev):
    """jobs past the 128-slot cap, each with several column CTAs: the stored matches are the first 128 of the full mutual set by image-2
    feature, the counter is the total"""
    cases = []
    for n in (300, 700, 1030):
        d1, d2, _ = synth.make_sift_pair(n, n + 17, n, noise=0.02, seed=n)
        cases.append((f"cap {n}", d1, d2))
    got = check_cases(dev, cases, offset=(0, 0))
    for (name, d1, d2), (gi, gd, gc) in zip(cases, got):
        ii, jj, dd = sc.closed_form_matches(sc.dot_of(d1, d2), 0.7, 0.8)
        assert gc == len(jj) > 128, name
        np.testing.assert_array_equal(gi.astype(np.int64), np.stack([ii[:128], jj[:128]], 1), err_msg=name)


def test_one_array_with_two_row_counts(dev):
    """one descriptor array in two jobs of a batch with 300 and 130 rows: the tensor maps are cached by (array, rows) and rows past a job's
    count are never read -- the image-2 set of the short job copies rows 200..259, which only a read past row 130 could match"""
    d1 = synth.make_sift_descriptors(300, seed=41)
    d2a = np.concatenate([synth.make_sift_descriptors(210, seed=42), d1[250:300]])
    d2b = np.concatenate([d1[200:260], synth.make_sift_descriptors(40, seed=43), d1[:20]])
    t1 = upload(dev, d1)
    jobs = [(t1, 300, upload(dev, d2a), len(d2a), (0, 0)), (t1, 130, upload(dev, d2b), len(d2b), (0, 0))]
    res = {sw: run_batch(dev, jobs, sw) for sw in SWEEPS}
    for sw in SWEEPS:
        assert_oracle(res[sw][0], d1, d2a, 0.7, 0.8, (0, 0))
        assert_oracle(res[sw][1], d1[:130], d2b, 0.7, 0.8, (0, 0))
        assert res[sw][0][2] > 0 and np.any(res[sw][0][0][:, 0] >= 250)
        assert res[sw][1][2] > 0 and np.all(res[sw][1][0][:, 0] < 130)
    for k in range(2):
        assert_same_bytes(res[SIFT_SWEEP_WGMMA][k], res[SIFT_SWEEP_MMA][k])


def test_two_streams_without_a_sync(dev):
    """two batches queued on two streams (bfSetStream through the stream the mirror binds) with no synchronisation in between: each equals
    its result alone"""
    import torch
    sets = []
    for k in range(2):
        pairs = [synth.make_sift_pair(n1, n2, 80, seed=50 + 10 * k + i) for i, (n1, n2) in enumerate([(700, 650), (129, 1025), (64, 64)])]
        sets.append([(f"stream {k} job {i}", d1, d2) for i, (d1, d2, _) in enumerate(pairs)])
    jobsets = [[(upload(dev, d1), len(d1), upload(dev, d2), len(d2), (1, 2)) for _, d1, d2 in cases] for cases in sets]
    for sw in SWEEPS:
        alone = [run_batch(dev, jobs, sw) for jobs in jobsets]
        set_match_sweep(sw)
        streams = [torch.cuda.Stream(dev), torch.cuda.Stream(dev)]
        outs = [[ImagePairMatch(dev) for _ in jobs] for jobs in jobsets]
        torch.cuda.synchronize()
        for s, jobs, ipms in zip(streams, jobsets, outs):
            with torch.cuda.stream(s):
                SiftMatchGPU(device=dev).matchBatch([(t1, n1, t2, n2, ipm, off) for (t1, n1, t2, n2, off), ipm in zip(jobs, ipms)])
        torch.cuda.synchronize()
        capi.lib().bfSetStream(None)
        for cases, a, ipms in zip(sets, alone, outs):
            for (name, d1, d2), ga, ipm in zip(cases, a, ipms):
                assert_same_bytes(ga, ipm.download(), name)
                assert_oracle(ga, d1, d2, 0.7, 0.8, (1, 2), name)


# ---- 5. the frame loop -----------------------------------------------------------------------------------------------------------------------
def test_frame_loop_under_both_sweeps(dev):
    """the 43-frame stream of test_solver_policies_gpu.py::test_frame_loop_under_every_policy under each forced sweep: every status field, the
    counters, the optimised trajectory and the heap are identical"""
    import torch
    from bundlefusion_b200.frame_loop import FrameLoop, default_params
    W, H = 320, 240
    frames = [synth.make_frame(2 * i, W, H, texture="rich") for i in range(43)]
    dev_frames = [(torch.from_numpy(d).to(dev), torch.from_numpy(c).to(dev)) for d, c, T in frames]
    out = {}
    for sw in SWEEPS:
        p = default_params(W, H)
        p.maxNumImages = 16; p.maxNumFrames = 64
        p.hash.m_hashNumBuckets = 100003; p.hash.m_numSDFBlocks = 90000
        set_match_sweep(sw)
        loop = FrameLoop(p, dev)
        try:
            sts = [loop.step(d, c).as_dict() for d, c in dev_frames]
            sts += [loop.step_past_end().as_dict() for _ in range(12)]
            torch.cuda.synchronize()
            assert match_info()[0] == sw
            out[sw] = (sts, loop.trajectory(43), loop.counters())
        finally:
            loop.close()
    s0, t0, c0 = out[SIFT_SWEEP_WGMMA]
    s1, t1, c1 = out[SIFT_SWEEP_MMA]
    assert c0["local_solves"] >= 4 and c0["global_solves"] >= 3
    assert c1 == c0
    assert len(s0) == len(s1)
    for a, b in zip(s0, s1):
        for k in a:
            if k == "transform":
                assert np.array_equal(a[k], b[k], equal_nan=True), a["frame"]
            else:
                assert a[k] == b[k], (a["frame"], k, a[k], b[k])
    assert np.array_equal(t0, t1, equal_nan=True)


# ---- 6. auto and the alignment contract ------------------------------------------------------------------------------------------------------
def test_auto_runs_wgmma_and_misaligned_arrays_are_refused(dev):
    """an aligned batch under AUTO runs the wgmma sweep; a batch with a live job whose descriptors start 1, 4 or 8 bytes past a 16-byte
    boundary returns cudaErrorInvalidValue and enqueues nothing (counters untouched, no launch counted, the last batch's info kept)"""
    import torch
    L = capi.lib()
    d1, d2, _ = synth.make_sift_pair(200, 150, 60, seed=61)
    t1, t2 = upload(dev, d1), upload(dev, d2)
    set_match_sweep(SIFT_SWEEP_AUTO)
    ipm = ImagePairMatch(dev)
    m = SiftMatchGPU(device=dev)
    m.matchBatch([(t1, 200, t2, 150, ipm, (0, 0))])
    assert match_info() == (SIFT_SWEEP_WGMMA, 1)
    torch.cuda.synchronize()
    assert_oracle(ipm.download(), d1, d2, 0.7, 0.8, (0, 0))
    raw = torch.zeros(150 * 128 + 64, dtype=torch.uint8, device=dev)
    for sweep in (SIFT_SWEEP_AUTO,) + SWEEPS:
        set_match_sweep(sweep)
        for off in (1, 4, 8):
            bad = ImagePairMatch(dev); bad.d_numMatches.fill_(GARBAGE)
            good = ImagePairMatch(dev); good.d_numMatches.fill_(GARBAGE)
            torch.cuda.synchronize()
            j_good, j_bad = m._job(t1, 200, t2, 150, good, (0, 0)), m._job(t1, 200, t2, 150, bad, (0, 0))
            j_bad.d_des2 = raw.data_ptr() + off
            launches, info = L.bfGetLaunchCount(), match_info()
            arr = (capi.BFSiftMatchJob * 2)(j_good, j_bad)
            assert L.bfSiftMatchBatch(arr, 2, C.c_float(0.7), C.c_float(0.8)) == 1          # cudaErrorInvalidValue
            torch.cuda.synchronize()
            assert L.bfGetLaunchCount() == launches and match_info() == info
            assert int(good.d_numMatches.item()) == GARBAGE and int(bad.d_numMatches.item()) == GARBAGE

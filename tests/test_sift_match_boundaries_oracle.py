"""The matcher's oracle (oracle/sift_oracle.c) against a closed-form numpy statement of the matching rule (tests/_sift_cases.py), on the tie
lattices and extreme values that test_sift_match_sweeps_gpu.py sends to both CUDA sweeps, and at sizes up to 4096 where the reference's 32
lanes hold many positions each; and bfSiftMatchBatch's host-side refusal of descriptor arrays that are not 16-byte aligned.  No GPU."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as orc
from tests import _sift_cases as sc
from tests.cuda_emu import run_without_device


def assert_oracle_is_closed_form(d1, d2, distmax, ratiomax, what=""):
    """orc.sift_match (counter, the first 128 matches in its ascending image-2 order, distances) equals the closed form; returns its matches"""
    ii, jj, dd = sc.closed_form_matches(sc.dot_of(d1, d2), distmax, ratiomax)
    oi, od, oc = orc.sift_match(d1, d2, distmax, ratiomax)
    assert oc == len(jj), what
    k = min(len(jj), 128)
    np.testing.assert_array_equal(oi.astype(np.int64), np.stack([ii[:k], jj[:k]], 1).reshape(k, 2), err_msg=what)
    np.testing.assert_allclose(od, dd[:k], rtol=0, atol=2e-7, err_msg=what)
    return set(zip(ii.tolist(), jj.tolist()))


def test_closed_form_on_hand_cases():
    """the statement itself, by hand: rows -- lane = column % 32, smaller bit-reversed lane first, then the smaller column; columns -- lane =
    (row / 4) % 32; the second value is the multiset's; a maximum of 0 has no winner"""
    m = np.array([[5, 5, 0, 0], [0, 5, 5, 0], [0, 3, 5, 5], [0, 0, 0, 0], [7, 7, 7, 9]], np.int64)
    win, v1, v2 = sc.best_second(m, sc.tie_keys(4, column=False))
    assert win.tolist() == [0, 2, 2, -1, 3]                  # brev5: lane 1 -> 16, lane 2 -> 8, lane 3 -> 24
    assert v1.tolist() == [5, 5, 5, 0, 9] and v2.tolist() == [5, 5, 5, 0, 7]
    keys = sc.tie_keys(1200, column=True)
    col = np.zeros((1, 1200), np.int64)
    col[0, [1, 3]] = 4
    assert sc.best_second(col, keys)[0][0] == 1              # one 4-row block: the first row
    col[0, [4, 8]] = 4
    assert sc.best_second(col, keys)[0][0] == 1 and sc.col_winner((1, 3, 4, 8)) == 1      # lanes 0, 0, 1, 2 -> 0, 0, 16, 8: lane 0 beats them all
    col[0, [1, 3]] = 0
    assert sc.best_second(col, keys)[0][0] == 8 and sc.col_winner((4, 8)) == 8
    col[0, :] = 0; col[0, [4, 8, 512 + 4]] = 4
    assert sc.best_second(col, keys)[0][0] == 8              # rows 4 and 516 share lane 1 (128-row cycle); lane 2 wins
    assert sc.row_winner((33, 1)) == 1 and sc.row_winner((2, 1, 1151)) == 2 and sc.row_winner((31, 1023, 63)) == 31


@pytest.mark.parametrize("n1,n2,levels,seed", [(8, 1, 3, 1), (40, 33, 2, 2), (16, 1152, 3, 3), (4, 4096, 2, 4), (3, 4096, 40, 5), (64, 513, 5, 6)])
def test_row_rule_on_tie_matrices(n1, n2, levels, seed):
    """orc.sift_row_match on integer matrices with ties everywhere (few distinct values, zeros included) equals the closed form"""
    rng = np.random.default_rng(seed)
    dot = rng.integers(0, levels, (n1, n2)).astype(np.int64) * 60000
    dot[0] = 0
    for distmax, ratiomax in ((0.7, 0.8), (4.0, 1.5), (4.0, 1.0), (1.2, 1.01)):
        res, dist = orc.sift_row_match(dot, distmax, ratiomax)
        cres, cdist = sc.row_rule(dot, distmax, ratiomax)
        np.testing.assert_array_equal(res, cres)
        np.testing.assert_allclose(dist, cdist, rtol=0, atol=2e-7)
        if (distmax, ratiomax) == (4.0, 1.5) and 60000 * (levels - 1) < 2 ** 18:
            assert np.count_nonzero(res >= 0) > n1 // 2           # ties below 2^18 are accepted above ratio 1


@pytest.mark.parametrize("n1,n2,levels,seed", [(1, 6, 3, 1), (33, 40, 2, 2), (1152, 16, 3, 3), (4096, 4, 2, 4), (4096, 3, 40, 5), (513, 64, 5, 6)])
def test_column_rule_on_tie_matrices(n1, n2, levels, seed):
    """the oracle's column pass (orc_sift_col_match after orc.sift_row_match) on integer matrices with ties everywhere equals the closed
    form: counter, the first 128 matches, distances"""
    rng = np.random.default_rng(seed)
    dot = rng.integers(0, levels, (n1, n2)).astype(np.int64) * 60000
    L = orc.lib()
    L.orc_sift_col_match.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
    L.orc_sift_col_match.restype = C.c_int
    d32 = np.ascontiguousarray(dot, np.int32)
    for distmax, ratiomax in ((0.7, 0.8), (4.0, 1.5), (4.0, 1.0)):
        rr, rd = orc.sift_row_match(dot, distmax, ratiomax)
        idx = np.zeros((128, 2), np.uint32); dist = np.zeros(128, np.float32)
        c = L.orc_sift_col_match(d32.ctypes.data, n1, n2, distmax, ratiomax, rr.ctypes.data, rd.ctypes.data, 0, 0, idx.ctypes.data, dist.ctypes.data)
        ii, jj, dd = sc.closed_form_matches(dot, distmax, ratiomax)
        assert c == len(jj)
        k = min(c, 128)
        np.testing.assert_array_equal(idx[:k].astype(np.int64), np.stack([ii[:k], jj[:k]], 1).reshape(k, 2))
        np.testing.assert_allclose(dist[:k], dd[:k], rtol=0, atol=2e-7)


def test_lattices_follow_the_closed_form():
    """every lattice of the GPU tie batch: the oracle's matches are the closed form's at ratiomax 1.5 and 0.8; at 1.5 each lattice reveals the
    pair it was built for, and a pure tie is never accepted at 0.8"""
    jobs = sc.lattice_jobs()
    assert len(jobs) > 600
    for lat in jobs:
        got15 = assert_oracle_is_closed_form(lat.d1, lat.d2, 0.7, 1.5, lat.name)
        got08 = assert_oracle_is_closed_form(lat.d1, lat.d2, 0.7, 0.8, lat.name)
        if lat.reveal is not None:
            assert lat.reveal in got15, lat.name
        if lat.pure_tie:
            assert lat.reveal not in got08, lat.name


@pytest.mark.parametrize("P", [(5, 37, 1029, 4069), (0, 2048, 4095), (31, 4064, 4095), (1, 2, 3, 4, 3000), (4092, 4093, 4094, 4095), (96, 3968)])
def test_row_ties_at_4096(P):
    """row ties across 4096 image-2 features, where each reference lane holds 128 positions (several in one lane: the earliest wins)"""
    rng = np.random.default_rng(sum(P))
    for q, n1 in ((0, 1), (3, 7)):
        d1, d2 = sc.lattice(rng, P, (q,), n1, 4096)
        assert (q, sc.row_winner(P)) in assert_oracle_is_closed_form(d1, d2, 0.7, 1.5)
        assert (q, sc.row_winner(P)) not in assert_oracle_is_closed_form(d1, d2, 0.7, 0.8)


@pytest.mark.parametrize("Q", [(5, 517, 1029, 4069), (0, 4, 4095), (1, 2, 3), (128, 256, 4092), (4, 2052), (127, 3968, 4000)])
def test_column_ties_at_4096(Q):
    """column ties across 4096 image-1 rows: 4-row blocks, the 128-row lane cycle repeated 32 times"""
    rng = np.random.default_rng(sum(Q))
    for p, n2 in ((0, 1), (2, 5)):
        d1, d2 = sc.lattice(rng, (p,), Q, 4096, n2)
        assert (sc.col_winner(Q), p) in assert_oracle_is_closed_form(d1, d2, 0.7, 1.5)
        assert (sc.col_winner(Q), p) not in assert_oracle_is_closed_form(d1, d2, 0.7, 0.8)


def test_extreme_values_follow_the_closed_form():
    """the packing bound, products above 2^18, single bins, zeros, orthogonal sets under every distmax / ratiomax of the GPU test"""
    seen = 0
    for name, d1, d2 in sc.extreme_cases():
        dot = sc.dot_of(d1, d2)
        if name.startswith("full"):
            assert dot.max() == 255 * 255 * 128 < 2 ** 23
        if name.startswith("above"):
            assert np.count_nonzero(dot > 2 ** 18) >= (2 if name == "above_2_18" else 1)
        for distmax in sc.DISTMAX:
            for ratiomax in sc.RATIOMAX:
                seen += len(assert_oracle_is_closed_form(d1, d2, distmax, ratiomax, f"{name} {distmax} {ratiomax}"))
    assert seen > 0


# ---- the alignment contract -------------------------------------------------------------------------------------------------------------
# Run in a child process that sees no CUDA device: a library without the host-side check would go on to the CUDA runtime and fail there
# instead of touching memory, on any machine.
_CHILD = r"""
import ctypes as C, json, sys
sys.path.insert(0, sys.argv[1])
from bundlefusion_b200 import _capi as capi
L = capi.lib()
def job(p1, n1, p2, n2):
    j = capi.BFSiftMatchJob()
    j.d_des1, j.num1, j.d_des2, j.num2 = p1, n1, p2, n2
    j.out.d_numMatches, j.out.d_distances, j.out.d_keyPointIndices = 0x7f0000000000, 0x7f0000001000, 0x7f0000002000
    return j
base = 0x7f0000100000
def run(*jobs):
    arr = (capi.BFSiftMatchJob * len(jobs))(*jobs)
    return L.bfSiftMatchBatch(arr, len(jobs), 0.7, 0.8)
out = {}
for off in (1, 4, 8):
    out["des1+%d" % off] = run(job(base + off, 10, base + 0x10000, 20))
    out["des2+%d" % off] = run(job(base, 10, base + 0x10000 + off, 20))
    out["second_job+%d" % off] = run(job(base, 10, base + 0x10000, 20), job(base + 0x20000, 5, base + 0x30000 + off, 7))
out["empty_null_next_to_aligned"] = run(job(None, 0, None, 0), job(base, 10, base + 0x10000, 20), job(base + 3, 0, None, 4))
print(json.dumps(out))
"""


def test_misaligned_descriptor_arrays_are_refused_on_the_host():
    """a live job whose d_des1 or d_des2 is 1, 4 or 8 bytes past a 16-byte boundary makes bfSiftMatchBatch return cudaErrorInvalidValue before
    any CUDA call; empty jobs (NULL or misaligned pointers, never read) next to a live aligned one are not refused by that check"""
    out = run_without_device(_CHILD)
    for k, rc in out.items():
        if k == "empty_null_next_to_aligned":
            assert rc != 1, (k, rc)                      # goes on to the CUDA runtime, which has no device here
        else:
            assert rc == 1, (k, rc)                      # cudaErrorInvalidValue

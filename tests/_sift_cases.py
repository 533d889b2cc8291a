"""Descriptor sets at the descriptor matcher's boundaries (row a18), shared by test_sift_match_boundaries_oracle.py (the oracle against a
closed-form statement of the matching rule) and test_sift_match_sweeps_gpu.py (both CUDA sweeps against the oracle and each other).

The closed form is written from the rule, not from the oracle's lanes and tree nor from the kernels' packed words:
  * a row's (column's) winner among equal maxima is the index with the smallest (brev5(lane) << 24) | index, lane = index % 32 for rows
    and (index / 4) % 32 for columns; a maximum of 0 has no winner (a product must be > 0 to be a candidate);
  * "second" is the second largest value of the multiset (a duplicated maximum is its own second; 0 when there is no other value);
  * dist = acos(min(v / 2^18, 1)) in float32; accepted iff dist < distmax and dist < dist(second) * ratiomax; a match is a column whose
    accepted winner row has that column as its accepted winner (the mutual check of test_sift_oracle.numpy_matches)."""
import itertools

import numpy as np

from bundlefusion_b200 import synth

F = np.float32

# image-2 positions of a row tie: 32-column slices (0..4, 16, 31 | 32, 33), mma.sync steps of 64, wgmma tiles of 128 and the 4-stage ring
# (512 = the first refill, 1024 / 1151 = the third phase of stages 0 and 0 / 0), lane 0 recurring at 32 k
P_SET = (0, 1, 2, 3, 4, 16, 31, 32, 33, 63, 64, 96, 127, 128, 129, 160, 255, 256, 384, 511, 512, 513, 640, 1023, 1024, 1151)
# image-1 rows of a column tie: 4-row blocks (0 1 3 | 4 5 7 | 8), the 128-row lane cycle (0 / 128, 4 / 132, 124), the 64- and 128-row CTA and
# warpgroup splits, and the column pass's ring over image 1 (511 / 512 / 513, 640, 1023 / 1024, 1151)
Q_SET = (0, 1, 3, 4, 5, 7, 8, 31, 32, 63, 64, 65, 124, 127, 128, 129, 131, 132, 255, 256, 384, 511, 512, 513, 516, 640, 1023, 1024, 1151)
DISTMAX = (0.0, 0.7, 4.0)
RATIOMAX = (0.0, 0.8, 1.0, 1.5)


# ---- the closed form ------------------------------------------------------------------------------------------------------------------------
def brev5(x):
    x = np.asarray(x, np.int64)
    return ((x & 1) << 4) | ((x & 2) << 2) | (x & 4) | ((x & 8) >> 2) | ((x & 16) >> 4)


def tie_keys(n: int, column: bool) -> np.ndarray:
    idx = np.arange(n, dtype=np.int64)
    lane = ((idx >> 2) if column else idx) & 31
    return (brev5(lane) << 24) | idx


def best_second(m: np.ndarray, keys: np.ndarray):
    """per row of m (int64 [r, c]): winner index (-1 when the maximum is 0), best value, second value of the multiset"""
    r, c = m.shape
    v1 = m.max(axis=1)
    win = np.where(m == v1[:, None], keys[None, :], np.iinfo(np.int64).max).min(axis=1) & 0xFFFFFF
    win = np.where(v1 > 0, win, -1)
    v2 = np.partition(m, c - 2, axis=1)[:, c - 2] if c > 1 else np.zeros(r, np.int64)
    return win, v1, v2


def dist_of(v):
    return np.arccos(np.minimum(np.asarray(v).astype(F) * F(2.0 ** -18), F(1.0))).astype(F)


def dot_of(d1, d2) -> np.ndarray:
    """exact int64 products (float64 sums of < 2^24 terms of < 2^16 are exact)"""
    return np.rint(np.asarray(d1, np.float64) @ np.asarray(d2, np.float64).T).astype(np.int64)


def row_rule(dot: np.ndarray, distmax: float, ratiomax: float, column: bool = False):
    """(accepted winner or -1, dist of the best) per row of dot; column=True applies the column lane rule to the rows of dot"""
    win, v1, v2 = best_second(dot, tie_keys(dot.shape[1], column))
    dist, distn = dist_of(v1), dist_of(v2)
    ok = (dist < F(distmax)) & (dist < distn * F(ratiomax))
    return np.where(ok, win, -1), dist


def closed_form_matches(dot: np.ndarray, distmax: float, ratiomax: float):
    """every mutual match (image-1 feature, image-2 feature, dist), ascending image-2 feature"""
    n1, n2 = dot.shape
    if n1 == 0 or n2 == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, F)
    rres, rdist = row_rule(dot, distmax, ratiomax)
    cres, _ = row_rule(dot.T, distmax, ratiomax, column=True)
    j = np.nonzero((cres >= 0) & (rres[np.maximum(cres, 0)] == np.arange(n2)))[0]
    return cres[j], j, rdist[cres[j]]


# ---- descriptor sets ------------------------------------------------------------------------------------------------------------------------
def tie_descriptor(rng) -> np.ndarray:
    """the lattice's descriptor D: supported on bins 0..63, norm ~480, so that 0 < dist(D . D) < 0.7 (a tie can be accepted at ratiomax > 1)"""
    v = (0.3 + rng.random(64)) * (rng.random(64) < 0.8)
    v[0] += 0.5
    d = np.zeros(128, np.uint8)
    d[:64] = np.clip(np.floor(v / np.linalg.norm(v) * 480.0 + 0.5), 0, 255)
    dd = int(d.astype(np.int64) @ d)
    assert 0 < dist_of(dd) < 0.6 and dd + 8 * int(d.sum()) < 2 ** 18
    return d


def fill(rng, n: int, zero_low: bool = False) -> np.ndarray:
    """unrelated SiftGPU-normalised descriptors with bins 0..63 halved (zeroed: zero_low), so that none reaches D . D against D"""
    f = synth.make_sift_descriptors(n, seed=int(rng.integers(1 << 30)))
    f[:, :64] = 0 if zero_low else f[:, :64] // 2
    return f


def boosted(d: np.ndarray) -> np.ndarray:
    """a descriptor whose product with d is larger than d . d (a unique best above a tie)"""
    e = d.astype(np.int64)
    e[:64] = np.minimum(e[:64] + (e[:64] > 0) * 4, 255)
    return e.astype(np.uint8)


def _assert_ties(dot, rows, cols, second=False, zero=False):
    """the lattice's constructed value really ties: the maximum (second=True: the second value, under a unique maximum) of each listed row
    (and of each listed column) occurs at least twice; zero=True: that maximum is 0"""
    for m, idx in ((dot, rows), (dot.T, cols)):
        for i in idx:
            line = m[i]
            top = line.max()
            if zero:
                assert top == 0 and len(line) >= 2
            elif second:
                assert np.count_nonzero(line == top) == 1
                nxt = line[line < top].max()
                assert np.count_nonzero(line == nxt) >= 2, "second value does not tie"
            else:
                assert top > 0 and np.count_nonzero(line == top) >= 2, "maximum does not tie"


def lattice(rng, P, Q, n1, n2, kind="tie", best_at=None):
    """one job: D at image-2 positions P and image-1 rows Q, unrelated descriptors elsewhere.  kind "tie": the rows of Q tie over P when
    |P| >= 2, the columns of P tie over Q when |Q| >= 2; "second_row" / "second_col": a boosted descriptor at image-2 position (image-1 row)
    best_at is the unique best of the rows of Q (columns of P) and the tie over P (Q) is their second value; "zero_row" / "zero_col": every
    product of the rows of Q (columns of P) is 0.  Returns (d1, d2); asserts the tie it was built for."""
    zr, zc = kind == "zero_row", kind == "zero_col"
    d1, d2 = fill(rng, n1, zero_low=zc), fill(rng, n2, zero_low=zr)
    D = tie_descriptor(rng)
    d2[list(P)] = D
    d1[list(Q)] = D
    if kind == "second_row":
        d2[best_at] = boosted(D)
    if kind == "second_col":
        d1[best_at] = boosted(D)
    dot = dot_of(d1, d2)
    if kind == "tie":
        _assert_ties(dot, Q if len(P) >= 2 else (), P if len(Q) >= 2 else ())
        assert len(P) >= 2 or len(Q) >= 2
    elif kind == "second_row":
        _assert_ties(dot, Q, (), second=True)
    elif kind == "second_col":
        _assert_ties(dot, (), P, second=True)
    else:
        _assert_ties(dot, Q if zr else (), P if zc else (), zero=True)
    return d1, d2


def row_winner(P) -> int:
    """the closed form's winner among tied image-2 positions P"""
    return min(P, key=lambda p: (int(brev5(p & 31)) << 24) | p)


def col_winner(Q) -> int:
    """the closed form's winner among tied image-1 rows Q"""
    return min(Q, key=lambda q: (int(brev5((q >> 2) & 31)) << 24) | q)


class Lattice:
    """one job of the tie batch: reveal = the (image-1, image-2) match it must produce at ratiomax > 1 (None: none), pure_tie = that match
    exists only because a tie was accepted (it must vanish at ratiomax < 1)"""

    def __init__(self, name, d1, d2, reveal=None, pure_tie=False):
        self.name, self.d1, self.d2, self.reveal, self.pure_tie = name, d1, d2, reveal, pure_tie


def lattice_jobs(seed: int = 0, triples: int = 24, both: int = 6):
    """the tie lattices of one batch: every pair and some random triples of P_SET (one image-1 row holds D), the same of Q_SET (one image-2
    feature holds D), a few with ties on both sides, seconds that tie under a unique best, ties at 0.  Returns [Lattice]."""
    rng = np.random.default_rng(seed)
    out = []
    sets_p = list(itertools.combinations(P_SET, 2)) + [tuple(sorted(rng.choice(P_SET, 3, replace=False).tolist())) for _ in range(triples)]
    for P in sets_p:
        n1 = int(rng.integers(1, 9)); n2 = max(P) + 1 + int(rng.integers(0, 40)); q = int(rng.integers(0, n1))
        out.append(Lattice(f"P{P}", *lattice(rng, P, (q,), n1, n2), (q, row_winner(P)), True))
    sets_q = list(itertools.combinations(Q_SET, 2)) + [tuple(sorted(rng.choice(Q_SET, 3, replace=False).tolist())) for _ in range(triples)]
    for Q in sets_q:
        n2 = int(rng.integers(1, 9)); n1 = max(Q) + 1 + int(rng.integers(0, 40)); p = int(rng.integers(0, n2))
        out.append(Lattice(f"Q{Q}", *lattice(rng, (p,), Q, n1, n2), (col_winner(Q), p), True))
    for _ in range(both):
        P = tuple(sorted(rng.choice(P_SET, 3, replace=False).tolist())); Q = tuple(sorted(rng.choice(Q_SET, 3, replace=False).tolist()))
        out.append(Lattice(f"P{P}Q{Q}", *lattice(rng, P, Q, max(Q) + 1 + int(rng.integers(0, 9)), max(P) + 1 + int(rng.integers(0, 9))),
                           (col_winner(Q), row_winner(P)), True))
    for P, Q, b in (((0, 1151), (2,), 600), ((31, 33, 640), (0, 5), 7), ((127, 129), (3,), 128), ((511, 512, 1024), (1,), 0)):
        out.append(Lattice(f"second_row P{P}", *lattice(rng, P, Q, max(Q) + 4, max(max(P), b) + 3, "second_row", b), (col_winner(Q), b)))
    for Q, P, b in (((0, 1151), (2,), 600), ((4, 132, 640), (0, 5), 7), ((127, 129), (3,), 128), ((511, 512, 1024), (1,), 0)):
        out.append(Lattice(f"second_col Q{Q}", *lattice(rng, P, Q, max(max(Q), b) + 3, max(P) + 4, "second_col", b), (b, row_winner(P))))
    out.append(Lattice("zero_row", *lattice(rng, (), (0, 3, 700), 701, 1100, "zero_row")))
    out.append(Lattice("zero_col", *lattice(rng, (2, 129, 1151), (), 900, 1152, "zero_col")))
    return out


def extreme_cases(seed: int = 0):
    """values at the edges: the packing bound, products above 2^18, single bins, zeros, orthogonal sets.  Returns [(name, d1, d2)]."""
    rng = np.random.default_rng(seed)
    full = np.full(128, 255, np.uint8)

    def single_bins(n, step, value=255):
        d = np.zeros((n, 128), np.uint8)
        d[np.arange(n), (np.arange(n) * step) % 128] = value
        return d
    out = []
    # 255 x 255 x 128 = 8 323 200 (< 2^23, the packed word's bound) as a unique best; the single-bin columns give 65 025 < 2^18 as the second
    sparse = single_bins(200, 3)
    d1 = np.concatenate([sparse[:70], full[None], single_bins(60, 5)])
    d2 = np.concatenate([sparse[:100], full[None], sparse[100:]])
    out.append(("full_one_row", d1, d2))
    d1m = d1.copy(); d1m[[3, 129, 70]] = full                                               # several all-255 rows: the column ties at the bound
    out.append(("full_rows", d1m, d2))
    # products above 2^18: distance clamps to 0 -- a best and a second both above it never match, a best above it over a second below does
    flat = lambda v, n: np.full((n, 128), v, np.uint8)                                      # noqa: E731
    out.append(("above_2_18", np.concatenate([flat(60, 3), flat(70, 2), synth.make_sift_descriptors(40, 3)]),
                np.concatenate([flat(60, 2), flat(20, 1), flat(80, 1), synth.make_sift_descriptors(50, 4)])))
    out.append(("above_over_below", np.concatenate([flat(60, 1), synth.make_sift_descriptors(20, 5)]),
                np.concatenate([flat(20, 1), synth.make_sift_descriptors(30, 6), flat(60, 1)])))
    # single-bin descriptors: every product is 65 025 or 0 -- ties everywhere
    out.append(("single_bin", single_bins(300, 7), single_bins(290, 5)))
    out.append(("single_bin_unique", single_bins(128, 1, 200), single_bins(128, 1, 200)[rng.permutation(128)]))
    # zero descriptors (every product 0: no candidate)
    z = np.zeros((70, 128), np.uint8)
    out.append(("zero_rows", z, synth.make_sift_descriptors(200, 7)))
    out.append(("zero_cols", synth.make_sift_descriptors(150, 8), z[:33]))
    out.append(("zero_both", z[:40], z))
    # mutually orthogonal sets: image 1 on bins 0..63, image 2 on 64..127
    a = synth.make_sift_descriptors(150, 9); a[:, 64:] = 0
    b = synth.make_sift_descriptors(170, 10); b[:, :64] = 0
    out.append(("orthogonal", a, b))
    # SiftGPU-normalised sets with planted matches, to see distmax / ratiomax decide
    p1, p2, _ = synth.make_sift_pair(260, 300, 120, noise=0.05, seed=11)
    out.append(("planted", p1, p2))
    return out

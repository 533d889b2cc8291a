"""Host side of the all-pairs keyframe search (include/bf_keyframe_search.h): the canonical pair numbering, the balanced split of the pairs
(bfKeyframePairRanges), every argument refusal of bfKeyframeSearch (answered before any CUDA call, so no GPU is needed), and the
rank-order gather of search_sharded on a two-process gloo group with the oracle's chain in place of the device search."""
import ctypes as C
import os

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from bundlefusion_b200 import keyframe_search as ks

INVALID = 1      # cudaErrorInvalidValue


def test_pair_numbering_at_every_j_boundary():
    p = 0
    for j in range(1, 200):
        for i in range(j):
            assert ks.pair_index(i, j) == p and ks.pair_of(p) == (i, j)
            p += 1
    for j in (2047, 2048, 4095):                             # large j: the square root must not round across a boundary
        for i in (0, j - 1):
            assert ks.pair_of(ks.pair_index(i, j)) == (i, j)


def _cost(nk, p):
    i, j = ks.pair_of(p)
    return int(nk[i]) * int(nk[j]) + ks.PAIR_COST


@pytest.mark.parametrize("case", ["uniform", "random", "zeros", "two", "one_heavy"])
def test_pair_ranges_cover_every_pair_once_and_balance(case):
    rng = np.random.default_rng(5)
    nk = {"uniform": np.full(40, 500), "random": rng.integers(0, 1025, 57), "zeros": np.where(np.arange(30) % 3 == 0, 0, 300),
          "two": np.array([7, 1024]), "one_heavy": np.r_[np.full(20, 3), 1024]}[case].astype(np.int32)
    P = ks.num_pairs(len(nk))
    costs = np.array([_cost(nk, p) for p in range(P)], np.int64)
    for parts in list(range(1, 9)) + [P + 3]:
        r = ks.pair_ranges(nk, parts)
        assert len(r) == parts and r[0][0] == 0 and r[-1][1] == P
        for (a, b), (c, d) in zip(r, r[1:]):
            assert a <= b == c <= d                              # contiguous, ascending
        share = costs.sum() / parts
        for a, b in r:
            assert abs(costs[a:b].sum() - share) <= costs.max(), (case, parts, a, b)


def _set(numImages=8, maxKeys=64, keys=0x10000, des=0x20000, counts=0x30000, frames=0x40000, cw=80, ch=60):
    s = ks.BFKeyframeSet()
    s.numImages, s.maxKeys, s.d_keyPoints, s.d_descriptors, s.d_numKeys, s.d_cacheFrames = numImages, maxKeys, keys, des, counts, frames
    s.cacheWidth, s.cacheHeight = cw, ch
    return s


def test_refusals_without_a_gpu():
    L = ks._bind(capi.lib())
    prm = ks.BFKeyframeSearchParams()
    L.bfKeyframeSearchDefaultParams(C.byref(prm))
    assert abs(prm.siftMatchThresh - 0.7) < 1e-7 and prm.minNumMatches == 5
    out = (0x50000, 0x60000, 0x70000)

    def call(s, p0=0, p1=1, params=prm, o=out, raw=None):
        return L.bfKeyframeSearch(C.byref(s) if s is not None else None, C.byref(params) if params is not None else None, p0, p1, o[0], o[1], o[2], 16,
                                  None, raw, None)
    assert call(_set(numImages=1)) == INVALID
    assert call(_set(numImages=0)) == INVALID
    assert call(_set(numImages=4097)) == INVALID
    assert call(_set(numImages=8), 0, 29) == INVALID             # 28 pairs
    assert call(_set(numImages=8), 5, 4) == INVALID
    assert call(_set(maxKeys=1025)) == INVALID
    assert call(_set(maxKeys=0)) == INVALID
    for off in (1, 4, 8):
        assert call(_set(des=0x20000 + off)) == INVALID
        assert call(_set(keys=0x10000 + off)) == INVALID
    for f in ("keys", "des", "counts", "frames"):
        assert call(_set(**{f: 0})) == INVALID
    assert call(None) == INVALID and call(_set(), params=None) == INVALID
    for k in range(3):
        o = list(out); o[k] = 0
        assert call(_set(), o=tuple(o)) == INVALID
    assert call(_set(), raw=C.byref(ks.BFKeyframeRawMatches(0x1000, 0, 0x2000))) == INVALID
    assert call(_set(cw=81)) == INVALID                          # verification block not a whole number of warps
    nk = np.full(4, 10, np.int32); b = np.zeros(3, np.uint64)
    assert L.bfKeyframePairRanges(nk.ctypes.data, 1, 2, b.ctypes.data) == INVALID
    assert L.bfKeyframePairRanges(nk.ctypes.data, 4, 0, b.ctypes.data) == INVALID
    assert L.bfKeyframePairRanges(np.array([3, -1, 2, 2], np.int32).ctypes.data, 4, 2, b.ctypes.data) == INVALID
    assert L.bfKeyframeSearchReserveWorkspace(1, 64) == INVALID and L.bfKeyframeSearchReserveWorkspace(8, 2048) == INVALID


# ---- search_sharded's range and gather logic on gloo -----------------------------------------------------------------------------------------
def _host_search(kf, params, pair_range):
    import torch
    from tests import _keyframe_cases as kc
    e, ei, _ = kc.oracle_range(*kf, pair_range)
    return {"entries": torch.from_numpy(e), "key_indices": torch.from_numpy(ei.view(np.int32))}


class _HostSet(tuple):
    """the keyframe set as search_sharded reads it on the host: num_keys and the tuple the oracle chain takes"""
    @property
    def num_keys(self):
        return self[2]


def _worker(rank, world, port, path):
    import torch.distributed as dist
    from tests import _keyframe_cases as kc
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        kf = _HostSet(kc.make_set([40, 0, 35, 60, 1, 50, 45, 30], 64, seed=3))
        res = ks.search_sharded(kf, None, search_fn=_host_search)
        np.savez(f"{path}.{rank}.npz", entries=res["entries"].numpy(), key_indices=res["key_indices"].numpy(), count=res["count"], range=np.array(res["range"]))
    finally:
        dist.destroy_process_group()


def test_search_sharded_gathers_the_unsharded_list_on_gloo(tmp_path):
    import socket

    import torch.multiprocessing as mp
    from tests import _keyframe_cases as kc
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]
    path = str(tmp_path / "out")
    mp.start_processes(_worker, args=(2, port, path), nprocs=2, join=True, start_method="spawn")
    keys, des, nk, cache = kc.make_set([40, 0, 35, 60, 1, 50, 45, 30], 64, seed=3)
    want_e, want_i, _ = kc.oracle_range(keys, des, nk, cache, (0, ks.num_pairs(len(nk))))
    assert len(want_e) > 100                                        # most pairs survive: the comparison is not vacuous
    ranges = ks.pair_ranges(nk, 2)
    for r in range(2):
        got = np.load(f"{path}.{r}.npz")
        assert tuple(got["range"]) == ranges[r] and ranges[r][0] < ranges[r][1]
        assert int(got["count"]) == len(want_e)
        np.testing.assert_array_equal(got["entries"], want_e)
        np.testing.assert_array_equal(got["key_indices"].view(np.uint32), want_i)

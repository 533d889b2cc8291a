"""The all-pairs keyframe search (bfKeyframeSearch) on the device against what it restates:
  * raw matches equal bfSiftMatchBatch's bytes for every pair (key counts 0, 1, 127-129, 1024 = the limit, the 128 cap, wave boundaries);
  * the whole search equals the per-image composition of the existing calls (bfSiftMatchBatch over 0..j-1, sort, Kabsch, surface area, dense
    verify, bfSiftAddCurrToResiduals) byte for byte, and the oracle's chain on a small set;
  * sub-ranges concatenate to the whole range; an undersized list holds the prefix and the counter the full count;
  * over the frame loop's own keyframes it reproduces the loop's global correspondence list;
  * after a reservation, calls do not grow the workspace."""
import ctypes as C

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from bundlefusion_b200 import keyframe_search as ks
from tests import _keyframe_cases as kc

pytestmark = pytest.mark.gpu
RAW = 128
FILT = 25


def upload(dev, keys, des, nk, cache):
    import torch
    t = {k: torch.from_numpy(np.ascontiguousarray(cache[k], np.float32)).to(dev) for k in ("depth", "campos", "normals")}
    rec = capi.BFCUDACachedFrame()
    rec.d_depthDownsampled, rec.d_cameraposDownsampled, rec.d_normalsDownsampled = t["depth"].data_ptr(), t["campos"].data_ptr(), t["normals"].data_ptr()
    recs = np.frombuffer(bytes(rec) * len(nk), np.uint8).copy()
    K, Kinv, Kc = kc.intrinsics()
    return ks.KeyframeSet(torch.from_numpy(keys).to(dev), torch.from_numpy(des).to(dev), torch.from_numpy(np.asarray(nk, np.int32)).to(dev),
                          torch.from_numpy(recs).to(dev), kc.CW, kc.CH, Kc, Kinv, owner=t)


def compose(kf, nk):
    """the frame loop's global chain per image j with the existing entry points: (entries [n, 32], key indices [n, 2], filtered count per pair,
    raw (counter, distances, indices) per pair)"""
    import torch
    L = capi.lib()
    dev = kf.device
    N, MK = kf.descriptors.shape[:2]
    _, Kinv, Kc = kc.intrinsics()
    Kinv_c, Kc_c = (C.c_float * 16)(*Kinv.reshape(-1)), (C.c_float * 16)(*Kc.reshape(-1))
    P = kc.PARAMS
    cap = 25 * ks.num_pairs(N) + 1
    glob = torch.zeros((cap, 32), dtype=torch.uint8, device=dev); gidx = torch.zeros((cap, 2), dtype=torch.int32, device=dev)
    gnum = torch.zeros(1, dtype=torch.int32, device=dev)
    nfs, raws = [], []
    base = kf.descriptors.data_ptr()
    for j in range(1, N):
        nm = torch.zeros(j + 1, dtype=torch.int32, device=dev); dd = torch.zeros((j + 1, RAW), device=dev); ix = torch.zeros((j + 1, RAW, 2), dtype=torch.int32, device=dev)
        nf = torch.zeros(j + 1, dtype=torch.int32, device=dev); fd = torch.zeros((j + 1, FILT), device=dev); fi = torch.zeros((j + 1, FILT, 2), dtype=torch.int32, device=dev)
        T = torch.zeros((j + 1, 16), device=dev); Ti = torch.zeros((j + 1, 16), device=dev)
        jobs = (capi.BFSiftMatchJob * j)()
        for i in range(j):
            jb = jobs[i]
            jb.d_des1, jb.num1, jb.d_des2, jb.num2 = base + i * MK * 128, int(nk[i]), base + j * MK * 128, int(nk[j])
            jb.out.d_numMatches, jb.out.d_distances, jb.out.d_keyPointIndices = nm.data_ptr() + 4 * i, dd.data_ptr() + 4 * RAW * i, ix.data_ptr() + 8 * RAW * i
            jb.keyPointOffset[0], jb.keyPointOffset[1] = i * MK, j * MK
        capi.check(L.bfSiftMatchBatch(jobs, j, C.c_float(P["distmax"]), C.c_float(P["ratiomax"])), "bfSiftMatchBatch")
        raws.append((nm[:j].clone(), dd[:j].clone(), ix[:j].clone()))
        kp = kf.keys.data_ptr()
        capi.check(L.bfSiftSortKeyPointMatches(j, 0, j + 1, nm.data_ptr(), dd.data_ptr(), ix.data_ptr()), "sort")
        capi.check(L.bfSiftFilterKeyPointMatches(j, 0, j + 1, kp, nm.data_ptr(), dd.data_ptr(), ix.data_ptr(), nf.data_ptr(), fd.data_ptr(), fi.data_ptr(),
                                                 T.data_ptr(), Ti.data_ptr(), Kinv_c, P["min_matches"], P["max_res2"]), "filter")
        capi.check(L.bfSiftFilterMatchesBySurfaceArea(j, 0, j + 1, kp, nf.data_ptr(), fi.data_ptr(), Kinv_c, P["area"], None), "area")
        capi.check(L.bfSiftFilterMatchesByDenseVerify(j, 0, j + 1, kc.CW, kc.CH, Kc_c, nf.data_ptr(), T.data_ptr(), kf.cache_frames.data_ptr(), P["dist"], P["normal"],
                                                      P["color"], P["err"], P["corr"], P["dmin"], P["dmax"], None), "verify")
        capi.check(L.bfSiftAddCurrToResiduals(j, 0, j + 1, glob.data_ptr(), gidx.data_ptr(), gnum.data_ptr(), nf.data_ptr(), fi.data_ptr(), kp, Kinv_c), "add")
        nfs.append(nf[:j].clone())
    torch.cuda.synchronize()
    n = int(gnum.item())
    raw = tuple(torch.cat([r[k] for r in raws]) for k in range(3))
    return glob[:n].cpu().numpy(), gidx[:n].cpu().numpy(), torch.cat(nfs).cpu().numpy(), tuple(r.cpu().numpy() for r in raw)


def _dview(ptr, shape, typestr, dev):
    import torch

    class _V:
        __cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (int(ptr), False), "version": 3, "strides": None}
    return torch.as_tensor(_V(), device=dev)


def assert_raw_equal(res, want_raw, what=""):
    gn, gd, gi = (res[k].cpu().numpy() for k in ("raw_num", "raw_dist", "raw_idx"))
    wn, wd, wi = want_raw
    np.testing.assert_array_equal(gn, wn, err_msg=what)
    for p in range(len(wn)):
        m = min(int(wn[p]), RAW)
        if m:
            assert np.array_equal(gi[p, :m], wi[p, :m]) and np.array_equal(gd[p, :m].view(np.uint32), wd[p, :m].view(np.uint32)), (what, p)


def assert_search_equal(res, want, what=""):
    we, wi, wnf, wraw = want
    assert res["count"] == len(we), what
    np.testing.assert_array_equal(res["entries"].cpu().numpy(), we, err_msg=what)
    np.testing.assert_array_equal(res["key_indices"].cpu().numpy(), wi, err_msg=what)
    np.testing.assert_array_equal(res["num_filtered"].cpu().numpy(), wnf, err_msg=what)
    assert_raw_equal(res, wraw, what)


# key counts at the boundaries of the sweep (1, 127-129, the 1024 limit), zero-key images, pairs over the 128 cap
SETS = {
    "boundaries": ([1, 127, 128, 129, 1024, 0, 300, 1024, 0, 129, 700, 64, 1, 1000], 1024, 300),
    "wave_crossing": ([int(x) for x in np.random.default_rng(9).integers(0, 60, 100)], 64, 120),       # 4950 pairs: two waves, the second partial
}


@pytest.fixture(scope="module")
def sets(cuda_device):
    out = {}
    for name, (nk, mk, pool) in SETS.items():
        host = kc.make_set(nk, mk, seed=len(nk), pool=pool)
        kf = upload(cuda_device, *host)
        out[name] = (host, kf, compose(kf, host[2]))
    return out


@pytest.mark.parametrize("name", list(SETS))
def test_whole_search_equals_the_composition_of_the_existing_calls(sets, name):
    host, kf, want = sets[name]
    res = ks.search(kf, ks.search_params(), raw=True)
    assert_search_equal(res, want, name)
    info = res["info"]
    N = kf.num_images
    assert info["pairs"] == ks.num_pairs(N) and info["waves"] == -(-ks.num_pairs(N) // ks.WAVE) and info["launches"] == 9 * info["waves"]
    assert info["entries"] == len(want[0]) and info["pairsSurviving"] == int((want[2] > 0).sum()) and info["pairsWithRawMatches"] == int((want[3][0] > 0).sum())
    assert info["pairsSurviving"] > 0
    if name == "boundaries":
        assert int(want[3][0].max()) > RAW                        # the 128 cap is reached


@pytest.mark.parametrize("name", list(SETS))
def test_sub_ranges_concatenate_and_undersized_lists_hold_the_prefix(sets, name):
    host, kf, want = sets[name]
    P = ks.num_pairs(kf.num_images)
    cuts = sorted({0, 1, P // 3, ks.WAVE if ks.WAVE < P else P // 2, P - 1, P})
    parts = [ks.search(kf, None, (a, b), raw=True) for a, b in zip(cuts, cuts[1:])]
    ents = np.concatenate([p["entries"].cpu().numpy() for p in parts])
    np.testing.assert_array_equal(ents, want[0])
    np.testing.assert_array_equal(np.concatenate([p["key_indices"].cpu().numpy() for p in parts]), want[1])
    np.testing.assert_array_equal(np.concatenate([p["num_filtered"].cpu().numpy() for p in parts]), want[2])
    for ranges in (ks.pair_ranges(host[2], 3), ks.pair_ranges(host[2], 8)):
        ents = np.concatenate([ks.search(kf, None, r)["entries"].cpu().numpy() for r in ranges])
        np.testing.assert_array_equal(ents, want[0])
    cap = len(want[0]) // 3
    small = ks.search(kf, None, capacity=cap)
    assert small["count"] == len(want[0]) and len(small["entries"]) == cap
    np.testing.assert_array_equal(small["entries"].cpu().numpy(), want[0][:cap])


def test_oracle_chain_on_a_small_set(cuda_device):
    host = kc.make_set([40, 0, 35, 60, 1, 50, 45, 30, 64, 20, 55, 33], 64, seed=3)
    res = ks.search(upload(cuda_device, *host), None)
    e, ei, nf = kc.oracle_range(*host, (0, ks.num_pairs(12)))
    assert len(e) > 100
    np.testing.assert_array_equal(res["num_filtered"].cpu().numpy(), nf)
    np.testing.assert_array_equal(res["key_indices"].cpu().numpy().view(np.uint32), ei)
    ge = res["entries"].cpu().numpy()
    np.testing.assert_array_equal(ge[:, :8], e[:, :8])            # image pair
    np.testing.assert_allclose(ge[:, 8:].view(np.float32), e[:, 8:].view(np.float32), rtol=0, atol=1e-6)


def test_reserved_workspace_does_not_grow(sets):
    host, kf, want = sets["boundaries"]
    ks.reserve_workspace(64, 1024)
    before = ks.workspace_bytes()
    assert before > 0
    for r in ((0, 10), (0, ks.num_pairs(kf.num_images))):
        ks.search(kf, None, r)
        assert ks.workspace_bytes() == before


def test_frame_loop_keyframes_reproduce_the_loops_global_list(cuda_device):
    import torch
    from bundlefusion_b200 import synth
    from bundlefusion_b200.frame_loop import FrameLoop, default_params
    W, H = 320, 240
    p = default_params(W, H)
    p.maxNumImages = 64; p.maxNumFrames = 512
    p.hash.m_hashNumBuckets = 100003; p.hash.m_numSDFBlocks = 90000
    loop = FrameLoop(p, cuda_device)
    try:
        for i in range(300):
            d, c, _ = synth.make_frame(2 * i, W, H, texture="rich")
            loop.step(torch.from_numpy(d).to(cuda_device), torch.from_numpy(c).to(cuda_device))
        torch.cuda.synchronize()
        gp = loop.global_problem()
        kf = loop.keyframes()
        N = kf.num_images
        assert N == gp.numKeyframes >= 20
        vimg = _dview(gp.d_validImages, (N,), "<i4", cuda_device).cpu().numpy()
        assert vimg.all(), "an invalid keyframe: the loop's list would hold retry pairs"
        loop_e = _dview(gp.d_correspondences, (gp.numCorrespondences, 32), "|u1", cuda_device).cpu().numpy()
        res = ks.search(kf, ks.search_params(p))
        got = res["entries"].cpu().numpy()
        ij = loop_e[:, :8].copy().view(np.uint32)
        live = ij[:, 0] != 0xFFFFFFFF
        gij = got[:, :8].copy().view(np.uint32)
        assert np.all(gij[:, 0] < gij[:, 1])
        assert np.all(ij[live, 0] < ij[live, 1]), "a retry pair (i > j) in the loop's list"
        assert len(got) == len(loop_e) and live.sum() > 0
        np.testing.assert_array_equal(got[live], loop_e[live])      # entries the loop invalidated (max-residual removal) are compared by position only
    finally:
        loop.close()

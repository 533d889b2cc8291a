"""Synthetic keyframe sets for the all-pairs search tests, and the oracle's per-frame composition of the match-filter chain over a pair range.

A set observes one pool of features: every image holds a subset of the pool at the same pixel and depth (a static camera), with its own
descriptor noise, so the pairs' matches fit the identity transform and most pairs survive every filter; all images share one dense-cache
frame of a textured plane."""
import numpy as np

from bundlefusion_b200 import synth
from bundlefusion_b200.keyframe_search import ENTRY_BYTES, pair_of

W, H, CW, CH = 640, 480, 80, 60
PARAMS = dict(distmax=0.7, ratiomax=0.8, min_matches=5, max_res2=0.0004, area=0.032, dist=0.15, normal=0.97, color=0.1, err=0.075, corr=0.02,
              dmin=0.1, dmax=4.0)


def intrinsics():
    K = np.eye(4, dtype=np.float32)
    K[0, 0] = K[1, 1] = 525.0; K[0, 2] = (W - 1) / 2.0; K[1, 2] = (H - 1) / 2.0
    Kc = K.copy()
    Kc[0, 0] *= CW / W; Kc[1, 1] *= CH / H; Kc[0, 2] *= (CW - 1) / (W - 1); Kc[1, 2] *= (CH - 1) / (H - 1)
    return K, np.linalg.inv(K.astype(np.float64)).astype(np.float32), Kc


def make_set(num_keys, max_keys, seed=0, pool=None):
    """host keyframe set: keys float32 [N, max_keys, 4], descriptors uint8 [N, max_keys, 128], num_keys int32 [N], cache frame dict"""
    rng = np.random.default_rng(seed)
    num_keys = np.asarray(num_keys, np.int32)
    M = int(pool or max(int(num_keys.max()) * 2, 64))
    base = synth.make_sift_descriptors(M, seed=seed + 1).astype(np.float64)
    xy = np.stack([rng.uniform(8, W - 8, M), rng.uniform(8, H - 8, M)], 1)
    depth = rng.uniform(1.0, 3.0, M)
    N = len(num_keys)
    keys = np.zeros((N, max_keys, 4), np.float32)
    des = np.zeros((N, max_keys, 128), np.uint8)
    for i, n in enumerate(num_keys):
        sel = np.sort(rng.choice(M, size=int(n), replace=False)) if n <= M else rng.choice(M, size=int(n), replace=True)
        keys[i, :n, 0:2] = xy[sel]; keys[i, :n, 2] = 2.0; keys[i, :n, 3] = depth[sel]
        v = base[sel] + rng.normal(0, 0.02, (int(n), 128)) * (base[sel] > 0)
        v = np.clip(v, 0, None)
        v /= np.maximum(np.linalg.norm(v, axis=1, keepdims=True), 1e-12)
        des[i, :n] = synth.quantize_descriptors(v)
    d, c, _ = synth.make_frame(0, 160, 120, texture="rich", noise=False, dropout=0.0)
    cache = synth.make_cache_frame(d, c, CW, CH)
    return keys, des, num_keys, cache


def oracle_range(keys, des, num_keys, cache, pair_range):
    """the frame loop's global chain (match, sort, Kabsch, surface area, dense verify, append) per image j on the oracle, restricted to the pairs of
    pair_range: (entries uint8 [n, 32], key indices uint32 [n, 2], filtered count per pair of the range)"""
    from oracle import oracle as orc
    p0, p1 = pair_range
    N, MK = des.shape[:2]
    K, Kinv, Kc = intrinsics()
    kp = keys.reshape(-1, 4)
    ents, idxs, nfs = [], [], []
    if p1 <= p0:
        return np.zeros((0, ENTRY_BYTES), np.uint8), np.zeros((0, 2), np.uint32), np.zeros(0, np.int32)
    j0, j1 = pair_of(p0)[1], pair_of(p1 - 1)[1]
    P = PARAMS
    for j in range(j0, j1 + 1):
        lo = max(p0, j * (j - 1) // 2) - j * (j - 1) // 2
        hi = min(p1, j * (j + 1) // 2) - j * (j - 1) // 2
        nm = np.zeros(j + 1, np.int32); dd = np.zeros((j + 1, 128), np.float32); ix = np.zeros((j + 1, 128, 2), np.uint32)
        for i in range(j):
            if num_keys[i] > 0 and num_keys[j] > 0:
                oi, od, oc = orc.sift_match(des[i, :num_keys[i]], des[j, :num_keys[j]], P["distmax"], P["ratiomax"], (i * MK, j * MK))
                nm[i] = oc; dd[i, :len(od)] = od; ix[i, :len(oi)] = oi
        dd, ix = orc.sift_sort_matches(j, 0, j + 1, nm, dd, ix)
        nf, fd, fi, T, Ti = orc.sift_filter_matches(j, 0, j + 1, kp, nm, dd, ix, Kinv, P["min_matches"], P["max_res2"])
        nf, _ = orc.sift_filter_surface_area(j, 0, j + 1, kp, nf, fi, Kinv, P["area"])
        nf, _ = orc.sift_filter_dense_verify(j, 0, j + 1, CW, CH, Kc, nf, T, [cache] * (j + 1), P["dist"], P["normal"], P["color"], P["err"], P["corr"],
                                             P["dmin"], P["dmax"])
        keep = np.zeros(j + 1, bool); keep[lo:hi] = True
        nf = np.where(keep, nf, 0).astype(np.int32)
        nfs.append(nf[lo:hi])
        e, ei = orc.sift_add_residuals(j, 0, j + 1, nf, fi, kp, Kinv)
        ents.append(e.view(np.uint8).reshape(-1, ENTRY_BYTES)); idxs.append(ei)
    return np.concatenate(ents), np.concatenate(idxs), np.concatenate(nfs)

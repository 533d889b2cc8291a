"""All-pairs correspondence search over a keyframe set (include/bf_keyframe_search.h; csrc/keyframe_search.cu).

``search`` returns the global correspondence list of every keyframe pair (i < j) in the canonical order p(i, j) = j (j - 1) / 2 + i, matched
and filtered as the frame loop's global bundler does it.  ``search_sharded`` splits the pairs over the ranks of a process group
(``pair_ranges``), searches each rank's range and all-gathers the parts in rank order, so every rank ends with the whole list."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _capi as capi

MAX_IMAGES = 4096
MAX_KEYS = 1024
WAVE = 4096
PAIR_COST = 16384
ENTRY_BYTES = 32              # BFEntryJ
ROW_BYTES = ENTRY_BYTES + 8   # an entry and its key-index pair, as search_sharded gathers them


class BFKeyframeSet(C.Structure):
    _fields_ = [("numImages", C.c_uint32), ("maxKeys", C.c_uint32), ("d_keyPoints", C.c_void_p), ("d_descriptors", C.c_void_p), ("d_numKeys", C.c_void_p),
                ("d_cacheFrames", C.c_void_p), ("cacheWidth", C.c_uint32), ("cacheHeight", C.c_uint32), ("cacheIntrinsics", C.c_float * 16),
                ("siftIntrinsicsInv", C.c_float * 16)]


class BFKeyframeSearchParams(C.Structure):
    _fields_ = [("siftMatchThresh", C.c_float), ("siftMatchRatioMax", C.c_float), ("minNumMatches", C.c_uint32), ("maxKabschResidual2", C.c_float),
                ("surfAreaPcaThresh", C.c_float), ("projCorrDistThres", C.c_float), ("projCorrNormalThres", C.c_float), ("projCorrColorThresh", C.c_float),
                ("verifySiftErrThresh", C.c_float), ("verifySiftCorrThresh", C.c_float), ("sensorDepthMin", C.c_float), ("sensorDepthMax", C.c_float)]


class BFKeyframeRawMatches(C.Structure):
    _fields_ = [("d_numMatches", C.c_void_p), ("d_distances", C.c_void_p), ("d_keyPointIndices", C.c_void_p)]


class BFKeyframeSearchInfo(C.Structure):
    _fields_ = [("pairs", C.c_uint64), ("waves", C.c_uint32), ("launches", C.c_uint32), ("pairsWithRawMatches", C.c_uint64), ("pairsSurviving", C.c_uint64),
                ("entries", C.c_uint64)]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


assert C.sizeof(BFKeyframeSet) == 176 and C.sizeof(BFKeyframeSearchParams) == 48 and C.sizeof(BFKeyframeSearchInfo) == 40


def _bind(L):
    if getattr(L, "_keyframe_search_bound", False):
        return L
    vp, P = C.c_void_p, C.POINTER
    L.bfKeyframeSearchDefaultParams.argtypes = [P(BFKeyframeSearchParams)]
    L.bfKeyframeSearchDefaultParams.restype = None
    L.bfKeyframeSearch.argtypes = [P(BFKeyframeSet), P(BFKeyframeSearchParams), C.c_uint64, C.c_uint64, vp, vp, vp, C.c_uint32, vp, P(BFKeyframeRawMatches),
                                   P(BFKeyframeSearchInfo)]
    L.bfKeyframePairRanges.argtypes = [vp, C.c_uint32, C.c_uint32, vp]
    L.bfKeyframeSearchReserveWorkspace.argtypes = [C.c_uint32, C.c_uint32]
    L.bfKeyframeSearchWorkspaceBytes.restype = C.c_size_t
    L._keyframe_search_bound = True
    return L


def pair_index(i: int, j: int) -> int:
    """canonical number of pair (i, j), i < j"""
    return j * (j - 1) // 2 + i


def pair_of(p: int) -> tuple[int, int]:
    """(i, j) of canonical pair p"""
    j = int((1 + np.sqrt(1 + 8 * float(p))) / 2)
    while j * (j - 1) // 2 > p:
        j -= 1
    while (j + 1) * j // 2 <= p:
        j += 1
    return p - j * (j - 1) // 2, j


def num_pairs(n: int) -> int:
    return n * (n - 1) // 2


def pair_ranges(num_keys, parts: int) -> list[tuple[int, int]]:
    """bfKeyframePairRanges: the balanced split of the canonical pair order into `parts` contiguous ranges (cost n_i n_j + PAIR_COST per pair)"""
    nk = np.ascontiguousarray(np.asarray(num_keys), np.int32)
    bounds = np.zeros(parts + 1, np.uint64)
    capi.check(_bind(capi.lib()).bfKeyframePairRanges(nk.ctypes.data, len(nk), parts, bounds.ctypes.data), "bfKeyframePairRanges")
    return [(int(bounds[k]), int(bounds[k + 1])) for k in range(parts)]


def search_params(loop_params=None) -> BFKeyframeSearchParams:
    """thresholds of the frame loop's global bundler, from frame_loop.default_params (or the given BFFrameLoopParams)"""
    if loop_params is None:
        from .frame_loop import default_params
        loop_params = default_params(640, 480)
    p = BFKeyframeSearchParams()
    lp = loop_params
    p.siftMatchThresh, p.siftMatchRatioMax, p.minNumMatches = lp.siftMatchThresh, lp.siftMatchRatioMaxGlobal, lp.minNumMatchesGlobal
    p.maxKabschResidual2, p.surfAreaPcaThresh = lp.maxKabschResidual2, lp.surfAreaPcaThresh
    p.projCorrDistThres, p.projCorrNormalThres, p.projCorrColorThresh = lp.projCorrDistThres, lp.projCorrNormalThres, lp.projCorrColorThresh
    p.verifySiftErrThresh, p.verifySiftCorrThresh = lp.verifySiftErrThresh, lp.verifySiftCorrThresh
    p.sensorDepthMin, p.sensorDepthMax = lp.sensorDepthMin, lp.sensorDepthMax
    return p


class KeyframeSet:
    """A keyframe set on one device: keys float32 [N, maxKeys, 4], descriptors uint8 [N, maxKeys, 128], num_keys int32 [N], cache_frames: the
    BFCUDACachedFrame records [N] (device bytes), cache size and 4x4 intrinsics, the inverse SIFT intrinsics (4x4).  ``owner`` keeps the memory
    behind the pointers alive (tensors, a cache, a frame loop)."""

    def __init__(self, keys, descriptors, num_keys, cache_frames, cache_width: int, cache_height: int, cache_intrinsics, sift_intrinsics_inv, owner=None):
        self.keys, self.descriptors, self.num_keys, self.cache_frames = keys, descriptors, num_keys, cache_frames
        self.owner = owner
        s = BFKeyframeSet()
        s.numImages, s.maxKeys = int(descriptors.shape[0]), int(descriptors.shape[1])
        s.d_keyPoints, s.d_descriptors, s.d_numKeys = keys.data_ptr(), descriptors.data_ptr(), num_keys.data_ptr()
        s.d_cacheFrames = cache_frames.data_ptr()
        s.cacheWidth, s.cacheHeight = int(cache_width), int(cache_height)
        for k, v in enumerate(np.asarray(cache_intrinsics, np.float32).reshape(16)):
            s.cacheIntrinsics[k] = float(v)
        for k, v in enumerate(np.asarray(sift_intrinsics_inv, np.float32).reshape(16)):
            s.siftIntrinsicsInv[k] = float(v)
        self.struct = s
        self.device = descriptors.device

    @classmethod
    def from_struct(cls, s: BFKeyframeSet, device, owner=None) -> "KeyframeSet":
        """views of device memory someone else owns (bfFrameLoopGetKeyframes)"""
        import torch
        N, K = int(s.numImages), int(s.maxKeys)

        def view(ptr, shape, typestr):
            class _V:
                __cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (int(ptr), False), "version": 3, "strides": None}
            return torch.as_tensor(_V(), device=device)
        kf = cls.__new__(cls)
        kf.keys = view(s.d_keyPoints, (N, K, 4), "<f4")
        kf.descriptors = view(s.d_descriptors, (N, K, 128), "|u1")
        kf.num_keys = view(s.d_numKeys, (N,), "<i4")
        kf.cache_frames = view(s.d_cacheFrames, (N * C.sizeof(capi.BFCUDACachedFrame),), "|u1")
        kf.owner, kf.struct, kf.device = owner, s, torch.device(device)
        return kf

    @property
    def num_images(self) -> int:
        return int(self.struct.numImages)


def search(kf: KeyframeSet, params: BFKeyframeSearchParams | None = None, pair_range=None, capacity: int | None = None, raw: bool = False,
           info: bool = True) -> dict:
    """bfKeyframeSearch over pair_range (default: every pair).  Returns device tensors: "entries" uint8 [n, 32] (BFEntryJ), "key_indices" int32 [n, 2],
    "num_filtered" int32 [pairs] (per pair after the last filter), "count" (entries of the range), "info" (bfKeyframeSearch's info) and, with raw,
    "raw_num" int32 [pairs], "raw_dist" float32 [pairs, 128], "raw_idx" int32 [pairs, 128, 2].  capacity: entries stored (default: enough for all;
    a first call sizes the list)."""
    import torch
    L = _bind(capi.lib())
    torch.cuda.set_device(kf.device)
    L.bfSetStream(C.c_void_p(torch.cuda.current_stream(kf.device).cuda_stream))
    if params is None:
        params = search_params()
    p0, p1 = (0, num_pairs(kf.num_images)) if pair_range is None else (int(pair_range[0]), int(pair_range[1]))
    n = max(p1 - p0, 0)
    dev = kf.device
    nf = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    rawm = None
    out = {}
    if raw:
        out["raw_num"] = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
        out["raw_dist"] = torch.zeros((max(n, 1), 128), dtype=torch.float32, device=dev)
        out["raw_idx"] = torch.zeros((max(n, 1), 128, 2), dtype=torch.int32, device=dev)
        rawm = BFKeyframeRawMatches(out["raw_num"].data_ptr(), out["raw_dist"].data_ptr(), out["raw_idx"].data_ptr())
    fixed = capacity is not None
    cap = int(capacity) if fixed else min(25 * n, 1 << 20)
    while True:
        ent = torch.zeros((max(cap, 1), ENTRY_BYTES), dtype=torch.uint8, device=dev)
        idx = torch.zeros((max(cap, 1), 2), dtype=torch.int32, device=dev)
        inf = BFKeyframeSearchInfo()
        capi.check(L.bfKeyframeSearch(C.byref(kf.struct), C.byref(params), p0, p1, ent.data_ptr(), idx.data_ptr(), cnt.data_ptr(), cap, nf.data_ptr(),
                                      C.byref(rawm) if rawm is not None else None, C.byref(inf) if info else None), "bfKeyframeSearch")
        total = int(cnt.item())
        if fixed or total <= cap:
            break
        cap = total
    m = min(total, cap)
    out.update({"entries": ent[:m], "key_indices": idx[:m], "num_filtered": nf[:n], "count": total, "info": inf.as_dict() if info else None})
    if raw:
        for k in ("raw_num", "raw_dist", "raw_idx"):
            out[k] = out[k][:n]
    return out


def search_sharded(kf: KeyframeSet, params: BFKeyframeSearchParams | None = None, group=None, search_fn=None) -> dict:
    """Every rank of `group` (torch.distributed, default group) holds the same keyframe set.  Each searches its range of pair_ranges(num_keys,
    world) and the parts are all-gathered in rank order -- first the counts, then the rows (entry + key-index pair) -- so every rank returns the
    whole canonical list: "entries" uint8 [n, 32], "key_indices" int32 [n, 2], "count", "range" (this rank's pairs).  search_fn(kf, params,
    pair_range) -> dict with "entries" and "key_indices" replaces bfKeyframeSearch (a test runs the oracle there)."""
    import torch
    import torch.distributed as dist
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    nk = kf.num_keys.cpu().numpy() if hasattr(kf.num_keys, "cpu") else np.asarray(kf.num_keys)
    ranges = pair_ranges(nk, world)
    mine = ranges[rank]
    res = (search_fn or search)(kf, params, mine)
    ent, idx = res["entries"], res["key_indices"]
    rows = torch.cat([ent.reshape(-1, ENTRY_BYTES), idx.reshape(-1, 2).contiguous().view(torch.uint8).reshape(-1, 8)], 1)
    counts = [torch.zeros(1, dtype=torch.int64, device=rows.device) for _ in range(world)]
    dist.all_gather(counts, torch.tensor([rows.shape[0]], dtype=torch.int64, device=rows.device), group=group)
    counts = [int(c.item()) for c in counts]
    width = max(max(counts), 1)
    padded = torch.zeros((width, ROW_BYTES), dtype=torch.uint8, device=rows.device)
    padded[:rows.shape[0]] = rows
    parts = [torch.empty_like(padded) for _ in range(world)]
    dist.all_gather(parts, padded, group=group)
    full = torch.cat([p[:c] for p, c in zip(parts, counts)], 0)
    return {"entries": full[:, :ENTRY_BYTES].contiguous(), "key_indices": full[:, ENTRY_BYTES:].contiguous().view(torch.int32).reshape(-1, 2),
            "count": int(sum(counts)), "range": mine}


def reserve_workspace(num_images: int, max_keys: int) -> None:
    capi.check(_bind(capi.lib()).bfKeyframeSearchReserveWorkspace(num_images, max_keys), "bfKeyframeSearchReserveWorkspace")


def workspace_bytes() -> int:
    return int(_bind(capi.lib()).bfKeyframeSearchWorkspaceBytes())

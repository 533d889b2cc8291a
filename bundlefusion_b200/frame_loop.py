"""Host-side handle of the frame-loop object (include/bf_frameloop.h; csrc/frame_loop.cu): one ``step`` per sensor frame runs what
FriedLiver's frame callback runs (FL/DepthSensing/DepthSensing.cpp:966-1129: ingest, OnlineBundler::processInput, reintegrate(),
integration of the current frame, OnlineBundler::process).  The sequencing is C++ inside the library; this file only carries pointers."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _capi as capi
from ._capi import BFHashParams


class BFFrameLoopParams(C.Structure):
    _fields_ = [("depthWidth", C.c_uint32), ("depthHeight", C.c_uint32), ("colorWidth", C.c_uint32), ("colorHeight", C.c_uint32),
                ("integrationWidth", C.c_uint32), ("integrationHeight", C.c_uint32), ("siftWidth", C.c_uint32), ("siftHeight", C.c_uint32),
                ("depthIntrinsics", C.c_float * 16), ("colorIntrinsics", C.c_float * 16),
                ("submapSize", C.c_uint32), ("maxNumImages", C.c_uint32), ("maxNumKeysPerImage", C.c_uint32), ("maxNumFrames", C.c_uint32), ("maxGlobalResiduals", C.c_uint32),
                ("numLocalNonLinIterations", C.c_uint32), ("numLocalLinIterations", C.c_uint32), ("numGlobalNonLinIterations", C.c_uint32), ("numGlobalLinIterations", C.c_uint32),
                ("numOptPerResidualRemoval", C.c_uint32),
                ("sensorDepthMin", C.c_float), ("sensorDepthMax", C.c_float), ("minKeyScale", C.c_float), ("featureCountThreshold", C.c_int32),
                ("siftMatchThresh", C.c_float), ("siftMatchRatioMaxLocal", C.c_float), ("siftMatchRatioMaxGlobal", C.c_float),
                ("minNumMatchesLocal", C.c_uint32), ("minNumMatchesGlobal", C.c_uint32),
                ("maxKabschResidual2", C.c_float), ("surfAreaPcaThresh", C.c_float),
                ("projCorrDistThres", C.c_float), ("projCorrNormalThres", C.c_float), ("projCorrColorThresh", C.c_float),
                ("verifySiftErrThresh", C.c_float), ("verifySiftCorrThresh", C.c_float), ("verifyOptErrThresh", C.c_float), ("verifyOptCorrThresh", C.c_float),
                ("optMaxResThresh", C.c_float),
                ("useLocalVerify", C.c_int32), ("useLocalDense", C.c_int32), ("useComprehensiveFrameInvalidation", C.c_int32),
                ("downsampledWidth", C.c_uint32), ("downsampledHeight", C.c_uint32),
                ("colorDownSigma", C.c_float), ("depthDownSigmaD", C.c_float), ("depthDownSigmaR", C.c_float),
                ("erodeSIFTdepth", C.c_int32), ("depthFilter", C.c_int32), ("depthSigmaD", C.c_float), ("depthSigmaR", C.c_float),
                ("maxFrameFixes", C.c_uint32), ("topNActive", C.c_uint32), ("minPoseDistSqrt", C.c_float),
                ("reconstructionEnabled", C.c_int32),
                ("hash", BFHashParams),
                ("renderDepthMin", C.c_float), ("renderDepthMax", C.c_float),
                ("hashMaxSDFBlocks", C.c_uint32), ("deviceFrameSlots", C.c_uint32)]


class BFFrameLoopStatus(C.Structure):
    _fields_ = [("frame", C.c_uint32), ("validTransform", C.c_int32), ("globalTrackingLost", C.c_int32), ("transform", C.c_float * 16),
                ("numKeyPoints", C.c_uint32), ("lastMatchedFrame", C.c_int32), ("numLocalCorrespondences", C.c_uint32), ("numReintegrated", C.c_uint32),
                ("localSolved", C.c_int32), ("localValid", C.c_int32), ("numKeyframes", C.c_uint32), ("numGlobalCorrespondences", C.c_uint32),
                ("globalSolved", C.c_int32), ("globalRemoved", C.c_int32), ("numOptimizedFrames", C.c_uint32)]

    def as_dict(self):
        d = {n: getattr(self, n) for n, _ in self._fields_ if n != "transform"}
        d["transform"] = np.array(list(self.transform), np.float32).reshape(4, 4)
        return d


class BFFrameLoopFinishInfo(C.Structure):
    _fields_ = [("turns", C.c_uint32), ("numFramesPastEnd", C.c_uint32), ("denseTurn", C.c_int32), ("denseKeyframes", C.c_uint32), ("densePairs", C.c_uint32),
                ("globalSolves", C.c_uint32), ("reintegrations", C.c_uint32), ("numTransforms", C.c_uint32), ("numValidTransforms", C.c_uint32),
                ("heapFreeCount", C.c_uint32), ("valid", C.c_int32), ("done", C.c_int32)]

    def as_dict(self):
        return {"turns": self.turns, "frames_past_end": self.numFramesPastEnd, "dense_turn": self.denseTurn, "dense_keyframes": self.denseKeyframes,
                "dense_pairs": self.densePairs, "global_solves": self.globalSolves, "reintegrations": self.reintegrations, "transforms": self.numTransforms,
                "valid_transforms": self.numValidTransforms, "heap_free": self.heapFreeCount, "valid": bool(self.valid), "done": bool(self.done)}


class BFFrameLoopFuseInfo(C.Structure):
    _fields_ = [("framesFused", C.c_uint32), ("framesSkipped", C.c_uint32), ("batches", C.c_uint32), ("heapFreeCount", C.c_uint32),
                ("insertsDropped", C.c_ulonglong)]

    def as_dict(self):
        return {"frames_fused": self.framesFused, "frames_skipped": self.framesSkipped, "batches": self.batches, "heap_free": self.heapFreeCount,
                "inserts_dropped": int(self.insertsDropped)}


class BFFrameLoopHashGrowth(C.Structure):
    _fields_ = [("growths", C.c_uint32), ("discarded", C.c_uint32), ("sdfBlocks", C.c_uint32), ("buckets", C.c_uint32), ("maxSDFBlocks", C.c_uint32),
                ("insertsDropped", C.c_ulonglong), ("ceilingReached", C.c_int32)]

    def as_dict(self):
        return {"growths": self.growths, "discarded": self.discarded, "sdf_blocks": self.sdfBlocks, "buckets": self.buckets, "max_sdf_blocks": self.maxSDFBlocks,
                "inserts_dropped": int(self.insertsDropped), "ceiling_reached": bool(self.ceilingReached)}


class BFFrameLoopFrameStore(C.Structure):
    _fields_ = [("slots", C.c_uint32), ("hostStore", C.c_int32), ("residentFrames", C.c_uint32), ("deviceBytes", C.c_ulonglong), ("hostBytes", C.c_ulonglong),
                ("writeBacks", C.c_ulonglong), ("fetches", C.c_ulonglong), ("hits", C.c_ulonglong), ("evictions", C.c_ulonglong),
                ("h2dBytes", C.c_ulonglong), ("d2hBytes", C.c_ulonglong), ("pinMs", C.c_double)]

    def as_dict(self):
        return {"slots": self.slots, "host_store": bool(self.hostStore), "resident_frames": self.residentFrames, "device_bytes": int(self.deviceBytes),
                "host_bytes": int(self.hostBytes), "write_backs": int(self.writeBacks), "fetches": int(self.fetches), "hits": int(self.hits),
                "evictions": int(self.evictions), "h2d_bytes": int(self.h2dBytes), "d2h_bytes": int(self.d2hBytes), "pin_ms": float(self.pinMs)}


class BFFrameLoopGlobalProblem(C.Structure):
    _fields_ = [("d_correspondences", C.c_void_p), ("numCorrespondences", C.c_uint32), ("numKeyframes", C.c_uint32), ("d_validImages", C.c_void_p),
                ("d_trajectory", C.c_void_p), ("d_cacheFrames", C.c_void_p), ("cacheWidth", C.c_uint32), ("cacheHeight", C.c_uint32),
                ("intrinsics", C.c_float * 4), ("maxNumImages", C.c_uint32), ("maxCorrPerImage", C.c_uint32)]


CUDA_ERROR_NOT_READY = 600


def default_params(width: int, height: int) -> BFFrameLoopParams:
    L = _bind(capi.lib())
    p = BFFrameLoopParams()
    L.bfFrameLoopDefaultParams(C.byref(p), width, height)
    return p


def growth_size(blocks: int, live: int, reserve: int, ceiling: int, init_blocks: int, init_buckets: int) -> tuple:
    """the loop's growth-size rule (bfFrameLoopHashGrowthSize): (new heap blocks, new bucket count)"""
    L = _bind(capi.lib())
    b, k = C.c_uint32(), C.c_uint32()
    L.bfFrameLoopHashGrowthSize(blocks, live, reserve, ceiling, init_blocks, init_buckets, C.byref(b), C.byref(k))
    return b.value, k.value


def _bind(L):
    if getattr(L, "_frameloop_bound", False):
        return L
    vp = C.c_void_p
    L.bfFrameLoopDefaultParams.argtypes = [C.POINTER(BFFrameLoopParams), C.c_uint32, C.c_uint32]
    L.bfFrameLoopDefaultParams.restype = None
    L.bfFrameLoopCreate.argtypes = [C.POINTER(BFFrameLoopParams), C.POINTER(vp)]
    L.bfFrameLoopDestroy.argtypes = [vp]
    L.bfFrameLoopDestroy.restype = None
    L.bfFrameLoopStep.argtypes = [vp, vp, vp, C.c_int, C.POINTER(BFFrameLoopStatus)]
    L.bfFrameLoopStepAhead.argtypes = [vp, vp, vp, vp, vp, C.c_int, C.POINTER(BFFrameLoopStatus)]
    L.bfFrameLoopStepPastEnd.argtypes = [vp, C.POINTER(BFFrameLoopStatus)]
    L.bfFrameLoopFinish.argtypes = [vp, C.c_uint32, C.c_uint32, C.POINTER(BFFrameLoopFinishInfo)]
    L.bfFrameLoopGetGlobalProblem.argtypes = [vp, C.POINTER(BFFrameLoopGlobalProblem)]
    L.bfFrameLoopFuse.argtypes = [vp, C.POINTER(capi.BFHashDataStruct), C.POINTER(BFHashParams), vp, C.c_uint32, C.POINTER(BFFrameLoopFuseInfo)]
    L.bfFrameLoopGetKeyframes.argtypes = [vp, vp]
    L.bfFrameLoopGetTrajectory.argtypes = [vp, vp, C.c_uint]
    L.bfFrameLoopGetTrajectory.restype = C.c_uint
    L.bfFrameLoopGetHashData.argtypes = [vp]
    L.bfFrameLoopGetHashData.restype = C.POINTER(capi.BFHashDataStruct)
    L.bfFrameLoopGetHashParams.argtypes = [vp]
    L.bfFrameLoopGetHashParams.restype = C.POINTER(BFHashParams)
    L.bfFrameLoopGetHashGrowth.argtypes = [vp, C.POINTER(BFFrameLoopHashGrowth)]
    L.bfFrameLoopHashGrowthSize.argtypes = [C.c_uint32, C.c_uint32, C.c_ulonglong, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    L.bfFrameLoopHashGrowthSize.restype = None
    L.bfFrameLoopGetCounters.argtypes = [vp, C.c_ulonglong * 8]
    L.bfFrameLoopGetCounters.restype = None
    L.bfFrameLoopSetOverlap.argtypes = [vp, C.c_int]
    L.bfFrameLoopJoin.argtypes = [vp]
    L.bfFrameLoopSetOpLog.argtypes = [vp, C.c_int]
    L.bfFrameLoopGetOpLog.argtypes = [vp, C.POINTER(capi.BFTsdfOp), C.POINTER(C.c_uint32), C.c_uint32]
    L.bfFrameLoopGetOpLog.restype = C.c_uint32
    L.bfFrameLoopGetFrame.argtypes = [vp, C.c_uint32, C.POINTER(vp), C.POINTER(vp)]
    L.bfFrameLoopFetchFrames.argtypes = [vp, C.POINTER(C.c_uint32), C.c_uint32, C.POINTER(vp), C.POINTER(vp)]
    L.bfFrameLoopGetFrameStore.argtypes = [vp, C.POINTER(BFFrameLoopFrameStore)]
    L.bfFrameLoopSetProfiling.argtypes = [vp, C.c_int]
    L.bfFrameLoopGetStageTimes.argtypes = [vp, C.c_double * 8]
    L.bfFrameLoopGetStageTimes.restype = C.c_ulonglong
    L._frameloop_bound = True
    return L


class FrameLoop:
    """One frame loop on one device.  ``step(depth, color)``: torch cuda tensors (float32 [H,W], uint8 [H,W,4]) or pinned / plain host tensors."""

    def __init__(self, params: BFFrameLoopParams, device="cuda:0"):
        import torch
        self._torch = torch
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("FrameLoop needs a CUDA device (no CPU fallback)")
        self.lib = _bind(capi.lib())
        self.params = params
        torch.cuda.set_device(self.device)
        self.lib.bfSetStream(C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream))
        h = C.c_void_p()
        capi.check(self.lib.bfFrameLoopCreate(C.byref(params), C.byref(h)), "bfFrameLoopCreate")
        self._h = h

    def _bind_stream(self):
        t = self._torch
        t.cuda.set_device(self.device)
        self.lib.bfSetStream(C.c_void_p(t.cuda.current_stream(self.device).cuda_stream))

    def step(self, depth, color, next_depth=None, next_color=None) -> BFFrameLoopStatus:
        """one frame; with (next_depth, next_color) -- the frame the NEXT call will pass -- that frame's upload, ingest, SIFT detection and dense cache
        are queued on the loop's feature stream during this call (bfFrameLoopStepAhead; same results)"""
        self._bind_stream()
        st = BFFrameLoopStatus()
        on_host = 0 if depth.is_cuda else 1
        if next_depth is None:
            capi.check(self.lib.bfFrameLoopStep(self._h, C.c_void_p(depth.data_ptr()), C.c_void_p(color.data_ptr()), on_host, C.byref(st)), "bfFrameLoopStep")
        else:
            if next_depth.is_cuda != depth.is_cuda:
                raise ValueError("the announced frame must live where the current one does (both device or both host)")
            capi.check(self.lib.bfFrameLoopStepAhead(self._h, C.c_void_p(depth.data_ptr()), C.c_void_p(color.data_ptr()), C.c_void_p(next_depth.data_ptr()),
                                                     C.c_void_p(next_color.data_ptr()), on_host, C.byref(st)), "bfFrameLoopStepAhead")
        return st

    def step_past_end(self) -> BFFrameLoopStatus:
        self._bind_stream()
        st = BFFrameLoopStatus()
        capi.check(self.lib.bfFrameLoopStepPastEnd(self._h, C.byref(st)), "bfFrameLoopStepPastEnd")
        return st

    def finish(self, solve_frames_before_exit: int = 30, max_turns: int | None = None) -> dict:
        """The end of the recording as the reference runs it (bfFrameLoopFinish): sparse global solves up to past-end turn K =
        solve_frames_before_exit (30 in the reference's shipped settings), the dense global solve at turn K, then re-integration only until every
        frame is fused at its final pose.  max_turns defaults to K + 2 + ceil(frames / maxFrameFixes): once solving stops no pose changes and each
        frame needs at most one operation.  Returns the call's info; "done" is False when max_turns ran out first (call again to continue)."""
        self._bind_stream()
        if max_turns is None:
            fixes = max(1, int(self.params.maxFrameFixes))
            max_turns = int(solve_frames_before_exit) + 2 + (self.counters()["frames"] + fixes - 1) // fixes
        info = BFFrameLoopFinishInfo()
        rc = self.lib.bfFrameLoopFinish(self._h, int(solve_frames_before_exit), int(max_turns), C.byref(info))
        if rc != CUDA_ERROR_NOT_READY:
            capi.check(rc, "bfFrameLoopFinish")
        return info.as_dict()

    def fuse(self, scene, poses=None, n: int | None = None) -> dict:
        """Fuse frames [0, n) of the frame store (default: every frame stepped) into ``scene`` (a CUDASceneRepHashSDF of any voxel size) along
        ``poses`` [n, 4, 4] camera-to-world (default: the loop's optimised trajectory) -- bfFrameLoopFuse: frames whose pose is not finite are
        skipped, the others go in batches of <= 16 with a garbage collection after each.  The loop itself does not change.  Returns the info."""
        self._bind_stream()
        scene._bind_stream()
        if n is None:
            n = self.counters()["frames"]
        T = None
        if poses is not None:
            T = np.ascontiguousarray(poses, dtype=np.float32).reshape(-1, 16)
            if len(T) < n:
                raise ValueError(f"{len(T)} poses for {n} frames")
        info = BFFrameLoopFuseInfo()
        capi.check(self.lib.bfFrameLoopFuse(self._h, C.byref(scene.m_hashData), C.byref(scene.m_hashParams), None if T is None else T.ctypes.data, int(n),
                                            C.byref(info)), "bfFrameLoopFuse")
        scene.m_numIntegratedFrames += info.framesFused
        return info.as_dict()

    def fit_hash_params(self, voxel_size: float, poses=None, n: int | None = None, max_table_bytes: int | None = None):
        """Hash parameters for fuse() of frames [0, n) (default: every frame stepped) along ``poses`` (default: the optimised trajectory) at
        voxel_size, sized from a count of the blocks that fusion will allocate (fuse.BlockCounter over the frame store; frames whose pose is not
        finite are skipped, as fuse() skips them): the loop's hash parameters at voxel_size with the heap and bucket count fuse.fit_hash_params
        picks.  The loop itself does not change.  Returns (BFHashParams, report)."""
        from . import fuse
        self.join()
        if n is None:
            n = self.counters()["frames"]
        if poses is None:
            T = np.full((n, 16), -np.inf, np.float32)
            traj = self.trajectory(n).reshape(-1, 16)
            T[:len(traj)] = traj
        else:
            T = np.ascontiguousarray(poses, dtype=np.float32).reshape(-1, 16)
            if len(T) < n:
                raise ValueError(f"{len(T)} poses for {n} frames")
        fin = [f for f in range(n) if np.isfinite(T[f]).all()]
        hp = BFHashParams()
        C.memmove(C.byref(hp), C.byref(self.params.hash), C.sizeof(BFHashParams))
        hp.m_virtualVoxelSize = voxel_size
        counter = fuse.BlockCounter(hp, self.device)
        cam = fuse.integration_camera(self.params)
        g = max(1, min(8, self.frame_store()["slots"] - 2))
        for s in range(0, len(fin), g):                # fetched frames' pointers hold until the next loop call: count them before it
            group = fin[s:s + g]
            depth, _ = self.fetch_frames(group)
            counter.add(depth, T[group], cam)
        return fuse.fit_hash_params(self.params.hash, voxel_size, counter, max_table_bytes)

    def global_problem(self) -> BFFrameLoopGlobalProblem:
        """the keyframe bundle-adjustment problem as the loop holds it (its device pointers, valid until the next loop call)"""
        out = BFFrameLoopGlobalProblem()
        capi.check(self.lib.bfFrameLoopGetGlobalProblem(self._h, C.byref(out)), "bfFrameLoopGetGlobalProblem")
        return out

    def keyframes(self):
        """the global SIFT manager's keyframe set as keyframe_search.KeyframeSet (views of the loop's device memory, valid until the next loop call)"""
        from .keyframe_search import BFKeyframeSet, KeyframeSet
        out = BFKeyframeSet()
        capi.check(self.lib.bfFrameLoopGetKeyframes(self._h, C.byref(out)), "bfFrameLoopGetKeyframes")
        return KeyframeSet.from_struct(out, self.device, owner=self)

    def trajectory(self, n: int) -> np.ndarray:
        out = np.zeros((n, 4, 4), np.float32)
        m = self.lib.bfFrameLoopGetTrajectory(self._h, out.ctypes.data, n)
        return out[:m]

    def counters(self) -> dict:
        c = (C.c_ulonglong * 8)()
        self.lib.bfFrameLoopGetCounters(self._h, c)
        return dict(zip(("frames", "integrations", "reintegrations", "local_solves", "global_solves", "global_pcg_iters", "host_syncs", "keyframes"), [int(x) for x in c]))

    STAGES = ("upload_ingest", "sift_detect", "dense_cache_and_count", "match_filters_sift_pose", "tsdf_reintegrate_integrate", "local_solve", "fuse_keyframe_match", "global_solve_trajectory")

    def set_overlap(self, enable: bool) -> bool:
        """TSDF work on the loop's second stream (the reference's reconstruction thread); returns the previous setting"""
        return bool(self.lib.bfFrameLoopSetOverlap(self._h, 1 if enable else 0))

    def join(self) -> None:
        self._bind_stream()
        capi.check(self.lib.bfFrameLoopJoin(self._h), "bfFrameLoopJoin")

    def set_op_log(self, enable: bool) -> bool:
        """record every TSDF op the loop runs (bfFrameLoopSetOpLog; enabling from off starts an empty log); returns the previous setting"""
        return bool(self.lib.bfFrameLoopSetOpLog(self._h, 1 if enable else 0))

    def op_log(self):
        """the recorded ops: (kinds int32 [n], frames int32 [n], poses float32 [n, 4, 4], turns uint32 [n])"""
        n = int(self.lib.bfFrameLoopGetOpLog(self._h, None, None, 0))
        ops, turns = (capi.BFTsdfOp * max(1, n))(), np.zeros(max(1, n), np.uint32)
        m = int(self.lib.bfFrameLoopGetOpLog(self._h, ops, turns.ctypes.data_as(C.POINTER(C.c_uint32)), n))
        raw = np.frombuffer(ops, np.uint8).reshape(-1, C.sizeof(capi.BFTsdfOp))[:m]
        words = raw.view(np.int32)
        return words[:, 0].copy(), words[:, 1].copy(), raw[:, 8:].copy().view(np.float32).reshape(m, 4, 4), turns[:m].copy()

    def _views(self, d, c):
        W, H = int(self.params.integrationWidth), int(self.params.integrationHeight)

        class _View:
            def __init__(self, ptr, shape, typestr):
                self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (int(ptr), False), "version": 3, "strides": None}
        t = self._torch
        return (t.as_tensor(_View(d, (H, W), "<f4"), device=self.device), t.as_tensor(_View(c, (H, W, 4), "|u1"), device=self.device))

    def frame(self, f: int):
        """frame f as the loop's frame store holds it (bfFrameLoopGetFrame): (depth float32 [H, W], colour uint8 [H, W, 4]) torch views of the
        loop's device memory at integration resolution, no copy.  With deviceFrameSlots = 0 they are valid while the loop lives.  With device
        frame slots the frame is fetched into a slot (bfFrameLoopFetchFrames) and the views are valid until the next call on the loop: read them
        on the current stream before it, or clone them."""
        self._bind_stream()
        d, c = C.c_void_p(), C.c_void_p()
        capi.check(self.lib.bfFrameLoopGetFrame(self._h, int(f), C.byref(d), C.byref(c)), "bfFrameLoopGetFrame")
        return self._views(d.value, c.value)

    def fetch_frames(self, frames):
        """frames (at most slots - 2) made resident in the frame store (bfFrameLoopFetchFrames): (depth pointers, colour pointers), device
        addresses valid until the next call on the loop; the current stream is ordered after the copies"""
        self._bind_stream()
        f = np.ascontiguousarray(frames, dtype=np.uint32).reshape(-1)
        d, c = (C.c_void_p * max(1, len(f)))(), (C.c_void_p * max(1, len(f)))()
        capi.check(self.lib.bfFrameLoopFetchFrames(self._h, f.ctypes.data_as(C.POINTER(C.c_uint32)), len(f), d, c), "bfFrameLoopFetchFrames")
        return [int(x or 0) for x in d[:len(f)]], [int(x or 0) for x in c[:len(f)]]

    def frame_store(self) -> dict:
        """slots, device and pinned host bytes, write-backs, fetches, hits, evictions and copy bytes of the frame store (bfFrameLoopGetFrameStore)"""
        out = BFFrameLoopFrameStore()
        capi.check(self.lib.bfFrameLoopGetFrameStore(self._h, C.byref(out)), "bfFrameLoopGetFrameStore")
        return out.as_dict()

    def set_profiling(self, enable: bool) -> None:
        capi.check(self.lib.bfFrameLoopSetProfiling(self._h, 1 if enable else 0), "bfFrameLoopSetProfiling")

    def stage_times(self) -> dict:
        """mean milliseconds per step and stage (device time line) since set_profiling(True)"""
        t = (C.c_double * 8)()
        n = int(self.lib.bfFrameLoopGetStageTimes(self._h, t))
        return {"steps": n, **{k: round(t[i] / max(1, n), 4) for i, k in enumerate(self.STAGES)}}

    def hash_growth(self) -> dict:
        """growths, current heap and bucket sizes, the ceiling, inserts dropped since creation and whether the ceiling stopped a growth
        (bfFrameLoopGetHashGrowth; synchronises)"""
        self._bind_stream()
        out = BFFrameLoopHashGrowth()
        capi.check(self.lib.bfFrameLoopGetHashGrowth(self._h, C.byref(out)), "bfFrameLoopGetHashGrowth")
        return out.as_dict()

    def heap_free(self) -> int:
        out = C.c_uint(0)
        capi.check(self.lib.bfTsdfGetHeapFreeCount(self.lib.bfFrameLoopGetHashData(self._h), C.byref(out)), "bfTsdfGetHeapFreeCount")
        return out.value

    def close(self):
        if getattr(self, "_h", None):
            self.lib.bfFrameLoopDestroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

"""Host-side mirror of ``CUDASceneRepHashSDF`` (FL/DepthSensing/CUDASceneRepHashSDF.h:29-423).

Same method names, argument meaning and sequencing as the reference class, but driving the
sync-free ``bfTsdf*`` entry points of the C-ABI.  torch is used only for device memory and the
current CUDA stream (plumbing); all compute is in libbundlefusion_b200.so.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _capi as capi
from ._capi import (BF_HASH_BUCKET_SIZE, BF_SDF_BLOCK_SIZE, BF_SDF_BLOCK_VOXELS, BFDepthCameraData,
                    BFDepthCameraParams, BFHashDataStruct, BFHashParams)


def mat4_to_c(m) -> capi.BFFloat4x4:
    out = capi.BFFloat4x4()
    flat = np.asarray(m, dtype=np.float32).reshape(16)
    for i in range(16):
        out.m[i] = float(flat[i])
    return out


def mat4_inverse_f32(m) -> np.ndarray:
    """fp32 inverse (the reference inverts on the host: cuda_SimpleMatrixUtil.h:980-1100)."""
    m = np.ascontiguousarray(np.asarray(m, dtype=np.float32).reshape(16))
    out = np.empty(16, dtype=np.float32)
    fp = C.POINTER(C.c_float)
    capi.lib().bfMat4Inverse(m.ctypes.data_as(fp), out.ctypes.data_as(fp))
    return out.reshape(4, 4)


def default_hash_params(num_buckets=800000, num_sdf_blocks=200000, voxel_size=0.010, truncation=0.06,
                        trunc_scale=0.02, max_integration_distance=3.0, max_list=7,
                        weight_sample=1, weight_max=99999999) -> BFHashParams:
    """``CUDASceneRepHashSDF::parametersFromGlobalAppState`` (h:39-59) with the defaults of
    FriedLiver/zParametersDefault.txt:39-50."""
    hp = BFHashParams()
    ident = np.eye(4, dtype=np.float32)
    hp.m_rigidTransform = mat4_to_c(ident)
    hp.m_rigidTransformInverse = mat4_to_c(ident)
    hp.m_hashNumBuckets = num_buckets
    hp.m_hashBucketSize = BF_HASH_BUCKET_SIZE
    hp.m_hashMaxCollisionLinkedListSize = max_list
    hp.m_numSDFBlocks = num_sdf_blocks
    hp.m_SDFBlockSize = BF_SDF_BLOCK_SIZE
    hp.m_virtualVoxelSize = voxel_size
    hp.m_numOccupiedBlocks = 0
    hp.m_maxIntegrationDistance = max_integration_distance
    hp.m_truncScale = trunc_scale
    hp.m_truncation = truncation
    hp.m_integrationWeightSample = weight_sample
    hp.m_integrationWeightMax = weight_max
    for i in range(3):
        hp.m_streamingVoxelExtents[i] = 1.0
        hp.m_streamingGridDimensions[i] = 257
        hp.m_streamingMinGridPos[i] = -128
    hp.m_streamingInitialChunkListSize = 2000
    return hp


def camera_params(width=640, height=480, fx=None, fy=None, mx=None, my=None, depth_min=0.1, depth_max=4.0) -> BFDepthCameraParams:
    """Pinhole intrinsics of SURVEY.md section 8d (fx = fy = 525*W/640, principal point at the centre);
    depth_min/max are the *render* depth range used by the frustum test (zParametersDefault.txt:35-36)."""
    cp = BFDepthCameraParams()
    cp.fx = 525.0 * width / 640.0 if fx is None else fx
    cp.fy = 525.0 * width / 640.0 if fy is None else fy
    cp.mx = (width - 1) / 2.0 if mx is None else mx
    cp.my = (height - 1) / 2.0 if my is None else my
    cp.m_imageWidth = width
    cp.m_imageHeight = height
    cp.m_sensorDepthWorldMin = depth_min
    cp.m_sensorDepthWorldMax = depth_max
    return cp


def set_pose(hp: BFHashParams, T) -> None:
    """``setLastRigidTransform`` (h:128-134): pose and its host-computed inverse."""
    T = np.asarray(T, dtype=np.float32).reshape(4, 4)
    hp.m_rigidTransform = mat4_to_c(T)
    hp.m_rigidTransformInverse = mat4_to_c(mat4_inverse_f32(T))


class CUDASceneRepHashSDF:
    """Voxel-hashed TSDF on one GPU.  Buffers are allocated here exactly as
    ``HashDataStruct::allocate`` does (VoxelUtilHashSDF.h:124-149) and handed to the library as
    raw device pointers."""

    def __init__(self, params: BFHashParams, device="cuda:0", arithmetic: str = "fast"):
        """arithmetic: "fast" (the library default: tolerance contract of bfTsdfSetArithmetic) or "exact" (bit-identical to the
        reference's IEEE build and to the oracle).  The library setting is process-wide; this object re-asserts its own before every call."""
        import torch
        if arithmetic not in ("fast", "exact"):
            raise ValueError("arithmetic must be 'fast' or 'exact'")
        self.arithmetic = arithmetic
        self._torch = torch
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("CUDASceneRepHashSDF needs a CUDA device (no CPU fallback)")
        self.lib = capi.lib()
        self.m_hashParams = BFHashParams()
        C.memmove(C.byref(self.m_hashParams), C.byref(params), C.sizeof(BFHashParams))
        self.m_hashData = self._allocate(self.m_hashParams)
        self.m_numIntegratedFrames = 0
        self.reset()

    # ---- plumbing -----------------------------------------------------------------------
    def _allocate(self, hp: BFHashParams) -> BFHashDataStruct:
        """the buffers of a hash of hp's sizes, as HashDataStruct::allocate sizes them (kept alive as attributes of this object)"""
        torch = self._torch
        n_entries = hp.m_hashNumBuckets * BF_HASH_BUCKET_SIZE
        n_blocks = hp.m_numSDFBlocks
        kw = dict(device=self.device)
        with torch.cuda.device(self.device):
            self.d_heap = torch.empty(n_blocks, dtype=torch.int32, **kw)
            self.d_heapCounter = torch.zeros(1, dtype=torch.int32, **kw)
            self.d_hash = torch.empty(n_entries * 8, dtype=torch.int32, **kw)
            self.d_hashDecision = torch.zeros(n_entries, dtype=torch.int32, **kw)
            self.d_hashDecisionPrefix = torch.zeros(n_entries, dtype=torch.int32, **kw)
            self.d_hashCompactified = torch.empty(n_entries * 8, dtype=torch.int32, **kw)
            self.d_hashCompactifiedCounter = torch.zeros(1, dtype=torch.int32, **kw)
            self.d_SDFBlocks = torch.empty(n_blocks * BF_SDF_BLOCK_VOXELS * 3, dtype=torch.int32, **kw)
            self.d_hashBucketMutex = torch.empty(hp.m_hashNumBuckets, dtype=torch.int32, **kw)
        hd = BFHashDataStruct()
        hd.d_heap = self.d_heap.data_ptr()
        hd.d_heapCounter = self.d_heapCounter.data_ptr()
        hd.d_hashDecision = self.d_hashDecision.data_ptr()
        hd.d_hashDecisionPrefix = self.d_hashDecisionPrefix.data_ptr()
        hd.d_hash = self.d_hash.data_ptr()
        hd.d_hashCompactified = self.d_hashCompactified.data_ptr()
        hd.d_hashCompactifiedCounter = self.d_hashCompactifiedCounter.data_ptr()
        hd.d_SDFBlocks = self.d_SDFBlocks.data_ptr()
        hd.d_hashBucketMutex = self.d_hashBucketMutex.data_ptr()
        hd.m_bIsOnGPU = 1
        return hd

    def _bind_stream(self):
        torch = self._torch
        torch.cuda.set_device(self.device)
        self.lib.bfSetStream(C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream))
        self.lib.bfTsdfSetArithmetic(1 if self.arithmetic == "fast" else 0)

    @staticmethod
    def _camera_data(depth, color) -> BFDepthCameraData:
        dd = BFDepthCameraData()
        dd.d_depthData = depth.data_ptr()
        dd.d_colorData = color.data_ptr() if color is not None else None
        return dd

    # ---- reference API ------------------------------------------------------------------
    def reset(self):
        """h:147-155"""
        self._bind_stream()
        self.m_numIntegratedFrames = 0
        set_pose(self.m_hashParams, np.eye(4, dtype=np.float32))
        self.m_hashParams.m_numOccupiedBlocks = 0
        capi.check(self.lib.bfTsdfReset(C.byref(self.m_hashData), C.byref(self.m_hashParams)), "bfTsdfReset")

    def integrate(self, lastRigidTransform, depth, color, cam: BFDepthCameraParams):
        """h:65-83: alloc -> compactify -> integrate (depth: float32 [H,W] cuda, color: uint8 [H,W,4] cuda)."""
        self._bind_stream()
        set_pose(self.m_hashParams, lastRigidTransform)
        dd = self._camera_data(depth, color)
        capi.check(self.lib.bfTsdfIntegrateFrame(C.byref(self.m_hashData), C.byref(self.m_hashParams), C.byref(dd), C.byref(cam), 0),
                   "bfTsdfIntegrateFrame")
        self.m_numIntegratedFrames += 1

    def deIntegrate(self, lastRigidTransform, depth, color, cam: BFDepthCameraParams):
        """h:85-108: compactify -> de-integrate."""
        self._bind_stream()
        set_pose(self.m_hashParams, lastRigidTransform)
        dd = self._camera_data(depth, color)
        capi.check(self.lib.bfTsdfIntegrateFrame(C.byref(self.m_hashData), C.byref(self.m_hashParams), C.byref(dd), C.byref(cam), 1),
                   "bfTsdfIntegrateFrame(deIntegrate)")
        self.m_numIntegratedFrames -= 1

    def integrateBatch(self, frames, poses, depth_ptrs, color_ptrs, cam: BFDepthCameraParams):
        """n <= 16 integrations in one pass (bfTsdfIntegrateBatch): frame frames[k] of the image arrays at camera-to-world pose poses[k] [n, 4, 4],
        bit-identical to n integrate() calls in that order.  depth_ptrs / color_ptrs: the frame images as cuda tensors or raw device pointers
        (indexed by frames[k]).  Asynchronous."""
        self._bind_stream()
        f = np.ascontiguousarray(frames, dtype=np.int32).reshape(-1)
        T = np.ascontiguousarray(poses, dtype=np.float32).reshape(-1, 16)
        if len(f) != len(T):
            raise ValueError("frames and poses differ in length")
        ptr = lambda x: x if isinstance(x, int) or x is None else x.data_ptr()
        dptr = (C.c_void_p * len(depth_ptrs))(*[ptr(x) for x in depth_ptrs])
        cptr = (C.c_void_p * len(color_ptrs))(*[ptr(x) for x in color_ptrs])
        capi.check(self.lib.bfTsdfIntegrateBatch(C.byref(self.m_hashData), C.byref(self.m_hashParams), C.byref(cam), f.ctypes.data, T.ctypes.data, len(f),
                                                  C.cast(dptr, C.c_void_p), C.cast(cptr, C.c_void_p)), "bfTsdfIntegrateBatch")
        self.m_numIntegratedFrames += len(f)

    def garbageCollect(self):
        """h:110-126 (identify + free over the last compactified list)."""
        self._bind_stream()
        capi.check(self.lib.bfTsdfGarbageCollect(C.byref(self.m_hashData), C.byref(self.m_hashParams)), "bfTsdfGarbageCollect")

    def getHeapFreeCount(self) -> int:
        """h:168-172 (synchronises)."""
        self._bind_stream()
        out = C.c_uint(0)
        capi.check(self.lib.bfTsdfGetHeapFreeCount(C.byref(self.m_hashData), C.byref(out)), "bfTsdfGetHeapFreeCount")
        return out.value

    def getNumOccupiedBlocks(self) -> int:
        self._bind_stream()
        out = C.c_uint(0)
        capi.check(self.lib.bfTsdfGetNumOccupiedBlocks(C.byref(self.m_hashData), C.byref(out)), "bfTsdfGetNumOccupiedBlocks")
        self.m_hashParams.m_numOccupiedBlocks = out.value
        return out.value

    def getLastFrameStats(self) -> dict:
        self._bind_stream()
        out = (C.c_ulonglong * 4)()
        capi.check(self.lib.bfTsdfGetLastFrameStats(C.byref(self.m_hashData), out), "bfTsdfGetLastFrameStats")
        return {"E": out[0], "U": out[2], "dropped": out[3]}

    def runOps(self, ops, depth_frames, color_frames, cam: BFDepthCameraParams):
        """Replay a list of (kind, frame, pose) TSDF operations in ONE library call (bfTsdfRunOps): the re-integration
        batch of DepthSensing.cpp:854-902 without a Python round trip per operation.  Asynchronous."""
        self.runPackedOps(self.packOps(ops), self.packFrames(depth_frames, color_frames), cam)

    @staticmethod
    def packOps(ops):
        """(kind, frame, pose) tuples -> BFTsdfOp array (host-side preparation, reusable)."""
        arr = (capi.BFTsdfOp * len(ops))()
        for i, (kind, frame, pose) in enumerate(ops):
            arr[i].kind, arr[i].frame = kind, frame
            if pose is not None:
                C.memmove(arr[i].pose, np.ascontiguousarray(pose, dtype=np.float32).ctypes.data, 64)
        return arr

    @staticmethod
    def packFrames(depth_frames, color_frames):
        dptr = (C.c_void_p * len(depth_frames))(*[t.data_ptr() for t in depth_frames])
        cptr = (C.c_void_p * len(color_frames))(*[t.data_ptr() for t in color_frames])
        return (dptr, cptr)

    def runPackedOps(self, arr, frames, cam: BFDepthCameraParams):
        self._bind_stream()
        self._op_keepalive = (arr, frames)
        capi.check(self.lib.bfTsdfRunOps(C.byref(self.m_hashData), C.byref(self.m_hashParams), C.byref(cam), arr, len(arr), frames[0], frames[1]),
                   "bfTsdfRunOps")

    def rehash(self, num_sdf_blocks: int, num_buckets: int) -> dict:
        """Move the model into a new table of num_sdf_blocks voxel blocks and num_buckets buckets (bfTsdfRehash): allocate it, reset it, move
        every live block with its voxels, live-voxel counter and the last compactified list, switch to it and free the old one.  Same block set
        and voxel words keyed by position; a garbage collection issued next frees what it would have freed before.  Synchronises.  Raises (and
        keeps the old table) when the new heap cannot hold the live blocks."""
        self._bind_stream()
        old_hd, old_hp = self.m_hashData, self.m_hashParams
        old_bufs = {k: getattr(self, k) for k in ("d_heap", "d_heapCounter", "d_hash", "d_hashDecision", "d_hashDecisionPrefix", "d_hashCompactified",
                                                   "d_hashCompactifiedCounter", "d_SDFBlocks", "d_hashBucketMutex")}
        hp = BFHashParams()
        C.memmove(C.byref(hp), C.byref(old_hp), C.sizeof(BFHashParams))
        hp.m_numSDFBlocks, hp.m_hashNumBuckets = int(num_sdf_blocks), int(num_buckets)
        hd = self._allocate(hp)
        out = (C.c_ulonglong * 2)()
        rc = self.lib.bfTsdfReset(C.byref(hd), C.byref(hp))
        if rc == 0:
            rc = self.lib.bfTsdfRehash(C.byref(old_hd), C.byref(old_hp), C.byref(hd), C.byref(hp), out)
        if rc != 0:
            self.lib.bfTsdfReleaseAux(C.byref(hd))
            for k, v in old_bufs.items():
                setattr(self, k, v)
            capi.check(rc, "bfTsdfRehash")
        self.lib.bfTsdfReleaseAux(C.byref(old_hd))
        self.m_hashData, self.m_hashParams = hd, hp
        return {"moved": int(out[0]), "refused": int(out[1])}

    def getHashData(self) -> BFHashDataStruct:
        return self.m_hashData

    def getHashParams(self) -> BFHashParams:
        return self.m_hashParams

    def getNumIntegratedFrames(self) -> int:
        return self.m_numIntegratedFrames

    # ---- test helpers (device -> host snapshots) ----------------------------------------
    def download(self) -> dict:
        """Host copies of the boundary buffers in their C layouts (numpy structured arrays)."""
        t = self._torch
        t.cuda.synchronize(self.device)
        n_entries = self.m_hashParams.m_hashNumBuckets * BF_HASH_BUCKET_SIZE
        return {
            "hash": self.d_hash.cpu().numpy().reshape(n_entries, 8),
            "compactified": self.d_hashCompactified.cpu().numpy().reshape(n_entries, 8),
            "compactified_count": int(self.d_hashCompactifiedCounter.cpu().numpy()[0]),
            "heap": self.d_heap.cpu().numpy().view(np.uint32),
            "heap_counter": int(self.d_heapCounter.cpu().numpy().view(np.uint32)[0]),
            "voxels": self.d_SDFBlocks.cpu().numpy().reshape(-1, BF_SDF_BLOCK_VOXELS, 3),
            "decision": self.d_hashDecision.cpu().numpy(),
            "mutex": self.d_hashBucketMutex.cpu().numpy(),
        }

    def close(self):
        if getattr(self, "lib", None) is not None:
            self.lib.bfTsdfReleaseAux(C.byref(self.m_hashData))

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

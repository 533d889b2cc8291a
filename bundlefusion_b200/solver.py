"""Host-side mirror of ``CUDASolverBundling`` (FL/Solver/CUDASolverBundling.{h,cpp}) and of the pose-conversion part of
``SBA`` (FL/SBA.cpp:53-115): same constructor arguments, ``solve`` / ``getMaxResidual`` / ``useVerification`` semantics,
buffers allocated as the reference constructor does (CUDASolverBundling.cpp:42-86) and handed to the C-ABI as raw device
pointers.  torch is plumbing (device memory, stream)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _capi as capi
from ._capi import BFSolverInput, BFSolverParameters, BFSolverState, BFSolverStateAnalysis


# Gauss-Newton grid policies (include/bf_solver.h: bfSolverSetGridPolicy).  Every policy gives the same bits; AUTO picks by problem size.
GRID_POLICY_AUTO, GRID_POLICY_GRID, GRID_POLICY_ONE_CTA, GRID_POLICY_CLUSTER = 0, 1, 2, 3


def set_grid_policy(policy: int) -> int:
    """Force the Gauss-Newton grid policy of every later solve in this process (GRID_POLICY_AUTO restores the default).  Returns the
    previous policy.  A forced policy that cannot run a solve makes that solve fail; it never falls back."""
    rc = capi.lib().bfSolverSetGridPolicy(int(policy))
    if policy not in (GRID_POLICY_AUTO, GRID_POLICY_GRID, GRID_POLICY_ONE_CTA, GRID_POLICY_CLUSTER):
        capi.check(rc, "bfSolverSetGridPolicy")
    return rc


class DeviceCache:
    """Device-side array of ``CUDACachedFrame`` structs (FL/CUDACacheUtil.h:41-53) -- what ``CUDACache::getCacheFramesGPU()``
    hands the solver.  Built here from host arrays (dict per frame: depth, campos, intensity, intensityDerivs, normalsU, normals)."""

    def __init__(self, caches, intrinsics, device):
        import torch
        self.width, self.height = caches[0]["depth"].shape[1], caches[0]["depth"].shape[0]
        self.intrinsics = tuple(float(x) for x in intrinsics)
        self._keep = []
        arr = (capi.BFCUDACachedFrame * len(caches))()
        names = {"depth": "d_depthDownsampled", "campos": "d_cameraposDownsampled", "intensity": "d_intensityDownsampled",
                 "intensityDerivs": "d_intensityDerivsDownsampled", "normalsU": "d_normalsDownsampledUCHAR4", "normals": "d_normalsDownsampled"}
        for k, c in enumerate(caches):
            for src, dst in names.items():
                t = torch.from_numpy(np.ascontiguousarray(c[src])).to(device)
                self._keep.append(t)
                setattr(arr[k], dst, t.data_ptr())
        raw = np.frombuffer(bytes(arr), dtype=np.uint8).copy()
        self.d_frames = torch.from_numpy(raw).to(device)

    def getCacheFramesGPU(self):
        return self.d_frames


class CUDASolverBundling:
    def __init__(self, maxNumberOfImages: int, maxNumResiduals: int, device="cuda:0", max_res_thresh: float = 0.08):
        import torch
        self._torch = torch
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("CUDASolverBundling needs a CUDA device (no CPU fallback)")
        self.lib = capi.lib()
        self.m_maxNumberOfImages = maxNumberOfImages
        self.m_maxNumResiduals = maxNumResiduals
        self.m_maxCorrPerImage = int(min(max(maxNumResiduals // maxNumberOfImages, 1000), 4000))   # cpp:39
        self.m_verifyOptDistThresh, self.m_verifyOptPercentThresh = 0.02, 0.05                       # cpp:35-36
        self.m_maxResidualThresh = max_res_thresh                                                    # s_optMaxResThresh
        N, R = maxNumberOfImages, maxNumResiduals
        f = lambda n: torch.zeros(n, dtype=torch.float32, device=self.device)
        i32 = lambda n: torch.zeros(n, dtype=torch.int32, device=self.device)
        self._bufs = {}
        st = BFSolverState()
        for name in ("d_deltaRot", "d_deltaTrans", "d_rRot", "d_rTrans", "d_zRot", "d_zTrans", "d_pRot", "d_pTrans", "d_Ap_XRot", "d_Ap_XTrans",
                     "d_precondionerRot", "d_precondionerTrans"):
            self._bufs[name] = f(3 * N)
        self._bufs["d_Jp"] = f(8)                      # matrix-free J p is not used by this implementation (accepted, not needed)
        self._bufs["d_scanAlpha"] = f(2)
        self._bufs["d_rDotzOld"] = f(N)
        self._bufs["d_sumResidual"] = f(1)
        self._bufs["d_countHighResidual"] = i32(1)
        self._bufs["d_denseJtJ"] = f(8)                # the dense (6N)^2 matrix is replaced by private block-sparse storage
        self._bufs["d_denseJtr"] = f(6 * N)
        self._bufs["d_denseCorrCounts"] = f(max(1, N * (N - 1) // 2))
        self._bufs["d_xTransforms"] = f(16 * N)
        self._bufs["d_xTransformInverses"] = f(16 * N)
        self._bufs["d_denseOverlappingImages"] = i32(max(2, N * (N - 1)))
        self._bufs["d_numDenseOverlappingImages"] = i32(1)
        self._bufs["d_corrCount"] = i32(1)
        self._bufs["d_corrCountColor"] = i32(1)
        self._bufs["d_sumResidualColor"] = f(1)
        for k, v in self._bufs.items():
            setattr(st, k, v.data_ptr())
        self.m_solverState = st
        self.d_variablesToCorrespondences = i32(N * self.m_maxCorrPerImage)
        self.d_numEntriesPerRow = i32(N)
        nblk = (R + 511) // 512
        self.d_maxResidual, self.d_maxResidualIndex = f(max(nblk, 2)), i32(max(nblk, 2))
        self.d_maxOut = f(2)
        self._maxRes = (0.0, 0)
        self._keep = None

    def _bind_stream(self):
        t = self._torch
        t.cuda.set_device(self.device)
        self.lib.bfSetStream(C.c_void_p(t.cuda.current_stream(self.device).cuda_stream))

    def _make_input(self, d_corr, nCorr, d_valid, nImages, wS, wD, wC, cudaCache=None):
        si = BFSolverInput()
        si.d_correspondences = d_corr.data_ptr()
        si.d_variablesToCorrespondences = self.d_variablesToCorrespondences.data_ptr()
        si.d_numEntriesPerRow = self.d_numEntriesPerRow.data_ptr()
        si.numberOfCorrespondences, si.numberOfImages = nCorr, nImages
        si.maxNumberOfImages, si.maxCorrPerImage = self.m_maxNumberOfImages, self.m_maxCorrPerImage
        si.d_validImages = d_valid.data_ptr() if d_valid is not None else None
        if cudaCache is not None:       # cpp:237-244
            si.d_cacheFrames = cudaCache.getCacheFramesGPU().data_ptr()
            si.denseDepthWidth, si.denseDepthHeight = cudaCache.width, cudaCache.height
            for k in range(4):
                si.intrinsics[k] = cudaCache.intrinsics[k]
            self._cache_keep = cudaCache
        else:
            si.d_cacheFrames = None
        si.maxNumDenseImPairs = self.m_maxNumberOfImages * (self.m_maxNumberOfImages - 1) // 2
        arrs = [np.ascontiguousarray(w, np.float32) for w in (wS, wD, wC)]
        fp = C.POINTER(C.c_float)
        si.weightsSparse, si.weightsDenseDepth, si.weightsDenseColor = (a.ctypes.data_as(fp) for a in arrs)
        self._keep = arrs
        return si

    def _params(self, nNonLin, nLin, wS, wD, wC):
        p = BFSolverParameters()
        p.nNonLinearIterations, p.nLinIterations = nNonLin, nLin
        p.verifyOptDistThresh, p.verifyOptPercentThresh = self.m_verifyOptDistThresh, self.m_verifyOptPercentThresh
        p.highResidualThresh = float("inf")
        p.denseDistThresh, p.denseNormalThresh, p.denseColorThresh, p.denseColorGradientMin = 0.15, 0.97, 0.1, 0.005
        p.denseDepthMin, p.denseDepthMax, p.denseOverlapCheckSubsampleFactor = 0.5, 4.0, 4
        p.weightSparse, p.weightDenseDepth, p.weightDenseColor = float(wS[0]), float(wD[0]), float(wC[0])
        p.useDense = 1 if (p.weightDenseDepth > 0 or p.weightDenseColor > 0) else 0
        p.useDenseDepthAllPairwise = 1
        return p

    def solve(self, d_correspondences, numberOfCorrespondences, d_validImages, numberOfImages, nNonLinearIterations, nLinearIterations,
              weightsSparse, weightsDenseDepth=None, weightsDenseColor=None, d_rotationAnglesUnknowns=None, d_translationUnknowns=None,
              rebuildJT=True, findMaxResidual=False, cudaCache=None, usePairwiseDense=True):
        """CUDASolverBundling::solve (cpp:187-284).  d_correspondences: uint8/int32 cuda tensor holding EntryJ[]; unknowns: float32
        cuda tensors [N,3] updated in place.  Asynchronous unless findMaxResidual."""
        self._bind_stream()
        nNonLin = min(nNonLinearIterations, len(weightsSparse))
        wD = weightsDenseDepth if weightsDenseDepth is not None else [0.0] * len(weightsSparse)
        wC = weightsDenseColor if weightsDenseColor is not None else [0.0] * len(weightsSparse)
        self.m_solverState.d_xRot = d_rotationAnglesUnknowns.data_ptr()
        self.m_solverState.d_xTrans = d_translationUnknowns.data_ptr()
        si = self._make_input(d_correspondences, numberOfCorrespondences, d_validImages, numberOfImages, weightsSparse, wD, wC, cudaCache)
        par = self._params(nNonLin, nLinearIterations, weightsSparse, wD, wC)
        par.useDenseDepthAllPairwise = 1 if usePairwiseDense else 0
        capi.check(self.lib.bfSolverSolve(C.byref(si), C.byref(self.m_solverState), C.byref(par)), "bfSolverSolve")
        if findMaxResidual:
            capi.check(self.lib.bfSolverMaxResidual(C.byref(si), C.byref(self.m_solverState), C.byref(par), self.d_maxOut.data_ptr()), "bfSolverMaxResidual")
            out = self.d_maxOut.cpu().numpy()
            self._maxRes = (float(out[0]), int(out[1:2].view(np.int32)[0]))
        self._last = (si, par)

    def connect_peers(self, group=None):
        """Shard this solver's PCG over the ranks of a torch.distributed group (one process per GPU of one box): exchange regions are opened through
        CUDA IPC, rows are dealt to the ranks, every rank then calls solve() with identical inputs (include/bf_solver.h: bfSolverPeer*)."""
        import torch.distributed as dist
        self._bind_stream()
        h = (C.c_char * 64)()
        capi.check(self.lib.bfSolverPeerCreate(C.byref(self.m_solverState), C.c_uint(self.m_maxNumberOfImages), C.c_uint(self.m_maxNumResiduals), h), "bfSolverPeerCreate")
        world = dist.get_world_size(group); rank = dist.get_rank(group)
        handles = [None] * world
        dist.all_gather_object(handles, bytes(h.raw), group=group)
        blob = b"".join(handles)
        capi.check(self.lib.bfSolverPeerConnect(C.byref(self.m_solverState), rank, world, blob), "bfSolverPeerConnect")
        dist.barrier(group=group)
        return rank, world

    def disconnect_peers(self):
        capi.check(self.lib.bfSolverPeerDisconnect(C.byref(self.m_solverState)), "bfSolverPeerDisconnect")

    def getMaxResidual(self):
        """(max residual, correspondence index), cpp:41-44."""
        return self._maxRes

    def shouldRemove(self, imgIdx_i: int, imgIdx_j: int) -> bool:
        """the decision of CUDASolverBundling::getMaxResidual(curFrame, ...) (cpp:429-452)."""
        return (not (imgIdx_i == 0 and imgIdx_j < 10)) and self._maxRes[0] > self.m_maxResidualThresh

    def useVerification(self, d_correspondences, numberOfCorrespondences) -> bool:
        """cpp:454-476 (synchronises)."""
        self._bind_stream()
        si, par = self._last
        si.d_correspondences = d_correspondences.data_ptr()
        si.numberOfCorrespondences = numberOfCorrespondences
        n = self.lib.countHighResiduals(C.byref(si), C.byref(self.m_solverState), C.byref(par), None)
        return (n / max(1, numberOfCorrespondences)) >= self.m_verifyOptPercentThresh

    def getStats(self) -> dict:
        self._bind_stream()
        out = (C.c_ulonglong * 8)()
        capi.check(self.lib.bfSolverGetStats(C.byref(self.m_solverState), out), "bfSolverGetStats")
        return {"gn": out[0], "pcg": out[1], "pairs": out[2], "max_delta": out[4] * 1e-6, "error": out[5], "converged": out[6],
                "dense_overlap_pairs": out[3], "dense_weighted_pairs": out[7]}

    def getLaunchInfo(self) -> dict:
        """The last Gauss-Newton launch of this solver (host-side record, no synchronisation): policy that ran, G (the cooperative grid's
        CTA count every policy reproduces), the device's cluster cap and the resident kernel's dynamic shared memory limit in bytes."""
        out = (C.c_int * 4)()
        capi.check(self.lib.bfSolverGetLaunchInfo(C.byref(self.m_solverState), out), "bfSolverGetLaunchInfo")
        return {"policy": out[0], "ctas": out[1], "cluster_cap": out[2], "dyn_smem": out[3]}

    def getVarToCorrNumEntriesPerRow(self):
        return self.d_numEntriesPerRow

    def close(self):
        if getattr(self, "lib", None) is not None:
            self.lib.bfSolverReleaseWorkspace(C.byref(self.m_solverState))

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

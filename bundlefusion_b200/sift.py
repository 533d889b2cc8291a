"""Host-side mirror of ``SiftMatchGPU`` (FL/SiftGPU/SiftMatch.{h,cpp}) and of the pair loop of ``Bundler::matchAndFilter``
(FL/Bundler.cpp:103-137): ``SetDescriptors`` / ``GetSiftMatch`` with the reference's argument meaning, plus the batched call
that replaces the per-pair loop.  torch is plumbing (device memory, stream)."""
from __future__ import annotations

import ctypes as C

from . import _capi as capi
from ._capi import BFSiftMatchJob

MAX_MATCHES_PER_IMAGE_PAIR_RAW = 128      # FL/GlobalDefines.h:8

# Descriptor-match sweeps (include/bf_sift.h: bfSiftSetMatchSweep).  Both give the same bytes; AUTO runs wgmma + TMA where tensor maps can be encoded.
SIFT_SWEEP_AUTO, SIFT_SWEEP_WGMMA, SIFT_SWEEP_MMA = 0, 1, 2


def set_match_sweep(sweep: int) -> int:
    """Force the sweep of every later bfSiftMatchBatch in this process (SIFT_SWEEP_AUTO restores the default).  Returns the previous
    setting.  A forced wgmma sweep that cannot map a batch makes that batch fail; it never falls back."""
    rc = capi.lib().bfSiftSetMatchSweep(int(sweep))
    if sweep not in (SIFT_SWEEP_AUTO, SIFT_SWEEP_WGMMA, SIFT_SWEEP_MMA):
        capi.check(rc, "bfSiftSetMatchSweep")
    return rc


def match_info() -> tuple[int, int]:
    """(sweep that ran, number of jobs) of the last bfSiftMatchBatch that enqueued work; recorded on the host."""
    out = (C.c_int * 2)()
    capi.check(capi.lib().bfSiftGetMatchInfo(out), "bfSiftGetMatchInfo")
    return out[0], out[1]


class ImagePairMatch:
    """FL/SiftGPU/SIFTImageManager.h:38-42 -- device buffers of one image pair's raw matches."""

    def __init__(self, device):
        import torch
        self.d_numMatches = torch.zeros(1, dtype=torch.int32, device=device)
        self.d_distances = torch.zeros(MAX_MATCHES_PER_IMAGE_PAIR_RAW, dtype=torch.float32, device=device)
        self.d_keyPointIndices = torch.zeros(MAX_MATCHES_PER_IMAGE_PAIR_RAW, 2, dtype=torch.int32, device=device)

    def download(self):
        """(indices [n,2] uint32, distances [n]) of the stored matches, n = min(counter, cap)."""
        n = min(int(self.d_numMatches.item()), MAX_MATCHES_PER_IMAGE_PAIR_RAW)
        import numpy as np
        return self.d_keyPointIndices[:n].cpu().numpy().view(np.uint32), self.d_distances[:n].cpu().numpy(), int(self.d_numMatches.item())


class SiftMatchGPU:
    def __init__(self, max_sift: int = 1024, device="cuda:0"):
        import torch
        self._torch = torch
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("SiftMatchGPU needs a CUDA device (no CPU fallback)")
        self.lib = capi.lib()
        self._des = [None, None]
        self._num = [0, 0]

    def _bind_stream(self):
        t = self._torch
        t.cuda.set_device(self.device)
        self.lib.bfSetStream(C.c_void_p(t.cuda.current_stream(self.device).cuda_stream))

    def SetDescriptors(self, index: int, num: int, d_descriptors):
        """SiftMatch.cpp:110-131: d_descriptors = uint8 cuda tensor [num, 128], normalised to 512.  No copy is made, so the tensor's data must
        be 16-byte aligned (include/bf_sift.h); a misaligned one makes GetSiftMatch / matchBatch fail with cudaErrorInvalidValue."""
        self._des[index], self._num[index] = d_descriptors, int(num)

    def _job(self, des1, n1, des2, n2, ipm: ImagePairMatch, off):
        j = BFSiftMatchJob()
        j.d_des1, j.num1, j.d_des2, j.num2 = des1.data_ptr() if n1 > 0 else None, n1, des2.data_ptr() if n2 > 0 else None, n2
        j.out.d_numMatches, j.out.d_distances, j.out.d_keyPointIndices = ipm.d_numMatches.data_ptr(), ipm.d_distances.data_ptr(), ipm.d_keyPointIndices.data_ptr()
        j.keyPointOffset[0], j.keyPointOffset[1] = off
        return j

    def GetSiftMatch(self, max_match: int, imagePairMatch: ImagePairMatch, keyPointOffset=(0, 0), distmax: float = 0.7, ratiomax: float = 0.8,
                     mutual_best_match: int = 1):
        """SiftMatch.cpp:160-196 for the pair set with SetDescriptors(0, ..), SetDescriptors(1, ..).  Asynchronous."""
        if not mutual_best_match:
            raise NotImplementedError("the reference's GetBestMatch only implements the mutual-best mode (SiftMatch.cpp:176-196)")
        self._bind_stream()
        arr = (BFSiftMatchJob * 1)(self._job(self._des[0], self._num[0], self._des[1], self._num[1], imagePairMatch, keyPointOffset))
        capi.check(self.lib.bfSiftMatchBatch(arr, 1, distmax, ratiomax), "bfSiftMatchBatch")

    def matchBatch(self, pairs, distmax: float = 0.7, ratiomax: float = 0.8):
        """The pair loop of Bundler::matchAndFilter (FL/Bundler.cpp:116-137) as ONE call.
        pairs: iterable of (d_des1, num1, d_des2, num2, ImagePairMatch, keyPointOffset)."""
        self._bind_stream()
        pairs = list(pairs)
        arr = (BFSiftMatchJob * len(pairs))(*[self._job(*p) for p in pairs])
        capi.check(self.lib.bfSiftMatchBatch(arr, len(pairs), distmax, ratiomax), "bfSiftMatchBatch")


class SiftGPU:
    """Mirror of ``SiftGPU`` as ``Bundler`` drives it (FL/Bundler.cpp:55-100; FL/SiftGPU/SiftGPU.cpp): ``SetParams`` latches the image size,
    the feature-count threshold and the depth range, ``RunSIFT`` + ``GetKeyPointsAndDescriptorsCUDA`` become one asynchronous
    ``bfSiftDetect``.  The count stays on the device; ``GetFeatureNum`` synchronises to read it.
    STATUS: the CUDA path behind it has been verified under CPU emulation only (tests/test_sift_detect_emulated.py)."""

    def __init__(self, device="cuda:0"):
        import torch
        self._torch = torch
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("SiftGPU needs a CUDA device (no CPU fallback)")
        self.lib = capi.lib()
        self._p = None
        self._num = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._levels = torch.zeros(12, dtype=torch.int32, device=self.device)

    def SetParams(self, siftWidth: int, siftHeight: int, enableTiming: bool, featureCountThreshold: int, siftDepthMin: float, siftDepthMax: float,
                  depthWidth: int | None = None, depthHeight: int | None = None, minKeyScale: float = 3.0):
        """SiftGPU.cpp:224-254; depth size and minKeyScale are what the reference reads from c_siftCameraParams (FL/OnlineBundler.cpp:45-56)."""
        self._p = capi.BFSiftDetectParams(siftWidth, siftHeight, depthWidth or siftWidth, depthHeight or siftHeight, siftDepthMin, siftDepthMax, minKeyScale,
                                          int(featureCountThreshold), 0)

    def RunSIFT(self, d_intensity, d_depth, d_keyPoints, d_keyPointDescs, maxNumKeyPoints: int) -> int:
        """RunSIFT + GetKeyPointsAndDescriptorsCUDA: d_intensity float32 [H, W] in 0..1, d_depth float32 [Hd, Wd]; outputs float32
        [maxNumKeyPoints, 4] and uint8 [maxNumKeyPoints, 128] cuda tensors.  Returns 1 (launched) like the reference's success flag."""
        if self._p is None:
            raise RuntimeError("SetParams first")
        t = self._torch
        t.cuda.set_device(self.device)
        self.lib.bfSetStream(C.c_void_p(t.cuda.current_stream(self.device).cuda_stream))
        self._p.maxKeyPoints = int(maxNumKeyPoints)
        capi.check(self.lib.bfSiftDetect(C.byref(self._p), d_intensity.data_ptr(), d_depth.data_ptr(), d_keyPoints.data_ptr(), d_keyPointDescs.data_ptr(),
                                         self._num.data_ptr(), self._levels.data_ptr()), "bfSiftDetect")
        return 1

    def GetFeatureNum(self) -> int:
        return int(self._num.item())

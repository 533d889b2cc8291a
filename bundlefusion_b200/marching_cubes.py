"""Host-side mirror of the reference's ``CUDAMarchingCubesHashSDF`` (FL/DepthSensing/CUDAMarchingCubesHashSDF.{h,cpp}) over the C-ABI of
include/bf_marchingcubes.h: the triangle mesh of the fused model, its clean-up (mergeCloseVertices / removeDuplicateFaces) and the PLY file ``saveMesh`` writes."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _capi as capi
from ._capi import BFMarchingCubesParams


def marching_cubes_params(num_buckets: int, voxel_size: float = 0.01, max_num_triangles: int = 3000000, thresh_factor: float = 10.0) -> BFMarchingCubesParams:
    """CUDAMarchingCubesHashSDF::parametersFromGlobalAppState (h:21-30) with the values of zParametersDefault.txt (s_marchingCubesMaxNumTriangles, s_SDFMarchingCubeThreshFactor)"""
    p = BFMarchingCubesParams()
    p.m_maxNumTriangles = max_num_triangles
    p.m_threshMarchingCubes = p.m_threshMarchingCubes2 = np.float32(thresh_factor) * np.float32(voxel_size)
    p.m_sdfBlockSize, p.m_hashBucketSize, p.m_hashNumBuckets = 8, capi.BF_HASH_BUCKET_SIZE, num_buckets
    return p


def _bind(L):
    if getattr(L, "_mc_bound", False):
        return L
    vp, sz = C.c_void_p, C.c_size_t
    L.bfMarchingCubesCreate.argtypes = [vp, C.POINTER(vp)]
    L.bfMarchingCubesDestroy.argtypes = [vp]; L.bfMarchingCubesDestroy.restype = None
    L.bfMarchingCubesExtractIsoSurface.argtypes = [vp, vp, vp, vp, vp, C.c_int]
    L.bfMarchingCubesClearMeshBuffer.argtypes = [vp]; L.bfMarchingCubesClearMeshBuffer.restype = None
    L.bfMarchingCubesGetSoup.argtypes = [vp, C.POINTER(vp), C.POINTER(vp)]; L.bfMarchingCubesGetSoup.restype = sz
    L.bfMarchingCubesSaveMesh.argtypes = [vp, C.c_char_p, vp, C.c_int, C.c_char_p, sz]
    L.bfMarchingCubesExtract.argtypes = [vp, vp, vp, vp, vp]
    L.bfMeshMergeCloseVertices.argtypes = [vp, vp, sz, vp, sz, C.c_float, C.POINTER(sz), C.POINTER(sz)]
    L.bfMeshRemoveDuplicateFaces.argtypes = [vp, sz, C.POINTER(sz)]
    L.bfMeshSavePly.argtypes = [C.c_char_p, vp, vp, sz, vp, sz]
    L.bfMarchingCubesCount.argtypes = [vp, vp, vp, vp, vp]
    L.bfMarchingCubesExtractRange.argtypes = [vp, vp, vp, C.c_uint32, C.c_uint32, vp, vp]
    L.bfMarchingCubesExtractIsoSurfaceWhole.argtypes = [vp, vp, vp, vp, vp, C.c_int, vp]
    L.bfMarchingCubesGetLastExtraction.argtypes = [vp, C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong)]
    L._mc_bound = True
    return L


def num_chunks(num_buckets: int) -> int:
    """chunks of a table of num_buckets buckets: the count pass writes one triangle count per chunk"""
    return (int(num_buckets) * capi.BF_HASH_BUCKET_SIZE + capi.BF_MC_CHUNK_SLOTS - 1) // capi.BF_MC_CHUNK_SLOTS


def merge_close_vertices(positions: np.ndarray, colors: np.ndarray | None, faces: np.ndarray, thresh: float = 0.00001):
    """MeshData::mergeCloseVertices(thresh, approx=True) + removeDegeneratedFaces on host arrays -> (positions, colors, faces)"""
    L = _bind(capi.lib())
    pos = np.ascontiguousarray(positions, np.float32).copy(); f = np.ascontiguousarray(faces, np.uint32).copy()
    col = None if colors is None else np.ascontiguousarray(colors, np.float32).copy()
    nv, nf = C.c_size_t(0), C.c_size_t(0)
    if L.bfMeshMergeCloseVertices(pos.ctypes.data, None if col is None else col.ctypes.data, len(pos), f.ctypes.data, len(f), thresh, C.byref(nv), C.byref(nf)):
        raise ValueError("bfMeshMergeCloseVertices: invalid arguments")
    return pos[:nv.value], None if col is None else col[:nv.value], f[:nf.value]


def remove_duplicate_faces(faces: np.ndarray) -> np.ndarray:
    L = _bind(capi.lib())
    f = np.ascontiguousarray(faces, np.uint32).copy()
    nf = C.c_size_t(0)
    L.bfMeshRemoveDuplicateFaces(f.ctypes.data, len(f), C.byref(nf))
    return f[:nf.value]


def save_ply(path: str, positions: np.ndarray, colors: np.ndarray | None, faces: np.ndarray) -> None:
    L = _bind(capi.lib())
    pos = np.ascontiguousarray(positions, np.float32); f = np.ascontiguousarray(faces, np.uint32)
    col = None if colors is None else np.ascontiguousarray(colors, np.float32)
    if L.bfMeshSavePly(path.encode(), pos.ctypes.data, None if col is None else col.ctypes.data, len(pos), f.ctypes.data, len(f)):
        raise OSError(f"bfMeshSavePly({path}) failed")


class CUDAMarchingCubesHashSDF:
    def __init__(self, params: BFMarchingCubesParams, device="cuda:0"):
        import torch
        self._torch = torch
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("CUDAMarchingCubesHashSDF needs a CUDA device (no CPU fallback)")
        self.lib = _bind(capi.lib())
        self.m_params = BFMarchingCubesParams()
        C.memmove(C.byref(self.m_params), C.byref(params), C.sizeof(BFMarchingCubesParams))
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            capi.check(self.lib.bfMarchingCubesCreate(C.byref(self.m_params), C.byref(h)), "bfMarchingCubesCreate")
        self._h = h

    def _bind_stream(self):
        t = self._torch
        t.cuda.set_device(self.device)
        self.lib.bfSetStream(C.c_void_p(t.cuda.current_stream(self.device).cuda_stream))

    def extractIsoSurface(self, scene, min_corner=(0.0, 0.0, 0.0), max_corner=(0.0, 0.0, 0.0), box_enabled: bool = False) -> int:
        """scene: a ``CUDASceneRepHashSDF`` (its hash data and parameters); the triangles are appended to the mesh buffer; returns the buffer's vertex count"""
        self._bind_stream()
        lo = (C.c_float * 3)(*min_corner); hi = (C.c_float * 3)(*max_corner)
        capi.check(self.lib.bfMarchingCubesExtractIsoSurface(self._h, C.byref(scene.m_hashData), C.byref(scene.m_hashParams), lo, hi, 1 if box_enabled else 0), "bfMarchingCubesExtractIsoSurface")
        return int(self.lib.bfMarchingCubesGetSoup(self._h, None, None))

    def _box_params(self, scene, min_corner, max_corner, box_enabled):
        p = BFMarchingCubesParams()
        C.memmove(C.byref(p), C.byref(self.m_params), C.sizeof(BFMarchingCubesParams))
        p.m_boxEnabled = 1 if box_enabled else 0
        for k in range(3):
            p.m_minCorner[k], p.m_maxCorner[k] = min_corner[k], max_corner[k]
        p.m_hashNumBuckets = int(scene.m_hashParams.m_hashNumBuckets)
        return p

    def count(self, scene, min_corner=(0.0, 0.0, 0.0), max_corner=(0.0, 0.0, 0.0), box_enabled: bool = False):
        """the count pass (bfMarchingCubesCount) -> (total triangles, triangles per 512-slot chunk of the table: uint32 numpy array).  Synchronises once."""
        t = self._torch
        self._bind_stream()
        p = self._box_params(scene, min_corner, max_corner, box_enabled)
        counts = t.empty(num_chunks(p.m_hashNumBuckets), dtype=t.int32, device=self.device)
        total = t.empty(1, dtype=t.int64, device=self.device)
        capi.check(self.lib.bfMarchingCubesCount(C.byref(scene.m_hashData), C.byref(scene.m_hashParams), C.byref(p), counts.data_ptr(), total.data_ptr()),
                   "bfMarchingCubesCount")
        return int(total.item()), counts.cpu().numpy().view(np.uint32)

    def extractIsoSurfaceWhole(self, scene, min_corner=(0.0, 0.0, 0.0), max_corner=(0.0, 0.0, 0.0), box_enabled: bool = False) -> dict:
        """the whole mesh appended to the mesh buffer, in parts that fit the buffer (bfMarchingCubesExtractIsoSurfaceWhole): no triangle is dropped.
        Returns {"triangles_counted", "triangles_extracted", "chunks", "parts", "largest_part", "buffer_triangles", "buffer_enlarged", "host_syncs"}."""
        self._bind_stream()
        lo = (C.c_float * 3)(*min_corner); hi = (C.c_float * 3)(*max_corner)
        info = capi.BFMarchingCubesWholeInfo()
        capi.check(self.lib.bfMarchingCubesExtractIsoSurfaceWhole(self._h, C.byref(scene.m_hashData), C.byref(scene.m_hashParams), lo, hi, 1 if box_enabled else 0,
                                                                  C.byref(info)), "bfMarchingCubesExtractIsoSurfaceWhole")
        return {"triangles_counted": int(info.trianglesCounted), "triangles_extracted": int(info.trianglesExtracted), "chunks": int(info.chunks),
                "parts": int(info.parts), "largest_part": int(info.largestPart), "buffer_triangles": int(info.bufferTriangles),
                "buffer_enlarged": bool(info.bufferEnlarged), "host_syncs": int(info.hostSyncs)}

    def lastExtraction(self) -> tuple[int, int]:
        """(found, kept) of the last extraction: triangles its cells produced and triangles it appended; found > kept when a full buffer dropped some"""
        found, kept = C.c_ulonglong(0), C.c_ulonglong(0)
        capi.check(self.lib.bfMarchingCubesGetLastExtraction(self._h, C.byref(found), C.byref(kept)), "bfMarchingCubesGetLastExtraction")
        return int(found.value), int(kept.value)

    def soup(self):
        """the mesh buffer: (positions [n, 3], colours [n, 4]) float32 copies, three consecutive vertices per triangle"""
        pp, cp = C.c_void_p(), C.c_void_p()
        n = int(self.lib.bfMarchingCubesGetSoup(self._h, C.byref(pp), C.byref(cp)))
        if n == 0:
            return np.zeros((0, 3), np.float32), np.zeros((0, 4), np.float32)
        pos = np.ctypeslib.as_array(C.cast(pp, C.POINTER(C.c_float)), (n, 3)).copy()
        col = np.ctypeslib.as_array(C.cast(cp, C.POINTER(C.c_float)), (n, 4)).copy()
        return pos, col

    def clearMeshBuffer(self):
        self.lib.bfMarchingCubesClearMeshBuffer(self._h)

    def saveMesh(self, filename: str, transform=None, overwrite: bool = False) -> str:
        t = None if transform is None else np.ascontiguousarray(transform, np.float32)
        out = C.create_string_buffer(4096)
        if self.lib.bfMarchingCubesSaveMesh(self._h, filename.encode(), None if t is None else t.ctypes.data, 1 if overwrite else 0, out, 4096):
            raise OSError(f"bfMarchingCubesSaveMesh({filename}) failed")
        return out.value.decode()

    def close(self):
        if getattr(self, "_h", None):
            self.lib.bfMarchingCubesDestroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

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
    L.bfMeshApplyTransform.argtypes = [vp, sz, vp]
    L.bfMeshWeldWorkspaceBytes.argtypes = [C.c_uint64]; L.bfMeshWeldWorkspaceBytes.restype = sz
    L.bfMeshWeld.argtypes = [vp, C.c_uint64, C.c_float, vp, sz, vp, vp, vp, vp]
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


def apply_transform(positions: np.ndarray, transform) -> np.ndarray:
    """saveMesh's transform (bfMeshApplyTransform): p' = M (p, 1), de-homogenised, M a row-major 4x4; returns a new float32 array"""
    L = _bind(capi.lib())
    pos = np.ascontiguousarray(positions, np.float32).copy()
    t = np.ascontiguousarray(transform, np.float32)
    if t.shape != (4, 4) or L.bfMeshApplyTransform(pos.ctypes.data, len(pos), t.ctypes.data):
        raise ValueError("apply_transform: positions [n, 3] and a 4x4 transform")
    return pos


def _weld_report(info) -> dict:
    return {"triangles_in": int(info.trianglesIn), "vertices_out": int(info.verticesOut), "degenerate_faces": int(info.degenerateFaces),
            "duplicate_faces": int(info.duplicateFaces), "faces_out": int(info.facesOut), "cells": int(info.cells), "rounds": int(info.rounds),
            "host_syncs": int(info.hostSyncs)}


class Mesh:
    """an indexed mesh in device memory: positions [V, 3] float32, colors [V, 4] float32 (w = 1), faces [F, 3] int32, and the weld's report"""

    def __init__(self, positions, colors, faces, info: dict):
        self.positions, self.colors, self.faces, self.info = positions, colors, faces, info

    def save_ply(self, path: str, transform=None) -> str:
        """the binary PLY saveMesh writes for this mesh (bfMeshSavePly; with transform, bfMeshApplyTransform first); returns path"""
        pos = self.positions.cpu().numpy()
        if transform is not None:
            pos = apply_transform(pos, transform)
        save_ply(path, pos, self.colors.cpu().numpy(), self.faces.cpu().numpy().view(np.uint32))
        return path


def weld_workspace_bytes(num_triangles: int) -> int:
    return int(_bind(capi.lib()).bfMeshWeldWorkspaceBytes(int(num_triangles)))


def weld(soup, thresh: float = 0.00001) -> Mesh:
    """saveMesh's clean-up on the device (bfMeshWeld): soup is a contiguous CUDA float32 tensor [T, 3, 6] (per vertex position, colour), as the
    extraction writes it.  The result equals merge_close_vertices(thresh) + remove_duplicate_faces on the same soup with colours (c, 1), bit for
    bit.  Runs on the current stream of the soup's device and synchronises once per round of the vertex merge plus once."""
    import torch
    if not (isinstance(soup, torch.Tensor) and soup.is_cuda and soup.dtype == torch.float32 and soup.dim() == 3 and tuple(soup.shape[1:]) == (3, 6)
            and soup.is_contiguous()):
        raise ValueError("weld: soup must be a contiguous CUDA float32 tensor [T, 3, 6]")
    L = _bind(capi.lib())
    dev = soup.device
    T = int(soup.shape[0])
    ws_bytes = int(L.bfMeshWeldWorkspaceBytes(T))
    if T and ws_bytes == 0:
        raise ValueError(f"weld: {T} triangles: 3T must be below 2^31 (PLY indices are int)")
    with torch.cuda.device(dev):
        L.bfSetStream(C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
        pos = torch.empty((3 * T, 3), dtype=torch.float32, device=dev)
        col = torch.empty((3 * T, 4), dtype=torch.float32, device=dev)
        faces = torch.empty((T, 3), dtype=torch.int32, device=dev)
        info = capi.BFMeshWeldInfo()
        capi.check(L.bfMeshWeld(soup.data_ptr(), T, thresh, ws.data_ptr(), ws_bytes, pos.data_ptr(), col.data_ptr(), faces.data_ptr(), C.byref(info)), "bfMeshWeld")
        del ws
        V, F = int(info.verticesOut), int(info.facesOut)
        out = Mesh(pos[:V].clone(), col[:V].clone(), faces[:F].clone(), _weld_report(info))
    out.info["device_bytes"] = T * 72 + ws_bytes + 3 * T * (12 + 16) + T * 12              # soup, workspace and outputs: what the weld holds at once
    return out


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

    def extractSoup(self, scene, min_corner=(0.0, 0.0, 0.0), max_corner=(0.0, 0.0, 0.0), box_enabled: bool = False):
        """the whole triangle soup in device memory: the count pass (read back once), a soup tensor [T, 3, 6] of exactly that size, and one
        bfMarchingCubesExtractRange over every chunk.  No triangle is dropped; the mesh buffer is not touched."""
        t = self._torch
        total, _ = self.count(scene, min_corner, max_corner, box_enabled)
        soup = t.empty((total, 3, 6), dtype=t.float32, device=self.device)
        if total:
            p = self._box_params(scene, min_corner, max_corner, box_enabled)
            p.m_maxNumTriangles = total
            n = t.empty(1, dtype=t.int32, device=self.device)
            self._bind_stream()
            capi.check(self.lib.bfMarchingCubesExtractRange(C.byref(scene.m_hashData), C.byref(scene.m_hashParams), C.byref(p), 0, num_chunks(p.m_hashNumBuckets),
                                                            soup.data_ptr(), n.data_ptr()), "bfMarchingCubesExtractRange")
        return soup

    def extractMesh(self, scene, min_corner=(0.0, 0.0, 0.0), max_corner=(0.0, 0.0, 0.0), box_enabled: bool = False, thresh: float = 0.00001) -> Mesh:
        """weld(extractSoup(...)): the indexed mesh saveMesh would write, in device memory"""
        return weld(self.extractSoup(scene, min_corner, max_corner, box_enabled), thresh)

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

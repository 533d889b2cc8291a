"""ctypes loader for the CPU oracle (oracle/liboracle*.so).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package (bundlefusion_b200/) never imports
this module.  The struct definitions are shared with the product's ctypes view of include/*.h
(bundlefusion_b200/_capi.py) because both sides speak the same C-ABI PODs.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from bundlefusion_b200._capi import (BF_HASH_BUCKET_SIZE, BF_SDF_BLOCK_VOXELS, BFDepthCameraParams, BFHashDataStruct,
                                     BFHashParams)

_HERE = os.path.dirname(os.path.abspath(__file__))
_libs = {}


def build() -> None:
    subprocess.check_call(["make", "-C", _HERE, "--no-print-directory"], stdout=subprocess.DEVNULL)


def lib(fast: bool = False) -> C.CDLL:
    name = "liboracle_fast.so" if fast else "liboracle.so"
    if name in _libs:
        return _libs[name]
    path = os.path.join(_HERE, name)
    if not os.path.exists(path):
        build()
    L = C.CDLL(path)
    P = C.POINTER
    fp = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
    L.orc_tsdf_reset.argtypes = [P(BFHashDataStruct), P(BFHashParams)]
    L.orc_tsdf_reset.restype = None
    L.orc_tsdf_find.argtypes = [P(BFHashDataStruct), P(BFHashParams), C.c_int, C.c_int, C.c_int]
    L.orc_tsdf_find.restype = C.c_int
    L.orc_tsdf_alloc.argtypes = [P(BFHashDataStruct), P(BFHashParams), fp, P(BFDepthCameraParams)]
    L.orc_tsdf_alloc.restype = C.c_uint
    L.orc_tsdf_compactify.argtypes = [P(BFHashDataStruct), P(BFHashParams), P(BFDepthCameraParams)]
    L.orc_tsdf_compactify.restype = C.c_uint
    L.orc_tsdf_integrate.argtypes = [P(BFHashDataStruct), P(BFHashParams), fp, C.c_void_p, P(BFDepthCameraParams), C.c_uint, C.c_int]
    L.orc_tsdf_integrate.restype = C.c_ulonglong
    L.orc_tsdf_garbage_collect.argtypes = [P(BFHashDataStruct), P(BFHashParams), C.c_uint]
    L.orc_tsdf_garbage_collect.restype = C.c_uint
    L.orc_tsdf_integrate_dense.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_float * 3, P(BFHashParams), fp, C.c_void_p,
                                           P(BFDepthCameraParams), C.c_int]
    L.orc_tsdf_integrate_dense.restype = C.c_ulonglong
    _libs[name] = L
    return L


def mat4_inverse(T) -> np.ndarray:
    """the reference's host 4x4 inverse (float4x4::getInverse = mat4f::getInverse; oracle/solver_oracle.c: orc_mat4_inverse), float32 [4, 4]"""
    L = lib()
    fp = C.POINTER(C.c_float)
    m = np.ascontiguousarray(T, np.float32).reshape(16); out = np.zeros(16, np.float32)
    L.orc_mat4_inverse.argtypes = [fp, fp]; L.orc_mat4_inverse.restype = None
    L.orc_mat4_inverse(m.ctypes.data_as(fp), out.ctypes.data_as(fp))
    return out.reshape(4, 4)


class OracleSceneRepHashSDF:
    """The same call surface as bundlefusion_b200.scene_rep.CUDASceneRepHashSDF, on host arrays."""

    def __init__(self, params: BFHashParams, fast: bool = False):
        self.L = lib(fast)
        self.hp = BFHashParams()
        C.memmove(C.byref(self.hp), C.byref(params), C.sizeof(BFHashParams))
        n_entries = self.hp.m_hashNumBuckets * BF_HASH_BUCKET_SIZE
        n_blocks = self.hp.m_numSDFBlocks
        self.heap = np.zeros(n_blocks, np.uint32)
        self.heap_counter = np.zeros(1, np.uint32)
        self.hash = np.zeros((n_entries, 8), np.int32)
        self.decision = np.zeros(n_entries, np.int32)
        self.prefix = np.zeros(n_entries, np.int32)
        self.compactified = np.zeros((n_entries, 8), np.int32)
        self.compactified_counter = np.zeros(1, np.int32)
        self.voxels = np.zeros((n_blocks, BF_SDF_BLOCK_VOXELS, 3), np.int32)
        self.mutex = np.zeros(self.hp.m_hashNumBuckets, np.int32)
        hd = BFHashDataStruct()
        hd.d_heap = self.heap.ctypes.data
        hd.d_heapCounter = self.heap_counter.ctypes.data
        hd.d_hashDecision = self.decision.ctypes.data
        hd.d_hashDecisionPrefix = self.prefix.ctypes.data
        hd.d_hash = self.hash.ctypes.data
        hd.d_hashCompactified = self.compactified.ctypes.data
        hd.d_hashCompactifiedCounter = self.compactified_counter.ctypes.data
        hd.d_SDFBlocks = self.voxels.ctypes.data
        hd.d_hashBucketMutex = self.mutex.ctypes.data
        hd.m_bIsOnGPU = 0
        self.hd = hd
        self.num_occupied = 0
        self.last_U = 0
        self.dropped = 0      # block inserts that found no room (table over-full)
        self.reset()

    def reset(self):
        self.L.orc_tsdf_reset(C.byref(self.hd), C.byref(self.hp))
        self.num_occupied = 0

    def _set_pose(self, T):
        """setLastRigidTransform (FL/DepthSensing/CUDASceneRepHashSDF.h:128-134): the pose and its host-computed inverse (the reference's formula: orc_mat4_inverse)"""
        T = np.ascontiguousarray(T, np.float32).reshape(4, 4)
        inv = mat4_inverse(T)
        for k in range(16):
            self.hp.m_rigidTransform.m[k] = float(T.reshape(16)[k]); self.hp.m_rigidTransformInverse.m[k] = float(inv.reshape(16)[k])

    def integrate(self, T, depth: np.ndarray, color: np.ndarray | None, cam: BFDepthCameraParams):
        self._set_pose(T)
        depth = np.ascontiguousarray(depth, np.float32)
        self.dropped += self.L.orc_tsdf_alloc(C.byref(self.hd), C.byref(self.hp), depth, C.byref(cam))
        self.num_occupied = self.L.orc_tsdf_compactify(C.byref(self.hd), C.byref(self.hp), C.byref(cam))
        cptr = color.ctypes.data if color is not None else None
        self.last_U = self.L.orc_tsdf_integrate(C.byref(self.hd), C.byref(self.hp), depth, cptr, C.byref(cam), self.num_occupied, 0)

    def deIntegrate(self, T, depth: np.ndarray, color: np.ndarray | None, cam: BFDepthCameraParams):
        self._set_pose(T)
        depth = np.ascontiguousarray(depth, np.float32)
        self.num_occupied = self.L.orc_tsdf_compactify(C.byref(self.hd), C.byref(self.hp), C.byref(cam))
        cptr = color.ctypes.data if color is not None else None
        self.last_U = self.L.orc_tsdf_integrate(C.byref(self.hd), C.byref(self.hp), depth, cptr, C.byref(cam), self.num_occupied, 1)

    def garbageCollect(self) -> int:
        return self.L.orc_tsdf_garbage_collect(C.byref(self.hd), C.byref(self.hp), self.num_occupied)

    def getHeapFreeCount(self) -> int:
        return (int(self.heap_counter[0]) + 1) & 0xFFFFFFFF

    def download(self) -> dict:
        return {"hash": self.hash, "compactified": self.compactified, "compactified_count": self.num_occupied,
                "heap": self.heap, "heap_counter": int(self.heap_counter[0]), "voxels": self.voxels,
                "decision": self.decision, "mutex": self.mutex}


def canonical_blocks(snap: dict):
    """Sorted (N,3) block coordinates and the matching (N,512,3) voxel words, keyed by world block
    position -- the parity key SURVEY.md section 7 ("hard parts") prescribes: slot/ptr assignment is
    race-dependent in the reference, the block SET and per-voxel values are not."""
    h = snap["hash"]
    used = h[:, 3] != -2
    ent = h[used]
    order = np.lexsort((ent[:, 2], ent[:, 1], ent[:, 0]))
    ent = ent[order]
    slots = ent[:, 3] // BF_SDF_BLOCK_VOXELS
    return ent[:, :3].copy(), snap["voxels"][slots]


def block_hash(pos, num_buckets: int | None = None) -> np.ndarray:
    """VoxelUtilHashSDF.h:226-234 on (N, 3) block positions in uint32 arithmetic: (x*73856093) ^ (y*19349669) ^ (z*83492791), and with
    num_buckets its bucket (an unsigned modulo)"""
    p = np.asarray(pos, np.int64).reshape(-1, 3).astype(np.uint32)
    v = (p[:, 0] * np.uint32(73856093)) ^ (p[:, 1] * np.uint32(19349669)) ^ (p[:, 2] * np.uint32(83492791))
    return v if num_buckets is None else v % np.uint32(num_buckets)


def check_hash_invariants(snap: dict, hp: BFHashParams) -> None:
    """CUDASceneRepHashSDF::debugHash (h:179-314): no duplicate blocks, heap and table partition the slots,
    every chain entry reachable from its home bucket within the list limit, all mutexes released."""
    h = snap["hash"]
    n_blocks = hp.m_numSDFBlocks
    used = np.nonzero(h[:, 3] != -2)[0]
    assert not np.any(h[:, 3] == -1), "LOCK_ENTRY left in the table"
    pos = h[used, :3]
    assert len(np.unique(pos, axis=0)) == len(pos), "duplicate block positions"
    slots = h[used, 3] // BF_SDF_BLOCK_VOXELS
    assert np.all(h[used, 3] % BF_SDF_BLOCK_VOXELS == 0)
    n_free = (snap["heap_counter"] + 1) & 0xFFFFFFFF
    free = snap["heap"][:n_free].astype(np.int64)
    assert len(np.unique(free)) == n_free, "duplicate free slots"
    assert len(np.unique(slots)) == len(slots), "two entries share a slot"
    assert len(np.intersect1d(free, slots)) == 0, "slot both free and allocated"
    assert n_free + len(slots) == n_blocks, "slot leaked"
    assert np.all(snap["mutex"] == -2), "bucket mutex left locked"
    # reachability
    total = hp.m_hashNumBuckets * BF_HASH_BUCKET_SIZE
    hv = block_hash(pos, hp.m_hashNumBuckets)
    for idx, hb in zip(used, hv.astype(np.int64)):
        if idx // BF_HASH_BUCKET_SIZE == hb:
            continue
        last = hb * BF_HASH_BUCKET_SIZE + BF_HASH_BUCKET_SIZE - 1
        i, found = last, False
        for _ in range(hp.m_hashMaxCollisionLinkedListSize + 1):
            off = int(np.uint32(h[i, 4]))
            if off == 0:
                break
            i = (last + off) % total
            if i == idx:
                found = True
                break
        assert found, f"entry {idx} not reachable from bucket {hb}"


# ------------------------------------------------------------------------------------------------
# solver oracle
# ------------------------------------------------------------------------------------------------
def _bind_solver(L):
    if getattr(L, "_solver_bound", False):
        return L
    fp = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
    ip = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
    L.orc_pose_to_matrix.argtypes = [fp, fp, fp]
    L.orc_matrix_to_pose.argtypes = [fp, fp, fp]
    L.orc_mat4_inverse.argtypes = [fp, fp]
    L.orc_solver_build_table.argtypes = [C.c_void_p, C.c_uint, C.c_uint, ip, ip, C.c_uint]
    L.orc_solver_solve_sparse.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_uint, fp, fp, C.c_uint, C.c_uint, fp, C.c_int, ip, ip, C.c_uint * 4]
    L.orc_solver_solve_sparse.restype = C.c_int
    L.orc_solver_max_residual.argtypes = [C.c_void_p, C.c_uint, fp, fp, C.c_float, C.POINTER(C.c_int)]
    L.orc_solver_max_residual.restype = C.c_float
    L.orc_solver_energy.argtypes = [C.c_void_p, C.c_uint, fp, fp, C.c_float]
    L.orc_solver_energy.restype = C.c_double
    L.orc_solver_set_trace.argtypes = [C.c_void_p, C.c_uint]
    L.orc_solver_set_trace.restype = None
    L.orc_solver_trace_count.argtypes = []
    L.orc_solver_trace_count.restype = C.c_uint
    L._solver_bound = True
    return L


class _Trace:
    """Records the early-out decisions of one oracle solve (orc_solver_set_trace): list of (gn, p.Ap) and (-(gn+1), max|delta|)."""

    def __init__(self, L, cap=8192):
        self.L, self.buf = L, np.zeros(2 * cap, np.float32)
        L.orc_solver_set_trace(self.buf.ctypes.data, cap)

    def finish(self):
        n = min(self.L.orc_solver_trace_count(), len(self.buf) // 2)
        self.L.orc_solver_set_trace(None, 0)
        return self.buf[:2 * n].reshape(-1, 2).copy()


def decision_margin(trace) -> float:
    """Smallest relative distance of any recorded early-out decision from its threshold: p.Ap against 5e-7 (last iteration,
    SolverBundling.cu:1092) and 1e-6 (alpha guard, :959), max|delta| against 0.005 (:1206).  0.3 means every decision would survive
    a 30 % change of the value it tests -- float summation order moves these by ~1e-6 relative."""
    m = np.inf
    for k, v in trace:
        for thr in ((5e-7, 1e-6) if k >= 0 else (0.005,)):
            m = min(m, abs(abs(float(v)) - thr) / thr)
    return float(m)


def pose_to_matrix(rot, trans) -> np.ndarray:
    L = _bind_solver(lib())
    M = np.zeros(16, np.float32)
    L.orc_pose_to_matrix(np.ascontiguousarray(rot, np.float32), np.ascontiguousarray(trans, np.float32), M)
    return M.reshape(4, 4)


def matrix_to_pose(M):
    L = _bind_solver(lib())
    r, t = np.zeros(3, np.float32), np.zeros(3, np.float32)
    L.orc_matrix_to_pose(np.ascontiguousarray(M, np.float32).reshape(16), r, t)
    return r, t


def solve_sparse(corr: np.ndarray, rot0, trans0, n_gn: int, n_pcg: int, weights=None, max_corr_per_image: int = 4000, fast: bool = False):
    """CUDASolverBundling::solve for the sparse term.  `corr`: structured array in EntryJ layout (copied; entries the
    table build invalidates are reported back).  Returns dict(rot, trans, stats, corr)."""
    L = _bind_solver(lib(fast))
    corr = np.ascontiguousarray(corr).copy()
    N = len(rot0)
    rot = np.ascontiguousarray(rot0, np.float32).copy()
    trans = np.ascontiguousarray(trans0, np.float32).copy()
    w = np.ascontiguousarray(weights if weights is not None else np.ones(n_gn), np.float32)
    table = np.zeros(N * max_corr_per_image, np.int32)
    rows = np.zeros(N, np.int32)
    stats = (C.c_uint * 4)()
    tr = _Trace(L)
    rc = L.orc_solver_solve_sparse(corr.ctypes.data, len(corr), N, max_corr_per_image, rot, trans, n_gn, n_pcg, w, 1, table, rows, stats)
    trace = tr.finish()
    assert rc == 0
    return {"rot": rot, "trans": trans, "gn": stats[0], "pcg": stats[1], "corr": corr, "rows": rows, "trace": trace}


def max_residual(corr, rot, trans, w=1.0):
    L = _bind_solver(lib())
    idx = C.c_int(0)
    corr = np.ascontiguousarray(corr)
    v = L.orc_solver_max_residual(corr.ctypes.data, len(corr), np.ascontiguousarray(rot, np.float32), np.ascontiguousarray(trans, np.float32), w, C.byref(idx))
    return float(v), idx.value


def energy(corr, rot, trans, w=1.0) -> float:
    L = _bind_solver(lib())
    corr = np.ascontiguousarray(corr)
    return float(L.orc_solver_energy(corr.ctypes.data, len(corr), np.ascontiguousarray(rot, np.float32), np.ascontiguousarray(trans, np.float32), w))


class OrcCacheFrame(C.Structure):
    _fields_ = [("depth", C.c_void_p), ("campos", C.c_void_p), ("intensity", C.c_void_p), ("intensityDerivs", C.c_void_p),
                ("normalsU", C.c_void_p), ("normals", C.c_void_p)]


class OrcDenseParams(C.Structure):
    _fields_ = [("W", C.c_uint), ("H", C.c_uint), ("fx", C.c_float), ("fy", C.c_float), ("mx", C.c_float), ("my", C.c_float),
                ("distThresh", C.c_float), ("normalThresh", C.c_float), ("colorThresh", C.c_float), ("colorGradientMin", C.c_float),
                ("depthMin", C.c_float), ("depthMax", C.c_float), ("subsample", C.c_uint), ("usePairwise", C.c_int)]


def dense_params(intrinsics, W=80, H=60, pairwise=True) -> OrcDenseParams:
    """defaults of FriedLiver/zParametersBundlingDefault.txt:22-28"""
    d = OrcDenseParams()
    d.W, d.H = W, H
    d.fx, d.fy, d.mx, d.my = [float(x) for x in intrinsics]
    d.distThresh, d.normalThresh, d.colorThresh, d.colorGradientMin, d.depthMin, d.depthMax = 0.15, 0.97, 0.1, 0.005, 0.5, 4.0
    d.subsample, d.usePairwise = 4, 1 if pairwise else 0
    return d


def _pack_frames(caches):
    arr = (OrcCacheFrame * len(caches))()
    keep = []
    for k, c in enumerate(caches):
        for name in ("depth", "campos", "intensity", "intensityDerivs", "normalsU", "normals"):
            a = np.ascontiguousarray(c[name]); keep.append(a)
            setattr(arr[k], name, a.ctypes.data)
    return arr, keep


def solve(corr, rot0, trans0, n_gn, n_pcg, w_sparse, w_depth=None, w_color=None, caches=None, intrinsics=None, valid=None,
          max_corr_per_image=4000, pairwise=True, fast=False):
    """The complete solveBundlingStub (sparse + dense depth/colour)."""
    L = _bind_solver(lib(fast))
    fp = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
    ip = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
    L.orc_solver_solve.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_uint, fp, fp, C.c_uint, C.c_uint, fp, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_void_p, ip, ip, C.c_uint * 4]
    L.orc_solver_solve.restype = C.c_int
    corr = np.ascontiguousarray(corr).copy()
    N = len(rot0)
    rot, trans = np.ascontiguousarray(rot0, np.float32).copy(), np.ascontiguousarray(trans0, np.float32).copy()
    wS = np.ascontiguousarray(w_sparse, np.float32)
    wD = np.ascontiguousarray(w_depth if w_depth is not None else np.zeros(n_gn), np.float32)
    wC = np.ascontiguousarray(w_color if w_color is not None else np.zeros(n_gn), np.float32)
    table, rows = np.zeros(N * max_corr_per_image, np.int32), np.zeros(N, np.int32)
    stats = (C.c_uint * 4)()
    frames, keep, dp = None, None, None
    if caches is not None:
        frames, keep = _pack_frames(caches)
        dp = dense_params(intrinsics, caches[0]["depth"].shape[1], caches[0]["depth"].shape[0], pairwise)
    v = np.ascontiguousarray(valid, np.int32) if valid is not None else None
    tr = _Trace(L)
    rc = L.orc_solver_solve(corr.ctypes.data, len(corr), N, max_corr_per_image, rot, trans, n_gn, n_pcg, wS, wD.ctypes.data, wC.ctypes.data,
                            C.cast(frames, C.c_void_p) if frames is not None else None, C.cast(C.pointer(dp), C.c_void_p) if dp is not None else None,
                            v.ctypes.data if v is not None else None, table, rows, stats)
    trace = tr.finish()
    assert rc == 0
    return {"rot": rot, "trans": trans, "gn": stats[0], "pcg": stats[1], "overlap_pairs": stats[2], "weighted_pairs": stats[3], "corr": corr, "rows": rows,
            "trace": trace}


def build_dense(rot, trans, caches, intrinsics, w_depth, w_color, valid=None, pairwise=True):
    """dense J^T J [(6N)^2] and J^T r [6N] at the given poses (translation-first ordering per image)."""
    L = _bind_solver(lib())
    fp = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
    L.orc_solver_build_dense.argtypes = [fp, fp, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float, fp, fp, C.c_uint * 2]
    L.orc_solver_build_dense.restype = C.c_uint
    N = len(rot)
    frames, keep = _pack_frames(caches)
    dp = dense_params(intrinsics, caches[0]["depth"].shape[1], caches[0]["depth"].shape[0], pairwise)
    JtJ, Jtr = np.zeros((6 * N) ** 2, np.float32), np.zeros(6 * N, np.float32)
    pairs = (C.c_uint * 2)()
    v = np.ascontiguousarray(valid, np.int32) if valid is not None else None
    L.orc_solver_build_dense(np.ascontiguousarray(rot, np.float32), np.ascontiguousarray(trans, np.float32), N, C.cast(frames, C.c_void_p),
                             C.cast(C.pointer(dp), C.c_void_p), v.ctypes.data if v is not None else None, w_depth, w_color, JtJ, Jtr, pairs)
    return JtJ.reshape(6 * N, 6 * N), Jtr, (pairs[0], pairs[1])


# ---- SIFT descriptor matcher (oracle/sift_oracle.c) ----------------------------------------------------------------------
def sift_multiply(d1: np.ndarray, d2: np.ndarray) -> np.ndarray:
    L = lib()
    d1, d2 = np.ascontiguousarray(d1, np.uint8), np.ascontiguousarray(d2, np.uint8)
    dot = np.zeros((len(d1), len(d2)), np.int32)
    L.orc_sift_multiply.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    L.orc_sift_multiply.restype = None
    L.orc_sift_multiply(d1.ctypes.data, len(d1), d2.ctypes.data, len(d2), dot.ctypes.data)
    return dot


def sift_match(d1: np.ndarray, d2: np.ndarray, distmax: float = 0.7, ratiomax: float = 0.8, offset=(0, 0), fast: bool = False):
    """SiftMatchGPU::GetSiftMatch for one pair.  Returns (indices [n,2] uint32, distances [n] float32, counter)."""
    L = lib(fast)
    d1, d2 = np.ascontiguousarray(d1, np.uint8), np.ascontiguousarray(d2, np.uint8)
    idx = np.zeros((128, 2), np.uint32); dist = np.zeros(128, np.float32)
    L.orc_sift_match.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
    L.orc_sift_match.restype = C.c_int
    c = L.orc_sift_match(d1.ctypes.data, len(d1), d2.ctypes.data, len(d2), distmax, ratiomax, offset[0], offset[1], idx.ctypes.data, dist.ctypes.data)
    n = min(c, 128)
    return idx[:n].copy(), dist[:n].copy(), c


def sift_row_match(dot: np.ndarray, distmax: float = 0.7, ratiomax: float = 0.8):
    """RowMatch_Kernel on a given dot matrix: (best column or -1 per row, distance per row)."""
    L = lib()
    dot = np.ascontiguousarray(dot, np.int32)
    n1, n2 = dot.shape
    res = np.zeros(n1, np.int32); dist = np.zeros(n1, np.float32)
    L.orc_sift_row_match.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
    L.orc_sift_row_match.restype = None
    L.orc_sift_row_match(dot.ctypes.data, n1, n2, distmax, ratiomax, res.ctypes.data, dist.ctypes.data)
    return res, dist


# ---- dense cache frame (oracle/cache_oracle.c) ----------------------------------------------------------------------------
def cache_store_frame(depth: np.ndarray, color: np.ndarray, K, cw: int = 80, ch: int = 60, colorDownSigma: float = 2.5,
                      depthDownSigmaD: float = 1.0, depthDownSigmaR: float = 0.05) -> dict:
    """CUDACache::storeFrame for one frame; K = 4x4 input intrinsics.  Returns host arrays keyed like synth.make_cache_frame."""
    from bundlefusion_b200._capi import BFCacheParams
    L = lib()
    depth = np.ascontiguousarray(depth, np.float32); color = np.ascontiguousarray(color, np.uint8)
    p = BFCacheParams()
    p.inputDepthHeight, p.inputDepthWidth = depth.shape
    p.inputColorHeight, p.inputColorWidth = color.shape[:2]
    p.width, p.height = cw, ch
    Ki = mat4_inverse(np.asarray(K, np.float32).reshape(4, 4))          # m_inputIntrinsics.getInverse(), FL/CUDACache.cpp:38
    for k in range(16):
        p.inputIntrinsicsInv[k] = float(Ki.reshape(-1)[k])
    p.filterIntensitySigma, p.filterDepthSigmaD, p.filterDepthSigmaR = colorDownSigma, depthDownSigmaD, depthDownSigmaR
    out = {"depth": np.full((ch, cw), -np.inf, np.float32), "campos": np.full((ch, cw, 4), -np.inf, np.float32),
           "normals": np.full((ch, cw, 4), -np.inf, np.float32), "normalsU": np.zeros((ch, cw, 4), np.uint8),
           "intensity": np.zeros((ch, cw), np.float32), "intensityDerivs": np.full((ch, cw, 2), -np.inf, np.float32)}
    L.orc_cache_store_frame.argtypes = [C.c_void_p] * 9
    L.orc_cache_store_frame.restype = None
    L.orc_cache_store_frame(C.addressof(p), depth.ctypes.data, color.ctypes.data, out["depth"].ctypes.data, out["campos"].ctypes.data,
                            out["normals"].ctypes.data, out["normalsU"].ctypes.data, out["intensity"].ctypes.data, out["intensityDerivs"].ctypes.data)
    return out


# ---- frame ingest (oracle/ingest_oracle.c) ---------------------------------------------------------------------------------
def ingest_params(depth_shape, color_shape, wi, hi, erode=True, depth_filter=True, sigmaD=2.0, sigmaR=0.05):
    from bundlefusion_b200._capi import BFIngestParams
    p = BFIngestParams()
    p.depthHeight, p.depthWidth = depth_shape[:2]
    p.colorHeight, p.colorWidth = color_shape[:2]
    p.widthIntegration, p.heightIntegration = wi, hi
    p.erodeIterations, p.erodeStructureSize, p.erodeDThresh, p.erodeFracReq = (2 if erode else 0), 3, 0.05, 0.3
    p.depthSigmaD, p.depthSigmaR = (sigmaD if depth_filter else 0.0), sigmaR
    return p


def ingest_frame(depth: np.ndarray, color: np.ndarray, wi: int, hi: int, **kw):
    """Device part of CUDAImageManager::process: (depth [hi,wi] f32, colour [hi,wi,4] u8) at the integration resolution."""
    L = lib(kw.pop("fast", False))
    depth = np.ascontiguousarray(depth, np.float32); color = np.ascontiguousarray(color, np.uint8)
    p = ingest_params(depth.shape, color.shape, wi, hi, **kw)
    dout = np.full((hi, wi), -np.inf, np.float32); cout = np.zeros((hi, wi, 4), np.uint8)
    L.orc_ingest_frame.argtypes = [C.c_void_p] * 5
    L.orc_ingest_frame.restype = None
    L.orc_ingest_frame(C.addressof(p), depth.ctypes.data, color.ctypes.data, dout.ctypes.data, cout.ctypes.data)
    return dout, cout


# ---- trajectory glue (oracle/trajectory_oracle.c) ---------------------------------------------------------------------------
def compute_sift_transform(filteredInv, numFiltered, complete, lastValidComplete, siftTraj, curAll, cur):
    """getSiftTransformCU_Kernel: returns (updated siftTraj copy, currIntegrateTrans [4,4])."""
    L = lib()
    f = lambda a: np.ascontiguousarray(a, np.float32)
    filteredInv, complete, siftTraj = f(filteredInv), f(complete), f(siftTraj).copy()
    nf = np.ascontiguousarray(numFiltered, np.int32)
    out = np.zeros((4, 4), np.float32)
    L.orc_compute_sift_transform.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p, C.c_uint, C.c_uint, C.c_void_p]
    L.orc_compute_sift_transform.restype = None
    L.orc_compute_sift_transform(filteredInv.ctypes.data, nf.ctypes.data, complete.ctypes.data, lastValidComplete, siftTraj.ctypes.data, curAll, cur, out.ctypes.data)
    return siftTraj, out


def update_trajectory(globalT, local, perTraj, invalidate):
    L = lib()
    g, l = np.ascontiguousarray(globalT, np.float32), np.ascontiguousarray(local, np.float32)
    inv = np.ascontiguousarray(invalidate, np.int32)
    out = np.zeros((len(inv), 4, 4), np.float32)
    L.orc_update_trajectory.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p, C.c_uint, C.c_void_p]
    L.orc_update_trajectory.restype = None
    L.orc_update_trajectory(g.ctypes.data, out.ctypes.data, len(inv), l.ctypes.data, perTraj, inv.ctypes.data)
    return out


def init_next_global(globalT, numGlobal, initIdx, local, lastValidLocal, perTraj):
    L = lib()
    g = np.ascontiguousarray(globalT, np.float32).copy(); l = np.ascontiguousarray(local, np.float32)
    L.orc_init_next_global.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_uint, C.c_uint]
    L.orc_init_next_global.restype = None
    L.orc_init_next_global(g.ctypes.data, numGlobal, initIdx, l.ctypes.data, lastValidLocal, perTraj)
    return g


def select_reintegration(opt, integ, state, topN, minDist, scale=2.0):
    """(dist [n], list of frame indices) -- TrajectoryManager::generateUpdateLists, re-integration part."""
    L = lib()
    opt, integ = np.ascontiguousarray(opt, np.float32), np.ascontiguousarray(integ, np.float32)
    st = np.ascontiguousarray(state, np.int32)
    n = len(st)
    dist = np.zeros(n, np.float32); lst = np.zeros(max(topN, 1), np.int32)
    L.orc_select_reintegration.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
    L.orc_select_reintegration.restype = C.c_int
    c = L.orc_select_reintegration(opt.ctypes.data, integ.ctypes.data, st.ctypes.data, n, topN, minDist, scale, dist.ctypes.data, lst.ctypes.data)
    return dist, lst[:c].copy()


def sift_sort_matches(curFrame, startFrame, numFrames, numMatches, dists, idxs):
    """SortKeyPointMatchesCU on the manager-layout arrays ([pairs,128] distances, [pairs,128,2] indices); returns sorted copies."""
    L = lib()
    nm = np.ascontiguousarray(numMatches, np.int32); d = np.ascontiguousarray(dists, np.float32).copy(); ix = np.ascontiguousarray(idxs, np.uint32).copy()
    L.orc_sift_sort_matches.argtypes = [C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_sift_sort_matches.restype = None
    L.orc_sift_sort_matches(curFrame, startFrame, numFrames, nm.ctypes.data, d.ctypes.data, ix.ctypes.data)
    return d, ix


# ---- Kabsch match filter (oracle/filter_oracle.c) ---------------------------------------------------------------------------
def sift_filter_matches(curFrame, startFrame, numFrames, keyPoints, numMatches, dists, idxs, siftIntrinsicsInv, minNumMatches=5, maxKabschRes2=0.0004):
    """FilterKeyPointMatchesCU.  keyPoints [K,4] float32 (x, y, scale, depth); dists [P,128]; idxs [P,128,2] uint32 (global key indices).
    Returns (numFiltered [P], fDists [P,25], fIdxs [P,25,2], T [P,4,4], Tinv [P,4,4])."""
    L = lib()
    kp = np.ascontiguousarray(keyPoints, np.float32); nm = np.ascontiguousarray(numMatches, np.int32)
    d = np.ascontiguousarray(dists, np.float32); ix = np.ascontiguousarray(idxs, np.uint32)
    Ki = np.ascontiguousarray(siftIntrinsicsInv, np.float32)
    P = len(nm)
    nf = np.zeros(P, np.int32); fd = np.zeros((P, 25), np.float32); fi = np.zeros((P, 25, 2), np.uint32)
    T = np.zeros((P, 4, 4), np.float32); Ti = np.zeros((P, 4, 4), np.float32)
    L.orc_sift_filter_matches.argtypes = [C.c_uint, C.c_uint, C.c_uint] + [C.c_void_p] * 10 + [C.c_uint, C.c_float]
    L.orc_sift_filter_matches.restype = None
    L.orc_sift_filter_matches(curFrame, startFrame, numFrames, kp.ctypes.data, nm.ctypes.data, d.ctypes.data, ix.ctypes.data, nf.ctypes.data, fd.ctypes.data,
                              fi.ctypes.data, T.ctypes.data, Ti.ctypes.data, Ki.ctypes.data, minNumMatches, maxKabschRes2)
    return nf, fd, fi, T, Ti


def sift_add_residuals(curFrame, startFrame, numFrames, numFiltered, fIdxs, keyPoints, colorIntrinsicsInv, capacity=None):
    """AddCurrToResidualsCU: returns (EntryJ structured array, key index pairs [n,2])."""
    L = lib()
    nf = np.ascontiguousarray(numFiltered, np.int32); fi = np.ascontiguousarray(fIdxs, np.uint32); kp = np.ascontiguousarray(keyPoints, np.float32)
    Ki = np.ascontiguousarray(colorIntrinsicsInv, np.float32)
    cap = capacity or int(nf.clip(0).sum()) + 1
    ent = np.zeros(cap, dtype=[("i", "<u4"), ("j", "<u4"), ("pi", "<f4", 3), ("pj", "<f4", 3)]); eidx = np.zeros((cap, 2), np.uint32)
    L.orc_sift_add_residuals.argtypes = [C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_sift_add_residuals.restype = C.c_int
    n = L.orc_sift_add_residuals(curFrame, startFrame, numFrames, ent.ctypes.data, eidx.ctypes.data, 0, nf.ctypes.data, fi.ctypes.data, kp.ctypes.data, Ki.ctypes.data)
    return ent[:n].copy(), eidx[:n].copy()


def sift_filter_surface_area(curFrame, startFrame, numFrames, keyPoints, numFiltered, fIdxs, colorIntrinsicsInv, areaThresh):
    """FilterMatchesBySurfaceAreaCU.  Returns (numFiltered' [P], areas [P,2])."""
    L = lib()
    kp = np.ascontiguousarray(keyPoints, np.float32); nf = np.ascontiguousarray(numFiltered, np.int32).copy()
    fi = np.ascontiguousarray(fIdxs, np.uint32); Ki = np.ascontiguousarray(colorIntrinsicsInv, np.float32)
    areas = np.full((len(nf), 2), -1.0, np.float32)
    L.orc_sift_filter_surface_area.argtypes = [C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p]
    L.orc_sift_filter_surface_area.restype = None
    L.orc_sift_filter_surface_area(curFrame, startFrame, numFrames, kp.ctypes.data, nf.ctypes.data, fi.ctypes.data, Ki.ctypes.data, areaThresh, areas.ctypes.data)
    return nf, areas


class _CachedFrame(C.Structure):
    _fields_ = [("depth", C.c_void_p), ("campos", C.c_void_p), ("intensity", C.c_void_p), ("intensityDerivs", C.c_void_p), ("normalsU4", C.c_void_p), ("normals", C.c_void_p)]


def sift_filter_dense_verify(curFrame, startFrame, numFrames, W, H, intrinsics, numFiltered, fT, frames, distThresh, normalThresh, colorThresh,
                             errThresh, corrThresh, dMin, dMax):
    """FilterMatchesByDenseVerifyCU.  frames: list of dicts with float32 arrays 'depth' [H,W], 'campos' [H,W,4], 'normals' [H,W,4].
    Returns (numFiltered' [P], stats [P,2] = (err, corr))."""
    L = lib()
    nf = np.ascontiguousarray(numFiltered, np.int32).copy(); T = np.ascontiguousarray(fT, np.float32); K = np.ascontiguousarray(intrinsics, np.float32)
    keep = [{k: np.ascontiguousarray(f[k], np.float32) for k in ("depth", "campos", "normals")} for f in frames]
    recs = (_CachedFrame * len(keep))()
    for r, f in zip(recs, keep):
        r.depth, r.campos, r.normals = f["depth"].ctypes.data, f["campos"].ctypes.data, f["normals"].ctypes.data
    stats = np.full((len(nf), 2), -1.0, np.float32)
    L.orc_sift_filter_dense_verify.argtypes = [C.c_uint] * 5 + [C.c_void_p] * 4 + [C.c_float] * 7 + [C.c_void_p]
    L.orc_sift_filter_dense_verify.restype = None
    L.orc_sift_filter_dense_verify(curFrame, startFrame, numFrames, W, H, K.ctypes.data, nf.ctypes.data, T.ctypes.data, C.addressof(recs),
                                   distThresh, normalThresh, colorThresh, errThresh, corrThresh, dMin, dMax, stats.ctypes.data)
    return nf, stats


def sift_verify_trajectory(numImages, validImages, trajectory, W, H, intrinsics, frames, distThresh, normalThresh, colorThresh, errThresh, corrThresh, dMin, dMax):
    """VerifyTrajectoryCU.  trajectory [N,4,4]; frames as for sift_filter_dense_verify.  Returns (valid 0/1, stats [N(N-1)/2, 2] by block index)."""
    L = lib()
    v = np.ascontiguousarray(validImages, np.int32); T = np.ascontiguousarray(trajectory, np.float32); K = np.ascontiguousarray(intrinsics, np.float32)
    keep = [{k: np.ascontiguousarray(f[k], np.float32) for k in ("depth", "campos", "normals")} for f in frames]
    recs = (_CachedFrame * len(keep))()
    for r, f in zip(recs, keep):
        r.depth, r.campos, r.normals = f["depth"].ctypes.data, f["campos"].ctypes.data, f["normals"].ctypes.data
    stats = np.full((max(1, numImages * (numImages - 1) // 2), 2), -1.0, np.float32)
    L.orc_sift_verify_trajectory.argtypes = [C.c_uint, C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p] + [C.c_float] * 7 + [C.c_void_p]
    L.orc_sift_verify_trajectory.restype = C.c_int
    ok = L.orc_sift_verify_trajectory(numImages, v.ctypes.data, T.ctypes.data, W, H, K.ctypes.data, C.addressof(recs), distThresh, normalThresh, colorThresh,
                                      errThresh, corrThresh, dMin, dMax, stats.ctypes.data)
    return int(ok), stats


def sift_fuse_to_global(corr, keyIdx, transforms, keys, descs, numKeysPerImage, keyStride, K, maxKeys=1024):
    """SIFTImageManager::fuseToGlobal (+ computeTracks).  corr: EntryJ structured array [C]; keyIdx [C,2] uint32 global key indices (image *
    keyStride + key); transforms [N,4,4]; keys [N*keyStride,4] (x, y, scale, depth); descs [N*keyStride,128] uint8.  Returns (keys [n,4], descs [n,128])."""
    L = lib()
    corr = np.ascontiguousarray(corr); ki = np.ascontiguousarray(keyIdx, np.uint32); T = np.ascontiguousarray(transforms, np.float32)
    kp = np.ascontiguousarray(keys, np.float32); ds = np.ascontiguousarray(descs, np.uint8); nk = np.ascontiguousarray(numKeysPerImage, np.int32)
    Kc = np.ascontiguousarray(K, np.float32)
    ok, od = np.zeros((maxKeys, 4), np.float32), np.zeros((maxKeys, 128), np.uint8)
    L.orc_sift_fuse_to_global.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint]
    L.orc_sift_fuse_to_global.restype = C.c_int
    n = L.orc_sift_fuse_to_global(corr.ctypes.data, ki.ctypes.data, len(corr), T.ctypes.data, len(T), kp.ctypes.data, ds.ctypes.data, nk.ctypes.data, keyStride,
                                  Kc.ctypes.data, ok.ctypes.data, od.ctypes.data, maxKeys)
    return ok[:n], od[:n]


# ---- SIFT detection (oracle/sift_detect_oracle.c) -----------------------------------------------------------------------------------
class SiftDetectParams(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("depthWidth", C.c_uint32), ("depthHeight", C.c_uint32), ("depthMin", C.c_float),
                ("depthMax", C.c_float), ("minKeyScale", C.c_float), ("featureCountThreshold", C.c_int32), ("maxKeyPoints", C.c_uint32)]


def sift_detect(intensity, depth, depthMin=0.1, depthMax=3.0, minKeyScale=3.0, featureCountThreshold=150, maxKeyPoints=1024):
    """SiftGPU::RunSIFT + GetKeyPointsAndDescriptorsCUDA.  intensity [H,W] float32 in 0..1, depth [Hd,Wd] float32 (-inf invalid).
    Returns (keyPoints [n,4] = (x, y, scale, depth), descriptors [n,128] uint8, levelCounts [12])."""
    L = lib()
    I = np.ascontiguousarray(intensity, np.float32); D = np.ascontiguousarray(depth, np.float32)
    P = SiftDetectParams(I.shape[1], I.shape[0], D.shape[1], D.shape[0], depthMin, depthMax, minKeyScale, featureCountThreshold, maxKeyPoints)
    kp = np.zeros((maxKeyPoints, 4), np.float32); des = np.zeros((maxKeyPoints, 128), np.uint8); lc = np.zeros(12, np.int32)
    L.orc_sift_detect.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(SiftDetectParams), C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_sift_detect.restype = C.c_int
    n = L.orc_sift_detect(I.ctypes.data, D.ctypes.data, C.byref(P), kp.ctypes.data, des.ctypes.data, lc.ctypes.data)
    if n < 0:
        raise ValueError("unsupported image size")
    return kp[:n].copy(), des[:n].copy(), lc


def sift_filter_bank():
    L = lib()
    s = np.zeros(6, np.float32); w = np.zeros(6, np.int32); t = np.zeros((6, 33), np.float32)
    L.orc_sift_filter_bank.argtypes = [C.c_void_p] * 3
    L.orc_sift_filter_bank(s.ctypes.data, w.ctypes.data, t.ctypes.data)
    return s, w, t


def sift_invalidate_image_to_image(entries, imgI, imgJ):
    """InvalidateImageToImageCU on a structured EntryJ array (copy returned)."""
    L = lib()
    e = np.ascontiguousarray(entries).copy()
    L.orc_sift_invalidate_image_to_image.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_uint]
    L.orc_sift_invalidate_image_to_image.restype = None
    L.orc_sift_invalidate_image_to_image(e.ctypes.data, len(e), imgI, imgJ)
    return e


def sift_check_invalid_frames(numEntriesPerRow, validImages, entries, comprehensive):
    """CheckForInvalidFrames(Simple)CU: returns (validImages', entries')."""
    L = lib()
    n = np.ascontiguousarray(numEntriesPerRow, np.int32); v = np.ascontiguousarray(validImages, np.int32).copy(); e = np.ascontiguousarray(entries).copy()
    L.orc_sift_check_invalid_frames.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p, C.c_uint, C.c_int]
    L.orc_sift_check_invalid_frames.restype = None
    L.orc_sift_check_invalid_frames(n.ctypes.data, v.ctypes.data, len(n), e.ctypes.data, len(e), int(comprehensive))
    return v, e


def sift_filter_frames(curFrame, startFrame, numFrames, numFiltered, validImages):
    """SIFTImageManager::filterFrames: returns (lastMatchedFrame or -1, validImages')."""
    L = lib()
    nf = np.ascontiguousarray(numFiltered, np.int32); v = np.ascontiguousarray(validImages, np.int32).copy()
    L.orc_sift_filter_frames.argtypes = [C.c_uint, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p]
    L.orc_sift_filter_frames.restype = C.c_int
    return L.orc_sift_filter_frames(curFrame, startFrame, numFrames, nf.ctypes.data, v.ctypes.data), v


# ---- ray cast of the hashed TSDF (oracle/raycast_oracle.c; SURVEY.md section 8f, row N3) ----------------------------------------------
def raycast_set_pose(p, T):
    """CUDARayCastSDF::rayIntervalSplatting (cpp:86-98): view matrix = inverse of the rigid transform (float32 cofactor inverse, as the host's mat4f)"""
    T = np.ascontiguousarray(T, np.float32).reshape(4, 4)
    inv = mat4_inverse(T)
    for k in range(16):
        p.m_viewMatrixInverse.m[k] = float(T.reshape(16)[k]); p.m_viewMatrix.m[k] = float(inv.reshape(16)[k])


def raycast_splat(scene: "OracleSceneRepHashSDF", cam, p, splat_minimum: int) -> np.ndarray:
    """one interval image ([height, width] float32, -inf = nothing drawn) from the scene's last compactified list"""
    L = lib()
    out = np.zeros((p.m_height, p.m_width), np.float32)
    p.m_splatMinimum = splat_minimum
    L.orc_raycast_splat.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p]
    L.orc_raycast_splat.restype = None
    L.orc_raycast_splat(C.addressof(scene.hp), C.addressof(cam), C.addressof(p), scene.compactified.ctypes.data, int(scene.num_occupied), out.ctypes.data)
    return out


def raycast_render(scene: "OracleSceneRepHashSDF", p, ray_min: np.ndarray, ray_max: np.ndarray) -> dict:
    L = lib()
    H, W = p.m_height, p.m_width
    o = {"depth": np.zeros((H, W), np.float32), "depth4": np.zeros((H, W, 4), np.float32), "normals": np.zeros((H, W, 4), np.float32), "colors": np.zeros((H, W, 4), np.float32)}
    L.orc_raycast_render.argtypes = [C.c_void_p] * 9
    L.orc_raycast_render.restype = None
    rmin, rmax = np.ascontiguousarray(ray_min, np.float32), np.ascontiguousarray(ray_max, np.float32)
    L.orc_raycast_render(C.addressof(scene.hd), C.addressof(scene.hp), C.addressof(p), rmin.ctypes.data, rmax.ctypes.data, o["depth"].ctypes.data, o["depth4"].ctypes.data,
                         o["normals"].ctypes.data, o["colors"].ctypes.data)
    if not p.m_useGradients:
        L.orc_raycast_normals.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_void_p]
        L.orc_raycast_normals.restype = None
        L.orc_raycast_normals(o["depth4"].ctypes.data, W, H, o["normals"].ctypes.data)
    return o


def raycast_frame(scene: "OracleSceneRepHashSDF", cam, p, T) -> dict:
    """CUDARayCastSDF::render: interval splat (both directions), ray march, normals"""
    raycast_set_pose(p, T)
    rmin = raycast_splat(scene, cam, p, 1)
    rmax = raycast_splat(scene, cam, p, 0)
    o = raycast_render(scene, p, rmin, rmax)
    o["ray_min"], o["ray_max"] = rmin, rmax
    return o


# ---- iso-surface extraction (oracle/marchingcubes_oracle.c; SURVEY.md section 8f, row N4, second half) ------------------------------------
def marchingcubes_tables():
    """(edgeTable [256], triTable [256, 16]) as the reference's Tables.h lays them out (-1 padded)"""
    L = lib()
    edge = np.zeros(256, np.int32); tri = np.zeros((256, 16), np.int32)
    L.orc_marchingcubes_tables.argtypes = [C.c_void_p, C.c_void_p]
    L.orc_marchingcubes_tables.restype = None
    L.orc_marchingcubes_tables(edge.ctypes.data, tri.ctypes.data)
    return edge, tri


def marchingcubes_extract(scene: "OracleSceneRepHashSDF", p):
    """extractIsoSurfaceKernel over the scene's hash table -> (triangles [n, 3, 6] float32: position xyz + colour rgb per vertex, triangles the cells produced)"""
    L = lib()
    tri = np.zeros((int(p.m_maxNumTriangles), 3, 6), np.float32)
    found = C.c_ulonglong(0)
    L.orc_marchingcubes_extract.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_marchingcubes_extract.restype = C.c_uint
    n = L.orc_marchingcubes_extract(C.addressof(scene.hd), C.addressof(scene.hp), C.addressof(p), tri.ctypes.data, C.byref(found))
    return tri[:n].copy(), int(found.value)

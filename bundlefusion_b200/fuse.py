"""Fusion along a fixed trajectory: a recording's frames integrated at given poses into a voxel hash of any voxel size, then meshed -- no
bundling.  What the reference does with ``s_binaryDumpSensorUseTrajectory`` (FL/DepthSensing/DepthSensing.cpp:1036-1040, FL/SensorDataReader.cpp:131:
integrate along the poses stored with the frames), and the usual last step after a scan: fuse again along the final, optimised trajectory at a
finer voxel size (4-5 mm) and mesh that.

    fuse_recording(sens_path, ply_path, voxel_size=0.004, poses="recorded")      # a .sens file along its own poses
    FrameLoop.fuse(scene, poses=None)                                              # the loop's frame store along its optimised trajectory
    fuse_recording(..., fit_hash=True)                                             # the hash sized from a count of the blocks it will hold

Sizing: BlockCounter counts on the device the union of the blocks the fusion's alloc launches will insert (bfTsdfCountBlocks), and
fit_hash_params sizes the hash from it -- a heap of exactly that many blocks and the fewest buckets (of a fixed sequence) in which no bucket
receives more than BF_HASH_BUCKET_SIZE of them.  The blocks live in the fused hash are always a subset of that union, so such a hash never
drops an insert and its heap never runs out (include/bf_tsdf.h).

Host glue only: each frame is decoded (the next one while the device works), ingested exactly as the frame loop ingests it (bfIngestFrame) into
a ring of 16 device slots, and every 16 frames with a finite pose go into the hash in one bfTsdfIntegrateBatch pass, with a garbage collection
after each batch; the mesh comes from CUDAMarchingCubesHashSDF."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _capi as capi
from .frame_loop import default_params
from .marching_cubes import CUDAMarchingCubesHashSDF, marching_cubes_params
from .scene_rep import CUDASceneRepHashSDF
from .sens import SensorDataReader

BATCH = 16                       # bfTsdfIntegrateBatch's limit
# the bytes per bucket CUDASceneRepHashSDF allocates: the hash and compactified entries, the decision and prefix ints, one mutex int
TABLE_BYTES_PER_BUCKET = capi.BF_HASH_BUCKET_SIZE * (2 * C.sizeof(capi.BFHashEntry) + 2 * 4) + 4
BUCKET_GROWTH = 1.25             # ratio of fit_hash_params' bucket-count sequence
MAX_BUCKETS = (2 ** 32 - 1) // capi.BF_HASH_BUCKET_SIZE        # entry indices are 32-bit in the kernels
# fit_hash_params' bucket cap when no max_table_bytes is given.  The reference's bucket function maps many distinct blocks to the same 32-bit
# value, so on large scans no bucket count removes every overflow (a 1.4 M-block surface keeps 32 blocks over at any count; an 800 k-block
# box needs more than 55 buckets per block); the cap keeps the table finite and the fit reports what remains as "predicted_overflow".
DEFAULT_BUCKETS_PER_BLOCK = 32


def recording_params(header, n: int):
    """the frame loop's parameters for a recording of n frames (its sizes and intrinsics; frame store and keyframe capacity for n frames)"""
    P = default_params(header.depthWidth, header.depthHeight)
    P.colorWidth, P.colorHeight = header.colorWidth, header.colorHeight          # the ingest resamples colour to the integration size, as CUDAImageManager::process does
    for k in range(16):
        P.depthIntrinsics[k] = header.depthIntrinsic[k]; P.colorIntrinsics[k] = header.colorIntrinsic[k]
    P.maxNumFrames = max(32, n + int(P.submapSize))                                  # frame store / trajectories: the sequence plus one chunk of slack
    P.maxNumImages = max(8, (int(P.maxNumFrames) + int(P.submapSize) - 1) // int(P.submapSize) + 1)      # one keyframe per chunk
    return P


def ingest_params(P) -> capi.BFIngestParams:
    """the BFIngestParams the frame loop derives from its parameters (bfFrameLoopCreate)"""
    p = capi.BFIngestParams()
    p.depthWidth, p.depthHeight, p.colorWidth, p.colorHeight = P.depthWidth, P.depthHeight, P.colorWidth, P.colorHeight
    p.widthIntegration, p.heightIntegration = P.integrationWidth, P.integrationHeight
    p.erodeIterations, p.erodeStructureSize, p.erodeDThresh, p.erodeFracReq = (2 if P.erodeSIFTdepth else 0), 3, 0.05, 0.3
    p.depthSigmaD, p.depthSigmaR = (P.depthSigmaD if P.depthFilter else 0.0), P.depthSigmaR
    return p


def integration_camera(P) -> capi.BFDepthCameraParams:
    """the frame loop's integration camera: the depth intrinsics scaled to the integration size, in float32 as bfFrameLoopCreate forms them"""
    f = np.float32
    K = np.array(list(P.depthIntrinsics), f)
    Wi, Hi, Wd, Hd = f(P.integrationWidth), f(P.integrationHeight), f(P.depthWidth), f(P.depthHeight)
    cam = capi.BFDepthCameraParams()
    cam.fx, cam.fy = float(K[0] * Wi / Wd), float(K[5] * Hi / Hd)
    cam.mx, cam.my = float(K[2] * (Wi - f(1)) / (Wd - f(1))), float(K[6] * (Hi - f(1)) / (Hd - f(1)))
    cam.m_imageWidth, cam.m_imageHeight = P.integrationWidth, P.integrationHeight
    cam.m_sensorDepthWorldMin, cam.m_sensorDepthWorldMax = P.renderDepthMin, P.renderDepthMax
    return cam


def fine_hash_params(P, voxel_size: float, hash_buckets: int | None = None, sdf_blocks: int | None = None) -> capi.BFHashParams:
    """the loop's hash parameters at another voxel size; without explicit sizes the bucket and block counts grow with the surface area a block
    covers, (loop voxel / voxel_size)^2"""
    hp = capi.BFHashParams()
    C.memmove(C.byref(hp), C.byref(P.hash), C.sizeof(capi.BFHashParams))
    s = (float(P.hash.m_virtualVoxelSize) / voxel_size) ** 2
    hp.m_virtualVoxelSize = voxel_size
    hp.m_hashNumBuckets = int(hash_buckets) if hash_buckets is not None else int(P.hash.m_hashNumBuckets * s) | 1
    hp.m_numSDFBlocks = int(sdf_blocks) if sdf_blocks is not None else int(P.hash.m_numSDFBlocks * s)
    return hp


def table_bytes(buckets: int) -> int:
    """device bytes of a hash table of `buckets` buckets, as CUDASceneRepHashSDF allocates it (the heap and voxel blocks not included)"""
    return int(buckets) * TABLE_BYTES_PER_BUCKET


def bucket_candidates(count: int, max_buckets: int = MAX_BUCKETS):
    """the odd bucket counts fit_hash_params tries, in order: floor(max(count, 1) * BUCKET_GROWTH^k) | 1 for k = 0, 1, ..., repeats dropped,
    up to max_buckets"""
    base, k, last = max(int(count), 1), 0, 0
    while True:
        b = int(base * BUCKET_GROWTH ** k) | 1
        k += 1
        if b > max_buckets:
            return
        if b > last:
            last = b
            yield b


class BlockCounter:
    """The union of the SDF blocks that bfTsdfIntegrateBatch's alloc launches would insert for the frames given to add(), kept on the device
    (bfTsdfCountBlocks into a BFBlockKeySet in torch storage).  hash_params: the fusion's parameters -- voxel size, truncation,
    m_maxIntegrationDistance and the m_dummy shard setting; its table sizes are not read.  The set grows by itself: add() merges it into one
    twice as large, and counts the frames again, whenever a key was refused or the set is more than half full."""

    def __init__(self, hash_params, device="cuda:0", capacity: int = 1 << 16):
        import torch
        if capacity < 1 or capacity & (capacity - 1) or capacity > 1 << 31:
            raise ValueError("capacity: a power of two <= 2^31")
        self._torch = torch
        self.device = torch.device(device)
        self.lib = capi.lib()
        self.hash_params = capi.BFHashParams()
        C.memmove(C.byref(self.hash_params), C.byref(hash_params), C.sizeof(capi.BFHashParams))
        self._set, self._keys, self._ctrs = self._new(capacity)
        self._load, self._out = None, torch.zeros(3, dtype=torch.int32, device=self.device)

    def _new(self, capacity: int):
        t = self._torch
        keys = t.zeros(capacity, dtype=t.int64, device=self.device)
        ctrs = t.zeros(3, dtype=t.int32, device=self.device)
        s = capi.BFBlockKeySet()
        s.d_keys, s.d_counters, s.capacity = keys.data_ptr(), ctrs.data_ptr(), capacity
        return s, keys, ctrs

    def _bind_stream(self):
        t = self._torch
        t.cuda.set_device(self.device)
        self.lib.bfSetStream(C.c_void_p(t.cuda.current_stream(self.device).cuda_stream))

    def _counters(self):
        stored, refused, out_of_range = (int(x) for x in self._ctrs.cpu().tolist())
        if out_of_range:
            raise RuntimeError(f"{out_of_range} blocks lie more than 2^20 blocks from the origin: the key set cannot hold them")
        return stored, refused

    def _grow(self, need: int):
        cap = self._set.capacity
        while cap < 2 * need:
            cap *= 2
        if cap > 1 << 31:
            raise RuntimeError(f"{need} blocks: more than the key set's 2^30")
        s, keys, ctrs = self._new(cap)
        capi.check(self.lib.bfTsdfBlockKeyMerge(C.byref(s), C.byref(self._set)), "bfTsdfBlockKeyMerge")
        self._set, self._keys, self._ctrs = s, keys, ctrs

    @property
    def capacity(self) -> int:
        return int(self._set.capacity)

    def add(self, depth_ptrs, poses, cam, frames=None) -> None:
        """counts frame frames[k] of depth_ptrs (cuda tensors or raw device pointers; default frames = 0..n-1) at camera-to-world pose poses[k]
        [n, 4, 4]; any n.  Synchronises once per 16 frames."""
        T = np.ascontiguousarray(poses, dtype=np.float32).reshape(-1, 16)
        f = np.arange(len(T), dtype=np.int32) if frames is None else np.ascontiguousarray(frames, dtype=np.int32).reshape(-1)
        if len(f) != len(T):
            raise ValueError("frames and poses differ in length")
        ptr = lambda x: x if isinstance(x, int) or x is None else x.data_ptr()
        dptr = (C.c_void_p * len(depth_ptrs))(*[ptr(x) for x in depth_ptrs])
        self._bind_stream()
        for s in range(0, len(f), BATCH):
            fk, Tk = f[s:s + BATCH].copy(), T[s:s + BATCH].copy()
            while True:
                capi.check(self.lib.bfTsdfCountBlocks(C.byref(self._set), C.byref(self.hash_params), C.byref(cam), fk.ctypes.data, Tk.ctypes.data, len(fk),
                                                      C.cast(dptr, C.c_void_p)), "bfTsdfCountBlocks")
                stored, refused = self._counters()
                if refused or 2 * stored > self.capacity:
                    self._grow(stored + refused)
                if not refused:
                    break

    @property
    def count(self) -> int:
        """distinct blocks counted so far (synchronises)"""
        return self._counters()[0]

    def bucket_load(self, buckets: int) -> dict:
        """{"keys", "max_load", "over"} of the counted blocks in `buckets` buckets of the hash's bucket function (bfTsdfBlockKeyLoad); over = sum
        over buckets of max(0, load - BF_HASH_BUCKET_SIZE).  Synchronises."""
        t = self._torch
        if self._load is None or self._load.numel() < buckets:
            self._load = t.empty(int(buckets), dtype=t.int32, device=self.device)
        self._bind_stream()
        capi.check(self.lib.bfTsdfBlockKeyLoad(C.byref(self._set), int(buckets), self._load.data_ptr(), self._out.data_ptr()), "bfTsdfBlockKeyLoad")
        keys, mx, over = (int(x) for x in self._out.cpu().tolist())
        return {"keys": keys, "max_load": mx, "over": over}

    def keys(self) -> np.ndarray:
        """the counted block positions, int32 [count, 3], in lexicographic order"""
        k = self._keys.cpu().numpy().view(np.uint64)
        k = np.sort(k[k != 0])
        lim = 1 << 20
        pos = np.stack([(k >> np.uint64(42)) & np.uint64(0x1FFFFF), (k >> np.uint64(21)) & np.uint64(0x1FFFFF), k & np.uint64(0x1FFFFF)], axis=1)
        return (pos.astype(np.int64) - lim).astype(np.int32)


def fit_hash_params(base_hp, voxel_size: float, counter, max_table_bytes: int | None = None):
    """Hash parameters for a fusion of the blocks `counter` (a BlockCounter) counted: base_hp's parameters at voxel_size, a heap of exactly the
    count, and the first bucket count of bucket_candidates(count) under which no bucket holds more than BF_HASH_BUCKET_SIZE counted blocks
    (over == 0: no insert of the fusion can be dropped).  When no such bucket count fits in max_table_bytes (table_bytes; default: the table of
    DEFAULT_BUCKETS_PER_BLOCK buckets per counted block), the largest odd one that fits is taken and its over reported as "predicted_overflow".
    Returns (BFHashParams, report)."""
    if np.float32(voxel_size) != np.float32(counter.hash_params.m_virtualVoxelSize):
        raise ValueError(f"the counter counted {counter.hash_params.m_virtualVoxelSize} m voxels, not {voxel_size} m")
    count = counter.count
    if max_table_bytes is None:
        max_table_bytes = table_bytes(DEFAULT_BUCKETS_PER_BLOCK * max(count, 1) + 1)
    cap = min(MAX_BUCKETS, int(max_table_bytes) // TABLE_BYTES_PER_BUCKET)
    if cap < 1:
        raise ValueError(f"max_table_bytes {max_table_bytes}: less than one bucket ({TABLE_BYTES_PER_BUCKET} bytes)")
    buckets, load, tried = None, None, 0
    for b in bucket_candidates(count, cap):
        load, tried = counter.bucket_load(b), tried + 1
        if load["over"] == 0:
            buckets = b
            break
    if buckets is None:
        buckets = cap if cap & 1 else cap - 1
        load, tried = counter.bucket_load(buckets), tried + 1
    hp = capi.BFHashParams()
    C.memmove(C.byref(hp), C.byref(base_hp), C.sizeof(capi.BFHashParams))
    hp.m_virtualVoxelSize = voxel_size
    hp.m_hashNumBuckets = buckets
    hp.m_numSDFBlocks = max(1, count)
    report = {"blocks_counted": count, "buckets": buckets, "sdf_blocks": int(hp.m_numSDFBlocks), "table_bytes": table_bytes(buckets),
              "max_load": load["max_load"], "predicted_overflow": load["over"], "candidates_tried": tried}
    return hp, report


def mesh_scene(scene, ply_path: str, device="cuda:0", max_num_triangles: int = 6_000_000, whole: bool = False, device_mesh: bool = False) -> dict:
    """iso-surface of a scene (threshold 10 x voxel, the reference's s_SDFMarchingCubeThreshFactor) saved as PLY.  Returns {"triangles" (in the
    mesh), "triangles_found" (the cells produced), "triangles_dropped" (found - kept: what a full buffer of max_num_triangles lost), "mesh_path"}.
    whole=True extracts through CUDAMarchingCubesHashSDF.extractIsoSurfaceWhole -- counted first, then in parts that fit the buffer, so nothing
    is dropped -- and adds its report under "mesh".
    device_mesh=True extracts the whole soup into device memory (CUDAMarchingCubesHashSDF.extractSoup) and cleans it up there (weld): the same
    PLY as saveMesh, written from the device mesh; the weld's report and the bytes the path holds at once go under "mesh".  It trades device
    memory (soup, workspace and outputs together) for time, so it is an option."""
    if whole and device_mesh:
        raise ValueError("mesh_scene: whole and device_mesh are two different paths; pick one")
    hp = scene.m_hashParams
    mc = CUDAMarchingCubesHashSDF(marching_cubes_params(int(hp.m_hashNumBuckets), float(hp.m_virtualVoxelSize), max_num_triangles), device)
    try:
        out = {}
        if device_mesh:
            mesh = mc.extractMesh(scene)
            n = int(mesh.info["triangles_in"])
            out.update(mesh={**mesh.info, "peak_device_bytes": mesh.info.pop("device_bytes")}, triangles=n, triangles_found=n, triangles_dropped=0,
                       mesh_path=mesh.save_ply(ply_path))
            return out
        if whole:
            out["mesh"] = mc.extractIsoSurfaceWhole(scene)
        else:
            mc.extractIsoSurface(scene)
        found, kept = mc.lastExtraction()
        out.update(triangles=kept, triangles_found=found, triangles_dropped=found - kept, mesh_path=mc.saveMesh(ply_path, overwrite=True))
        return out
    finally:
        mc.close()


def fuse_recording(sens_path: str, ply_path: str | None = None, voxel_size: float = 0.004, poses="recorded", hash_buckets: int | None = None,
                   sdf_blocks: int | None = None, device="cuda:0", max_frames: int | None = None, scene: CUDASceneRepHashSDF | None = None,
                   max_num_triangles: int = 6_000_000, fit_hash: bool = False, max_table_bytes: int | None = None, whole_mesh: bool = False,
                   device_mesh: bool = False) -> dict:
    """Fuses a .sens recording along fixed camera-to-world poses -- "recorded" (the poses stored with the frames) or an array [n, 4, 4] --
    into a voxel hash of voxel_size (or into ``scene``, a reset CUDASceneRepHashSDF), with no bundling.  Frames whose pose is not finite are
    skipped.  Returns {"frames", "fused", "skipped", "batches", "inserts_dropped" (block inserts the hash had no room for), "heap_free",
    "triangles", "mesh_path", "scene"}.
    fit_hash=True sizes the hash from the blocks the fusion will allocate: a first pass decodes and ingests every frame as the fusion does and
    counts them (BlockCounter), fit_hash_params sizes the hash (within max_table_bytes), and the fusion runs as a second pass.  The result then
    also holds "blocks_counted", "buckets", "predicted_overflow" (0 unless max_table_bytes was too small to avoid overflow) and the whole
    report under "fit".  fit_hash excludes hash_buckets, sdf_blocks and scene.
    The mesh: "triangles_found" and "triangles_dropped" as mesh_scene reports them; whole_mesh=True meshes through mesh_scene(whole=True), which
    drops nothing however small max_num_triangles is, and adds its report under "mesh"; device_mesh=True meshes through
    mesh_scene(device_mesh=True)."""
    import torch
    if whole_mesh and device_mesh:
        raise ValueError("whole_mesh and device_mesh are two different mesh paths: pick one")
    if fit_hash and (hash_buckets is not None or sdf_blocks is not None or scene is not None):
        raise ValueError("fit_hash sizes the hash itself: pass no hash_buckets, sdf_blocks or scene")
    dev = torch.device(device)
    r = SensorDataReader(sens_path)
    try:
        n = len(r) if max_frames is None else min(len(r), max_frames)
        P = recording_params(r.header, n)
        if isinstance(poses, str):
            if poses != "recorded":
                raise ValueError("poses: 'recorded' or an array of camera-to-world poses")
            T = np.stack([r.frame_pose(i) for i in range(n)]) if n else np.zeros((0, 4, 4), np.float32)
        else:
            T = np.ascontiguousarray(poses, np.float32).reshape(-1, 4, 4)
            if len(T) < n:
                raise ValueError(f"{len(T)} poses for {n} frames")
        cam, ip, lib = integration_camera(P), ingest_params(P), capi.lib()
        Wi, Hi = int(P.integrationWidth), int(P.integrationHeight)
        raw_d = torch.empty((int(P.depthHeight), int(P.depthWidth)), dtype=torch.float32, device=dev)
        raw_c = torch.empty((int(P.colorHeight), int(P.colorWidth), 4), dtype=torch.uint8, device=dev)
        ring_d = torch.empty((BATCH, Hi, Wi), dtype=torch.float32, device=dev)
        ring_c = torch.empty((BATCH, Hi, Wi, 4), dtype=torch.uint8, device=dev)
        dptr, cptr = [ring_d[k] for k in range(BATCH)], [ring_c[k] for k in range(BATCH)]
        todo = [i for i in range(n) if np.isfinite(T[i]).all()]

        def batches(bind_stream):
            """decodes and ingests the frames of `todo` into the ring; yields the recording's frame indices of each full ring (or the last)"""
            cur = r.frame(todo[0], pinned=True) if todo else None
            for j, i in enumerate(todo):
                nxt = r.frame(todo[j + 1], pinned=True) if j + 1 < len(todo) else None        # decode the next frame while the device works on this one
                bind_stream()
                raw_d.copy_(cur[0], non_blocking=True); raw_c.copy_(cur[1], non_blocking=True)
                k = j % BATCH
                capi.check(lib.bfIngestFrame(C.byref(ip), raw_d.data_ptr(), raw_c.data_ptr(), ring_d[k].data_ptr(), ring_c[k].data_ptr()), "bfIngestFrame")
                if k == BATCH - 1 or j + 1 == len(todo):
                    yield todo[j - k:j + 1]
                cur = nxt

        fit = None
        if fit_hash:
            counter = BlockCounter(fine_hash_params(P, voxel_size), dev)
            for idx in batches(counter._bind_stream):
                counter.add(dptr[:len(idx)], T[idx], cam)
            hp, fit = fit_hash_params(P.hash, voxel_size, counter, max_table_bytes)
            del counter
            scene = CUDASceneRepHashSDF(hp, dev)
        elif scene is None:
            scene = CUDASceneRepHashSDF(fine_hash_params(P, voxel_size, hash_buckets, sdf_blocks), dev)
        out = {"frames": n, "fused": len(todo), "skipped": n - len(todo), "batches": 0}
        for idx in batches(scene._bind_stream):
            scene.integrateBatch(np.arange(len(idx)), T[idx], dptr, cptr, cam)
            scene.garbageCollect()
            out["batches"] += 1
        torch.cuda.synchronize(dev)
        out["inserts_dropped"] = scene.getLastFrameStats()["dropped"] if out["batches"] else 0
        out["heap_free"] = scene.getHeapFreeCount()
        if fit is not None:
            out.update(blocks_counted=fit["blocks_counted"], buckets=fit["buckets"], predicted_overflow=fit["predicted_overflow"], fit=fit)
        out.update(triangles=0, triangles_found=0, triangles_dropped=0, mesh_path=None, scene=scene)
        if ply_path is not None:
            out.update(mesh_scene(scene, ply_path, device, max_num_triangles, whole=whole_mesh, device_mesh=device_mesh))
        return out
    finally:
        r.close()

"""Fusion along a fixed trajectory: a recording's frames integrated at given poses into a voxel hash of any voxel size, then meshed -- no
bundling.  What the reference does with ``s_binaryDumpSensorUseTrajectory`` (FL/DepthSensing/DepthSensing.cpp:1036-1040, FL/SensorDataReader.cpp:131:
integrate along the poses stored with the frames), and the usual last step after a scan: fuse again along the final, optimised trajectory at a
finer voxel size (4-5 mm) and mesh that.

    fuse_recording(sens_path, ply_path, voxel_size=0.004, poses="recorded")      # a .sens file along its own poses
    FrameLoop.fuse(scene, poses=None)                                              # the loop's frame store along its optimised trajectory

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


def mesh_scene(scene, ply_path: str, device="cuda:0", max_num_triangles: int = 6_000_000) -> dict:
    """iso-surface of a scene (threshold 10 x voxel, the reference's s_SDFMarchingCubeThreshFactor) saved as PLY"""
    hp = scene.m_hashParams
    mc = CUDAMarchingCubesHashSDF(marching_cubes_params(int(hp.m_hashNumBuckets), float(hp.m_virtualVoxelSize), max_num_triangles), device)
    try:
        tri = mc.extractIsoSurface(scene) // 3
        return {"triangles": tri, "mesh_path": mc.saveMesh(ply_path, overwrite=True)}
    finally:
        mc.close()


def fuse_recording(sens_path: str, ply_path: str | None = None, voxel_size: float = 0.004, poses="recorded", hash_buckets: int | None = None,
                   sdf_blocks: int | None = None, device="cuda:0", max_frames: int | None = None, scene: CUDASceneRepHashSDF | None = None,
                   max_num_triangles: int = 6_000_000) -> dict:
    """Fuses a .sens recording along fixed camera-to-world poses -- "recorded" (the poses stored with the frames) or an array [n, 4, 4] --
    into a voxel hash of voxel_size (or into ``scene``, a reset CUDASceneRepHashSDF), with no bundling.  Frames whose pose is not finite are
    skipped.  Returns {"frames", "fused", "skipped", "batches", "inserts_dropped" (block inserts the hash had no room for: size it up when
    non-zero), "heap_free", "triangles", "mesh_path", "scene"}."""
    import torch
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
        if scene is None:
            scene = CUDASceneRepHashSDF(fine_hash_params(P, voxel_size, hash_buckets, sdf_blocks), dev)
        cam, ip, lib = integration_camera(P), ingest_params(P), capi.lib()
        Wi, Hi = int(P.integrationWidth), int(P.integrationHeight)
        raw_d = torch.empty((int(P.depthHeight), int(P.depthWidth)), dtype=torch.float32, device=dev)
        raw_c = torch.empty((int(P.colorHeight), int(P.colorWidth), 4), dtype=torch.uint8, device=dev)
        ring_d = torch.empty((BATCH, Hi, Wi), dtype=torch.float32, device=dev)
        ring_c = torch.empty((BATCH, Hi, Wi, 4), dtype=torch.uint8, device=dev)
        dptr, cptr = [ring_d[k] for k in range(BATCH)], [ring_c[k] for k in range(BATCH)]
        todo = [i for i in range(n) if np.isfinite(T[i]).all()]
        out = {"frames": n, "fused": len(todo), "skipped": n - len(todo), "batches": 0}
        cur = r.frame(todo[0], pinned=True) if todo else None
        for j, i in enumerate(todo):
            nxt = r.frame(todo[j + 1], pinned=True) if j + 1 < len(todo) else None        # decode the next frame while the device works on this one
            scene._bind_stream()
            raw_d.copy_(cur[0], non_blocking=True); raw_c.copy_(cur[1], non_blocking=True)
            k = j % BATCH
            capi.check(lib.bfIngestFrame(C.byref(ip), raw_d.data_ptr(), raw_c.data_ptr(), ring_d[k].data_ptr(), ring_c[k].data_ptr()), "bfIngestFrame")
            if k == BATCH - 1 or j + 1 == len(todo):
                idx = todo[j - k:j + 1]
                scene.integrateBatch(np.arange(k + 1), T[idx], dptr, cptr, cam)
                scene.garbageCollect()
                out["batches"] += 1
            cur = nxt
        torch.cuda.synchronize(dev)
        out["inserts_dropped"] = scene.getLastFrameStats()["dropped"] if out["batches"] else 0
        out["heap_free"] = scene.getHeapFreeCount()
        out.update(triangles=0, mesh_path=None, scene=scene)
        if ply_path is not None:
            out.update(mesh_scene(scene, ply_path, device, max_num_triangles))
        return out
    finally:
        r.close()

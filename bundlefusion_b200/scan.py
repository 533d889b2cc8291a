"""A recorded sequence in, a mesh and a trajectory out: the application-level path of the reference (FriedLiver's main loop over a ``SensorDataReader``: every frame through
``OnlineBundler::processInput`` / ``process`` and ``reintegrate`` / ``integrate``, then ``CUDAMarchingCubesHashSDF::extractIsoSurface`` + ``saveMesh`` and the optimised
trajectory; FL/FriedLiver.cpp, FL/DepthSensing/DepthSensing.cpp:966-1129, 1180-1230) over this library's pieces: ``sens.SensorDataReader`` -> ``FrameLoop.step`` (look-ahead on
the next decoded frame) -> ``CUDAMarchingCubesHashSDF``.  Host glue only; every stage is the C-ABI's.

    python -m bundlefusion_b200.scan scan.sens out.ply [--frames N] [--device cuda:0] [--solve-frames-before-exit 30]
        [--mesh-voxel-size V]       after the loop, fuse its frames along the final trajectory into a V-sized hash and mesh that (bundlefusion_b200.fuse)
        [--poses recorded]          no loop: fuse along the poses stored with the frames (the reference's s_binaryDumpSensorUseTrajectory)
        [--fit-hash]                size that fused hash from a count of the blocks it will hold (fuse.fit_hash_params), so it drops nothing
        [--grow-hash MAX_BLOCKS]    start the online hash at --sdf-blocks and let the loop grow it up to MAX_BLOCKS voxel blocks while it scans
        [--device-frames N]         keep N frame slots on the device and every frame in pinned host memory (same results, less device memory)
        [--whole-mesh]              count the mesh's triangles first and extract them in parts that fit the triangle buffer, so none is dropped
        [--device-mesh]             extract the whole soup into device memory and merge its vertices and faces there (same PLY, more device memory)

The JSON summary always carries "triangles_found" (what the iso-surface's cells produced) and "triangles_dropped" (what a full triangle buffer
lost: found - kept); with --whole-mesh it is 0, and the extraction's report (parts, buffer, synchronisations) goes under "mesh"; with
--device-mesh it is 0 too, and the weld's report (vertices, faces, rounds, synchronisations, peak device bytes) goes under "mesh".
"""
from __future__ import annotations

import argparse
import ctypes as C
import json

import numpy as np

from . import _capi as capi
from . import fuse
from .frame_loop import FrameLoop, default_params
from .scene_rep import CUDASceneRepHashSDF
from .sens import SensorDataReader


class _LoopScene:
    """what CUDAMarchingCubesHashSDF.extractIsoSurface reads of a scene: the loop's hash data and parameters"""

    def __init__(self, loop: FrameLoop):
        self.m_hashData = loop.lib.bfFrameLoopGetHashData(loop._h).contents
        self.m_hashParams = loop.lib.bfFrameLoopGetHashParams(loop._h).contents


def reconstruct(sens_path: str, ply_path: str | None = None, device="cuda:0", max_frames: int | None = None, hash_buckets: int | None = None,
                sdf_blocks: int | None = None, max_num_triangles: int = 6_000_000, tweak=None, solve_frames_before_exit: int | None = None,
                mesh_voxel_size: float | None = None, fit_hash: bool = False, grow_hash: int | None = None,
                device_frames: int | None = None, whole_mesh: bool = False, device_mesh: bool = False) -> dict:
    """runs the sequence; returns {"frames", "valid", "keyframes", "trajectory" [n, 4, 4], "mesh_path", "triangles", "status" (per frame)}.
    solve_frames_before_exit=K ends the recording as the reference does (FrameLoop.finish: sparse global solves to past-end turn K, the dense
    global solve at turn K, then re-integration until every frame is fused at its final pose) and adds that call's info under "finish";
    None runs a fixed submapSize + 2 past-end turns.  mesh_voxel_size=V: the loop's frames are then fused along its final trajectory into a
    fresh hash of voxel size V (FrameLoop.fuse) and that model is meshed instead of the online one; that call's info goes under "fuse".  With
    fit_hash that hash is sized by FrameLoop.fit_hash_params, whose report goes under "fit".  grow_hash=MAX_BLOCKS: the online hash starts at
    sdf_blocks (default: the loop's) and the loop may grow it up to MAX_BLOCKS voxel blocks (hashMaxSDFBlocks); FrameLoop.hash_growth() goes
    under "hash".  device_frames=N keeps N frame slots on the device over a pinned host store of every frame (deviceFrameSlots); the results
    do not change, and FrameLoop.frame_store() goes under "frame_store".  The mesh adds "triangles_found" and "triangles_dropped"
    (fuse.mesh_scene); whole_mesh=True extracts it counted and in parts that fit the buffer, dropping nothing, and adds the report under "mesh";
    device_mesh=True extracts the whole soup to the device and welds it there (fuse.mesh_scene(device_mesh=True)), report under "mesh"."""
    r = SensorDataReader(sens_path)
    n = len(r) if max_frames is None else min(len(r), max_frames)
    P = fuse.recording_params(r.header, n)
    if hash_buckets is not None:
        P.hash.m_hashNumBuckets = hash_buckets
    if sdf_blocks is not None:
        P.hash.m_numSDFBlocks = sdf_blocks
    if grow_hash is not None:
        P.hashMaxSDFBlocks = int(grow_hash)
    if device_frames is not None:
        P.deviceFrameSlots = int(device_frames)
    if tweak is not None:
        tweak(P)
    loop = FrameLoop(P, device)
    status = []
    cur = r.frame(0, pinned=True) if n else None
    for i in range(n):
        nxt = r.frame(i + 1, pinned=True) if i + 1 < n else None                      # decode the next frame while the device works on this one
        st = loop.step(cur[0], cur[1], *((nxt[0], nxt[1]) if nxt is not None else (None, None)))
        status.append(st.as_dict())
        cur = nxt
    # after the last frame the reference keeps turning its loop without input (FL/OnlineBundler.cpp:170-197) until the last, partial chunk is solved and the
    # re-integration list is empty
    finish = None
    if solve_frames_before_exit is not None:
        finish = loop.finish(solve_frames_before_exit)
    else:                                                                              # one chunk's worth of turns plus the frames one solve may move
        for _ in range(int(P.submapSize) + 2):
            loop.step_past_end()
    loop.join()
    out = {"frames": n, "valid": int(sum(s["validTransform"] for s in status)), "keyframes": loop.counters()["keyframes"], "trajectory": loop.trajectory(n), "status": status,
           "mesh_path": None, "triangles": 0, "triangles_found": 0, "triangles_dropped": 0}
    if finish is not None:
        out["finish"] = finish
    if grow_hash is not None:
        out["hash"] = loop.hash_growth()
    if mesh_voxel_size is not None:
        if fit_hash:
            hp, out["fit"] = loop.fit_hash_params(mesh_voxel_size, n=n)
        else:
            hp = fuse.fine_hash_params(P, mesh_voxel_size)
        scene = CUDASceneRepHashSDF(hp, device)
        out["fuse"] = loop.fuse(scene, n=n)
        if ply_path is not None:
            out.update(fuse.mesh_scene(scene, ply_path, device, max_num_triangles, whole=whole_mesh, device_mesh=device_mesh))
        scene.close()
    elif ply_path is not None:
        # the table the loop holds now: a grown one has more buckets than P.hash
        out.update(fuse.mesh_scene(_LoopScene(loop), ply_path, device, max_num_triangles, whole=whole_mesh, device_mesh=device_mesh))
    if device_frames is not None:
        out["frame_store"] = loop.frame_store()
    loop.close(); r.close()
    return out


def ate(estimated, recorded) -> dict:
    """Absolute trajectory error of camera-to-world poses [n, 4, 4] against the poses recorded with the sequence (the `.sens` frames carry them, e.g. ScanNet's): the
    camera centres of the frames valid in both are aligned by the least-squares rigid transform (Horn / Kabsch, float64, no scale), then RMSE / mean / max of the residual
    distances in metres.  Frames whose pose is not finite on either side (lost tracking: -inf) are left out."""
    E, R = np.asarray(estimated, np.float64), np.asarray(recorded, np.float64)
    n = min(len(E), len(R))
    ok = np.array([np.isfinite(E[i]).all() and np.isfinite(R[i]).all() for i in range(n)], bool)
    if ok.sum() < 3:
        return {"frames": int(ok.sum()), "rmse": float("nan"), "mean": float("nan"), "max": float("nan")}
    a, b = E[:n][ok][:, :3, 3], R[:n][ok][:, :3, 3]
    ca, cb = a.mean(0), b.mean(0)
    U, _, Vt = np.linalg.svd((a - ca).T @ (b - cb))
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(Vt.T @ U.T))])
    Rot = Vt.T @ D @ U.T
    d = np.linalg.norm((Rot @ (a - ca).T).T + cb - b, axis=1)
    return {"frames": int(ok.sum()), "rmse": float(np.sqrt((d * d).mean())), "mean": float(d.mean()), "max": float(d.max())}


def recorded_poses(sens_path: str, max_frames: int | None = None) -> np.ndarray:
    """the camera-to-world poses stored with the frames ([n, 4, 4]; all -inf where the recorder had none)"""
    r = SensorDataReader(sens_path)
    n = len(r) if max_frames is None else min(len(r), max_frames)
    out = np.stack([r.frame_pose(i) for i in range(n)]) if n else np.zeros((0, 4, 4), np.float32)
    r.close()
    return out


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("sens"); ap.add_argument("ply")
    ap.add_argument("--frames", type=int, default=None); ap.add_argument("--device", default="cuda:0")
    ap.add_argument("--hash-buckets", type=int, default=None); ap.add_argument("--sdf-blocks", type=int, default=None)
    ap.add_argument("--trajectory", default=None, help="write the camera-to-world poses here (one 4x4 per frame, text)")
    ap.add_argument("--solve-frames-before-exit", type=int, default=None, metavar="K",
                    help="end the recording as the reference does: global solves for K turns past the last frame, the dense global solve at turn K, then "
                         "re-integration until every frame is fused at its final pose (the reference's value is 30); without it, a fixed 12 past-end turns")
    ap.add_argument("--mesh-voxel-size", type=float, default=None, metavar="V",
                    help="fuse the frames again along the final trajectory into a hash of voxel size V (metres, e.g. 0.004) and mesh that instead of the online model")
    ap.add_argument("--poses", choices=("recorded",), default=None,
                    help="'recorded': no bundling -- fuse along the poses stored with the frames (at --mesh-voxel-size, default the loop's 1 cm) and mesh that")
    ap.add_argument("--fit-hash", action="store_true",
                    help="with --mesh-voxel-size or --poses recorded: count the blocks the fusion will allocate and size its hash from the count, so that "
                         "no insert is dropped (the JSON summary carries the report under 'fit')")
    ap.add_argument("--grow-hash", type=int, default=None, metavar="MAX_BLOCKS",
                    help="start the online hash at --sdf-blocks (default: the loop's) and grow it while scanning, up to MAX_BLOCKS voxel blocks "
                         "(the JSON summary carries growths, sizes and dropped inserts under 'hash')")
    ap.add_argument("--device-frames", type=int, default=None, metavar="N",
                    help="keep N frame slots on the device over a pinned host store of every frame, N >= 16 (the results do not change; the JSON "
                         "summary carries slots, bytes, fetches and hits under 'frame_store')")
    ap.add_argument("--whole-mesh", action="store_true",
                    help="count the iso-surface's triangles on the device and extract them in parts that fit the triangle buffer, so that none is "
                         "dropped (the JSON summary carries the extraction's report under 'mesh')")
    ap.add_argument("--device-mesh", action="store_true",
                    help="extract the whole triangle soup into device memory and merge its vertices and faces there: the same PLY, cleaned up on the device, "
                         "for the device memory of soup, workspace and mesh at once (the JSON summary carries the weld's report under 'mesh')")
    a = ap.parse_args(argv)
    if a.whole_mesh and a.device_mesh:
        ap.error("--whole-mesh and --device-mesh are two different mesh paths: pick one")
    if a.fit_hash and a.poses != "recorded" and a.mesh_voxel_size is None:
        ap.error("--fit-hash sizes a fused hash: use it with --mesh-voxel-size or --poses recorded")
    if a.poses == "recorded":
        if a.fit_hash and (a.hash_buckets is not None or a.sdf_blocks is not None):
            ap.error("--fit-hash sizes the fused hash itself: drop --hash-buckets / --sdf-blocks")
        voxel = a.mesh_voxel_size if a.mesh_voxel_size is not None else float(default_params(16, 16).hash.m_virtualVoxelSize)
        o = fuse.fuse_recording(a.sens, a.ply, voxel, "recorded", a.hash_buckets, a.sdf_blocks, a.device, a.frames, fit_hash=a.fit_hash,
                                whole_mesh=a.whole_mesh, device_mesh=a.device_mesh)
        o["scene"].close()
        summary = {"frames": o["frames"], "fuse": {k: o[k] for k in ("fused", "skipped", "batches", "inserts_dropped", "heap_free")},
                   "triangles": o["triangles"], "mesh_path": o["mesh_path"], "triangles_found": o["triangles_found"],
                   "triangles_dropped": o["triangles_dropped"]}
        if "fit" in o:
            summary["fit"] = o["fit"]
        if "mesh" in o:
            summary["mesh"] = o["mesh"]
        print(json.dumps(summary))
        return 0
    o = reconstruct(a.sens, a.ply, a.device, a.frames, a.hash_buckets, a.sdf_blocks, solve_frames_before_exit=a.solve_frames_before_exit,
                    mesh_voxel_size=a.mesh_voxel_size, fit_hash=a.fit_hash, grow_hash=a.grow_hash,
                    device_frames=a.device_frames, whole_mesh=a.whole_mesh, device_mesh=a.device_mesh)
    if a.trajectory:
        np.savetxt(a.trajectory, o["trajectory"].reshape(-1, 16))
    summary = {k: o[k] for k in ("frames", "valid", "keyframes", "triangles", "mesh_path", "triangles_found", "triangles_dropped")}
    if "mesh" in o:
        summary["mesh"] = o["mesh"]
    if "finish" in o:
        summary["finish"] = o["finish"]                     # its "valid": StopScanningAndExit's verdict on the reconstruction
    if "fuse" in o:
        summary["fuse"] = {k: o["fuse"][k] for k in ("frames_fused", "frames_skipped", "batches", "inserts_dropped", "heap_free")}
    if "fit" in o:
        summary["fit"] = o["fit"]
    if "hash" in o:
        summary["hash"] = {k: o["hash"][k] for k in ("growths", "sdf_blocks", "buckets", "inserts_dropped")}
    if "frame_store" in o:
        summary["frame_store"] = o["frame_store"]
    gt = recorded_poses(a.sens, a.frames)
    if np.isfinite(gt).all(axis=(1, 2)).sum() >= 3:
        summary["ate"] = ate(o["trajectory"], gt[:len(o["trajectory"])])
    print(json.dumps(summary))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())

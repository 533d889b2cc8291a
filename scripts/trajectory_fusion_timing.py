"""Fusion rate along a fixed trajectory (FrameLoop.fuse, bfFrameLoopFuse) on bench.py's stream configuration (development aid).

usage: trajectory_fusion_timing.py [--preroll 250] [--frames 1000] [--stride 2] [--reps 2] [--out FILE]

The synthetic 640x480 stream of bench.py's loop workload (rich texture, 1 cm voxels, 4 M-block heap, two streams, look-ahead) is stepped for
preroll + frames frames and finished (bfFrameLoopFinish, K = 30); its frame store is then fused along the final trajectory into a fresh hash at
1 cm and at 4 mm:
  rate:     frames per second of whole FrameLoop.fuse calls (wall clock around a call that ends in a device synchronise), batched
            (bfTsdfIntegrateBatch, 16 frames a pass) and one op per call (bfTsdfSetBatching(0), the BF_TSDF_BATCH=0 path), alternated, `reps` each;
  stencil:  one profiled call per mode -- the stencil launches' summed CUDA-event time and their algorithmic bytes (DESIGN §3b: 24 B x U + 20 B x E
            + 2 W H 4 B per pass, summed over the passes a batch launch performs) over that time;
  union:    one batched pass through CUDASceneRepHashSDF.integrateBatch with the union list's size read after every batch, against the mean E
            (in-frustum blocks) of the frames in it.
The target hashes are sized from the blocks the loop's own 1 cm model uses (x 1.5 at 1 cm, x 8 at 4 mm); inserts_dropped says whether that was
enough.  Prints one JSON line with the card's name and power limit read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bundlefusion_b200 import _capi as capi  # noqa: E402
from bundlefusion_b200 import synth_gpu  # noqa: E402
from bundlefusion_b200.frame_loop import FrameLoop, default_params  # noqa: E402
from bundlefusion_b200.fuse import integration_camera  # noqa: E402
from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF  # noqa: E402

W, H = 640, 480


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                  # the name from torch is still reported
        q = f"nvidia-smi unavailable: {e}"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.splitlines()[0] if q else ""}


def stream_bank(n, stride, dev):
    depth = torch.empty(n, H, W, dtype=torch.float32, device=dev); color = torch.empty(n, H, W, 4, dtype=torch.uint8, device=dev)
    for s0 in range(0, n, 64):
        idx = [stride * i for i in range(s0, min(n, s0 + 64))]
        d, c, _ = synth_gpu.make_frames(idx, W, H, device=str(dev), texture="rich")
        depth[s0:s0 + len(idx)] = d; color[s0:s0 + len(idx)] = c
    return depth, color


def target_params(loop, voxel, blocks):
    hp = capi.BFHashParams()
    C.memmove(C.byref(hp), C.byref(loop.lib.bfFrameLoopGetHashParams(loop._h).contents), C.sizeof(capi.BFHashParams))
    hp.m_virtualVoxelSize = voxel; hp.m_numSDFBlocks = blocks; hp.m_hashNumBuckets = (2 * blocks) | 1
    return hp


def algorithmic_bytes(U, E, frames):
    return 24 * U + 20 * E + 2 * W * H * 4 * frames


def profiled(lib, loop, scene, batching):
    lib.bfTsdfSetBatching(batching)
    scene.reset()
    lib.bfTsdfSetProfiling(1)
    info = loop.fuse(scene)
    out = (C.c_ulonglong * 16)()
    capi.check(lib.bfTsdfGetProfileEx(C.byref(scene.m_hashData), out), "bfTsdfGetProfileEx")
    lib.bfTsdfSetProfiling(0)
    launches, timed, ns, U, E, frames = (int(out[k]) for k in range(6))
    assert timed == launches, "not every stencil launch was timed"
    ms = ns / 1e6
    return {"launches": launches, "stencil_ms": round(ms, 3), "U": U, "E": E, "frames_read": frames,
            "algorithmic_GBps": round(algorithmic_bytes(U, E, frames) / (ms * 1e-3) / 1e9, 1) if ms else None,
            "batch_launches": int(out[8]), "culled_probes": int(out[15]), "frames_fused": info["frames_fused"]}


def union_vs_e(lib, loop, scene, n):
    """one batched pass through integrateBatch: the union list's size after every batch against the summed / mean E of its frames"""
    traj = loop.trajectory(n)
    fin = [f for f in range(n) if np.isfinite(traj[f]).all()]
    frames = [loop.frame(f) for f in range(n)]
    cam = integration_camera(loop.params)
    scene.reset()
    lib.bfTsdfSetProfiling(1)
    union, esum, nfr = [], 0, 0
    out = (C.c_ulonglong * 16)()
    for s in range(0, len(fin), 16):
        idx = fin[s:s + 16]
        scene.integrateBatch(idx, traj[idx], [f[0] for f in frames], [f[1] for f in frames], cam)
        union.append(scene.getLastFrameStats()["E"])
        capi.check(lib.bfTsdfGetProfileEx(C.byref(scene.m_hashData), out), "bfTsdfGetProfileEx")
        esum += int(out[12]); nfr += int(out[13])
        scene.garbageCollect()
    lib.bfTsdfSetProfiling(0)
    mean_union = float(np.mean(union)) if union else 0.0
    mean_e = esum / max(1, nfr)
    return {"batches": len(union), "mean_union_blocks": round(mean_union, 1), "mean_frame_E": round(mean_e, 1),
            "union_over_frame_E": round(mean_union / mean_e, 3) if mean_e else None, "voxel_passes_saved": round(16 * mean_e / mean_union, 2) if mean_union else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preroll", type=int, default=250); ap.add_argument("--frames", type=int, default=1000); ap.add_argument("--stride", type=int, default=2)
    ap.add_argument("--reps", type=int, default=2); ap.add_argument("--K", type=int, default=30); ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("trajectory_fusion_timing.py needs a CUDA device")
    dev = torch.device("cuda:0")
    n = a.preroll + a.frames
    depth, color = stream_bank(n, a.stride, dev)
    P = default_params(W, H)
    P.maxNumFrames = n + 8; P.maxNumImages = n // 10 + 8; P.maxGlobalResiduals = 25 * P.maxNumImages * 48          # bench.py run_loop's sizing
    P.hash.m_hashNumBuckets = 4_000_000; P.hash.m_numSDFBlocks = 4_000_000
    loop = FrameLoop(P, dev)
    loop.set_overlap(True)
    t0 = time.perf_counter()
    for f in range(n):
        loop.step(depth[f], color[f], *((depth[f + 1], color[f + 1]) if f + 1 < n else (None, None)))
    finish = loop.finish(a.K)
    loop.join(); torch.cuda.synchronize()
    loop_s = time.perf_counter() - t0
    del depth, color
    torch.cuda.empty_cache()
    used = int(P.hash.m_numSDFBlocks) - loop.heap_free()
    lib = capi.lib()
    prev = lib.bfTsdfSetBatching(1)
    res = {}
    try:
        for voxel, scale in ((0.01, 1.5), (0.004, 8.0)):
            scene = CUDASceneRepHashSDF(target_params(loop, voxel, int(used * scale) + 20000), dev)
            runs = {"batched": [], "one_op_per_call": []}
            infos = {}
            for _ in range(a.reps):
                for mode, b in (("batched", 1), ("one_op_per_call", 0)):
                    lib.bfTsdfSetBatching(b)
                    scene.reset(); torch.cuda.synchronize()
                    t = time.perf_counter()
                    info = loop.fuse(scene)                     # ends in a device synchronise (the heap free count)
                    dt = time.perf_counter() - t
                    runs[mode].append(round(info["frames_fused"] / dt, 1))
                    infos[mode] = info
            res["%gmm" % (voxel * 1000)] = {
                "blocks": int(scene.m_hashParams.m_numSDFBlocks), "fps": runs,
                "speedup_median": round(float(np.median(runs["batched"]) / np.median(runs["one_op_per_call"])), 3),
                "info": infos, "same_heap_free": infos["batched"]["heap_free"] == infos["one_op_per_call"]["heap_free"],
                "stencil": {"batched": profiled(lib, loop, scene, 1), "one_op_per_call": profiled(lib, loop, scene, 0)},
                "union": union_vs_e(lib, loop, scene, n),
            }
            scene.close(); del scene
            torch.cuda.empty_cache()
    finally:
        lib.bfTsdfSetBatching(prev)
    out = {"card": card(), "frames": n, "preroll": a.preroll, "stride": a.stride, "loop_and_finish_s": round(loop_s, 2), "finish_done": finish["done"],
           "loop_blocks_used": used, "fusion": res}
    loop.close()
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()

"""Cost and effect of sizing a fusion's hash from a block count (FrameLoop.fit_hash_params) on bench.py's stream configuration (development aid).

usage: hash_fit_timing.py [--preroll 250] [--frames 1000] [--stride 2] [--reps 2] [--out FILE]

The loop runs and finishes as in scripts/trajectory_fusion_timing.py (the same stream, hash and K = 30); its frame store is then fused along the
final trajectory at 1 cm and at 4 mm, alternating, `reps` times each:
  fit:    FrameLoop.fit_hash_params -- the count pass over the frame store (bfTsdfCountBlocks) plus the bucket-count search
          (bfTsdfBlockKeyLoad per candidate) -- wall clock around the call, which ends in a device synchronise;
  fused:  FrameLoop.fuse into the fitted hash, wall clock around the call (it ends in a device synchronise);
  hand:   FrameLoop.fuse into trajectory_fusion_timing.py's hand-sized hash (x 1.5 / x 8 the loop's 1 cm blocks, 2 buckets per block).
Reported per voxel size: the count, the chosen bucket count and table bytes, both hashes' inserts_dropped, and the medians of the times.
Prints one JSON line with the card's name and power limit read in the same run."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bundlefusion_b200 import fuse  # noqa: E402
from bundlefusion_b200.frame_loop import FrameLoop, default_params  # noqa: E402
from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF  # noqa: E402
from trajectory_fusion_timing import W, H, card, stream_bank, target_params  # noqa: E402


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preroll", type=int, default=250); ap.add_argument("--frames", type=int, default=1000); ap.add_argument("--stride", type=int, default=2)
    ap.add_argument("--reps", type=int, default=2); ap.add_argument("--K", type=int, default=30); ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("hash_fit_timing.py needs a CUDA device")
    dev = torch.device("cuda:0")
    n = a.preroll + a.frames
    depth, color = stream_bank(n, a.stride, dev)
    P = default_params(W, H)
    P.maxNumFrames = n + 8; P.maxNumImages = n // 10 + 8; P.maxGlobalResiduals = 25 * P.maxNumImages * 48          # bench.py run_loop's sizing
    P.hash.m_hashNumBuckets = 4_000_000; P.hash.m_numSDFBlocks = 4_000_000
    loop = FrameLoop(P, dev)
    loop.set_overlap(True)
    for f in range(n):
        loop.step(depth[f], color[f], *((depth[f + 1], color[f + 1]) if f + 1 < n else (None, None)))
    finish = loop.finish(a.K)
    loop.join(); torch.cuda.synchronize()
    del depth, color
    torch.cuda.empty_cache()
    used = int(P.hash.m_numSDFBlocks) - loop.heap_free()
    res = {}
    for voxel, scale in ((0.01, 1.5), (0.004, 8.0)):
        fit_s, fused_s, hand_s, rep, fit_info, hand_info = [], [], [], None, None, None
        hand_hp = target_params(loop, voxel, int(used * scale) + 20000)
        for _ in range(a.reps):
            (hp, rep), dt = timed(lambda: loop.fit_hash_params(voxel))
            fit_s.append(dt)
            scene = CUDASceneRepHashSDF(hp, dev)
            fit_info, dt = timed(lambda: loop.fuse(scene))
            fused_s.append(dt)
            scene.close(); del scene
            torch.cuda.empty_cache()
            scene = CUDASceneRepHashSDF(hand_hp, dev)
            hand_info, dt = timed(lambda: loop.fuse(scene))
            hand_s.append(dt)
            scene.close(); del scene
            torch.cuda.empty_cache()
        res["%gmm" % (voxel * 1000)] = {
            "fit_hash_params_s": round(float(np.median(fit_s)), 4), "fused_call_s": round(float(np.median(fused_s)), 4),
            "fit_over_fused": round(float(np.median(fit_s) / np.median(fused_s)), 3), "hand_sized_fused_call_s": round(float(np.median(hand_s)), 4),
            "fit": rep, "fitted_inserts_dropped": fit_info["inserts_dropped"], "frames_fused": fit_info["frames_fused"],
            "hand_sized": {"sdf_blocks": int(hand_hp.m_numSDFBlocks), "buckets": int(hand_hp.m_hashNumBuckets),
                           "table_bytes": fuse.table_bytes(int(hand_hp.m_hashNumBuckets)), "inserts_dropped": hand_info["inserts_dropped"]},
            "times_s": {"fit": [round(x, 4) for x in fit_s], "fused": [round(x, 4) for x in fused_s], "hand": [round(x, 4) for x in hand_s]},
        }
    out = {"card": card(), "frames": n, "preroll": a.preroll, "stride": a.stride, "finish_done": finish["done"], "loop_blocks_used": used, "fusion": res}
    loop.close()
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()

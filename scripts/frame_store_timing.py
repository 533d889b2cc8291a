"""Cost of keeping the frame loop's frames in pinned host memory behind a few device slots (deviceFrameSlots), on bench.py's stream (development aid).

usage: frame_store_timing.py [--preroll 250] [--frames 1000] [--stride 2] [--reps 2] [--slots 64,256] [--out FILE]

The bench stream at 640 x 480 (preroll + frames at 1 cm, overlap and look-ahead on), then finish(30) and a 1 cm fuse() of every frame along the
final trajectory, through a resident store (deviceFrameSlots = 0) and each --slots value, alternated, `reps` times each.  Per run: frames/s of
the steps after the preroll (wall clock ending in a device synchronise), finish and fuse wall time, fetches per turn and the hit rate (during the
steps, during finish, during fuse), copy bytes, device and pinned host bytes of the store, and the host time the create spent pinning.
H2D rate: after the run, groups of slots - 2 frames that are not resident are fetched with bfFrameLoopFetchFrames; CUDA events on the library
stream around each call, which waits for the copy stream's copies, give bytes / time.  Prints one JSON line with the card's name and power
limit read in the same run."""
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
from trajectory_fusion_timing import W, H, card, stream_bank  # noqa: E402


def rates(a, b, turns):
    fetched, hits = b["fetches"] - a["fetches"], b["hits"] - a["hits"]
    return {"fetches": fetched, "fetches_per_turn": round(fetched / max(1, turns), 3), "hit_rate": round(hits / max(1, hits + fetched), 4),
            "h2d_bytes": b["h2d_bytes"] - a["h2d_bytes"], "d2h_bytes": b["d2h_bytes"] - a["d2h_bytes"]}


def h2d_rate(loop, n, slots):
    """fetch groups of slots - 2 frames not resident now (the first frames, evicted long ago): bytes / event time"""
    res, g = [], slots - 2
    lib_stream = torch.cuda.current_stream()
    for s in range(0, min(n, 4 * g), g):
        frames = list(range(s, min(n, s + g)))
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        before = loop.frame_store()
        e0.record(lib_stream)
        loop.fetch_frames(frames)
        e1.record(lib_stream); torch.cuda.synchronize()
        b = loop.frame_store()["h2d_bytes"] - before["h2d_bytes"]
        ms = e0.elapsed_time(e1)
        if b:
            res.append({"frames": len(frames), "bytes": b, "event_ms": round(ms, 3), "gb_s": round(b / (ms * 1e-3) / 1e9, 2)})
    return res


def run(depth, color, pre, n, K, slots, dev):
    P = default_params(W, H)
    P.maxNumFrames = n + 8; P.maxNumImages = n // 10 + 8; P.maxGlobalResiduals = 25 * P.maxNumImages * 48          # bench.py run_loop's sizing
    P.hash.m_hashNumBuckets = 4_000_001; P.hash.m_numSDFBlocks = 2_000_000
    P.deviceFrameSlots = slots
    torch.cuda.synchronize()
    t = time.perf_counter()
    loop = FrameLoop(P, dev)
    torch.cuda.synchronize()
    create_s = time.perf_counter() - t
    loop.set_overlap(True)
    step = lambda f: loop.step(depth[f], color[f], *((depth[f + 1], color[f + 1]) if f + 1 < n else (None, None)))
    for f in range(pre):
        step(f)
    loop.join(); torch.cuda.synchronize()
    s0, t0 = loop.frame_store(), time.perf_counter()
    for f in range(pre, n):
        step(f)
    loop.join(); torch.cuda.synchronize()
    steps_s = time.perf_counter() - t0
    s1, t1 = loop.frame_store(), time.perf_counter()
    fin = loop.finish(K)
    loop.join(); torch.cuda.synchronize()
    finish_s = time.perf_counter() - t1
    s2 = loop.frame_store()
    scene = CUDASceneRepHashSDF(fuse.fine_hash_params(P, 0.01), dev)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    info = loop.fuse(scene)
    torch.cuda.synchronize()
    fuse_s = time.perf_counter() - t2
    s3 = loop.frame_store()
    scene.close()
    out = {"slots": slots, "fps": round((n - pre) / steps_s, 2), "steps_s": round(steps_s, 3), "finish_s": round(finish_s, 3), "fuse_s": round(fuse_s, 3),
           "finish_turns": fin["turns"], "fuse_batches": info["batches"], "create_s": round(create_s, 3),
           "steps": rates(s0, s1, n - pre), "finish": rates(s1, s2, fin["turns"]), "fuse": rates(s2, s3, info["batches"]),
           "device_bytes": s3["device_bytes"], "host_bytes": s3["host_bytes"], "pin_ms": round(s3["pin_ms"], 1), "store_end": s3,
           "h2d_fetch_calls": h2d_rate(loop, n, slots) if slots else None}
    return loop, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preroll", type=int, default=250); ap.add_argument("--frames", type=int, default=1000); ap.add_argument("--stride", type=int, default=2)
    ap.add_argument("--reps", type=int, default=2); ap.add_argument("--K", type=int, default=30); ap.add_argument("--slots", default="64,256")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("frame_store_timing.py needs a CUDA device")
    dev = torch.device("cuda:0")
    n = a.preroll + a.frames
    depth, color = stream_bank(n, a.stride, dev)
    kinds = [0] + [int(x) for x in a.slots.split(",")]
    runs = {str(k): [] for k in kinds}
    for _ in range(a.reps):
        for k in kinds:
            loop, o = run(depth, color, a.preroll, n, a.K, k, dev)
            loop.close(); torch.cuda.synchronize(); torch.cuda.empty_cache()
            runs[str(k)].append(o)
            print(k, json.dumps(o), flush=True)
    out = {"card": card(), "frames": n, "preroll": a.preroll, "runs": runs,
           "fps_median": {k: float(np.median([r["fps"] for r in v])) for k, v in runs.items()},
           "finish_s_median": {k: float(np.median([r["finish_s"] for r in v])) for k, v in runs.items()},
           "fuse_s_median": {k: float(np.median([r["fuse_s"] for r in v])) for k, v in runs.items()}}
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

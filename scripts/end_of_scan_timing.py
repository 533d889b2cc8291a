"""CUDA-event timing of the end of a recording (FrameLoop.finish, bfFrameLoopFinish) on bench.py's stream configuration (development aid).

usage: end_of_scan_timing.py [--preroll 250] [--stride 2] [--K 30] [--out FILE]

The synthetic 640x480 stream of bench.py's loop workload (rich texture, 1 cm voxels, 4 M-block heap, 4 M buckets, two streams, look-ahead) is
stepped for `preroll` frames, then finished with s_numSolveFramesBeforeExit = K, twice on fresh loops over the same frames:
  pass 1, one turn per call with the stage profile on: each turn's time (events around the call) and its global-solve and re-integration stage
          times -- turns 0 .. K-1 are the sparse global solves, turn K the dense end solve, the rest the drain;
  pass 2, one call, profile off: the whole finish.
Prints one JSON line with the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bundlefusion_b200 import synth_gpu  # noqa: E402
from bundlefusion_b200.frame_loop import FrameLoop, default_params  # noqa: E402

W, H = 640, 480


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                  # the name from torch is still reported
        q = f"nvidia-smi unavailable: {e}"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.splitlines()[0] if q else ""}


def new_loop(n, dev):
    P = default_params(W, H)
    P.maxNumFrames = n + 8; P.maxNumImages = n // 10 + 8; P.maxGlobalResiduals = 25 * P.maxNumImages * 48          # bench.py run_loop's sizing
    P.hash.m_hashNumBuckets = 4_000_000; P.hash.m_numSDFBlocks = 4_000_000
    loop = FrameLoop(P, dev)
    loop.set_overlap(True)
    return loop


def preroll(loop, depth, color):
    n = depth.shape[0]
    for f in range(n):
        loop.step(depth[f], color[f], *((depth[f + 1], color[f + 1]) if f + 1 < n else (None, None)))
    torch.cuda.synchronize()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preroll", type=int, default=250); ap.add_argument("--stride", type=int, default=2); ap.add_argument("--K", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("end_of_scan_timing.py needs a CUDA device")
    dev = torch.device("cuda:0")
    n, K = a.preroll, a.K
    depth = torch.empty(n, H, W, dtype=torch.float32, device=dev); color = torch.empty(n, H, W, 4, dtype=torch.uint8, device=dev)
    for s0 in range(0, n, 64):
        idx = [a.stride * i for i in range(s0, min(n, s0 + 64))]
        d, c, _ = synth_gpu.make_frames(idx, W, H, device=str(dev), texture="rich")
        depth[s0:s0 + len(idx)] = d; color[s0:s0 + len(idx)] = c
    ev = lambda: torch.cuda.Event(enable_timing=True)

    # pass 1: one turn per call, stage profile on
    loop = new_loop(n, dev)
    preroll(loop, depth, color)
    keyframes = loop.counters()["keyframes"]
    turns = []
    info = {"done": False}
    while not info["done"] and len(turns) < K + 2 + (n + 9) // 10 + 50:
        loop.set_profiling(True)
        e0, e1 = ev(), ev()
        e0.record()
        info = loop.finish(K, max_turns=1)
        e1.record(); torch.cuda.synchronize()
        st = loop.stage_times()
        turns.append({"turn": info["frames_past_end"] - 1, "ms": e0.elapsed_time(e1), "solve_ms": st["global_solve_trajectory"],
                      "reint_ms": st["tsdf_reintegrate_integrate"], "reint": info["reintegrations"], "global_solves": info["global_solves"]})
    loop.set_profiling(False)
    final1 = info
    traj1 = loop.trajectory(n)
    loop.close(); del loop
    sparse = [t for t in turns if t["turn"] < K]
    dense = [t for t in turns if t["turn"] == K]
    drain = [t for t in turns if t["turn"] > K]

    # pass 2: the whole finish in one call
    loop = new_loop(n, dev)
    preroll(loop, depth, color)
    e0, e1 = ev(), ev()
    e0.record()
    info2 = loop.finish(K)
    e1.record(); torch.cuda.synchronize()
    finish_ms = e0.elapsed_time(e1)
    same = bool(np.array_equal(loop.trajectory(n), traj1, equal_nan=True))
    loop.close()

    r = 3
    out = {
        "card": card(), "frames": n, "stride": a.stride, "K": K, "keyframes_after_preroll": keyframes,
        "sparse_solves": {"turns": len(sparse), "ms_total": round(sum(t["ms"] for t in sparse), r), "solve_stage_ms_total": round(sum(t["solve_ms"] for t in sparse), r),
                          "solve_stage_ms_median": round(sorted(t["solve_ms"] for t in sparse)[len(sparse) // 2], r) if sparse else None},
        "dense_end_solve": {"turn": final1["dense_turn"], "N": final1["dense_keyframes"], "dense_pairs": final1["dense_pairs"],
                            "turn_ms": round(dense[0]["ms"], r) if dense else None, "solve_stage_ms": round(dense[0]["solve_ms"], r) if dense else None},
        "drain": {"turns": len(drain), "reintegrations": sum(t["reint"] for t in drain), "ms_total": round(sum(t["ms"] for t in drain), r),
                  "reint_stage_ms_total": round(sum(t["reint_ms"] for t in drain), r)},
        "finish_one_call": {"ms": round(finish_ms, r), "turns": info2["turns"], "frames_past_end": info2["frames_past_end"], "done": info2["done"],
                            "valid": info2["valid"], "dense_pairs": info2["dense_pairs"], "same_trajectory_as_pass_1": same},
        "pass_1_done": final1["done"], "per_turn": [{k: (round(v, r) if isinstance(v, float) else v) for k, v in t.items()} for t in turns],
    }
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()

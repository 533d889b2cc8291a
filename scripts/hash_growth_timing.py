"""Cost of growing the frame loop's voxel hash on bench.py's stream configuration (development aid).

usage: hash_growth_timing.py [--preroll 250] [--frames 1000] [--stride 2] [--reps 2] [--start 16384] [--out FILE]

The bench stream (preroll + frames at 1 cm, overlap and look-ahead on, then finish(30)) through two loops, alternated, `reps` times each:
  fixed:  4 M buckets / 4 M blocks, as bench.py sizes the table;
  grown:  --start blocks and 4 buckets per block, growth ceiling 4 M blocks (hashMaxSDFBlocks).
Per run: frames/s of the steps (wall clock, ending in a device synchronise), finish time, hash growth report, and the hash + heap bytes the
loop holds at the end.  Per growth during the steps (the step after which the loop's heap size changed): blocks before and after, the step's
wall time.  The grown loop starts with 4 buckets per block (the reference's default ratio) and keeps that ratio.
Rehash cost: the final grown model moved by bfTsdfRehash into a table of twice its heap, CUDA events around the call; algorithmic bytes = slot
table scan (16 B per slot up to the high-water mark, bounded here by the heap) + 2 x 6144 B per live block + 32 B per destination entry written,
against 3.35 TB/s.  Prints one JSON line with the card's name and power limit read in the same run."""
import argparse
import ctypes as C
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bundlefusion_b200 import _capi as capi  # noqa: E402
from bundlefusion_b200 import fuse  # noqa: E402
from bundlefusion_b200.frame_loop import FrameLoop, default_params  # noqa: E402
from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF  # noqa: E402
from trajectory_fusion_timing import W, H, card, stream_bank  # noqa: E402

HBM = 3.35e12
ENTRY, VOXEL_BLOCK = 32, 512 * 12


def table_bytes(hp):
    """the table's buckets (fuse.table_bytes), plus per heap block its heap word and voxel block"""
    return fuse.table_bytes(int(hp.m_hashNumBuckets)) + (4 + VOXEL_BLOCK) * int(hp.m_numSDFBlocks)


def hp_of(loop):
    return loop.lib.bfFrameLoopGetHashParams(loop._h).contents


def run(depth, color, n, K, start, dev):
    P = default_params(W, H)
    P.maxNumFrames = n + 8; P.maxNumImages = n // 10 + 8; P.maxGlobalResiduals = 25 * P.maxNumImages * 48          # bench.py run_loop's sizing
    P.hash.m_hashNumBuckets = 4_000_000; P.hash.m_numSDFBlocks = 4_000_000
    if start:
        P.hashMaxSDFBlocks = 4_000_000
        P.hash.m_hashNumBuckets = (4 * start) | 1             # the reference's 4 buckets per block (800 000 / 200 000)
        P.hash.m_numSDFBlocks = start
    loop = FrameLoop(P, dev)
    loop.set_overlap(True)
    growth_steps = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for f in range(n):
        b0, ts = hp_of(loop).m_numSDFBlocks, time.perf_counter()
        loop.step(depth[f], color[f], *((depth[f + 1], color[f + 1]) if f + 1 < n else (None, None)))
        if hp_of(loop).m_numSDFBlocks != b0:
            growth_steps.append({"frame": f, "blocks": [int(b0), int(hp_of(loop).m_numSDFBlocks)], "step_ms": round((time.perf_counter() - ts) * 1e3, 2)})
    loop.join(); torch.cuda.synchronize()
    steps_s = time.perf_counter() - t0
    t1 = time.perf_counter()
    loop.finish(K)
    loop.join(); torch.cuda.synchronize()
    g = loop.hash_growth()
    hp = loop.lib.bfFrameLoopGetHashParams(loop._h).contents
    out = {"fps": round(n / steps_s, 2), "steps_s": round(steps_s, 3), "finish_s": round(time.perf_counter() - t1, 3), "growth": g,
           "live_blocks": int(hp.m_numSDFBlocks) - loop.heap_free(), "table_bytes_end": table_bytes(hp), "growth_steps": growth_steps}
    return loop, out


def rehash_cost(loop, dev, reps=3):
    """the loop's model moved into a fresh table of twice its heap, the source untouched"""
    hd = loop.lib.bfFrameLoopGetHashData(loop._h).contents
    hp_src = loop.lib.bfFrameLoopGetHashParams(loop._h).contents
    live = int(hp_src.m_numSDFBlocks) - loop.heap_free()
    res = []
    for _ in range(reps):
        hp = capi.BFHashParams()
        C.memmove(C.byref(hp), C.byref(hp_src), C.sizeof(capi.BFHashParams))
        hp.m_numSDFBlocks = 2 * int(hp_src.m_numSDFBlocks); hp.m_hashNumBuckets = (2 * int(hp_src.m_hashNumBuckets)) | 1
        dst = CUDASceneRepHashSDF(hp, dev)
        torch.cuda.synchronize()
        lib = capi.lib()
        lib.bfSetStream(C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        o = (C.c_ulonglong * 2)()
        e0.record()
        capi.check(lib.bfTsdfRehash(C.byref(hd), C.byref(hp_src), C.byref(dst.m_hashData), C.byref(dst.m_hashParams), o), "bfTsdfRehash")
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        nbytes = 16 * int(hp_src.m_numSDFBlocks) + 2 * VOXEL_BLOCK * live + ENTRY * live
        res.append({"moved": int(o[0]), "refused": int(o[1]), "event_ms": round(ms, 3), "bytes": nbytes, "tb_s": round(nbytes / (ms * 1e-3) / 1e12, 3),
                    "share_of_3_35_tb_s": round(nbytes / (ms * 1e-3) / HBM, 4)})
        dst.close(); del dst
    return {"src_blocks": int(hp_src.m_numSDFBlocks), "src_buckets": int(hp_src.m_hashNumBuckets), "live": live, "runs": res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preroll", type=int, default=250); ap.add_argument("--frames", type=int, default=1000); ap.add_argument("--stride", type=int, default=2)
    ap.add_argument("--reps", type=int, default=2); ap.add_argument("--K", type=int, default=30); ap.add_argument("--start", type=int, default=16384)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("hash_growth_timing.py needs a CUDA device")
    dev = torch.device("cuda:0")
    n = a.preroll + a.frames
    depth, color = stream_bank(n, a.stride, dev)
    runs = {"fixed": [], "grown": []}
    rehash = None
    for _ in range(a.reps):
        for kind in ("fixed", "grown"):
            loop, o = run(depth, color, n, a.K, a.start if kind == "grown" else 0, dev)
            if kind == "grown" and rehash is None:
                rehash = rehash_cost(loop, dev)
            loop.close(); torch.cuda.synchronize(); torch.cuda.empty_cache()
            runs[kind].append(o)
            print(kind, json.dumps(o), flush=True)
    out = {"card": card(), "frames": n, "start_blocks": a.start, "runs": runs, "rehash_final_model": rehash,
           "fps_median": {k: float(np.median([r["fps"] for r in v])) for k, v in runs.items()}}
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

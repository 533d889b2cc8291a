"""Cost of meshing a model whole (CUDAMarchingCubesHashSDF.extractIsoSurfaceWhole) on bench.py's stream configuration (development aid).

usage: mesh_timing.py [--preroll 250] [--frames 1000] [--stride 2] [--reps 5] [--out FILE]

The loop runs and finishes as in scripts/hash_fit_timing.py (the same stream, hash and K = 30).  Two models are meshed: the loop's own model at
1 cm, and the loop's frames fused along the final trajectory at 4 mm into a hash sized by FrameLoop.fit_hash_params.  For each:
  blocks, triangles found (the count pass's total), chunks and the largest chunk;
  count:   bfMarchingCubesCount, CUDA events around the launch pair, median of `reps` after one warm-up;
  whole:   at buffers of 6 M and 1 M triangles, the parts of the whole-mesh call (the same greedy cut of the chunk counts), each part's
           bfMarchingCubesExtractRange and its device-to-host copy into pinned memory timed with CUDA events (summed over the parts), and
           the whole-mesh call itself, wall clock (count, parts, copies, host appends);
  save:    saveMesh of the whole soup (index buffer, mergeCloseVertices, removeDuplicateFaces, PLY to a temporary file), wall clock.
Prints one JSON line with the card's name and power limit read in the same run."""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bundlefusion_b200.frame_loop import FrameLoop, default_params  # noqa: E402
from bundlefusion_b200.marching_cubes import CUDAMarchingCubesHashSDF, marching_cubes_params  # noqa: E402
from bundlefusion_b200.scan import _LoopScene  # noqa: E402
from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF  # noqa: E402
from trajectory_fusion_timing import W, H, card, stream_bank  # noqa: E402


def parts_of(chunks, cap):
    """the whole-mesh call's cut: consecutive chunks, greedily, into parts of at most cap triangles; empty parts are not extracted"""
    out, begin, s = [], 0, 0
    for c, n in enumerate(list(chunks) + [None]):
        if n is not None and s + int(n) <= cap:
            s += int(n)
            continue
        if s:
            out.append((begin, c, s))
        begin, s = c, (int(n) if n is not None else 0)
    return out


def measure(scene, blocks, reps, dev):
    hp = scene.m_hashParams
    res = {"blocks": int(blocks), "buckets": int(hp.m_hashNumBuckets), "voxel_m": float(hp.m_virtualVoxelSize)}
    mc = CUDAMarchingCubesHashSDF(marching_cubes_params(int(hp.m_hashNumBuckets), float(hp.m_virtualVoxelSize), 1000), dev)
    L = mc.lib
    found, chunks = mc.count(scene)
    res.update(triangles_found=found, chunks=len(chunks), largest_chunk=int(chunks.max()))
    # the count pass
    d_counts = torch.empty(len(chunks), dtype=torch.int32, device=dev)
    d_total = torch.empty(1, dtype=torch.int64, device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    times = []
    mc._bind_stream()
    for _ in range(reps + 1):
        torch.cuda.synchronize(dev)
        ev[0].record()
        capi_rc = L.bfMarchingCubesCount(C.byref(scene.m_hashData), C.byref(hp), C.byref(mc.m_params), d_counts.data_ptr(), d_total.data_ptr())
        ev[1].record()
        torch.cuda.synchronize(dev)
        assert capi_rc == 0
        times.append(ev[0].elapsed_time(ev[1]))
    res["count_ms"] = round(float(np.median(times[1:])), 3)
    res["count_ms_all"] = [round(t, 3) for t in times[1:]]
    assert int(d_total.item()) == found
    mc.close()
    # whole extraction at two buffer sizes
    res["whole"] = {}
    for cap in (6_000_000, 1_000_000):
        parts = parts_of(chunks, max(cap, int(chunks.max())))
        tri = torch.empty((max(p[2] for p in parts) if parts else 1) * 18, dtype=torch.float32, device=dev)
        host = torch.empty(tri.numel(), dtype=torch.float32, pin_memory=True)
        cnt = torch.zeros(1, dtype=torch.int32, device=dev)
        mp = marching_cubes_params(int(hp.m_hashNumBuckets), float(hp.m_virtualVoxelSize), max(cap, int(chunks.max())))
        extract_ms, copy_ms, got = 0.0, 0.0, 0
        torch.cuda.synchronize(dev)
        mc2 = CUDAMarchingCubesHashSDF(mp, dev)
        mc2._bind_stream()
        for b, e, want in parts:
            ev[0].record()
            assert L.bfMarchingCubesExtractRange(C.byref(scene.m_hashData), C.byref(hp), C.byref(mp), b, e, tri.data_ptr(), cnt.data_ptr()) == 0
            ev[1].record()
            host[:want * 18].copy_(tri[:want * 18], non_blocking=True)
            ev[2].record()
            torch.cuda.synchronize(dev)
            extract_ms += ev[0].elapsed_time(ev[1]); copy_ms += ev[1].elapsed_time(ev[2]); got += int(cnt.item())
        del tri, host
        torch.cuda.synchronize(dev)
        t = time.perf_counter()
        info = mc2.extractIsoSurfaceWhole(scene)
        torch.cuda.synchronize(dev)
        wall = time.perf_counter() - t
        entry = {"parts": info["parts"], "largest_part": info["largest_part"], "buffer_enlarged": info["buffer_enlarged"], "host_syncs": info["host_syncs"],
                 "triangles_extracted": info["triangles_extracted"], "parts_device_ms": round(extract_ms, 3), "parts_copy_ms": round(copy_ms, 3),
                 "copy_GBps": round(72.0 * got / (copy_ms * 1e6), 2) if copy_ms else None, "whole_call_s": round(wall, 4)}
        assert got == found == info["triangles_extracted"], (got, found, info)
        if cap == 6_000_000:
            with tempfile.TemporaryDirectory() as d:
                t = time.perf_counter()
                mc2.saveMesh(os.path.join(d, "mesh.ply"), overwrite=True)
                entry["save_mesh_s"] = round(time.perf_counter() - t, 3)
                entry["ply_bytes"] = os.path.getsize(os.path.join(d, "mesh.ply"))
        res["whole"]["%dM" % (cap // 1_000_000)] = entry
        mc2.close()
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preroll", type=int, default=250); ap.add_argument("--frames", type=int, default=1000); ap.add_argument("--stride", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5); ap.add_argument("--K", type=int, default=30); ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("mesh_timing.py needs a CUDA device")
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
    models = {"1cm_loop": measure(_LoopScene(loop), int(P.hash.m_numSDFBlocks) - loop.heap_free(), a.reps, dev)}
    hp, fit = loop.fit_hash_params(0.004)
    scene = CUDASceneRepHashSDF(hp, dev)
    fused = loop.fuse(scene)
    models["4mm_fused"] = measure(scene, int(hp.m_numSDFBlocks) - scene.getHeapFreeCount(), a.reps, dev)
    models["4mm_fused"].update(inserts_dropped=fused["inserts_dropped"], fit_predicted_overflow=fit["predicted_overflow"])
    scene.close()
    out = {"card": card(), "frames": n, "preroll": a.preroll, "stride": a.stride, "finish_done": finish["done"], "models": models,
           "4mm_exceeds_6M": models["4mm_fused"]["triangles_found"] > 6_000_000}
    loop.close()
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()

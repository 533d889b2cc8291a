"""Cost of the device mesh path (CUDAMarchingCubesHashSDF.extractSoup + weld) against saveMesh's host clean-up, on the models of
scripts/mesh_timing.py (development aid).

usage: mesh_weld_timing.py [--preroll 250] [--frames 1000] [--stride 2] [--reps 3] [--check] [--out FILE]

The loop runs and finishes as in scripts/mesh_timing.py (bench.py's stream, K = 30).  Two models: the loop's own at 1 cm, and its frames fused
along the final trajectory at 4 mm into a hash sized by FrameLoop.fit_hash_params.  For each:
  count, soup, weld:  bfMarchingCubesCount, bfMarchingCubesExtractRange over every chunk, bfMeshWeld (its rounds and host synchronisations
                      included), each between CUDA events; median of `reps` after one warm-up;
  download + PLY:     Mesh.save_ply to a temporary file, wall clock;
  device path:        extractMesh + save_ply, wall clock;
  saveMesh:           the whole-mesh call, then saveMesh (index buffer, host clean-up, PLY), wall clock of saveMesh alone;
  device bytes:       soup + workspace + outputs, and torch's peak allocation over the device path.
--check compares the weld with bfMeshMergeCloseVertices + bfMeshRemoveDuplicateFaces on the same soup, and the two PLY files, byte for byte.
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

from bundlefusion_b200 import _capi as capi  # noqa: E402
from bundlefusion_b200 import marching_cubes as mcm  # noqa: E402
from bundlefusion_b200.frame_loop import FrameLoop, default_params  # noqa: E402
from bundlefusion_b200.marching_cubes import CUDAMarchingCubesHashSDF, marching_cubes_params, num_chunks  # noqa: E402
from bundlefusion_b200.scan import _LoopScene  # noqa: E402
from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF  # noqa: E402
from trajectory_fusion_timing import W, H, card, stream_bank  # noqa: E402


def measure(scene, reps, dev, check):
    hp = scene.m_hashParams
    res = {"buckets": int(hp.m_hashNumBuckets), "voxel_m": float(hp.m_virtualVoxelSize)}
    mc = CUDAMarchingCubesHashSDF(marching_cubes_params(int(hp.m_hashNumBuckets), float(hp.m_virtualVoxelSize), 6_000_000), dev)
    L = mc.lib
    T, _ = mc.count(scene)
    p = mc._box_params(scene, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), False)
    p.m_maxNumTriangles = T
    chunks = num_chunks(p.m_hashNumBuckets)
    d_counts = torch.empty(chunks, dtype=torch.int32, device=dev); d_total = torch.empty(1, dtype=torch.int64, device=dev)
    soup = torch.empty((T, 3, 6), dtype=torch.float32, device=dev); cnt = torch.empty(1, dtype=torch.int32, device=dev)
    ws_bytes = int(L.bfMeshWeldWorkspaceBytes(T))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    pos = torch.empty((3 * T, 3), dtype=torch.float32, device=dev); col = torch.empty((3 * T, 4), dtype=torch.float32, device=dev)
    faces = torch.empty((T, 3), dtype=torch.int32, device=dev)
    info = capi.BFMeshWeldInfo()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    times = {"count_ms": [], "soup_ms": [], "weld_ms": []}
    mc._bind_stream()
    for _ in range(reps + 1):
        torch.cuda.synchronize(dev)
        ev[0].record()
        assert L.bfMarchingCubesCount(C.byref(scene.m_hashData), C.byref(hp), C.byref(p), d_counts.data_ptr(), d_total.data_ptr()) == 0
        ev[1].record()
        assert L.bfMarchingCubesExtractRange(C.byref(scene.m_hashData), C.byref(hp), C.byref(p), 0, chunks, soup.data_ptr(), cnt.data_ptr()) == 0
        ev[2].record()
        capi.check(L.bfMeshWeld(soup.data_ptr(), T, 0.00001, ws.data_ptr(), ws_bytes, pos.data_ptr(), col.data_ptr(), faces.data_ptr(), C.byref(info)), "bfMeshWeld")
        ev[3].record()
        torch.cuda.synchronize(dev)
        for k, (a, b) in zip(times, ((0, 1), (1, 2), (2, 3))):
            times[k].append(ev[a].elapsed_time(ev[b]))
    assert int(d_total.item()) == int(cnt.item()) == T
    for k, v in times.items():
        res[k] = round(float(np.median(v[1:])), 3)
        res[k + "_all"] = [round(x, 3) for x in v[1:]]
    res["weld"] = mcm._weld_report(info)
    res["device_bytes"] = {"soup": T * 72, "workspace": ws_bytes, "outputs": 3 * T * 28 + T * 12}
    res["device_bytes"]["total"] = sum(res["device_bytes"].values())
    if check:                                                                          # the last timed weld against the host clean-up of the same soup
        V, F = int(info.verticesOut), int(info.facesOut)
        tri = soup.cpu().numpy()
        hpos = np.ascontiguousarray(tri[..., :3].reshape(-1, 3))
        hcol = np.concatenate([tri[..., 3:].reshape(-1, 3), np.ones((len(hpos), 1), np.float32)], axis=1)
        wp, wc, wf = mcm.merge_close_vertices(hpos, hcol, np.arange(len(hpos), dtype=np.uint32).reshape(-1, 3), 0.00001)
        wf = mcm.remove_duplicate_faces(wf)
        gp, gc, gf = pos[:V].cpu().numpy(), col[:V].cpu().numpy(), faces[:F].cpu().numpy().view(np.uint32)
        same = gp.shape == wp.shape and gf.shape == wf.shape and np.array_equal(gp.view(np.uint32), wp.view(np.uint32)) and \
            np.array_equal(gc.view(np.uint32), wc.view(np.uint32)) and np.array_equal(gf, wf)
        with tempfile.TemporaryDirectory() as d:
            mcm.save_ply(os.path.join(d, "host.ply"), wp, wc, wf)
            mcm.save_ply(os.path.join(d, "device.ply"), gp, gc, gf)
            res["check"] = {"arrays_equal": bool(same),
                            "ply_equal": open(os.path.join(d, "host.ply"), "rb").read() == open(os.path.join(d, "device.ply"), "rb").read()}
    del soup, ws, pos, col, faces
    torch.cuda.empty_cache()
    with tempfile.TemporaryDirectory() as d:
        # the device path end to end, and its download + PLY alone
        torch.cuda.synchronize(dev)
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        t = time.perf_counter()
        mesh = mc.extractMesh(scene)
        t1 = time.perf_counter()
        mesh.save_ply(os.path.join(d, "device.ply"))
        t2 = time.perf_counter()
        res.update(device_path_s=round(t2 - t, 4), download_ply_s=round(t2 - t1, 4), torch_peak_bytes=int(torch.cuda.max_memory_allocated(dev) - base),
                   ply_bytes=os.path.getsize(os.path.join(d, "device.ply")))
        # saveMesh on the same model
        whole = mc.extractIsoSurfaceWhole(scene)
        assert whole["triangles_extracted"] == T
        t = time.perf_counter()
        mc.saveMesh(os.path.join(d, "host.ply"), overwrite=True)
        res["save_mesh_s"] = round(time.perf_counter() - t, 3)
    del mesh
    mc.close()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preroll", type=int, default=250); ap.add_argument("--frames", type=int, default=1000); ap.add_argument("--stride", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3); ap.add_argument("--K", type=int, default=30); ap.add_argument("--check", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("mesh_weld_timing.py needs a CUDA device")
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
    loop.finish(a.K)
    loop.join(); torch.cuda.synchronize()
    del depth, color
    torch.cuda.empty_cache()
    models = {"1cm_loop": measure(_LoopScene(loop), a.reps, dev, a.check)}
    hp, _ = loop.fit_hash_params(0.004)
    scene = CUDASceneRepHashSDF(hp, dev)
    loop.fuse(scene)
    models["4mm_fused"] = measure(scene, a.reps, dev, a.check)
    scene.close()
    loop.close()
    line = json.dumps({"card": card(), "frames": n, "preroll": a.preroll, "stride": a.stride, "models": models})
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()

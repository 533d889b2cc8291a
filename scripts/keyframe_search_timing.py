"""Times the all-pairs keyframe search (bfKeyframeSearch, search_sharded) on configs[4] of BASELINE.json: N frames of the synthetic Lissajous
stream (synth_gpu) at 640x480 and 1280x960, each detected with bfSiftDetect (no feature-count limit, up to 1024 keys) and cached with
bfCacheStoreFrame.  Every rank builds the same set; a hash all-reduce confirms it.  One JSON line per (size, world) from rank 0.

    torchrun --nproc_per_node G scripts/keyframe_search_timing.py [--frames 2000] [--sizes 640x480,1280x960] [--check] [--compare]

--check: every rank's gathered list must equal the single-GPU search byte for byte (exit code 1 otherwise).
--compare (world 1): the same pairs through the per-image path -- bfSiftMatchBatch over 0..j-1 plus the per-image filter chain -- timed beside it."""
import argparse
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bundlefusion_b200 import _capi as capi                      # noqa: E402
from bundlefusion_b200 import keyframe_search as ks              # noqa: E402
from bundlefusion_b200 import synth_gpu                          # noqa: E402

DATASHEET_INT8_TOPS = 1979.0          # H100 SXM, dense, 700 W card (data-sheet figure, not a measurement)


def build_set(N, W, H, dev):
    import torch
    L = capi.lib()
    MK, CW, CH = 1024, 80, 60
    fx = 525.0 * W / 640.0
    K = np.eye(4, dtype=np.float32); K[0, 0] = K[1, 1] = fx; K[0, 2] = (W - 1) / 2.0; K[1, 2] = (H - 1) / 2.0
    Kc = K.copy(); Kc[0, 0] *= CW / W; Kc[1, 1] *= CH / H; Kc[0, 2] *= (CW - 1) / (W - 1); Kc[1, 2] *= (CH - 1) / (H - 1)
    Kinv = np.linalg.inv(K.astype(np.float64)).astype(np.float32)
    keys = torch.zeros((N, MK, 4), dtype=torch.float32, device=dev); des = torch.zeros((N, MK, 128), dtype=torch.uint8, device=dev)
    nk = torch.zeros(N, dtype=torch.int32, device=dev)
    P = capi.BFSiftDetectParams(W, H, W, H, 0.1, 4.0, 3.0, 0, MK)
    cp = capi.BFCacheParams()
    cp.inputDepthWidth, cp.inputDepthHeight, cp.inputColorWidth, cp.inputColorHeight, cp.width, cp.height = W, H, W, H, CW, CH
    for k, v in enumerate(np.linalg.inv(K.astype(np.float64)).astype(np.float32).reshape(-1)):
        cp.inputIntrinsicsInv[k] = float(v)
    cp.filterIntensitySigma, cp.filterDepthSigmaD, cp.filterDepthSigmaR = 2.5, 1.0, 0.05
    n = CW * CH
    planes = [torch.zeros((N, n * w), dtype=torch.float32, device=dev) for w in (1, 4, 1, 2)] + [torch.zeros((N, n * 4), dtype=torch.uint8, device=dev),
                                                                                            torch.zeros((N, n * 4), dtype=torch.float32, device=dev)]
    recs = (capi.BFCUDACachedFrame * N)()
    L.bfSetStream(C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    for i in range(N):
        d, c, _ = synth_gpu.make_frames([i], W, H, n_total=N, device=dev, texture="rich")
        d, c = d[0].contiguous(), c[0].contiguous()
        inten = ((0.299 * c[..., 0].float() + 0.587 * c[..., 1].float() + 0.114 * c[..., 2].float()) / 255.0).contiguous()
        capi.check(L.bfSiftDetect(C.byref(P), inten.data_ptr(), d.data_ptr(), keys[i].data_ptr(), des[i].data_ptr(), nk[i:].data_ptr(), None), "bfSiftDetect")
        r = recs[i]
        r.d_depthDownsampled, r.d_cameraposDownsampled, r.d_intensityDownsampled = planes[0][i].data_ptr(), planes[1][i].data_ptr(), planes[2][i].data_ptr()
        r.d_intensityDerivsDownsampled, r.d_normalsDownsampledUCHAR4, r.d_normalsDownsampled = planes[3][i].data_ptr(), planes[4][i].data_ptr(), planes[5][i].data_ptr()
        capi.check(L.bfCacheStoreFrame(C.byref(cp), d.data_ptr(), c.data_ptr(), C.byref(r)), "bfCacheStoreFrame")
    torch.cuda.synchronize()
    rec_t = torch.from_numpy(np.frombuffer(bytes(recs), np.uint8).copy()).to(dev)
    return ks.KeyframeSet(keys, des, nk, rec_t, CW, CH, Kc, Kinv, owner=planes)


def set_hash(kf):
    h = hashlib.sha256()
    nk = kf.num_keys.cpu().numpy()
    h.update(nk.tobytes())
    for i in range(kf.num_images):
        h.update(kf.descriptors[i, :nk[i]].cpu().numpy().tobytes()); h.update(kf.keys[i, :nk[i]].cpu().numpy().tobytes())
    return int.from_bytes(h.digest()[:7], "little")


def events_ms(fn, reps):
    import torch
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def per_image_path(kf, params):
    """today's path: bfSiftMatchBatch over 0..j-1 (one legal batch per j) and the per-image filter chain, per image j"""
    import torch
    L = capi.lib()
    dev = kf.device
    N, MK = kf.descriptors.shape[:2]
    nk = kf.num_keys.cpu().numpy()
    s = kf.struct
    Ki, Kc = (C.c_float * 16)(*s.siftIntrinsicsInv), (C.c_float * 16)(*s.cacheIntrinsics)
    nm = torch.zeros(N, dtype=torch.int32, device=dev); dd = torch.zeros((N, 128), device=dev); ix = torch.zeros((N, 128, 2), dtype=torch.int32, device=dev)
    nf = torch.zeros(N, dtype=torch.int32, device=dev); fd = torch.zeros((N, 25), device=dev); fi = torch.zeros((N, 25, 2), dtype=torch.int32, device=dev)
    T = torch.zeros((N, 16), device=dev); Ti = torch.zeros((N, 16), device=dev)
    cap = 1 << 22
    glob = torch.zeros((cap, 32), dtype=torch.uint8, device=dev); gidx = torch.zeros((cap, 2), dtype=torch.int32, device=dev); gnum = torch.zeros(1, dtype=torch.int32, device=dev)
    base, kp = kf.descriptors.data_ptr(), kf.keys.data_ptr()
    jobs_all = [(capi.BFSiftMatchJob * max(j, 1))() for j in range(N)]
    for j in range(1, N):
        for i in range(j):
            jb = jobs_all[j][i]
            jb.d_des1, jb.num1, jb.d_des2, jb.num2 = base + i * MK * 128, int(nk[i]), base + j * MK * 128, int(nk[j])
            jb.out.d_numMatches, jb.out.d_distances, jb.out.d_keyPointIndices = nm.data_ptr() + 4 * i, dd.data_ptr() + 512 * i, ix.data_ptr() + 1024 * i
            jb.keyPointOffset[0], jb.keyPointOffset[1] = i * MK, j * MK

    def run():
        gnum.zero_()
        for j in range(1, N):
            capi.check(L.bfSiftMatchBatch(jobs_all[j], j, C.c_float(params.siftMatchThresh), C.c_float(params.siftMatchRatioMax)), "bfSiftMatchBatch")
            L.bfSiftSortKeyPointMatches(j, 0, j + 1, nm.data_ptr(), dd.data_ptr(), ix.data_ptr())
            L.bfSiftFilterKeyPointMatches(j, 0, j + 1, kp, nm.data_ptr(), dd.data_ptr(), ix.data_ptr(), nf.data_ptr(), fd.data_ptr(), fi.data_ptr(), T.data_ptr(),
                                          Ti.data_ptr(), Ki, params.minNumMatches, C.c_float(params.maxKabschResidual2))
            L.bfSiftFilterMatchesBySurfaceArea(j, 0, j + 1, kp, nf.data_ptr(), fi.data_ptr(), Ki, C.c_float(params.surfAreaPcaThresh), None)
            L.bfSiftFilterMatchesByDenseVerify(j, 0, j + 1, s.cacheWidth, s.cacheHeight, Kc, nf.data_ptr(), T.data_ptr(), s.d_cacheFrames, params.projCorrDistThres,
                                               params.projCorrNormalThres, params.projCorrColorThresh, params.verifySiftErrThresh, params.verifySiftCorrThresh,
                                               params.sensorDepthMin, params.sensorDepthMax, None)
            L.bfSiftAddCurrToResiduals(j, 0, j + 1, glob.data_ptr(), gidx.data_ptr(), gnum.data_ptr(), nf.data_ptr(), fi.data_ptr(), kp, Ki)
    return run, gnum, glob


def main():
    import torch
    import torch.distributed as dist
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--sizes", default="640x480,1280x960")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--compare", action="store_true")
    a = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1")); rank = int(os.environ.get("RANK", "0")); local = int(os.environ.get("LOCAL_RANK", "0"))
    dev = torch.device(f"cuda:{local}")
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    else:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1"); os.environ.setdefault("MASTER_PORT", "29533")
        dist.init_process_group("gloo", rank=0, world_size=1)
    ok = True
    try:
        import subprocess
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
        gpu = q[local] if local < len(q) else (q[0] if q else torch.cuda.get_device_name(dev))
        params = ks.search_params()
        for size in a.sizes.split(","):
            W, H = (int(x) for x in size.split("x"))
            kf = build_set(a.frames, W, H, dev)
            h = set_hash(kf)
            hs = torch.tensor([h, -h], dtype=torch.int64, device=dev if world > 1 else "cpu")
            dist.all_reduce(hs, op=dist.ReduceOp.MAX)
            assert int(hs[0]) == h and int(hs[1]) == -h, "ranks built different keyframe sets"
            nk = kf.num_keys.cpu().numpy().astype(np.int64)
            N = a.frames
            pairs = ks.num_pairs(N)
            ops = 128 * (int(nk.sum()) ** 2 - int((nk * nk).sum()))          # 2 * 128 * sum_{i<j} n_i n_j: each product counted once
            ks.reserve_workspace(N, 1024)
            ranges = ks.pair_ranges(nk, world)
            mine = ranges[rank]
            res = ks.search(kf, params, mine)                                  # warm-up, sizes the list
            cap = max(res["count"], 1)
            search_ms = events_ms(lambda: ks.search(kf, params, mine, capacity=cap, info=False), a.repeats)
            gather_ms = events_ms(lambda: ks.search_sharded(kf, params, search_fn=lambda k, p, r: res) if world > 1 else None, a.repeats)
            full = ks.search_sharded(kf, params) if world > 1 else {"entries": res["entries"], "key_indices": res["key_indices"], "count": res["count"]}
            t = torch.tensor([search_ms, gather_ms], dtype=torch.float64, device=dev if world > 1 else "cpu")
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            line = {"config": "configs[4] keyframe all-pairs search", "size": [W, H], "world": world, "gpu": gpu, "keyframes": N,
                    "keys_mean": float(nk.mean()), "keys_min": int(nk.min()), "keys_max": int(nk.max()), "pairs": pairs, "int8_ops_algorithmic": ops,
                    "entries": full["count"], "info_rank0": res["info"], "search_ms_max_over_ranks": round(float(t[0]), 3),
                    "gather_ms_max_over_ranks": round(float(t[1]), 3) if world > 1 else None,
                    "sweep_filters_emission_split": "not measured (one call)",
                    "achieved_tops_int8": round(ops / (float(t[0]) * 1e-3) / 1e12, 2) if ops else None,
                    "datasheet_int8_tops": DATASHEET_INT8_TOPS, "repeats_median_of": a.repeats}
            if a.check or a.compare:
                one = ks.search(kf, params) if world > 1 else res
                same = (full["count"] == one["count"] and torch.equal(full["entries"].cpu(), one["entries"].cpu())
                        and torch.equal(full["key_indices"].cpu(), one["key_indices"].cpu()))
                line["gathered_equals_single_gpu"] = bool(same)
                ok &= same
            if a.compare and world == 1:
                run, gnum, glob = per_image_path(kf, params)
                run()
                per_ms = events_ms(run, 1)
                n = int(gnum.item())
                line["per_image_path_ms"] = round(per_ms, 3)
                line["per_image_path_equal"] = bool(n == res["count"] and torch.equal(glob[:n].cpu(), res["entries"].cpu()))
                ok &= line["per_image_path_equal"]
            if rank == 0:
                print(json.dumps(line), flush=True)
            del kf
            torch.cuda.empty_cache()
    finally:
        dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()

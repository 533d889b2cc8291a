"""The frame store with device slots over a pinned host store (BFFrameLoopParams.deviceFrameSlots), on the GPU, against the resident store
(deviceFrameSlots = 0) on the 43-frame stream of test_frame_loop_model_gpu.py with look-ahead, overlap and the op log on: statuses, trajectory,
op log, model, finish info and host synchronisations bit for bit at N = 16 (the minimum) and N = 24, with frames evicted and fetched back;
fuse() at 1 cm and 4 mm from N = 16 (fetch and integrate alternate) and N = 32 (the next batch is fetched while one integrates); the bytes of
every frame through FetchFrames / GetFrame and the fit_hash_params report; the refusals; the device bytes; scan.py --device-frames."""
import ctypes as C
import json

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from bundlefusion_b200 import fuse
from bundlefusion_b200.frame_loop import FrameLoop
from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF
from oracle import oracle as orc
from tests.test_frame_loop_model_gpu import W, H, loop_model, loop_params, stream
from tests.test_trajectory_fusion_gpu import recording  # noqa: F401  (a fixture)

pytestmark = pytest.mark.gpu
N_LOOP, K_FINISH = 43, 30
SLOTS = (16, 24, 32)


def _params(slots):
    p = loop_params(N_LOOP)
    p.deviceFrameSlots = slots
    return p


def _run(slots, dev):
    """the stream with look-ahead and overlap on, then finish(30); the loop stays open for the fusion and frame-access tests"""
    loop = FrameLoop(_params(slots), dev)
    loop.set_op_log(True)
    loop.set_overlap(True)
    frames = stream(N_LOOP, dev)
    status = []
    for i, (d, c) in enumerate(frames):
        nxt = frames[i + 1] if i + 1 < N_LOOP else (None, None)
        status.append(loop.step(d, c, *nxt).as_dict())
    loop.join()
    r = {"loop": loop, "status": status, "traj": loop.trajectory(N_LOOP), "model": loop_model(loop, dev)[0], "syncs": loop.counters()["host_syncs"],
         "store": loop.frame_store()}
    r["finish"] = loop.finish(K_FINISH)
    loop.join()
    r.update({"traj_end": loop.trajectory(N_LOOP), "model_end": loop_model(loop, dev)[0], "syncs_end": loop.counters()["host_syncs"],
              "log": loop.op_log(), "store_end": loop.frame_store()})
    return r


@pytest.fixture(scope="module")
def runs(cuda_device):
    out = {0: _run(0, cuda_device)}
    for n in SLOTS:
        out[n] = _run(n, cuda_device)
        print("N = %d: %s" % (n, out[n]["store_end"]))
    yield out
    for r in out.values():
        r["loop"].close()


def _same_model(a, b, what):
    (ba, va), (bb, vb) = a, b
    assert ba.shape == bb.shape and np.array_equal(ba, bb), (what, "block set", len(ba), len(bb))
    assert np.array_equal(va, vb), (what, "voxel words differ in %d voxels" % int((va != vb).any(-1).sum()))


@pytest.mark.parametrize("slots", [16, 24])
def test_slot_loop_equals_resident_loop(runs, slots):
    res, got = runs[0], runs[slots]
    for a, b in zip(res["status"], got["status"]):
        assert a.keys() == b.keys() and all((a[k].tobytes() == b[k].tobytes()) if k == "transform" else a[k] == b[k] for k in a), (a, b)
    assert len(res["status"]) == len(got["status"]) == N_LOOP
    assert res["traj"].tobytes() == got["traj"].tobytes() and res["traj_end"].tobytes() == got["traj_end"].tobytes()
    assert all(x.tobytes() == y.tobytes() for x, y in zip(res["log"], got["log"])) and len(res["log"][0]) == len(got["log"][0])
    assert res["finish"] == got["finish"]
    _same_model(got["model"], res["model"], "N = %d after the steps" % slots)
    _same_model(got["model_end"], res["model_end"], "N = %d after finish(%d)" % (slots, K_FINISH))
    assert got["syncs"] == res["syncs"] and got["syncs_end"] == res["syncs_end"]
    # the slots were exercised: more frames than slots, every frame written back, frames evicted and fetched back for the ops that read them
    s = got["store_end"]
    assert N_LOOP > slots and s["slots"] == slots and s["host_store"]
    assert s["write_backs"] == N_LOOP and s["evictions"] > 0 and s["fetches"] > 0 and s["hits"] > 0
    assert s["h2d_bytes"] == s["fetches"] * W * H * 8 and s["d2h_bytes"] == N_LOOP * W * H * 8
    r = runs[0]["store_end"]
    assert not r["host_store"] and r["fetches"] == r["evictions"] == r["write_backs"] == 0 and r["host_bytes"] == 0


def _fuse(r, voxel, dev):
    hp = fuse.fine_hash_params(r["loop"].params, voxel)
    scene = CUDASceneRepHashSDF(hp, dev)
    info = r["loop"].fuse(scene)
    model = orc.canonical_blocks(scene.download())
    scene.close()
    return info, model


@pytest.mark.parametrize("voxel", [0.01, 0.004])
def test_fuse_from_slots_equals_resident(runs, cuda_device, voxel):
    ref_info, ref_model = _fuse(runs[0], voxel, cuda_device)
    assert ref_info["inserts_dropped"] == 0 and ref_info["batches"] >= 3
    for n in (16, 32):
        before = runs[n]["loop"].frame_store()
        info, model = _fuse(runs[n], voxel, cuda_device)
        assert info == ref_info, (n, info, ref_info)
        _same_model(model, ref_model, "fuse at %g m from N = %d" % (voxel, n))
        assert runs[n]["loop"].frame_store()["fetches"] > before["fetches"]


def test_frame_access_equals_resident(runs, cuda_device):
    import torch
    res = runs[0]["loop"]
    want = [tuple(t.clone() for t in res.frame(f)) for f in range(N_LOOP)]
    for n in (16, 24):
        loop = runs[n]["loop"]
        for f in range(N_LOOP):                                     # GetFrame: one frame per call, frames far apart evict each other
            d, c = loop.frame(f)
            assert torch.equal(d, want[f][0]) and torch.equal(c, want[f][1]), (n, f)
        g = n - 2
        for s in range(0, N_LOOP, g):                               # FetchFrames: groups of slots - 2
            frames = list(range(N_LOOP - 1 - s, max(-1, N_LOOP - 1 - s - g), -1))
            dp, cp = loop.fetch_frames(frames)
            for f, dd, cc in zip(frames, dp, cp):
                d, c = loop._views(dd, cc)
                assert torch.equal(d, want[f][0]) and torch.equal(c, want[f][1]), (n, f)
    for voxel in (0.01, 0.004):
        ref = res.fit_hash_params(voxel)[1]
        for n in (16, 24):
            assert runs[n]["loop"].fit_hash_params(voxel)[1] == ref, (n, voxel)


def test_refusals(runs, cuda_device):
    p = _params(0)
    lo = max(int(p.maxFrameFixes) + 2, 16)
    lib = capi.lib()
    for n in (1, lo - 1):
        p.deviceFrameSlots = n
        with pytest.raises(RuntimeError, match="error 1"):
            FrameLoop(p, cuda_device)
    p.maxFrameFixes = 20
    p.deviceFrameSlots = 21
    with pytest.raises(RuntimeError, match="error 1"):
        FrameLoop(p, cuda_device)
    p.deviceFrameSlots = 22
    FrameLoop(p, cuda_device).close()
    loop = runs[16]["loop"]
    before = loop.frame_store()
    frames = (C.c_uint32 * 15)(*range(15))
    d, c = (C.c_void_p * 15)(), (C.c_void_p * 15)()
    assert lib.bfFrameLoopFetchFrames(loop._h, frames, 15, d, c) == 1
    assert lib.bfGetLastErrorString().decode().startswith("bfFrameLoopFetchFrames: more than deviceFrameSlots - 2 frames")
    frames[0] = N_LOOP
    assert lib.bfFrameLoopFetchFrames(loop._h, frames, 14, d, c) == 1
    assert loop.frame_store() == before, "a refused fetch changed the store"
    assert all(x is None for x in d)


def test_device_bytes(runs, cuda_device):
    import torch
    for n in (0,) + SLOTS:
        s = runs[n]["store_end"]
        slots = n if n else N_LOOP + 16
        assert s["slots"] == slots and s["device_bytes"] == slots * W * H * 8
        assert s["host_bytes"] == (0 if n == 0 else (N_LOOP + 16) * W * H * 8)
    # the allocation itself, at a frame count where the store dominates: 2000 frames of 320 x 240 = 1.23 GB resident, 16 slots = 9.8 MB

    def used(p):
        torch.cuda.synchronize(cuda_device)
        free0 = torch.cuda.mem_get_info(cuda_device)[0]
        loop = FrameLoop(p, cuda_device)
        torch.cuda.synchronize(cuda_device)
        free1 = torch.cuda.mem_get_info(cuda_device)[0]
        loop.close()
        return free0 - free1
    p = loop_params(N_LOOP)
    p.maxNumFrames = 2000
    resident = used(p)
    p.deviceFrameSlots = 16
    slots = used(p)
    saved = (2000 - 16) * W * H * 8
    assert resident - slots > 0.9 * saved, (resident, slots, saved)


def test_scan_device_frames(cuda_device, recording, tmp_path, capsys):  # noqa: F811
    from bundlefusion_b200 import scan
    path, _ = recording
    dev = str(cuda_device)
    traj = {}
    for tag, extra in (("resident", []), ("slots", ["--device-frames", "16"])):
        assert scan.main([path, str(tmp_path / (tag + ".ply")), "--solve-frames-before-exit", "3", "--trajectory", str(tmp_path / (tag + ".txt")),
                          "--device", dev] + extra) == 0
        traj[tag] = (json.loads(capsys.readouterr().out.strip().splitlines()[-1]), np.loadtxt(tmp_path / (tag + ".txt")))
    (a, ta), (b, tb) = traj["resident"], traj["slots"]
    assert "frame_store" not in a and b["frame_store"]["slots"] == 16 and b["frame_store"]["host_store"]
    assert b["triangles"] == a["triangles"] > 0 and b["finish"] == a["finish"]
    assert ta.tobytes() == tb.tobytes()

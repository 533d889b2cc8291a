"""The frame loop as ONE call per frame (bfFrameLoopStep: ingest -> SIFT detect -> cache -> match + filters -> SIFT pose -> re-integration ->
integration -> local BA (+ verification) -> fuse to keyframe -> global match -> global BA -> trajectory update), on a synthetic stream with a
world-anchored texture and known camera poses.  This is an end-to-end behaviour test: there is no oracle of the whole loop (the reference
has no CPU path for it), every stage has its own parity test; here the loop must track, solve, and keep its trajectory near the truth."""
import numpy as np
import pytest

from bundlefusion_b200 import synth
from bundlefusion_b200.frame_loop import FrameLoop, default_params

pytestmark = pytest.mark.gpu
W, H = 320, 240


def rel_pose(T0, T):
    return np.linalg.inv(T0.astype(np.float64)) @ T.astype(np.float64)


def canonical_model(loop, dev):
    """the loop's fused model as oracle.canonical_blocks keys it: block positions and their raw sdf / weight / colour words"""
    import torch
    from oracle import oracle as orc
    hd = loop.lib.bfFrameLoopGetHashData(loop._h).contents
    hp = loop.lib.bfFrameLoopGetHashParams(loop._h).contents
    torch.cuda.synchronize(dev)

    def host(ptr, nbytes):
        class _View:
            pass
        v = _View()
        v.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False), "version": 3, "strides": None}
        return torch.as_tensor(v, device=dev).cpu().numpy().view(np.int32)
    n_entries = int(hp.m_hashNumBuckets) * 4
    return orc.canonical_blocks({"hash": host(hd.d_hash, n_entries * 32).reshape(n_entries, 8),
                                 "voxels": host(hd.d_SDFBlocks, int(hp.m_numSDFBlocks) * 512 * 12).reshape(-1, 512, 3)})


def test_frame_loop_tracks_solves_and_reintegrates(cuda_device):
    import torch
    p = default_params(W, H)
    p.maxNumImages = 16; p.maxNumFrames = 64
    p.hash.m_hashNumBuckets = 100003; p.hash.m_numSDFBlocks = 90000
    n_frames = 43                                         # 4 full chunks + a partial one
    frames = [synth.make_frame(2 * i, W, H, texture="rich") for i in range(n_frames)]
    loop = FrameLoop(p, cuda_device)
    free0 = loop.heap_free()
    stats = []
    for d, c, T in frames:
        st = loop.step(torch.from_numpy(d).to(cuda_device), torch.from_numpy(c).to(cuda_device))
        stats.append(st.as_dict())
    # every frame found features and (after the first) matched an earlier frame of its chunk; every frame was integrated
    assert all(s["numKeyPoints"] > 60 for s in stats)
    assert all(s["validTransform"] == 1 for s in stats), [s["frame"] for s in stats if not s["validTransform"]]
    assert all(s["lastMatchedFrame"] >= 0 for s in stats if s["frame"] > 0)
    # SIFT poses (what the frame was integrated with) stay within a few cm of the truth over the whole stream
    for s, (d, c, T) in zip(stats, frames):
        want = rel_pose(frames[0][2], T)
        assert np.abs(s["transform"] - want)[:3, 3].max() < 0.08 and np.abs(s["transform"] - want)[:3, :3].max() < 0.05, (s["frame"], s["transform"], want)
    # chunks were solved and accepted, keyframes accumulated, global solves ran
    solved = [s for s in stats if s["localSolved"] >= 0]
    assert len(solved) == 4 and all(s["localValid"] == 1 for s in solved), [(s["frame"], s["localSolved"], s["localValid"]) for s in solved]
    assert stats[-1]["numKeyframes"] == 4 and stats[-1]["numGlobalCorrespondences"] > 20
    assert sum(s["globalSolved"] for s in stats) >= 3
    c = loop.counters()
    assert c["frames"] == n_frames and c["integrations"] == n_frames and c["local_solves"] == 4 and c["global_solves"] >= 3
    assert c["reintegrations"] > 0, "pose updates from the solves must trigger re-integration"
    assert loop.heap_free() < free0
    # drain: the partial last chunk gets solved, re-integration runs out of work
    for _ in range(12):
        st = loop.step_past_end().as_dict()
    traj = loop.trajectory(n_frames)
    assert len(traj) >= 40
    err = []
    for f in range(len(traj)):
        if np.isfinite(traj[f]).all():
            want = rel_pose(frames[0][2], frames[f][2])
            err.append(np.abs(traj[f] - want)[:3, 3].max())
    assert len(err) >= 38 and max(err) < 0.05, (len(err), max(err))
    print("frame loop: max translation error of the optimised trajectory %.4f m over %d frames; counters %s" % (max(err), len(err), loop.counters()))
    loop.close()


def test_frame_loop_loses_and_flags_a_frame_without_texture(cuda_device):
    """a frame with nothing to match (uniform colour) gets no SIFT pose: it is not integrated and the loop reports it"""
    import torch
    p = default_params(W, H)
    p.maxNumImages = 8; p.maxNumFrames = 32
    p.hash.m_hashNumBuckets = 50021; p.hash.m_numSDFBlocks = 40000
    loop = FrameLoop(p, cuda_device)
    for i in range(4):
        d, c, T = synth.make_frame(2 * i, W, H, texture="rich")
        if i == 2:
            c = np.full_like(c, 128); c[..., 3] = 255
        st = loop.step(torch.from_numpy(d).to(cuda_device), torch.from_numpy(c).to(cuda_device)).as_dict()
        if i == 2:
            assert st["validTransform"] == 0 and st["numKeyPoints"] == 0 and np.isneginf(st["transform"]).all()
        else:
            assert st["validTransform"] == 1
    assert loop.counters()["integrations"] == 3
    loop.close()


def test_two_stream_loop_equals_single_stream(cuda_device):
    """bfFrameLoopSetOverlap: the reconstruction work on the loop's second stream changes when kernels run, not what they compute -- statuses,
    trajectory and the fused model (canonical voxel words) are those of the single-stream loop."""
    import torch
    from bundlefusion_b200 import _capi as capi
    from oracle import oracle as orc
    frames = [synth.make_frame(2 * i, W, H, texture="rich") for i in range(25)]
    out = []
    for overlap in (False, True):
        p = default_params(W, H)
        p.maxNumImages = 8; p.maxNumFrames = 40
        p.hash.m_hashNumBuckets = 100003; p.hash.m_numSDFBlocks = 90000
        loop = FrameLoop(p, cuda_device)
        loop.set_overlap(overlap)
        sts = [loop.step(torch.from_numpy(d).to(cuda_device), torch.from_numpy(c).to(cuda_device)).as_dict() for d, c, T in frames]
        loop.join()
        torch.cuda.synchronize()
        traj = loop.trajectory(25)
        free = loop.heap_free()
        out.append((sts, traj, free, loop.counters(), canonical_model(loop, cuda_device)))
        loop.close()
    (s0, t0, f0, c0, m0), (s1, t1, f1, c1, m1) = out
    assert f0 == f1 and c0["reintegrations"] == c1["reintegrations"] > 0 and c0["integrations"] == c1["integrations"]
    assert np.array_equal(m0[0], m1[0]) and np.array_equal(m0[1], m1[1]), "the two-stream loop fused another model"
    for a, b in zip(s0, s1):
        assert a["validTransform"] == b["validTransform"] and a["numReintegrated"] == b["numReintegrated"] and a["localSolved"] == b["localSolved"]
        assert np.array_equal(a["transform"], b["transform"], equal_nan=True)
    assert np.array_equal(t0, t1, equal_nan=True)


def test_lookahead_loop_equals_plain_loop(cuda_device):
    """bfFrameLoopStepAhead: the next frame's upload / ingest / SIFT detection / dense cache run on the loop's feature stream while the current frame is
    matched, solved and fused.  Same kernels, same inputs, destinations fixed one frame early: every status field, the trajectory, the heap, the
    counters and the fused model (canonical voxel words) are those of the plain loop -- over two chunk boundaries (where the chunk the next frame belongs to changes), with device and with pinned
    host frames, with and without the reconstruction stream."""
    import torch
    frames = [synth.make_frame(2 * i, W, H, texture="rich") for i in range(25)]
    dev_frames = [(torch.from_numpy(d).to(cuda_device), torch.from_numpy(c).to(cuda_device)) for d, c, T in frames]
    host_frames = [(torch.from_numpy(d).pin_memory(), torch.from_numpy(c).pin_memory()) for d, c, T in frames]
    out = []
    for mode in ("plain", "ahead", "ahead+overlap", "ahead-host", "ahead-every-other"):
        p = default_params(W, H)
        p.maxNumImages = 8; p.maxNumFrames = 40
        p.hash.m_hashNumBuckets = 100003; p.hash.m_numSDFBlocks = 90000
        loop = FrameLoop(p, cuda_device)
        loop.set_overlap(mode == "ahead+overlap")
        fr = host_frames if mode == "ahead-host" else dev_frames
        sts = []
        for i, (d, c) in enumerate(fr):
            announce = mode != "plain" and i + 1 < len(fr) and not (mode == "ahead-every-other" and i % 2)
            sts.append(loop.step(d, c, *(fr[i + 1] if announce else (None, None))).as_dict())
        loop.join()
        torch.cuda.synchronize()
        out.append((mode, sts, loop.trajectory(25), loop.heap_free(), loop.counters(), canonical_model(loop, cuda_device)))
        loop.close()
    _, s0, t0, f0, c0, m0 = out[0]
    assert c0["local_solves"] == 2 and c0["reintegrations"] > 0
    for mode, s1, t1, f1, c1, m1 in out[1:]:
        assert f0 == f1, mode
        assert np.array_equal(m0[0], m1[0]) and np.array_equal(m0[1], m1[1]), (mode, "another fused model")
        for k in ("frames", "integrations", "reintegrations", "local_solves", "global_solves", "keyframes"):
            assert c0[k] == c1[k], (mode, k)
        for a, b in zip(s0, s1):
            for k in a:
                if k == "transform":
                    assert np.array_equal(a[k], b[k], equal_nan=True), (mode, a["frame"])
                else:
                    assert a[k] == b[k], (mode, a["frame"], k, a[k], b[k])
        assert np.array_equal(t0, t1, equal_nan=True), mode


def test_lookahead_rejects_a_frame_that_was_not_announced(cuda_device):
    import torch
    from bundlefusion_b200 import _capi as capi
    p = default_params(W, H)
    p.maxNumImages = 8; p.maxNumFrames = 16
    p.hash.m_hashNumBuckets = 50021; p.hash.m_numSDFBlocks = 40000
    loop = FrameLoop(p, cuda_device)
    fr = [synth.make_frame(2 * i, W, H, texture="rich") for i in range(3)]
    t = [(torch.from_numpy(d).to(cuda_device), torch.from_numpy(c).to(cuda_device)) for d, c, T in fr]
    loop.step(t[0][0], t[0][1], t[1][0], t[1][1])
    with pytest.raises(Exception):
        loop.step(t[2][0], t[2][1])                      # frame 1 was announced
    with pytest.raises(Exception):
        loop.step_past_end()
    st = loop.step(t[1][0], t[1][1]).as_dict()           # the announced frame is still accepted
    assert st["frame"] == 1 and st["validTransform"] == 1
    loop.close()

"""The model the frame loop builds, checked exactly: the loop records every TSDF op it hands to bfTsdfRunOps (bfFrameLoopSetOpLog), and the
model must be the replay of that log -- on the CPU oracle in the bit-exact arithmetic, and through bfTsdfRunOps one re-integration item per call (no batch
pass, one lane) in the default arithmetic, bit for bit.  The replays read the loop's own frame store (bfFrameLoopGetFrame).

The ledger walks the same log: per frame, the multiset of poses it currently contributes at.  Every de-integration must remove a contribution
that is there, bit for bit; every turn is <= maxFrameFixes re-integration items, one GARBAGE_COLLECT, then at most the INTEGRATE of the current
frame at its status pose; at the end each frame contributes once at its trajectory pose, or not at all when that pose is -inf -- but for
stranded contributions: a frame whose pose turned -inf while it was queued for re-integration is skipped by the TrajectoryManager and never
de-integrated (the reference's behaviour, tests/test_trajectory_manager.py).

Streams (bfFrameLoopSetOverlap), look-ahead, the batch pass and the two lanes change when kernels run, not the model nor the op list.
Replayed one op per call the default arithmetic leaves the fused re-integration pass out, whose sdf is the two passes' composition up to the
rounding of a shared numerator: there the comparison is weights and blocks exact, sdf close.

Finally the difference between the model and a fresh fusion F of the returned trajectory is accounted for: R' = the replay plus a
de-integration of every stranded contribution, compared with F.  On the synthetic stream of test_frame_loop_finish_gpu.py (320 x 240,
synth.make_frame(2 i), texture "rich")."""
import ctypes as C

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from bundlefusion_b200 import synth
from bundlefusion_b200.frame_loop import FrameLoop, default_params

pytestmark = pytest.mark.gpu
W, H = 320, 240
K_TEST = 3
SDF_TOL = 1e-3                    # metres: the "sdf differs" line of the accounting table
INT, DEINT, GC = capi.BF_TSDF_OP_INTEGRATE, capi.BF_TSDF_OP_DEINTEGRATE, capi.BF_TSDF_OP_GARBAGE_COLLECT
EXACT, FAST = 0, 1

_STREAMS = {}


def stream(n, dev):
    """n raw frames (device tensors): synth.make_frame every second pose of the Lissajous path"""
    import torch
    if n not in _STREAMS:
        fr = [synth.make_frame(2 * i, W, H, texture="rich") for i in range(n)]
        _STREAMS[n] = [(torch.from_numpy(d).to(dev), torch.from_numpy(c).to(dev)) for d, c, _ in fr]
    return _STREAMS[n]


def loop_params(n):
    p = default_params(W, H)
    p.maxNumImages = max(16, n // 10 + 8); p.maxNumFrames = n + 16
    p.hash.m_hashNumBuckets = 100003 if n <= 64 else 200003
    p.hash.m_numSDFBlocks = 90000 if n <= 64 else 200000
    return p


class Run:
    pass


def run_loop(n, dev, arith=FAST, overlap=False, ahead=False, batching=1, lanes=1, finish=True):
    """the n-frame stream through the loop with the op log on, then (finish) bfFrameLoopFinish(K_TEST) one turn per call; the trajectory is read
    after every turn (host state only: it changes nothing the loop computes)"""
    import torch
    lib = capi.lib()
    prev = (lib.bfTsdfSetArithmetic(arith), lib.bfTsdfSetBatching(batching), lib.bfTsdfSetLanes(lanes))
    try:
        r = Run()
        r.loop = loop = FrameLoop(loop_params(n), dev)
        loop.set_op_log(True)
        loop.set_overlap(overlap)
        frames = stream(n, dev)
        r.status, r.traj, r.info = [], [], None
        for i, (d, c) in enumerate(frames):
            nxt = frames[i + 1] if ahead and i + 1 < n else (None, None)
            r.status.append(loop.step(d, c, *nxt).as_dict())
            r.traj.append(loop.trajectory(n))
        while finish:
            r.info = loop.finish(K_TEST, max_turns=1)
            r.traj.append(loop.trajectory(n))
            if r.info["done"]:
                break
            assert len(r.traj) < n + K_TEST + 2 + n, "finish does not end"
        loop.join()
        torch.cuda.synchronize(dev)
    finally:
        lib.bfTsdfSetArithmetic(prev[0]); lib.bfTsdfSetBatching(prev[1]); lib.bfTsdfSetLanes(prev[2])
    r.kinds, r.frames, r.poses, r.turns = loop.op_log()
    r.final = loop.trajectory(n)
    return r


def device_bytes(ptr, nbytes, dev):
    import torch

    class _View:
        pass
    v = _View()
    v.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False), "version": 3, "strides": None}
    return torch.as_tensor(v, device=dev)


def hash_snapshot(hd, hp, dev):
    """the hash table and voxel blocks of a device hash in the layout oracle.canonical_blocks reads, and its heap free count"""
    import torch
    torch.cuda.synchronize(dev)
    n_entries = int(hp.m_hashNumBuckets) * 4
    h = device_bytes(hd.d_hash, n_entries * 32, dev).cpu().numpy().view(np.int32).reshape(n_entries, 8)
    vox = device_bytes(hd.d_SDFBlocks, int(hp.m_numSDFBlocks) * 512 * 12, dev).cpu().numpy().view(np.int32).reshape(-1, 512, 3)
    counter = int(device_bytes(hd.d_heapCounter, 4, dev).cpu().numpy().view(np.uint32)[0])
    return {"hash": h, "voxels": vox}, (counter + 1) & 0xFFFFFFFF


def loop_model(loop, dev):
    from oracle import oracle as orc
    hd = loop.lib.bfFrameLoopGetHashData(loop._h).contents
    snap, free = hash_snapshot(hd, loop.lib.bfFrameLoopGetHashParams(loop._h).contents, dev)
    assert free == loop.heap_free()
    return orc.canonical_blocks(snap), free


def hash_params_of(loop):
    hp = capi.BFHashParams()
    C.memmove(C.byref(hp), C.byref(loop.lib.bfFrameLoopGetHashParams(loop._h).contents), C.sizeof(capi.BFHashParams))
    return hp


def assert_same_model(a, b, what):
    ((ba, va), fa), ((bb, vb), fb) = a, b
    assert ba.shape == bb.shape and np.array_equal(ba, bb), (what, "block set", len(ba), len(bb))
    diff = np.nonzero((va != vb).any(axis=-1))
    assert len(diff[0]) == 0, (what, "voxel words differ in %d voxels of %d blocks" % (len(diff[0]), len(np.unique(diff[0]))))
    assert fa == fb, (what, "heap free", fa, fb)


def assert_same_log(a, b, what):
    assert len(a.kinds) == len(b.kinds), (what, len(a.kinds), len(b.kinds))
    for x, y, name in ((a.kinds, b.kinds, "kind"), (a.frames, b.frames, "frame"), (a.turns, b.turns, "turn")):
        assert np.array_equal(x, y), (what, name, int(np.argmax(x != y)))
    assert np.array_equal(a.poses.view(np.uint32), b.poses.view(np.uint32)), (what, "pose")


# ---- the ledger -----------------------------------------------------------------------------------------------------------------------
def ledger(r, max_fixes):
    """walks the op log; returns (violations, stranded [(frame, turn, pose)], non-finite ops [(index, turn, kind, frame)], stats)"""
    bad, nonfinite = [], []
    contrib = {}                                     # frame -> [(pose bytes, turn it went in)]
    n_turns = len(r.traj)
    assert np.array_equal(np.unique(r.turns), np.arange(n_turns)), ("every turn issues ops, numbered 0 ..", n_turns, np.unique(r.turns)[-5:])
    for t in range(n_turns):
        idx = np.nonzero(r.turns == t)[0]
        k, fr = r.kinds[idx], r.frames[idx]
        gcs = np.nonzero(k == GC)[0]
        if len(gcs) != 1:
            bad.append(("turn %d: %d GARBAGE_COLLECT ops" % (t, len(gcs)))); continue
        g = gcs[0]
        items, j = 0, 0
        while j < g:                                 # re-integration items: lone ops and (DEINTEGRATE, INTEGRATE) pairs of one frame
            pair = j + 1 < g and k[j] == DEINT and k[j + 1] == INT and fr[j] == fr[j + 1]
            j += 2 if pair else 1
            items += 1
        if items > max_fixes:
            bad.append("turn %d: %d re-integration items" % (t, items))
        tail = idx[g + 1:]
        if len(tail) > 1 or (len(tail) == 1 and r.kinds[tail[0]] != INT):
            bad.append("turn %d: %d ops after the GARBAGE_COLLECT" % (t, len(tail)))
        if t < len(r.status):
            st = r.status[t]
            if st["validTransform"]:
                if len(tail) != 1 or r.frames[tail[0]] != t or not np.array_equal(r.poses[tail[0]].view(np.uint32), st["transform"].view(np.uint32)):
                    bad.append("turn %d: the INTEGRATE of the current frame is not at its status pose" % t)
            elif len(tail):
                bad.append("turn %d: an invalid frame was integrated" % t)
        elif len(tail):
            bad.append("past-end turn %d integrates" % t)
    for i in range(len(r.kinds)):
        kind, f, T, t = int(r.kinds[i]), int(r.frames[i]), r.poses[i], int(r.turns[i])
        if kind == GC:
            continue
        if not np.isfinite(T).all():
            nonfinite.append((i, t, "INTEGRATE" if kind == INT else "DEINTEGRATE", f))
        lst = contrib.setdefault(f, [])
        if kind == INT:
            lst.append((T.tobytes(), t))
        else:
            hit = [j for j, (p, _) in enumerate(lst) if p == T.tobytes()]
            if hit:
                lst.pop(hit[0])
            else:
                bad.append("op %d (turn %d): DEINTEGRATE of frame %d at a pose it does not contribute at" % (i, t, f))
    stranded = []
    for f in range(len(r.final)):
        lst = [(p, t) for p, t in contrib.get(f, []) if np.isfinite(np.frombuffer(p, np.float32)).all()]
        want = r.final[f]
        if np.isfinite(want).all():
            hit = [j for j, (p, _) in enumerate(lst) if p == want.tobytes()]
            if not hit:
                bad.append("frame %d does not contribute at its trajectory pose" % f); continue
            lst.pop(hit[0])
        for p, t in lst:                             # stranded: the frame's reported pose was -inf after some later turn
            later = [u for u in range(t, len(r.traj)) if len(r.traj[u]) > f and np.isneginf(r.traj[u][f]).all()]
            if later:
                stranded.append((f, t, np.frombuffer(p, np.float32).reshape(4, 4)))
            else:
                bad.append("frame %d: an extra contribution from turn %d that is not stranded" % (f, t))
    stats = {"ops": len(r.kinds), "turns": n_turns, "integrate": int((r.kinds == INT).sum()), "deintegrate": int((r.kinds == DEINT).sum()),
             "stranded": [(f, t) for f, t, _ in stranded], "nonfinite": nonfinite,
             "invalid_at_end": int(sum(1 for f in range(len(r.final)) if not np.isfinite(r.final[f]).all()))}
    return bad, stranded, nonfinite, stats


def check_ledger(r, what, max_fixes=10):
    bad, stranded, nonfinite, stats = ledger(r, max_fixes)
    print("ledger %s: %s" % (what, stats))
    assert not bad, (what, bad[:10])
    return stranded


# ---- replays ------------------------------------------------------------------------------------------------------------------------------
def replay_on_oracle(r, dev):
    """the log op by op on OracleSceneRepHashSDF (bit-exact arithmetic), from the loop's frame store downloaded"""
    import time
    from bundlefusion_b200.scene_rep import camera_params
    from oracle import oracle as orc
    cam = camera_params(W, H)
    o = orc.OracleSceneRepHashSDF(hash_params_of(r.loop))
    host = {}
    t0 = time.perf_counter()
    for kind, f, T in zip(r.kinds, r.frames, r.poses):
        if kind == GC:
            o.garbageCollect(); continue
        if f not in host:
            d, c = r.loop.frame(int(f))
            host[f] = (d.cpu().numpy(), np.ascontiguousarray(c.cpu().numpy()))
        (o.integrate if kind == INT else o.deIntegrate)(T, host[f][0], host[f][1], cam)
    secs = time.perf_counter() - t0
    return (orc.canonical_blocks(o.download()), o.getHeapFreeCount()), secs


class DeviceReplay:
    """a fresh hash with the loop's parameters; ops through bfTsdfRunOps one call per op -- or, with pairs=True, one call per re-integration
    item, so that a (DEINTEGRATE, INTEGRATE) pair of a frame takes the fused pass -- batching and lanes off, on the current stream"""

    def __init__(self, r, dev):
        from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF, camera_params
        self.scene = CUDASceneRepHashSDF(hash_params_of(r.loop), dev, arithmetic="fast")
        self.cam = camera_params(W, H)
        n = len(r.final)
        ptrs = [r.loop.frame(f) for f in range(n)]
        self.keep = ptrs
        self.d = (C.c_void_p * n)(*[p[0].data_ptr() for p in ptrs])
        self.c = (C.c_void_p * n)(*[p[1].data_ptr() for p in ptrs])
        self.dev = dev

    def run(self, ops, pairs=False):
        s, lib = self.scene, self.scene.lib
        ops = list(ops)
        s._bind_stream()
        prev = (lib.bfTsdfSetBatching(0), lib.bfTsdfSetLanes(0))
        try:
            i = 0
            while i < len(ops):
                m = 2 if pairs and i + 1 < len(ops) and ops[i][0] == DEINT and ops[i + 1][0] == INT and ops[i][1] == ops[i + 1][1] else 1
                arr = (capi.BFTsdfOp * m)()
                for j, (kind, f, T) in enumerate(ops[i:i + m]):
                    arr[j].kind, arr[j].frame = int(kind), int(f)
                    C.memmove(arr[j].pose, np.ascontiguousarray(T, np.float32).ctypes.data, 64)
                capi.check(lib.bfTsdfRunOps(C.byref(s.m_hashData), C.byref(s.m_hashParams), C.byref(self.cam), arr, m, self.d, self.c), "bfTsdfRunOps")
                i += m
        finally:
            lib.bfTsdfSetBatching(prev[0]); lib.bfTsdfSetLanes(prev[1])

    def model(self):
        from oracle import oracle as orc
        snap = self.scene.download()
        return orc.canonical_blocks(snap), self.scene.getHeapFreeCount()

    def close(self):
        self.scene.close()


def fresh_fusion(r, dev):
    """F: a fresh hash, every frame with a finite final pose integrated at it (the loop's frame store), in frame order"""
    rep = DeviceReplay(r, dev)
    rep.run([(INT, f, r.final[f]) for f in range(len(r.final)) if np.isfinite(r.final[f]).all()])
    m = rep.model()
    rep.close()
    return m


def model_difference(a, b):
    """voxels with weight > 0 in one model only (split: the other model has the block / never allocated it), with another weight, and
    with |d sdf| > SDF_TOL where the weights agree"""
    ((ba, va), _), ((bb, vb), _) = a, b
    pack = lambda k: ((k[:, 0].astype(np.int64) + 32768) * 65536 + (k[:, 1] + 32768)) * 65536 + (k[:, 2] + 32768)
    common, ia, ib = np.intersect1d(pack(ba), pack(bb), assume_unique=True, return_indices=True)
    wa, wb = va[..., 1].view(np.float32), vb[..., 1].view(np.float32)
    sa, sb = va[..., 0].view(np.float32), vb[..., 0].view(np.float32)
    ca, cb = np.ones(len(ba), bool), np.ones(len(bb), bool)
    ca[ia] = False; cb[ib] = False
    no_block = int((wa[ca] > 0).sum() + (wb[cb] > 0).sum())
    wa_c, wb_c = wa[ia], wb[ib]
    with_block = int(((wa_c > 0) != (wb_c > 0)).sum())
    both = (wa_c > 0) & (wb_c > 0)
    other_w = int((both & (wa_c != wb_c)).sum())
    same = both & (wa_c == wb_c)
    far = int((np.abs(sa[ia] - sb[ib])[same] > SDF_TOL).sum())
    n = int((wb > 0).sum())
    return {"voxels": n, "one_model_only": no_block + with_block, "one_only_block_absent": no_block, "one_only_block_in_both": with_block,
            "other_weight": other_w, "sdf_above_1mm": far}


# ---- tests --------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [43, 23])
def test_model_is_the_exact_replay_of_its_op_log(cuda_device, n):
    """the loop in the bit-exact TSDF arithmetic, through finish(3); its op log replayed on the CPU oracle from the loop's frame store gives the
    same block set, the same sdf / weight / colour words and the same heap free count.  43 frames: the ledger holds as well."""
    r = run_loop(n, cuda_device, arith=EXACT)
    assert r.info["done"] and r.info["valid"], r.info
    if n == 43:
        check_ledger(r, "43 frames, exact")
    got = loop_model(r.loop, cuda_device)
    want, secs = replay_on_oracle(r, cuda_device)
    print("%d frames: %d ops replayed on the CPU oracle in %.1f s; %d blocks" % (n, len(r.kinds), secs, len(got[0][0])))
    assert_same_model(got, want, "%d frames: loop vs oracle replay" % n)
    r.loop.close()


def test_200_frame_model_is_the_replay_of_its_op_log_and_accounts_for_the_fresh_fusion(cuda_device):
    """200 frames through finish(3) in the default arithmetic: the ledger holds; the log replayed one re-integration item per bfTsdfRunOps call
    (no batch pass, one lane) is the model bit for bit -- the batch pass, its cull and the two lanes on the op lists the loop really produces;
    replayed one op per call (no fused pair either) it is the model but for the fused pass's shared rounding of the sdf numerator (include/bf_tsdf.h,
    csrc/tsdf_fast.cu: the default arithmetic's fused pair is the composition of the two passes up to < 2e-7 m a pair); R' (the replay plus a
    de-integration of every stranded contribution) against the fresh fusion F of the trajectory"""
    r = run_loop(200, cuda_device)
    assert r.info["done"] and r.info["valid"], r.info
    stranded = check_ledger(r, "200 frames")
    got = loop_model(r.loop, cuda_device)
    rep = DeviceReplay(r, cuda_device)
    rep.run(zip(r.kinds, r.frames, r.poses), pairs=True)
    assert_same_model(got, rep.model(), "200 frames: loop vs replay, one re-integration item per call")
    single = DeviceReplay(r, cuda_device)
    single.run(zip(r.kinds, r.frames, r.poses))
    assert_close_model(got, single.model(), "200 frames: loop vs replay, one op per call")
    single.close()
    account(r, rep, stranded, got, "200 frames", cuda_device)
    rep.close()
    r.loop.close()


def assert_close_model(a, b, what, sdf_tol=1e-4):
    """same block set, heap and weights; sdf within sdf_tol (the fused pass against the two passes it fuses, accumulated over the run)"""
    ((ba, va), fa), ((bb, vb), fb) = a, b
    assert np.array_equal(ba, bb) and fa == fb, (what, "block set / heap")
    wa, wb = va[..., 1].view(np.float32), vb[..., 1].view(np.float32)
    assert np.array_equal(wa, wb), (what, "weights differ in %d voxels" % int((wa != wb).sum()))
    d = np.abs(va[..., 0].view(np.float32) - vb[..., 0].view(np.float32))[wa > 0]
    print("%s: %d of %d voxels differ in sdf, max %.3g m" % (what, int((d > 0).sum()), d.size, float(d.max())))
    assert float(d.max()) <= sdf_tol, what


def account(r, rep, stranded, model, what, dev):
    """model vs F and R' vs F; and both against F0, the fresh fusion run twice (every frame integrated, de-integrated, integrated again at its
    final pose: every block any frame allocates exists before the first voxel update that counts)"""
    F = fresh_fusion(r, dev)
    m_vs_f = model_difference(model, F)
    rep.run([(DEINT, f, T) for f, _, T in stranded])
    r2 = rep.model()
    r_vs_f = model_difference(r2, F)
    valid = [f for f in range(len(r.final)) if np.isfinite(r.final[f]).all()]
    pre = DeviceReplay(r, dev)
    pre.run([(INT, f, r.final[f]) for f in valid] + [(DEINT, f, r.final[f]) for f in valid] + [(INT, f, r.final[f]) for f in valid])
    F0 = pre.model()
    pre.close()
    r_vs_f0 = model_difference(r2, F0)
    print("%s accounting: %d stranded contributions\n  model vs F  %s\n  R' vs F    %s\n  model vs F0 %s\n  R' vs F0   %s\n  F vs F0     %s"
          % (what, len(stranded), m_vs_f, r_vs_f, model_difference(model, F0), r_vs_f0, model_difference(F, F0)))
    # measured on an H100 (43 / 200 frames, no stranded contribution): R' vs F 18 / 428 voxels in one model only, 123 / 10395 with another weight,
    # 0 / 690 with |d sdf| > 1 mm; against F0 no sdf difference is left: what remains is which blocks existed when a frame was integrated
    assert r_vs_f0["sdf_above_1mm"] == 0, r_vs_f0
    return m_vs_f, r_vs_f


def test_streams_lookahead_batching_and_lanes_do_not_change_the_model(cuda_device):
    """43 frames through finish(3): overlap off / on, look-ahead announcing every frame, batching off, lanes off -- identical op logs and
    identical canonical blocks and heap; the model against the oracle's replay of the log under the tolerance contract of the default
    arithmetic (DESIGN section 3b); and the fresh-fusion accounting at 43 frames"""
    base = run_loop(43, cuda_device)
    assert base.info["done"] and base.info["valid"], base.info
    stranded = check_ledger(base, "43 frames")
    want = loop_model(base.loop, cuda_device)
    for name, kw in (("overlap", dict(overlap=True)), ("look-ahead", dict(ahead=True)), ("look-ahead + overlap", dict(ahead=True, overlap=True)),
                     ("batching off", dict(batching=0)), ("lanes off", dict(lanes=0))):
        r = run_loop(43, cuda_device, **kw)
        assert_same_log(base, r, name)
        assert_same_model(loop_model(r.loop, cuda_device), want, name)
        r.loop.close()
    (ob, ov), ofree = replay_on_oracle(base, cuda_device)[0]
    (gb, gv), gfree = want
    assert np.array_equal(gb, ob) and gfree == ofree, "block set / heap differ from the oracle's replay"
    gw, ow = gv[..., 1].view(np.float32), ov[..., 1].view(np.float32)
    n = gw.size
    w_mismatch = int((gw != ow).sum())
    touched = (gw == ow) & (gw > 0)
    dsdf = np.abs(gv[..., 0].view(np.float32) - ov[..., 0].view(np.float32))[touched]
    flips = int((dsdf > 1e-4).sum())
    print("43 frames, default arithmetic vs the oracle's replay: %d of %d voxel weights differ, %d of %d touched voxels |d sdf| > 1e-4 m, max %.3g"
          % (w_mismatch, n, flips, dsdf.size, float(dsdf.max())))
    # the per-op contract (<= 1e-4 of the voxels on a decision boundary) accumulated over 358 ops; measured on an H100: 9.3e-5 of the weights,
    # 4.0e-4 of the touched voxels
    assert w_mismatch <= 3e-4 * n and flips <= 1.5e-3 * dsdf.size
    rep = DeviceReplay(base, cuda_device)
    rep.run(zip(base.kinds, base.frames, base.poses), pairs=True)
    assert_same_model(want, rep.model(), "43 frames: loop vs replay, one re-integration item per call")
    account(base, rep, stranded, want, "43 frames", cuda_device)
    rep.close()
    base.loop.close()

"""Pins the host TrajectoryManager of the library (csrc/trajectory_host.cu, bfTrajectory*) and its Python restatement against the REFERENCE's
own class: FL/TrajectoryManager.{h,cpp} with the Lie pose maps of FL/PoseHelper.h, compiled by g++ against minimal mLib types
(oracle/build_ref.py build_trajectory_host -> oracle/_ref/libref_trajectory_host.so) and driven through application-like sessions (frames
arrive, the optimiser rewrites the trajectory, DepthSensing.cpp's reintegrate() pops one operation per turn in its priority order).  What the
reference returned -- every popped operation with its transforms, the frame types and the number of queued operations after every frame --
is committed as tests/golden/trajectory_manager_reference.npz (scripts/make_golden_trajectory_manager.py) and replayed here.
Pose distances agree to ~1e-5 relative (the host's SE(3) logarithm differs from the device one in operation order); the sessions are built so
that no ordering decision sits closer than that."""
import os

import numpy as np

from bundlefusion_b200.trajectory_manager import TrajectoryManager
from oracle import oracle as orc
from oracle.trajectory_manager_oracle import TrajectoryManagerOracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "trajectory_manager_reference.npz")
NEG = np.full((4, 4), -np.inf, np.float32)
SESSIONS, N = 12, 60


def rand_pose(rng, rot=0.3, trans=0.5):
    return orc.pose_to_matrix(rng.normal(0, rot, 3).astype(np.float32), rng.normal(0, trans, 3).astype(np.float32))


class Recorder:
    """Wraps the live reference: forwards every call and records what it returned."""

    def __init__(self, ref):
        self.ref, self.log = ref, []

    def __getattr__(self, name):
        fn = getattr(self.ref, name)

        def call(*a):
            r = fn(*a)
            if name.startswith("get") or name in ("types", "active"):
                self.log.append((name, r))
            return r
        return call


class Replay:
    """Stands in for the reference: mutators do nothing, queries return the recorded answers in order."""

    def __init__(self, log):
        self.log, self.pos = log, 0

    def __getattr__(self, name):
        def call(*a):
            if name.startswith("get") or name in ("types", "active"):
                rec = self.log[self.pos]; self.pos += 1
                assert rec[0] == name, (rec[0], name)
                return rec[1]
            return None
        return call


def same_pop(a, b):
    if b is None:
        return a is None
    return a is not None and len(a) == len(b) and all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(a, b))


def run_session(seed, impls, ref):
    """impls: objects with the TrajectoryManager method names (the library's class, the Python restatement); ref: Recorder or Replay."""
    rng = np.random.default_rng(500 + seed)
    topN, minD = int(rng.integers(1, 8)), float(rng.choice([0.0, 1e-4, 1e-2]))
    made = [make(N, topN, minD) for make in impls]
    ref.create(N, topN, minD)
    traj = np.zeros((N, 4, 4), np.float32)
    added = nOpt = 0
    for frame in range(N):
        valid = rng.random() < 0.9
        T = rand_pose(rng) if valid else NEG.copy()
        kind = 0 if valid else 1
        for m in made:
            m.addFrame(kind, T, added)
        ref.addFrame(kind, T, added)
        traj[added] = T; added += 1
        if rng.random() < 0.7:
            n = nOpt = int(min(N, max(nOpt, added - int(rng.integers(0, 3)))))
            for i in range(min(n, added)):
                r = rng.random()
                if r < 0.05:
                    traj[i] = -np.inf
                elif r < 0.4 or np.isneginf(traj[i, 0, 0]):
                    base = traj[i] if not np.isneginf(traj[i, 0, 0]) else rand_pose(rng)
                    traj[i] = (rand_pose(rng, 0.02, 0.05) @ base).astype(np.float32); traj[i, 3] = [0, 0, 0, 1]
            for m in made:
                m.updateOptimizedTransform(traj, n)
            ref.updateOptimizedTransform(traj, n)
        for m in made:
            m.generateUpdateLists()
        ref.generateUpdateLists()
        for _ in range(int(rng.integers(0, 6))):                      # DepthSensing.cpp:871-899: one operation per turn, in this priority
            b = ref.getTopFromDeIntegrateList()
            for m in made:
                assert same_pop(m.getTopFromDeIntegrateList(), b), (seed, frame, "de-integrate")
            if b is not None:
                continue
            b = ref.getTopFromIntegrateList()
            for m in made:
                assert same_pop(m.getTopFromIntegrateList(), b), (seed, frame, "integrate")
            if b is not None:
                if not np.isneginf(b[0][0, 0]):
                    for m in made:
                        m.confirmIntegration(b[1])
                    ref.confirmIntegration(b[1])
                continue
            b = ref.getTopFromReIntegrateList()
            for m in made:
                assert same_pop(m.getTopFromReIntegrateList(), b), (seed, frame, "re-integrate")
            if b is not None:
                if not np.isneginf(b[1][0, 0]):
                    for m in made:
                        m.confirmIntegration(b[2])
                    ref.confirmIntegration(b[2])
                continue
            break
        types, active = ref.types(added), ref.active()
        for m in made:
            mine = [m.frameType(i) for i in range(added)] if hasattr(m, "frameType") else [m.frames[i].type for i in range(added)]
            assert mine == list(types), (seed, frame)
            assert m.getNumActiveOperations() == active, (seed, frame)


EXTRA_SESSIONS = ("stranded", "all_lost")


def run_extra_session(name, impls, ref):
    """Two scripted sessions around a frame that loses its pose while it waits in the re-integration list.  "stranded": frames 0-5 integrated,
    0-3 moved (queued 0, 1, 2, 3), one pop, frames 1-2 set to -inf, pops until empty, generateUpdateLists, 1-2 finite again, drain -- 1 and 2
    are never de-integrated and are integrated a second time.  "all_lost": every queued frame set to -inf; the pop returns the last one with
    newT = -inf."""
    rng = np.random.default_rng(900 + EXTRA_SESSIONS.index(name))
    n = 6 if name == "stranded" else 3
    made = [make(8, 8, 0.0) for make in impls]
    ref.create(8, 8, 0.0)
    everyone = made + [ref]
    poses = np.stack([rand_pose(rng) for _ in range(n)])

    def each(fn):
        for m in everyone:
            fn(m)

    def check(what):
        types, active = ref.types(n), ref.active()
        for m in made:
            mine = [m.frameType(i) for i in range(n)] if hasattr(m, "frameType") else [m.frames[i].type for i in range(n)]
            assert mine == list(types) and m.getNumActiveOperations() == active, (name, what)

    def pop(limit):
        for _ in range(limit):
            for kind in ("getTopFromDeIntegrateList", "getTopFromIntegrateList", "getTopFromReIntegrateList"):
                b = getattr(ref, kind)()
                for m in made:
                    assert same_pop(getattr(m, kind)(), b), (name, kind)
                if b is not None:
                    break
            if b is None:
                return
            new = b[1] if kind == "getTopFromReIntegrateList" else b[0]
            if kind != "getTopFromDeIntegrateList" and not np.isneginf(new[0, 0]):
                each(lambda m: m.confirmIntegration(b[-1]))
            check(kind)

    for i in range(n):
        each(lambda m: m.addFrame(0, poses[i], i))
    each(lambda m: m.updateOptimizedTransform(poses, n)); each(lambda m: m.generateUpdateLists())
    moved = poses.copy()
    for i, dx in enumerate((0.4, 0.3, 0.2, 0.1)[:min(4, n)]):
        moved[i, 0, 3] += np.float32(dx)
    each(lambda m: m.updateOptimizedTransform(moved, n)); each(lambda m: m.generateUpdateLists())
    check("queued")
    gone = moved.copy()
    if name == "stranded":
        pop(1)
        gone[1:3] = -np.inf
    else:
        gone[:] = -np.inf
    each(lambda m: m.updateOptimizedTransform(gone, n))
    pop(20)
    each(lambda m: m.generateUpdateLists())
    check("invalidated")
    pop(20)
    back = moved.copy()
    if name == "stranded":
        back[1, 1, 3] += np.float32(0.05); back[2, 1, 3] -= np.float32(0.05)
    each(lambda m: m.updateOptimizedTransform(back, n)); each(lambda m: m.generateUpdateLists())
    check("back")
    pop(20)
    each(lambda m: m.generateUpdateLists())
    check("drained")


def load_log(g, s):
    names = ["getTopFromDeIntegrateList", "getTopFromIntegrateList", "getTopFromReIntegrateList", "types", "active"]
    log = []
    p = f"s{s}" if isinstance(s, int) else s
    kinds, found, idx, T = g[f"{p}_kind"], g[f"{p}_found"], g[f"{p}_idx"], g[f"{p}_T"]
    types, tpos = g[f"{p}_types"], 0
    for k in range(len(kinds)):
        name = names[kinds[k]]
        if name == "types":
            n = int(idx[k]); log.append((name, types[tpos:tpos + n].tolist())); tpos += n
        elif name == "active":
            log.append((name, int(idx[k])))
        elif not found[k]:
            log.append((name, None))
        elif name == "getTopFromReIntegrateList":
            log.append((name, (T[k, 0].reshape(4, 4), T[k, 1].reshape(4, 4), int(idx[k]))))
        else:
            log.append((name, (T[k, 0].reshape(4, 4), int(idx[k]))))
    return log


def test_library_and_restatement_replay_the_reference_sessions():
    g = np.load(GOLDEN)
    ops = 0
    for s in range(SESSIONS):
        log = load_log(g, s)
        rp = Replay(log)
        run_session(s, [TrajectoryManager, TrajectoryManagerOracle], rp)
        assert rp.pos == len(log)
        ops += sum(1 for name, r in log if name.startswith("get") and r is not None)
    assert ops > 1000


def test_library_and_restatement_replay_the_reference_on_a_frame_lost_while_queued():
    """the reference's own class on the two scripted sessions of run_extra_session: what it pops, its frame types and queue sizes after every
    pop, replayed against the library's class and the restatement"""
    g = np.load(GOLDEN)
    for name in EXTRA_SESSIONS:
        log = load_log(g, name)
        rp = Replay(log)
        run_extra_session(name, [TrajectoryManager, TrajectoryManagerOracle], rp)
        assert rp.pos == len(log), name
    stranded = load_log(g, "stranded")
    re_pops = [r for name, r in stranded if name == "getTopFromReIntegrateList" and r is not None]
    assert [r[2] for r in re_pops] == [0, 3]                              # frames 1 and 2 were skipped, never popped
    assert not [r for name, r in stranded if name == "getTopFromDeIntegrateList" and r is not None]
    assert sorted(r[1] for name, r in stranded if name == "getTopFromIntegrateList" and r is not None) == [1, 2]
    lost = [r for name, r in load_log(g, "all_lost") if name == "getTopFromReIntegrateList" and r is not None]
    assert lost[0][2] == 2 and np.all(np.isneginf(lost[0][1]))

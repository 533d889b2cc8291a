"""Host-side TrajectoryManager (csrc/trajectory_host.cu behind include/bf_bundler.h) against the plain-Python restatement of
FL/TrajectoryManager.cpp (oracle/trajectory_manager_oracle.py).  Pure host logic: runs without a GPU."""
import numpy as np
import pytest

from bundlefusion_b200 import trajectory_manager as tmod
from bundlefusion_b200.trajectory_manager import TrajectoryManager
from oracle import oracle as orc
from oracle.trajectory_manager_oracle import TrajectoryManagerOracle

NEG = np.full((4, 4), -np.inf, np.float32)


def rand_pose(rng, rot=0.3, trans=0.5):
    return orc.pose_to_matrix(rng.normal(0, rot, 3).astype(np.float32), rng.normal(0, trans, 3).astype(np.float32))


def same_state(tm, ref, n):
    assert tm.getNumAddedFrames() == ref.numAdded and tm.getNumOptimizedFrames() == ref.numOptimized
    assert tm.getNumActiveOperations() == ref.getNumActiveOperations()
    for i in range(n):
        assert tm.frameType(i) == ref.frames[i].type, i
    a, b = tm.getOptimizedTransforms(), ref.getOptimizedTransforms()
    assert a.shape == b.shape and np.array_equal(a, b)


def same_pop(a, b):
    if b is None:
        assert a is None
        return
    assert a is not None and len(a) == len(b)
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y))


def test_constructor_and_empty_lists():
    tm = TrajectoryManager(16, topNActive=3, minPoseDistSqrt=0.01)
    assert tm.getNumAddedFrames() == 0 and tm.getNumOptimizedFrames() == 0 and tm.getNumActiveOperations() == 0
    assert tm.getTopFromIntegrateList() is None and tm.getTopFromDeIntegrateList() is None and tm.getTopFromReIntegrateList() is None
    assert all(tm.frameType(i) == tmod.NOT_INTEGRATED_NO_TRANSFORM for i in range(16))
    tm.generateUpdateLists()                                  # nothing added: no-op
    assert tm.getNumActiveOperations() == 0 and tm.getOptimizedTransforms().shape == (0, 4, 4)
    with pytest.raises(IndexError):
        tm.addFrame(tmod.INTEGRATED, np.eye(4), 16)


def test_reintegration_selection_by_pose_distance():
    """Five integrated frames; the optimiser moves #1 a lot, #3 a little, #4 below the threshold: the list is (#1, #3), capped by topN."""
    rng = np.random.default_rng(1)
    poses = [rand_pose(rng) for _ in range(5)]
    tm = TrajectoryManager(8, topNActive=2, minPoseDistSqrt=1e-3)
    for i, T in enumerate(poses):
        tm.addFrame(tmod.INTEGRATED, T, i)
    opt = np.stack(poses).copy()
    opt[1, :3, 3] += np.float32(0.5)
    opt[3, :3, 3] += np.float32(0.1)
    opt[4, 0, 3] += np.float32(0.01)                          # dist 4e-4 < 1e-3
    opt[2, 1, 3] += np.float32(0.05)                          # dist 1e-2: third largest, cut by topN = 2
    tm.updateOptimizedTransform(opt, 5)
    tm.generateUpdateLists()
    assert [tm.frameType(i) for i in range(5)] == [tmod.INTEGRATED, tmod.REINTEGRATION, tmod.INTEGRATED, tmod.REINTEGRATION, tmod.INTEGRATED]
    # the distance is taken between Lie-algebra poses (t_lie = V^-1 t), so it is |dt|^2 only up to the rotation's V^-1: a few percent here
    for i, want in ((1, 4 * 0.75), (3, 4 * 0.03), (4, 4 * 1e-4), (2, 4 * 2.5e-3)):          # the factor 2 multiplies the translation part of the pose
        assert abs(tm.frameDist(i) - want) < 0.15 * want, (i, tm.frameDist(i))
    assert tm.frameDist(0) == 0.0
    assert tm.getNumActiveOperations() == 2
    old, new, idx = tm.getTopFromReIntegrateList()
    assert idx == 1 and np.array_equal(old, poses[1]) and np.array_equal(new, opt[1])
    tm.confirmIntegration(1)
    tm.generateUpdateLists()                                  # #1 is now integrated with its optimised pose (dist 0)
    # Reference quirk kept (cpp:97): the refill loop starts at sorted[len(list)], not sorted[0] -- with #3 still queued it looks at the
    # SECOND-largest integrated frame (#4, below the threshold) and stops, so #2 is not picked yet.
    assert tm.frameDist(1) == 0.0 and tm.frameType(2) == tmod.INTEGRATED and tm.getNumActiveOperations() == 1
    assert tm.getTopFromReIntegrateList()[2] == 3
    tm.confirmIntegration(3)
    tm.generateUpdateLists()                                  # list empty -> starts at sorted[0] = #2
    assert tm.frameType(2) == tmod.REINTEGRATION and tm.getTopFromReIntegrateList()[2] == 2
    assert tm.getTopFromReIntegrateList() is None


def test_invalidation_and_revalidation():
    rng = np.random.default_rng(2)
    poses = np.stack([rand_pose(rng) for _ in range(4)])
    tm = TrajectoryManager(4, topNActive=4, minPoseDistSqrt=0.0)
    tm.addFrame(tmod.INTEGRATED, poses[0], 0)
    tm.addFrame(tmod.INTEGRATED, poses[1], 1)
    tm.addFrame(tmod.NOT_INTEGRATED_NO_TRANSFORM, NEG, 2)     # a frame that could not be aligned (Bundler marks it -inf)
    tm.addFrame(tmod.INTEGRATED, poses[3], 3)
    opt = poses.copy(); opt[1] = -np.inf; opt[2] = -np.inf
    tm.updateOptimizedTransform(opt, 4)
    tm.generateUpdateLists()
    assert tm.frameType(1) == tmod.INVALID and tm.frameType(2) == tmod.INVALID
    T, idx = tm.getTopFromDeIntegrateList()                   # only the frame that WAS integrated is de-integrated, with the pose it went in with
    assert idx == 1 and np.array_equal(T, poses[1]) and tm.getTopFromDeIntegrateList() is None
    out = tm.getOptimizedTransforms()
    assert np.all(np.isneginf(out[1])) and np.all(np.isneginf(out[2])) and np.array_equal(out[0], poses[0])
    opt[2] = poses[2]                                         # the optimiser recovers frame 2
    tm.updateOptimizedTransform(opt, 4)
    tm.generateUpdateLists()
    assert tm.frameType(2) == tmod.NOT_INTEGRATED_WITH_TRANSFORM
    T, idx = tm.getTopFromIntegrateList()
    assert idx == 2 and np.array_equal(T, poses[2])
    tm.confirmIntegration(2)
    assert tm.frameType(2) == tmod.INTEGRATED and tm.getNumActiveOperations() == 0


def test_reintegrate_list_skips_frames_invalidated_while_queued():
    """getTopFromReIntegrateList pops entries whose optimised pose went invalid meanwhile and returns the first valid one (cpp:121-133)."""
    rng = np.random.default_rng(3)
    poses = np.stack([rand_pose(rng) for _ in range(3)])
    tm = TrajectoryManager(3, topNActive=3, minPoseDistSqrt=0.0)
    ref = TrajectoryManagerOracle(3, 3, 0.0)
    for m in (tm, ref):
        for i in range(3):
            m.addFrame(tmod.INTEGRATED, poses[i], i)
    opt = poses.copy(); opt[:, 0, 3] += np.float32([0.3, 0.2, 0.1])
    for m in (tm, ref):
        m.updateOptimizedTransform(opt, 3); m.generateUpdateLists()
    opt2 = opt.copy(); opt2[0] = -np.inf
    for m in (tm, ref):
        m.updateOptimizedTransform(opt2, 3)
    a, b = tm.getTopFromReIntegrateList(), ref.getTopFromReIntegrateList()
    same_pop(a, b)
    assert a[2] == 1 and tm.getNumActiveOperations() == 1
    same_state(tm, ref, 3)


@pytest.mark.parametrize("seed", [0, 1, 2, 3, 4])
def test_random_sessions_match_the_restatement(seed):
    """A scanning session in miniature: frames arrive, the optimiser rewrites the trajectory (sometimes marking frames invalid, sometimes
    for fewer / more frames than were added), the fusion thread pops one operation of each kind per frame and confirms it."""
    rng = np.random.default_rng(100 + seed)
    N, topN, minD = 40, int(rng.integers(1, 6)), float(rng.choice([0.0, 1e-4, 1e-2]))
    tm, ref = TrajectoryManager(N, topN, minD), TrajectoryManagerOracle(N, topN, minD)
    traj = np.zeros((N, 4, 4), np.float32)
    added, nOpt = 0, 0
    for step in range(3 * N):
        op = rng.random()
        if added < N and (op < 0.35 or added == 0):
            valid = rng.random() < 0.85
            T = rand_pose(rng) if valid else NEG.copy()
            kind = tmod.INTEGRATED if valid else tmod.NOT_INTEGRATED_NO_TRANSFORM
            tm.addFrame(kind, T, added); ref.addFrame(kind, T, added)
            traj[added] = T
            added += 1
        elif op < 0.6:
            # the optimised-frame count only grows in the application (with a shrinking count the reference sorts on stale distances)
            n = nOpt = int(min(N, max(nOpt, added + rng.integers(-2, 2))))
            for i in range(min(n, added)):
                r = rng.random()
                if r < 0.1:
                    traj[i] = -np.inf
                elif r < 0.5 or np.isneginf(traj[i, 0, 0]):
                    base = traj[i] if not np.isneginf(traj[i, 0, 0]) else rand_pose(rng)
                    traj[i] = (rand_pose(rng, 0.02, 0.05) @ base).astype(np.float32)
                    traj[i, 3] = [0, 0, 0, 1]
            tm.updateOptimizedTransform(traj, n); ref.updateOptimizedTransform(traj, n)
            tm.generateUpdateLists(); ref.generateUpdateLists()
            for i in range(min(n, added)):
                if ref.frames[i].type in (tmod.INTEGRATED, tmod.REINTEGRATION) and np.isfinite(ref.frames[i].dist):
                    assert tm.frameDist(i) == ref.frames[i].dist, (i, tm.frameDist(i), ref.frames[i].dist)
        else:
            a, b = tm.getTopFromDeIntegrateList(), ref.getTopFromDeIntegrateList()
            same_pop(a, b)
            a, b = tm.getTopFromReIntegrateList(), ref.getTopFromReIntegrateList()
            same_pop(a, b)
            if b is not None and not np.isneginf(b[1][0, 0]):
                tm.confirmIntegration(b[2]); ref.confirmIntegration(b[2])
            a, b = tm.getTopFromIntegrateList(), ref.getTopFromIntegrateList()
            same_pop(a, b)
            if b is not None:
                tm.confirmIntegration(b[1]); ref.confirmIntegration(b[1])
        same_state(tm, ref, added)


def reconstruct_turn(m, ops, max_fixes=10):
    """the pops of one reintegrate() turn as the frame loop makes them (csrc/frame_loop.cu reconstruct, DepthSensing.cpp:867-899): de-integrate list
    first, then integrate list, then re-integration list (a pair: de-integrate at the old pose, integrate at the new one); each integration confirmed.
    Appends (kind, frame, pose) to ops, kind 'D' or 'I'; returns the raw pops."""
    pops = []
    for _ in range(max_fixes):
        r = m.getTopFromDeIntegrateList()
        if r is not None:
            pops.append(("de", r)); ops.append(("D", r[1], r[0])); continue
        r = m.getTopFromIntegrateList()
        if r is not None:
            pops.append(("in", r)); ops.append(("I", r[1], r[0])); m.confirmIntegration(r[1]); continue
        r = m.getTopFromReIntegrateList()
        if r is not None:
            pops.append(("re", r)); ops.append(("D", r[2], r[0])); ops.append(("I", r[2], r[1])); m.confirmIntegration(r[2]); continue
        break
    return pops


def test_frame_invalidated_while_queued_for_reintegration_is_stranded():
    """A frame whose optimised pose turns -inf while it waits in the re-integration list is popped and skipped
    (TrajectoryManager.cpp:116-136): it stays of type REINTEGRATION, so the next generateUpdateLists marks it INVALID without queueing a
    de-integration (cpp:201-210 queues one only for INTEGRATED).  Its old contribution stays in the model; when its pose comes back it is
    integrated a second time.  The library's class and the restatement agree op for op; the reference's own class is pinned on the same
    session by test_trajectory_manager_reference.py."""
    rng = np.random.default_rng(7)
    poses = np.stack([rand_pose(rng) for _ in range(6)])
    tm, ref = TrajectoryManager(8, topNActive=8, minPoseDistSqrt=0.0), TrajectoryManagerOracle(8, 8, 0.0)
    streams = {}
    for m in (tm, ref):
        ops = streams.setdefault(id(m), [])
        for i in range(6):                                               # 1. frames 0-5 integrated
            m.addFrame(tmod.INTEGRATED, poses[i], i); ops.append(("I", i, poses[i]))
        m.updateOptimizedTransform(poses, 6); m.generateUpdateLists()
        assert m.getNumActiveOperations() == 0
    moved = poses.copy()
    for i, dx in enumerate((0.4, 0.3, 0.2, 0.1)):                      # 2. frames 0-3 move (0 most): queued for re-integration in that order
        moved[i, 0, 3] += np.float32(dx)
    for m in (tm, ref):
        m.updateOptimizedTransform(moved, 6); m.generateUpdateLists()
    assert [tm.frameType(i) for i in range(6)] == [tmod.REINTEGRATION] * 4 + [tmod.INTEGRATED] * 2
    pops = {id(m): reconstruct_turn(m, streams[id(m)], max_fixes=1) for m in (tm, ref)}      # 3. one re-integration: frame 0
    assert pops[id(tm)][0][1][2] == 0
    gone = moved.copy(); gone[1:3] = -np.inf                              # 4. frames 1-2 lose their pose while queued
    for m in (tm, ref):
        m.updateOptimizedTransform(gone, 6)
        more = reconstruct_turn(m, streams[id(m)])                       # 5. pop until empty: 1 and 2 are skipped, 3 is re-integrated
        assert [(k, r[-1]) for k, r in more] == [("re", 3)], more
        pops[id(m)] += more
        assert m.getTopFromReIntegrateList() is None
    assert tm.frameType(1) == tm.frameType(2) == tmod.REINTEGRATION
    for m in (tm, ref):
        m.generateUpdateLists()                                          # 6. invalid now, and nothing queued to take them out
        assert m.getNumActiveOperations() == 0
    assert tm.frameType(1) == tm.frameType(2) == tmod.INVALID
    back = moved.copy(); back[1, 1, 3] += np.float32(0.05); back[2, 1, 3] -= np.float32(0.05)
    for m in (tm, ref):
        m.updateOptimizedTransform(back, 6); m.generateUpdateLists()      # 7. the poses come back
        assert m.getNumActiveOperations() == 2
        while reconstruct_turn(m, streams[id(m)]):                        # 8. drain
            pass
        m.generateUpdateLists()
        assert m.getNumActiveOperations() == 0
    same_state(tm, ref, 6)
    a, b = streams[id(tm)], streams[id(ref)]
    assert len(a) == len(b) and all(x[:2] == y[:2] and np.array_equal(x[2], y[2]) for x, y in zip(a, b))
    # what that op stream leaves in the model: frames 1 and 2 are never de-integrated and are integrated twice
    assert not [op for op in a if op[0] == "D" and op[1] in (1, 2)]
    for f in (1, 2):
        ins = [op[2] for op in a if op[0] == "I" and op[1] == f]
        assert len(ins) == 2 and np.array_equal(ins[0], poses[f]) and np.array_equal(ins[1], back[f])
    contributions = {}
    for k, f, T in a:
        lst = contributions.setdefault(f, [])
        if k == "I":
            lst.append(T)
        else:
            hit = [j for j, U in enumerate(lst) if np.array_equal(U, T)]
            assert hit, (f, "de-integration of a contribution that is not in the model")
            lst.pop(hit[0])
    final = tm.getOptimizedTransforms()
    for f in range(6):
        want = 2 if f in (1, 2) else 1
        assert len(contributions[f]) == want and np.array_equal(contributions[f][-1], final[f]), f


def test_reintegration_list_of_invalid_frames_only_returns_a_non_finite_pose():
    """Every frame left in the re-integration list has lost its pose: the pop still returns 1 (cpp:116-136), with the last skipped frame's index,
    its integrated pose as the old pose and newT = -inf; the frame loop then queues DEINTEGRATE(old) and INTEGRATE(-inf) for it."""
    rng = np.random.default_rng(8)
    poses = np.stack([rand_pose(rng) for _ in range(3)])
    tm, ref = TrajectoryManager(4, topNActive=4, minPoseDistSqrt=0.0), TrajectoryManagerOracle(4, 4, 0.0)
    moved = poses.copy(); moved[:, 2, 3] += np.float32([0.3, 0.2, 0.1])
    gone = np.full_like(poses, -np.inf)
    for m in (tm, ref):
        for i in range(3):
            m.addFrame(tmod.INTEGRATED, poses[i], i)
        m.updateOptimizedTransform(poses, 3); m.generateUpdateLists()
        m.updateOptimizedTransform(moved, 3); m.generateUpdateLists()
        assert m.getNumActiveOperations() == 3
        m.updateOptimizedTransform(gone, 3)
    a, b = tm.getTopFromReIntegrateList(), ref.getTopFromReIntegrateList()
    same_pop(a, b)
    old, new, idx = a
    assert idx == 2 and np.array_equal(old, poses[2]) and np.all(np.isneginf(new))
    assert tm.getNumActiveOperations() == 0 and tm.getTopFromReIntegrateList() is None
    ops = []
    tm.confirmIntegration(idx); ref.confirmIntegration(idx)
    same_state(tm, ref, 3)
    assert tm.frameType(2) == tmod.INTEGRATED and [tm.frameType(i) for i in (0, 1)] == [tmod.REINTEGRATION] * 2
    for m in (tm, ref):
        m.generateUpdateLists()                                          # the -inf frame 2 is INTEGRATED: de-integrated again at its old pose
        ops.append(m.getTopFromDeIntegrateList())
    same_pop(ops[0], ops[1])
    assert ops[0][1] == 2 and np.array_equal(ops[0][0], poses[2])

"""Generates tests/golden/trajectory_manager_reference.npz: what the REFERENCE's own TrajectoryManager (oracle/_ref/libref_trajectory_host.so, built
by oracle/build_ref.py from FL/TrajectoryManager.{h,cpp} + FL/PoseHelper.h with g++) returns on the sessions of
tests/test_trajectory_manager_reference.py.

    python oracle/build_ref.py && python scripts/make_golden_trajectory_manager.py < /dev/null
"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.test_trajectory_manager_reference import EXTRA_SESSIONS, SESSIONS, Recorder, run_extra_session, run_session         # noqa: E402


class Ref:
    def __init__(self):
        R = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libref_trajectory_host.so"))
        vp, u, f = C.c_void_p, C.c_uint, C.c_float
        R.refTrajCreate.argtypes = [u, u, f]; R.refTrajCreate.restype = vp
        R.refTrajAddFrame.argtypes = [vp, C.c_int, vp, u]; R.refTrajUpdateOptimizedTransform.argtypes = [vp, vp, u]; R.refTrajGenerateUpdateLists.argtypes = [vp]
        R.refTrajConfirmIntegration.argtypes = [vp, u]
        R.refTrajGetTopFromReIntegrateList.argtypes = [vp, vp, vp, vp]; R.refTrajGetTopFromIntegrateList.argtypes = [vp, vp, vp]; R.refTrajGetTopFromDeIntegrateList.argtypes = [vp, vp, vp]
        R.refTrajGetNumActiveOperations.argtypes = [vp]; R.refTrajGetNumActiveOperations.restype = u
        R.refTrajGetFrameType.argtypes = [vp, u]
        self.R, self.h = R, None

    def create(self, n, topN, minD): self.h = self.R.refTrajCreate(n, topN, minD)
    def addFrame(self, kind, T, idx): self.R.refTrajAddFrame(self.h, kind, np.ascontiguousarray(T, np.float32).ctypes.data, idx)
    def updateOptimizedTransform(self, traj, n): self.R.refTrajUpdateOptimizedTransform(self.h, np.ascontiguousarray(traj, np.float32).ctypes.data, n)
    def generateUpdateLists(self): self.R.refTrajGenerateUpdateLists(self.h)
    def confirmIntegration(self, i): self.R.refTrajConfirmIntegration(self.h, i)

    def _pop2(self, fn):
        o = np.zeros(16, np.float32); i = C.c_uint(0)
        return (o.reshape(4, 4), i.value) if fn(self.h, o.ctypes.data, C.addressof(i)) else None

    def getTopFromDeIntegrateList(self): return self._pop2(self.R.refTrajGetTopFromDeIntegrateList)
    def getTopFromIntegrateList(self): return self._pop2(self.R.refTrajGetTopFromIntegrateList)

    def getTopFromReIntegrateList(self):
        o, n, i = np.zeros(16, np.float32), np.zeros(16, np.float32), C.c_uint(0)
        return (o.reshape(4, 4), n.reshape(4, 4), i.value) if self.R.refTrajGetTopFromReIntegrateList(self.h, o.ctypes.data, n.ctypes.data, C.addressof(i)) else None

    def types(self, n): return [self.R.refTrajGetFrameType(self.h, i) for i in range(n)]
    def active(self): return self.R.refTrajGetNumActiveOperations(self.h)


def main():
    names = {"getTopFromDeIntegrateList": 0, "getTopFromIntegrateList": 1, "getTopFromReIntegrateList": 2, "types": 3, "active": 4}
    out = {}
    for s in list(range(SESSIONS)) + list(EXTRA_SESSIONS):
        rec = Recorder(Ref())
        if isinstance(s, int):
            run_session(s, [], rec)
        else:
            run_extra_session(s, [], rec)
        p = f"s{s}" if isinstance(s, int) else s
        kinds, found, idx, T, types = [], [], [], [], []
        for name, r in rec.log:
            kinds.append(names[name]); t = np.zeros((2, 16), np.float32)
            if name == "types":
                found.append(1); idx.append(len(r)); types += list(r)
            elif name == "active":
                found.append(1); idx.append(r)
            elif r is None:
                found.append(0); idx.append(0)
            else:
                found.append(1); idx.append(r[-1]); t[0] = r[0].reshape(16)
                if len(r) == 3:
                    t[1] = r[1].reshape(16)
            T.append(t)
        out[f"{p}_kind"], out[f"{p}_found"], out[f"{p}_idx"] = np.array(kinds, np.int8), np.array(found, np.int8), np.array(idx, np.int32)
        out[f"{p}_T"], out[f"{p}_types"] = np.stack(T), np.array(types, np.int8)
        print("session", s, len(kinds), "records")
    path = os.path.join(ROOT, "tests", "golden", "trajectory_manager_reference.npz")
    np.savez_compressed(path, **out)
    print("written", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

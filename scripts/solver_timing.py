"""CUDA-event timing of the solver at local / global sizes (development aid).

usage: solver_timing.py [POSE_DIR]  -- with POSE_DIR, the solved poses of every size are also saved there as
poses_N<N>.npz (rot, trans; poses_N11_dense.npz for the local solve), so that two builds can be compared bit for bit.

The N = 11 dense case is bench.py's local solve: sparse weight 1, dense depth weights 1, 2, colour 0, 2 x 100 iterations."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from bundlefusion_b200 import synth
from bundlefusion_b200.solver import CUDASolverBundling, DeviceCache
dev = torch.device("cuda:0")
for (N, deg, gn, pcg) in [("11d", 0, 2, 100), (11, 10, 2, 100), (32, 10, 3, 150), (64, 12, 3, 150), (128, 15, 3, 150), (500, 15, 3, 150), (2000, 15, 3, 150)]:
    dense = N == "11d"
    if dense:
        N = 11
        prob = synth.make_dense_ba_problem(11, stride=3, start=100, corr_per_pair=25, noise=0.002, seed=31)
        cache = DeviceCache(prob["caches"], prob["intrinsics"], dev)
        weights = dict(weightsDenseDepth=[1.0, 2.0], weightsDenseColor=[0.0, 0.0], cudaCache=cache)
    else:
        prob = synth.make_ba_problem(N, degree=deg, corr_per_pair=25, noise=0.002, seed=32, stride=10 if N <= 500 else 2)
        weights = {}
    corr = torch.from_numpy(prob["corr"].view(np.uint8).reshape(-1).copy()).to(dev)
    r0 = torch.from_numpy(prob["init_rot"]).to(dev); t0 = torch.from_numpy(prob["init_trans"]).to(dev)
    valid = torch.ones(N, dtype=torch.int32, device=dev)
    sol = CUDASolverBundling(N, max(len(prob["corr"]), 1000 * N), dev)
    rot, trans = r0.clone(), t0.clone()
    def run():
        rot.copy_(r0); trans.copy_(t0)
        sol.solve(corr, len(prob["corr"]), valid, N, gn, pcg, [1.0] * gn, d_rotationAnglesUnknowns=rot, d_translationUnknowns=trans, **weights)
    for _ in range(3): run()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(10): run()
    b.record(); torch.cuda.synchronize()
    st = sol.getStats()
    ms = a.elapsed_time(b) / 10
    if len(sys.argv) > 1:
        os.makedirs(sys.argv[1], exist_ok=True)
        np.savez(os.path.join(sys.argv[1], f"poses_N{N}{'_dense' if dense else ''}.npz"), rot=rot.cpu().numpy(), trans=trans.cpu().numpy())
    print(json.dumps({"N": N, "dense": dense, "C": len(prob["corr"]), "ms_per_solve": ms, "gn": st["gn"], "pcg": st["pcg"], "us_per_pcg_iter": ms * 1e3 / max(1, st["pcg"]), "pairs": st["pairs"]}))

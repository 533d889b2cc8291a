"""Where do the stencil's voxel probes fail?  Replays the bench's warm model, takes the in-frustum list of one bank frame and
classifies all E*512 probes with torch float32 math (diagnostic, approximate at decision boundaries)."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from bundlefusion_b200 import synth_gpu
from bundlefusion_b200.scene_rep import CUDASceneRepHashSDF, camera_params, default_hash_params
dev = torch.device("cuda:0")
W, H, B = 640, 480, 128
cam = camera_params(W, H)
hp = default_hash_params(num_buckets=4_000_000, num_sdf_blocks=4_000_000, voxel_size=0.01)
scene = CUDASceneRepHashSDF(hp, dev)
depth, color, poses = synth_gpu.make_frames([8 * i for i in range(B)], W, H, device=str(dev))
dl, cl = [depth[i] for i in range(B)], [color[i] for i in range(B)]
scene.runOps([(0, i, poses[i]) for i in range(B)], dl, cl, cam)
torch.cuda.synchronize()
for r in (5, 60, 127):
    scene.integrate(poses[r], dl[r], cl[r], cam)
    snap = scene.download()
    E = snap["compactified_count"]
    ent = torch.from_numpy(snap["compactified"][:E].astype(np.int32)).to(dev)           # (E, 8): pos xyz, offset, ptr
    bpos = ent[:, :3]
    l = torch.arange(512, device=dev)
    loc = torch.stack([l & 7, (l >> 3) & 7, l >> 6], 1)                                    # (512, 3)
    vox = (bpos[:, None, :] * 8 + loc[None]).float() * hp.m_virtualVoxelSize               # (E, 512, 3)
    Tinv = torch.from_numpy(np.linalg.inv(poses[r].astype(np.float64)).astype(np.float32)).to(dev)
    pc = vox @ Tinv[:3, :3].T + Tinv[:3, 3]
    sx = pc[..., 0] * cam.fx / pc[..., 2] + cam.mx; sy = pc[..., 1] * cam.fy / pc[..., 2] + cam.my
    px = (sx + 0.5).trunc().long(); py = (sy + 0.5).trunc().long()
    on = (px >= 0) & (px < W) & (py >= 0) & (py < H) & (sx + 0.5 >= 0) & (sy + 0.5 >= 0)
    d = torch.full_like(sx, float("-inf"))
    d[on] = dl[r].reshape(-1)[(py[on] * W + px[on])]
    valid = on & torch.isfinite(d) & (d < hp.m_maxIntegrationDistance)
    sdf = d - pc[..., 2]
    trunc = hp.m_truncation + hp.m_truncScale * d
    ok = valid & (sdf.abs() < trunc)
    n = ok.numel()
    blk_any = ok.any(1)
    out = {"frame": r, "E": E, "offscreen": float((~on).sum() / n), "invalid_or_far_depth": float((on & ~valid).sum() / n),
           "behind_surface": float((valid & ~ok & (sdf < 0)).sum() / n), "in_front_of_band": float((valid & ~ok & (sdf > 0)).sum() / n),
           "pass": float(ok.sum() / n), "blocks_with_no_passing_voxel": float((~blk_any).sum() / E),
           "pass_within_live_blocks": float(ok[blk_any].float().mean())}
    # 16-byte piece granularity: thread = 4 consecutive voxels
    q = ok.reshape(E, 128, 4).any(2)
    out["quads_touched"] = float(q.float().mean())
    print(json.dumps(out), flush=True)

"""The device mesh path on the GPU: CUDAMarchingCubesHashSDF.extractSoup against the oracle and the whole-mesh call (triangle multisets),
weld against the host clean-up (bfMeshMergeCloseVertices + bfMeshRemoveDuplicateFaces on soup.cpu(), bit for bit, and the PLY byte for
byte) on those soups and on a soup of over 2 M triangles, and the device_mesh option of fuse_recording and scan.py."""
import json

import numpy as np
import pytest

from bundlefusion_b200 import marching_cubes as mcm
from bundlefusion_b200.marching_cubes import CUDAMarchingCubesHashSDF, marching_cubes_params
from oracle import oracle as orc
from tests.test_marchingcubes_gpu import BUCKETS, build, soup_triangles
from tests.test_marchingcubes_reference_emulated import canon
from tests.test_trajectory_fusion_gpu import _face_count, recording  # noqa: F401  (recording: a module fixture)

pytestmark = pytest.mark.gpu
FUSE = dict(voxel_size=0.005, poses="recorded", hash_buckets=100003, sdf_blocks=90000)


@pytest.fixture(scope="module")
def scene_soup(cuda_device):
    gpu, cpu = build(cuda_device, n_frames=5)
    p = marching_cubes_params(BUCKETS, voxel_size=float(cpu.hp.m_virtualVoxelSize), max_num_triangles=1_000_000)
    want, found = orc.marchingcubes_extract(cpu, p)
    assert found == len(want) >= 75_000
    mc = CUDAMarchingCubesHashSDF(p, cuda_device)
    soup = mc.extractSoup(gpu)
    mc.close(); gpu.close()
    assert np.array_equal(canon(soup.cpu().numpy()), canon(want))
    return soup


@pytest.fixture(scope="module")
def fused_soup(cuda_device, recording):  # noqa: F811
    from bundlefusion_b200 import fuse
    path, _ = recording
    o = fuse.fuse_recording(path, None, device=cuda_device, **FUSE)
    scene = o["scene"]
    hp = scene.m_hashParams
    mc = CUDAMarchingCubesHashSDF(marching_cubes_params(int(hp.m_hashNumBuckets), float(hp.m_virtualVoxelSize), 5000), cuda_device)
    soup = mc.extractSoup(scene)
    info = mc.extractIsoSurfaceWhole(scene)
    whole, _ = soup_triangles(mc)
    mc.close(); scene.close()
    assert info["triangles_extracted"] == len(soup) > 20000 and info["parts"] > 1
    assert np.array_equal(canon(soup.cpu().numpy()), canon(whole))
    return soup


def host_mesh(tri, thresh=0.00001):
    pos = np.ascontiguousarray(tri[..., :3].reshape(-1, 3))
    col = np.concatenate([tri[..., 3:].reshape(-1, 3), np.ones((len(pos), 1), np.float32)], axis=1)
    p, c, f = mcm.merge_close_vertices(pos, col, np.arange(len(pos), dtype=np.uint32).reshape(-1, 3), thresh)
    return p, c, mcm.remove_duplicate_faces(f)


def check_weld(soup, tmp_path):
    mesh = mcm.weld(soup)
    wp, wc, wf = host_mesh(soup.cpu().numpy())
    gp, gc, gf = mesh.positions.cpu().numpy(), mesh.colors.cpu().numpy(), mesh.faces.cpu().numpy().view(np.uint32)
    assert gp.shape == wp.shape and gf.shape == wf.shape
    assert np.array_equal(gp.view(np.uint32), wp.view(np.uint32)) and np.array_equal(gc.view(np.uint32), wc.view(np.uint32)) and np.array_equal(gf, wf)
    info = mesh.info
    assert info["triangles_in"] == len(soup) and info["faces_out"] == len(wf) and info["vertices_out"] == len(wp)
    assert info["host_syncs"] == info["rounds"] + 1
    mesh.save_ply(str(tmp_path / "device.ply"))
    mcm.save_ply(str(tmp_path / "host.ply"), wp, wc, wf)
    assert open(str(tmp_path / "device.ply"), "rb").read() == open(str(tmp_path / "host.ply"), "rb").read()
    again = mcm.weld(soup)
    for a, b in ((mesh.positions, again.positions), (mesh.colors, again.colors), (mesh.faces, again.faces)):
        assert a.shape == b.shape and a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
    assert again.info == info
    return info


def test_weld_the_oracle_scene(scene_soup, tmp_path):
    info = check_weld(scene_soup, tmp_path)
    assert info["vertices_out"] < 3 * info["triangles_in"] // 4


def test_weld_the_fused_recording(fused_soup, tmp_path):
    check_weld(fused_soup, tmp_path)


def test_weld_over_two_million_triangles(scene_soup, tmp_path):
    import torch
    base = scene_soup
    copies = 2_000_000 // len(base) + 1
    g = torch.Generator(device=base.device).manual_seed(7)
    tiles = []
    for k in range(copies):
        t = base.clone()
        t[..., 0] += 0.5 * (k % 8) - 1.0
        t[..., 1] += 0.5 * (k // 8) - 1.0
        if k % 2:                                                                      # jitter around the merge threshold
            t[..., :3] += (torch.rand(t[..., :3].shape, generator=g, device=base.device) - 0.5) * 2.4e-5
        tiles.append(t)
    soup = torch.cat(tiles).contiguous()
    assert len(soup) > 2_000_000
    check_weld(soup, tmp_path)


def test_weld_refuses_a_non_finite_position(cuda_device):
    import torch
    soup = torch.zeros((4, 3, 6), dtype=torch.float32, device=cuda_device)
    soup[2, 1, 0] = float("nan")
    with pytest.raises(RuntimeError, match="not finite"):
        mcm.weld(soup)
    assert mcm.weld(soup[:2].contiguous()).info["vertices_out"] == 1


def test_fuse_recording_device_mesh(cuda_device, recording, tmp_path):  # noqa: F811
    from bundlefusion_b200 import fuse
    path, _ = recording
    whole = fuse.fuse_recording(path, str(tmp_path / "whole.ply"), device=cuda_device, whole_mesh=True, **FUSE)
    whole["scene"].close()
    dm = fuse.fuse_recording(path, str(tmp_path / "device.ply"), device=cuda_device, device_mesh=True, **FUSE)
    dm["scene"].close()
    assert dm["triangles_found"] == dm["triangles"] == whole["triangles_found"] > 20000 and dm["triangles_dropped"] == 0
    assert _face_count(dm["mesh_path"]) == dm["mesh"]["faces_out"] > 0
    assert dm["mesh"]["peak_device_bytes"] > 72 * dm["triangles"]
    with pytest.raises(ValueError):
        fuse.fuse_recording(path, str(tmp_path / "x.ply"), device=cuda_device, whole_mesh=True, device_mesh=True, **FUSE)


def test_scan_device_mesh(cuda_device, recording, tmp_path, capsys):  # noqa: F811
    from bundlefusion_b200 import scan
    path, _ = recording
    sizes = ["--hash-buckets", "100003", "--sdf-blocks", "90000", "--device", str(cuda_device), "--poses", "recorded", "--mesh-voxel-size", "0.005"]
    whole, device = str(tmp_path / "whole.ply"), str(tmp_path / "device.ply")
    assert scan.main([path, whole, "--whole-mesh"] + sizes) == 0
    w = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert scan.main([path, device, "--device-mesh"] + sizes) == 0
    d = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert d["triangles_found"] == d["triangles"] == w["triangles_found"] > 0 and d["triangles_dropped"] == 0
    assert _face_count(device) == d["mesh"]["faces_out"] > 0 and d["mesh"]["host_syncs"] == d["mesh"]["rounds"] + 1
    with pytest.raises(SystemExit):
        scan.main([path, device, "--device-mesh", "--whole-mesh"] + sizes)

"""The whole mesh on the GPU: the count pass against oracle/marchingcubes_oracle.c, the whole-mesh call of CUDAMarchingCubesHashSDF in several
parts against the oracle's soup and one extraction into an ample buffer (triangle multisets, bit for bit), the buffer rule, the loss the fixed
buffer now reports, and the options of fuse_recording and scan.py that mesh through the whole-mesh call.  The product's model is fused by the
library's bit-exact TSDF kernels, the oracle's by its own: hash slots differ, voxel values do not (so totals are compared, not chunks)."""
import json

import numpy as np
import pytest

from bundlefusion_b200.marching_cubes import CUDAMarchingCubesHashSDF, marching_cubes_params, num_chunks
from oracle import oracle as orc
from tests.test_marchingcubes_gpu import BUCKETS, build, soup_triangles
from tests.test_marchingcubes_reference_emulated import canon
from tests.test_trajectory_fusion_gpu import N_SENS, SKIP, _face_count, recording  # noqa: F401  (recording: a module fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def scenes(cuda_device):
    gpu, cpu = build(cuda_device, n_frames=5)
    p = marching_cubes_params(BUCKETS, voxel_size=float(cpu.hp.m_virtualVoxelSize), max_num_triangles=1_000_000)
    want, found = orc.marchingcubes_extract(cpu, p)
    assert found == len(want) >= 75_000
    yield gpu, cpu, want
    gpu.close()


def mesher(dev, cpu, cap):
    return CUDAMarchingCubesHashSDF(marching_cubes_params(BUCKETS, voxel_size=float(cpu.hp.m_virtualVoxelSize), max_num_triangles=cap), dev)


def test_count_equals_the_oracle(cuda_device, scenes):
    gpu, cpu, want = scenes
    mc = mesher(cuda_device, cpu, 5000)
    total, chunks = mc.count(gpu)
    assert total == len(want) and len(chunks) == num_chunks(BUCKETS) and int(chunks.astype(np.int64).sum()) == total
    again, chunks2 = mc.count(gpu)
    assert again == total and np.array_equal(chunks, chunks2)                        # plain stores of CTA-local sums: the same counts every time
    # with a box: the oracle's box count
    lo, hi = want[..., :3].reshape(-1, 3).min(0), want[..., :3].reshape(-1, 3).max(0)
    box = ((float(lo[0]) - 1.0, float(lo[1]) - 1.0, float(lo[2]) - 1.0), (float(0.5 * (lo[0] + hi[0])), float(hi[1]) + 1.0, float(hi[2]) + 1.0))
    pb = marching_cubes_params(BUCKETS, voxel_size=float(cpu.hp.m_virtualVoxelSize), max_num_triangles=1_000_000)
    pb.m_boxEnabled = 1
    for k in range(3):
        pb.m_minCorner[k], pb.m_maxCorner[k] = box[0][k], box[1][k]
    _, foundb = orc.marchingcubes_extract(cpu, pb)
    assert 0 < mc.count(gpu, box[0], box[1], True)[0] == foundb < total
    mc.close()


def test_whole_mesh_in_parts_equals_the_oracle_and_an_ample_buffer(cuda_device, scenes):
    gpu, cpu, want = scenes
    ample = mesher(cuda_device, cpu, 1_000_000)
    assert ample.extractIsoSurface(gpu) == 3 * len(want)
    assert ample.lastExtraction() == (len(want), len(want))
    one, _ = soup_triangles(ample)
    ample.close()
    mc = mesher(cuda_device, cpu, 5000)
    _, chunks = mc.count(gpu)
    assert chunks.max() <= 5000
    info = mc.extractIsoSurfaceWhole(gpu)
    assert info["triangles_counted"] == info["triangles_extracted"] == len(want)
    assert info["parts"] > 1 and info["host_syncs"] == 1 + info["parts"] and info["largest_part"] <= 5000
    assert info["buffer_triangles"] == 5000 and not info["buffer_enlarged"]
    got, col = soup_triangles(mc)
    assert len(got) == len(want) and np.array_equal(canon(got), canon(want)) and np.array_equal(canon(got), canon(one)) and np.all(col[:, 3] == 1.0)
    assert mc.lastExtraction() == (len(want), len(want))
    # the fixed path with the same small buffer: the loss is on record -- found = the oracle's count, kept = the capacity
    mc.clearMeshBuffer()
    assert mc.extractIsoSurface(gpu) == 3 * 5000
    assert mc.lastExtraction() == (len(want), 5000)
    mc.close()


def test_a_buffer_below_the_largest_chunk_is_enlarged(cuda_device, scenes):
    gpu, cpu, want = scenes
    mc = mesher(cuda_device, cpu, 64)
    _, chunks = mc.count(gpu)
    assert chunks.max() > 64
    info = mc.extractIsoSurfaceWhole(gpu)
    assert info["buffer_enlarged"] and info["buffer_triangles"] == int(chunks.max()) and info["triangles_extracted"] == len(want)
    assert info["parts"] > 1 and info["largest_part"] <= int(chunks.max())
    assert np.array_equal(canon(soup_triangles(mc)[0]), canon(want))
    # the enlarged buffer stays: a second call needs no enlargement
    mc.clearMeshBuffer()
    again = mc.extractIsoSurfaceWhole(gpu)
    assert not again["buffer_enlarged"] and again["buffer_triangles"] == info["buffer_triangles"] and again["parts"] == info["parts"]
    mc.close()


def test_fuse_recording_whole_mesh_drops_nothing(cuda_device, recording, tmp_path):  # noqa: F811
    from bundlefusion_b200 import fuse
    path, _ = recording
    kw = dict(voxel_size=0.005, poses="recorded", hash_buckets=100003, sdf_blocks=90000, device=cuda_device)
    ample = fuse.fuse_recording(path, str(tmp_path / "ample.ply"), **kw)
    ample["scene"].close()
    assert ample["triangles"] == ample["triangles_found"] > 20000 and ample["triangles_dropped"] == 0 and "mesh" not in ample
    small = ample["triangles"] // 10
    whole = fuse.fuse_recording(path, str(tmp_path / "whole.ply"), max_num_triangles=small, whole_mesh=True, **kw)
    whole["scene"].close()
    assert whole["triangles"] == whole["triangles_found"] == ample["triangles"] and whole["triangles_dropped"] == 0
    assert whole["mesh"]["parts"] >= 10 and whole["mesh"]["triangles_counted"] == ample["triangles"]
    fixed = fuse.fuse_recording(path, str(tmp_path / "fixed.ply"), max_num_triangles=small, **kw)
    fixed["scene"].close()
    assert fixed["triangles"] == small and fixed["triangles_found"] == ample["triangles"] and fixed["triangles_dropped"] == ample["triangles"] - small


def test_scan_whole_mesh(cuda_device, recording, tmp_path, capsys):  # noqa: F811
    from bundlefusion_b200 import scan
    path, _ = recording
    sizes = ["--hash-buckets", "100003", "--sdf-blocks", "90000", "--device", str(cuda_device)]
    ample, whole = str(tmp_path / "ample.ply"), str(tmp_path / "whole.ply")
    assert scan.main([path, ample, "--poses", "recorded", "--mesh-voxel-size", "0.005"] + sizes) == 0
    a = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert a["triangles_dropped"] == 0 and a["triangles_found"] == a["triangles"] > 0 and "mesh" not in a
    assert scan.main([path, whole, "--poses", "recorded", "--mesh-voxel-size", "0.005", "--whole-mesh"] + sizes) == 0
    w = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert w["triangles_dropped"] == 0 and w["triangles_found"] == w["triangles"] == a["triangles"]
    assert w["mesh"]["triangles_extracted"] == a["triangles"] and w["mesh"]["parts"] == 1
    assert _face_count(whole) == _face_count(ample)
    # the online model of the loop, meshed whole
    online = str(tmp_path / "online.ply")
    assert scan.main([path, online, "--solve-frames-before-exit", "3", "--whole-mesh"] + sizes) == 0
    o = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert o["triangles_dropped"] == 0 and o["triangles"] == o["triangles_found"] == o["mesh"]["triangles_counted"] > 0 and o["mesh_path"] == online
    assert _face_count(online) > 0

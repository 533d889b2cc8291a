import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device")


# Collection order of the GPU tests (the driver runs `pytest -x`): the voxel-hash tests first, then the other rows against the oracle,
# then the comparisons with the recorded outputs of the reference's own CUDA build (tests/reference_cuda.py), last the kernels with the
# shortest hardware history.  One failure must hide as little verified work as possible.
_ORDER = {"test_tsdf_gpu.py": 0, "test_tsdf_vs_reference_gpu.py": 1, "test_solver_vs_reference_gpu.py": 5,
          "test_zz_sift_prune_gpu.py": 6, "test_zz_sift_detect_gpu.py": 7, "test_marchingcubes_gpu.py": 8, "test_sens_frame_loop_gpu.py": 9, "test_zz_scan_to_mesh_gpu.py": 10}          # 8 - 10: written after the round's last GPU minute -- first hardware run is the driver's


def pytest_collection_modifyitems(config, items):
    items.sort(key=lambda it: _ORDER.get(os.path.basename(str(it.fspath)), 3))          # stable: the order inside each group is unchanged


@pytest.fixture(scope="session")
def oracle_lib():
    from oracle import oracle
    oracle.build()
    return oracle.lib()


@pytest.fixture(scope="session")
def cuda_device():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")

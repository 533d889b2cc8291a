"""search_sharded on 2 and 4 ranks (NCCL): scripts/keyframe_search_timing.py --check under torchrun; every rank's gathered list must equal the
single-GPU search byte for byte.  Skipped below two GPUs."""
import os
import subprocess
import sys

import pytest

from tests._cudart import device_count

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_search_equals_single_gpu(world):
    if device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc_per_node={world}",
                        os.path.join(ROOT, "scripts", "keyframe_search_timing.py"), "--frames", "120", "--sizes", "640x480", "--repeats", "1", "--check"],
                       cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert '"gathered_equals_single_gpu": true' in r.stdout

"""Outputs of the reference's own CUDA build (oracle/_ref, see oracle/build_ref.py) for the parity tests, stored under tests/golden/ so that
the tests need neither the reference's sources nor a build of them.  With BF_RECORD_REFERENCE_CUDA=<directory> set (and oracle/_ref built)
the tests run the reference live, check against what it computed, and write the recorded outputs to that directory:
scripts/make_golden_reference_cuda.sh."""
import hashlib
import os
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
RECORD_DIR = os.environ.get("BF_RECORD_REFERENCE_CUDA")


class Recorded:
    def __init__(self, name):
        self.name = name
        self.data = None

    def get(self, key, live):
        """the arrays stored under `key`; when recording, live() computes them with the reference's build first"""
        if self.data is None:
            self.data = {} if RECORD_DIR else dict(np.load(os.path.join(HERE, "golden", self.name)))
        if RECORD_DIR:
            for k, v in live().items():
                self.data[f"{key}/{k}"] = np.asarray(v)
        prefix = key + "/"
        out = {k[len(prefix):]: v for k, v in self.data.items() if k.startswith(prefix)}
        assert out, f"{key} is not in tests/golden/{self.name}"
        return out

    def save(self):
        if RECORD_DIR and self.data:
            os.makedirs(RECORD_DIR, exist_ok=True)
            np.savez_compressed(os.path.join(RECORD_DIR, self.name), **self.data)


def saving_fixture(rec):
    """module fixture: writes what the module recorded once its tests have run"""
    @pytest.fixture(scope="module", autouse=True)
    def _save():
        yield
        rec.save()
    return _save


# Voxel states: the block set and a CRC-32 of every block's voxel words are stored whole (bit-exact comparisons), the voxel words themselves at a
# fixed, seeded set of positions of the canonical order (oracle.canonical_blocks) -- for the tolerance statistics; most among the voxels the
# reference touched, a quarter of that number elsewhere.
VOXEL_SAMPLE = 12000


def sample_state(snap):
    from oracle import oracle as orc
    blocks, vox = orc.canonical_blocks(snap)
    flat = vox.reshape(-1, vox.shape[-1])
    w = flat[:, 1].view(np.float32)
    rng = np.random.default_rng(7)
    touched, rest = np.flatnonzero(w > 0), np.flatnonzero(w == 0)
    idx = np.sort(np.r_[rng.choice(touched, min(VOXEL_SAMPLE, touched.size), replace=False),
                        rng.choice(rest, min(VOXEL_SAMPLE // 4, rest.size), replace=False)]).astype(np.int64)
    return {"blocks": blocks, "idx": idx, "vox": flat[idx], "crc": block_crcs(vox)}


def block_crcs(vox):
    """CRC-32 of every block's voxel words (canonical order): the whole state, for the bit-exact comparison"""
    return np.array([zlib.crc32(np.ascontiguousarray(b).tobytes()) for b in vox], np.uint32)


def digest(a):
    """SHA-256 of an array's shape, dtype and bytes: large golden outputs that are only ever compared for equality are stored as this"""
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(f"{a.shape}{a.dtype.str}".encode())
    h.update(a.tobytes())
    return np.frombuffer(h.digest(), np.uint8)

"""Sizing a fusion's voxel hash, on the CPU: the device key set and bucket-load kernels of bundlefusion_b200/csrc/tsdf_keys.cuh compiled by g++
against tests/cuda_emu (one OS thread per CUDA thread, atomics under a lock) and checked against a numpy statement of the hash's bucket
function; the refusals of bfTsdfCountBlocks / bfTsdfBlockKeyLoad / bfTsdfBlockKeyMerge in a process that sees no CUDA device; and
fuse.fit_hash_params' bucket sequence and byte accounting on synthetic counts."""
import ctypes as C

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from bundlefusion_b200 import fuse
from oracle import oracle as orc
from tests.cuda_emu import build_emulated, run_without_device

LIM = 1 << 20

_GLUE = r'''
extern "C" void emu_bucket_load(const unsigned long long* keys, unsigned n, unsigned numBuckets, unsigned* load, unsigned* out, unsigned grid, unsigned block) {
    EMU_LAUNCH(bf::bucket_load_kernel, grid, block, keys, n, numBuckets, load, out);
}
extern "C" void emu_merge(unsigned long long* keys, unsigned capacity, unsigned* ctrs, const unsigned long long* src, unsigned n, unsigned grid, unsigned block) {
    EMU_LAUNCH(bf::keyset_merge_kernel, grid, block, keys, capacity - 1u, ctrs, src, n);
}
extern "C" unsigned long long emu_pack(int x, int y, int z) { return bf::pack_block_key(bf::I3{ x, y, z }); }
'''


@pytest.fixture(scope="module")
def emu():
    L = build_emulated("tsdf_keys.cuh", 0, glue=_GLUE)
    vp, u = C.c_void_p, C.c_uint
    L.emu_bucket_load.argtypes = [vp, u, u, vp, vp, u, u]
    L.emu_merge.argtypes = [vp, u, vp, vp, u, u, u]
    L.emu_pack.argtypes = [C.c_int] * 3
    L.emu_pack.restype = C.c_ulonglong
    return L


def pack(pos):
    p = np.asarray(pos, np.int64).reshape(-1, 3) + LIM
    return (np.uint64(1) << np.uint64(63)) | (p[:, 0].astype(np.uint64) << np.uint64(42)) | (p[:, 1].astype(np.uint64) << np.uint64(21)) | p[:, 2].astype(np.uint64)


def expected_load(pos, buckets):
    load = np.bincount(orc.block_hash(pos, buckets).astype(np.int64), minlength=buckets)
    return load, int(load.max()) if len(pos) else 0, int(np.maximum(load - capi.BF_HASH_BUCKET_SIZE, 0).sum())


def _run_load(L, keys, buckets, grid=3, block=64):
    k = np.ascontiguousarray(keys, np.uint64)
    load, out = np.zeros(buckets, np.uint32), np.zeros(3, np.uint32)
    L.emu_bucket_load(k.ctypes.data, len(k), buckets, load.ctypes.data, out.ctypes.data, grid, block)
    return load, out


def _random_positions(rng, n, spread):
    return np.unique(rng.integers(-spread, spread, size=(n, 3)), axis=0)


def test_pack_matches_the_numpy_statement(emu):
    for p in [(0, 0, 0), (-1, 2, -3), (LIM - 1, -LIM, 5), (-LIM, -LIM, -LIM)]:
        assert emu.emu_pack(*p) == int(pack(p)[0])


@pytest.mark.parametrize("kind", ["random", "clustered"])
@pytest.mark.parametrize("buckets", [1, 2, 3, 7, 61, 1021, 40009])
def test_bucket_load_equals_numpy(emu, kind, buckets):
    rng = np.random.default_rng(buckets)
    if kind == "random":
        pos = _random_positions(rng, 3000, 1 << 19)
    else:                                                  # a surface band: the block layout a fusion produces
        g = np.stack(np.meshgrid(np.arange(-20, 20), np.arange(-15, 15), np.arange(0, 3), indexing="ij"), -1).reshape(-1, 3)
        pos = np.unique(g + rng.integers(-1, 2, size=g.shape), axis=0)
    keys = np.zeros(2 * len(pos) + 7, np.uint64)           # the keys scattered among empty slots, as in a key set
    keys[rng.permutation(len(keys))[:len(pos)]] = pack(pos)
    load, out = _run_load(emu, keys, buckets)
    want, mx, over = expected_load(pos, buckets)
    np.testing.assert_array_equal(load, want)
    assert (int(out[0]), int(out[1]), int(out[2])) == (len(pos), mx, over)


def test_bucket_load_at_four_and_five_keys_per_bucket(emu):
    """loads of exactly BF_HASH_BUCKET_SIZE (no overflow) and one more (overflow 1 per such bucket), found by the numpy hash itself"""
    B = 101
    rng = np.random.default_rng(7)
    cand = _random_positions(rng, 20000, 1 << 12)
    h = orc.block_hash(cand, B)
    by = [cand[h == b] for b in range(B)]
    four = np.concatenate([by[b][:4] for b in range(0, 40)])
    five = np.concatenate([by[b][:5] for b in range(40, 43)])
    for pos, mx, over in ((four, 4, 0), (np.concatenate([four, five]), 5, 3)):
        _, out = _run_load(emu, pack(pos), B)
        assert (int(out[0]), int(out[1]), int(out[2])) == (len(pos), mx, over)
        assert expected_load(pos, B)[1:] == (mx, over)


def test_key_set_stores_each_key_once(emu):
    rng = np.random.default_rng(3)
    pos = _random_positions(rng, 500, 1000)
    src = np.concatenate([pack(pos), pack(pos[:200]), np.zeros(50, np.uint64), pack(pos[::-1])])
    src = src[rng.permutation(len(src))]
    cap = 1024
    keys, ctrs = np.zeros(cap, np.uint64), np.zeros(3, np.uint32)
    emu.emu_merge(keys.ctypes.data, cap, ctrs.ctypes.data, src.ctypes.data, len(src), 4, 32)
    assert list(ctrs) == [len(pos), 0, 0]
    np.testing.assert_array_equal(np.sort(keys[keys != 0]), np.sort(pack(pos)))
    # a second pass over the same keys stores nothing new
    emu.emu_merge(keys.ctypes.data, cap, ctrs.ctypes.data, src.ctypes.data, len(src), 2, 16)
    assert list(ctrs) == [len(pos), 0, 0]


def test_full_key_set_refuses_without_writing_past_its_capacity(emu):
    rng = np.random.default_rng(5)
    pos = _random_positions(rng, 40, 1000)[:37]
    cap, guard = 16, 8
    buf = np.full(cap + 2 * guard, 0xA5A5A5A5A5A5A5A5, np.uint64)
    buf[guard:guard + cap] = 0
    ctrs = np.zeros(3, np.uint32)
    src = np.concatenate([pack(pos), pack(pos)])           # every key twice
    emu.emu_merge(buf[guard:].ctypes.data, cap, ctrs.ctypes.data, src.ctypes.data, len(src), 3, 8)
    stored = buf[guard:guard + cap]
    assert ctrs[0] == cap and (stored != 0).all() and len(np.unique(stored)) == cap
    assert set(stored.tolist()) <= set(pack(pos).tolist())
    # each of the 37 - 16 keys that found no slot is refused both times it came
    assert ctrs[1] == 2 * (len(pos) - cap) and ctrs[2] == 0
    assert (buf[:guard] == 0xA5A5A5A5A5A5A5A5).all() and (buf[guard + cap:] == 0xA5A5A5A5A5A5A5A5).all()


_REFUSALS = r'''
import ctypes as C, json, sys
sys.path.insert(0, sys.argv[1])
from bundlefusion_b200 import _capi as capi
from bundlefusion_b200.scene_rep import camera_params, default_hash_params
L = capi.lib()
hp, cam = default_hash_params(num_buckets=101, num_sdf_blocks=64), camera_params(64, 48)
def ks(keys=0x1000, ctrs=0x2000, cap=1024):
    s = capi.BFBlockKeySet(); s.d_keys, s.d_counters, s.capacity = keys, ctrs, cap; return s
fake = (C.c_void_p * 4)(0x1000, 0x2000, None, 0x4000)          # never dereferenced: every case is refused first
frames = (C.c_int32 * 17)(*([0, 1] + [3] * 15))
poses = (C.c_float * (17 * 16))()
vp = lambda x: C.cast(x, C.c_void_p)
good = ks()
N = lambda s, fr, po, n, d, h=hp, c=cam: L.bfTsdfCountBlocks(None if s is None else C.byref(s), None if h is None else C.byref(h), None if c is None else C.byref(c), fr, po, n, d)
Ld = lambda s, b, load=0x3000, out=0x4000: L.bfTsdfBlockKeyLoad(None if s is None else C.byref(s), b, load, out)
M = lambda d, s: L.bfTsdfBlockKeyMerge(None if d is None else C.byref(d), None if s is None else C.byref(s))
out = {
    "count_n0": N(good, vp(frames), vp(poses), 0, vp(fake)),
    "count_n17": N(good, vp(frames), vp(poses), 17, vp(fake)),
    "count_null_set": N(None, vp(frames), vp(poses), 2, vp(fake)),
    "count_null_keys": N(ks(keys=0), vp(frames), vp(poses), 2, vp(fake)),
    "count_null_counters": N(ks(ctrs=0), vp(frames), vp(poses), 2, vp(fake)),
    "count_capacity0": N(ks(cap=0), vp(frames), vp(poses), 2, vp(fake)),
    "count_capacity_not_pow2": N(ks(cap=1000), vp(frames), vp(poses), 2, vp(fake)),
    "count_capacity_2_32m": N(ks(cap=(1 << 32) - (1 << 30)), vp(frames), vp(poses), 2, vp(fake)),
    "count_null_frames": N(good, None, vp(poses), 2, vp(fake)),
    "count_null_poses": N(good, vp(frames), None, 2, vp(fake)),
    "count_null_depth_array": N(good, vp(frames), vp(poses), 2, None),
    "count_null_hash_params": N(good, vp(frames), vp(poses), 2, vp(fake), h=None),
    "count_null_camera": N(good, vp(frames), vp(poses), 2, vp(fake), c=None),
    "count_null_depth_ptr": N(good, vp((C.c_int32 * 3)(0, 2, 1)), vp(poses), 3, vp(fake)),
    "count_negative_frame": N(good, vp((C.c_int32 * 2)(0, -1)), vp(poses), 2, vp(fake)),
    "load_null_set": Ld(None, 7),
    "load_null_keys": Ld(ks(keys=0), 7),
    "load_capacity_not_pow2": Ld(ks(cap=3), 7),
    "load_zero_buckets": Ld(good, 0),
    "load_null_scratch": Ld(good, 7, load=0),
    "load_null_out": Ld(good, 7, out=0),
    "merge_null_dst": M(None, good),
    "merge_null_src": M(good, None),
    "merge_bad_dst": M(ks(cap=6), good),
    "merge_bad_src": M(good, ks(keys=0x5000, cap=0)),
    "merge_into_itself": M(good, ks()),
}
print(json.dumps(out))
'''


def test_count_and_load_refusals_enqueue_nothing():
    """each malformed call returns cudaErrorInvalidValue (1) before any CUDA call: run in a child process that sees no CUDA device, where a call
    that went on to the runtime would fail with another code (or touch the fake pointers)"""
    out = run_without_device(_REFUSALS)
    assert out == {k: 1 for k in out}, out


# ---- fit_hash_params on synthetic counts -----------------------------------------------------------------------------------------------------
class _Counter:
    """what fit_hash_params reads of a BlockCounter, on host positions (the bucket loads from the numpy hash)"""

    def __init__(self, pos, voxel=0.004):
        from bundlefusion_b200.scene_rep import default_hash_params
        self.pos, self.hash_params, self.calls = pos, default_hash_params(voxel_size=voxel), []

    @property
    def count(self):
        return len(self.pos)

    def bucket_load(self, b):
        self.calls.append(b)
        _, mx, over = expected_load(self.pos, b)
        return {"keys": len(self.pos), "max_load": mx, "over": over}


def test_table_bytes_follow_the_scene_allocation():
    # CUDASceneRepHashSDF: d_hash and d_hashCompactified 8 int32 per entry, d_hashDecision and d_hashDecisionPrefix one int32 per entry, one mutex
    # int32 per bucket; 4 entries per bucket
    assert fuse.TABLE_BYTES_PER_BUCKET == 4 * (32 + 32 + 4 + 4) + 4 == 292
    assert fuse.table_bytes(1000003) == 292 * 1000003


def test_bucket_candidates_are_odd_increasing_and_geometric():
    c = list(fuse.bucket_candidates(1000, 10 ** 6))
    assert c[0] == 1001 and all(b & 1 for b in c) and all(a < b for a, b in zip(c, c[1:]))
    assert c == sorted({int(1000 * 1.25 ** k) | 1 for k in range(80) if int(1000 * 1.25 ** k) | 1 <= 10 ** 6})
    assert list(fuse.bucket_candidates(0, 10))[:3] == [1, 3, 5]


def test_fit_picks_the_first_candidate_without_overflow():
    rng = np.random.default_rng(11)
    pos = _random_positions(rng, 5000, 300)
    ctr = _Counter(pos)
    base = capi.BFHashParams()
    base.m_truncation, base.m_virtualVoxelSize = 0.06, 0.01
    hp, rep = fuse.fit_hash_params(base, 0.004, ctr)
    want = next(b for b in fuse.bucket_candidates(len(pos)) if expected_load(pos, b)[2] == 0)
    assert hp.m_hashNumBuckets == rep["buckets"] == want and ctr.calls[-1] == want
    assert ctr.calls == [b for b in fuse.bucket_candidates(len(pos)) if b <= want]
    assert hp.m_numSDFBlocks == rep["sdf_blocks"] == rep["blocks_counted"] == len(pos)
    assert rep["predicted_overflow"] == 0 and rep["max_load"] <= 4 and rep["table_bytes"] == 292 * want
    assert np.float32(hp.m_virtualVoxelSize) == np.float32(0.004) and np.float32(hp.m_truncation) == np.float32(0.06)
    assert rep["candidates_tried"] == len(ctr.calls)


def test_fit_stops_at_the_table_cap_and_predicts_the_overflow():
    rng = np.random.default_rng(12)
    pos = _random_positions(rng, 4000, 300)
    ctr = _Counter(pos)
    cap_bytes = fuse.table_bytes(len(pos) // 8) + 100       # a quarter of the buckets the keys need at the very least
    hp, rep = fuse.fit_hash_params(capi.BFHashParams(), 0.004, ctr, max_table_bytes=cap_bytes)
    b = cap_bytes // 292
    b = b if b & 1 else b - 1
    assert hp.m_hashNumBuckets == rep["buckets"] == b and rep["table_bytes"] <= cap_bytes
    assert rep["predicted_overflow"] == expected_load(pos, b)[2] > 0
    assert ctr.calls == [b]                                   # no candidate of the sequence fits under the cap
    with pytest.raises(ValueError):
        fuse.fit_hash_params(capi.BFHashParams(), 0.004, ctr, max_table_bytes=291)


def test_fit_without_a_cap_stops_at_the_default_buckets_per_block():
    """blocks of a surface-like lattice whose 32-bit hash values coincide five or more at a time: no bucket count separates them, the default
    cap ends the search and the overflow that remains is reported"""
    g = np.stack(np.meshgrid(np.arange(-300, 300), np.arange(-300, 300), np.arange(-2, 2), indexing="ij"), -1).reshape(-1, 3)
    _, inv, cnt = np.unique(orc.block_hash(g), return_inverse=True, return_counts=True)
    pos = g[cnt[inv] >= 5]
    floor = int(np.maximum(cnt - 4, 0).sum())
    assert floor > 0 and len(pos) > 0
    ctr = _Counter(pos)
    hp, rep = fuse.fit_hash_params(capi.BFHashParams(), 0.004, ctr)
    cap = fuse.DEFAULT_BUCKETS_PER_BLOCK * len(pos) + 1
    assert hp.m_hashNumBuckets == rep["buckets"] == cap and rep["table_bytes"] == fuse.table_bytes(cap)
    assert rep["predicted_overflow"] == expected_load(pos, cap)[2] >= floor
    assert ctr.calls == list(fuse.bucket_candidates(len(pos), cap)) + [cap]


def test_fit_refuses_a_counter_of_another_voxel_size():
    with pytest.raises(ValueError):
        fuse.fit_hash_params(capi.BFHashParams(), 0.005, _Counter(np.zeros((1, 3), np.int64), voxel=0.004))


def test_fuse_recording_refuses_explicit_sizes_with_fit_hash():
    for kw in ({"hash_buckets": 1001}, {"sdf_blocks": 1000}):
        with pytest.raises(ValueError):
            fuse.fuse_recording("never-opened.sens", None, 0.004, fit_hash=True, **kw)

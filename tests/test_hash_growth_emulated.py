"""Growing the voxel hash, on the CPU: the rehash kernels of bundlefusion_b200/csrc/tsdf_hash.cuh compiled by g++ against tests/cuda_emu (one
OS thread per CUDA thread, atomics under a lock), with the source table built by the same header's alloc_block / delete_entry.  Random and
clustered blocks in a table small enough for overflow lists, freed holes, a last list that holds a freed block; rehashed into a larger, a
same-size and a smaller table.  Also the refusals of bfTsdfRehash in a process that sees no CUDA device, and the frame loop's growth-size rule."""
import ctypes as C

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from bundlefusion_b200.scene_rep import default_hash_params
from oracle import oracle as orc
from tests.cuda_emu import build_emulated, run_without_device

FREE, LIST_LIMIT = capi.BF_FREE_ENTRY, 7
# the counter layout of csrc/tsdf_shared.cuh (pinned by test_counter_layout_is_the_librarys)
CTR_HIGH_WATER, CTR_E, CTR_FREED, CTR_HEAP_FAIL, CTR_DROPPED, CTR_SET1, SET_COUNT, CTR_NUM = 0, 3, 8, 9, 10, 24, 0, 32
VEC = 512 * 3                                              # 32-bit words per voxel block

_GLUE = r'''
using namespace bf;
static void insert_kernel(BFHashDataStruct hd, BFHashParams hp, int4* slotInfo, unsigned* ctrs, const int* pos, unsigned n) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) alloc_block(hd, hp, slotInfo, ctrs, I3{ pos[3 * i], pos[3 * i + 1], pos[3 * i + 2] });
}
static void delete_kernel(BFHashDataStruct hd, BFHashParams hp, int4* slotInfo, const int* pos, unsigned n) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) delete_entry(hd, hp, slotInfo, I3{ pos[3 * i], pos[3 * i + 1], pos[3 * i + 2] });
}
extern "C" void emu_insert(const BFHashDataStruct* hd, const BFHashParams* hp, int4* slotInfo, unsigned* ctrs, const int* pos, unsigned n) {
    EMU_LAUNCH(insert_kernel, (n + 63) / 64, 64, *hd, *hp, slotInfo, ctrs, pos, n);
}
extern "C" void emu_delete(const BFHashDataStruct* hd, const BFHashParams* hp, int4* slotInfo, const int* pos, unsigned n) {
    EMU_LAUNCH(delete_kernel, (n + 63) / 64, 64, *hd, *hp, slotInfo, pos, n);
}
extern "C" void emu_rehash(const BFHashDataStruct* src, const BFHashDataStruct* dst, const BFHashParams* dhp, const int4* srcSlotInfo, const unsigned* srcCtrs,
                           const int* srcLive, int4* dstSlotInfo, unsigned* dstCtrs, int* dstLive, unsigned* slotMap, unsigned* out, unsigned grid) {
    EMU_LAUNCH(rehash_kernel, grid, BF_REHASH_CHUNK, *src, *dst, *dhp, srcSlotInfo, srcCtrs, srcLive, dstSlotInfo, dstCtrs, dstLive, slotMap, out);
}
extern "C" void emu_list(const BFHashDataStruct* src, const BFHashDataStruct* dst, const unsigned* srcCtrs, unsigned* dstCtrs, int set, const int4* dstSlotInfo,
                         const unsigned* slotMap, const unsigned char* srcFlags, unsigned char* dstFlags, unsigned grid, unsigned block) {
    EMU_LAUNCH(rehash_list_kernel, grid, block, *src, *dst, srcCtrs, dstCtrs, set, dstSlotInfo, slotMap, srcFlags, dstFlags);
}
extern "C" void emu_counter_layout(unsigned* out) {
    const unsigned v[] = { CTR_HIGH_WATER, CTR_E, CTR_FREED, CTR_HEAP_FAIL, CTR_DROPPED, CTR_SET1, SET_COUNT, CTR_NUM };
    memcpy(out, v, sizeof v);
}
'''


@pytest.fixture(scope="module")
def emu():
    L = build_emulated("tsdf_hash.cuh", 0, glue=_GLUE)
    vp, u = C.c_void_p, C.c_uint
    L.emu_insert.argtypes = [vp, vp, vp, vp, vp, u]
    L.emu_delete.argtypes = [vp, vp, vp, vp, u]
    L.emu_rehash.argtypes = [vp] * 11 + [u]
    L.emu_list.argtypes = [vp, vp, vp, vp, C.c_int, vp, vp, vp, vp, u, u]
    L.emu_counter_layout.argtypes = [vp]
    return L


def test_counter_layout_is_the_librarys(emu):
    got = np.zeros(8, np.uint32)
    emu.emu_counter_layout(got.ctypes.data)
    assert got.tolist() == [CTR_HIGH_WATER, CTR_E, CTR_FREED, CTR_HEAP_FAIL, CTR_DROPPED, CTR_SET1, SET_COUNT, CTR_NUM]


class Table:
    """a reset hash (bfTsdfReset's state) with its library-private side arrays, as numpy buffers the emulated kernels write in place"""

    def __init__(self, blocks, buckets):
        self.hp = default_hash_params(num_buckets=buckets, num_sdf_blocks=blocks)
        self.hp.m_hashMaxCollisionLinkedListSize = LIST_LIMIT
        n = buckets * 4
        self.heap = np.arange(blocks - 1, -1, -1, dtype=np.uint32)
        self.counter = np.array([blocks - 1], np.uint32)
        self.hash = np.zeros((n, 8), np.int32); self.hash[:, 3] = FREE
        self.comp = np.zeros((n, 8), np.int32); self.comp[:, 3] = FREE
        self.comp_count = np.zeros(1, np.int32)
        self.dec = np.zeros(n, np.int32); self.decp = np.zeros(n, np.int32)
        self.vox = np.zeros((blocks, VEC), np.uint32)
        self.mutex = np.full(buckets, FREE, np.int32)
        self.slot_info = np.zeros((blocks, 4), np.int32); self.slot_info[:, 3] = -1
        self.ctrs = np.zeros(CTR_NUM, np.uint32)
        self.live = np.zeros(blocks, np.int32)
        self.flags = np.zeros(blocks, np.uint8)
        hd = capi.BFHashDataStruct()
        hd.d_heap, hd.d_heapCounter, hd.d_hashDecision, hd.d_hashDecisionPrefix = self.heap.ctypes.data, self.counter.ctypes.data, self.dec.ctypes.data, self.decp.ctypes.data
        hd.d_hash, hd.d_hashCompactified, hd.d_hashCompactifiedCounter = self.hash.ctypes.data, self.comp.ctypes.data, self.comp_count.ctypes.data
        hd.d_SDFBlocks, hd.d_hashBucketMutex, hd.m_bIsOnGPU = self.vox.ctypes.data, self.mutex.ctypes.data, 1
        self.hd = hd

    def live_blocks(self):
        """{block position: slot} of the occupied entries"""
        e = self.hash[self.hash[:, 3] >= 0]
        return {tuple(int(v) for v in r[:3]): int(r[3]) // 512 for r in e}


def _positions(kind, rng):
    if kind == "random":
        return np.unique(rng.integers(-400, 400, size=(700, 3)), axis=0).astype(np.int32)
    g = np.stack(np.meshgrid(np.arange(-12, 12), np.arange(-10, 10), np.arange(0, 2), indexing="ij"), -1).reshape(-1, 3)
    return np.unique(g + rng.integers(-1, 2, size=g.shape), axis=0).astype(np.int32)


def _source(L, kind, seed):
    """a table with overflow lists, freed holes, voxel words, live counts, drop counters and a last list that holds a freed block"""
    rng = np.random.default_rng(seed)
    pos = _positions(kind, rng)
    src = Table(len(pos) + 64, len(pos) | 1)               # ~1 block per bucket of 4: some overflow-list entries, headroom in the probe windows
    pos = pos[rng.permutation(len(pos))]
    L.emu_insert(C.byref(src.hd), C.byref(src.hp), src.slot_info.ctypes.data, src.ctrs.ctypes.data, np.ascontiguousarray(pos).ctypes.data, len(pos))
    gone = np.ascontiguousarray(pos[rng.permutation(len(pos))[:len(pos) // 6]])
    L.emu_delete(C.byref(src.hd), C.byref(src.hp), src.slot_info.ctypes.data, gone.ctypes.data, len(gone))
    live = src.live_blocks()
    assert len(live) >= len(pos) - len(gone) - 8              # a block whose probe window was full is dropped, as the table's rule says
    assert (src.hash[:, 4] != 0).any(), "no overflow-list entry: the case does not test the lists"
    for p, s in live.items():
        src.vox[s] = rng.integers(0, 2 ** 32, VEC, dtype=np.uint32)
        src.live[s] = rng.integers(-3, 512)
    src.ctrs[CTR_HEAP_FAIL], src.ctrs[CTR_DROPPED], src.ctrs[CTR_E], src.ctrs[CTR_FREED] = 2, 3, 77, len(gone)
    # the last list (counter set 1): live blocks in a shuffled order and one freed block, as a GC leaves its list behind
    items = list(live.items())
    pick = [items[i] for i in rng.permutation(len(items))[:len(items) // 2]]
    freed = tuple(int(v) for v in gone[0])
    freed_slot = next(s for s in range(len(src.slot_info)) if src.slot_info[s, 3] < 0 and s < src.ctrs[CTR_HIGH_WATER])
    pick.insert(len(pick) // 2, (freed, freed_slot))
    for k, (p, s) in enumerate(pick):
        src.comp[k, :3], src.comp[k, 3], src.comp[k, 4] = p, s * 512, 0
        src.flags[k] = rng.integers(0, 4)
    src.ctrs[CTR_SET1 + SET_COUNT] = len(pick)
    src.comp_count[0] = len(pick)
    return src, pick, freed_slot


def _reachable(t, p):
    """find_entry's rule: the home bucket, then the list hanging off its last entry, within the list limit"""
    B = t.hp.m_hashNumBuckets
    h = int(orc.block_hash(p, B)[0])
    for j in range(4):
        if tuple(t.hash[h * 4 + j, :3]) == p and t.hash[h * 4 + j, 3] != FREE:
            return h * 4 + j
    last = h * 4 + 3
    i = last
    for _ in range(LIST_LIMIT):
        if tuple(t.hash[i, :3]) == p and t.hash[i, 3] != FREE:
            return i
        if t.hash[i, 4] == 0:
            break
        i = (last + int(t.hash[i, 4])) % (4 * B)
    return -1


@pytest.mark.parametrize("kind", ["random", "clustered"])
@pytest.mark.parametrize("size", ["larger", "same", "smaller"])
def test_rehash_moves_every_block_and_the_last_list(emu, kind, size):
    src, pick, freed_slot = _source(emu, kind, 17 if kind == "random" else 23)
    live = src.live_blocks()
    nb, nk = len(src.heap), src.hp.m_hashNumBuckets
    blocks, buckets = {"larger": (2 * nb + 5, 3 * nk + 2), "same": (nb, nk), "smaller": (len(live) + 3, nk - 2)}[size]
    dst = Table(blocks, buckets)
    slot_map, out = np.zeros(nb, np.uint32), np.zeros(2, np.uint32)
    slot_map[:] = 0xFFFFFFFF
    emu.emu_rehash(C.byref(src.hd), C.byref(dst.hd), C.byref(dst.hp), src.slot_info.ctypes.data, src.ctrs.ctypes.data, src.live.ctypes.data, dst.slot_info.ctypes.data,
                   dst.ctrs.ctypes.data, dst.live.ctypes.data, slot_map.ctypes.data, out.ctypes.data, 3)
    emu.emu_list(C.byref(src.hd), C.byref(dst.hd), src.ctrs.ctypes.data, dst.ctrs.ctypes.data, CTR_SET1, dst.slot_info.ctypes.data, slot_map.ctypes.data,
                 src.flags.ctypes.data, dst.flags.ctypes.data, 2, 64)
    assert list(out) == [len(live), 0]
    got = dst.live_blocks()
    assert got.keys() == live.keys()
    used = set()
    for p, s in got.items():
        assert np.array_equal(dst.vox[s], src.vox[live[p]]), p
        assert dst.live[s] == src.live[live[p]] and slot_map[live[p]] == s
        e = _reachable(dst, p)
        assert e >= 0 and int(dst.hash[e, 3]) == s * 512, p
        assert tuple(dst.slot_info[s]) == (*p, e)
        used.add(s)
    # heap: the counter and the free stack partition the slots with the table
    free = int(dst.counter[0]) + 1
    assert free == blocks - len(live) and set(int(x) for x in dst.heap[:free]) == set(range(blocks)) - used
    assert (dst.slot_info[sorted(set(range(blocks)) - used), 3] == -1).all()
    assert (dst.mutex == FREE).all() and dst.ctrs[CTR_HIGH_WATER] == max(used) + 1
    # the last list: same order, count and flags; ptr translated; the freed block's entry on a free slot
    n = len(pick)
    assert dst.ctrs[CTR_SET1 + SET_COUNT] == n and dst.comp_count[0] == n
    assert np.array_equal(dst.flags[:n], src.flags[:n]) and np.array_equal(dst.comp[:n, :3], src.comp[:n, :3])
    for k, (p, s) in enumerate(pick):
        d = int(dst.comp[k, 3]) // 512
        if s == freed_slot:
            assert d == int(dst.heap[dst.counter[0]]) and d not in used and dst.live[d] == 0 and not dst.vox[d].any()
        else:
            assert d == got[p] and dst.comp[k, 4] == dst.hash[dst.slot_info[d, 3], 4]
    # counters: copied, the drop counters summed into dst's (0 here)
    assert dst.ctrs[CTR_HEAP_FAIL] == 2 and dst.ctrs[CTR_DROPPED] == 3 and dst.ctrs[CTR_E] == 77 and dst.ctrs[CTR_FREED] == src.ctrs[CTR_FREED]


def test_a_table_too_small_refuses_what_it_cannot_take(emu):
    src, _, _ = _source(emu, "random", 5)
    live = src.live_blocks()
    dst = Table(len(live) - 10, 257)
    slot_map, out = np.full(len(src.heap), 0xFFFFFFFF, np.uint32), np.zeros(2, np.uint32)
    emu.emu_rehash(C.byref(src.hd), C.byref(dst.hd), C.byref(dst.hp), src.slot_info.ctypes.data, src.ctrs.ctypes.data, src.live.ctypes.data, dst.slot_info.ctypes.data,
                   dst.ctrs.ctypes.data, dst.live.ctypes.data, slot_map.ctypes.data, out.ctypes.data, 2)
    got = dst.live_blocks()
    assert out[0] == len(got) and out[0] + out[1] == len(live) and out[1] >= 10
    assert dst.ctrs[CTR_HEAP_FAIL] + dst.ctrs[CTR_DROPPED] == out[1]
    for p, s in got.items():
        assert np.array_equal(dst.vox[s], src.vox[live[p]])
    assert int((slot_map != 0xFFFFFFFF).sum()) == len(got)


_REFUSALS = r'''
import ctypes as C, json, sys
sys.path.insert(0, sys.argv[1])
from bundlefusion_b200 import _capi as capi
from bundlefusion_b200.scene_rep import default_hash_params
L = capi.lib()
def hd(base):
    h = capi.BFHashDataStruct()
    for i, n in enumerate(("d_heap", "d_heapCounter", "d_hashDecision", "d_hashDecisionPrefix", "d_hash", "d_hashCompactified", "d_hashCompactifiedCounter",
                           "d_SDFBlocks", "d_hashBucketMutex")):
        setattr(h, n, base + 0x1000 * i)          # never dereferenced: every case is refused first
    return h
def hp(**kw):
    p = default_hash_params(num_buckets=101, num_sdf_blocks=64)
    for k, v in kw.items():
        setattr(p, k, v)
    return p
s, d, out = hd(0x100000), hd(0x200000), (C.c_ulonglong * 2)()
R = lambda s_, sp, d_, dp, o=out: L.bfTsdfRehash(None if s_ is None else C.byref(s_), None if sp is None else C.byref(sp),
                                                 None if d_ is None else C.byref(d_), None if dp is None else C.byref(dp), o)
shared = hd(0x200000); shared.d_SDFBlocks = s.d_SDFBlocks
nulled = hd(0x200000); nulled.d_hash = None
cases = {
    "null_src": lambda: R(None, hp(), d, hp()), "null_src_params": lambda: R(s, None, d, hp()), "null_dst": lambda: R(s, hp(), None, hp()),
    "null_dst_params": lambda: R(s, hp(), d, None), "null_out": lambda: R(s, hp(), d, hp(), None), "src_is_dst": lambda: R(s, hp(), s, hp()),
    "shared_buffer": lambda: R(s, hp(), shared, hp()), "null_buffer": lambda: R(s, hp(), nulled, hp()),
    "voxel_size": lambda: R(s, hp(), d, hp(m_virtualVoxelSize=0.005)), "truncation": lambda: R(s, hp(), d, hp(m_truncation=0.05)),
    "trunc_scale": lambda: R(s, hp(), d, hp(m_truncScale=0.03)), "max_distance": lambda: R(s, hp(), d, hp(m_maxIntegrationDistance=2.0)),
    "block_size": lambda: R(s, hp(), d, hp(m_SDFBlockSize=4)), "bucket_size": lambda: R(s, hp(), d, hp(m_hashBucketSize=2)),
    "list_limit": lambda: R(s, hp(), d, hp(m_hashMaxCollisionLinkedListSize=9)), "shard": lambda: R(s, hp(), d, hp(m_dummy=1 | (2 << 32))),
    "zero_buckets": lambda: R(s, hp(), d, hp(m_hashNumBuckets=0)), "zero_blocks": lambda: R(s, hp(), d, hp(m_numSDFBlocks=0)),
    "too_many_buckets": lambda: R(s, hp(), d, hp(m_hashNumBuckets=(1 << 30) + 1)),
    "not_reset": lambda: R(s, hp(), d, hp()),
}
res = {k: [f(), L.bfGetLastErrorString().decode()] for k, f in cases.items()}
print(json.dumps(res))
'''


def test_rehash_refusals_enqueue_nothing():
    """each malformed call returns cudaErrorInvalidValue (1) before any CUDA call, in a child process that sees no CUDA device, and names the
    check that refused it.  That nothing is written to dst, and the refusal of a dst heap smaller than src's live blocks (which needs a read of
    src), are checked on real tables on the GPU (tests/test_hash_growth_gpu.py)."""
    out = run_without_device(_REFUSALS)
    assert all(rc == 1 for rc, _ in out.values()), out
    # each case is refused by its own check: a case whose check were missing would fall through to a later one and report that one's reason
    assert {k: msg for k, (_, msg) in out.items()} == {k: "bfTsdfRehash: " + why for k, why in _REASONS.items()}, out


_REASONS = {
    "null_src": "NULL argument", "null_src_params": "NULL argument", "null_dst": "NULL argument", "null_dst_params": "NULL argument",
    "null_out": "NULL argument", "src_is_dst": "src == dst", "shared_buffer": "src and dst share a buffer", "null_buffer": "NULL buffer",
    "voxel_size": "voxel size differs", "truncation": "truncation differs", "trunc_scale": "truncation scale differs",
    "max_distance": "max integration distance differs", "block_size": "block size differs", "bucket_size": "bucket size differs",
    "list_limit": "linked-list limit differs", "shard": "shard setting (m_dummy) differs", "zero_buckets": "dst bucket count 0 or beyond 32-bit entry indices",
    "zero_blocks": "dst heap size 0", "too_many_buckets": "dst bucket count 0 or beyond 32-bit entry indices",
    "not_reset": "src is not a hash this library maintains (bfTsdfReset)",
}


def test_growth_size_rule():
    from bundlefusion_b200.frame_loop import growth_size
    cap = (2 ** 32 - 1) // 4
    # doubling wins when the reserve is small; live + 2 x reserve when it is not; the ceiling caps both
    assert growth_size(1000, 900, 100, 10 ** 6, 1000, 1111) == (2000, 2222 | 1)
    assert growth_size(1000, 900, 800, 10 ** 6, 1000, 1111) == (2500, (1111 * 2500 // 1000) | 1)
    assert growth_size(1000, 900, 800, 1800, 1000, 1111) == (1800, (1111 * 1800 // 1000) | 1)
    assert growth_size(1800, 1700, 50, 1800, 1000, 1111)[0] == 1800             # at the ceiling: no larger heap
    # buckets keep the initial ratio, odd, within the 32-bit entry-index limit
    b, k = growth_size(2 ** 30, 2 ** 30 - 5, 10, 2 ** 32 - 1, 1000, 4000)
    assert b == 2 ** 31 and k == cap and k & 1
    assert growth_size(16384, 16000, 4000, 4 * 10 ** 6, 16384, 16411)[1] == (16411 * 32768 // 16384) | 1

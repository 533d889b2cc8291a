"""The count pass, the chunk-range extraction and the whole-mesh call of csrc/marching_cubes.cu without a GPU: the product's kernels executed on the CPU
through tests/cuda_emu (as tests/test_marchingcubes_oracle.py runs them) on the seeded scene of tests/test_marchingcubes_reference_emulated.py, against
oracle/marchingcubes_oracle.c block by block.  Both run on the same hash table, so a chunk of the product is a range of the oracle's slots.

The oracle extracts the whole table; the triangles of one slot's block come from it through its own box test: a cell is meshed only when its
centre lies in the box, and the box from the block's first cell centre to its last (each computed as the kernels compute it, (float)index *
voxel size) admits exactly that block's 512 cells.  Intersected with the extraction's own box, it admits the cells both admit."""
import ctypes as C
import os

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from oracle import oracle as orc
from tests.test_marchingcubes_reference_emulated import canon, golden_params, golden_scene, scene_box

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK = capi.BF_MC_CHUNK_SLOTS

_EXTRA = r'''
#include <string>
#include "%s"
#include "%s"
#include "%s"
namespace bf { static BFHashParams g_emuHp; const BFHashParams* bound_hash_params() { return &g_emuHp; }
               static std::string g_emuError; static inline void set_last_error(const char* where, int) { g_emuError = where; } }
extern "C" const char* emu_last_error() { return bf::g_emuError.c_str(); }
extern "C" void emu_clear_error() { bf::g_emuError.clear(); }
extern "C" void updateConstantHashParams(const BFHashParams* p) { bf::g_emuHp = *p; }
enum { cudaMemcpyDeviceToHost = 2 };
static inline int cudaMallocHost(void** p, size_t n) { *p = calloc(1, n); return *p ? 0 : 2; }
template <class T> static inline int cudaMallocHost(T** p, size_t n) { return cudaMallocHost(reinterpret_cast<void**>(p), n); }
static inline int cudaFreeHost(void* p) { free(p); return 0; }
static inline int cudaMemcpyAsync(void* d, const void* s, size_t n, int, cudaStream_t) { memcpy(d, s, n); return 0; }
static inline int cudaStreamSynchronize(cudaStream_t) { return 0; }
'''


@pytest.fixture(scope="module")
def emu():
    from tests.cuda_emu import build_emulated
    inc = os.path.join(ROOT, "include")
    L = build_emulated("marching_cubes.cu", 4, extra_pre=_EXTRA % (os.path.join(inc, "bf_tsdf.h"), os.path.join(inc, "bf_raycast.h"), os.path.join(inc, "bf_marchingcubes.h")))
    vp = C.c_void_p
    L.bfMarchingCubesExtract.argtypes = [vp] * 5
    L.bfMarchingCubesCount.argtypes = [vp] * 5
    L.bfMarchingCubesExtractRange.argtypes = [vp, vp, vp, C.c_uint32, C.c_uint32, vp, vp]
    L.bfMarchingCubesCreate.argtypes = [vp, C.POINTER(vp)]
    L.bfMarchingCubesExtractIsoSurface.argtypes = [vp, vp, vp, vp, vp, C.c_int]
    L.bfMarchingCubesExtractIsoSurfaceWhole.argtypes = [vp, vp, vp, vp, vp, C.c_int, vp]
    L.bfMarchingCubesGetLastExtraction.argtypes = [vp, C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong)]
    L.bfMarchingCubesGetSoup.argtypes = [vp, C.POINTER(vp), C.POINTER(vp)]; L.bfMarchingCubesGetSoup.restype = C.c_size_t
    L.bfMarchingCubesClearMeshBuffer.argtypes = [vp]; L.bfMarchingCubesClearMeshBuffer.restype = None
    L.bfMarchingCubesDestroy.argtypes = [vp]; L.bfMarchingCubesDestroy.restype = None
    L.emu_last_error.restype = C.c_char_p
    return L


@pytest.fixture(scope="module")
def scene():
    sc, cam, frames = golden_scene(small=True)
    return sc


def chunks_of(sc):
    return (int(sc.hp.m_hashNumBuckets) * capi.BF_HASH_BUCKET_SIZE + CHUNK - 1) // CHUNK


def slots_of(sc, begin, end):
    total = int(sc.hp.m_hashNumBuckets) * capi.BF_HASH_BUCKET_SIZE
    return min(begin * CHUNK, total), min(end * CHUNK, total)


def oracle_by_slot(sc, p):
    """{slot: the oracle's triangles of that slot's block} for every occupied slot, under p (its box, if enabled, included)"""
    f32 = np.float32
    vs = f32(sc.hp.m_virtualVoxelSize)
    out = {}
    for s in np.flatnonzero(sc.hash[:, 3] != capi.BF_FREE_ENTRY):
        q = capi.BFMarchingCubesParams.from_buffer_copy(p)
        q.m_boxEnabled, q.m_maxNumTriangles = 1, 512 * 5                            # room for every triangle of one block
        for k in range(3):
            lo, hi = f32(f32(int(sc.hash[s, k]) * 8) * vs), f32(f32(int(sc.hash[s, k]) * 8 + 7) * vs)
            if p.m_boxEnabled:
                lo, hi = max(lo, f32(p.m_minCorner[k])), min(hi, f32(p.m_maxCorner[k]))
            q.m_minCorner[k], q.m_maxCorner[k] = float(lo), float(hi)
        tri, found = orc.marchingcubes_extract(sc, q)
        assert found == len(tri)
        out[int(s)] = tri
    return out


def oracle_per_slot(sc, by_slot):
    """triangles per slot of the table"""
    n = np.zeros(int(sc.hp.m_hashNumBuckets) * capi.BF_HASH_BUCKET_SIZE, np.int64)
    for s, tri in by_slot.items():
        n[s] = len(tri)
    return n


def oracle_range(by_slot, begin, end):
    """the oracle's triangles of the blocks in slots [begin, end)"""
    parts = [tri for s, tri in sorted(by_slot.items()) if begin <= s < end]
    return np.concatenate(parts) if parts else np.zeros((0, 3, 6), np.float32)


def count(L, sc, p):
    n = chunks_of(sc)
    counts = np.full(n + 4, 0xDEADBEEF, np.uint32)
    total = np.full(1, 77, np.uint64)
    assert L.bfMarchingCubesCount(C.addressof(sc.hd), C.addressof(sc.hp), C.addressof(p), counts.ctypes.data, total.ctypes.data) == 0
    assert np.all(counts[n:] == 0xDEADBEEF)                                         # one entry per chunk, nothing past them
    return int(total[0]), counts[:n].copy()


def extract_range(L, sc, p, begin, end):
    tri = np.zeros((int(p.m_maxNumTriangles), 3, 6), np.float32)
    n = np.full(1, 77, np.uint32)
    assert L.bfMarchingCubesExtractRange(C.addressof(sc.hd), C.addressof(sc.hp), C.addressof(p), begin, end, tri.ctypes.data, n.ctypes.data) == 0
    return tri[:int(n[0])].copy()


def test_chunk_counts_equal_the_oracles_per_slot_counts(emu, scene):
    sc = scene
    assert chunks_of(sc) == 4 and int(sc.hp.m_hashNumBuckets) * 4 % CHUNK != 0          # the last chunk is partial
    for p in (golden_params(sc.hp), golden_params(sc.hp, scene_box(sc)), golden_params(sc.hp, cap=10)):
        want, found = orc.marchingcubes_extract(sc, golden_params(sc.hp, scene_box(sc) if p.m_boxEnabled else None))
        by_slot = oracle_by_slot(sc, p)
        per_slot = oracle_per_slot(sc, by_slot)
        # the blocks' triangles make up the whole soup: the block boxes split the oracle's extraction exactly
        assert np.array_equal(canon(oracle_range(by_slot, 0, len(per_slot))), canon(want))
        total, counts = count(emu, sc, p)
        per_chunk = np.add.reduceat(per_slot.astype(np.int64), np.arange(0, len(per_slot), CHUNK))
        assert np.array_equal(counts.astype(np.int64), per_chunk) and total == found == int(per_slot.sum()) > 100
        assert np.count_nonzero(counts) >= 2                                           # the triangles are spread over several chunks
    # the box rejects cells: fewer triangles, still counted per chunk
    assert count(emu, sc, golden_params(sc.hp, scene_box(sc)))[0] < count(emu, sc, golden_params(sc.hp))[0]


@pytest.mark.parametrize("box", [False, True])
def test_range_extractions_partition_the_soup(emu, scene, box):
    sc = scene
    p = golden_params(sc.hp, scene_box(sc) if box else None)
    full, found = orc.marchingcubes_extract(sc, p)
    assert len(full) == found
    by_slot = oracle_by_slot(sc, p)
    n = chunks_of(sc)
    partitions = [[(0, n)], [(0, 1), (1, 1), (1, 3), (3, n)], [(0, 2), (2, n)], [(k, k + 1) for k in range(n)], [(0, 0), (0, n - 1), (n - 1, n), (n, n)]]
    for parts in partitions:
        got = []
        for b, e in parts:
            part = extract_range(emu, sc, p, b, e)
            want = oracle_range(by_slot, *slots_of(sc, b, e))
            assert np.array_equal(canon(part), canon(want)), (parts, b, e)
            if b == e:
                assert len(part) == 0
            got.append(part)
        assert np.array_equal(canon(np.concatenate(got)), canon(full)), parts
    # the full range is bfMarchingCubesExtract's extraction
    tri = np.zeros((int(p.m_maxNumTriangles), 3, 6), np.float32)
    cnt = np.full(1, 5, np.uint32)
    assert emu.bfMarchingCubesExtract(C.addressof(sc.hd), C.addressof(sc.hp), C.addressof(p), tri.ctypes.data, cnt.ctypes.data) == 0
    assert np.array_equal(canon(tri[:int(cnt[0])]), canon(full))


def test_refusals_write_nothing(emu, scene):
    sc = scene
    p = golden_params(sc.hp)
    n = chunks_of(sc)
    tri = np.full((8, 3, 6), 3.0, np.float32)
    cnt = np.full(1, 77, np.uint32)
    counts = np.full(n, 99, np.uint32)
    total = np.full(1, 99, np.uint64)
    hd, hp, pp = C.addressof(sc.hd), C.addressof(sc.hp), C.addressof(p)
    bad = golden_params(sc.hp)
    bad.m_hashNumBuckets = int(sc.hp.m_hashNumBuckets) + 2
    R = emu.bfMarchingCubesExtractRange
    cases = {
        "range past the table": (lambda: R(hd, hp, pp, 0, n + 1, tri.ctypes.data, cnt.ctypes.data), "bfMarchingCubesExtractRange: chunk range past the table"),
        "empty range past the table": (lambda: R(hd, hp, pp, n + 1, n + 1, tri.ctypes.data, cnt.ctypes.data), "bfMarchingCubesExtractRange: chunk range past the table"),
        "begin > end": (lambda: R(hd, hp, pp, 3, 2, tri.ctypes.data, cnt.ctypes.data), "bfMarchingCubesExtractRange: chunkBegin > chunkEnd"),
        "null counter": (lambda: R(hd, hp, pp, 0, n, tri.ctypes.data, None), "bfMarchingCubesExtractRange: NULL counter"),
        "null triangles": (lambda: R(hd, hp, pp, 0, n, None, cnt.ctypes.data), "bfMarchingCubesExtractRange: NULL argument"),
        "null hash": (lambda: R(None, hp, pp, 0, n, tri.ctypes.data, cnt.ctypes.data), "bfMarchingCubesExtractRange: NULL argument"),
        "range: other table": (lambda: R(hd, hp, C.addressof(bad), 0, n, tri.ctypes.data, cnt.ctypes.data), "bfMarchingCubesExtractRange: hash or cell parameters"),
        "count: null counts": (lambda: emu.bfMarchingCubesCount(hd, hp, pp, None, total.ctypes.data), "bfMarchingCubesCount: NULL argument"),
        "count: null total": (lambda: emu.bfMarchingCubesCount(hd, hp, pp, counts.ctypes.data, None), "bfMarchingCubesCount: NULL counter"),
        "count: null params": (lambda: emu.bfMarchingCubesCount(hd, hp, None, counts.ctypes.data, total.ctypes.data), "bfMarchingCubesCount: NULL argument"),
        "count: other table": (lambda: emu.bfMarchingCubesCount(hd, hp, C.addressof(bad), counts.ctypes.data, total.ctypes.data), "bfMarchingCubesCount: hash or cell parameters"),
    }
    for name, (call, why) in cases.items():
        emu.emu_clear_error()
        assert call() == 1, name                                                       # cudaErrorInvalidValue
        assert emu.emu_last_error().decode().startswith(why), (name, emu.emu_last_error())
        assert np.all(tri == 3.0) and cnt[0] == 77 and np.all(counts == 99) and total[0] == 99, name
    h = C.c_void_p()
    assert emu.bfMarchingCubesCreate(C.addressof(p), C.byref(h)) == 0
    info = capi.BFMarchingCubesWholeInfo()
    emu.emu_clear_error()
    assert emu.bfMarchingCubesExtractIsoSurfaceWhole(h, hd, hp, None, None, 0, None) == 1
    assert emu.emu_last_error().decode() == "bfMarchingCubesExtractIsoSurfaceWhole: NULL argument"
    assert emu.bfMarchingCubesExtractIsoSurfaceWhole(None, hd, hp, None, None, 0, C.byref(info)) == 1
    assert emu.bfMarchingCubesGetSoup(h, None, None) == 0
    emu.bfMarchingCubesDestroy(h)


def soup_of(L, h):
    pp, cp = C.c_void_p(), C.c_void_p()
    nv = L.bfMarchingCubesGetSoup(h, C.byref(pp), C.byref(cp))
    pos = np.ctypeslib.as_array(C.cast(pp, C.POINTER(C.c_float)), (nv, 3)); col = np.ctypeslib.as_array(C.cast(cp, C.POINTER(C.c_float)), (nv, 4))
    return np.concatenate([pos, col[:, :3]], axis=1).reshape(-1, 3, 6).copy()


def test_whole_mesh_call_and_the_fixed_paths_loss(emu, scene):
    sc = scene
    full, found = orc.marchingcubes_extract(sc, golden_params(sc.hp))
    per_slot = oracle_per_slot(sc, oracle_by_slot(sc, golden_params(sc.hp)))
    per_chunk = np.add.reduceat(per_slot.astype(np.int64), np.arange(0, len(per_slot), CHUNK))
    hd, hp = C.addressof(sc.hd), C.addressof(sc.hp)
    last = lambda h: (lambda f, k: (emu.bfMarchingCubesGetLastExtraction(h, C.byref(f), C.byref(k)), f.value, k.value))(C.c_ulonglong(), C.c_ulonglong())
    # a buffer that holds the largest chunk but not the mesh: several parts, no triangle lost, the buffer unchanged
    cap = int(per_chunk.max()) + 1
    assert cap < found
    h = C.c_void_p()
    assert emu.bfMarchingCubesCreate(C.addressof(golden_params(sc.hp, cap=cap)), C.byref(h)) == 0
    info = capi.BFMarchingCubesWholeInfo()
    assert emu.bfMarchingCubesExtractIsoSurfaceWhole(h, hd, hp, None, None, 0, C.byref(info)) == 0
    assert info.trianglesCounted == info.trianglesExtracted == found and info.chunks == len(per_chunk)
    assert info.parts >= 2 and info.hostSyncs == 1 + info.parts and info.largestPart <= cap and info.bufferTriangles == cap and info.bufferEnlarged == 0
    assert np.array_equal(canon(soup_of(emu, h)), canon(full))
    assert last(h) == (0, found, found)
    # the fixed path into the same buffer: appended after the whole mesh; found = the oracle's count, kept = the capacity
    assert emu.bfMarchingCubesExtractIsoSurface(h, hd, hp, None, None, 0) == 0
    assert len(soup_of(emu, h)) == found + cap and last(h) == (0, found, cap)
    emu.bfMarchingCubesDestroy(h)
    # a buffer smaller than the largest chunk: enlarged to that chunk, then every part fits
    small = int(per_chunk.max()) - 1
    assert emu.bfMarchingCubesCreate(C.addressof(golden_params(sc.hp, cap=small)), C.byref(h)) == 0
    assert emu.bfMarchingCubesExtractIsoSurfaceWhole(h, hd, hp, None, None, 0, C.byref(info)) == 0
    assert info.bufferEnlarged == 1 and info.bufferTriangles == per_chunk.max() and info.trianglesExtracted == found
    assert 2 <= info.parts <= np.count_nonzero(per_chunk)
    assert np.array_equal(canon(soup_of(emu, h)), canon(full))
    # with the box: the box's triangles, in parts
    box = scene_box(sc)
    wantb, foundb = orc.marchingcubes_extract(sc, golden_params(sc.hp, box))
    emu.bfMarchingCubesClearMeshBuffer(h)
    lo, hi = (C.c_float * 3)(*box[0]), (C.c_float * 3)(*box[1])
    assert emu.bfMarchingCubesExtractIsoSurfaceWhole(h, hd, hp, lo, hi, 1, C.byref(info)) == 0
    assert info.trianglesCounted == info.trianglesExtracted == foundb < found
    assert np.array_equal(canon(soup_of(emu, h)), canon(wantb))
    emu.bfMarchingCubesDestroy(h)

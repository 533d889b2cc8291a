"""bfMeshWeld (csrc/mesh_weld.cu) without a GPU: the product's kernels executed on the CPU through tests/cuda_emu, against the host clean-up
bfMeshMergeCloseVertices + bfMeshRemoveDuplicateFaces of the built library (itself pinned to the reference's mLib classes by
tests/test_mesh_reference_host.py) on the same soup, bit for bit."""
import ctypes as C
import os

import numpy as np
import pytest

from bundlefusion_b200 import _capi as capi
from bundlefusion_b200 import marching_cubes as mc
from tests.test_mesh_reference_host import GOLDEN, REF_SO, TRANSFORM, reference_save, soups

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

_EXTRA = r'''
#include <string>
#include "%s"
namespace bf { static std::string g_emuError; static inline void set_last_error(const char* where, int) { g_emuError = where; } }
extern "C" const char* emu_last_error() { return bf::g_emuError.c_str(); }
extern "C" void emu_clear_error() { bf::g_emuError.clear(); }
enum { cudaMemcpyDeviceToHost = 2 };
static inline int cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { memset(p, v, n); return 0; }
static inline int cudaMemcpyAsync(void* d, const void* s, size_t n, int, cudaStream_t) { memcpy(d, s, n); return 0; }
static inline int cudaStreamSynchronize(cudaStream_t) { return 0; }
// the cell index's individually rounded operations: the emulated build is compiled with -ffp-contract=off, so plain float * and + are rounded one by one
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
'''


@pytest.fixture(scope="module")
def emu():
    from tests.cuda_emu import build_emulated
    L = build_emulated("mesh_weld.cu", 9, extra_pre=_EXTRA % os.path.join(ROOT, "include", "bf_marchingcubes.h"))
    vp = C.c_void_p
    L.bfMeshWeldWorkspaceBytes.argtypes = [C.c_uint64]; L.bfMeshWeldWorkspaceBytes.restype = C.c_size_t
    L.bfMeshWeld.argtypes = [vp, C.c_uint64, C.c_float, vp, C.c_size_t, vp, vp, vp, vp]
    L.emu_last_error.restype = C.c_char_p
    return L


def weld(L, tri, thresh):
    """the emulated weld of soup tri [T, 3, 6] -> (positions, colours, faces uint32, info)"""
    tri = np.ascontiguousarray(tri, np.float32)
    T = len(tri)
    ws = np.full(max(int(L.bfMeshWeldWorkspaceBytes(T)), 1), 0xAB, np.uint8)
    pos, col, faces = np.full((3 * T, 3), np.nan, np.float32), np.full((3 * T, 4), np.nan, np.float32), np.full((T, 3), 0xFFFFFFFF, np.uint32)
    info = capi.BFMeshWeldInfo()
    assert L.bfMeshWeld(tri.ctypes.data if T else None, T, thresh, ws.ctypes.data, ws.nbytes, pos.ctypes.data, col.ctypes.data, faces.ctypes.data, C.byref(info)) == 0
    V, F = int(info.verticesOut), int(info.facesOut)
    assert info.trianglesIn == T and info.degenerateFaces + info.duplicateFaces + F == T
    assert info.hostSyncs == (info.rounds + 1 if T else 0)
    return pos[:V], col[:V], faces[:F], info


def host(tri, thresh):
    """saveMesh's clean-up on the host: bfMeshMergeCloseVertices then bfMeshRemoveDuplicateFaces, colours (c, 1)"""
    pos = np.ascontiguousarray(tri[..., :3].reshape(-1, 3))
    col = np.concatenate([tri[..., 3:].reshape(-1, 3), np.ones((len(pos), 1), np.float32)], axis=1)
    p, c, f = mc.merge_close_vertices(pos, col, np.arange(len(pos), dtype=np.uint32).reshape(-1, 3), thresh)
    return p, c, mc.remove_duplicate_faces(f)


def assert_same(got, want):
    p, c, f = got[:3]
    wp, wc, wf = want
    assert p.shape == wp.shape and f.shape == wf.shape, (p.shape, wp.shape, f.shape, wf.shape)
    assert np.array_equal(p.view(np.uint32), wp.view(np.uint32)) and np.array_equal(c.view(np.uint32), wc.view(np.uint32)) and np.array_equal(f, wf)


def check(L, tri, thresh):
    got = weld(L, tri, thresh)
    assert_same(got, host(tri, thresh))
    return got[3]


@pytest.mark.parametrize("name,transform", [("a", None), ("b", None), ("b", TRANSFORM)])
def test_golden_soups_and_their_ply(emu, tmp_path, name, transform):
    g = np.load(GOLDEN)
    key = name + ("_t" if transform is not None else "")
    tri = soups()[name]
    assert np.array_equal(tri, g["soup_" + name])
    p, c, f, info = weld(emu, tri, 0.00001)
    assert_same((p, c, f), host(tri, 0.00001))
    if transform is None:
        assert np.array_equal(p.view(np.uint32), g["pos_" + key].view(np.uint32))
    assert np.array_equal(c, g["col_" + key]) and np.array_equal(f, g["faces_" + key])
    if transform is not None:
        p = mc.apply_transform(p, transform)
        assert np.array_equal(p.view(np.uint32), g["pos_" + key].view(np.uint32))
    path = str(tmp_path / "weld.ply")
    mc.save_ply(path, p, c, f)
    assert open(path, "rb").read() == g["ply_" + key].tobytes()
    assert info.verticesOut < 3 * len(tri) / 2 and info.rounds >= 1


@pytest.fixture(scope="module")
def scene_soup():
    from oracle import oracle as orc
    from tests.test_marchingcubes_reference_emulated import golden_params, golden_scene
    sc, cam, frames = golden_scene()
    tri, found = orc.marchingcubes_extract(sc, golden_params(sc.hp))
    assert len(tri) == found > 1000
    return np.ascontiguousarray(tri)


@pytest.mark.parametrize("thresh", [0.00001, 0.001])
def test_seeded_scene(emu, scene_soup, thresh):
    info = check(emu, scene_soup, thresh)
    if thresh == 0.001:                                                                  # a fifth of the voxel: many merges, some faces collapse
        assert info.verticesOut < info.trianglesIn and info.degenerateFaces > 0
    else:
        assert info.degenerateFaces + info.duplicateFaces < info.trianglesIn // 10


THRESH = 2.0 ** -10                                                                      # exact cell boundaries: x * 1024 is exact


def chain(order):
    """vertices on the x axis, vertex order[i] at cell i: neighbouring cells one apart"""
    n = len(order)
    x = np.zeros(n, np.float32)
    x[np.asarray(order)] = np.arange(n, dtype=np.float32) * np.float32(THRESH)
    tri = np.zeros((n // 3, 3, 6), np.float32)
    tri[..., 0] = x.reshape(-1, 3)
    tri[..., 3:] = np.linspace(0, 1, n * 3, dtype=np.float32).reshape(-1, 3, 3)
    return tri


def test_chain_in_index_order_takes_a_round_per_link(emu):
    n = 30
    info = check(emu, chain(np.arange(n)), THRESH)
    assert info.cells == n and info.rounds == n and info.hostSyncs == n + 1
    assert info.verticesOut == (n + 1) // 2                                               # every other cell keeps its vertex


def test_chain_with_even_cells_first_decides_in_two_rounds(emu):
    n = 30
    cells = np.concatenate([np.arange(0, n, 2), np.arange(1, n, 2)])                      # vertex v sits at cell cells[v]: the even cells first
    inv = np.empty(n, np.int64); inv[cells] = np.arange(n)
    info = check(emu, chain(inv), THRESH)
    assert info.cells == n and info.rounds == 2 and info.hostSyncs == 3 and info.verticesOut == n // 2


def test_special_soups(emu):
    rng = np.random.default_rng(3)
    # every vertex in one cell: one vertex, every face degenerate
    one = np.zeros((7, 3, 6), np.float32)
    one[..., :3] = rng.uniform(0.1, 0.4, (7, 3, 3)).astype(np.float32) * np.float32(THRESH)
    one[..., 3:] = rng.uniform(0, 1, (7, 3, 3)).astype(np.float32)
    info = check(emu, one, THRESH)
    assert info.verticesOut == 1 and info.facesOut == 0 and info.degenerateFaces == 7
    # every triangle degenerate (two corners equal), vertices far apart
    deg = rng.uniform(-1, 1, (12, 3, 6)).astype(np.float32)
    deg[:, 2] = deg[:, 0]
    info = check(emu, deg, THRESH)
    assert info.facesOut == 0 and info.degenerateFaces == 12
    # duplicate faces: rotated and flipped copies, interleaved
    base = rng.uniform(-1, 1, (10, 3, 6)).astype(np.float32)
    dup = np.concatenate([base, base[:, [1, 2, 0]], base[:, [2, 1, 0]], base[3:6], base[:, [0, 2, 1]]])
    dup = dup[rng.permutation(len(dup))]
    info = check(emu, dup, THRESH)
    assert info.facesOut == 10 and info.duplicateFaces == len(dup) - 10
    # both sides of 0, on and next to cell boundaries (x * inv + 0.5 sign lands on and next to integers), -0 and +0
    k = np.arange(-4, 5, dtype=np.float32)
    vals = np.concatenate([(k + np.float32(0.5)) * np.float32(THRESH), np.nextafter((k + np.float32(0.5)) * np.float32(THRESH), np.float32(np.inf)),
                           np.nextafter((k + np.float32(0.5)) * np.float32(THRESH), np.float32(-np.inf)), k * np.float32(THRESH), np.float32([0.0, -0.0, 1e-30, -1e-30])])
    m = len(vals)
    coords = np.stack(np.meshgrid(np.arange(m), np.arange(m) % 5, np.arange(m) % 3, indexing="ij"), -1).reshape(-1, 3)
    coords = coords[rng.permutation(len(coords))][: 3 * (len(coords) // 3)]
    bnd = np.zeros((len(coords) // 3, 3, 6), np.float32)
    bnd[..., :3] = vals[coords].reshape(-1, 3, 3)
    bnd[..., 3:] = rng.uniform(0, 1, bnd[..., 3:].shape).astype(np.float32)
    info = check(emu, bnd, THRESH)
    assert info.rounds >= 2 and 0 < info.verticesOut < 3 * len(bnd)
    # the same at a threshold whose inverse is not exact, with jitter around it
    info = check(emu, bnd + rng.uniform(-1e-5, 1e-5, bnd.shape).astype(np.float32) * np.float32([1, 1, 1, 0, 0, 0]), 0.0003)
    # T = 1 and T = 0
    check(emu, base[:1], THRESH)
    p, c, f, info = weld(emu, np.zeros((0, 3, 6), np.float32), THRESH)
    assert len(p) == len(f) == 0 and info.rounds == 0 and info.hostSyncs == 0


@pytest.mark.skipif(not os.path.exists(REF_SO), reason="oracle/_ref/libref_mesh_host.so not built (needs the reference: python oracle/build_ref.py)")
def test_live_against_the_references_mesh_classes(emu, tmp_path):
    rng = np.random.default_rng(17)
    for it in range(3):
        tri = soups()["a"][rng.permutation(1200)[:500]].copy()
        tri[..., :3] += rng.uniform(-1.2e-5, 1.2e-5, tri[..., :3].shape).astype(np.float32) * (it % 2)
        tri[..., :3] *= np.float32(1 - 2 * (it // 2))
        p, c, f, _ = weld(emu, tri, 0.00001)
        transform = TRANSFORM if it == 2 else None
        wp, wc, wf = reference_save(tri, transform, str(tmp_path / "r.ply"))
        if transform is not None:
            p = mc.apply_transform(p, transform)
        assert np.array_equal(p.view(np.uint32), wp.view(np.uint32)) and np.array_equal(c, wc) and np.array_equal(f, wf)
        mc.save_ply(str(tmp_path / "w.ply"), p, c, f)
        assert open(str(tmp_path / "w.ply"), "rb").read() == open(str(tmp_path / "r.ply"), "rb").read()


def test_refusals_on_the_device_write_nothing(emu):
    tri = soups()["a"][:40].copy()
    for bad, thresh in ((np.nan, 0.00001), (np.inf, 0.00001), (3e4, 0.00001), (-3e4, 0.00001), (1.0, 1e-38)):
        t = tri.copy()
        t[17, 1, 2] = bad
        T = len(t)
        ws = np.zeros(int(emu.bfMeshWeldWorkspaceBytes(T)), np.uint8)
        pos, col, faces = np.full((3 * T, 3), 7.0, np.float32), np.full((3 * T, 4), 7.0, np.float32), np.full((T, 3), 7, np.uint32)
        info = capi.BFMeshWeldInfo(trianglesIn=99, rounds=99)
        emu.emu_clear_error()
        assert emu.bfMeshWeld(t.ctypes.data, T, thresh, ws.ctypes.data, ws.nbytes, pos.ctypes.data, col.ctypes.data, faces.ctypes.data, C.byref(info)) == 1, bad
        assert emu.emu_last_error().decode().startswith("bfMeshWeld: a vertex position is not finite")
        assert bytes(info) == bytes(capi.BFMeshWeldInfo()) and np.all(pos == 7.0) and np.all(col == 7.0) and np.all(faces == 7)


_REFUSALS = r'''
import ctypes as C, json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from bundlefusion_b200 import _capi as capi
from bundlefusion_b200 import marching_cubes as mc
L = mc._bind(capi.lib())
T = 4
tri = np.zeros((T, 3, 6), np.float32)
ws_bytes = int(L.bfMeshWeldWorkspaceBytes(T))
ws = np.full(ws_bytes, 5, np.uint8)
pos, col, faces = np.full((3 * T, 3), 7.0, np.float32), np.full((3 * T, 4), 7.0, np.float32), np.full((T, 3), 7, np.uint32)
out = {"ws_bytes": ws_bytes, "big": int(L.bfMeshWeldWorkspaceBytes((1 << 31) // 3 + 1)), "ok_below": int(L.bfMeshWeldWorkspaceBytes((1 << 31) // 3)) > 0}
def call(soup, n, thresh, w, wb, p, c, f, info):
    L.bfGetLastErrorString.restype = C.c_char_p
    rc = L.bfMeshWeld(soup, n, thresh, w, wb, p, c, f, info)
    return [rc, L.bfGetLastErrorString().decode()]
info = capi.BFMeshWeldInfo(trianglesIn=99)
a = (tri.ctypes.data, T, 1e-5, ws.ctypes.data, ws_bytes, pos.ctypes.data, col.ctypes.data, faces.ctypes.data, C.byref(info))
cases = {"null soup": (None,) + a[1:], "null workspace": a[:3] + (None,) + a[4:], "null positions": a[:5] + (None,) + a[6:],
         "null colours": a[:6] + (None,) + a[7:], "null faces": a[:7] + (None,) + a[8:], "null info": a[:8] + (None,),
         "thresh 0": a[:2] + (0.0,) + a[3:], "thresh < 0": a[:2] + (-1e-5,) + a[3:], "thresh nan": a[:2] + (float("nan"),) + a[3:],
         "thresh inf": a[:2] + (float("inf"),) + a[3:], "3T >= 2^31": a[:1] + ((1 << 31) // 3 + 1,) + a[2:],
         "workspace small": a[:4] + (ws_bytes - 1,) + a[5:]}
out["cases"] = {k: call(*v) for k, v in cases.items()}
out["untouched"] = bool(np.all(ws == 5) and np.all(pos == 7.0) and np.all(col == 7.0) and np.all(faces == 7) and info.trianglesIn == 99)
print(json.dumps(out))
'''


def test_host_refusals_enqueue_nothing():
    from tests.cuda_emu import run_without_device
    r = run_without_device(_REFUSALS)
    assert r["big"] == 0 and r["ok_below"] and r["ws_bytes"] > 0
    why = {"null soup": "NULL argument", "null workspace": "NULL argument", "null positions": "NULL argument", "null colours": "NULL argument",
           "null faces": "NULL argument", "null info": "NULL info", "thresh 0": "thresh must be finite and > 0", "thresh < 0": "thresh must be finite and > 0",
           "thresh nan": "thresh must be finite and > 0", "thresh inf": "thresh must be finite and > 0", "3T >= 2^31": "3 x numTriangles >= 2^31",
           "workspace small": "workspace smaller than"}
    assert set(r["cases"]) == set(why)
    for k, (rc, msg) in r["cases"].items():
        assert rc == 1 and msg.startswith("bfMeshWeld: " + why[k]), (k, rc, msg)
    assert r["untouched"]

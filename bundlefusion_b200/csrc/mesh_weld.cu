// mesh_weld.cu -- the mesh clean-up of saveMesh on the device: mergeCloseVertices(thresh, approx) + removeDegeneratedFaces + removeDuplicateFaces
// (csrc/marching_cubes.cu: merge_close_vertices, remove_duplicate_faces) over a triangle soup in device memory.  Implements bfMeshWeld of
// include/bf_marchingcubes.h; the output is the host functions' output, bit for bit, for any finite thresh > 0 (DESIGN.md section 4i).
//
// The host visits vertices in order: a vertex whose cell (or one of the 26 around it, probed dx, dy, dz from -1 to 1) already holds a kept vertex
// maps to the first such; otherwise it is kept and claims its cell.  Here:
//   1. insert: every vertex's cell into an open-addressing table keyed by a claimed vertex index; smin[slot] = m(C), the first vertex of the cell.
//      Only m(C) can be kept, so the kept cells are the lexicographically first maximal independent set of the occupied cells (order: m,
//      adjacency: Chebyshev distance 1).
//   2. rounds: an undecided cell becomes OUT when an earlier adjacent cell is IN, IN when every earlier adjacent cell is OUT; each round reads the
//      previous round's states only, so the number of rounds does not depend on scheduling.  The earliest undecided cell decides every round.
//   3. map: a vertex maps to the first IN cell of the host's probe order with m < v; none found: it is m of an IN cell and is kept.
//      Kept vertices are ranked by a scan in vertex order.
//   4. faces: re-indexed; a face survives if not degenerate and it is the first face with its sorted triple (a second table keyed by a claimed
//      face index); survivors are compacted in order by a second scan.
// No grid-wide barrier, no CUB: each step is a launch; the scans are tile sums, one CTA's scan of the sums, and a per-tile scan that writes.
// Arithmetic: the cell index is computed as the host computes it, each float operation rounded on its own (__fmul_rn, __fadd_rn, truncation).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>

#include "../../include/bf_marchingcubes.h"
#include "bf_common.cuh"

namespace bf {

extern unsigned long long g_launchCount;

#define BF_WELD_THREADS 256
#define BF_WELD_ITEMS 4
#define BF_WELD_TILE (BF_WELD_THREADS * BF_WELD_ITEMS)
#define BF_WELD_NONE 0xFFFFFFFFu
enum : unsigned char { kUndecided = 0, kIn = 1, kOut = 2 };
enum { kCtrUndecided, kCtrBad, kCtrCells, kCtrNonDegenerate, kCtrVertices, kCtrFaces, kCtrCount };

struct WeldCell { int x, y, z; };

// the host's cell index: (int)(p * inv + 0.5 * sign(p)) per axis; false if p is not finite or the index is outside int32 (less one cell, so the
// neighbours' indices are too)
__device__ __forceinline__ bool weld_cell(const float* soup, unsigned v, float inv, WeldCell& c) {
    const float* p = soup + 6ull * v;
    float t[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float x = __ldg(p + k);
        t[k] = __fadd_rn(__fmul_rn(x, inv), x > 0.0f ? 0.5f : (x < 0.0f ? -0.5f : 0.0f));
    }
    if (!(fabsf(t[0]) < 2147483648.0f && fabsf(t[1]) < 2147483648.0f && fabsf(t[2]) < 2147483648.0f)) return false;
    c = WeldCell{ (int)t[0], (int)t[1], (int)t[2] };
    return true;
}
__device__ __forceinline__ unsigned weld_mix(unsigned h) { h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16; return h; }
__device__ __forceinline__ unsigned weld_hash3(unsigned a, unsigned b, unsigned c) { return weld_mix((a * 73856093u) ^ (b * 19349669u) ^ (c * 83492791u)); }
// vertex o (a claimant of the table: its cell is valid) lies in cell c
__device__ __forceinline__ bool weld_in_cell(const float* soup, unsigned o, float inv, WeldCell c) {
    WeldCell d;
    weld_cell(soup, o, inv, d);
    return d.x == c.x && d.y == c.y && d.z == c.z;
}
// the slot of cell c, or BF_WELD_NONE
__device__ __forceinline__ unsigned weld_find(const float* soup, float inv, const int* slot, unsigned mask, WeldCell c) {
    for (unsigned h = weld_hash3((unsigned)c.x, (unsigned)c.y, (unsigned)c.z) & mask;; h = (h + 1u) & mask) {
        const int o = __ldg(slot + h);
        if (o < 0) return BF_WELD_NONE;
        if (weld_in_cell(soup, (unsigned)o, inv, c)) return h;
    }
}
__device__ __forceinline__ WeldCell weld_offset(WeldCell c, int k) { return WeldCell{ c.x + k / 9 - 1, c.y + (k / 3) % 3 - 1, c.z + k % 3 - 1 }; }   // k = 0..26: the host's probe order
// exclusive scan of one value per thread over the CTA (s: BF_WELD_THREADS words of shared memory); total = the CTA's sum
__device__ __forceinline__ unsigned weld_cta_scan(unsigned v, unsigned* s, unsigned& total) {
    const unsigned tid = threadIdx.x;
    s[tid] = v;
    __syncthreads();
    for (unsigned off = 1; off < BF_WELD_THREADS; off <<= 1) {
        const unsigned x = tid >= off ? s[tid - off] : 0u;
        __syncthreads();
        s[tid] += x;
        __syncthreads();
    }
    total = s[BF_WELD_THREADS - 1];
    const unsigned r = s[tid] - v;
    __syncthreads();
    return r;
}

// 1. every vertex's cell into the table: claim an empty slot or find the cell's slot, then smin = the smallest vertex of the cell
__global__ void __launch_bounds__(BF_WELD_THREADS) weld_insert_kernel(const float* soup, unsigned n, float inv, int* slot, unsigned* smin, unsigned mask, unsigned* ctr) {
    __shared__ unsigned sCells;
    if (threadIdx.x == 0) sCells = 0;
    __syncthreads();
    unsigned claimed = 0;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
        WeldCell c;
        if (!weld_cell(soup, v, inv, c)) { atomicMax(&ctr[kCtrBad], 1u); continue; }
        for (unsigned h = weld_hash3((unsigned)c.x, (unsigned)c.y, (unsigned)c.z) & mask;; h = (h + 1u) & mask) {
            const int o = atomicCAS(&slot[h], -1, (int)v);
            if (o == -1) ++claimed;
            if (o == -1 || weld_in_cell(soup, (unsigned)o, inv, c)) { atomicMin(&smin[h], v); break; }
        }
    }
    if (claimed) atomicAdd(&sCells, claimed);
    __syncthreads();
    if (threadIdx.x == 0 && sCells) atomicAdd(&ctr[kCtrCells], sCells);
}

// 2. one round of the maximal independent set over the occupied slots, from stIn to stOut
__global__ void __launch_bounds__(BF_WELD_THREADS) weld_round_kernel(const float* soup, float inv, const int* slot, const unsigned* smin, unsigned slots, unsigned mask,
                                                                    const unsigned char* stIn, unsigned char* stOut, unsigned* ctr) {
    for (unsigned h = blockIdx.x * blockDim.x + threadIdx.x; h < slots; h += gridDim.x * blockDim.x) {
        if (__ldg(slot + h) < 0) continue;
        unsigned char s = stIn[h];
        if (s == kUndecided) {
            const unsigned m = __ldg(smin + h);
            WeldCell c;
            weld_cell(soup, m, inv, c);
            bool allOut = true;
            for (int k = 0; k < 27; ++k) {
                if (k == 13) continue;
                const unsigned g = weld_find(soup, inv, slot, mask, weld_offset(c, k));
                if (g == BF_WELD_NONE || __ldg(smin + g) > m) continue;                                    // absent, or later than this cell
                const unsigned char t = stIn[g];
                if (t == kIn) { s = kOut; break; }
                if (t == kUndecided) allOut = false;
            }
            if (s == kUndecided && allOut) s = kIn;
            if (s == kUndecided) atomicAdd(&ctr[kCtrUndecided], 1u);
        }
        stOut[h] = s;
    }
}

// 3a. kept[v] = 1 for a vertex that starts a cell of the set; otherwise vmap[v] = the vertex it becomes (m of the first IN cell in probe order with m < v)
__global__ void __launch_bounds__(BF_WELD_THREADS) weld_map_kernel(const float* soup, unsigned n, float inv, const int* slot, const unsigned* smin, unsigned mask,
                                                                  const unsigned char* st, unsigned* kept, unsigned* vmap) {
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
        WeldCell c;
        weld_cell(soup, v, inv, c);
        unsigned target = BF_WELD_NONE;
        for (int k = 0; k < 27; ++k) {
            const unsigned g = weld_find(soup, inv, slot, mask, weld_offset(c, k));
            if (g != BF_WELD_NONE && st[g] == kIn && __ldg(smin + g) < v) { target = __ldg(smin + g); break; }
        }
        kept[v] = target == BF_WELD_NONE ? 1u : 0u;
        vmap[v] = target;
    }
}

// the scans: per tile of BF_WELD_TILE flags their sum, then one CTA turns the sums into exclusive offsets and writes the total
__global__ void __launch_bounds__(BF_WELD_THREADS) weld_tile_sums_kernel(const unsigned* flag, unsigned n, unsigned tiles, unsigned* tileSums) {
    __shared__ unsigned s[BF_WELD_THREADS];
    for (unsigned tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const unsigned base = tile * BF_WELD_TILE + threadIdx.x * BF_WELD_ITEMS;
        unsigned sum = 0;
        for (unsigned i = 0; i < BF_WELD_ITEMS; ++i) if (base + i < n) sum += flag[base + i];
        unsigned total;
        weld_cta_scan(sum, s, total);
        if (threadIdx.x == 0) tileSums[tile] = total;
    }
}
__global__ void __launch_bounds__(BF_WELD_THREADS) weld_scan_sums_kernel(unsigned* tileSums, unsigned tiles, unsigned* total) {
    __shared__ unsigned s[BF_WELD_THREADS];
    unsigned carry = 0;
    for (unsigned base = 0; base < tiles; base += BF_WELD_THREADS) {
        const unsigned i = base + threadIdx.x;
        unsigned sum;
        const unsigned ex = weld_cta_scan(i < tiles ? tileSums[i] : 0u, s, sum);
        if (i < tiles) tileSums[i] = carry + ex;
        carry += sum;
    }
    if (threadIdx.x == 0) *total = carry;
}

// 3b. the kept vertices in vertex order: vmap[v] = rank, position, colour with w = 1
__global__ void __launch_bounds__(BF_WELD_THREADS) weld_emit_vertices_kernel(const float* soup, unsigned n, unsigned tiles, const unsigned* kept, const unsigned* tileSums,
                                                                            unsigned* vmap, float* pos, float* col) {
    __shared__ unsigned s[BF_WELD_THREADS];
    for (unsigned tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const unsigned base = tile * BF_WELD_TILE + threadIdx.x * BF_WELD_ITEMS;
        unsigned f[BF_WELD_ITEMS], sum = 0;
        for (unsigned i = 0; i < BF_WELD_ITEMS; ++i) { f[i] = base + i < n ? kept[base + i] : 0u; sum += f[i]; }
        unsigned total;
        unsigned r = weld_cta_scan(sum, s, total) + tileSums[tile];
        for (unsigned i = 0; i < BF_WELD_ITEMS; ++i) {
            if (!f[i]) continue;
            const unsigned v = base + i;
            const float* p = soup + 6ull * v;
            vmap[v] = r;
            pos[3ull * r] = p[0]; pos[3ull * r + 1] = p[1]; pos[3ull * r + 2] = p[2];
            col[4ull * r] = p[3]; col[4ull * r + 1] = p[4]; col[4ull * r + 2] = p[5]; col[4ull * r + 3] = 1.0f;
            ++r;
        }
    }
}

// face t re-indexed: a kept vertex's rank, or the rank of the vertex it became
__device__ __forceinline__ void weld_face(const unsigned* kept, const unsigned* vmap, unsigned t, unsigned f[3]) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const unsigned v = 3u * t + (unsigned)k;
        f[k] = kept[v] ? vmap[v] : vmap[vmap[v]];
    }
}
__device__ __forceinline__ void weld_sorted(const unsigned f[3], unsigned s[3]) {
    const unsigned lo = min(f[0], min(f[1], f[2])), hi = max(f[0], max(f[1], f[2]));
    s[0] = lo; s[2] = hi; s[1] = f[0] ^ f[1] ^ f[2] ^ lo ^ hi;
}

// 4a. every non-degenerate face's sorted triple into the table (reset): fslot[t] = its slot, smin = the first face with that triple; degenerate: BF_WELD_NONE
__global__ void __launch_bounds__(BF_WELD_THREADS) weld_face_insert_kernel(unsigned numFaces, const unsigned* kept, const unsigned* vmap, int* slot, unsigned* smin,
                                                                          unsigned mask, unsigned* fslot, unsigned* ctr) {
    __shared__ unsigned sCount;
    if (threadIdx.x == 0) sCount = 0;
    __syncthreads();
    unsigned mine = 0;
    for (unsigned t = blockIdx.x * blockDim.x + threadIdx.x; t < numFaces; t += gridDim.x * blockDim.x) {
        unsigned f[3], s[3];
        weld_face(kept, vmap, t, f);
        if (f[0] == f[1] || f[0] == f[2] || f[1] == f[2]) { fslot[t] = BF_WELD_NONE; continue; }
        ++mine;
        weld_sorted(f, s);
        for (unsigned h = weld_hash3(s[0], s[1], s[2]) & mask;; h = (h + 1u) & mask) {
            const int o = atomicCAS(&slot[h], -1, (int)t);
            bool same = o == -1;
            if (!same) {
                unsigned g[3], q[3];
                weld_face(kept, vmap, (unsigned)o, g);
                weld_sorted(g, q);
                same = q[0] == s[0] && q[1] == s[1] && q[2] == s[2];
            }
            if (same) { atomicMin(&smin[h], t); fslot[t] = h; break; }
        }
    }
    if (mine) atomicAdd(&sCount, mine);
    __syncthreads();
    if (threadIdx.x == 0 && sCount) atomicAdd(&ctr[kCtrNonDegenerate], sCount);
}
// 4b. fslot[t] <- 1 if face t survives (the first of its triple), else 0
__global__ void __launch_bounds__(BF_WELD_THREADS) weld_face_flag_kernel(unsigned numFaces, const unsigned* smin, unsigned* fslot) {
    for (unsigned t = blockIdx.x * blockDim.x + threadIdx.x; t < numFaces; t += gridDim.x * blockDim.x) {
        const unsigned h = fslot[t];
        fslot[t] = (h != BF_WELD_NONE && smin[h] == t) ? 1u : 0u;
    }
}
// 4c. the survivors in face order, in their own vertex order
__global__ void __launch_bounds__(BF_WELD_THREADS) weld_emit_faces_kernel(unsigned numFaces, unsigned tiles, const unsigned* survive, const unsigned* tileSums,
                                                                         const unsigned* kept, const unsigned* vmap, unsigned* faces) {
    __shared__ unsigned s[BF_WELD_THREADS];
    for (unsigned tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const unsigned base = tile * BF_WELD_TILE + threadIdx.x * BF_WELD_ITEMS;
        unsigned f[BF_WELD_ITEMS], sum = 0;
        for (unsigned i = 0; i < BF_WELD_ITEMS; ++i) { f[i] = base + i < numFaces ? survive[base + i] : 0u; sum += f[i]; }
        unsigned total;
        unsigned r = weld_cta_scan(sum, s, total) + tileSums[tile];
        for (unsigned i = 0; i < BF_WELD_ITEMS; ++i) {
            if (!f[i]) continue;
            unsigned g[3];
            weld_face(kept, vmap, base + i, g);
            faces[3ull * r] = g[0]; faces[3ull * r + 1] = g[1]; faces[3ull * r + 2] = g[2];
            ++r;
        }
    }
}

// ---- host side ----
// the workspace, carved from the caller's buffer in this order; base == NULL only measures it
struct WeldWs {
    int* slot; unsigned* smin; unsigned char* st[2];      // the table (cells, then faces) and the round states, `slots` entries each
    unsigned* vmap; unsigned* kept;                       // per vertex
    unsigned* fslot;                                      // per face
    unsigned* tileSums; unsigned* ctr;
    unsigned slots, tiles;
};
static size_t weld_layout(uint64_t numTriangles, char* base, WeldWs* w) {
    const uint64_t n = 3 * numTriangles;
    uint64_t slots = 1024;
    while (slots < 2 * n && slots < (1ull << 31)) slots <<= 1;                                                       // load <= 1/2 (n < 2^31 = the cap)
    const uint64_t tiles = (n + BF_WELD_TILE - 1) / BF_WELD_TILE;
    size_t off = 0;
    auto take = [&](uint64_t bytes) { char* p = base ? base + off : nullptr; off += (size_t)((bytes + 255) & ~255ull); return p; };
    char* slot = take(4 * slots); char* smin = take(4 * slots); char* st0 = take(slots); char* st1 = take(slots);
    char* vmap = take(4 * n); char* kept = take(4 * n); char* fslot = take(4 * numTriangles);
    char* sums = take(4 * (tiles + 1)); char* ctr = take(4 * kCtrCount);
    if (w) {
        w->slot = reinterpret_cast<int*>(slot); w->smin = reinterpret_cast<unsigned*>(smin);
        w->st[0] = reinterpret_cast<unsigned char*>(st0); w->st[1] = reinterpret_cast<unsigned char*>(st1);
        w->vmap = reinterpret_cast<unsigned*>(vmap); w->kept = reinterpret_cast<unsigned*>(kept); w->fslot = reinterpret_cast<unsigned*>(fslot);
        w->tileSums = reinterpret_cast<unsigned*>(sums); w->ctr = reinterpret_cast<unsigned*>(ctr);
        w->slots = (unsigned)slots; w->tiles = (unsigned)tiles;
    }
    return off;
}

static unsigned weld_grid(uint64_t items) {
    const uint64_t blocks = (items + BF_WELD_THREADS - 1) / BF_WELD_THREADS;
    return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(blocks, (uint64_t)num_sms() * 8));
}
// exclusive offsets of the tiles of flag[0, n), and *total
static void weld_scan(const unsigned* flag, unsigned n, unsigned tiles, unsigned* tileSums, unsigned* total) {
    const unsigned grid = std::min<unsigned>(tiles, (unsigned)num_sms() * 8);
    g_launchCount += 2;
    weld_tile_sums_kernel<<<grid, BF_WELD_THREADS, 0, stream()>>>(flag, n, tiles, tileSums);
    weld_scan_sums_kernel<<<1, BF_WELD_THREADS, 0, stream()>>>(tileSums, tiles, total);
}

static int weld_refuse(const char* why) {
    set_last_error((std::string("bfMeshWeld: ") + why).c_str(), cudaErrorInvalidValue);
    return (int)cudaErrorInvalidValue;
}

}  // namespace bf

using namespace bf;

BF_API size_t bfMeshWeldWorkspaceBytes(uint64_t numTriangles) {
    if (numTriangles >= (1ull << 31) / 3 + 1) return 0;                                                              // refused by bfMeshWeld
    return weld_layout(numTriangles, nullptr, nullptr);
}

BF_API int bfMeshWeld(const BFMarchingCubesTriangle* d_soup, uint64_t numTriangles, float thresh, void* d_workspace, size_t workspaceBytes,
                      float* d_positions, float* d_colors, uint32_t* d_faces, BFMeshWeldInfo* info) {
    if (!info) return weld_refuse("NULL info");
    if (numTriangles > 0 && (!d_soup || !d_workspace || !d_positions || !d_colors || !d_faces)) return weld_refuse("NULL argument");
    if (!std::isfinite(thresh) || !(thresh > 0.0f)) return weld_refuse("thresh must be finite and > 0");
    if (numTriangles >= (1ull << 31) / 3 + 1) return weld_refuse("3 x numTriangles >= 2^31 (PLY indices are int)");
    if (workspaceBytes < bfMeshWeldWorkspaceBytes(numTriangles)) return weld_refuse("workspace smaller than bfMeshWeldWorkspaceBytes(numTriangles)");
    BFMeshWeldInfo r;
    memset(&r, 0, sizeof(r));
    r.trianglesIn = numTriangles;
    if (numTriangles == 0) { *info = r; return 0; }
    WeldWs w;
    weld_layout(numTriangles, static_cast<char*>(d_workspace), &w);
    const float* soup = reinterpret_cast<const float*>(d_soup);
    const unsigned n = (unsigned)(3 * numTriangles), numFaces = (unsigned)numTriangles, mask = w.slots - 1;
    const float inv = 1.0f / thresh;                                                                                 // as the host function computes it
    cudaStream_t s = stream();
    unsigned h_ctr[kCtrCount];
    // 1. the cells
    BF_CHECK(cudaMemsetAsync(w.slot, 0xFF, 4ull * w.slots, s));
    BF_CHECK(cudaMemsetAsync(w.smin, 0xFF, 4ull * w.slots, s));
    BF_CHECK(cudaMemsetAsync(w.st[0], 0, w.slots, s));
    BF_CHECK(cudaMemsetAsync(w.ctr, 0, 4 * kCtrCount, s));
    ++g_launchCount;
    weld_insert_kernel<<<weld_grid(n), BF_WELD_THREADS, 0, stream()>>>(soup, n, inv, w.slot, w.smin, mask, w.ctr);
    // 2. rounds until no cell is undecided, one host synchronisation each; the first also reads the key pass's refusal
    int cur = 0;
    for (;;) {
        BF_CHECK(cudaMemsetAsync(w.ctr + kCtrUndecided, 0, 4, s));
        ++g_launchCount;
        weld_round_kernel<<<weld_grid(w.slots), BF_WELD_THREADS, 0, stream()>>>(soup, inv, w.slot, w.smin, w.slots, mask, w.st[cur], w.st[cur ^ 1], w.ctr);
        cur ^= 1;
        BF_CHECK(cudaGetLastError());
        BF_CHECK(cudaMemcpyAsync(h_ctr, w.ctr, sizeof(h_ctr), cudaMemcpyDeviceToHost, s));
        BF_CHECK(cudaStreamSynchronize(s));
        r.rounds += 1;
        r.hostSyncs += 1;
        if (h_ctr[kCtrBad]) {
            memset(info, 0, sizeof(*info));
            return weld_refuse("a vertex position is not finite, or its cell index at this thresh is outside int32");
        }
        if (h_ctr[kCtrUndecided] == 0) break;
    }
    const unsigned char* st = w.st[cur];
    // 3. the vertices
    ++g_launchCount;
    weld_map_kernel<<<weld_grid(n), BF_WELD_THREADS, 0, stream()>>>(soup, n, inv, w.slot, w.smin, mask, st, w.kept, w.vmap);
    weld_scan(w.kept, n, w.tiles, w.tileSums, w.ctr + kCtrVertices);
    const unsigned vertexGrid = std::min<unsigned>(w.tiles, (unsigned)num_sms() * 8);
    ++g_launchCount;
    weld_emit_vertices_kernel<<<vertexGrid, BF_WELD_THREADS, 0, stream()>>>(soup, n, w.tiles, w.kept, w.tileSums, w.vmap, d_positions, d_colors);
    // 4. the faces, through the same table
    const unsigned faceTiles = (numFaces + BF_WELD_TILE - 1) / BF_WELD_TILE;
    BF_CHECK(cudaMemsetAsync(w.slot, 0xFF, 4ull * w.slots, s));
    BF_CHECK(cudaMemsetAsync(w.smin, 0xFF, 4ull * w.slots, s));
    ++g_launchCount;
    weld_face_insert_kernel<<<weld_grid(numFaces), BF_WELD_THREADS, 0, stream()>>>(numFaces, w.kept, w.vmap, w.slot, w.smin, mask, w.fslot, w.ctr);
    ++g_launchCount;
    weld_face_flag_kernel<<<weld_grid(numFaces), BF_WELD_THREADS, 0, stream()>>>(numFaces, w.smin, w.fslot);
    weld_scan(w.fslot, numFaces, faceTiles, w.tileSums, w.ctr + kCtrFaces);
    const unsigned faceGrid = std::min<unsigned>(faceTiles, (unsigned)num_sms() * 8);
    ++g_launchCount;
    weld_emit_faces_kernel<<<faceGrid, BF_WELD_THREADS, 0, stream()>>>(numFaces, faceTiles, w.fslot, w.tileSums, w.kept, w.vmap, d_faces);
    BF_CHECK(cudaGetLastError());
    BF_CHECK(cudaMemcpyAsync(h_ctr, w.ctr, sizeof(h_ctr), cudaMemcpyDeviceToHost, s));
    BF_CHECK(cudaStreamSynchronize(s));
    r.hostSyncs += 1;
    r.verticesOut = h_ctr[kCtrVertices];
    r.facesOut = h_ctr[kCtrFaces];
    r.degenerateFaces = numTriangles - h_ctr[kCtrNonDegenerate];
    r.duplicateFaces = (uint64_t)h_ctr[kCtrNonDegenerate] - h_ctr[kCtrFaces];
    r.cells = h_ctr[kCtrCells];
    *info = r;
    return 0;
}

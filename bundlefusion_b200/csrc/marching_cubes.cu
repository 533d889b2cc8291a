// marching_cubes.cu -- iso-surface extraction of the hashed TSDF for sm_90a and the host-side mesh clean-up / PLY writer.  Implements
// include/bf_marchingcubes.h (SURVEY.md section 8f, row N4, second half).
//
// Behavioural sources (what, not how; FL/ = /root/reference/FriedLiver/Source/, mLib = /root/reference/external/mLib/include):
//   extractIsoSurfaceKernel, resetMarchingCubesKernel                        FL/DepthSensing/CUDAMarchingCubesSDF.cu:10-52
//   MarchingCubesData::extractIsoSurfaceAtPosition, vertexInterp, appendTriangle   FL/DepthSensing/MarchingCubesSDFUtil.h:121-271
//   CUDAMarchingCubesHashSDF::extractIsoSurface, copyTrianglesToCPU, saveMesh FL/DepthSensing/CUDAMarchingCubesHashSDF.cpp:13-115
//   MeshData::mergeCloseVertices (approx), removeDegeneratedFaces, removeDuplicateFaces   mLib core-mesh/meshData.cpp:40-100, 200-300
//   MeshIO::saveToPLY                                                        mLib core-mesh/meshIO.cpp:556-640
// How it differs from the reference's organisation:
//   * the reference launches one 512-thread CTA per HASH SLOT (buckets x bucket size: millions of CTAs for the default table, nearly all of which read one entry and
//     leave); here a resident grid (a multiple of the SM count) strides over the table in 512-entry chunks -- one coalesced 16-byte load per thread -- and
//     gives every occupied entry of its chunk to the whole CTA;
//   * a cell's eight corner values are trilinear samples of 2 x 2 x 2 voxels each: 64 voxel reads through the hash per cell in the reference.  A block's 512
//     cells only touch the block and a one-voxel shell around it, so the CTA resolves the 27 neighbouring blocks ONCE and stages those 10^3 voxels (12 KB)
//     in shared memory; every sample then reads shared memory.  Values and arithmetic are the reference's (same voxel index rounding, same weights, same order);
//   * triangles are appended with one global atomicAdd per block instead of one per triangle: cells count their triangles, the CTA reserves a contiguous range.
//     (The reference's soup order is whatever its atomics produce; so is the order of the blocks here.)
// Arithmetic contract (bit-exact with oracle/marchingcubes_oracle.c): TU built -fmad=false -prec-div=true, expressions in the reference's order.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include <sys/stat.h>

#include "../../include/bf_marchingcubes.h"
#include "bf_common.cuh"
#include "hash_read.cuh"
#include "mc_tables.cuh"

namespace bf {

extern unsigned long long g_launchCount;
const BFHashParams* bound_hash_params();                 // tsdf.cu: what updateConstantHashParams latched

#define BF_MC_THREADS 512
#define BF_MC_TILE 10                                    // a block and its one-voxel shell

struct McArgs {
    BFHashDataStruct hd; BFHashParams hp; BFMarchingCubesParams p;
    const BFMarchingCubesParams* d_params;               // non-NULL: the cell parameters are read from the device copy (the reference-named stub)
    BFMarchingCubesTriangle* tri; unsigned* count;
};

struct McTile { const unsigned* w; I3 origin; };         // staged voxels (3 words each) and the voxel position of tile entry (0, 0, 0)

// a voxel by world position: the reference's index rounding, then the staged copy; a position outside the tile (cannot happen for a cell of this block unless
// coordinates exceed float's integer range) falls back to the hash
__device__ __forceinline__ VoxelW mc_voxel(const McTile& t, const BFHashDataStruct& hd, const BFHashParams& hp, F3 pos, BlockCache& bc) {
    const I3 v = world_to_voxel(hp, pos);
    const unsigned rx = (unsigned)(v.x - t.origin.x), ry = (unsigned)(v.y - t.origin.y), rz = (unsigned)(v.z - t.origin.z);
    if (rx < BF_MC_TILE && ry < BF_MC_TILE && rz < BF_MC_TILE) {
        const unsigned* w = t.w + 3u * ((rz * BF_MC_TILE + ry) * BF_MC_TILE + rx);
        return VoxelW{ __uint_as_float(w[0]), __uint_as_float(w[1]), w[2] };
    }
    return get_voxel_at(hd, hp, v, bc);
}

// MarchingCubesData::vertexInterp, MarchingCubesSDFUtil.h:211-233 (both colours are the cell's voxel colour)
__device__ __forceinline__ BFMarchingCubesVertex mc_vertex(float isolevel, F3 p1, F3 p2, float d1, float d2, unsigned color) {
    const float cr = (float)(color & 0xffu), cg = (float)((color >> 8) & 0xffu), cb = (float)((color >> 16) & 0xffu);
    BFMarchingCubesVertex r;
    r.c[0] = cr / 255.f; r.c[1] = cg / 255.f; r.c[2] = cb / 255.f;
    if (fabsf(isolevel - d1) < 0.00001f) { r.p[0] = p1.x; r.p[1] = p1.y; r.p[2] = p1.z; return r; }
    if (fabsf(isolevel - d2) < 0.00001f) { r.p[0] = p2.x; r.p[1] = p2.y; r.p[2] = p2.z; return r; }
    if (fabsf(d1 - d2) < 0.00001f) { r.p[0] = p1.x; r.p[1] = p1.y; r.p[2] = p1.z; return r; }
    const float mu = (isolevel - d1) / (d2 - d1);
    r.p[0] = p1.x + mu * (p2.x - p1.x); r.p[1] = p1.y + mu * (p2.y - p1.y); r.p[2] = p1.z + mu * (p2.z - p1.z);
    const float zero = (float)0;                                        // (float)(c2 - c1) of two equal uchar colours
    r.c[0] = (cr + mu * zero) / 255.f; r.c[1] = (cg + mu * zero) / 255.f; r.c[2] = (cb + mu * zero) / 255.f;
    return r;
}

// offsets (in half voxels) of cube corner v in Bourke's numbering, see mc_tables.cuh
__device__ __forceinline__ F3 mc_corner(F3 c, float P, int v) {
    const float M = -P;
    const bool px = (v == 1 || v == 2 || v == 5 || v == 6), py = (v == 0 || v == 1 || v == 4 || v == 5), pz = v >= 4;
    return F3{ c.x + (px ? P : M), c.y + (py ? P : M), c.z + (pz ? P : M) };
}

__global__ void __launch_bounds__(BF_MC_THREADS)
mc_extract_kernel(const __grid_constant__ McArgs a) {
    __shared__ unsigned sTile[BF_MC_TILE * BF_MC_TILE * BF_MC_TILE * 3];
    __shared__ unsigned long long sTri[256];
    __shared__ unsigned sOcc[BF_MC_THREADS];
    __shared__ int sPtr[27];
    __shared__ unsigned sNumOcc, sTotal, sBase;
    const unsigned tid = threadIdx.x;
    if (tid < 256) sTri[tid] = kMcTriangles[tid];
    const BFMarchingCubesParams P = a.d_params ? *a.d_params : a.p;
    const unsigned total = a.hp.m_hashNumBuckets * BF_HASH_BUCKET_SIZE;
    const float vs = a.hp.m_virtualVoxelSize, half = vs / 2.0f;
    const float isolevel = 0.0f;
    for (unsigned chunk = blockIdx.x; (size_t)chunk * BF_MC_THREADS < total; chunk += gridDim.x) {
        if (tid == 0) sNumOcc = 0;
        __syncthreads();
        const unsigned e = chunk * BF_MC_THREADS + tid;
        if (e < total && __ldg(&a.hd.d_hash[e].ptr) != BF_FREE_ENTRY) sOcc[atomicAdd(&sNumOcc, 1u)] = e;
        __syncthreads();
        const unsigned numOcc = sNumOcc;
        for (unsigned o = 0; o < numOcc; ++o) {
            const BFHashEntry* he = &a.hd.d_hash[sOcc[o]];
            const I3 bpos = { __ldg(&he->pos[0]), __ldg(&he->pos[1]), __ldg(&he->pos[2]) };
            // ---- the 27 blocks around this one, then the 10^3 voxels the block's cells read ----
            if (tid < 27) {
                const I3 nb = { bpos.x + (int)(tid % 3) - 1, bpos.y + (int)((tid / 3) % 3) - 1, bpos.z + (int)(tid / 9) - 1 };
                sPtr[tid] = (tid == 13) ? __ldg(&he->ptr) : find_block(a.hd, a.hp, nb);
            }
            if (tid == 0) sTotal = 0;
            __syncthreads();
            for (unsigned t = tid; t < BF_MC_TILE * BF_MC_TILE * BF_MC_TILE; t += BF_MC_THREADS) {
                const unsigned tx = t % BF_MC_TILE, ty = (t / BF_MC_TILE) % BF_MC_TILE, tz = t / (BF_MC_TILE * BF_MC_TILE);
                const unsigned nx = tx == 0 ? 0u : (tx == BF_MC_TILE - 1 ? 2u : 1u), ny = ty == 0 ? 0u : (ty == BF_MC_TILE - 1 ? 2u : 1u), nz = tz == 0 ? 0u : (tz == BF_MC_TILE - 1 ? 2u : 1u);
                const int ptr = sPtr[nx + 3 * ny + 9 * nz];
                unsigned w0 = 0, w1 = 0, w2 = 0;                                               // a missing block reads as the empty voxel (getVoxel, VoxelUtilHashSDF.h:407-418)
                if (ptr != BF_FREE_ENTRY) {
                    const unsigned lx = (tx + 7u) & 7u, ly = (ty + 7u) & 7u, lz = (tz + 7u) & 7u;
                    const unsigned* w = reinterpret_cast<const unsigned*>(a.hd.d_SDFBlocks + (size_t)ptr + (size_t)((lz * BF_SDF_BLOCK_SIZE + ly) * BF_SDF_BLOCK_SIZE + lx));
                    w0 = __ldg(w); w1 = __ldg(w + 1); w2 = __ldg(w + 2);
                }
                sTile[3 * t] = w0; sTile[3 * t + 1] = w1; sTile[3 * t + 2] = w2;
            }
            __syncthreads();
            // ---- one cell per thread: MarchingCubesSDFUtil.h:121-209 ----
            const I3 base = { bpos.x * BF_SDF_BLOCK_SIZE, bpos.y * BF_SDF_BLOCK_SIZE, bpos.z * BF_SDF_BLOCK_SIZE };       // SDFBlockToVirtualVoxelPos
            const McTile tile = { sTile, I3{ base.x - 1, base.y - 1, base.z - 1 } };
            const I3 pi = { base.x + (int)(tid & 7u), base.y + (int)((tid >> 3) & 7u), base.z + (int)(tid >> 6) };
            const F3 worldPos = { (float)pi.x * vs, (float)pi.y * vs, (float)pi.z * vs };                                 // virtualVoxelPosToWorld
            BlockCache bc = { I3{ 0, 0, 0 }, 0, false };
            float d[8];                                                                                                 // corner values in the table's numbering
            unsigned cube = 0, nTri = 0, off = 0, cellColor = 0;
            bool live = !(P.m_boxEnabled == 1 && (worldPos.x < P.m_minCorner[0] || worldPos.x > P.m_maxCorner[0] || worldPos.y < P.m_minCorner[1] || worldPos.y > P.m_maxCorner[1] ||
                                                  worldPos.z < P.m_minCorner[2] || worldPos.z > P.m_maxCorner[2]));
            if (live) {
#pragma unroll
                for (int v = 0; v < 8; ++v) {
                    unsigned col;
                    const bool ok = trilinear_with(a.hp, mc_corner(worldPos, half, v), d[v], col, [&](F3 q) { return mc_voxel(tile, a.hd, a.hp, q, bc); });
                    live = live && ok;
                }
            }
            if (live) {
#pragma unroll
                for (int v = 0; v < 8; ++v) if (d[v] < isolevel) cube |= 1u << v;
                // the reference's order of the corner array is 000 100 010 001 110 011 101 111 = v3 v2 v0 v7 v1 v4 v6 v5; the pair test is symmetric
                const float thres = P.m_threshMarchingCubes;
#pragma unroll
                for (int k = 0; k < 8; ++k)
#pragma unroll
                    for (int l = 0; l < 8; ++l) {
                        if (d[k] * d[l] < 0.0f) { if (fabsf(d[k]) + fabsf(d[l]) > thres) live = false; }
                        else if (fabsf(d[k] - d[l]) > thres) live = false;
                    }
#pragma unroll
                for (int v = 0; v < 8; ++v) if (fabsf(d[v]) > P.m_threshMarchingCubes2) live = false;
                const unsigned mask = mc_edge_mask(cube);
                if (mask == 0u || mask == 255u) live = false;
            }
            if (live) {
                const unsigned long long row = sTri[cube];
                while (nTri < 5u && ((row >> (12u * nTri)) & 15ull) != 15ull) ++nTri;
                cellColor = mc_voxel(tile, a.hd, a.hp, worldPos, bc).color;                                               // Voxel v = hashData.getVoxel(worldPos)
                off = atomicAdd(&sTotal, nTri);
            }
            __syncthreads();
            if (tid == 0 && sTotal != 0u) sBase = atomicAdd(a.count, sTotal);
            __syncthreads();
            if (nTri != 0u) {
                const unsigned long long row = sTri[cube];
                for (unsigned i = 0; i < nTri; ++i) {
                    const unsigned addr = sBase + off + i;
                    if (addr >= P.m_maxNumTriangles) break;                                                              // appendTriangle: a full buffer drops the rest
                    BFMarchingCubesVertex vtx[3];
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const unsigned edge = (unsigned)((row >> (4u * (3u * i + (unsigned)c))) & 15ull);
                        // edge e joins corners (e, e + 1 mod 4), (4 + e, 4 + (e + 1) mod 4), (e - 8, e - 4)
                        const int va = edge < 8u ? (int)edge : (int)edge - 8, vb = edge < 4u ? (int)((edge + 1u) & 3u) : (edge < 8u ? 4 + (int)((edge + 1u) & 3u) : (int)edge - 4);
                        vtx[c] = mc_vertex(isolevel, mc_corner(worldPos, half, va), mc_corner(worldPos, half, vb), d[va], d[vb], cellColor);
                    }
                    BFMarchingCubesTriangle* tr = a.tri + addr;
                    tr->v0 = vtx[0]; tr->v1 = vtx[1]; tr->v2 = vtx[2];
                }
            }
            __syncthreads();                                                                                           // the tile and the counters are reused
        }
    }
}

__global__ void mc_reset_kernel(unsigned* count) { *count = 0; }
__global__ void mc_clamp_kernel(unsigned* count, unsigned maxNumTriangles, const BFMarchingCubesParams* d_params) {
    const unsigned cap = d_params ? d_params->m_maxNumTriangles : maxNumTriangles;
    if (*count > cap) *count = cap;                                                                                     // appendTriangle, MarchingCubesSDFUtil.h:252-263
}

// the kernel is written for the reference's compile-time geometry (SDF_BLOCK_SIZE 8, HASH_BUCKET_SIZE 4: VoxelUtilHashSDF.h:38-41); parameters that say otherwise are refused
static int check_args(const BFHashDataStruct* hd, const BFHashParams* hp, const BFMarchingCubesParams* p, const BFMarchingCubesTriangle* tri, const unsigned* count) {
    if (!hd || !hp || !p || !tri || !count) return (int)cudaErrorInvalidValue;
    if (hp->m_hashNumBuckets == 0 || !(hp->m_virtualVoxelSize > 0.0f)) return (int)cudaErrorInvalidValue;
    if ((p->m_sdfBlockSize != 0 && p->m_sdfBlockSize != BF_SDF_BLOCK_SIZE) || (p->m_hashBucketSize != 0 && p->m_hashBucketSize != BF_HASH_BUCKET_SIZE)) return (int)cudaErrorInvalidValue;
    if (p->m_hashNumBuckets != 0 && p->m_hashNumBuckets != hp->m_hashNumBuckets) return (int)cudaErrorInvalidValue;          // the grid of the reference's launch and the table disagree
    return 0;
}

static int do_extract(const BFHashDataStruct* hd, const BFHashParams* hp, const BFMarchingCubesParams* p, const BFMarchingCubesParams* d_params, BFMarchingCubesTriangle* tri, unsigned* count) {
    const int bad = check_args(hd, hp, p, tri, count);
    if (bad) return bad;
    McArgs a;
    a.hd = *hd; a.hp = *hp; a.p = *p; a.d_params = d_params; a.tri = tri; a.count = count;
    const size_t chunks = ((size_t)hp->m_hashNumBuckets * BF_HASH_BUCKET_SIZE + BF_MC_THREADS - 1) / BF_MC_THREADS;
    const unsigned grid = (unsigned)std::min<size_t>(chunks, (size_t)num_sms() * 2);
    g_launchCount += 2;
    mc_extract_kernel<<<grid, BF_MC_THREADS, 0, stream()>>>(a);
    mc_clamp_kernel<<<1, 1, 0, stream()>>>(count, p->m_maxNumTriangles, d_params);
    BF_CHECK(cudaGetLastError());
    return 0;
}

// ---- host side: the mesh clean-up of CUDAMarchingCubesHashSDF::saveMesh ------------------------------------------------------------------
struct CoordHash {
    size_t operator()(const I3& v) const { return ((size_t)(unsigned)v.x * 73856093u) ^ ((size_t)(unsigned)v.y * 19349669u) ^ ((size_t)(unsigned)v.z * 83492791u); }
};
struct CoordEq { bool operator()(const I3& a, const I3& b) const { return a.x == b.x && a.y == b.y && a.z == b.z; } };
static inline int sign_of(float v) { return (0.0f < v) - (v < 0.0f); }

// MeshData::mergeCloseVertices(thresh, approx = true) followed by removeDegeneratedFaces (meshData.cpp:217-300): vertices are visited in order; a vertex whose
// cell of size `thresh` (index = (int)(v * (1 / thresh) + 0.5 * sign(v))) or one of its 26 neighbours -- probed in the order x, y, z from -1 to 1 -- already holds a vertex
// becomes that vertex; faces are re-indexed and those with a repeated index dropped
static void merge_close_vertices(std::vector<float>& pos, std::vector<float>& col, std::vector<uint32_t>& faces, float thresh) {
    const size_t numV = pos.size() / 3;
    const bool hasColors = col.size() == numV * 4;
    std::vector<uint32_t> lookUp(numV);
    std::vector<float> newPos, newCol;
    newPos.reserve(pos.size()); if (hasColors) newCol.reserve(col.size());
    std::unordered_map<I3, uint32_t, CoordHash, CoordEq> grid;
    grid.reserve(numV * 2);
    const float inv = 1.0f / thresh;                                                                                     // vec3 / scalar multiplies by the inverse (mLib core-math/vec3.h:142-147)
    uint32_t cnt = 0;
    for (size_t v = 0; v < numV; ++v) {
        const float* p = &pos[3 * v];
        const I3 c = { (int)(p[0] * inv + 0.5f * (float)sign_of(p[0])), (int)(p[1] * inv + 0.5f * (float)sign_of(p[1])), (int)(p[2] * inv + 0.5f * (float)sign_of(p[2])) };
        uint32_t nn = (uint32_t)-1;
        for (int i = -1; i <= 1 && nn == (uint32_t)-1; ++i)
            for (int j = -1; j <= 1 && nn == (uint32_t)-1; ++j)
                for (int k = -1; k <= 1; ++k) {
                    const auto it = grid.find(I3{ c.x + i, c.y + j, c.z + k });
                    if (it != grid.end()) { nn = it->second; break; }
                }
        if (nn == (uint32_t)-1) {
            grid[c] = cnt;
            newPos.insert(newPos.end(), p, p + 3);
            if (hasColors) newCol.insert(newCol.end(), &col[4 * v], &col[4 * v] + 4);
            lookUp[v] = cnt++;
        } else lookUp[v] = nn;
    }
    for (uint32_t& f : faces) f = lookUp[f];
    pos.swap(newPos); if (hasColors) col.swap(newCol);
    size_t out = 0;                                                                                                     // removeDegeneratedFaces
    for (size_t f = 0; f + 2 < faces.size(); f += 3) {
        const uint32_t a = faces[f], b = faces[f + 1], c = faces[f + 2];
        if (a == b || a == c || b == c) continue;
        faces[out] = a; faces[out + 1] = b; faces[out + 2] = c; out += 3;
    }
    faces.resize(out);
}

struct Face3 { uint32_t a, b, c; };
struct Face3Hash { size_t operator()(const Face3& f) const { return ((size_t)f.a * 73856093u) ^ ((size_t)f.b * 19349669u) ^ ((size_t)f.c * 83492791u); } };
struct Face3Eq { bool operator()(const Face3& x, const Face3& y) const { return x.a == y.a && x.b == y.b && x.c == y.c; } };
// MeshData::removeDuplicateFaces (meshData.cpp:40-100): the first face of every set of faces with the same (unordered) vertex set stays, in its own vertex order
static void remove_duplicate_faces(std::vector<uint32_t>& faces) {
    std::unordered_map<Face3, char, Face3Hash, Face3Eq> seen;
    seen.reserve(faces.size() / 3 * 2);
    size_t out = 0;
    for (size_t f = 0; f + 2 < faces.size(); f += 3) {
        uint32_t s[3] = { faces[f], faces[f + 1], faces[f + 2] };
        std::sort(s, s + 3);
        if (!seen.emplace(Face3{ s[0], s[1], s[2] }, 1).second) continue;
        const uint32_t a = faces[f], b = faces[f + 1], c = faces[f + 2];
        faces[out] = a; faces[out + 1] = b; faces[out + 2] = c; out += 3;
    }
    faces.resize(out);
}

// MeshIO::saveToPLY (meshIO.cpp:556-640): binary little-endian, float positions, uchar rgba = (uchar)(colour * 255), faces as uchar count + int indices
static int save_ply(const char* filename, const float* pos, const float* col, size_t numV, const uint32_t* faces, size_t numF) {
    FILE* f = fopen(filename, "wb");
    if (!f) return 1;
    fprintf(f, "ply\nformat binary_little_endian 1.0\ncomment MLIB generated\nelement vertex %zu\nproperty float x\nproperty float y\nproperty float z\n", numV);
    if (col) fprintf(f, "property uchar red\nproperty uchar green\nproperty uchar blue\nproperty uchar alpha\n");
    fprintf(f, "element face %zu\nproperty list uchar int vertex_indices\nend_header\n", numF);
    std::vector<unsigned char> buf;
    buf.reserve(numV * (col ? 16 : 12) + numF * 13);
    for (size_t v = 0; v < numV; ++v) {
        const unsigned char* p = reinterpret_cast<const unsigned char*>(pos + 3 * v);
        buf.insert(buf.end(), p, p + 12);
        if (col) for (int k = 0; k < 4; ++k) buf.push_back((unsigned char)(col[4 * v + k] * 255));
    }
    for (size_t t = 0; t < numF; ++t) {
        buf.push_back(3);
        const unsigned char* p = reinterpret_cast<const unsigned char*>(faces + 3 * t);
        buf.insert(buf.end(), p, p + 12);
    }
    const bool ok = fwrite(buf.data(), 1, buf.size(), f) == buf.size();
    return (fclose(f) == 0 && ok) ? 0 : 1;
}

static bool file_exists(const std::string& p) { struct stat st; return stat(p.c_str(), &st) == 0; }

}  // namespace bf

using namespace bf;

struct BFMarchingCubes {
    BFMarchingCubesParams params;
    BFMarchingCubesTriangle* d_triangles = nullptr;
    unsigned* d_numTriangles = nullptr;
    unsigned* h_numTriangles = nullptr;                  // pinned
    std::vector<float> positions, colors;                // m_meshData: soup, three vertices per triangle
    std::vector<BFMarchingCubesTriangle> staging;
};

BF_API void resetMarchingCubesCUDA(BFMarchingCubesData* data) {
    if (!data || !data->d_numTriangles) BF_SAFE((int)cudaErrorInvalidValue);
    ++g_launchCount;
    mc_reset_kernel<<<1, 1, 0, stream()>>>(data->d_numTriangles);
    BF_SAFE((int)cudaGetLastError());
}
BF_API void extractIsoSurfaceCUDA(const BFHashDataStruct* hashData, const BFRayCastData*, const BFMarchingCubesParams* params, BFMarchingCubesData* data) {
    if (!data || !data->d_params) BF_SAFE((int)cudaErrorInvalidValue);
    BF_SAFE(do_extract(hashData, bound_hash_params(), params, data->d_params, data->d_triangles, data->d_numTriangles));
}
BF_API int bfMarchingCubesExtract(const BFHashDataStruct* hashData, const BFHashParams* hashParams, const BFMarchingCubesParams* params, BFMarchingCubesTriangle* d_triangles,
                                  uint32_t* d_numTriangles) {
    const int bad = check_args(hashData, hashParams, params, d_triangles, d_numTriangles);
    if (bad) return bad;
    ++g_launchCount;
    mc_reset_kernel<<<1, 1, 0, stream()>>>(d_numTriangles);
    return do_extract(hashData, hashParams, params, nullptr, d_triangles, d_numTriangles);
}

BF_API int bfMarchingCubesCreate(const BFMarchingCubesParams* params, BFMarchingCubes** out) {
    if (!params || !out || params->m_maxNumTriangles == 0) return (int)cudaErrorInvalidValue;
    BFMarchingCubes* mc = new BFMarchingCubes();
    mc->params = *params;
    cudaError_t e = cudaMalloc(&mc->d_triangles, sizeof(BFMarchingCubesTriangle) * (size_t)params->m_maxNumTriangles);
    if (e == cudaSuccess) e = cudaMalloc(&mc->d_numTriangles, sizeof(unsigned));
    if (e == cudaSuccess) e = cudaMallocHost(&mc->h_numTriangles, sizeof(unsigned));
    if (e != cudaSuccess) { bfMarchingCubesDestroy(mc); set_last_error("bfMarchingCubesCreate", e); return (int)e; }
    *out = mc;
    return 0;
}
BF_API void bfMarchingCubesDestroy(BFMarchingCubes* mc) {
    if (!mc) return;
    cudaFree(mc->d_triangles); cudaFree(mc->d_numTriangles); cudaFreeHost(mc->h_numTriangles);
    delete mc;
}
BF_API int bfMarchingCubesExtractIsoSurface(BFMarchingCubes* mc, const BFHashDataStruct* hashData, const BFHashParams* hashParams, const float* minCorner, const float* maxCorner,
                                            int boxEnabled) {
    if (!mc) return (int)cudaErrorInvalidValue;
    for (int k = 0; k < 3; ++k) { mc->params.m_minCorner[k] = minCorner ? minCorner[k] : 0.0f; mc->params.m_maxCorner[k] = maxCorner ? maxCorner[k] : 0.0f; }
    mc->params.m_boxEnabled = boxEnabled ? 1 : 0;
    const int rc = bfMarchingCubesExtract(hashData, hashParams, &mc->params, mc->d_triangles, mc->d_numTriangles);
    if (rc) return rc;
    // copyTrianglesToCPU: the count first, then only the triangles there are (the reference copies the whole buffer)
    BF_CHECK(cudaMemcpyAsync(mc->h_numTriangles, mc->d_numTriangles, sizeof(unsigned), cudaMemcpyDeviceToHost, stream()));
    BF_CHECK(cudaStreamSynchronize(stream()));
    const unsigned n = *mc->h_numTriangles;
    if (n == 0) return 0;
    mc->staging.resize(n);
    BF_CHECK(cudaMemcpyAsync(mc->staging.data(), mc->d_triangles, sizeof(BFMarchingCubesTriangle) * (size_t)n, cudaMemcpyDeviceToHost, stream()));
    BF_CHECK(cudaStreamSynchronize(stream()));
    const size_t base = mc->positions.size() / 3;
    mc->positions.resize((base + 3 * (size_t)n) * 3); mc->colors.resize((base + 3 * (size_t)n) * 4);
    const BFMarchingCubesVertex* v = reinterpret_cast<const BFMarchingCubesVertex*>(mc->staging.data());
    for (size_t i = 0; i < 3 * (size_t)n; ++i) {
        float* p = &mc->positions[(base + i) * 3]; float* c = &mc->colors[(base + i) * 4];
        p[0] = v[i].p[0]; p[1] = v[i].p[1]; p[2] = v[i].p[2];
        c[0] = v[i].c[0]; c[1] = v[i].c[1]; c[2] = v[i].c[2]; c[3] = 1.0f;                   // vec4f(vec3f): w = 1
    }
    return 0;
}
BF_API void bfMarchingCubesClearMeshBuffer(BFMarchingCubes* mc) { if (mc) { mc->positions.clear(); mc->colors.clear(); } }
BF_API size_t bfMarchingCubesGetSoup(const BFMarchingCubes* mc, const float** positions, const float** colors) {
    if (!mc) return 0;
    if (positions) *positions = mc->positions.data();
    if (colors) *colors = mc->colors.data();
    return mc->positions.size() / 3;
}

BF_API int bfMeshMergeCloseVertices(float* positions, float* colors, size_t numVertices, uint32_t* faces, size_t numFaces, float thresh, size_t* numVerticesOut, size_t* numFacesOut) {
    if (!positions || !faces || !(thresh > 0.0f)) return 1;
    for (size_t i = 0; i < 3 * numFaces; ++i) if (faces[i] >= numVertices) return 1;
    std::vector<float> pos(positions, positions + 3 * numVertices), col;
    if (colors) col.assign(colors, colors + 4 * numVertices);
    std::vector<uint32_t> f(faces, faces + 3 * numFaces);
    merge_close_vertices(pos, col, f, thresh);
    std::copy(pos.begin(), pos.end(), positions);
    if (colors) std::copy(col.begin(), col.end(), colors);
    std::copy(f.begin(), f.end(), faces);
    if (numVerticesOut) *numVerticesOut = pos.size() / 3;
    if (numFacesOut) *numFacesOut = f.size() / 3;
    return 0;
}
BF_API int bfMeshRemoveDuplicateFaces(uint32_t* faces, size_t numFaces, size_t* numFacesOut) {
    if (!faces) return 1;
    std::vector<uint32_t> f(faces, faces + 3 * numFaces);
    remove_duplicate_faces(f);
    std::copy(f.begin(), f.end(), faces);
    if (numFacesOut) *numFacesOut = f.size() / 3;
    return 0;
}
BF_API int bfMeshSavePly(const char* filename, const float* positions, const float* colors, size_t numVertices, const uint32_t* faces, size_t numFaces) {
    if (!filename || (!positions && numVertices) || (!faces && numFaces)) return 1;
    return save_ply(filename, positions, colors, numVertices, faces, numFaces);
}

BF_API int bfMarchingCubesSaveMesh(BFMarchingCubes* mc, const char* filename, const float* transform, int overwrite, char* actualPath, size_t actualPathCapacity) {
    if (!mc || !filename) return 1;
    std::string name = filename;
    const size_t slash = name.find_last_of('/');
    if (slash != std::string::npos && slash > 0) {                                                                      // util::makeDirectory(folder)
        const std::string folder = name.substr(0, slash);
        if (!file_exists(folder)) mkdir(folder.c_str(), 0777);
    }
    if (!overwrite) {
        // scan.ply, scan1.ply, scan2.ply, ...: the numeric suffix of the base name counts up until the name is free (CUDAMarchingCubesHashSDF.cpp:55-68)
        while (file_exists(name)) {
            const size_t sl = name.find_last_of('/');
            const std::string path = sl == std::string::npos ? "" : name.substr(0, sl + 1);
            std::string curr = sl == std::string::npos ? name : name.substr(sl + 1);
            const size_t dot = curr.find_last_of('.');
            const std::string ext = dot == std::string::npos ? "" : curr.substr(dot + 1);
            if (dot != std::string::npos) curr = curr.substr(0, dot);
            size_t digits = curr.size();
            while (digits > 0 && curr[digits - 1] >= '0' && curr[digits - 1] <= '9') --digits;
            const unsigned num = digits == curr.size() ? 0u : (unsigned)strtoul(curr.c_str() + digits, nullptr, 10);
            name = path + curr.substr(0, digits) + std::to_string(num + 1) + "." + ext;
        }
    }
    const size_t numV = mc->positions.size() / 3;
    std::vector<uint32_t> faces(numV / 3 * 3);
    for (size_t i = 0; i < faces.size(); ++i) faces[i] = (uint32_t)i;
    merge_close_vertices(mc->positions, mc->colors, faces, 0.00001f);
    remove_duplicate_faces(faces);
    if (transform) {                                                     // MeshData::applyTransform: p' = M * (p, 1), de-homogenised (mLib core-math/matrix4x4.h:479-488)
        for (size_t v = 0; v < mc->positions.size() / 3; ++v) {
            float* p = &mc->positions[3 * v];
            const float x = p[0], y = p[1], z = p[2];
            float r[4];
            for (int k = 0; k < 4; ++k) r[k] = transform[4 * k] * x + transform[4 * k + 1] * y + transform[4 * k + 2] * z + transform[4 * k + 3];
            p[0] = r[0] / r[3]; p[1] = r[1] / r[3]; p[2] = r[2] / r[3];
        }
    }
    const int rc = save_ply(name.c_str(), mc->positions.data(), mc->colors.empty() ? nullptr : mc->colors.data(), mc->positions.size() / 3, faces.data(), faces.size() / 3);
    if (actualPath && actualPathCapacity) { strncpy(actualPath, name.c_str(), actualPathCapacity - 1); actualPath[actualPathCapacity - 1] = 0; }
    bfMarchingCubesClearMeshBuffer(mc);
    return rc;
}

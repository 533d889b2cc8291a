/*
 * tsdf_oracle.c -- CPU restatement of the reference's hashed-voxel TSDF path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under bundlefusion_b200/ may include, link
 * or call this file; only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs use it (as the checker / the timed CPU
 * baseline, never as the product).
 *
 * PARITY STATUS: PINNED against the reference itself.  The reference ships no golden vectors or tests for this path (SURVEY.md
 * section 4 / 8c) and its .cu files neither compile with CUDA 12.9 as they are nor run without a GPU, so the pin is made of
 * (a) tests/golden/tsdf_reference_ieee.npz -- outputs of the reference's OWN kernels (oracle/_ref: CUDASceneRepHashSDF.cu built
 *     for sm_90a from /root/reference with the mechanical compat patch of oracle/build_ref.py, IEEE build) on a seeded stream
 *     (3 integrations, a re-integration, GC), produced on a GPU by scripts/make_golden_from_reference.py and replayed through
 *     this file by tests/test_golden_reference.py in the CPU-only suite: block set, heap count and EVERY voxel word bit-identical;
 * (b) tests/test_tsdf_vs_reference_gpu.py on the GPU box (this oracle's contract = the CUDA library = the reference's kernels);
 * (c) analytic known-answer tests we author (tests/test_tsdf_oracle.py).
 *
 * Every function cites the reference lines it restates.  FL/ = FriedLiver/Source/.
 *
 * Arithmetic contract (shared with bundlefusion_b200/csrc/tsdf.cu so the two can
 * be compared BIT-exactly): IEEE-754 binary32, round-to-nearest-even; + - * / are
 * individually rounded EXCEPT where fmaf() is written out, and fmaf() is written
 * exactly where nvcc 12.9 -O3 (without --use_fast_math) fuses the reference's
 * expressions -- read off the SASS of oracle/_ref/libref_tsdf.so: the 4x4 * float3
 * product (t = y*m1; t = fma(x, m0, t); t = fma(z, m2, t); t + m3), the truncation
 * fma(scale, z, trunc), the block centre fma(float(8b), voxelSize, off), and the voxel
 * update (fma(oldSdf, oldW, +-sdf), fma(cur, 0.2, old*0.8), fma(old, oldW, -cur)).
 * With that, the integrate / de-integrate stencil is bit-identical not only to tsdf.cu
 * but to the reference's own kernels in the IEEE build (tests/test_tsdf_vs_reference_gpu.py).
 * Built with -ffp-contract=off here and -fmad=false there so that nothing ELSE fuses.
 * 1/sqrt(x) is a correctly rounded sqrt followed by a correctly rounded divide (the
 * reference uses the approximate rsqrtf, FL/../Include/cutil/inc/cutil_math.h:1207-1211,
 * which no CPU can reproduce: the alloc walk is therefore equal as a SET of blocks, not
 * operation by operation), float->int conversion is CUDA's cvt.rzi.s32.f32 (truncate,
 * saturate, NaN -> 0).
 * Sequential semantics: where the reference resolves races with try-locks and a
 * host retry loop (FL/DepthSensing/CUDASceneRepHashSDF.h:335-348) the oracle simply
 * performs every insertion, which is the fixed point of that loop.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "../include/bf_tsdf.h"

#define ORC_API __attribute__((visibility("default")))

typedef struct { float x, y, z; } f3;
typedef struct { int x, y, z; } i3;

static const float ORC_MINF = -INFINITY;

/* CUDA cvt.rzi.s32.f32 */
static inline int f2i(float v) {
    if (v != v) return 0;
    if (v >= 2147483648.0f) return INT32_MAX;
    if (v <= -2147483648.0f) return INT32_MIN;
    return (int)v;
}
/* CUDA cvt.rzi.u8.f32 (used by make_uchar4(float,...)) */
static inline uint8_t f2u8(float v) {
    if (v != v) return 0;
    if (v <= 0.0f) return 0;
    if (v >= 255.0f) return 255;
    return (uint8_t)v;
}
/* cutil_math.h:31-33 */
static inline int isign(float v) { return (0.0f < v) - (v < 0.0f); }

/* cuda_SimpleMatrixUtil.h:937-944 : affine transform, implicit w = 1; `m0*x + m1*y + m2*z + m3*1` as nvcc fuses it */
static inline f3 xform(const BFFloat4x4* M, f3 v) {
    const float* m = M->m;
    f3 r;
    r.x = fmaf(v.z, m[2], fmaf(v.x, m[0], v.y * m[1])) + m[3];
    r.y = fmaf(v.z, m[6], fmaf(v.x, m[4], v.y * m[5])) + m[7];
    r.z = fmaf(v.z, m[10], fmaf(v.x, m[8], v.y * m[9])) + m[11];
    return r;
}

/* VoxelUtilHashSDF.h:226-234.  `int % unsigned` promotes the int to unsigned, so the
 * modulo is an unsigned one and the "res < 0" fix-up in the reference is dead code. */
static inline uint32_t hash_pos(const BFHashParams* hp, i3 p) {
    const uint32_t p0 = 73856093u, p1 = 19349669u, p2 = 83492791u;
    uint32_t v = ((uint32_t)p.x * p0) ^ ((uint32_t)p.y * p1) ^ ((uint32_t)p.z * p2);
    return v % hp->m_hashNumBuckets;
}

/* VoxelUtilHashSDF.h:272-274 */
static inline float truncation(const BFHashParams* hp, float z) {
    return fmaf(hp->m_truncScale, z, hp->m_truncation);
}
/* VoxelUtilHashSDF.h:283-287 */
static inline i3 world_to_voxel(const BFHashParams* hp, f3 pos) {
    f3 p = { pos.x / hp->m_virtualVoxelSize, pos.y / hp->m_virtualVoxelSize, pos.z / hp->m_virtualVoxelSize };
    i3 r = { f2i(p.x + (float)isign(p.x) * 0.5f), f2i(p.y + (float)isign(p.y) * 0.5f), f2i(p.z + (float)isign(p.z) * 0.5f) };
    return r;
}
/* VoxelUtilHashSDF.h:290-299 */
static inline i3 voxel_to_block(i3 v) {
    if (v.x < 0) v.x -= BF_SDF_BLOCK_SIZE - 1;
    if (v.y < 0) v.y -= BF_SDF_BLOCK_SIZE - 1;
    if (v.z < 0) v.z -= BF_SDF_BLOCK_SIZE - 1;
    i3 r = { v.x / BF_SDF_BLOCK_SIZE, v.y / BF_SDF_BLOCK_SIZE, v.z / BF_SDF_BLOCK_SIZE };
    return r;
}
/* VoxelUtilHashSDF.h:303-315 */
static inline f3 voxel_to_world(const BFHashParams* hp, i3 v) {
    f3 r = { (float)v.x * hp->m_virtualVoxelSize, (float)v.y * hp->m_virtualVoxelSize, (float)v.z * hp->m_virtualVoxelSize };
    return r;
}
static inline f3 block_to_world(const BFHashParams* hp, i3 b) {
    i3 v = { b.x * BF_SDF_BLOCK_SIZE, b.y * BF_SDF_BLOCK_SIZE, b.z * BF_SDF_BLOCK_SIZE };
    return voxel_to_world(hp, v);
}
static inline i3 world_to_block(const BFHashParams* hp, f3 w) { return voxel_to_block(world_to_voxel(hp, w)); }

/* DepthCameraUtil.h:71-76 */
static inline void cam_to_screen_f(const BFDepthCameraParams* cp, f3 pos, float* sx, float* sy) {
    *sx = pos.x * cp->fx / pos.z + cp->mx;
    *sy = pos.y * cp->fy / pos.z + cp->my;
}
/* DepthCameraUtil.h:91-93 */
static inline float proj_z(const BFDepthCameraParams* cp, float z) {
    return (z - cp->m_sensorDepthWorldMin) / (cp->m_sensorDepthWorldMax - cp->m_sensorDepthWorldMin);
}
/* DepthCameraUtil.h:113-119 */
static inline f3 depth_to_skeleton(const BFDepthCameraParams* cp, unsigned ux, unsigned uy, float depth) {
    const float x = ((float)ux - cp->mx) / cp->fx;
    const float y = ((float)uy - cp->my) / cp->fy;
    f3 r = { depth * x, depth * y, depth };
    return r;
}
/* DepthCameraUtil.h:95-107 + :137-144 */
static inline int in_frustum_approx(const BFDepthCameraParams* cp, const BFFloat4x4* viewInv, f3 pos) {
    f3 pc = xform(viewInv, pos);
    float px, py;
    cam_to_screen_f(cp, pc, &px, &py);
    float w1 = (float)cp->m_imageWidth - 1.0f, h1 = (float)cp->m_imageHeight - 1.0f;
    float ix = (2.0f * px - w1) / w1;
    float iy = (h1 - 2.0f * py) / h1;
    float iz = proj_z(cp, pc.z);
    ix *= 0.95f; iy *= 0.95f; iz *= 0.95f;
    return !(ix < -1.0f || ix > 1.0f || iy < -1.0f || iy > 1.0f || iz < 0.0f || iz > 1.0f);
}
/* VoxelUtilHashSDF.h:322-326 */
static inline int block_in_frustum(const BFHashParams* hp, const BFDepthCameraParams* cp, i3 b) {
    const float vs = hp->m_virtualVoxelSize;
    const float off = vs * 0.5f * ((float)BF_SDF_BLOCK_SIZE - 1.0f);
    f3 w = { fmaf((float)(b.x * BF_SDF_BLOCK_SIZE), vs, off), fmaf((float)(b.y * BF_SDF_BLOCK_SIZE), vs, off), fmaf((float)(b.z * BF_SDF_BLOCK_SIZE), vs, off) };
    return in_frustum_approx(cp, &hp->m_rigidTransformInverse, w);
}

/* ---------------------------------------------------------------------- */
/* reset: CUDASceneRepHashSDF.cu:27-65                                     */
ORC_API void orc_tsdf_reset(BFHashDataStruct* hd, const BFHashParams* hp) {
    const uint32_t N = hp->m_numSDFBlocks;
    hd->d_heapCounter[0] = N - 1;
    for (uint32_t i = 0; i < N; ++i) hd->d_heap[i] = N - i - 1;
    memset(hd->d_SDFBlocks, 0, (size_t)N * BF_SDF_BLOCK_VOXELS * sizeof(BFVoxel));
    const uint32_t E = hp->m_hashNumBuckets * BF_HASH_BUCKET_SIZE;
    for (uint32_t i = 0; i < E; ++i) {
        BFHashEntry e = { {0, 0, 0}, BF_FREE_ENTRY, 0 };
        hd->d_hash[i] = e;
        hd->d_hashCompactified[i] = e;
    }
    for (uint32_t i = 0; i < hp->m_hashNumBuckets; ++i) hd->d_hashBucketMutex[i] = BF_FREE_ENTRY;
}

static inline int entry_is(const BFHashEntry* e, i3 p) {
    return e->pos[0] == p.x && e->pos[1] == p.y && e->pos[2] == p.z && e->ptr != BF_FREE_ENTRY;
}

/* VoxelUtilHashSDF.h:440-485 ; returns entry index or -1 */
ORC_API int orc_tsdf_find(const BFHashDataStruct* hd, const BFHashParams* hp, int bx, int by, int bz) {
    i3 p = { bx, by, bz };
    const uint32_t h = hash_pos(hp, p), hpz = h * BF_HASH_BUCKET_SIZE;
    const uint32_t total = BF_HASH_BUCKET_SIZE * hp->m_hashNumBuckets;
    for (uint32_t j = 0; j < BF_HASH_BUCKET_SIZE; ++j)
        if (entry_is(&hd->d_hash[hpz + j], p)) return (int)(hpz + j);
    const uint32_t last = (h + 1) * BF_HASH_BUCKET_SIZE - 1;
    uint32_t i = last;
    for (uint32_t it = 0; it < hp->m_hashMaxCollisionLinkedListSize; ++it) {
        const BFHashEntry* c = &hd->d_hash[i];
        if (entry_is(c, p)) return (int)i;
        if (c->offset == 0) break;
        i = (last + c->offset) % total;
    }
    return -1;
}

/* VoxelUtilHashSDF.h:535-540 consumeHeap.  Guard added: the reference has no
 * exhaustion check ("TODO MATTHIAS"); the oracle refuses to pop an empty heap and
 * returns 0 so the caller skips the insertion (the product does the same). */
static int heap_pop(BFHashDataStruct* hd, uint32_t* slot) {
    uint32_t c = hd->d_heapCounter[0];
    if (c == 0xFFFFFFFFu) return 0;           /* counter = top index; -1 = empty */
    *slot = hd->d_heap[c];
    hd->d_heapCounter[0] = c - 1;
    return 1;
}
/* VoxelUtilHashSDF.h:541-546 appendHeap */
static void heap_push(BFHashDataStruct* hd, uint32_t slot) {
    uint32_t c = hd->d_heapCounter[0];
    hd->d_heap[c + 1] = slot;
    hd->d_heapCounter[0] = c + 1;
}

/* VoxelUtilHashSDF.h:549-655 allocBlock, with every try-lock succeeding.
 * Returns 1 if the block had to be DROPPED (no heap slot, or no free entry inside the probe window). */
static int alloc_block(BFHashDataStruct* hd, const BFHashParams* hp, i3 pos) {
    const uint32_t h = hash_pos(hp, pos), hpz = h * BF_HASH_BUCKET_SIZE;
    const uint32_t total = BF_HASH_BUCKET_SIZE * hp->m_hashNumBuckets;
    int firstEmpty = -1;
    for (uint32_t j = 0; j < BF_HASH_BUCKET_SIZE; ++j) {
        const BFHashEntry* c = &hd->d_hash[hpz + j];
        if (entry_is(c, pos)) return 0;
        if (firstEmpty == -1 && c->ptr == BF_FREE_ENTRY) firstEmpty = (int)(hpz + j);
    }
    const uint32_t last = (h + 1) * BF_HASH_BUCKET_SIZE - 1;
    uint32_t i = last;
    const uint32_t maxLoop = hp->m_hashMaxCollisionLinkedListSize;
    for (uint32_t it = 0; it < maxLoop; ++it) {
        const BFHashEntry* c = &hd->d_hash[i];
        if (entry_is(c, pos)) return 0;
        if (c->offset == 0) break;
        i = (last + c->offset) % total;
    }
    uint32_t slot;
    if (firstEmpty != -1) {
        if (!heap_pop(hd, &slot)) return 1;
        BFHashEntry* e = &hd->d_hash[firstEmpty];
        e->pos[0] = pos.x; e->pos[1] = pos.y; e->pos[2] = pos.z;
        e->offset = BF_NO_OFFSET;
        e->ptr = (int32_t)(slot * BF_SDF_BLOCK_VOXELS);
        return 0;
    }
    /* linear probe for a free non-bucket-last slot, splice into the list (:614-654) */
    uint32_t offset = 0, it = 0;
    while (it < maxLoop) {
        offset++;
        i = (last + offset) % total;
        if ((offset % BF_HASH_BUCKET_SIZE) == 0) continue;
        if (hd->d_hash[i].ptr == BF_FREE_ENTRY) {
            if (!heap_pop(hd, &slot)) return 1;
            BFHashEntry lastE = hd->d_hash[last];
            BFHashEntry* e = &hd->d_hash[i];
            e->pos[0] = pos.x; e->pos[1] = pos.y; e->pos[2] = pos.z;
            e->offset = lastE.offset;
            e->ptr = (int32_t)(slot * BF_SDF_BLOCK_VOXELS);
            hd->d_hash[last].offset = offset;
            return 0;
        }
        it++;
    }
    return 1;
}

/* Multi-GPU spatial shard of the voxel hash (not in the reference; SURVEY.md section 8e, tsdf.cu owns_block): with
 * hp->m_dummy = {rank, world}, world > 1, a device allocates -- and therefore integrates -- only the blocks it owns:
 * a 3-D checkerboard of cubes of 8^3 blocks, owner = (cx + cy + cz) mod world. */
static inline int floor_div_cube(int v) { return (v >= 0) ? v / 8 : -((-v + 7) / 8); }
static inline int owns_block(const BFHashParams* hp, i3 b) {
    const int world = (int)hp->m_dummy[1];
    if (world <= 1) return 1;
    int m = (floor_div_cube(b.x) + floor_div_cube(b.y) + floor_div_cube(b.z)) % world;
    if (m < 0) m += world;
    return (uint32_t)m == hp->m_dummy[0];
}

/* allocKernel: CUDASceneRepHashSDF.cu:165-251 (d_bitMask == NULL: streaming is disabled
 * for BundleFusion, zParametersDefault.txt:99). */
/* the in-frustum (owned) blocks one pixel's DDA visits, in walk order (allocKernel, CUDASceneRepHashSDF.cu:165-251) */
static unsigned pixel_blocks(const BFHashParams* hp, const float* depth, const BFDepthCameraParams* cp, unsigned x, unsigned y, i3* out /*[1024]*/) {
    const unsigned W = cp->m_imageWidth;
    const float vs = hp->m_virtualVoxelSize;
    unsigned n = 0;
    {
        float d = depth[y * W + x];
        if (d == ORC_MINF || d == 0.0f) return n;
        if (d >= hp->m_maxIntegrationDistance) return n;
        float t = truncation(hp, d);
        float minDepth = fminf(hp->m_maxIntegrationDistance, d - t);
        float maxDepth = fminf(hp->m_maxIntegrationDistance, d + t);
        if (minDepth >= maxDepth) return n;

        f3 rayMin = xform(&hp->m_rigidTransform, depth_to_skeleton(cp, x, y, minDepth));
        f3 rayMax = xform(&hp->m_rigidTransform, depth_to_skeleton(cp, x, y, maxDepth));
        f3 dv = { rayMax.x - rayMin.x, rayMax.y - rayMin.y, rayMax.z - rayMin.z };
        float inv = 1.0f / sqrtf(dv.x * dv.x + dv.y * dv.y + dv.z * dv.z);
        f3 dir = { dv.x * inv, dv.y * inv, dv.z * inv };

        i3 cur = world_to_block(hp, rayMin);
        i3 end = world_to_block(hp, rayMax);
        f3 step = { (float)isign(dir.x), (float)isign(dir.y), (float)isign(dir.z) };
        i3 nb = { cur.x + f2i(fminf(fmaxf(step.x, 0.0f), 1.0f)),
                  cur.y + f2i(fminf(fmaxf(step.y, 0.0f), 1.0f)),
                  cur.z + f2i(fminf(fmaxf(step.z, 0.0f), 1.0f)) };
        f3 bw = block_to_world(hp, nb);
        float half = 0.5f * vs;
        f3 boundary = { bw.x - half, bw.y - half, bw.z - half };
        f3 tMax = { (boundary.x - rayMin.x) / dir.x, (boundary.y - rayMin.y) / dir.y, (boundary.z - rayMin.z) / dir.z };
        f3 tDelta = { (step.x * (float)BF_SDF_BLOCK_SIZE * vs) / dir.x,
                      (step.y * (float)BF_SDF_BLOCK_SIZE * vs) / dir.y,
                      (step.z * (float)BF_SDF_BLOCK_SIZE * vs) / dir.z };
        i3 bound = { f2i((float)end.x + step.x), f2i((float)end.y + step.y), f2i((float)end.z + step.z) };
        if (dir.x == 0.0f) { tMax.x = INFINITY; tDelta.x = INFINITY; }
        if (boundary.x - rayMin.x == 0.0f) { tMax.x = INFINITY; tDelta.x = INFINITY; }
        if (dir.y == 0.0f) { tMax.y = INFINITY; tDelta.y = INFINITY; }
        if (boundary.y - rayMin.y == 0.0f) { tMax.y = INFINITY; tDelta.y = INFINITY; }
        if (dir.z == 0.0f) { tMax.z = INFINITY; tDelta.z = INFINITY; }
        if (boundary.z - rayMin.z == 0.0f) { tMax.z = INFINITY; tDelta.z = INFINITY; }

        for (unsigned iter = 0; iter < 1024; ++iter) {
            if (block_in_frustum(hp, cp, cur) && owns_block(hp, cur) && n < 1024) out[n++] = cur;
            if (tMax.x < tMax.y && tMax.x < tMax.z) {
                cur.x = f2i((float)cur.x + step.x);
                if (cur.x == bound.x) break;
                tMax.x += tDelta.x;
            } else if (tMax.z < tMax.y) {
                cur.z = f2i((float)cur.z + step.z);
                if (cur.z == bound.z) break;
                tMax.z += tDelta.z;
            } else {
                cur.y = f2i((float)cur.y + step.y);
                if (cur.y == bound.y) break;
                tMax.y += tDelta.y;
            }
        }
    }
    return n;
}

ORC_API unsigned orc_tsdf_alloc(BFHashDataStruct* hd, const BFHashParams* hp,
                            const float* depth, const BFDepthCameraParams* cp) {
    const unsigned W = cp->m_imageWidth, H = cp->m_imageHeight;
    unsigned dropped = 0;
#ifdef _OPENMP
    /* timing build (liboracle_fast.so, bench.py's CPU arm): every host thread walks rows and collects the blocks its pixels visit;
     * the insertions -- the only part that touches the table -- then run in one thread.  Same SET of blocks as the serial walk (the
     * slot a block receives may differ, which no comparison keys on; the drop count differs only in an over-full table). */
    const int nt = omp_get_max_threads();
    i3** lists = (i3**)calloc((size_t)nt, sizeof(i3*));
    size_t* cnt = (size_t*)calloc((size_t)nt, sizeof(size_t)); size_t* cap = (size_t*)calloc((size_t)nt, sizeof(size_t));
#pragma omp parallel
    {
        const int t = omp_get_thread_num();
        i3 buf[1024];
#pragma omp for schedule(dynamic, 4)
        for (unsigned y = 0; y < H; ++y) for (unsigned x = 0; x < W; ++x) {
            const unsigned n = pixel_blocks(hp, depth, cp, x, y, buf);
            for (unsigned k = 0; k < n; ++k) {
                if (cnt[t] && lists[t][cnt[t] - 1].x == buf[k].x && lists[t][cnt[t] - 1].y == buf[k].y && lists[t][cnt[t] - 1].z == buf[k].z) continue;
                if (cnt[t] == cap[t]) { cap[t] = cap[t] ? 2 * cap[t] : 4096; lists[t] = (i3*)realloc(lists[t], cap[t] * sizeof(i3)); }
                lists[t][cnt[t]++] = buf[k];
            }
        }
    }
    for (int t = 0; t < nt; ++t) { for (size_t k = 0; k < cnt[t]; ++k) dropped += (unsigned)alloc_block(hd, hp, lists[t][k]); free(lists[t]); }
    free(lists); free(cnt); free(cap);
#else
    i3 buf[1024];
    for (unsigned y = 0; y < H; ++y) for (unsigned x = 0; x < W; ++x) {
        const unsigned n = pixel_blocks(hp, depth, cp, x, y, buf);
        for (unsigned k = 0; k < n; ++k) dropped += (unsigned)alloc_block(hd, hp, buf[k]);
    }
#endif
    return dropped;   /* insert attempts that found no room (0 in any sanely sized table) */
}

/* compactifyHashAllInOneKernel: CUDASceneRepHashSDF.cu:324-384 (table order) */
ORC_API unsigned orc_tsdf_compactify(BFHashDataStruct* hd, const BFHashParams* hp, const BFDepthCameraParams* cp) {
    const uint32_t E = hp->m_hashNumBuckets * BF_HASH_BUCKET_SIZE;
    unsigned n = 0;
    for (uint32_t i = 0; i < E; ++i) {
        const BFHashEntry* e = &hd->d_hash[i];
        if (e->ptr == BF_FREE_ENTRY) continue;
        i3 b = { e->pos[0], e->pos[1], e->pos[2] };
        if (block_in_frustum(hp, cp, b)) hd->d_hashCompactified[n++] = *e;
    }
    hd->d_hashCompactifiedCounter[0] = (int32_t)n;
    return n;
}

static inline float clamp_color(float v) { return fmaxf(0.0f, fminf(v, 254.5f)); }

/* integrateDepthMapKernel<deIntegrate>: CUDASceneRepHashSDF.cu:420-521.
 * Returns U, the number of voxels that passed the truncation test (were rewritten). */
ORC_API unsigned long long orc_tsdf_integrate(BFHashDataStruct* hd, const BFHashParams* hp,
                                              const float* depthImg, const uint8_t* colorImg,
                                              const BFDepthCameraParams* cp, unsigned numOccupied, int deIntegrate) {
    unsigned long long U = 0;
    const unsigned W = cp->m_imageWidth, H = cp->m_imageHeight;
    /* blocks own disjoint voxels, so the timing build (liboracle_fast.so, -fopenmp) may split them */
#pragma omp parallel for schedule(dynamic, 64) reduction(+ : U)
    for (unsigned b = 0; b < numOccupied; ++b) {
        const BFHashEntry* e = &hd->d_hashCompactified[b];
        for (unsigned i = 0; i < BF_SDF_BLOCK_VOXELS; ++i) {
            i3 pi = { e->pos[0] * BF_SDF_BLOCK_SIZE + (int)(i % 8), e->pos[1] * BF_SDF_BLOCK_SIZE + (int)((i % 64) / 8),
                      e->pos[2] * BF_SDF_BLOCK_SIZE + (int)(i / 64) };
            f3 pf = xform(&hp->m_rigidTransformInverse, voxel_to_world(hp, pi));
            float sx, sy;
            cam_to_screen_f(cp, pf, &sx, &sy);
            unsigned px = (unsigned)f2i(sx + 0.5f), py = (unsigned)f2i(sy + 0.5f);
            if (!(px < W && py < H)) continue;
            float depth = depthImg[py * W + px];
            float cr = ORC_MINF, cg = 0, cb = 0;
            if (colorImg) { const uint8_t* c = &colorImg[4 * (py * W + px)]; cr = c[0]; cg = c[1]; cb = c[2]; }
            if (!(cr != ORC_MINF && depth != ORC_MINF)) continue;
            if (!(depth < hp->m_maxIntegrationDistance)) continue;
            float sdf = depth - pf.z;
            float trunc = truncation(hp, depth);
            if (!(fabsf(sdf) < trunc)) continue;
            if (sdf >= 0.0f) sdf = fminf(trunc, sdf); else sdf = fmaxf(-trunc, sdf);
            const float cw = 1.0f;                      /* weightUpdate forced to 1, :465-466 (Q2) */
            uint8_t cur[3];
            if (colorImg) { cur[0] = f2u8(cr); cur[1] = f2u8(cg); cur[2] = f2u8(cb); }
            else { cur[0] = 0; cur[1] = 255; cur[2] = 0; }
            BFVoxel* v = &hd->d_SDFBlocks[(size_t)(uint32_t)e->ptr + i];
            const BFVoxel old = *v;
            BFVoxel nv;
            float oc[3] = { old.color[0], old.color[1], old.color[2] };
            float cc[3] = { cur[0], cur[1], cur[2] };
            if (!deIntegrate) {
                for (int k = 0; k < 3; ++k) {
                    float r = (old.weight == 0) ? cc[k] : fmaf(cc[k], 0.2f, 0.8f * oc[k]);
                    nv.color[k] = f2u8(clamp_color(roundf(r)));
                }
                nv.color[3] = 255;
                nv.sdf = fmaf(old.sdf, old.weight, sdf * cw) / (cw + old.weight);
                nv.weight = fminf((float)hp->m_integrationWeightMax, cw + old.weight);
            } else {
                for (int k = 0; k < 3; ++k) {
                    float r = fmaf(oc[k], old.weight, -(cc[k] * cw)) / (old.weight - cw);
                    nv.color[k] = f2u8(clamp_color(roundf(r)));
                }
                nv.color[3] = 255;
                nv.sdf = fmaf(old.sdf, old.weight, -(sdf * cw)) / (old.weight - cw);
                nv.weight = fmaxf(0.0f, old.weight - cw);
                if (nv.weight <= 0.001f) { nv.sdf = 0.0f; nv.weight = 0.0f; nv.color[0] = nv.color[1] = nv.color[2] = nv.color[3] = 0; }
            }
            *v = nv;
            ++U;
        }
    }
    return U;
}

/* deleteHashEntryElement: VoxelUtilHashSDF.h:739-826, all try-locks succeeding */
static int delete_entry(BFHashDataStruct* hd, const BFHashParams* hp, i3 p) {
    const uint32_t h = hash_pos(hp, p), hpz = h * BF_HASH_BUCKET_SIZE;
    const uint32_t total = BF_HASH_BUCKET_SIZE * hp->m_hashNumBuckets;
    const BFHashEntry freeE = { {0, 0, 0}, BF_FREE_ENTRY, 0 };
    for (uint32_t j = 0; j < BF_HASH_BUCKET_SIZE; ++j) {
        uint32_t i = hpz + j;
        BFHashEntry c = hd->d_hash[i];
        if (entry_is(&c, p)) {
            heap_push(hd, (uint32_t)c.ptr / BF_SDF_BLOCK_VOXELS);
            if (c.offset != 0) {
                uint32_t next = (i + c.offset) % total;
                hd->d_hash[i] = hd->d_hash[next];
                hd->d_hash[next] = freeE;
            } else {
                hd->d_hash[i] = freeE;
            }
            return 1;
        }
    }
    const uint32_t last = (h + 1) * BF_HASH_BUCKET_SIZE - 1;
    BFHashEntry c = hd->d_hash[last];
    uint32_t prev = last;
    uint32_t i = (last + c.offset) % total;
    for (uint32_t it = 0; it < hp->m_hashMaxCollisionLinkedListSize; ++it) {
        c = hd->d_hash[i];
        if (entry_is(&c, p)) {
            heap_push(hd, (uint32_t)c.ptr / BF_SDF_BLOCK_VOXELS);
            hd->d_hash[i] = freeE;
            hd->d_hash[prev].offset = c.offset;
            return 1;
        }
        if (c.offset == 0) return 0;
        prev = i;
        i = (last + c.offset) % total;
    }
    return 0;
}

/* garbageCollectIdentifyKernel + garbageCollectFreeKernel: CUDASceneRepHashSDF.cu:584-668.
 * The block maximum is taken through a uint shared array (:581,606 -- quirk Q13), i.e. the
 * block is garbage iff trunc(max weight) == 0.  Returns the number of blocks freed. */
ORC_API unsigned orc_tsdf_garbage_collect(BFHashDataStruct* hd, const BFHashParams* hp, unsigned numOccupied) {
    unsigned freed = 0;
    for (unsigned b = 0; b < numOccupied; ++b) {
        const BFHashEntry e = hd->d_hashCompactified[b];
        uint32_t mw = 0;
        for (unsigned i = 0; i < BF_SDF_BLOCK_VOXELS; i += 2) {
            float m = fmaxf(hd->d_SDFBlocks[(size_t)(uint32_t)e.ptr + i].weight, hd->d_SDFBlocks[(size_t)(uint32_t)e.ptr + i + 1].weight);
            uint32_t u = (m != m || m <= 0.0f) ? 0u : (m >= 4294967296.0f ? 0xFFFFFFFFu : (uint32_t)m);   /* cvt.rzi.u32.f32 */
            if (u > mw) mw = u;
        }
        hd->d_hashDecision[b] = (mw == 0) ? 1 : 0;
    }
    for (unsigned b = 0; b < numOccupied; ++b) {
        if (!hd->d_hashDecision[b]) continue;
        const BFHashEntry e = hd->d_hashCompactified[b];
        i3 p = { e.pos[0], e.pos[1], e.pos[2] };
        if (delete_entry(hd, hp, p)) {
            memset(&hd->d_SDFBlocks[(size_t)(uint32_t)e.ptr], 0, BF_SDF_BLOCK_VOXELS * sizeof(BFVoxel));
            ++freed;
        }
    }
    return freed;
}

/* ---------------------------------------------------------------------- */
/* BASELINE.json configs[0]: one frame into a dense D^3 grid ("mLib VoxelGrid" stand-in,
 * ml::Grid3 x-fastest layout external/mLib/include/core-base/grid3.h:42-45) with the same
 * per-voxel rule as integrateDepthMapKernel.  origin = world position of voxel (0,0,0). */
ORC_API unsigned long long orc_tsdf_integrate_dense(BFVoxel* grid, int D, float voxelSize, const float origin[3],
                                                    const BFHashParams* hp, const float* depthImg, const uint8_t* colorImg,
                                                    const BFDepthCameraParams* cp, int deIntegrate) {
    /* express the dense grid as D/8 ^3 pseudo-blocks sharing the hashed-path voxel rule */
    unsigned long long U = 0;
    const unsigned W = cp->m_imageWidth, H = cp->m_imageHeight;
    for (int z = 0; z < D; ++z) for (int y = 0; y < D; ++y) for (int x = 0; x < D; ++x) {
        f3 w = { origin[0] + (float)x * voxelSize, origin[1] + (float)y * voxelSize, origin[2] + (float)z * voxelSize };
        f3 pf = xform(&hp->m_rigidTransformInverse, w);
        float sx, sy;
        cam_to_screen_f(cp, pf, &sx, &sy);
        unsigned px = (unsigned)f2i(sx + 0.5f), py = (unsigned)f2i(sy + 0.5f);
        if (!(px < W && py < H)) continue;
        float depth = depthImg[py * W + px];
        if (depth == ORC_MINF || !(depth < hp->m_maxIntegrationDistance)) continue;
        float sdf = depth - pf.z;
        float trunc = truncation(hp, depth);
        if (!(fabsf(sdf) < trunc)) continue;
        if (sdf >= 0.0f) sdf = fminf(trunc, sdf); else sdf = fmaxf(-trunc, sdf);
        BFVoxel* v = &grid[((size_t)z * D + y) * D + x];
        const BFVoxel old = *v;
        BFVoxel nv;
        const uint8_t* c = colorImg ? &colorImg[4 * (py * W + px)] : NULL;
        for (int k = 0; k < 3; ++k) {
            float cc = c ? (float)c[k] : (k == 1 ? 255.0f : 0.0f), oc = old.color[k], r;
            if (!deIntegrate) r = (old.weight == 0) ? cc : fmaf(cc, 0.2f, 0.8f * oc);
            else r = fmaf(oc, old.weight, -cc) / (old.weight - 1.0f);
            nv.color[k] = f2u8(clamp_color(roundf(r)));
        }
        nv.color[3] = 255;
        if (!deIntegrate) {
            nv.sdf = fmaf(old.sdf, old.weight, sdf) / (1.0f + old.weight);
            nv.weight = fminf((float)hp->m_integrationWeightMax, 1.0f + old.weight);
        } else {
            nv.sdf = fmaf(old.sdf, old.weight, -sdf) / (old.weight - 1.0f);
            nv.weight = fmaxf(0.0f, old.weight - 1.0f);
            if (nv.weight <= 0.001f) { memset(&nv, 0, sizeof nv); }
        }
        *v = nv;
        ++U;
    }
    return U;
}

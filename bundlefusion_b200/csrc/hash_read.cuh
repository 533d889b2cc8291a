// hash_read.cuh -- read-only access to the hashed TSDF shared by the ray cast (raycast.cu) and the iso-surface extraction (marching_cubes.cu): block look-up,
// voxel fetch by world position, and the trilinear sample both walk the volume with; the block geometry and the bucket walk are voxel_hash.cuh's.
// Reference (FL/ = FriedLiver/Source/):
//   HashDataStruct::getVoxel(float3)                                                                                         FL/DepthSensing/VoxelUtilHashSDF.h:407-418
//   RayCastData::trilinearInterpolationSimpleFastFast                                                                        FL/DepthSensing/RayCastSDFUtil.h:100-121
// Arithmetic contract: IEEE binary32, every operation individually rounded (TUs built -fmad=false, -prec-div=true), the reference's expression order.
#pragma once
#include "../../include/bf_tsdf.h"
#include "bf_common.cuh"
#include "voxel_hash.cuh"

namespace bf {

__device__ __forceinline__ F3 add3(F3 a, F3 b) { return F3{ a.x + b.x, a.y + b.y, a.z + b.z }; }
__device__ __forceinline__ F3 sub3(F3 a, F3 b) { return F3{ a.x - b.x, a.y - b.y, a.z - b.z }; }
__device__ __forceinline__ F3 scale3(float s, F3 a) { return F3{ s * a.x, s * a.y, s * a.z }; }
__device__ __forceinline__ float dot3(F3 a, F3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ F3 normalize3(F3 v) { const float inv = 1.0f / sqrtf(dot3(v, v)); return F3{ v.x * inv, v.y * inv, v.z * inv }; }
__device__ __forceinline__ F3 mul_point(const float* M, F3 v) {      // float4x4 * float3 (w = 1), cuda_SimpleMatrixUtil.h:937-944
    return F3{ M[0] * v.x + M[1] * v.y + M[2] * v.z + M[3] * 1.0f, M[4] * v.x + M[5] * v.y + M[6] * v.z + M[7] * 1.0f, M[8] * v.x + M[9] * v.y + M[10] * v.z + M[11] * 1.0f };
}
__device__ __forceinline__ F3 mul_dir(const float* M, F3 v) {        // xyz of float4x4 * float4(v, 0), :925-933
    return F3{ M[0] * v.x + M[1] * v.y + M[2] * v.z + M[3] * 0.0f, M[4] * v.x + M[5] * v.y + M[6] * v.z + M[7] * 0.0f, M[8] * v.x + M[9] * v.y + M[10] * v.z + M[11] * 0.0f };
}
__device__ __forceinline__ int f2i_rz(float v) { return __float2int_rz(v); }                 // cvt.rzi.s32.f32: truncate, saturate, NaN -> 0

// ---- read-only hash access ----------------------------------------------------------------------------------------------------------
// an entry read through the read-only path: pos.xyz and ptr in one 16-byte load (entries are 16-byte aligned), the offset only when the walk
// follows it
struct LdgEntry { int4 q; const BFHashEntry* e; };
__device__ __forceinline__ bool entry_holds(const LdgEntry& e, I3 b) { return e.q.x == b.x && e.q.y == b.y && e.q.z == b.z && e.q.w != BF_FREE_ENTRY; }
__device__ __forceinline__ unsigned entry_offset(const LdgEntry& e) { return __ldg(&e.e->offset); }
// the block's first-voxel index or BF_FREE_ENTRY
__device__ inline int find_block(const BFHashDataStruct& hd, const BFHashParams& hp, I3 b) {
    const auto load = [&](unsigned i) { return LdgEntry{ __ldg(reinterpret_cast<const int4*>(&hd.d_hash[i])), &hd.d_hash[i] }; };
    return walk_bucket(hp, b, hash_pos(hp.m_hashNumBuckets, b), load, [](const LdgEntry& e, unsigned) { return e.q.w; }, (int)BF_FREE_ENTRY);
}
struct BlockCache { I3 b; int ptr; bool valid; };
struct VoxelW { float sdf, weight; unsigned color; };
// the voxel at integer position v, with the thread's last block kept; a missing block reads as the empty voxel
__device__ __forceinline__ VoxelW get_voxel_at(const BFHashDataStruct& hd, const BFHashParams& hp, I3 v, BlockCache& c) {
    const I3 b = voxel_to_block(v);
    if (!(c.valid && c.b.x == b.x && c.b.y == b.y && c.b.z == b.z)) { c.b = b; c.ptr = find_block(hd, hp, b); c.valid = true; }
    VoxelW r = { 0.0f, 0.0f, 0u };
    if (c.ptr == BF_FREE_ENTRY) return r;
    const int k = voxel_local_index(v);
    const unsigned* w = reinterpret_cast<const unsigned*>(hd.d_SDFBlocks + (size_t)c.ptr + (size_t)k);
    r.sdf = __uint_as_float(__ldg(w)); r.weight = __uint_as_float(__ldg(w + 1)); r.color = __ldg(w + 2);
    return r;
}
// HashDataStruct::getVoxel(const float3&), :407-418
__device__ __forceinline__ VoxelW get_voxel(const BFHashDataStruct& hd, const BFHashParams& hp, F3 pos, BlockCache& c) { return get_voxel_at(hd, hp, world_to_voxel(hp, pos), c); }
__device__ __forceinline__ float frac1(float v) { return v - floorf(v); }

// trilinearInterpolationSimpleFastFast, RayCastSDFUtil.h:100-121: false at the first empty corner, the partial sum stays in dist.  fetch(F3 worldPos) -> VoxelW is
// how a voxel is read (through the hash, or from a staged tile).
template <class Fetch>
__device__ __forceinline__ bool trilinear_with(const BFHashParams& hp, F3 pos, float& dist, unsigned& colorOut, Fetch fetch) {
    const float oSet = hp.m_virtualVoxelSize;
    const F3 half = { oSet / 2.0f, oSet / 2.0f, oSet / 2.0f };
    const F3 posDual = sub3(pos, half);
    const F3 w = { frac1(pos.x / oSet), frac1(pos.y / oSet), frac1(pos.z / oSet) };
    dist = 0.0f;
    float cx = 0.0f, cy = 0.0f, cz = 0.0f;
    // corners in the reference's order: 000 100 010 001 110 011 101 111
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int ox = (k == 1 || k == 4 || k == 6 || k == 7), oy = (k == 2 || k == 4 || k == 5 || k == 7), oz = (k == 3 || k == 5 || k == 6 || k == 7);
        const F3 off = { ox ? oSet : 0.0f, oy ? oSet : 0.0f, oz ? oSet : 0.0f };
        const VoxelW v = fetch(add3(posDual, off));
        if (v.weight == 0) return false;
        const float wx = ox ? w.x : (1.0f - w.x), wy = oy ? w.y : (1.0f - w.y), wz = oz ? w.z : (1.0f - w.z);
        const float ww = wx * wy * wz;
        dist += ww * v.sdf;
        cx += ww * (float)(v.color & 0xffu); cy += ww * (float)((v.color >> 8) & 0xffu); cz += ww * (float)((v.color >> 16) & 0xffu);
    }
    colorOut = ((unsigned)f2i_rz(cx) & 0xffu) | (((unsigned)f2i_rz(cy) & 0xffu) << 8) | (((unsigned)f2i_rz(cz) & 0xffu) << 16);          // make_uchar3(float, float, float)
    return true;
}
__device__ inline bool trilinear(const BFHashDataStruct& hd, const BFHashParams& hp, F3 pos, float& dist, unsigned& colorOut, BlockCache& bc) {
    return trilinear_with(hp, pos, dist, colorOut, [&](F3 q) { return get_voxel(hd, hp, q, bc); });
}

}  // namespace bf

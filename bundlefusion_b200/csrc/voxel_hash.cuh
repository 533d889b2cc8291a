// voxel_hash.cuh -- the voxel hash's block geometry and look-up, stated once for every kernel that writes or reads the hash: the TSDF
// (tsdf.cu, tsdf_hash.cuh), the block keys (tsdf_keys.cuh), the ray cast and the iso-surface extraction (hash_read.cuh).  Reference
// (FL/ = FriedLiver/Source/): computeHashPos, worldToVirtualVoxelPos, virtualVoxelPosToSDFBlock, SDFBlockToVirtualVoxelPos,
// virtualVoxelPosToWorld, virtualVoxelPosToLocalSDFBlockIndex, getHashEntryForSDFBlockPos   FL/DepthSensing/VoxelUtilHashSDF.h:226-358, 440-485
// The float conversions are the reference's expressions, one rounding each, so FMA contraction cannot change them; the translation units
// that use them are built -prec-div=true.  The CPU suite compiles this header against tests/cuda_emu.
#pragma once
#include <cuda_runtime.h>

#include "../../include/bf_tsdf.h"

namespace bf {

struct I3 { int x, y, z; };
struct F3 { float x, y, z; };

__device__ __forceinline__ int isign(float v) { return (0.0f < v) - (v < 0.0f); }

// computeHashPos, :226-234 (unsigned modulo, see oracle note)
__device__ __forceinline__ unsigned hash_pos(unsigned numBuckets, I3 p) {
    return (((unsigned)p.x * 73856093u) ^ ((unsigned)p.y * 19349669u) ^ ((unsigned)p.z * 83492791u)) % numBuckets;
}

// worldToVirtualVoxelPos, :283-287 (cvt.rzi.s32.f32: truncate, saturate, NaN -> 0)
__device__ __forceinline__ I3 world_to_voxel(const BFHashParams& hp, F3 pos) {
    const float vs = hp.m_virtualVoxelSize;
    const F3 p = { pos.x / vs, pos.y / vs, pos.z / vs };
    return I3{ __float2int_rz(p.x + (float)isign(p.x) * 0.5f), __float2int_rz(p.y + (float)isign(p.y) * 0.5f), __float2int_rz(p.z + (float)isign(p.z) * 0.5f) };
}
// virtualVoxelPosToSDFBlock, :290-299
__device__ __forceinline__ I3 voxel_to_block(I3 v) {
    if (v.x < 0) v.x -= BF_SDF_BLOCK_SIZE - 1;
    if (v.y < 0) v.y -= BF_SDF_BLOCK_SIZE - 1;
    if (v.z < 0) v.z -= BF_SDF_BLOCK_SIZE - 1;
    return I3{ v.x / BF_SDF_BLOCK_SIZE, v.y / BF_SDF_BLOCK_SIZE, v.z / BF_SDF_BLOCK_SIZE };
}
// SDFBlockToVirtualVoxelPos, :303-305
__device__ __forceinline__ I3 block_to_voxel(I3 b) { return I3{ b.x * BF_SDF_BLOCK_SIZE, b.y * BF_SDF_BLOCK_SIZE, b.z * BF_SDF_BLOCK_SIZE }; }
// virtualVoxelPosToWorld, :308-310
__device__ __forceinline__ F3 voxel_to_world(const BFHashParams& hp, I3 v) {
    return F3{ (float)v.x * hp.m_virtualVoxelSize, (float)v.y * hp.m_virtualVoxelSize, (float)v.z * hp.m_virtualVoxelSize };
}
__device__ __forceinline__ F3 block_to_world(const BFHashParams& hp, I3 b) { return voxel_to_world(hp, block_to_voxel(b)); }
__device__ __forceinline__ I3 world_to_block(const BFHashParams& hp, F3 w) { return voxel_to_block(world_to_voxel(hp, w)); }
// virtualVoxelPosToLocalSDFBlockIndex, :347-358: the voxel's index in its block's BF_SDF_BLOCK_VOXELS
__device__ __forceinline__ int voxel_local_index(I3 v) {
    I3 l = { v.x % BF_SDF_BLOCK_SIZE, v.y % BF_SDF_BLOCK_SIZE, v.z % BF_SDF_BLOCK_SIZE };
    if (l.x < 0) l.x += BF_SDF_BLOCK_SIZE;
    if (l.y < 0) l.y += BF_SDF_BLOCK_SIZE;
    if (l.z < 0) l.z += BF_SDF_BLOCK_SIZE;
    return l.z * BF_SDF_BLOCK_SIZE * BF_SDF_BLOCK_SIZE + l.y * BF_SDF_BLOCK_SIZE + l.x;
}

// ---- look-up ------------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool entry_holds(const BFHashEntry& e, I3 b) {
    return e.pos[0] == b.x && e.pos[1] == b.y && e.pos[2] == b.z && e.ptr != BF_FREE_ENTRY;
}
__device__ __forceinline__ unsigned entry_offset(const BFHashEntry& e) { return e.offset; }

// getHashEntryForSDFBlockPos, :440-485: bucket h's entries, then the overflow list that starts at its last entry.  load(i) gives entry i and
// the walk reads it through entry_holds and entry_offset, so the caller picks its loads by what load returns: a reference into the table
// (plain loads; a bucket entry's fields are read only as far as the test needs them, a list entry is copied whole, offset included), a copy
// it loaded itself (__ldcg), or a type of its own with its own entry_holds / entry_offset.  found(e, i) is the result for the entry e at
// index i that holds block b, `missing` the result when no entry does.
template <class Load, class Found, class R>
__device__ __forceinline__ R walk_bucket(const BFHashParams& hp, I3 b, unsigned h, Load load, Found found, R missing) {
    const unsigned hpz = h * BF_HASH_BUCKET_SIZE, total = BF_HASH_BUCKET_SIZE * hp.m_hashNumBuckets;
#pragma unroll
    for (unsigned j = 0; j < BF_HASH_BUCKET_SIZE; ++j) {
        const auto& e = load(hpz + j);
        if (entry_holds(e, b)) return found(e, hpz + j);
    }
    const unsigned last = hpz + BF_HASH_BUCKET_SIZE - 1;
    unsigned i = last;
    for (unsigned it = 0; it < hp.m_hashMaxCollisionLinkedListSize; ++it) {
        const auto e = load(i);
        if (entry_holds(e, b)) return found(e, i);
        const unsigned off = entry_offset(e);
        if (off == 0) break;
        i = (last + off) % total;
    }
    return missing;
}

}  // namespace bf

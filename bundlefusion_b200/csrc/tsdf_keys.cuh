// tsdf_keys.cuh -- SDF-block positions as packed 64-bit keys, bucket loads under the voxel hash's bucket function, and the device key set that
// bfTsdfCountBlocks fills and bfTsdfBlockKeyLoad / bfTsdfBlockKeyMerge read (include/bf_tsdf.h).  Integer code only, so tsdf.cu
// (built -fmad=false) includes it unchanged and the CPU suite compiles it against tests/cuda_emu.
#pragma once
#include <cuda_runtime.h>

#include "../../include/bf_tsdf.h"
#include "voxel_hash.cuh"

namespace bf {

// key = bit 63 | three 21-bit fields biased by 2^20 (x, y, z from the top): a block with every coordinate in [-2^20, 2^20) packs, and
// no key is 0, the key set's empty slot
#define BF_BLOCK_KEY_LIM (1 << 20)
__device__ __forceinline__ bool block_key_packable(I3 b) {
    return b.x >= -BF_BLOCK_KEY_LIM && b.x < BF_BLOCK_KEY_LIM && b.y >= -BF_BLOCK_KEY_LIM && b.y < BF_BLOCK_KEY_LIM &&
           b.z >= -BF_BLOCK_KEY_LIM && b.z < BF_BLOCK_KEY_LIM;
}
__device__ __forceinline__ unsigned long long pack_block_key(I3 b) {
    const int lim = BF_BLOCK_KEY_LIM;
    return (1ull << 63) | ((unsigned long long)(unsigned)(b.x + lim) << 42) | ((unsigned long long)(unsigned)(b.y + lim) << 21) |
           (unsigned long long)(unsigned)(b.z + lim);
}
__device__ __forceinline__ I3 unpack_block_key(unsigned long long key) {
    const int lim = 1 << 20;
    I3 b = { (int)((key >> 42) & 0x1FFFFF) - lim, (int)((key >> 21) & 0x1FFFFF) - lim, (int)(key & 0x1FFFFF) - lim };
    return b;
}

// ---- the key set: open addressing over a power-of-two capacity, linear probing over every slot ---------------------------------------
enum { KEYSET_STORED = 0, KEYSET_REFUSED = 1, KEYSET_OUT_OF_RANGE = 2 };

__device__ __forceinline__ unsigned keyset_home(unsigned long long key, unsigned mask) {
    key ^= key >> 33; key *= 0xff51afd7ed558ccdull; key ^= key >> 33;       // the fields are dense small integers: mix before masking
    return (unsigned)key & mask;
}
// stores `key` once; a key that finds every slot taken by other keys is refused and counted, nothing is written
__device__ __forceinline__ void keyset_insert(unsigned long long* keys, unsigned mask, unsigned* ctrs, unsigned long long key) {
    unsigned i = keyset_home(key, mask);
    for (unsigned n = 0; n <= mask; ++n, i = (i + 1u) & mask) {
        unsigned long long cur = __ldcg(&keys[i]);
        if (cur == 0ull) {
            cur = atomicCAS(&keys[i], 0ull, key);
            if (cur == 0ull) { atomicAdd(&ctrs[KEYSET_STORED], 1u); return; }
        }
        if (cur == key) return;
    }
    atomicAdd(&ctrs[KEYSET_REFUSED], 1u);
}
__device__ __forceinline__ void keyset_insert_block(unsigned long long* keys, unsigned mask, unsigned* ctrs, I3 b) {
    if (!block_key_packable(b)) { atomicAdd(&ctrs[KEYSET_OUT_OF_RANGE], 1u); return; }
    keyset_insert(keys, mask, ctrs, pack_block_key(b));
}

// every key of src[0, n) into the set (bfTsdfBlockKeyMerge: growing a set)
__global__ void __launch_bounds__(256) keyset_merge_kernel(unsigned long long* keys, unsigned mask, unsigned* ctrs, const unsigned long long* __restrict__ src, unsigned n) {
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long key = src[i];
        if (key != 0ull) keyset_insert(keys, mask, ctrs, key);
    }
}

// bucket loads of the keys of slots [0, n) for numBuckets buckets of hash_pos: load[h] (zeroed by the caller) and out = { keys, largest load,
// sum over buckets of max(0, load - BF_HASH_BUCKET_SIZE) } (zeroed by the caller).  A key that arrives in its bucket when the bucket already
// holds BF_HASH_BUCKET_SIZE or more adds one to the overflow sum, so the sum comes out of the same atomic that counts the load.
__global__ void __launch_bounds__(256) bucket_load_kernel(const unsigned long long* __restrict__ keys, unsigned n, unsigned numBuckets, unsigned* load, unsigned* out) {
    unsigned cnt = 0, over = 0, mx = 0;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long key = keys[i];
        if (key == 0ull) continue;
        const unsigned before = atomicAdd(&load[hash_pos(numBuckets, unpack_block_key(key))], 1u);
        ++cnt;
        if (before >= BF_HASH_BUCKET_SIZE) ++over;
        if (before + 1u > mx) mx = before + 1u;
    }
    if (cnt) { atomicAdd(&out[0], cnt); atomicMax(&out[1], mx); }
    if (over) atomicAdd(&out[2], over);
}

}  // namespace bf

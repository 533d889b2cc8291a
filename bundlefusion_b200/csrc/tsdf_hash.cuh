// tsdf_hash.cuh -- the voxel hash's entry primitives (lookup, bucket locks, heap pop, the insertion rule alloc_block) and the rehash
// kernels of bfTsdfRehash (include/bf_tsdf.h), which move a table's live blocks into another table through that same insertion rule.
// Integer code only: tsdf.cu (built -fmad=false) includes it, and the CPU suite compiles it against tests/cuda_emu.
#pragma once
#include <cuda_runtime.h>

#include "../../include/bf_tsdf.h"
#include "tsdf_shared.cuh"
#include "tsdf_keys.cuh"          // and through it voxel_hash.cuh

namespace bf {

// ------------------------------------------------------------------------------------------
// hash table primitives.  Entry = 5 ints (20 B).  Loads on the lock-free fast path may come
// from L1 (possibly stale => at worst a spurious miss that is re-checked under the lock);
// loads under a bucket lock use ld.global.cg (L2), stores are followed by __threadfence().
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ BFHashEntry load_entry_cg(const BFHashEntry* e) {
    BFHashEntry r;
    const int* s = reinterpret_cast<const int*>(e);
    r.pos[0] = __ldcg(s + 0); r.pos[1] = __ldcg(s + 1); r.pos[2] = __ldcg(s + 2); r.ptr = __ldcg(s + 3);
    r.offset = (unsigned)__ldcg(s + 4);
    return r;
}

// the entry index of block p in bucket h or its overflow list, or -1.  kCoherent: read through L2.
template <bool kCoherent>
__device__ int find_entry(const BFHashEntry* __restrict__ hash, const BFHashParams& hp, I3 p, unsigned h) {
    const auto index = [](const BFHashEntry&, unsigned i) { return (int)i; };
    if constexpr (kCoherent) return walk_bucket(hp, p, h, [&](unsigned i) { return load_entry_cg(&hash[i]); }, index, -1);
    else return walk_bucket(hp, p, h, [&](unsigned i) -> const BFHashEntry& { return hash[i]; }, index, -1);
}

__device__ __forceinline__ bool try_lock(int* mutex) { return atomicCAS(mutex, BF_FREE_ENTRY, BF_LOCK_ENTRY) == BF_FREE_ENTRY; }
__device__ __forceinline__ void unlock(int* mutex) { __threadfence(); atomicExch(mutex, BF_FREE_ENTRY); }

// VoxelUtilHashSDF.h:535-540 consumeHeap, plus an exhaustion guard (the reference has none)
__device__ __forceinline__ bool heap_pop(unsigned* heap, unsigned* heapCounter, unsigned* slot) {
    unsigned addr = atomicSub(heapCounter, 1u);
    if (addr == 0xFFFFFFFFu || addr >= 0x80000000u) { atomicAdd(heapCounter, 1u); return false; }
    *slot = __ldcg(&heap[addr]);
    return true;
}

__device__ __forceinline__ void write_entry(BFHashEntry* e, I3 p, unsigned offset, int ptr) {
    int* d = reinterpret_cast<int*>(e);
    __stcg(d + 0, p.x); __stcg(d + 1, p.y); __stcg(d + 2, p.z); __stcg(d + 4, (int)offset);
    __threadfence();
    __stcg(d + 3, ptr);       // ptr last: a reader that sees a valid ptr sees a valid pos
}

// Insert `pos` (VoxelUtilHashSDF.h:549-655 semantics: bucket slot first, else splice into the
// bucket's overflow list).  Unlike the reference (try-lock, give up, host retries) this spins
// until the block is present, so one launch reaches the reference's fixed point.
// slotEpoch / tag (optional): batch re-integration -- a block inserted by THIS launch is tagged with (batch id << 8 | op index), so that the
// multi-op stencil can tell which operations of the batch saw the block exist (tsdf_reintegrate_batch)
struct AllocEpoch { unsigned* slotEpoch; unsigned tag; };
__device__ void alloc_block(const BFHashDataStruct& hd, const BFHashParams& hp, int4* slotInfo, unsigned* ctrs, I3 pos, AllocEpoch ep = AllocEpoch{nullptr, 0u}) {
    const unsigned h = hash_pos(hp.m_hashNumBuckets, pos);
    if (find_entry<false>(hd.d_hash, hp, pos, h) >= 0) return;      // fast path, no lock

    const unsigned hpz = h * BF_HASH_BUCKET_SIZE;
    const unsigned last = hpz + BF_HASH_BUCKET_SIZE - 1;
    const unsigned total = BF_HASH_BUCKET_SIZE * hp.m_hashNumBuckets;
    const unsigned maxLoop = hp.m_hashMaxCollisionLinkedListSize;
    int* mutexH = &hd.d_hashBucketMutex[h];

    bool done = false;
    unsigned backoff = 32;
    while (!done) {
        if (try_lock(mutexH)) {
            __threadfence();
            if (find_entry<true>(hd.d_hash, hp, pos, h) >= 0) { unlock(mutexH); return; }
            // first free slot of the home bucket
            int firstEmpty = -1;
#pragma unroll
            for (unsigned j = 0; j < BF_HASH_BUCKET_SIZE; ++j) {
                int p = __ldcg(&hd.d_hash[hpz + j].ptr);
                if (firstEmpty == -1 && p == BF_FREE_ENTRY) firstEmpty = (int)(hpz + j);
            }
            if (firstEmpty != -1) {
                unsigned slot;
                if (heap_pop(hd.d_heap, hd.d_heapCounter, &slot)) {
                    slotInfo[slot] = make_int4(pos.x, pos.y, pos.z, firstEmpty);
                    if (ep.slotEpoch) ep.slotEpoch[slot] = ep.tag;
                    atomicMax(&ctrs[CTR_HIGH_WATER], slot + 1u);
                    write_entry(&hd.d_hash[firstEmpty], pos, BF_NO_OFFSET, (int)(slot * BF_SDF_BLOCK_VOXELS));
                } else {
                    atomicAdd(&ctrs[CTR_HEAP_FAIL], 1u);
                }
                unlock(mutexH);
                return;
            }
            // overflow: probe forward for a free non-bucket-last slot (:614-654)
            unsigned offset = 0, it = 0;
            bool retry = false;
            while (it < maxLoop) {
                offset++;
                const unsigned i = (last + offset) % total;
                if ((offset % BF_HASH_BUCKET_SIZE) == 0) continue;
                if (__ldcg(&hd.d_hash[i].ptr) == BF_FREE_ENTRY) {
                    const unsigned h2 = i / BF_HASH_BUCKET_SIZE;
                    int* mutex2 = &hd.d_hashBucketMutex[h2];
                    const bool same = (h2 == h);
                    if (!same && !try_lock(mutex2)) { retry = true; break; }   // avoid lock-order deadlock
                    __threadfence();
                    if (__ldcg(&hd.d_hash[i].ptr) == BF_FREE_ENTRY) {
                        unsigned slot;
                        if (heap_pop(hd.d_heap, hd.d_heapCounter, &slot)) {
                            const unsigned lastOffset = (unsigned)__ldcg(reinterpret_cast<const int*>(&hd.d_hash[last]) + 4);
                            slotInfo[slot] = make_int4(pos.x, pos.y, pos.z, (int)i);
                            if (ep.slotEpoch) ep.slotEpoch[slot] = ep.tag;
                            atomicMax(&ctrs[CTR_HIGH_WATER], slot + 1u);
                            write_entry(&hd.d_hash[i], pos, lastOffset, (int)(slot * BF_SDF_BLOCK_VOXELS));
                            __threadfence();
                            __stcg(reinterpret_cast<int*>(&hd.d_hash[last]) + 4, (int)offset);   // publish: head -> new
                        } else {
                            atomicAdd(&ctrs[CTR_HEAP_FAIL], 1u);
                        }
                        if (!same) unlock(mutex2);
                        unlock(mutexH);
                        return;
                    }
                    if (!same) unlock(mutex2);
                    // slot was taken meanwhile: keep probing (does not count as an iteration)
                    continue;
                }
                it++;
            }
            unlock(mutexH);
            if (!retry) { atomicAdd(&ctrs[CTR_DROPPED], 1u); return; }   // no room within the probe window: dropped (as the reference)
        }
        __nanosleep(backoff + ((threadIdx.x * 7u) & 63u));     // jitter: break lock-step livelock inside a warp
        if (backoff < 1024) backoff <<= 1;
    }
}

// deleteHashEntryElement (VoxelUtilHashSDF.h:739-826) under the home bucket's spin lock.
__device__ bool delete_entry(const BFHashDataStruct& hd, const BFHashParams& hp, int4* slotInfo, I3 p) {
    const unsigned h = hash_pos(hp.m_hashNumBuckets, p);
    const unsigned hpz = h * BF_HASH_BUCKET_SIZE;
    const unsigned last = hpz + BF_HASH_BUCKET_SIZE - 1;
    const unsigned total = BF_HASH_BUCKET_SIZE * hp.m_hashNumBuckets;
    int* mutexH = &hd.d_hashBucketMutex[h];
    unsigned backoff = 32;
    while (!try_lock(mutexH)) { __nanosleep(backoff); if (backoff < 1024) backoff <<= 1; }
    __threadfence();
    bool ok = false;
    BFHashEntry freeE; freeE.pos[0] = freeE.pos[1] = freeE.pos[2] = 0; freeE.ptr = BF_FREE_ENTRY; freeE.offset = 0;
    for (unsigned j = 0; j < BF_HASH_BUCKET_SIZE && !ok; ++j) {
        const unsigned i = hpz + j;
        const BFHashEntry c = load_entry_cg(&hd.d_hash[i]);
        if (entry_holds(c, p)) {
            const unsigned slot = (unsigned)c.ptr / BF_SDF_BLOCK_VOXELS;
            const unsigned addr = atomicAdd(hd.d_heapCounter, 1u);            // appendHeap :541-546
            hd.d_heap[addr + 1] = slot;
            slotInfo[slot] = make_int4(0, 0, 0, -1);
            if (c.offset != 0) {
                const unsigned next = (i + c.offset) % total;
                const BFHashEntry n = load_entry_cg(&hd.d_hash[next]);
                hd.d_hash[i] = n;
                if (n.ptr >= 0) slotInfo[(unsigned)n.ptr / BF_SDF_BLOCK_VOXELS].w = (int)i;   // the moved entry changed index
                hd.d_hash[next] = freeE;
            } else {
                hd.d_hash[i] = freeE;
            }
            ok = true;
        }
    }
    if (!ok) {
        BFHashEntry c = load_entry_cg(&hd.d_hash[last]);
        unsigned prev = last;
        unsigned i = (last + c.offset) % total;
        for (unsigned it = 0; it < hp.m_hashMaxCollisionLinkedListSize; ++it) {
            c = load_entry_cg(&hd.d_hash[i]);
            if (entry_holds(c, p)) {
                const unsigned slot = (unsigned)c.ptr / BF_SDF_BLOCK_VOXELS;
                const unsigned addr = atomicAdd(hd.d_heapCounter, 1u);
                hd.d_heap[addr + 1] = slot;
                slotInfo[slot] = make_int4(0, 0, 0, -1);
                hd.d_hash[i] = freeE;
                hd.d_hash[prev].offset = c.offset;
                ok = true;
                break;
            }
            if (c.offset == 0) break;
            prev = i;
            i = (last + c.offset) % total;
        }
    }
    unlock(mutexH);
    return ok;
}


// ---- rehash (bfTsdfRehash) ----------------------------------------------------------------------------------------------------------------
// One CTA walks the source's slot table (slotInfo: 16 B per ever-allocated slot, dense, read coalesced up to its high-water mark -- the
// entry table of a large hash is mostly empty and 32 B per entry) in chunks of BF_REHASH_CHUNK slots.  The chunk's live slots are compacted
// in shared memory; one thread per live block inserts it into dst through alloc_block, the insertion rule of every alloc launch, and looks up
// the slot it landed in; then the whole CTA moves the chunk's voxel blocks with 16-byte loads and stores, four in flight per thread.
// slotMap[src slot] = dst slot (0xFFFFFFFF: no block moved from it); out[0] += blocks moved, out[1] += blocks dst could not take.
#define BF_REHASH_CHUNK 256
#define BF_BLOCK_VEC (BF_SDF_BLOCK_VOXELS * (int)sizeof(BFVoxel) / 16)      // 384 16-byte words per voxel block
__global__ void __launch_bounds__(BF_REHASH_CHUNK)
rehash_kernel(BFHashDataStruct src, BFHashDataStruct dst, const __grid_constant__ BFHashParams dhp, const int4* __restrict__ srcSlotInfo,
              const unsigned* __restrict__ srcCtrs, const int* __restrict__ srcLive, int4* dstSlotInfo, unsigned* dstCtrs, int* __restrict__ dstLive,
              unsigned* __restrict__ slotMap, unsigned* out) {
    __shared__ int4 sInfo[BF_REHASH_CHUNK];     // {x, y, z, source slot} of the chunk's live blocks
    __shared__ int sDst[BF_REHASH_CHUNK];       // their slots in dst (-1: not taken)
    __shared__ unsigned sN;
    const unsigned highWater = srcCtrs[CTR_HIGH_WATER];
    const unsigned tid = threadIdx.x, lane = tid & 31u;
    for (unsigned base = blockIdx.x * BF_REHASH_CHUNK; base < highWater; base += gridDim.x * BF_REHASH_CHUNK) {
        if (tid == 0) sN = 0;
        __syncthreads();
        const unsigned slot = base + tid;
        const int4 info = slot < highWater ? srcSlotInfo[slot] : make_int4(0, 0, 0, -1);
        const unsigned ballot = __ballot_sync(0xffffffffu, info.w >= 0);
        unsigned wbase = 0;
        if (lane == 0 && ballot) wbase = atomicAdd(&sN, (unsigned)__popc(ballot));
        wbase = __shfl_sync(0xffffffffu, wbase, 0);
        if (info.w >= 0) sInfo[wbase + __popc(ballot & ((1u << lane) - 1u))] = make_int4(info.x, info.y, info.z, (int)slot);
        __syncthreads();
        const unsigned n = sN;
        if (tid < n) {
            const int4 s = sInfo[tid];
            const I3 p = { s.x, s.y, s.z };
            alloc_block(dst, dhp, dstSlotInfo, dstCtrs, p);
            const int e = find_entry<true>(dst.d_hash, dhp, p, hash_pos(dhp.m_hashNumBuckets, p));
            const int d = e >= 0 ? __ldcg(&dst.d_hash[e].ptr) / BF_SDF_BLOCK_VOXELS : -1;
            sDst[tid] = d;
            slotMap[s.w] = d >= 0 ? (unsigned)d : 0xFFFFFFFFu;
            if (d >= 0) dstLive[d] = srcLive[s.w];
            atomicAdd(&out[d >= 0 ? 0 : 1], 1u);
        }
        __syncthreads();
        const uint4* __restrict__ sv = reinterpret_cast<const uint4*>(src.d_SDFBlocks);
        uint4* __restrict__ dv = reinterpret_cast<uint4*>(dst.d_SDFBlocks);
        const unsigned total = n * BF_BLOCK_VEC;
        for (unsigned j0 = tid; j0 < total; j0 += 4 * BF_REHASH_CHUNK) {
            uint4 v[4];
            size_t to[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const unsigned j = j0 + u * BF_REHASH_CHUNK;
                to[u] = ~(size_t)0;
                if (j < total) {
                    const unsigned b = j / BF_BLOCK_VEC, w = j - b * BF_BLOCK_VEC;
                    const int d = sDst[b];
                    if (d >= 0) { v[u] = sv[(size_t)sInfo[b].w * BF_BLOCK_VEC + w]; to[u] = (size_t)d * BF_BLOCK_VEC + w; }
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (to[u] != ~(size_t)0) dv[to[u]] = v[u];
        }
        __syncthreads();
    }
}

// src's last compactified list in dst, entry for entry in the same order: each ptr moved to the slot its block went to, the offset of the entry
// that now holds the block, the GC flags as they were.  An entry whose source slot no longer holds a block (a block the last GC freed) points at
// a free slot of dst, whose zero voxels and zero live count decide as the freed slot's do.  Thread 0 also copies the list count and every counter
// but the slot high-water mark, which dst's inserts set, and adds src's dropped-insert counters to dst's.  One thread per list entry.
__global__ void __launch_bounds__(256)
rehash_list_kernel(BFHashDataStruct src, BFHashDataStruct dst, const unsigned* __restrict__ srcCtrs, unsigned* dstCtrs, int set,
                   const int4* __restrict__ dstSlotInfo, const unsigned* __restrict__ slotMap, const unsigned char* __restrict__ srcFlags,
                   unsigned char* __restrict__ dstFlags) {
    const unsigned count = srcCtrs[set + SET_COUNT];
    const unsigned tid = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned top = __ldcg(dst.d_heapCounter);
    const unsigned freeSlot = top < 0x80000000u ? __ldcg(&dst.d_heap[top]) : 0u;
    for (unsigned k = tid; k < count; k += gridDim.x * blockDim.x) {
        BFHashEntry e = src.d_hashCompactified[k];
        const unsigned m = slotMap[(unsigned)e.ptr / BF_SDF_BLOCK_VOXELS];
        const unsigned d = m != 0xFFFFFFFFu ? m : freeSlot;
        e.ptr = (int)(d * BF_SDF_BLOCK_VOXELS);
        const int w = dstSlotInfo[d].w;
        e.offset = w >= 0 ? dst.d_hash[w].offset : 0u;
        dst.d_hashCompactified[k] = e;
        dstFlags[k] = srcFlags[k];
    }
    if (tid == 0) {
        for (int i = 0; i < CTR_NUM; ++i)
            if (i != CTR_HIGH_WATER) dstCtrs[i] = (i == CTR_HEAP_FAIL || i == CTR_DROPPED) ? dstCtrs[i] + srcCtrs[i] : srcCtrs[i];
        dst.d_hashCompactifiedCounter[0] = src.d_hashCompactifiedCounter[0];
    }
}

}  // namespace bf

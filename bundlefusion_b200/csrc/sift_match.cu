// sift_match.cu -- SIFT descriptor matching for sm_90a.  Implements include/bf_sift.h (row a18 of SURVEY.md section 8).
//
// Behavioural source (what, not how): FL/SiftGPU/ProgramCU.cu:1634-1938 (MultiplyDescriptor / RowMatch / ColMatch kernels),
// FL/SiftGPU/SiftMatch.cpp:160-196, FL/Bundler.cpp:116-137.
//
// Design:
//  * the n1 x n2 dot-product matrix is NEVER written to memory.  The reference writes it (4 MB per pair at 1024 keys), re-reads it
//    in RowMatch, and keeps a second (n1/4) x n2 int4 array for the column pass; here each CTA sweeps the u8 x u8 -> s32 tensor-core
//    products (wgmma, exact) of 128 features against ALL features of the other image and keeps, per feature, the two largest
//    (value, index) in registers;
//  * the column direction is the same kernel with the two images swapped (the contraction is ~2 % of the kernel's instructions, the
//    best / second bookkeeping is the cost) and the reference's column tie-break, followed in the same CTA by the distance / ratio
//    tests, the mutual-best check against the row pass, and the append;
//  * all pairs of a frame are ONE batch: two launches in total instead of (2 copies + 3 launches + 1 memset) per pair.
#include <cuda.h>

#include <atomic>
#include <cstring>
#include <map>
#include <mutex>
#include <vector>

#include "../../include/bf_sift.h"
#include "bf_common.cuh"
#include "sift_pairs.cuh"
#include "sift_sweep.cuh"

namespace bf {

extern unsigned long long g_launchCount;

// Winner among equal maxima, exactly as the reference's 32 strided lanes + fold-upper-half-into-lower tree pick it (see
// oracle/sift_oracle.c): smallest (bit-reversed lane, position), lane = col % 32 for rows and (row / 4) % 32 for columns.
template <bool kColumnPass>
__device__ __forceinline__ unsigned tie_key(unsigned idx) {
    const unsigned lane = kColumnPass ? ((idx >> 2) & 31u) : (idx & 31u);
    return ((__brev(lane) >> 27) << 24) | idx;
}
// Per-feature running state: the largest value with the tie key of its index, and the second largest VALUE of the multiset (its
// index never matters).  A product can only change the state if it beats the second value or ties the first, which after the first
// few tiles almost none does: the common case is two integer compares.
struct Top2 { int v1; unsigned k1; int v2; };
template <bool kColumnPass>
__device__ __forceinline__ void top2_update(Top2& s, int v, unsigned idx) {
    if (v > s.v2 || (v == s.v1 && v > 0)) {
        const unsigned key = tie_key<kColumnPass>(idx);
        if (v > s.v1) { s.v2 = s.v1; s.v1 = v; s.k1 = key; }
        else if (v == s.v1) { s.v2 = v; if (key < s.k1) s.k1 = key; }
        else s.v2 = v;
    }
}
// union of two states (order-independent)
__device__ __forceinline__ void top2_merge(Top2& s, int ov1, unsigned ok1, int ov2) {
    if (ov1 > s.v1) { s.v2 = max(s.v1, ov2); s.v1 = ov1; s.k1 = ok1; }
    else if (ov1 == s.v1) { if (ov1 > 0) { s.v2 = ov1; if (ok1 < s.k1) s.k1 = ok1; } }
    else s.v2 = max(s.v2, ov1);
}
__device__ __forceinline__ float dist_of(int dot) { return acosf(fminf((float)dot * 0.000003814697265625f, 1.0f)); }

// the end of a feature's sweep: distance / ratio tests, then the row result (RowMatch_Kernel, ProgramCU.cu:1823-1829) or the mutual-best check of
// the column pass (ColMatch_Kernel, :1900-1915; here A = image 2, r = its feature)
template <bool kColumnPass>
__device__ __forceinline__ void finish_feature(const SiftJobDev& job, int r, const Top2& st, float distmax, float ratiomax) {
    if (r >= job.nA) return;
    const int vmax = st.v1, vnxt = st.v2;
    const int idx = (vmax > 0) ? (int)(st.k1 & 0x00FFFFFFu) : -1;
    const float dist = dist_of(vmax), distn = dist_of(vnxt);
    const int res = (dist < distmax && dist < distn * ratiomax) ? idx : -1;
    if (!kColumnPass) { job.rowResult[r] = res; job.rowDist[r] = dist; }
    else job.colResult[r] = (res >= 0 && job.rowResult[res] == r) ? res : -1;
}
// The reference appends its matches with an atomicAdd: beyond the 128-slot cap the kept subset depends on the scheduling.  Here the job's last
// CTA to finish compacts the per-feature results in ascending image-2 feature: the first 128 are kept, the counter still holds the total.
// Any block of <= 16 warps (all of them call); ctasOfJob: CTAs of this launch that work on the job.
__device__ __forceinline__ void compact_job(const SiftJobDev& job, int ctasOfJob) {
    __shared__ int sLast, sWarp[16];
    const unsigned t = threadIdx.x, lane = t & 31, warp = t >> 5, nWarps = blockDim.x >> 5;
    const int nA = job.nA;
    __threadfence();
    __syncthreads();
    if (t == 0) sLast = (atomicAdd(job.done, 1) == ctasOfJob - 1) ? 1 : 0;
    __syncthreads();
    if (!sLast) return;
    __threadfence();
    int base = 0;
    for (int r0 = 0; r0 < nA; r0 += (int)blockDim.x) {
        const int r = r0 + (int)t;
        const int res = (r < nA) ? __ldcg(&job.colResult[r]) : -1;
        const unsigned bal = __ballot_sync(0xffffffffu, res >= 0);
        if (lane == 0) sWarp[warp] = __popc(bal);
        __syncthreads();
        int off = base;
        for (unsigned w = 0; w < warp; ++w) off += sWarp[w];
        const int slot = off + __popc(bal & ((1u << lane) - 1u));
        if (res >= 0 && slot < BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW) {
            job.outIdx[slot] = make_uint2((unsigned)res + job.offset.x, (unsigned)r + job.offset.y);
            job.outDist[slot] = job.rowDist[res];
        }
        for (unsigned w = 0; w < nWarps; ++w) base += sWarp[w];
        __syncthreads();
    }
    if (t == 0) { *job.numMatches = base; *job.done = 0; }
}

#define SM_BM 64              // features of A per CTA (4 warps x 16)
#define SM_BN 64              // features of B per sweep step
#define SM_PITCH 144          // bytes per staged descriptor row: 128 + 16 -> the 8 rows a fragment load touches hit 32 distinct banks

__device__ __forceinline__ void mma_u8(int (&c)[4], const unsigned (&a)[4], unsigned b0, unsigned b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// grid = (ceil(maxNA / 64), numJobs), 128 threads
template <bool kColumnPass>
__global__ void __launch_bounds__(128)
sift_best_kernel(const SiftJobDev* __restrict__ jobs, float distmax, float ratiomax) {
    const SiftJobDev job = jobs[blockIdx.y];
    const int nA = job.nA, nB = job.nB;
    const int row0 = blockIdx.x * SM_BM;
    if (!kColumnPass && blockIdx.x == 0 && threadIdx.x == 0) *job.numMatches = 0;       // SiftMatch.cpp:163 / ProgramCU.cu:1928
    if (nA <= 0 || nB <= 0 || row0 >= nA) return;

    __shared__ __align__(16) unsigned char sBuf[2][SM_BN * SM_PITCH];          // double-buffered tile of B
    const unsigned t = threadIdx.x, lane = t & 31, warp = t >> 5, g = lane >> 2, q = lane & 3;

    // A fragments of this warp's 16 features, all of K = 128 (4 k-steps), kept in registers for the whole sweep
    unsigned a[4][4];
    {
        const int r0 = row0 + (int)warp * 16 + (int)g, r1 = r0 + 8;
        const unsigned* p0 = reinterpret_cast<const unsigned*>(job.desA + (size_t)(r0 < nA ? r0 : 0) * 128);
        const unsigned* p1 = reinterpret_cast<const unsigned*>(job.desA + (size_t)(r1 < nA ? r1 : 0) * 128);
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            a[ks][0] = (r0 < nA) ? __ldg(p0 + ks * 8 + q) : 0u;
            a[ks][1] = (r1 < nA) ? __ldg(p1 + ks * 8 + q) : 0u;
            a[ks][2] = (r0 < nA) ? __ldg(p0 + ks * 8 + 4 + q) : 0u;
            a[ks][3] = (r1 < nA) ? __ldg(p1 + ks * 8 + 4 + q) : 0u;
        }
    }
    // running best / second of this thread's two features (rows g and g + 8 of the warp tile); a dot product must be > 0 to be a
    // candidate (the reference starts from max = 0 with a strict '>')
    Top2 st[2] = { { 0, 0xFFFFFFFFu, 0 }, { 0, 0xFFFFFFFFu, 0 } };

    // stage 64 descriptors of B per step: 64 x 128 B = 512 uint4, 4 per thread, coalesced; the NEXT tile's global loads are issued
    // before the current tile's products so that their latency hides behind the tensor-core work (one barrier per step)
    uint4 pf[4];
    auto fetch = [&](int col0) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const unsigned v = t + 128u * k, r = v >> 3, c16 = v & 7u;
            pf[k] = (col0 + (int)r < nB) ? __ldg(reinterpret_cast<const uint4*>(job.desB + (size_t)(col0 + r) * 128) + c16) : make_uint4(0u, 0u, 0u, 0u);
        }
    };
    auto stash = [&](unsigned char* dst) {
#pragma unroll
        for (int k = 0; k < 4; ++k) { const unsigned v = t + 128u * k, r = v >> 3, c16 = v & 7u; *reinterpret_cast<uint4*>(&dst[r * SM_PITCH + c16 * 16]) = pf[k]; }
    };
    fetch(0);
    stash(sBuf[0]);
    __syncthreads();
    int buf = 0;
    for (int col0 = 0; col0 < nB; col0 += SM_BN) {
        const bool more = col0 + SM_BN < nB;
        if (more) fetch(col0 + SM_BN);
        const unsigned char* sB = sBuf[buf];
        int acc[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) { acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0; }
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const unsigned char* bp = &sB[(nt * 8 + g) * SM_PITCH + ks * 32 + q * 4];
                const unsigned bb0 = *reinterpret_cast<const unsigned*>(bp), bb1 = *reinterpret_cast<const unsigned*>(bp + 16);
                mma_u8(acc[nt], a[ks], bb0, bb1);
            }
        }
        // bookkeeping: acc[nt][0..1] belong to feature g, acc[nt][2..3] to feature g + 8; columns col0 + nt*8 + 2q + {0,1}
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const int c = col0 + nt * 8 + 2 * (int)q;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                if (c + e < nB) {
                    top2_update<kColumnPass>(st[0], acc[nt][e], (unsigned)(c + e));
                    top2_update<kColumnPass>(st[1], acc[nt][2 + e], (unsigned)(c + e));
                }
            }
        }
        if (more) stash(sBuf[buf ^ 1]);
        __syncthreads();
        buf ^= 1;
    }
    // merge the four lanes (q = 0..3) that share a feature
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
            const int ov1 = __shfl_xor_sync(0xffffffffu, st[h].v1, o), ov2 = __shfl_xor_sync(0xffffffffu, st[h].v2, o);
            const unsigned ok1 = __shfl_xor_sync(0xffffffffu, st[h].k1, o);
            top2_merge(st[h], ov1, ok1, ov2);
        }
    }
    if (q == 0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) finish_feature<kColumnPass>(job, row0 + (int)warp * 16 + (int)g + 8 * h, st[h], distmax, ratiomax);
    }
    if (kColumnPass) compact_job(job, (nA + SM_BM - 1) / SM_BM);
}

// ---- branch-free best / second best over the products of one 32-column slice (the wgmma read-back) ----------------------------------------------
// A product v (< 2^23: 128 x 255 x 255) and the preference of its column among equal products are packed into ONE 32-bit word, x = 32 v + R(e), so that
// the running best and the second largest value of the multiset cost three integer min / max per product (m = max(b, x); s = max(s, min(b, x)); b = m)
// plus one multiply-add on the FMA pipe for the packing -- the per-product `if` of top2_update costs a divergent branch and a 64-bit (value, key) compare,
// and the integer pipe is what bounds the read-back.
// The reference's tie rule (tie_key): among equal products the smallest (bit-reversed "lane", column) wins, lane = column % 32 for rows and
// (column / 4) % 32 for columns.  Inside a 32-column slice (first column a multiple of 32) that is a fixed 5-bit rank R(e) of the slice position e; across
// slices it is decided once per slice (top2q_slice): rows -- same rank order, then the earlier slice; columns -- the two low bits of the bit-reversed lane
// come from the slice's position in its 128-column tile, then the earlier tile.
struct Top2Q { int kBest; int bBest; int slice; int s2; };           // merge key and packed word of the best product, its slice, packed second
__host__ __device__ constexpr int brev5_c(int x) { return ((x & 1) << 4) | ((x & 2) << 2) | (x & 4) | ((x & 8) >> 2) | ((x & 16) >> 4); }
__host__ __device__ constexpr int brev3_c(int x) { return ((x & 1) << 2) | (x & 2) | ((x & 4) >> 2); }
template <bool kColumnPass> __host__ __device__ constexpr int rank_of(int e) { return kColumnPass ? (((7 - brev3_c(e >> 2)) << 2) | (3 - (e & 3))) : (31 - brev5_c(e)); }
__device__ __forceinline__ int mad_fma_pipe(int a, int b, int c) { int d; asm("mad.lo.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
// x: packed words of distinct slice positions of slice `sliceIdx` (slices arrive in ascending order)
template <bool kColumnPass, int N>
__device__ __forceinline__ void top2q_slice(Top2Q& st, const int (&x)[N], int sliceIdx) {
    int b[2] = { 0, 0 }, s[2] = { 0, 0 };
#pragma unroll
    for (int e = 0; e < N; ++e) {
        const int k = e & 1;
        s[k] = max(s[k], min(b[k], x[e]));
        b[k] = max(b[k], x[e]);
    }
    // two chains -> one (packed words are distinct unless zero, so max / min on them is the multiset's best / second)
    const int bb = max(b[0], b[1]), ss = max(max(s[0], s[1]), min(b[0], b[1]));
    // into the running state
    const int key = kColumnPass ? ((bb & ~3) | (3 - (((sliceIdx & 1) << 1) | ((sliceIdx >> 1) & 1)))) : bb;       // columns: 3 - brev2(slice position in its tile)
    const bool gt = key > st.kBest;                                       // equal keys: the earlier slice keeps it
    st.s2 = max(max(st.s2, ss), min(st.bBest, bb));
    st.kBest = gt ? key : st.kBest; st.bBest = gt ? bb : st.bBest; st.slice = gt ? sliceIdx : st.slice;
}
// union of two states over disjoint column sets: larger key wins; equal keys -> the earlier slice, then (same slice: columns of one lane of the
// reference, which differ in their two low bits) the larger packed word, i.e. the smaller column
__device__ __forceinline__ void top2q_merge(Top2Q& st, const Top2Q& o) {
    const bool gt = (o.kBest > st.kBest) | ((o.kBest == st.kBest) & ((o.slice < st.slice) | ((o.slice == st.slice) & (o.bBest > st.bBest))));
    st.s2 = max(max(st.s2, o.s2), min(st.bBest, o.bBest));
    st.kBest = gt ? o.kBest : st.kBest; st.bBest = gt ? o.bBest : st.bBest; st.slice = gt ? o.slice : st.slice;
}
// back to the (value, tie key, second value) form finish_feature takes
template <bool kColumnPass>
__device__ __forceinline__ Top2 top2q_finish(const Top2Q& st) {
    Top2 r;
    r.v1 = st.bBest >> 5; r.v2 = st.s2 >> 5;
    const int rank = st.bBest & 31;
    int e = 0;
    if (kColumnPass) { const int hi = 7 - (rank >> 2); e = (brev3_c(hi) << 2) | (3 - (rank & 3)); }
    else e = brev5_c(31 - rank);
    const unsigned col = (unsigned)st.slice * 32u + (unsigned)e;
    r.k1 = tie_key<kColumnPass>(col);
    return r;
}

// ---- wgmma + TMA version: warp-specialised ---------------------------------------------------------------------------------------------------
// One CTA = 128 features of A against all of B in tiles of 128.  288 threads: warp 8's first lane is the whole data path -- it asks the TMA unit for the
// A tile and, four tiles ahead, for the B tiles (cp.async.bulk.tensor.2d straight into the 128-byte-swizzled K-major layout wgmma reads; rows past the end
// of a descriptor array arrive as zeros).  Warps 0-7 are two warpgroups; warpgroup w owns features 64 w .. 64 w + 63 and computes their 64 x 128 x 128
// u8 x u8 -> s32 products of a tile as four wgmma m64n128k32 (exact), A and B both read from shared memory, the accumulators in registers.  A thread
// holds 32 products of each of two features (rows g and g + 8 of its warp's 16, columns 8 i + 2 q + {0, 1}), folds them slice by slice into its running
// best / second best, and the four lanes that share a feature merge at the end.  The hand-offs are mbarriers (TMA -> wgmma: full[s]; wgmma -> TMA:
// empty[s], one arrival per consumer warp once its warpgroup's products of the stage have completed).
#define TC_BM 128
#define TC_BN 128
#define TC_TILE_BYTES (128 * 128)
#define TMA_STAGES 4
#define TMA_SMEM_BYTES ((1 + TMA_STAGES) * TC_TILE_BYTES + 1024)     // A + four B stages + alignment slack (81 KB: two CTAs per SM)

__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr) {           // K-major, SWIZZLE_128B: LBO field 1 (unused), SBO 1024 B (8 rows)
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok = 0;
    for (unsigned spin = 0; !ok; ++spin) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
        if (spin > (1u << 28)) __trap();                     // a lost completion must not hang the device
    }
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count)); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void tma_load_tile(uint32_t dst, const CUtensorMap* map, int row, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 :: "r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(0), "r"(row) : "memory");
}
// d (+)= A (64 x 32 bytes at descA) . B (128 x 32 bytes at descB)^T
__device__ __forceinline__ void wgmma_u8_m64n128k32(int (&d)[64], uint64_t descA, uint64_t descB, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.u8 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
                 "%64, %65, p;\n\t}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]),
                   "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
                   "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]),
                   "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
                   "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]),
                   "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
                 : "l"(descA), "l"(descB), "r"(accumulate) : "memory");
}

template <bool kColumnPass>
__global__ void __launch_bounds__(288, 2)
sift_best_wgmma_kernel(const SiftJobDev* __restrict__ jobs, float distmax, float ratiomax) {
    const SiftJobDev job = jobs[blockIdx.y];
    const int nA = job.nA, nB = job.nB;
    const int row0 = blockIdx.x * TC_BM;
    if (!kColumnPass && blockIdx.x == 0 && threadIdx.x == 0) *job.numMatches = 0;       // SiftMatch.cpp:163 / ProgramCU.cu:1928
    if (nA <= 0 || nB <= 0 || row0 >= nA) return;

    extern __shared__ unsigned char tcSmemRaw[];
    __shared__ __align__(8) unsigned long long sBar[1 + 2 * TMA_STAGES];     // fullA, full[S], empty[S]
    unsigned char* const smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(tcSmemRaw) + 1023) & ~(uintptr_t)1023);
    const uint32_t sA = smem_u32(smem), sB = sA + TC_TILE_BYTES;
    const unsigned t = threadIdx.x, warp = t >> 5, lane = t & 31;
    const uint32_t bFullA = smem_u32(&sBar[0]), bFull = smem_u32(&sBar[1]), bEmpty = smem_u32(&sBar[1 + TMA_STAGES]);
    if (t == 0) {
        mbar_init(bFullA, 1);
        for (int s = 0; s < TMA_STAGES; ++s) { mbar_init(bFull + 8 * s, 1); mbar_init(bEmpty + 8 * s, 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int T = (nB + TC_BN - 1) / TC_BN;

    if (warp == 8) {
        if (lane == 0) {
            asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" :: "l"(reinterpret_cast<uint64_t>(job.mapA)) : "memory");
            asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" :: "l"(reinterpret_cast<uint64_t>(job.mapB)) : "memory");
            mbar_expect_tx(bFullA, TC_TILE_BYTES);
            tma_load_tile(sA, job.mapA, row0, bFullA);
            const int nPre = T < TMA_STAGES ? T : TMA_STAGES;
            for (int j = 0; j < nPre; ++j) { mbar_expect_tx(bFull + 8 * j, TC_TILE_BYTES); tma_load_tile(sB + (uint32_t)j * TC_TILE_BYTES, job.mapB, j * TC_BN, bFull + 8 * j); }
            for (int j = 0; j + TMA_STAGES < T; ++j) {
                const int s = j % TMA_STAGES;
                mbar_wait(bEmpty + 8 * s, (uint32_t)((j / TMA_STAGES) & 1));                 // tile j's products have read stage s
                mbar_expect_tx(bFull + 8 * s, TC_TILE_BYTES);
                tma_load_tile(sB + (uint32_t)s * TC_TILE_BYTES, job.mapB, (j + TMA_STAGES) * TC_BN, bFull + 8 * s);
            }
        }
    } else {
        const unsigned wg = warp >> 2, g = lane >> 2, q = lane & 3;
        // packing constants of this thread's slice positions: m = 2 (i % 4) + e <-> position 8 (i % 4) + 2 q + e
        int rk[8];
    #pragma unroll
        for (int m = 0; m < 8; ++m) rk[m] = rank_of<kColumnPass>(8 * (m >> 1) + 2 * (int)q + (m & 1));
        Top2Q st[2] = { { 0, 0, 0, 0 }, { 0, 0, 0, 0 } };       // a dot product must be > 0 to be a candidate (the reference starts from max = 0 with a strict '>')
        const int thirtyTwo = 32 + (nA >> 30);                  // 32, opaque to the compiler
        const uint32_t aRows = sA + wg * 64u * 128u;            // this warpgroup's 64 rows of A (a multiple of 1024 bytes: the swizzle pattern is unchanged)
        mbar_wait(bFullA, 0);
        for (int j = 0; j < T; ++j) {
            const int s = j % TMA_STAGES;
            const uint32_t bRows = sB + (uint32_t)s * TC_TILE_BYTES;
            mbar_wait(bFull + 8 * s, (uint32_t)((j / TMA_STAGES) & 1));
            int d[64];
            asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
    #pragma unroll
            for (int k = 0; k < 4; ++k)                         // K = 128 bytes = 4 x 32: the descriptors advance 32 bytes inside the swizzled row
                wgmma_u8_m64n128k32(d, wgmma_desc_sw128(aRows + 32u * k), wgmma_desc_sw128(bRows + 32u * k), k ? 1u : 0u);
            asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
            asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(bEmpty + 8 * s);
    #pragma unroll
            for (int h = 0; h < 2; ++h) {
    #pragma unroll
                for (int p = 0; p < 4; ++p) {                   // slice p of the tile: products d[4 i + 2 h + e], i = 4 p .. 4 p + 3
                    int x[8];
    #pragma unroll
                    for (int m = 0; m < 8; ++m) x[m] = mad_fma_pipe(d[4 * (4 * p + (m >> 1)) + 2 * h + (m & 1)], thirtyTwo, rk[m]);
                    top2q_slice<kColumnPass>(st[h], x, 4 * j + p);          // rows past nB are zero-filled by the TMA: never a candidate
                }
            }
        }
        // merge the four lanes (q = 0..3) that share a feature
    #pragma unroll
        for (int h = 0; h < 2; ++h) {
    #pragma unroll
            for (int o = 1; o <= 2; o <<= 1) {
                Top2Q ot;
                ot.kBest = __shfl_xor_sync(0xffffffffu, st[h].kBest, o); ot.bBest = __shfl_xor_sync(0xffffffffu, st[h].bBest, o);
                ot.slice = __shfl_xor_sync(0xffffffffu, st[h].slice, o); ot.s2 = __shfl_xor_sync(0xffffffffu, st[h].s2, o);
                top2q_merge(st[h], ot);
            }
        }
        if (q == 0) {
    #pragma unroll
            for (int h = 0; h < 2; ++h) finish_feature<kColumnPass>(job, row0 + (int)(wg * 64 + (warp & 3) * 16 + g) + 8 * h, top2q_finish<kColumnPass>(st[h]), distmax, ratiomax);
        }
    }
    if (kColumnPass) compact_job(job, (nA + TC_BM - 1) / TC_BM);
}


// SortKeyPointMatchesCU_Kernel (SIFTImageManager.cu:59-145): one CTA per image pair, 128 slots, bitonic network in shared memory on
// the total order (distance, image-2 feature, image-1 feature); padding sorts last.
__global__ void __launch_bounds__(BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW)
sift_sort_kernel(const PairList pl, const int* __restrict__ numMatches, float* dists, uint2* idxs) {
    const PairRef pr = pair_of(pl, blockIdx.x);
    if (pr.skip) return;
    const unsigned pair = pr.slot;
    const int n = min(BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW, numMatches[pair]);
    if (n <= 0) return;
    __shared__ float sD[BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW];
    __shared__ uint2 sI[BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW];
    const unsigned t = threadIdx.x;
    float* d = dists + (size_t)pair * BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW;
    uint2* ix = idxs + (size_t)pair * BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW;
    sD[t] = ((int)t < n) ? d[t] : INFINITY;
    sI[t] = ((int)t < n) ? ix[t] : make_uint2(0xFFFFFFFFu, 0xFFFFFFFFu);
    __syncthreads();
    for (unsigned k = 2; k <= BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW; k <<= 1)
        for (unsigned j = k >> 1; j > 0; j >>= 1) {
            const unsigned o = t ^ j;
            if (o > t) {
                const float a = sD[t], b = sD[o];
                const uint2 ia = sI[t], ib = sI[o];
                const bool aAfterB = (a > b) || (a == b && (ia.y > ib.y || (ia.y == ib.y && ia.x > ib.x)));      // NaN distances do not occur (acosf of a clamped value)
                const bool up = ((t & k) == 0);
                if (aAfterB == up) { sD[t] = b; sD[o] = a; sI[t] = ib; sI[o] = ia; }
            }
            __syncthreads();
        }
    if ((int)t < n) { d[t] = sD[t]; ix[t] = sI[t]; }
}

// ---- host ----------------------------------------------------------------------------------------------------------
struct SiftWs {
    SiftJobDev* dJobs = nullptr; size_t jobCap = 0;
    SiftJobDev* hJobs = nullptr;                 // pinned staging for the job table; evCopied = its last upload has left it
    cudaEvent_t evCopied = nullptr;
    cudaEvent_t evDone = nullptr;                // the last batch's column pass has finished (the workspace is shared by every caller)
    int* rowResult = nullptr; float* rowDist = nullptr; size_t rowCap = 0;
    int* colResult = nullptr; size_t colCap = 0;
    int* done = nullptr;
    CUtensorMap* dMaps = nullptr; CUtensorMap* hMaps = nullptr; size_t mapCap = 0;      // two tensor maps per job (device table + pinned staging)
    std::vector<CUtensorMap> mapStage;                                                  // a batch's maps, encoded before anything is enqueued
    std::map<std::pair<const void*, int>, CUtensorMap> mapCache;                        // encoded maps by (array, rows): a keyframe's descriptors recur every frame
};
static SiftWs g_sift;
// Which sweep runs a batch (bfSiftSetMatchSweep): auto = wgmma + TMA unless the batch's arrays cannot be described by tensor maps (no driver
// entry point), then mma.sync.  The setting starts as BF_SIFT_MATCH gives it ("mma": the mma.sync sweep).  A forced sweep never falls back, so
// that a test can run one batch under both and compare the bytes.
static std::atomic<int>& sweep_setting() {
    static std::atomic<int> s{ [] { const char* e = getenv("BF_SIFT_MATCH"); return (e && e[0] == 'm') ? BF_SIFT_SWEEP_MMA : BF_SIFT_SWEEP_AUTO; }() };
    return s;
}
static bool g_wgmmaAttrSet = false;                // the wgmma kernels' dynamic shared memory limit has been raised (at their first use)
static int g_matchInfo[2] = { 0, 0 };              // the last batch: sweep that ran, jobs (bfSiftGetMatchInfo)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr; static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr; cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
        (void)cudaGetLastError();
    }
    return fn;
}
// [rows][128] bytes, box 128 bytes x 128 rows, 128-byte swizzle, rows past the end read as zeros
bool sift_encode_descriptor_map(const uint8_t* base, int rows, CUtensorMap* out) {
    EncodeTiledFn fn = encode_tiled_fn();
    if (!fn || (reinterpret_cast<uintptr_t>(base) & 15u) || rows <= 0) return false;
    const cuuint64_t dims[2] = { 128, (cuuint64_t)rows }, strides[1] = { 128 };
    const cuuint32_t box[2] = { 128, 128 }, estr[2] = { 1, 1 };
    return fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
              CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
static bool descriptor_map(const uint8_t* base, int rows, CUtensorMap* out) {
    auto key = std::make_pair((const void*)base, rows);
    auto it = g_sift.mapCache.find(key);
    if (it != g_sift.mapCache.end()) { *out = it->second; return true; }
    if (!sift_encode_descriptor_map(base, rows, out)) return false;
    if (g_sift.mapCache.size() > 65536) g_sift.mapCache.clear();
    g_sift.mapCache.emplace(key, *out);
    return true;
}
static std::mutex g_siftMutex;

int sift_wgmma_sweep(const SiftJobDev* dJobs, int numJobs, int gx1, int gx2, float distmax, float ratiomax, cudaStream_t s) {
    if (!g_wgmmaAttrSet) {
        BF_CHECK(cudaFuncSetAttribute(sift_best_wgmma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, TMA_SMEM_BYTES));
        BF_CHECK(cudaFuncSetAttribute(sift_best_wgmma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, TMA_SMEM_BYTES));
        g_wgmmaAttrSet = true;
    }
    g_launchCount += 2;
    sift_best_wgmma_kernel<false><<<dim3(gx1, numJobs), 288, TMA_SMEM_BYTES, s>>>(dJobs, distmax, ratiomax);
    BF_CHECK(cudaGetLastError());
    sift_best_wgmma_kernel<true><<<dim3(gx2, numJobs), 288, TMA_SMEM_BYTES, s>>>(dJobs + numJobs, distmax, ratiomax);
    BF_CHECK(cudaGetLastError());
    return 0;
}
int sift_sort_pairs(const PairList& L, unsigned nBlocks, const int32_t* numMatches, float* dists, uint32_t* idxs) {
    if (!nBlocks) return 0;
    ++g_launchCount;
    sift_sort_kernel<<<nBlocks, BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW, 0, stream()>>>(L, numMatches, dists, reinterpret_cast<uint2*>(idxs));
    BF_CHECK(cudaGetLastError());
    return 0;
}

// grows the matcher's scratch to hold `jobs` jobs with `rows` image-1 and `cols` image-2 features in total; `exact`: called with a batch's own numbers
// (capacities double so that a growing keyframe set rarely reallocates), else a reservation (bfSiftReserveWorkspace: capacities as given)
static int sift_reserve(cudaStream_t s, size_t jobs, size_t rows, size_t cols, bool fromBatch) {
    if (jobs > g_sift.jobCap) {
        if (g_sift.dJobs) { BF_CHECK(cudaStreamSynchronize(s)); BF_CHECK(cudaFree(g_sift.dJobs)); BF_CHECK(cudaFreeHost(g_sift.hJobs)); BF_CHECK(cudaFree(g_sift.done)); }
        g_sift.jobCap = fromBatch ? jobs * 2 : jobs;
        BF_CHECK(cudaMalloc(&g_sift.done, sizeof(int) * g_sift.jobCap));
        BF_CHECK(cudaMemsetAsync(g_sift.done, 0, sizeof(int) * g_sift.jobCap, s));          // each job's last CTA leaves its counter at 0 again
        BF_CHECK(cudaMalloc(&g_sift.dJobs, sizeof(SiftJobDev) * 2 * g_sift.jobCap));      // [row-pass jobs | column-pass jobs]
        BF_CHECK(cudaMallocHost(&g_sift.hJobs, sizeof(SiftJobDev) * 2 * g_sift.jobCap));
        if (!g_sift.evCopied) BF_CHECK(cudaEventCreateWithFlags(&g_sift.evCopied, cudaEventDisableTiming));
    } else if (fromBatch) {
        BF_CHECK(cudaEventSynchronize(g_sift.evCopied));      // the previous call's upload (normally long done) before the staging is rewritten
    }
    if (rows > g_sift.rowCap) {
        if (g_sift.rowResult) { BF_CHECK(cudaStreamSynchronize(s)); BF_CHECK(cudaFree(g_sift.rowResult)); BF_CHECK(cudaFree(g_sift.rowDist)); }
        g_sift.rowCap = fromBatch ? rows * 2 : rows;
        BF_CHECK(cudaMalloc(&g_sift.rowResult, sizeof(int) * g_sift.rowCap));
        BF_CHECK(cudaMalloc(&g_sift.rowDist, sizeof(float) * g_sift.rowCap));
    }
    if (cols > g_sift.colCap) {
        if (g_sift.colResult) { BF_CHECK(cudaStreamSynchronize(s)); BF_CHECK(cudaFree(g_sift.colResult)); }
        g_sift.colCap = fromBatch ? cols * 2 : cols;
        BF_CHECK(cudaMalloc(&g_sift.colResult, sizeof(int) * g_sift.colCap));
    }
    return 0;
}
static int sift_reserve_maps(cudaStream_t s, size_t jobs, bool fromBatch) {
    if (jobs > g_sift.mapCap) {
        if (g_sift.dMaps) { BF_CHECK(cudaStreamSynchronize(s)); BF_CHECK(cudaFree(g_sift.dMaps)); BF_CHECK(cudaFreeHost(g_sift.hMaps)); }
        g_sift.mapCap = fromBatch ? jobs * 2 : jobs;
        BF_CHECK(cudaMalloc(&g_sift.dMaps, sizeof(CUtensorMap) * 2 * g_sift.mapCap));
        BF_CHECK(cudaMallocHost(&g_sift.hMaps, sizeof(CUtensorMap) * 2 * g_sift.mapCap));
    }
    return 0;
}

}  // namespace bf

using namespace bf;

BF_API int bfSiftMatchBatch(const BFSiftMatchJob* jobs, int numJobs, float distmax, float ratiomax) {
    if (numJobs <= 0) return 0;
    std::lock_guard<std::mutex> lk(g_siftMutex);
    size_t rows = 0, cols = 0;
    int maxN1 = 0, maxN2 = 0;
    for (int i = 0; i < numJobs; ++i) {
        const bool live = jobs[i].num1 > 0 && jobs[i].num2 > 0;
        if (live) { rows += (size_t)jobs[i].num1; cols += (size_t)jobs[i].num2; maxN1 = jobs[i].num1 > maxN1 ? jobs[i].num1 : maxN1; maxN2 = jobs[i].num2 > maxN2 ? jobs[i].num2 : maxN2; }
        if (jobs[i].num1 >= (1 << 24) || jobs[i].num2 >= (1 << 24)) return (int)cudaErrorInvalidValue;       // index field of the packed key
        // both sweeps read descriptor rows in 16-byte units (TMA boxes, uint4 loads): a misaligned array is refused before anything is enqueued
        if (live && ((reinterpret_cast<uintptr_t>(jobs[i].d_des1) | reinterpret_cast<uintptr_t>(jobs[i].d_des2)) & 15u)) {
            set_last_error("bfSiftMatchBatch: descriptor array not 16-byte aligned", cudaErrorInvalidValue);
            return (int)cudaErrorInvalidValue;
        }
    }
    // tensor maps of the batch (wgmma + TMA sweep), encoded on the host before anything is enqueued: a forced wgmma sweep that cannot map a batch
    // fails it here; auto runs such a batch (no driver entry point) with the mma.sync sweep, which computes the same matches
    const int sweep = sweep_setting().load();
    bool useTc = sweep != BF_SIFT_SWEEP_MMA;
    if (useTc) {
        g_sift.mapStage.resize(2 * (size_t)numJobs);
        for (int i = 0; i < numJobs && useTc; ++i) {
            const BFSiftMatchJob& j = jobs[i];
            if (j.num1 > 0 && j.num2 > 0)
                useTc = descriptor_map(j.d_des1, j.num1, &g_sift.mapStage[2 * (size_t)i]) && descriptor_map(j.d_des2, j.num2, &g_sift.mapStage[2 * (size_t)i + 1]);
        }
        if (!useTc && sweep == BF_SIFT_SWEEP_WGMMA) {
            set_last_error("bfSiftMatchBatch: the forced wgmma sweep cannot map this batch", cudaErrorNotSupported);
            return (int)cudaErrorNotSupported;
        }
    }
    cudaStream_t s = stream();
    if (!g_sift.evDone) BF_CHECK(cudaEventCreateWithFlags(&g_sift.evDone, cudaEventDisableTiming));
    BF_CHECK(cudaStreamWaitEvent(s, g_sift.evDone, 0));       // a previous batch (possibly on another stream) still owns rowResult / the job table
    { const int rcR = sift_reserve(s, (size_t)numJobs, rows, cols, true); if (rcR) return rcR; }
    if (useTc) {
        const int rcM = sift_reserve_maps(s, (size_t)numJobs, true); if (rcM) return rcM;
        memcpy(g_sift.hMaps, g_sift.mapStage.data(), sizeof(CUtensorMap) * 2 * (size_t)numJobs);      // staging is free: sift_reserve waited for evCopied
    }
    SiftJobDev* h = g_sift.hJobs;
    size_t off = 0, coff = 0;
    for (int i = 0; i < numJobs; ++i) {
        const BFSiftMatchJob& j = jobs[i];
        const bool live = j.num1 > 0 && j.num2 > 0;
        SiftJobDev r;
        r.desA = j.d_des1; r.nA = live ? j.num1 : 0; r.desB = j.d_des2; r.nB = live ? j.num2 : 0;
        r.rowResult = g_sift.rowResult + off; r.rowDist = g_sift.rowDist + off;
        r.numMatches = j.out.d_numMatches; r.outDist = j.out.d_distances; r.outIdx = reinterpret_cast<uint2*>(j.out.d_keyPointIndices);
        r.offset = make_uint2(j.keyPointOffset[0], j.keyPointOffset[1]);
        r.colResult = g_sift.colResult + coff; r.done = g_sift.done + i;
        r.mapA = nullptr; r.mapB = nullptr;
        if (useTc && live) { r.mapA = g_sift.dMaps + 2 * i; r.mapB = g_sift.dMaps + 2 * i + 1; }
        SiftJobDev c = r;                                   // column pass: image 2 owns the sweep, image 1 is swept
        c.desA = j.d_des2; c.nA = r.nB; c.desB = j.d_des1; c.nB = r.nA; c.mapA = r.mapB; c.mapB = r.mapA;
        h[i] = r; h[(size_t)numJobs + i] = c;
        if (live) { off += (size_t)j.num1; coff += (size_t)j.num2; }
    }
    if (useTc) BF_CHECK(cudaMemcpyAsync(g_sift.dMaps, g_sift.hMaps, sizeof(CUtensorMap) * 2 * (size_t)numJobs, cudaMemcpyHostToDevice, s));
    BF_CHECK(cudaMemcpyAsync(g_sift.dJobs, h, sizeof(SiftJobDev) * 2 * (size_t)numJobs, cudaMemcpyHostToDevice, s));
    BF_CHECK(cudaEventRecord(g_sift.evCopied, s));
    g_matchInfo[0] = useTc ? BF_SIFT_SWEEP_WGMMA : BF_SIFT_SWEEP_MMA; g_matchInfo[1] = numJobs;
    if (useTc) {
        const int gx1 = maxN1 > 0 ? (maxN1 + TC_BM - 1) / TC_BM : 1, gx2 = maxN2 > 0 ? (maxN2 + TC_BM - 1) / TC_BM : 1;
        const int rcS = sift_wgmma_sweep(g_sift.dJobs, numJobs, gx1, gx2, distmax, ratiomax, s); if (rcS) return rcS;
    } else {
        g_launchCount += 2;
        const int gx1 = maxN1 > 0 ? (maxN1 + SM_BM - 1) / SM_BM : 1, gx2 = maxN2 > 0 ? (maxN2 + SM_BM - 1) / SM_BM : 1;
        sift_best_kernel<false><<<dim3(gx1, numJobs), 128, 0, s>>>(g_sift.dJobs, distmax, ratiomax);
        BF_CHECK(cudaGetLastError());
        sift_best_kernel<true><<<dim3(gx2, numJobs), 128, 0, s>>>(g_sift.dJobs + numJobs, distmax, ratiomax);
        BF_CHECK(cudaGetLastError());
    }
    BF_CHECK(cudaEventRecord(g_sift.evDone, s));
    return 0;
}

BF_API int bfSiftSortKeyPointMatches(unsigned int curFrame, unsigned int startFrame, unsigned int numFrames, const int32_t* d_numMatchesPerImagePair,
                                     float* d_matchDistances, uint32_t* d_matchKeyPointIndices) {
    if (numFrames <= startFrame) return 0;                                  // SIFTImageManager.cu:148
    return sift_sort_pairs(frame_pairs(curFrame, startFrame), numFrames - startFrame, d_numMatchesPerImagePair, d_matchDistances, d_matchKeyPointIndices);
}

BF_API size_t bfSiftWorkspaceBytes(void) {
    std::lock_guard<std::mutex> lk(g_siftMutex);
    return sizeof(SiftJobDev) * 2 * g_sift.jobCap + (sizeof(int) + sizeof(float)) * g_sift.rowCap + sizeof(int) * (g_sift.colCap + g_sift.jobCap);
}
BF_API int bfSiftReserveWorkspace(unsigned int maxJobs, unsigned int maxKeysPerImage) {
    if (maxJobs == 0 || maxKeysPerImage == 0) return (int)cudaErrorInvalidValue;
    std::lock_guard<std::mutex> lk(g_siftMutex);
    cudaStream_t s = stream();
    if (!g_sift.evDone) BF_CHECK(cudaEventCreateWithFlags(&g_sift.evDone, cudaEventDisableTiming));
    BF_CHECK(cudaStreamWaitEvent(s, g_sift.evDone, 0));
    const size_t n = (size_t)maxJobs * maxKeysPerImage;
    int rc = sift_reserve(s, maxJobs, n, n, false);
    if (!rc) rc = sift_reserve_maps(s, maxJobs, false);
    return rc;
}
BF_API int bfSiftReleaseWorkspace(void) {
    std::lock_guard<std::mutex> lk(g_siftMutex);
    cudaFree(g_sift.dJobs); cudaFree(g_sift.rowResult); cudaFree(g_sift.rowDist); cudaFree(g_sift.colResult); cudaFree(g_sift.done); cudaFree(g_sift.dMaps);
    if (g_sift.hMaps) cudaFreeHost(g_sift.hMaps);
    if (g_sift.hJobs) cudaFreeHost(g_sift.hJobs);
    if (g_sift.evCopied) cudaEventDestroy(g_sift.evCopied);
    if (g_sift.evDone) cudaEventDestroy(g_sift.evDone);
    g_sift = SiftWs();
    return 0;
}
BF_API int bfSiftSetMatchSweep(int sweep) {
    if (sweep < BF_SIFT_SWEEP_AUTO || sweep > BF_SIFT_SWEEP_MMA) return (int)cudaErrorInvalidValue;
    return sweep_setting().exchange(sweep);
}
BF_API int bfSiftGetMatchInfo(int out[2]) {
    if (!out) return (int)cudaErrorInvalidValue;
    std::lock_guard<std::mutex> lk(g_siftMutex);
    out[0] = g_matchInfo[0]; out[1] = g_matchInfo[1];
    return 0;
}

// solver.cu -- sparse bundle adjustment (Gauss-Newton + Jacobi-PCG in Lie space) for sm_90a.
// Implements include/bf_solver.h (rows a10-a12, a14-a16 of SURVEY.md section 8).
//
// Behavioural source: FL/Solver/SolverBundling.cu:756-1264, FL/Solver/SolverBundlingEquationsLie.h:27-228,
// FL/Solver/LieDerivUtil.h:19-307, FL/SBA.cu:75-119.
//
// Design (DESIGN.md section "Solver"):
//  * the reference applies the sparse term matrix-free, J^T(J p), touching every correspondence twice per PCG
//    iteration (~140 B/correspondence/iteration) and needs ~9 launches + a blocking device->host copy per
//    iteration.  Here the correspondences of one image pair are folded ONCE per Gauss-Newton iteration into a
//    6x6 block (block-sparse J^T J, both (i,j) and (j,i) stored so a row never needs a transpose), and a PCG
//    iteration is a block-sparse mat-vec over ~144 B per image pair -- ~25x less traffic, L2-resident;
//  * one persistent kernel (a cooperative grid; one CTA at N <= 16; at 17 <= N <= 128 one thread-block cluster with the PCG system
//    resident in shared memory) runs a whole Gauss-Newton iteration: pose -> matrix, block build, row reduction, PCG init, all PCG iterations
//    (2 grid barriers each on the grid, none in the cluster), Lie update, convergence test.  The early-outs
//    (|p.Ap| < 5e-7, max|delta| < 0.005) are evaluated on the device; later GN launches see a "done" flag;
//  * every floating-point reduction has a fixed shape (per-segment serial sums, fixed warp trees, partials summed
//    in CTA order), so results are run-to-run deterministic -- the reference's atomics are not.
#include <cooperative_groups.h>

#include <atomic>
#include <cstring>
#include <map>
#include <mutex>

#include "../../include/bf_solver.h"
#include "bf_common.cuh"
#include "se3.cuh"

namespace cg = cooperative_groups;

namespace bf {

extern unsigned long long g_launchCount;      // defined in tsdf.cu (bfGetLaunchCount)

#define BF_FLOAT_EPSILON 0.000001f      // FL/SolverUtil.h:9
#define BF_MAX_ROW 8192                 // longest variable row the in-smem row sort handles
#define BF_SOLVER_THREADS 256
#define BF_SOLVER_MAX_PEERS 8
#define BF_SOLVER_ONE_CTA_MAX_N 16u      // largest N whose Gauss-Newton iterations run as one CTA (OneCtaGrid)
#define BF_DENSE_MAX_IMAGES 4096        // dense term: N^2 pair tables + one 90-sum record per image pair (allocated on first use, sized by the workspace)

__device__ void mat4_mul(const float* a, const float* b, float* o) {
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) o[r * 4 + c] = a[r * 4] * b[c] + a[r * 4 + 1] * b[4 + c] + a[r * 4 + 2] * b[8 + c] + a[r * 4 + 3] * b[12 + c];
}
// general 4x4 inverse (adjugate / determinant), cuda_SimpleMatrixUtil.h:980-1100
__device__ void mat4_inverse(const float* m, float* out) {
    const float s0 = m[0] * m[5] - m[4] * m[1], s1 = m[0] * m[6] - m[4] * m[2], s2 = m[0] * m[7] - m[4] * m[3];
    const float s3 = m[1] * m[6] - m[5] * m[2], s4 = m[1] * m[7] - m[5] * m[3], s5 = m[2] * m[7] - m[6] * m[3];
    const float c5 = m[10] * m[15] - m[14] * m[11], c4 = m[9] * m[15] - m[13] * m[11], c3 = m[9] * m[14] - m[13] * m[10];
    const float c2 = m[8] * m[15] - m[12] * m[11], c1 = m[8] * m[14] - m[12] * m[10], c0 = m[8] * m[13] - m[12] * m[9];
    const float r = 1.0f / (s0 * c5 - s1 * c4 + s2 * c3 + s3 * c2 - s4 * c1 + s5 * c0);
    out[0] = (m[5] * c5 - m[6] * c4 + m[7] * c3) * r;   out[1] = (-m[1] * c5 + m[2] * c4 - m[3] * c3) * r;
    out[2] = (m[13] * s5 - m[14] * s4 + m[15] * s3) * r; out[3] = (-m[9] * s5 + m[10] * s4 - m[11] * s3) * r;
    out[4] = (-m[4] * c5 + m[6] * c2 - m[7] * c1) * r;  out[5] = (m[0] * c5 - m[2] * c2 + m[3] * c1) * r;
    out[6] = (-m[12] * s5 + m[14] * s2 - m[15] * s1) * r; out[7] = (m[8] * s5 - m[10] * s2 + m[11] * s1) * r;
    out[8] = (m[4] * c4 - m[5] * c2 + m[7] * c0) * r;   out[9] = (-m[0] * c4 + m[1] * c2 - m[3] * c0) * r;
    out[10] = (m[12] * s4 - m[13] * s2 + m[15] * s0) * r; out[11] = (-m[8] * s4 + m[9] * s2 - m[11] * s0) * r;
    out[12] = (-m[4] * c3 + m[5] * c1 - m[6] * c0) * r; out[13] = (m[0] * c3 - m[1] * c1 + m[2] * c0) * r;
    out[14] = (-m[12] * s3 + m[13] * s1 - m[14] * s0) * r; out[15] = (m[8] * s3 - m[9] * s1 + m[10] * s0) * r;
}

// ---- workspace --------------------------------------------------------------------------------------------
struct Segment { int nbr; int start; int count; int _pad; };      // one (row image, neighbour image) run of a row
enum { SC_DONE = 0, SC_GN_RUN = 1, SC_PCG_RUN = 2, SC_NUM_SEG = 3, SC_NUM_VALID = 4, SC_MAXDELTA_BITS = 5, SC_ERROR = 6, SC_DENSE_ON = 7, SC_DENSE_OVERLAP = 8, SC_DENSE_PAIRS = 9, SC_NUM = 16 };
// values of scal[SC_ERROR] (bfSolverGetStats out[5])
#define BF_SOLVER_ERR_EXCHANGE_TIMEOUT 2u      // pcg_resident: the bytes of a PCG iteration did not all arrive within BF_MBAR_TIMEOUT_NS

struct SolverWs {
    unsigned maxImages = 0, maxCorr = 0;
    int* rowCount = nullptr;      // [N]   arrivals per image
    int* rowStart = nullptr;      // [N+1] CSR offsets
    int* cursor = nullptr;        // [N]
    int* entries = nullptr;       // [2*maxCorr] correspondence indices, per row sorted by (neighbour, index)
    int* nbrs = nullptr;          // [2*maxCorr] the other image of each row entry, written with it (never re-read from the correspondence)
    int* segCount = nullptr;      // [N]   segments of each row
    Segment* segs = nullptr;      // [2*maxCorr] segments of row v live at rowStart[v] ...
    float* offBlk = nullptr;      // [2*maxCorr][36] off-diagonal 6x6 blocks, aligned with segs
    float* segMom = nullptr;      // [2*maxCorr][20] per-segment diagonal moments + rhs
    float* diagBlk = nullptr;     // [N][36]
    float* partials = nullptr;    // [2][maxGrid]
    float* p2 = nullptr;          // [2][N][3] second search-direction buffer (rot, trans): p ping-pongs so that the update of p
                                  // can be fused into the next mat-vec (2 grid barriers per PCG iteration instead of 3)
    // dense depth / colour term, block-sparse: the reference keeps a dense (6N)^2 matrix (576 MB at N = 2000, read in full by every PCG
    // iteration); here only the image pairs that carry weight exist.  Allocated by ensure_dense() on the first dense solve, Nd = maxImages.
    unsigned denseCap = 0;        // Nd the dense buffers were sized for (0: not allocated)
    float* pairW = nullptr;       // [Nd*Nd]   weight of pair (i < j), 0 = none
    int*   pairIdx = nullptr;     // [Nd*Nd]   index of pair (i < j) in the pair list
    int*   pairCnt = nullptr;     // [2][Nd]   per image: pairs it leads (j > i), pairs it is part of
    int*   pairRowStart = nullptr;// [Nd+1]    pair list offsets by leading image (the list is sorted by (i, j))
    int2*  pairIJ = nullptr;      // [maxPairs]
    float* pairOut = nullptr;     // [maxPairs][90] per pair: J_i^T J_i (21, upper triangle), J_j^T J_j (21), J_i^T J_j (36), J_i^T r (6), J_j^T r (6)
    int*   dnbrStart = nullptr;   // [Nd+1]    per image: its pairs, ascending in the other image
    int2*  dnbr = nullptr;        // [2 maxPairs] {other image, pair index}
    float* denseDiag = nullptr;   // [Nd][36]  diagonal 6x6 blocks (translation-first ordering per image, as the reference)
    float* denseJtr = nullptr;    // [6 Nd]
    unsigned* scal = nullptr;     // [SC_NUM]
    int maxGrid = 0;
    // sharded solve (bfSolverPeerCreate / Connect): this rank's exchange region (cudaMalloc'd, opened by the peers through CUDA IPC) and theirs
    int rank = 0, world = 1; float* region = nullptr; float* peer[BF_SOLVER_MAX_PEERS] = {}; bool peerOpened[BF_SOLVER_MAX_PEERS] = {}; unsigned peerSeq = 0;
    const void* owner[4] = { nullptr, nullptr, nullptr, nullptr };   // the caller's d_deltaTrans / d_rRot / d_pRot / d_Ap_XRot: a recycled
                                                                     // d_deltaRot address with other neighbours is another solver object
    int launchInfo[4] = { 0, 0, 0, 0 };                              // last GN launch: policy, G, cluster cap, resident smem limit (bfSolverGetLaunchInfo)
};
static void free_ws(SolverWs& w) {
    cudaFree(w.rowCount); cudaFree(w.rowStart); cudaFree(w.cursor); cudaFree(w.entries); cudaFree(w.nbrs); cudaFree(w.segCount); cudaFree(w.segs);
    cudaFree(w.offBlk); cudaFree(w.segMom); cudaFree(w.diagBlk); cudaFree(w.partials); cudaFree(w.p2); cudaFree(w.scal);
    cudaFree(w.pairW); cudaFree(w.pairIdx); cudaFree(w.pairCnt); cudaFree(w.pairRowStart); cudaFree(w.pairIJ); cudaFree(w.pairOut); cudaFree(w.dnbrStart); cudaFree(w.dnbr);
    cudaFree(w.denseDiag); cudaFree(w.denseJtr);
    for (int g = 0; g < BF_SOLVER_MAX_PEERS; ++g) if (w.peerOpened[g]) cudaIpcCloseMemHandle(w.peer[g]);
    cudaFree(w.region);
}
static std::mutex g_wsMutex;
static std::map<const void*, SolverWs> g_ws;

static int get_ws(const BFSolverState* st, unsigned maxImages, unsigned maxCorr, SolverWs** out) {
    std::lock_guard<std::mutex> lk(g_wsMutex);
    auto it = g_ws.find(st->d_deltaRot);
    const void* owner[4] = { st->d_deltaTrans, st->d_rRot, st->d_pRot, st->d_Ap_XRot };
    if (it != g_ws.end() && it->second.maxImages >= maxImages && it->second.maxCorr >= maxCorr && memcmp(it->second.owner, owner, sizeof(owner)) == 0) {
        *out = &it->second; return 0;
    }
    if (it != g_ws.end()) { free_ws(it->second); g_ws.erase(it); }
    SolverWs w;
    w.maxImages = maxImages; w.maxCorr = maxCorr ? maxCorr : 1;
    w.maxGrid = num_sms() * 4;
    memcpy(w.owner, owner, sizeof(owner));
    const size_t E = 2 * (size_t)w.maxCorr;
    // every buffer is zeroed once at creation: nothing a kernel reads before writing can depend on what the allocator hands back
#define BF_WS_ALLOC(ptr, bytes) do { BF_CHECK(cudaMalloc(&(ptr), (bytes))); BF_CHECK(cudaMemsetAsync((ptr), 0, (bytes), stream())); } while (0)
    BF_WS_ALLOC(w.rowCount, sizeof(int) * maxImages);
    BF_WS_ALLOC(w.rowStart, sizeof(int) * (maxImages + 1));
    BF_WS_ALLOC(w.cursor, sizeof(int) * maxImages);
    BF_WS_ALLOC(w.entries, sizeof(int) * E);
    BF_WS_ALLOC(w.nbrs, sizeof(int) * E);
    BF_WS_ALLOC(w.segCount, sizeof(int) * maxImages);
    BF_WS_ALLOC(w.segs, sizeof(Segment) * E);
    BF_WS_ALLOC(w.offBlk, sizeof(float) * 36 * E);
    BF_WS_ALLOC(w.segMom, sizeof(float) * 20 * E);
    BF_WS_ALLOC(w.diagBlk, sizeof(float) * 36 * maxImages);
    BF_WS_ALLOC(w.partials, sizeof(float) * 2 * w.maxGrid);
    BF_WS_ALLOC(w.p2, sizeof(float) * 6 * maxImages);
    BF_WS_ALLOC(w.scal, sizeof(unsigned) * SC_NUM);
    auto res = g_ws.emplace(st->d_deltaRot, w);
    *out = &res.first->second;
    return 0;
}
static int ensure_dense(SolverWs* w) {
    if (w->denseCap >= w->maxImages) return 0;
    const size_t Nd = w->maxImages, maxPairs = Nd * (Nd - 1) / 2 + 1;
    BF_WS_ALLOC(w->pairW, sizeof(float) * Nd * Nd);
    BF_WS_ALLOC(w->pairIdx, sizeof(int) * Nd * Nd);
    BF_WS_ALLOC(w->pairCnt, sizeof(int) * 2 * Nd);
    BF_WS_ALLOC(w->pairRowStart, sizeof(int) * (Nd + 1));
    BF_WS_ALLOC(w->pairIJ, sizeof(int2) * maxPairs);
    BF_WS_ALLOC(w->pairOut, sizeof(float) * 90 * maxPairs);
    BF_WS_ALLOC(w->dnbrStart, sizeof(int) * (Nd + 1));
    BF_WS_ALLOC(w->dnbr, sizeof(int2) * 2 * maxPairs);
    BF_WS_ALLOC(w->denseDiag, sizeof(float) * 36 * Nd);
    BF_WS_ALLOC(w->denseJtr, sizeof(float) * 6 * Nd);
    w->denseCap = (unsigned)Nd;
    return 0;
}
#undef BF_WS_ALLOC

// ---- preparation: variable rows (CSR), reference-format table, neighbour segments ----------------------------
__device__ __forceinline__ bool corr_valid(const BFEntryJ& c) { return c.imgIdx_i != 0xFFFFFFFFu; }

__global__ void prep_count_kernel(const BFEntryJ* __restrict__ corr, unsigned C, int* rowCount) {
    const unsigned x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= C) return;
    const unsigned i = corr[x].imgIdx_i, j = corr[x].imgIdx_j;
    if (i == 0xFFFFFFFFu) return;
    atomicAdd(&rowCount[i], 1);
    atomicAdd(&rowCount[j], 1);
}
// single CTA: exclusive scan of rowCount -> rowStart, publish counts in the reference's d_numEntriesPerRow
__global__ void prep_scan_kernel(const int* __restrict__ rowCount, int* rowStart, int* cursor, int* numEntriesPerRow, unsigned N, unsigned* scal) {
    __shared__ int sSum[1024];
    const unsigned t = threadIdx.x;
    const unsigned per = (N + blockDim.x - 1) / blockDim.x;
    int local = 0;
    for (unsigned k = 0; k < per; ++k) { const unsigned i = t * per + k; if (i < N) local += rowCount[i]; }
    sSum[t] = local;
    __syncthreads();
    for (unsigned off = 1; off < blockDim.x; off <<= 1) {
        int v = (t >= off) ? sSum[t - off] : 0;
        __syncthreads();
        sSum[t] += v;
        __syncthreads();
    }
    int run = sSum[t] - local;
    for (unsigned k = 0; k < per; ++k) {
        const unsigned i = t * per + k;
        if (i < N) { rowStart[i] = run; cursor[i] = 0; if (numEntriesPerRow) numEntriesPerRow[i] = rowCount[i]; run += rowCount[i]; }
    }
    if (t == blockDim.x - 1) rowStart[N] = sSum[t];
    if (t == 0) { scal[SC_DONE] = 0; scal[SC_GN_RUN] = 0; scal[SC_PCG_RUN] = 0; scal[SC_ERROR] = 0; }
}
__global__ void prep_scatter_kernel(const BFEntryJ* __restrict__ corr, unsigned C, const int* __restrict__ rowStart, int* cursor, int* entries, int* nbrs) {
    const unsigned x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= C) return;
    const unsigned i = corr[x].imgIdx_i, j = corr[x].imgIdx_j;
    if (i == 0xFFFFFFFFu) return;
    const int pi = rowStart[i] + atomicAdd(&cursor[i], 1), pj = rowStart[j] + atomicAdd(&cursor[j], 1);
    entries[pi] = (int)x; nbrs[pi] = (int)j;
    entries[pj] = (int)x; nbrs[pj] = (int)i;
}
// bitonic sort of n 64-bit keys held in shared memory (n padded to a power of two with ~0 keys)
__device__ void bitonic_sort_smem(unsigned long long* keys, unsigned nPow2) {
    for (unsigned k = 2; k <= nPow2; k <<= 1) {
        for (unsigned j = k >> 1; j > 0; j >>= 1) {
            for (unsigned i = threadIdx.x; i < nPow2; i += blockDim.x) {
                const unsigned ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long a = keys[i], b = keys[ixj];
                    const bool up = ((i & k) == 0);
                    if ((a > b) == up) { keys[i] = b; keys[ixj] = a; }
                }
            }
            __syncthreads();
        }
    }
}
// one CTA per image row: (1) sort the row by correspondence index -> reference-format table row + overflow
// invalidation (SolverBundling.cu:1237-1245 with arrival rank = ascending index); (2) sort by (neighbour, index) and
// cut the row into neighbour segments.  The neighbour of a row entry comes from the array the scatter kernel wrote, never from
// the correspondence itself: another row's CTA may be invalidating that correspondence at this moment (two separate stores).
// Rows longer than BF_MAX_ROW (> maxCorrPerImage, checked by the host) keep their maxCorrPerImage smallest indices, found by
// a bisection on the index value over the row in global memory; the rest is invalidated as the reference does.
__global__ void __launch_bounds__(256)
prep_rows_kernel(BFEntryJ* corr, const int* __restrict__ rowStart, int* entries, int* nbrs, int* segCount, Segment* segs,
                 int* varToCorr, unsigned maxCorrPerImage, unsigned* scal) {
    extern __shared__ unsigned long long sKeys[];
    __shared__ unsigned sCnt;
    const unsigned v = blockIdx.x;
    const int start = rowStart[v];
    int n = rowStart[v + 1] - start;
    if (threadIdx.x == 0) segCount[v] = 0;
    if (n <= 0) return;
    if (n > BF_MAX_ROW) {
        // smallest T with #{entries <= T} >= maxCorrPerImage (indices within a row are distinct)
        unsigned lo = 0u, hi = 0x7FFFFFFFu;
        while (lo < hi) {
            const unsigned mid = lo + (hi - lo) / 2;
            if (threadIdx.x == 0) sCnt = 0;
            __syncthreads();
            unsigned c = 0;
            for (int i = threadIdx.x; i < n; i += blockDim.x) c += ((unsigned)entries[start + i] <= mid) ? 1u : 0u;
            c = warp_sum_u(c);
            if ((threadIdx.x & 31) == 0 && c) atomicAdd(&sCnt, c);
            __syncthreads();
            const unsigned tot = sCnt;
            __syncthreads();
            if (tot >= maxCorrPerImage) hi = mid; else lo = mid + 1;
        }
        if (threadIdx.x == 0) sCnt = 0;
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const unsigned c = (unsigned)entries[start + i];
            if (c <= lo) sKeys[atomicAdd(&sCnt, 1u)] = ((unsigned long long)c << 32) | (unsigned)nbrs[start + i];
            else { corr[c].imgIdx_i = 0xFFFFFFFFu; corr[c].imgIdx_j = 0xFFFFFFFFu; }
        }
        __syncthreads();
        n = (int)sCnt;                                       // == maxCorrPerImage <= BF_MAX_ROW
    } else {
        for (int i = threadIdx.x; i < n; i += blockDim.x) sKeys[i] = ((unsigned long long)(unsigned)entries[start + i] << 32) | (unsigned)nbrs[start + i];
    }
    unsigned nPow2 = 1; while (nPow2 < (unsigned)n) nPow2 <<= 1;
    for (unsigned i = n + threadIdx.x; i < nPow2; i += blockDim.x) sKeys[i] = ~0ull;
    __syncthreads();
    bitonic_sort_smem(sKeys, nPow2);
    // (1) table row + invalidation of the overflow tail; the kept part is re-keyed (neighbour, index), the tail parked at the end
    for (unsigned i = threadIdx.x; i < (unsigned)n; i += blockDim.x) {
        const unsigned c = (unsigned)(sKeys[i] >> 32), nb = (unsigned)sKeys[i];
        if (i < maxCorrPerImage) { if (varToCorr) varToCorr[(size_t)v * maxCorrPerImage + i] = (int)c; sKeys[i] = ((unsigned long long)nb << 32) | c; }
        else { corr[c].imgIdx_i = 0xFFFFFFFFu; corr[c].imgIdx_j = 0xFFFFFFFFu; sKeys[i] = ((unsigned long long)0x7FFFFFFFu << 32) | c; }      // setInvalid (both rows may do it; same value)
    }
    __syncthreads();
    // (2) An entry the OTHER row of its correspondence invalidates keeps its place: the block build skips invalid entries whatever
    // segment they sit in.
    bitonic_sort_smem(sKeys, nPow2);
    for (unsigned i = threadIdx.x; i < (unsigned)n; i += blockDim.x) { entries[start + i] = (int)(unsigned)sKeys[i]; nbrs[start + i] = (int)(unsigned)(sKeys[i] >> 32); }
    // segment heads, in order: serial over the row by one warp-sized stride would reorder, so thread 0 walks it
    __syncthreads();
    if (threadIdx.x == 0) {
        int ns = 0, segStart = 0;
        unsigned cur = (unsigned)(sKeys[0] >> 32);
        for (int i = 1; i <= n; ++i) {
            const unsigned nb = (i < n) ? (unsigned)(sKeys[i] >> 32) : 0xFFFFFFFFu;
            if (nb != cur) {
                if (cur != 0x7FFFFFFFu) { Segment s; s.nbr = (int)cur; s.start = start + segStart; s.count = i - segStart; s._pad = 0; segs[start + ns] = s; ++ns; }
                segStart = i; cur = nb;
            }
        }
        segCount[v] = ns;
        atomicAdd(&scal[SC_NUM_SEG], (unsigned)ns);
    }
}

// ---- the Gauss-Newton iteration kernel (persistent) ------------------------------------------------------------
struct GnArgs {
    const BFEntryJ* corr;
    unsigned N, C;
    const int* validImages;
    float* xRot; float* xTrans;
    float* deltaRot; float* deltaTrans; float* rRot; float* rTrans; float* zRot; float* zTrans; float* pRot; float* pTrans;
    float* ApRot; float* ApTrans; float* precRot; float* precTrans;
    float* T; float* Tinv;
    const int* rowStart; const int* entries; const int* segCount; const Segment* segs;
    float* offBlk; float* segMom; float* diagBlk; float* partials; unsigned* scal;
    float* p2Rot; float* p2Trans;
    float wSparse; unsigned nLin; int isLastGn; int maxGrid;
    const int* dnbrStart; const int2* dnbr; const float* pairOut; const float* denseDiag; const float* denseJtr; int useDense;       // dense term, block-sparse (NULL / 0 when off)
    // rows sharded over GPUs (world > 1): this rank computes A p for the rows v with v % world == rank and stores them straight into EVERY rank's exchange
    // region over NVLink; peer[g] = base of rank g's region (peer[rank]: the local one).  seqBase: barrier sequence numbers already used.
    int rank, world; float* peer[BF_SOLVER_MAX_PEERS]; unsigned seqBase; unsigned peerMaxN;
};
// exchange region of a rank (floats): ap[2][6 maxN] (rot 3 maxN, trans 3 maxN; double-buffered by PCG iteration parity), partials[2][MAX_PEERS * maxGrid], flags[MAX_PEERS]
__host__ __device__ inline size_t peer_region_floats(unsigned maxN, int maxGrid) { return (size_t)12 * maxN + (size_t)2 * BF_SOLVER_MAX_PEERS * maxGrid + BF_SOLVER_MAX_PEERS; }
__device__ __forceinline__ float* peer_ap(float* base, unsigned maxN, unsigned par) { return base + (size_t)par * 6 * maxN; }
__device__ __forceinline__ float* peer_partials(float* base, unsigned maxN, int maxGrid, unsigned par) { return base + (size_t)12 * maxN + (size_t)par * BF_SOLVER_MAX_PEERS * maxGrid; }
__device__ __forceinline__ unsigned* peer_flags(float* base, unsigned maxN, int maxGrid) { return reinterpret_cast<unsigned*>(base + (size_t)12 * maxN + (size_t)2 * BF_SOLVER_MAX_PEERS * maxGrid); }

// 6x6 block times 6-vector (rot,trans order)
__device__ __forceinline__ void blk_mv(const float* __restrict__ B, V3 pr, V3 pt, float* y) {
#pragma unroll
    for (int r = 0; r < 6; ++r)
        y[r] += B[r * 6 + 0] * pr.x + B[r * 6 + 1] * pr.y + B[r * 6 + 2] * pr.z + B[r * 6 + 3] * pt.x + B[r * 6 + 4] * pt.y + B[r * 6 + 5] * pt.z;
}

// deterministic grid-wide sum: every CTA writes its partial, after the barrier every thread sums them in CTA order
__device__ __forceinline__ float block_sum(float v, float* sRed) {
    v = warp_sum(v);
    const unsigned t = threadIdx.x;
    if ((t & 31) == 0) sRed[t >> 5] = v;
    __syncthreads();
    float tot = 0.0f;
    if (t == 0) { for (unsigned w = 0; w < blockDim.x / 32; ++w) tot += sRed[w]; sRed[0] = tot; }
    __syncthreads();
    tot = sRed[0];
    __syncthreads();
    return tot;
}
// every CTA evaluates the same fixed-shape sum of the per-CTA partials: lane l adds partials[l], [l+32], ... in order, then a
// fixed shuffle tree -- one L2 round trip instead of gridDim.x dependent ones, and identical bits in every CTA
__device__ __forceinline__ float grid_sum_after_sync(const float* partials, unsigned grid, float* sRed) {
    if (threadIdx.x < 32) {
        float v = 0.0f;
        for (unsigned b = threadIdx.x; b < grid; b += 32) v += __ldcg(&partials[b]);
        v = warp_sum(v);
        if (threadIdx.x == 0) sRed[0] = v;
    }
    __syncthreads();
    const float tot = sRed[0];
    __syncthreads();
    return tot;
}

// How gn_iteration_kernel's G CTAs of BF_SOLVER_THREADS threads run.  Every order-sensitive float sum of the kernel depends only on
// that partition: a thread's serial sum, the warp tree, a CTA's warp sums added in order (block_sum), the G CTA partials combined by
// grid_sum_after_sync.
//  * CoopGrid: G real CTAs, cooperative launch, grid barriers (any N).  Every PCG operand is read from L2.
//  * OneCtaGrid: ONE CTA of G x BF_SOLVER_THREADS threads (G <= 4).  Thread t is the cooperative grid's thread t, so rows map to
//    threads and warps as there; barriers are __syncthreads, and sum() forms the G partials and their total in exactly the shape
//    above -- bit-identical results.  At the local solve's size the PCG iteration is barrier- and L2-latency-bound.
//  * ResidentCluster: the same G CTAs as ONE thread-block cluster (G <= the cluster cap, 16 where the device allows it, else 8;
//    sharded solves excluded).  Steps (0)-(2) and (4) are the grid's with cluster barriers.  The PCG (pcg_resident) first copies
//    each warp's row -- its segment blocks, dense pair blocks and diagonal blocks -- into the CTA's shared memory, and every CTA
//    keeps full-length copies of z, p, r, delta, the preconditioner and Ap.  In a PCG iteration
//    the mat-vec rows store Ap and the p.Ap partials into every CTA's copy (distributed shared memory, st.async), and every CTA
//    runs the step / residual / z.r phase for all rows itself once its copy is complete.  Every sum keeps the grid's shape, so results are bit-identical.
struct CoopGrid {
    static constexpr int kThreads = BF_SOLVER_THREADS;
    static constexpr bool kPeers = true;
    static constexpr bool kResident = false;
    __device__ __forceinline__ void sync() const { cg::this_grid().sync(); }
    // grid-wide sum of every thread's v, the same bits in every thread; partials: [gridDim.x] scratch
    __device__ __forceinline__ float sum(float v, float* partials, float* sRed) const {
        v = block_sum(v, sRed);
        if (threadIdx.x == 0) partials[blockIdx.x] = v;
        sync();
        return grid_sum_after_sync(partials, gridDim.x, sRed);
    }
};
struct OneCtaGrid {
    static constexpr int kThreads = 4 * BF_SOLVER_THREADS;
    static constexpr bool kPeers = false;
    static constexpr bool kResident = false;
    __device__ __forceinline__ void sync() const { __syncthreads(); }
    __device__ __forceinline__ float sum(float v, float*, float* sRed) const {
        v = warp_sum(v);
        if ((threadIdx.x & 31) == 0) sRed[threadIdx.x >> 5] = v;
        __syncthreads();
        if (threadIdx.x < 32) {
            const unsigned G = blockDim.x / BF_SOLVER_THREADS, b = threadIdx.x;
            float g = 0.0f;                                      // grid_sum_after_sync: lane b adds partial b (G <= 32)
            if (b < G) {
                float tot = 0.0f;                                // block_sum of virtual CTA b
                for (unsigned w = 0; w < BF_SOLVER_THREADS / 32; ++w) tot += sRed[b * (BF_SOLVER_THREADS / 32) + w];
                g += tot;
            }
            g = warp_sum(g);
            if (b == 0) sRed[0] = g;
        }
        __syncthreads();
        const float tot = sRed[0];
        __syncthreads();
        return tot;
    }
};
struct ResidentCluster {
    static constexpr int kThreads = BF_SOLVER_THREADS;
    static constexpr bool kPeers = false;
    static constexpr bool kResident = true;
    __device__ __forceinline__ void sync() const { __threadfence(); cg::this_cluster().sync(); }
    __device__ __forceinline__ float sum(float v, float* partials, float* sRed) const {
        v = block_sum(v, sRed);
        if (threadIdx.x == 0) partials[blockIdx.x] = v;
        sync();
        return grid_sum_after_sync(partials, gridDim.x, sRed);
    }
};
#define BF_RESIDENT_MAX_CLUSTER 16
#define BF_RESIDENT_ROWS (BF_SOLVER_THREADS / 32)      // rows per CTA: warp w of CTA c owns row 1 + 8c + w
// Dynamic shared memory of pcg_resident, in 4-byte words; S = N slots per row (a row's segments and dense pairs have distinct
// neighbours in [0, N)).  Blocks first so that they are 16-byte aligned:
//   off [R][S][36], dense [R][S][36] (when on), diag [R][2][36] (sparse, dense), vec [8][6N] (z, p0, p1, r, delta, prec, Ap[2];
//   each rot [N][3] then trans [N][3]), part [2][32], nbr [R][S] int, dnb [R][S] int (when on)
__host__ __device__ inline size_t resident_smem_words(unsigned N, bool dense) {
    const size_t R = BF_RESIDENT_ROWS, S = N;
    return R * S * 36 * (dense ? 2 : 1) + R * 72 + (size_t)48 * N + 64 + R * S * (dense ? 2 : 1);
}

// Barrier over all GPUs of a sharded solve.  Every thread's remote stores are made visible system-wide, the local grid arrives, one CTA publishes this
// rank's sequence number in every rank's flag array (release), every CTA waits on its OWN region until all ranks have published it (acquire).
template <class Grid>
__device__ __forceinline__ void peer_barrier(const GnArgs& a, unsigned seq, Grid& grid) {
    __threadfence_system();
    grid.sync();
    if (blockIdx.x == 0 && threadIdx.x < (unsigned)a.world) {
        unsigned* f = peer_flags(a.peer[threadIdx.x], a.peerMaxN, a.maxGrid) + a.rank;
        asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(f), "r"(seq) : "memory");
    }
    if (threadIdx.x < (unsigned)a.world) {
        const unsigned* f = peer_flags(a.peer[a.rank], a.peerMaxN, a.maxGrid) + threadIdx.x;
        unsigned v, spins = 0;
        do {
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
            if (++spins > (1u << 27)) __trap();                 // a missing rank must not hang the device
        } while ((int)(v - seq) < 0);
    }
    __syncthreads();
}

// 6x6 block times 6-vector, the block in shared memory (16-byte aligned): nine 128-bit loads, then blk_mv's arithmetic
__device__ __forceinline__ void blk_mv_smem(const float* B, V3 pr, V3 pt, float* y) {
    float b[36];
#pragma unroll
    for (int q = 0; q < 9; ++q) { const float4 f = reinterpret_cast<const float4*>(B)[q]; b[4 * q] = f.x; b[4 * q + 1] = f.y; b[4 * q + 2] = f.z; b[4 * q + 3] = f.w; }
    blk_mv(b, pr, pt, y);
}
// dense pair block M (row orientation: M[r*6+c] couples row image coordinate r to the other image's coordinate c, translation
// first) times p of the other image, the expression of the grid's mat-vec
__device__ __forceinline__ void dense_mv(const float* M, V3 pr, V3 pt, float* y) {
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        y[3 + r] += M[r * 6 + 0] * pt.x + M[r * 6 + 1] * pt.y + M[r * 6 + 2] * pt.z + M[r * 6 + 3] * pr.x + M[r * 6 + 4] * pr.y + M[r * 6 + 5] * pr.z;
        y[r] += M[(3 + r) * 6 + 0] * pt.x + M[(3 + r) * 6 + 1] * pt.y + M[(3 + r) * 6 + 2] * pt.z + M[(3 + r) * 6 + 3] * pr.x + M[(3 + r) * 6 + 4] * pr.y + M[(3 + r) * 6 + 5] * pr.z;
    }
}

// Distributed-shared-memory exchange without a cluster barrier: a cluster barrier's release compiles to a GPU-scope memory barrier
// (MEMBAR.ALL.GPU), which alone costs more than the rest of a small PCG iteration.  Instead every value goes out with st.async,
// which counts its bytes off the RECEIVING CTA's transaction barrier; a CTA waits on its own barrier until all bytes of an
// iteration have landed.
__device__ __forceinline__ unsigned cluster_addr(unsigned a, unsigned rank) {
    unsigned r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(rank));
    return r;
}
__device__ __forceinline__ void st_async(unsigned addr, float v, unsigned mbar) {
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" :: "r"(addr), "r"(__float_as_uint(v)), "r"(mbar) : "memory");
}
__device__ __forceinline__ void mbar_expect(unsigned mbar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(mbar), "r"(bytes) : "memory");
}
// up to 1024 probes of the phase in one tight PTX loop (written in C++, the loop's exits cost convergence barriers on every probe)
__device__ __forceinline__ bool mbar_try_wait(unsigned mbar, unsigned parity) {
    unsigned done;
    asm volatile("{\n\t.reg .pred p;\n\t.reg .u32 k;\n\tmov.u32 k, 1024;\n"
                 "BF_MBAR_PROBE_%=:\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                 "@p bra BF_MBAR_DONE_%=;\n\t"
                 "sub.u32 k, k, 1;\n\t"
                 "setp.ne.u32 p, k, 0;\n\t"
                 "@p bra BF_MBAR_PROBE_%=;\n"
                 "BF_MBAR_DONE_%=:\n\t"
                 "selp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(mbar), "r"(parity) : "memory");
    return done != 0;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// A legitimate wait is a few microseconds.  The bound turns a wrong byte count or a missing sender into an error flag instead of a hung device.
#define BF_MBAR_TIMEOUT_NS 1000000000ull
// false: the phase did not complete within BF_MBAR_TIMEOUT_NS.  The clock is read once per 1024 probes, off the path of the common short wait.
__device__ __forceinline__ bool mbar_wait(unsigned mbar, unsigned parity) {
    if (mbar_try_wait(mbar, parity)) return true;
    const unsigned long long t0 = globaltimer_ns();
    while (!mbar_try_wait(mbar, parity))
        if (globaltimer_ns() - t0 > BF_MBAR_TIMEOUT_NS) return false;
    return true;
}

// x(v) <- exp(delta(v)) x(v) (LieDerivUtil.h:301-307), for the resident PCG.  Not inlined: compiled on its own, the float contraction of
// this branchy code does not depend on the surrounding kernel, and it then rounds exactly as the cooperative grid's inlined copy does;
// inlined into pcg_resident it rounded differently in the last bit for some rows.
__device__ __noinline__ void lie_update_row(const GnArgs& a, unsigned v) {
    float U[16], Cm[16], P[16];
    pose_to_matrix(ld3(a.deltaRot, v), ld3(a.deltaTrans, v), U);
    pose_to_matrix(ld3(a.xRot, v), ld3(a.xTrans, v), Cm);
    mat4_mul(U, Cm, P);
    V3 nr, nt;
    matrix_to_pose(P, nr, nt);
    st3(a.xRot, v, nr); st3(a.xTrans, v, nt);
}
// Step (3) of gn_iteration_kernel<ResidentCluster>: all PCG iterations with the system in shared memory (layout: resident_smem_words).
// Thread and warp roles are the grid's: warp w of CTA c owns row 1 + 8c + w in the mat-vec, and row v of the step phase is thread v
// -- of CTA 0 in the grid (N <= 128 < 256), of EVERY CTA here, each on its own copies.  The other CTAs' z.r partials are therefore +0
// in the grid, and each CTA forms the total in the grid's shape locally.  Called after the barrier that ends step (2); returns the
// number of PCG iterations run.  On exit delta and the Lie update of x are in global memory, written by CTA 0's thread v.
__device__ unsigned pcg_resident(const GnArgs& a, bool denseOn, float rDotzOld) {
    extern __shared__ float4 sDyn4[];
    __shared__ float sRedA[BF_RESIDENT_ROWS], sRedB[BF_RESIDENT_ROWS];
    __shared__ unsigned sTimedOut;                                                // a thread's wait on sMbar timed out (mbar_wait)
    __shared__ __align__(8) unsigned long long sMbar[2];                         // transaction barriers of the Ap / partial buffers, by parity
    cg::cluster_group cluster = cg::this_cluster();
    const unsigned N = a.N, S = N, R = BF_RESIDENT_ROWS, C = gridDim.x;
    const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & 31, t = threadIdx.x;
    float* const sOff = reinterpret_cast<float*>(sDyn4);
    float* const sDen = sOff + (size_t)R * S * 36;                              // only when denseOn
    float* const sDiag = sDen + (denseOn ? (size_t)R * S * 36 : 0);
    float* const sVec = sDiag + R * 72;
    float* const sZ = sVec, * const sP0 = sVec + 6 * N, * const sP1 = sVec + 12 * N, * const sR = sVec + 18 * N, * const sDelta = sVec + 24 * N,
                 * const sPrec = sVec + 30 * N, * const sAp = sVec + 36 * N;        // sAp: [2][6N] by iteration parity
    float* const sPart = sVec + 48 * N;                                           // [2][32] p.Ap partials by iteration parity
    int* const sNbr = reinterpret_cast<int*>(sPart + 64);
    int* const sDnb = sNbr + (size_t)R * S;                                        // only when denseOn

    // ---- residency: this warp's row, the full vectors ----
    const unsigned v = 1 + blockIdx.x * R + warp;
    int ns = 0, nd = 0;
    if (v < N) {
        // a row's segments have distinct neighbours and its dense pairs distinct other images, all in [0, N): at most S of each
        const int rs = a.rowStart[v];
        ns = min(a.segCount[v], (int)S);
        for (int sI = (int)lane; sI < ns; sI += 32) sNbr[warp * S + sI] = __ldcg(&a.segs[rs + sI].nbr);
        const float4* gOff = reinterpret_cast<const float4*>(a.offBlk + 36 * (size_t)rs);
        float4* lOff = reinterpret_cast<float4*>(sOff + 36 * (size_t)warp * S);
        for (int q = (int)lane; q < ns * 9; q += 32) lOff[q] = __ldcg(&gOff[q]);
        for (unsigned q = lane; q < 36; q += 32) sDiag[warp * 72 + q] = __ldcg(&a.diagBlk[36 * (size_t)v + q]);
        if (denseOn) {
            const int e0 = a.dnbrStart[v];
            nd = min(a.dnbrStart[v + 1] - e0, (int)S);
            for (int q = (int)lane; q < nd * 36; q += 32) {
                const int e = q / 36, rc = q % 36, r = rc / 6, c = rc % 6;
                const int2 nb = a.dnbr[e0 + e];
                if (rc == 0) sDnb[warp * S + e] = nb.x;
                sDen[36 * ((size_t)warp * S + e) + rc] = a.pairOut[(size_t)nb.y * 90 + 42 + ((v < (unsigned)nb.x) ? r * 6 + c : c * 6 + r)];   // v is the pair's hi image: the transposed block
            }
            for (unsigned q = lane; q < 36; q += 32) sDiag[warp * 72 + 36 + q] = a.denseDiag[36 * (size_t)v + q];
        }
    }
    for (unsigned i = t; i < 3 * N; i += blockDim.x) {
        sP0[i] = __ldcg(&a.pRot[i]); sP0[3 * N + i] = __ldcg(&a.pTrans[i]);
        sR[i] = __ldcg(&a.rRot[i]); sR[3 * N + i] = __ldcg(&a.rTrans[i]);
        sPrec[i] = __ldcg(&a.precRot[i]); sPrec[3 * N + i] = __ldcg(&a.precTrans[i]);
        sDelta[i] = 0.0f; sDelta[3 * N + i] = 0.0f;
    }
    // per iteration every CTA receives Ap of the N - 1 rows and the C partials; buffer par serves iterations par, par + 2, ...
    const unsigned bytesPerIter = 24u * (N - 1) + 4u * C;
    const unsigned mbar0 = smem_u32(&sMbar[0]);
    if (t == 0) {
        sTimedOut = 0u;
        for (unsigned p = 0; p < 2; ++p) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(mbar0 + 8 * p) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbar_expect(mbar0, bytesPerIter); mbar_expect(mbar0 + 8, bytesPerIter);
    }
    cluster.sync();                                                     // every CTA's barriers are armed before the first store

    unsigned pcgRun = 0;
    float beta = 0.0f;
    for (unsigned lin = 0; lin < a.nLin; ++lin) {
        bool last = (lin == a.nLin - 1);
        ++pcgRun;
        const bool fly = lin > 0;
        const unsigned par = lin & 1u;
        const float* const curP = par ? sP1 : sP0;                                 // p_k of this iteration (formed below when fly)
        const float* const prvP = par ? sP0 : sP1;                                 // p_{k-1}
        float* const ap = sAp + par * 6 * N;
        float* const part = sPart + par * 32;
        // A: Ap = H p for this warp's row into every CTA's copy, this CTA's partial p.Ap into every CTA's copy
        float pAp = 0.0f;
        if (v < N) {
            float y[6] = { 0, 0, 0, 0, 0, 0 };
            for (int sI = (int)lane; sI < ns; sI += 32) {
                const unsigned o = (unsigned)sNbr[warp * S + sI];
                if (o == 0 || o >= N) continue;                         // variable 0 is fixed: its p is zero by construction
                const V3 pr = fly ? ld3(sZ, o) + ld3(prvP, o) * beta : ld3(sP0, o);
                const V3 pt = fly ? ld3(sZ + 3 * N, o) + ld3(prvP + 3 * N, o) * beta : ld3(sP0 + 3 * N, o);
                blk_mv_smem(&sOff[36 * ((size_t)warp * S + sI)], pr, pt, y);
            }
            for (int e = (int)lane; e < nd; e += 32) {                  // nd = 0 without the dense term
                const unsigned o = (unsigned)sDnb[warp * S + e];
                if (o == 0) continue;
                const V3 pr = fly ? ld3(sZ, o) + ld3(prvP, o) * beta : ld3(sP0, o);
                const V3 pt = fly ? ld3(sZ + 3 * N, o) + ld3(prvP + 3 * N, o) * beta : ld3(sP0 + 3 * N, o);
                dense_mv(&sDen[36 * ((size_t)warp * S + e)], pr, pt, y);
            }
#pragma unroll
            for (int k = 0; k < 6; ++k) y[k] = warp_sum(y[k]);
            if (lane == 0) {
                const V3 pr = fly ? ld3(sZ, v) + ld3(prvP, v) * beta : ld3(sP0, v);
                const V3 pt = fly ? ld3(sZ + 3 * N, v) + ld3(prvP + 3 * N, v) * beta : ld3(sP0 + 3 * N, v);
                blk_mv(&sDiag[warp * 72], pr, pt, y);
                if (denseOn) dense_mv(&sDiag[warp * 72 + 36], pr, pt, y);
                pAp += pr.x * y[0] + pr.y * y[1] + pr.z * y[2] + pt.x * y[3] + pt.y * y[4] + pt.z * y[5];
            }
#pragma unroll
            for (int k = 0; k < 6; ++k) y[k] = __shfl_sync(0xffffffffu, y[k], 0);      // lane 0's sums (the tree's bits differ by lane)
            for (unsigned c = lane; c < C; c += 32) {
                const unsigned dst = cluster_addr(smem_u32(ap), c), mb = cluster_addr(mbar0 + 8 * par, c);
#pragma unroll
                for (int k = 0; k < 3; ++k) { st_async(dst + 4 * (3 * v + k), y[k], mb); st_async(dst + 4 * (3 * N + 3 * v + k), y[3 + k], mb); }
            }
        }
        pAp = warp_sum(pAp);
        if (lane == 0) sRedA[warp] = pAp;
        __syncthreads();
        if (t < C) {                                                      // block_sum's total, stored into CTA t's partials
            float tot = 0.0f;
            for (unsigned w = 0; w < R; ++w) tot += sRedA[w];
            st_async(cluster_addr(smem_u32(part + blockIdx.x), t), tot, cluster_addr(mbar0 + 8 * par, t));
        }
        // every row's Ap and every partial of this iteration have landed here.  A CTA reaches iteration lin + 2 (the next use of this
        // buffer) only after receiving this CTA's rows of lin + 1, which are sent after this CTA's last read of the buffer below.
        const bool arrived = mbar_wait(mbar0 + 8 * par, (lin >> 1) & 1u);
        if (t == 0) mbar_expect(mbar0 + 8 * par, bytesPerIter);          // re-arm for lin + 2
        float dotProduct;
        {                                                                 // grid_sum_after_sync, in every warp
            float g = 0.0f;
            if (lane < C) g += part[lane];
            g = warp_sum(g);
            dotProduct = __shfl_sync(0xffffffffu, g, 0);
        }
        // B: step, residual, preconditioned residual, z.r -- every row, in every CTA
        float alpha = 0.0f;
        if (dotProduct > BF_FLOAT_EPSILON) alpha = rDotzOld / dotProduct;
        float zr = 0.0f;
        if (t < N && t != 0) {
            V3 pkR, pkT;
            if (fly) {
                float* const cur = par ? sP1 : sP0;
                pkR = ld3(sZ, t) + ld3(prvP, t) * beta; pkT = ld3(sZ + 3 * N, t) + ld3(prvP + 3 * N, t) * beta;
                st3(cur, t, pkR); st3(cur + 3 * N, t, pkT);
            } else { pkR = ld3(curP, t); pkT = ld3(curP + 3 * N, t); }
            st3(sDelta, t, ld3(sDelta, t) + pkR * alpha);
            st3(sDelta + 3 * N, t, ld3(sDelta + 3 * N, t) + pkT * alpha);
            const V3 rR = ld3(sR, t) - ld3(ap, t) * alpha, rT = ld3(sR + 3 * N, t) - ld3(ap + 3 * N, t) * alpha;
            st3(sR, t, rR); st3(sR + 3 * N, t, rT);
            const V3 zR = mulv(ld3(sPrec, t), rR), zT = mulv(ld3(sPrec + 3 * N, t), rT);
            st3(sZ, t, zR); st3(sZ + 3 * N, t, zT);
            zr += dot(zR, rR) + dot(zT, rT);
        }
        zr = warp_sum(zr);
        if (lane == 0) sRedB[warp] = zr;
        if (!arrived) sTimedOut = 1u;
        __syncthreads();
        // A timed-out wait leaves the PCG in the whole CTA, before the Lie update.  The other CTAs then time out on this CTA's missing
        // rows; every CTA passes the cluster barrier of step (4) before it exits, so no store targets an exited CTA's shared memory.
        // H100 80GB HBM3, 400 W limit, scripts/solver_timing.py against the unbounded wait: +10 / 20 / 30 ns per PCG iteration at
        // N = 32 / 64 / 128 (2.33 -> 2.34, 3.22 -> 3.24, 3.53 -> 3.56 us).  __syncthreads_or in place of the flag cost ~60 ns, and
        // this test placed after the beta update ~40 ns.
        if (sTimedOut) {
            if (t == 0) a.scal[SC_ERROR] = BF_SOLVER_ERR_EXCHANGE_TIMEOUT;
            break;
        }
        float rDotzNew;
        {                                                                 // the grid's shape: partial 0 = this CTA's rows, partials 1..C-1 = +0
            float tot = 0.0f;
            for (unsigned w = 0; w < R; ++w) tot += sRedB[w];
            float g = 0.0f;
            if (lane < C) g += (lane == 0) ? tot : 0.0f;
            g = warp_sum(g);
            rDotzNew = __shfl_sync(0xffffffffu, g, 0);
        }
        if (fabsf(dotProduct) < 5e-7f) last = true;                     // ENABLE_EARLY_OUT (:1088-1093)
        beta = 0.0f;
        if (rDotzOld > BF_FLOAT_EPSILON) beta = rDotzNew / rDotzOld;
        if (last && blockIdx.x == 0 && t < N && t != 0) {
            st3(a.deltaRot, t, ld3(sDelta, t)); st3(a.deltaTrans, t, ld3(sDelta + 3 * N, t));
            lie_update_row(a, t);
        }
        rDotzOld = rDotzNew;
        if (last) break;
    }
    return pcgRun;
}

template <class Grid>
__global__ void __launch_bounds__(Grid::kThreads)
gn_iteration_kernel(const GnArgs a) {
    Grid grid;
    __shared__ float sRed[32];
    if (__ldcg(&a.scal[SC_DONE]) != 0) return;                 // an earlier GN iteration converged (uniform for the grid)
    const unsigned tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
    const unsigned N = a.N;
    const float w = a.wSparse;

    // (0) pose -> matrix (+ inverse for the dense term), convertLiePosesToMatricesCU (SolverBundling.cu:1114-1121)
    for (unsigned k = tid; k < N; k += nth) {
        float M[16], Mi[16];
        pose_to_matrix(ld3(a.xRot, k), ld3(a.xTrans, k), M);
        mat4_inverse(M, Mi);
#pragma unroll
        for (int e = 0; e < 16; ++e) { a.T[16 * k + e] = M[e]; a.Tinv[16 * k + e] = Mi[e]; }
    }
    grid.sync();

    // (1) one thread per (row, neighbour) segment: fold the segment's correspondences into the off-diagonal 6x6 block
    //     H_vo = -w G_v^T G_o and the row's diagonal / rhs moments, G(P) = [-[P]x | I], P = T * p.
    {
        // segments are addressed through their row: flatten (row, local segment) over the grid
        const unsigned gw = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5), nw = gridDim.x * (blockDim.x / 32);
        for (unsigned v = gw; v < N; v += nw) {                      // a warp per row, lanes over the row's segments
            const int ns = a.segCount[v], rs = a.rowStart[v];
            for (int sI = threadIdx.x & 31; sI < ns; sI += 32) {
                const Segment sg = a.segs[rs + sI];
                float nCnt = 0.0f, sumPP = 0.0f, sPvPo = 0.0f;
                V3 sPv = mk(0, 0, 0), sPo = mk(0, 0, 0), gRot = mk(0, 0, 0);
                float vv[6] = { 0, 0, 0, 0, 0, 0 };          // sum Pv Pv^T (xx,xy,xz,yy,yz,zz)
                float ov[9] = { 0, 0, 0, 0, 0, 0, 0, 0, 0 }; // sum Po Pv^T
                for (int e = 0; e < sg.count; ++e) {
                    const BFEntryJ c = a.corr[a.entries[sg.start + e]];
                    if (!corr_valid(c)) continue;
                    const bool vIsI = (c.imgIdx_i == v);
                    const V3 pv = vIsI ? mk(c.pos_i[0], c.pos_i[1], c.pos_i[2]) : mk(c.pos_j[0], c.pos_j[1], c.pos_j[2]);
                    const V3 po = vIsI ? mk(c.pos_j[0], c.pos_j[1], c.pos_j[2]) : mk(c.pos_i[0], c.pos_i[1], c.pos_i[2]);
                    const V3 Pv = xf(&a.T[16 * v], pv), Po = xf(&a.T[16 * (unsigned)sg.nbr], po);
                    nCnt += 1.0f; sumPP += dot(Pv, Pv); sPvPo += dot(Pv, Po);
                    sPv = sPv + Pv; sPo = sPo + Po;
                    gRot = gRot + cross(Po, Pv);             // J_v^T r (rot part) = Po x Pv, independent of the i/j role
                    vv[0] += Pv.x * Pv.x; vv[1] += Pv.x * Pv.y; vv[2] += Pv.x * Pv.z; vv[3] += Pv.y * Pv.y; vv[4] += Pv.y * Pv.z; vv[5] += Pv.z * Pv.z;
                    ov[0] += Po.x * Pv.x; ov[1] += Po.x * Pv.y; ov[2] += Po.x * Pv.z;
                    ov[3] += Po.y * Pv.x; ov[4] += Po.y * Pv.y; ov[5] += Po.y * Pv.z;
                    ov[6] += Po.z * Pv.x; ov[7] += Po.z * Pv.y; ov[8] += Po.z * Pv.z;
                }
                // off-diagonal block: -w [[ (Pv.Po) I - Po Pv^T , [Pv]x ],[ -[Po]x , I ]] summed over the segment
                float* B = &a.offBlk[36 * (size_t)(rs + sI)];
                const float mw = -w;
                B[0] = mw * (sPvPo - ov[0]); B[1] = mw * (-ov[1]);        B[2] = mw * (-ov[2]);
                B[6] = mw * (-ov[3]);        B[7] = mw * (sPvPo - ov[4]); B[8] = mw * (-ov[5]);
                B[12] = mw * (-ov[6]);       B[13] = mw * (-ov[7]);       B[14] = mw * (sPvPo - ov[8]);
                // [Pv]x = [[0,-z,y],[z,0,-x],[-y,x,0]]
                B[3] = 0.0f;          B[4] = mw * (-sPv.z); B[5] = mw * (sPv.y);
                B[9] = mw * (sPv.z);  B[10] = 0.0f;         B[11] = mw * (-sPv.x);
                B[15] = mw * (-sPv.y); B[16] = mw * (sPv.x); B[17] = 0.0f;
                // -[Po]x
                B[18] = 0.0f;          B[19] = mw * (sPo.z);  B[20] = mw * (-sPo.y);
                B[24] = mw * (-sPo.z); B[25] = 0.0f;          B[26] = mw * (sPo.x);
                B[30] = mw * (sPo.y);  B[31] = mw * (-sPo.x); B[32] = 0.0f;
                B[21] = mw * nCnt; B[22] = 0.0f; B[23] = 0.0f; B[27] = 0.0f; B[28] = mw * nCnt; B[29] = 0.0f; B[33] = 0.0f; B[34] = 0.0f; B[35] = mw * nCnt;
                float* m = &a.segMom[20 * (size_t)(rs + sI)];
                m[0] = nCnt; m[1] = sPv.x; m[2] = sPv.y; m[3] = sPv.z; m[4] = sumPP;
                m[5] = vv[0]; m[6] = vv[1]; m[7] = vv[2]; m[8] = vv[3]; m[9] = vv[4]; m[10] = vv[5];
                m[11] = gRot.x; m[12] = gRot.y; m[13] = gRot.z;
                m[14] = sPv.x - sPo.x; m[15] = sPv.y - sPo.y; m[16] = sPv.z - sPo.z;
            }
        }
    }
    grid.sync();

    const bool denseOn = a.useDense && (__ldcg(&a.scal[SC_DENSE_ON]) != 0);      // BuildDenseSystem found overlapping pairs (:1167)
    // (2) one thread per row: sum the row's segment moments in segment order -> diagonal block, -J^T f, Jacobi
    //     preconditioner from the UNWEIGHTED diagonal (SolverBundlingEquationsLie.h:105-147), PCG init (:756-794)
    float part = 0.0f;
    for (unsigned v = tid; v < N; v += nth) {
        if (v == 0) continue;
        const int ns = a.segCount[v], rs = a.rowStart[v];
        float m[17];
#pragma unroll
        for (int k = 0; k < 17; ++k) m[k] = 0.0f;
        for (int sI = 0; sI < ns; ++sI) {
            const float* sm = &a.segMom[20 * (size_t)(rs + sI)];
#pragma unroll
            for (int k = 0; k < 17; ++k) m[k] += sm[k];
        }
        float* D = &a.diagBlk[36 * (size_t)v];
        // w * [[ |P|^2 I - P P^T , [P]x ],[ [P]x^T , n I ]]
        D[0] = w * (m[4] - m[5]); D[1] = w * (-m[6]);       D[2] = w * (-m[7]);
        D[6] = w * (-m[6]);       D[7] = w * (m[4] - m[8]); D[8] = w * (-m[9]);
        D[12] = w * (-m[7]);      D[13] = w * (-m[9]);      D[14] = w * (m[4] - m[10]);
        D[3] = 0.0f;         D[4] = w * (-m[3]); D[5] = w * (m[2]);
        D[9] = w * (m[3]);   D[10] = 0.0f;       D[11] = w * (-m[1]);
        D[15] = w * (-m[2]); D[16] = w * (m[1]); D[17] = 0.0f;
        D[18] = 0.0f;        D[19] = w * (m[3]);  D[20] = w * (-m[2]);
        D[24] = w * (-m[3]); D[25] = 0.0f;        D[26] = w * (m[1]);
        D[30] = w * (m[2]);  D[31] = w * (-m[1]); D[32] = 0.0f;
        D[21] = w * m[0]; D[22] = 0.0f; D[23] = 0.0f; D[27] = 0.0f; D[28] = w * m[0]; D[29] = 0.0f; D[33] = 0.0f; D[34] = 0.0f; D[35] = w * m[0];
        V3 resRot = mk(-w * m[11], -w * m[12], -w * m[13]), resTrans = mk(-w * m[14], -w * m[15], -w * m[16]);
        if (denseOn) {      // minus since -J^T f, weight already built in (SolverBundlingEquationsLie.h:114-118)
            resRot = resRot - mk(a.denseJtr[v * 6 + 3], a.denseJtr[v * 6 + 4], a.denseJtr[v * 6 + 5]);
            resTrans = resTrans - mk(a.denseJtr[v * 6 + 0], a.denseJtr[v * 6 + 1], a.denseJtr[v * 6 + 2]);
        }
        const V3 pr = mk(m[4] - m[5], m[4] - m[8], m[4] - m[10]);            // sum (da.da, db.db, dc.dc)
        const V3 precR = mk(pr.x > BF_FLOAT_EPSILON ? 1.0f / pr.x : 1.0f, pr.y > BF_FLOAT_EPSILON ? 1.0f / pr.y : 1.0f, pr.z > BF_FLOAT_EPSILON ? 1.0f / pr.z : 1.0f);
        const float pt = (m[0] > BF_FLOAT_EPSILON) ? 1.0f / m[0] : 1.0f;
        const V3 precT = mk(pt, pt, pt);
        st3(a.precRot, v, precR); st3(a.precTrans, v, precT);
        st3(a.deltaRot, v, mk(0, 0, 0)); st3(a.deltaTrans, v, mk(0, 0, 0));
        st3(a.rRot, v, resRot); st3(a.rTrans, v, resTrans);
        const V3 p0r = mulv(precR, resRot), p0t = mulv(precT, resTrans);
        st3(a.pRot, v, p0r); st3(a.pTrans, v, p0t);
        part += dot(resRot, p0r) + dot(resTrans, p0t);
    }
    float rDotzOld = grid.sum(part, a.partials + a.maxGrid, sRed);        // second array: the first is rewritten by PCG step A

    const bool peerMode = Grid::kPeers && a.world > 1;
    // (3) PCG iterations (SolverBundling.cu:1024-1108): rows are dealt to warps; lanes split a row's segments
    const unsigned warpsPerBlock = blockDim.x / 32, gwarp = blockIdx.x * warpsPerBlock + (threadIdx.x >> 5), nwarps = gridDim.x * warpsPerBlock;
    const unsigned lane = threadIdx.x & 31;
    unsigned pcgRun = 0;
    // Two grid barriers per iteration.  The textbook third one (p <- z + beta p must be complete before the next mat-vec) is
    // removed by never materialising p before it is needed: a reader forms p_k(o) = z(o) + beta p_{k-1}(o) on the fly from two
    // vectors that ARE complete, and each row's owner stores its own p_k(v) into the other of two ping-pong buffers (nobody
    // reads that buffer during this mat-vec).  The expression, and therefore every bit, is the one the stored update had.
    float beta = 0.0f;
    if constexpr (Grid::kResident) pcgRun = pcg_resident(a, denseOn, rDotzOld);
    for (unsigned lin = 0; !Grid::kResident && lin < a.nLin; ++lin) {      // the grid's PCG, operands in L2
        bool last = (lin == a.nLin - 1);
        ++pcgRun;
        const bool fly = lin > 0;
        float* const curR = (lin & 1) ? a.p2Rot : a.pRot;   float* const curT = (lin & 1) ? a.p2Trans : a.pTrans;    // p_k of the rows this thread owns
        const float* const prvR = (lin & 1) ? a.pRot : a.p2Rot; const float* const prvT = (lin & 1) ? a.pTrans : a.p2Trans;    // p_{k-1}, complete
        // A: Ap = H p, partial p.Ap.  Sharded: this rank's rows only (v = rank + world k), each result stored into every rank's exchange region.
        float pAp = 0.0f;
        const unsigned par = lin & 1u;
        for (unsigned kRow = gwarp; ; kRow += nwarps) {
            const unsigned v = peerMode ? (unsigned)a.rank + (unsigned)a.world * (kRow + (a.rank == 0 ? 1u : 0u)) : 1u + kRow;
            if (v >= N) break;
            const int ns = a.segCount[v], rs = a.rowStart[v];
            float y[6] = { 0, 0, 0, 0, 0, 0 };
            for (int sI = lane; sI < ns; sI += 32) {
                const unsigned o = (unsigned)a.segs[rs + sI].nbr;
                if (o == 0 || o >= N) continue;                         // variable 0 is fixed: its p is zero by construction
                const V3 pr = fly ? ld3(a.zRot, o) + ld3(prvR, o) * beta : ld3(a.pRot, o);
                const V3 pt = fly ? ld3(a.zTrans, o) + ld3(prvT, o) * beta : ld3(a.pTrans, o);
                blk_mv(&a.offBlk[36 * (size_t)(rs + sI)], pr, pt, y);
            }
            if (denseOn) {      // dense J^T J p (applyJTJDenseDevice, SolverBundlingDenseUtil.h:371-411) over the pairs image v is part of; record
                                // coordinates are translation-first: p_rec = (trans, rot), y_rec[0..2] -> trans rows, y_rec[3..5] -> rot rows
                const int e1 = a.dnbrStart[v + 1];
                for (int e = a.dnbrStart[v] + (int)lane; e < e1; e += 32) {
                    const int2 nb = a.dnbr[e];
                    const unsigned o = (unsigned)nb.x;
                    if (o == 0) continue;
                    const float* B = &a.pairOut[(size_t)nb.y * 90 + 42];                 // J_lo^T J_hi, [a over lo][b over hi]
                    const V3 pr = fly ? ld3(a.zRot, o) + ld3(prvR, o) * beta : ld3(a.pRot, o);
                    const V3 pt = fly ? ld3(a.zTrans, o) + ld3(prvT, o) * beta : ld3(a.pTrans, o);
                    const int sa = (v < o) ? 6 : 1, sb = (v < o) ? 1 : 6;               // v is the pair's hi image: the transposed block
#pragma unroll
                    for (int r = 0; r < 3; ++r) {
                        y[3 + r] += B[r * sa + 0 * sb] * pt.x + B[r * sa + 1 * sb] * pt.y + B[r * sa + 2 * sb] * pt.z + B[r * sa + 3 * sb] * pr.x + B[r * sa + 4 * sb] * pr.y + B[r * sa + 5 * sb] * pr.z;
                        y[r] += B[(3 + r) * sa + 0 * sb] * pt.x + B[(3 + r) * sa + 1 * sb] * pt.y + B[(3 + r) * sa + 2 * sb] * pt.z + B[(3 + r) * sa + 3 * sb] * pr.x + B[(3 + r) * sa + 4 * sb] * pr.y + B[(3 + r) * sa + 5 * sb] * pr.z;
                    }
                }
            }
#pragma unroll
            for (int k = 0; k < 6; ++k) y[k] = warp_sum(y[k]);
            if (lane == 0) {
                const V3 pr = fly ? ld3(a.zRot, v) + ld3(prvR, v) * beta : ld3(a.pRot, v);
                const V3 pt = fly ? ld3(a.zTrans, v) + ld3(prvT, v) * beta : ld3(a.pTrans, v);
                if (fly && !peerMode) { st3(curR, v, pr); st3(curT, v, pt); }       // sharded: step B forms and stores p_k for every row itself
                blk_mv(&a.diagBlk[36 * (size_t)v], pr, pt, y);
                if (denseOn) {
                    const float* D = &a.denseDiag[36 * (size_t)v];
#pragma unroll
                    for (int r = 0; r < 3; ++r) {
                        y[3 + r] += D[r * 6 + 0] * pt.x + D[r * 6 + 1] * pt.y + D[r * 6 + 2] * pt.z + D[r * 6 + 3] * pr.x + D[r * 6 + 4] * pr.y + D[r * 6 + 5] * pr.z;
                        y[r] += D[(3 + r) * 6 + 0] * pt.x + D[(3 + r) * 6 + 1] * pt.y + D[(3 + r) * 6 + 2] * pt.z + D[(3 + r) * 6 + 3] * pr.x + D[(3 + r) * 6 + 4] * pr.y + D[(3 + r) * 6 + 5] * pr.z;
                    }
                }
                if (!peerMode) { st3(a.ApRot, v, mk(y[0], y[1], y[2])); st3(a.ApTrans, v, mk(y[3], y[4], y[5])); }
                else
                    for (int g = 0; g < a.world; ++g) {           // 24 bytes per row and rank over NVLink; ordered before the flag by the fence in peer_barrier
                        float* ap = peer_ap(a.peer[g], a.peerMaxN, par);
                        st3(ap, v, mk(y[0], y[1], y[2])); st3(ap + 3 * (size_t)a.peerMaxN, v, mk(y[3], y[4], y[5]));
                    }
                pAp += pr.x * y[0] + pr.y * y[1] + pr.z * y[2] + pt.x * y[3] + pt.y * y[4] + pt.z * y[5];
            }
        }
        float dotProduct;
        if (!peerMode) {
            dotProduct = grid.sum(pAp, a.partials, sRed);
        } else {
            pAp = block_sum(pAp, sRed);
            if (threadIdx.x < (unsigned)a.world) peer_partials(a.peer[threadIdx.x], a.peerMaxN, a.maxGrid, par)[(size_t)a.rank * a.maxGrid + blockIdx.x] = pAp;   // pAp is uniform in the CTA
            peer_barrier(a, a.seqBase + lin + 1u, grid);
            // every rank adds the same world x grid partial sums in the same order: identical bits everywhere
            const float* pp = peer_partials(a.peer[a.rank], a.peerMaxN, a.maxGrid, par);
            if (threadIdx.x < 32) {
                float acc = 0.0f;
                for (unsigned e = threadIdx.x; e < (unsigned)a.world * gridDim.x; e += 32) acc += __ldcg(&pp[(size_t)(e / gridDim.x) * a.maxGrid + (e % gridDim.x)]);
                acc = warp_sum(acc);
                if (threadIdx.x == 0) sRed[0] = acc;
            }
            __syncthreads();
            dotProduct = sRed[0];
            __syncthreads();
        }
        // B: step, residual, preconditioned residual, partial z.r
        float alpha = 0.0f;
        if (dotProduct > BF_FLOAT_EPSILON) alpha = rDotzOld / dotProduct;
        float zr = 0.0f;
        const float* const apR = peerMode ? peer_ap(a.peer[a.rank], a.peerMaxN, par) : a.ApRot;
        const float* const apT = peerMode ? peer_ap(a.peer[a.rank], a.peerMaxN, par) + 3 * (size_t)a.peerMaxN : a.ApTrans;
        for (unsigned v = tid; v < N; v += nth) {
            if (v == 0) continue;
            V3 pkR, pkT;
            if (peerMode) {      // the expression the mat-vec read: p_k = z + beta p_{k-1}, materialised here for every row (the owner-only store does not reach the other ranks)
                pkR = fly ? ld3(a.zRot, v) + ld3(prvR, v) * beta : ld3(a.pRot, v);
                pkT = fly ? ld3(a.zTrans, v) + ld3(prvT, v) * beta : ld3(a.pTrans, v);
                if (fly) { st3(curR, v, pkR); st3(curT, v, pkT); }
            } else { pkR = ld3(curR, v); pkT = ld3(curT, v); }
            st3(a.deltaRot, v, ld3(a.deltaRot, v) + pkR * alpha);
            st3(a.deltaTrans, v, ld3(a.deltaTrans, v) + pkT * alpha);
            const V3 rR = ld3(a.rRot, v) - V3(mk(__ldcg(&apR[3 * v]), __ldcg(&apR[3 * v + 1]), __ldcg(&apR[3 * v + 2]))) * alpha, rT = ld3(a.rTrans, v) - V3(mk(__ldcg(&apT[3 * v]), __ldcg(&apT[3 * v + 1]), __ldcg(&apT[3 * v + 2]))) * alpha;
            st3(a.rRot, v, rR); st3(a.rTrans, v, rT);
            const V3 zR = mulv(ld3(a.precRot, v), rR), zT = mulv(ld3(a.precTrans, v), rT);
            st3(a.zRot, v, zR); st3(a.zTrans, v, zT);
            zr += dot(zR, rR) + dot(zT, rT);
        }
        const float rDotzNew = grid.sum(zr, a.partials + a.maxGrid, sRed);
        if (fabsf(dotProduct) < 5e-7f) last = true;                     // ENABLE_EARLY_OUT (:1088-1093)
        // C: the new direction's coefficient; the direction itself is formed by the next mat-vec (+ Lie update on the last
        //    iteration, LieDerivUtil.h:301-307)
        beta = 0.0f;
        if (rDotzOld > BF_FLOAT_EPSILON) beta = rDotzNew / rDotzOld;
        if (last) {
            for (unsigned v = tid; v < N; v += nth) {
                if (v == 0) continue;
                float U[16], Cm[16], P[16];
                pose_to_matrix(ld3(a.deltaRot, v), ld3(a.deltaTrans, v), U);
                pose_to_matrix(ld3(a.xRot, v), ld3(a.xTrans, v), Cm);
                mat4_mul(U, Cm, P);
                V3 nr, nt;
                matrix_to_pose(P, nr, nt);
                st3(a.xRot, v, nr); st3(a.xTrans, v, nt);
            }
        }
        rDotzOld = rDotzNew;
        if (last) break;
    }

    // (4) GN convergence: max |delta| over valid variables (SolverBundling.cu:694-749, 1206)
    float md = 0.0f;
    for (unsigned v = tid; v < N; v += nth) {
        if (v == 0 || (a.validImages && a.validImages[v] == 0)) continue;
        const V3 dr = ld3(a.deltaRot, v), dt = ld3(a.deltaTrans, v);
        md = fmaxf(md, fmaxf(fmaxf(fabsf(dr.x), fabsf(dr.y)), fabsf(dr.z)));
        md = fmaxf(md, fmaxf(fmaxf(fabsf(dt.x), fabsf(dt.y)), fabsf(dt.z)));
    }
    md = warp_max(md);
    if ((threadIdx.x & 31) == 0) sRed[threadIdx.x >> 5] = md;
    __syncthreads();
    if (threadIdx.x == 0) {
        float m2 = 0.0f;
        for (unsigned wI = 0; wI < blockDim.x / 32; ++wI) m2 = fmaxf(m2, sRed[wI]);
        a.partials[blockIdx.x] = m2;
    }
    grid.sync();
    if (tid == 0) {
        float m2 = 0.0f;
        for (unsigned b = 0; b < gridDim.x; ++b) m2 = fmaxf(m2, __ldcg(&a.partials[b]));
        a.scal[SC_MAXDELTA_BITS] = __float_as_uint(m2);
        a.scal[SC_GN_RUN] += 1;
        a.scal[SC_PCG_RUN] += pcgRun;
        if (!a.isLastGn && m2 < 0.005f) a.scal[SC_DONE] = 1;
    }
}

// ---- dense depth / colour term (SURVEY.md row a13) -------------------------------------------------------------------
// FindImageImageCorr / FindDenseCorrespondences / Weight / BuildDenseSystem (SolverBundling.cu:30-471) restructured: one CTA
// per candidate pair decides overlap, counts and weights without a host round trip; one CTA per weighted pair reduces its 90
// sums (6x6 blocks ii, jj, ij + two 6-vectors) in registers with a fixed tree; an assemble kernel lays the dense system out
// in pair order.  No atomics: deterministic.
struct DenseArgs {
    const BFCUDACachedFrame* frames; const int* valid; const float* T; const float* Tinv;
    unsigned N, W, H; float fx, fy, mx, my;
    float distThresh, normalThresh, colorThresh, colorGradientMin, depthMin, depthMax;
    unsigned subsample; int usePairwise; float wDepth, wColor;
    float* pairW; int* pairIdx; int* pairCnt; int* pairRowStart; int2* pairIJ; float* pairOut; int* dnbrStart; int2* dnbr; float* diag; float* Jtr; unsigned* scal;
};
__device__ __forceinline__ V3 rot3(const float* m, V3 v) { return mk(m[0] * v.x + m[1] * v.y + m[2] * v.z, m[4] * v.x + m[5] * v.y + m[6] * v.z, m[8] * v.x + m[9] * v.y + m[10] * v.z); }
__device__ __forceinline__ V3 depth_to_cam(const DenseArgs& d, int x, int y, float depth) {
    const float fx = ((float)x - d.mx) / d.fx, fy = ((float)y - d.my) / d.fy;
    return mk(depth * fx, depth * fy, depth);
}
// ICPUtil.h:56-110 (nc channels, validity on channel 0)
template <int NC>
__device__ bool bilinear(const float* __restrict__ img, float x, float y, unsigned W, unsigned H, float* out) {
    const int x0 = (int)floorf(x), y0 = (int)floorf(y);
    const float alpha = x - (float)x0, beta = y - (float)y0;
    float s0[NC], s1[NC], w0 = 0.0f, w1 = 0.0f;
#pragma unroll
    for (int c = 0; c < NC; ++c) { s0[c] = 0.0f; s1[c] = 0.0f; }
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const int xs = x0 + k;
        const float wgt = k ? alpha : (1.0f - alpha);
        if ((unsigned)xs < W && (unsigned)y0 < H) { const float* v = &img[((size_t)y0 * W + xs) * NC]; if (v[0] != -INFINITY) { for (int c = 0; c < NC; ++c) s0[c] += wgt * v[c]; w0 += wgt; } }
        if ((unsigned)xs < W && (unsigned)(y0 + 1) < H) { const float* v = &img[((size_t)(y0 + 1) * W + xs) * NC]; if (v[0] != -INFINITY) { for (int c = 0; c < NC; ++c) s1[c] += wgt * v[c]; w1 += wgt; } }
    }
    float ww = 0.0f;
#pragma unroll
    for (int c = 0; c < NC; ++c) out[c] = 0.0f;
    if (w0 > 0.0f) { for (int c = 0; c < NC; ++c) out[c] += (1.0f - beta) * (s0[c] / w0); ww += (1.0f - beta); }
    if (w1 > 0.0f) { for (int c = 0; c < NC; ++c) out[c] += beta * (s1[c] / w1); ww += beta; }
    if (ww > 0.0f) { for (int c = 0; c < NC; ++c) out[c] = out[c] / ww; return true; }
    for (int c = 0; c < NC; ++c) out[c] = -INFINITY;
    return false;
}
__device__ __forceinline__ int block_sum_int(int v, int* sRed) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sRed[threadIdx.x >> 5] = v;
    __syncthreads();
    int tot = 0;
    for (unsigned w = 0; w < blockDim.x / 32; ++w) tot += sRed[w];
    __syncthreads();
    return tot;
}
__global__ void __launch_bounds__(512)
dense_pair_weight_kernel(const DenseArgs d) {
    __shared__ int sRed[16];
    const unsigned i = blockIdx.x, j = blockIdx.y, N = d.N;
    if (d.scal[SC_DONE] != 0) return;
    if (i >= j) { if (threadIdx.x == 0 && i < N && j < N) d.pairW[i * N + j] = 0.0f; return; }
    float weight = 0.0f; int overlap = 0;
    bool cand = d.usePairwise || (j == i + 1);
    if (cand && d.valid && (d.valid[i] == 0 || d.valid[j] == 0)) cand = false;
    float tr[16];
    if (cand) {
        mat4_mul(&d.Tinv[16 * i], &d.T[16 * j], tr);
        const float inv = 1.0f / sqrtf(3.0f);
        const V3 x = mk(inv, inv, inv), vv = rot3(tr, x);
        const float angle = acosf(fminf(fmaxf(dot(x, vv), -1.0f), 1.0f));
        if (!(fabsf(angle) < 0.52f)) cand = false;                       // computeAngleDiff, ~30 degrees (:60)
    }
    if (cand) {
        const BFCUDACachedFrame fi = d.frames[i], fj = d.frames[j];
        // overlap pre-filter on the sub-sampled grid (SolverBundlingDenseUtil.h:22-42)
        int hit = 0;
        {
            const unsigned subW = d.W / d.subsample, t = threadIdx.x;
            const unsigned x = (t % subW) * d.subsample, y = (t / subW) * d.subsample, idx = y * d.W + x;
            if (idx < d.W * d.H) {
                const V3 cj = depth_to_cam(d, (int)x, (int)y, fj.d_depthDownsampled[idx]);
                if (cj.z > d.depthMin && cj.z < d.depthMax) {
                    const V3 s2t = xf(tr, cj);
                    const int tx = (int)roundf(s2t.x * d.fx / s2t.z + d.mx), ty = (int)roundf(s2t.y * d.fy / s2t.z + d.my);
                    if (tx >= 0 && ty >= 0 && tx < (int)d.W && ty < (int)d.H) {
                        const V3 ct = depth_to_cam(d, tx, ty, fi.d_depthDownsampled[ty * d.W + tx]);
                        if (ct.z > d.depthMin && ct.z < d.depthMax && length(s2t - ct) <= d.distThresh) hit = 1;
                    }
                }
            }
        }
        const int found = block_sum_int(hit, sRed);
        if (found > 10) {
            overlap = 1;
            // full-resolution count with the uchar4 normals (SolverBundlingDenseUtil.h:152-184)
            int cnt = 0;
            for (unsigned idx = threadIdx.x; idx < d.W * d.H; idx += blockDim.x) {
                const unsigned x = idx % d.W, y = idx / d.W;
                const V3 cj = depth_to_cam(d, (int)x, (int)y, fj.d_depthDownsampled[idx]);
                if (!(cj.z > d.depthMin && cj.z < d.depthMax)) continue;
                const uchar4 nu = reinterpret_cast<const uchar4*>(fj.d_normalsDownsampledUCHAR4)[idx];
                if ((nu.x | nu.y | nu.z | nu.w) == 0) continue;
                const V3 nj = rot3(tr, mk((float)nu.x / 255.0f * 2.0f - 1.0f, (float)nu.y / 255.0f * 2.0f - 1.0f, (float)nu.z / 255.0f * 2.0f - 1.0f));
                const V3 s2t = xf(tr, cj);
                const int tx = (int)roundf(s2t.x * d.fx / s2t.z + d.mx), ty = (int)roundf(s2t.y * d.fy / s2t.z + d.my);
                if (!(tx >= 0 && ty >= 0 && tx < (int)d.W && ty < (int)d.H)) continue;
                const V3 ct = depth_to_cam(d, tx, ty, fi.d_depthDownsampled[ty * d.W + tx]);
                if (!(ct.z > d.depthMin && ct.z < d.depthMax)) continue;
                const uchar4 tu = reinterpret_cast<const uchar4*>(fi.d_normalsDownsampledUCHAR4)[ty * d.W + tx];
                if ((tu.x | tu.y | tu.z | tu.w) == 0) continue;
                const V3 nt = mk((float)tu.x / 255.0f * 2.0f - 1.0f, (float)tu.y / 255.0f * 2.0f - 1.0f, (float)tu.z / 255.0f * 2.0f - 1.0f);
                if (dot(nj, nt) >= d.normalThresh && length(s2t - ct) <= d.distThresh) ++cnt;
            }
            const float count = (float)block_sum_int(cnt, sRed);
            if (count > 0) weight = (count < 800) ? 0.0f : 1.0f / fminf(logf(count), 9.0f);      // (:162-180)
        }
    }
    if (threadIdx.x == 0) {
        d.pairW[i * N + j] = weight;
        if (overlap) atomicAdd(&d.scal[SC_DENSE_OVERLAP], 1u);
        if (weight != 0.0f) atomicAdd(&d.scal[SC_DENSE_PAIRS], 1u);
    }
}

// rows of one dense correspondence: depth row = -n^T d(s2t)/de, colour row = dI^T dProj d(s2t)/de, with d(s2t)/de for image i
// (evalLie_derivI, A = Tj^-1, D = Ti) and image j (evalLie_derivJ, A = Ti^-1, D = Tj) in closed form (LieDerivUtil.h:247-295):
//   J_i = [ -M | rows_k = d_k x q + (M skew(t_D))_k ],  M = R_T^T R_A, T = A D, q = R_A^T (p - t_T), d_k = k-th column of R_D
//   J_j = [ R_A | -R_A skew(D p) ]
__device__ void lie_jac_i(const float* A, const float* D, V3 p, float J[18]) {
    float T[16]; mat4_mul(A, D, T);
    const V3 pt = p - mk(T[3], T[7], T[11]);
    const V3 q = mk(A[0] * pt.x + A[4] * pt.y + A[8] * pt.z, A[1] * pt.x + A[5] * pt.y + A[9] * pt.z, A[2] * pt.x + A[6] * pt.y + A[10] * pt.z);
    float M[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) M[r * 3 + c] = T[0 * 4 + r] * A[0 * 4 + c] + T[1 * 4 + r] * A[1 * 4 + c] + T[2 * 4 + r] * A[2 * 4 + c];
    const V3 tD = mk(D[3], D[7], D[11]);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        J[k * 6 + 0] = -M[k * 3 + 0]; J[k * 6 + 1] = -M[k * 3 + 1]; J[k * 6 + 2] = -M[k * 3 + 2];
        const V3 dk = mk(D[0 * 4 + k], D[1 * 4 + k], D[2 * 4 + k]);
        const V3 c1 = cross(dk, q);
        // (M skew(t))_k = row_k(M) * [[0,-tz,ty],[tz,0,-tx],[-ty,tx,0]]
        const float m0 = M[k * 3 + 0], m1 = M[k * 3 + 1], m2 = M[k * 3 + 2];
        J[k * 6 + 3] = c1.x + (m1 * tD.z - m2 * tD.y);
        J[k * 6 + 4] = c1.y + (-m0 * tD.z + m2 * tD.x);
        J[k * 6 + 5] = c1.z + (m0 * tD.y - m1 * tD.x);
    }
}
__device__ void lie_jac_j(const float* A, const float* D, V3 p, float J[18]) {
    const V3 a = xf(D, p);
    const float G[3][3] = { { 0.0f, a.z, -a.y }, { -a.z, 0.0f, a.x }, { a.y, -a.x, 0.0f } };
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        J[r * 6 + 0] = A[r * 4 + 0]; J[r * 6 + 1] = A[r * 4 + 1]; J[r * 6 + 2] = A[r * 4 + 2];
#pragma unroll
        for (int c = 0; c < 3; ++c) J[r * 6 + 3 + c] = A[r * 4 + 0] * G[0][c] + A[r * 4 + 1] * G[1][c] + A[r * 4 + 2] * G[2][c];
    }
}
// one 128-thread CTA per weighted pair; 90 sums per thread: ii (21, a<=b), jj (21), ij (36, a over i, b over j), gi (6), gj (6)
__device__ __forceinline__ void accum_rows(float* acc, const float* ri, const float* rj, float res, float w, bool hasI, bool hasJ) {
    int k = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int b = a; b < 6; ++b) { if (hasI) acc[k] += ri[a] * ri[b] * w; if (hasJ) acc[21 + k] += rj[a] * rj[b] * w; ++k; }
    if (hasI && hasJ) {
#pragma unroll
        for (int a = 0; a < 6; ++a)
#pragma unroll
            for (int b = 0; b < 6; ++b) acc[42 + a * 6 + b] += ri[a] * rj[b] * w;
    }
#pragma unroll
    for (int a = 0; a < 6; ++a) { if (hasI) acc[78 + a] += ri[a] * res * w; if (hasJ) acc[84 + a] += rj[a] * res * w; }
}
// ---- pair list: the weighted pairs in (i, j) order, and per image the pairs it is part of ----
// one warp per image v: pairs it leads (j > v) and pairs it is part of
__global__ void dense_pair_count_kernel(const DenseArgs d) {
    if (d.scal[SC_DONE] != 0) return;
    const unsigned v = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31, N = d.N;
    if (v >= N) return;
    int lead = 0, all = 0;
    for (unsigned o = lane; o < N; o += 32) {
        if (o == v) continue;
        const bool w = (o < v ? d.pairW[o * N + v] : d.pairW[v * N + o]) != 0.0f;
        all += w ? 1 : 0; lead += (w && o > v) ? 1 : 0;
    }
    for (int s = 16; s > 0; s >>= 1) { lead += __shfl_xor_sync(0xffffffffu, lead, s); all += __shfl_xor_sync(0xffffffffu, all, s); }
    if (lane == 0) { d.pairCnt[v] = lead; d.pairCnt[N + v] = all; }
}
// exclusive scans of the two counts (one CTA; N <= 4096)
__global__ void __launch_bounds__(1024)
dense_pair_scan_kernel(const DenseArgs d) {
    if (d.scal[SC_DONE] != 0) return;
    __shared__ int sA[1024], sB[1024];
    const unsigned N = d.N, t = threadIdx.x, per = (N + 1023) / 1024;
    int a = 0, b = 0;
    for (unsigned k = t * per; k < N && k < (t + 1) * per; ++k) { a += d.pairCnt[k]; b += d.pairCnt[N + k]; }
    sA[t] = a; sB[t] = b;
    __syncthreads();
    if (t == 0) { int ra = 0, rb = 0; for (int k = 0; k < 1024; ++k) { const int x = sA[k], y = sB[k]; sA[k] = ra; sB[k] = rb; ra += x; rb += y; } d.pairRowStart[N] = ra; d.dnbrStart[N] = rb; }
    __syncthreads();
    a = sA[t]; b = sB[t];
    for (unsigned k = t * per; k < N && k < (t + 1) * per; ++k) { d.pairRowStart[k] = a; d.dnbrStart[k] = b; a += d.pairCnt[k]; b += d.pairCnt[N + k]; }
}
// one warp per image i: its pairs (i, j > i) in ascending j
__global__ void dense_pair_fill_kernel(const DenseArgs d) {
    if (d.scal[SC_DONE] != 0) return;
    const unsigned i = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31, N = d.N;
    if (i >= N) return;
    int k = d.pairRowStart[i];
    for (unsigned j0 = i + 1; j0 < N; j0 += 32) {
        const unsigned j = j0 + lane;
        const bool w = j < N && d.pairW[i * N + j] != 0.0f;
        const unsigned bal = __ballot_sync(0xffffffffu, w);
        if (w) { const int kk = k + __popc(bal & ((1u << lane) - 1u)); d.pairIJ[kk] = make_int2((int)i, (int)j); d.pairIdx[i * N + j] = kk; }
        k += __popc(bal);
    }
}
__global__ void __launch_bounds__(128)
dense_build_kernel(const DenseArgs d) {
    __shared__ float sAcc[4][90];
    const unsigned N = d.N;
    if (d.scal[SC_DONE] != 0) return;
    const int P = d.pairRowStart[N];
  for (int pk = (int)blockIdx.x; pk < P; pk += (int)gridDim.x) {
    const int2 ij = d.pairIJ[pk];
    const unsigned i = (unsigned)ij.x, j = (unsigned)ij.y;
    const float pairW = d.pairW[i * N + j];
    const BFCUDACachedFrame fi = d.frames[i], fj = d.frames[j];
    const float* Ti = &d.T[16 * i]; const float* Tj = &d.T[16 * j]; const float* Tii = &d.Tinv[16 * i]; const float* Tji = &d.Tinv[16 * j];
    float tr[16]; mat4_mul(Tii, Tj, tr);
    float acc[90];
#pragma unroll
    for (int k = 0; k < 90; ++k) acc[k] = 0.0f;
    const bool hasI = i > 0, hasJ = j > 0;
    for (unsigned idx = threadIdx.x; idx < d.W * d.H; idx += blockDim.x) {
        // findDenseCorr, camera-position version with float4 normals (SolverBundlingDenseUtil.h:79-113)
        const float4 cp = reinterpret_cast<const float4*>(fj.d_cameraposDownsampled)[idx];
        if (!(cp.z > d.depthMin && cp.z < d.depthMax)) continue;
        const V3 cps = mk(cp.x, cp.y, cp.z);
        const float4 nj4 = reinterpret_cast<const float4*>(fj.d_normalsDownsampled)[idx];
        if (nj4.x == -INFINITY) continue;
        const float n4[4] = { tr[0] * nj4.x + tr[1] * nj4.y + tr[2] * nj4.z + tr[3] * nj4.w, tr[4] * nj4.x + tr[5] * nj4.y + tr[6] * nj4.z + tr[7] * nj4.w,
                              tr[8] * nj4.x + tr[9] * nj4.y + tr[10] * nj4.z + tr[11] * nj4.w, tr[12] * nj4.x + tr[13] * nj4.y + tr[14] * nj4.z + tr[15] * nj4.w };
        const V3 s2t = xf(tr, cps);
        const float sx = s2t.x * d.fx / s2t.z + d.mx, sy = s2t.y * d.fy / s2t.z + d.my;
        const int tx = (int)roundf(sx), ty = (int)roundf(sy);
        if (!(tx >= 0 && ty >= 0 && tx < (int)d.W && ty < (int)d.H)) continue;
        float ci[4], ni[4];
        bilinear<4>(fi.d_cameraposDownsampled, sx, sy, d.W, d.H, ci);
        if (!(ci[2] > d.depthMin && ci[2] < d.depthMax)) continue;
        bilinear<4>(fi.d_normalsDownsampled, sx, sy, d.W, d.H, ni);
        if (ni[0] == -INFINITY) continue;
        const V3 cpt = mk(ci[0], ci[1], ci[2]), nt = mk(ni[0], ni[1], ni[2]);
        const float dist = length(s2t - cpt);
        const float dNormal = n4[0] * ni[0] + n4[1] * ni[1] + n4[2] * ni[2] + n4[3] * ni[3];
        if (!(dNormal >= d.normalThresh && dist <= d.distThresh)) continue;
        float Ji[18], Jj[18];
        if (hasI) lie_jac_i(Tji, Ti, cps, Ji);
        if (hasJ) lie_jac_j(Tii, Tj, cps, Jj);
        if (d.wDepth > 0.0f) {
            const float res = dot(cpt - s2t, nt);
            const float w = d.wDepth * pairW * powf(fmaxf(0.0f, 1.0f - cpt.z / 2.0f), 2.5f);       // (:256)
            float ri[6], rj[6];
#pragma unroll
            for (int c = 0; c < 6; ++c) {
                ri[c] = hasI ? -(Ji[c] * nt.x + Ji[6 + c] * nt.y + Ji[12 + c] * nt.z) : 0.0f;
                rj[c] = hasJ ? -(Jj[c] * nt.x + Jj[6 + c] * nt.y + Jj[12 + c] * nt.z) : 0.0f;
            }
            accum_rows(acc, ri, rj, res, w, hasI, hasJ);
        }
        if (d.wColor > 0.0f) {
            float dI[2], It;
            bilinear<2>(fi.d_intensityDerivsDownsampled, sx, sy, d.W, d.H, dI);
            bilinear<1>(fi.d_intensityDownsampled, sx, sy, d.W, d.H, &It);
            const float cres = It - fj.d_intensityDownsampled[idx];
            if (dI[0] != -INFINITY && fabsf(cres) < d.colorThresh && sqrtf(dI[0] * dI[0] + dI[1] * dI[1]) > d.colorGradientMin) {
                const float z2 = s2t.z * s2t.z;
                const float P00 = d.fx / s2t.z, P02 = -d.fx * s2t.x / z2, P11 = d.fy / s2t.z, P12 = -d.fy * s2t.y / z2;
                float ri[6], rj[6];
#pragma unroll
                for (int c = 0; c < 6; ++c) {
                    ri[c] = hasI ? dI[0] * (P00 * Ji[c] + P02 * Ji[12 + c]) + dI[1] * (P11 * Ji[6 + c] + P12 * Ji[12 + c]) : 0.0f;
                    rj[c] = hasJ ? dI[0] * (P00 * Jj[c] + P02 * Jj[12 + c]) + dI[1] * (P11 * Jj[6 + c] + P12 * Jj[12 + c]) : 0.0f;
                }
                const float w = d.wColor * pairW * fmaxf(0.0f, 1.0f - fabsf(cres) / (1.15f * d.colorThresh));   // (:294)
                accum_rows(acc, ri, rj, cres, w, hasI, hasJ);
            }
        }
    }
    // fixed-shape reduction: warp tree, then the 4 warps in order
#pragma unroll
    for (int k = 0; k < 90; ++k) { const float v = warp_sum(acc[k]); if ((threadIdx.x & 31) == 0) sAcc[threadIdx.x >> 5][k] = v; }
    __syncthreads();
    if (threadIdx.x < 90) d.pairOut[(size_t)pk * 90 + threadIdx.x] = sAcc[0][threadIdx.x] + sAcc[1][threadIdx.x] + sAcc[2][threadIdx.x] + sAcc[3][threadIdx.x];
    __syncthreads();
  }
}
// Per image v (one 64-thread CTA): its pair list {other image, pair index} in ascending other image, the diagonal 6x6 block and J^T r as the sums of
// its pairs' records in that order (the order the dense (6N)^2 assembly of the reference's layout sums them in) -- translation first per image.
__device__ __forceinline__ int tri_index(int a, int b) { if (a > b) { const int t = a; a = b; b = t; } return a * 6 - (a * (a - 1)) / 2 + (b - a); }   // (a<=b) -> 0..20
__global__ void __launch_bounds__(64)
dense_assemble_kernel(const DenseArgs d) {
    const unsigned N = d.N, v = blockIdx.x, t = threadIdx.x;
    if (d.scal[SC_DONE] != 0) return;
    const int e0 = d.dnbrStart[v], e1 = d.dnbrStart[v + 1];
    if (t < 32) {
        int k = e0;
        for (unsigned o0 = 0; o0 < N; o0 += 32) {
            const unsigned o = o0 + t;
            const bool w = o < N && o != v && (o < v ? d.pairW[o * N + v] : d.pairW[v * N + o]) != 0.0f;
            const unsigned bal = __ballot_sync(0xffffffffu, w);
            if (w) d.dnbr[k + __popc(bal & ((1u << t) - 1u))] = make_int2((int)o, o < v ? d.pairIdx[o * N + v] : d.pairIdx[v * N + o]);
            k += __popc(bal);
        }
    }
    __syncthreads();
    if (t < 36) {
        const int a = (int)t / 6, b = (int)t % 6, tri = tri_index(a, b);
        float val = 0.0f;
        for (int e = e0; e < e1; ++e) { const int2 nb = d.dnbr[e]; val += d.pairOut[(size_t)nb.y * 90 + ((unsigned)nb.x > v ? 0 : 21) + tri]; }
        d.diag[36 * (size_t)v + t] = val;
    } else if (t < 42) {
        const int a = (int)t - 36;
        float sum = 0.0f;
        for (int e = e0; e < e1; ++e) { const int2 nb = d.dnbr[e]; sum += d.pairOut[(size_t)nb.y * 90 + ((unsigned)nb.x > v ? 78 : 84) + a]; }
        d.Jtr[6 * v + a] = sum;
    }
    if (v == 0 && t == 0) d.scal[SC_DENSE_ON] = (d.scal[SC_DENSE_OVERLAP] > 0) ? 1u : 0u;
}
// test accessor: the block-sparse system scattered into the reference's dense layout ((6N)^2 row-major, zeroed by the caller)
__global__ void dense_scatter_kernel(unsigned N, const int* dnbrStart, const int2* dnbr, const float* pairOut, const float* diag, float* JtJ) {
    const unsigned v = blockIdx.x, dim = 6 * N;
    for (unsigned t = threadIdx.x; t < 36; t += blockDim.x) JtJ[(size_t)(6 * v + t / 6) * dim + 6 * v + t % 6] = diag[36 * (size_t)v + t];
    for (int e = dnbrStart[v]; e < dnbrStart[v + 1]; ++e) {
        const int2 nb = dnbr[e];
        const unsigned o = (unsigned)nb.x;
        for (unsigned t = threadIdx.x; t < 36; t += blockDim.x) {
            const unsigned ra = t / 6, cb = t % 6;
            JtJ[(size_t)(6 * v + ra) * dim + 6 * o + cb] = pairOut[(size_t)nb.y * 90 + 42 + (v < o ? ra * 6 + cb : cb * 6 + ra)];
        }
    }
}

// ---- small kernels behind the reference-named stubs -------------------------------------------------------------
__global__ void poses_to_matrices_kernel(const float* rot, const float* trans, unsigned n, float* T, float* Tinv, const int* valid) {
    const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n || (valid && valid[k] == 0)) return;
    float M[16];
    pose_to_matrix(ld3(rot, k), ld3(trans, k), M);
    for (int e = 0; e < 16; ++e) T[16 * k + e] = M[e];
    if (Tinv) { float Mi[16]; mat4_inverse(M, Mi); for (int e = 0; e < 16; ++e) Tinv[16 * k + e] = Mi[e]; }
}
// first kernel of a dense GN iteration: matrices for this iteration's poses + reset of the pair counters -- skipped once an
// earlier iteration has converged, so the statistics of the last iteration that ran stay readable
__global__ void dense_begin_kernel(const float* rot, const float* trans, unsigned n, float* T, float* Tinv, unsigned* scal) {
    if (scal[SC_DONE] != 0) return;
    const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k == 0) { scal[SC_DENSE_ON] = 0; scal[SC_DENSE_OVERLAP] = 0; scal[SC_DENSE_PAIRS] = 0; }
    if (k >= n) return;
    float M[16], Mi[16];
    pose_to_matrix(ld3(rot, k), ld3(trans, k), M);
    mat4_inverse(M, Mi);
    for (int e = 0; e < 16; ++e) { T[16 * k + e] = M[e]; Tinv[16 * k + e] = Mi[e]; }
}
__global__ void matrices_to_poses_kernel(const float* T, unsigned n, float* rot, float* trans, const int* valid) {
    const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n || (valid && valid[k] == 0)) return;
    V3 r, t;
    matrix_to_pose(&T[16 * k], r, t);
    st3(rot, k, r); st3(trans, k, t);
}
// evalAbsMaxResidualDevice (SolverBundlingEquationsLie.h:27-40)
__device__ __forceinline__ float abs_max_residual(const BFEntryJ& c, const float* xRot, const float* xTrans, float w) {
    if (!corr_valid(c)) return 0.0f;
    float TI[16], TJ[16];
    pose_to_matrix(ld3(xRot, c.imgIdx_i), ld3(xTrans, c.imgIdx_i), TI);
    pose_to_matrix(ld3(xRot, c.imgIdx_j), ld3(xTrans, c.imgIdx_j), TJ);
    const V3 d = xf(TI, mk(c.pos_i[0], c.pos_i[1], c.pos_i[2])) - xf(TJ, mk(c.pos_j[0], c.pos_j[1], c.pos_j[2]));
    return fmaxf(w * fabsf(d.z), fmaxf(w * fabsf(d.x), w * fabsf(d.y)));
}
// per-512-correspondence block maximum + first index attaining it (SolverBundling.cu:511-550)
__global__ void __launch_bounds__(512)
eval_max_residual_kernel(const BFEntryJ* corr, unsigned C, const float* xRot, const float* xTrans, float w, float* maxRes, int* maxIdx) {
    __shared__ float sV[16]; __shared__ int sI[16];
    const unsigned x = blockIdx.x * blockDim.x + threadIdx.x;
    float v = 0.0f; int idx = 0;
    if (x < C) { v = abs_max_residual(corr[x], xRot, xTrans, w); idx = (int)x; }
    // warp arg-max, ties to the lower index (the reference's strict '<' keeps the earlier entry)
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_down_sync(0xffffffffu, v, o); const int oi = __shfl_down_sync(0xffffffffu, idx, o);
        if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
    }
    if ((threadIdx.x & 31) == 0) { sV[threadIdx.x >> 5] = v; sI[threadIdx.x >> 5] = idx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < 16; ++k) if (sV[k] > v || (sV[k] == v && sI[k] < idx)) { v = sV[k]; idx = sI[k]; }
        maxRes[blockIdx.x] = v; maxIdx[blockIdx.x] = idx;
    }
}
// grid-wide maximum in one launch (single CTA over the block maxima): d_out = {max, index bits}
__global__ void reduce_max_kernel(const float* maxRes, const int* maxIdx, unsigned n, float* out2) {
    __shared__ float sV[32]; __shared__ int sI[32];
    float v = 0.0f; int idx = 0;
    for (unsigned k = threadIdx.x; k < n; k += blockDim.x) if (maxRes[k] > v) { v = maxRes[k]; idx = maxIdx[k]; }
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_down_sync(0xffffffffu, v, o); const int oi = __shfl_down_sync(0xffffffffu, idx, o);
        if (ov > v || (ov == v && ov > 0.0f && oi < idx)) { v = ov; idx = oi; }
    }
    if ((threadIdx.x & 31) == 0) { sV[threadIdx.x >> 5] = v; sI[threadIdx.x >> 5] = idx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (unsigned k = 1; k < blockDim.x / 32; ++k) if (sV[k] > v || (sV[k] == v && v > 0.0f && sI[k] < idx)) { v = sV[k]; idx = sI[k]; }
        out2[0] = v; out2[1] = __int_as_float(idx);
    }
}
__global__ void count_high_residuals_kernel(const BFEntryJ* corr, unsigned C, const float* xRot, const float* xTrans, float w, float thresh, int* count) {
    const unsigned x = blockIdx.x * blockDim.x + threadIdx.x;
    int hit = 0;
    if (x < C) hit = abs_max_residual(corr[x], xRot, xTrans, w) > thresh ? 1 : 0;
    const unsigned b = __ballot_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(count, __popc(b));
}
__global__ void collect_high_residuals_kernel(const BFEntryJ* corr, unsigned C, const float* xRot, const float* xTrans, float w, float thresh,
                                              int* count, float* outRes, int* outIdx, unsigned maxOut) {
    const unsigned x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= C) return;
    const float r = abs_max_residual(corr[x], xRot, xTrans, w);
    if (r > thresh) { const int k = atomicAdd(count, 1); if ((unsigned)k < maxOut) { outRes[k] = r; outIdx[k] = (int)x; } }
}
__global__ void energy_kernel(const BFEntryJ* corr, unsigned C, const float* xRot, const float* xTrans, float w, float* sum) {
    const unsigned x = blockIdx.x * blockDim.x + threadIdx.x;
    float e = 0.0f;
    if (x < C && corr_valid(corr[x])) {
        const BFEntryJ c = corr[x];
        float TI[16], TJ[16];
        pose_to_matrix(ld3(xRot, c.imgIdx_i), ld3(xTrans, c.imgIdx_i), TI);
        pose_to_matrix(ld3(xRot, c.imgIdx_j), ld3(xTrans, c.imgIdx_j), TJ);
        const V3 d = xf(TI, mk(c.pos_i[0], c.pos_i[1], c.pos_i[2])) - xf(TJ, mk(c.pos_j[0], c.pos_j[1], c.pos_j[2]));
        e = w * dot(d, d);
    }
    e = warp_sum(e);
    if ((threadIdx.x & 31) == 0) atomicAdd(sum, e);
}

// BuildVariablesToCorrespondencesTableDevice (SolverBundling.cu:1226-1248), arrival-order slots
__global__ void table_arrival_kernel(BFEntryJ* corr, unsigned C, unsigned maxPerImage, int* table, int* rows) {
    const unsigned x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= C || !corr_valid(corr[x])) return;
    const unsigned i = corr[x].imgIdx_i, j = corr[x].imgIdx_j;
    const int o0 = atomicAdd(&rows[i], 1), o1 = atomicAdd(&rows[j], 1);
    if ((unsigned)o0 < maxPerImage && (unsigned)o1 < maxPerImage) { table[(size_t)i * maxPerImage + o0] = (int)x; table[(size_t)j * maxPerImage + o1] = (int)x; }
    else { corr[x].imgIdx_i = 0xFFFFFFFFu; corr[x].imgIdx_j = 0xFFFFFFFFu; }
}

// ---- host side ------------------------------------------------------------------------------------------------------
static int run_prep(const BFSolverInput* in, const BFSolverState* st, SolverWs* ws) {
    const unsigned N = in->numberOfImages, C = in->numberOfCorrespondences;
    BF_CHECK(cudaMemsetAsync(ws->rowCount, 0, sizeof(int) * N, stream()));
    BF_CHECK(cudaMemsetAsync(ws->scal + SC_NUM_SEG, 0, sizeof(unsigned), stream()));
    if (C > 0) prep_count_kernel<<<(C + 255) / 256, 256, 0, stream()>>>(in->d_correspondences, C, ws->rowCount);
    prep_scan_kernel<<<1, 1024, 0, stream()>>>(ws->rowCount, ws->rowStart, ws->cursor, in->d_numEntriesPerRow, N, ws->scal);
    if (C > 0) prep_scatter_kernel<<<(C + 255) / 256, 256, 0, stream()>>>(in->d_correspondences, C, ws->rowStart, ws->cursor, ws->entries, ws->nbrs);
    g_launchCount += (C > 0 ? 4 : 2);
    static bool attrSet = false;
    if (!attrSet) { BF_CHECK(cudaFuncSetAttribute(prep_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BF_MAX_ROW * 8)); attrSet = true; }
    prep_rows_kernel<<<N, 256, BF_MAX_ROW * 8, stream()>>>(in->d_correspondences, ws->rowStart, ws->entries, ws->nbrs, ws->segCount, ws->segs,
                                                          in->d_variablesToCorrespondences, in->maxCorrPerImage, ws->scal);
    BF_CHECK(cudaGetLastError());
    (void)st;
    return 0;
}

// ---- Gauss-Newton launch policy -------------------------------------------------------------------------------------------
// Which Grid runs gn_iteration_kernel.  Auto picks by size; bfSolverSetGridPolicy forces one process-wide, so that a test can solve one
// problem under every policy and compare the bits.  A forced policy that cannot run a solve fails it (cudaErrorNotSupported), never falls back.
enum { BF_POLICY_AUTO = 0, BF_POLICY_GRID = 1, BF_POLICY_ONE_CTA = 2, BF_POLICY_CLUSTER = 3 };
static std::atomic<int> g_gridPolicy{ BF_POLICY_AUTO };

struct LaunchLimits { int maxCoResident = 0, clusterCap = 0, maxDynSmem = 0; };
// Probed once per process: the co-resident CTAs of the cooperative grid, the largest launchable cluster of the resident kernel (16 where
// the device allows non-portable sizes, else 8) and the dynamic shared memory it may use.
static int launch_limits(LaunchLimits* out) {
    static std::mutex mu;
    static LaunchLimits lim;
    std::lock_guard<std::mutex> lk(mu);
    if (!lim.clusterCap) {
        LaunchLimits l;
        int perSm = 0;
        BF_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, gn_iteration_kernel<CoopGrid>, BF_SOLVER_THREADS, 0));
        l.maxCoResident = perSm * num_sms();
        auto kern = gn_iteration_kernel<ResidentCluster>;
        int dev = 0, optin = 0;
        cudaFuncAttributes fa;
        BF_CHECK(cudaGetDevice(&dev));
        BF_CHECK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
        BF_CHECK(cudaFuncGetAttributes(&fa, kern));
        l.maxDynSmem = optin - (int)fa.sharedSizeBytes;
        BF_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, l.maxDynSmem));
        l.clusterCap = 8;
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess) {
            const unsigned n16 = BF_RESIDENT_MAX_CLUSTER * BF_RESIDENT_ROWS;
            cudaLaunchConfig_t cfg = {};
            cfg.gridDim = dim3(BF_RESIDENT_MAX_CLUSTER); cfg.blockDim = dim3(BF_SOLVER_THREADS); cfg.dynamicSmemBytes = sizeof(float) * resident_smem_words(n16, false);
            cudaLaunchAttribute at; at.id = cudaLaunchAttributeClusterDimension; at.val.clusterDim.x = BF_RESIDENT_MAX_CLUSTER; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
            cfg.attrs = &at; cfg.numAttrs = 1;
            int nClusters = 0;
            if (cudaOccupancyMaxActiveClusters(&nClusters, kern, &cfg) == cudaSuccess && nClusters >= 1) l.clusterCap = BF_RESIDENT_MAX_CLUSTER;
        }
        (void)cudaGetLastError();
        lim = l;
    }
    *out = lim;
    return 0;
}
// G CTAs: enough to give every row a warp, never more than are co-resident
static int gn_grid(unsigned N, const SolverWs* ws, const LaunchLimits& lim) {
    int grid = (int)((N + (BF_SOLVER_THREADS / 32) - 1) / (BF_SOLVER_THREADS / 32));
    if (grid > num_sms()) grid = num_sms();
    if (grid > lim.maxCoResident) grid = lim.maxCoResident;
    if (grid > ws->maxGrid) grid = ws->maxGrid;
    if (grid < 1) grid = 1;
    return grid;
}
static bool gn_dense(const BFSolverInput* in, unsigned k) {
    const float wDepth = in->weightsDenseDepth ? in->weightsDenseDepth[k] : 0.0f, wColor = in->weightsDenseColor ? in->weightsDenseColor[k] : 0.0f;
    return (wDepth > 0.0f || wColor > 0.0f) && in->d_cacheFrames != nullptr;
}
static bool one_cta_can_run(int grid, const SolverWs* ws) { return ws->world == 1 && grid * BF_SOLVER_THREADS <= OneCtaGrid::kThreads; }
// pcg_resident gives each warp one row (rows 1 .. 8G) and every row's Ap to every CTA: G = ceil(N / 8) CTAs in one cluster
static bool cluster_can_run(unsigned N, bool dense, int grid, const SolverWs* ws, const LaunchLimits& lim) {
    return ws->world == 1 && grid <= lim.clusterCap && (unsigned)grid * BF_RESIDENT_ROWS + 1 >= N &&
           sizeof(float) * resident_smem_words(N, dense) <= (size_t)lim.maxDynSmem;
}
static int pick_policy(unsigned N, bool dense, int grid, const SolverWs* ws, const LaunchLimits& lim) {
    const int forced = g_gridPolicy.load();
    if (forced != BF_POLICY_AUTO) return forced;          // solve_impl has checked that it can run
    // Small problems: the G CTAs as one CTA (same bits, no grid barrier).  H100: 5.9 vs 9.3 us per PCG iteration at N = 11, but
    // 7.8 vs 7.4 at N = 32, where the mat-vec of 32 rows on one SM costs more than the barriers it saves.
    if (N <= BF_SOLVER_ONE_CTA_MAX_N && one_cta_can_run(grid, ws)) return BF_POLICY_ONE_CTA;
    // Up to 128 images: the G CTAs as one cluster with the PCG system in shared memory (same bits, no barrier in the PCG loop).
    // H100 80GB HBM3, 400 W limit, scripts/solver_timing.py, solve time / PCG iterations against the cooperative grid: 2.3 vs 7.3 us
    // at N = 32, 3.2 vs 8.2 at 64, 3.5 vs 8.4 at 128.  At N = 11 the cluster also beat the one-CTA kernel (4.2 vs 5.4 us).  One bench
    // frame-loop run once differed between a cluster build and the one-CTA build, but the bench's outputs also vary between runs of one build.
    // On frame-loop inputs the policies agree bit for bit: tests/test_solver_policies_gpu.py runs a 43-frame stream (local solves at N = 11,
    // dense term on) under each policy and compares every status field and the trajectory.  Moving N <= 16 to the cluster is a
    // performance change of its own; until then it stays on one CTA.
    if (cluster_can_run(N, dense, grid, ws, lim)) return BF_POLICY_CLUSTER;
    return BF_POLICY_GRID;
}
// cudaErrorNotSupported when the forced policy cannot run one of this solve's GN iterations; checked before anything is enqueued
static int check_forced_policy(const BFSolverInput* in, const BFSolverParameters* par, const SolverWs* ws) {
    const int forced = g_gridPolicy.load();
    if (forced == BF_POLICY_AUTO || forced == BF_POLICY_GRID) return 0;
    LaunchLimits lim;
    { const int rc = launch_limits(&lim); if (rc) return rc; }
    const unsigned N = in->numberOfImages;
    const int grid = gn_grid(N, ws, lim);
    bool ok = true;
    if (forced == BF_POLICY_ONE_CTA) ok = one_cta_can_run(grid, ws);
    else
        for (unsigned k = 0; k < par->nNonLinearIterations; ++k) ok = ok && cluster_can_run(N, gn_dense(in, k), grid, ws, lim);
    if (ok) return 0;
    set_last_error(forced == BF_POLICY_ONE_CTA ? "bfSolverSolve: the forced one-CTA policy needs ceil(N / 8) <= 4 and an unsharded solve"
                                               : "bfSolverSolve: the forced cluster policy needs ceil(N / 8) <= the cluster cap, the resident system within "
                                                 "the shared memory limit and an unsharded solve", cudaErrorNotSupported);
    return (int)cudaErrorNotSupported;
}

static int run_gn(const BFSolverInput* in, const BFSolverState* st, const BFSolverParameters* par, SolverWs* ws, unsigned nIter, bool isLast) {
    GnArgs a;
    a.corr = in->d_correspondences; a.N = in->numberOfImages; a.C = in->numberOfCorrespondences; a.validImages = in->d_validImages;
    a.xRot = st->d_xRot; a.xTrans = st->d_xTrans; a.deltaRot = st->d_deltaRot; a.deltaTrans = st->d_deltaTrans;
    a.rRot = st->d_rRot; a.rTrans = st->d_rTrans; a.zRot = st->d_zRot; a.zTrans = st->d_zTrans; a.pRot = st->d_pRot; a.pTrans = st->d_pTrans;
    a.ApRot = st->d_Ap_XRot; a.ApTrans = st->d_Ap_XTrans; a.precRot = st->d_precondionerRot; a.precTrans = st->d_precondionerTrans;
    a.T = st->d_xTransforms; a.Tinv = st->d_xTransformInverses;
    a.rowStart = ws->rowStart; a.entries = ws->entries; a.segCount = ws->segCount; a.segs = ws->segs;
    a.offBlk = ws->offBlk; a.segMom = ws->segMom; a.diagBlk = ws->diagBlk; a.partials = ws->partials; a.scal = ws->scal;
    a.p2Rot = ws->p2; a.p2Trans = ws->p2 + 3 * (size_t)ws->maxImages;
    a.wSparse = in->weightsSparse[nIter]; a.nLin = par->nLinIterations; a.isLastGn = isLast ? 1 : 0; a.maxGrid = ws->maxGrid;
    const float wDepth = in->weightsDenseDepth ? in->weightsDenseDepth[nIter] : 0.0f, wColor = in->weightsDenseColor ? in->weightsDenseColor[nIter] : 0.0f;
    const bool dense = (wDepth > 0.0f || wColor > 0.0f) && in->d_cacheFrames != nullptr;
    a.dnbrStart = nullptr; a.dnbr = nullptr; a.pairOut = nullptr; a.denseDiag = nullptr; a.denseJtr = nullptr; a.useDense = dense ? 1 : 0;
    a.rank = ws->rank; a.world = ws->world; a.seqBase = ws->peerSeq; a.peerMaxN = ws->maxImages;
    for (int g = 0; g < BF_SOLVER_MAX_PEERS; ++g) a.peer[g] = ws->peer[g];
    if (ws->world > 1) ws->peerSeq += par->nLinIterations + 2;          // every rank launches the same sequence: the numbers agree
    if (dense) {
        { const int rc = ensure_dense(ws); if (rc) return rc; }
        a.dnbrStart = ws->dnbrStart; a.dnbr = ws->dnbr; a.pairOut = ws->pairOut; a.denseDiag = ws->denseDiag; a.denseJtr = ws->denseJtr;
        // BuildDenseSystem (SolverBundling.cu:308-471) for this iteration's poses: 1 pose kernel + 3 dense kernels, no host sync
        DenseArgs d;
        d.frames = in->d_cacheFrames; d.valid = in->d_validImages; d.T = st->d_xTransforms; d.Tinv = st->d_xTransformInverses;
        d.N = a.N; d.W = in->denseDepthWidth; d.H = in->denseDepthHeight;
        d.fx = in->intrinsics[0]; d.fy = in->intrinsics[1]; d.mx = in->intrinsics[2]; d.my = in->intrinsics[3];
        d.distThresh = par->denseDistThresh; d.normalThresh = par->denseNormalThresh; d.colorThresh = par->denseColorThresh;
        d.colorGradientMin = par->denseColorGradientMin; d.depthMin = par->denseDepthMin; d.depthMax = par->denseDepthMax;
        d.subsample = par->denseOverlapCheckSubsampleFactor ? par->denseOverlapCheckSubsampleFactor : 1; d.usePairwise = par->useDenseDepthAllPairwise ? 1 : 0;
        d.wDepth = wDepth; d.wColor = wColor;
        d.pairW = ws->pairW; d.pairIdx = ws->pairIdx; d.pairCnt = ws->pairCnt; d.pairRowStart = ws->pairRowStart; d.pairIJ = ws->pairIJ; d.pairOut = ws->pairOut;
        d.dnbrStart = ws->dnbrStart; d.dnbr = ws->dnbr; d.diag = ws->denseDiag; d.Jtr = ws->denseJtr; d.scal = ws->scal;
        dense_begin_kernel<<<(a.N + 127) / 128, 128, 0, stream()>>>(st->d_xRot, st->d_xTrans, a.N, st->d_xTransforms, st->d_xTransformInverses, ws->scal);
        dense_pair_weight_kernel<<<dim3(a.N, a.N), 512, 0, stream()>>>(d);
        dense_pair_count_kernel<<<(a.N + 7) / 8, 256, 0, stream()>>>(d);
        dense_pair_scan_kernel<<<1, 1024, 0, stream()>>>(d);
        dense_pair_fill_kernel<<<(a.N + 7) / 8, 256, 0, stream()>>>(d);
        const unsigned long long maxPairs = (unsigned long long)a.N * (a.N - 1) / 2;
        const unsigned buildGrid = (unsigned)std::min<unsigned long long>(maxPairs, (unsigned long long)num_sms() * 8);
        dense_build_kernel<<<buildGrid ? buildGrid : 1, 128, 0, stream()>>>(d);
        dense_assemble_kernel<<<a.N, 64, 0, stream()>>>(d);
        BF_CHECK(cudaGetLastError());
        g_launchCount += 7;
    }
    void* args[] = { (void*)&a };
    ++g_launchCount;
    LaunchLimits lim;
    { const int rc = launch_limits(&lim); if (rc) return rc; }
    const int grid = gn_grid(a.N, ws, lim);
    const int policy = pick_policy(a.N, dense, grid, ws, lim);
    ws->launchInfo[0] = policy; ws->launchInfo[1] = grid; ws->launchInfo[2] = lim.clusterCap; ws->launchInfo[3] = lim.maxDynSmem;
    if (policy == BF_POLICY_ONE_CTA) {
        gn_iteration_kernel<OneCtaGrid><<<1, grid * BF_SOLVER_THREADS, 0, stream()>>>(a);
        BF_CHECK(cudaGetLastError());
        return 0;
    }
    if (policy == BF_POLICY_CLUSTER) {
        const size_t smem = sizeof(float) * resident_smem_words(a.N, dense);
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(grid); cfg.blockDim = dim3(BF_SOLVER_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = stream();
        cudaLaunchAttribute at; at.id = cudaLaunchAttributeClusterDimension; at.val.clusterDim.x = grid; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
        cfg.attrs = &at; cfg.numAttrs = 1;
        BF_CHECK(cudaLaunchKernelEx(&cfg, gn_iteration_kernel<ResidentCluster>, a));
        return 0;
    }
    BF_CHECK(cudaLaunchCooperativeKernel((void*)gn_iteration_kernel<CoopGrid>, dim3(grid), dim3(BF_SOLVER_THREADS), args, 0, stream()));
    return 0;
}

static int solve_impl(const BFSolverInput* in, const BFSolverState* st, const BFSolverParameters* par, bool rebuild) {
    if (in->numberOfImages < 2 || par->nNonLinearIterations == 0) return 0;
    for (unsigned k = 0; k < par->nNonLinearIterations; ++k)
        if (((in->weightsDenseDepth && in->weightsDenseDepth[k] > 0.0f) || (in->weightsDenseColor && in->weightsDenseColor[k] > 0.0f)) &&
            in->d_cacheFrames != nullptr && in->numberOfImages > BF_DENSE_MAX_IMAGES) {
            set_last_error("bfSolverSolve: the dense depth/colour term keeps N^2 pair tables: <= 4096 images", cudaErrorNotSupported);
            return (int)cudaErrorNotSupported;
        }
    if (in->maxCorrPerImage == 0 || in->maxCorrPerImage > BF_MAX_ROW) {      // CUDASolverBundling.cpp:39 clamps it to [1000, 4000]
        set_last_error("bfSolverSolve: maxCorrPerImage must be in [1, 8192]", cudaErrorInvalidValue);
        return (int)cudaErrorInvalidValue;
    }
    SolverWs* ws;
    unsigned cap = 1024;                                  // grow geometrically so a growing problem rarely reallocates
    while (cap < in->numberOfCorrespondences) cap <<= 1;
    int rc = get_ws(st, in->maxNumberOfImages > in->numberOfImages ? in->maxNumberOfImages : in->numberOfImages, cap, &ws);
    if (rc) return rc;
    rc = check_forced_policy(in, par, ws);
    if (rc) return rc;
    if (rebuild) { rc = run_prep(in, st, ws); if (rc) return rc; }
    else BF_CHECK(cudaMemsetAsync(ws->scal, 0, sizeof(unsigned) * 3, stream()));   // done / counters
    for (unsigned k = 0; k < par->nNonLinearIterations; ++k) {
        rc = run_gn(in, st, par, ws, k, k == par->nNonLinearIterations - 1);
        if (rc) return rc;
    }
    return 0;
}

}  // namespace bf

using namespace bf;

// ======================================================================================================================
BF_API int bfSolverSolve(const BFSolverInput* in, const BFSolverState* st, const BFSolverParameters* par) { return solve_impl(in, st, par, true); }

BF_API int bfSolverGetStats(const BFSolverState* st, unsigned long long out[8]) {
    SolverWs* ws = nullptr;
    { std::lock_guard<std::mutex> lk(g_wsMutex); auto it = g_ws.find(st->d_deltaRot); if (it != g_ws.end()) ws = &it->second; }
    if (!ws) return (int)cudaErrorInvalidValue;
    unsigned s[SC_NUM];
    BF_CHECK(cudaMemcpyAsync(s, ws->scal, sizeof(s), cudaMemcpyDeviceToHost, stream()));
    BF_CHECK(cudaStreamSynchronize(stream()));
    float md; memcpy(&md, &s[SC_MAXDELTA_BITS], 4);
    out[0] = s[SC_GN_RUN]; out[1] = s[SC_PCG_RUN]; out[2] = s[SC_NUM_SEG] / 2; out[3] = s[SC_DENSE_OVERLAP];
    out[4] = (unsigned long long)(md * 1e6f); out[5] = s[SC_ERROR]; out[6] = s[SC_DONE]; out[7] = s[SC_DENSE_PAIRS];
    return 0;
}

BF_API int bfSolverSetGridPolicy(int policy) {
    if (policy < BF_POLICY_AUTO || policy > BF_POLICY_CLUSTER) return (int)cudaErrorInvalidValue;
    return g_gridPolicy.exchange(policy);
}

BF_API int bfSolverGetLaunchInfo(const BFSolverState* st, int out[4]) {
    if (!st || !out) return (int)cudaErrorInvalidValue;
    std::lock_guard<std::mutex> lk(g_wsMutex);
    auto it = g_ws.find(st->d_deltaRot);
    if (it == g_ws.end()) return (int)cudaErrorInvalidValue;
    memcpy(out, it->second.launchInfo, sizeof(it->second.launchInfo));
    return 0;
}

BF_API int bfSolverMaxResidual(const BFSolverInput* in, const BFSolverState* st, const BFSolverParameters* par, float* d_out2) {
    const unsigned C = in->numberOfCorrespondences;
    SolverWs* ws;
    int rc = get_ws(st, in->maxNumberOfImages, C, &ws);
    if (rc) return rc;
    if (C == 0) { BF_CHECK(cudaMemsetAsync(d_out2, 0, 8, stream())); return 0; }
    const unsigned nb = (C + 511) / 512;
    // block maxima go to the (large enough) segment-moment scratch
    float* bm = ws->segMom; int* bi = reinterpret_cast<int*>(ws->segMom) + nb;
    eval_max_residual_kernel<<<nb, 512, 0, stream()>>>(in->d_correspondences, C, st->d_xRot, st->d_xTrans, par->weightSparse, bm, bi);
    reduce_max_kernel<<<1, 1024, 0, stream()>>>(bm, bi, nb, d_out2);
    BF_CHECK(cudaGetLastError());
    return 0;
}

BF_API int bfSolverReserveWorkspace(const BFSolverState* st, unsigned int maxImages, unsigned int maxRes, int withDenseTerm) {
    if (!st || maxImages < 1) return (int)cudaErrorInvalidValue;
    SolverWs* ws;
    unsigned cap = 1024;                                  // the capacity bfSolverSolve would ask for at maxRes correspondences
    while (cap < maxRes) cap <<= 1;
    const int rc = get_ws(st, maxImages, cap, &ws);
    if (rc) return rc;
    return withDenseTerm ? ensure_dense(ws) : 0;
}

BF_API size_t bfSolverWorkspaceBytes(unsigned int maxImages, unsigned int maxRes) {
    const size_t E = 2 * (size_t)maxRes;
    return sizeof(int) * (3 * (size_t)maxImages + 1 + 2 * E + maxImages) + sizeof(Segment) * E + sizeof(float) * (36 + 20) * E + sizeof(float) * 36 * maxImages;
}
BF_API int bfSolverReleaseWorkspace(const BFSolverState* st) {
    std::lock_guard<std::mutex> lk(g_wsMutex);
    auto it = g_ws.find(st->d_deltaRot);
    if (it == g_ws.end()) return 0;
    free_ws(it->second);
    g_ws.erase(it);
    return 0;
}

// ---- sharded solve over the GPUs of one box ---------------------------------------------------------------------------------------------------------
BF_API int bfSolverPeerCreate(const BFSolverState* st, unsigned int maxImages, unsigned int maxCorr, void* ipcHandleOut64) {
    SolverWs* ws;
    unsigned cap = 1024;
    while (cap < maxCorr) cap <<= 1;
    int rc = get_ws(st, maxImages, cap, &ws);
    if (rc) return rc;
    if (!ws->region) {
        const size_t bytes = sizeof(float) * peer_region_floats(ws->maxImages, ws->maxGrid);
        BF_CHECK(cudaMalloc(&ws->region, bytes));
        BF_CHECK(cudaMemset(ws->region, 0, bytes));
    }
    cudaIpcMemHandle_t h;
    BF_CHECK(cudaIpcGetMemHandle(&h, ws->region));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    memcpy(ipcHandleOut64, &h, 64);
    return 0;
}
BF_API int bfSolverPeerConnect(const BFSolverState* st, int rank, int world, const void* ipcHandles) {
    SolverWs* ws = nullptr;
    { std::lock_guard<std::mutex> lk(g_wsMutex); auto it = g_ws.find(st->d_deltaRot); if (it != g_ws.end()) ws = &it->second; }
    if (!ws || !ws->region || world < 1 || world > BF_SOLVER_MAX_PEERS || rank < 0 || rank >= world) return (int)cudaErrorInvalidValue;
    for (int g = 0; g < world; ++g) {
        if (g == rank) { ws->peer[g] = ws->region; continue; }
        cudaIpcMemHandle_t h; memcpy(&h, static_cast<const char*>(ipcHandles) + 64 * (size_t)g, 64);
        void* p = nullptr;
        BF_CHECK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
        ws->peer[g] = static_cast<float*>(p); ws->peerOpened[g] = true;
    }
    ws->rank = rank; ws->world = world; ws->peerSeq = 0;
    return 0;
}
BF_API int bfSolverPeerDisconnect(const BFSolverState* st) {
    SolverWs* ws = nullptr;
    { std::lock_guard<std::mutex> lk(g_wsMutex); auto it = g_ws.find(st->d_deltaRot); if (it != g_ws.end()) ws = &it->second; }
    if (!ws) return 0;
    BF_CHECK(cudaStreamSynchronize(stream()));
    for (int g = 0; g < BF_SOLVER_MAX_PEERS; ++g) { if (ws->peerOpened[g]) { cudaIpcCloseMemHandle(ws->peer[g]); ws->peerOpened[g] = false; } ws->peer[g] = nullptr; }
    ws->rank = 0; ws->world = 1;
    return 0;
}

// Test / diagnosis accessor: the dense normal equations of the LAST Gauss-Newton iteration that built them, in the reference's
// layout (FL/Solver/SolverBundling.cu:308-471: (6N)^2 row-major, translation first per image; J^T r [6N]) -- what the
// reference keeps in SolverState::d_denseJtJ / d_denseJtr.  Device-to-device copies on the library stream.
BF_API int bfSolverDebugDenseSystem(const BFSolverState* st, unsigned int numImages, float* d_JtJ, float* d_Jtr) {
    SolverWs* ws = nullptr;
    { std::lock_guard<std::mutex> lk(g_wsMutex); auto it = g_ws.find(st->d_deltaRot); if (it != g_ws.end()) ws = &it->second; }
    if (!ws || !ws->denseCap || numImages > ws->denseCap) return (int)cudaErrorInvalidValue;
    const size_t dim = 6 * (size_t)numImages;
    if (d_JtJ) {
        BF_CHECK(cudaMemsetAsync(d_JtJ, 0, sizeof(float) * dim * dim, stream()));
        dense_scatter_kernel<<<numImages, 64, 0, stream()>>>(numImages, ws->dnbrStart, ws->dnbr, ws->pairOut, ws->denseDiag, d_JtJ);
        BF_CHECK(cudaGetLastError());
    }
    if (d_Jtr) BF_CHECK(cudaMemcpyAsync(d_Jtr, ws->denseJtr, sizeof(float) * dim, cudaMemcpyDeviceToDevice, stream()));
    return 0;
}

// ---- reference-named stubs ---------------------------------------------------------------------------------------------
BF_API void solveBundlingStub(BFSolverInput* in, BFSolverState* st, BFSolverParameters* par, BFSolverStateAnalysis* analysis, float* conv, void* timer) {
    (void)analysis; (void)timer;
    auto energy = [&](float w) -> float {
        float e = 0.0f;
        if (in->numberOfCorrespondences == 0) return 0.0f;
        BF_SAFE((int)cudaMemsetAsync(st->d_sumResidual, 0, sizeof(float), stream()));
        energy_kernel<<<(in->numberOfCorrespondences + 255) / 256, 256, 0, stream()>>>(in->d_correspondences, in->numberOfCorrespondences, st->d_xRot, st->d_xTrans, w, st->d_sumResidual);
        BF_SAFE((int)cudaMemcpyAsync(&e, st->d_sumResidual, sizeof(float), cudaMemcpyDeviceToHost, stream()));
        BF_SAFE((int)cudaStreamSynchronize(stream()));
        return e;
    };
    if (!conv) { BF_SAFE(solve_impl(in, st, par, true)); return; }
    // convergence recording (s_recordSolverConvergence): one GN iteration at a time with an energy read-back
    conv[0] = energy(par->weightSparse);
    BFSolverParameters one = *par; one.nNonLinearIterations = 1;
    for (unsigned k = 0; k < par->nNonLinearIterations; ++k) {
        BFSolverInput ik = *in; ik.weightsSparse = in->weightsSparse + k; ik.weightsDenseDepth = in->weightsDenseDepth + k; ik.weightsDenseColor = in->weightsDenseColor + k;
        BF_SAFE(solve_impl(&ik, st, &one, k == 0));
        conv[k + 1] = energy(in->weightsSparse[k]);
    }
}

BF_API void buildVariablesToCorrespondencesTableCUDA(BFEntryJ* d_corr, unsigned int C, unsigned int maxPerImage, int* d_table, int* d_rows, void* timer) {
    (void)timer;
    // The caller has zeroed d_rows (CUDASolverBundling.cpp:288).  The image count is not part of this signature, so this
    // entry fills the table the way the reference does (arrival order); solveBundlingStub / bfSolverSolve rebuild rows
    // and table in ascending-index order before they solve.
    if (C) table_arrival_kernel<<<(C + 255) / 256, 256, 0, stream()>>>(d_corr, C, maxPerImage, d_table, d_rows);
    BF_SAFE((int)cudaGetLastError());
}

BF_API void evalMaxResidual(BFSolverInput* in, BFSolverState* st, BFSolverStateAnalysis* an, BFSolverParameters* par, void* timer) {
    (void)timer;
    const unsigned C = in->numberOfCorrespondences;
    if (C == 0) return;
    eval_max_residual_kernel<<<(C + 511) / 512, 512, 0, stream()>>>(in->d_correspondences, C, st->d_xRot, st->d_xTrans, par->weightSparse, an->d_maxResidual, an->d_maxResidualIndex);
    BF_SAFE((int)cudaGetLastError());
}
BF_API int countHighResiduals(BFSolverInput* in, BFSolverState* st, BFSolverParameters* par, void* timer) {
    (void)timer;
    const unsigned C = in->numberOfCorrespondences;
    int count = 0;
    BF_SAFE((int)cudaMemsetAsync(st->d_countHighResidual, 0, sizeof(int), stream()));
    if (C) count_high_residuals_kernel<<<(C + 511) / 512, 512, 0, stream()>>>(in->d_correspondences, C, st->d_xRot, st->d_xTrans, par->weightSparse, par->verifyOptDistThresh, st->d_countHighResidual);
    BF_SAFE((int)cudaMemcpyAsync(&count, st->d_countHighResidual, sizeof(int), cudaMemcpyDeviceToHost, stream()));
    BF_SAFE((int)cudaStreamSynchronize(stream()));
    return count;
}
BF_API void collectHighResiduals(BFSolverInput* in, BFSolverState* st, BFSolverStateAnalysis* an, BFSolverParameters* par, void* timer) {
    (void)timer;
    const unsigned C = in->numberOfCorrespondences;
    BF_SAFE((int)cudaMemsetAsync(st->d_countHighResidual, 0, sizeof(int), stream()));
    const unsigned maxOut = (in->maxCorrPerImage * in->maxNumberOfImages + 511) / 512;
    if (C) collect_high_residuals_kernel<<<(C + 511) / 512, 512, 0, stream()>>>(in->d_correspondences, C, st->d_xRot, st->d_xTrans, par->weightSparse, par->highResidualThresh,
                                                                               st->d_countHighResidual, an->d_maxResidual, an->d_maxResidualIndex, maxOut);
    BF_SAFE((int)cudaGetLastError());
}
BF_API void convertLiePosesToMatricesCU(const float* d_rot, const float* d_trans, unsigned int n, float* d_T, float* d_Tinv) {
    if (n) poses_to_matrices_kernel<<<(n + 127) / 128, 128, 0, stream()>>>(d_rot, d_trans, n, d_T, d_Tinv, nullptr);
    BF_SAFE((int)cudaGetLastError());
}
BF_API void convertMatricesToPosesCU(const float* d_T, unsigned int n, float* d_rot, float* d_trans, const int* d_valid) {
    if (n) matrices_to_poses_kernel<<<(n + 127) / 128, 128, 0, stream()>>>(d_T, n, d_rot, d_trans, d_valid);
    BF_SAFE((int)cudaGetLastError());
}
BF_API void convertPosesToMatricesCU(const float* d_rot, const float* d_trans, unsigned int n, float* d_T, const int* d_valid) {
    if (n) poses_to_matrices_kernel<<<(n + 127) / 128, 128, 0, stream()>>>(d_rot, d_trans, n, d_T, nullptr, d_valid);
    BF_SAFE((int)cudaGetLastError());
}

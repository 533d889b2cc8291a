// tsdf_fast.cu -- the integrate / de-integrate / fused re-integration stencil in TOLERANCE arithmetic (the library default).
//
// Behavioural source: integrateDepthMapKernel<deIntegrate>, FL/DepthSensing/CUDASceneRepHashSDF.cu:420-521 (per-voxel rule),
// DepthCameraUtil.h:71-82 (projection), the re-integration loop of FL/DepthSensing/DepthSensing.cpp:854-902.
//
// Why a second stencil.  tsdf.cu reproduces the reference's IEEE build bit for bit (individually rounded operations, two IEEE
// divides per voxel probe, the full 4x4 product per voxel): ~130 thread-instructions per probe, issue-bound far below the HBM
// roof on the re-integration stream.  The reference itself ships --use_fast_math
// and BASELINE's north star asks for "weights/sdf within a stated fp32 tolerance", so the product path is this one:
//   * the voxel -> camera transform is affine in the integer voxel coordinate: one FMA chain per (thread, block) and three adds
//     per further x-consecutive voxel instead of a 4x4 product per voxel;
//   * one approximate reciprocal (MUFU.RCP) of z per probe instead of two IEEE divides;
//   * the truncation clamp is dropped (|sdf| < trunc makes it the identity), the colour blend 0.2 c + 0.8 o is evaluated in
//     exact integer arithmetic (its fraction is a multiple of 0.2, never a rounding tie: identical to the float expression),
//     byte <-> float moves use PRMT / magic-number adds, no conversion instructions;
//   * a fused re-integration shares everything but the two poses' projections; each voxel is read and written once.
// Contract (tests/test_tsdf_fast_gpu.py): allocated block set identical (alloc / compactify stay in tsdf.cu), weights identical,
// |d sdf| <= 1e-5 m, colour +-1, except for a <= 1e-4 fraction of voxels whose projected pixel or truncation test sits within
// rounding distance of its decision boundary -- the same kind and size of difference the reference's own --use_fast_math build
// shows against its IEEE build (tests/test_tsdf_vs_reference_gpu.py).  bfTsdfSetArithmetic(BF_TSDF_ARITH_EXACT)
// selects tsdf.cu's kernels.
#include "bf_common.cuh"
#include "tsdf_shared.cuh"

namespace bf {

struct FastPose {
    // camera-space z of a voxel = cz[0] vx + cz[1] vy + cz[2] vz + cz[3] (row of Tinv * diag(voxelSize)); cx / cy: the rows for x / y times the focal
    // length, so that the pixel coordinate is (cx . v) / z + mx -- one multiply-add after the reciprocal
    float cx[4], cy[4], cz[4];
    float maxDist, trunc0, truncScale, wMax;
};
struct FastCam { unsigned W, H; float fx, fy, mx5, my5; };     // mx + 0.5, my + 0.5: the reference's int(proj + 0.5)
struct FastArgs {
    BFVoxel* blocks; const BFHashEntry* list; int* listCounterOut; const int4* work;
    const float* depth; const uchar4* color; unsigned* ctrs; int* live;
    int set; int useListCount; unsigned countOverride;
    FastCam cam;
    FastPose A, B;                   // MODE 0 / 1: A.  MODE 2: A = old pose (de-integrated), B = new pose (integrated)
};
struct MultiOp { FastPose A, B; const float* depth; const unsigned* color; };
struct MultiArgs {
    BFVoxel* blocks; const int4* workA; const int4* workB; const unsigned* maskA; const unsigned* maskB; unsigned* ctrs; int* live; int* listCounterOut;
    int set; int nOps; unsigned workCap;
    unsigned long long* ktime;       // optional {min CTA start, max CTA end} in %globaltimer ns (measurement only)
    FastCam cam;
    MultiOp ops[BF_MULTI_MAX_OPS];
};

// resident CTAs per SM the kernels are compiled for: the fused pass keeps two poses' probe sets live (<= 64 registers), the others 48
#define BF_FAST_MINBLOCKS 10
#define BF_FAST_MINBLOCKS_FUSED 8

#ifdef BF_EMU_SEQUENTIAL      // tests/test_tsdf_fast_emulated.py: this source executed on the CPU, one CUDA thread after the other
__device__ __forceinline__ float rcp_approx(float x) { return 1.0f / x; }
#else
__device__ __forceinline__ float rcp_approx(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
#endif
// byte k of w as a float, exactly: bits 0x4B0000bb = 2^23 + b
template <int K> __device__ __forceinline__ float byte_to_float(unsigned w) {
    return __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7440u | K)) - 8388608.0f;
}
template <int K> __device__ __forceinline__ unsigned put_byte(unsigned acc, unsigned v) {
    return __byte_perm(acc, v, K == 0 ? 0x3214u : (K == 1 ? 0x3240u : 0x3410u));
}

// ---- probe phase, branch-free: projections and the depth gathers of all four voxels of a thread are independent of each other, so
// the compiler can issue the loads back to back (memory-level parallelism) and interleave the arithmetic of the four chains ----
struct ProbeSet {
    float sdf[4];          // after decide(): depth - z of the voxels that pass
    unsigned idx[4];       // pixel index (0 when the voxel projects outside the image; such a voxel never passes)
    unsigned mask;         // bit k: voxel k passes the truncation test
};
// the image pointer in an ordinary (non-uniform) register pair: the gather's address is then one IMAD.WIDE (base + 4 idx) instead of a LEA / LEA.HI.X
// pair off a uniform base
__device__ __forceinline__ const float* in_vector_regs(const float* p) {
#ifndef BF_EMU_SEQUENTIAL
    asm("" : "+l"(p));
#endif
    return p;
}
// (vx, vy, vz): integer voxel coordinates of the thread's first voxel, as floats.  Every fast kernel evaluates the SAME expression here, so a
// voxel's pass / fail decision for a given (pose, frame) is the same bit for bit whichever kernel asks (integrate now, de-integrate later in a batch)
__device__ __forceinline__ void project4(const FastCam& a, const float* __restrict__ depthU, const FastPose& p, float vx, float vy, float vz, ProbeSet& ps, float (&z)[4]) {
    const float* const depth = in_vector_regs(depthU);
    const float X = fmaf(vx, p.cx[0], fmaf(vy, p.cx[1], fmaf(vz, p.cx[2], p.cx[3])));
    const float Y = fmaf(vx, p.cy[0], fmaf(vy, p.cy[1], fmaf(vz, p.cy[2], p.cy[3])));
    const float Z = fmaf(vx, p.cz[0], fmaf(vy, p.cz[1], fmaf(vz, p.cz[2], p.cz[3])));
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float Xk = k ? fmaf((float)k, p.cx[0], X) : X, Yk = k ? fmaf((float)k, p.cy[0], Y) : Y, Zk = k ? fmaf((float)k, p.cz[0], Z) : Z;
        const float rz = rcp_approx(Zk);
        const float sx = fmaf(Xk, rz, a.mx5), sy = fmaf(Yk, rz, a.my5);
        const unsigned ix = (unsigned)__float2int_rz(sx), iy = (unsigned)__float2int_rz(sy);   // cvt.rzi: (-1, 0) -> 0, NaN -> 0, as the reference's (int)
        const bool on = (ix < a.W) & (iy < a.H);
        const unsigned idx = on ? iy * a.W + ix : 0u;
        ps.idx[k] = idx;
        z[k] = Zk;
        const float d = __ldg(&depth[idx]);                              // unconditional load from a safe address
        ps.sdf[k] = on ? d : -INFINITY;                                  // holds the DEPTH until decide(); off screen = no depth
    }
}
// truncation test (.cu:433-463 without the identity clamp): depth valid, below the integration distance, |depth - z| < truncation(depth).
// An invalid depth (-inf) fails the band test by itself: |sdf| = inf is not below trunc0 + truncScale * (-inf) = -inf (or trunc0 when the scale is 0).
__device__ __forceinline__ void decide4(const FastPose& p, ProbeSet& ps, const float (&z)[4]) {
    ps.mask = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float d = ps.sdf[k];
        const float sdf = d - z[k];
        const bool pass = (d < p.maxDist) & (fabsf(sdf) < fmaf(p.truncScale, d, p.trunc0));
        ps.sdf[k] = sdf;
        ps.mask |= pass ? (1u << k) : 0u;
    }
}

// integrate one sample into (sdf, weight, colour) words; .cu:486-500
__device__ __forceinline__ void integrate_fast(const FastPose& p, float sdf, unsigned col, unsigned& wSdf, unsigned& wWeight, unsigned& wColor) {
    const float oldSdf = __uint_as_float(wSdf), oldW = __uint_as_float(wWeight);
    const float den = oldW + 1.0f;
    const float nSdf = fmaf(oldSdf, oldW, sdf) * rcp_approx(den);
    unsigned nc = 0xFF000000u;
    // oldW == 0: colour = the sample (through clamp [0, 254.5] and the byte conversion: 255 -> 254); else
    // round(0.2 c + 0.8 o) = floor((2 c + 8 o + 5) / 10): the fraction of (c + 4 o) / 5 is a multiple of 0.2, never a tie
    const bool first = (oldW == 0.0f);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const unsigned c = (col >> (8 * k)) & 0xffu, o = (wColor >> (8 * k)) & 0xffu;
        const unsigned q = first ? c : __umulhi(8u * o + 2u * c + 5u, 429496730u);
        const unsigned v = min(q, 254u);
        nc = (k == 0) ? put_byte<0>(nc, v) : (k == 1 ? put_byte<1>(nc, v) : put_byte<2>(nc, v));
    }
    wSdf = __float_as_uint(nSdf); wWeight = __float_as_uint(fminf(p.wMax, den)); wColor = nc;
}

// de-integrate one sample; .cu:501-514
__device__ __forceinline__ void deintegrate_fast(float sdf, unsigned col, unsigned& wSdf, unsigned& wWeight, unsigned& wColor) {
    const float oldSdf = __uint_as_float(wSdf), oldW = __uint_as_float(wWeight);
    const float den = oldW - 1.0f;
    if (!(den > 0.001f)) { wSdf = 0u; wWeight = 0u; wColor = 0u; return; }           // weight max(0, w - 1) <= 0.001: the voxel is cleared
    const float r = rcp_approx(den);
    const float nSdf = fmaf(oldSdf, oldW, -sdf) * r;
    // round((o w - c) / (w - 1)), half away from zero, clamped to [0, 254.5] -> byte.  The quotient is biased up by 2^-20 so that the
    // exact ties (w - 1 = 2, 4, ...) fall on the reference's side under an approximate reciprocal; then round-to-nearest via 2^23.
    const float rb = r * 1.00000095367431640625f;
    unsigned nc = 0xFF000000u;
    {
        const float q = fminf(fmaxf(fmaf(byte_to_float<0>(wColor), oldW, -byte_to_float<0>(col)) * rb, 0.0f), 254.4f);
        nc = put_byte<0>(nc, __float_as_uint(q + 8388608.0f));
    }
    {
        const float q = fminf(fmaxf(fmaf(byte_to_float<1>(wColor), oldW, -byte_to_float<1>(col)) * rb, 0.0f), 254.4f);
        nc = put_byte<1>(nc, __float_as_uint(q + 8388608.0f));
    }
    {
        const float q = fminf(fmaxf(fmaf(byte_to_float<2>(wColor), oldW, -byte_to_float<2>(col)) * rb, 0.0f), 254.4f);
        nc = put_byte<2>(nc, __float_as_uint(q + 8388608.0f));
    }
    wSdf = __float_as_uint(nSdf); wWeight = __float_as_uint(den); wColor = nc;
}

// The three cases of a re-integration pair on one voxel -- only the old pose passes (de-integrate), only the new one (integrate), both (composed) --
// as ONE branch-free expression, a = passA, b = passB as 0 / 1:  sdf = (s w - a sD + b sI) / (w - a + b), weight = w - a, + 1 clamped to wMax if b,
// colour de-integrated if a (kept as a whole level in a float), then blended if b.  A warp whose lanes disagree on the case (voxels at the edge of
// either pose's truncation band: about every second warp) executes this once instead of up to three divergent bodies.  Each case evaluates to the
// same value as integrate_fast / deintegrate_fast (and, for both, their composition with one reciprocal: ((s w - sD) / (w - 1) (w - 1) + sI) / w) up to the rounding of the shared sdf numerator (< 2e-7 m).
__device__ __forceinline__ void update_pair(const FastPose& pB, bool passA, float sdfD, unsigned colD, bool passB, float sdfI, unsigned colI,
                                            unsigned& wSdf, unsigned& wWeight, unsigned& wColor, int& liveDelta) {
    const float oldSdf = __uint_as_float(wSdf), oldW = __uint_as_float(wWeight);
    const bool wasLive = oldW > 0.0f;
    const float wd0 = passA ? oldW - 1.0f : oldW;
    const bool cleared = passA & !(wd0 > 0.001f);                       // the de-integration empties the voxel (.cu:505-513)
    const float wd = cleared ? 0.0f : wd0;
    const float num = cleared ? (passB ? sdfI : 0.0f) : fmaf(oldSdf, oldW, (passB ? sdfI : 0.0f) - (passA ? sdfD : 0.0f));
    const float den = passB ? wd + 1.0f : wd;
    const float nSdf = (den > 0.0f) ? num * rcp_approx(den) : 0.0f;
    const float nW = passB ? fminf(pB.wMax, den) : wd;
    const float rb = rcp_approx(wd0) * 1.00000095367431640625f;          // see deintegrate_fast; unused (selected away) when !passA or cleared
    const bool first = (wd == 0.0f);
    unsigned nc = 0xFF000000u;
#define BF_PAIR_CHANNEL(K)                                                                                                                    \
    {                                                                                                                                         \
        const float c0 = byte_to_float<K>(wColor);                                                                                            \
        const float qd = fminf(fmaxf(fmaf(c0, oldW, -byte_to_float<K>(colD)) * rb, 0.0f), 254.4f);                                            \
        const float c1 = passA ? (cleared ? 0.0f : (qd + 8388608.0f) - 8388608.0f) : c0;      /* whole level <= 254 */                        \
        const float ci = byte_to_float<K>(colI);                                                                                              \
        const float q = first ? fminf(ci, 254.0f) : fmaf(0.2f, ci, 0.8f * c1);                 /* fraction a multiple of 0.2: never a tie */    \
        nc = put_byte<K>(nc, __float_as_uint((passB ? q : c1) + 8388608.0f));                                                                \
    }
    BF_PAIR_CHANNEL(0) BF_PAIR_CHANNEL(1) BF_PAIR_CHANNEL(2)
#undef BF_PAIR_CHANNEL
    const bool zero = cleared & !passB;                                  // cleared voxels are all-zero words (.cu:509-512)
    wSdf = zero ? 0u : __float_as_uint(nSdf); wWeight = zero ? 0u : __float_as_uint(nW); wColor = zero ? 0u : nc;
    liveDelta += (int)(nW > 0.0f) - (int)wasLive;
}

template <int MODE>
__device__ __forceinline__ void update_fast(const FastPose& pA, const FastPose& pB, bool passA, float sdfA, unsigned colA, bool passB, float sdfB, unsigned colB,
                                            unsigned& wSdf, unsigned& wWeight, unsigned& wColor, int& liveDelta) {
    if (MODE == 2) { update_pair(pB, passA, sdfA, colA, passB, sdfB, colB, wSdf, wWeight, wColor, liveDelta); return; }
    const bool wasLive = __uint_as_float(wWeight) > 0.0f;
    if (MODE == 0) integrate_fast(pA, sdfA, colA, wSdf, wWeight, wColor);
    else deintegrate_fast(sdfA, colA, wSdf, wWeight, wColor);
    liveDelta += (int)(__uint_as_float(wWeight) > 0.0f) - (int)wasLive;
}

struct ThreadVoxel { int lx, ly, lz; };          // this thread's first voxel inside a block: i = 4t -> x = (4t) % 8, y = (4t % 64) / 8, z = 4t / 64

__device__ __forceinline__ void live_delta_commit(int* live, unsigned slot, unsigned t, int liveDelta) {
    // live-voxel bookkeeping for the O(E) garbage collection: one RED per warp, only when a weight crossed zero
#ifdef BF_EMU_SEQUENTIAL
    if (liveDelta != 0) atomicAdd(&live[slot], liveDelta);
#else
    if (__any_sync(0xffffffffu, liveDelta != 0)) {
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) liveDelta += __shfl_xor_sync(0xffffffffu, liveDelta, s);
        if ((t & 31) == 0 && liveDelta != 0) atomicAdd(&live[slot], liveDelta);
    }
#endif
}

// one SDF block: 128 threads, 4 x-consecutive voxels (48 B = three 16-byte vectors) per thread
template <int MODE>
__device__ __forceinline__ void process_block(const FastArgs& a, const ThreadVoxel& o, unsigned t, int bx, int by, int bz, unsigned ptr, unsigned fl, unsigned& passed) {
    const float vx = (float)(bx * BF_SDF_BLOCK_SIZE + o.lx), vy = (float)(by * BF_SDF_BLOCK_SIZE + o.ly), vz = (float)(bz * BF_SDF_BLOCK_SIZE + o.lz);
    ProbeSet pA, pB;
    float zA[4], zB[4];
    pA.mask = 0; pB.mask = 0;
    if (a.color == nullptr) return;                        // without colour nothing passes (.cu:441-448)
    if (fl & 1u) project4(a.cam, a.depth, a.A, vx, vy, vz, pA, zA);
    if (MODE == 2 && (fl & 2u)) project4(a.cam, a.depth, a.B, vx, vy, vz, pB, zB);
    if (fl & 1u) decide4(a.A, pA, zA);
    if (MODE == 2 && (fl & 2u)) decide4(a.B, pB, zB);
    const unsigned mask = pA.mask | pB.mask;
    int liveDelta = 0;
    if (mask) {
        // colour gathers of the passing voxels (safe address otherwise) and the voxel quad: one batch of independent loads
        const unsigned* colImg = reinterpret_cast<const unsigned*>(a.color);
        unsigned cA[4], cB[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            cA[k] = __ldg(&colImg[(pA.mask >> k) & 1u ? pA.idx[k] : 0u]);
            if (MODE == 2) cB[k] = __ldg(&colImg[(pB.mask >> k) & 1u ? pB.idx[k] : 0u]);
        }
        uint4* const vp = reinterpret_cast<uint4*>(a.blocks + (size_t)ptr) + 3 * t;      // 48 B per thread, 16-B aligned
        uint4 qa = vp[0], qb = vp[1], qc = vp[2];
        // 4 voxels = 12 words: v0{a.x,a.y,a.z} v1{a.w,b.x,b.y} v2{b.z,b.w,c.x} v3{c.y,c.z,c.w}
        if (mask & 1u) update_fast<MODE>(a.A, a.B, pA.mask & 1u, pA.sdf[0], cA[0], pB.mask & 1u, pB.sdf[0], cB[0], qa.x, qa.y, qa.z, liveDelta);
        if (mask & 2u) update_fast<MODE>(a.A, a.B, pA.mask & 2u, pA.sdf[1], cA[1], pB.mask & 2u, pB.sdf[1], cB[1], qa.w, qb.x, qb.y, liveDelta);
        if (mask & 4u) update_fast<MODE>(a.A, a.B, pA.mask & 4u, pA.sdf[2], cA[2], pB.mask & 4u, pB.sdf[2], cB[2], qb.z, qb.w, qc.x, liveDelta);
        if (mask & 8u) update_fast<MODE>(a.A, a.B, pA.mask & 8u, pA.sdf[3], cA[3], pB.mask & 8u, pB.sdf[3], cB[3], qc.y, qc.z, qc.w, liveDelta);
        if (mask & 0x3u) vp[0] = qa;                      // only the 16-byte pieces that hold an updated voxel
        if (mask & 0x6u) vp[1] = qb;
        if (mask & 0xCu) vp[2] = qc;
        passed += __popc(pA.mask) + __popc(pB.mask);
    }
    live_delta_commit(a.live, ptr / BF_SDF_BLOCK_VOXELS, t, liveDelta);
}

// one SDF block of a batch: the ops whose mask bits are set are applied in order to the voxel quad held in registers.  kOldPose = false: a batch of
// integrations only (bfTsdfIntegrateBatch) -- no op has an old pose, its mask bit 0 is never set, and each passing voxel takes integrate_fast, the
// very update the one-frame stencil (MODE 0) applies, so the batch is bit-identical to the frames integrated one by one
template <bool kOldPose>
__device__ __forceinline__ void process_block_multi(const MultiArgs& a, const ThreadVoxel& o, unsigned t, int4 w, unsigned opMask, unsigned& passed) {
    const float vx = (float)(w.x * BF_SDF_BLOCK_SIZE + o.lx), vy = (float)(w.y * BF_SDF_BLOCK_SIZE + o.ly), vz = (float)(w.z * BF_SDF_BLOCK_SIZE + o.lz);
    uint4* const vp = reinterpret_cast<uint4*>(a.blocks + (size_t)(unsigned)w.w * BF_SDF_BLOCK_VOXELS) + 3 * t;
    uint4 qa = make_uint4(0, 0, 0, 0), qb = qa, qc = qa;
    bool loaded = false;
    unsigned dirty = 0;
    int liveDelta = 0;
#pragma unroll 1
    for (int k = 0; k < a.nOps; ++k) {
        const unsigned fl = (opMask >> (2 * k)) & (kOldPose ? 3u : 2u);
        if (!fl) continue;                                   // uniform for the CTA
        const MultiOp& op = a.ops[k];
        ProbeSet pA, pB;
        float zA[4], zB[4];
        pA.mask = 0; pB.mask = 0;
        if (kOldPose && (fl & 1u)) project4(a.cam, op.depth, op.A, vx, vy, vz, pA, zA);
        if (fl & 2u) project4(a.cam, op.depth, op.B, vx, vy, vz, pB, zB);
        if (kOldPose && (fl & 1u)) decide4(op.A, pA, zA);
        if (fl & 2u) decide4(op.B, pB, zB);
        const unsigned mask = pA.mask | pB.mask;
        if (mask) {
            unsigned cA[4], cB[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                cA[j] = kOldPose ? __ldg(&op.color[(pA.mask >> j) & 1u ? pA.idx[j] : 0u]) : 0u;
                cB[j] = __ldg(&op.color[(pB.mask >> j) & 1u ? pB.idx[j] : 0u]);
            }
            if (!loaded) { qa = vp[0]; qb = vp[1]; qc = vp[2]; loaded = true; }
            if (kOldPose) {
                if (mask & 1u) update_pair(op.B, pA.mask & 1u, pA.sdf[0], cA[0], pB.mask & 1u, pB.sdf[0], cB[0], qa.x, qa.y, qa.z, liveDelta);
                if (mask & 2u) update_pair(op.B, pA.mask & 2u, pA.sdf[1], cA[1], pB.mask & 2u, pB.sdf[1], cB[1], qa.w, qb.x, qb.y, liveDelta);
                if (mask & 4u) update_pair(op.B, pA.mask & 4u, pA.sdf[2], cA[2], pB.mask & 4u, pB.sdf[2], cB[2], qb.z, qb.w, qc.x, liveDelta);
                if (mask & 8u) update_pair(op.B, pA.mask & 8u, pA.sdf[3], cA[3], pB.mask & 8u, pB.sdf[3], cB[3], qc.y, qc.z, qc.w, liveDelta);
            } else {
                if (mask & 1u) update_fast<0>(op.B, op.B, true, pB.sdf[0], cB[0], false, 0.0f, 0u, qa.x, qa.y, qa.z, liveDelta);
                if (mask & 2u) update_fast<0>(op.B, op.B, true, pB.sdf[1], cB[1], false, 0.0f, 0u, qa.w, qb.x, qb.y, liveDelta);
                if (mask & 4u) update_fast<0>(op.B, op.B, true, pB.sdf[2], cB[2], false, 0.0f, 0u, qb.z, qb.w, qc.x, liveDelta);
                if (mask & 8u) update_fast<0>(op.B, op.B, true, pB.sdf[3], cB[3], false, 0.0f, 0u, qc.y, qc.z, qc.w, liveDelta);
            }
            dirty |= mask;
            passed += __popc(pA.mask) + __popc(pB.mask);
        }
    }
    if (dirty & 0x3u) vp[0] = qa;
    if (dirty & 0x6u) vp[1] = qb;
    if (dirty & 0xCu) vp[2] = qc;
    live_delta_commit(a.live, (unsigned)w.w, t, liveDelta);
}

// Persistent grid.  With a work list (the library's own compactify) blocks are dealt out dynamically: a CTA starts on block blockIdx.x and
// then draws tickets from a per-list counter (zeroed with the list's counter set), two iterations ahead, so that the atomic and the work-item
// load it feeds are in flight while a block is being processed -- blocks differ 3x in cost (none / all voxels pass), a static deal leaves
// a quarter of the SM-time idle at the tail.  Without a work list (reference-named stubs: d_hashCompactified, count from the caller) the
// deal is static.
template <int MODE, bool DYN>
__global__ void __launch_bounds__(128, MODE == 2 ? BF_FAST_MINBLOCKS_FUSED : BF_FAST_MINBLOCKS)
stencil_fast_kernel(const __grid_constant__ FastArgs a) {
    const unsigned listCount = a.useListCount ? a.ctrs[a.set + SET_COUNT] : a.countOverride;
    const unsigned count = DYN ? a.ctrs[a.set + SET_WORK] : listCount;
    const unsigned t = threadIdx.x;
    if (blockIdx.x == 0 && t == 0) {
        if (a.useListCount) { a.listCounterOut[0] = (int)listCount; a.ctrs[CTR_E] = listCount; }
        if (!DYN) atomicAdd(reinterpret_cast<unsigned long long*>(&a.ctrs[CTR_E_TOT_LO]), (unsigned long long)listCount);
    }
    ThreadVoxel o;
    o.lx = (int)((4 * t) & 7); o.ly = (int)(((4 * t) & 63) >> 3); o.lz = (int)((4 * t) >> 6);
    unsigned passed = 0;
    if (DYN) {
#ifndef BF_EMU_SEQUENTIAL
        __shared__ int4 sWork[2];
        const int4 kEnd = make_int4(0, 0, 0, -1);
        unsigned* const ticket = &a.ctrs[a.set + SET_TICKET];
        int4 wCur = (blockIdx.x < count) ? __ldg(&a.work[blockIdx.x]) : kEnd;
        int4 wNext = kEnd; unsigned iAfter = 0xFFFFFFFFu;
        if (t == 0) {
            const unsigned i1 = gridDim.x + atomicAdd(ticket, 1u);
            wNext = (i1 < count) ? __ldg(&a.work[i1]) : kEnd;
            iAfter = gridDim.x + atomicAdd(ticket, 1u);
        }
        unsigned parity = 0;
        while (wCur.w != -1) {
            process_block<MODE>(a, o, t, wCur.x, wCur.y, wCur.z, ((unsigned)wCur.w & 0x0FFFFFFFu) * BF_SDF_BLOCK_VOXELS, MODE == 2 ? ((unsigned)wCur.w >> 28) : 3u, passed);
            if (t == 0) {
                sWork[parity] = wNext;
                wNext = (iAfter < count) ? __ldg(&a.work[iAfter]) : kEnd;
                iAfter = (iAfter < count) ? gridDim.x + atomicAdd(ticket, 1u) : 0xFFFFFFFFu;
            }
            __syncthreads();
            wCur = sWork[parity];
            parity ^= 1u;
        }
#else
        for (unsigned b = blockIdx.x; b < count; b += gridDim.x) {      // sequential emulation: static deal (same set of blocks)
            const int4 w = a.work[b];
            process_block<MODE>(a, o, t, w.x, w.y, w.z, ((unsigned)w.w & 0x0FFFFFFFu) * BF_SDF_BLOCK_VOXELS, MODE == 2 ? ((unsigned)w.w >> 28) : 3u, passed);
        }
#endif
    } else {
        for (unsigned b = blockIdx.x; b < count; b += gridDim.x) {
            const BFHashEntry* ep = &a.list[b];
            process_block<MODE>(a, o, t, __ldg(&ep->pos[0]), __ldg(&ep->pos[1]), __ldg(&ep->pos[2]), (unsigned)__ldg(&ep->ptr), 3u, passed);
        }
    }
    // U statistics (voxel updates, the roofline's byte count): one 64-bit atomic per warp, no barrier at the end of the kernel
#ifdef BF_EMU_SEQUENTIAL
    if (passed) { atomicAdd(reinterpret_cast<unsigned long long*>(&a.ctrs[a.set + SET_U_LO]), (unsigned long long)passed); atomicAdd(reinterpret_cast<unsigned long long*>(&a.ctrs[CTR_U_TOT_LO]), (unsigned long long)passed); }
#else
    passed = warp_sum_u(passed);
    if ((t & 31) == 0 && passed) {
        atomicAdd(reinterpret_cast<unsigned long long*>(&a.ctrs[a.set + SET_U_LO]), (unsigned long long)passed);
        atomicAdd(reinterpret_cast<unsigned long long*>(&a.ctrs[CTR_U_TOT_LO]), (unsigned long long)passed);
    }
#endif
}

// batch re-integration (kOldPose) or batch integration: the same persistent grid and dynamic deal over the union list, every block visited once
// for up to 16 ops
template <bool kOldPose>
__global__ void __launch_bounds__(128, kOldPose ? BF_FAST_MINBLOCKS_FUSED : BF_FAST_MINBLOCKS)
stencil_multi_kernel(const __grid_constant__ MultiArgs a) {
    // ticket i -> work item: the four cost buckets in order, costliest first (layout: tsdf_shared.cuh)
    const unsigned n3 = a.ctrs[a.set + SET_WORK], n2 = a.ctrs[a.set + SET_Q2], n1 = a.ctrs[a.set + SET_Q1], n0 = a.ctrs[a.set + SET_Q0];
    const unsigned e3 = n3, e2 = n3 + n2, e1 = e2 + n1, count = e1 + n0;
    const unsigned t = threadIdx.x;
    if (blockIdx.x == 0 && t == 0) { const unsigned listCount = a.ctrs[a.set + SET_COUNT]; a.listCounterOut[0] = (int)listCount; a.ctrs[CTR_E] = listCount; }
    ThreadVoxel o;
    o.lx = (int)((4 * t) & 7); o.ly = (int)(((4 * t) & 63) >> 3); o.lz = (int)((4 * t) >> 6);
    unsigned passed = 0;
#ifndef BF_EMU_SEQUENTIAL
    if (a.ktime && t == 0) { unsigned long long g; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g)); atomicMin(&a.ktime[0], g); }
#endif
#define BF_MULTI_LOAD(i, W, M)                                                                                              \
    do {                                                                                                                    \
        const unsigned _i = (i);                                                                                            \
        if (_i < e3)      { W = __ldg(&a.workA[_i]);                          M = __ldg(&a.maskA[_i]); }                    \
        else if (_i < e2) { const unsigned _j = a.workCap - 1u - (_i - e3); W = __ldg(&a.workA[_j]); M = __ldg(&a.maskA[_j]); } \
        else if (_i < e1) { const unsigned _j = _i - e2;                     W = __ldg(&a.workB[_j]); M = __ldg(&a.maskB[_j]); } \
        else              { const unsigned _j = a.workCap - 1u - (_i - e1); W = __ldg(&a.workB[_j]); M = __ldg(&a.maskB[_j]); } \
    } while (0)
#ifndef BF_EMU_SEQUENTIAL
    __shared__ int4 sWork[2];
    __shared__ unsigned sMask[2];
    const int4 kEnd = make_int4(0, 0, 0, -1);
    unsigned* const ticket = &a.ctrs[a.set + SET_TICKET];
    int4 wCur = kEnd; unsigned mCur = 0;
    if (blockIdx.x < count) BF_MULTI_LOAD(blockIdx.x, wCur, mCur);
    int4 wNext = kEnd; unsigned mNext = 0, iAfter = 0xFFFFFFFFu;
    if (t == 0) {
        const unsigned i1 = gridDim.x + atomicAdd(ticket, 1u);
        if (i1 < count) BF_MULTI_LOAD(i1, wNext, mNext);
        iAfter = gridDim.x + atomicAdd(ticket, 1u);
    }
    unsigned parity = 0;
    while (wCur.w != -1) {
        process_block_multi<kOldPose>(a, o, t, wCur, mCur, passed);
        if (t == 0) {
            sWork[parity] = wNext; sMask[parity] = mNext;
            wNext = kEnd; mNext = 0;
            if (iAfter < count) { BF_MULTI_LOAD(iAfter, wNext, mNext); iAfter = gridDim.x + atomicAdd(ticket, 1u); }
            else iAfter = 0xFFFFFFFFu;
        }
        __syncthreads();
        wCur = sWork[parity]; mCur = sMask[parity];
        parity ^= 1u;
    }
    passed = warp_sum_u(passed);
    if ((t & 31) == 0 && passed) {
        atomicAdd(reinterpret_cast<unsigned long long*>(&a.ctrs[a.set + SET_U_LO]), (unsigned long long)passed);
        atomicAdd(reinterpret_cast<unsigned long long*>(&a.ctrs[CTR_U_TOT_LO]), (unsigned long long)passed);
        atomicAdd(reinterpret_cast<unsigned long long*>(&a.ctrs[CTR_UB_TOT_LO]), (unsigned long long)passed);
    }
    if (a.ktime && t == 0) { unsigned long long g; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g)); atomicMax(&a.ktime[1], g); }
#else
    for (unsigned b = blockIdx.x; b < count; b += gridDim.x) { int4 w; unsigned m; BF_MULTI_LOAD(b, w, m); process_block_multi<kOldPose>(a, o, t, w, m, passed); }
    if (passed) { atomicAdd(reinterpret_cast<unsigned long long*>(&a.ctrs[a.set + SET_U_LO]), (unsigned long long)passed); atomicAdd(reinterpret_cast<unsigned long long*>(&a.ctrs[CTR_U_TOT_LO]), (unsigned long long)passed); }
#endif
#undef BF_MULTI_LOAD
}

// ---- host side ----------------------------------------------------------------------------------------------------------
static void make_pose(const BFHashParams* hp, const BFDepthCameraParams* cp, FastPose* p) {
    const float* M = hp->m_rigidTransformInverse.m;
    const double vs = (double)hp->m_virtualVoxelSize;
    const double fx = cp->fx, fy = cp->fy;
    for (int c = 0; c < 4; ++c) {
        const double s = c < 3 ? vs : 1.0;
        const double rx = (double)M[0 + c] * s, ry = (double)M[4 + c] * s, rz = (double)M[8 + c] * s;
        p->cx[c] = (float)(fx * rx); p->cy[c] = (float)(fy * ry); p->cz[c] = (float)rz;
    }
    p->maxDist = hp->m_maxIntegrationDistance; p->trunc0 = hp->m_truncation; p->truncScale = hp->m_truncScale; p->wMax = (float)hp->m_integrationWeightMax;
}
static void make_args(FastArgs* a, const BFHashDataStruct* hd, const BFDepthCameraParams* cp, const float* depth, const void* color,
                      bool useListCount, unsigned countOverride, unsigned* ctrs, int* live, const int4* work, int set) {
    a->blocks = hd->d_SDFBlocks; a->list = hd->d_hashCompactified; a->listCounterOut = hd->d_hashCompactifiedCounter; a->work = work;
    a->depth = depth; a->color = reinterpret_cast<const uchar4*>(color); a->ctrs = ctrs; a->live = live;
    a->set = set; a->useListCount = useListCount ? 1 : 0; a->countOverride = countOverride;
    a->cam.W = cp->m_imageWidth; a->cam.H = cp->m_imageHeight; a->cam.fx = cp->fx; a->cam.fy = cp->fy; a->cam.mx5 = cp->mx + 0.5f; a->cam.my5 = cp->my + 0.5f;
}

int fast_stencil_ctas_per_sm(bool fused) { return fused ? BF_FAST_MINBLOCKS_FUSED : BF_FAST_MINBLOCKS; }

int launch_integrate_fast(const BFHashDataStruct* hd, const BFHashParams* hp, const BFDepthCameraParams* cp, const float* depth, const void* color,
                          bool deIntegrate, bool useListCount, unsigned countOverride, unsigned* ctrs, int* live, const int4* work, int set,
                          int grid, cudaStream_t s) {
    FastArgs a;
    make_args(&a, hd, cp, depth, color, useListCount, countOverride, ctrs, live, work, set);
    make_pose(hp, cp, &a.A); a.B = a.A;
    if (work) { if (deIntegrate) stencil_fast_kernel<1, true><<<grid, 128, 0, s>>>(a); else stencil_fast_kernel<0, true><<<grid, 128, 0, s>>>(a); }
    else      { if (deIntegrate) stencil_fast_kernel<1, false><<<grid, 128, 0, s>>>(a); else stencil_fast_kernel<0, false><<<grid, 128, 0, s>>>(a); }
    BF_CHECK(cudaGetLastError());
    return 0;
}

int launch_reintegrate_fast(const BFHashDataStruct* hd, const BFHashParams* hpOld, const BFHashParams* hpNew, const BFDepthCameraParams* cp,
                            const float* depth, const void* color, const int4* work, int set, unsigned* ctrs, int* live, int grid, cudaStream_t s) {
    FastArgs a;
    make_args(&a, hd, cp, depth, color, true, 0, ctrs, live, work, set);
    make_pose(hpOld, cp, &a.A); make_pose(hpNew, cp, &a.B);
    stencil_fast_kernel<2, true><<<grid, 128, 0, s>>>(a);
    BF_CHECK(cudaGetLastError());
    return 0;
}

int launch_reintegrate_multi_fast(const BFHashDataStruct* hd, const BFMultiOpDesc* ops, int nOps, const BFDepthCameraParams* cp, const int4* workA, const int4* workB,
                                  const unsigned* maskA, const unsigned* maskB, unsigned workCap, int set, unsigned* ctrs, int* live, int grid, cudaStream_t s,
                                  unsigned long long* ktime) {
    if (nOps < 1 || nOps > BF_MULTI_MAX_OPS) return (int)cudaErrorInvalidValue;
    static MultiArgs a;                      // ~2.5 KB: kept off the stack; filled and passed by value at the launch
    a.blocks = hd->d_SDFBlocks; a.workA = workA; a.workB = workB; a.maskA = maskA; a.maskB = maskB; a.ctrs = ctrs; a.live = live; a.listCounterOut = hd->d_hashCompactifiedCounter;
    a.set = set; a.nOps = nOps; a.workCap = workCap; a.ktime = ktime;
    a.cam.W = cp->m_imageWidth; a.cam.H = cp->m_imageHeight; a.cam.fx = cp->fx; a.cam.fy = cp->fy; a.cam.mx5 = cp->mx + 0.5f; a.cam.my5 = cp->my + 0.5f;
    const bool oldPose = ops[0].hpOld != nullptr;     // all ops of a batch alike: re-integration pairs, or integrations (hpOld NULL)
    for (int k = 0; k < nOps; ++k) {
        make_pose(ops[k].hpNew, cp, &a.ops[k].B);
        if (oldPose) make_pose(ops[k].hpOld, cp, &a.ops[k].A); else a.ops[k].A = a.ops[k].B;
        a.ops[k].depth = ops[k].depth; a.ops[k].color = reinterpret_cast<const unsigned*>(ops[k].color);
    }
    // one launch site for both instantiations, under the kernel's name: tests/test_tsdf_fast_emulated.py rewrites this launch to run the kernel on the CPU
    void (*const stencil_multi_kernel)(MultiArgs) = oldPose ? bf::stencil_multi_kernel<true> : bf::stencil_multi_kernel<false>;
    stencil_multi_kernel<<<grid, 128, 0, s>>>(a);
    BF_CHECK(cudaGetLastError());
    return 0;
}

}  // namespace bf

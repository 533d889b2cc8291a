// sift_filter.cu -- Kabsch match filter for sm_90a.  Implements bfSiftFilterKeyPointMatches of include/bf_sift.h (row a19, first filter).
//
// Behavioural source (what, not how): FL/SiftGPU/SIFTImageManager.cu:186-316 (FilterKeyPointMatchesCU), FL/SiftGPU/cuda_kabsch.h:110-502,
// FL/SiftGPU/cuda_EigenValue.h:9-39.  The per-pair algorithm is inherently sequential (greedy insertion with re-fits), so, as in the
// reference, a pair's raw matches are walked in order; pairs run in parallel, one warp each, arrays in shared memory -- and inside a fit the warp's
// lanes carry the independent sums (see "The per-pair algorithm on ONE WARP" below), each in the serial order.  The device functions follow
// oracle/filter_oracle.c operation for operation (this TU is built -fmad=false), including the reference's own 3x3 SVD (the fast approximate one of cuda_svd3.h, with rsqrt taken as 1 / sqrtf).
#include "../../include/bf_sift.h"
#include "bf_common.cuh"
#include "mat4.cuh"

namespace bf {

extern unsigned long long g_launchCount;

#define MAX_RAW BF_MAX_MATCHES_PER_IMAGE_PAIR_RAW
#define MAX_FILTERED BF_MAX_MATCHES_PER_IMAGE_PAIR_FILTERED
#define KABSCH_CONDITION_THRESH 100.0f  /* cuda_kabsch.h:231 */

struct KeyPoint { float px, py, scale, depth; };       // SIFTKeyPoint, FL/SiftGPU/SIFTImageManager.h:22-26
struct f3 { float x, y, z; };

/* cuda_EigenValue.h:9-39: eigenvalues of a symmetric 3x3, e0 >= e1 >= e2 */
__device__ void sym_eigenvalues(const float a[9], float e[3]) {
    const float PI = 3.14159265f;
    float p = a[1] * a[1] + a[2] * a[2] + a[5] * a[5];
    if (p == 0.0f) { e[0] = a[0]; e[1] = a[4]; e[2] = a[8]; return; }
    const float q = (a[0] + a[4] + a[8]) / 3.0f;
    p = (a[0] - q) * (a[0] - q) + (a[4] - q) * (a[4] - q) + (a[8] - q) * (a[8] - q) + 2.0f * p;
    p = sqrtf(p / 6.0f);
    float B[9];
    for (int k = 0; k < 9; ++k) B[k] = (a[k] - ((k % 4 == 0) ? q : 0.0f)) * (1.0f / p);
    const float det = B[0] * (B[4] * B[8] - B[5] * B[7]) - B[1] * (B[3] * B[8] - B[5] * B[6]) + B[2] * (B[3] * B[7] - B[4] * B[6]);
    const float r = det / 2.0f;
    float phi;
    if (r <= -1.0f) phi = PI / 3.0f; else if (r >= 1.0f) phi = 0.0f; else phi = acosf(r) / 3.0f;
    e[0] = q + 2.0f * p * cosf(phi);
    e[2] = q + 2.0f * p * cosf(phi + PI * (2.0f / 3.0f));
    e[1] = 3.0f * q - e[0] - e[2];
}

/* The reference's 3x3 SVD (FL/SiftGPU/cuda_svd3.h: E. Jang's version of McAdams et al., TR1690): four fixed sweeps with the approximate
 * Givens angle, quaternion accumulation, column sort (with the reference's rho2 over b12, b22, b23), Givens QR.  Operation for operation the
 * same as oracle/filter_oracle.c svd3_fast(), which is pinned bit for bit against the reference's own host build of that header
 * (tests/test_kabsch_reference_host.py).  rsqrt: the reference's device build calls CUDA's rsqrtf (2 ulp); here, as in the oracle,
 * 1 / sqrtf, individually rounded. */
__device__ __forceinline__ float rsqrt_exact(float x) { return 1.0f / sqrtf(x); }
__device__ void cond_swap(int c, float* X, float* Y) { const float Z = *X; *X = c ? *Y : *X; *Y = c ? Z : *Y; }
__device__ void cond_neg_swap(int c, float* X, float* Y) { const float Z = -*X; *X = c ? *Y : *X; *Y = c ? Z : *Y; }

__device__ void jacobi_conjugation(int x, int y, int z, float* s11, float* s21, float* s22, float* s31, float* s32, float* s33, float* qV) {    /* cuda_svd3.h:149-204 */
    float ch = 2.0f * (*s11 - *s22), sh = *s21;                                  /* approximateGivensQuaternion, :134-147 */
    const int big = 5.828427124f * sh * sh < ch * ch;
    const float w = rsqrt_exact(ch * ch + sh * sh);
    ch = big ? w * ch : 0.923879532f;
    sh = big ? w * sh : 0.3826834323f;
    const float scale = ch * ch + sh * sh;
    const float a = (ch * ch - sh * sh) / scale, b = (2.0f * sh * ch) / scale;
    float t11 = *s11, t21 = *s21, t22 = *s22, t31 = *s31, t32 = *s32, t33 = *s33;
    *s11 = a * (a * t11 + b * t21) + b * (a * t21 + b * t22);
    *s21 = a * (-b * t11 + a * t21) + b * (-b * t21 + a * t22);
    *s22 = -b * (-b * t11 + a * t21) + a * (-b * t21 + a * t22);
    *s31 = a * t31 + b * t32; *s32 = -b * t31 + a * t32; *s33 = t33;
    float tmp[3] = { qV[0] * sh, qV[1] * sh, qV[2] * sh };
    sh *= qV[3];
    qV[0] *= ch; qV[1] *= ch; qV[2] *= ch; qV[3] *= ch;
    qV[z] += sh; qV[3] -= tmp[z]; qV[x] += tmp[y]; qV[y] -= tmp[x];
    t11 = *s22; t21 = *s32; t22 = *s33; t31 = *s21; t32 = *s31; t33 = *s11;      /* re-arrange for the next rotation */
    *s11 = t11; *s21 = t21; *s22 = t22; *s31 = t31; *s32 = t32; *s33 = t33;
}
__device__ void qr_givens(float a1, float a2, float* ch, float* sh) {               /* QRGivensQuaternion, :265-281 */
    const float eps = 1e-6f, q = a1 * a1 + a2 * a2;
    const float rho = q * rsqrt_exact(q);                                              /* accurateSqrt */
    *sh = rho > eps ? a2 : 0.0f;
    *ch = fabsf(a1) + fmaxf(rho, eps);
    cond_swap(a1 < 0.0f, sh, ch);
    const float w = rsqrt_exact(*ch * *ch + *sh * *sh);
    *ch *= w; *sh *= w;
}
/* svd(A) -> U, S (upper triangular R of the QR, its diagonal = singular values up to sign), V; all row-major 3x3.  cuda_svd3.h:347-393 */
__device__ void svd3_fast(const float A[9], float U[9], float S[9], float V[9]) {
    const float a11 = A[0], a12 = A[1], a13 = A[2], a21 = A[3], a22 = A[4], a23 = A[5], a31 = A[6], a32 = A[7], a33 = A[8];
    /* A^T A (multAtB) */
    float s11 = a11 * a11 + a21 * a21 + a31 * a31;
    float s21 = a12 * a11 + a22 * a21 + a32 * a31, s22 = a12 * a12 + a22 * a22 + a32 * a32;
    float s31 = a13 * a11 + a23 * a21 + a33 * a31, s32 = a13 * a12 + a23 * a22 + a33 * a32, s33 = a13 * a13 + a23 * a23 + a33 * a33;
    float qV[4] = { 0.0f, 0.0f, 0.0f, 1.0f };
    for (int i = 0; i < 4; ++i) {                                                 /* jacobiEigenanlysis, :214-229 */
        jacobi_conjugation(0, 1, 2, &s11, &s21, &s22, &s31, &s32, &s33, qV);
        jacobi_conjugation(1, 2, 0, &s11, &s21, &s22, &s31, &s32, &s33, qV);
        jacobi_conjugation(2, 0, 1, &s11, &s21, &s22, &s31, &s32, &s33, qV);
    }
    /* quatToMat3, :102-131 */
    const float w = qV[3], x = qV[0], y = qV[1], z = qV[2];
    const float qxx = x * x, qyy = y * y, qzz = z * z, qxz = x * z, qxy = x * y, qyz = y * z, qwx = w * x, qwy = w * y, qwz = w * z;
    float v11 = 1 - 2 * (qyy + qzz), v12 = 2 * (qxy - qwz), v13 = 2 * (qxz + qwy);
    float v21 = 2 * (qxy + qwz), v22 = 1 - 2 * (qxx + qzz), v23 = 2 * (qyz - qwx);
    float v31 = 2 * (qxz - qwy), v32 = 2 * (qyz + qwx), v33 = 1 - 2 * (qxx + qyy);
    /* B = A V (multAB) */
    float b11 = a11 * v11 + a12 * v21 + a13 * v31, b12 = a11 * v12 + a12 * v22 + a13 * v32, b13 = a11 * v13 + a12 * v23 + a13 * v33;
    float b21 = a21 * v11 + a22 * v21 + a23 * v31, b22 = a21 * v12 + a22 * v22 + a23 * v32, b23 = a21 * v13 + a22 * v23 + a23 * v33;
    float b31 = a31 * v11 + a32 * v21 + a33 * v31, b32 = a31 * v12 + a32 * v22 + a33 * v32, b33 = a31 * v13 + a32 * v23 + a33 * v33;
    /* sortSingularValues, :231-262 (rho2 over b12, b22, b23 as written there) */
    float rho1 = b11 * b11 + b21 * b21 + b31 * b31, rho2 = b12 * b12 + b22 * b22 + b23 * b23, rho3 = b13 * b13 + b23 * b23 + b33 * b33;
    int c = rho1 < rho2;
    cond_neg_swap(c, &b11, &b12); cond_neg_swap(c, &v11, &v12); cond_neg_swap(c, &b21, &b22); cond_neg_swap(c, &v21, &v22); cond_neg_swap(c, &b31, &b32); cond_neg_swap(c, &v31, &v32);
    cond_swap(c, &rho1, &rho2);
    c = rho1 < rho3;
    cond_neg_swap(c, &b11, &b13); cond_neg_swap(c, &v11, &v13); cond_neg_swap(c, &b21, &b23); cond_neg_swap(c, &v21, &v23); cond_neg_swap(c, &b31, &b33); cond_neg_swap(c, &v31, &v33);
    cond_swap(c, &rho1, &rho3);
    c = rho2 < rho3;
    cond_neg_swap(c, &b12, &b13); cond_neg_swap(c, &v12, &v13); cond_neg_swap(c, &b22, &b23); cond_neg_swap(c, &v22, &v23); cond_neg_swap(c, &b32, &b33); cond_neg_swap(c, &v32, &v33);
    /* QRDecomposition, :283-345 */
    float ch1, sh1, ch2, sh2, ch3, sh3, r11, r12, r13, r21, r22, r23, r31, r32, r33;
    qr_givens(b11, b21, &ch1, &sh1);
    float a = 1 - 2 * sh1 * sh1, b = 2 * ch1 * sh1;
    r11 = a * b11 + b * b21; r12 = a * b12 + b * b22; r13 = a * b13 + b * b23;
    r21 = -b * b11 + a * b21; r22 = -b * b12 + a * b22; r23 = -b * b13 + a * b23;
    r31 = b31; r32 = b32; r33 = b33;
    qr_givens(r11, r31, &ch2, &sh2);
    a = 1 - 2 * sh2 * sh2; b = 2 * ch2 * sh2;
    b11 = a * r11 + b * r31; b12 = a * r12 + b * r32; b13 = a * r13 + b * r33;
    b21 = r21; b22 = r22; b23 = r23;
    b31 = -b * r11 + a * r31; b32 = -b * r12 + a * r32; b33 = -b * r13 + a * r33;
    qr_givens(b22, b32, &ch3, &sh3);
    a = 1 - 2 * sh3 * sh3; b = 2 * ch3 * sh3;
    r11 = b11; r12 = b12; r13 = b13;
    r21 = a * b21 + b * b31; r22 = a * b22 + b * b32; r23 = a * b23 + b * b33;
    r31 = -b * b21 + a * b31; r32 = -b * b22 + a * b32; r33 = -b * b23 + a * b33;
    const float sh12 = sh1 * sh1, sh22 = sh2 * sh2, sh32 = sh3 * sh3;
    U[0] = (-1 + 2 * sh12) * (-1 + 2 * sh22);
    U[1] = 4 * ch2 * ch3 * (-1 + 2 * sh12) * sh2 * sh3 + 2 * ch1 * sh1 * (-1 + 2 * sh32);
    U[2] = 4 * ch1 * ch3 * sh1 * sh3 - 2 * ch2 * (-1 + 2 * sh12) * sh2 * (-1 + 2 * sh32);
    U[3] = 2 * ch1 * sh1 * (1 - 2 * sh22);
    U[4] = -8 * ch1 * ch2 * ch3 * sh1 * sh2 * sh3 + (-1 + 2 * sh12) * (-1 + 2 * sh32);
    U[5] = -2 * ch3 * sh3 + 4 * sh1 * (ch3 * sh1 * sh3 + ch1 * ch2 * sh2 * (-1 + 2 * sh32));
    U[6] = 2 * ch2 * sh2;
    U[7] = 2 * ch3 * (1 - 2 * sh22) * sh3;
    U[8] = (-1 + 2 * sh22) * (-1 + 2 * sh32);
    S[0] = r11; S[1] = r12; S[2] = r13; S[3] = r21; S[4] = r22; S[5] = r23; S[6] = r31; S[7] = r32; S[8] = r33;
    V[0] = v11; V[1] = v12; V[2] = v13; V[3] = v21; V[4] = v22; V[5] = v23; V[6] = v31; V[7] = v32; V[8] = v33;
}
/* svd(m, v, s) + svdAbsEV, cuda_svd3.h:436-482: U, V and the ABSOLUTE diagonal of S (the columns of U follow the sign), unsorted */
__device__ void svd3(const float H[9], float U[9], float s[3], float V[9]) {
    float S[9];
    svd3_fast(H, U, S, V);
    s[0] = S[0]; s[1] = S[4]; s[2] = S[8];
    for (int i = 0; i < 3; ++i) if (s[i] < 0.0f) { s[i] *= -1.0f; for (int j = 0; j < 3; ++j) U[3 * j + i] *= -1.0f; }
}

/* matNxM<3,3>::det, cuda_SimpleMatrixUtil.h:1544-1559 */
__device__ float det3(const float m[9]) { return m[0] * m[4] * m[8] + m[1] * m[5] * m[6] + m[2] * m[3] * m[7] - m[6] * m[4] * m[2] - m[7] * m[5] * m[0] - m[8] * m[3] * m[1]; }

/* ---- The per-pair algorithm on ONE WARP ---------------------------------------------------------------------------------------------------
 * filterKeyPointMatches (cuda_kabsch.h:417-502) is a greedy loop -- add a match, re-fit, drop the worst while the fit is bad -- and the reference runs
 * it on one thread per image pair.  The loop is sequential, the work inside a fit is not: the 6 mean components, the 9 covariance entries of the Kabsch
 * fit, the n residuals, the ranks of the sort, the 2 x 9 covariance entries of the condition test and the `addMatch` distance tests are independent
 * chains.  Each chain goes to one lane and is evaluated there in the reference's order (ascending point index, one rounding per operation; this TU is
 * built -fmad=false), so every sum has the bits of the serial evaluation; the 3x3 SVD and the small matrix products run redundantly on all lanes
 * (uniform, nothing to broadcast).  Control flow is uniform across the warp (decisions come from shared memory or from ballots).  Arrays live in
 * shared memory, phases are separated by __syncwarp(). */
#define FULL 0xFFFFFFFFu

/* kabsch(), cuda_kabsch.h:110-176, from the means (p0 | q0) and the covariance H: T (4x4 row-major) with T src ~ tgt; evs = singular values, descending */
__device__ void kabsch_from_moments(const float m[6], const float H[9], float T[16], float evs[3]) {
    const float* p0 = m; const float* q0 = m + 3;
    float U[9], V[9];
    svd3(H, U, evs, V);
    { float t; if (evs[0] < evs[1]) { t = evs[0]; evs[0] = evs[1]; evs[1] = t; } if (evs[1] < evs[2]) { t = evs[1]; evs[1] = evs[2]; evs[2] = t; }
      if (evs[0] < evs[1]) { t = evs[0]; evs[0] = evs[1]; evs[1] = t; } }          /* cuda_kabsch.h:139-141 */
    /* R = V D U^T, D = diag(1, 1, -1) when det(U V^T) < 0 (cuda_kabsch.h:185-190): always the THIRD column, whatever the order of the values */
    float UVt[9];
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) UVt[3 * r + c] = U[3 * r] * V[3 * c] + U[3 * r + 1] * V[3 * c + 1] + U[3 * r + 2] * V[3 * c + 2];
    const float d = (det3(UVt) < 0.0f) ? -1.0f : 1.0f;
    float R[9];
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) R[3 * r + c] = V[3 * r] * U[3 * c] + V[3 * r + 1] * U[3 * c + 1] + (V[3 * r + 2] * d) * U[3 * c + 2];
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) T[4 * r + c] = R[3 * r + c];
        T[4 * r + 3] = q0[r] - (R[3 * r] * p0[0] + R[3 * r + 1] * p0[1] + R[3 * r + 2] * p0[2]);
    }
    T[12] = T[13] = T[14] = 0.0f; T[15] = 1.0f;
}
__device__ __forceinline__ float f3_get(const f3* p, unsigned i, int c) { return (&p[i].x)[c]; }

/* means of src (lanes 0..2) and tgt (lanes 3..5) over the first n points, every lane gets all six: p0[k] = (((0 + x0) + x1) + ...) / n as the serial loop */
__device__ __forceinline__ void warp_means(const f3* src, const f3* tgt, unsigned n, unsigned lane, float m[6]) {
    float acc = 0.0f;
    if (lane < 6) {
        const f3* pts = lane < 3 ? src : tgt; const int c = (int)(lane % 3);
        for (unsigned i = 0; i < n; ++i) acc += f3_get(pts, i, c);
        acc /= (float)n;
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) m[k] = __shfl_sync(FULL, acc, k);
}

/* ComputeReprojection(), cuda_kabsch.h:381-414, on one warp: fit, residuals, sort by residual, condition numbers.  T / the return value are uniform. */
__device__ int compute_reprojection(f3* src, f3* tgt, unsigned n, float* res, float T[16], uint32_t* idx /*[.][2]*/, float* dist, unsigned lane) {
    float m[6], H[9], evs[3];
    __syncwarp();
    warp_means(src, tgt, n, lane, m);
    {   /* covariance of the fit (cuda_kabsch.h:121-131): entry (r, c) on lane 3 r + c */
        float h = 0.0f;
        if (lane < 9) {
            const int r = (int)lane / 3, c = (int)lane % 3;
            for (unsigned i = 0; i < n; ++i) { const float p = f3_get(src, i, r) - m[r], q = f3_get(tgt, i, c) - m[3 + c]; h += p * q; }
            h /= (float)n;
        }
#pragma unroll
        for (int k = 0; k < 9; ++k) H[k] = __shfl_sync(FULL, h, k);
    }
    kabsch_from_moments(m, H, T, evs);
    /* residual of point `lane` and its rank.  sortKabschResiduals (:368-377) is an exchange sort; its result is the ascending order, and only among EQUAL
     * (or unordered: NaN) residuals does the arrangement depend on its particular swap sequence -- then that sequence is replayed, by one lane. */
    float r = 0.0f; f3 a = { 0, 0, 0 }, b = { 0, 0, 0 }; uint32_t ia = 0, ib = 0; float d = 0.0f;
    if (lane < n) {
        a = src[lane]; b = tgt[lane]; ia = idx[2 * lane]; ib = idx[2 * lane + 1]; d = dist[lane];
        const float dx = (T[0] * a.x + T[1] * a.y + T[2] * a.z + T[3]) - b.x;
        const float dy = (T[4] * a.x + T[5] * a.y + T[6] * a.z + T[7]) - b.y;
        const float dz = (T[8] * a.x + T[9] * a.y + T[10] * a.z + T[11]) - b.z;
        r = dx * dx + dy * dy + dz * dz;
        res[lane] = r;
    }
    __syncwarp();
    bool bad = false; unsigned rank = 0;
    if (lane < n) {
        bad = (r != r);
        for (unsigned j = 0; j < n; ++j) {
            const float rj = res[j];
            if (rj < r) ++rank;
            else if (j != lane && !(rj > r)) bad = true;                              /* equal or unordered */
        }
    }
    const bool replay = __ballot_sync(FULL, bad) != 0u;
    if (!replay) {
        if (lane < n) { res[rank] = r; src[rank] = a; tgt[rank] = b; idx[2 * rank] = ia; idx[2 * rank + 1] = ib; dist[rank] = d; }      /* all reads happened before the barrier above */
    } else if (lane == 0) {
        for (unsigned i = 0; i < n; ++i)
            for (unsigned j = i; j < n; ++j)
                if (res[i] > res[j]) {
                    float t = res[i]; res[i] = res[j]; res[j] = t;
                    f3 s = src[i]; src[i] = src[j]; src[j] = s;
                    s = tgt[i]; tgt[i] = tgt[j]; tgt[j] = s;
                    uint32_t x = idx[2 * i], y = idx[2 * i + 1]; idx[2 * i] = idx[2 * j]; idx[2 * i + 1] = idx[2 * j + 1]; idx[2 * j] = x; idx[2 * j + 1] = y;
                    t = dist[i]; dist[i] = dist[j]; dist[j] = t;
                }
    }
    __syncwarp();
    /* covarianceSVD() of the (sorted) source and target points, :178-198: entry (r, c) of the source covariance on lane 3 r + c, of the target's on lane 9 + 3 r + c */
    warp_means(src, tgt, n, lane, m);
    float cs = 0.0f;
    if (lane < 18) {
        const f3* pts = lane < 9 ? src : tgt; const float* p0 = lane < 9 ? m : m + 3;
        const int e = (int)lane % 9, rr = e / 3, cc = e % 3;
        for (unsigned i = 0; i < n; ++i) { const float p = f3_get(pts, i, rr) - p0[rr], q = f3_get(pts, i, cc) - p0[cc]; cs += p * q; }
        cs /= (float)n;
    }
    float C[9], e3[3];
    const int base = lane < 16 ? 0 : 9;                                               /* lanes 0..15 evaluate the source's eigenvalues, 16..31 the target's */
#pragma unroll
    for (int k = 0; k < 9; ++k) C[k] = __shfl_sync(FULL, cs, base + k);
    sym_eigenvalues(C, e3);
    const float ratio = e3[0] / e3[1];
    const float cp = __shfl_sync(FULL, ratio, 0), cq = __shfl_sync(FULL, ratio, 16);
    const float c1 = evs[0] / evs[1];
    if (c1 != c1 || cp != cp || cq != cq || fabsf(c1) > KABSCH_CONDITION_THRESH || fabsf(cp) > KABSCH_CONDITION_THRESH || fabsf(cq) > KABSCH_CONDITION_THRESH) return 0;
    return 1;
}
/* addMatch, :233-247: the candidate is refused when it lies within 5 pixels of a kept match in either image; kept match i on lane i */
__device__ int add_match(uint32_t ax, uint32_t ay, const KeyPoint* kp, const uint32_t* idx, unsigned cur, unsigned lane) {
    bool hit = false;
    if (lane < cur) {
        const float dix = kp[ax].px - kp[idx[2 * lane]].px, diy = kp[ax].py - kp[idx[2 * lane]].py;
        const float djx = kp[ay].px - kp[idx[2 * lane + 1]].px, djy = kp[ay].py - kp[idx[2 * lane + 1]].py;
        hit = sqrtf(dix * dix + diy * diy) <= 5.0f || sqrtf(djx * djx + djy * djy) <= 5.0f;
    }
    return __ballot_sync(FULL, hit) == 0u;
}
/* getKeySourceAndTargetPoints, :249-321, for matches [first, first + n): lane 2 i + s computes point i of image s */
__device__ void key_points_3d(const KeyPoint* kp, const uint32_t* idx, unsigned first, unsigned n, f3* src, f3* tgt, const float* Ki, unsigned lane) {
    if (lane < 2 * n) {
        const unsigned i = first + lane / 2; const int s = (int)(lane & 1u);
        const KeyPoint* k = &kp[idx[2 * i + s]];
        const float v[3] = { k->depth * k->px, k->depth * k->py, k->depth * 1.0f };
        f3 o = { Ki[0] * v[0] + Ki[1] * v[1] + Ki[2] * v[2] + Ki[3], Ki[4] * v[0] + Ki[5] * v[1] + Ki[6] * v[2] + Ki[7], Ki[8] * v[0] + Ki[9] * v[1] + Ki[10] * v[2] + Ki[11] };
        if (s == 0) src[i] = o; else tgt[i] = o;
    }
}

/* filterKeyPointMatches, cuda_kabsch.h:417-502.  idx / dist: the pair's raw matches (sorted by distance), modified in place; returns the
 * number of filtered matches (their indices / distances in the first slots), T = the transform estimate.  Called by all 32 lanes of the pair's warp. */
__device__ unsigned filter_pair(const KeyPoint* kp, uint32_t* idx, float* dist, unsigned numRaw, float T[16], const float* Ki, unsigned minNum, float maxRes2,
                                f3* src, f3* tgt, float* res, unsigned lane) {
    unsigned i0 = 0, cur = 0;
    float curMax = 100.0f;
    int valid = 0;
    for (int k = 0; k < 16; ++k) T[k] = (k % 5 == 0) ? 1.0f : 0.0f;
    for (;;) {
        if (i0 == numRaw || cur >= MAX_FILTERED) {
            if (cur < minNum || curMax >= maxRes2 || !valid) cur = 0;
            break;
        } else if (add_match(idx[2 * i0], idx[2 * i0 + 1], kp, idx, cur, lane)) {
            __syncwarp();
            if (lane == 0) { idx[2 * cur] = idx[2 * i0]; idx[2 * cur + 1] = idx[2 * i0 + 1]; dist[cur] = dist[i0]; }
            __syncwarp();
            ++cur;
            if (cur >= 3) {
                // getKeySourceAndTargetPoints recomputes all cur points from their indices; src / tgt follow idx through every sort, so only the points of
                // the first fit (cur == 3) and, afterwards, of the match just added are not in place already -- same values, 2 key-point loads instead of 2 cur
                if (cur == 3) key_points_3d(kp, idx, 0, 3, src, tgt, Ki, lane); else key_points_3d(kp, idx, cur - 1, 1, src, tgt, Ki, lane);
                valid = compute_reprojection(src, tgt, cur, res, T, idx, dist, lane);
                const int b = valid;
                float prevT[16]; for (int k = 0; k < 16; ++k) prevT[k] = T[k];
                curMax = res[cur - 1];
                if (curMax > maxRes2) {
                    float lastRes = -1.0f;
                    for (int i = (int)cur - 1; i >= 3; --i) {
                        lastRes = res[i];
                        --cur;
                        valid = compute_reprojection(src, tgt, cur, res, T, idx, dist, lane);
                        curMax = res[cur - 1];
                        if (cur == 3 && (curMax > maxRes2 || (b && !valid))) { ++cur; curMax = lastRes; valid = b; for (int k = 0; k < 16; ++k) T[k] = prevT[k]; break; }
                        if (curMax < maxRes2) break;
                    }
                }
            }
        }
        ++i0;
    }
    return cur;
}


struct FilterArgs {
    unsigned curFrame, startFrame;
    const KeyPoint* kp; const int* numMatches; const float* dists; const uint2* idxs;
    int* numFiltered; float* fDists; uint2* fIdxs; float* fT; float* fTinv;
    float Ki[16]; unsigned minNum; float maxRes2;
};

__global__ void __launch_bounds__(32)
sift_filter_kernel(const __grid_constant__ FilterArgs a) {
    const unsigned p = blockIdx.x + a.startFrame, t = threadIdx.x;
    if (p == a.curFrame) return;
    const int raw = a.numMatches[p];
    if (raw <= 0) { if (t == 0) a.numFiltered[p] = 0; return; }                    // SIFTImageManager.cu:211-216
    const unsigned n = (unsigned)min(MAX_RAW, raw);
    __shared__ uint32_t sIdx[2 * MAX_RAW];
    __shared__ float sDist[MAX_RAW];
    __shared__ f3 sSrc[MAX_FILTERED], sTgt[MAX_FILTERED];
    __shared__ float sRes[MAX_FILTERED];
    __shared__ unsigned sCount;
    for (unsigned k = t; k < n; k += 32) { const uint2 v = a.idxs[(size_t)p * MAX_RAW + k]; sIdx[2 * k] = v.x; sIdx[2 * k + 1] = v.y; sDist[k] = a.dists[(size_t)p * MAX_RAW + k]; }
    __syncwarp();
    {
        float T[16], Ti[16];
        const unsigned cnt = filter_pair(a.kp, sIdx, sDist, n, T, a.Ki, a.minNum, a.maxRes2, sSrc, sTgt, sRes, t);      // the whole warp; T and the count are uniform
        if (t == 0) {
            sCount = cnt;
            mat4_inverse_hd(T, Ti);
            for (int k = 0; k < 16; ++k) { a.fT[16 * (size_t)p + k] = T[k]; a.fTinv[16 * (size_t)p + k] = Ti[k]; }
            a.numFiltered[p] = (int)cnt;
        }
    }
    __syncwarp();
    const unsigned c = sCount;
    if (t < MAX_FILTERED) {                                                        // :243-250
        const size_t o = (size_t)p * MAX_FILTERED + t;
        a.fDists[o] = (t < c) ? sDist[t] : 999.0f;
        a.fIdxs[o] = (t < c) ? make_uint2(sIdx[2 * t], sIdx[2 * t + 1]) : make_uint2(0xFFFFFFFFu, 0xFFFFFFFFu);
    }
}

struct AddArgs {
    unsigned curFrame, startFrame, numFrames;
    BFEntryJ* glob; uint2* globIdx; int* globNum; const int* numFiltered; const uint2* fIdxs; const KeyPoint* kp;
    const int* lastMatched;           // optional device predicate (bfSiftFilterFrames): nothing is appended when *lastMatched < 0
    float Ki[16];
};
// SIFTImageManager::filterFrames (FL/SiftGPU/SIFTImageManager.cpp:551-575) without its host round trip: the LAST frame i in
// [startFrame, numFrames), i != curFrame, that is valid and has filtered matches; the current frame is valid iff there is one
__global__ void __launch_bounds__(256)
sift_filter_frames_kernel(unsigned curFrame, unsigned startFrame, unsigned numFrames, const int* __restrict__ numFiltered, int* validImages, int* lastMatched) {
    __shared__ int sBest[256];
    int best = -1;
    for (unsigned i = startFrame + threadIdx.x; i < numFrames; i += blockDim.x)
        if (i != curFrame && validImages[i] != 0 && numFiltered[i] > 0) best = (int)i;       // strided ascending: the last hit of a thread is its largest
    sBest[threadIdx.x] = best;
    __syncthreads();
    for (unsigned off = 128; off > 0; off >>= 1) {
        if (threadIdx.x < off && sBest[threadIdx.x + off] > sBest[threadIdx.x]) sBest[threadIdx.x] = sBest[threadIdx.x + off];
        __syncthreads();
    }
    if (threadIdx.x == 0) { validImages[curFrame] = sBest[0] >= 0 ? 1 : 0; *lastMatched = sBest[0]; }
}

// AddCurrToResidualsCU_Kernel (SIFTImageManager.cu:610-655), one CTA: slots are handed out in ascending pair order
__global__ void __launch_bounds__(1024)
sift_add_residuals_kernel(const __grid_constant__ AddArgs a) {
    __shared__ int sBase;             // running base while pairs are walked in chunks of blockDim.x
    __shared__ int sScan[1024];
    const unsigned t = threadIdx.x;
    if (a.lastMatched && *a.lastMatched < 0) return;            // Bundler::matchAndFilter: `if (lastMatchedFrame != -1) AddCurrToResidualsCU(...)`
    if (t == 0) sBase = *a.globNum;
    __syncthreads();
    for (unsigned p0 = a.startFrame; p0 < a.numFrames; p0 += blockDim.x) {
        const unsigned p = p0 + t;
        int cnt = 0;
        if (p < a.numFrames && p != a.curFrame) cnt = a.numFiltered[p];
        sScan[t] = cnt;
        __syncthreads();
        for (unsigned o = 1; o < blockDim.x; o <<= 1) {                 // inclusive Hillis-Steele scan
            const int v = (t >= o) ? sScan[t - o] : 0;
            __syncthreads();
            sScan[t] += v;
            __syncthreads();
        }
        const int base = sBase + sScan[t] - cnt;
        for (int k = 0; k < cnt; ++k) {
            const uint2 ij = a.fIdxs[(size_t)p * MAX_FILTERED + k];
            BFEntryJ e;
            e.imgIdx_i = p; e.imgIdx_j = a.curFrame;
            for (int s2 = 0; s2 < 2; ++s2) {
                const KeyPoint kq = a.kp[s2 == 0 ? ij.x : ij.y];
                const float v0 = kq.depth * kq.px, v1 = kq.depth * kq.py, v2 = kq.depth * 1.0f;
                float* o = (s2 == 0) ? e.pos_i : e.pos_j;
                o[0] = a.Ki[0] * v0 + a.Ki[1] * v1 + a.Ki[2] * v2 + a.Ki[3];
                o[1] = a.Ki[4] * v0 + a.Ki[5] * v1 + a.Ki[6] * v2 + a.Ki[7];
                o[2] = a.Ki[8] * v0 + a.Ki[9] * v1 + a.Ki[10] * v2 + a.Ki[11];
            }
            a.glob[base + k] = e;
            a.globIdx[base + k] = ij;
        }
        __syncthreads();
        if (t == blockDim.x - 1) sBase += sScan[t];
        __syncthreads();
    }
    if (t == 0) *a.globNum = sBase;
}

}  // namespace bf

using namespace bf;

BF_API int bfSiftFilterFrames(unsigned int curFrame, unsigned int startFrame, unsigned int numFrames, const int32_t* d_currNumFilteredMatchesPerImagePair,
                              int32_t* d_validImages, int32_t* d_lastMatchedFrame) {
    if (!d_currNumFilteredMatchesPerImagePair || !d_validImages || !d_lastMatchedFrame || curFrame >= numFrames) return (int)cudaErrorInvalidValue;
    ++g_launchCount;
    sift_filter_frames_kernel<<<1, 256, 0, stream()>>>(curFrame, startFrame, numFrames, d_currNumFilteredMatchesPerImagePair, d_validImages, d_lastMatchedFrame);
    BF_CHECK(cudaGetLastError());
    return 0;
}

static int add_curr_to_residuals(unsigned int curFrame, unsigned int startFrame, unsigned int numFrames, BFEntryJ* d_globMatches,
                                 uint32_t* d_globMatchesKeyPointIndices, int32_t* d_globNumResiduals, const int32_t* d_currNumFilteredMatchesPerImagePair,
                                 const uint32_t* d_currFilteredMatchKeyPointIndices, const BFSIFTKeyPoint* d_keyPoints, const float* colorIntrinsicsInv,
                                 const int32_t* d_lastMatchedFrame) {
    if (numFrames <= startFrame) return 0;
    AddArgs a;
    a.lastMatched = d_lastMatchedFrame;
    a.curFrame = curFrame; a.startFrame = startFrame; a.numFrames = numFrames;
    a.glob = d_globMatches; a.globIdx = reinterpret_cast<uint2*>(d_globMatchesKeyPointIndices); a.globNum = d_globNumResiduals;
    a.numFiltered = d_currNumFilteredMatchesPerImagePair; a.fIdxs = reinterpret_cast<const uint2*>(d_currFilteredMatchKeyPointIndices);
    a.kp = reinterpret_cast<const KeyPoint*>(d_keyPoints);
    for (int k = 0; k < 16; ++k) a.Ki[k] = colorIntrinsicsInv[k];
    ++g_launchCount;
    sift_add_residuals_kernel<<<1, 1024, 0, stream()>>>(a);
    BF_CHECK(cudaGetLastError());
    return 0;
}

BF_API int bfSiftAddCurrToResiduals(unsigned int curFrame, unsigned int startFrame, unsigned int numFrames, BFEntryJ* d_globMatches,
                                    uint32_t* d_globMatchesKeyPointIndices, int32_t* d_globNumResiduals, const int32_t* d_currNumFilteredMatchesPerImagePair,
                                    const uint32_t* d_currFilteredMatchKeyPointIndices, const BFSIFTKeyPoint* d_keyPoints, const float* colorIntrinsicsInv) {
    return add_curr_to_residuals(curFrame, startFrame, numFrames, d_globMatches, d_globMatchesKeyPointIndices, d_globNumResiduals, d_currNumFilteredMatchesPerImagePair,
                                 d_currFilteredMatchKeyPointIndices, d_keyPoints, colorIntrinsicsInv, nullptr);
}

BF_API int bfSiftAddCurrToResidualsIfMatched(unsigned int curFrame, unsigned int startFrame, unsigned int numFrames, BFEntryJ* d_globMatches,
                                             uint32_t* d_globMatchesKeyPointIndices, int32_t* d_globNumResiduals, const int32_t* d_currNumFilteredMatchesPerImagePair,
                                             const uint32_t* d_currFilteredMatchKeyPointIndices, const BFSIFTKeyPoint* d_keyPoints, const float* colorIntrinsicsInv,
                                             const int32_t* d_lastMatchedFrame) {
    if (!d_lastMatchedFrame) return (int)cudaErrorInvalidValue;
    return add_curr_to_residuals(curFrame, startFrame, numFrames, d_globMatches, d_globMatchesKeyPointIndices, d_globNumResiduals, d_currNumFilteredMatchesPerImagePair,
                                 d_currFilteredMatchKeyPointIndices, d_keyPoints, colorIntrinsicsInv, d_lastMatchedFrame);
}

BF_API int bfSiftFilterKeyPointMatches(unsigned int curFrame, unsigned int startFrame, unsigned int numFrames, const BFSIFTKeyPoint* d_keyPoints,
                                       const int32_t* d_numMatchesPerImagePair, const float* d_matchDistances, const uint32_t* d_matchKeyPointIndices,
                                       int32_t* d_numFilteredMatchesPerImagePair, float* d_filteredMatchDistances, uint32_t* d_filteredMatchKeyPointIndices,
                                       float* d_filteredTransforms, float* d_filteredTransformsInv, const float* siftIntrinsicsInv,
                                       unsigned int minNumMatches, float maxKabschRes2) {
    if (numFrames <= startFrame) return 0;                                         // SIFTImageManager.cu:267
    FilterArgs a;
    a.curFrame = curFrame; a.startFrame = startFrame;
    a.kp = reinterpret_cast<const KeyPoint*>(d_keyPoints); a.numMatches = d_numMatchesPerImagePair; a.dists = d_matchDistances;
    a.idxs = reinterpret_cast<const uint2*>(d_matchKeyPointIndices);
    a.numFiltered = d_numFilteredMatchesPerImagePair; a.fDists = d_filteredMatchDistances; a.fIdxs = reinterpret_cast<uint2*>(d_filteredMatchKeyPointIndices);
    a.fT = d_filteredTransforms; a.fTinv = d_filteredTransformsInv;
    for (int k = 0; k < 16; ++k) a.Ki[k] = siftIntrinsicsInv[k];
    a.minNum = minNumMatches; a.maxRes2 = maxKabschRes2;
    ++g_launchCount;
    sift_filter_kernel<<<numFrames - startFrame, 32, 0, stream()>>>(a);
    BF_CHECK(cudaGetLastError());
    return 0;
}

/*
 * solver_oracle.c -- CPU restatement of the reference's sparse bundle-adjustment solver (GN + Jacobi-PCG in
 * Lie space), float32, single thread.
 *
 * TEST INFRASTRUCTURE ONLY (see tsdf_oracle.c header for the rules).  PARITY STATUS: the reference has no tests
 * or golden vectors for this path and needs a GPU to run, so in the authoring container this file is pinned only
 * by the known-answer tests in tests/test_solver_oracle.py (SE(3) exp/log identities, recovery of known poses
 * from exact correspondences, agreement with an independent float64 dense Gauss-Newton written in numpy,
 * finite-difference rows of the dense Jacobian) AND by tests/golden/solver_reference_ieee.npz: poses solved by the reference's
 * own SolverBundling.cu (oracle/_ref, run on a GPU by scripts/make_golden_from_reference.py) for a sparse 11-image problem and a
 * sparse + dense 5-image problem, which tests/test_golden_reference.py requires this oracle to reproduce within 1e-4 relative L2
 * (and the dense overlap count exactly).  On the GPU box it is additionally pinned against the reference live:
 * tests/test_solver_vs_reference_gpu.py runs the reference's own SolverBundling.cu / SBA.cu (oracle/_ref, built
 * by oracle/build_ref.py) on the same inputs and requires this oracle's poses within 1e-4 relative L2 of them
 * (measured 1e-6 .. 5e-5) and its dense (6N)^2 system within 1e-4 relative Frobenius.
 *
 * Restates, function by function (FL/ = FriedLiver/Source/):
 *   exp / log of SE(3)          FL/Solver/LieDerivUtil.h:19-207
 *   generators, Lie update      FL/Solver/LieDerivUtil.h:231-242, 301-307
 *   -J^T f + preconditioner     FL/Solver/SolverBundlingEquationsLie.h:63-148
 *   J p, J^T (J p)              FL/Solver/SolverBundlingEquationsLie.h:154-228
 *   PCG init / iteration        FL/Solver/SolverBundling.cu:756-794, 894-1108
 *   GN loop + early-outs        FL/Solver/SolverBundling.cu:1137-1220 (5e-7 on p.Ap, 0.005 on max|delta|)
 *   variable -> corr table      FL/Solver/SolverBundling.cu:1226-1248 (slots in ascending correspondence order)
 *   max residual                FL/Solver/SolverBundlingEquationsLie.h:27-40, SolverBundling.cu:511-550
 * Sums run in the order a sequential reading of those kernels gives (ascending variable / correspondence).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>

#include "../include/bf_solver.h"

#define ORC_API __attribute__((visibility("default")))
#define FLOAT_EPSILON 0.000001f       /* FL/SolverUtil.h:9 */
/* Decision trace (tests): every early-out decision of the last solve -- per PCG iteration (GN index, p.Ap), per evaluated GN
 * convergence test (-(GN index + 1), max|delta|).  The parity tests use it to certify that a problem's decisions sit clear of their
 * thresholds (5e-7, 1e-6, 0.005), i.e. that a last-bit difference in a float sum cannot send two implementations down different paths. */
static float* g_trace = 0; static unsigned g_traceCap = 0, g_traceN = 0;
ORC_API void orc_solver_set_trace(float* buf, unsigned capPairs) { g_trace = buf; g_traceCap = capPairs; g_traceN = 0; }
ORC_API unsigned orc_solver_trace_count(void) { return g_traceN; }
static void trace_put(float a, float b) { if (g_trace && g_traceN < g_traceCap) { g_trace[2 * g_traceN] = a; g_trace[2 * g_traceN + 1] = b; } if (g_trace) ++g_traceN; }

typedef struct { float x, y, z; } v3;
static inline v3 V(float x, float y, float z) { v3 r = { x, y, z }; return r; }
static inline v3 add(v3 a, v3 b) { return V(a.x + b.x, a.y + b.y, a.z + b.z); }
static inline v3 sub(v3 a, v3 b) { return V(a.x - b.x, a.y - b.y, a.z - b.z); }
static inline v3 mul(v3 a, float s) { return V(a.x * s, a.y * s, a.z * s); }
static inline v3 mulv(v3 a, v3 b) { return V(a.x * b.x, a.y * b.y, a.z * b.z); }
static inline float dot(v3 a, v3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
static inline v3 cross(v3 a, v3 b) { return V(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
static inline float length(v3 a) { return sqrtf(dot(a, a)); }
static inline v3 ld3(const float* p, unsigned i) { return V(p[3 * i], p[3 * i + 1], p[3 * i + 2]); }
static inline void st3(float* p, unsigned i, v3 v) { p[3 * i] = v.x; p[3 * i + 1] = v.y; p[3 * i + 2] = v.z; }
/* affine transform of a point, implicit w = 1 (cuda_SimpleMatrixUtil.h:937-944) */
static inline v3 xf(const float* m, v3 v) {
    return V(m[0] * v.x + m[1] * v.y + m[2] * v.z + m[3] * 1.0f, m[4] * v.x + m[5] * v.y + m[6] * v.z + m[7] * 1.0f,
             m[8] * v.x + m[9] * v.y + m[10] * v.z + m[11] * 1.0f);
}

/* LieDerivUtil.h:19-47 */
static void rodrigues(v3 w, float A, float B, float R[9]) {
    const float wx2 = w.x * w.x, wy2 = w.y * w.y, wz2 = w.z * w.z;
    R[0] = 1.0f - B * (wy2 + wz2); R[4] = 1.0f - B * (wx2 + wz2); R[8] = 1.0f - B * (wx2 + wy2);
    float a = A * w.z, b = B * (w.x * w.y); R[1] = b - a; R[3] = b + a;
    a = A * w.y; b = B * (w.x * w.z); R[2] = b + a; R[6] = b - a;
    a = A * w.x; b = B * (w.y * w.z); R[5] = b - a; R[7] = b + a;
}
/* LieDerivUtil.h:50-76 */
static void exp_rotation(v3 w, float R[9]) {
    const float theta_sq = dot(w, w), theta = sqrtf(theta_sq);
    float A, B;
    if (theta_sq < 1e-8) { A = 1.0f - 0.16666667f * theta_sq; B = 0.5f; }
    else if (theta_sq < 1e-6) { B = 0.5f - 0.25f * 0.16666667f * theta_sq; A = 1.0f - theta_sq * 0.16666667f * (1.0f - 0.05f * theta_sq); }
    else { const float inv = 1.0f / theta; A = sinf(theta) * inv; B = (1 - cosf(theta)) * (inv * inv); }
    rodrigues(w, A, B, R);
}
/* LieDerivUtil.h:79-133 */
static v3 ln_rotation(const float* M /* 4x4 row-major, uses the 3x3 part */) {
#define Rm(r, c) M[(r) * 4 + (c)]
    const float cos_angle = (Rm(0, 0) + Rm(1, 1) + Rm(2, 2) - 1.0f) * 0.5f;
    v3 result = V((Rm(2, 1) - Rm(1, 2)) * 0.5f, (Rm(0, 2) - Rm(2, 0)) * 0.5f, (Rm(1, 0) - Rm(0, 1)) * 0.5f);
    const float sin_angle_abs = length(result);
    if (cos_angle > 0.70710678118654752440f) {
        if (sin_angle_abs > 0) result = mul(result, asinf(sin_angle_abs) / sin_angle_abs);
    } else if (cos_angle > -0.70710678118654752440f) {
        const float angle = acosf(cos_angle);
        result = mul(result, angle / sin_angle_abs);
    } else {
        const float angle = 3.14159265358979323846f - asinf(sin_angle_abs);
        const float d0 = Rm(0, 0) - cos_angle, d1 = Rm(1, 1) - cos_angle, d2 = Rm(2, 2) - cos_angle;
        v3 r2;
        if (fabsf(d0) > fabsf(d1) && fabsf(d0) > fabsf(d2)) r2 = V(d0, (Rm(1, 0) + Rm(0, 1)) * 0.5f, (Rm(0, 2) + Rm(2, 0)) * 0.5f);
        else if (fabsf(d1) > fabsf(d2)) r2 = V((Rm(1, 0) + Rm(0, 1)) * 0.5f, d1, (Rm(2, 1) + Rm(1, 2)) * 0.5f);
        else r2 = V((Rm(0, 2) + Rm(2, 0)) * 0.5f, (Rm(2, 1) + Rm(1, 2)) * 0.5f, d2);
        if (dot(r2, result) < 0) r2 = mul(r2, -1.0f);
        result = mul(r2, angle / length(r2));
    }
#undef Rm
    return result;
}
/* LieDerivUtil.h:160-207 */
ORC_API void orc_pose_to_matrix(const float rot3[3], const float trans3[3], float M[16]) {
    const v3 rot = V(rot3[0], rot3[1], rot3[2]), trans = V(trans3[0], trans3[1], trans3[2]);
    const float theta_sq = dot(rot, rot), theta = sqrtf(theta_sq);
    float A, B;
    v3 translation;
    const v3 cr = cross(rot, trans);
    if (theta_sq < 1e-8) {
        A = 1.0f - 0.16666667f * theta_sq; B = 0.5f;
        translation = add(trans, mul(cr, 0.5f));
    } else {
        float C;
        if (theta_sq < 1e-6) { C = 0.16666667f * (1.0f - 0.05f * theta_sq); A = 1.0f - theta_sq * C; B = 0.5f - 0.25f * 0.16666667f * theta_sq; }
        else { const float inv = 1.0f / theta; A = sinf(theta) * inv; B = (1 - cosf(theta)) * (inv * inv); C = (1 - A) * (inv * inv); }
        const v3 wc = cross(rot, cr);
        translation = add(add(trans, mul(cr, B)), mul(wc, C));
    }
    float R[9];
    rodrigues(rot, A, B, R);
    M[0] = R[0]; M[1] = R[1]; M[2] = R[2]; M[3] = translation.x;
    M[4] = R[3]; M[5] = R[4]; M[6] = R[5]; M[7] = translation.y;
    M[8] = R[6]; M[9] = R[7]; M[10] = R[8]; M[11] = translation.z;
    M[12] = 0; M[13] = 0; M[14] = 0; M[15] = 1;
}
/* LieDerivUtil.h:135-158 */
ORC_API void orc_matrix_to_pose(const float M[16], float rot3[3], float trans3[3]) {
    const v3 t = V(M[3], M[7], M[11]);
    v3 rot = ln_rotation(M);
    const float theta = length(rot);
    float shtot = 0.5f;
    if (theta > 0.00001f) shtot = sinf(theta * 0.5f) / theta;
    float H[9];
    exp_rotation(mul(rot, -0.5f), H);
    v3 trans = V(H[0] * t.x + H[1] * t.y + H[2] * t.z, H[3] * t.x + H[4] * t.y + H[5] * t.z, H[6] * t.x + H[7] * t.y + H[8] * t.z);
    if (theta > 0.001f) trans = sub(trans, mul(rot, dot(t, rot) * (1 - 2 * shtot) / dot(rot, rot)));
    else trans = sub(trans, mul(rot, dot(t, rot) / 24));
    trans = mul(trans, 1.0f / (2 * shtot));
    rot3[0] = rot.x; rot3[1] = rot.y; rot3[2] = rot.z;
    trans3[0] = trans.x; trans3[1] = trans.y; trans3[2] = trans.z;
}
static void mat4_mul(const float* a, const float* b, float* o) {
    for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c)
        o[r * 4 + c] = a[r * 4] * b[c] + a[r * 4 + 1] * b[4 + c] + a[r * 4 + 2] * b[8 + c] + a[r * 4 + 3] * b[12 + c];
}
/* general fp32 4x4 inverse (cuda_SimpleMatrixUtil.h:980-1100), adjugate / determinant */
ORC_API void orc_mat4_inverse(const float* m, float* out) {
    float inv[16];
    inv[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
    inv[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
    inv[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
    inv[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
    inv[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
    inv[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
    inv[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
    inv[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
    inv[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
    inv[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
    inv[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
    inv[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
    inv[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
    inv[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
    inv[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
    inv[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
    const float det = m[0] * inv[0] + m[1] * inv[4] + m[2] * inv[8] + m[3] * inv[12];
    const float r = 1.0f / det;
    for (int i = 0; i < 16; ++i) out[i] = inv[i] * r;
}

/* host-side view of the solver buffers (all HOST pointers here) */
typedef struct OrcSolver {
    unsigned N, C, maxCorrPerImage;
    BFEntryJ* corr;                 /* [C] (may be invalidated by the table build) */
    int* varToCorr;                 /* [N * maxCorrPerImage] */
    int* numEntriesPerRow;          /* [N] */
    float *xRot, *xTrans;           /* [N][3] unknowns */
    float *deltaRot, *deltaTrans, *rRot, *rTrans, *zRot, *zTrans, *pRot, *pTrans, *ApRot, *ApTrans, *precRot, *precTrans;
    float* Jp;                      /* [C][3] */
    float* T;                       /* [N][16] */
    float* Tinv;                    /* [N][16] */
    float* rDotzOld;                /* [N] */
} OrcSolver;

static inline int corr_valid(const BFEntryJ* c) { return c->imgIdx_i != 0xFFFFFFFFu; }

/* SolverBundling.cu:1226-1248 */
ORC_API void orc_solver_build_table(BFEntryJ* corr, unsigned C, unsigned maxCorrPerImage, int* varToCorr, int* numEntriesPerRow, unsigned N) {
    memset(numEntriesPerRow, 0, sizeof(int) * N);
    /* When only ONE of the two rows overflows, the reference leaves the other row's slot unwritten (it then holds whatever
     * the buffer held: -1 from the constructor's memset, i.e. an out-of-bounds read).  The oracle marks such slots -1 and
     * skips them -- the defined behaviour closest to the intent ("invalidate"). */
    memset(varToCorr, 0xff, sizeof(int) * (size_t)N * maxCorrPerImage);
    for (unsigned x = 0; x < C; ++x) {
        BFEntryJ* c = &corr[x];
        if (!corr_valid(c)) continue;
        int o0 = numEntriesPerRow[c->imgIdx_i]++;
        int o1 = numEntriesPerRow[c->imgIdx_j]++;
        if ((unsigned)o0 < maxCorrPerImage && (unsigned)o1 < maxCorrPerImage) {
            varToCorr[c->imgIdx_i * maxCorrPerImage + o0] = (int)x;
            varToCorr[c->imgIdx_j * maxCorrPerImage + o1] = (int)x;
        } else {
            c->imgIdx_i = 0xFFFFFFFFu; c->imgIdx_j = 0xFFFFFFFFu;
        }
    }
}

/* SolverBundlingEquationsLie.h:63-148 (sparse part) */
static void eval_minus_jtf(OrcSolver* s, unsigned v, float wSparse, v3* resRot, v3* resTrans) {
    v3 rRot = V(0, 0, 0), rTrans = V(0, 0, 0), pRot = V(0, 0, 0), pTrans = V(0, 0, 0);
    st3(s->deltaRot, v, V(0, 0, 0)); st3(s->deltaTrans, v, V(0, 0, 0));
    int n = s->numEntriesPerRow[v];
    if ((unsigned)n > s->maxCorrPerImage) n = (int)s->maxCorrPerImage;
    for (int k = 0; k < n; ++k) {
        const int ci0 = s->varToCorr[v * s->maxCorrPerImage + k];
        if (ci0 < 0) continue;
        const BFEntryJ* c = &s->corr[ci0];
        if (!corr_valid(c)) continue;
        const float* TI = &s->T[16 * c->imgIdx_i];
        const float* TJ = &s->T[16 * c->imgIdx_j];
        const v3 pi = V(c->pos_i[0], c->pos_i[1], c->pos_i[2]), pj = V(c->pos_j[0], c->pos_j[1], c->pos_j[2]);
        v3 wp; float sign = 1;
        if (v != c->imgIdx_i) { sign = -1; wp = xf(TJ, pj); } else wp = xf(TI, pi);
        const v3 da = V(0.0f, -wp.z, wp.y), db = V(wp.z, 0.0f, -wp.x), dc = V(-wp.y, wp.x, 0.0f);
        const v3 r = sub(xf(TI, pi), xf(TJ, pj));
        rRot = add(rRot, mul(V(dot(da, r), dot(db, r), dot(dc, r)), sign));
        rTrans = add(rTrans, mul(r, sign));
        pRot = add(pRot, V(dot(da, da), dot(db, db), dot(dc, dc)));
        pTrans = add(pTrans, V(1.0f, 1.0f, 1.0f));
    }
    *resRot = mul(rRot, -wSparse);
    *resTrans = mul(rTrans, -wSparse);
    st3(s->precRot, v, V(pRot.x > FLOAT_EPSILON ? 1.0f / pRot.x : 1.0f, pRot.y > FLOAT_EPSILON ? 1.0f / pRot.y : 1.0f, pRot.z > FLOAT_EPSILON ? 1.0f / pRot.z : 1.0f));
    st3(s->precTrans, v, V(pTrans.x > FLOAT_EPSILON ? 1.0f / pTrans.x : 1.0f, pTrans.y > FLOAT_EPSILON ? 1.0f / pTrans.y : 1.0f, pTrans.z > FLOAT_EPSILON ? 1.0f / pTrans.z : 1.0f));
}

/* SolverBundlingEquationsLie.h:195-228 */
static v3 apply_j(const OrcSolver* s, unsigned ci, float wSparse) {
    v3 b = V(0, 0, 0);
    const BFEntryJ* c = &s->corr[ci];
    if (!corr_valid(c)) return b;
    if (c->imgIdx_i > 0) {
        const v3 wp = xf(&s->T[16 * c->imgIdx_i], V(c->pos_i[0], c->pos_i[1], c->pos_i[2]));
        const v3 da = V(0.0f, -wp.z, wp.y), db = V(wp.z, 0.0f, -wp.x), dc = V(-wp.y, wp.x, 0.0f);
        const v3 pp = ld3(s->pRot, c->imgIdx_i);
        b = add(b, add(add(add(mul(da, pp.x), mul(db, pp.y)), mul(dc, pp.z)), ld3(s->pTrans, c->imgIdx_i)));
    }
    if (c->imgIdx_j > 0) {
        const v3 wp = xf(&s->T[16 * c->imgIdx_j], V(c->pos_j[0], c->pos_j[1], c->pos_j[2]));
        const v3 da = V(0.0f, -wp.z, wp.y), db = V(wp.z, 0.0f, -wp.x), dc = V(-wp.y, wp.x, 0.0f);
        const v3 pp = ld3(s->pRot, c->imgIdx_j);
        b = sub(b, add(add(add(mul(da, pp.x), mul(db, pp.y)), mul(dc, pp.z)), ld3(s->pTrans, c->imgIdx_j)));
    }
    return mul(b, wSparse);
}

/* SolverBundlingEquationsLie.h:154-193 */
static void apply_jt(const OrcSolver* s, unsigned v, v3* outRot, v3* outTrans) {
    v3 oR = V(0, 0, 0), oT = V(0, 0, 0);
    int n = s->numEntriesPerRow[v];
    if ((unsigned)n > s->maxCorrPerImage) n = (int)s->maxCorrPerImage;
    for (int k = 0; k < n; ++k) {
        const int ci = s->varToCorr[v * s->maxCorrPerImage + k];
        if (ci < 0) continue;
        const BFEntryJ* c = &s->corr[ci];
        if (!corr_valid(c)) continue;
        v3 wp; float sign = 1;
        if (v != c->imgIdx_i) { sign = -1; wp = xf(&s->T[16 * c->imgIdx_j], V(c->pos_j[0], c->pos_j[1], c->pos_j[2])); }
        else wp = xf(&s->T[16 * c->imgIdx_i], V(c->pos_i[0], c->pos_i[1], c->pos_i[2]));
        const v3 da = V(0.0f, -wp.z, wp.y), db = V(wp.z, 0.0f, -wp.x), dc = V(-wp.y, wp.x, 0.0f);
        const v3 jp = ld3(s->Jp, (unsigned)ci);
        oR = add(oR, mul(V(dot(da, jp), dot(db, jp), dot(dc, jp)), sign));
        oT = add(oT, mul(jp, sign));
    }
    *outRot = oR; *outTrans = oT;
}

/* Runs the whole solveBundlingStub for the SPARSE term (weightsDense* must be 0).
 * xRot / xTrans: in/out unknowns [N][3].  stats[0]=GN iterations, stats[1]=total PCG iterations.
 * Returns 0, or -1 on allocation failure. */
ORC_API int orc_solver_solve_sparse(BFEntryJ* corr, unsigned C, unsigned N, unsigned maxCorrPerImage,
                                    float* xRot, float* xTrans, unsigned nNonLinear, unsigned nLinear,
                                    const float* weightsSparse, int rebuildTable, int* varToCorr, int* numEntriesPerRow,
                                    unsigned stats[4]) {
    OrcSolver s;
    memset(&s, 0, sizeof s);
    s.N = N; s.C = C; s.maxCorrPerImage = maxCorrPerImage; s.corr = corr; s.varToCorr = varToCorr; s.numEntriesPerRow = numEntriesPerRow;
    s.xRot = xRot; s.xTrans = xTrans;
    float* buf = (float*)calloc((size_t)N * (3 * 12 + 32 + 1) + (size_t)C * 3 + 16, sizeof(float));
    if (!buf) return -1;
    float* p = buf;
    s.deltaRot = p; p += 3 * N; s.deltaTrans = p; p += 3 * N; s.rRot = p; p += 3 * N; s.rTrans = p; p += 3 * N;
    s.zRot = p; p += 3 * N; s.zTrans = p; p += 3 * N; s.pRot = p; p += 3 * N; s.pTrans = p; p += 3 * N;
    s.ApRot = p; p += 3 * N; s.ApTrans = p; p += 3 * N; s.precRot = p; p += 3 * N; s.precTrans = p; p += 3 * N;
    s.T = p; p += 16 * N; s.Tinv = p; p += 16 * N; s.rDotzOld = p; p += N; s.Jp = p;
    if (rebuildTable) orc_solver_build_table(corr, C, maxCorrPerImage, varToCorr, numEntriesPerRow, N);
    unsigned totalPcg = 0, gnRun = 0;
    for (unsigned nIter = 0; nIter < nNonLinear; ++nIter) {
        const float wS = weightsSparse[nIter];
        ++gnRun;
        for (unsigned k = 0; k < N; ++k) { orc_pose_to_matrix(&xRot[3 * k], &xTrans[3 * k], &s.T[16 * k]); orc_mat4_inverse(&s.T[16 * k], &s.Tinv[16 * k]); }
        /* Initialization (:756-794) */
        float scanAlpha0 = 0.0f, scanAlpha1 = 0.0f;
        for (unsigned x = 1; x < N; ++x) {
            v3 resRot, resTrans;
            eval_minus_jtf(&s, x, wS, &resRot, &resTrans);
            st3(s.rRot, x, resRot); st3(s.rTrans, x, resTrans);
            const v3 pR = mulv(ld3(s.precRot, x), resRot), pT = mulv(ld3(s.precTrans, x), resTrans);
            st3(s.pRot, x, pR); st3(s.pTrans, x, pT);
            scanAlpha0 += dot(resRot, pR) + dot(resTrans, pT);
            st3(s.ApRot, x, V(0, 0, 0)); st3(s.ApTrans, x, V(0, 0, 0));
        }
        for (unsigned x = 1; x < N; ++x) s.rDotzOld[x] = scanAlpha0;
        /* PCG (:1024-1108) */
        for (unsigned lin = 0; lin < nLinear; ++lin) {
            int last = (lin == nLinear - 1);
            ++totalPcg;
            scanAlpha0 = 0.0f; scanAlpha1 = 0.0f;
            for (unsigned c = 0; c < C; ++c) st3(s.Jp, c, apply_j(&s, c, wS));
            for (unsigned x = 1; x < N; ++x) {
                v3 r, t; apply_jt(&s, x, &r, &t);
                st3(s.ApRot, x, add(ld3(s.ApRot, x), r)); st3(s.ApTrans, x, add(ld3(s.ApTrans, x), t));
            }
            for (unsigned x = 1; x < N; ++x) scanAlpha0 += dot(ld3(s.pRot, x), ld3(s.ApRot, x)) + dot(ld3(s.pTrans, x), ld3(s.ApTrans, x));
            const float dotProduct = scanAlpha0;
            for (unsigned x = 1; x < N; ++x) {
                float alpha = 0.0f;
                if (dotProduct > FLOAT_EPSILON) alpha = s.rDotzOld[x] / dotProduct;
                st3(s.deltaRot, x, add(ld3(s.deltaRot, x), mul(ld3(s.pRot, x), alpha)));
                st3(s.deltaTrans, x, add(ld3(s.deltaTrans, x), mul(ld3(s.pTrans, x), alpha)));
                const v3 rR = sub(ld3(s.rRot, x), mul(ld3(s.ApRot, x), alpha)), rT = sub(ld3(s.rTrans, x), mul(ld3(s.ApTrans, x), alpha));
                st3(s.rRot, x, rR); st3(s.rTrans, x, rT);
                const v3 zR = mulv(ld3(s.precRot, x), rR), zT = mulv(ld3(s.precTrans, x), rT);
                st3(s.zRot, x, zR); st3(s.zTrans, x, zT);
                scanAlpha1 += dot(zR, rR) + dot(zT, rT);
            }
            if (getenv("ORC_DEBUG")) fprintf(stderr, "gn %u pcg %u pAp %.6e rz_old %.6e rz_new %.6e\n", nIter, lin, scanAlpha0, s.rDotzOld[1], scanAlpha1);
            trace_put((float)nIter, scanAlpha0);
            if (fabsf(scanAlpha0) < 5e-7f) last = 1;
            for (unsigned x = 1; x < N; ++x) {
                const float rDotzNew = scanAlpha1, rDotzOld = s.rDotzOld[x];
                float beta = 0.0f;
                if (rDotzOld > FLOAT_EPSILON) beta = rDotzNew / rDotzOld;
                s.rDotzOld[x] = rDotzNew;
                st3(s.pRot, x, add(ld3(s.zRot, x), mul(ld3(s.pRot, x), beta)));
                st3(s.pTrans, x, add(ld3(s.zTrans, x), mul(ld3(s.pTrans, x), beta)));
                st3(s.ApRot, x, V(0, 0, 0)); st3(s.ApTrans, x, V(0, 0, 0));
                if (last) {   /* computeLieUpdate, LieDerivUtil.h:301-307 */
                    float U[16], Cm[16], P[16];
                    orc_pose_to_matrix(&s.deltaRot[3 * x], &s.deltaTrans[3 * x], U);
                    orc_pose_to_matrix(&xRot[3 * x], &xTrans[3 * x], Cm);
                    mat4_mul(U, Cm, P);
                    orc_matrix_to_pose(P, &xRot[3 * x], &xTrans[3 * x]);
                }
            }
            if (last) break;
        }
        /* EvalGNConvergence (:694-749): max |delta| over variables > 0 (all images treated as valid here) */
        if (nIter < nNonLinear - 1) {
            float m = 0.0f;
            for (unsigned x = 1; x < N; ++x) for (int k = 0; k < 3; ++k) {
                m = fmaxf(m, fabsf(s.deltaRot[3 * x + k])); m = fmaxf(m, fabsf(s.deltaTrans[3 * x + k]));
            }
            trace_put(-(float)(nIter + 1), m);
            if (m < 0.005f) break;
        }
    }
    if (stats) { stats[0] = gnRun; stats[1] = totalPcg; }
    free(buf);
    return 0;
}

/* evalAbsMaxResidualDevice over all correspondences (SolverBundlingEquationsLie.h:27-40; SolverBundling.cu:511-550 +
 * CUDASolverBundling.cpp:313-329): returns the maximum and writes its correspondence index */
ORC_API float orc_solver_max_residual(const BFEntryJ* corr, unsigned C, const float* xRot, const float* xTrans, float wSparse, int* outIndex) {
    float best = 0.0f; int bi = 0;
    for (unsigned x = 0; x < C; ++x) {
        const BFEntryJ* c = &corr[x];
        if (!corr_valid(c)) continue;
        float TI[16], TJ[16];
        orc_pose_to_matrix(&xRot[3 * c->imgIdx_i], &xTrans[3 * c->imgIdx_i], TI);
        orc_pose_to_matrix(&xRot[3 * c->imgIdx_j], &xTrans[3 * c->imgIdx_j], TJ);
        const v3 d = sub(xf(TI, V(c->pos_i[0], c->pos_i[1], c->pos_i[2])), xf(TJ, V(c->pos_j[0], c->pos_j[1], c->pos_j[2])));
        const float r = fmaxf(wSparse * fabsf(d.z), fmaxf(wSparse * fabsf(d.x), wSparse * fabsf(d.y)));
        if (best < r) { best = r; bi = (int)x; }
    }
    if (outIndex) *outIndex = bi;
    return best;
}

/* sum of squared sparse residuals (evalFDevice, SolverBundlingEquationsLie.h:42-57) -- the GN energy */
ORC_API double orc_solver_energy(const BFEntryJ* corr, unsigned C, const float* xRot, const float* xTrans, float wSparse) {
    double e = 0.0;
    for (unsigned x = 0; x < C; ++x) {
        const BFEntryJ* c = &corr[x];
        if (!corr_valid(c)) continue;
        float TI[16], TJ[16];
        orc_pose_to_matrix(&xRot[3 * c->imgIdx_i], &xTrans[3 * c->imgIdx_i], TI);
        orc_pose_to_matrix(&xRot[3 * c->imgIdx_j], &xTrans[3 * c->imgIdx_j], TJ);
        const v3 d = sub(xf(TI, V(c->pos_i[0], c->pos_i[1], c->pos_i[2])), xf(TJ, V(c->pos_j[0], c->pos_j[1], c->pos_j[2])));
        e += (double)(wSparse * dot(d, d));
    }
    return e;
}

/* ======================================================================================================================
 * Dense depth / colour term (SURVEY.md section 8 row a13) and the full solveBundlingStub with it.
 *   FindImageImageCorr / FindDenseCorrespondences / Weight / BuildDenseSystem / FlipJtJ   FL/Solver/SolverBundling.cu:30-471
 *   findDenseCorr (3 of the 5 overloads are live), addToLocalSystem, applyJTJDenseDevice   FL/Solver/SolverBundlingDenseUtil.h:22-411
 *   evalLie_derivI / evalLie_derivJ                                                        FL/Solver/LieDerivUtil.h:247-295
 *   Jacobian rows (depth, intensity)                                                       FL/Solver/SolverBundlingEquationsLie.h:234-277
 *   bilinear lookups, dCameraToScreen                                                      FL/Solver/ICPUtil.h:14-110
 * Dense unknown order per image is [tx ty tz | wx wy wz] (translation first).  Image pairs are visited in ascending (i, j)
 * order and pixels in ascending index order (the reference's atomics fix no order).
 * ====================================================================================================================== */
typedef struct OrcCacheFrame {      /* host mirror of CUDACachedFrame (FL/CUDACacheUtil.h:41-53) */
    const float* depth; const float* campos; const float* intensity; const float* intensityDerivs; const uint8_t* normalsU; const float* normals;
} OrcCacheFrame;

typedef struct OrcDenseParams {
    unsigned W, H;
    float fx, fy, mx, my;
    float distThresh, normalThresh, colorThresh, colorGradientMin, depthMin, depthMax;
    unsigned subsample; int usePairwise;
} OrcDenseParams;

static const float MINF_ = -INFINITY;
static inline v3 rot3(const float* m, v3 v) { return V(m[0] * v.x + m[1] * v.y + m[2] * v.z, m[4] * v.x + m[5] * v.y + m[6] * v.z, m[8] * v.x + m[9] * v.y + m[10] * v.z); }
static inline void cam_to_depth(const OrcDenseParams* d, v3 p, float* sx, float* sy) { *sx = p.x * d->fx / p.z + d->mx; *sy = p.y * d->fy / p.z + d->my; }
static inline v3 depth_to_cam(const OrcDenseParams* d, int x, int y, float depth) {
    const float fx = ((float)x - d->mx) / d->fx, fy = ((float)y - d->my) / d->fy;
    return V(depth * fx, depth * fy, depth);
}
static inline int f2i_c(float v) { if (v != v) return 0; if (v >= 2147483648.0f) return INT32_MAX; if (v <= -2147483648.0f) return INT32_MIN; return (int)v; }

/* ICPUtil.h:56-110: bilinear lookup with MINF-aware renormalisation; nc = number of channels (1, 2 or 4), validity on channel 0 */
static int bilinear(const float* img, int nc, float x, float y, unsigned W, unsigned H, float* out) {
    const int x0 = f2i_c(floorf(x)), y0 = f2i_c(floorf(y));
    const float alpha = x - (float)x0, beta = y - (float)y0;
    float s0[4] = { 0, 0, 0, 0 }, s1[4] = { 0, 0, 0, 0 }, w0 = 0, w1 = 0;
    const int xs[2] = { x0, x0 + 1 };
    for (int k = 0; k < 2; ++k) {
        const float wgt = k ? alpha : (1.0f - alpha);
        if ((unsigned)xs[k] < W && (unsigned)y0 < H) { const float* v = &img[((size_t)y0 * W + xs[k]) * nc]; if (v[0] != MINF_) { for (int c = 0; c < nc; ++c) s0[c] += wgt * v[c]; w0 += wgt; } }
        if ((unsigned)xs[k] < W && (unsigned)(y0 + 1) < H) { const float* v = &img[((size_t)(y0 + 1) * W + xs[k]) * nc]; if (v[0] != MINF_) { for (int c = 0; c < nc; ++c) s1[c] += wgt * v[c]; w1 += wgt; } }
    }
    float ss[4] = { 0, 0, 0, 0 }, ww = 0;
    if (w0 > 0.0f) { for (int c = 0; c < nc; ++c) ss[c] += (1.0f - beta) * (s0[c] / w0); ww += (1.0f - beta); }
    if (w1 > 0.0f) { for (int c = 0; c < nc; ++c) ss[c] += beta * (s1[c] / w1); ww += beta; }
    if (ww > 0.0f) { for (int c = 0; c < nc; ++c) out[c] = ss[c] / ww; return 1; }
    for (int c = 0; c < nc; ++c) out[c] = MINF_;
    return 0;
}

/* SolverBundlingDenseUtil.h:22-42 (overlap pre-filter, depth maps, no normals) */
static int find_corr_prefilter(const OrcDenseParams* d, unsigned idx, const float* transform, const float* tgtDepth, const float* srcDepth) {
    const unsigned x = idx % d->W, y = idx / d->W;
    const v3 cposj = depth_to_cam(d, (int)x, (int)y, srcDepth[idx]);
    if (!(cposj.z > d->depthMin && cposj.z < d->depthMax)) return 0;
    const v3 s2t = xf(transform, cposj);
    float sx, sy; cam_to_depth(d, s2t, &sx, &sy);
    const int tx = f2i_c(roundf(sx)), ty = f2i_c(roundf(sy));
    if (!(tx >= 0 && ty >= 0 && tx < (int)d->W && ty < (int)d->H)) return 0;
    const v3 ct = depth_to_cam(d, tx, ty, tgtDepth[ty * d->W + tx]);
    if (!(ct.z > d->depthMin && ct.z < d->depthMax)) return 0;
    return length(sub(s2t, ct)) <= d->distThresh;
}
/* SolverBundlingDenseUtil.h:152-184 (counting pass: depth maps + uchar4 normals) */
static int find_corr_count(const OrcDenseParams* d, unsigned idx, const float* transform, const OrcCacheFrame* tgt, const OrcCacheFrame* src) {
    const unsigned x = idx % d->W, y = idx / d->W;
    const v3 cposj = depth_to_cam(d, (int)x, (int)y, src->depth[idx]);
    if (!(cposj.z > d->depthMin && cposj.z < d->depthMax)) return 0;
    const uint8_t* nu = &src->normalsU[4 * idx];
    if (nu[0] == 0 && nu[1] == 0 && nu[2] == 0 && nu[3] == 0) return 0;
    v3 nrmj = V((float)nu[0] / 255.0f * 2.0f - 1.0f, (float)nu[1] / 255.0f * 2.0f - 1.0f, (float)nu[2] / 255.0f * 2.0f - 1.0f);
    nrmj = rot3(transform, nrmj);
    const v3 s2t = xf(transform, cposj);
    float sx, sy; cam_to_depth(d, s2t, &sx, &sy);
    const int tx = f2i_c(roundf(sx)), ty = f2i_c(roundf(sy));
    if (!(tx >= 0 && ty >= 0 && tx < (int)d->W && ty < (int)d->H)) return 0;
    const v3 ct = depth_to_cam(d, tx, ty, tgt->depth[ty * d->W + tx]);
    if (!(ct.z > d->depthMin && ct.z < d->depthMax)) return 0;
    const uint8_t* tu = &tgt->normalsU[4 * (ty * d->W + tx)];
    if (tu[0] == 0 && tu[1] == 0 && tu[2] == 0 && tu[3] == 0) return 0;
    const v3 nt = V((float)tu[0] / 255.0f * 2.0f - 1.0f, (float)tu[1] / 255.0f * 2.0f - 1.0f, (float)tu[2] / 255.0f * 2.0f - 1.0f);
    return dot(nrmj, nt) >= d->normalThresh && length(sub(s2t, ct)) <= d->distThresh;
}
/* SolverBundlingDenseUtil.h:79-113 (build pass: camera positions + float4 normals, bilinear target lookups) */
static int find_corr_build(const OrcDenseParams* d, unsigned idx, const float* transform, const OrcCacheFrame* tgt, const OrcCacheFrame* src,
                           v3* camPosSrc, v3* s2t, float* sx, float* sy, v3* camPosTgt, v3* normalTgt) {
    const float* cp = &src->campos[4 * idx];
    if (!(cp[2] > d->depthMin && cp[2] < d->depthMax)) return 0;
    *camPosSrc = V(cp[0], cp[1], cp[2]);
    const float* nj = &src->normals[4 * idx];
    if (nj[0] == MINF_) return 0;
    /* float4x4 * float4 (cuda_SimpleMatrixUtil.h:925-933), w of a normal is 0 */
    const float n4[4] = { transform[0] * nj[0] + transform[1] * nj[1] + transform[2] * nj[2] + transform[3] * nj[3],
                          transform[4] * nj[0] + transform[5] * nj[1] + transform[6] * nj[2] + transform[7] * nj[3],
                          transform[8] * nj[0] + transform[9] * nj[1] + transform[10] * nj[2] + transform[11] * nj[3],
                          transform[12] * nj[0] + transform[13] * nj[1] + transform[14] * nj[2] + transform[15] * nj[3] };
    *s2t = xf(transform, *camPosSrc);
    cam_to_depth(d, *s2t, sx, sy);
    const int tx = f2i_c(roundf(*sx)), ty = f2i_c(roundf(*sy));
    if (!(tx >= 0 && ty >= 0 && tx < (int)d->W && ty < (int)d->H)) return 0;
    float ci[4];
    bilinear(tgt->campos, 4, *sx, *sy, d->W, d->H, ci);
    if (!(ci[2] > d->depthMin && ci[2] < d->depthMax)) return 0;
    *camPosTgt = V(ci[0], ci[1], ci[2]);
    float ni[4];
    bilinear(tgt->normals, 4, *sx, *sy, d->W, d->H, ni);
    if (ni[0] == MINF_) return 0;
    *normalTgt = V(ni[0], ni[1], ni[2]);
    const float dist = length(sub(*s2t, *camPosTgt));
    const float dNormal = n4[0] * ni[0] + n4[1] * ni[1] + n4[2] * ni[2] + n4[3] * ni[3];
    return dNormal >= d->normalThresh && dist <= d->distThresh;
}

/* LieDerivUtil.h:247-272 : 3x6 Jacobian of (A exp(e) D)^-1 p  w.r.t. e, columns [t | w] */
static void lie_deriv_i(const float* A, const float* D, v3 p, float jac[18]) {
    float T[16]; mat4_mul(A, D, T);
    const v3 pt = sub(p, V(T[3], T[7], T[11]));
    float j0[3][12], j1[12][6];
    memset(j0, 0, sizeof j0); memset(j1, 0, sizeof j1);
    j0[0][0] = pt.x; j0[0][1] = pt.y; j0[0][2] = pt.z; j0[1][3] = pt.x; j0[1][4] = pt.y; j0[1][5] = pt.z; j0[2][6] = pt.x; j0[2][7] = pt.y; j0[2][8] = pt.z;
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { j0[r][c + 9] = -T[c * 4 + r]; j1[r + 9][c] = A[r * 4 + c]; }
    for (int k = 0; k < 4; ++k) {
        const v3 dcol = V(D[0 * 4 + k], D[1 * 4 + k], D[2 * 4 + k]);
        /* m = RA * skew(dcol) * -1 ; skew(v) = [[0,-z,y],[z,0,-x],[-y,x,0]] */
        const float S[9] = { 0, -dcol.z, dcol.y, dcol.z, 0, -dcol.x, -dcol.y, dcol.x, 0 };
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) {
            const float m = (A[r * 4 + 0] * S[0 * 3 + c] + A[r * 4 + 1] * S[1 * 3 + c] + A[r * 4 + 2] * S[2 * 3 + c]) * -1.0f;
            j1[3 * k + r][3 + c] = m;
        }
    }
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 6; ++c) { float s = 0; for (int k = 0; k < 12; ++k) s += j0[r][k] * j1[k][c]; jac[r * 6 + c] = s; }
}
/* LieDerivUtil.h:277-295 : 3x6 Jacobian of (A exp(e) D) p */
static void lie_deriv_j(const float* A, const float* D, v3 p, float jac[18]) {
    const v3 dr1 = V(D[0], D[1], D[2]), dr2 = V(D[4], D[5], D[6]), dr3 = V(D[8], D[9], D[10]);
    const float dtx = D[3], dty = D[7], dtz = D[11];
    float J[3][6] = { { 1, 0, 0, 0.0f, dot(p, dr3) + dtz, -(dot(p, dr2) + dty) },
                      { 0, 1, 0, -(dot(p, dr3) + dtz), 0.0f, dot(p, dr1) + dtx },
                      { 0, 0, 1, dot(p, dr2) + dty, -(dot(p, dr1) + dtx), 0.0f } };
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 6; ++c) jac[r * 6 + c] = A[r * 4 + 0] * J[0][c] + A[r * 4 + 1] * J[1][c] + A[r * 4 + 2] * J[2][c];
}

/* accumulates one residual row pair into the dense lower-triangular system (SolverBundlingDenseUtil.h:229-298) */
static void add_to_system(float* JtJ, float* Jtr, unsigned dim, const float* ri, const float* rj, unsigned vi, unsigned vj, float res, float w) {
    for (unsigned a = 0; a < 6; ++a) {
        for (unsigned b = a; b < 6; ++b) {
            if (vi > 0) JtJ[(vi * 6 + b) * dim + (vi * 6 + a)] += ri[a] * ri[b] * w;
            if (vj > 0) JtJ[(vj * 6 + b) * dim + (vj * 6 + a)] += rj[a] * rj[b] * w;
            if (vi > 0 && vj > 0) {
                JtJ[(vj * 6 + b) * dim + (vi * 6 + a)] += ri[a] * rj[b] * w;
                if (a != b) JtJ[(vj * 6 + a) * dim + (vi * 6 + b)] += ri[b] * rj[a] * w;
            }
        }
        if (vi > 0) Jtr[vi * 6 + a] += ri[a] * res * w;
        if (vj > 0) Jtr[vj * 6 + a] += rj[a] * res * w;
    }
}

/* BuildDenseSystem (SolverBundling.cu:308-471).  Returns the number of overlapping pairs with non-zero weight; 0 => dense off. */
static unsigned build_dense_system(const OrcDenseParams* d, const OrcCacheFrame* frames, const int* valid, unsigned N, const float* T, const float* Tinv,
                                   float wDepth, float wColor, float* JtJ, float* Jtr, unsigned* outPairs) {
    const unsigned dim = 6 * N;
    memset(JtJ, 0, sizeof(float) * dim * dim); memset(Jtr, 0, sizeof(float) * dim);
    unsigned nOverlap = 0, nUsed = 0;
    const unsigned subW = d->W / d->subsample;
    for (unsigned i = 0; i < N; ++i) for (unsigned j = i + 1; j < N; ++j) {
        if (!d->usePairwise && j != i + 1) continue;
        if (valid && (valid[i] == 0 || valid[j] == 0)) continue;
        float transform[16]; mat4_mul(&Tinv[16 * i], &T[16 * j], transform);
        { /* computeAngleDiff(transform, 0.52) SolverBundlingDenseUtil.h:416-424 */
            const float inv = 1.0f / sqrtf(3.0f);
            const v3 x = V(inv, inv, inv), vv = rot3(transform, x);
            const float angle = acosf(fminf(fmaxf(dot(x, vv), -1.0f), 1.0f));
            if (!(fabsf(angle) < 0.52f)) continue;
        }
        int found = 0;
        for (unsigned tidx = 0; tidx < 512; ++tidx) {
            const unsigned x = (tidx % subW) * d->subsample, y = (tidx / subW) * d->subsample, idx = y * d->W + x;
            if (idx < d->W * d->H) found += find_corr_prefilter(d, idx, transform, frames[i].depth, frames[j].depth);
        }
        if (!(found > 10)) continue;
        ++nOverlap;
        float count = 0.0f;
        for (unsigned idx = 0; idx < d->W * d->H; ++idx) count += (float)find_corr_count(d, idx, transform, &frames[i], &frames[j]);
        float pairW = count;
        if (count > 0) pairW = (count < 800) ? 0.0f : 1.0f / fminf(logf(count), 9.0f);
        if (pairW == 0.0f) continue;
        ++nUsed;
        for (unsigned idx = 0; idx < d->W * d->H; ++idx) {
            v3 cps, s2t, cpt, nt; float sx, sy;
            const int foundCorr = find_corr_build(d, idx, transform, &frames[i], &frames[j], &cps, &s2t, &sx, &sy, &cpt, &nt);
            if (wDepth > 0.0f && foundCorr) {
                const float res = dot(sub(cpt, s2t), nt);
                const float w = wDepth * pairW * powf(fmaxf(0.0f, 1.0f - cpt.z / 2.0f), 2.5f);
                float ri[6] = { 0, 0, 0, 0, 0, 0 }, rj[6] = { 0, 0, 0, 0, 0, 0 }, jac[18];
                if (i > 0) { lie_deriv_i(&Tinv[16 * j], &T[16 * i], cps, jac); for (int c = 0; c < 6; ++c) ri[c] = -(jac[c] * nt.x + jac[6 + c] * nt.y + jac[12 + c] * nt.z); }
                if (j > 0) { lie_deriv_j(&Tinv[16 * i], &T[16 * j], cps, jac); for (int c = 0; c < 6; ++c) rj[c] = -(jac[c] * nt.x + jac[6 + c] * nt.y + jac[12 + c] * nt.z); }
                add_to_system(JtJ, Jtr, dim, ri, rj, i, j, res, w);
            }
            if (wColor > 0.0f && foundCorr) {
                float dI[2], It;
                bilinear(frames[i].intensityDerivs, 2, sx, sy, d->W, d->H, dI);
                bilinear(frames[i].intensity, 1, sx, sy, d->W, d->H, &It);
                const float cres = It - frames[j].intensity[idx];
                if (dI[0] != MINF_ && fabsf(cres) < d->colorThresh && sqrtf(dI[0] * dI[0] + dI[1] * dI[1]) > d->colorGradientMin) {
                    /* dColorB (1x2) * dProj (2x3) * jac (3x6), ICPUtil.h:14-25, EquationsLie.h:263-277 */
                    const float z2 = s2t.z * s2t.z;
                    const float P[2][3] = { { d->fx / s2t.z, 0.0f, -d->fx * s2t.x / z2 }, { 0.0f, d->fy / s2t.z, -d->fy * s2t.y / z2 } };
                    float ri[6] = { 0, 0, 0, 0, 0, 0 }, rj[6] = { 0, 0, 0, 0, 0, 0 }, jac[18];
                    for (int side = 0; side < 2; ++side) {
                        if (side == 0 && !(i > 0)) continue;
                        if (side == 1 && !(j > 0)) continue;
                        if (side == 0) lie_deriv_i(&Tinv[16 * j], &T[16 * i], cps, jac); else lie_deriv_j(&Tinv[16 * i], &T[16 * j], cps, jac);
                        for (int c = 0; c < 6; ++c) {
                            const float pj0 = P[0][0] * jac[c] + P[0][1] * jac[6 + c] + P[0][2] * jac[12 + c];
                            const float pj1 = P[1][0] * jac[c] + P[1][1] * jac[6 + c] + P[1][2] * jac[12 + c];
                            (side == 0 ? ri : rj)[c] = dI[0] * pj0 + dI[1] * pj1;
                        }
                    }
                    const float w = wColor * pairW * fmaxf(0.0f, 1.0f - fabsf(cres) / (1.15f * d->colorThresh));
                    add_to_system(JtJ, Jtr, dim, ri, rj, i, j, cres, w);
                }
            }
        }
    }
    /* FlipJtJ: mirror lower -> upper (:81-91) */
    for (unsigned y = 0; y < dim; ++y) for (unsigned x = y + 1; x < dim; ++x) JtJ[y * dim + x] = JtJ[x * dim + y];
    if (outPairs) { outPairs[0] = nOverlap; outPairs[1] = nUsed; }
    return nOverlap;
}

/* The complete solveBundlingStub (sparse + dense), SolverBundling.cu:1137-1220.  frames / dense may be NULL (sparse only).
 * stats: [0] GN iterations, [1] PCG iterations, [2] overlapping pairs (last GN), [3] pairs with weight (last GN). */
ORC_API int orc_solver_solve(BFEntryJ* corr, unsigned C, unsigned N, unsigned maxCorrPerImage, float* xRot, float* xTrans,
                             unsigned nNonLinear, unsigned nLinear, const float* weightsSparse, const float* weightsDenseDepth,
                             const float* weightsDenseColor, const OrcCacheFrame* frames, const OrcDenseParams* dense, const int* valid,
                             int* varToCorr, int* numEntriesPerRow, unsigned stats[4]) {
    OrcSolver s;
    memset(&s, 0, sizeof s);
    s.N = N; s.C = C; s.maxCorrPerImage = maxCorrPerImage; s.corr = corr; s.varToCorr = varToCorr; s.numEntriesPerRow = numEntriesPerRow;
    s.xRot = xRot; s.xTrans = xTrans;
    const unsigned dim = 6 * N;
    float* buf = (float*)calloc((size_t)N * (3 * 12 + 32 + 1) + (size_t)C * 3 + 16 + (frames ? (size_t)dim * dim + dim : 0), sizeof(float));
    if (!buf) return -1;
    float* p = buf;
    s.deltaRot = p; p += 3 * N; s.deltaTrans = p; p += 3 * N; s.rRot = p; p += 3 * N; s.rTrans = p; p += 3 * N;
    s.zRot = p; p += 3 * N; s.zTrans = p; p += 3 * N; s.pRot = p; p += 3 * N; s.pTrans = p; p += 3 * N;
    s.ApRot = p; p += 3 * N; s.ApTrans = p; p += 3 * N; s.precRot = p; p += 3 * N; s.precTrans = p; p += 3 * N;
    s.T = p; p += 16 * N; s.Tinv = p; p += 16 * N; s.rDotzOld = p; p += N; s.Jp = p; p += 3 * (size_t)C + 16;
    float* JtJ = frames ? p : NULL; float* Jtr = frames ? p + (size_t)dim * dim : NULL;
    orc_solver_build_table(corr, C, maxCorrPerImage, varToCorr, numEntriesPerRow, N);
    unsigned totalPcg = 0, gnRun = 0, pairInfo[2] = { 0, 0 };
    for (unsigned nIter = 0; nIter < nNonLinear; ++nIter) {
        const float wS = weightsSparse[nIter], wD = weightsDenseDepth ? weightsDenseDepth[nIter] : 0.0f, wC = weightsDenseColor ? weightsDenseColor[nIter] : 0.0f;
        int useDense = (wD > 0 || wC > 0) && frames != NULL;
        ++gnRun;
        for (unsigned k = 0; k < N; ++k) { orc_pose_to_matrix(&xRot[3 * k], &xTrans[3 * k], &s.T[16 * k]); orc_mat4_inverse(&s.T[16 * k], &s.Tinv[16 * k]); }
        if (useDense) useDense = build_dense_system(dense, frames, valid, N, s.T, s.Tinv, wD, wC, JtJ, Jtr, pairInfo) > 0;
        float scanAlpha0 = 0.0f, scanAlpha1 = 0.0f;
        for (unsigned x = 1; x < N; ++x) {
            v3 resRot, resTrans;
            eval_minus_jtf(&s, x, wS, &resRot, &resTrans);
            if (useDense) {   /* SolverBundlingEquationsLie.h:114-118 */
                resRot = sub(resRot, V(Jtr[x * 6 + 3], Jtr[x * 6 + 4], Jtr[x * 6 + 5]));
                resTrans = sub(resTrans, V(Jtr[x * 6 + 0], Jtr[x * 6 + 1], Jtr[x * 6 + 2]));
            }
            st3(s.rRot, x, resRot); st3(s.rTrans, x, resTrans);
            const v3 pR = mulv(ld3(s.precRot, x), resRot), pT = mulv(ld3(s.precTrans, x), resTrans);
            st3(s.pRot, x, pR); st3(s.pTrans, x, pT);
            scanAlpha0 += dot(resRot, pR) + dot(resTrans, pT);
            st3(s.ApRot, x, V(0, 0, 0)); st3(s.ApTrans, x, V(0, 0, 0));
        }
        for (unsigned x = 1; x < N; ++x) s.rDotzOld[x] = scanAlpha0;
        for (unsigned lin = 0; lin < nLinear; ++lin) {
            int last = (lin == nLinear - 1);
            ++totalPcg;
            scanAlpha0 = 0.0f; scanAlpha1 = 0.0f;
            if (wS > 0.0f) {
                for (unsigned c = 0; c < C; ++c) st3(s.Jp, c, apply_j(&s, c, wS));
                for (unsigned x = 1; x < N; ++x) { v3 r, t; apply_jt(&s, x, &r, &t); st3(s.ApRot, x, add(ld3(s.ApRot, x), r)); st3(s.ApTrans, x, add(ld3(s.ApTrans, x), t)); }
            }
            if (useDense) {   /* applyJTJDenseDevice, SolverBundlingDenseUtil.h:371-411 */
                for (unsigned x = 1; x < N; ++x) {
                    v3 oR = V(0, 0, 0), oT = V(0, 0, 0);
                    for (unsigned i = 1; i < N; ++i) {
                        const v3 pt = ld3(s.pTrans, i), pr = ld3(s.pRot, i);
                        const float* B = &JtJ[(x * 6) * dim + i * 6];
#define BR(r, c) B[(r) * dim + (c)]
                        oT = add(oT, V(BR(0, 0) * pt.x + BR(0, 1) * pt.y + BR(0, 2) * pt.z + BR(0, 3) * pr.x + BR(0, 4) * pr.y + BR(0, 5) * pr.z,
                                       BR(1, 0) * pt.x + BR(1, 1) * pt.y + BR(1, 2) * pt.z + BR(1, 3) * pr.x + BR(1, 4) * pr.y + BR(1, 5) * pr.z,
                                       BR(2, 0) * pt.x + BR(2, 1) * pt.y + BR(2, 2) * pt.z + BR(2, 3) * pr.x + BR(2, 4) * pr.y + BR(2, 5) * pr.z));
                        oR = add(oR, V(BR(3, 0) * pt.x + BR(3, 1) * pt.y + BR(3, 2) * pt.z + BR(3, 3) * pr.x + BR(3, 4) * pr.y + BR(3, 5) * pr.z,
                                       BR(4, 0) * pt.x + BR(4, 1) * pt.y + BR(4, 2) * pt.z + BR(4, 3) * pr.x + BR(4, 4) * pr.y + BR(4, 5) * pr.z,
                                       BR(5, 0) * pt.x + BR(5, 1) * pt.y + BR(5, 2) * pt.z + BR(5, 3) * pr.x + BR(5, 4) * pr.y + BR(5, 5) * pr.z));
#undef BR
                    }
                    st3(s.ApRot, x, add(ld3(s.ApRot, x), oR)); st3(s.ApTrans, x, add(ld3(s.ApTrans, x), oT));
                }
            }
            for (unsigned x = 1; x < N; ++x) scanAlpha0 += dot(ld3(s.pRot, x), ld3(s.ApRot, x)) + dot(ld3(s.pTrans, x), ld3(s.ApTrans, x));
            const float dotProduct = scanAlpha0;
            for (unsigned x = 1; x < N; ++x) {
                float alpha = 0.0f;
                if (dotProduct > FLOAT_EPSILON) alpha = s.rDotzOld[x] / dotProduct;
                st3(s.deltaRot, x, add(ld3(s.deltaRot, x), mul(ld3(s.pRot, x), alpha)));
                st3(s.deltaTrans, x, add(ld3(s.deltaTrans, x), mul(ld3(s.pTrans, x), alpha)));
                const v3 rR = sub(ld3(s.rRot, x), mul(ld3(s.ApRot, x), alpha)), rT = sub(ld3(s.rTrans, x), mul(ld3(s.ApTrans, x), alpha));
                st3(s.rRot, x, rR); st3(s.rTrans, x, rT);
                const v3 zR = mulv(ld3(s.precRot, x), rR), zT = mulv(ld3(s.precTrans, x), rT);
                st3(s.zRot, x, zR); st3(s.zTrans, x, zT);
                scanAlpha1 += dot(zR, rR) + dot(zT, rT);
            }
            trace_put((float)nIter, scanAlpha0);
            if (fabsf(scanAlpha0) < 5e-7f) last = 1;
            for (unsigned x = 1; x < N; ++x) {
                const float rDotzNew = scanAlpha1, rDotzOld = s.rDotzOld[x];
                float beta = 0.0f;
                if (rDotzOld > FLOAT_EPSILON) beta = rDotzNew / rDotzOld;
                s.rDotzOld[x] = rDotzNew;
                st3(s.pRot, x, add(ld3(s.zRot, x), mul(ld3(s.pRot, x), beta)));
                st3(s.pTrans, x, add(ld3(s.zTrans, x), mul(ld3(s.pTrans, x), beta)));
                st3(s.ApRot, x, V(0, 0, 0)); st3(s.ApTrans, x, V(0, 0, 0));
                if (last) {
                    float U[16], Cm[16], P[16];
                    orc_pose_to_matrix(&s.deltaRot[3 * x], &s.deltaTrans[3 * x], U);
                    orc_pose_to_matrix(&xRot[3 * x], &xTrans[3 * x], Cm);
                    mat4_mul(U, Cm, P);
                    orc_matrix_to_pose(P, &xRot[3 * x], &xTrans[3 * x]);
                }
            }
            if (last) break;
        }
        if (nIter < nNonLinear - 1) {
            float m = 0.0f;
            for (unsigned x = 1; x < N; ++x) {
                if (valid && valid[x] == 0) continue;
                for (int k = 0; k < 3; ++k) { m = fmaxf(m, fabsf(s.deltaRot[3 * x + k])); m = fmaxf(m, fabsf(s.deltaTrans[3 * x + k])); }
            }
            trace_put(-(float)(nIter + 1), m);
            if (m < 0.005f) break;
        }
    }
    if (stats) { stats[0] = gnRun; stats[1] = totalPcg; stats[2] = pairInfo[0]; stats[3] = pairInfo[1]; }
    free(buf);
    return 0;
}

/* dense system only (for tests of the dense builder): fills JtJ [(6N)^2] and Jtr [6N] for the given poses */
ORC_API unsigned orc_solver_build_dense(const float* xRot, const float* xTrans, unsigned N, const OrcCacheFrame* frames, const OrcDenseParams* dense,
                                        const int* valid, float wDepth, float wColor, float* JtJ, float* Jtr, unsigned outPairs[2]) {
    float* T = (float*)malloc(sizeof(float) * 32 * N);
    for (unsigned k = 0; k < N; ++k) { orc_pose_to_matrix(&xRot[3 * k], &xTrans[3 * k], &T[16 * k]); orc_mat4_inverse(&T[16 * k], &T[16 * N + 16 * k]); }
    unsigned r = build_dense_system(dense, frames, valid, N, T, T + 16 * N, wDepth, wColor, JtJ, Jtr, outPairs);
    free(T);
    return r;
}

/* test hook: the two 1x6 point-to-plane Jacobian rows of one dense correspondence (SolverBundlingEquationsLie.h:234-250) */
ORC_API void orc_dense_depth_rows(const float* Ti, const float* Tj, const float p[3], const float n[3], float rowI[6], float rowJ[6]) {
    float Tii[16], Tji[16], jac[18];
    orc_mat4_inverse(Ti, Tii); orc_mat4_inverse(Tj, Tji);
    const v3 cps = V(p[0], p[1], p[2]), nt = V(n[0], n[1], n[2]);
    lie_deriv_i(Tji, Ti, cps, jac); for (int c = 0; c < 6; ++c) rowI[c] = -(jac[c] * nt.x + jac[6 + c] * nt.y + jac[12 + c] * nt.z);
    lie_deriv_j(Tii, Tj, cps, jac); for (int c = 0; c < 6; ++c) rowJ[c] = -(jac[c] * nt.x + jac[6 + c] * nt.y + jac[12 + c] * nt.z);
}

// host_api.cu -- host-side C-ABI helpers (include/bf_host.h): pose inverse and the TSDF op replay loop.
#include "../../include/bf_host.h"
#include "bf_common.cuh"
#include "mat4.cuh"

// 4x4 inverse by cofactor expansion in fp32, as the reference's float4x4::getInverse does on the host
// (FL/SiftGPU/cuda_SimpleMatrixUtil.h:980-1100).  Written from the textbook adjugate formula:
// inv = adj(M) / det(M), cofactors expanded as 2x2 sub-determinant products.
BF_API void bfMat4Inverse(const float* m, float* out) { bf::mat4_inverse_ref(m, out); }          // the reference's host formula, bit for bit (mat4.cuh)

namespace bf {
int tsdf_lanes_begin(const BFHashDataStruct* hd, const BFHashParams* hp);     // tsdf.cu: two-lane replay bracket
int tsdf_lanes_end(const BFHashDataStruct* hd);
int tsdf_batching_usable();                                                     // tsdf.cu: batching on and fast arithmetic selected
}

static int run_ops(BFHashDataStruct* hd, BFHashParams* hp, const BFDepthCameraParams* cam, const BFTsdfOp* ops, int numOps,
                   const float* const* d_depthFrames, const uint8_t* const* d_colorFrames);

// One call replays a whole batch of TSDF operations.  Inside, the stencil of op k runs on the library's back lane while alloc +
// compactify of op k+1 run on the caller's stream (tsdf.cu, "two lanes"); on return the caller's stream is ordered after all of it.
BF_API int bfTsdfRunOps(BFHashDataStruct* hd, BFHashParams* hp, const BFDepthCameraParams* cam, const BFTsdfOp* ops, int numOps,
                        const float* const* d_depthFrames, const uint8_t* const* d_colorFrames) {
    int rc = bf::tsdf_lanes_begin(hd, hp);
    if (rc) return rc;
    rc = run_ops(hd, hp, cam, ops, numOps, d_depthFrames, d_colorFrames);
    const int rc2 = bf::tsdf_lanes_end(hd);
    return rc ? rc : rc2;
}

static int run_ops(BFHashDataStruct* hd, BFHashParams* hp, const BFDepthCameraParams* cam, const BFTsdfOp* ops, int numOps,
                   const float* const* d_depthFrames, const uint8_t* const* d_colorFrames) {
    const bool batch = d_colorFrames != nullptr && bf::tsdf_batching_usable() != 0;
    for (int i = 0; i < numOps; ++i) {
        const BFTsdfOp& op = ops[i];
        if (batch) {
            // a run of re-integration pairs (DepthSensing.cpp:867-895: up to s_maxFrameFixes of them per frame): one batch pass per <= 16 pairs
            int n = 0;
            while (i + 2 * n + 1 < numOps && n < 16 && ops[i + 2 * n].kind == BF_TSDF_OP_DEINTEGRATE && ops[i + 2 * n + 1].kind == BF_TSDF_OP_INTEGRATE &&
                   ops[i + 2 * n + 1].frame == ops[i + 2 * n].frame && d_colorFrames[ops[i + 2 * n].frame] != nullptr) ++n;
            if (n >= 2) {
                BFTsdfReintegration pairs[16];
                for (int k = 0; k < n; ++k) {
                    pairs[k].frame = ops[i + 2 * k].frame;
                    for (int e = 0; e < 16; ++e) { pairs[k].oldPose[e] = ops[i + 2 * k].pose[e]; pairs[k].newPose[e] = ops[i + 2 * k + 1].pose[e]; }
                }
                int rc = bfTsdfReintegrateBatch(hd, hp, cam, pairs, n, d_depthFrames, d_colorFrames);
                if (rc) return rc;
                i += 2 * n - 1;
                continue;
            }
        }
        if (op.kind == BF_TSDF_OP_DEINTEGRATE && i + 1 < numOps && ops[i + 1].kind == BF_TSDF_OP_INTEGRATE && ops[i + 1].frame == op.frame) {
            // the reference's re-integration pair: one fused pass (bfTsdfReintegrateFrame)
            BFHashParams hpOld = *hp;
            for (int k = 0; k < 16; ++k) hpOld.m_rigidTransform.m[k] = op.pose[k];
            bfMat4Inverse(op.pose, hpOld.m_rigidTransformInverse.m);
            const BFTsdfOp& nx = ops[i + 1];
            for (int k = 0; k < 16; ++k) hp->m_rigidTransform.m[k] = nx.pose[k];
            bfMat4Inverse(nx.pose, hp->m_rigidTransformInverse.m);
            BFDepthCameraData dd;
            dd.d_depthData = d_depthFrames[op.frame];
            dd.d_colorData = d_colorFrames ? d_colorFrames[op.frame] : nullptr;
            int rc = bfTsdfReintegrateFrame(hd, &hpOld, hp, &dd, cam);
            if (rc) return rc;
            ++i;
            continue;
        }
        if (op.kind == BF_TSDF_OP_GARBAGE_COLLECT) {
            int rc = bfTsdfGarbageCollect(hd, hp);
            if (rc) return rc;
            continue;
        }
        for (int k = 0; k < 16; ++k) hp->m_rigidTransform.m[k] = op.pose[k];
        bfMat4Inverse(op.pose, hp->m_rigidTransformInverse.m);
        BFDepthCameraData dd;
        dd.d_depthData = d_depthFrames[op.frame];
        dd.d_colorData = d_colorFrames ? d_colorFrames[op.frame] : nullptr;
        int rc = bfTsdfIntegrateFrame(hd, hp, &dd, cam, op.kind == BF_TSDF_OP_DEINTEGRATE ? 1 : 0);
        if (rc) return rc;
    }
    return 0;
}

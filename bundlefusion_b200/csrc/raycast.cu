// raycast.cu -- ray cast of the hashed TSDF for sm_90a.  Implements include/bf_raycast.h (SURVEY.md section 8f, row N3).
//
// Behavioural sources (what, not how; FL/ = /root/reference/FriedLiver/Source/):
//   renderKernel, rayIntervalSplatKernel, resetRayIntervalSplatKernel      FL/DepthSensing/CUDARayCastSDF.cu:17-191
//   RayCastData (trilinear sample, bisection, gradient, projections)       FL/DepthSensing/RayCastSDFUtil.h:87-294
//   HashDataStruct::getVoxel / getHashEntryForSDFBlockPos                  FL/DepthSensing/VoxelUtilHashSDF.h:276-358, 407-485
//   the Direct3D 11 draw of the quads                                      FL/DepthSensing/DX11RayIntervalSplatting.cpp:137-229
//   computeNormals_Kernel                                                  FL/CUDAImageUtil.cu:404-431
// How it differs from the reference's organisation:
//   * the interval images are built by ONE CUDA kernel (a warp per in-frustum block walks the pixels of the block's screen rectangle, atomic min /
//     max on the float bits), for both directions at once, from the device-side list count -- the reference round-trips through Direct3D 11 (two
//     kernel launches that write a vertex buffer, two draws, two render targets mapped back as textures);
//   * the ray march keeps the last block it looked up per thread: the eight corners of a trilinear sample and consecutive samples of a ray mostly fall
//     into the same block, so seven of eight hash probes go away; values are the same loads;
//   * one thread per pixel in 8 x 8 tiles, as the reference (neighbouring rays walk neighbouring voxels).
// Arithmetic contract (bit-exact with oracle/raycast_oracle.c): TU built -fmad=false, expressions in the reference's order, normalize() as
// v * (1 / sqrtf(v.v)) (the reference's rsqrtf is an approximate instruction).
#include <cmath>

#include <cstring>

#include "../../include/bf_host.h"
#include "../../include/bf_raycast.h"
#include "bf_common.cuh"
#include "hash_read.cuh"

namespace bf {

extern unsigned long long g_launchCount;
const BFHashParams* bound_hash_params();                 // tsdf.cu: what updateConstantHashParams / updateConstantDepthCameraParams latched
const BFDepthCameraParams* bound_camera_params();

struct RcArgs {
    BFHashDataStruct hd; BFHashParams hp; BFDepthCameraParams cp; BFRayCastParams p; BFRayCastData d;
};

// findIntersectionBisection, :148-170
__device__ bool bisection(const RcArgs& a, F3 camPos, F3 dir, float d0, float r0, float d1, float r1, float& alpha, unsigned& color, BlockCache& bc) {
    float lo = r0, loDist = d0, hi = r1, hiDist = d1, c = 0.0f;
#pragma unroll 1
    for (unsigned i = 0; i < 3; ++i) {
        c = lo + (loDist / (loDist - hiDist)) * (hi - lo);
        float cDist;
        if (!trilinear(a.hd, a.hp, add3(camPos, scale3(c, dir)), cDist, color, bc)) return false;
        if (loDist * cDist > 0.0f) { lo = c; loDist = cDist; } else { hi = c; hiDist = cDist; }
    }
    alpha = c;
    return true;
}

// gradientForPoint, :173-199
__device__ F3 gradient(const RcArgs& a, F3 pos, BlockCache& bc) {
    const float vs = a.hp.m_virtualVoxelSize;
    unsigned col;
    float dm[3], dp[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { const F3 o = { k == 0 ? 0.5f * vs : 0.0f, k == 1 ? 0.5f * vs : 0.0f, k == 2 ? 0.5f * vs : 0.0f }; trilinear(a.hd, a.hp, sub3(pos, o), dm[k], col, bc); }
#pragma unroll
    for (int k = 0; k < 3; ++k) { const F3 o = { k == 0 ? 0.5f * vs : 0.0f, k == 1 ? 0.5f * vs : 0.0f, k == 2 ? 0.5f * vs : 0.0f }; trilinear(a.hd, a.hp, add3(pos, o), dp[k], col, bc); }
    const F3 g = { (dm[0] - dp[0]) / vs, (dm[1] - dp[1]) / vs, (dm[2] - dp[2]) / vs };
    const float l = sqrtf(dot3(g, g));
    if (l == 0.0f) return F3{ 0.0f, 0.0f, 0.0f };
    return F3{ -g.x / l, -g.y / l, -g.z / l };
}
__device__ __forceinline__ F3 depth_to_camera(const BFRayCastParams& p, unsigned ux, unsigned uy, float depth) {        // :207-212
    const float x = ((float)ux - p.mx) / p.fx, y = ((float)uy - p.my) / p.fy;
    return F3{ depth * x, depth * y, depth };
}

// renderKernel (CUDARayCastSDF.cu:17-58) + traverseCoarseGridSimpleSampleAll (RayCastSDFUtil.h:231-294)
__global__ void __launch_bounds__(64)
raycast_render_kernel(const __grid_constant__ RcArgs a) {
    const unsigned x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    const BFRayCastParams& p = a.p;
    if (x >= p.m_width || y >= p.m_height) return;
    const size_t i = (size_t)y * p.m_width + x;
    const float4 minf4 = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    float outDepth = -INFINITY; float4 outPos = minf4, outNrm = minf4, outCol = minf4;
    const F3 camDir = normalize3(depth_to_camera(p, x, y, 1.0f));
    const F3 camPos = mul_point(p.m_viewMatrixInverse.m, F3{ 0.0f, 0.0f, 0.0f });
    const F3 dir = normalize3(mul_dir(p.m_viewMatrixInverse.m, camDir));
    float mn = __ldg(&a.d.d_rayIntervalSplatMin[i]), mx = __ldg(&a.d.d_rayIntervalSplatMax[i]);
    const bool have = !(mn == 0 || mn == -INFINITY) && !(mx == 0 || mx == -INFINITY);
    if (have) {
        mn = fmaxf(mn, p.m_minDepth); mx = fminf(mx, p.m_maxDepth);
        float lastSdf = 0.0f, lastAlpha = 0.0f; unsigned lastWeight = 0;
        const float depthToRayLength = 1.0f / camDir.z;
        float rayCurrent = depthToRayLength * fmaxf(p.m_minDepth, mn);
        const float rayEnd = depthToRayLength * fminf(p.m_maxDepth, mx);
        BlockCache bc; bc.valid = false; bc.ptr = BF_FREE_ENTRY; bc.b = I3{ 0, 0, 0 };
#pragma unroll 1
        while (rayCurrent < rayEnd) {
            const F3 cur = add3(camPos, scale3(rayCurrent, dir));
            float dist; unsigned col;
            if (trilinear(a.hd, a.hp, cur, dist, col, bc)) {
                if (lastWeight > 0 && lastSdf > 0.0f && dist < 0.0f) {
                    float alpha = 0.0f; unsigned col2 = 0;
                    const bool b = bisection(a, camPos, dir, lastSdf, lastAlpha, dist, rayCurrent, alpha, col2, bc);
                    if (b && fabsf(lastSdf - dist) < p.m_thresSampleDist && fabsf(dist) < p.m_thresDist) {
                        const float d = alpha / depthToRayLength;
                        outDepth = d;
                        const F3 c3 = depth_to_camera(p, x, y, d);
                        outPos = make_float4(c3.x, c3.y, c3.z, 1.0f);
                        outCol = make_float4((float)(col2 & 0xffu) / 255.f, (float)((col2 >> 8) & 0xffu) / 255.f, (float)((col2 >> 16) & 0xffu) / 255.f, 1.0f);
                        if (p.m_useGradients) {
                            const F3 g = gradient(a, add3(camPos, scale3(alpha, dir)), bc);
                            const F3 n = mul_dir(p.m_viewMatrix.m, F3{ -g.x, -g.y, -g.z });
                            outNrm = make_float4(n.x, n.y, n.z, 1.0f);
                        }
                        break;
                    }
                }
                lastSdf = dist; lastAlpha = rayCurrent; lastWeight = 1;
            } else lastWeight = 0;
            rayCurrent += p.m_rayIncrement;
        }
    }
    a.d.d_depth[i] = outDepth;
    reinterpret_cast<float4*>(a.d.d_depth4)[i] = outPos;
    reinterpret_cast<float4*>(a.d.d_normals)[i] = outNrm;
    reinterpret_cast<float4*>(a.d.d_colors)[i] = outCol;
}

// computeNormals_Kernel, FL/CUDAImageUtil.cu:404-431
__global__ void __launch_bounds__(64)
raycast_normals_kernel(float4* __restrict__ out, const float4* __restrict__ in, unsigned W, unsigned H) {
    const unsigned x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= W || y >= H) return;
    float4 o = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    if (x > 0 && x < W - 1 && y > 0 && y < H - 1) {
        const float4 CC = in[(size_t)y * W + x], PC = in[(size_t)(y + 1) * W + x], CP = in[(size_t)y * W + x + 1], MC = in[(size_t)(y - 1) * W + x], CM = in[(size_t)y * W + x - 1];
        if (CC.x != -INFINITY && PC.x != -INFINITY && CP.x != -INFINITY && MC.x != -INFINITY && CM.x != -INFINITY) {
            const float ax = PC.x - MC.x, ay = PC.y - MC.y, az = PC.z - MC.z, bx = CP.x - CM.x, by = CP.y - CM.y, bz = CP.z - CM.z;
            const float nx = ay * bz - az * by, ny = az * bx - ax * bz, nz = ax * by - ay * bx;
            const float l = sqrtf((nx * nx + ny * ny) + nz * nz);
            if (l > 0.0f) o = make_float4(nx / -l, ny / -l, nz / -l, 0.0f);
        }
    }
    out[(size_t)y * W + x] = o;
}

// ---- interval splat --------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ F3 camera_to_depth_proj(const BFRayCastParams& p, F3 pos) {       // RayCastSDFUtil.h:213-228
    const float px = pos.x * p.fx / pos.z + p.mx, py = pos.y * p.fy / pos.z + p.my;
    F3 r;
    r.x = (2.0f * px - ((float)p.m_width - 1.0f)) / ((float)p.m_width - 1.0f);
    r.y = (((float)p.m_height - 1.0f) - 2.0f * py) / ((float)p.m_height - 1.0f);
    r.z = (pos.z - p.m_minDepth) / (p.m_maxDepth - p.m_minDepth);
    return r;
}
__device__ bool block_in_frustum(const BFHashParams& hp, const BFDepthCameraParams& cp, I3 b) {        // VoxelUtilHashSDF.h:322-326, DepthCameraUtil.h:138-144
    const float vs = hp.m_virtualVoxelSize, off = vs * 0.5f * ((float)BF_SDF_BLOCK_SIZE - 1.0f);
    const F3 w = { (float)(b.x * BF_SDF_BLOCK_SIZE) * vs + off, (float)(b.y * BF_SDF_BLOCK_SIZE) * vs + off, (float)(b.z * BF_SDF_BLOCK_SIZE) * vs + off };
    const F3 pc = mul_point(hp.m_rigidTransformInverse.m, w);
    const float px = pc.x * cp.fx / pc.z + cp.mx, py = pc.y * cp.fy / pc.z + cp.my;
    const float w1 = (float)cp.m_imageWidth - 1.0f, h1 = (float)cp.m_imageHeight - 1.0f;
    float ix = (2.0f * px - w1) / w1, iy = (h1 - 2.0f * py) / h1;
    float iz = (pc.z - cp.m_sensorDepthWorldMin) / (cp.m_sensorDepthWorldMax - cp.m_sensorDepthWorldMin);
    ix *= 0.95f; iy *= 0.95f; iz *= 0.95f;
    return !(ix < -1.0f || ix > 1.0f || iy < -1.0f || iy > 1.0f || iz < 0.0f || iz > 1.0f);
}
// rayIntervalSplatKernel for one entry (CUDARayCastSDF.cu:90-172): lo / hi of the eight projected corners
__device__ bool block_quad(const RcArgs& a, const BFHashEntry* e, F3& lo, F3& hi) {
    const int4 q = __ldg(reinterpret_cast<const int4*>(e));
    if (q.w == BF_FREE_ENTRY) return false;
    const I3 b = { q.x, q.y, q.z };
    if (!block_in_frustum(a.hp, a.cp, b)) return false;
    const float vs = a.hp.m_virtualVoxelSize;
    const F3 wv = block_to_world(a.hp, b);
    const F3 mn = { wv.x - vs / 2.0f, wv.y - vs / 2.0f, wv.z - vs / 2.0f };
    const F3 mx = { mn.x + (float)BF_SDF_BLOCK_SIZE * vs, mn.y + (float)BF_SDF_BLOCK_SIZE * vs, mn.z + (float)BF_SDF_BLOCK_SIZE * vs };
    lo = F3{ INFINITY, INFINITY, INFINITY }; hi = F3{ -INFINITY, -INFINITY, -INFINITY };
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const F3 c = { (k & 1) ? mx.x : mn.x, (k & 2) ? mx.y : mn.y, (k & 4) ? mx.z : mn.z };
        const F3 s = camera_to_depth_proj(a.p, mul_point(a.p.m_viewMatrix.m, c));
        lo.x = fminf(lo.x, s.x); lo.y = fminf(lo.y, s.y); lo.z = fminf(lo.z, s.z);
        hi.x = fmaxf(hi.x, s.x); hi.y = fmaxf(hi.y, s.y); hi.z = fmaxf(hi.z, s.z);
    }
    return true;
}
__device__ __forceinline__ float depth_proj_to_camera_z(const BFRayCastParams& p, float z) { return z * (p.m_maxDepth - p.m_minDepth) + p.m_minDepth; }

__global__ void raycast_fill_kernel(float* a, float* b, unsigned n, float v) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { a[i] = v; if (b) b[i] = v; }
}
// the reference's vertex buffer, for callers that rasterise themselves: six vertices per entry
__global__ void raycast_quads_kernel(const __grid_constant__ RcArgs a, unsigned count) {
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count) return;
    F3 lo, hi;
    if (!block_quad(a, &a.hd.d_hashCompactified[idx], lo, hi)) return;
    const float depth = a.p.m_splatMinimum == 1 ? lo.z : hi.z, dw = depth_proj_to_camera_z(a.p, depth);
    float4* v = reinterpret_cast<float4*>(a.d.d_vertexBuffer) + (size_t)idx * 6;
    v[0] = make_float4(hi.x, lo.y, depth, dw); v[1] = make_float4(lo.x, lo.y, depth, dw); v[2] = make_float4(hi.x, hi.y, depth, dw);
    v[3] = make_float4(lo.x, lo.y, depth, dw); v[4] = make_float4(hi.x, hi.y, depth, dw); v[5] = make_float4(lo.x, hi.y, depth, dw);
}
// Both interval images in one pass: a warp per list entry; a pixel belongs to the block's rectangle when its centre lies in [x0, x1) x [y0, y1) of the
// viewport rectangle (Direct3D's top-left rule on exact coordinates); constant depth per quad, LESS into the min image, GREATER into the max image;
// a quad whose depth leaves [0, 1] is clipped away.  Empty pixels hold -inf: as UNSIGNED bits -inf is above every positive float (atomicMin takes any
// depth), as SIGNED bits it is below (atomicMax takes any depth).
__global__ void __launch_bounds__(256)
raycast_splat_kernel(const __grid_constant__ RcArgs a) {
    const unsigned count = (unsigned)max(0, a.hd.d_hashCompactifiedCounter[0]);
    const unsigned lane = threadIdx.x & 31u, warpsPerGrid = (gridDim.x * blockDim.x) >> 5;
    const int W = (int)a.p.m_width, H = (int)a.p.m_height;
    for (unsigned e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < count; e += warpsPerGrid) {
        F3 lo, hi;
        if (!block_quad(a, &a.hd.d_hashCompactified[e], lo, hi)) continue;                  // uniform for the warp
        const float X0 = (lo.x + 1.0f) * 0.5f * (float)W, X1 = (hi.x + 1.0f) * 0.5f * (float)W;
        const float Y0 = (1.0f - hi.y) * 0.5f * (float)H, Y1 = (1.0f - lo.y) * 0.5f * (float)H;
        if (!(X0 < X1) || !(Y0 < Y1)) continue;
        float fi0 = ceilf(X0 - 0.5f), fi1 = ceilf(X1 - 0.5f), fj0 = ceilf(Y0 - 0.5f), fj1 = ceilf(Y1 - 0.5f);
        if (fi0 < 0.0f) fi0 = 0.0f;
        if (fj0 < 0.0f) fj0 = 0.0f;
        if (fi1 > (float)W) fi1 = (float)W;
        if (fj1 > (float)H) fj1 = (float)H;
        const int i0 = (int)fi0, i1 = (int)fi1, j0 = (int)fj0, j1 = (int)fj1;
        if (i1 <= i0 || j1 <= j0) continue;
        const bool nearOk = lo.z >= 0.0f && lo.z <= 1.0f, farOk = hi.z >= 0.0f && hi.z <= 1.0f;
        const float dNear = depth_proj_to_camera_z(a.p, lo.z), dFar = depth_proj_to_camera_z(a.p, hi.z);
        const int nx = i1 - i0, n = nx * (j1 - j0);
        for (int k = (int)lane; k < n; k += 32) {
            const size_t px = (size_t)(j0 + k / nx) * W + (size_t)(i0 + k % nx);
            if (nearOk) atomicMin(reinterpret_cast<unsigned*>(a.d.d_rayIntervalSplatMin) + px, __float_as_uint(dNear));
            if (farOk) atomicMax(reinterpret_cast<int*>(a.d.d_rayIntervalSplatMax) + px, (int)__float_as_uint(dFar));
        }
    }
}

static BFRayCastParams g_rayCastParams;        // updateConstantRayCastParams

static int fill_args(RcArgs* a, const BFHashDataStruct* hd, const BFHashParams* hp, const BFDepthCameraParams* cp, const BFRayCastData* d, const BFRayCastParams* p) {
    if (!hd || !hp || !d || !p) return (int)cudaErrorInvalidValue;
    if (p->m_width == 0 || p->m_height == 0) return (int)cudaErrorInvalidValue;
    a->hd = *hd; a->hp = *hp; a->p = *p; a->d = *d;
    if (cp) a->cp = *cp; else memset(&a->cp, 0, sizeof(a->cp));
    return 0;
}
static int do_splat(const BFHashDataStruct* hd, const BFHashParams* hp, const BFDepthCameraParams* cp, const BFRayCastData* d, const BFRayCastParams* p) {
    RcArgs a;
    const int rc = fill_args(&a, hd, hp, cp, d, p);
    if (rc) return rc;
    if (!cp || !d->d_rayIntervalSplatMin || !d->d_rayIntervalSplatMax) return (int)cudaErrorInvalidValue;
    const unsigned n = p->m_width * p->m_height;
    g_launchCount += 2;
    raycast_fill_kernel<<<(n + 255) / 256, 256, 0, stream()>>>(d->d_rayIntervalSplatMin, d->d_rayIntervalSplatMax, n, -INFINITY);
    raycast_splat_kernel<<<num_sms() * 4, 256, 0, stream()>>>(a);
    BF_CHECK(cudaGetLastError());
    return 0;
}
static int do_render(const BFHashDataStruct* hd, const BFHashParams* hp, const BFRayCastData* d, const BFRayCastParams* p) {
    RcArgs a;
    const int rc = fill_args(&a, hd, hp, nullptr, d, p);
    if (rc) return rc;
    if (!d->d_depth || !d->d_depth4 || !d->d_normals || !d->d_colors || !d->d_rayIntervalSplatMin || !d->d_rayIntervalSplatMax) return (int)cudaErrorInvalidValue;
    ++g_launchCount;
    const dim3 block(8, 8), grid((p->m_width + 7) / 8, (p->m_height + 7) / 8);
    raycast_render_kernel<<<grid, block, 0, stream()>>>(a);
    BF_CHECK(cudaGetLastError());
    return 0;
}
static int do_normals(const BFRayCastData* d, unsigned W, unsigned H) {
    if (!d || !d->d_normals || !d->d_depth4 || W == 0 || H == 0) return (int)cudaErrorInvalidValue;
    ++g_launchCount;
    const dim3 block(8, 8), grid((W + 7) / 8, (H + 7) / 8);
    raycast_normals_kernel<<<grid, block, 0, stream()>>>(reinterpret_cast<float4*>(d->d_normals), reinterpret_cast<const float4*>(d->d_depth4), W, H);
    BF_CHECK(cudaGetLastError());
    return 0;
}

}  // namespace bf

using namespace bf;

BF_API void updateConstantRayCastParams(const BFRayCastParams* params) { g_rayCastParams = *params; }

BF_API void rayIntervalSplatCUDA(const BFHashDataStruct* hashData, const BFRayCastData* rayCastData, const BFRayCastParams* rayCastParams) {
    RcArgs a;
    BF_SAFE(fill_args(&a, hashData, bound_hash_params(), bound_camera_params(), rayCastData, rayCastParams));
    if (!rayCastData->d_vertexBuffer) BF_SAFE((int)cudaErrorInvalidValue);
    const unsigned n = rayCastParams->m_numOccupiedSDFBlocks;
    if (n == 0) return;
    ++g_launchCount;
    raycast_quads_kernel<<<(n + 127) / 128, 128, 0, stream()>>>(a, n);
    BF_SAFE((int)cudaGetLastError());
}
BF_API void resetRayIntervalSplatCUDA(BFRayCastData* data, const BFRayCastParams* params) {          // every vertex (-inf, -inf, -inf, -inf)
    if (!data || !params || !data->d_vertexBuffer) BF_SAFE((int)cudaErrorInvalidValue);
    const unsigned n = params->m_maxNumVertices * 4;
    if (n == 0) return;
    ++g_launchCount;
    raycast_fill_kernel<<<(n + 255) / 256, 256, 0, stream()>>>(data->d_vertexBuffer, nullptr, n, -INFINITY);
    BF_SAFE((int)cudaGetLastError());
}
BF_API void renderCS(const BFHashDataStruct* hashData, const BFRayCastData* rayCastData, const BFRayCastParams* rayCastParams) {
    BF_SAFE(do_render(hashData, bound_hash_params(), rayCastData, rayCastParams));
}

BF_API int bfRayCastSplat(const BFHashDataStruct* hashData, const BFHashParams* hashParams, const BFDepthCameraParams* cameraParams, const BFRayCastData* rayCastData,
                          const BFRayCastParams* rayCastParams) {
    return do_splat(hashData, hashParams, cameraParams, rayCastData, rayCastParams);
}
BF_API int bfRayCastRender(const BFHashDataStruct* hashData, const BFHashParams* hashParams, const BFRayCastData* rayCastData, const BFRayCastParams* rayCastParams) {
    return do_render(hashData, hashParams, rayCastData, rayCastParams);
}
BF_API int bfRayCastComputeNormals(const BFRayCastData* rayCastData, unsigned int width, unsigned int height) { return do_normals(rayCastData, width, height); }

BF_API int bfRayCastRenderPose(const BFHashDataStruct* hashData, const BFHashParams* hashParams, const BFDepthCameraParams* cameraParams, const BFRayCastData* rayCastData,
                               BFRayCastParams* rayCastParams, const float* rigidTransform) {
    if (!rayCastParams || !rigidTransform) return (int)cudaErrorInvalidValue;
    // CUDARayCastSDF::rayIntervalSplatting (cpp:86-98): view = inverse of the rigid transform
    float inv[16];
    for (int k = 0; k < 16; ++k) rayCastParams->m_viewMatrixInverse.m[k] = rigidTransform[k];
    bfMat4Inverse(rigidTransform, inv);                    // mat4f::getInverse as the host does it (include/bf_host.h)
    for (int k = 0; k < 16; ++k) rayCastParams->m_viewMatrix.m[k] = inv[k];
    int rc = do_splat(hashData, hashParams, cameraParams, rayCastData, rayCastParams);
    if (!rc) rc = do_render(hashData, hashParams, rayCastData, rayCastParams);
    if (!rc && !rayCastParams->m_useGradients) rc = do_normals(rayCastData, rayCastParams->m_width, rayCastParams->m_height);
    return rc;
}

// Projection and SH math of the rasterizer, stated once for the forward (raster_project.cu), the single-view backward
// (raster_project_bwd.cu) and the multi-view backward (raster_project_bwd_multi.cu).  The kernels are compositions of these
// helpers, each the arithmetic its callers used before, expression for expression.  The quaternion normalisation stays at
// the call sites: the forward uses 1 / sqrtf (compiled -fmad=false, it feeds the bit-exact tile keys), the backward rsqrtf,
// whose result it also needs for the normalisation gradient.
// Formulas: SURVEY.md App. B.1 (projection), B.2 (SH), B.6 (backward), pinned against torch.autograd by the tests.
#pragma once
#include "raster_common.cuh"

namespace {

// 3x3 row-major products: C = A B, C = A B^T, C = A^T B
__device__ __forceinline__ void mat3_mul(const float* A, const float* B, float* C) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            C[i * 3 + j] = A[i * 3 + 0] * B[0 * 3 + j] + A[i * 3 + 1] * B[1 * 3 + j] + A[i * 3 + 2] * B[2 * 3 + j];
}
__device__ __forceinline__ void mat3_mul_bt(const float* A, const float* B, float* C) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            C[i * 3 + j] = A[i * 3 + 0] * B[j * 3 + 0] + A[i * 3 + 1] * B[j * 3 + 1] + A[i * 3 + 2] * B[j * 3 + 2];
}
__device__ __forceinline__ void mat3_mul_at(const float* A, const float* B, float* C) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            C[i * 3 + j] = A[0 * 3 + i] * B[0 * 3 + j] + A[1 * 3 + i] * B[1 * 3 + j] + A[2 * 3 + i] * B[2 * 3 + j];
}

// Rotation matrix of the unit quaternion (w, x, y, z); the caller normalises.
__device__ __forceinline__ void quat_to_rotmat(float w, float qx, float qy, float qz, float* Rq) {
    const float x2 = qx * qx, y2 = qy * qy, z2 = qz * qz;
    const float xy = qx * qy, xz = qx * qz, yz = qy * qz, wx = w * qx, wy = w * qy, wz = w * qz;
    Rq[0] = 1.0f - 2.0f * (y2 + z2); Rq[1] = 2.0f * (xy - wz);        Rq[2] = 2.0f * (xz + wy);
    Rq[3] = 2.0f * (xy + wz);        Rq[4] = 1.0f - 2.0f * (x2 + z2); Rq[5] = 2.0f * (yz - wx);
    Rq[6] = 2.0f * (xz - wy);        Rq[7] = 2.0f * (yz + wx);        Rq[8] = 1.0f - 2.0f * (x2 + y2);
}

// World covariance: M = Rq diag(s), Sigma = M M^T
__device__ __forceinline__ void world_cov(const float* Rq, const float* s, float* M, float* Sigma) {
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) M[a * 3 + b] = Rq[a * 3 + b] * s[b];
    mat3_mul_bt(M, M, Sigma);
}

// Camera covariance: RS = R Sigma, Sc = R Sigma R^T (R: the view matrix's rotation)
__device__ __forceinline__ void cam_cov(const float* R, const float* Sigma, float* RS, float* Sc) {
    mat3_mul(R, Sigma, RS);
    mat3_mul_bt(RS, R, Sc);
}

// gsplat's perspective Jacobian at the camera-space point (x, y, z), with x / z and y / z clamped to the field of view
// widened by 0.3 tan(fov / 2) on each side.  J is the 2x3 Jacobian (row-major, J[1] = J[3] = 0); (tx, ty) the clamped
// point; clamp_x / clamp_y whether the clamp bit (its gradient then stops at the limit).
struct PerspJacobian {
    float rz, rz2, rz3, tx, ty;
    float J[6];
    bool clamp_x, clamp_y;
};
__device__ __forceinline__ PerspJacobian persp_jacobian(float x, float y, float z, float fx, float fy, float cx, float cy,
                                                        float W, float H) {
    PerspJacobian p;
    const float tanx = 0.5f * W / fx, tany = 0.5f * H / fy;
    const float lxp = (W - cx) / fx + 0.3f * tanx, lxn = cx / fx + 0.3f * tanx;
    const float lyp = (H - cy) / fy + 0.3f * tany, lyn = cy / fy + 0.3f * tany;
    p.rz = 1.0f / z;
    p.rz2 = p.rz * p.rz;
    p.rz3 = p.rz2 * p.rz;
    const float xr = x * p.rz, yr = y * p.rz;
    p.clamp_x = !(xr <= lxp && xr >= -lxn);
    p.clamp_y = !(yr <= lyp && yr >= -lyn);
    p.tx = z * fminf(lxp, fmaxf(-lxn, xr));
    p.ty = z * fminf(lyp, fmaxf(-lyn, yr));
    p.J[0] = fx * p.rz; p.J[1] = 0.f; p.J[2] = -fx * p.tx * p.rz2;
    p.J[3] = 0.f;       p.J[4] = fy * p.rz; p.J[5] = -fy * p.ty * p.rz2;
    return p;
}

// Real SH basis of degree <= 3 at the unit direction (x, y, z); B[k] = 0 above the degree.
__device__ __forceinline__ void sh_basis(int deg, float x, float y, float z, float* B) {
#pragma unroll
    for (int k = 0; k < 16; ++k) B[k] = 0.f;
    B[0] = 0.2820947917738781f;
    if (deg < 1) return;
    B[1] = -0.48860251190292f * y; B[2] = 0.48860251190292f * z; B[3] = -0.48860251190292f * x;
    if (deg < 2) return;
    const float z2 = z * z, fT0B = -1.092548430592079f * z;
    const float fC1 = x * x - y * y, fS1 = 2.f * x * y;
    B[4] = 0.5462742152960395f * fS1; B[5] = fT0B * y; B[6] = 0.9461746957575601f * z2 - 0.3153915652525201f;
    B[7] = fT0B * x; B[8] = 0.5462742152960395f * fC1;
    if (deg < 3) return;
    const float fT0C = -2.285228997322329f * z2 + 0.4570457994644658f, fT1B = 1.445305721320277f * z;
    const float fC2 = x * fC1 - y * fS1, fS2 = x * fS1 + y * fC1;
    B[9] = -0.5900435899266435f * fS2; B[10] = fT1B * fS1; B[11] = fT0C * y;
    B[12] = z * (1.865881662950577f * z2 - 1.119528997770346f); B[13] = fT0C * x; B[14] = fT1B * fC1;
    B[15] = -0.5900435899266435f * fC2;
}

// The same basis and its gradient (Bx, By, Bz) w.r.t. the unit direction.
__device__ __forceinline__ void sh_basis_grad(int deg, float x, float y, float z, float* B, float* Bx, float* By, float* Bz) {
#pragma unroll
    for (int k = 0; k < 16; ++k) B[k] = Bx[k] = By[k] = Bz[k] = 0.f;
    B[0] = 0.2820947917738781f;
    if (deg < 1) return;
    B[1] = -0.48860251190292f * y; B[2] = 0.48860251190292f * z; B[3] = -0.48860251190292f * x;
    By[1] = -0.48860251190292f; Bz[2] = 0.48860251190292f; Bx[3] = -0.48860251190292f;
    if (deg < 2) return;
    const float z2 = z * z, fT0B = -1.092548430592079f * z, fT0B_z = -1.092548430592079f;
    const float fC1 = x * x - y * y, fS1 = 2.f * x * y;
    const float fC1_x = 2.f * x, fC1_y = -2.f * y, fS1_x = 2.f * y, fS1_y = 2.f * x;
    B[4] = 0.5462742152960395f * fS1; B[5] = fT0B * y; B[6] = 0.9461746957575601f * z2 - 0.3153915652525201f;
    B[7] = fT0B * x; B[8] = 0.5462742152960395f * fC1;
    Bx[4] = 0.5462742152960395f * fS1_x; By[4] = 0.5462742152960395f * fS1_y;
    By[5] = fT0B; Bz[5] = fT0B_z * y;
    Bz[6] = 2.f * 0.9461746957575601f * z;
    Bx[7] = fT0B; Bz[7] = fT0B_z * x;
    Bx[8] = 0.5462742152960395f * fC1_x; By[8] = 0.5462742152960395f * fC1_y;
    if (deg < 3) return;
    const float fT0C = -2.285228997322329f * z2 + 0.4570457994644658f, fT0C_z = -2.285228997322329f * 2.f * z;
    const float fT1B = 1.445305721320277f * z, fT1B_z = 1.445305721320277f;
    const float fC2 = x * fC1 - y * fS1, fS2 = x * fS1 + y * fC1;
    const float fC2_x = fC1 + x * fC1_x - y * fS1_x, fC2_y = x * fC1_y - fS1 - y * fS1_y;
    const float fS2_x = fS1 + x * fS1_x + y * fC1_x, fS2_y = x * fS1_y + fC1 + y * fC1_y;
    B[9] = -0.5900435899266435f * fS2; B[10] = fT1B * fS1; B[11] = fT0C * y;
    B[12] = z * (1.865881662950577f * z2 - 1.119528997770346f); B[13] = fT0C * x; B[14] = fT1B * fC1;
    B[15] = -0.5900435899266435f * fC2;
    Bx[9] = -0.5900435899266435f * fS2_x; By[9] = -0.5900435899266435f * fS2_y;
    Bx[10] = fT1B * fS1_x; By[10] = fT1B * fS1_y; Bz[10] = fT1B_z * fS1;
    By[11] = fT0C; Bz[11] = fT0C_z * y;
    Bz[12] = 3.f * 1.865881662950577f * z2 - 1.119528997770346f;
    Bx[13] = fT0C; Bz[13] = fT0C_z * x;
    Bx[14] = fT1B * fC1_x; By[14] = fT1B * fC1_y; Bz[14] = fT1B_z * fC1;
    Bx[15] = -0.5900435899266435f * fC2_x; By[15] = -0.5900435899266435f * fC2_y;
}

// The 16x3 SH coefficients of Gaussian i, read by `readers` warps: more than one, an ordinary read-only load (the others
// read the same lines next); otherwise a streaming load that does not allocate in L1.
__device__ __forceinline__ void load_sh_coeffs(const float* sh, int i, int readers, float* c48) {
    const float4* sp = reinterpret_cast<const float4*>(sh + (size_t)i * 48);
#pragma unroll
    for (int k = 0; k < 12; ++k) {
        const float4 q = readers > 1 ? __ldg(sp + k) : adb_ldg_stream4(sp + k);
        c48[4 * k] = q.x; c48[4 * k + 1] = q.y; c48[4 * k + 2] = q.z; c48[4 * k + 3] = q.w;
    }
}

// ---- staging a CTA's parameter rows in shared memory -------------------------------------------------------------------
// One lane per Gaussian reading its own 192 B SH row makes every 16 B load instruction touch 32 different 128 B lines; copying
// a CTA's contiguous rows with consecutive threads on consecutive 16 B pieces touches each line once.  Staged SH rows are
// SH_ROW floats apart: 13 16-byte bank groups, odd, so 8 consecutive lanes' 16 B accesses to the same offset of their own rows
// fall in 8 distinct groups (48 floats would be a 16-way conflict).
constexpr int SH_ROW = 52;

// Asynchronous global -> shared copies (cp.async): 16 B bypassing L1, 4 B through it.  cp_async_wait_all waits for the
// calling thread's copies; a barrier then makes every thread's copies visible to the CTA.
__device__ __forceinline__ void cp_async16(void* s, const void* g) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(s)), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async4(void* s, const void* g) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(s)), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// Rows [first, first + n) of a [*, 48] table into shared rows of SH_ROW floats, by all threads of the CTA (asynchronous: the
// caller waits and synchronises).
__device__ __forceinline__ void stage_sh_rows(float* s, const float* g, int first, int n) {
    const float4* src = reinterpret_cast<const float4*>(g + (size_t)first * 48);
    for (int j = threadIdx.x; j < 12 * n; j += blockDim.x) {
        const int r = j / 12;
        cp_async16(s + r * SH_ROW + 4 * (j - 12 * r), src + j);
    }
}

// The reverse, after a barrier: shared rows of SH_ROW floats -> rows [first, first + n) of a [*, 48] table.
__device__ __forceinline__ void store_sh_rows(float* g, const float* s, int first, int n) {
    float4* dst = reinterpret_cast<float4*>(g + (size_t)first * 48);
    for (int j = threadIdx.x; j < 12 * n; j += blockDim.x) {
        const int r = j / 12;
        dst[j] = *reinterpret_cast<const float4*>(s + r * SH_ROW + 4 * (j - 12 * r));
    }
}

// n consecutive floats (4 B copies, for rows of 1 or 3 floats whose start need not be 16 B aligned).
__device__ __forceinline__ void stage_floats(float* s, const float* g, int n) {
    for (int j = threadIdx.x; j < n; j += blockDim.x) cp_async4(s + j, g + j);
}

// dL/dSigma -> dL/d(scales) and dL/d(quats) through Sigma = M M^T, M = Rq diag(s) (world_cov) and the normalisation of
// q = (w, qx, qy, qz) / qinv.
__device__ __forceinline__ void world_cov_bwd(const float* vSigma, const float* M, const float* Rq, const float* s, float w,
                                              float qx, float qy, float qz, float qinv, float* vs, float* vq) {
    float vM[9], vRq[9];
    mat3_mul(vSigma, M, vM);
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) {
            vM[a * 3 + b] *= 2.0f;
            vRq[a * 3 + b] = vM[a * 3 + b] * s[b];
        }
#pragma unroll
    for (int b = 0; b < 3; ++b) vs[b] = vM[b] * Rq[b] + vM[3 + b] * Rq[3 + b] + vM[6 + b] * Rq[6 + b];
    float vn[4];
    vn[0] = 2.0f * (qx * (vRq[7] - vRq[5]) + qy * (vRq[2] - vRq[6]) + qz * (vRq[3] - vRq[1]));
    vn[1] = 2.0f * (-2.0f * qx * (vRq[4] + vRq[8]) + qy * (vRq[1] + vRq[3]) + qz * (vRq[2] + vRq[6]) + w * (vRq[7] - vRq[5]));
    vn[2] = 2.0f * (qx * (vRq[1] + vRq[3]) - 2.0f * qy * (vRq[0] + vRq[8]) + qz * (vRq[5] + vRq[7]) + w * (vRq[2] - vRq[6]));
    vn[3] = 2.0f * (qx * (vRq[2] + vRq[6]) + qy * (vRq[5] + vRq[7]) - 2.0f * qz * (vRq[0] + vRq[4]) + w * (vRq[3] - vRq[1]));
    const float dotq = vn[0] * w + vn[1] * qx + vn[2] * qy + vn[3] * qz;
    vq[0] = (vn[0] - dotq * w) * qinv; vq[1] = (vn[1] - dotq * qx) * qinv;
    vq[2] = (vn[2] - dotq * qy) * qinv; vq[3] = (vn[3] - dotq * qz) * qinv;
}

}  // namespace

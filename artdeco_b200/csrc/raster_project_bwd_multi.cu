// Multi-view backward of projection + SH: C cameras of the SAME Gaussians in one pass per stage.
//
// The reference renders one view per optimiser step (h3dgsv3.py:406-464) and lets autograd sum nothing; BASELINE config 4
// ("8-view batch optimise", SURVEY.md §8e) sums the gradients of C views.  Running the single-view backward C times costs
// C x (236 B read + 236 B written + a [N,59] accumulate) per Gaussian.  Here:
//   project_bwd_multi  one thread per Gaussian loops over the C cameras: parameters are read once, the camera-independent
//                      parts (quaternion rotation, Sigma) are computed once, the 11 geometry gradients are summed in
//                      registers and written once; per camera it reads only the 48 B record + 48 B accumulator and emits
//                      the 12 B clamp-masked colour gradient g_rgb[c][i];
//   sh_bwd_multi       v_sh[i] = sum_c basis(dir_c) (x) g_rgb[c][i] in registers, one 192 B write per Gaussian; the
//                      direction term is added to v_means.
// The split is also what makes the multi-GPU exchange cheap (artdeco_b200/parallel.py): ranks all-gather g_rgb (12 B per view
// and Gaussian) and all-reduce only the 11 geometry floats instead of all-reducing 59 floats; every rank then expands the SH
// gradient of ALL views locally.  Formulas: raster_project_bwd.cu (SURVEY.md App. B.6), pinned by tests against the sum of
// single-view backward passes.
#include "raster_common.cuh"

namespace {

__device__ __forceinline__ void m3_mul(const float* A, const float* B, float* C) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            C[i * 3 + j] = A[i * 3 + 0] * B[0 * 3 + j] + A[i * 3 + 1] * B[1 * 3 + j] + A[i * 3 + 2] * B[2 * 3 + j];
}
__device__ __forceinline__ void m3_mul_bt(const float* A, const float* B, float* C) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            C[i * 3 + j] = A[i * 3 + 0] * B[j * 3 + 0] + A[i * 3 + 1] * B[j * 3 + 1] + A[i * 3 + 2] * B[j * 3 + 2];
}
__device__ __forceinline__ void m3_mul_at(const float* A, const float* B, float* C) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            C[i * 3 + j] = A[0 * 3 + i] * B[0 * 3 + j] + A[1 * 3 + i] * B[1 * 3 + j] + A[2 * 3 + i] * B[2 * 3 + j];
}

constexpr int PB = 128;

__global__ void __launch_bounds__(PB)
project_bwd_multi_kernel(int N, int C, const float* __restrict__ means, const float* __restrict__ quats,
                         const float* __restrict__ scales, const float* __restrict__ viewmats,
                         const float* __restrict__ Ks, int W, int H, const int32_t* __restrict__ radii,
                         const float* __restrict__ splats, const float* __restrict__ v_splats,
                         float* __restrict__ v_means, float* __restrict__ v_quats, float* __restrict__ v_scales,
                         float* __restrict__ v_opac, float* __restrict__ g_rgb, float* __restrict__ v_viewmats) {
    __shared__ float sRed[PB / 32][12];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = i < N;
    float mu[3] = {0.f, 0.f, 0.f}, s[3] = {1.f, 1.f, 1.f};
    float w = 1.f, qx = 0.f, qy = 0.f, qz = 0.f, qinv = 1.f;
    if (in) {
        mu[0] = means[3 * i]; mu[1] = means[3 * i + 1]; mu[2] = means[3 * i + 2];
        const float4 q4 = reinterpret_cast<const float4*>(quats)[i];
        qinv = rsqrtf(q4.x * q4.x + q4.y * q4.y + q4.z * q4.z + q4.w * q4.w);
        w = q4.x * qinv; qx = q4.y * qinv; qy = q4.z * qinv; qz = q4.w * qinv;
        s[0] = scales[3 * i]; s[1] = scales[3 * i + 1]; s[2] = scales[3 * i + 2];
    }
    float Rq[9], M[9], Sigma[9];
    {
        const float x2 = qx * qx, y2 = qy * qy, z2 = qz * qz;
        const float xy = qx * qy, xz = qx * qz, yz = qy * qz, wx = w * qx, wy = w * qy, wz = w * qz;
        Rq[0] = 1.0f - 2.0f * (y2 + z2); Rq[1] = 2.0f * (xy - wz);        Rq[2] = 2.0f * (xz + wy);
        Rq[3] = 2.0f * (xy + wz);        Rq[4] = 1.0f - 2.0f * (x2 + z2); Rq[5] = 2.0f * (yz - wx);
        Rq[6] = 2.0f * (xz - wy);        Rq[7] = 2.0f * (yz + wx);        Rq[8] = 1.0f - 2.0f * (x2 + y2);
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int b = 0; b < 3; ++b) M[a * 3 + b] = Rq[a * 3 + b] * s[b];
        m3_mul_bt(M, M, Sigma);
    }
    float vm[3] = {0.f, 0.f, 0.f}, vo = 0.f;
    float vSigma_acc[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) vSigma_acc[k] = 0.f;

    for (int c = 0; c < C; ++c) {
        float red[12];
#pragma unroll
        for (int k = 0; k < 12; ++k) red[k] = 0.f;
        bool live = false;
        if (in) {
            const int2 r = reinterpret_cast<const int2*>(radii)[(size_t)c * N + i];
            live = (r.x > 0 || r.y > 0);
        }
        float grgb[3] = {0.f, 0.f, 0.f};
        if (live) {
            const float* V = viewmats + 16 * c;
            const float* K = Ks + 9 * c;
            const float R[9] = {V[0], V[1], V[2], V[4], V[5], V[6], V[8], V[9], V[10]};
            const float t[3] = {V[3], V[7], V[11]};
            const float fx = K[0], fy = K[4], cx = K[2], cy = K[5];
            const float x = R[0] * mu[0] + R[1] * mu[1] + R[2] * mu[2] + t[0];
            const float y = R[3] * mu[0] + R[4] * mu[1] + R[5] * mu[2] + t[1];
            const float z = R[6] * mu[0] + R[7] * mu[1] + R[8] * mu[2] + t[2];
            float RS[9], Sc[9];
            m3_mul(R, Sigma, RS);
            m3_mul_bt(RS, R, Sc);
            const float Wf = (float)W, Hf = (float)H;
            const float tanx = 0.5f * Wf / fx, tany = 0.5f * Hf / fy;
            const float lxp = (Wf - cx) / fx + 0.3f * tanx, lxn = cx / fx + 0.3f * tanx;
            const float lyp = (Hf - cy) / fy + 0.3f * tany, lyn = cy / fy + 0.3f * tany;
            const float rz = 1.0f / z, rz2 = rz * rz, rz3 = rz2 * rz;
            const float xr = x * rz, yr = y * rz;
            const bool clamp_x = !(xr <= lxp && xr >= -lxn), clamp_y = !(yr <= lyp && yr >= -lyn);
            const float tx = z * fminf(lxp, fmaxf(-lxn, xr)), ty = z * fminf(lyp, fmaxf(-lyn, yr));
            const float J[6] = {fx * rz, 0.f, -fx * tx * rz2, 0.f, fy * rz, -fy * ty * rz2};

            const size_t off = ((size_t)c * N + i) * ADB_SPLAT_STRIDE;
            const float4 rec0 = reinterpret_cast<const float4*>(splats + off)[0];
            const float4 rec1 = reinterpret_cast<const float4*>(splats + off)[1];
            const float4 rec2 = reinterpret_cast<const float4*>(splats + off)[2];
            const float4 g0 = reinterpret_cast<const float4*>(v_splats + off)[0];
            const float4 g1 = reinterpret_cast<const float4*>(v_splats + off)[1];
            const float4 g2 = reinterpret_cast<const float4*>(v_splats + off)[2];
            const float A = rec0.z, B = rec0.w, Cc = rec1.x;
            const float vu = A * g0.x + B * g0.y, vv = B * g0.x + Cc * g0.y;
            const float gA = 0.5f * g0.z, gB = 0.5f * g0.w, gC = 0.5f * g1.x;
            vo += -g1.y / rec1.y;
            grgb[0] = rec2.x > 0.f ? g1.z : 0.f;
            grgb[1] = rec2.y > 0.f ? g1.w : 0.f;
            grgb[2] = rec2.z > 0.f ? g2.x : 0.f;
            const float v_depth = g2.y;
            const float q00 = A * gA + B * gB, q01 = A * gB + B * gC, q10 = B * gA + Cc * gB, q11 = B * gB + Cc * gC;
            const float V00 = -(q00 * A + q01 * B), V01 = -(q00 * B + q01 * Cc), V10 = -(q10 * A + q11 * B),
                        V11 = -(q10 * B + q11 * Cc);
            float VJ[6];
#pragma unroll
            for (int b = 0; b < 3; ++b) {
                VJ[b] = V00 * J[b] + V01 * J[3 + b];
                VJ[3 + b] = V10 * J[b] + V11 * J[3 + b];
            }
            float vSc[9], vJ[6];
#pragma unroll
            for (int a = 0; a < 3; ++a)
#pragma unroll
                for (int b = 0; b < 3; ++b) vSc[a * 3 + b] = J[a] * VJ[b] + J[3 + a] * VJ[3 + b];
#pragma unroll
            for (int a = 0; a < 2; ++a)
#pragma unroll
                for (int b = 0; b < 3; ++b)
                    vJ[a * 3 + b] = 2.0f * (VJ[a * 3 + 0] * Sc[0 * 3 + b] + VJ[a * 3 + 1] * Sc[1 * 3 + b] + VJ[a * 3 + 2] * Sc[2 * 3 + b]);
            float vp[3];
            vp[0] = fx * rz * vu;
            vp[1] = fy * rz * vv;
            vp[2] = -(fx * x * vu + fy * y * vv) * rz2 + v_depth;
            vp[2] += -fx * rz2 * vJ[0] - fy * rz2 * vJ[4];
            if (!clamp_x) { vp[0] += -fx * rz2 * vJ[2]; vp[2] += 2.0f * fx * tx * rz3 * vJ[2]; }
            else          { vp[2] += fx * tx * rz3 * vJ[2]; }
            if (!clamp_y) { vp[1] += -fy * rz2 * vJ[5]; vp[2] += 2.0f * fy * ty * rz3 * vJ[5]; }
            else          { vp[2] += fy * ty * rz3 * vJ[5]; }
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                vm[a] += R[0 * 3 + a] * vp[0] + R[1 * 3 + a] * vp[1] + R[2 * 3 + a] * vp[2];
                red[9 + a] = vp[a];
#pragma unroll
                for (int b = 0; b < 3; ++b) red[a * 3 + b] = vp[a] * mu[b];
            }
            float tmp[9], vSigma[9], add[9];
            m3_mul_at(R, vSc, tmp);
            m3_mul(tmp, R, vSigma);
            m3_mul(vSc, RS, add);
#pragma unroll
            for (int k = 0; k < 9; ++k) { red[k] += 2.0f * add[k]; vSigma_acc[k] += vSigma[k]; }
        }
        if (in && g_rgb) {
            float* o = g_rgb + ((size_t)c * N + i) * 3;
            o[0] = grgb[0]; o[1] = grgb[1]; o[2] = grgb[2];
        }
        // block reduction of this camera's 12 view-matrix gradient terms
#pragma unroll
        for (int k = 0; k < 12; ++k) red[k] = adb_warp_sum(red[k]);
        const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
        __syncthreads();
        if (lane == 0)
#pragma unroll
            for (int k = 0; k < 12; ++k) sRed[wid][k] = red[k];
        __syncthreads();
        if (threadIdx.x < 12) {
            float v = 0.f;
#pragma unroll
            for (int w_ = 0; w_ < PB / 32; ++w_) v += sRed[w_][threadIdx.x];
            if (v != 0.f) {
                const int k = threadIdx.x;
                float* vv_ = v_viewmats + 16 * c;
                if (k < 9) atomicAdd(vv_ + (k / 3) * 4 + (k % 3), v);
                else atomicAdd(vv_ + (k - 9) * 4 + 3, v);
            }
        }
    }
    if (!in) return;
    // Sigma = M M^T chain, once for the summed v_Sigma (linear in v_Sigma)
    float vM[9], vRq[9], vs[3], vq[4];
    m3_mul(vSigma_acc, M, vM);
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
    v_means[3 * i] = vm[0]; v_means[3 * i + 1] = vm[1]; v_means[3 * i + 2] = vm[2];
    reinterpret_cast<float4*>(v_quats)[i] = make_float4(vq[0], vq[1], vq[2], vq[3]);
    v_scales[3 * i] = vs[0]; v_scales[3 * i + 1] = vs[1]; v_scales[3 * i + 2] = vs[2];
    v_opac[i] = vo;
}

// basis and its gradient w.r.t. the unit direction, degree <= 3 (same polynomials as raster_project_bwd.cu)
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

__global__ void __launch_bounds__(PB)
sh_bwd_multi_kernel(int N, int C, const float* __restrict__ means, const float* __restrict__ sh, int sh_degree,
                    const float* __restrict__ campos, const float* __restrict__ g_rgb, float* __restrict__ v_sh,
                    float* __restrict__ v_means, int accumulate, int skip_mod, int skip_val,
                    float* __restrict__ v_campos) {
    __shared__ float sRed[PB / 32][3];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = i < N;
    float mu[3] = {0.f, 0.f, 0.f};
    float c48[48], o48[48];
#pragma unroll
    for (int k = 0; k < 48; ++k) { c48[k] = 0.f; o48[k] = 0.f; }
    if (in) {
        mu[0] = means[3 * i]; mu[1] = means[3 * i + 1]; mu[2] = means[3 * i + 2];
        const float4* sp = reinterpret_cast<const float4*>(sh + (size_t)i * 48);
#pragma unroll
        for (int k = 0; k < 12; ++k) {
            const float4 q = adb_ldg_stream4(sp + k);
            c48[4 * k] = q.x; c48[4 * k + 1] = q.y; c48[4 * k + 2] = q.z; c48[4 * k + 3] = q.w;
        }
        if (accumulate & 2) {            // second pass of a split expansion: continue from the stored partial sums
            const float4* op0 = reinterpret_cast<const float4*>(v_sh + (size_t)i * 48);
#pragma unroll
            for (int k = 0; k < 12; ++k) {
                const float4 q = op0[k];
                o48[4 * k] = q.x; o48[4 * k + 1] = q.y; o48[4 * k + 2] = q.z; o48[4 * k + 3] = q.w;
            }
        }
    }
    float gm[3] = {0.f, 0.f, 0.f};
    // software pipeline: the colour gradient of view c+1 is in flight while view c is expanded.  (A two-lanes-per-Gaussian
    // split of the 16 coefficients duplicates the basis evaluation, which costs more than the halved register footprint buys.)
    float gn[3] = {0.f, 0.f, 0.f};
    if (in) {
        const float* gp = g_rgb + (size_t)i * 3;
        gn[0] = gp[0]; gn[1] = gp[1]; gn[2] = gp[2];
    }
    for (int c = 0; c < C; ++c) {
        float red[3] = {0.f, 0.f, 0.f};
        const float g[3] = {gn[0], gn[1], gn[2]};
        if (in && c + 1 < C) {
            const float* gp = g_rgb + ((size_t)(c + 1) * N + i) * 3;
            gn[0] = gp[0]; gn[1] = gp[1]; gn[2] = gp[2];
        }
        const bool skip = skip_mod > 0 && (c % skip_mod) == skip_val;     // views already expanded by the first pass
        if (!skip && (g[0] != 0.f || g[1] != 0.f || g[2] != 0.f)) {
            const float dx = mu[0] - campos[3 * c], dy = mu[1] - campos[3 * c + 1], dz = mu[2] - campos[3 * c + 2];
            const float inv = rsqrtf(dx * dx + dy * dy + dz * dz);
            const float nx = dx * inv, ny = dy * inv, nz = dz * inv;
            float Bs[16], Bx[16], By[16], Bz[16];
            sh_basis_grad(sh_degree, nx, ny, nz, Bs, Bx, By, Bz);
            float vnx = 0.f, vny = 0.f, vnz = 0.f;
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                // s_k = <coefficients of band k, g>: one dot product feeds the three direction-gradient sums
                const float sk = fmaf(c48[3 * k], g[0], fmaf(c48[3 * k + 1], g[1], c48[3 * k + 2] * g[2]));
                vnx = fmaf(Bx[k], sk, vnx); vny = fmaf(By[k], sk, vny); vnz = fmaf(Bz[k], sk, vnz);
                o48[3 * k] = fmaf(Bs[k], g[0], o48[3 * k]);
                o48[3 * k + 1] = fmaf(Bs[k], g[1], o48[3 * k + 1]);
                o48[3 * k + 2] = fmaf(Bs[k], g[2], o48[3 * k + 2]);
            }
            const float dot = vnx * nx + vny * ny + vnz * nz;
            const float gx = (vnx - dot * nx) * inv, gy = (vny - dot * ny) * inv, gz = (vnz - dot * nz) * inv;
            gm[0] += gx; gm[1] += gy; gm[2] += gz;
            red[0] = -gx; red[1] = -gy; red[2] = -gz;
        }
        if (v_campos) {
#pragma unroll
            for (int k = 0; k < 3; ++k) red[k] = adb_warp_sum(red[k]);
            const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
            __syncthreads();
            if (lane == 0) { sRed[wid][0] = red[0]; sRed[wid][1] = red[1]; sRed[wid][2] = red[2]; }
            __syncthreads();
            if (threadIdx.x < 3) {
                float v = 0.f;
#pragma unroll
                for (int w_ = 0; w_ < PB / 32; ++w_) v += sRed[w_][threadIdx.x];
                if (v != 0.f) atomicAdd(v_campos + 3 * c + threadIdx.x, v);
            }
        }
    }
    if (!in) return;
    float4* op = reinterpret_cast<float4*>(v_sh + (size_t)i * 48);
#pragma unroll
    for (int k = 0; k < 12; ++k) op[k] = make_float4(o48[4 * k], o48[4 * k + 1], o48[4 * k + 2], o48[4 * k + 3]);
    if (accumulate & 1) { v_means[3 * i] += gm[0]; v_means[3 * i + 1] += gm[1]; v_means[3 * i + 2] += gm[2]; }
    else                { v_means[3 * i] = gm[0];  v_means[3 * i + 1] = gm[1];  v_means[3 * i + 2] = gm[2]; }
}


// ---- split form of the SH backward for the multi-GPU step -------------------------------------------------------------------
// The fused kernel above does two things per (Gaussian, view): the outer product basis(dir) (x) g into v_sh, and the gradient of
// the colour through the view DIRECTION into v_means.  Only the first needs the other ranks' colour gradients; the second is
// linear in the views, so each rank computes it for its LOCAL views and the geometry all-reduce sums it.  That leaves the
// replicated part — the expansion of ALL views on every rank — without the 192 B coefficient read, the basis gradients and
// half of the registers.

// basis values only, degree <= 3
__device__ __forceinline__ void sh_basis_values(int deg, float x, float y, float z, float* B) {
#pragma unroll
    for (int k = 1; k < 16; ++k) B[k] = 0.f;
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

// v_sh[i] = sum_c basis(dir_c(i)) (x) g_rgb[c][i]   (overwritten)
__global__ void __launch_bounds__(PB)
sh_expand_multi_kernel(int N, int C, const float* __restrict__ means, int sh_degree, const float* __restrict__ campos,
                       const float* __restrict__ g_rgb, float* __restrict__ v_sh) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const float mx = means[3 * i], my = means[3 * i + 1], mz = means[3 * i + 2];
    float o48[48];
#pragma unroll
    for (int k = 0; k < 48; ++k) o48[k] = 0.f;
    const float* gp = g_rgb + (size_t)i * 3;
    float gn0 = gp[0], gn1 = gp[1], gn2 = gp[2];
    for (int c = 0; c < C; ++c) {
        const float g0 = gn0, g1 = gn1, g2 = gn2;
        if (c + 1 < C) {                                  // next view's colour gradient in flight while this one is expanded
            const float* gq = g_rgb + ((size_t)(c + 1) * N + i) * 3;
            gn0 = gq[0]; gn1 = gq[1]; gn2 = gq[2];
        }
        if (g0 == 0.f && g1 == 0.f && g2 == 0.f) continue;
        const float dx = mx - campos[3 * c], dy = my - campos[3 * c + 1], dz = mz - campos[3 * c + 2];
        const float inv = rsqrtf(dx * dx + dy * dy + dz * dz);
        float Bs[16];
        sh_basis_values(sh_degree, dx * inv, dy * inv, dz * inv, Bs);
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            o48[3 * k] = fmaf(Bs[k], g0, o48[3 * k]);
            o48[3 * k + 1] = fmaf(Bs[k], g1, o48[3 * k + 1]);
            o48[3 * k + 2] = fmaf(Bs[k], g2, o48[3 * k + 2]);
        }
    }
    float4* op = reinterpret_cast<float4*>(v_sh + (size_t)i * 48);
#pragma unroll
    for (int k = 0; k < 12; ++k) op[k] = make_float4(o48[4 * k], o48[4 * k + 1], o48[4 * k + 2], o48[4 * k + 3]);
}

// v_means[i] += sum over the LOCAL views of the colour gradient pulled back through the view direction; v_campos[c] gets the
// opposite.  The colour gradient of view c is taken from the blend backward's accumulators with the SH clamp mask applied
// (splats[c][i].rgb > 0 ? v_splats[c][i][6:9] : 0 — raster.mask_rgb_grad).
__global__ void __launch_bounds__(PB)
sh_dir_bwd_multi_kernel(int N, int C, const float* __restrict__ means, const float* __restrict__ sh, int sh_degree,
                        const float* __restrict__ campos, const float* __restrict__ splats, const float* __restrict__ v_splats,
                        float* __restrict__ v_means, float* __restrict__ v_campos) {
    __shared__ float sRed[PB / 32][3];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = i < N;
    float mu[3] = {0.f, 0.f, 0.f};
    float c48[48];
#pragma unroll
    for (int k = 0; k < 48; ++k) c48[k] = 0.f;
    if (in) {
        mu[0] = means[3 * i]; mu[1] = means[3 * i + 1]; mu[2] = means[3 * i + 2];
        const float4* sp = reinterpret_cast<const float4*>(sh + (size_t)i * 48);
#pragma unroll
        for (int k = 0; k < 12; ++k) {
            const float4 q = adb_ldg_stream4(sp + k);
            c48[4 * k] = q.x; c48[4 * k + 1] = q.y; c48[4 * k + 2] = q.z; c48[4 * k + 3] = q.w;
        }
    }
    float gm[3] = {0.f, 0.f, 0.f};
    for (int c = 0; c < C; ++c) {
        float red[3] = {0.f, 0.f, 0.f};
        float g[3] = {0.f, 0.f, 0.f};
        if (in) {
            const size_t rec = ((size_t)c * N + i) * ADB_SPLAT_STRIDE;
            const float4 Cc = __ldg(reinterpret_cast<const float4*>(splats + rec) + 2);
            const float4 v1 = __ldg(reinterpret_cast<const float4*>(v_splats + rec) + 1);
            const float4 v2 = __ldg(reinterpret_cast<const float4*>(v_splats + rec) + 2);
            g[0] = Cc.x > 0.f ? v1.z : 0.f;
            g[1] = Cc.y > 0.f ? v1.w : 0.f;
            g[2] = Cc.z > 0.f ? v2.x : 0.f;
        }
        if (g[0] != 0.f || g[1] != 0.f || g[2] != 0.f) {
            const float dx = mu[0] - campos[3 * c], dy = mu[1] - campos[3 * c + 1], dz = mu[2] - campos[3 * c + 2];
            const float inv = rsqrtf(dx * dx + dy * dy + dz * dz);
            const float nx = dx * inv, ny = dy * inv, nz = dz * inv;
            float Bs[16], Bx[16], By[16], Bz[16];
            sh_basis_grad(sh_degree, nx, ny, nz, Bs, Bx, By, Bz);
            float vnx = 0.f, vny = 0.f, vnz = 0.f;
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                const float sk = fmaf(c48[3 * k], g[0], fmaf(c48[3 * k + 1], g[1], c48[3 * k + 2] * g[2]));
                vnx = fmaf(Bx[k], sk, vnx); vny = fmaf(By[k], sk, vny); vnz = fmaf(Bz[k], sk, vnz);
            }
            const float dot = vnx * nx + vny * ny + vnz * nz;
            const float gx = (vnx - dot * nx) * inv, gy = (vny - dot * ny) * inv, gz = (vnz - dot * nz) * inv;
            gm[0] += gx; gm[1] += gy; gm[2] += gz;
            red[0] = -gx; red[1] = -gy; red[2] = -gz;
        }
        if (v_campos) {
#pragma unroll
            for (int k = 0; k < 3; ++k) red[k] = adb_warp_sum(red[k]);
            const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
            __syncthreads();
            if (lane == 0) { sRed[wid][0] = red[0]; sRed[wid][1] = red[1]; sRed[wid][2] = red[2]; }
            __syncthreads();
            if (threadIdx.x < 3) {
                float v = 0.f;
#pragma unroll
                for (int w_ = 0; w_ < PB / 32; ++w_) v += sRed[w_][threadIdx.x];
                if (v != 0.f) atomicAdd(v_campos + 3 * c + threadIdx.x, v);
            }
        }
    }
    if (!in) return;
    v_means[3 * i] += gm[0]; v_means[3 * i + 1] += gm[1]; v_means[3 * i + 2] += gm[2];
}

}  // namespace

// Geometry gradients of C views summed per Gaussian.  radii [C,N,2], splats / v_splats [C,N,12] (stacked per camera),
// viewmats [C,16], Ks [C,9] on the device.  v_means / v_quats / v_scales / v_opac [N,*] are OVERWRITTEN with the sum over
// cameras; g_rgb [C,N,3] (may be NULL) receives the colour gradient masked by the SH clamp and by visibility;
// v_viewmats [C,16] is ACCUMULATED (caller zeroes it).
ADB_API int adb_raster_project_bwd_multi(int N, int C, const float* means, const float* quats, const float* scales,
                                         const float* viewmats, const float* Ks, int W, int H, const int32_t* radii,
                                         const float* splats, const float* v_splats, float* v_means, float* v_quats,
                                         float* v_scales, float* v_opac, float* g_rgb, float* v_viewmats,
                                         cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && C >= 1 && W > 0 && H > 0, "adb_raster_project_bwd_multi: bad sizes");
    if (N == 0) return ADB_OK;
    ADB_REQUIRE(means && quats && scales && viewmats && Ks && radii && splats && v_splats && v_means && v_quats &&
                    v_scales && v_opac && v_viewmats,
                "adb_raster_project_bwd_multi: null pointer");
    project_bwd_multi_kernel<<<adb_cdiv(N, PB), PB, 0, stream>>>(N, C, means, quats, scales, viewmats, Ks, W, H, radii,
                                                                splats, v_splats, v_means, v_quats, v_scales, v_opac,
                                                                g_rgb, v_viewmats);
    ADB_CHECK_LAUNCH("project_bwd_multi_kernel");
    return ADB_OK;
}

// v_sh [N,48] = sum_c basis(dir_c) (x) g_rgb[c]; the direction term goes to v_means [N,3].  accumulate bit 0: v_means += (else
// =: a separate buffer, so that an all-reduce of the geometry gradients can be in flight meanwhile); bit 1: v_sh += (else =).
// skip_mod > 0 skips the views c with c % skip_mod == skip_val — the second pass of a split expansion (multi-GPU: the local
// views are expanded while the other ranks' colour gradients are still being gathered; in the view-major gathered table
// [C_local, world] the local entries are those with c % world == rank).  v_campos [C,3] (may be NULL) accumulated.  g_rgb
// may hold views rendered on OTHER GPUs: only their campos[C,3] is needed.
ADB_API int adb_raster_sh_bwd_multi(int N, int C, const float* means, const float* sh, int sh_degree,
                                    const float* campos, const float* g_rgb, float* v_sh, float* v_means,
                                    int accumulate, int skip_mod, int skip_val, float* v_campos, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && C >= 1 && sh_degree >= 0 && sh_degree <= 3, "adb_raster_sh_bwd_multi: bad sizes");
    if (N == 0) return ADB_OK;
    ADB_REQUIRE(means && sh && campos && g_rgb && v_sh && v_means, "adb_raster_sh_bwd_multi: null pointer");
    sh_bwd_multi_kernel<<<adb_cdiv(N, PB), PB, 0, stream>>>(N, C, means, sh, sh_degree, campos, g_rgb, v_sh, v_means,
                                                           accumulate, skip_mod, skip_val, v_campos);
    ADB_CHECK_LAUNCH("sh_bwd_multi_kernel");
    return ADB_OK;
}

// Split form for the multi-GPU step (see the kernels): adb_raster_sh_dir_bwd_multi adds the LOCAL views' direction term to
// v_means [N,3] (and v_campos [C,3], may be NULL) straight from the blend backward's accumulators splats / v_splats [C,N,12];
// adb_raster_sh_expand_multi overwrites v_sh [N,48] with sum_c basis(dir_c) (x) g_rgb[c] over ALL views (g_rgb [C,N,3] and
// campos [C,3] may hold views rendered on other GPUs).  Together they equal adb_raster_sh_bwd_multi.
ADB_API int adb_raster_sh_dir_bwd_multi(int N, int C, const float* means, const float* sh, int sh_degree, const float* campos,
                                        const float* splats, const float* v_splats, float* v_means, float* v_campos,
                                        cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && C >= 1 && sh_degree >= 0 && sh_degree <= 3, "adb_raster_sh_dir_bwd_multi: bad sizes");
    if (N == 0) return ADB_OK;
    ADB_REQUIRE(means && sh && campos && splats && v_splats && v_means, "adb_raster_sh_dir_bwd_multi: null pointer");
    sh_dir_bwd_multi_kernel<<<adb_cdiv(N, PB), PB, 0, stream>>>(N, C, means, sh, sh_degree, campos, splats, v_splats, v_means,
                                                               v_campos);
    ADB_CHECK_LAUNCH("sh_dir_bwd_multi_kernel");
    return ADB_OK;
}
ADB_API int adb_raster_sh_expand_multi(int N, int C, const float* means, int sh_degree, const float* campos, const float* g_rgb,
                                       float* v_sh, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && C >= 1 && sh_degree >= 0 && sh_degree <= 3, "adb_raster_sh_expand_multi: bad sizes");
    if (N == 0) return ADB_OK;
    ADB_REQUIRE(means && campos && g_rgb && v_sh, "adb_raster_sh_expand_multi: null pointer");
    sh_expand_multi_kernel<<<adb_cdiv(N, PB), PB, 0, stream>>>(N, C, means, sh_degree, campos, g_rgb, v_sh);
    ADB_CHECK_LAUNCH("sh_expand_multi_kernel");
    return ADB_OK;
}

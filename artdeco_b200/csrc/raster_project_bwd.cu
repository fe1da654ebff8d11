// Per-Gaussian backward of projection + SH: v_splats (accumulated by blend_bwd) -> gradients of the
// Gaussian parameters, the view matrix and the camera centre.  One streaming pass: the forward
// intermediates (Sigma, J, ...) are recomputed from the 44 B of geometry instead of being stored.
//
// Replaces gsplat's fully_fused_projection_bwd + spherical_harmonics_bwd reached through autograd of
// Reconstruct/scene/scene_models/h3dgsv3.py:664-680 (SURVEY.md App. B.6).  Formulas are the analytic
// backward pinned against torch.autograd in tests/test_oracle_raster.py; the projection, covariance and SH pieces
// shared with the forward and the multi-view backward are in raster_geom.cuh.
#include "raster_geom.cuh"

namespace {

constexpr int PB = 128;  // threads per block (register heavy kernel)

__global__ void __launch_bounds__(PB)
project_bwd_kernel(int N, const float* __restrict__ means, const float* __restrict__ quats,
                   const float* __restrict__ scales, const float* __restrict__ sh, int sh_degree, AdbCam cam,
                   const int32_t* __restrict__ radii, const float* __restrict__ splats,
                   const float* __restrict__ v_splats, float* __restrict__ v_means, float* __restrict__ v_quats,
                   float* __restrict__ v_scales, float* __restrict__ v_opac, float* __restrict__ v_sh,
                   float* __restrict__ v_viewmat, float* __restrict__ v_campos) {
    __shared__ float sRed[PB / 32][15];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float red[15];
#pragma unroll
    for (int k = 0; k < 15; ++k) red[k] = 0.f;

    bool live = false;
    if (i < N) {
        const int2 r = reinterpret_cast<const int2*>(radii)[i];
        live = (r.x > 0 || r.y > 0);
    }
    float vm[3] = {0.f, 0.f, 0.f}, vq[4] = {0.f, 0.f, 0.f, 0.f}, vs[3] = {0.f, 0.f, 0.f}, vo = 0.f;
    if (live) {
        const float* V = cam.viewmat;
        const float R[9] = {V[0], V[1], V[2], V[4], V[5], V[6], V[8], V[9], V[10]};
        const float t[3] = {V[3], V[7], V[11]};
        const float fx = cam.K[0], fy = cam.K[4], cx = cam.K[2], cy = cam.K[5];
        const float mu[3] = {means[3 * i], means[3 * i + 1], means[3 * i + 2]};
        const float x = R[0] * mu[0] + R[1] * mu[1] + R[2] * mu[2] + t[0];
        const float y = R[3] * mu[0] + R[4] * mu[1] + R[5] * mu[2] + t[1];
        const float z = R[6] * mu[0] + R[7] * mu[1] + R[8] * mu[2] + t[2];
        const float4 q4 = reinterpret_cast<const float4*>(quats)[i];
        const float qinv = rsqrtf(q4.x * q4.x + q4.y * q4.y + q4.z * q4.z + q4.w * q4.w);
        const float w = q4.x * qinv, qx = q4.y * qinv, qy = q4.z * qinv, qz = q4.w * qinv;
        float Rq[9], M[9], Sigma[9], RS[9], Sc[9];
        quat_to_rotmat(w, qx, qy, qz, Rq);
        const float s[3] = {scales[3 * i], scales[3 * i + 1], scales[3 * i + 2]};
        world_cov(Rq, s, M, Sigma);
        cam_cov(R, Sigma, RS, Sc);
        const PerspJacobian pj = persp_jacobian(x, y, z, fx, fy, cx, cy, (float)cam.W, (float)cam.H);

        const float4 rec0 = reinterpret_cast<const float4*>(splats + (size_t)i * ADB_SPLAT_STRIDE)[0];
        const float4 rec1 = reinterpret_cast<const float4*>(splats + (size_t)i * ADB_SPLAT_STRIDE)[1];
        const float4 rec2 = reinterpret_cast<const float4*>(splats + (size_t)i * ADB_SPLAT_STRIDE)[2];
        const float4 g0 = reinterpret_cast<const float4*>(v_splats + (size_t)i * ADB_SPLAT_STRIDE)[0];
        const float4 g1 = reinterpret_cast<const float4*>(v_splats + (size_t)i * ADB_SPLAT_STRIDE)[1];
        const float4 g2 = reinterpret_cast<const float4*>(v_splats + (size_t)i * ADB_SPLAT_STRIDE)[2];
        const float* J = pj.J;
        const float rz = pj.rz, rz2 = pj.rz2, rz3 = pj.rz3, tx = pj.tx, ty = pj.ty;
        const bool clamp_x = pj.clamp_x, clamp_y = pj.clamp_y;
        const float A = rec0.z, B = rec0.w, C = rec1.x;
        // blend_bwd accumulates raw moments of v_sigma about the splat centre (slots 0..5 = M1x M1y M2xx M2xy M2yy M0):
        //   v_mean2d = conic * (M1x, M1y);  v_conic = (M2xx/2, M2xy, M2yy/2);  v_opacity = -M0 / opacity
        const float vu = A * g0.x + B * g0.y, vv = B * g0.x + C * g0.y;
        const float gA = 0.5f * g0.z, gB = 0.5f * g0.w, gC = 0.5f * g1.x;
        vo = -g1.y / rec1.y;
        const float v_rgb[3] = {g1.z, g1.w, g2.x};
        const float v_depth = g2.y;

        // conic -> covariance: V2 = -Q G Q
        const float q00 = A * gA + B * gB, q01 = A * gB + B * gC, q10 = B * gA + C * gB, q11 = B * gB + C * gC;
        const float V00 = -(q00 * A + q01 * B), V01 = -(q00 * B + q01 * C), V10 = -(q10 * A + q11 * B),
                    V11 = -(q10 * B + q11 * C);
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
        else             { vp[2] += fx * tx * rz3 * vJ[2]; }
        if (!clamp_y) { vp[1] += -fy * rz2 * vJ[5]; vp[2] += 2.0f * fy * ty * rz3 * vJ[5]; }
        else             { vp[2] += fy * ty * rz3 * vJ[5]; }
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            vm[a] = R[0 * 3 + a] * vp[0] + R[1 * 3 + a] * vp[1] + R[2 * 3 + a] * vp[2];
            red[9 + a] = vp[a];
#pragma unroll
            for (int b = 0; b < 3; ++b) red[a * 3 + b] = vp[a] * mu[b];
        }
        float tmp[9], vSigma[9], add[9];
        mat3_mul_at(R, vSc, tmp);
        mat3_mul(tmp, R, vSigma);
        mat3_mul(vSc, RS, add);
#pragma unroll
        for (int k = 0; k < 9; ++k) red[k] += 2.0f * add[k];
        world_cov_bwd(vSigma, M, Rq, s, w, qx, qy, qz, qinv, vs, vq);

        // SH backward (+ its contribution to v_means / v_campos)
        if (sh) {
            const float dx = mu[0] - cam.campos[0], dy = mu[1] - cam.campos[1], dz = mu[2] - cam.campos[2];
            const float inv = rsqrtf(dx * dx + dy * dy + dz * dz);
            const float nx = dx * inv, ny = dy * inv, nz = dz * inv;
            float Bs[16], Bx[16], By[16], Bz[16];
            sh_basis_grad(sh_degree, nx, ny, nz, Bs, Bx, By, Bz);
            const float rgb[3] = {rec2.x, rec2.y, rec2.z};
            float gch[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) gch[c] = rgb[c] > 0.f ? v_rgb[c] : 0.f;
            float4* op = reinterpret_cast<float4*>(v_sh + (size_t)i * 48);
            float vnx = 0.f, vny = 0.f, vnz = 0.f;
            float c48[48];
            load_sh_coeffs(sh, i, 1, c48);
            float o48[48];
#pragma unroll
            for (int k = 0; k < 16; ++k)
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float sv = c48[3 * k + c] * gch[c];
                    o48[3 * k + c] = Bs[k] * gch[c];
                    vnx += Bx[k] * sv; vny += By[k] * sv; vnz += Bz[k] * sv;
                }
#pragma unroll
            for (int k = 0; k < 12; ++k) op[k] = make_float4(o48[4 * k], o48[4 * k + 1], o48[4 * k + 2], o48[4 * k + 3]);
            const float dot = vnx * nx + vny * ny + vnz * nz;
            const float gx = (vnx - dot * nx) * inv, gy = (vny - dot * ny) * inv, gz = (vnz - dot * nz) * inv;
            vm[0] += gx; vm[1] += gy; vm[2] += gz;
            red[12] = -gx; red[13] = -gy; red[14] = -gz;
        }
    } else if (i < N && v_sh) {
        float4* op = reinterpret_cast<float4*>(v_sh + (size_t)i * 48);
#pragma unroll
        for (int k = 0; k < 12; ++k) op[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (i < N) {
        v_means[3 * i] = vm[0]; v_means[3 * i + 1] = vm[1]; v_means[3 * i + 2] = vm[2];
        reinterpret_cast<float4*>(v_quats)[i] = make_float4(vq[0], vq[1], vq[2], vq[3]);
        v_scales[3 * i] = vs[0]; v_scales[3 * i + 1] = vs[1]; v_scales[3 * i + 2] = vs[2];
        v_opac[i] = vo;
    }
    // block reduction of the 15 camera-gradient terms
#pragma unroll
    for (int k = 0; k < 15; ++k) red[k] = adb_warp_sum(red[k]);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < 15; ++k) sRed[wid][k] = red[k];
    __syncthreads();
    if (threadIdx.x < 15) {
        float v = 0.f;
#pragma unroll
        for (int w_ = 0; w_ < PB / 32; ++w_) v += sRed[w_][threadIdx.x];
        if (v != 0.f) {
            const int k = threadIdx.x;
            if (k < 9) atomicAdd(v_viewmat + (k / 3) * 4 + (k % 3), v);
            else if (k < 12) atomicAdd(v_viewmat + (k - 9) * 4 + 3, v);
            else if (v_campos) atomicAdd(v_campos + (k - 12), v);
        }
    }
}

}  // namespace

// v_viewmat[16] and v_campos[3] are ACCUMULATED (caller zeroes them); all per-Gaussian outputs are overwritten.
ADB_API int adb_raster_project_bwd(int N, const float* means, const float* quats, const float* scales,
                                   const float* sh, int sh_degree, const float* viewmat, const float* K,
                                   const float* campos, int W, int H, float eps2d, float near_plane,
                                   float far_plane, float radius_clip, const int32_t* radii, const float* splats,
                                   const float* v_splats, float* v_means, float* v_quats, float* v_scales,
                                   float* v_opac, float* v_sh, float* v_viewmat, float* v_campos,
                                   cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && W > 0 && H > 0, "adb_raster_project_bwd: bad sizes");
    if (N == 0) return ADB_OK;
    ADB_REQUIRE(means && quats && scales && viewmat && K && radii && splats && v_splats && v_means && v_quats &&
                    v_scales && v_opac && v_viewmat,
                "adb_raster_project_bwd: null pointer");
    ADB_REQUIRE(!sh || (campos && v_sh && v_campos), "adb_raster_project_bwd: sh needs campos, v_sh, v_campos");
    AdbCam cam{viewmat, K, campos, W, H, eps2d, near_plane, far_plane, radius_clip};
    project_bwd_kernel<<<adb_cdiv(N, PB), PB, 0, stream>>>(N, means, quats, scales, sh, sh_degree, cam, radii, splats,
                                                          v_splats, v_means, v_quats, v_scales, v_opac, v_sh,
                                                          v_viewmat, v_campos);
    ADB_CHECK_LAUNCH("project_bwd_kernel");
    return ADB_OK;
}

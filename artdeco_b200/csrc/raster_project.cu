// Per-Gaussian projection + SH colour + tile count, fused into one streaming pass (compiled with
// -fmad=false: the values that feed the integer tile keys must be bit-identical to the C oracle).
//
// Replaces what the reference reaches through gsplat.rendering.rasterization at
// Reconstruct/scene/scene_models/h3dgsv3.py:664-680: the projection (SURVEY.md App. B.1), the degree-3 SH
// evaluation with the +0.5 / clamp (App. B.2) and the tile count of isect_tiles (App. B.3).  gsplat runs
// these as three kernels with [N]-sized round trips through HBM between them; here one thread per
// Gaussian reads the 236 B of parameters once and writes one 48 B splat record + radii + count.  The projection and SH
// math shared with the backward kernels is in raster_geom.cuh.
#include "raster_geom.cuh"
#include "adb_detmath.h"
#include <stdio.h>

namespace {

// C cameras (viewmat / K / campos point at [C,16] / [C,9] / [C,3]); outputs are [C,N,...] stacks and tile_counts holds C
// consecutive counter blocks of 2 * COPIES * T.  Work split: warp w of the grid handles view (w % C) of the 32 Gaussians of
// chunk (w / C).  The C warps of a chunk are consecutive, so the C per-view chains run in parallel.  Each view warp recomputes
// the quaternion rotation and world-space covariance (a few dozen FP32 ops, against a chain of several hundred per view).
// One thread looping over the views, with that work and the SH coefficients kept in registers, needed 110 registers (2 CTAs
// per SM) and measured 1.48 ms per 8-view batch at 1M Gaussians / 1080p on an H100 SXM at 400 W — no faster than 8
// single-view launches (1.42 ms); this split measured 0.78 ms with every lane loading its own rows from global memory.
// For C = 1 it is the single-view kernel thread for thread.  Everything per view is expression for expression the
// single-view arithmetic, so C = 1 and C > 1 produce the same bits.
//
// When C divides 8 (the 8-view batch, the single view) or is a multiple of 8, a CTA's warps cover whole chunks, proj_rows(C)
// consecutive Gaussians; the CTA first copies their parameter rows into shared memory with coalesced copies (raster_geom.cuh:
// the per-lane 192 B SH rows touched 32 lines per load instruction, and every view warp repeated that), and each view warp
// reads its lane's row from there.  On an H100 SXM at 700 W this took the 8-view batch from 0.785 to 0.600 ms and the single
// view from 0.175 to 0.141 ms.  For any other C a chunk straddles two CTAs and the lanes read global memory directly.
constexpr int PROJ_WARPS = 8;
constexpr int PROJ_ROW_FLOATS = SH_ROW + 4 + 3 + 3 + 1;        // staged row: SH, quat, mean, scale, opacity
__host__ __device__ constexpr int proj_rows(int C) {
    return (C <= PROJ_WARPS && PROJ_WARPS % C == 0) ? PROJ_WARPS * 32 / C : (C % PROJ_WARPS == 0 ? 32 : 0);
}
__global__ void __launch_bounds__(PROJ_WARPS * 32)
project_fwd_kernel(int N, int C, const float* __restrict__ means, const float* __restrict__ quats,
                   const float* __restrict__ scales, const float* __restrict__ opacities,
                   const float* __restrict__ sh, int sh_degree, AdbCam cam,
                   int32_t* __restrict__ radii, float* __restrict__ splats, int32_t* __restrict__ tiles_per_gauss,
                   int32_t* __restrict__ tile_counts) {
    extern __shared__ float4 proj_smem[];
    const unsigned gw = blockIdx.x * PROJ_WARPS + (threadIdx.x >> 5);     // < 2^32: checked at launch
    const int c = C == 1 ? 0 : (int)(gw % (unsigned)C);                     // C = 1: no integer division
    const unsigned chunk = C == 1 ? gw : gw / (unsigned)C;
    const int i = (int)(chunk * 32u + (threadIdx.x & 31));                 // < N + 32 <= 2^31 - 1: checked at launch
    // staged rows [first, first + rows): SH rows of SH_ROW floats, then quats, means, scales, opacities
    const int rows = proj_rows(C);
    const int first = (int)((blockIdx.x * PROJ_WARPS) / (unsigned)C * 32u);
    float* const sSH = reinterpret_cast<float*>(proj_smem);
    float4* const sQ = proj_smem + rows * (SH_ROW / 4);
    float* const sM = reinterpret_cast<float*>(sQ + rows);
    float* const sS = sM + 3 * rows;
    float* const sO = sS + 3 * rows;
    if (rows) {
        const int n = min(rows, N - first);                 // > 0: the CTA's first warp has Gaussians
        if (sh) stage_sh_rows(sSH, sh, first, n);
        const float4* q4 = reinterpret_cast<const float4*>(quats) + first;
        for (int j = threadIdx.x; j < n; j += blockDim.x) cp_async16(sQ + j, q4 + j);
        stage_floats(sM, means + 3 * (size_t)first, 3 * n);
        stage_floats(sS, scales + 3 * (size_t)first, 3 * n);
        stage_floats(sO, opacities + first, n);
        cp_async_wait_all();
        __syncthreads();
    }
    if (i >= N) return;
    const int row = i - first;                             // staged row of Gaussian i
    const size_t ci = (size_t)c * N + i;
    int tr_x0 = 0, tr_x1 = 0, tr_y0 = 0, tr_y1 = 0;    // tile rectangle (for the fused per-tile counting)
    const float* V = cam.viewmat + 16 * c;
    const float* Kc = cam.K + 9 * c;
    const float R[9] = {V[0], V[1], V[2], V[4], V[5], V[6], V[8], V[9], V[10]};
    const float t[3] = {V[3], V[7], V[11]};
    const float fx = Kc[0], fy = Kc[4], cx = Kc[2], cy = Kc[5];
    const float m0 = rows ? sM[3 * row] : means[3 * i], m1 = rows ? sM[3 * row + 1] : means[3 * i + 1],
                m2 = rows ? sM[3 * row + 2] : means[3 * i + 2];

    int rx_i = 0, ry_i = 0, count = 0, cull_rx = 0, cull_ry = 0;
    float u = 0.f, v = 0.f, ca = 0.f, cb = 0.f, cc = 0.f, lg = 0.f;
    const float x = R[0] * m0 + R[1] * m1 + R[2] * m2 + t[0];
    const float y = R[3] * m0 + R[4] * m1 + R[5] * m2 + t[1];
    const float z = R[6] * m0 + R[7] * m1 + R[8] * m2 + t[2];
    const float opacity = rows ? sO[row] : opacities[i];
    bool ok = !(z < cam.near_plane || z > cam.far_plane);
    if (ok) {
        float Rq[9];
        {
            const float4 q = rows ? sQ[row] : reinterpret_cast<const float4*>(quats)[i];
            const float inv = 1.0f / sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
            quat_to_rotmat(q.x * inv, q.y * inv, q.z * inv, q.w * inv, Rq);
        }
        const float s[3] = {rows ? sS[3 * row] : scales[3 * i], rows ? sS[3 * row + 1] : scales[3 * i + 1],
                            rows ? sS[3 * row + 2] : scales[3 * i + 2]};
        float M[9], Sigma[9], RS[9], Sc[9];
        world_cov(Rq, s, M, Sigma);
        cam_cov(R, Sigma, RS, Sc);

        const float W = (float)cam.W, H = (float)cam.H;
        const PerspJacobian pj = persp_jacobian(x, y, z, fx, fy, cx, cy, W, H);
        const float rz = pj.rz, J0 = pj.J[0], J2 = pj.J[2], J4 = pj.J[4], J5 = pj.J[5];
        float k00 = J0 * Sc[0] + J2 * Sc[6], k01 = J0 * Sc[1] + J2 * Sc[7], k02 = J0 * Sc[2] + J2 * Sc[8];
        float k11 = J4 * Sc[4] + J5 * Sc[7], k12 = J4 * Sc[5] + J5 * Sc[8];
        float a = k00 * J0 + k02 * J2;
        float b = k01 * J4 + k02 * J5;
        float c = k11 * J4 + k12 * J5;
        a = a + cam.eps2d;
        c = c + cam.eps2d;
        float det = a * c - b * b;
        if (cam.convention == ADB_CONV_INRIA) {
            ok = det > 0.f;
            if (ok) {
                u = fx * x * rz + cx;
                v = fy * y * rz + cy;
                const float mid = 0.5f * (a + c);
                const float lam1 = mid + sqrtf(fmaxf(0.1f, mid * mid - det));
                const int rI = (int)fminf(ceilf(3.0f * sqrtf(lam1)), 1.0e9f);
                int x0, x1, y0, y1;
                adb_tile_rect(u, v, rI, rI, cam.W, cam.H, ADB_CONV_INRIA, x0, x1, y0, y1);
                count = (x1 - x0) * (y1 - y0);
                tr_x0 = x0; tr_x1 = x1; tr_y0 = y0; tr_y1 = y1;
                ok = count > 0;          // Inria leaves radii = 0 when no tile is touched
                if (ok) {
                    rx_i = ry_i = rI;
                    ca = c / det; cb = -b / det; cc = a / det;
                    if (opacity < ADB_ALPHA_THRESHOLD) {
                        // alpha can never reach 1/255: keeps its radius (visibility filter) and a record (so the
                        // backward reads defined values) but emits no keys
                        count = 0;
                    } else {
                        // conservative extent for the blend kernels' block-level culling (alpha < 1/255 outside it)
                        lg = adb_det_logf(opacity / ADB_ALPHA_THRESHOLD);
                        const float ext = fminf(3.33f, sqrtf(2.0f * lg));
                        const float r1 = ext * sqrtf(lam1);
                        cull_rx = (int)fminf(ceilf(fminf(ext * sqrtf(a), r1)), 65535.f);
                        cull_ry = (int)fminf(ceilf(fminf(ext * sqrtf(c), r1)), 65535.f);
                    }
                }
            }
        } else {
        ok = det > 0.f && !(opacity < ADB_ALPHA_THRESHOLD);
        if (ok) {
            u = fx * x * rz + cx;
            v = fy * y * rz + cy;
            lg = adb_det_logf(opacity / ADB_ALPHA_THRESHOLD);
            float ext = sqrtf(2.0f * lg);
            ext = fminf(3.33f, ext);
            float bb = 0.5f * (a + c);
            float lam = bb + sqrtf(fmaxf(0.01f, bb * bb - det));
            float r1 = ext * sqrtf(lam);
            float rx = ceilf(fminf(ext * sqrtf(a), r1));
            float ry = ceilf(fminf(ext * sqrtf(c), r1));
            ok = !(rx <= cam.radius_clip && ry <= cam.radius_clip) &&
                 !(u + rx <= 0.f || u - rx >= W || v + ry <= 0.f || v - ry >= H);
            if (ok) {
                rx_i = (int)rx; ry_i = (int)ry;
                cull_rx = rx_i; cull_ry = ry_i;
                ca = c / det; cb = -b / det; cc = a / det;
                // tile count (same arithmetic as the emit kernel and the oracle's tile_bounds)
                int x0, x1, y0, y1;
                adb_tile_rect(u, v, rx_i, ry_i, cam.W, cam.H, ADB_CONV_GSPLAT, x0, x1, y0, y1);
                count = (x1 - x0) * (y1 - y0);
                tr_x0 = x0; tr_x1 = x1; tr_y0 = y0; tr_y1 = y1;
            }
        }
        }
    }
    reinterpret_cast<int2*>(radii)[ci] = make_int2(rx_i, ry_i);
    tiles_per_gauss[ci] = count;
    if (tile_counts && count > 0) {
        // fused first stage of the tile-bucketed intersection (raster_isect.cu): fire-and-forget REDs into the replicated
        // per-tile counters, overlapped with the SH loads below instead of a separate pass over radii / means2d
        // (the counter copy must be the one tile_scatter_kernel picks for Gaussian i: its CTA index i / 256)
        const int tw = (cam.W + ADB_TILE - 1) / ADB_TILE;
        const int cp = (i >> 8) & (ADB_TILE_COUNTER_COPIES - 1);
        int32_t* counts = tile_counts + (size_t)c * 2 * ADB_TILE_COUNTER_COPIES * tw * ((cam.H + ADB_TILE - 1) / ADB_TILE);
        for (int ty = tr_y0; ty < tr_y1; ++ty)
            for (int tx = tr_x0; tx < tr_x1; ++tx) atomicAdd(counts + (ty * tw + tx) * ADB_TILE_COUNTER_COPIES + cp, 1);
    }
    if (!ok) return;

    float r = 0.f, g = 0.f, bl = 0.f;
    if (sh) {
        const float* P = cam.campos + 3 * c;
        float dx = m0 - P[0], dy = m1 - P[1], dz = m2 - P[2];
        float inv = 1.0f / sqrtf(dx * dx + dy * dy + dz * dz);
        float B[16];
        sh_basis(sh_degree, dx * inv, dy * inv, dz * inv, B);
        if (rows) {
            const float* sc = sSH + row * SH_ROW;
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                r += B[k] * sc[3 * k]; g += B[k] * sc[3 * k + 1]; bl += B[k] * sc[3 * k + 2];
            }
        } else {
            float c48[48];
            load_sh_coeffs(sh, i, C, c48);      // C > 1: the chunk's C view warps read the same lines
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                r += B[k] * c48[3 * k]; g += B[k] * c48[3 * k + 1]; bl += B[k] * c48[3 * k + 2];
            }
        }
        r = fmaxf(r + 0.5f, 0.f); g = fmaxf(g + 0.5f, 0.f); bl = fmaxf(bl + 0.5f, 0.f);
    }
    float4* out = reinterpret_cast<float4*>(splats + ci * ADB_SPLAT_STRIDE);
    // sigma <= ln(255*opacity) <=> alpha >= 1/255; the margin keeps the pre-test a strict superset of the exact test
    const float sigma_max = lg + 0.02f;
    const unsigned packed_radii = (unsigned)min(cull_rx, 65535) | ((unsigned)min(cull_ry, 65535) << 16);
    out[0] = make_float4(u, v, ca, cb);
    out[1] = make_float4(cc, opacity, sigma_max, __uint_as_float(packed_radii));
    out[2] = make_float4(r, g, bl, z);
}

}  // namespace

static int refuse(const char* name, const char* what) {
    char msg[160];
    snprintf(msg, sizeof(msg), "%s: %s", name, what);
    adb_set_error_msg(msg);
    return ADB_ERR_INVALID;
}

// C cameras.  `sh` may be NULL (then rgb = 0 and campos is ignored).  viewmats/Ks/camposs are DEVICE pointers to [C,16] /
// [C,9] / [C,3]; outputs are [C,N,...] stacks and tile_counts (may be NULL) holds C counter blocks.
static int project_fwd_impl(const char* name, int convention, int N, int C, const float* means, const float* quats,
                            const float* scales, const float* opacities, const float* sh, int sh_degree,
                            const float* viewmats, const float* Ks, const float* camposs, int W, int H,
                            float eps2d, float near_plane, float far_plane, float radius_clip,
                            int32_t* radii, float* splats, int32_t* tiles_per_gauss, int32_t* tile_counts,
                            cudaStream_t stream) {
    if (!(N >= 0 && C > 0 && W > 0 && H > 0)) return refuse(name, "bad sizes");
    if (N == 0) return ADB_OK;
    if (!(means && quats && scales && opacities && viewmats && Ks && radii && splats && tiles_per_gauss))
        return refuse(name, "null pointer");
    if (sh && !camposs) return refuse(name, "sh needs campos");
    if (!(sh_degree >= 0 && sh_degree <= 3)) return refuse(name, "sh_degree must be 0..3");
    AdbCam cam{viewmats, Ks, camposs, W, H, eps2d, near_plane, far_plane, radius_clip, convention};
    const long long warps = (long long)adb_cdiv(N, 32) * C;
    if (warps >= (1LL << 32) - PROJ_WARPS || N > 2147483647 - 32) return refuse(name, "too many (Gaussian, view) pairs");
    const unsigned blocks = (unsigned)((warps + PROJ_WARPS - 1) / PROJ_WARPS);
    constexpr int max_smem = proj_rows(1) * PROJ_ROW_FLOATS * (int)sizeof(float);     // 63 KB: above the 48 KB default
    static AdbDeviceOnce once;
    const int rc = once.ensure([]() -> int {
        ADB_CUDA(cudaFuncSetAttribute(project_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
        return ADB_OK;
    });
    if (rc != ADB_OK) return rc;
    const size_t smem = (size_t)proj_rows(C) * PROJ_ROW_FLOATS * sizeof(float);
    project_fwd_kernel<<<blocks, PROJ_WARPS * 32, smem, stream>>>(N, C, means, quats, scales, opacities, sh, sh_degree, cam,
                                                              radii, splats, tiles_per_gauss, tile_counts);
    ADB_CHECK_LAUNCH("project_fwd_kernel");
    return ADB_OK;
}

ADB_API int adb_raster_project_fwd(int N, const float* means, const float* quats, const float* scales,
                                   const float* opacities, const float* sh, int sh_degree,
                                   const float* viewmat, const float* K, const float* campos, int W, int H,
                                   float eps2d, float near_plane, float far_plane, float radius_clip,
                                   int32_t* radii, float* splats, int32_t* tiles_per_gauss, cudaStream_t stream) {
    return project_fwd_impl("adb_raster_project_fwd", ADB_CONV_GSPLAT, N, 1, means, quats, scales, opacities, sh, sh_degree,
                            viewmat, K, campos, W, H, eps2d, near_plane, far_plane, radius_clip, radii, splats,
                            tiles_per_gauss, nullptr, stream);
}

// Same, plus the first stage of the tile-bucketed intersection fused in: tile_counts (int32 [2*4*T], first half zero on entry,
// see adb_raster_tile_count_scan) receives one RED per (Gaussian, touched tile); pass counts_ready = 1 to the scan afterwards.
ADB_API int adb_raster_project_fwd_counts(int N, const float* means, const float* quats, const float* scales,
                                          const float* opacities, const float* sh, int sh_degree,
                                          const float* viewmat, const float* K, const float* campos, int W, int H,
                                          float eps2d, float near_plane, float far_plane, float radius_clip,
                                          int32_t* radii, float* splats, int32_t* tiles_per_gauss, int32_t* tile_counts,
                                          cudaStream_t stream) {
    ADB_REQUIRE(tile_counts, "adb_raster_project_fwd_counts: null tile_counts");
    return project_fwd_impl("adb_raster_project_fwd_counts", ADB_CONV_GSPLAT, N, 1, means, quats, scales, opacities, sh,
                            sh_degree, viewmat, K, campos, W, H, eps2d, near_plane, far_plane, radius_clip, radii, splats,
                            tiles_per_gauss, tile_counts, stream);
}

// C cameras of the same Gaussians in one pass (the multi-view batch): parameters read once, per view the records of
// adb_raster_project_fwd_counts bit for bit.  radii [C,N,2], splats [C,N,12], tiles_per_gauss [C,N], tile_counts
// [C, 2*4*T] (first half of every view's block zero on entry).
ADB_API int adb_raster_project_fwd_multi(int N, int C, const float* means, const float* quats, const float* scales,
                                         const float* opacities, const float* sh, int sh_degree,
                                         const float* viewmats, const float* Ks, const float* camposs, int W, int H,
                                         float eps2d, float near_plane, float far_plane, float radius_clip,
                                         int32_t* radii, float* splats, int32_t* tiles_per_gauss, int32_t* tile_counts,
                                         cudaStream_t stream) {
    ADB_REQUIRE(tile_counts, "adb_raster_project_fwd_multi: null tile_counts");
    return project_fwd_impl("adb_raster_project_fwd_multi", ADB_CONV_GSPLAT, N, C, means, quats, scales, opacities, sh,
                            sh_degree, viewmats, Ks, camposs, W, H, eps2d, near_plane, far_plane, radius_clip, radii, splats,
                            tiles_per_gauss, tile_counts, stream);
}

// Legacy (Inria / diff_gaussian_rasterization) conventions: radii[:,0] == radii[:,1] == ceil(3 sqrt(lambda_max)); the
// caller passes eps2d = 0.3 and near_plane = 0.2.  Same record layout (slot 11 stays the camera-space depth z).
ADB_API int adb_raster_project_fwd_legacy(int N, const float* means, const float* quats, const float* scales,
                                          const float* opacities, const float* sh, int sh_degree,
                                          const float* viewmat, const float* K, const float* campos, int W, int H,
                                          float eps2d, float near_plane, float far_plane,
                                          int32_t* radii, float* splats, int32_t* tiles_per_gauss, cudaStream_t stream) {
    return project_fwd_impl("adb_raster_project_fwd_legacy", ADB_CONV_INRIA, N, 1, means, quats, scales, opacities, sh,
                            sh_degree, viewmat, K, campos, W, H, eps2d, near_plane, far_plane, 0.f, radii, splats,
                            tiles_per_gauss, nullptr, stream);
}

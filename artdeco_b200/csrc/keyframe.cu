// Key-frame hand-off from the Backend to the mapper, for sm_90a.
//
// Replaces, once per key frame:
//   VSLAM/Backend.py:117-193      prepare_for_mapper / compute_dense_point: ~30 torch and pypose kernels at SLAM resolution
//                                 and blocking .cpu() copies of densePoint, T_WC and T_CkC
//   run_system.py:161-192         the copies back to the mapper's device and Tcw = quat2unit(SE3(T_WC[:7])).Inv().matrix()
//   Reconstruct/scene/keyframe.py:64-127   Keyframe.__init__ (training branch): the 1/z prior, its bilinear resize to the
//                                 mapper image, and the average-pool pyramids of the image and of the inverse depth
//
// Design:
//  * dense_point_kernel: one thread per SLAM pixel, one 16 B store of (point xyz in key-frame order, channel 3 in
//    last-key-frame order).  The reference also scatters each matched point back to its key-frame pixel; every scattered
//    value is the same function of the same input as the value already there, so each point is computed once.  Block 0
//    writes T_CkC.  An idx_k2l entry outside [0, HW) (the reference faults or raises) is not read: its pixel is NaN in all
//    four channels and counted in a caller-zeroed device int32;
//  * mapper_inputs_kernel: one block per 32x32 tile of the mapper image.  Tiles are aligned to 2^(pyr_levels-1), so every
//    pooled pixel of every level lies in one tile: level 0 of the inverse depth is computed from the dense point's z at the
//    four bilinear taps and kept in shared memory, level 1 of the image is pooled from global memory, and the deeper
//    levels are pooled in shared memory.  Thread 0 of block (0, 0) writes the mapper pose;
//  * arithmetic as PyTorch evaluates it on CUDA: IEEE division, upsample_bilinear2d's index arithmetic and blend, and
//    avg_pool2d's window-order sum (resample.cuh).
#include <cstdint>

#include "backproject.cuh"
#include "common.cuh"
#include "mapper_pose.cuh"
#include "resample.cuh"

namespace {

using adb_backproject::on_ray;

constexpr int DP_THREADS = 256;
constexpr int TILE = 32;               // mapper tile edge at level 0
constexpr int MI_ROWS = 8;             // block 32x8
constexpr int MI_THREADS = TILE * MI_ROWS;
constexpr int MAX_LEVELS = 6;          // 2^(MAX_LEVELS - 1) == TILE
constexpr long long MAX_PIXELS = 1LL << 28;

// The per-pixel arithmetic rounds once per operation, in the order of oracle/keyframe_ref.py's elementwise statements: the
// confidence 1 / (r - 2) turns one rounding of the reprojected pixel into up to ~1e-4 of the result.

// a x b: each product rounded, then the difference
__device__ __forceinline__ void cross_rn(const float* a, const float* b, float* c) {
    c[0] = __fsub_rn(__fmul_rn(a[1], b[2]), __fmul_rn(a[2], b[1]));
    c[1] = __fsub_rn(__fmul_rn(a[2], b[0]), __fmul_rn(a[0], b[2]));
    c[2] = __fsub_rn(__fmul_rn(a[0], b[1]), __fmul_rn(a[1], b[0]));
}

// pypose's Sim3 Act on an [8] pose (t, q xyzw, s): s (X + w uv + q x uv) + t with uv = 2 q x X
__device__ __forceinline__ void sim3_act(const float* T, const float X[3], float Y[3]) {
    float c[3], uv[3], c2[3];
    cross_rn(T + 3, X, c);
#pragma unroll
    for (int i = 0; i < 3; ++i) uv[i] = __fmul_rn(2.f, c[i]);
    cross_rn(T + 3, uv, c2);
#pragma unroll
    for (int i = 0; i < 3; ++i)
        Y[i] = __fadd_rn(__fmul_rn(__fadd_rn(__fadd_rn(X[i], __fmul_rn(T[6], uv[i])), c2[i]), T[7]), T[i]);
}

// T^-1 = (-(1/s) q^-1 t, q^-1, 1/s)
__device__ __forceinline__ void sim3_inv(const float* T, float* I) {
    const float si = __fdiv_rn(1.f, T[7]);
    const float R[8] = {0.f, 0.f, 0.f, -T[3], -T[4], -T[5], T[6], 1.f};
    float r[3];
    sim3_act(R, T, r);
#pragma unroll
    for (int i = 0; i < 3; ++i) I[i] = __fmul_rn(-si, r[i]);
#pragma unroll
    for (int i = 3; i < 7; ++i) I[i] = R[i];
    I[7] = si;
}

// A B = (A.Act(B.t), A.q B.q, A.s B.s), the quaternion product summed left to right as gn_ref.quat_comp writes it
__device__ __forceinline__ void sim3_mul(const float* A, const float* B, float* T) {
    sim3_act(A, B, T);
    const float* a = A + 3;
    const float* b = B + 3;
    T[3] = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(a[3], b[0]), __fmul_rn(a[0], b[3])), __fmul_rn(a[1], b[2])), __fmul_rn(a[2], b[1]));
    T[4] = __fadd_rn(__fadd_rn(__fsub_rn(__fmul_rn(a[3], b[1]), __fmul_rn(a[0], b[2])), __fmul_rn(a[1], b[3])), __fmul_rn(a[2], b[0]));
    T[5] = __fadd_rn(__fsub_rn(__fadd_rn(__fmul_rn(a[3], b[2]), __fmul_rn(a[0], b[1])), __fmul_rn(a[1], b[0])), __fmul_rn(a[2], b[3]));
    T[6] = __fsub_rn(__fsub_rn(__fsub_rn(__fmul_rn(a[3], b[3]), __fmul_rn(a[0], b[0])), __fmul_rn(a[1], b[1])), __fmul_rn(a[2], b[2]));
    T[7] = __fmul_rn(A[7], B[7]);
}

__global__ void __launch_bounds__(DP_THREADS)
dense_point_kernel(int H, int W, const float* __restrict__ X, const float* __restrict__ C, const int* __restrict__ N,
                   const float* __restrict__ Twk_g, const float* __restrict__ Twl_g, const long long* __restrict__ idx,
                   const float* __restrict__ K, float4* __restrict__ out, float* __restrict__ T_CkC, int* __restrict__ n_bad) {
    const int HW = H * W;
    const int p = blockIdx.x * DP_THREADS + threadIdx.x;
    float k[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) k[i] = __ldg(K + i);
    if (!Twl_g) {
        // first key frame: the points on their rays, channel 3 = float(C / N > 1.5) with N a Python int
        if (p >= HW) return;
        const float inv_n = 1.0f / (float)__ldg(N);
        float P[3];
        on_ray(X, k, p, W, P);
        const float c = __fmul_rn(__ldg(C + p), inv_n);
        out[p] = make_float4(P[0], P[1], P[2], c > 1.5f ? 1.f : 0.f);
        return;
    }
    float Twk[8], Tlk[8], Tkw[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) Twk[i] = __ldg(Twk_g + i);
    {
        float Twl[8], Tlw[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) Twl[i] = __ldg(Twl_g + i);
        sim3_inv(Twl, Tlw);
        sim3_mul(Tlw, Twk, Tlk);
        // SE3(Twk[:7]).Inv(): the quaternion as it is, the scale dropped
        const float se3[8] = {Twk[0], Twk[1], Twk[2], Twk[3], Twk[4], Twk[5], Twk[6], 1.f};
        sim3_inv(se3, Tkw);
    }
    if (p == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) T_CkC[i] = Tlk[i];
    }
    bool bad = false;
    if (p < HW) {
        const long long j = __ldg(idx + p);
        float4 o;
        if (j < 0 || j >= HW) {
            bad = true;
            const float nan = __int_as_float(0x7fffffff);
            o = make_float4(nan, nan, nan, nan);
        } else {
            // point: Tkw_se3.Act(Twk.Act(Xc))
            float Xc[3], Xw[3], P[3];
            on_ray(X, k, p, W, Xc);
            sim3_act(Twk, Xc, Xw);
            sim3_act(Tkw, Xw, P);
            // channel 3: reprojection residual of the matched key-frame point in the last key frame
            float Xj[3], Y[3];
            on_ray(X, k, (int)j, W, Xj);
            sim3_act(Tlk, Xj, Y);
            const float pk[3] = {__fdiv_rn(Y[0], Y[2]), __fdiv_rn(Y[1], Y[2]), __fdiv_rn(Y[2], Y[2])};
            const float u = __fadd_rn(__fadd_rn(__fmul_rn(k[0], pk[0]), __fmul_rn(k[1], pk[1])), __fmul_rn(k[2], pk[2]));
            const float v = __fadd_rn(__fadd_rn(__fmul_rn(k[3], pk[0]), __fmul_rn(k[4], pk[1])), __fmul_rn(k[5], pk[2]));
            const float du = __fsub_rn(u, (float)(p % W)), dv = __fsub_rn(v, (float)(p / W));
            const float res = __fsqrt_rn(__fadd_rn(__fmul_rn(du, du), __fmul_rn(dv, dv)));
            const float conf = res < 3.f ? 1.f : __fdiv_rn(1.f, __fadd_rn(__fsub_rn(res, 3.f), 1.f));
            o = make_float4(P[0], P[1], P[2], conf);
        }
        out[p] = o;
    }
    const unsigned m = __ballot_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(n_bad, __popc(m));
}

struct MiParams {
    int H, W, Hs, Ws, L;
    float sy, sx;                           // fp32 (Hs - 1) / (H - 1), (Ws - 1) / (W - 1); 0 for an output of size 1
    long long cs, ys, xs;                   // image strides (elements): channel, row, column
    int h[MAX_LEVELS], w[MAX_LEVELS];       // level sizes, floored level by level
    long long id_off[MAX_LEVELS];           // offsets of the levels in the packed inverse-depth pyramid
    long long im_off[MAX_LEVELS];           // offsets of levels 1.. in the packed image pyramid (3 planes per level)
};

// where(z != 0, 1 / (z + 1e-4), 1e4)
__device__ __forceinline__ float prior(float z) { return z != 0.f ? 1.0f / __fadd_rn(z, 1e-4f) : 1e4f; }

__device__ __forceinline__ float tap(const float4* __restrict__ dp, int Ws, int y, int x) {
    return prior(__ldg(&dp[(size_t)y * Ws + x].z));
}

// shared-memory offset of level l (level l of a tile is (TILE >> l)^2 floats)
__host__ __device__ constexpr int lvl_off(int l) {
    int o = 0;
    for (int i = 0; i < l; ++i) o += (TILE >> i) * (TILE >> i);
    return o;
}

__global__ void __launch_bounds__(MI_THREADS)
mapper_inputs_kernel(MiParams p, const float* __restrict__ image, const float4* __restrict__ dp,
                     const float* __restrict__ T_WC, float* __restrict__ idepth, float* __restrict__ img_out,
                     float* __restrict__ rW2C, float* __restrict__ tW2C, float* __restrict__ approx, float* __restrict__ Rout) {
    __shared__ float s_id[lvl_off(MAX_LEVELS)];
    __shared__ float s_im[3][lvl_off(MAX_LEVELS)];      // level 0 of the image is not kept (index 0 unused)
    const int tid = threadIdx.y * TILE + threadIdx.x;
    const int X0 = blockIdx.x * TILE, Y0 = blockIdx.y * TILE;
    if (tid == 0 && blockIdx.x == 0 && blockIdx.y == 0) {
        // Rt = quat2unit(SE3(T_WC[:7])).Inv().matrix()
        float t[3] = {T_WC[0], T_WC[1], T_WC[2]}, q[4] = {T_WC[3], T_WC[4], T_WC[5], T_WC[6]};
        adb_pose::quat_unit(q);
        float R[3][3], ti[3], c[3];
        adb_pose::se3_inverse_Rt(t, q, R, ti);
        adb_pose::centre_of(R, ti, c);
        float r6[6];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            r6[2 * i] = R[i][0];
            r6[2 * i + 1] = R[i][1];
            tW2C[i] = ti[i];
            approx[i] = c[i];
        }
#pragma unroll
        for (int i = 0; i < 6; ++i) rW2C[i] = r6[i];
        float Rs[3][3];
        adb_pose::six_d_to_R(r6, Rs);
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) Rout[3 * i + j] = Rs[i][j];
    }
    // level 0 of the inverse depth: the prior at the four taps, then upsample_bilinear2d
    for (int i = tid; i < TILE * TILE; i += MI_THREADS) {
        const int y = Y0 + i / TILE, x = X0 + i % TILE;
        if (y >= p.H || x >= p.W) continue;
        int y0, yp, x0, xp;
        float ly, lx;
        adb_resample::lin_src(p.sy, y, p.Hs, &y0, &yp, &ly);
        adb_resample::lin_src(p.sx, x, p.Ws, &x0, &xp, &lx);
        const float v = adb_resample::blend4(1.f - ly, ly, 1.f - lx, lx, tap(dp, p.Ws, y0, x0), tap(dp, p.Ws, y0, x0 + xp),
                                             tap(dp, p.Ws, y0 + yp, x0), tap(dp, p.Ws, y0 + yp, x0 + xp));
        s_id[i] = v;
        idepth[(size_t)y * p.W + x] = v;
    }
    // level 1 of the image, pooled from the input through its strides
    if (p.L > 1) {
        constexpr int T1 = TILE / 2;
        const size_t plane = (size_t)p.h[1] * p.w[1];
        for (int i = tid; i < T1 * T1; i += MI_THREADS) {
            const int y = Y0 / 2 + i / T1, x = X0 / 2 + i % T1;
            if (y >= p.h[1] || x >= p.w[1]) continue;
            const float* a = image + (2 * y) * p.ys + (2 * x) * p.xs;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float* q = a + c * p.cs;
                const float v = adb_resample::pool4(q[0], q[p.xs], q[p.ys], q[p.ys + p.xs]);
                s_im[c][lvl_off(1) + i] = v;
                img_out[p.im_off[1] + c * plane + (size_t)y * p.w[1] + x] = v;
            }
        }
    }
    __syncthreads();
    for (int l = 1; l < p.L; ++l) {
        const int T = TILE >> l, Tp = TILE >> (l - 1);
        const int oy = Y0 >> l, ox = X0 >> l;
        const float* prev = s_id + lvl_off(l - 1);
        for (int i = tid; i < T * T; i += MI_THREADS) {
            const int ly = i / T, lx = i % T;
            const int y = oy + ly, x = ox + lx;
            if (y >= p.h[l] || x >= p.w[l]) continue;
            const float* a = prev + (2 * ly) * Tp + 2 * lx;
            const float v = adb_resample::pool4(a[0], a[1], a[Tp], a[Tp + 1]);
            s_id[lvl_off(l) + i] = v;
            idepth[p.id_off[l] + (size_t)y * p.w[l] + x] = v;
            if (l >= 2) {
                const size_t plane = (size_t)p.h[l] * p.w[l];
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float* b = s_im[c] + lvl_off(l - 1) + (2 * ly) * Tp + 2 * lx;
                    const float u = adb_resample::pool4(b[0], b[1], b[Tp], b[Tp + 1]);
                    s_im[c][lvl_off(l) + i] = u;
                    img_out[p.im_off[l] + c * plane + (size_t)y * p.w[l] + x] = u;
                }
            }
        }
        __syncthreads();
    }
}

}  // namespace

ADB_API int adb_kf_dense_point(int height, int width, const float* X_canon, const float* C, const int32_t* N,
                               const float* T_WC, const float* last_T_WC, const long long* idx_k2l, const float* K,
                               float* dense_point, float* T_CkC, int32_t* n_bad, cudaStream_t stream) {
    ADB_REQUIRE(height >= 1 && width >= 1 && (long long)height * width <= MAX_PIXELS, "adb_kf_dense_point: bad size");
    ADB_REQUIRE(X_canon && K && dense_point, "adb_kf_dense_point: null pointer");
    if (last_T_WC) {
        ADB_REQUIRE(T_WC && idx_k2l && T_CkC && n_bad, "adb_kf_dense_point: null pointer");
    } else {
        ADB_REQUIRE(C && N, "adb_kf_dense_point: null pointer (the first key frame needs C and N)");
    }
    ADB_REQUIRE(((uintptr_t)dense_point & 15) == 0, "adb_kf_dense_point: dense_point must be 16-byte aligned");
    const int HW = height * width;
    dense_point_kernel<<<adb_cdiv(HW, DP_THREADS), DP_THREADS, 0, stream>>>(
        height, width, X_canon, C, N, T_WC, last_T_WC, idx_k2l, K, (float4*)dense_point, T_CkC, n_bad);
    ADB_CHECK_LAUNCH("dense_point_kernel");
    return ADB_OK;
}

ADB_API int adb_kf_pyramid_floats(int height, int width, int pyr_levels, long long* idepth_floats, long long* image_floats) {
    ADB_REQUIRE(idepth_floats && image_floats, "adb_kf_pyramid_floats: null pointer");
    ADB_REQUIRE(pyr_levels >= 1 && pyr_levels <= MAX_LEVELS, "adb_kf_pyramid_floats: pyr_levels must lie in [1, 6]");
    ADB_REQUIRE(height >= 1 && width >= 1 && (height >> (pyr_levels - 1)) >= 1 && (width >> (pyr_levels - 1)) >= 1,
                "adb_kf_pyramid_floats: the coarsest level must be at least 1x1");
    long long a = 0, b = 0;
    for (int l = 0; l < pyr_levels; ++l) {
        const long long n = (long long)(height >> l) * (width >> l);
        a += n;
        if (l > 0) b += 3 * n;
    }
    *idepth_floats = a;
    *image_floats = b;
    return ADB_OK;
}

ADB_API int adb_kf_mapper_inputs(int height, int width, int Hs, int Ws, int pyr_levels, const float* image,
                                 const long long* image_strides, const float* dense_point, const float* T_WC,
                                 float* idepth_pyr, float* image_pyr, float* rW2C, float* tW2C, float* approx_centre, float* R,
                                 cudaStream_t stream) {
    ADB_REQUIRE(pyr_levels >= 1 && pyr_levels <= MAX_LEVELS, "adb_kf_mapper_inputs: pyr_levels must lie in [1, 6]");
    ADB_REQUIRE(height >= 1 && width >= 1 && (long long)height * width <= MAX_PIXELS && Hs >= 1 && Ws >= 1 &&
                    (long long)Hs * Ws <= MAX_PIXELS,
                "adb_kf_mapper_inputs: bad size");
    ADB_REQUIRE((height >> (pyr_levels - 1)) >= 1 && (width >> (pyr_levels - 1)) >= 1,
                "adb_kf_mapper_inputs: the coarsest level must be at least 1x1");
    ADB_REQUIRE(image && image_strides && dense_point && T_WC && idepth_pyr && (image_pyr || pyr_levels == 1) && rW2C &&
                    tW2C && approx_centre && R,
                "adb_kf_mapper_inputs: null pointer");
    ADB_REQUIRE(((uintptr_t)dense_point & 15) == 0, "adb_kf_mapper_inputs: dense_point must be 16-byte aligned");
    MiParams p{};
    p.H = height; p.W = width; p.Hs = Hs; p.Ws = Ws; p.L = pyr_levels;
    p.sy = height > 1 ? (float)(Hs - 1) / (float)(height - 1) : 0.f;
    p.sx = width > 1 ? (float)(Ws - 1) / (float)(width - 1) : 0.f;
    p.cs = image_strides[0]; p.ys = image_strides[1]; p.xs = image_strides[2];
    long long a = 0, b = 0;
    for (int l = 0; l < pyr_levels; ++l) {
        p.h[l] = height >> l;
        p.w[l] = width >> l;
        p.id_off[l] = a;
        p.im_off[l] = b;
        a += (long long)p.h[l] * p.w[l];
        if (l > 0) b += 3LL * p.h[l] * p.w[l];
    }
    const dim3 grid(adb_cdiv(width, TILE), adb_cdiv(height, TILE));
    mapper_inputs_kernel<<<grid, dim3(TILE, MI_ROWS), 0, stream>>>(p, image, (const float4*)dense_point, T_WC, idepth_pyr,
                                                                   image_pyr, rW2C, tW2C, approx_centre, R);
    ADB_CHECK_LAUNCH("mapper_inputs_kernel");
    return ADB_OK;
}

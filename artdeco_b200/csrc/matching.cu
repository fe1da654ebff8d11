// Dense matching after a MASt3R pair (SURVEY.md §8f rank 1): the reference's mast3r_slam_backends.iter_proj /
// refine_matches (VSLAM/backend/src/matching_kernels.cu:26-116, 119-316; bindings gn.cpp:84-112) and the PyTorch glue around
// them in VSLAM/utils_matching.py:59-190 (ray image + Scharr-like gradients, point normalisation, occlusion test, linear
// index), as four streaming kernels:
//   match_prep      X11 -> rays_with_grad [B,H,W,9] (normalised ray, d/du, d/dv; reflect padding), X21 -> unit vectors,
//                   initial pixel guesses from a linear index (utils_matching.py:61-97,120-145) -- one pass instead of
//                   normalize + pad + 2 grouped conv2d + cat + permute + contiguous;
//   iter_proj       per-pixel Levenberg-Marquardt on the bilinear ray image (matching_kernels.cu:119-276);
//   match_finalize  integer pixel (truncation, as .long()), occlusion test ||X11[p] - X21|| < dist_thresh, AND with the LM
//                   convergence flag (utils_matching.py:166-174);
//   refine_matches  descriptor search in a dilated window (matching_kernels.cu:26-83) with the reference's fp16 arithmetic
//                   reproduced exactly (product and running sum each rounded to half, sequential over the feature dim), two
//                   candidates per HMUL2/HADD2, 128-bit descriptor gathers; also emits the linear index u + W v.
// The reference launches 16-thread blocks (BLOCK 16, matching_kernels.cu:14); here 128 threads per CTA.
#include "common.cuh"
#include <cuda_fp16.h>

namespace {

__device__ __forceinline__ float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }

__device__ __forceinline__ int reflect(int i, int n) {   // F.pad(mode="reflect") by one pixel
    if (i < 0) return -i;
    if (i >= n) return 2 * n - 2 - i;
    return i;
}

__device__ __forceinline__ void unit3(const float* __restrict__ p, float* o) {   // F.normalize(dim=-1), eps 1e-12
    const float x = p[0], y = p[1], z = p[2];
    const float n = fmaxf(sqrtf(x * x + y * y + z * z), 1e-12f);
    o[0] = x / n; o[1] = y / n; o[2] = z / n;
}

__global__ void __launch_bounds__(128)
match_prep_kernel(int H, int W, const float* __restrict__ X11, const float* __restrict__ X21,
                  const long long* __restrict__ idx_init, float* __restrict__ rays, float* __restrict__ pts,
                  float* __restrict__ p_init) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= H * W) return;
    const int v = n / W, u = n - v * W;
    const float* X = X11 + (size_t)b * H * W * 3;
    float r[3][3][3];
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dx = 0; dx < 3; ++dx)
            unit3(X + ((size_t)reflect(v + dy - 1, H) * W + reflect(u + dx - 1, W)) * 3, r[dy][dx]);
    float* o = rays + ((size_t)b * H * W + n) * 9;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        // utils_matching.py:66-83: gx = [[-3,0,3],[-10,0,10],[-3,0,3]]/32, gy its transpose
        const float gx = (-3.f * r[0][0][c] + 3.f * r[0][2][c] - 10.f * r[1][0][c] + 10.f * r[1][2][c] -
                          3.f * r[2][0][c] + 3.f * r[2][2][c]) * (1.0f / 32.0f);
        const float gy = (-3.f * r[0][0][c] - 10.f * r[0][1][c] - 3.f * r[0][2][c] + 3.f * r[2][0][c] +
                          10.f * r[2][1][c] + 3.f * r[2][2][c]) * (1.0f / 32.0f);
        o[c] = r[1][1][c];
        o[3 + c] = gx;
        o[6 + c] = gy;
    }
    const size_t q = (size_t)b * H * W + n;
    unit3(X21 + q * 3, pts + q * 3);
    const long long li = idx_init ? idx_init[q] : (long long)n;
    // lin_to_pixel (utils_matching.py:99-103) is torch's % and //, which floor: a negative index maps to
    // (li mod W in [0, W), floor(li / W)), not C's truncated quotient and signed remainder
    long long vi = li / W, ui = li - vi * W;
    if (ui < 0) { ui += W; --vi; }
    p_init[q * 2] = (float)ui;
    p_init[q * 2 + 1] = (float)vi;
}

struct Bilin {
    const float *r11, *r12, *r21, *r22;
    float w11, w12, w21, w22;
};
__device__ __forceinline__ Bilin bilin_setup(const float* __restrict__ img, int W, float u, float v) {
    // matching_kernels.cu:153-170: weights are named after the OPPOSITE corner's area
    const int u11 = (int)floorf(u), v11 = (int)floorf(v);
    const float du = u - (float)u11, dv = v - (float)v11;
    Bilin s;
    s.w11 = du * dv; s.w12 = (1.0f - du) * dv; s.w21 = du * (1.0f - dv); s.w22 = (1.0f - du) * (1.0f - dv);
    s.r11 = img + ((size_t)(v11 + 1) * W + u11 + 1) * 9;
    s.r12 = img + ((size_t)(v11 + 1) * W + u11) * 9;
    s.r21 = img + ((size_t)v11 * W + u11 + 1) * 9;
    s.r22 = img + ((size_t)v11 * W + u11) * 9;
    return s;
}
__device__ __forceinline__ float bilin(const Bilin& s, int j) {
    return s.w11 * __ldg(s.r11 + j) + s.w12 * __ldg(s.r12 + j) + s.w21 * __ldg(s.r21 + j) + s.w22 * __ldg(s.r22 + j);
}

__global__ void __launch_bounds__(128)
iter_proj_kernel(int H, int W, int n_pts, const float* __restrict__ rays, const float* __restrict__ pts,
                 const float* __restrict__ p_init, int max_iter, float lambda_init, float cost_thresh,
                 float* __restrict__ p_new, unsigned char* __restrict__ converged) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= n_pts) return;
    const float* img = rays + (size_t)b * H * W * 9;
    const size_t q = (size_t)b * n_pts + n;
    const float t0 = pts[q * 3], t1 = pts[q * 3 + 1], t2 = pts[q * 3 + 2];
    float u = clampf(p_init[q * 2], 1.f, (float)(W - 2));
    float v = clampf(p_init[q * 2 + 1], 1.f, (float)(H - 2));
    float lambda = lambda_init;
    bool conv = false;
    for (int it = 0; it < max_iter; ++it) {
        float r[3], gx[3], gy[3];
        {
            const Bilin s = bilin_setup(img, W, u, v);
#pragma unroll
            for (int j = 0; j < 3; ++j) { r[j] = bilin(s, j); gx[j] = bilin(s, 3 + j); gy[j] = bilin(s, 6 + j); }
        }
        float inv = 1.0f / sqrtf(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
        const float e0 = r[0] * inv - t0, e1 = r[1] * inv - t1, e2 = r[2] * inv - t2;
        const float cost = e0 * e0 + e1 * e1 + e2 * e2;
        const float A00 = gx[0] * gx[0] + gx[1] * gx[1] + gx[2] * gx[2] + lambda;
        const float A01 = gx[0] * gy[0] + gx[1] * gy[1] + gx[2] * gy[2];
        const float A11 = gy[0] * gy[0] + gy[1] * gy[1] + gy[2] * gy[2] + lambda;
        const float b0 = -(e0 * gx[0] + e1 * gx[1] + e2 * gx[2]);
        const float b1 = -(e0 * gy[0] + e1 * gy[1] + e2 * gy[2]);
        const float det_inv = 1.0f / (A00 * A11 - A01 * A01);
        const float un = clampf(u + det_inv * (A11 * b0 - A01 * b1), 1.f, (float)(W - 2));
        const float vn = clampf(v + det_inv * (-A01 * b0 + A00 * b1), 1.f, (float)(H - 2));
        float new_cost;
        {
            const Bilin s = bilin_setup(img, W, un, vn);
            const float a0 = bilin(s, 0), a1 = bilin(s, 1), a2 = bilin(s, 2);
            inv = 1.0f / sqrtf(a0 * a0 + a1 * a1 + a2 * a2);
            const float f0 = a0 * inv - t0, f1 = a1 * inv - t1, f2 = a2 * inv - t2;
            new_cost = f0 * f0 + f1 * f1 + f2 * f2;
        }
        if (new_cost < cost) {            // matching_kernels.cu:255-264
            u = un; v = vn;
            lambda = (float)((double)lambda * 0.1);     // the reference multiplies by a double literal
            conv = new_cost < cost_thresh;
        } else {
            lambda = (float)((double)lambda * 10.0);
            conv = cost < cost_thresh;
        }
    }
    p_new[q * 2] = u;
    p_new[q * 2 + 1] = v;
    converged[q] = conv ? 1 : 0;
}

__global__ void __launch_bounds__(128)
match_finalize_kernel(int H, int W, const float* __restrict__ X11, const float* __restrict__ X21,
                      const float* __restrict__ p, const unsigned char* __restrict__ converged, float dist_thresh,
                      long long* __restrict__ p1, unsigned char* __restrict__ valid) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= H * W) return;
    const size_t q = (size_t)b * H * W + n;
    const long long u = (long long)p[q * 2], v = (long long)p[q * 2 + 1];     // .long(): truncation
    p1[q * 2] = u;
    p1[q * 2 + 1] = v;
    const float* a = X11 + ((size_t)b * H * W + (size_t)v * W + u) * 3;
    const float* c = X21 + q * 3;
    const float dx = a[0] - c[0], dy = a[1] - c[1], dz = a[2] - c[2];
    const float d = sqrtf(dx * dx + dy * dy + dz * dz);
    valid[q] = (converged[q] && d < dist_thresh) ? 1 : 0;
}

// F halfs per descriptor, F % 8 == 0 (16-byte gathers).  Scores are formed exactly as the reference's c10::Half arithmetic
// does (Half.h operator*, operator+=: float op, result rounded to half == HMUL / HADD in round-to-nearest): per candidate
// s = 0; for k: s = rn16(s + rn16(d21[k] * d11[k])).  Two candidates ride in the two halves of a __half2.
// PLANAR: descriptors stored chunk-planar [b][F/8][pixels][8 halfs] (adb_desc_pack_f16): the 32 lanes of a warp, which
// look at 32 neighbouring pixels, then read 512 contiguous bytes per 128-bit load (4 lines) instead of 16 B at a 48 B
// stride (12 lines) -- the row-major kernel is bound by L1 wavefronts, not by arithmetic.
template <int F, bool PLANAR>
__global__ void __launch_bounds__(128)
refine_matches_kernel(int H, int W, int n_pts, const __half* __restrict__ D11, const __half* __restrict__ D21,
                      const long long* __restrict__ p1, int radius, int dilation_max, long long* __restrict__ p1_new,
                      long long* __restrict__ lin_idx) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= n_pts) return;
    const size_t q = (size_t)b * n_pts + n;
    __half2 d2[F];   // query feature k duplicated in both halves
    {
        const uint4* src = reinterpret_cast<const uint4*>(D21) + (PLANAR ? ((size_t)b * (F / 8) * n_pts + n) : q * (F / 8));
        const size_t qstep = PLANAR ? (size_t)n_pts : 1;
#pragma unroll
        for (int k8 = 0; k8 < F / 8; ++k8) {
            const uint4 w = __ldg(src + k8 * qstep);
            const __half* hh = reinterpret_cast<const __half*>(&w);
#pragma unroll
            for (int k = 0; k < 8; ++k) d2[k8 * 8 + k] = __half2half2(hh[k]);
        }
    }
    const uint4* img = reinterpret_cast<const uint4*>(D11) + (size_t)b * H * W * (F / 8);
    const size_t cstep = PLANAR ? (size_t)H * W : 1;      // distance between a pixel's consecutive 16-byte chunks
    const size_t pstep = PLANAR ? 1 : (F / 8);           // distance between neighbouring pixels' first chunks
    long long u0 = p1[q * 2], v0 = p1[q * 2 + 1];
    long long u_new = u0, v_new = v0;
    // matching_kernels.cu:47 starts from ::cuda::std::numeric_limits<c10::Half>::min(); libcu++ does not specialise
    // numeric_limits for c10::Half, so that is Half() == 0: any positive score wins, a score <= 0 never does
    float max_score = 0.f;
    for (int d = dilation_max; d > 0; --d) {
        const int rd = radius * d;
        const int cnt = (2 * rd) / d + 1;     // i = 0, d, 2d, .. < 2rd+1
        for (int i = 0; i < cnt; ++i) {
            const long long uu = u0 - rd + (long long)i * d;
            const bool u_ok = uu >= 0 && uu < W;
            for (int j = 0; j < cnt; j += 2) {
                // candidates (i, j) and (i, j+1): the reference visits j in increasing order with a strict '>' update
                const long long va = v0 - rd + (long long)j * d, vb = va + d;
                const bool a_ok = u_ok && va >= 0 && va < H;
                const bool b_ok = u_ok && (j + 1 < cnt) && vb >= 0 && vb < H;
                if (!a_ok && !b_ok) continue;
                const uint4* pa = img + ((size_t)(a_ok ? va : vb) * W + uu) * pstep;
                const uint4* pb = img + ((size_t)(b_ok ? vb : va) * W + uu) * pstep;
                __half2 s = __float2half2_rn(0.f);
#pragma unroll
                for (int k8 = 0; k8 < F / 8; ++k8) {
                    const uint4 wa = __ldg(pa + k8 * cstep), wb = __ldg(pb + k8 * cstep);
                    const __half* ha = reinterpret_cast<const __half*>(&wa);
                    const __half* hb = reinterpret_cast<const __half*>(&wb);
#pragma unroll
                    for (int k = 0; k < 8; ++k)
                        s = __hadd2_rn(s, __hmul2_rn(d2[k8 * 8 + k], __halves2half2(ha[k], hb[k])));   // _rn: never contracted to FMA
                }
                const float sa = __low2float(s), sb = __high2float(s);
                if (a_ok && sa > max_score) { max_score = sa; u_new = uu; v_new = va; }
                if (b_ok && sb > max_score) { max_score = sb; u_new = uu; v_new = vb; }
            }
        }
        u0 = u_new;
        v0 = v_new;
    }
    p1_new[q * 2] = u_new;
    p1_new[q * 2 + 1] = v_new;
    if (lin_idx) lin_idx[q] = u_new + (long long)W * v_new;
}

// fp32 [b, pixels, F] -> fp16 (round to nearest, == .half()) in the chunk-planar layout [b][F/8][pixels][8]
template <int F>
__global__ void __launch_bounds__(256)
desc_pack_kernel(long long n_pix, const float* __restrict__ src, __half* __restrict__ dst) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // (pixel, chunk) pairs, chunk fastest
    const int b = blockIdx.y;
    if (i >= n_pix * (F / 8)) return;
    const long long pix = i / (F / 8);
    const int k8 = (int)(i - pix * (F / 8));
    const float4* s4 = reinterpret_cast<const float4*>(src + ((size_t)b * n_pix + pix) * F + k8 * 8);
    const float4 x = __ldg(s4), y = __ldg(s4 + 1);
    __half2 h[4] = {__floats2half2_rn(x.x, x.y), __floats2half2_rn(x.z, x.w), __floats2half2_rn(y.x, y.y),
                    __floats2half2_rn(y.z, y.w)};
    reinterpret_cast<uint4*>(dst)[((size_t)b * (F / 8) + k8) * n_pix + pix] = *reinterpret_cast<uint4*>(h);
}

}  // namespace

ADB_API int adb_desc_pack_f16(int B, long long n_pix, int fdim, const float* src, void* dst_f16, cudaStream_t stream) {
    ADB_REQUIRE(B >= 0 && n_pix >= 0, "adb_desc_pack_f16: bad sizes");
    ADB_REQUIRE(fdim == 16 || fdim == 24 || fdim == 32, "adb_desc_pack_f16: descriptor dim must be 16, 24 or 32");
    if (B == 0 || n_pix == 0) return ADB_OK;
    ADB_REQUIRE(src && dst_f16, "adb_desc_pack_f16: null pointer");
    ADB_REQUIRE(((uintptr_t)src | (uintptr_t)dst_f16) % 16 == 0, "adb_desc_pack_f16: buffers must be 16-byte aligned");
    dim3 grid((unsigned)adb_cdiv(n_pix * (fdim / 8), 256), B);
    __half* d = (__half*)dst_f16;
    if (fdim == 16) desc_pack_kernel<16><<<grid, 256, 0, stream>>>(n_pix, src, d);
    else if (fdim == 24) desc_pack_kernel<24><<<grid, 256, 0, stream>>>(n_pix, src, d);
    else desc_pack_kernel<32><<<grid, 256, 0, stream>>>(n_pix, src, d);
    ADB_CHECK_LAUNCH("desc_pack_kernel");
    return ADB_OK;
}

ADB_API int adb_match_prep(int B, int H, int W, const float* X11, const float* X21, const long long* idx_init,
                           float* rays_with_grad, float* pts3d_norm, float* p_init, cudaStream_t stream) {
    ADB_REQUIRE(B >= 0 && H >= 2 && W >= 2, "adb_match_prep: bad sizes (reflect padding needs H, W >= 2)");
    if (B == 0) return ADB_OK;
    ADB_REQUIRE(X11 && X21 && rays_with_grad && pts3d_norm && p_init, "adb_match_prep: null pointer");
    dim3 grid(adb_cdiv(H * W, 128), B);
    match_prep_kernel<<<grid, 128, 0, stream>>>(H, W, X11, X21, idx_init, rays_with_grad, pts3d_norm, p_init);
    ADB_CHECK_LAUNCH("match_prep_kernel");
    return ADB_OK;
}

ADB_API int adb_iter_proj(int B, int H, int W, int n_pts, const float* rays_with_grad, const float* pts3d_norm,
                          const float* p_init, int max_iter, float lambda_init, float cost_thresh, float* p_new,
                          unsigned char* converged, cudaStream_t stream) {
    ADB_REQUIRE(B >= 0 && H >= 3 && W >= 3 && n_pts >= 0 && max_iter >= 0, "adb_iter_proj: bad sizes (needs H, W >= 3)");
    if (B == 0 || n_pts == 0) return ADB_OK;
    ADB_REQUIRE(rays_with_grad && pts3d_norm && p_init && p_new && converged, "adb_iter_proj: null pointer");
    dim3 grid(adb_cdiv(n_pts, 128), B);
    iter_proj_kernel<<<grid, 128, 0, stream>>>(H, W, n_pts, rays_with_grad, pts3d_norm, p_init, max_iter, lambda_init,
                                              cost_thresh, p_new, converged);
    ADB_CHECK_LAUNCH("iter_proj_kernel");
    return ADB_OK;
}

ADB_API int adb_match_finalize(int B, int H, int W, const float* X11, const float* X21, const float* p,
                               const unsigned char* converged, float dist_thresh, long long* p1, unsigned char* valid,
                               cudaStream_t stream) {
    ADB_REQUIRE(B >= 0 && H > 0 && W > 0, "adb_match_finalize: bad sizes");
    if (B == 0) return ADB_OK;
    ADB_REQUIRE(X11 && X21 && p && converged && p1 && valid, "adb_match_finalize: null pointer");
    dim3 grid(adb_cdiv(H * W, 128), B);
    match_finalize_kernel<<<grid, 128, 0, stream>>>(H, W, X11, X21, p, converged, dist_thresh, p1, valid);
    ADB_CHECK_LAUNCH("match_finalize_kernel");
    return ADB_OK;
}

ADB_API int adb_refine_matches(int B, int H, int W, int fdim, int n_pts, const void* D11_f16, const void* D21_f16,
                               int planar, const long long* p1, int radius, int dilation_max, long long* p1_new,
                               long long* lin_idx, cudaStream_t stream) {
    ADB_REQUIRE(B >= 0 && H > 0 && W > 0 && n_pts >= 0 && radius >= 0 && dilation_max >= 0, "adb_refine_matches: bad sizes");
    ADB_REQUIRE(fdim == 16 || fdim == 24 || fdim == 32, "adb_refine_matches: descriptor dim must be 16, 24 or 32");
    if (B == 0 || n_pts == 0) return ADB_OK;
    ADB_REQUIRE(D11_f16 && D21_f16 && p1 && p1_new, "adb_refine_matches: null pointer");
    ADB_REQUIRE(((uintptr_t)D11_f16 | (uintptr_t)D21_f16) % 16 == 0, "adb_refine_matches: descriptors must be 16-byte aligned");
    dim3 grid(adb_cdiv(n_pts, 128), B);
    const __half* a = (const __half*)D11_f16;
    const __half* c = (const __half*)D21_f16;
#define ADB_REFINE(FD, PL) refine_matches_kernel<FD, PL><<<grid, 128, 0, stream>>>(H, W, n_pts, a, c, p1, radius, dilation_max, p1_new, lin_idx)
    if (planar) {
        if (fdim == 16) ADB_REFINE(16, true); else if (fdim == 24) ADB_REFINE(24, true); else ADB_REFINE(32, true);
    } else {
        if (fdim == 16) ADB_REFINE(16, false); else if (fdim == 24) ADB_REFINE(24, false); else ADB_REFINE(32, false);
    }
#undef ADB_REFINE
    ADB_CHECK_LAUNCH("refine_matches_kernel");
    return ADB_OK;
}

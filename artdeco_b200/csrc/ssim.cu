// Fused differentiable SSIM (11x11 separable Gaussian window, zero padding) for sm_90a.
//
// Replaces the reference's fused-ssim extension:
//   Reconstruct/submodules/fused-ssim/ssim.cu:62   fusedssimCUDA
//   Reconstruct/submodules/fused-ssim/ssim.cu:286  fusedssim_backwardCUDA
//   Reconstruct/submodules/fused-ssim/ssim.cu:434  fusedssim (host)       -> adb_ssim_forward
//   Reconstruct/submodules/fused-ssim/ssim.cu:480  fusedssim_backward     -> adb_ssim_backward
//
// Design differences (not a translation):
//  * 32x32 output tile per CTA (halo read amplification 1.72x instead of 2.64x), one CTA per
//    (tile, batch*channel) plane so the grid is ~3.1k CTAs at 1080p x 3ch (24 waves over 132 SMs).
//  * no memsets: every output element is written exactly once by the kernel (the reference
//    zero-fills four tensors first, ssim.cu:455-460).
//  * optional fused mean: the per-CTA sum of the SSIM map is reduced in-kernel and added to a
//    scalar, so the training path never has to write or re-read the map itself.
//  * backward accepts a uniform upstream gradient (dL/dmap == const, which is what `map.mean()`
//    produces) without reading a dL_dmap tensor.
// Arithmetic follows the reference's summation order (symmetric tap pairs, then centre) with IEEE
// division (the reference is built with --use_fast_math; we are not).
#include "common.cuh"

namespace {

constexpr int TILE = 32;
constexpr int HALO = 5;
constexpr int SH = TILE + 2 * HALO;  // 42
constexpr int SPITCH = SH + 1;       // 43, odd pitch
constexpr int NTHREADS = 256;

__constant__ float cG[11] = {
    0.001028380123898387f, 0.0075987582094967365f, 0.036000773310661316f, 0.10936068743467331f,
    0.21300552785396576f,  0.26601171493530273f,   0.21300552785396576f,  0.10936068743467331f,
    0.036000773310661316f, 0.0075987582094967365f, 0.001028380123898387f};

template <bool TRAIN>
__global__ void __launch_bounds__(NTHREADS)
ssim_fwd_kernel(int H, int W, float C1, float C2,
                const float* __restrict__ img1, const float* __restrict__ img2,
                float* __restrict__ ssim_map, float* __restrict__ dm_dmu1,
                float* __restrict__ dm_dsigma1_sq, float* __restrict__ dm_dsigma12,
                float* __restrict__ ssim_sum) {
    __shared__ float sX[SH][SPITCH];
    __shared__ float sY[SH][SPITCH];
    __shared__ float sC[5][SH][TILE];
    __shared__ float sRed[NTHREADS / 32];

    const int tid = threadIdx.x;
    const int tx = tid & 31, ty = tid >> 5;
    const size_t plane = (size_t)blockIdx.z * H * W;
    const float* p1 = img1 + plane;
    const float* p2 = img2 + plane;
    const int x0 = blockIdx.x * TILE - HALO;
    const int y0 = blockIdx.y * TILE - HALO;

    // 1) halo tile of both images, zero padded
    for (int i = tid; i < SH * SH; i += NTHREADS) {
        int ly = i / SH, lx = i - ly * SH;
        int gy = y0 + ly, gx = x0 + lx;
        float a = 0.f, b = 0.f;
        if (gx >= 0 && gx < W && gy >= 0 && gy < H) {
            a = __ldg(p1 + (size_t)gy * W + gx);
            b = __ldg(p2 + (size_t)gy * W + gx);
        }
        sX[ly][lx] = a;
        sY[ly][lx] = b;
    }
    __syncthreads();

    // 2) horizontal 11-tap for the five statistics
    for (int row = ty; row < SH; row += NTHREADS / 32) {
        const int lx = tx + HALO;
        float sx = 0.f, sx2 = 0.f, sy = 0.f, sy2 = 0.f, sxy = 0.f;
#pragma unroll
        for (int d = 1; d <= HALO; ++d) {
            float w = cG[HALO - d];
            float xl = sX[row][lx - d], yl = sY[row][lx - d];
            float xr = sX[row][lx + d], yr = sY[row][lx + d];
            sx += (xl + xr) * w;
            sx2 += ((xl * xl) + (xr * xr)) * w;
            sy += (yl + yr) * w;
            sy2 += ((yl * yl) + (yr * yr)) * w;
            sxy += ((xl * yl) + (xr * yr)) * w;
        }
        {
            float xc = sX[row][lx], yc = sY[row][lx], wc = cG[HALO];
            sx += xc * wc;
            sx2 += (xc * xc) * wc;
            sy += yc * wc;
            sy2 += (yc * yc) * wc;
            sxy += (xc * yc) * wc;
        }
        sC[0][row][tx] = sx;
        sC[1][row][tx] = sx2;
        sC[2][row][tx] = sy;
        sC[3][row][tx] = sy2;
        sC[4][row][tx] = sxy;
    }
    __syncthreads();

    // 3) vertical 11-tap + SSIM + partial derivatives
    float local_sum = 0.f;
#pragma unroll
    for (int k = 0; k < TILE / (NTHREADS / 32); ++k) {
        const int oy = ty + k * (NTHREADS / 32);
        const int ly = oy + HALO;
        float o0 = 0.f, o1 = 0.f, o2 = 0.f, o3 = 0.f, o4 = 0.f;
#pragma unroll
        for (int d = 1; d <= HALO; ++d) {
            float w = cG[HALO - d];
            o0 += (sC[0][ly - d][tx] + sC[0][ly + d][tx]) * w;
            o1 += (sC[1][ly - d][tx] + sC[1][ly + d][tx]) * w;
            o2 += (sC[2][ly - d][tx] + sC[2][ly + d][tx]) * w;
            o3 += (sC[3][ly - d][tx] + sC[3][ly + d][tx]) * w;
            o4 += (sC[4][ly - d][tx] + sC[4][ly + d][tx]) * w;
        }
        {
            float wc = cG[HALO];
            o0 += sC[0][ly][tx] * wc;
            o1 += sC[1][ly][tx] * wc;
            o2 += sC[2][ly][tx] * wc;
            o3 += sC[3][ly][tx] * wc;
            o4 += sC[4][ly][tx] * wc;
        }
        const int px = blockIdx.x * TILE + tx, py = blockIdx.y * TILE + oy;
        if (px < W && py < H) {
            float mu1 = o0, mu2 = o2;
            float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2;
            float sigma1_sq = o1 - mu1_sq;
            float sigma2_sq = o3 - mu2_sq;
            float sigma12 = o4 - mu1 * mu2;
            float A = mu1_sq + mu2_sq + C1;
            float B = sigma1_sq + sigma2_sq + C2;
            float C_ = 2.f * mu1 * mu2 + C1;
            float D_ = 2.f * sigma12 + C2;
            float val = (C_ * D_) / (A * B);
            size_t gi = plane + (size_t)py * W + px;
            if (ssim_map) ssim_map[gi] = val;
            local_sum += val;
            if (TRAIN) {
                float AB = A * B;
                float d_mu1 = (mu2 * 2.f * D_) / AB - (mu2 * 2.f * C_) / AB -
                              (mu1 * 2.f * C_ * D_) / (A * AB) + (mu1 * 2.f * C_ * D_) / (AB * B);
                dm_dmu1[gi] = d_mu1;
                dm_dsigma1_sq[gi] = (-C_ * D_) / (AB * B);
                dm_dsigma12[gi] = (2.f * C_) / AB;
            }
        }
    }
    if (ssim_sum) {
        local_sum = adb_warp_sum(local_sum);
        if (tx == 0) sRed[ty] = local_sum;
        __syncthreads();
        if (tid < 32) {
            float v = tid < NTHREADS / 32 ? sRed[tid] : 0.f;
            v = adb_warp_sum(v);
            if (tid == 0) atomicAdd(ssim_sum, v);
        }
    }
}

__global__ void __launch_bounds__(NTHREADS)
ssim_bwd_kernel(int H, int W,
                const float* __restrict__ img1, const float* __restrict__ img2,
                const float* __restrict__ dL_dmap, const float* __restrict__ dL_scalar, float dL_scale,
                const float* __restrict__ dm_dmu1, const float* __restrict__ dm_dsigma1_sq,
                const float* __restrict__ dm_dsigma12, float* __restrict__ dL_dimg1) {
    __shared__ float sD[3][SH][SPITCH];
    __shared__ float sS[3][SH][TILE];

    const int tid = threadIdx.x;
    const int tx = tid & 31, ty = tid >> 5;
    const size_t plane = (size_t)blockIdx.z * H * W;
    const int x0 = blockIdx.x * TILE - HALO;
    const int y0 = blockIdx.y * TILE - HALO;
    const float dL_uniform = (dL_scalar ? __ldg(dL_scalar) : 1.f) * dL_scale;

    for (int i = tid; i < SH * SH; i += NTHREADS) {
        int ly = i / SH, lx = i - ly * SH;
        int gy = y0 + ly, gx = x0 + lx;
        float a = 0.f, b = 0.f, c = 0.f;
        if (gx >= 0 && gx < W && gy >= 0 && gy < H) {
            size_t gi = plane + (size_t)gy * W + gx;
            float chain = dL_dmap ? __ldg(dL_dmap + gi) : dL_uniform;
            a = __ldg(dm_dmu1 + gi) * chain;
            b = __ldg(dm_dsigma1_sq + gi) * chain;
            c = __ldg(dm_dsigma12 + gi) * chain;
        }
        sD[0][ly][lx] = a;
        sD[1][ly][lx] = b;
        sD[2][ly][lx] = c;
    }
    __syncthreads();

    for (int row = ty; row < SH; row += NTHREADS / 32) {
        const int lx = tx + HALO;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll
        for (int d = 1; d <= HALO; ++d) {
            float w = cG[HALO - d];
            a0 += (sD[0][row][lx - d] + sD[0][row][lx + d]) * w;
            a1 += (sD[1][row][lx - d] + sD[1][row][lx + d]) * w;
            a2 += (sD[2][row][lx - d] + sD[2][row][lx + d]) * w;
        }
        float wc = cG[HALO];
        a0 += sD[0][row][lx] * wc;
        a1 += sD[1][row][lx] * wc;
        a2 += sD[2][row][lx] * wc;
        sS[0][row][tx] = a0;
        sS[1][row][tx] = a1;
        sS[2][row][tx] = a2;
    }
    __syncthreads();

#pragma unroll
    for (int k = 0; k < TILE / (NTHREADS / 32); ++k) {
        const int oy = ty + k * (NTHREADS / 32);
        const int ly = oy + HALO;
        const int px = blockIdx.x * TILE + tx, py = blockIdx.y * TILE + oy;
        if (px < W && py < H) {
            float s0 = 0.f, s1 = 0.f, s2 = 0.f;
#pragma unroll
            for (int d = 1; d <= HALO; ++d) {
                float w = cG[HALO - d];
                s0 += (sS[0][ly - d][tx] + sS[0][ly + d][tx]) * w;
                s1 += (sS[1][ly - d][tx] + sS[1][ly + d][tx]) * w;
                s2 += (sS[2][ly - d][tx] + sS[2][ly + d][tx]) * w;
            }
            float wc = cG[HALO];
            s0 += sS[0][ly][tx] * wc;
            s1 += sS[1][ly][tx] * wc;
            s2 += sS[2][ly][tx] * wc;
            size_t gi = plane + (size_t)py * W + px;
            float q1 = __ldg(img1 + gi), q2 = __ldg(img2 + gi);
            dL_dimg1[gi] = s0 + (2.f * q1) * s1 + q2 * s2;
        }
    }
}

}  // namespace

// ssim_map / ssim_sum may each be NULL (but not both); derivative pointers must be non-NULL iff train.
ADB_API int adb_ssim_forward(int B, int CH, int H, int W, float C1, float C2,
                             const float* img1, const float* img2, int train,
                             float* ssim_map, float* dm_dmu1, float* dm_dsigma1_sq,
                             float* dm_dsigma12, float* ssim_sum, cudaStream_t stream) {
    ADB_REQUIRE(B >= 0 && CH >= 0 && H >= 0 && W >= 0, "adb_ssim_forward: negative dimension");
    if ((long long)B * CH * H * W == 0) return ADB_OK;
    ADB_REQUIRE(img1 && img2, "adb_ssim_forward: null image pointer");
    ADB_REQUIRE(ssim_map || ssim_sum, "adb_ssim_forward: need ssim_map or ssim_sum");
    ADB_REQUIRE((long long)B * CH <= 65535, "adb_ssim_forward: B*CH exceeds grid.z limit");
    if (train) ADB_REQUIRE(dm_dmu1 && dm_dsigma1_sq && dm_dsigma12, "adb_ssim_forward: train needs derivative buffers");
    dim3 grid(adb_cdiv(W, TILE), adb_cdiv(H, TILE), B * CH);
    if (train)
        ssim_fwd_kernel<true><<<grid, NTHREADS, 0, stream>>>(H, W, C1, C2, img1, img2, ssim_map, dm_dmu1,
                                                            dm_dsigma1_sq, dm_dsigma12, ssim_sum);
    else
        ssim_fwd_kernel<false><<<grid, NTHREADS, 0, stream>>>(H, W, C1, C2, img1, img2, ssim_map, nullptr,
                                                             nullptr, nullptr, ssim_sum);
    ADB_CHECK_LAUNCH("ssim_fwd_kernel");
    return ADB_OK;
}

// dL_dmap may be NULL: then the upstream gradient of every map element is the constant
// (dL_scalar ? *dL_scalar : 1) * dL_scale, with dL_scalar a DEVICE pointer (no host sync needed).
ADB_API int adb_ssim_backward(int B, int CH, int H, int W, float C1, float C2,
                              const float* img1, const float* img2, const float* dL_dmap,
                              const float* dL_scalar, float dL_scale, const float* dm_dmu1, const float* dm_dsigma1_sq,
                              const float* dm_dsigma12, float* dL_dimg1, cudaStream_t stream) {
    (void)C1; (void)C2;
    ADB_REQUIRE(B >= 0 && CH >= 0 && H >= 0 && W >= 0, "adb_ssim_backward: negative dimension");
    if ((long long)B * CH * H * W == 0) return ADB_OK;
    ADB_REQUIRE(img1 && img2 && dm_dmu1 && dm_dsigma1_sq && dm_dsigma12 && dL_dimg1,
                "adb_ssim_backward: null pointer");
    ADB_REQUIRE((long long)B * CH <= 65535, "adb_ssim_backward: B*CH exceeds grid.z limit");
    dim3 grid(adb_cdiv(W, TILE), adb_cdiv(H, TILE), B * CH);
    ssim_bwd_kernel<<<grid, NTHREADS, 0, stream>>>(H, W, img1, img2, dL_dmap, dL_scalar, dL_scale, dm_dmu1,
                                                  dm_dsigma1_sq, dm_dsigma12, dL_dimg1);
    ADB_CHECK_LAUNCH("ssim_bwd_kernel");
    return ADB_OK;
}

// The mapper's per-step pixel loss, forward and backward, for sm_90a.
//
// Replaces the eager-PyTorch loss block of SceneModel.optimization_step:
//   Reconstruct/scene/scene_models/h3dgsv3.py:682-686  background composite and 1/D (SceneModel.render)
//   Reconstruct/scene/scene_models/h3dgsv3.py:611-614  exposure affine map and clamp(0, 1) (render_from_id)
//   Reconstruct/scene/scene_models/h3dgsv3.py:430-450  radial-weighted L1, the is_important=False error mask,
//                                                       1 - fused_ssim, the inverse-depth term, the weighted sum
//   and the autograd mirror of all of it.
//
// Design:
//  * one streaming pass per pixel reads the rasterizer's channels-last outputs directly (colors [h,w,4] as one 16 B load,
//    alphas [h,w]) and writes the two SSIM operands; the existing adb_ssim_forward / adb_ssim_backward do the window work;
//  * sums are per-CTA partials added by a single-CTA launch in a fixed order (double accumulation), never float atomics, so
//    the loss and the exposure gradient are bitwise reproducible;
//  * the backward recomputes the composite, exposure, clamp and mask from the inputs instead of saving them, and writes
//    v_colors [h,w,4] / v_alphas [h,w] in the layout the rasterizer's backward consumes.
// Element-wise arithmetic is rounded as PyTorch's separate eager kernels round it (no contraction across the composite),
// the 3x3 map as an FMA chain.
#include "common.cuh"

namespace {

constexpr int NT = 256;
constexpr int PPT = 4;                 // pixels per thread
constexpr int PIX_PER_CTA = NT * PPT;  // 1024
constexpr int NPART_FWD = 3;           // l1 sum, depth sum, ssim-map sum
constexpr int NPART_BWD = 12;          // dL/dE [3,4]

__host__ __device__ inline long long n_blocks(long long hw) { return (hw + PIX_PER_CTA - 1) / PIX_PER_CTA; }

// torch.sgn for real values: sgn(0) = 0 and sgn(NaN) = 0.
__device__ __forceinline__ float sgnf(float x) { return (float)(x > 0.f) - (float)(x < 0.f); }

// torch.clamp(x, 0, 1): NaN propagates.
__device__ __forceinline__ float clamp01(float x) { return isnan(x) ? x : fminf(fmaxf(x, 0.f), 1.f); }

struct Pixel {
    float c[3];   // composite colour
    float y[3];   // exposed, before the clamp
    float e[3];   // exposed, clamped
    float g[3];   // ground truth
    float inv;    // 1 / D (unmasked)
    float mono;
    float r;      // radial weight
    float m;      // mask as the float the reference multiplies by (1 or 0)
};

__device__ __forceinline__ void load_pixel(long long p, long long hw, const float4* __restrict__ colors,
                                           const float* __restrict__ alphas, const float* __restrict__ gt,
                                           const float* __restrict__ mono, const float* __restrict__ rdk,
                                           const float* sE, const float* sBg, int important, Pixel& px, float& depth) {
    const float4 c4 = adb_ldg_stream4(colors + p);
    const float om = __fsub_rn(1.f, __ldg(alphas + p));
    px.c[0] = __fadd_rn(c4.x, __fmul_rn(om, sBg[0]));
    px.c[1] = __fadd_rn(c4.y, __fmul_rn(om, sBg[1]));
    px.c[2] = __fadd_rn(c4.z, __fmul_rn(om, sBg[2]));
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float* e = sE + 4 * k;
        px.y[k] = __fadd_rn(fmaf(e[2], px.c[2], fmaf(e[1], px.c[1], __fmul_rn(e[0], px.c[0]))), e[3]);
        px.e[k] = clamp01(px.y[k]);
        px.g[k] = __ldg(gt + k * hw + p);
    }
    depth = c4.w;
    px.inv = 1.f / c4.w;
    px.mono = __ldg(mono + p);
    px.r = __ldg(rdk + p);
    px.m = 1.f;
    if (!important) {
        // h3dgsv3.py:433-435 verbatim: channel 1 is tested twice, channel 2 never.
        const float err0 = __fmul_rn(px.r, fabsf(__fsub_rn(px.e[0], px.g[0])));
        const float err1 = __fmul_rn(px.r, fabsf(__fsub_rn(px.e[1], px.g[1])));
        const bool drop = (err0 > 0.2f) | (err1 > 0.2f) | (err1 > 0.2f);
        px.m = drop ? 0.f : 1.f;
    }
}

// Deterministic block sum of NV values per thread into out[0..NV) (thread 0 of the block holds the result).
template <int NV>
__device__ __forceinline__ void block_sum(float (&v)[NV], float (*sRed)[NT / 32], float* out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const float s = adb_warp_sum(v[i]);
        if (lane == 0) sRed[i][warp] = s;
    }
    __syncthreads();
    if (threadIdx.x < NV) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < NT / 32; ++w) s += sRed[threadIdx.x][w];
        out[threadIdx.x] = s;
    }
}

__global__ void __launch_bounds__(NT)
mapper_loss_fwd_kernel(long long hw, const float4* __restrict__ colors, const float* __restrict__ alphas,
                       const float* __restrict__ gt, const float* __restrict__ mono, const float* __restrict__ exposure,
                       const float* __restrict__ bg, const float* __restrict__ rdk, int important,
                       float* __restrict__ img, float* __restrict__ gt_m, float* __restrict__ inv_out,
                       float* __restrict__ part) {
    __shared__ float sE[12], sBg[3];
    __shared__ float sRed[2][NT / 32];
    if (threadIdx.x < 12) sE[threadIdx.x] = __ldg(exposure + threadIdx.x);
    if (threadIdx.x < 3) sBg[threadIdx.x] = __ldg(bg + threadIdx.x);
    __syncthreads();
    float acc[2] = {0.f, 0.f};
#pragma unroll
    for (int k = 0; k < PPT; ++k) {
        const long long p = (long long)blockIdx.x * PIX_PER_CTA + k * NT + threadIdx.x;
        if (p >= hw) break;
        Pixel px;
        float depth;
        load_pixel(p, hw, colors, alphas, gt, mono, rdk, sE, sBg, important, px, depth);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float em = __fmul_rn(px.e[c], px.m), gm = __fmul_rn(px.g[c], px.m);
            img[c * hw + p] = em;
            gt_m[c * hw + p] = gm;
            acc[0] += __fmul_rn(px.r, fabsf(__fsub_rn(em, gm)));
        }
        const float invm = __fmul_rn(px.inv, px.m), mom = __fmul_rn(px.mono, px.m);
        if (inv_out) inv_out[p] = invm;
        acc[1] += __fmul_rn(px.r, fabsf(__fsub_rn(invm, mom)));
    }
    block_sum<2>(acc, sRed, part + (size_t)blockIdx.x * NPART_FWD);
}

// Per-CTA sums of the SSIM map over the same pixel blocks (3 channels each) into part[b*3 + 2].
__global__ void __launch_bounds__(NT)
ssim_map_partial_kernel(long long hw, const float* __restrict__ ssim_map, float* __restrict__ part) {
    __shared__ float sRed[1][NT / 32];
    float acc[1] = {0.f};
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int k = 0; k < PPT; ++k) {
            const long long p = (long long)blockIdx.x * PIX_PER_CTA + k * NT + threadIdx.x;
            if (p < hw) acc[0] += __ldg(ssim_map + c * hw + p);
        }
    block_sum<1>(acc, sRed, part + (size_t)blockIdx.x * NPART_FWD + 2);
}

// sums[j] = sum over b of part[b*stride + j], j < ncols, in a fixed order (warp j%8 strides the rows, lanes in double).
__device__ void column_sums(long long nrows, int stride, int ncols, const float* __restrict__ part, double* sums) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int j = warp; j < ncols; j += NT / 32) {
        double s = 0.0;
        for (long long b = lane; b < nrows; b += 32) s += (double)part[b * stride + j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) sums[j] = s;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(NT)
mapper_loss_fwd_final_kernel(long long hw, long long nblk, const float* __restrict__ part, float lambda_dssim,
                             float depth_weight, float* __restrict__ terms) {
    __shared__ double sums[NPART_FWD];
    column_sums(nblk, NPART_FWD, NPART_FWD, part, sums);
    if (threadIdx.x == 0) {
        const float l1 = (float)(sums[0] / (3.0 * (double)hw));
        const float depth = (float)(sums[1] / (double)hw);
        const float ssim = (float)(sums[2] / (3.0 * (double)hw));
        // h3dgsv3.py:441,445-448 (scaling_reg is per-Gaussian and stays with the caller)
        const float ssim_loss = 1.f - ssim;
        terms[0] = lambda_dssim * ssim_loss + (1.f - lambda_dssim) * l1 + depth_weight * depth;
        terms[1] = l1;
        terms[2] = ssim;
        terms[3] = depth;
    }
}

__global__ void __launch_bounds__(NT)
mapper_loss_bwd_kernel(long long hw, const float4* __restrict__ colors, const float* __restrict__ alphas,
                       const float* __restrict__ gt, const float* __restrict__ mono, const float* __restrict__ exposure,
                       const float* __restrict__ bg, const float* __restrict__ rdk, int important,
                       const float* __restrict__ dssim, const float* __restrict__ dL, float lambda_dssim,
                       float depth_weight, float4* __restrict__ v_colors, float* __restrict__ v_alphas,
                       float* __restrict__ part) {
    __shared__ float sE[12], sBg[3];
    __shared__ float sRed[NPART_BWD][NT / 32];
    if (threadIdx.x < 12) sE[threadIdx.x] = __ldg(exposure + threadIdx.x);
    if (threadIdx.x < 3) sBg[threadIdx.x] = __ldg(bg + threadIdx.x);
    __syncthreads();
    const float g = __ldg(dL);
    // d loss / d (per-element |.|) after the means: (g * w) / n, as the mul and mean backward compute it
    const float a_l1 = __fdiv_rn(__fmul_rn(g, 1.f - lambda_dssim), (float)(3 * hw));
    const float a_d = __fdiv_rn(__fmul_rn(g, depth_weight), (float)hw);
    float acc[NPART_BWD];
#pragma unroll
    for (int i = 0; i < NPART_BWD; ++i) acc[i] = 0.f;
#pragma unroll 1
    for (int k = 0; k < PPT; ++k) {
        const long long p = (long long)blockIdx.x * PIX_PER_CTA + k * NT + threadIdx.x;
        if (p >= hw) break;
        Pixel px;
        float depth;
        load_pixel(p, hw, colors, alphas, gt, mono, rdk, sE, sBg, important, px, depth);
        (void)depth;
        float dy[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float em = __fmul_rn(px.e[c], px.m), gm = __fmul_rn(px.g[c], px.m);
            const float d_img = __fadd_rn(__fmul_rn(__fmul_rn(a_l1, px.r), sgnf(__fsub_rn(em, gm))),
                                          __ldg(dssim + c * hw + p));
            const float d_e = __fmul_rn(d_img, px.m);
            dy[c] = (px.y[c] >= 0.f && px.y[c] <= 1.f) ? d_e : 0.f;   // clamp backward: inclusive bounds
        }
        const float invm = __fmul_rn(px.inv, px.m), mom = __fmul_rn(px.mono, px.m);
        const float d_inv = __fmul_rn(__fmul_rn(__fmul_rn(a_d, px.r), sgnf(__fsub_rn(invm, mom))), px.m);
        const float d_D = __fmul_rn(d_inv, -__fmul_rn(px.inv, px.inv));   // reciprocal backward: -g / D^2 = -g inv^2
        float dc[3];
#pragma unroll
        for (int j = 0; j < 3; ++j)
            dc[j] = fmaf(sE[8 + j], dy[2], fmaf(sE[4 + j], dy[1], __fmul_rn(sE[j], dy[0])));
        const float d_om = fmaf(dc[2], sBg[2], fmaf(dc[1], sBg[1], __fmul_rn(dc[0], sBg[0])));
        v_colors[p] = make_float4(dc[0], dc[1], dc[2], d_D);
        v_alphas[p] = -d_om;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            acc[4 * r + 0] = fmaf(dy[r], px.c[0], acc[4 * r + 0]);
            acc[4 * r + 1] = fmaf(dy[r], px.c[1], acc[4 * r + 1]);
            acc[4 * r + 2] = fmaf(dy[r], px.c[2], acc[4 * r + 2]);
            acc[4 * r + 3] += dy[r];
        }
    }
    block_sum<NPART_BWD>(acc, sRed, part + (size_t)blockIdx.x * NPART_BWD);
}

__global__ void __launch_bounds__(NT)
mapper_loss_bwd_final_kernel(long long nblk, const float* __restrict__ part, float* __restrict__ v_exposure) {
    __shared__ double sums[NPART_BWD];
    column_sums(nblk, NPART_BWD, NPART_BWD, part, sums);
    if (threadIdx.x < NPART_BWD) v_exposure[threadIdx.x] = (float)sums[threadIdx.x];
}

size_t part_bytes(long long hw, int ncols) { return (size_t)n_blocks(hw) * ncols * sizeof(float); }
size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// Workspace: [forward partials nblk x 3][backward partials nblk x 12], each 256 B aligned.
size_t ws_bytes_for(long long hw) { return align256(part_bytes(hw, NPART_FWD)) + align256(part_bytes(hw, NPART_BWD)); }

int check_size(int height, int width, const char* who) {
    if (height <= 0 || width <= 0) {
        adb_set_error_msg(who);
        return ADB_ERR_INVALID;
    }
    if (3LL * height * width > 0x7fffffffLL) {
        adb_set_error_msg(who);
        return ADB_ERR_INVALID;
    }
    return ADB_OK;
}

}  // namespace

ADB_API int adb_mapper_loss_workspace_bytes(int height, int width, size_t* bytes) {
    ADB_REQUIRE(bytes, "adb_mapper_loss_workspace_bytes: null bytes");
    if (int rc = check_size(height, width, "adb_mapper_loss_workspace_bytes: height and width must be > 0 and 3hw < 2^31"))
        return rc;
    *bytes = ws_bytes_for((long long)height * width);
    return ADB_OK;
}

ADB_API int adb_mapper_loss_forward(int height, int width, const float* colors, const float* alphas, const float* gt,
                                    const float* mono_idepth, const float* exposure, const float* bg, const float* rdk,
                                    int is_important, float* image, float* gt_masked, float* invdepth, void* ws,
                                    size_t ws_bytes, cudaStream_t stream) {
    if (int rc = check_size(height, width, "adb_mapper_loss_forward: height and width must be > 0 and 3hw < 2^31"))
        return rc;
    ADB_REQUIRE(colors && alphas && gt && mono_idepth && exposure && bg && rdk && image && gt_masked && ws,
                "adb_mapper_loss_forward: null pointer");
    ADB_REQUIRE(((uintptr_t)colors & 15) == 0, "adb_mapper_loss_forward: colors must be 16-byte aligned");
    const long long hw = (long long)height * width;
    if (ws_bytes < ws_bytes_for(hw)) {
        adb_set_error_msg("adb_mapper_loss_forward: workspace too small");
        return ADB_ERR_WORKSPACE;
    }
    const long long nblk = n_blocks(hw);
    mapper_loss_fwd_kernel<<<(unsigned)nblk, NT, 0, stream>>>(hw, (const float4*)colors, alphas, gt, mono_idepth, exposure,
                                                              bg, rdk, is_important != 0, image, gt_masked, invdepth,
                                                              (float*)ws);
    ADB_CHECK_LAUNCH("mapper_loss_fwd_kernel");
    return ADB_OK;
}

ADB_API int adb_mapper_loss_reduce(int height, int width, const float* ssim_map, float lambda_dssim, float depth_weight,
                                   float* terms, void* ws, size_t ws_bytes, cudaStream_t stream) {
    if (int rc = check_size(height, width, "adb_mapper_loss_reduce: height and width must be > 0 and 3hw < 2^31"))
        return rc;
    ADB_REQUIRE(ssim_map && terms && ws, "adb_mapper_loss_reduce: null pointer");
    const long long hw = (long long)height * width;
    if (ws_bytes < ws_bytes_for(hw)) {
        adb_set_error_msg("adb_mapper_loss_reduce: workspace too small");
        return ADB_ERR_WORKSPACE;
    }
    const long long nblk = n_blocks(hw);
    ssim_map_partial_kernel<<<(unsigned)nblk, NT, 0, stream>>>(hw, ssim_map, (float*)ws);
    ADB_CHECK_LAUNCH("ssim_map_partial_kernel");
    mapper_loss_fwd_final_kernel<<<1, NT, 0, stream>>>(hw, nblk, (const float*)ws, lambda_dssim, depth_weight, terms);
    ADB_CHECK_LAUNCH("mapper_loss_fwd_final_kernel");
    return ADB_OK;
}

ADB_API int adb_mapper_loss_backward(int height, int width, const float* colors, const float* alphas, const float* gt,
                                     const float* mono_idepth, const float* exposure, const float* bg, const float* rdk,
                                     int is_important, const float* dssim, const float* dL, float lambda_dssim,
                                     float depth_weight, float* v_colors, float* v_alphas, float* v_exposure, void* ws,
                                     size_t ws_bytes, cudaStream_t stream) {
    if (int rc = check_size(height, width, "adb_mapper_loss_backward: height and width must be > 0 and 3hw < 2^31"))
        return rc;
    ADB_REQUIRE(colors && alphas && gt && mono_idepth && exposure && bg && rdk && dssim && dL && v_colors && v_alphas &&
                    v_exposure && ws,
                "adb_mapper_loss_backward: null pointer");
    ADB_REQUIRE(((uintptr_t)colors & 15) == 0 && ((uintptr_t)v_colors & 15) == 0,
                "adb_mapper_loss_backward: colors and v_colors must be 16-byte aligned");
    const long long hw = (long long)height * width;
    if (ws_bytes < ws_bytes_for(hw)) {
        adb_set_error_msg("adb_mapper_loss_backward: workspace too small");
        return ADB_ERR_WORKSPACE;
    }
    const long long nblk = n_blocks(hw);
    float* part = (float*)((char*)ws + align256(part_bytes(hw, NPART_FWD)));
    mapper_loss_bwd_kernel<<<(unsigned)nblk, NT, 0, stream>>>(hw, (const float4*)colors, alphas, gt, mono_idepth, exposure,
                                                              bg, rdk, is_important != 0, dssim, dL, lambda_dssim,
                                                              depth_weight, (float4*)v_colors, v_alphas, part);
    ADB_CHECK_LAUNCH("mapper_loss_bwd_kernel");
    mapper_loss_bwd_final_kernel<<<1, NT, 0, stream>>>(nblk, part, v_exposure);
    ADB_CHECK_LAUNCH("mapper_loss_bwd_final_kernel");
    return ADB_OK;
}

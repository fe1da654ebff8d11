// Held-out key-frame evaluation for sm_90a: exposure harmonisation, PSNR, SSIM and LPIPS-VGG.
//
// Replaces the quality evaluation of the mapper:
//   Reconstruct/scene/scene_models/h3dgsv3.py:507-520   SceneModel.harmonize_test_exposure
//   Reconstruct/scene/scene_models/h3dgsv3.py:523-558   SceneModel.evaluate (render_from_id's exposure :611-614, bg = 0)
//   Reconstruct/utils.py:86-87                          psnr
//   Reconstruct/scene/scene_models/h3dgsv3.py:98        lpips.LPIPS(net="vgg") (version 0.1, spatial=False)
//
// Design:
//  * one streaming pass over the T stacked views reads the rasterizer's channels-last colors [T,h,w,4] / alphas [T,h,w],
//    applies the exposure and clamp, writes the planar image and per-CTA partials of the squared error; the existing
//    adb_ssim_forward writes the SSIM map of all T views in one launch and a second pass takes per-CTA partials of it
//    (its own ssim_sum is a float atomic, so it is not used: the metrics must be bitwise reproducible);
//  * LPIPS: conv1_1 (3 -> 64, K = 27) is a direct fp32 kernel with the ScalingLayer fused in; the other twelve 3x3
//    convolutions are adb_conv3x3_bf16 (wgmma, bf16x3, bias + ReLU epilogue); the 2x2 max-pool reads the fp32 tap and
//    writes the next layer's bf16 split; one head kernel per tap takes the channel norm, the squared difference and the
//    1x1 lin layer per pixel and writes per-CTA partials of the spatial mean;
//  * every sum is a per-CTA partial added by one single-CTA launch in a fixed order in double: no float atomics;
//  * nothing synchronises the device or allocates; the caller's evaluation workspace holds every partial.
#include "common.cuh"
#include "artdeco_b200.h"
#include <cuda_bf16.h>

namespace {

constexpr int NT = 256;
constexpr int PPT = 4;
constexpr int PIX_PER_CTA = NT * PPT;   // image-metric pass: 1024 pixels per CTA
constexpr int HEAD_PIX = 64;            // LPIPS head: 64 pixels per CTA (8 per warp)
constexpr int COUNT_PER_CTA = NT * 16;  // visibility count: 4096 flags per CTA
constexpr int NTAP = 5;
constexpr int NCONV = 13;
constexpr int N_METRICS = ADB_EVAL_N_METRICS;
constexpr int N_SUMS = 2 + NTAP + 1;    // per view: squared error, ssim map, five tap sums, visible count

// VGG16 up to relu5_3 (torchvision features[0:30]): channels per conv, which convs are taps (followed by a pool except
// the last).
constexpr int VGG_COUT[NCONV] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512};
constexpr bool VGG_TAP[NCONV] = {false, true, false, true, false, false, true, false, false, true, false, false, true};

__host__ __device__ inline long long cdivll(long long a, long long b) { return (a + b - 1) / b; }

struct Level {
    int H[NTAP], W[NTAP];
};
__host__ __device__ inline Level levels(int h, int w) {
    Level L;
    for (int l = 0; l < NTAP; ++l) {
        L.H[l] = h;
        L.W[l] = w;
        h /= 2;   // MaxPool2d(2, 2), ceil_mode=False
        w /= 2;
    }
    return L;
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// Evaluation workspace: per-view partial rows, then the double sums.
struct EvalLayout {
    long long nblk_img, nblk_cnt, nblk_tap[NTAP];
    size_t off_img, off_cnt, off_tap[NTAP], off_sums, total;
};
EvalLayout eval_layout(int T, int h, int w, long long n) {
    EvalLayout e;
    const Level L = levels(h, w);
    e.nblk_img = cdivll((long long)h * w, PIX_PER_CTA);
    e.nblk_cnt = n > 0 ? cdivll(n, COUNT_PER_CTA) : 1;
    size_t off = 0;
    e.off_img = off;
    off += align256((size_t)T * e.nblk_img * 2 * sizeof(float));
    e.off_cnt = off;
    off += align256((size_t)T * e.nblk_cnt * sizeof(unsigned long long));
    for (int l = 0; l < NTAP; ++l) {
        e.nblk_tap[l] = cdivll((long long)L.H[l] * L.W[l], HEAD_PIX);
        e.off_tap[l] = off;
        off += align256((size_t)T * e.nblk_tap[l] * sizeof(float));
    }
    e.off_sums = off;
    off += align256((size_t)T * N_SUMS * sizeof(double));
    e.total = off;
    return e;
}

// LPIPS activation workspace for nf frames (2 nf images): two bf16 split buffers (hi, lo) and one fp32 tap buffer.
struct LpipsLayout {
    size_t split_a, split_b, tap, total;   // element counts of A and B (each of hi and lo) and of the tap buffer
};
LpipsLayout lpips_layout(int nf, int h, int w) {
    constexpr int LEVEL_C[NTAP] = {64, 128, 256, 512, 512};
    const Level L = levels(h, w);
    LpipsLayout s{};
    // A holds conv1_1's output and every pool output, B the other non-tap outputs from level 1 on (conv3_2, 4_2 and 5_2
    // write A again), the tap buffer every tap; each level's activations are [2 nf, H_l, W_l, C_l]
    for (int l = 0; l < NTAP; ++l) {
        const size_t n = (size_t)2 * nf * L.H[l] * L.W[l] * LEVEL_C[l];
        s.split_a = n > s.split_a ? n : s.split_a;
        if (l > 0) s.split_b = n > s.split_b ? n : s.split_b;
        s.tap = n > s.tap ? n : s.tap;
    }
    s.total = 2 * align256(s.split_a * 2) + 2 * align256(s.split_b * 2) + align256(s.tap * 4);
    return s;
}

// torch.clamp(x, 0, 1): NaN propagates.
__device__ __forceinline__ float clamp01(float x) { return isnan(x) ? x : fminf(fmaxf(x, 0.f), 1.f); }

__device__ __forceinline__ void split2(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
    hi = __float2bfloat16_rn(v);
    lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// Deterministic block sum of one value per thread; thread 0 returns the result.
__device__ __forceinline__ float block_sum1(float v, float* sRed) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = adb_warp_sum(v);
    if (lane == 0) sRed[warp] = v;
    __syncthreads();
    float s = 0.f;
    if (threadIdx.x == 0)
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += sRed[i];
    return s;
}

// ---- exposure harmonisation: one thread walks the K key frames in order, exactly as the Python loop does ----
__global__ void harmonize_kernel(int K, float* __restrict__ E, const uint8_t* __restrict__ is_test, int* __restrict__ n_bad) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    int bad = 0;
    for (int i = 0; i < K; ++i) {
        if (!is_test[i]) continue;
        int im = i != 0 ? i - 1 : 1;
        int ip = i != K - 1 ? i + 1 : K - 2;
        // Python list indexing: [-K, K) is valid, negatives wrap; anything else raises IndexError, which stops the loop
        if (im < -K || im >= K || ip < -K || ip >= K) {
            bad = 1;
            break;
        }
        if (im < 0) im += K;
        if (ip < 0) ip += K;
        for (int j = 0; j < 12; ++j) E[12 * i + j] = __fdiv_rn(__fadd_rn(E[12 * im + j], E[12 * ip + j]), 2.f);
    }
    *n_bad = bad;
}

// ---- visible-Gaussian count of one view: per-CTA integer partials ----
__global__ void __launch_bounds__(NT)
count_visible_kernel(long long n, const uint8_t* __restrict__ mask, unsigned long long* __restrict__ part) {
    __shared__ unsigned sRed[NT / 32];
    unsigned c = 0;
    const long long base = (long long)blockIdx.x * COUNT_PER_CTA;
#pragma unroll 4
    for (int k = 0; k < COUNT_PER_CTA / NT; ++k) {
        const long long i = base + (long long)k * NT + threadIdx.x;
        if (i < n) c += mask[i] != 0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) sRed[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long s = 0;
        for (int i = 0; i < NT / 32; ++i) s += sRed[i];
        part[blockIdx.x] = s;
    }
}

// ---- image metrics: exposure, clamp, planar image and squared-error partials ----
__global__ void __launch_bounds__(NT)
image_pass_kernel(long long hw, long long nblk, const float4* __restrict__ colors, const float* __restrict__ alphas,
                  const float* __restrict__ E, const int* __restrict__ view_frame, const float* __restrict__ gt,
                  float* __restrict__ image, float* __restrict__ part) {
    __shared__ float sE[12];
    __shared__ float sRed[NT / 32];
    const int t = blockIdx.y;
    if (threadIdx.x < 12) sE[threadIdx.x] = E[12LL * view_frame[t] + threadIdx.x];
    __syncthreads();
    const float4* col = colors + (size_t)t * hw;
    const float* alp = alphas + (size_t)t * hw;
    const float* g = gt + (size_t)t * 3 * hw;
    float* img = image + (size_t)t * 3 * hw;
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < PPT; ++k) {
        const long long p = (long long)blockIdx.x * PIX_PER_CTA + k * NT + threadIdx.x;
        if (p >= hw) break;
        const float4 c4 = adb_ldg_stream4(col + p);
        const float om0 = __fmul_rn(__fsub_rn(1.f, __ldg(alp + p)), 0.f);   // render's (1 - alpha) * bg with bg = 0
        const float c[3] = {__fadd_rn(c4.x, om0), __fadd_rn(c4.y, om0), __fadd_rn(c4.z, om0)};
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            const float* e = sE + 4 * ch;
            const float y = __fadd_rn(fmaf(e[2], c[2], fmaf(e[1], c[1], __fmul_rn(e[0], c[0]))), e[3]);
            const float v = clamp01(y);
            img[ch * hw + p] = v;
            const float d = __fsub_rn(v, __ldg(g + ch * hw + p));
            acc = fmaf(d, d, acc);
        }
    }
    const float s = block_sum1(acc, sRed);
    if (threadIdx.x == 0) part[((size_t)t * nblk + blockIdx.x) * 2] = s;
}

__global__ void __launch_bounds__(NT)
ssim_partial_kernel(long long hw, long long nblk, const float* __restrict__ ssim_map, float* __restrict__ part) {
    __shared__ float sRed[NT / 32];
    const int t = blockIdx.y;
    const float* m = ssim_map + (size_t)t * 3 * hw;
    float acc = 0.f;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch)
#pragma unroll
        for (int k = 0; k < PPT; ++k) {
            const long long p = (long long)blockIdx.x * PIX_PER_CTA + k * NT + threadIdx.x;
            if (p < hw) acc += __ldg(m + ch * hw + p);
        }
    const float s = block_sum1(acc, sRed);
    if (threadIdx.x == 0) part[((size_t)t * nblk + blockIdx.x) * 2 + 1] = s;
}

// ---- LPIPS conv1_1: ScalingLayer + 3x3 conv (3 -> 64) + bias + ReLU, fp32, written as the NHWC bf16 split ----
// Network image n = 2 f + s: s = 0 the render (in0), s = 1 the ground truth (in1) of frame f.
constexpr int C1_NT = 128;
__global__ void __launch_bounds__(C1_NT)
lpips_conv1_kernel(int h, int w, const float* __restrict__ img0, const float* __restrict__ img1,
                   const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ shift,
                   const float* __restrict__ scale, __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo) {
    __shared__ float sW[27][64];   // [ci*9 + ky*3 + kx][co]
    __shared__ float sB[64];
    for (int i = threadIdx.x; i < 27 * 64; i += C1_NT) sW[i % 27][i / 27] = __ldg(w1 + i);
    if (threadIdx.x < 64) sB[threadIdx.x] = __ldg(b1 + threadIdx.x);
    __syncthreads();
    const long long hw = (long long)h * w;
    const long long p = (long long)blockIdx.x * C1_NT + threadIdx.x;
    if (p >= hw) return;
    const int n = blockIdx.y, f = n >> 1;
    const float* src = ((n & 1) ? img1 : img0) + (size_t)f * 3 * hw;
    const int y = (int)(p / w), x = (int)(p % w);
    float in[27];
#pragma unroll
    for (int ci = 0; ci < 3; ++ci) {
        const float sh = __ldg(shift + ci), sc = __ldg(scale + ci);
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int yy = y + ky - 1, xx = x + kx - 1;
                // zero padding applies to the scaled input (ScalingLayer runs before the conv)
                in[ci * 9 + ky * 3 + kx] = (yy >= 0 && yy < h && xx >= 0 && xx < w)
                                               ? __fdiv_rn(__fsub_rn(__ldg(src + ci * hw + (long long)yy * w + xx), sh), sc)
                                               : 0.f;
            }
    }
    const size_t o = ((size_t)n * hw + p) * 64;
#pragma unroll 1
    for (int c0 = 0; c0 < 64; c0 += 8) {
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = sB[c0 + j];
#pragma unroll
        for (int k = 0; k < 27; ++k)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = fmaf(sW[k][c0 + j], in[k], acc[j]);
        __align__(16) __nv_bfloat16 hi[8], lo[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) split2(fmaxf(acc[j], 0.f), hi[j], lo[j]);
        *reinterpret_cast<uint4*>(out_hi + o + c0) = *reinterpret_cast<const uint4*>(hi);
        *reinterpret_cast<uint4*>(out_lo + o + c0) = *reinterpret_cast<const uint4*>(lo);
    }
}

// ---- 2x2 / stride 2 max-pool (floor) of an fp32 NHWC tap into the next layer's bf16 split ----
__device__ __forceinline__ float maxnan(float a, float b) { return (a > b || isnan(a)) ? a : b; }   // NaN propagates

__global__ void __launch_bounds__(NT)
maxpool_kernel(long long total4, int H, int W, int C, const float* __restrict__ x, __nv_bfloat16* __restrict__ hi,
               __nv_bfloat16* __restrict__ lo) {
    const int Ho = H / 2, Wo = W / 2, C4 = C / 4;
    for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < total4; i += (long long)gridDim.x * NT) {
        const int c = (int)(i % C4) * 4;
        long long r = i / C4;
        const int xo = (int)(r % Wo);
        r /= Wo;
        const int yo = (int)(r % Ho);
        const long long n = r / Ho;
        const float* b = x + ((n * H + 2 * yo) * W + 2 * xo) * C + c;
        const float4 a = __ldg(reinterpret_cast<const float4*>(b));
        const float4 bb = __ldg(reinterpret_cast<const float4*>(b + C));
        const float4 cc = __ldg(reinterpret_cast<const float4*>(b + (long long)W * C));
        const float4 d = __ldg(reinterpret_cast<const float4*>(b + (long long)W * C + C));
        const float v[4] = {maxnan(maxnan(a.x, bb.x), maxnan(cc.x, d.x)), maxnan(maxnan(a.y, bb.y), maxnan(cc.y, d.y)),
                            maxnan(maxnan(a.z, bb.z), maxnan(cc.z, d.z)), maxnan(maxnan(a.w, bb.w), maxnan(cc.w, d.w))};
        __align__(8) __nv_bfloat16 h4[4], l4[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) split2(v[j], h4[j], l4[j]);
        const size_t o = (size_t)i * 4;
        *reinterpret_cast<uint2*>(hi + o) = *reinterpret_cast<const uint2*>(h4);
        *reinterpret_cast<uint2*>(lo + o) = *reinterpret_cast<const uint2*>(l4);
    }
}

// ---- LPIPS head of one tap: per pixel sum_c lin_c (x0/(|x0|+eps) - x1/(|x1|+eps))^2, per-CTA partials ----
__global__ void __launch_bounds__(NT)
lpips_head_kernel(long long hw, int C, long long nblk, const float* __restrict__ feat, const float* __restrict__ lin,
                  float* __restrict__ part) {
    __shared__ float sRed[NT / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int f = blockIdx.y;
    const float* f0 = feat + (size_t)(2 * f) * hw * C;
    const float* f1 = feat + (size_t)(2 * f + 1) * hw * C;
    float acc = 0.f;   // lane 0: this warp's pixels in order
    for (int k = 0; k < HEAD_PIX / (NT / 32); ++k) {
        const long long p = (long long)blockIdx.x * HEAD_PIX + warp * (HEAD_PIX / (NT / 32)) + k;
        if (p >= hw) break;
        const float* a = f0 + p * C;
        const float* b = f1 + p * C;
        float s0 = 0.f, s1 = 0.f;
        for (int c = lane; c < C; c += 32) {
            const float u = __ldg(a + c), v = __ldg(b + c);
            s0 = fmaf(u, u, s0);
            s1 = fmaf(v, v, s1);
        }
        s0 = adb_warp_sum(s0);
        s1 = adb_warp_sum(s1);
        const float n0 = __fadd_rn(__fsqrt_rn(s0), 1e-10f), n1 = __fadd_rn(__fsqrt_rn(s1), 1e-10f);
        float d = 0.f;
        for (int c = lane; c < C; c += 32) {
            const float e = __fsub_rn(__fdiv_rn(__ldg(a + c), n0), __fdiv_rn(__ldg(b + c), n1));
            d = fmaf(__ldg(lin + c), __fmul_rn(e, e), d);
        }
        d = adb_warp_sum(d);
        acc += d;
    }
    const float s = block_sum1(lane == 0 ? acc : 0.f, sRed);
    if (threadIdx.x == 0) part[(size_t)f * nblk + blockIdx.x] = s;
}

// ---- final reduction: one CTA adds every view's partial rows in a fixed order in double and writes the table ----
__global__ void __launch_bounds__(NT)
eval_reduce_kernel(int T, long long hw, long long n_gauss, EvalLayout e, const char* __restrict__ ws, int with_lpips,
                   double* __restrict__ sums, double* __restrict__ table) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float* pimg = (const float*)(ws + e.off_img);
    const unsigned long long* pcnt = (const unsigned long long*)(ws + e.off_cnt);
    for (int job = warp; job < T * N_SUMS; job += NT / 32) {
        const int t = job / N_SUMS, k = job % N_SUMS;
        double s = 0.0;
        if (k < 2) {
            for (long long b = lane; b < e.nblk_img; b += 32) s += (double)pimg[((size_t)t * e.nblk_img + b) * 2 + k];
        } else if (k < 2 + NTAP) {
            if (with_lpips) {
#pragma unroll
                for (int l = 0; l < NTAP; ++l)   // static indices keep the layout in the parameter bank
                    if (k == 2 + l) {
                        const float* p = (const float*)(ws + e.off_tap[l]) + (size_t)t * e.nblk_tap[l];
                        for (long long b = lane; b < e.nblk_tap[l]; b += 32) s += (double)p[b];
                    }
            }
        } else {
            for (long long b = lane; b < e.nblk_cnt; b += 32) s += (double)pcnt[(size_t)t * e.nblk_cnt + b];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) sums[(size_t)t * N_SUMS + k] = s;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < T; t += NT) {
        const double* S = sums + (size_t)t * N_SUMS;
        double* R = table + (size_t)t * N_METRICS;
        const float mse = (float)(S[0] / (3.0 * (double)hw));
        // psnr (utils.py:86-87) in fp32, as the tensor expression 10 * log10(1 / mse) evaluates it
        const float psnr = __fmul_rn(10.f, log10f(__frcp_rn(mse)));
        const float ssim = (float)(S[1] / (3.0 * (double)hw));
        R[0] = psnr;
        R[1] = ssim;
        R[3] = (double)S[2 + NTAP];   // Render: visibility_filter.sum()
        R[4] = (double)n_gauss;       // GS: len(visibility_filter)
        R[5] = mse;
        for (int l = 0; l < NTAP; ++l) R[6 + l] = NAN;
        R[2] = with_lpips ? 0.0 : NAN;   // filled by lpips_finish_kernel
    }
}

__global__ void __launch_bounds__(NT)
lpips_finish_kernel(int T, int h, int w, const double* __restrict__ sums, double* __restrict__ table) {
    const Level L = levels(h, w);
    for (int t = threadIdx.x; t < T; t += NT) {
        const double* S = sums + (size_t)t * N_SUMS;
        double* R = table + (size_t)t * N_METRICS;
        float val = 0.f;   // lpips.LPIPS.forward: val = 0; val += res[l] for l in 0..4, in fp32
        for (int l = 0; l < NTAP; ++l) {
            const float m = (float)(S[2 + l] / ((double)L.H[l] * L.W[l]));   // spatial_average
            R[6 + l] = m;
            val = l == 0 ? m : __fadd_rn(val, m);
        }
        R[2] = val;
    }
}

int check_eval(int T, int h, int w, long long n, const char* who) {
    if (T <= 0 || h <= 0 || w <= 0 || n < 0 || 3LL * T * h * w > 0x7fffffffLL * 8LL || (long long)T > 65535) {
        adb_set_error_msg(who);
        return ADB_ERR_INVALID;
    }
    return ADB_OK;
}

}  // namespace

ADB_API int adb_eval_workspace_bytes(int T, int height, int width, long long n_gaussians, size_t* bytes) {
    ADB_REQUIRE(bytes, "adb_eval_workspace_bytes: null bytes");
    if (int rc = check_eval(T, height, width, n_gaussians, "adb_eval_workspace_bytes: need T in [1, 65535], h, w > 0, n >= 0"))
        return rc;
    *bytes = eval_layout(T, height, width, n_gaussians).total;
    return ADB_OK;
}

ADB_API int adb_eval_harmonize(int K, float* exposure, const uint8_t* is_test, int* n_bad, cudaStream_t stream) {
    ADB_REQUIRE(K >= 1, "adb_eval_harmonize: K must be >= 1");
    ADB_REQUIRE(exposure && is_test && n_bad, "adb_eval_harmonize: null pointer");
    harmonize_kernel<<<1, 32, 0, stream>>>(K, exposure, is_test, n_bad);
    ADB_CHECK_LAUNCH("harmonize_kernel");
    return ADB_OK;
}

ADB_API int adb_eval_count_visible(int T, int height, int width, long long n_gaussians, int t, const uint8_t* mask,
                                   void* ws, size_t ws_bytes, cudaStream_t stream) {
    if (int rc = check_eval(T, height, width, n_gaussians, "adb_eval_count_visible: need T in [1, 65535], h, w > 0, n >= 0"))
        return rc;
    ADB_REQUIRE(t >= 0 && t < T, "adb_eval_count_visible: view index out of range");
    ADB_REQUIRE(ws && (mask || n_gaussians == 0), "adb_eval_count_visible: null pointer");
    const EvalLayout e = eval_layout(T, height, width, n_gaussians);
    if (ws_bytes < e.total) {
        adb_set_error_msg("adb_eval_count_visible: workspace too small");
        return ADB_ERR_WORKSPACE;
    }
    unsigned long long* part = (unsigned long long*)((char*)ws + e.off_cnt) + (size_t)t * e.nblk_cnt;
    if (n_gaussians == 0) {
        ADB_CUDA(cudaMemsetAsync(part, 0, sizeof(unsigned long long), stream));
        return ADB_OK;
    }
    count_visible_kernel<<<(unsigned)e.nblk_cnt, NT, 0, stream>>>(n_gaussians, mask, part);
    ADB_CHECK_LAUNCH("count_visible_kernel");
    return ADB_OK;
}

ADB_API int adb_eval_image_metrics(int T, int height, int width, long long n_gaussians, const float* colors,
                                   const float* alphas, const float* exposure, const int* view_frame, const float* gt,
                                   float* image, float* ssim_map, void* ws, size_t ws_bytes, cudaStream_t stream) {
    if (int rc = check_eval(T, height, width, n_gaussians, "adb_eval_image_metrics: need T in [1, 65535], h, w > 0, n >= 0"))
        return rc;
    ADB_REQUIRE(colors && alphas && exposure && view_frame && gt && image && ssim_map && ws,
                "adb_eval_image_metrics: null pointer");
    ADB_REQUIRE(((uintptr_t)colors & 15) == 0, "adb_eval_image_metrics: colors must be 16-byte aligned");
    const EvalLayout e = eval_layout(T, height, width, n_gaussians);
    if (ws_bytes < e.total) {
        adb_set_error_msg("adb_eval_image_metrics: workspace too small");
        return ADB_ERR_WORKSPACE;
    }
    const long long hw = (long long)height * width;
    float* part = (float*)((char*)ws + e.off_img);
    image_pass_kernel<<<dim3((unsigned)e.nblk_img, T), NT, 0, stream>>>(hw, e.nblk_img, (const float4*)colors, alphas,
                                                                        exposure, view_frame, gt, image, part);
    ADB_CHECK_LAUNCH("image_pass_kernel");
    // fused_ssim(image, gt, train=False): C1 = 0.01^2, C2 = 0.03^2 (fused_ssim/__init__.py)
    if (int rc = adb_ssim_forward(T, 3, height, width, 0.01f * 0.01f, 0.03f * 0.03f, image, gt, 0, ssim_map, nullptr,
                                  nullptr, nullptr, nullptr, stream))
        return rc;
    ssim_partial_kernel<<<dim3((unsigned)e.nblk_img, T), NT, 0, stream>>>(hw, e.nblk_img, ssim_map, part);
    ADB_CHECK_LAUNCH("ssim_partial_kernel");
    return ADB_OK;
}

ADB_API int adb_lpips_workspace_bytes(int n_frames, int height, int width, size_t* bytes) {
    ADB_REQUIRE(bytes, "adb_lpips_workspace_bytes: null bytes");
    ADB_REQUIRE(n_frames >= 1 && height >= 16 && width >= 16, "adb_lpips_workspace_bytes: need n_frames >= 1, h, w >= 16");
    *bytes = lpips_layout(n_frames, height, width).total;
    return ADB_OK;
}

ADB_API int adb_lpips_vgg_forward(int T, int height, int width, long long n_gaussians, int frame0, int n_frames,
                                  const float* img0, const float* img1, const float* w1, const float* b1,
                                  const float* shift, const float* scale, const void* const* w_hi, const void* const* w_lo,
                                  const float* const* bias, const float* const* lin, float* const* taps, void* lws,
                                  size_t lws_bytes, void* ews, size_t ews_bytes, cudaStream_t stream) {
    if (int rc = check_eval(T, height, width, n_gaussians, "adb_lpips_vgg_forward: need T in [1, 65535], h, w > 0, n >= 0"))
        return rc;
    ADB_REQUIRE(height >= 16 && width >= 16, "adb_lpips_vgg_forward: h and w must be >= 16 (four 2x2 pools)");
    ADB_REQUIRE(frame0 >= 0 && n_frames >= 1 && frame0 + n_frames <= T, "adb_lpips_vgg_forward: frame range outside [0, T)");
    ADB_REQUIRE(img0 && img1 && w1 && b1 && shift && scale && w_hi && w_lo && bias && lin && lws && ews,
                "adb_lpips_vgg_forward: null pointer");
    for (int i = 0; i < NCONV - 1; ++i)
        ADB_REQUIRE(w_hi[i] && w_lo[i] && bias[i], "adb_lpips_vgg_forward: null conv weight");
    for (int l = 0; l < NTAP; ++l) ADB_REQUIRE(lin[l], "adb_lpips_vgg_forward: null lin weight");
    const EvalLayout e = eval_layout(T, height, width, n_gaussians);
    const LpipsLayout s = lpips_layout(n_frames, height, width);
    if (ews_bytes < e.total || lws_bytes < s.total) {
        adb_set_error_msg("adb_lpips_vgg_forward: workspace too small");
        return ADB_ERR_WORKSPACE;
    }
    const Level L = levels(height, width);
    const int N = 2 * n_frames;
    char* base = (char*)lws;
    __nv_bfloat16* a_hi = (__nv_bfloat16*)base;
    __nv_bfloat16* a_lo = (__nv_bfloat16*)(base + align256(s.split_a * 2));
    __nv_bfloat16* b_hi = (__nv_bfloat16*)(base + 2 * align256(s.split_a * 2));
    __nv_bfloat16* b_lo = (__nv_bfloat16*)(base + 2 * align256(s.split_a * 2) + align256(s.split_b * 2));
    float* tapbuf = (float*)(base + 2 * align256(s.split_a * 2) + 2 * align256(s.split_b * 2));
    const long long hw = (long long)height * width;
    const float* in0 = img0 + (size_t)frame0 * 3 * hw;
    const float* in1 = img1 + (size_t)frame0 * 3 * hw;

    lpips_conv1_kernel<<<dim3((unsigned)cdivll(hw, C1_NT), N), C1_NT, 0, stream>>>(height, width, in0, in1, w1, b1, shift,
                                                                                    scale, a_hi, a_lo);
    ADB_CHECK_LAUNCH("lpips_conv1_kernel");
    // the current input split: which buffer, its channel count and level
    bool in_a = true;
    int cin = 64, lvl = 0, tap = 0;
    for (int i = 1; i < NCONV; ++i) {
        const int H = L.H[lvl], W = L.W[lvl], cout = VGG_COUT[i];
        const void* xh = in_a ? (const void*)a_hi : (const void*)b_hi;
        const void* xl = in_a ? (const void*)a_lo : (const void*)b_lo;
        if (VGG_TAP[i]) {
            float* D = taps && taps[tap] ? taps[tap] : tapbuf;
            if (int rc = adb_conv3x3_bf16(N, H, W, cin, cout, xh, xl, w_hi[i - 1], w_lo[i - 1], bias[i - 1], nullptr, D,
                                          nullptr, nullptr, 2, 0, stream))
                return rc;
            const long long nb = cdivll((long long)H * W, HEAD_PIX);
            float* part = (float*)((char*)ews + e.off_tap[tap]) + (size_t)frame0 * nb;
            lpips_head_kernel<<<dim3((unsigned)nb, n_frames), NT, 0, stream>>>((long long)H * W, cout, nb, D, lin[tap], part);
            ADB_CHECK_LAUNCH("lpips_head_kernel");
            if (tap < NTAP - 1) {
                const long long total4 = (long long)N * (H / 2) * (W / 2) * (cout / 4);
                const unsigned grid = (unsigned)min(cdivll(total4, NT), 132LL * 16);
                maxpool_kernel<<<grid, NT, 0, stream>>>(total4, H, W, cout, D, a_hi, a_lo);
                ADB_CHECK_LAUNCH("maxpool_kernel");
                in_a = true;
                ++lvl;
            }
            ++tap;
        } else {
            if (int rc = adb_conv3x3_bf16(N, H, W, cin, cout, xh, xl, w_hi[i - 1], w_lo[i - 1], bias[i - 1], nullptr,
                                          nullptr, in_a ? b_hi : a_hi, in_a ? b_lo : a_lo, 2, 0, stream))
                return rc;
            in_a = !in_a;
        }
        cin = cout;
    }
    return ADB_OK;
}

ADB_API int adb_eval_reduce(int T, int height, int width, long long n_gaussians, int with_lpips, void* ws,
                            size_t ws_bytes, double* table, cudaStream_t stream) {
    if (int rc = check_eval(T, height, width, n_gaussians, "adb_eval_reduce: need T in [1, 65535], h, w > 0, n >= 0"))
        return rc;
    ADB_REQUIRE(ws && table, "adb_eval_reduce: null pointer");
    const EvalLayout e = eval_layout(T, height, width, n_gaussians);
    if (ws_bytes < e.total) {
        adb_set_error_msg("adb_eval_reduce: workspace too small");
        return ADB_ERR_WORKSPACE;
    }
    double* sums = (double*)((char*)ws + e.off_sums);
    eval_reduce_kernel<<<1, NT, 0, stream>>>(T, (long long)height * width, n_gaussians, e, (const char*)ws,
                                             with_lpips != 0, sums, table);
    ADB_CHECK_LAUNCH("eval_reduce_kernel");
    if (with_lpips) {
        lpips_finish_kernel<<<1, NT, 0, stream>>>(T, height, width, sums, table);
        ADB_CHECK_LAUNCH("lpips_finish_kernel");
    }
    return ADB_OK;
}

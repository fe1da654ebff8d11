// Pi3-specific kernels (VSLAM/thirdparty/Pi3/pi3/models/).  Everything dense runs on the wgmma GEMM and the fused
// attention kernel; these are the stages that do not fit them:
//   pi3_patch14      ImageNet normalisation + 14x14/s14 im2col into the bf16 split GEMM operand   pi3.py:174, patch_embed.py:75
//   pi3_tokens       [cls + pos0, 4 registers, patches + pos] token assembly              vision_transformer.py:215-234
//   qknorm_rope      per-head LayerNorm(64, eps) of q or k, RoPE2D, head split            layers/attention.py:326-334
//   pi3_point_head   pixel-shuffle(14), local_points = (xy e^z, e^z), points = pose [lp, 1]   pi3.py:193-209, transformer_head.py:70-80
//   pi3_camera_tail  token average pool, 512-wide ReLU MLP, fc_t / fc_rot in fp32         layers/camera_head.py:48-61
//   pi3_svd_pose     row-normalise, R = V diag(1,1,det(V U^T)) U^T by fp64 Jacobi SVD, 4x4 pose   camera_head.py:66-93
//   pi3_window_input inverse_normalize + bilinear resize (align_corners=False)            mast3r_slam/retrieval_database.py:21-41
#include "common.cuh"
#include <cuda_bf16.h>

#include "pi3_svd.cuh"

namespace {

constexpr int P14 = 14;
constexpr int K14 = 3 * P14 * P14;       // 588 taps per patch
constexpr int K14_PAD = 592;             // GEMM row stride: a multiple of 8 elements (16 bytes of bf16)

__device__ __forceinline__ void split_store(__nv_bfloat16* hi, __nv_bfloat16* lo, size_t i, float v) {
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    hi[i] = h;
    if (lo) lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
}

// out[(bn * n + p) * 592 + (c, ky, kx)] = (img[bn, c, py*14+ky, px*14+kx] - mean[c]) / std[c]; columns 588..591 are 0.
__global__ void __launch_bounds__(256)
patch14_kernel(int BN, int H, int W, const float* __restrict__ img, __nv_bfloat16* __restrict__ hi,
               __nv_bfloat16* __restrict__ lo) {
    const int gw = W / P14, n = (H / P14) * gw;
    const long long total = (long long)BN * n * K14_PAD;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(i % K14_PAD);
        const long long row = i / K14_PAD;
        float v = 0.f;
        if (k < K14) {
            const int p = (int)(row % n), bn = (int)(row / n);
            const int c = k / (P14 * P14), r = k % (P14 * P14);
            const int y = (p / gw) * P14 + r / P14, x = (p % gw) * P14 + r % P14;
            const float mean = c == 0 ? 0.485f : (c == 1 ? 0.456f : 0.406f);
            const float stdv = c == 0 ? 0.229f : (c == 1 ? 0.224f : 0.225f);
            v = __fdiv_rn(img[(((size_t)bn * 3 + c) * H + y) * W + x] - mean, stdv);
        }
        split_store(hi, lo, (size_t)i, v);
    }
}

// x[bn, 0] = cls + pos[0]; x[bn, 1..4] = reg; x[bn, 5 + p] = patch[bn * n + p] + pos[1 + p]   (C % 4 == 0)
__global__ void __launch_bounds__(256)
tokens_kernel(int BN, int n, int C, const float* __restrict__ patch, const float* __restrict__ cls,
              const float* __restrict__ reg, const float* __restrict__ pos, float* __restrict__ x) {
    const int C4 = C / 4, T = n + 5;
    const long long total = (long long)BN * T * C4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4) * 4;
        const long long bt = i / C4;
        const int t = (int)(bt % T), bn = (int)(bt / T);
        float4 v;
        if (t == 0) {
            const float4 a = *reinterpret_cast<const float4*>(cls + c), b = *reinterpret_cast<const float4*>(pos + c);
            v = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
        } else if (t < 5) {
            v = *reinterpret_cast<const float4*>(reg + (size_t)(t - 1) * C + c);
        } else {
            const float4 a = *reinterpret_cast<const float4*>(patch + ((size_t)bn * n + (t - 5)) * C + c);
            const float4 b = *reinterpret_cast<const float4*>(pos + (size_t)(t - 4) * C + c);
            v = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
        }
        *reinterpret_cast<float4*>(x + (size_t)bt * C + c) = v;
    }
}

// One warp per (token, head): lane owns dims (lane, lane + 32), i.e. the same index of the y half and the x half.
// LayerNorm over the 64 dims, then rotate_half RoPE inside each 32-dim half (partner dim = lane ^ 16).
// x: fp32 [B*N, ld], this section's heads start at col0; out: bf16 split [B, h, N, 64].
__global__ void __launch_bounds__(256)
qknorm_rope_kernel(int B, int N, int h, long long ld, int col0, const float* __restrict__ x,
                   const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                   const long long* __restrict__ pos, const float2* __restrict__ table, int n_pos,
                   __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= (long long)B * N * h) return;
    const int hh = (int)(warp % h);
    const long long bn = warp / h;
    const int n = (int)(bn % N), b = (int)(bn / N);
    const float* xr = x + (size_t)bn * ld + col0 + hh * 64;
    float a = xr[lane], c = xr[lane + 32];
    if (gamma) {
        const float mean = adb_warp_sum(a + c) / 64.f;
        const float da = a - mean, dc = c - mean;
        const float var = adb_warp_sum(da * da + dc * dc) / 64.f;
        const float rstd = 1.0f / sqrtf(var + eps);
        a = da * rstd * gamma[lane] + beta[lane];
        c = dc * rstd * gamma[lane + 32] + beta[lane + 32];
    }
    const float pa = __shfl_xor_sync(0xffffffffu, a, 16), pc = __shfl_xor_sync(0xffffffffu, c, 16);
    long long py = pos[(size_t)bn * 2], px = pos[(size_t)bn * 2 + 1];
    py = py < 0 ? 0 : (py >= n_pos ? n_pos - 1 : py);
    px = px < 0 ? 0 : (px >= n_pos ? n_pos - 1 : px);
    const int j = lane & 15;
    const float2 cy = table[py * 16 + j], cx = table[px * 16 + j];
    const bool first = lane < 16;
    const float ya = first ? a * cy.x - pa * cy.y : a * cy.x + pa * cy.y;
    const float xc = first ? c * cx.x - pc * cx.y : c * cx.x + pc * cx.y;
    const size_t o = (((size_t)b * h + hh) * N + n) * 64;
    split_store(hi, lo, o + lane, ya);
    split_store(hi, lo, o + lane + 32, xc);
}

// One thread per output pixel.  pts: [BN * hw, 588] (token row bn*hw + skip + p; column c*196 + iy*14 + ix),
// cf: [BN * hw, 196], pose: [BN, 4, 4]; outputs [BN, H, W, 3|3|1].
__global__ void __launch_bounds__(256)
point_head_kernel(int BN, int H, int W, int hw, int skip, const float* __restrict__ pts, const float* __restrict__ cf,
                  const float* __restrict__ pose, float* __restrict__ points, float* __restrict__ local_points,
                  float* __restrict__ conf) {
    const long long total = (long long)BN * H * W;
    const int gw = W / P14;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int X = (int)(i % W);
        const long long r = i / W;
        const int Y = (int)(r % H), bn = (int)(r / H);
        const size_t row = (size_t)bn * hw + skip + (Y / P14) * gw + X / P14;
        const int j = (Y % P14) * P14 + X % P14;
        const float* f = pts + row * K14;
        const float z = expf(f[2 * P14 * P14 + j]);
        const float l0 = f[j] * z, l1 = f[P14 * P14 + j] * z;
        const float* P = pose + (size_t)bn * 16;
        local_points[i * 3 + 0] = l0;
        local_points[i * 3 + 1] = l1;
        local_points[i * 3 + 2] = z;
#pragma unroll
        for (int a = 0; a < 3; ++a) points[i * 3 + a] = P[a * 4 + 0] * l0 + P[a * 4 + 1] * l1 + P[a * 4 + 2] * z + P[a * 4 + 3];
        conf[i] = cf[row * (P14 * P14) + j];
    }
}

// One 512-thread block per view: mean over the hw - skip patch tokens, relu(W0 f + b0), relu(W2 . + b2), then
// fc_t (3) and fc_rot (9), all fp32.  w0t / w2t are the MLP weights transposed ([in][out]) so thread o reads row k
// of every matrix coalesced.
__global__ void __launch_bounds__(512)
camera_tail_kernel(int hw, int skip, const float* __restrict__ feat, const float* __restrict__ w0t,
                   const float* __restrict__ b0, const float* __restrict__ w2t, const float* __restrict__ b2,
                   const float* __restrict__ wt, const float* __restrict__ bt, const float* __restrict__ wr,
                   const float* __restrict__ br, float* __restrict__ rot, float* __restrict__ trans) {
    __shared__ float f[512], g[512];
    const int bn = blockIdx.x, o = threadIdx.x;
    const float* fr = feat + (size_t)bn * hw * 512;
    float s = 0.f;
    for (int p = skip; p < hw; ++p) s += fr[(size_t)p * 512 + o];
    f[o] = s / (float)(hw - skip);
    __syncthreads();
    float acc = b0[o];
    for (int k = 0; k < 512; ++k) acc += f[k] * w0t[(size_t)k * 512 + o];
    g[o] = fmaxf(acc, 0.f);
    __syncthreads();
    acc = b2[o];
    for (int k = 0; k < 512; ++k) acc += g[k] * w2t[(size_t)k * 512 + o];
    __syncthreads();
    f[o] = fmaxf(acc, 0.f);
    __syncthreads();
    if (o < 12) {
        const bool is_t = o < 3;
        const int q = is_t ? o : o - 3;
        const float* w = (is_t ? wt : wr) + (size_t)q * 512;
        float a = is_t ? bt[q] : br[q];
        for (int k = 0; k < 512; ++k) a += f[k] * w[k];
        if (is_t) trans[(size_t)bn * 3 + q] = a;
        else rot[(size_t)bn * 9 + q] = a;
    }
}

__global__ void svd_pose_kernel(int BN, const float* __restrict__ rot, const float* __restrict__ trans,
                                float* __restrict__ pose) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= BN) return;
    double m[9], R[9];
    for (int e = 0; e < 9; ++e) m[e] = rot[(size_t)i * 9 + e];
    adb_pi3_svd_orthogonalize(m, R);
    float* P = pose + (size_t)i * 16;
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) P[r * 4 + c] = (float)R[r * 3 + c];
        P[r * 4 + 3] = trans ? trans[(size_t)i * 3 + r] : 0.f;
    }
    P[12] = 0.f; P[13] = 0.f; P[14] = 0.f; P[15] = 1.f;
}

// out[n, c, y, x] = bilinear (align_corners=False, no antialias) of clamp(img * 0.5 + 0.5, 0, 1), as
// F.interpolate(mode='bilinear') computes it (source index scale * (dst + 0.5) - 0.5, clamped at 0).
__global__ void __launch_bounds__(256)
window_input_kernel(int N, int Hi, int Wi, const float* __restrict__ img, int Ho, int Wo, float* __restrict__ out) {
    const long long total = (long long)N * 3 * Ho * Wo;
    const float sh = (float)Hi / (float)Ho, sw = (float)Wi / (float)Wo;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % Wo);
        const long long r = i / Wo;
        const int y = (int)(r % Ho);
        const long long nc = r / Ho;
        float hr = sh * (y + 0.5f) - 0.5f, wr = sw * (x + 0.5f) - 0.5f;
        hr = hr < 0.f ? 0.f : hr;
        wr = wr < 0.f ? 0.f : wr;
        const int h1 = (int)hr, w1 = (int)wr;
        const int h1p = h1 < Hi - 1 ? 1 : 0, w1p = w1 < Wi - 1 ? 1 : 0;
        const float h1l = hr - h1, h0l = 1.f - h1l, w1l = wr - w1, w0l = 1.f - w1l;
        const float* src = img + (size_t)nc * Hi * Wi;
        auto px = [&](int yy, int xx) { return fminf(fmaxf(src[(size_t)yy * Wi + xx] * 0.5f + 0.5f, 0.f), 1.f); };
        out[i] = h0l * (w0l * px(h1, w1) + w1l * px(h1, w1 + w1p)) + h1l * (w0l * px(h1 + h1p, w1) + w1l * px(h1 + h1p, w1 + w1p));
    }
}

inline int grid_for(long long n, int per_block = 256) {
    long long b = (n + per_block - 1) / per_block;
    return (int)(b > 132LL * 16 ? 132LL * 16 : (b < 1 ? 1 : b));
}

inline bool al16(const void* p) { return ((uintptr_t)p % 16) == 0; }

}  // namespace

ADB_API int adb_pi3_patch14(int BN, int H, int W, const float* img, void* hi, void* lo, cudaStream_t stream) {
    ADB_REQUIRE(BN >= 1, "adb_pi3_patch14: need at least one frame");
    ADB_REQUIRE(H >= P14 && W >= P14 && H % P14 == 0 && W % P14 == 0, "adb_pi3_patch14: H, W must be multiples of 14");
    ADB_REQUIRE(img && hi, "adb_pi3_patch14: null pointer");
    ADB_REQUIRE(al16(hi) && al16(lo), "adb_pi3_patch14: outputs must be 16-byte aligned");
    const long long total = (long long)BN * (H / P14) * (W / P14) * K14_PAD;
    patch14_kernel<<<grid_for(total), 256, 0, stream>>>(BN, H, W, img, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo);
    ADB_CHECK_LAUNCH("pi3_patch14_kernel");
    return ADB_OK;
}

ADB_API int adb_pi3_tokens(int BN, int n, int C, const float* patch, const float* cls, const float* reg, const float* pos,
                           float* x, cudaStream_t stream) {
    ADB_REQUIRE(BN >= 1 && n >= 1 && C >= 4 && C % 4 == 0, "adb_pi3_tokens: bad sizes");
    ADB_REQUIRE(patch && cls && reg && pos && x, "adb_pi3_tokens: null pointer");
    ADB_REQUIRE(al16(patch) && al16(cls) && al16(reg) && al16(pos) && al16(x), "adb_pi3_tokens: pointers must be 16-byte aligned");
    tokens_kernel<<<grid_for((long long)BN * (n + 5) * (C / 4)), 256, 0, stream>>>(BN, n, C, patch, cls, reg, pos, x);
    ADB_CHECK_LAUNCH("pi3_tokens_kernel");
    return ADB_OK;
}

ADB_API int adb_qknorm_rope(int B, int N, int h, long long ld, int col0, const float* x, const float* gamma,
                            const float* beta, float eps, const long long* pos, const float* table, int n_pos, void* hi,
                            void* lo, cudaStream_t stream) {
    ADB_REQUIRE(B >= 1 && N >= 1 && h >= 1 && n_pos >= 1 && col0 >= 0 && ld >= (long long)col0 + h * 64,
                "adb_qknorm_rope: bad sizes");
    ADB_REQUIRE(x && pos && table && hi, "adb_qknorm_rope: null pointer");
    ADB_REQUIRE((gamma == nullptr) == (beta == nullptr), "adb_qknorm_rope: give gamma and beta together");
    ADB_REQUIRE(al16(x) && al16(hi) && al16(lo) && ((uintptr_t)pos % 8) == 0 && ((uintptr_t)table % 8) == 0,
                "adb_qknorm_rope: misaligned pointer");
    const long long threads = (long long)B * N * h * 32;
    qknorm_rope_kernel<<<(int)((threads + 255) / 256), 256, 0, stream>>>(B, N, h, ld, col0, x, gamma, beta, eps, pos,
                                                                         (const float2*)table, n_pos,
                                                                         (__nv_bfloat16*)hi, (__nv_bfloat16*)lo);
    ADB_CHECK_LAUNCH("qknorm_rope_kernel");
    return ADB_OK;
}

ADB_API int adb_pi3_point_head(int BN, int H, int W, int hw, int skip, const float* pts, const float* cf,
                               const float* pose, float* points, float* local_points, float* conf, cudaStream_t stream) {
    ADB_REQUIRE(BN >= 1, "adb_pi3_point_head: need at least one frame");
    ADB_REQUIRE(H >= P14 && W >= P14 && H % P14 == 0 && W % P14 == 0, "adb_pi3_point_head: H, W must be multiples of 14");
    ADB_REQUIRE(skip >= 0 && hw == skip + (H / P14) * (W / P14), "adb_pi3_point_head: hw must be skip + patch count");
    ADB_REQUIRE(pts && cf && pose && points && local_points && conf, "adb_pi3_point_head: null pointer");
    ADB_REQUIRE((((uintptr_t)pts | (uintptr_t)cf | (uintptr_t)pose | (uintptr_t)points | (uintptr_t)local_points |
                  (uintptr_t)conf) % 4) == 0, "adb_pi3_point_head: misaligned pointer");
    point_head_kernel<<<grid_for((long long)BN * H * W), 256, 0, stream>>>(BN, H, W, hw, skip, pts, cf, pose, points,
                                                                           local_points, conf);
    ADB_CHECK_LAUNCH("pi3_point_head_kernel");
    return ADB_OK;
}

ADB_API int adb_pi3_camera_tail(int BN, int hw, int skip, const float* feat, const float* w0t, const float* b0,
                                const float* w2t, const float* b2, const float* wt, const float* bt, const float* wr,
                                const float* br, float* rot, float* trans, cudaStream_t stream) {
    ADB_REQUIRE(BN >= 1 && skip >= 0 && hw > skip, "adb_pi3_camera_tail: bad sizes");
    ADB_REQUIRE(feat && w0t && b0 && w2t && b2 && wt && bt && wr && br && rot && trans, "adb_pi3_camera_tail: null pointer");
    ADB_REQUIRE((((uintptr_t)feat | (uintptr_t)w0t | (uintptr_t)w2t | (uintptr_t)wt | (uintptr_t)wr | (uintptr_t)rot |
                  (uintptr_t)trans) % 4) == 0, "adb_pi3_camera_tail: misaligned pointer");
    camera_tail_kernel<<<BN, 512, 0, stream>>>(hw, skip, feat, w0t, b0, w2t, b2, wt, bt, wr, br, rot, trans);
    ADB_CHECK_LAUNCH("pi3_camera_tail_kernel");
    return ADB_OK;
}

ADB_API int adb_pi3_svd_pose(int BN, const float* rot, const float* trans, float* pose, cudaStream_t stream) {
    ADB_REQUIRE(BN >= 1, "adb_pi3_svd_pose: need at least one view");
    ADB_REQUIRE(rot && pose, "adb_pi3_svd_pose: null pointer");
    ADB_REQUIRE((((uintptr_t)rot | (uintptr_t)trans | (uintptr_t)pose) % 4) == 0, "adb_pi3_svd_pose: misaligned pointer");
    svd_pose_kernel<<<adb_cdiv(BN, 64), 64, 0, stream>>>(BN, rot, trans, pose);
    ADB_CHECK_LAUNCH("pi3_svd_pose_kernel");
    return ADB_OK;
}

ADB_API int adb_pi3_window_input(int N, int Hi, int Wi, const float* img, int Ho, int Wo, float* out, cudaStream_t stream) {
    ADB_REQUIRE(N >= 1 && Hi >= 1 && Wi >= 1, "adb_pi3_window_input: bad input size");
    ADB_REQUIRE(Ho >= P14 && Wo >= P14 && Ho % P14 == 0 && Wo % P14 == 0, "adb_pi3_window_input: H, W must be multiples of 14");
    ADB_REQUIRE(img && out, "adb_pi3_window_input: null pointer");
    ADB_REQUIRE((((uintptr_t)img | (uintptr_t)out) % 4) == 0, "adb_pi3_window_input: misaligned pointer");
    window_input_kernel<<<grid_for((long long)N * 3 * Ho * Wo), 256, 0, stream>>>(N, Hi, Wi, img, Ho, Wo, out);
    ADB_CHECK_LAUNCH("pi3_window_input_kernel");
    return ADB_OK;
}

// Memory-bound companions of the tensor-core GEMM on the MASt3R path.  Every kernel that feeds a GEMM writes the
// bf16 (hi, lo) split of its fp32 result directly (hi = rn(x), lo = rn(x - hi)), so no activation makes an extra
// fp32 round trip through HBM just to be converted.
//   layernorm      nn.LayerNorm(eps=1e-6)                 croco/models/croco.py:34, blocks.py:127-130,186-191
//   rope_heads     RoPE2D (base 100) + head split/transpose   croco/models/pos_embed.py:112-159, curope/kernels.cu:18-82
//   softmax        attn.softmax(dim=-1)                   blocks.py:106,163
//   im2col_patch   PatchEmbedDust3R's 16x16/s16 conv as a GEMM operand   dust3r/patch_embed.py:19-29
//   split          fp32 -> bf16 (hi, lo)
#include "common.cuh"
#include <cuda_bf16.h>

namespace {

__device__ __forceinline__ void split_store(__nv_bfloat16* hi, __nv_bfloat16* lo, size_t i, float v) {
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    hi[i] = h;
    if (lo) lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
}

// one warp per row; lane owns 8 consecutive channels per 256-channel chunk (two LDG.128 in, one 128-bit bf16 store out)
template <int CHUNKS>
__global__ void __launch_bounds__(256)
layernorm_kernel(long long rows, int C, const float* __restrict__ x, const float* __restrict__ gamma,
                 const float* __restrict__ beta, float eps, float* __restrict__ y, __nv_bfloat16* __restrict__ yhi,
                 __nv_bfloat16* __restrict__ ylo) {
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float* xr = x + (size_t)row * C;
    float v[CHUNKS][8];
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < CHUNKS; ++k) {
        const int c = k * 256 + lane * 8;
        if (c < C) {
            const float4 a = *reinterpret_cast<const float4*>(xr + c), b = *reinterpret_cast<const float4*>(xr + c + 4);
            v[k][0] = a.x; v[k][1] = a.y; v[k][2] = a.z; v[k][3] = a.w; v[k][4] = b.x; v[k][5] = b.y; v[k][6] = b.z; v[k][7] = b.w;
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e) v[k][e] = 0.f;
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) sum += v[k][e];
    }
    sum = adb_warp_sum(sum);
    const float mean = sum / (float)C;
    float var = 0.f;
#pragma unroll
    for (int k = 0; k < CHUNKS; ++k) {
        if (k * 256 + lane * 8 < C) {
#pragma unroll
            for (int e = 0; e < 8; ++e) { const float d = v[k][e] - mean; var += d * d; }
        }
    }
    var = adb_warp_sum(var) / (float)C;
    const float rstd = 1.0f / sqrtf(var + eps);
#pragma unroll
    for (int k = 0; k < CHUNKS; ++k) {
        const int c = k * 256 + lane * 8;
        if (c < C) {
            const float4 g0 = *reinterpret_cast<const float4*>(gamma + c), g1 = *reinterpret_cast<const float4*>(gamma + c + 4);
            const float4 b0 = *reinterpret_cast<const float4*>(beta + c), b1 = *reinterpret_cast<const float4*>(beta + c + 4);
            const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
            const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
            float o[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) o[e] = (v[k][e] - mean) * rstd * gg[e] + bb[e];
            const size_t i = (size_t)row * C + c;
            if (y) {
                *reinterpret_cast<float4*>(y + i) = make_float4(o[0], o[1], o[2], o[3]);
                *reinterpret_cast<float4*>(y + i + 4) = make_float4(o[4], o[5], o[6], o[7]);
            }
            if (yhi) {
                uint32_t hw[4], lw[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const __nv_bfloat16 ah = __float2bfloat16_rn(o[2 * e]), bh = __float2bfloat16_rn(o[2 * e + 1]);
                    const __nv_bfloat16 al = __float2bfloat16_rn(o[2 * e] - __bfloat162float(ah));
                    const __nv_bfloat16 bl = __float2bfloat16_rn(o[2 * e + 1] - __bfloat162float(bh));
                    hw[e] = (uint32_t)__bfloat16_as_ushort(ah) | ((uint32_t)__bfloat16_as_ushort(bh) << 16);
                    lw[e] = (uint32_t)__bfloat16_as_ushort(al) | ((uint32_t)__bfloat16_as_ushort(bl) << 16);
                }
                *reinterpret_cast<uint4*>(yhi + i) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
                if (ylo) *reinterpret_cast<uint4*>(ylo + i) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
            }
        }
    }
}

__global__ void __launch_bounds__(256)
split_kernel(long long n, const float* __restrict__ x, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        split_store(hi, lo, (size_t)i, x[i]);
}

// x: fp32 [B, N, ld] (this head group starts at column col0), pos: int64 [B, N, 2] (y, x),
// table: float2 [n_pos][16] = (cos, sin)(p * base^(-j/16)) computed by the caller exactly as the reference does
// (pos_embed.py:118-127).  mode 0: RoPE, mode 1: plain; out [B, h, N, 64].  One thread per 8 consecutive dims.
__global__ void __launch_bounds__(256)
rope_heads_kernel(int B, int N, int h, long long ld, int col0, const float* __restrict__ x,
                  const long long* __restrict__ pos, const float2* __restrict__ table, int n_pos, int mode,
                  __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
    const long long total = (long long)B * N * h * 8;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int d0 = (int)(i & 7) * 8;
        const int hh = (int)((i >> 3) % h);
        const long long bn = (i >> 3) / h;
        const int n = (int)(bn % N);
        const int b = (int)(bn / N);
        const float* xr = x + (size_t)bn * ld + col0 + hh * 64;
        float v[8];
        {
            const float4 a = *reinterpret_cast<const float4*>(xr + d0), c = *reinterpret_cast<const float4*>(xr + d0 + 4);
            v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = c.x; v[5] = c.y; v[6] = c.z; v[7] = c.w;
        }
        if (mode == 0) {
            const int half = d0 >> 5, j0 = d0 & 31, jj0 = j0 & 15;
            const bool first = j0 < 16;
            const float* xp = xr + (half << 5) + (first ? j0 + 16 : j0 - 16);
            const float4 a = *reinterpret_cast<const float4*>(xp), c = *reinterpret_cast<const float4*>(xp + 4);
            const float o[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
            long long pz = pos[(size_t)bn * 2 + half];
            pz = pz < 0 ? 0 : (pz >= n_pos ? n_pos - 1 : pz);
            const float2* tb = table + (size_t)pz * 16 + jj0;
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float2 cs = __ldg(tb + e);
                v[e] = first ? v[e] * cs.x - o[e] * cs.y : v[e] * cs.x + o[e] * cs.y;
            }
        }
        uint32_t hw[4], lw[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const __nv_bfloat16 ah = __float2bfloat16_rn(v[2 * e]), bh = __float2bfloat16_rn(v[2 * e + 1]);
            const __nv_bfloat16 al = __float2bfloat16_rn(v[2 * e] - __bfloat162float(ah));
            const __nv_bfloat16 bl = __float2bfloat16_rn(v[2 * e + 1] - __bfloat162float(bh));
            hw[e] = (uint32_t)__bfloat16_as_ushort(ah) | ((uint32_t)__bfloat16_as_ushort(bh) << 16);
            lw[e] = (uint32_t)__bfloat16_as_ushort(al) | ((uint32_t)__bfloat16_as_ushort(bl) << 16);
        }
        const size_t o8 = (((size_t)b * h + hh) * N + n) * 64 + d0;
        *reinterpret_cast<uint4*>(hi + o8) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
        if (lo) *reinterpret_cast<uint4*>(lo + o8) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
    }
}

// mode 2: plain values, transposed output [B, h, 64, Npad] through a shared-memory tile (coalesced on both sides).
// grid = (ceil(N/64), h, B), block = 256.
__global__ void __launch_bounds__(256)
heads_transpose_kernel(int N, int h, long long ld, int col0, const float* __restrict__ x, int Npad,
                       __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
    __shared__ float tile[64][65];
    const int n0 = blockIdx.x * 64, hh = blockIdx.y, b = blockIdx.z;
    const int t = threadIdx.x;
    {
        const int tok = t >> 2, dq = (t & 3) * 16;
        const int n = n0 + tok;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
            if (n < N) q = *reinterpret_cast<const float4*>(x + ((size_t)b * N + n) * ld + col0 + hh * 64 + dq + 4 * e);
            tile[dq + 4 * e][tok] = q.x; tile[dq + 4 * e + 1][tok] = q.y; tile[dq + 4 * e + 2][tok] = q.z; tile[dq + 4 * e + 3][tok] = q.w;
        }
    }
    __syncthreads();
    const int d = t >> 2, tq = (t & 3) * 16;
#pragma unroll
    for (int g = 0; g < 2; ++g) {
        const int n = n0 + tq + 8 * g;
        if (n >= Npad) continue;          // Npad is a multiple of 8, so an 8-token group never straddles it
        uint32_t hw[4], lw[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float f0 = tile[d][tq + 8 * g + 2 * e], f1 = tile[d][tq + 8 * g + 2 * e + 1];
            const __nv_bfloat16 ah = __float2bfloat16_rn(f0), bh = __float2bfloat16_rn(f1);
            const __nv_bfloat16 al = __float2bfloat16_rn(f0 - __bfloat162float(ah));
            const __nv_bfloat16 bl = __float2bfloat16_rn(f1 - __bfloat162float(bh));
            hw[e] = (uint32_t)__bfloat16_as_ushort(ah) | ((uint32_t)__bfloat16_as_ushort(bh) << 16);
            lw[e] = (uint32_t)__bfloat16_as_ushort(al) | ((uint32_t)__bfloat16_as_ushort(bl) << 16);
        }
        const size_t o = (((size_t)b * h + hh) * 64 + d) * Npad + n;
        *reinterpret_cast<uint4*>(hi + o) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
        if (lo) *reinterpret_cast<uint4*>(lo + o) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
    }
}

// one warp per row of length L (row stride ld_in for the fp32 input, ld_out for the bf16 outputs).  The row is read
// ONCE into registers (4 values per lane per 128-column chunk, LDG.128) when L <= 128*CH and L % 4 == 0.
template <int CH>
__global__ void __launch_bounds__(256)
softmax_reg_kernel(long long rows, int L, long long ld_in, long long ld_out, const float* __restrict__ s,
                   __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float* sr = s + (size_t)row * ld_in;
    float v[CH][4];
    float m = -INFINITY;          // not a finite floor: a row of finfo.min logits would underflow every term to 0
#pragma unroll
    for (int k = 0; k < CH; ++k) {
        const int c = k * 128 + lane * 4;
        if (c < L) {
            const float4 a = *reinterpret_cast<const float4*>(sr + c);
            v[k][0] = a.x; v[k][1] = a.y; v[k][2] = a.z; v[k][3] = a.w;
            m = fmaxf(m, fmaxf(fmaxf(a.x, a.y), fmaxf(a.z, a.w)));
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < CH; ++k)
        if (k * 128 + lane * 4 < L) {
#pragma unroll
            for (int e = 0; e < 4; ++e) { v[k][e] = expf(v[k][e] - m); sum += v[k][e]; }
        }
    sum = adb_warp_sum(sum);
    const float inv = 1.0f / sum;
#pragma unroll
    for (int k = 0; k < CH; ++k) {
        const int c = k * 128 + lane * 4;
        if (c < L) {
            uint32_t hw[2], lw[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const float a = v[k][2 * e] * inv, b = v[k][2 * e + 1] * inv;
                const __nv_bfloat16 ah = __float2bfloat16_rn(a), bh = __float2bfloat16_rn(b);
                const __nv_bfloat16 al = __float2bfloat16_rn(a - __bfloat162float(ah));
                const __nv_bfloat16 bl = __float2bfloat16_rn(b - __bfloat162float(bh));
                hw[e] = (uint32_t)__bfloat16_as_ushort(ah) | ((uint32_t)__bfloat16_as_ushort(bh) << 16);
                lw[e] = (uint32_t)__bfloat16_as_ushort(al) | ((uint32_t)__bfloat16_as_ushort(bl) << 16);
            }
            const size_t o = (size_t)row * ld_out + c;
            *reinterpret_cast<uint2*>(hi + o) = make_uint2(hw[0], hw[1]);
            if (lo) *reinterpret_cast<uint2*>(lo + o) = make_uint2(lw[0], lw[1]);
        }
    }
}

// generic fallback (any L / alignment): three passes over the row
__global__ void __launch_bounds__(256)
softmax_kernel(long long rows, int L, long long ld_in, long long ld_out, const float* __restrict__ s,
               __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float* sr = s + (size_t)row * ld_in;
    float m = -INFINITY;
    for (int c = lane; c < L; c += 32) m = fmaxf(m, sr[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float sum = 0.f;
    for (int c = lane; c < L; c += 32) sum += expf(sr[c] - m);
    sum = adb_warp_sum(sum);
    const float inv = 1.0f / sum;
    for (int c = lane; c < L; c += 32) split_store(hi, lo, (size_t)row * ld_out + c, expf(sr[c] - m) * inv);
}

// img fp32 [B, 3, H, W] -> A [B * (H/16) * (W/16), 768] with column = c*256 + py*16 + px (the conv weight's flattening)
__global__ void __launch_bounds__(256)
im2col_patch_kernel(int B, int H, int W, const float* __restrict__ img, __nv_bfloat16* __restrict__ hi,
                    __nv_bfloat16* __restrict__ lo) {
    const int gw = W / 16, gh = H / 16;
    const long long total = (long long)B * gh * gw * 768;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int col = (int)(i % 768);
        const long long patch = i / 768;
        const int pxx = (int)(patch % gw), pyy = (int)((patch / gw) % gh), b = (int)(patch / ((long long)gw * gh));
        const int c = col >> 8, py = (col >> 4) & 15, px = col & 15;
        const float v = img[(((size_t)b * 3 + c) * H + (pyy * 16 + py)) * W + pxx * 16 + px];
        split_store(hi, lo, (size_t)i, v);
    }
}

inline int grid_for(long long n) { long long g = (n + 255) / 256; return (int)(g < 132LL * 32 ? g : 132LL * 32); }

// NULL passes: optional outputs are checked only when given
inline bool aligned(const void* p, unsigned bytes) { return ((uintptr_t)p % bytes) == 0; }

}  // namespace

// ---- DPT head companions (round 2): the last eager PyTorch ops of the head ------------------------------------------
// Bilinear x2 upsampling, align_corners=True (croco/models/dpt_block.py:215-216,320: F.interpolate(scale_factor=2,
// mode="bilinear", align_corners=True)), NHWC fp32 in.  Same arithmetic as torch's upsample_bilinear2d: src = dst*(in-1)/(out-1),
// out = (1-ly)[(1-lx) v00 + lx v01] + ly[(1-lx) v10 + lx v11].  Fused with what follows it in the head: an optional addend
// (the skip connection "x0 + RCU1(x1)" of FeatureFusionBlock is out = up(x) + addend), an optional crop (dpt_head.py:57) and
// the bf16 (hi, lo) split the next implicit-GEMM conv consumes.  One thread per (output pixel, 4 channels).
__global__ void __launch_bounds__(256)
upsample2x_kernel(int B, int Hin, int Win, int C, int Hout, int Wout, const float* __restrict__ x,
                  const float* __restrict__ addend, float* __restrict__ y, __nv_bfloat16* __restrict__ hi,
                  __nv_bfloat16* __restrict__ lo) {
    const int C4 = C >> 2;
    const long long total = (long long)B * Hout * Wout * C4;
    const float sh = (float)(Hin - 1) / (float)(2 * Hin - 1), sw = (float)(Win - 1) / (float)(2 * Win - 1);
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int c4 = (int)(t % C4);
        long long r = t / C4;
        const int ox = (int)(r % Wout);
        r /= Wout;
        const int oy = (int)(r % Hout), b = (int)(r / Hout);
        const float fy = sh * (float)oy, fx = sw * (float)ox;
        const int y0 = (int)fy, x0 = (int)fx;
        const int y1 = y0 + (y0 < Hin - 1 ? 1 : 0), x1 = x0 + (x0 < Win - 1 ? 1 : 0);
        const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.0f - ly, hx = 1.0f - lx;
        const float4* base = reinterpret_cast<const float4*>(x) + (size_t)b * Hin * Win * C4 + c4;
        const float4 v00 = base[((size_t)y0 * Win + x0) * C4], v01 = base[((size_t)y0 * Win + x1) * C4];
        const float4 v10 = base[((size_t)y1 * Win + x0) * C4], v11 = base[((size_t)y1 * Win + x1) * C4];
        float4 o;
        o.x = hy * (hx * v00.x + lx * v01.x) + ly * (hx * v10.x + lx * v11.x);
        o.y = hy * (hx * v00.y + lx * v01.y) + ly * (hx * v10.y + lx * v11.y);
        o.z = hy * (hx * v00.z + lx * v01.z) + ly * (hx * v10.z + lx * v11.z);
        o.w = hy * (hx * v00.w + lx * v01.w) + ly * (hx * v10.w + lx * v11.w);
        const size_t oi = (size_t)t;            // float4 index into [B, Hout, Wout, C4]
        if (addend) {
            const float4 a = reinterpret_cast<const float4*>(addend)[oi];
            o.x += a.x; o.y += a.y; o.z += a.z; o.w += a.w;
        }
        if (y) reinterpret_cast<float4*>(y)[oi] = o;
        if (hi) {
            const float v[4] = {o.x, o.y, o.z, o.w};
            __nv_bfloat16 h4[4], l4[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                h4[k] = __float2bfloat16_rn(v[k]);
                l4[k] = __float2bfloat16_rn(v[k] - __bfloat162float(h4[k]));
            }
            reinterpret_cast<uint2*>(hi)[oi] = *reinterpret_cast<uint2*>(h4);
            if (lo) reinterpret_cast<uint2*>(lo)[oi] = *reinterpret_cast<uint2*>(l4);
        }
    }
}

// Head epilogue (mast3r/catmlp_dpt_head.py:25-39,87-96 + dust3r/heads/postprocess.py:22-58) in one pass: reads the 4-channel
// DPT map (NHWC) and the local-feature MLP output [B*S, 25*256] in its PRE-pixel-shuffle layout (channel c of pixel (Y,X) is
// column c*256 + (Y%16)*16 + X%16 of token (Y/16)*(W/16) + X/16), and writes the post-processed dict directly:
//   pts3d = xyz / max(|xyz|, 1e-8) * expm1(|xyz|)   conf = 1 + exp(c)   desc = d / |d|   desc_conf = exp(q).
// Replaces pixel_shuffle + cat + 8 elementwise/reduction torch kernels and the [B,29,H,W] intermediate.
template <int ND>
__global__ void __launch_bounds__(256)
head_postprocess_kernel(int B, int H, int W, const float* __restrict__ pts, const float* __restrict__ lf, long long ld_lf,
                        float* __restrict__ pts3d, float* __restrict__ conf, float* __restrict__ desc,
                        float* __restrict__ desc_conf) {
    const long long total = (long long)B * H * W;
    const int tw = W >> 4, S = (H >> 4) * tw;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int X = (int)(t % W);
        const long long r = t / W;
        const int Y = (int)(r % H), b = (int)(r / H);
        const float4 p = reinterpret_cast<const float4*>(pts)[t];
        const float d = sqrtf(p.x * p.x + p.y * p.y + p.z * p.z);
        const float sc = expm1f(d) / fmaxf(d, 1e-8f);
        pts3d[3 * t] = p.x * sc; pts3d[3 * t + 1] = p.y * sc; pts3d[3 * t + 2] = p.z * sc;
        conf[t] = 1.0f + expf(p.w);
        const float* row = lf + ((size_t)b * S + (size_t)(Y >> 4) * tw + (X >> 4)) * ld_lf + (Y & 15) * 16 + (X & 15);
        float dv[ND];
        float nrm = 0.f;
#pragma unroll
        for (int c = 0; c < ND; ++c) {
            dv[c] = row[(size_t)c * 256];
            nrm += dv[c] * dv[c];
        }
        const float inv = 1.0f / sqrtf(nrm);
        float4* dp = reinterpret_cast<float4*>(desc + (size_t)t * ND);
#pragma unroll
        for (int c = 0; c < ND; c += 4) dp[c >> 2] = make_float4(dv[c] * inv, dv[c + 1] * inv, dv[c + 2] * inv, dv[c + 3] * inv);
        desc_conf[t] = expf(row[(size_t)ND * 256]);
    }
}

ADB_API int adb_layernorm(long long rows, int C, const float* x, const float* gamma, const float* beta, float eps,
                          float* y, void* y_hi, void* y_lo, cudaStream_t stream) {
    ADB_REQUIRE(rows >= 0 && C >= 8 && C <= 2048 && C % 8 == 0, "adb_layernorm: C must be a multiple of 8 in [8, 2048]");
    if (rows == 0) return ADB_OK;
    ADB_REQUIRE(x && gamma && beta && (y || y_hi), "adb_layernorm: null pointer");
    ADB_REQUIRE(aligned(x, 16) && aligned(gamma, 16) && aligned(beta, 16) && aligned(y, 16) && aligned(y_hi, 16) &&
                    aligned(y_lo, 16), "adb_layernorm: x, gamma, beta, y, y_hi and y_lo must be 16-byte aligned");
    const int blocks = (int)((rows + 7) / 8);
    if (C <= 1024)
        layernorm_kernel<4><<<blocks, 256, 0, stream>>>(rows, C, x, gamma, beta, eps, y, (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo);
    else
        layernorm_kernel<8><<<blocks, 256, 0, stream>>>(rows, C, x, gamma, beta, eps, y, (__nv_bfloat16*)y_hi, (__nv_bfloat16*)y_lo);
    ADB_CHECK_LAUNCH("layernorm_kernel");
    return ADB_OK;
}

ADB_API int adb_split_bf16(long long n, const float* x, void* hi, void* lo, cudaStream_t stream) {
    ADB_REQUIRE(n >= 0, "adb_split_bf16: bad n");
    if (n == 0) return ADB_OK;
    ADB_REQUIRE(x && hi, "adb_split_bf16: null pointer");
    split_kernel<<<grid_for(n), 256, 0, stream>>>(n, x, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo);
    ADB_CHECK_LAUNCH("split_kernel");
    return ADB_OK;
}

ADB_API int adb_rope_heads(int B, int N, int h, long long ld, int col0, const float* x, const long long* pos,
                           const float* table, int n_pos, int mode, int Npad, void* hi, void* lo, cudaStream_t stream) {
    ADB_REQUIRE(B >= 0 && N >= 0 && h >= 1 && mode >= 0 && mode <= 2, "adb_rope_heads: bad args");
    if ((long long)B * N == 0) return ADB_OK;
    ADB_REQUIRE(x && hi && (mode != 0 || (pos && table && n_pos > 0)), "adb_rope_heads: null pointer");
    ADB_REQUIRE(col0 >= 0 && ld >= (long long)col0 + h * 64, "adb_rope_heads: need ld >= col0 + h*64");
    ADB_REQUIRE(ld % 4 == 0 && col0 % 4 == 0 && ((uintptr_t)x % 16 == 0), "adb_rope_heads: x must allow 128-bit loads");
    ADB_REQUIRE(aligned(hi, 16) && aligned(lo, 16) && aligned(pos, 8) && aligned(table, 8),
                "adb_rope_heads: hi and lo must be 16-byte aligned, pos and table 8-byte aligned");
    if (mode == 2) {
        ADB_REQUIRE(Npad >= N && Npad % 8 == 0, "adb_rope_heads: Npad must be a multiple of 8 and >= N");
        dim3 grid(adb_cdiv(Npad, 64), h, B);
        heads_transpose_kernel<<<grid, 256, 0, stream>>>(N, h, ld, col0, x, Npad, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo);
        ADB_CHECK_LAUNCH("heads_transpose_kernel");
        return ADB_OK;
    }
    rope_heads_kernel<<<grid_for((long long)B * N * h * 8), 256, 0, stream>>>(B, N, h, ld, col0, x, pos,
                                                                             (const float2*)table, n_pos, mode,
                                                                             (__nv_bfloat16*)hi, (__nv_bfloat16*)lo);
    ADB_CHECK_LAUNCH("rope_heads_kernel");
    return ADB_OK;
}

ADB_API int adb_softmax_rows(long long rows, int L, long long ld_in, long long ld_out, const float* s, void* hi, void* lo,
                             cudaStream_t stream) {
    ADB_REQUIRE(rows >= 0 && L >= 1, "adb_softmax_rows: bad sizes");
    if (rows == 0) return ADB_OK;
    ADB_REQUIRE(s && hi, "adb_softmax_rows: null pointer");
    const bool fast = (L % 4 == 0) && (ld_in % 4 == 0) && (ld_out % 4 == 0) && ((uintptr_t)s % 16 == 0) &&
                      ((uintptr_t)hi % 8 == 0) && ((uintptr_t)lo % 8 == 0) && L <= 2048;
    const int blocks = (int)((rows + 7) / 8);
    if (fast && L <= 1024)
        softmax_reg_kernel<8><<<blocks, 256, 0, stream>>>(rows, L, ld_in, ld_out, s, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo);
    else if (fast)
        softmax_reg_kernel<16><<<blocks, 256, 0, stream>>>(rows, L, ld_in, ld_out, s, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo);
    else
        softmax_kernel<<<blocks, 256, 0, stream>>>(rows, L, ld_in, ld_out, s, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo);
    ADB_CHECK_LAUNCH("softmax_kernel");
    return ADB_OK;
}

ADB_API int adb_im2col_patch16(int B, int H, int W, const float* img, void* hi, void* lo, cudaStream_t stream) {
    ADB_REQUIRE(B >= 0 && H > 0 && W > 0 && H % 16 == 0 && W % 16 == 0, "adb_im2col_patch16: H, W must be multiples of 16");
    if (B == 0) return ADB_OK;
    ADB_REQUIRE(img && hi, "adb_im2col_patch16: null pointer");
    im2col_patch_kernel<<<grid_for((long long)B * (H / 16) * (W / 16) * 768), 256, 0, stream>>>(B, H, W, img, (__nv_bfloat16*)hi,
                                                                                               (__nv_bfloat16*)lo);
    ADB_CHECK_LAUNCH("im2col_patch_kernel");
    return ADB_OK;
}

// ---- curope.rope_2d: in-place RoPE2D on tokens [B,N,H,D] (VSLAM/thirdparty/mast3r/dust3r/croco/models/curope/
// kernels.cu:18-108, curope.cpp:49-68).  One head = [u_Y (Q) | v_Y (Q) | u_X (Q) | v_X (Q)], Q = D/4;
// inv_freq_i = F0 / base^(i/Q); (u,v) <- (u c - v s, v c + u s) with the angle pos_{y|x} * inv_freq_i.
// One CTA per token: the D/2 (cos,sin) pairs are computed once (precise powf/sincosf; the reference build uses
// --use_fast_math intrinsics, its PyTorch fallback pos_embed.py:112-159 is exact) and reused by all H heads.
namespace {
__global__ void __launch_bounds__(256)
rope2d_inplace_kernel(float* __restrict__ tok, const long long* __restrict__ pos, int N, int H, int D,
                      long long sb, long long sn, float base, float F0) {
    const int b = blockIdx.x / N, n = blockIdx.x % N;
    const int half = D / 2, Q = D / 4;
    const int p = threadIdx.x % half;          // pair index: [0,Q) -> Y, [Q,2Q) -> X
    const int hl = threadIdx.x / half, hstep = blockDim.x / half;
    const int X = p >= Q, i = p - X * Q;
    const float ang = (float)pos[((long long)b * N + n) * 2 + X] * (F0 / powf(base, (float)i / (float)Q));
    float s, c;
    sincosf(ang, &s, &c);
    float* t = tok + b * sb + n * sn + X * half + i;
    for (int h = hl; h < H; h += hstep) {
        float* q = t + (long long)h * D;
        const float u = q[0], v = q[Q];
        q[0] = u * c - v * s;
        q[Q] = v * c + u * s;
    }
}
}  // namespace

ADB_API int adb_rope2d_inplace(int B, int N, int H, int D, long long stride_b, long long stride_n, float* tokens,
                               const long long* positions, float base, float F0, cudaStream_t stream) {
    ADB_REQUIRE(B >= 0 && N >= 0 && H > 0 && D > 0, "adb_rope2d_inplace: bad sizes");
    ADB_REQUIRE(D % 4 == 0 && D <= 512, "adb_rope2d_inplace: token dim must be a multiple of 4 (and <= 512)");
    if ((long long)B * N == 0) return ADB_OK;
    ADB_REQUIRE(tokens && positions, "adb_rope2d_inplace: null pointer");
    const int half = D / 2;
    int hy = 256 / half;
    if (hy < 1) hy = 1;
    if (hy > H) hy = H;
    rope2d_inplace_kernel<<<(unsigned)((long long)B * N), half * hy, 0, stream>>>(tokens, positions, N, H, D, stride_b,
                                                                                stride_n, base, F0);
    ADB_CHECK_LAUNCH("rope2d_inplace_kernel");
    return ADB_OK;
}

// x [B,Hin,Win,C] fp32 NHWC (C % 4 == 0) -> bilinear x2 (align_corners=True), cropped to [Hout<=2Hin, Wout<=2Win];
// + addend [B,Hout,Wout,C] (may be NULL); y fp32 and/or (hi, lo) bf16 split outputs (each may be NULL).
ADB_API int adb_upsample2x_nhwc(int B, int Hin, int Win, int C, int Hout, int Wout, const float* x, const float* addend,
                                float* y, void* hi, void* lo, cudaStream_t stream) {
    ADB_REQUIRE(B >= 0 && Hin >= 1 && Win >= 1 && C >= 4 && C % 4 == 0 && Hout >= 1 && Hout <= 2 * Hin && Wout >= 1 &&
                    Wout <= 2 * Win, "adb_upsample2x_nhwc: bad sizes");
    if (B == 0) return ADB_OK;
    ADB_REQUIRE(x && (y || hi), "adb_upsample2x_nhwc: null pointer");
    ADB_REQUIRE(!lo || hi, "adb_upsample2x_nhwc: lo without hi");
    ADB_REQUIRE(aligned(x, 16) && aligned(addend, 16) && aligned(y, 16) && aligned(hi, 8) && aligned(lo, 8),
                "adb_upsample2x_nhwc: x, addend and y must be 16-byte aligned, hi and lo 8-byte aligned");
    upsample2x_kernel<<<grid_for((long long)B * Hout * Wout * (C / 4)), 256, 0, stream>>>(
        B, Hin, Win, C, Hout, Wout, x, addend, y, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo);
    ADB_CHECK_LAUNCH("upsample2x_kernel");
    return ADB_OK;
}

// pts [B,H,W,4] fp32, lf [B*(H/16)*(W/16), ld_lf >= (n_desc+1)*256] fp32 -> pts3d [B,H,W,3], conf [B,H,W],
// desc [B,H,W,n_desc], desc_conf [B,H,W].  H, W multiples of 16; n_desc == 24 (the checkpoint ARTDECO loads).
ADB_API int adb_head_postprocess(int B, int H, int W, const float* pts, const float* lf, long long ld_lf, int n_desc,
                                 float* pts3d, float* conf, float* desc, float* desc_conf, cudaStream_t stream) {
    ADB_REQUIRE(B >= 0 && H >= 16 && W >= 16 && H % 16 == 0 && W % 16 == 0 && ld_lf >= (long long)(n_desc + 1) * 256,
                "adb_head_postprocess: bad sizes");
    ADB_REQUIRE(n_desc == 24, "adb_head_postprocess: only the desc24 head (output_mode pts3d+desc24) is built");
    if (B == 0) return ADB_OK;
    ADB_REQUIRE(pts && lf && pts3d && conf && desc && desc_conf, "adb_head_postprocess: null pointer");
    ADB_REQUIRE(aligned(pts, 16) && aligned(desc, 16) && aligned(lf, 4) && aligned(pts3d, 4) && aligned(conf, 4) &&
                    aligned(desc_conf, 4), "adb_head_postprocess: pts and desc must be 16-byte aligned, the rest 4-byte aligned");
    head_postprocess_kernel<24><<<grid_for((long long)B * H * W), 256, 0, stream>>>(B, H, W, pts, lf, ld_lf, pts3d, conf,
                                                                                   desc, desc_conf);
    ADB_CHECK_LAUNCH("head_postprocess_kernel");
    return ADB_OK;
}

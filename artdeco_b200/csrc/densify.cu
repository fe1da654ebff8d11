// Key-frame densification: the sampler of SceneModel.add_new_gaussians (Reconstruct/scene/scene_models/h3dgsv3.py:766-940).
//
// The reference spends ~60 small torch kernels and ~5 host syncs per LoD on this (two bilinear resizes, two Laplacian /
// disc filters, a Bernoulli draw, boolean indexing, two grid_samples, torch.quantile(...).item(), back-projection, the
// initial parameters).  Here one LoD is
//   densify_stencil_kernel   img / render resize, both get_lapla_norm filters, the draw, the depth / conf samples and the
//                            validity test on a shared-memory tile; per-(row, 32-column segment) counts of emitted rows
//   cub InclusiveSum         of the segment counts (row-major segment order = the order of the reference's boolean masks)
//   densify_emit_kernel      xyz, f_dc, scaling, opacity, d_max of every emitted pixel at its row-major rank
// with one host read (the row count) between the scan and the emission, which sizes the outputs.  Per call:
//   depth quantile           torch.quantile(point_map[:, 2], 0.02) by the exact two-level radix selection of select.cuh
//   densify_prune_kernel     the valid_gs_mask of the existing Gaussians
// Arithmetic follows what PyTorch evaluates on CUDA: a division by a Python scalar is a multiplication by the fp32
// reciprocal, and the steps the reference runs as separate kernels are rounded separately here (__fmul_rn / __fadd_rn).
#include "common.cuh"
#include "select.cuh"
#include "artdeco_b200.h"

#include <cub/device/device_scan.cuh>

namespace {

using adb_select::HIST_BINS;
using adb_select::SEL_THREADS;

constexpr int DS_TX = 32, DS_TY = 16, DS_ROWS = 8;      // output tile 32x16, block 32x8 (two rows per thread)
constexpr int DS_HALO = 4;                              // 1 (3x3 Laplacian) + 3 (7x7 disc)
constexpr int IN_W = DS_TX + 2 * DS_HALO, IN_H = DS_TY + 2 * DS_HALO;
constexpr int LP_W = DS_TX + 6, LP_H = DS_TY + 6;
constexpr int DS_THREADS = DS_TX * DS_ROWS;
constexpr int Q_THREADS = 256;
constexpr int MAX_PIXELS = 1 << 28;

struct SampleParams {
    int H, W, lod, h, w, Hs, Ws, nsx;
    float scale_img_y, scale_img_x;   // pooled (H/2, W/2) -> (h, w), align_corners=True
    float scale_r_y, scale_r_x;       // full (H, W) -> (h, w)
    float grid_sx, grid_sy;           // fp32(2 / (w - 1)), fp32(2 / (h - 1)) (make_torch_sampler)
    float scaler, ratio;
    long long r_cs, r_ys, r_xs;       // render strides (elements): channel, row, column
    int has_render;
};

struct EmitParams {
    float cx, cy;                     // centre / lod
    float inv_f;                      // 1 / fp32(f / lod)
    float inv_f_full;                 // fp32(1 / f)
    float wmax;                       // fp32(W / 10)
    float lod_f;
    float inv_c0;                     // 1 / fp32(C0)
};

__device__ __forceinline__ float clampf(float x, float lo, float hi) {        // torch.clamp: NaN propagates
    return x != x ? x : fminf(fmaxf(x, lo), hi);
}

// upsample_bilinear2d (align_corners=True) source index: (index, neighbour offset, lambda)
__device__ __forceinline__ void lin_src(float scale, int dst, int in_size, int* i0, int* ip, float* l1) {
    const float r = scale * (float)dst;
    const int i = (int)r;
    *i0 = i;
    *ip = (i < in_size - 1) ? 1 : 0;
    *l1 = r - (float)i;
}

// avg_pool2d(image, 2) at pooled pixel (py, px) of channel c
__device__ __forceinline__ float pooled(const float* __restrict__ img, int W, size_t plane, int c, int py, int px) {
    const float* p = img + c * plane + (size_t)(2 * py) * W + 2 * px;
    float a = 0.f;
    a = __fadd_rn(a, p[0]);
    a = __fadd_rn(a, p[1]);
    a = __fadd_rn(a, p[W]);
    a = __fadd_rn(a, p[W + 1]);
    return a / 4.0f;
}

__device__ __forceinline__ float blend4(float h0l, float h1l, float w0l, float w1l, float a, float b, float c, float d) {
    return h0l * (w0l * a + w1l * b) + h1l * (w0l * c + w1l * d);
}

// img = interpolate(avg_pool2d(image, 2), (h, w), bilinear, align_corners=True)  at LoD pixel (y, x), 3 channels
__device__ __forceinline__ void lod_image(const SampleParams& p, const float* __restrict__ image, int y, int x, float* out) {
    const int Hp = p.H / 2, Wp = p.W / 2;
    int y0, yp, x0, xp;
    float ly, lx;
    lin_src(p.scale_img_y, y, Hp, &y0, &yp, &ly);
    lin_src(p.scale_img_x, x, Wp, &x0, &xp, &lx);
    const size_t plane = (size_t)p.H * p.W;
#pragma unroll
    for (int c = 0; c < 3; ++c)
        out[c] = blend4(1.f - ly, ly, 1.f - lx, lx, pooled(image, p.W, plane, c, y0, x0), pooled(image, p.W, plane, c, y0, x0 + xp),
                        pooled(image, p.W, plane, c, y0 + yp, x0), pooled(image, p.W, plane, c, y0 + yp, x0 + xp));
}

// clamp(E[:3,:3] @ rgb + E[:3,3], 0, 1) of one full-resolution render pixel (render_from_id, h3dgsv3.py:611-614)
__device__ __forceinline__ void exposed(const SampleParams& p, const float* __restrict__ rnd, const float* E, int y, int x,
                                        float* out) {
    const float* q = rnd + (long long)y * p.r_ys + (long long)x * p.r_xs;
    const float r0 = q[0], r1 = q[p.r_cs], r2 = q[2 * p.r_cs];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float m = fmaf(E[c * 4 + 2], r2, fmaf(E[c * 4 + 1], r1, E[c * 4 + 0] * r0));
        out[c] = clampf(__fadd_rn(m, E[c * 4 + 3]), 0.f, 1.f);
    }
}

// interpolate(exposed render, (h, w), bilinear, align_corners=True) at LoD pixel (y, x)
__device__ __forceinline__ void lod_render(const SampleParams& p, const float* __restrict__ rnd, const float* E, int y, int x,
                                           float* out) {
    int y0, yp, x0, xp;
    float ly, lx;
    lin_src(p.scale_r_y, y, p.H, &y0, &yp, &ly);
    lin_src(p.scale_r_x, x, p.W, &x0, &xp, &lx);
    float a[3], b[3], c[3], d[3];
    exposed(p, rnd, E, y0, x0, a);
    exposed(p, rnd, E, y0, x0 + xp, b);
    exposed(p, rnd, E, y0 + yp, x0, c);
    exposed(p, rnd, E, y0 + yp, x0 + xp, d);
#pragma unroll
    for (int k = 0; k < 3; ++k) out[k] = blend4(1.f - ly, ly, 1.f - lx, lx, a[k], b[k], c[k], d[k]);
}

// sample(map, uv, w, h) = grid_sample(map, uv * (2 / (size - 1)) - 1, bilinear, zeros, align_corners=True)
__device__ __forceinline__ float grid_sample(const float* __restrict__ map, int Hs, int Ws, float gx, float gy) {
    const float ix = __fmul_rn(__fadd_rn(gx, 1.f) / 2, (float)(Ws - 1));
    const float iy = __fmul_rn(__fadd_rn(gy, 1.f) / 2, (float)(Hs - 1));
    const float fx = floorf(ix), fy = floorf(iy);
    const int x0 = (int)fx, y0 = (int)fy;
    const float nw = (fx + 1.f - ix) * (fy + 1.f - iy), ne = (ix - fx) * (fy + 1.f - iy);
    const float sw = (fx + 1.f - ix) * (iy - fy), se = (ix - fx) * (iy - fy);
    auto in = [&](int yy, int xx) { return yy >= 0 && yy < Hs && xx >= 0 && xx < Ws; };
    float out = 0.f;
    if (in(y0, x0)) out += map[(size_t)y0 * Ws + x0] * nw;
    if (in(y0, x0 + 1)) out += map[(size_t)y0 * Ws + x0 + 1] * ne;
    if (in(y0 + 1, x0)) out += map[(size_t)(y0 + 1) * Ws + x0] * sw;
    if (in(y0 + 1, x0 + 1)) out += map[(size_t)(y0 + 1) * Ws + x0 + 1] * se;
    return out;
}

__device__ __forceinline__ void depth_conf(const SampleParams& p, const float* __restrict__ depth, const float* __restrict__ conf,
                                           int y, int x, float* d, float* c) {
    const float gx = __fsub_rn(__fmul_rn((float)x, p.grid_sx), 1.f);
    const float gy = __fsub_rn(__fmul_rn((float)y, p.grid_sy), 1.f);
    *d = grid_sample(depth, p.Hs, p.Ws, gx, gy);
    *c = grid_sample(conf, p.Hs, p.Ws, gx, gy);
}

// ---- (a) probability, penalty and decision on a 32x16 tile ----
__global__ void __launch_bounds__(DS_THREADS)
densify_stencil_kernel(SampleParams p, const float* __restrict__ image, const float* __restrict__ rnd,
                       const float* __restrict__ expo, const float* __restrict__ depth, const float* __restrict__ conf,
                       const float* __restrict__ uni, const float* __restrict__ qmin_dev, float* __restrict__ init_proba,
                       float* __restrict__ penalty, unsigned char* __restrict__ flags, int* __restrict__ seg_count) {
    __shared__ float s_in[2][3][IN_H][IN_W];
    __shared__ float s_lap[2][LP_H][LP_W];
    __shared__ float E[12];
    const int tid = threadIdx.y * DS_TX + threadIdx.x;
    if (tid < 12) E[tid] = p.has_render ? expo[tid] : 0.f;
    __syncthreads();
    const int x0 = blockIdx.x * DS_TX, y0 = blockIdx.y * DS_TY;
    const int n_src = p.has_render ? 2 : 1;
    for (int i = tid; i < IN_H * IN_W; i += DS_THREADS) {
        const int sy = i / IN_W, sx = i % IN_W;
        const int gy = y0 - DS_HALO + sy, gx = x0 - DS_HALO + sx;
        const bool inside = gy >= 0 && gy < p.h && gx >= 0 && gx < p.w;       // conv2d "same": zero padding
        float v[3] = {0.f, 0.f, 0.f};
        if (inside) lod_image(p, image, gy, gx, v);
#pragma unroll
        for (int c = 0; c < 3; ++c) s_in[0][c][sy][sx] = v[c];
        if (p.has_render) {
            float r[3] = {0.f, 0.f, 0.f};
            if (inside) lod_render(p, rnd, E, gy, gx, r);
#pragma unroll
            for (int c = 0; c < 3; ++c) s_in[1][c][sy][sx] = r[c];
        }
    }
    __syncthreads();
    // |sum over channels of the 3x3 Laplacian|, with rows / columns 0 and -1 zeroed and zero outside the image
    for (int i = tid; i < LP_H * LP_W; i += DS_THREADS) {
        const int sy = i / LP_W, sx = i % LP_W;
        const int gy = y0 - 3 + sy, gx = x0 - 3 + sx;
        const bool live = gy > 0 && gy < p.h - 1 && gx > 0 && gx < p.w - 1;
        for (int s = 0; s < n_src; ++s) {
            float l = 0.f;
            if (live) {
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float ctr = s_in[s][c][sy + 1][sx + 1];
                    float a = s_in[s][c][sy][sx + 1];
                    a = __fadd_rn(a, s_in[s][c][sy + 1][sx]);
                    a = fmaf(-4.f, ctr, a);
                    a = __fadd_rn(a, s_in[s][c][sy + 1][sx + 2]);
                    a = __fadd_rn(a, s_in[s][c][sy + 2][sx + 1]);
                    l = __fadd_rn(l, a);
                }
                l = fabsf(l);
            }
            s_lap[s][sy][sx] = l;
        }
    }
    __syncthreads();
    const float qmin = *qmin_dev;
    const float tap = 1.0f / 37.0f;
    const int x = x0 + threadIdx.x;
#pragma unroll
    for (int k = 0; k < DS_TY / DS_ROWS; ++k) {
        const int ty = threadIdx.y + k * DS_ROWS;
        const int y = y0 + ty;
        const bool in = x < p.w && y < p.h;
        bool keep = false;
        if (in) {
            float dsum[2] = {0.f, 0.f};
            for (int s = 0; s < n_src; ++s) {
                float a = 0.f;
#pragma unroll
                for (int dy = -3; dy <= 3; ++dy)
#pragma unroll
                    for (int dx = -3; dx <= 3; ++dx)
                        if (dx * dx + dy * dy <= 12) a = fmaf(s_lap[s][ty + 3 + dy][threadIdx.x + 3 + dx], tap, a);
                dsum[s] = a;
            }
            const float pr = __fmul_rn(clampf(dsum[0], 0.f, 1.f), p.scaler);
            const float pe = p.has_render ? __fmul_rn(clampf(dsum[1], 0.f, 1.f), p.scaler) : 0.f;
            const size_t pix = (size_t)y * p.w + x;
            init_proba[pix] = pr;
            if (penalty) penalty[pix] = pe;
            const bool sampled = uni[pix] < __fmul_rn(__fsub_rn(pr, pe), p.ratio);
            bool valid = false;
            if (sampled) {
                float d, c;
                depth_conf(p, depth, conf, y, x, &d, &c);
                valid = (c >= 0.f) && (d > qmin);
            }
            keep = sampled && valid;
            flags[pix] = (unsigned char)((sampled ? 1 : 0) | (valid ? 2 : 0));
        }
        const unsigned int b = __ballot_sync(0xffffffffu, keep);
        if (threadIdx.x == 0 && y < p.h) seg_count[(size_t)y * p.nsx + blockIdx.x] = __popc(b);
    }
}

// ---- (b) emission at the row-major rank ----
__global__ void __launch_bounds__(DS_THREADS)
densify_emit_kernel(SampleParams p, EmitParams e, const float* __restrict__ image, const float* __restrict__ depth,
                    const float* __restrict__ conf, const float* __restrict__ init_proba, const unsigned char* __restrict__ flags,
                    const int* __restrict__ seg_count, const int* __restrict__ seg_incl, const float* __restrict__ cam,
                    float* __restrict__ xyz, float* __restrict__ f_dc, float* __restrict__ scaling, float* __restrict__ opacity,
                    float* __restrict__ d_max) {
    const int x = blockIdx.x * DS_TX + threadIdx.x, y = blockIdx.y * DS_ROWS + threadIdx.y;
    const bool in = x < p.w && y < p.h;
    const size_t pix = (size_t)y * p.w + x;
    const bool keep = in && flags[pix] == 3;
    const unsigned int b = __ballot_sync(0xffffffffu, keep);
    if (!keep) return;
    const size_t seg = (size_t)y * p.nsx + blockIdx.x;
    const long long row = (long long)(seg_incl[seg] - seg_count[seg]) + __popc(b & ((1u << threadIdx.x) - 1u));
    float d, c;
    depth_conf(p, depth, conf, y, x, &d, &c);
    // depth2points (utils.py:188-190) then (P - t) @ R
    const float P[3] = {__fmul_rn(d, __fmul_rn(__fsub_rn((float)x, e.cx), e.inv_f)),
                        __fmul_rn(d, __fmul_rn(__fsub_rn((float)y, e.cy), e.inv_f)), d};
    const float a[3] = {__fsub_rn(P[0], cam[9]), __fsub_rn(P[1], cam[10]), __fsub_rn(P[2], cam[11])};
    float X[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) X[j] = fmaf(a[2], cam[6 + j], fmaf(a[1], cam[3 + j], a[0] * cam[j]));
#pragma unroll
    for (int j = 0; j < 3; ++j) xyz[row * 3 + j] = X[j];
    float v[3];
    lod_image(p, image, y, x, v);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) f_dc[row * 3 + ch] = __fmul_rn(__fsub_rn(v[ch], 0.5f), e.inv_c0);
    const float dx = __fsub_rn(X[0], cam[12]), dy = __fsub_rn(X[1], cam[13]), dz = __fsub_rn(X[2], cam[14]);
    const float dist = sqrtf(fmaf(dz, dz, fmaf(dy, dy, dx * dx)));
    float s = 1.0f / sqrtf(init_proba[pix]);
    s = clampf(s, 1.f, e.wmax);
    s = __fmul_rn(s, e.inv_f_full);
    s = __fmul_rn(s, dist);
    s = logf(__fmul_rn(e.lod_f, clampf(s, 1e-6f, 1e6f)));
#pragma unroll
    for (int j = 0; j < 3; ++j) scaling[row * 3 + j] = s;
    const float o = __fmul_rn(0.2f, c);
    opacity[row] = logf(o / __fsub_rn(1.f, o));
    d_max[row] = __fmul_rn(d, e.lod_f);
}

// ---- (c) depth quantile ----
struct QSel {
    unsigned int bin[2];
    unsigned int rank_in_bin[2];
    int has_nan;
    int pad;
};

__device__ __forceinline__ void q_ranks(long long n, float q, unsigned int* r, float* w) {
    const float rk = q * (float)(n - 1);
    const float lo = floorf(rk);
    r[0] = (unsigned int)lo;
    r[1] = (unsigned int)ceilf(rk);
    *w = rk - lo;
}

__global__ void __launch_bounds__(Q_THREADS)
dq_hist_hi_kernel(long long n, const float* __restrict__ v, unsigned int* __restrict__ hist_hi, QSel* __restrict__ sel) {
    for (long long i = (long long)blockIdx.x * Q_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * Q_THREADS) {
        const float f = v[i];
        if (f != f) atomicOr(&sel->has_nan, 1);
        adb_select::hist_add(hist_hi, adb_select::order_key(f) >> 16);
    }
}

__global__ void __launch_bounds__(SEL_THREADS)
dq_select_hi_kernel(long long n, float q, unsigned int* __restrict__ hist_hi, QSel* __restrict__ sel) {
    __shared__ unsigned int s_tot[SEL_THREADS];
    __shared__ unsigned int s_bins[2], s_in[2];
    unsigned int r[2];
    float w;
    q_ranks(n, q, r, &w);
    if (threadIdx.x < 2) { s_bins[threadIdx.x] = 0u; s_in[threadIdx.x] = 0u; }
    __syncthreads();
    adb_select::hist_find(hist_hi, r, s_bins, s_in, 2, s_tot);
    __syncthreads();
    if (threadIdx.x < 2) { sel->bin[threadIdx.x] = s_bins[threadIdx.x]; sel->rank_in_bin[threadIdx.x] = s_in[threadIdx.x]; }
}

__global__ void __launch_bounds__(Q_THREADS)
dq_hist_lo_kernel(long long n, const float* __restrict__ v, const QSel* __restrict__ sel, unsigned int* __restrict__ hist_lo) {
    const unsigned int b0 = sel->bin[0], b1 = sel->bin[1];
    for (long long i = (long long)blockIdx.x * Q_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * Q_THREADS) {
        const unsigned int k = adb_select::order_key(v[i]);
        if ((k >> 16) == b0) adb_select::hist_add(hist_lo, k & 0xFFFFu);
        if ((k >> 16) == b1) adb_select::hist_add(hist_lo + HIST_BINS, k & 0xFFFFu);
    }
}

// out[0] = torch.quantile(v, q) (NaN if any value is NaN), out[1] = fp32(min(0.01, out[0])) as Python's min evaluates it
__global__ void __launch_bounds__(SEL_THREADS)
dq_select_lo_kernel(long long n, float q, unsigned int* __restrict__ hist_lo, QSel* __restrict__ sel, float* __restrict__ out) {
    __shared__ unsigned int s_tot[SEL_THREADS];
    __shared__ unsigned int s_bins[2], s_in[2];
    unsigned int r[2];
    float w;
    q_ranks(n, q, r, &w);
    if (threadIdx.x < 2) s_bins[threadIdx.x] = 0u;
    __syncthreads();
    const unsigned int r0[1] = {sel->rank_in_bin[0]}, r1[1] = {sel->rank_in_bin[1]};
    adb_select::hist_find(hist_lo, r0, s_bins, s_in, 1, s_tot);
    adb_select::hist_find(hist_lo + HIST_BINS, r1, s_bins + 1, s_in + 1, 1, s_tot);
    __syncthreads();
    if (threadIdx.x != 0) return;
    const float a = adb_select::key_value((sel->bin[0] << 16) | s_bins[0]);
    const float b = adb_select::key_value((sel->bin[1] << 16) | s_bins[1]);
    const float d = b - a;
    float qv = fabsf(w) < 0.5f ? fmaf(w, d, a) : fmaf(-d, 1.0f - w, b);     // ATen lerp
    if (sel->has_nan) qv = __int_as_float(0x7fffffff);
    out[0] = qv;
    out[1] = ((double)qv < 0.01) ? qv : 0.01f;                               // min(1e-2, q): NaN < x is false
}

// ---- (d) prune mask of the existing Gaussians ----
__global__ void __launch_bounds__(256)
densify_prune_kernel(long long N, const float* __restrict__ xyz, const float* __restrict__ opacity,
                     const float* __restrict__ scaling, const float* __restrict__ centre, float f, float half_w,
                     unsigned char* __restrict__ mask) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= N) return;
    const float sig = 1.0f / (1.0f + expf(-opacity[i]));
    const float smax = fmaxf(fmaxf(expf(scaling[i * 3]), expf(scaling[i * 3 + 1])), expf(scaling[i * 3 + 2]));
    const float dx = __fsub_rn(xyz[i * 3], centre[0]), dy = __fsub_rn(xyz[i * 3 + 1], centre[1]),
                dz = __fsub_rn(xyz[i * 3 + 2], centre[2]);
    const float dist = sqrtf(fmaf(dz, dz, fmaf(dy, dy, dx * dx)));
    const float screen = __fmul_rn(f, smax) / dist;
    mask[i] = (sig > 0.05f) && (screen < half_w);
}

// ---- workspace ----
struct DensifyWs {
    int* seg_count;
    int* seg_incl;
    void* scan_tmp;
    size_t scan_bytes;
    unsigned int* hist;          // [3][HIST_BINS]: level 0, then the two level-1 histograms
    QSel* sel;
};
size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

int ws_layout(long long n_seg, unsigned char* base, DensifyWs* w, size_t* bytes) {
    size_t scan_bytes = 0;
    ADB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (const int*)nullptr, (int*)nullptr, (int)n_seg));
    size_t off = 0;
    auto take = [&](size_t b) { unsigned char* q = base ? base + off : nullptr; off += align256(b); return q; };
    DensifyWs t;
    t.seg_count = (int*)take((size_t)n_seg * 4);
    t.seg_incl = (int*)take((size_t)n_seg * 4);
    t.scan_bytes = scan_bytes;
    t.scan_tmp = take(scan_bytes);
    t.hist = (unsigned int*)take((size_t)HIST_BINS * 12);
    t.sel = (QSel*)take(sizeof(QSel));
    if (w) *w = t;
    *bytes = off;
    return ADB_OK;
}

long long n_segments(int h, int w) { return (long long)h * adb_cdiv(w, DS_TX); }

int get_ws(long long n_seg, void* ws, size_t ws_bytes, DensifyWs* w, const char* who) {
    size_t need = 0;
    int rc = ws_layout(n_seg, nullptr, nullptr, &need);
    if (rc != ADB_OK) return rc;
    if (!ws || need > ws_bytes) { adb_set_error_msg(who); return ADB_ERR_WORKSPACE; }
    return ws_layout(n_seg, (unsigned char*)ws, w, &need);
}

SampleParams sample_params(int H, int W, int lod, int Hs, int Ws, float scaler, float ratio, const long long* rstr, bool rnd) {
    SampleParams p{};
    p.H = H; p.W = W; p.lod = lod; p.h = H / lod; p.w = W / lod; p.Hs = Hs; p.Ws = Ws;
    p.nsx = adb_cdiv(p.w, DS_TX);
    const int Hp = H / 2, Wp = W / 2;
    p.scale_img_y = p.h > 1 ? (float)(Hp - 1) / (float)(p.h - 1) : 0.f;
    p.scale_img_x = p.w > 1 ? (float)(Wp - 1) / (float)(p.w - 1) : 0.f;
    p.scale_r_y = p.h > 1 ? (float)(H - 1) / (float)(p.h - 1) : 0.f;
    p.scale_r_x = p.w > 1 ? (float)(W - 1) / (float)(p.w - 1) : 0.f;
    p.grid_sx = (float)(2.0 / (double)(p.w - 1));
    p.grid_sy = (float)(2.0 / (double)(p.h - 1));
    p.scaler = scaler; p.ratio = ratio;
    p.has_render = rnd ? 1 : 0;
    if (rnd) { p.r_cs = rstr[0]; p.r_ys = rstr[1]; p.r_xs = rstr[2]; }
    return p;
}

const char* check_sizes(int H, int W, int lod, int Hs, int Ws) {
    if (!(lod == 1 || lod == 2 || lod == 4 || lod == 8)) return "lod must be 1, 2, 4 or 8";
    if (H < 2 || W < 2 || H / lod < 2 || W / lod < 2) return "the LoD image must be at least 2x2 (make_torch_sampler divides by size - 1)";
    if ((long long)H * W > MAX_PIXELS) return "image too large";
    if (Hs < 1 || Ws < 1 || (long long)Hs * Ws > MAX_PIXELS) return "bad point-map size";
    return nullptr;
}

}  // namespace

ADB_API int adb_densify_workspace_bytes(int height, int width, size_t* bytes) {
    ADB_REQUIRE(bytes && height >= 1 && width >= 1 && (long long)height * width <= MAX_PIXELS,
                "adb_densify_workspace_bytes: bad args");
    return ws_layout(n_segments(height, width), nullptr, nullptr, bytes);
}

ADB_API int adb_densify_depth_quantile(long long n, const float* values, float q, float* out, void* ws, size_t ws_bytes,
                                       cudaStream_t stream) {
    ADB_REQUIRE(n >= 1 && n <= MAX_PIXELS && values && out, "adb_densify_depth_quantile: bad args");
    ADB_REQUIRE(q >= 0.f && q <= 1.f, "adb_densify_depth_quantile: q must lie in [0, 1]");
    DensifyWs w;
    const int rc = get_ws(1, ws, ws_bytes, &w, "adb_densify_depth_quantile: workspace too small");
    if (rc != ADB_OK) return rc;
    ADB_CUDA(cudaMemsetAsync(w.hist, 0, (size_t)HIST_BINS * 12, stream));
    ADB_CUDA(cudaMemsetAsync(w.sel, 0, sizeof(QSel), stream));
    long long nb = (n + Q_THREADS - 1) / Q_THREADS;
    if (nb > 132 * 16) nb = 132 * 16;
    dq_hist_hi_kernel<<<(int)nb, Q_THREADS, 0, stream>>>(n, values, w.hist, w.sel);
    ADB_CHECK_LAUNCH("dq_hist_hi_kernel");
    dq_select_hi_kernel<<<1, SEL_THREADS, 0, stream>>>(n, q, w.hist, w.sel);
    ADB_CHECK_LAUNCH("dq_select_hi_kernel");
    dq_hist_lo_kernel<<<(int)nb, Q_THREADS, 0, stream>>>(n, values, w.sel, w.hist + HIST_BINS);
    ADB_CHECK_LAUNCH("dq_hist_lo_kernel");
    dq_select_lo_kernel<<<1, SEL_THREADS, 0, stream>>>(n, q, w.hist + HIST_BINS, w.sel, out);
    ADB_CHECK_LAUNCH("dq_select_lo_kernel");
    return ADB_OK;
}

ADB_API int adb_densify_sample(int height, int width, int lod, const float* image, const float* render,
                               const long long* render_strides, const float* exposure, int Hs, int Ws, const float* depth,
                               const float* conf, const float* uniforms, const float* qmin, float init_proba_scaler,
                               float gs_add_ratio, float* init_proba, float* penalty, unsigned char* flags, int32_t* n_rows,
                               void* ws, size_t ws_bytes, cudaStream_t stream) {
    const char* bad = check_sizes(height, width, lod, Hs, Ws);
    ADB_REQUIRE(!bad, bad ? bad : "");
    ADB_REQUIRE(image && depth && conf && uniforms && qmin && init_proba && flags && n_rows, "adb_densify_sample: null pointer");
    ADB_REQUIRE(!render || (render_strides && exposure), "adb_densify_sample: a render needs its strides and the exposure");
    const SampleParams p = sample_params(height, width, lod, Hs, Ws, init_proba_scaler, gs_add_ratio, render_strides,
                                         render != nullptr);
    const long long n_seg = (long long)p.h * p.nsx;
    DensifyWs w;
    const int rc = get_ws(n_seg, ws, ws_bytes, &w, "adb_densify_sample: workspace too small");
    if (rc != ADB_OK) return rc;
    densify_stencil_kernel<<<dim3(p.nsx, adb_cdiv(p.h, DS_TY)), dim3(DS_TX, DS_ROWS), 0, stream>>>(
        p, image, render, exposure, depth, conf, uniforms, qmin, init_proba, penalty, flags, w.seg_count);
    ADB_CHECK_LAUNCH("densify_stencil_kernel");
    size_t sb = w.scan_bytes;
    ADB_CUDA(cub::DeviceScan::InclusiveSum(w.scan_tmp, sb, w.seg_count, w.seg_incl, (int)n_seg, stream));
    ADB_CUDA(cudaMemcpyAsync(n_rows, w.seg_incl + (n_seg - 1), sizeof(int32_t), cudaMemcpyDeviceToDevice, stream));
    return ADB_OK;
}

ADB_API int adb_densify_emit(int height, int width, int lod, const float* image, int Hs, int Ws, const float* depth,
                             const float* conf, const float* init_proba, const unsigned char* flags, const float* cam, double f,
                             float* xyz, float* f_dc, float* scaling, float* opacity, float* d_max, void* ws, size_t ws_bytes,
                             cudaStream_t stream) {
    const char* bad = check_sizes(height, width, lod, Hs, Ws);
    ADB_REQUIRE(!bad, bad ? bad : "");
    ADB_REQUIRE(image && depth && conf && init_proba && flags && cam && xyz && f_dc && scaling && opacity && d_max,
                "adb_densify_emit: null pointer");
    ADB_REQUIRE(f > 0.0, "adb_densify_emit: f must be positive");
    const SampleParams p = sample_params(height, width, lod, Hs, Ws, 1.f, 1.f, nullptr, false);
    DensifyWs w;
    const int rc = get_ws((long long)p.h * p.nsx, ws, ws_bytes, &w, "adb_densify_emit: workspace too small");
    if (rc != ADB_OK) return rc;
    EmitParams e;
    const float inv_lod = 1.0f / (float)lod;
    e.cx = (float)((width - 1) / 2.0) * inv_lod;
    e.cy = (float)((height - 1) / 2.0) * inv_lod;
    e.inv_f = 1.0f / (float)(f / lod);
    e.inv_f_full = (float)(1.0 / f);
    e.wmax = (float)(width / 10.0);
    e.lod_f = (float)lod;
    e.inv_c0 = 1.0f / (float)0.28209479177387814;
    densify_emit_kernel<<<dim3(p.nsx, adb_cdiv(p.h, DS_ROWS)), dim3(DS_TX, DS_ROWS), 0, stream>>>(
        p, e, image, depth, conf, init_proba, flags, w.seg_count, w.seg_incl, cam, xyz, f_dc, scaling, opacity, d_max);
    ADB_CHECK_LAUNCH("densify_emit_kernel");
    return ADB_OK;
}

ADB_API int adb_densify_prune_mask(long long N, const float* xyz, const float* opacity, const float* scaling,
                                   const float* approx_centre, double f, int width, unsigned char* mask, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && width >= 1 && f > 0.0, "adb_densify_prune_mask: bad args");
    if (N == 0) return ADB_OK;
    ADB_REQUIRE(xyz && opacity && scaling && approx_centre && mask, "adb_densify_prune_mask: null pointer");
    densify_prune_kernel<<<(unsigned)((N + 255) / 256), 256, 0, stream>>>(N, xyz, opacity, scaling, approx_centre, (float)f,
                                                                       (float)(0.5 * width), mask);
    ADB_CHECK_LAUNCH("densify_prune_kernel");
    return ADB_OK;
}

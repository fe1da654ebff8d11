// Frame tracking: the calibrated Sim(3) pose tracker of ARTDECO's Frontend, CameraTracker.track after matching
// (VSLAM/CameraTracker.py:53-155, opt_pose_calib_sim3 :296-396, nonlinear_optimizer.py:5-33, utils_uncertainty.py:5-50).
//
// The reference runs every Gauss-Newton iteration over all H*W points as some tens of small torch kernels, a sort for
// torch.quantile, a cuSOLVER Cholesky and a `.item()` host sync.  Here one iteration is a fixed sequence of launches that
// turn into no-ops once the device flag `state->done` is set, so the whole solve (and the frame) can be captured in a graph:
//   track_det_hist    (filter on) det of the projected covariance in closed form, order-preserving 16-bit radix histogram
//   track_select  x2  exact selection of the two order statistics torch.quantile interpolates (high then low 16 bits)
//   track_hist_lo     (filter on) histogram of the low 16 bits inside the two selected high bins
//   track_reduce      residuals, Jacobians, Huber weights; 28 + 7 + 1 sums per CTA in fp32, written without atomics
//   track_step        one CTA: CTA partials summed in fp64 in a fixed order, 7x7 Cholesky in fp64, Exp(tau) T, quat2unit,
//                     check_convergence.
// Every sum has a fixed order and the histograms count integers, so results are bitwise reproducible run to run.
#include "common.cuh"
#include "select.cuh"
#include "sim3.cuh"
#include "artdeco_b200.h"

namespace {

using adb_sim3::act_so3;
using adb_sim3::quat_comp;
using adb_select::HIST_BINS;
using adb_select::SEL_THREADS;
using adb_select::hist_add;
using adb_select::hist_find;
using adb_select::key_value;
using adb_select::order_key;

constexpr int TR_THREADS = 256;
constexpr int TR_MAX_BLOCKS = 1024;       // reduce grid cap: fixed by N only, so the summation order is device-independent
constexpr int TR_NSUM = 36;               // 28 (upper triangle of A^T A) + 7 (A^T b) + 1 (b^T b)

struct Sel {                               // selection state (workspace)
    unsigned int bin[2];                   // high 16 bits of the two order statistics
    unsigned int rank_in_bin[2];
    int has_nan;
    int pad;
};

// ---- Sim(3) on [8] = (t, q xyzw, s), as pypose stores it ----
__device__ __forceinline__ void quat2unit(float* T) {
    const float n = fmaxf(sqrtf(T[3] * T[3] + T[4] * T[4] + T[5] * T[5] + T[6] * T[6]), 1e-12f);
    T[3] /= n; T[4] /= n; T[5] /= n; T[6] /= n;
}
__device__ __forceinline__ void act_sim3(const float* T, const float* X, float* Y) {
    act_so3(T + 3, X, Y);
    Y[0] = Y[0] * T[7] + T[0]; Y[1] = Y[1] * T[7] + T[1]; Y[2] = Y[2] * T[7] + T[2];
}
__device__ __forceinline__ void mul_sim3(const float* A, const float* B, float* out) {     // A * B
    float t[3], q[4];
    act_sim3(A, B, t);
    quat_comp(A + 3, B + 3, q);
    const float s = A[7] * B[7];
    out[0] = t[0]; out[1] = t[1]; out[2] = t[2];
    out[3] = q[0]; out[4] = q[1]; out[5] = q[2]; out[6] = q[3]; out[7] = s;
}
__device__ __forceinline__ void inv_sim3(const float* A, float* out) {
    const float qi[4] = {-A[3], -A[4], -A[5], A[6]};
    const float si = 1.0f / A[7];
    float t[3];
    act_so3(qi, A, t);
    out[0] = -si * t[0]; out[1] = -si * t[1]; out[2] = -si * t[2];
    out[3] = qi[0]; out[4] = qi[1]; out[5] = qi[2]; out[6] = qi[3]; out[7] = si;
}

// ================================ preparation ================================

// local_diag_cov_from_X1 (utils_uncertainty.py:5-50) on the frame's ray-constrained pointmap, frame pixel order.
// Box filter 5x5 with reflect padding, summed row by row in fp32 and divided by 25 like avg_pool2d; validity
// finite & z > 0 enters as a 0/1 factor (so a non-finite point still poisons its neighbours, as in the reference).
constexpr int COV_TX = 32, COV_TY = 8, COV_R = 2;
constexpr int COV_SW = COV_TX + 2 * COV_R, COV_SH = COV_TY + 2 * COV_R;

__global__ void __launch_bounds__(COV_TX * COV_TY)
track_cov_kernel(int H, int W, const float* __restrict__ Kd, const float* __restrict__ Xff, float* __restrict__ cov_f) {
    __shared__ float sm[7][COV_SH][COV_SW];
    const float fx = Kd[0], fy = Kd[4], cx = Kd[2], cy = Kd[5];
    const int x0 = blockIdx.x * COV_TX, y0 = blockIdx.y * COV_TY;
    const int tid = threadIdx.y * COV_TX + threadIdx.x;
    for (int c = tid; c < COV_SH * COV_SW; c += COV_TX * COV_TY) {
        const int sy = c / COV_SW, sx = c % COV_SW;
        int gy = y0 - COV_R + sy, gx = x0 - COV_R + sx;
        gy = gy < 0 ? -gy : (gy >= H ? 2 * H - 2 - gy : gy);
        gx = gx < 0 ? -gx : (gx >= W ? 2 * W - 2 - gx : gx);
        gy = min(max(gy, 0), H - 1);           // rows / columns past a partial tile feed no output
        gx = min(max(gx, 0), W - 1);
        const float z = Xff[((size_t)gy * W + gx) * 3 + 2];
        const float x = ((float)gx - cx) / fx * z, y = ((float)gy - cy) / fy * z;
        const float v = (isfinite(x) && isfinite(y) && isfinite(z) && z > 0.f) ? 1.f : 0.f;
        sm[0][sy][sx] = v;
        sm[1][sy][sx] = x * v; sm[2][sy][sx] = y * v; sm[3][sy][sx] = z * v;
        sm[4][sy][sx] = (x * x) * v; sm[5][sy][sx] = (y * y) * v; sm[6][sy][sx] = (z * z) * v;
    }
    __syncthreads();
    const int ox = x0 + threadIdx.x, oy = y0 + threadIdx.y;
    if (ox >= W || oy >= H) return;
    float s[7];
#pragma unroll
    for (int ch = 0; ch < 7; ++ch) {
        float a = 0.f;
#pragma unroll
        for (int dy = 0; dy < 5; ++dy)
#pragma unroll
            for (int dx = 0; dx < 5; ++dx) a += sm[ch][threadIdx.y + dy][threadIdx.x + dx];
        s[ch] = a / 25.0f;
    }
    const float denom = fmaxf(s[0], 1e-9f);
    float* out = cov_f + ((size_t)oy * W + ox) * 3;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const float mean = s[1 + d] / denom, ex2 = s[4 + d] / denom;
        out[d] = fmaxf(__fsub_rn(ex2, __fmul_rn(mean, mean)), 1e-12f);   // no FMA: E[X^2] - E[X]^2 cancels
    }
}

struct PrepParams {
    int H, W, n;
    float C_conf, Q_conf, depth_eps;
};

// get_points_poses (:189-219) + the masks of :83-87, key-frame pixel order.  Counts by warp ballots (integers).
__global__ void __launch_bounds__(TR_THREADS)
track_gather_kernel(PrepParams p, const float* __restrict__ Kd, const long long* __restrict__ idx,
                    const unsigned char* __restrict__ vmatch, const float* __restrict__ Xff, const float* __restrict__ Cff,
                    const float* __restrict__ Qff, const float* __restrict__ Qkf, const float* __restrict__ kfX,
                    const float* __restrict__ kfC, const int* __restrict__ kfN, const float* __restrict__ cov_f,
                    unsigned int* __restrict__ seen, float* __restrict__ Xf, float* __restrict__ Xf_cov,
                    float* __restrict__ Qk_out, float* __restrict__ meas, unsigned char* __restrict__ vmeas_out,
                    unsigned char* __restrict__ vopt_out, unsigned char* __restrict__ vkf_out, adb_track_state* st) {
    const int i = blockIdx.x * TR_THREADS + threadIdx.x;
    const bool in = i < p.n;
    bool vo = false, vk = false, first = false;
    if (in) {
        const float fx = Kd[0], fy = Kd[4], cx = Kd[2], cy = Kd[5];
        long long jl = idx[i];
        jl = jl < 0 ? 0 : (jl >= p.n ? p.n - 1 : jl);    // memory safety only: matching emits indices in [0, N)
        const int j = (int)jl;
        const int uj = j % p.W, vj = j / p.W, ui = i % p.W, vi = i / p.W;
        const float z = Xff[(size_t)j * 3 + 2];
        Xf[(size_t)i * 3 + 0] = ((float)uj - cx) / fx * z;
        Xf[(size_t)i * 3 + 1] = ((float)vj - cy) / fy * z;
        Xf[(size_t)i * 3 + 2] = z;
#pragma unroll
        for (int d = 0; d < 3; ++d) Xf_cov[(size_t)i * 3 + d] = cov_f[(size_t)j * 3 + d];
        const float q = sqrtf(Qff[j] * Qkf[i]);
        Qk_out[i] = q;
        const float cf = Cff[j];                            // the frame's update_pointmap with N = 0: C = Cff, N = 1
        const float ck = kfC[i] / (float)(*kfN);            // keyframe.get_average_conf()
        const float zk = kfX[(size_t)i * 3 + 2];
        const bool vm_k = zk > p.depth_eps;
        meas[(size_t)i * 3 + 0] = vm_k ? (float)ui : 0.f;
        meas[(size_t)i * 3 + 1] = vm_k ? (float)vi : 0.f;
        meas[(size_t)i * 3 + 2] = vm_k ? logf(zk) : 0.f;
        vmeas_out[i] = vm_k;
        const bool vm = vmatch[i] != 0;
        vo = vm && (cf > p.C_conf) && (ck > p.C_conf) && (q > p.Q_conf);
        vk = vm && (q > p.Q_conf);
        vopt_out[i] = vo;
        vkf_out[i] = vk;
        if (vm) {
            const unsigned int bit = 1u << (j & 31);
            first = (atomicOr(seen + (j >> 5), bit) & bit) == 0u;
        }
    }
    const unsigned int bo = __ballot_sync(0xffffffffu, vo), bk = __ballot_sync(0xffffffffu, vk),
                       bu = __ballot_sync(0xffffffffu, first);
    if ((threadIdx.x & 31) == 0) {
        if (bo) atomicAdd(&st->n_valid_opt, __popc(bo));
        if (bk) atomicAdd(&st->n_valid_kf, __popc(bk));
        if (bu) atomicAdd(&st->n_unique, __popc(bu));
    }
}

// match_frac < min_match_frac -> lost before any solve (:90-118)
__global__ void track_match_check_kernel(int n, float min_match_frac, adb_track_state* st) {
    if (threadIdx.x != 0) return;
    const float frac = (float)st->n_valid_opt / (float)n;
    if (frac < min_match_frac) { st->lost = ADB_TRACK_LOST_MATCHES; st->done = 1; }
}

// ================================ exact quantile selection ================================
// torch.quantile(v, q) with linear interpolation: r = q (n-1) in fp32, the order statistics floor(r) and ceil(r), lerp by
// r - floor(r) (ATen's lerp, small-weight branch).  Level 0 finds the high-16-bit bin of both order statistics, level 1
// the exact keys inside those bins; each level zeroes the histogram it consumed.  mode 0: covariance filter (n = N, gated
// by state->done; threshold = max(quantile, 1), NaN if any value is NaN).  mode 1: key-frame displacement (n = n_valid_opt,
// gated by state->lost; the decision of check_keyframe_map).
struct SelParams {
    int mode, n_all;
    float q;
    double min_displacement, last_dist;
};

__device__ bool sel_active(int mode, const adb_track_state* st) { return mode == 0 ? st->done == 0 : st->lost == 0; }

__device__ __forceinline__ void sel_ranks(const SelParams& p, const adb_track_state* st, int* n_out, unsigned int* r,
                                          float* w) {
    const int n = p.mode == 0 ? p.n_all : st->n_valid_opt;
    *n_out = n;
    const float rk = p.q * (float)(n > 0 ? n - 1 : 0);
    const float lo = floorf(rk);
    r[0] = (unsigned int)lo;
    r[1] = (unsigned int)ceilf(rk);
    *w = rk - lo;
}

__global__ void __launch_bounds__(SEL_THREADS)
track_select_hi_kernel(SelParams p, unsigned int* __restrict__ hist_hi, Sel* __restrict__ sel, const adb_track_state* st) {
    if (!sel_active(p.mode, st)) return;
    __shared__ unsigned int s_tot[SEL_THREADS];
    __shared__ unsigned int s_bins[2], s_in[2];
    int n;
    unsigned int r[2];
    float w;
    sel_ranks(p, st, &n, r, &w);
    if (threadIdx.x < 2) { s_bins[threadIdx.x] = 0u; s_in[threadIdx.x] = 0u; }
    __syncthreads();
    hist_find(hist_hi, r, s_bins, s_in, n > 0 ? 2 : 0, s_tot);
    __syncthreads();
    if (threadIdx.x < 2) { sel->bin[threadIdx.x] = s_bins[threadIdx.x]; sel->rank_in_bin[threadIdx.x] = s_in[threadIdx.x]; }
}

__global__ void __launch_bounds__(SEL_THREADS)
track_select_lo_kernel(SelParams p, unsigned int* __restrict__ hist_lo, Sel* __restrict__ sel, adb_track_state* st) {
    if (!sel_active(p.mode, st)) return;
    __shared__ unsigned int s_tot[SEL_THREADS];
    __shared__ unsigned int s_bins[2], s_in[2];
    int n;
    unsigned int r[2];
    float w;
    sel_ranks(p, st, &n, r, &w);
    if (threadIdx.x < 2) s_bins[threadIdx.x] = 0u;
    __syncthreads();
    const unsigned int r0[1] = {sel->rank_in_bin[0]}, r1[1] = {sel->rank_in_bin[1]};
    hist_find(hist_lo, r0, s_bins, s_in, n > 0 ? 1 : 0, s_tot);
    hist_find(hist_lo + HIST_BINS, r1, s_bins + 1, s_in + 1, n > 0 ? 1 : 0, s_tot);
    __syncthreads();
    if (threadIdx.x != 0) return;
    const int has_nan = sel->has_nan;
    sel->has_nan = 0;
    float qv;
    if (n <= 0) {
        qv = __int_as_float(0x7fffffff);     // empty selection (the reference would raise)
    } else {
        const float a = key_value((sel->bin[0] << 16) | s_bins[0]), b = key_value((sel->bin[1] << 16) | s_bins[1]);
        const float d = b - a;
        qv = fabsf(w) < 0.5f ? fmaf(w, d, a) : fmaf(-d, 1.0f - w, b);
    }
    if (p.mode == 0) {
        if (has_nan) qv = __int_as_float(0x7fffffff);
        st->cov_threshold = (1.0f > qv) ? 1.0f : qv;      // Python max(q, 1) keeps q unless 1 > q (so NaN stays NaN)
    } else {
        st->dist_quantile = qv;
        if (!st->is_keyframe) {
            const bool add = ((double)qv - p.last_dist) > p.min_displacement;
            st->is_keyframe_map = add;
            st->last_dist = add ? (double)qv : p.last_dist;
        }
    }
}

// values whose high 16 bits are one of the two selected bins -> histograms of their low 16 bits
__global__ void __launch_bounds__(TR_THREADS)
track_hist_lo_kernel(int n, int mode, const float* __restrict__ vals, const Sel* __restrict__ sel,
                     unsigned int* __restrict__ hist_lo, const adb_track_state* st) {
    if (!sel_active(mode, st)) return;
    const int i = blockIdx.x * TR_THREADS + threadIdx.x;
    if (i >= n) return;
    const unsigned int k = order_key(vals[i]);
    const unsigned int b0 = sel->bin[0], b1 = sel->bin[1];
    if ((k >> 16) == b0) hist_add(hist_lo, k & 0xFFFFu);
    if ((k >> 16) == b1) hist_add(hist_lo + HIST_BINS, k & 0xFFFFu);
}

// ================================ Gauss-Newton ================================
struct SolveParams {
    int n, H, W;
    int filter;
    float border, u_max, v_max, depth_eps;
    float inv_sp, inv_sd, huber_k;
    double rel_error;
    float delta_norm;
};

// Projected-covariance determinant (:336-345) in closed form: T.matrix()[:3,:3] = sR and Sigma is diagonal, so
// det(JCOV (sR) Sigma (sR)^T JCOV^T) = (fx fy / Z^3)^2 s^6 vx vy vz.
__global__ void __launch_bounds__(TR_THREADS)
track_det_hist_kernel(SolveParams p, const float* __restrict__ Kd, const float* __restrict__ Xf, const float* __restrict__ cov,
                      float* __restrict__ vals, unsigned int* __restrict__ hist_hi, Sel* __restrict__ sel,
                      const adb_track_state* st) {
    if (st->done) return;
    __shared__ float T[8];
    if (threadIdx.x < 8) T[threadIdx.x] = st->T_CkCf[threadIdx.x];
    __syncthreads();
    const int i = blockIdx.x * TR_THREADS + threadIdx.x;
    if (i >= p.n) return;
    const float X[3] = {Xf[(size_t)i * 3], Xf[(size_t)i * 3 + 1], Xf[(size_t)i * 3 + 2]};
    float P[3];
    act_sim3(T, X, P);
    const float Z = P[2], s = T[7];
    const float jd = Kd[0] * Kd[4] / (Z * Z * Z), s3 = s * s * s;
    const float det = (jd * jd) * (s3 * s3) * cov[(size_t)i * 3] * cov[(size_t)i * 3 + 1] * cov[(size_t)i * 3 + 2];
    vals[i] = det;
    if (det != det) atomicOr(&sel->has_nan, 1);
    hist_add(hist_hi, order_key(det) >> 16);
}

__global__ void __launch_bounds__(TR_THREADS)
track_reduce_kernel(SolveParams p, const float* __restrict__ Kd, const float* __restrict__ Xf, const float* __restrict__ Qk,
                    const unsigned char* __restrict__ valid, const float* __restrict__ meas,
                    const unsigned char* __restrict__ vmeas, const float* __restrict__ det, float* __restrict__ partial,
                    const adb_track_state* st) {
    if (st->done) return;
    __shared__ float T[8];
    __shared__ float sRed[TR_THREADS / 32][TR_NSUM];
    if (threadIdx.x < 8) T[threadIdx.x] = st->T_CkCf[threadIdx.x];
    __syncthreads();
    const float thr = st->cov_threshold;
    const float k00 = Kd[0], k01 = Kd[1], k02 = Kd[2], k10 = Kd[3], k11 = Kd[4], k12 = Kd[5], k20 = Kd[6], k21 = Kd[7],
                k22 = Kd[8];
    float acc[TR_NSUM];
#pragma unroll
    for (int l = 0; l < TR_NSUM; ++l) acc[l] = 0.f;
    for (int i = blockIdx.x * TR_THREADS + threadIdx.x; i < p.n; i += gridDim.x * TR_THREADS) {
        const float X[3] = {Xf[(size_t)i * 3], Xf[(size_t)i * 3 + 1], Xf[(size_t)i * 3 + 2]};
        float P[3];
        act_sim3(T, X, P);
        const float x = P[0], y = P[1], z = P[2];
        // project_calib (geometry.py:66-113)
        const float p0 = k00 * x + k01 * y + k02 * z, p1 = k10 * x + k11 * y + k12 * z, p2 = k20 * x + k21 * y + k22 * z;
        const float u = p0 / p2, v = p1 / p2;
        const bool vz = z > p.depth_eps;
        const bool vproj = (u > p.border) && (u < p.u_max) && (v > p.border) && (v < p.v_max) && vz;
        const float logz = vz ? logf(z) : 0.f;
        const bool vcov = p.filter ? (det[i] < thr) : true;
        const float w2 = (vproj && vmeas[i] && vcov) ? 1.f : 0.f;          // valid2
        const float vo = valid[i] ? 1.f : 0.f;
        const float sq = sqrtf(Qk[i]);
        const float s_pix = w2 * ((p.inv_sp * vo) * sq), s_dep = w2 * ((p.inv_sd * vo) * sq);   // valid2 * sqrt_info
        const float r[3] = {meas[(size_t)i * 3] - u, meas[(size_t)i * 3 + 1] - v, meas[(size_t)i * 3 + 2] - logz};
        const float zi = 1.0f / z;
        const float a = k00 * zi, c = (-k00 * x * zi) * zi, b = k11 * zi, e = (-k11 * y * zi) * zi;
        // J = -dpz/dP [I | -[P]x | P]
        const float J[3][7] = {{-a, 0.f, -c, -(c * y), -(a * z - c * x), a * y, -(a * x + c * z)},
                               {0.f, -b, -e, -(e * y - b * z), e * x, -(b * x), -(b * y + e * z)},
                               {0.f, 0.f, -zi, -(zi * y), zi * x, 0.f, -(zi * z)}};
#pragma unroll
        for (int row = 0; row < 3; ++row) {
            const float s2 = row < 2 ? s_pix : s_dep;
            const float rob = s2 * sqrtf(adb_sim3::huber(s2 * r[row], p.huber_k));
            const float br = rob * r[row];
            float A[7];
#pragma unroll
            for (int m = 0; m < 7; ++m) A[m] = rob * J[row][m];
            int l = 0;
#pragma unroll
            for (int m = 0; m < 7; ++m)
#pragma unroll
                for (int k = m; k < 7; ++k) acc[l++] += A[m] * A[k];
#pragma unroll
            for (int m = 0; m < 7; ++m) acc[28 + m] += A[m] * br;
            acc[35] += br * br;
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int l = 0; l < TR_NSUM; ++l) {
        const float s = adb_warp_sum(acc[l]);
        if (lane == 0) sRed[warp][l] = s;
    }
    __syncthreads();
    if (threadIdx.x < TR_NSUM) {
        float s = 0.f;
#pragma unroll
        for (int w_ = 0; w_ < TR_THREADS / 32; ++w_) s += sRed[w_][threadIdx.x];
        partial[(size_t)blockIdx.x * TR_NSUM + threadIdx.x] = s;
    }
}

constexpr int STEP_SPLIT = 8;
// One CTA of TR_NSUM * STEP_SPLIT threads.  solve() (:223-238) + Exp(tau) T + quat2unit + check_convergence.
__global__ void __launch_bounds__(TR_NSUM * STEP_SPLIT)
track_step_kernel(SolveParams p, int n_blocks, const float* __restrict__ partial, adb_track_state* st) {
    if (st->done) return;
    __shared__ double sPart[STEP_SPLIT][TR_NSUM];
    const int v = threadIdx.x % TR_NSUM, part = threadIdx.x / TR_NSUM;
    double s = 0.0;
    for (int b = part; b < n_blocks; b += STEP_SPLIT) s += (double)partial[(size_t)b * TR_NSUM + v];
    sPart[part][v] = s;
    __syncthreads();
    if (threadIdx.x != 0) return;
    double sum[TR_NSUM];
    for (int l = 0; l < TR_NSUM; ++l) {
        double t = 0.0;
        for (int q = 0; q < STEP_SPLIT; ++q) t += sPart[q][l];
        sum[l] = t;
    }
    double H[7][7], g[7];
    int l = 0;
    for (int m = 0; m < 7; ++m)
        for (int k = m; k < 7; ++k) { H[m][k] = sum[l]; H[k][m] = sum[l]; ++l; }
    for (int m = 0; m < 7; ++m) g[m] = -sum[28 + m];
    const double cost = 0.5 * sum[35];
    for (int m = 0; m < 7; ++m) {
        st->g[m] = g[m];
        for (int k = 0; k < 7; ++k) st->H[m * 7 + k] = H[m][k];
    }
    st->cost = cost;
    // Cholesky H = L L^T in place (lower triangle); a pivot that is not positive (or NaN) is the reference's exception
    double L[7][7];
    for (int j = 0; j < 7; ++j) {
        double d = H[j][j];
        for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k];
        if (!(d > 0.0)) { st->lost = ADB_TRACK_LOST_CHOLESKY; st->done = 1; return; }
        L[j][j] = sqrt(d);
        for (int i = j + 1; i < 7; ++i) {
            double a = H[i][j];
            for (int k = 0; k < j; ++k) a -= L[i][k] * L[j][k];
            L[i][j] = a / L[j][j];
        }
    }
    double y[7], x[7];
    for (int i = 0; i < 7; ++i) {
        double a = g[i];
        for (int k = 0; k < i; ++k) a -= L[i][k] * y[k];
        y[i] = a / L[i][i];
    }
    for (int i = 6; i >= 0; --i) {
        double a = y[i];
        for (int k = i + 1; k < 7; ++k) a -= L[k][i] * x[k];
        x[i] = a / L[i][i];
    }
    float tau[7], nrm2 = 0.f;
    for (int m = 0; m < 7; ++m) { tau[m] = (float)x[m]; nrm2 += tau[m] * tau[m]; }
    const float tau_norm = sqrtf(nrm2);
    // T <- quat2unit(Exp(tau) T)
    float E[8], Tn[8];
    adb_sim3::exp_sim3(tau, E, E + 3, E + 7);
    mul_sim3(E, st->T_CkCf, Tn);
    quat2unit(Tn);
    for (int m = 0; m < 8; ++m) st->T_CkCf[m] = Tn[m];
    // check_convergence (nonlinear_optimizer.py:5-25): rel_dec is NaN on the first iteration (old_cost = inf); an old cost
    // of exactly 0 raises ZeroDivisionError in the reference, which track() reports as lost
    const int it = st->iters;
    st->iters = it + 1;
    st->tau_norm = tau_norm;
    bool conv;
    if (it == 0) {
        conv = tau_norm < p.delta_norm;
    } else {
        const double old = st->prev_cost;
        if (old == 0.0) { st->lost = ADB_TRACK_LOST_ZERO_COST; st->done = 1; return; }
        const double rel = fabs((old - cost) / old);
        conv = (rel < p.rel_error) || (tau_norm < p.delta_norm);
    }
    st->prev_cost = cost;
    if (conv) { st->converged = 1; st->done = 1; }
}

// T_CkCf = quat2unit(T_WCk)^-1 quat2unit(T_WCf) (get_points_poses :194-195, :303); resets the solver fields
__global__ void track_init_kernel(const float* __restrict__ T_WCf, const float* __restrict__ T_WCk,
                                  float* __restrict__ T_CkCf_out, adb_track_state* st) {
    if (threadIdx.x != 0) return;
    float Tf[8], Tk[8], Ti[8], T[8];
    for (int m = 0; m < 8; ++m) { Tf[m] = T_WCf[m]; Tk[m] = T_WCk[m]; }
    quat2unit(Tf);
    quat2unit(Tk);
    inv_sim3(Tk, Ti);
    mul_sim3(Ti, Tf, T);
    for (int m = 0; m < 8; ++m) { st->T_CkCf[m] = T[m]; st->T_WCk[m] = Tk[m]; T_CkCf_out[m] = T[m]; }
    st->iters = 0; st->converged = 0; st->tau_norm = 0.f; st->cost = 0.0; st->prev_cost = 0.0;
    st->cov_threshold = 0.f;
    st->done = st->lost != 0;
}

// T_WCf = quat2unit(T_WCk T_CkCf) (:395, :134); nothing is written on a lost outcome
__global__ void track_out_kernel(float* __restrict__ T_WCf_out, float* __restrict__ T_CkCf_out, const adb_track_state* st) {
    if (threadIdx.x != 0 || st->lost) return;
    float T[8];
    mul_sim3(st->T_WCk, st->T_CkCf, T);
    quat2unit(T);
    for (int m = 0; m < 8; ++m) { T_WCf_out[m] = T[m]; T_CkCf_out[m] = st->T_CkCf[m]; }
}

// ================================ after the solve ================================
// check_keyframe (:159-167): min(valid_kf.sum() / N, |unique| / N) < match_frac_thresh, with the reference's mixed
// float32-tensor / Python-float comparisons
__global__ void track_keyframe_kernel(int n, double match_frac_thresh, double last_dist, adb_track_state* st) {
    if (threadIdx.x != 0 || st->lost) return;
    const float a = (float)st->n_valid_kf / (float)n;
    const double b = (double)st->n_unique / (double)n;
    const bool take_b = a > (float)b;                    // min(a, b) evaluates b < a
    const bool kf = take_b ? (b < match_frac_thresh) : (a < (float)match_frac_thresh);
    st->is_keyframe = kf;
    st->is_keyframe_map = kf;
    st->last_dist = kf ? 0.0 : last_dist;
}

// check_keyframe_map (:170-186): pixel displacement of every valid_opt match; +inf elsewhere sorts past the n selected ranks
__global__ void __launch_bounds__(TR_THREADS)
track_dist_hist_kernel(int n, int W, const long long* __restrict__ idx, const unsigned char* __restrict__ vopt,
                       float* __restrict__ vals, unsigned int* __restrict__ hist_hi, const adb_track_state* st) {
    if (st->lost) return;
    const int i = blockIdx.x * TR_THREADS + threadIdx.x;
    if (i >= n) return;
    float d = __int_as_float(0x7f800000);
    if (vopt[i]) {
        const long long j = idx[i];
        const long long du = j % W - i % W, dv = j / W - i / W;
        d = sqrtf((float)(du * du + dv * dv));
    }
    vals[i] = d;
    hist_add(hist_hi, order_key(d) >> 16);
}

// update_pointmap (ImageFrame.py:42-46) with Xkk = T_CkCf.Act(Xkf): X <- (C X + Ckf Xkk) / (C + Ckf), C += Ckf, N += 1.
// Each product and sum rounded separately, as the reference's elementwise kernels do.
__global__ void __launch_bounds__(TR_THREADS)
track_fuse_kernel(int n, const float* __restrict__ Xkf, const float* __restrict__ Ckf, float* __restrict__ kfX,
                  float* __restrict__ kfC, int* __restrict__ kfN, const adb_track_state* st) {
    if (st->lost) return;
    const int i = blockIdx.x * TR_THREADS + threadIdx.x;
    if (i == 0) *kfN += 1;
    if (i >= n) return;
    const float Xs[3] = {Xkf[(size_t)i * 3], Xkf[(size_t)i * 3 + 1], Xkf[(size_t)i * 3 + 2]};
    float Xk[3];
    act_sim3(st->T_CkCf, Xs, Xk);
    const float c = kfC[i], ck = Ckf[i];
    const float den = __fadd_rn(c, ck);
#pragma unroll
    for (int d = 0; d < 3; ++d)
        kfX[(size_t)i * 3 + d] = __fdiv_rn(__fadd_rn(__fmul_rn(c, kfX[(size_t)i * 3 + d]), __fmul_rn(ck, Xk[d])), den);
    kfC[i] = den;
}

// ---- workspace ----
struct TrackWs {
    float* cov_f;            // [N,3] frame-order variances (prepare)
    float* vals;             // [N] values being selected (determinants, displacements)
    unsigned int* seen;      // [ceil(N/32)] frame pixels already matched (unique count)
    unsigned int* hist_hi;   // [65536]
    unsigned int* hist_lo;   // [2][65536]
    float* partial;          // [TR_MAX_BLOCKS][36]
    Sel* sel;
};
size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
size_t ws_layout(int n, unsigned char* base, TrackWs* w) {
    size_t off = 0;
    auto take = [&](size_t bytes) { unsigned char* p = base ? base + off : nullptr; off += align256(bytes); return p; };
    TrackWs t;
    t.cov_f = (float*)take((size_t)n * 12);
    t.vals = (float*)take((size_t)n * 4);
    t.seen = (unsigned int*)take(((size_t)n + 31) / 32 * 4);
    t.hist_hi = (unsigned int*)take((size_t)HIST_BINS * 4);
    t.hist_lo = (unsigned int*)take((size_t)HIST_BINS * 8);
    t.partial = (float*)take((size_t)TR_MAX_BLOCKS * TR_NSUM * 4);
    t.sel = (Sel*)take(sizeof(Sel));
    if (w) *w = t;
    return off;
}
constexpr int TR_MAX_PTS = 1 << 26;

int check_ws(int n, void* ws, size_t ws_bytes, TrackWs* w, const char* who) {
    const size_t need = ws_layout(n, nullptr, nullptr);
    if (need > ws_bytes) {
        adb_set_error_msg(who);
        return ADB_ERR_WORKSPACE;
    }
    ws_layout(n, (unsigned char*)ws, w);
    return ADB_OK;
}

}  // namespace

ADB_API int adb_track_workspace_bytes(int n_pts, size_t* ws_bytes, size_t* state_bytes) {
    ADB_REQUIRE(ws_bytes && state_bytes && n_pts >= 1 && n_pts <= TR_MAX_PTS, "adb_track_workspace_bytes: bad args");
    *ws_bytes = ws_layout(n_pts, nullptr, nullptr);
    *state_bytes = sizeof(adb_track_state);
    return ADB_OK;
}

ADB_API int adb_track_prepare(int height, int width, const float* K3x3, const long long* idx_f2k,
                              const unsigned char* valid_match_k, const float* Xff, const float* Cff, const float* Qff,
                              const float* Qkf, const float* kf_X, const float* kf_C, const int32_t* kf_N, float C_conf,
                              float Q_conf, float depth_eps, float min_match_frac, float* Xf, float* Xf_cov, float* Qk,
                              float* meas_k, unsigned char* valid_meas_k, unsigned char* valid_opt, unsigned char* valid_kf,
                              adb_track_state* state, void* ws, size_t ws_bytes, cudaStream_t stream) {
    ADB_REQUIRE(height >= 3 && width >= 3 && (long long)height * width <= TR_MAX_PTS,
                "adb_track_prepare: height and width must be >= 3 (5x5 reflect-padded box filter)");
    ADB_REQUIRE(K3x3 && idx_f2k && valid_match_k && Xff && Cff && Qff && Qkf && kf_X && kf_C && kf_N,
                "adb_track_prepare: null input pointer");
    ADB_REQUIRE(Xf && Xf_cov && Qk && meas_k && valid_meas_k && valid_opt && valid_kf && state && ws,
                "adb_track_prepare: null output pointer");
    const int n = height * width;
    TrackWs w;
    const int rc = check_ws(n, ws, ws_bytes, &w, "adb_track_prepare: workspace too small");
    if (rc != ADB_OK) return rc;
    ADB_CUDA(cudaMemsetAsync(state, 0, sizeof(adb_track_state), stream));
    ADB_CUDA(cudaMemsetAsync(w.seen, 0, ((size_t)n + 31) / 32 * 4, stream));
    track_cov_kernel<<<dim3(adb_cdiv(width, COV_TX), adb_cdiv(height, COV_TY)), dim3(COV_TX, COV_TY), 0, stream>>>(
        height, width, K3x3, Xff, w.cov_f);
    ADB_CHECK_LAUNCH("track_cov_kernel");
    PrepParams p{height, width, n, C_conf, Q_conf, depth_eps};
    track_gather_kernel<<<adb_cdiv(n, TR_THREADS), TR_THREADS, 0, stream>>>(p, K3x3, idx_f2k, valid_match_k, Xff, Cff, Qff,
                                                                          Qkf, kf_X, kf_C, kf_N, w.cov_f, w.seen, Xf, Xf_cov,
                                                                          Qk, meas_k, valid_meas_k, valid_opt, valid_kf,
                                                                          state);
    ADB_CHECK_LAUNCH("track_gather_kernel");
    track_match_check_kernel<<<1, 32, 0, stream>>>(n, min_match_frac, state);
    ADB_CHECK_LAUNCH("track_match_check_kernel");
    return ADB_OK;
}

ADB_API int adb_track_solve(int n_pts, int height, int width, const float* K3x3, const float* Xf, const float* Xf_cov,
                            const float* Qk, const unsigned char* valid, const float* meas_k,
                            const unsigned char* valid_meas_k, const float* T_WCf, const float* T_WCk, int max_iters,
                            int covariance_filter, int pixel_border, float depth_eps, float sigma_pixel, float sigma_depth,
                            float huber_k, double rel_error, float delta_norm, float* T_WCf_out, float* T_CkCf_out,
                            adb_track_state* state, void* ws, size_t ws_bytes, cudaStream_t stream) {
    ADB_REQUIRE(n_pts >= 1 && n_pts <= TR_MAX_PTS && height >= 1 && width >= 1 && max_iters >= 0,
                "adb_track_solve: bad sizes");
    ADB_REQUIRE(K3x3 && Xf && Qk && valid && meas_k && valid_meas_k && T_WCf && T_WCk && T_WCf_out && T_CkCf_out && state &&
                    ws && (Xf_cov || !covariance_filter),
                "adb_track_solve: null pointer");
    ADB_REQUIRE(sigma_pixel > 0.f && sigma_depth > 0.f && huber_k > 0.f, "adb_track_solve: sigmas and huber_k must be positive");
    TrackWs w;
    const int rc = check_ws(n_pts, ws, ws_bytes, &w, "adb_track_solve: workspace too small");
    if (rc != ADB_OK) return rc;
    SolveParams p{};
    p.n = n_pts; p.H = height; p.W = width; p.filter = covariance_filter != 0;
    p.border = (float)pixel_border;
    p.u_max = (float)(width - 1 - pixel_border);
    p.v_max = (float)(height - 1 - pixel_border);
    p.depth_eps = depth_eps;
    p.inv_sp = (float)(1.0 / (double)sigma_pixel);
    p.inv_sd = (float)(1.0 / (double)sigma_depth);
    p.huber_k = huber_k; p.rel_error = rel_error; p.delta_norm = delta_norm;
    const int nb = adb_cdiv(n_pts, TR_THREADS);
    const int n_red = nb < TR_MAX_BLOCKS ? nb : TR_MAX_BLOCKS;
    SelParams sp{0, n_pts, 0.9f, 0.0, 0.0};
    if (p.filter) ADB_CUDA(cudaMemsetAsync(w.hist_hi, 0, (size_t)HIST_BINS * 12, stream));   // hist_hi and hist_lo
    ADB_CUDA(cudaMemsetAsync(w.sel, 0, sizeof(Sel), stream));
    track_init_kernel<<<1, 32, 0, stream>>>(T_WCf, T_WCk, T_CkCf_out, state);
    ADB_CHECK_LAUNCH("track_init_kernel");
    for (int it = 0; it < max_iters; ++it) {
        if (p.filter) {
            track_det_hist_kernel<<<nb, TR_THREADS, 0, stream>>>(p, K3x3, Xf, Xf_cov, w.vals, w.hist_hi, w.sel, state);
            ADB_CHECK_LAUNCH("track_det_hist_kernel");
            track_select_hi_kernel<<<1, SEL_THREADS, 0, stream>>>(sp, w.hist_hi, w.sel, state);
            ADB_CHECK_LAUNCH("track_select_hi_kernel");
            track_hist_lo_kernel<<<nb, TR_THREADS, 0, stream>>>(n_pts, 0, w.vals, w.sel, w.hist_lo, state);
            ADB_CHECK_LAUNCH("track_hist_lo_kernel");
            track_select_lo_kernel<<<1, SEL_THREADS, 0, stream>>>(sp, w.hist_lo, w.sel, state);
            ADB_CHECK_LAUNCH("track_select_lo_kernel");
        }
        track_reduce_kernel<<<n_red, TR_THREADS, 0, stream>>>(p, K3x3, Xf, Qk, valid, meas_k, valid_meas_k, w.vals, w.partial,
                                                              state);
        ADB_CHECK_LAUNCH("track_reduce_kernel");
        track_step_kernel<<<1, TR_NSUM * STEP_SPLIT, 0, stream>>>(p, n_red, w.partial, state);
        ADB_CHECK_LAUNCH("track_step_kernel");
    }
    track_out_kernel<<<1, 32, 0, stream>>>(T_WCf_out, T_CkCf_out, state);
    ADB_CHECK_LAUNCH("track_out_kernel");
    return ADB_OK;
}

ADB_API int adb_track_finish(int height, int width, const long long* idx_f2k, const unsigned char* valid_opt,
                             const float* Xkf, const float* Ckf, float* kf_X, float* kf_C, int32_t* kf_N, int point_fusion,
                             double match_frac_thresh, float thres_keyframe, double min_displacement, double last_dist,
                             adb_track_state* state, void* ws, size_t ws_bytes, cudaStream_t stream) {
    ADB_REQUIRE(height >= 1 && width >= 1 && (long long)height * width <= TR_MAX_PTS, "adb_track_finish: bad sizes");
    ADB_REQUIRE(idx_f2k && valid_opt && state && ws, "adb_track_finish: null pointer");
    ADB_REQUIRE(!point_fusion || (Xkf && Ckf && kf_X && kf_C && kf_N), "adb_track_finish: point fusion needs Xkf, Ckf and the key frame");
    ADB_REQUIRE(thres_keyframe >= 0.f && thres_keyframe <= 1.f, "adb_track_finish: thres_keyframe must lie in [0, 1]");
    const int n = height * width;
    TrackWs w;
    const int rc = check_ws(n, ws, ws_bytes, &w, "adb_track_finish: workspace too small");
    if (rc != ADB_OK) return rc;
    const int nb = adb_cdiv(n, TR_THREADS);
    if (point_fusion) {
        track_fuse_kernel<<<nb, TR_THREADS, 0, stream>>>(n, Xkf, Ckf, kf_X, kf_C, kf_N, state);
        ADB_CHECK_LAUNCH("track_fuse_kernel");
    }
    track_keyframe_kernel<<<1, 32, 0, stream>>>(n, match_frac_thresh, last_dist, state);
    ADB_CHECK_LAUNCH("track_keyframe_kernel");
    SelParams sp{1, n, thres_keyframe, min_displacement, last_dist};
    ADB_CUDA(cudaMemsetAsync(w.hist_hi, 0, (size_t)HIST_BINS * 12, stream));
    ADB_CUDA(cudaMemsetAsync(w.sel, 0, sizeof(Sel), stream));
    track_dist_hist_kernel<<<nb, TR_THREADS, 0, stream>>>(n, width, idx_f2k, valid_opt, w.vals, w.hist_hi, state);
    ADB_CHECK_LAUNCH("track_dist_hist_kernel");
    track_select_hi_kernel<<<1, SEL_THREADS, 0, stream>>>(sp, w.hist_hi, w.sel, state);
    ADB_CHECK_LAUNCH("track_select_hi_kernel");
    track_hist_lo_kernel<<<nb, TR_THREADS, 0, stream>>>(n, 1, w.vals, w.sel, w.hist_lo, state);
    ADB_CHECK_LAUNCH("track_hist_lo_kernel");
    track_select_lo_kernel<<<1, SEL_THREADS, 0, stream>>>(sp, w.hist_lo, w.sel, state);
    ADB_CHECK_LAUNCH("track_select_lo_kernel");
    return ADB_OK;
}

// The Backend's factor graph on the device, for sm_90a: FactorGraph (VSLAM/mast3r_slam/global_opt.py) minus the solve,
// which is gn.cu's.
//
// Replaces:
//   global_opt.py:56-110   add_factors after matching: Qj / Qi, the Q_conf gate, match fractions, the edge decision and
//                          eight torch.cat's that copy the whole edge store for every new key frame
//   global_opt.py:113-136  get_unique_kf_idx / get_poses_points / prep_two_way_edges: every key frame of the graph copied
//                          to the device and re-derived on every solve, and a full copy of the edge store
//   global_opt.py:143-220  constrain_points_to_ray and update_T_WCs around the solve
//
// Design:
//  * two-way edge table: edge e is rows 2e (i, j, idx_i2j, valid_match_j, Qj) and 2e+1 (j, i, idx_j2i, valid_match_i, Qi),
//    so the first 2E rows are the arrays adb_gauss_newton reads.  The caller owns the table and grows it geometrically;
//  * gating is three launches.  fg_gate_kernel writes every candidate b to the provisional rows of edge E+b (past the
//    E edges in use, so nothing the solve reads changes) and counts valid_j, valid_i and out-of-range indices per CTA in
//    integers.  fg_decide_kernel (one CTA) sums the CTA counts in a fixed order, decides, ranks the accepted edges and
//    writes their (i, j) columns.  fg_compact_kernel moves accepted rows down over rejected ones, each thread walking
//    its pixels through the candidates in increasing order: an accepted row only moves down, onto a row already read;
//  * key-frame mirror: one launch over the rows to refresh.  A row whose (dataset_idx, N_updates) equals the stamp of
//    its last refresh returns at once; every CTA compares against the stamps of the previous launch and block 0 of a row
//    writes the new stamp to the other buffer, so no CTA can see a stamp of its own launch;
//  * poses: one gather (quat2unit, rank order) before the solve, one scatter of ranks >= pin after it.
#include <cstdint>

#include "backproject.cuh"
#include "common.cuh"
#include "artdeco_b200.h"

namespace {

constexpr int FG_THREADS = 256;
constexpr int FG_MAX_B = 1024;             // candidate edges per call: one thread of fg_decide_kernel each
constexpr int MIR_CTAS_PER_ROW = 64;       // a refreshed row is 64 CTAs striding over its pixels
constexpr long long MAX_PIXELS = 1LL << 28;

__global__ void __launch_bounds__(FG_THREADS)
fg_gate_kernel(int n, long long E, const long long* __restrict__ idx_i2j, const long long* __restrict__ idx_j2i,
               const unsigned char* __restrict__ vm_j, const unsigned char* __restrict__ vm_i, const float* __restrict__ Qii,
               const float* __restrict__ Qjj, const float* __restrict__ Qji, const float* __restrict__ Qij, float Q_conf,
               long long* __restrict__ rows_idx, unsigned char* __restrict__ rows_valid, float* __restrict__ rows_Q,
               int* __restrict__ partial) {
    __shared__ int s_cnt[3];
    if (threadIdx.x < 3) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const int b = blockIdx.y;
    const int p = blockIdx.x * FG_THREADS + threadIdx.x;
    bool vj = false, vi = false;
    int bad = 0;
    if (p < n) {
        const size_t o = (size_t)b * n + p;
        const float nan = __int_as_float(0x7fffffff);
        // Qj = sqrt(Qii[b, idx_i2j] * Qji): the key frame i's own confidence at the match, times j's in i's frame
        const long long a = __ldg(idx_i2j + o), c = __ldg(idx_j2i + o);
        const bool ok_a = a >= 0 && a < n, ok_c = c >= 0 && c < n;
        const float qj = ok_a ? __fsqrt_rn(__fmul_rn(__ldg(Qii + (size_t)b * n + a), __ldg(Qji + o))) : nan;
        const float qi = ok_c ? __fsqrt_rn(__fmul_rn(__ldg(Qjj + (size_t)b * n + c), __ldg(Qij + o))) : nan;
        vj = ok_a && __ldg(vm_j + o) != 0 && qj > Q_conf;
        vi = ok_c && __ldg(vm_i + o) != 0 && qi > Q_conf;
        bad = (int)!ok_a + (int)!ok_c;
        const size_t r0 = (size_t)(2 * (E + b)) * n + p, r1 = r0 + n;
        // the table keeps the matcher's mask, as the reference does (the solve applies Q_conf itself); a pixel whose
        // index is out of range is kept out of the solve
        rows_idx[r0] = a;
        rows_valid[r0] = ok_a && __ldg(vm_j + o) != 0;
        rows_Q[r0] = qj;
        rows_idx[r1] = c;
        rows_valid[r1] = ok_c && __ldg(vm_i + o) != 0;
        rows_Q[r1] = qi;
    }
    const unsigned bj = __ballot_sync(0xffffffffu, vj), bi = __ballot_sync(0xffffffffu, vi);
    const int bb = __reduce_add_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0) {
        if (bj) atomicAdd(&s_cnt[0], __popc(bj));
        if (bi) atomicAdd(&s_cnt[1], __popc(bi));
        if (bb) atomicAdd(&s_cnt[2], bb);
    }
    __syncthreads();
    if (threadIdx.x < 3) partial[((size_t)b * gridDim.x + blockIdx.x) * 3 + threadIdx.x] = s_cnt[threadIdx.x];
}

__global__ void __launch_bounds__(FG_MAX_B)
fg_decide_kernel(int B, int n, int n_blk, long long E, const long long* __restrict__ cand_ij, float min_match_frac,
                 int is_reloc, const int* __restrict__ partial, long long* __restrict__ rows_i, long long* __restrict__ rows_j,
                 int* __restrict__ dest, int* __restrict__ accepted, int* __restrict__ counts, int* __restrict__ n_bad) {
    __shared__ int s_ok[FG_MAX_B];
    __shared__ int s_any_invalid, s_bad;
    const int b = threadIdx.x;
    if (b == 0) { s_any_invalid = 0; s_bad = 0; }
    __syncthreads();
    if (b < B) {
        long long cj = 0, ci = 0, cb = 0;
        const int* q = partial + (size_t)b * n_blk * 3;
        for (int k = 0; k < n_blk; ++k) { cj += q[3 * k]; ci += q[3 * k + 1]; cb += q[3 * k + 2]; }
        // valid.sum() / n on CUDA: the int64 count converted to fp32, times the fp32 reciprocal of n
        const float inv_n = 1.0f / (float)n;
        const float fj = __fmul_rn((float)cj, inv_n), fi = __fmul_rn((float)ci, inv_n);
        const bool consecutive = cand_ij[2 * b] == cand_ij[2 * b + 1] - 1;
        const bool invalid = !consecutive && fminf(fj, fi) < min_match_frac;
        s_ok[b] = !invalid;
        counts[2 * b] = (int)cj;
        counts[2 * b + 1] = (int)ci;
        if (invalid) atomicOr(&s_any_invalid, 1);
        atomicAdd(&s_bad, (int)cb);
    }
    __syncthreads();
    if (b == 0 && s_bad) atomicAdd(n_bad, s_bad);
    if (b < B) {
        // strict relocalisation: one invalid edge rejects them all
        const bool ok = s_ok[b] && !(is_reloc && s_any_invalid);
        int r = 0;
        for (int k = 0; k < b; ++k) r += s_ok[k];
        accepted[b] = ok;
        dest[b] = ok ? r : -1;
        if (ok) {
            const long long i = cand_ij[2 * b], j = cand_ij[2 * b + 1];
            const long long row = 2 * (E + r);
            rows_i[row] = i;
            rows_j[row] = j;
            rows_i[row + 1] = j;
            rows_j[row + 1] = i;
        }
    }
}

__global__ void __launch_bounds__(FG_THREADS)
fg_compact_kernel(int B, int n, long long E, const int* __restrict__ dest, long long* __restrict__ rows_idx,
                  unsigned char* __restrict__ rows_valid, float* __restrict__ rows_Q) {
    const int p = blockIdx.x * FG_THREADS + threadIdx.x;
    if (p >= n) return;
    for (int b = 0; b < B; ++b) {
        const int r = dest[b];
        if (r < 0 || r == b) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const size_t src = (size_t)(2 * (E + b) + h) * n + p, dst = (size_t)(2 * (E + r) + h) * n + p;
            rows_idx[dst] = rows_idx[src];
            rows_valid[dst] = rows_valid[src];
            rows_Q[dst] = rows_Q[src];
        }
    }
}

struct MirParams {
    int mode, n, W, staged, mirror_rows;
};

// Row r of the launch: source row r (staged) or ids[r] (the frames' own tensors), mirror row ids ? ids[r] : r.
__global__ void __launch_bounds__(FG_THREADS)
fg_mirror_kernel(MirParams p, const long long* __restrict__ ids, const float* __restrict__ X, const float* __restrict__ C,
                 const int* __restrict__ N, const int* __restrict__ dataset_idx, const int* __restrict__ N_updates,
                 const int2* __restrict__ seen, int2* __restrict__ seen_next, const float* __restrict__ K,
                 float* __restrict__ Xm, float* __restrict__ Cm) {
    const int r = blockIdx.y;
    const long long d = ids ? __ldg(ids + r) : r;
    if (d < 0 || d >= p.mirror_rows) return;
    const long long s = p.staged ? r : d;
    if (seen) {
        const int2 now = make_int2(__ldg(dataset_idx + s), __ldg(N_updates + s));
        if (blockIdx.x == 0 && threadIdx.x == 0) seen_next[d] = now;
        const int2 was = seen[d];
        if (was.x == now.x && was.y == now.y) return;
    }
    float k[9];
    if (p.mode == 1) {
#pragma unroll
        for (int i = 0; i < 9; ++i) k[i] = __ldg(K + i);
    }
    // get_average_conf(): C / N with N a Python int, which CUDA evaluates as C times the fp32 reciprocal of N
    const float inv_n = 1.0f / (float)__ldg(N + s);
    const float* Xs = X + (size_t)s * p.n * 3;
    const float* Cs = C + (size_t)s * p.n;
    float* Xd = Xm + (size_t)d * p.n * 3;
    float* Cd = Cm + (size_t)d * p.n;
    for (int q = blockIdx.x * FG_THREADS + threadIdx.x; q < p.n; q += gridDim.x * FG_THREADS) {
        float P[3];
        if (p.mode == 1) {
            adb_backproject::on_ray(Xs, k, q, p.W, P);
        } else {
#pragma unroll
            for (int i = 0; i < 3; ++i) P[i] = __ldg(Xs + 3 * (size_t)q + i);
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) Xd[3 * (size_t)q + i] = P[i];
        Cd[q] = __fmul_rn(__ldg(Cs + q), inv_n);
    }
}

// pp.quat2unit: q / max(|q|, 1e-12)
__global__ void fg_pose_gather_kernel(int U, int src_rows, const long long* __restrict__ ids, const float* __restrict__ T_WC,
                                      float* __restrict__ poses) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= U) return;
    const long long s = ids ? ids[r] : r;
    float T[8];
    if (s < 0 || s >= src_rows) {
#pragma unroll
        for (int i = 0; i < 8; ++i) T[i] = __int_as_float(0x7fffffff);
    } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) T[i] = T_WC[8 * s + i];
        const float nq = fmaxf(__fsqrt_rn(T[3] * T[3] + T[4] * T[4] + T[5] * T[5] + T[6] * T[6]), 1e-12f);
#pragma unroll
        for (int i = 3; i < 7; ++i) T[i] = __fdiv_rn(T[i], nq);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) poses[8 * (size_t)r + i] = T[i];
}

__global__ void fg_pose_scatter_kernel(int U, int pin, int dst_rows, const long long* __restrict__ ids,
                                       const float* __restrict__ poses, float* __restrict__ T_WC) {
    const int r = pin + blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= U) return;
    const long long d = ids ? ids[r] : r;
    if (d < 0 || d >= dst_rows) return;
#pragma unroll
    for (int i = 0; i < 8; ++i) T_WC[8 * d + i] = poses[8 * (size_t)r + i];
}

int gate_blocks(int n) { return adb_cdiv(n, FG_THREADS); }

}  // namespace

ADB_API int adb_fg_gate_workspace_bytes(int B, int n, size_t* bytes) {
    ADB_REQUIRE(bytes, "adb_fg_gate_workspace_bytes: null pointer");
    ADB_REQUIRE(B >= 1 && B <= FG_MAX_B && n >= 1 && n <= MAX_PIXELS, "adb_fg_gate_workspace_bytes: bad size");
    *bytes = sizeof(int) * ((size_t)B * gate_blocks(n) * 3 + B);
    return ADB_OK;
}

ADB_API int adb_fg_gate(int B, int n, long long n_edges, long long capacity, const long long* cand_ij,
                        const long long* idx_i2j, const long long* idx_j2i, const unsigned char* valid_match_j,
                        const unsigned char* valid_match_i, const float* Qii, const float* Qjj, const float* Qji,
                        const float* Qij, float Q_conf, float min_match_frac, int is_reloc, long long* rows_i,
                        long long* rows_j, long long* rows_idx, unsigned char* rows_valid, float* rows_Q, int* accepted,
                        int* counts, int* n_bad, void* ws, size_t ws_bytes, cudaStream_t stream) {
    ADB_REQUIRE(B >= 1 && B <= FG_MAX_B && n >= 1 && n <= MAX_PIXELS, "adb_fg_gate: bad size");
    ADB_REQUIRE(n_edges >= 0 && capacity >= n_edges + B && capacity <= (1LL << 40) / n,
                "adb_fg_gate: bad size (the table must hold n_edges + B edges)");
    ADB_REQUIRE(cand_ij && idx_i2j && idx_j2i && valid_match_j && valid_match_i && Qii && Qjj && Qji && Qij && rows_i &&
                    rows_j && rows_idx && rows_valid && rows_Q && accepted && counts && n_bad && ws,
                "adb_fg_gate: null pointer");
    const int n_blk = gate_blocks(n);
    const size_t need = sizeof(int) * ((size_t)B * n_blk * 3 + B);
    if (ws_bytes < need) { adb_set_error_msg("adb_fg_gate: workspace too small"); return ADB_ERR_WORKSPACE; }
    int* partial = (int*)ws;
    int* dest = partial + (size_t)B * n_blk * 3;
    fg_gate_kernel<<<dim3(n_blk, B), FG_THREADS, 0, stream>>>(n, n_edges, idx_i2j, idx_j2i, valid_match_j, valid_match_i,
                                                              Qii, Qjj, Qji, Qij, Q_conf, rows_idx, rows_valid, rows_Q,
                                                              partial);
    ADB_CHECK_LAUNCH("fg_gate_kernel");
    fg_decide_kernel<<<1, FG_MAX_B, 0, stream>>>(B, n, n_blk, n_edges, cand_ij, min_match_frac, is_reloc, partial, rows_i,
                                                 rows_j, dest, accepted, counts, n_bad);
    ADB_CHECK_LAUNCH("fg_decide_kernel");
    if (B > 1) {
        fg_compact_kernel<<<n_blk, FG_THREADS, 0, stream>>>(B, n, n_edges, dest, rows_idx, rows_valid, rows_Q);
        ADB_CHECK_LAUNCH("fg_compact_kernel");
    }
    return ADB_OK;
}

ADB_API int adb_fg_mirror_refresh(int mode, int rows, int height, int width, int mirror_rows, const long long* ids,
                                  int staged, const float* X, const float* C, const int32_t* N,
                                  const int32_t* dataset_idx, const int32_t* N_updates, const int32_t* seen,
                                  int32_t* seen_next, const float* K, float* Xm, float* Cm, cudaStream_t stream) {
    ADB_REQUIRE(mode == 0 || mode == 1, "adb_fg_mirror_refresh: mode must be 0 (rays) or 1 (calib)");
    ADB_REQUIRE(height >= 1 && width >= 1 && (long long)height * width <= MAX_PIXELS && rows >= 0 && rows <= 65535 &&
                    mirror_rows >= 0,
                "adb_fg_mirror_refresh: bad size");
    ADB_REQUIRE(X && C && N && Xm && Cm && (mode == 0 || K), "adb_fg_mirror_refresh: null pointer");
    ADB_REQUIRE(!seen || (seen_next && dataset_idx && N_updates), "adb_fg_mirror_refresh: null pointer (stamps)");
    ADB_REQUIRE(staged || ids || rows <= mirror_rows, "adb_fg_mirror_refresh: more rows than the mirror holds");
    if (rows == 0) return ADB_OK;
    MirParams p{mode, height * width, width, staged ? 1 : 0, mirror_rows};
    const int gx = min(MIR_CTAS_PER_ROW, adb_cdiv(p.n, FG_THREADS));
    fg_mirror_kernel<<<dim3(gx, rows), FG_THREADS, 0, stream>>>(p, ids, X, C, N, dataset_idx, N_updates, (const int2*)seen,
                                                                (int2*)seen_next, K, Xm, Cm);
    ADB_CHECK_LAUNCH("fg_mirror_kernel");
    return ADB_OK;
}

ADB_API int adb_fg_pose_gather(int n_unique, int src_rows, const long long* ids, const float* T_WC, float* poses,
                               cudaStream_t stream) {
    ADB_REQUIRE(n_unique >= 0 && src_rows >= 0 && (ids || n_unique <= src_rows), "adb_fg_pose_gather: bad size");
    ADB_REQUIRE(T_WC && poses, "adb_fg_pose_gather: null pointer");
    if (n_unique == 0) return ADB_OK;
    fg_pose_gather_kernel<<<adb_cdiv(n_unique, 128), 128, 0, stream>>>(n_unique, src_rows, ids, T_WC, poses);
    ADB_CHECK_LAUNCH("fg_pose_gather_kernel");
    return ADB_OK;
}

ADB_API int adb_fg_pose_scatter(int n_unique, int pin, int dst_rows, const long long* ids, const float* poses, float* T_WC,
                                cudaStream_t stream) {
    ADB_REQUIRE(n_unique >= 0 && pin >= 0 && dst_rows >= 0 && (ids || n_unique <= dst_rows),
                "adb_fg_pose_scatter: bad size");
    ADB_REQUIRE(T_WC && poses, "adb_fg_pose_scatter: null pointer");
    if (n_unique <= pin) return ADB_OK;
    fg_pose_scatter_kernel<<<adb_cdiv(n_unique - pin, 128), 128, 0, stream>>>(n_unique, pin, dst_rows, ids, poses, T_WC);
    ADB_CHECK_LAUNCH("fg_pose_scatter_kernel");
    return ADB_OK;
}

// Global Gauss-Newton over Sim(3) key-frame poses: `mast3r_slam_backends.gauss_newton_rays / gauss_newton_calib`
// (VSLAM/backend/src/gn_kernels.cu:813-1230 ray_align_kernel + host loop, :1231-1637 calib_proj_kernel + host loop;
// called from VSLAM/mast3r_slam/global_opt.py:158,208).  SURVEY.md §8f rank 4.
//
// Reference flow per iteration: one kernel builds per-edge 14x14 normal-equation blocks with 119 shared-memory block
// reductions, then the blocks are copied to the HOST, assembled into an Eigen sparse matrix in double, factorised with
// SimplicialLLT, the step is copied back, a retraction kernel updates the poses and `delta_norm.item()` syncs again.
//
// Here the whole solve stays on the device and no iteration touches the host:
//   gn_edge_kernel      several CTAs per edge (the points are split so that the GPU is full).  The reference's two Jacobian halves satisfy Ji = -Jj exactly (it computes Jj by the
//                       adjoint and negates it), so the 14x14 block is [[S,-S],[-S,S]] with ONE symmetric 7x7 S: 28 + 7
//                       accumulators per thread instead of 105 + 14, reduced with warp shuffles (35 values) instead of 119
//                       block-wide shared-memory trees.
//   gn_assemble_kernel  adds the blocks into a DENSE double-precision system of the free poses (7 (K-1) unknowns; key-frame
//                       graphs have tens to a few hundred poses, so dense fits L2) — the precision the reference solves in.
//   gn_solve_kernel     one CTA: left-looking Cholesky in double, forward/back substitution, dx = -x (zeros when a pivot is
//                       not positive, as the reference returns zeros when SimplicialLLT fails).
//   gn_retract_kernel   Sim(3) retraction of every free pose (same expSim3 series as the reference), |dx| and the
//                       convergence flag on the device; once set, the kernels of later iterations return immediately.
#include "common.cuh"
#include "sim3.cuh"

namespace {

using adb_sim3::act_so3;
using adb_sim3::exp_sim3;
using adb_sim3::quat_comp;

constexpr int GN_THREADS = 256;

__device__ __forceinline__ float huber(float r) { return adb_sim3::huber(r, 1.345f); }
__device__ __forceinline__ float dot3(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// relative pose T_i^-1 T_j (gn_kernels.cu:244-265)
__device__ void rel_sim3(const float* ti, const float* qi, float si, const float* tj, const float* qj, float sj, float* tij,
                         float* qij, float* sij) {
    const float si_inv = 1.0f / si;
    *sij = si_inv * sj;
    const float qi_inv[4] = {-qi[0], -qi[1], -qi[2], qi[3]};
    quat_comp(qi_inv, qj, qij);
    float d[3] = {tj[0] - ti[0], tj[1] - ti[1], tj[2] - ti[2]};
    act_so3(qi_inv, d, tij);
    tij[0] *= si_inv; tij[1] *= si_inv; tij[2] *= si_inv;
}

// row vector times the inverse adjoint (order tau, omega, s) — gn_kernels.cu:267-290
__device__ __forceinline__ void apply_sim3_adj_inv(const float* t, const float* q, float s, const float* X, float* Y) {
    const float s_inv = 1.0f / s;
    float Ra[3];
    act_so3(q, X, Ra);
    Y[0] = s_inv * Ra[0]; Y[1] = s_inv * Ra[1]; Y[2] = s_inv * Ra[2];
    act_so3(q, X + 3, Y + 3);
    Y[3] += s_inv * (t[1] * Ra[2] - t[2] * Ra[1]);
    Y[4] += s_inv * (t[2] * Ra[0] - t[0] * Ra[2]);
    Y[5] += s_inv * (t[0] * Ra[1] - t[1] * Ra[0]);
    Y[6] = X[6] + s_inv * dot3(t, Ra);
}

struct GnParams {
    int mode;            // 0 rays, 1 calib
    float sigma_a_inv, sigma_b_inv;   // rays: 1/sigma_ray, 1/sigma_dist;  calib: 1/sigma_pixel, 1/sigma_depth
    float C_thresh, Q_thresh;
    const float* Kdev;   // calib: device pointer to the 3x3 intrinsics (row-major), read in the kernel as the reference does
    float z_eps;
    int height, width, pixel_border;
};

// S (28 lower-triangle entries, row-major n >= m) += w J J^T,  v += w e J
__device__ __forceinline__ void accumulate(float* S, float* v, const float* J, float w, float e) {
    int l = 0;
#pragma unroll
    for (int n = 0; n < 7; ++n) {
        const float wn = w * J[n];
#pragma unroll
        for (int m = 0; m <= n; ++m) S[l++] += wn * J[m];
    }
    const float we = w * e;
#pragma unroll
    for (int n = 0; n < 7; ++n) v[n] += we * J[n];
}

// poses [K,8] = t(3) q(4, xyzw) s(1); Xs [K,n,3]; Cs [K,n]; ii/jj [E] positions into the pose table; idx [E,n] int64;
// valid [E,n] bool; Q [E,n].  Writes S_out [E,28] and v_out [E,7] (the j-side; the i-side is its negative).
__global__ void __launch_bounds__(GN_THREADS)
gn_edge_kernel(GnParams p, int n_pts, const float* __restrict__ poses, const float* __restrict__ Xs,
               const float* __restrict__ Cs, const long long* __restrict__ ii, const long long* __restrict__ jj,
               const long long* __restrict__ idx, const unsigned char* __restrict__ valid_match,
               const float* __restrict__ Q, const int* __restrict__ done, float* __restrict__ S_out,
               float* __restrict__ v_out) {
    if (*done) return;
    const int e = blockIdx.x, tid = threadIdx.x;
    const int n_split = gridDim.y, part = blockIdx.y;       // an edge's points are split over gridDim.y CTAs
    const int ix = (int)ii[e], jx = (int)jj[e];
    __shared__ float ti[3], tj[3], tij[3], qi[4], qj[4], qij[4], sc[3];
    __shared__ float sRed[GN_THREADS / 32][35];
    if (tid < 3) { ti[tid] = poses[ix * 8 + tid]; tj[tid] = poses[jx * 8 + tid]; }
    if (tid < 4) { qi[tid] = poses[ix * 8 + 3 + tid]; qj[tid] = poses[jx * 8 + 3 + tid]; }
    if (tid == 0) { sc[0] = poses[ix * 8 + 7]; sc[1] = poses[jx * 8 + 7]; }
    __syncthreads();
    if (tid == 0) rel_sim3(ti, qi, sc[0], tj, qj, sc[1], tij, qij, &sc[2]);
    __syncthreads();
    const float si = sc[0], sij = sc[2];

    float S[28], v[7];
#pragma unroll
    for (int l = 0; l < 28; ++l) S[l] = 0.f;
#pragma unroll
    for (int l = 0; l < 7; ++l) v[l] = 0.f;

    const float* Xi_base = Xs + (size_t)ix * n_pts * 3;
    const float* Xj_base = Xs + (size_t)jx * n_pts * 3;
    const int chunk = (n_pts + n_split - 1) / n_split;
    const int k_end = min(n_pts, (part + 1) * chunk);
    for (int k = part * chunk + tid; k < k_end; k += GN_THREADS) {
        const bool vm = valid_match[(size_t)e * n_pts + k] != 0;
        const long long ind = vm ? idx[(size_t)e * n_pts + k] : 0;
        const float Xi[3] = {Xi_base[ind * 3], Xi_base[ind * 3 + 1], Xi_base[ind * 3 + 2]};
        const float Xj[3] = {Xj_base[(size_t)k * 3], Xj_base[(size_t)k * 3 + 1], Xj_base[(size_t)k * 3 + 2]};
        float P[3];                                   // Xj in camera i
        act_so3(qij, Xj, P);
        P[0] = P[0] * sij + tij[0]; P[1] = P[1] * sij + tij[1]; P[2] = P[2] * sij + tij[2];
        const float q = Q[(size_t)e * n_pts + k];
        const float ci = Cs[(size_t)ix * n_pts + ind], cj = Cs[(size_t)jx * n_pts + k];
        bool valid = vm & (q > p.Q_thresh) & (ci > p.C_thresh) & (cj > p.C_thresh);
        float Ji[7], Jj[7];
        if (p.mode == 0) {
            // ---- rays (gn_kernels.cu:924-1095): unit-ray difference (3) + distance difference (1) ----
            const float n2i = Xi[0] * Xi[0] + Xi[1] * Xi[1] + Xi[2] * Xi[2];
            const float n1i = sqrtf(n2i), n1i_inv = 1.0f / n1i;
            const float n2j = P[0] * P[0] + P[1] * P[1] + P[2] * P[2];
            const float n1j = sqrtf(n2j), n1j_inv = 1.0f / n1j;
            const float r[3] = {n1j_inv * P[0], n1j_inv * P[1], n1j_inv * P[2]};
            const float err[4] = {r[0] - n1i_inv * Xi[0], r[1] - n1i_inv * Xi[1], r[2] - n1i_inv * Xi[2], n1j - n1i};
            const float sw_a = valid ? p.sigma_a_inv * sqrtf(q) : 0.f, sw_b = valid ? p.sigma_b_inv * sqrtf(q) : 0.f;
            const float w[4] = {huber(sw_a * err[0]) * sw_a * sw_a, huber(sw_a * err[1]) * sw_a * sw_a,
                                huber(sw_a * err[2]) * sw_a * sw_a, huber(sw_b * err[3]) * sw_b * sw_b};
            const float n3 = n1j_inv / n2j;
            const float dxx = n1j_inv - P[0] * P[0] * n3, dyy = n1j_inv - P[1] * P[1] * n3, dzz = n1j_inv - P[2] * P[2] * n3;
            const float dxy = -P[0] * P[1] * n3, dxz = -P[0] * P[2] * n3, dyz = -P[1] * P[2] * n3;
            Ji[0] = dxx; Ji[1] = dxy; Ji[2] = dxz; Ji[3] = 0.f; Ji[4] = r[2]; Ji[5] = -r[1]; Ji[6] = 0.f;
            apply_sim3_adj_inv(ti, qi, si, Ji, Jj);
            accumulate(S, v, Jj, w[0], err[0]);
            Ji[0] = dxy; Ji[1] = dyy; Ji[2] = dyz; Ji[3] = -r[2]; Ji[4] = 0.f; Ji[5] = r[0]; Ji[6] = 0.f;
            apply_sim3_adj_inv(ti, qi, si, Ji, Jj);
            accumulate(S, v, Jj, w[1], err[1]);
            Ji[0] = dxz; Ji[1] = dyz; Ji[2] = dzz; Ji[3] = r[1]; Ji[4] = -r[0]; Ji[5] = 0.f; Ji[6] = 0.f;
            apply_sim3_adj_inv(ti, qi, si, Ji, Jj);
            accumulate(S, v, Jj, w[2], err[2]);
            Ji[0] = r[0]; Ji[1] = r[1]; Ji[2] = r[2]; Ji[3] = 0.f; Ji[4] = 0.f; Ji[5] = 0.f; Ji[6] = n1j;
            apply_sim3_adj_inv(ti, qi, si, Ji, Jj);
            accumulate(S, v, Jj, w[3], err[3]);
        } else {
            // ---- calibrated projection (gn_kernels.cu:1346-1500): pixel difference (2) + log-depth difference (1) ----
            const int u_t = (int)(ind % p.width), v_t = (int)(ind / p.width);
            const bool vz = (P[2] > p.z_eps) && (Xi[2] > p.z_eps);
            const float zj_inv = vz ? 1.0f / P[2] : 0.f, zj_log = vz ? logf(P[2]) : 0.f, zi_log = vz ? logf(Xi[2]) : 0.f;
            const float xz = P[0] * zj_inv, yz = P[1] * zj_inv;
            const float fx = p.Kdev[0], fy = p.Kdev[4], cx = p.Kdev[2], cy = p.Kdev[5];
            const float u = fx * xz + cx, vv = fy * yz + cy;
            const bool vu = (u > p.pixel_border) && (u < p.width - 1 - p.pixel_border);
            const bool vvv = (vv > p.pixel_border) && (vv < p.height - 1 - p.pixel_border);
            valid = valid & vu & vvv & vz;
            const float err[3] = {u - (float)u_t, vv - (float)v_t, zj_log - zi_log};
            const float sw_a = valid ? p.sigma_a_inv * sqrtf(q) : 0.f, sw_b = valid ? p.sigma_b_inv * sqrtf(q) : 0.f;
            const float w[3] = {huber(sw_a * err[0]) * sw_a * sw_a, huber(sw_a * err[1]) * sw_a * sw_a,
                                huber(sw_b * err[2]) * sw_b * sw_b};
            Ji[0] = fx * zj_inv; Ji[1] = 0.f; Ji[2] = -fx * xz * zj_inv; Ji[3] = -fx * xz * yz;
            Ji[4] = fx * (1.f + xz * xz); Ji[5] = -fx * yz; Ji[6] = 0.f;
            apply_sim3_adj_inv(ti, qi, si, Ji, Jj);
            accumulate(S, v, Jj, w[0], err[0]);
            Ji[0] = 0.f; Ji[1] = fy * zj_inv; Ji[2] = -fy * yz * zj_inv; Ji[3] = -fy * (1.f + yz * yz);
            Ji[4] = fy * xz * yz; Ji[5] = fy * xz; Ji[6] = 0.f;
            apply_sim3_adj_inv(ti, qi, si, Ji, Jj);
            accumulate(S, v, Jj, w[1], err[1]);
            Ji[0] = 0.f; Ji[1] = 0.f; Ji[2] = zj_inv; Ji[3] = yz; Ji[4] = -xz; Ji[5] = 0.f; Ji[6] = 1.f;
            apply_sim3_adj_inv(ti, qi, si, Ji, Jj);
            accumulate(S, v, Jj, w[2], err[2]);
        }
    }
    // 35 sums: warp shuffles, then 8 partials per value through shared memory
    const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int l = 0; l < 28; ++l) {
        const float r = adb_warp_sum(S[l]);
        if (lane == 0) sRed[warp][l] = r;
    }
#pragma unroll
    for (int l = 0; l < 7; ++l) {
        const float r = adb_warp_sum(v[l]);
        if (lane == 0) sRed[warp][28 + l] = r;
    }
    __syncthreads();
    if (tid < 35) {
        float r = 0.f;
#pragma unroll
        for (int w_ = 0; w_ < GN_THREADS / 32; ++w_) r += sRed[w_][tid];
        // S_out / v_out are zeroed per iteration; the CTAs of one edge add their partial sums
        if (tid < 28) atomicAdd(S_out + (size_t)e * 28 + tid, r);
        else atomicAdd(v_out + (size_t)e * 7 + tid - 28, r);
    }
}

// Dense system of the free poses: H [D,D], b [D], D = 7 (K - num_fix).  Block (i,i) += S, (i,j) -= S, (j,i) -= S, (j,j) += S;
// b_i -= v, b_j += v (the i-side Jacobian is the negated j-side one); rows / columns of fixed poses are dropped, exactly as
// SparseBlock::update_lhs / update_rhs skip negative indices (gn_kernels.cu:71-113).
__global__ void __launch_bounds__(64)
gn_assemble_kernel(int E, int D, int num_fix, const long long* __restrict__ ii, const long long* __restrict__ jj,
                   const float* __restrict__ S_in, const float* __restrict__ v_in, const int* __restrict__ done,
                   double* __restrict__ H, double* __restrict__ b) {
    if (*done) return;
    const int e = blockIdx.x, t = threadIdx.x;
    if (e >= E) return;
    const int io = (int)ii[e] - num_fix, jo = (int)jj[e] - num_fix;
    if (t < 49) {
        const int n = t / 7, m = t % 7;
        const int a = n >= m ? n : m, c = n >= m ? m : n;
        const double s = (double)S_in[(size_t)e * 28 + a * (a + 1) / 2 + c];
        if (io >= 0) atomicAdd(H + (size_t)(io * 7 + n) * D + io * 7 + m, s);
        if (jo >= 0) atomicAdd(H + (size_t)(jo * 7 + n) * D + jo * 7 + m, s);
        if (io >= 0 && jo >= 0) {
            atomicAdd(H + (size_t)(io * 7 + n) * D + jo * 7 + m, -s);
            atomicAdd(H + (size_t)(jo * 7 + n) * D + io * 7 + m, -s);
        }
    } else if (t < 56) {
        const int n = t - 49;
        const double vv = (double)v_in[(size_t)e * 7 + n];
        if (io >= 0) atomicAdd(b + io * 7 + n, -vv);
        if (jo >= 0) atomicAdd(b + jo * 7 + n, vv);
    }
}

// One CTA.  In-place left-looking Cholesky of H (lower triangle), then L y = b, L^T x = y, dx = -x (float).  `ok` = 0 and
// dx = 0 when a pivot is not positive (SimplicialLLT failure path, gn_kernels.cu:141-151).
__global__ void __launch_bounds__(1024)
gn_solve_kernel(int D, double* __restrict__ H, double* __restrict__ b, const int* __restrict__ done, float* __restrict__ dx,
                int* __restrict__ ok) {
    if (*done) return;
    __shared__ double s_piv;
    __shared__ int s_fail;
    const int tid = threadIdx.x, nt = blockDim.x;
    if (tid == 0) s_fail = 0;
    __syncthreads();
    for (int j = 0; j < D; ++j) {
        // row j of L (columns < j) is final; every thread needs it: read through L2 (rows are contiguous)
        const double* Lj = H + (size_t)j * D;
        if (tid == 0) {
            double s = Lj[j];
            for (int k = 0; k < j; ++k) s -= Lj[k] * Lj[k];
            if (!(s > 0.0)) s_fail = 1;
            s_piv = s > 0.0 ? sqrt(s) : 1.0;
        }
        __syncthreads();
        if (s_fail) break;
        const double piv = s_piv, inv = 1.0 / piv;
        for (int i = j + 1 + tid; i < D; i += nt) {
            double* Li = H + (size_t)i * D;
            double s = Li[j];
            for (int k = 0; k < j; ++k) s -= Li[k] * Lj[k];
            Li[j] = s * inv;
        }
        if (tid == 0) H[(size_t)j * D + j] = piv;
        __syncthreads();
    }
    if (s_fail) {
        for (int i = tid; i < D; i += nt) dx[i] = 0.f;
        if (tid == 0) *ok = 0;
        return;
    }
    // forward substitution L y = b (sequential over rows, parallel dot products are not worth it at these sizes: one warp)
    if (tid < 32) {
        for (int i = 0; i < D; ++i) {
            const double* Li = H + (size_t)i * D;
            double s = 0.0;
            for (int k = tid; k < i; k += 32) s += Li[k] * b[k];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (tid == 0) b[i] = (b[i] - s) / Li[i];
            __syncwarp();
        }
        for (int i = D - 1; i >= 0; --i) {
            double s = 0.0;
            for (int k = i + 1 + tid; k < D; k += 32) s += H[(size_t)k * D + i] * b[k];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (tid == 0) b[i] = (b[i] - s) / H[(size_t)i * D + i];
            __syncwarp();
        }
    }
    __syncthreads();
    for (int i = tid; i < D; i += nt) dx[i] = (float)(-b[i]);
    if (tid == 0) *ok = 1;
}

// poses[k] <- exp(dx[k - num_fix]) * poses[k] for k >= num_fix (gn_kernels.cu:387-452); |dx| -> *delta; sets *done when
// |dx| < delta_thresh (the update of this iteration is still applied, as in the reference loop).
__global__ void __launch_bounds__(256)
gn_retract_kernel(int K, int num_fix, float* __restrict__ poses, const float* __restrict__ dx, float delta_thresh,
                  int* __restrict__ done, float* __restrict__ delta, int* __restrict__ iters) {
    if (*done) return;
    __shared__ float sN[8];
    const int tid = threadIdx.x;
    float acc = 0.f;
    for (int k = num_fix + tid; k < K; k += blockDim.x) {
        float xi[7], t[3], q[4], t1[3], q1[4], dt[3], dq[4], ds;
        for (int n = 0; n < 7; ++n) { xi[n] = dx[(k - num_fix) * 7 + n]; acc += xi[n] * xi[n]; }
        for (int n = 0; n < 3; ++n) t[n] = poses[k * 8 + n];
        for (int n = 0; n < 4; ++n) q[n] = poses[k * 8 + 3 + n];
        const float s = poses[k * 8 + 7];
        exp_sim3(xi, dt, dq, &ds);
        quat_comp(dq, q, q1);
        act_so3(dq, t, t1);
        for (int n = 0; n < 3; ++n) poses[k * 8 + n] = t1[n] * ds + dt[n];
        for (int n = 0; n < 4; ++n) poses[k * 8 + 3 + n] = q1[n];
        poses[k * 8 + 7] = ds * s;
    }
    acc = adb_warp_sum(acc);
    if ((tid & 31) == 0) sN[tid >> 5] = acc;
    __syncthreads();
    if (tid == 0) {
        float tot = 0.f;
        for (int w_ = 0; w_ < (int)(blockDim.x >> 5); ++w_) tot += sN[w_];
        const float nrm = sqrtf(tot);
        *delta = nrm;
        *iters += 1;
        if (nrm < delta_thresh) *done = 1;
    }
}

}  // namespace

// Workspace (bytes): S [E,28] f32 + v [E,7] f32 + H [D,D] f64 + b [D] f64 + dx [D] f32 + 4 ints/floats of state.
ADB_API int adb_gn_workspace_bytes(int n_poses, int n_edges, size_t* bytes) {
    ADB_REQUIRE(bytes && n_poses >= 1 && n_edges >= 0, "adb_gn_workspace_bytes: bad args");
    const size_t D = (size_t)7 * (size_t)(n_poses - 1);
    *bytes = (size_t)n_edges * 35 * 4 + D * D * 8 + D * 8 + D * 4 + 256 + 64;
    return ADB_OK;
}

// mode 0 = gauss_newton_rays (sigma_a = sigma_ray, sigma_b = sigma_dist; K4 / image size ignored),
// mode 1 = gauss_newton_calib (sigma_a = sigma_pixel, sigma_b = sigma_depth; K4 = DEVICE pointer to the row-major 3x3 K).
// poses [K,8] are updated IN PLACE (pose 0 is fixed, num_fix = 1 as in the reference).  ii / jj: int64 [E] POSITIONS of the
// edge's key frames in the pose table.  dx_out [K-1,7] receives the last step; state_out (device, 4 x 32 bit):
// [0] iterations run, [1] converged flag, [2] last |dx| (float bits), [3] last Cholesky ok flag.  No host sync inside.
ADB_API int adb_gauss_newton(int mode, int n_poses, int n_pts, int n_edges, float* poses, const float* Xs, const float* Cs,
                             const float* K4, const long long* ii, const long long* jj, const long long* idx_ii2jj,
                             const unsigned char* valid_match, const float* Q, int height, int width, int pixel_border,
                             float z_eps, float sigma_a, float sigma_b, float C_thresh, float Q_thresh, int max_iter,
                             float delta_thresh, float* dx_out, int* state_out, void* ws, size_t ws_bytes,
                             cudaStream_t stream) {
    ADB_REQUIRE((mode == 0 || mode == 1) && n_poses >= 1 && n_pts >= 0 && n_edges >= 0 && max_iter >= 0, "adb_gauss_newton: bad sizes");
    ADB_REQUIRE(poses && dx_out && state_out && ws, "adb_gauss_newton: null pointer");
    ADB_REQUIRE(sigma_a > 0.f && sigma_b > 0.f, "adb_gauss_newton: sigmas must be positive");
    const int num_fix = 1;
    const int Kf = n_poses - num_fix, D = 7 * Kf;
    size_t need = 0;
    adb_gn_workspace_bytes(n_poses, n_edges, &need);
    if (need > ws_bytes) { adb_set_error_msg("adb_gauss_newton: workspace too small"); return ADB_ERR_WORKSPACE; }
    ADB_CUDA(cudaMemsetAsync(state_out, 0, 4 * sizeof(int), stream));
    if (D == 0 || n_edges == 0 || max_iter == 0) return ADB_OK;
    ADB_REQUIRE(Xs && Cs && ii && jj && idx_ii2jj && valid_match && Q, "adb_gauss_newton: null pointer");
    ADB_REQUIRE(mode == 0 || (K4 && height > 0 && width > 0), "adb_gauss_newton: calib mode needs K and the image size");
    unsigned char* w = (unsigned char*)ws;
    double* H = (double*)w;                          w += (size_t)D * D * 8;
    double* b = (double*)w;                          w += (size_t)D * 8;
    float* S = (float*)w;                            w += (size_t)n_edges * 28 * 4;
    float* v = (float*)w;                            w += (size_t)n_edges * 7 * 4;
    float* dx = dx_out;
    GnParams p{};
    p.mode = mode; p.sigma_a_inv = 1.0f / sigma_a; p.sigma_b_inv = 1.0f / sigma_b; p.C_thresh = C_thresh; p.Q_thresh = Q_thresh;
    p.z_eps = z_eps; p.height = height; p.width = width; p.pixel_border = pixel_border;
    int* it_p = state_out, *done_p = state_out + 1, *ok_p = state_out + 3;
    float* delta_p = (float*)(state_out + 2);
    p.Kdev = K4;
    // enough CTAs to fill the GPU: the reference launches one 256-thread CTA per edge (128 edges = 128 CTAs on 132 SMs);
    // here every edge's points are split so that about 8 CTAs per SM of an H100 are in flight
    int n_split = (132 * 8 + n_edges - 1) / n_edges;
    const int max_split = (n_pts + 4 * GN_THREADS - 1) / (4 * GN_THREADS);
    if (n_split > max_split) n_split = max_split;
    if (n_split < 1) n_split = 1;
    for (int it = 0; it < max_iter; ++it) {
        ADB_CUDA(cudaMemsetAsync(S, 0, (size_t)n_edges * 35 * 4, stream));     // S and v are contiguous
        gn_edge_kernel<<<dim3(n_edges, n_split), GN_THREADS, 0, stream>>>(p, n_pts, poses, Xs, Cs, ii, jj, idx_ii2jj,
                                                                        valid_match, Q, done_p, S, v);
        ADB_CHECK_LAUNCH("gn_edge_kernel");
        ADB_CUDA(cudaMemsetAsync(H, 0, ((size_t)D * D + D) * 8, stream));
        gn_assemble_kernel<<<n_edges, 64, 0, stream>>>(n_edges, D, num_fix, ii, jj, S, v, done_p, H, b);
        ADB_CHECK_LAUNCH("gn_assemble_kernel");
        gn_solve_kernel<<<1, 1024, 0, stream>>>(D, H, b, done_p, dx, ok_p);
        ADB_CHECK_LAUNCH("gn_solve_kernel");
        gn_retract_kernel<<<1, 256, 0, stream>>>(n_poses, num_fix, poses, dx, delta_thresh, done_p, delta_p, it_p);
        ADB_CHECK_LAUNCH("gn_retract_kernel");
    }
    return ADB_OK;
}

// Re-anchoring the map after the Backend's global Gauss-Newton has moved its Sim(3) key frames, for sm_90a.
//
// Replaces, on every SLAM key frame:
//   run_system.py:194-227                               the per-mapper-key-frame pose loop (pypose SE3 / quat2unit / mul /
//                                                       Inv / matrix, get_Rt, set_Rt and three torch.linalg.inv per frame)
//   Reconstruct/scene/scene_models/h3dgsv3.py:955-966   SceneModel.rigid_transform_gs
//   Reconstruct/utils.py:28-60                          update_gaussians (gather of two [N,4,4] tables, batched inverse, bmm,
//                                                       einsum, kornia's quaternion <-> rotation-matrix conversions)
//
// Design:
//  * adb_reanchor_keyframes: one thread per mapper key frame computes the whole loop body; no host round trip;
//  * adb_reanchor_gaussians: the reference inverts one 4x4 per Gaussian although only K distinct ones exist.  Here one
//    launch over K writes the per-frame delta new_c2w * inv(old_c2w) (3x4, plus a validity flag) to the workspace, and one
//    streaming launch over N reads id / xyz / rotation (36 B), the delta through the read-only cache (neighbouring rows
//    share a key frame) and writes xyz / rotation (28 B);
//  * closed forms exact in real arithmetic: the rigid inverse [R^T | -R^T t] for the matrices built from rotations
//    (get_Rt, the SE3 matrix and both c2w of the pose loop); the c2w tables given to adb_reanchor_gaussians can come from
//    anywhere, so that inverse is a general Gauss-Jordan elimination with partial pivoting;
//  * rows the reference would fault or raise on (an index out of range, a singular old_c2w) are left unchanged and counted
//    in a caller-zeroed device int32, never trapped.
#include <cfloat>

#include "common.cuh"
#include "mapper_pose.cuh"
#include "sim3.cuh"

namespace {

constexpr int NT_FRAMES = 128;
constexpr int NT_ROWS = 256;
constexpr int DELTA_FLOATS = 16;   // rows 0..2 of the 4x4 delta, then [12] = 1 if the frame has a delta, 0 if singular

using adb_pose::centre_of;
using adb_pose::six_d_to_R;

// out [4,4] = inverse of [R | t; 0 0 0 1] = [R^T | -R^T t; 0 0 0 1]
__device__ __forceinline__ void store_rigid_inverse(const float R[3][3], const float t[3], float* out) {
    float c[3];
    centre_of(R, t, c);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        out[4 * i + 0] = R[0][i];
        out[4 * i + 1] = R[1][i];
        out[4 * i + 2] = R[2][i];
        out[4 * i + 3] = c[i];
    }
    out[12] = 0.f; out[13] = 0.f; out[14] = 0.f; out[15] = 1.f;
}

__global__ void __launch_bounds__(NT_FRAMES)
reanchor_keyframes_kernel(int K, int K_slam, const float* __restrict__ slam_T_WC, const long long* __restrict__ last_kf,
                          const unsigned char* __restrict__ is_slam, const float* __restrict__ T_CkCf, float* rW2C,
                          float* tW2C, float* __restrict__ old_c2w, float* __restrict__ new_c2w,
                          float* __restrict__ cam_centres, float* __restrict__ approx_centres, int* __restrict__ n_bad) {
    const int k = blockIdx.x * NT_FRAMES + threadIdx.x;
    if (k >= K) return;
    float* r6 = rW2C + 6 * (size_t)k;
    float* tk = tW2C + 3 * (size_t)k;
    float R_old[3][3];
    six_d_to_R(r6, R_old);
    const float t_old[3] = {tk[0], tk[1], tk[2]};
    store_rigid_inverse(R_old, t_old, old_c2w + 16 * (size_t)k);            // torch.linalg.inv(old_Rt)
    const long long li = last_kf[k];
    if (li < 0 || li >= K_slam) {
        // keyframes[last_keyframe_index] would fault: the frame keeps its pose, so its Gaussians stay where they are
        atomicAdd(n_bad, 1);
        store_rigid_inverse(R_old, t_old, new_c2w + 16 * (size_t)k);
        float c[3];
        centre_of(R_old, t_old, c);
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            cam_centres[3 * (size_t)k + i] = c[i];
            approx_centres[3 * (size_t)k + i] = c[i];
        }
        return;
    }
    const float* A = slam_T_WC + 8 * li;
    float t[3], q[4];
    if (is_slam[k]) {
        // quat2unit(SE3(T_WC[:7]))
        t[0] = A[0]; t[1] = A[1]; t[2] = A[2];
        q[0] = A[3]; q[1] = A[4]; q[2] = A[5]; q[3] = A[6];
    } else {
        // SE3(quat2unit(T_WCk . T_CkCf)[:7]): the Sim(3) product scales the translation before the scale is dropped
        const float* B = T_CkCf + 8 * (size_t)k;
        const float qa[4] = {A[3], A[4], A[5], A[6]}, qb[4] = {B[3], B[4], B[5], B[6]}, tb[3] = {B[0], B[1], B[2]};
        float y[3];
        adb_sim3::act_so3(qa, tb, y);
#pragma unroll
        for (int i = 0; i < 3; ++i) t[i] = y[i] * A[7] + A[i];
        adb_sim3::quat_comp(qa, qb, q);
    }
    adb_pose::quat_unit(q);
    // new_Rt = T_WCf.Inv().matrix()
    float ti[3], R_new[3][3];
    adb_pose::se3_inverse_Rt(t, q, R_new, ti);
    store_rigid_inverse(R_new, ti, new_c2w + 16 * (size_t)k);               // torch.linalg.inv(new_Rt)
    // set_Rt(new_Rt)
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        r6[2 * i + 0] = R_new[i][0];
        r6[2 * i + 1] = R_new[i][1];
        tk[i] = ti[i];
    }
    float c[3];
    centre_of(R_new, ti, c);                                                 // approx_centre: new_Rt's own R
#pragma unroll
    for (int i = 0; i < 3; ++i) approx_centres[3 * (size_t)k + i] = c[i];
    // inverse(get_Rt().T)[3, :3] after set_Rt: the re-orthonormalised sixD2mtx R
    const float r_new[6] = {R_new[0][0], R_new[0][1], R_new[1][0], R_new[1][1], R_new[2][0], R_new[2][1]};
    float R_re[3][3];
    six_d_to_R(r_new, R_re);
    centre_of(R_re, ti, c);
#pragma unroll
    for (int i = 0; i < 3; ++i) cam_centres[3 * (size_t)k + i] = c[i];
}

// delta[k] = new_c2w[k] . inv(old_c2w[k]), rows 0..2; a zero pivot (torch.inverse raises) marks the frame as singular.
__global__ void __launch_bounds__(NT_FRAMES)
reanchor_delta_kernel(int K, const float* __restrict__ old_c2w, const float* __restrict__ new_c2w,
                      float* __restrict__ delta) {
    const int k = blockIdx.x * NT_FRAMES + threadIdx.x;
    if (k >= K) return;
    float a[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            a[i][j] = old_c2w[16 * (size_t)k + 4 * i + j];
            a[i][4 + j] = i == j ? 1.f : 0.f;
        }
    bool singular = false;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        // partial pivoting; every index is a compile-time constant so the matrix stays in registers
        int p = c;
        float best = fabsf(a[c][c]);
#pragma unroll
        for (int r = c + 1; r < 4; ++r)
            if (fabsf(a[r][c]) > best) { best = fabsf(a[r][c]); p = r; }
#pragma unroll
        for (int r = c + 1; r < 4; ++r)
            if (r == p)
#pragma unroll
                for (int j = 0; j < 8; ++j) { const float s = a[c][j]; a[c][j] = a[r][j]; a[r][j] = s; }
        const float piv = a[c][c];
        singular |= piv == 0.f;
        const float inv_piv = 1.f / piv;
#pragma unroll
        for (int j = 0; j < 8; ++j) a[c][j] *= inv_piv;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            if (r == c) continue;
            const float f = a[r][c];
#pragma unroll
            for (int j = 0; j < 8; ++j) a[r][j] = fmaf(-f, a[c][j], a[r][j]);
        }
    }
    float* d = delta + DELTA_FLOATS * (size_t)k;
    if (singular) {
#pragma unroll
        for (int j = 0; j < DELTA_FLOATS; ++j) d[j] = 0.f;
        return;
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        float n[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) n[j] = new_c2w[16 * (size_t)k + 4 * i + j];
#pragma unroll
        for (int j = 0; j < 4; ++j)
            d[4 * i + j] = fmaf(n[3], a[3][4 + j], fmaf(n[2], a[2][4 + j], fmaf(n[1], a[1][4 + j], n[0] * a[0][4 + j])));
    }
    d[12] = 1.f; d[13] = 0.f; d[14] = 0.f; d[15] = 0.f;
}

// kornia.geometry.conversions.quaternion_to_rotation_matrix (wxyz): F.normalize(q, eps=1e-12) first.
__device__ __forceinline__ void quat_to_R(float4 q4, float m[3][3]) {
    const float n = sqrtf(q4.x * q4.x + q4.y * q4.y + q4.z * q4.z + q4.w * q4.w);
    const float den = fmaxf(n, 1e-12f);
    const float w = q4.x / den, x = q4.y / den, y = q4.z / den, z = q4.w / den;
    const float tx = 2.f * x, ty = 2.f * y, tz = 2.f * z;
    const float twx = tx * w, twy = ty * w, twz = tz * w;
    const float txx = tx * x, txy = ty * x, txz = tz * x;
    const float tyy = ty * y, tyz = tz * y, tzz = tz * z;
    m[0][0] = 1.f - (tyy + tzz); m[0][1] = txy - twz;         m[0][2] = txz + twy;
    m[1][0] = txy + twz;         m[1][1] = 1.f - (txx + tzz); m[1][2] = tyz - twx;
    m[2][0] = txz - twy;         m[2][1] = tyz + twx;         m[2][2] = 1.f - (txx + tyy);
}

// kornia's safe_zero_division: num / clamp(den, min=FLT_MIN); clamp propagates NaN
__device__ __forceinline__ float safe_div(float num, float den) { return num / (den < FLT_MIN ? FLT_MIN : den); }

// kornia.geometry.conversions.rotation_matrix_to_quaternion (eps = 1e-8), wxyz; the branch is kornia's torch.where chain.
__device__ __forceinline__ float4 R_to_quat(const float m[3][3]) {
    const float eps = 1e-8f;
    const float m00 = m[0][0], m01 = m[0][1], m02 = m[0][2];
    const float m10 = m[1][0], m11 = m[1][1], m12 = m[1][2];
    const float m20 = m[2][0], m21 = m[2][1], m22 = m[2][2];
    const float trace = (m00 + m11) + m22;
    if (trace > 0.f) {
        const float sq = sqrtf((trace + 1.f) + eps) * 2.f;
        return make_float4(0.25f * sq, safe_div(m21 - m12, sq), safe_div(m02 - m20, sq), safe_div(m10 - m01, sq));
    }
    if ((m00 > m11) & (m00 > m22)) {
        const float sq = sqrtf((((1.f + m00) - m11) - m22) + eps) * 2.f;
        return make_float4(safe_div(m21 - m12, sq), 0.25f * sq, safe_div(m01 + m10, sq), safe_div(m02 + m20, sq));
    }
    if (m11 > m22) {
        const float sq = sqrtf((((1.f + m11) - m00) - m22) + eps) * 2.f;
        return make_float4(safe_div(m02 - m20, sq), safe_div(m01 + m10, sq), 0.25f * sq, safe_div(m12 + m21, sq));
    }
    const float sq = sqrtf((((1.f + m22) - m00) - m11) + eps) * 2.f;
    return make_float4(safe_div(m10 - m01, sq), safe_div(m02 + m20, sq), safe_div(m12 + m21, sq), 0.25f * sq);
}

__global__ void __launch_bounds__(NT_ROWS)
reanchor_gaussians_kernel(long long N, int K, const long long* __restrict__ ids, const float* __restrict__ xyz,
                          const float4* __restrict__ rot, const float4* __restrict__ delta, float* __restrict__ xyz_out,
                          float4* __restrict__ rot_out, int* __restrict__ n_bad) {
    const long long i = (long long)blockIdx.x * NT_ROWS + threadIdx.x;
    const bool live = i < N;
    bool bad = false;
    if (live) {
        const long long id = __ldg(ids + i);
        const float p[3] = {__ldg(xyz + 3 * i), __ldg(xyz + 3 * i + 1), __ldg(xyz + 3 * i + 2)};
        const float4 q = adb_ldg_stream4(rot + i);
        float4 d0 = make_float4(0.f, 0.f, 0.f, 0.f), d1 = d0, d2 = d0, d3 = d0;
        if (id >= 0 && id < K) {
            const float4* d = delta + (DELTA_FLOATS / 4) * id;
            d3 = __ldg(d + 3);
            d0 = __ldg(d);
            d1 = __ldg(d + 1);
            d2 = __ldg(d + 2);
        }
        bad = d3.x == 0.f;   // out-of-range id or singular old_c2w: the row is copied unchanged
        float o[3] = {p[0], p[1], p[2]};
        float4 qo = q;
        if (!bad) {
            const float D[3][4] = {{d0.x, d0.y, d0.z, d0.w}, {d1.x, d1.y, d1.z, d1.w}, {d2.x, d2.y, d2.z, d2.w}};
#pragma unroll
            for (int r = 0; r < 3; ++r) o[r] = fmaf(D[r][2], p[2], fmaf(D[r][1], p[1], D[r][0] * p[0])) + D[r][3];
            float m[3][3], n[3][3];
            quat_to_R(q, m);
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int c = 0; c < 3; ++c) n[r][c] = fmaf(D[r][2], m[2][c], fmaf(D[r][1], m[1][c], D[r][0] * m[0][c]));
            qo = R_to_quat(n);
        }
        xyz_out[3 * i] = o[0];
        xyz_out[3 * i + 1] = o[1];
        xyz_out[3 * i + 2] = o[2];
        rot_out[i] = qo;
    }
    const unsigned m = __ballot_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(n_bad, __popc(m));
}

}  // namespace

ADB_API int adb_reanchor_workspace_bytes(int K, size_t* bytes) {
    ADB_REQUIRE(bytes, "adb_reanchor_workspace_bytes: null bytes");
    ADB_REQUIRE(K >= 0, "adb_reanchor_workspace_bytes: K must be >= 0");
    *bytes = (size_t)K * DELTA_FLOATS * sizeof(float);
    return ADB_OK;
}

ADB_API int adb_reanchor_keyframes(int K, int K_slam, const float* slam_T_WC, const long long* last_keyframe_index,
                                   const unsigned char* is_slam_keyframe, const float* T_CkCf, float* rW2C, float* tW2C,
                                   float* old_c2w, float* new_c2w, float* cam_centres, float* approx_centres, int* n_bad,
                                   cudaStream_t stream) {
    ADB_REQUIRE(K >= 0 && K_slam >= 0, "adb_reanchor_keyframes: K and K_slam must be >= 0");
    if (K == 0) return ADB_OK;
    ADB_REQUIRE((slam_T_WC || K_slam == 0) && last_keyframe_index && is_slam_keyframe && T_CkCf && rW2C && tW2C &&
                    old_c2w && new_c2w && cam_centres && approx_centres && n_bad,
                "adb_reanchor_keyframes: null pointer");
    reanchor_keyframes_kernel<<<adb_cdiv(K, NT_FRAMES), NT_FRAMES, 0, stream>>>(
        K, K_slam, slam_T_WC, last_keyframe_index, is_slam_keyframe, T_CkCf, rW2C, tW2C, old_c2w, new_c2w, cam_centres,
        approx_centres, n_bad);
    ADB_CHECK_LAUNCH("reanchor_keyframes_kernel");
    return ADB_OK;
}

ADB_API int adb_reanchor_gaussians(long long N, int K, const long long* ids, const float* xyz, const float* rotation,
                                   const float* old_c2w, const float* new_c2w, float* xyz_out, float* rotation_out,
                                   int* n_bad, void* ws, size_t ws_bytes, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && K >= 0, "adb_reanchor_gaussians: N and K must be >= 0");
    ADB_REQUIRE(N <= 0x7fffffffLL, "adb_reanchor_gaussians: N must be < 2^31");
    if (N == 0) return ADB_OK;
    ADB_REQUIRE(ids && xyz && rotation && xyz_out && rotation_out && n_bad && (K == 0 || (old_c2w && new_c2w && ws)),
                "adb_reanchor_gaussians: null pointer");
    ADB_REQUIRE(((uintptr_t)rotation & 15) == 0 && ((uintptr_t)rotation_out & 15) == 0 && ((uintptr_t)ws & 15) == 0,
                "adb_reanchor_gaussians: rotation, rotation_out and ws must be 16-byte aligned");
    if (ws_bytes < (size_t)K * DELTA_FLOATS * sizeof(float)) {
        adb_set_error_msg("adb_reanchor_gaussians: workspace too small");
        return ADB_ERR_WORKSPACE;
    }
    if (K > 0) {
        reanchor_delta_kernel<<<adb_cdiv(K, NT_FRAMES), NT_FRAMES, 0, stream>>>(K, old_c2w, new_c2w, (float*)ws);
        ADB_CHECK_LAUNCH("reanchor_delta_kernel");
    }
    reanchor_gaussians_kernel<<<(unsigned)((N + NT_ROWS - 1) / NT_ROWS), NT_ROWS, 0, stream>>>(
        N, K, ids, xyz, (const float4*)rotation, (const float4*)ws, xyz_out, (float4*)rotation_out, n_bad);
    ADB_CHECK_LAUNCH("reanchor_gaussians_kernel");
    return ADB_OK;
}

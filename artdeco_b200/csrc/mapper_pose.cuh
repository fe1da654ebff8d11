// Mapper key-frame pose helpers shared by the map re-anchoring (reanchor.cu) and the key-frame hand-off (keyframe.cu).
// A mapper key frame stores its world-to-camera pose as the 6-D rotation rW2C [3,2] and tW2C [3] (Reconstruct/scene/keyframe.py).
#pragma once
#include <cuda_runtime.h>

#include "sim3.cuh"

namespace adb_pose {

// sixD2mtx (Reconstruct/utils.py:223-229) of r [3,2] row-major: columns b1, b2, b3 = b1 x b2.
__device__ __forceinline__ void six_d_to_R(const float* r, float R[3][3]) {
    float b1[3] = {r[0], r[2], r[4]};
    const float c[3] = {r[1], r[3], r[5]};
    const float n1 = sqrtf(b1[0] * b1[0] + b1[1] * b1[1] + b1[2] * b1[2]);
#pragma unroll
    for (int i = 0; i < 3; ++i) b1[i] = b1[i] / n1;
    const float d = b1[0] * c[0] + b1[1] * c[1] + b1[2] * c[2];
    float b2[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) b2[i] = c[i] - d * b1[i];
    const float n2 = sqrtf(b2[0] * b2[0] + b2[1] * b2[1] + b2[2] * b2[2]);
#pragma unroll
    for (int i = 0; i < 3; ++i) b2[i] = b2[i] / n2;
    const float b3[3] = {b1[1] * b2[2] - b1[2] * b2[1], b1[2] * b2[0] - b1[0] * b2[2], b1[0] * b2[1] - b1[1] * b2[0]};
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        R[i][0] = b1[i];
        R[i][1] = b2[i];
        R[i][2] = b3[i];
    }
}

// c = -R^T t
__device__ __forceinline__ void centre_of(const float R[3][3], const float t[3], float c[3]) {
#pragma unroll
    for (int j = 0; j < 3; ++j) c[j] = -(R[0][j] * t[0] + R[1][j] * t[1] + R[2][j] * t[2]);
}

// pypose's quat2unit: q / max(|q|, 1e-12)
__device__ __forceinline__ void quat_unit(float q[4]) {
    const float n = fmaxf(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
#pragma unroll
    for (int i = 0; i < 4; ++i) q[i] = q[i] / n;
}

// SE3(t, q).Inv().matrix() for a unit q (xyzw): q^-1 = conj(q), t^-1 = -(q^-1 t), columns of R = q^-1 e_c.
__device__ __forceinline__ void se3_inverse_Rt(const float t[3], const float q[4], float R[3][3], float ti[3]) {
    const float qi[4] = {-q[0], -q[1], -q[2], q[3]};
    adb_sim3::act_so3(qi, t, ti);
    ti[0] = -ti[0]; ti[1] = -ti[1]; ti[2] = -ti[2];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float e[3] = {c == 0 ? 1.f : 0.f, c == 1 ? 1.f : 0.f, c == 2 ? 1.f : 0.f};
        float col[3];
        adb_sim3::act_so3(qi, e, col);
        R[0][c] = col[0]; R[1][c] = col[1]; R[2][c] = col[2];
    }
}

}  // namespace adb_pose

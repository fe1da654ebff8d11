// Sim(3) device helpers shared by the global Gauss-Newton (gn.cu) and the frame tracker (track.cu).
// Poses are stored as (t[3], q[4] xyzw, s); tangent vectors as [tau(3), phi(3), sigma].
#pragma once
#include <cuda_runtime.h>

namespace adb_sim3 {

constexpr float EPS = 1e-6f;

// Huber weight of a whitened residual: 1 inside k, k/|r| outside.
__device__ __forceinline__ float huber(float r, float k) {
    const float a = fabsf(r);
    return a < k ? 1.0f : k / a;
}
__device__ __forceinline__ void quat_comp(const float* qi, const float* qj, float* out) {
    out[0] = qi[3] * qj[0] + qi[0] * qj[3] + qi[1] * qj[2] - qi[2] * qj[1];
    out[1] = qi[3] * qj[1] - qi[0] * qj[2] + qi[1] * qj[3] + qi[2] * qj[0];
    out[2] = qi[3] * qj[2] + qi[0] * qj[1] - qi[1] * qj[0] + qi[2] * qj[3];
    out[3] = qi[3] * qj[3] - qi[0] * qj[0] - qi[1] * qj[1] - qi[2] * qj[2];
}
__device__ __forceinline__ void act_so3(const float* q, const float* X, float* Y) {
    float uv[3];
    uv[0] = 2.0f * (q[1] * X[2] - q[2] * X[1]);
    uv[1] = 2.0f * (q[2] * X[0] - q[0] * X[2]);
    uv[2] = 2.0f * (q[0] * X[1] - q[1] * X[0]);
    const float y0 = X[0] + q[3] * uv[0] + (q[1] * uv[2] - q[2] * uv[1]);
    const float y1 = X[1] + q[3] * uv[1] + (q[2] * uv[0] - q[0] * uv[2]);
    const float y2 = X[2] + q[3] * uv[2] + (q[0] * uv[1] - q[1] * uv[0]);
    Y[0] = y0; Y[1] = y1; Y[2] = y2;
}

__device__ __forceinline__ void exp_so3(const float* phi, float* q) {
    const float th2 = phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2];
    float imag, real;
    if (th2 < EPS) {
        const float th4 = th2 * th2;
        imag = 0.5f - (1.0f / 48.0f) * th2 + (1.0f / 3840.0f) * th4;
        real = 1.0f - (1.0f / 8.0f) * th2 + (1.0f / 384.0f) * th4;
    } else {
        const float th = sqrtf(th2);
        imag = sinf(0.5f * th) / th;
        real = cosf(0.5f * th);
    }
    q[0] = imag * phi[0]; q[1] = imag * phi[1]; q[2] = imag * phi[2]; q[3] = real;
}
__device__ __forceinline__ void cross_inplace(const float* a, float* b) {
    const float x0 = a[1] * b[2] - a[2] * b[1], x1 = a[2] * b[0] - a[0] * b[2], x2 = a[0] * b[1] - a[1] * b[0];
    b[0] = x0; b[1] = x1; b[2] = x2;
}
// Exp of sim(3): t = W(phi, sigma) tau, q = exp(phi), s = e^sigma (lietorch's closed form with its small-angle and
// small-sigma branches; VSLAM/backend/src/gn_kernels.cu:316-385).  pypose's sim3.Exp is the same map.
__device__ __forceinline__ void exp_sim3(const float* xi, float* t, float* q, float* s) {
    float tau[3] = {xi[0], xi[1], xi[2]};
    const float phi[3] = {xi[3], xi[4], xi[5]};
    const float sigma = xi[6];
    const float scale = expf(sigma);
    exp_so3(phi, q);
    *s = scale;
    const float th2 = phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2];
    const float th = sqrtf(th2);
    float A, B, C;
    if (fabsf(sigma) < EPS) {
        C = 1.0f;
        if (fabsf(th) < EPS) { A = 0.5f; B = 1.0f / 6.0f; }
        else { A = (1.0f - cosf(th)) / th2; B = (th - sinf(th)) / (th2 * th); }
    } else {
        C = (scale - 1.0f) / sigma;
        if (fabsf(th) < EPS) {
            const float s2 = sigma * sigma;
            A = ((sigma - 1.0f) * scale + 1.0f) / s2;
            B = (scale * 0.5f * s2 + scale - 1.0f - sigma * scale) / (s2 * sigma);
        } else {
            const float a = scale * sinf(th), b = scale * cosf(th), c = th2 + sigma * sigma;
            A = (a * sigma + (1.0f - b) * th) / (th * c);
            B = (C - ((b - 1.0f) * sigma + a * th) / c) / th2;
        }
    }
    t[0] = C * tau[0]; t[1] = C * tau[1]; t[2] = C * tau[2];
    cross_inplace(phi, tau);
    t[0] += A * tau[0]; t[1] += A * tau[1]; t[2] += A * tau[2];
    cross_inplace(phi, tau);
    t[0] += B * tau[0]; t[1] += B * tau[1]; t[2] += B * tau[2];
}

}  // namespace adb_sim3

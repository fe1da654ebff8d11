// Pixel back-projection shared by the frame tracker (track.cu), the key-frame hand-off (keyframe.cu) and the factor graph
// (factor_graph.cu): backproject / constrain_points_to_ray (VSLAM/mast3r_slam/geometry.py:38-43,116-124), the point at
// depth z on the ray through pixel (u, v).  Each operation rounds once, in the reference's order: (u - cx) / fx, then
// times z.
#pragma once
#include <cuda_runtime.h>

namespace adb_backproject {

__device__ __forceinline__ void ray_point(float u, float v, float z, float fx, float fy, float cx, float cy, float P[3]) {
    P[0] = __fmul_rn(z, __fdiv_rn(__fsub_rn(u, cx), fx));
    P[1] = __fmul_rn(z, __fdiv_rn(__fsub_rn(v, cy), fy));
    P[2] = z;
}

// constrain_points_to_ray of pixel p of a width-W image whose point map X is [HW,3]; K row-major [3,3]
__device__ __forceinline__ void on_ray(const float* __restrict__ X, const float* k, long long p, int W, float P[3]) {
    ray_point((float)(p % W), (float)(p / W), __ldg(X + 3 * (size_t)p + 2), k[0], k[4], k[2], k[5], P);
}

}  // namespace adb_backproject

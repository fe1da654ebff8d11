// Resampling arithmetic as PyTorch's CUDA kernels evaluate it, shared by the densification (densify.cu) and the key-frame
// hand-off (keyframe.cu).
#pragma once
#include <cuda_runtime.h>

namespace adb_resample {

// upsample_bilinear2d (align_corners=True) source index: (index, neighbour offset, lambda)
__device__ __forceinline__ void lin_src(float scale, int dst, int in_size, int* i0, int* ip, float* l1) {
    const float r = scale * (float)dst;
    const int i = (int)r;
    *i0 = i;
    *ip = (i < in_size - 1) ? 1 : 0;
    *l1 = r - (float)i;
}

// upsample_bilinear2d's blend of the four taps a (i0, j0), b (i0, j0 + jp), c (i0 + ip, j0), d (i0 + ip, j0 + jp)
__device__ __forceinline__ float blend4(float h0l, float h1l, float w0l, float w1l, float a, float b, float c, float d) {
    return h0l * (w0l * a + w1l * b) + h1l * (w0l * c + w1l * d);
}

// avg_pool2d(x, 2) of one window: the sum in window order (0,0), (0,1), (1,0), (1,1) from 0, then / 4
__device__ __forceinline__ float pool4(float a, float b, float c, float d) {
    float s = 0.f;
    s = __fadd_rn(s, a);
    s = __fadd_rn(s, b);
    s = __fadd_rn(s, c);
    s = __fadd_rn(s, d);
    return s / 4.0f;
}

}  // namespace adb_resample

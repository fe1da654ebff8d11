// Sparse (visibility-masked) Adam without bias correction, in place.
//
// Replaces diff_gaussian_rasterization.adamUpdate / adamUpdateBasic (on-the-fly-nvs fork, un-vendored; the
// contract is pinned by the call sites Reconstruct/scene/optimizers.py:48-57, 90-99, 116-128, 144-156 and
// SURVEY.md App. B.8):   m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;  p -= lr * m / (sqrt(v) + eps)
// rows with visible[row] == 0 are skipped entirely (moments untouched).  `lr` is a DEVICE tensor of numel 1, N
// or N*M (optimizers.py:71-73,185-192; h3dgsv3.py:1241-1247) or, when lr_dev is NULL, the host scalar lr_scalar
// (adamUpdateBasic gets a Python float, optimizers.py:41).
// HBM-bound: 16 B read + 12 B written per visible element; rows are processed as float4 when M % 4 == 0.
#include "common.cuh"

namespace {

__device__ __forceinline__ void adam1(float& p, float g, float& m, float& v, float lr, float b1, float b2, float eps) {
    m = b1 * m + (1.0f - b1) * g;
    v = b2 * v + (1.0f - b2) * g * g;
    p -= lr * m / (sqrtf(v) + eps);
}

// lr_mode: 0 scalar (host), 1 device numel 1, 2 per row, 3 per element
// DECAY (lr_mode 3 only): after the update the element's own learning rate becomes max(lr * lr_decay, lr_min) -- the
// per-primitive schedule SparseGaussianAdam.step applies with `lr[visibility] *= decay; lr.clamp_min_(0.1 lr_init)`
// (optimizers.py:130-133,158-161), fused so the lr tensor is read and written in the same pass.
template <int VEC, bool DECAY>
__global__ void __launch_bounds__(256)
adam_kernel(long long N, long long M, float* __restrict__ param, const float* __restrict__ grad,
            float* __restrict__ m1, float* __restrict__ m2, const unsigned char* __restrict__ visible,
            const float* lr_dev, int lr_mode, float lr_scalar, float b1, float b2, float eps,
            float* lr_mut, float lr_decay, float lr_min) {
    const long long total = N * M / VEC;
    const long long mv = M / VEC;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / mv;
        if (visible && !visible[row]) continue;
        float lr = lr_scalar;
        if (lr_mode == 1) lr = __ldg(lr_dev);
        else if (lr_mode == 2) lr = __ldg(lr_dev + row);
        if (VEC == 4) {
            float4 p = reinterpret_cast<float4*>(param)[i];
            const float4 g = reinterpret_cast<const float4*>(grad)[i];
            float4 a = reinterpret_cast<float4*>(m1)[i];
            float4 v = reinterpret_cast<float4*>(m2)[i];
            float4 l = make_float4(lr, lr, lr, lr);
            if (lr_mode == 3) l = reinterpret_cast<const float4*>(lr_dev)[i];
            adam1(p.x, g.x, a.x, v.x, l.x, b1, b2, eps);
            adam1(p.y, g.y, a.y, v.y, l.y, b1, b2, eps);
            adam1(p.z, g.z, a.z, v.z, l.z, b1, b2, eps);
            adam1(p.w, g.w, a.w, v.w, l.w, b1, b2, eps);
            reinterpret_cast<float4*>(param)[i] = p;
            reinterpret_cast<float4*>(m1)[i] = a;
            reinterpret_cast<float4*>(m2)[i] = v;
            if (DECAY)
                reinterpret_cast<float4*>(lr_mut)[i] = make_float4(fmaxf(l.x * lr_decay, lr_min), fmaxf(l.y * lr_decay, lr_min),
                                                                   fmaxf(l.z * lr_decay, lr_min), fmaxf(l.w * lr_decay, lr_min));
        } else {
            if (lr_mode == 3) lr = lr_dev[i];
            float p = param[i], a = m1[i], v = m2[i];
            adam1(p, grad[i], a, v, lr, b1, b2, eps);
            param[i] = p; m1[i] = a; m2[i] = v;
            if (DECAY) lr_mut[i] = fmaxf(lr * lr_decay, lr_min);
        }
    }
}

}  // namespace

// param/grad/m1/m2: [N, M] fp32.  visible: uint8/bool [N] or NULL (all rows).  lr_dev: NULL (use lr_scalar) or a
// device tensor with lr_numel in {1, N, N*M}.
ADB_API int adb_adam_update(long long N, long long M, float* param, const float* grad, float* m1, float* m2,
                            const unsigned char* visible, const float* lr_dev, long long lr_numel, float lr_scalar,
                            float b1, float b2, float eps, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && M >= 0, "adb_adam_update: negative size");
    if (N * M == 0) return ADB_OK;
    ADB_REQUIRE(param && grad && m1 && m2, "adb_adam_update: null pointer");
    int lr_mode = 0;
    if (lr_dev) {
        if (lr_numel == 1) lr_mode = 1;
        else if (lr_numel == N) lr_mode = 2;       // (N == N*M only when M == 1: per-row == per-element)
        else if (lr_numel == N * M) lr_mode = 3;
        else { adb_set_error_msg("adb_adam_update: lr numel must be 1, N or N*M"); return ADB_ERR_INVALID; }
    }
    const bool vec = (M % 4 == 0) && ((((uintptr_t)param | (uintptr_t)grad | (uintptr_t)m1 | (uintptr_t)m2 |
                                        (uintptr_t)lr_dev) & 15) == 0);
    const long long work = vec ? N * M / 4 : N * M;
    const int blocks = (int)((work + 255) / 256 < 132LL * 16 ? (work + 255) / 256 : 132LL * 16);
    if (vec)
        adam_kernel<4, false><<<blocks, 256, 0, stream>>>(N, M, param, grad, m1, m2, visible, lr_dev, lr_mode, lr_scalar,
                                                         b1, b2, eps, nullptr, 1.f, 0.f);
    else
        adam_kernel<1, false><<<blocks, 256, 0, stream>>>(N, M, param, grad, m1, m2, visible, lr_dev, lr_mode, lr_scalar,
                                                         b1, b2, eps, nullptr, 1.f, 0.f);
    ADB_CHECK_LAUNCH("adam_kernel");
    return ADB_OK;
}

// Adam step + per-element learning-rate decay in one pass.  lr [N,M] (same shape as param) is read, used, and overwritten
// with max(lr * lr_decay, lr_min) on visible rows (optimizers.py:116-133,144-161).
ADB_API int adb_adam_update_decay(long long N, long long M, float* param, const float* grad, float* m1, float* m2,
                                  const unsigned char* visible, float* lr, float b1, float b2, float eps,
                                  float lr_decay, float lr_min, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && M >= 0, "adb_adam_update_decay: negative size");
    if (N * M == 0) return ADB_OK;
    ADB_REQUIRE(param && grad && m1 && m2 && lr, "adb_adam_update_decay: null pointer");
    const bool vec = (M % 4 == 0) && ((((uintptr_t)param | (uintptr_t)grad | (uintptr_t)m1 | (uintptr_t)m2 |
                                        (uintptr_t)lr) & 15) == 0);
    const long long work = vec ? N * M / 4 : N * M;
    const int blocks = (int)((work + 255) / 256 < 132LL * 16 ? (work + 255) / 256 : 132LL * 16);
    if (vec)
        adam_kernel<4, true><<<blocks, 256, 0, stream>>>(N, M, param, grad, m1, m2, visible, lr, 3, 0.f, b1, b2, eps, lr,
                                                        lr_decay, lr_min);
    else
        adam_kernel<1, true><<<blocks, 256, 0, stream>>>(N, M, param, grad, m1, m2, visible, lr, 3, 0.f, b1, b2, eps, lr,
                                                        lr_decay, lr_min);
    ADB_CHECK_LAUNCH("adam_kernel<decay>");
    return ADB_OK;
}

// LoD d_max cull: fused distance test + selection mask + alpha ratio + stream compaction of the selected ids.
//
// Replaces the ~12 full-N0 torch kernels of SceneModel.render's cull
// (Reconstruct/scene/scene_models/h3dgsv3.py:626-645) and the per-keyframe count of weed_out_gaussians (:942-953):
//   dist = ||xyz - cam||;  selected = dist < 2*d_max;
//   alpha_ratio = (2*d_max - dist)/d_max  where d_max < dist < 2*d_max, else 1.
// One streaming pass over 16 B/Gaussian (xyz + d_max) writes mask (1 B), ratio (4 B) and, through a
// decoupled-look-back select, the ascending list of selected ids — the order boolean-mask indexing produces.
#include "common.cuh"
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

namespace {

__global__ void __launch_bounds__(256)
lod_mask_kernel(long long N, const float* __restrict__ xyz, const float* __restrict__ d_max,
                const float* __restrict__ cam, unsigned char* __restrict__ mask, float* __restrict__ ratio) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const float dx = xyz[3 * i] - cam[0], dy = xyz[3 * i + 1] - cam[1], dz = xyz[3 * i + 2] - cam[2];
    const float dist = sqrtf(dx * dx + dy * dy + dz * dz);
    const float d = d_max[i];
    const bool sel = dist < 2.0f * d;
    const bool fade = dist > d && sel;
    mask[i] = sel ? 1 : 0;
    if (ratio) ratio[i] = fade ? (2.0f * d - dist) / d : 1.0f;
}

// weed_out_gaussians (h3dgsv3.py:942-953): the reference loops over every key frame in Python and streams all N rows once per
// key frame (K x ~6 torch kernels).  Here one pass over the 16 B/Gaussian counts the key frames that see each Gaussian
// (camera centres staged in shared memory) and applies the keep rule  count / K > visible_threshold  in fp32 as torch does
// on the device: an int tensor over a Python int is count * fl32(1 / K), which differs from a correctly rounded division at
// some counts (K = 500, count = 5 at threshold 0.01: the reference keeps that Gaussian).
constexpr int WEED_MAX_CAMS_SMEM = 1024;
__global__ void __launch_bounds__(256)
weed_out_kernel(long long N, const float* __restrict__ xyz, const float* __restrict__ d_max, int K,
                const float* __restrict__ cams, float visible_threshold, int32_t* __restrict__ visible_count,
                unsigned char* __restrict__ keep) {
    __shared__ float sCam[WEED_MAX_CAMS_SMEM * 3];
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    float x = 0.f, y = 0.f, z = 0.f, two_d = 0.f;
    if (i < N) { x = xyz[3 * i]; y = xyz[3 * i + 1]; z = xyz[3 * i + 2]; two_d = 2.0f * d_max[i]; }
    int cnt = 0;
    for (int k0 = 0; k0 < K; k0 += WEED_MAX_CAMS_SMEM) {
        const int kn = min(WEED_MAX_CAMS_SMEM, K - k0);
        __syncthreads();
        for (int t = threadIdx.x; t < kn * 3; t += blockDim.x) sCam[t] = cams[(size_t)k0 * 3 + t];
        __syncthreads();
        for (int k = 0; k < kn; ++k) {
            const float dx = x - sCam[3 * k], dy = y - sCam[3 * k + 1], dz = z - sCam[3 * k + 2];
            cnt += (sqrtf(dx * dx + dy * dy + dz * dz) < two_d) ? 1 : 0;
        }
    }
    if (i < N) {
        if (visible_count) visible_count[i] = cnt;
        keep[i] = (__fmul_rn((float)cnt, __fdiv_rn(1.0f, (float)K)) > visible_threshold) ? 1 : 0;
    }
}

}  // namespace

// xyz [N,3], d_max [N], cams [K,3] (device) -> keep [N] uint8/bool = (count/K > visible_threshold), visible_count [N] int32
// (may be NULL).  Replaces the per-key-frame Python loop of weed_out_gaussians (h3dgsv3.py:942-953).
ADB_API int adb_lod_weed_out(long long N, const float* xyz, const float* d_max, int K, const float* cams,
                             float visible_threshold, int32_t* visible_count, unsigned char* keep, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && K >= 1, "adb_lod_weed_out: bad sizes");
    if (N == 0) return ADB_OK;
    ADB_REQUIRE(xyz && d_max && cams && keep, "adb_lod_weed_out: null pointer");
    weed_out_kernel<<<adb_cdiv(N, 256), 256, 0, stream>>>(N, xyz, d_max, K, cams, visible_threshold, visible_count, keep);
    ADB_CHECK_LAUNCH("weed_out_kernel");
    return ADB_OK;
}

ADB_API int adb_lod_select_workspace_bytes(long long N, size_t* bytes) {
    ADB_REQUIRE(bytes && N >= 0 && N < 2147483647LL, "adb_lod_select_workspace_bytes: bad args");
    size_t b = 0;
    cub::CountingInputIterator<int32_t> ids(0);
    ADB_CUDA(cub::DeviceSelect::Flagged(nullptr, b, ids, (const unsigned char*)nullptr, (int32_t*)nullptr,
                                        (int32_t*)nullptr, (int)N));
    *bytes = b + 256;
    return ADB_OK;
}

// mask [N] (uint8 / torch.bool), ratio [N] (may be NULL), ids [N] capacity (first *count valid, ascending),
// count: DEVICE int32.  cam: DEVICE float[3].
ADB_API int adb_lod_select(long long N, const float* xyz, const float* d_max, const float* cam,
                           unsigned char* mask, float* ratio, int32_t* ids, int32_t* count, void* ws,
                           size_t ws_bytes, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && N < 2147483647LL, "adb_lod_select: bad N");
    ADB_REQUIRE(count, "adb_lod_select: null count");
    if (N == 0) { ADB_CUDA(cudaMemsetAsync(count, 0, sizeof(int32_t), stream)); return ADB_OK; }
    ADB_REQUIRE(xyz && d_max && cam && mask && ids && ws, "adb_lod_select: null pointer");
    lod_mask_kernel<<<adb_cdiv(N, 256), 256, 0, stream>>>(N, xyz, d_max, cam, mask, ratio);
    ADB_CHECK_LAUNCH("lod_mask_kernel");
    cub::CountingInputIterator<int32_t> it(0);
    size_t need = 0;
    ADB_CUDA(cub::DeviceSelect::Flagged(nullptr, need, it, mask, ids, count, (int)N));
    if (need > ws_bytes) { adb_set_error_msg("adb_lod_select: workspace too small"); return ADB_ERR_WORKSPACE; }
    ADB_CUDA(cub::DeviceSelect::Flagged(ws, need, it, mask, ids, count, (int)N, stream));
    return ADB_OK;
}

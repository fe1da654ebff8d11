// Densification bookkeeping of SparseGaussianAdam.add_and_prune (Reconstruct/scene/optimizers.py:163-219; SURVEY.md §8a R6,
// §8f rank 3): every per-Gaussian tensor -- each parameter, both Adam moments and the per-element learning rates -- becomes
// cat(t[valid_mask], extension).  The reference does this tensor by tensor with boolean indexing (a nonzero + host sync +
// gather each), a torch.cat and a .contiguous(): ~25 syncs and ~60 copy kernels per key frame, 3-4 passes over all state.
// Here: ONE plan (stream compaction of the row indices, a single count read back) and ONE gather launch for all tensors:
//   out[r] = src[src_of[r]]            r <  n_keep
//          = ext[r - n_keep] | fill    r >= n_keep          (fill: 0 for the moments, lr_init for learning rates)
// Rows are moved as 32-bit words (every state tensor is fp32 or int64), reads are row-contiguous, writes fully coalesced.
#include "common.cuh"
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#define ADB_COMPACT_MAX_TENSORS 32

namespace {

struct CompactTable {
    const uint32_t* src[ADB_COMPACT_MAX_TENSORS];
    uint32_t* dst[ADB_COMPACT_MAX_TENSORS];
    const uint32_t* ext[ADB_COMPACT_MAX_TENSORS];
    int row_words[ADB_COMPACT_MAX_TENSORS];
    uint32_t fill[ADB_COMPACT_MAX_TENSORS];
};

__global__ void __launch_bounds__(256)
compact_gather_kernel(long long n_keep, long long n_ext, const int32_t* __restrict__ src_of,
                      const __grid_constant__ CompactTable tab) {
    const int t = blockIdx.y;
    const int rw = tab.row_words[t];
    const long long total = (n_keep + n_ext) * rw;
    const uint32_t* __restrict__ src = tab.src[t];
    const uint32_t* __restrict__ ext = tab.ext[t];
    uint32_t* __restrict__ dst = tab.dst[t];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / rw;
        const int w = (int)(i - r * rw);
        uint32_t v;
        if (r < n_keep) v = __ldg(src + (long long)__ldg(src_of + r) * rw + w);
        else v = ext ? __ldg(ext + (r - n_keep) * rw + w) : tab.fill[t];
        dst[i] = v;
    }
}

}  // namespace

ADB_API int adb_compact_workspace_bytes(long long N, size_t* bytes) {
    ADB_REQUIRE(bytes && N >= 0 && N < 2147483647LL, "adb_compact_workspace_bytes: bad args");
    size_t b = 0;
    cub::CountingInputIterator<int32_t> it(0);
    ADB_CUDA(cub::DeviceSelect::Flagged(nullptr, b, it, (const unsigned char*)nullptr, (int32_t*)nullptr, (int32_t*)nullptr,
                                        (int)N));
    *bytes = b + 256;
    return ADB_OK;
}

// src_of[0..n_keep) = indices i with mask[i] != 0, ascending (the order boolean indexing keeps); *n_keep_dev = their count.
ADB_API int adb_compact_plan(long long N, const unsigned char* mask, int32_t* src_of, int32_t* n_keep_dev, void* ws,
                             size_t ws_bytes, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && N < 2147483647LL, "adb_compact_plan: bad N");
    ADB_REQUIRE(n_keep_dev, "adb_compact_plan: null pointer");
    if (N == 0) { ADB_CUDA(cudaMemsetAsync(n_keep_dev, 0, sizeof(int32_t), stream)); return ADB_OK; }
    ADB_REQUIRE(mask && src_of && ws, "adb_compact_plan: null pointer");
    cub::CountingInputIterator<int32_t> it(0);
    size_t need = 0;
    ADB_CUDA(cub::DeviceSelect::Flagged(nullptr, need, it, mask, src_of, n_keep_dev, (int)N));
    if (need > ws_bytes) { adb_set_error_msg("adb_compact_plan: workspace too small"); return ADB_ERR_WORKSPACE; }
    ADB_CUDA(cub::DeviceSelect::Flagged(ws, need, it, mask, src_of, n_keep_dev, (int)N, stream));
    return ADB_OK;
}

// All arrays are HOST arrays of n_tensors entries.  srcs[t]: [N, row_words[t]] words; dsts[t]: [n_keep+n_ext, row_words[t]];
// exts[t]: [n_ext, row_words[t]] or NULL (then the tail rows are filled with fill_words[t]).
ADB_API int adb_compact_gather(long long n_keep, long long n_ext, const int32_t* src_of, int n_tensors,
                               const void* const* srcs, void* const* dsts, const void* const* exts, const int* row_words,
                               const unsigned* fill_words, cudaStream_t stream) {
    ADB_REQUIRE(n_keep >= 0 && n_ext >= 0 && n_tensors >= 0, "adb_compact_gather: bad sizes");
    ADB_REQUIRE(n_tensors <= ADB_COMPACT_MAX_TENSORS, "adb_compact_gather: at most 32 tensors per call");
    if (n_tensors == 0 || n_keep + n_ext == 0) return ADB_OK;
    ADB_REQUIRE(srcs && dsts && exts && row_words && fill_words && (src_of || n_keep == 0), "adb_compact_gather: null pointer");
    CompactTable tab;
    long long max_words = 0;
    for (int t = 0; t < n_tensors; ++t) {
        ADB_REQUIRE(dsts[t] && (srcs[t] || n_keep == 0) && row_words[t] > 0, "adb_compact_gather: bad tensor entry");
        tab.src[t] = (const uint32_t*)srcs[t];
        tab.dst[t] = (uint32_t*)dsts[t];
        tab.ext[t] = (const uint32_t*)exts[t];
        tab.row_words[t] = row_words[t];
        tab.fill[t] = fill_words[t];
        const long long wds = (n_keep + n_ext) * row_words[t];
        if (wds > max_words) max_words = wds;
    }
    long long bx = (max_words + 255) / 256;
    if (bx > 132LL * 8) bx = 132LL * 8;
    dim3 grid((unsigned)bx, n_tensors);
    compact_gather_kernel<<<grid, 256, 0, stream>>>(n_keep, n_ext, src_of, tab);
    ADB_CHECK_LAUNCH("compact_gather_kernel");
    return ADB_OK;
}

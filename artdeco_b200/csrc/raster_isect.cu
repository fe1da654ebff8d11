// Tile intersection: scan of per-Gaussian tile counts, (key,value) emission, radix sort, tile ranges.
// Integer / byte work with a BIT-EXACT contract against the oracle (SURVEY.md §8a R2c-R2e, App. B.3):
//   key = (cam << (32+tile_bits)) | (tile << 32) | float_bits(depth),  val = cam*N + gaussian,
//   emission order: Gaussian-major, then ty outer / tx inner; stable ascending sort over the live bits only.
// Replaces gsplat's isect_tiles / radix sort / isect_offset_encode that the reference reaches through
// Reconstruct/scene/scene_models/h3dgsv3.py:664-680.
//
// Compiled with -fmad=false like raster_project.cu would not matter here (only /16, floor, ceil) but the tile
// bound arithmetic below must stay textually identical to project_fwd_kernel's count.
#include "raster_common.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

namespace {

struct ToI64 {
    __host__ __device__ __forceinline__ int64_t operator()(const int32_t& v) const { return (int64_t)v; }
};

__global__ void __launch_bounds__(256)
isect_emit_kernel(int N, const int32_t* __restrict__ radii, const float* __restrict__ splats,
                  const int64_t* __restrict__ cum_tiles, int W, int H, int cam_id, int tile_bits, int convention,
                  int64_t* __restrict__ keys, int32_t* __restrict__ vals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int2 r = reinterpret_cast<const int2*>(radii)[i];
    if (r.x <= 0 && r.y <= 0) return;
    const float4 rec0 = reinterpret_cast<const float4*>(splats + (size_t)i * ADB_SPLAT_STRIDE)[0];
    const float depth = splats[(size_t)i * ADB_SPLAT_STRIDE + 11];
    const int tw = (W + ADB_TILE - 1) / ADB_TILE;
    int x0, x1, y0, y1;
    adb_tile_rect(rec0.x, rec0.y, r.x, r.y, W, H, convention, x0, x1, y0, y1);
    int64_t o = (i == 0) ? 0 : cum_tiles[i - 1];
    if (convention != ADB_CONV_GSPLAT && cum_tiles[i] == o) return;  // kept its radius but was given no tiles
    const uint64_t hi = (uint64_t)cam_id << (32 + tile_bits);
    const uint64_t dbits = (uint64_t)__float_as_uint(depth);
    const int32_t val = cam_id * N + i;
    for (int ty = y0; ty < y1; ++ty)
        for (int tx = x0; tx < x1; ++tx) {
            uint64_t tile = (uint64_t)(ty * tw + tx);
            keys[o] = (int64_t)(hi | (tile << 32) | dbits);
            vals[o] = val;
            ++o;
        }
}

// offsets[t] = first sorted index whose tile id >= t; offsets[T] = n.
__global__ void __launch_bounds__(256)
tile_offsets_kernel(int64_t n, const int64_t* __restrict__ keys, int tile_bits, int T, int32_t* __restrict__ offsets) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t mask = ((uint64_t)1 << tile_bits) - 1;
    if (n == 0) {
        if (i <= T) offsets[i] = 0;
        return;
    }
    if (i >= n) return;
    const int cur = (int)((((uint64_t)keys[i]) >> 32) & mask);
    if (i == 0) {
        for (int t = 0; t <= cur; ++t) offsets[t] = 0;
    } else {
        const int prev = (int)((((uint64_t)keys[i - 1]) >> 32) & mask);
        for (int t = prev + 1; t <= cur; ++t) offsets[t] = (int32_t)i;
    }
    if (i == n - 1)
        for (int t = cur + 1; t <= T; ++t) offsets[t] = (int32_t)n;
}

}  // namespace

ADB_API int adb_raster_scan_workspace_bytes(int N, size_t* bytes) {
    ADB_REQUIRE(bytes && N >= 0, "adb_raster_scan_workspace_bytes: bad args");
    size_t b = 0;
    cub::TransformInputIterator<int64_t, ToI64, const int32_t*> it((const int32_t*)nullptr, ToI64());
    ADB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, b, it, (int64_t*)nullptr, N));
    *bytes = b + 256;
    return ADB_OK;
}

// cum_tiles[i] = sum_{j<=i} tiles_per_gauss[j]  (int64).  The caller reads cum_tiles[N-1] to size keys/vals.
ADB_API int adb_raster_isect_scan(int N, const int32_t* tiles_per_gauss, int64_t* cum_tiles, void* ws,
                                  size_t ws_bytes, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0, "adb_raster_isect_scan: bad N");
    if (N == 0) return ADB_OK;
    ADB_REQUIRE(tiles_per_gauss && cum_tiles && ws, "adb_raster_isect_scan: null pointer");
    cub::TransformInputIterator<int64_t, ToI64, const int32_t*> it(tiles_per_gauss, ToI64());
    size_t need = 0;
    ADB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, need, it, cum_tiles, N));
    if (need > ws_bytes) { adb_set_error_msg("adb_raster_isect_scan: workspace too small"); return ADB_ERR_WORKSPACE; }
    ADB_CUDA(cub::DeviceScan::InclusiveSum(ws, need, it, cum_tiles, N, stream));
    return ADB_OK;
}

static int isect_emit_impl(int convention, int N, const int32_t* radii, const float* splats, const int64_t* cum_tiles,
                           int W, int H, int cam_id, int n_cams, int64_t* keys, int32_t* vals, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && W > 0 && H > 0 && cam_id >= 0 && n_cams > cam_id, "adb_raster_isect_emit: bad sizes");
    if (N == 0) return ADB_OK;
    ADB_REQUIRE(radii && splats && cum_tiles && keys && vals, "adb_raster_isect_emit: null pointer");
    isect_emit_kernel<<<adb_cdiv(N, 256), 256, 0, stream>>>(N, radii, splats, cum_tiles, W, H, cam_id,
                                                           adb_tile_bits(W, H), convention, keys, vals);
    ADB_CHECK_LAUNCH("isect_emit_kernel");
    return ADB_OK;
}

ADB_API int adb_raster_isect_emit(int N, const int32_t* radii, const float* splats, const int64_t* cum_tiles,
                                  int W, int H, int cam_id, int n_cams, int64_t* keys, int32_t* vals,
                                  cudaStream_t stream) {
    return isect_emit_impl(ADB_CONV_GSPLAT, N, radii, splats, cum_tiles, W, H, cam_id, n_cams, keys, vals, stream);
}

// Legacy (Inria) tile rectangle; everything else (key layout, emission order) as above.
ADB_API int adb_raster_isect_emit_legacy(int N, const int32_t* radii, const float* splats, const int64_t* cum_tiles,
                                         int W, int H, int cam_id, int n_cams, int64_t* keys, int32_t* vals,
                                         cudaStream_t stream) {
    return isect_emit_impl(ADB_CONV_INRIA, N, radii, splats, cum_tiles, W, H, cam_id, n_cams, keys, vals, stream);
}

ADB_API int adb_raster_sort_workspace_bytes(long long n_isect, size_t* bytes) {
    ADB_REQUIRE(bytes && n_isect >= 0, "adb_raster_sort_workspace_bytes: bad args");
    size_t b = 0;
    cub::DoubleBuffer<int64_t> dk(nullptr, nullptr);
    cub::DoubleBuffer<int32_t> dv(nullptr, nullptr);
    ADB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b, dk, dv, (int64_t)n_isect, 0, 64));
    *bytes = b + 256;
    return ADB_OK;
}

// Stable ascending sort over the live key bits.  keys_a/vals_a hold the input; the sorted result lands in
// whichever buffer pair *sorted_in_b reports (0 -> a, 1 -> b); both pairs must hold n_isect elements.
ADB_API int adb_raster_sort(long long n_isect, int W, int H, int n_cams, int64_t* keys_a, int32_t* vals_a,
                            int64_t* keys_b, int32_t* vals_b, void* ws, size_t ws_bytes, int* sorted_in_b,
                            cudaStream_t stream) {
    ADB_REQUIRE(n_isect >= 0 && sorted_in_b, "adb_raster_sort: bad args");
    *sorted_in_b = 0;
    if (n_isect == 0) return ADB_OK;
    ADB_REQUIRE(keys_a && vals_a && keys_b && vals_b && ws, "adb_raster_sort: null pointer");
    const int end_bit = 32 + adb_tile_bits(W, H) + adb_cam_bits(n_cams);
    cub::DoubleBuffer<int64_t> dk(keys_a, keys_b);
    cub::DoubleBuffer<int32_t> dv(vals_a, vals_b);
    size_t need = 0;
    ADB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, need, dk, dv, (int64_t)n_isect, 0, end_bit));
    if (need > ws_bytes) { adb_set_error_msg("adb_raster_sort: workspace too small"); return ADB_ERR_WORKSPACE; }
    ADB_CUDA(cub::DeviceRadixSort::SortPairs(ws, need, dk, dv, (int64_t)n_isect, 0, end_bit, stream));
    *sorted_in_b = (dk.Current() == keys_b) ? 1 : 0;
    return ADB_OK;
}

// tile_offsets has T+1 entries (T = ceil(W/16)*ceil(H/16)); entry T is n_isect.
ADB_API int adb_raster_tile_offsets(long long n_isect, const int64_t* keys_sorted, int W, int H,
                                    int32_t* tile_offsets, cudaStream_t stream) {
    ADB_REQUIRE(n_isect >= 0 && W > 0 && H > 0 && tile_offsets, "adb_raster_tile_offsets: bad args");
    ADB_REQUIRE(n_isect < 2147483647LL, "adb_raster_tile_offsets: more than 2^31 intersections");
    const int T = adb_cdiv(W, ADB_TILE) * adb_cdiv(H, ADB_TILE);
    long long threads = n_isect > 0 ? n_isect : (long long)T + 1;
    tile_offsets_kernel<<<adb_cdiv(threads, 256), 256, 0, stream>>>(n_isect, keys_sorted, adb_tile_bits(W, H), T,
                                                                   tile_offsets);
    ADB_CHECK_LAUNCH("tile_offsets_kernel");
    return ADB_OK;
}


// =====================================================================================================================
// Tile-bucketed intersection (round 2): no library sort, no host sync, bit-identical output.
//
//   count    per Gaussian: one RED.ADD per touched tile into tile_counts[tile][copy]            (16 B read / Gaussian)
//   scan     one CTA: exclusive scan of the T x COPIES counters -> per-(tile,copy) segment starts + tile_offsets[T+1]
//            (clamped to the caller's capacity; the true total and an overflow flag stay on the device)
//   scatter  per Gaussian: slot = start[tile][copy] + atomicSub(counter) - 1 -> packed[slot] = depth_bits<<32 | gaussian
//            (arbitrary order inside a tile; the counters return to zero, so the buffer needs no memset between calls;
//            four atomics are in flight per thread before the first dependent store)
//   sort     one CTA per tile: bitonic sort of the tile's 64-bit words — the 64-element sub-networks run in REGISTERS with
//            warp shuffles, only the wider exchanges go through shared memory (global memory for tiles beyond 4096
//            entries) — then keys = cam|tile|depth_bits and vals = cam*N + gaussian are written out.
//
// COPIES = 4 replicas of every tile counter (selected by CTA index) cut the same-address serialisation of the L2 atomics
// that a single counter per tile suffers.
//
// Why the order equals the reference's stable radix sort of (tile, depth): the reference emits keys Gaussian-major, so
// inside one (tile, depth) tie the stable sort leaves ascending Gaussian ids — exactly the ascending order of the
// composite word (depth_bits, gaussian).  A Gaussian touches a tile at most once, so the words of a tile are distinct
// and the result does not depend on the scatter order.  (SURVEY.md App. B.3; oracle: adbo_isect_sort.)
// The global 45-bit onesweep radix sort this replaces moved 6 x 24 B per intersection and was 12.6 % of the round-1 step.
namespace {

constexpr int COPIES = ADB_TILE_COUNTER_COPIES;
static_assert(COPIES == 4, "the scan kernel reads one tile's counters as an int4");

__global__ void __launch_bounds__(256)
tile_count_kernel(int N, const int32_t* __restrict__ radii, const float* __restrict__ splats,
                  const int32_t* __restrict__ tiles_per_gauss, int W, int H, int convention,
                  int32_t* __restrict__ tile_counts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    if (tiles_per_gauss[i] <= 0) return;
    const int2 r = reinterpret_cast<const int2*>(radii)[i];
    const float2 m = reinterpret_cast<const float2*>(splats + (size_t)i * ADB_SPLAT_STRIDE)[0];
    const int tw = (W + ADB_TILE - 1) / ADB_TILE;
    const int cp = blockIdx.x & (COPIES - 1);
    int x0, x1, y0, y1;
    adb_tile_rect(m.x, m.y, r.x, r.y, W, H, convention, x0, x1, y0, y1);
    for (int ty = y0; ty < y1; ++ty)
        for (int tx = x0; tx < x1; ++tx) atomicAdd(tile_counts + (ty * tw + tx) * COPIES + cp, 1);
}

// Single CTA, 1024 threads, over the T*COPIES counters in (tile-major, copy-minor) order.
// starts[e] = min(capacity, sum_{f<e} counts[f]);  offsets[t] = starts[t*COPIES];  offsets[T] = min(capacity, total).
// Each thread owns 16 consecutive counters (4 tiles x 4 copies): four 128-bit loads in flight, one block-wide scan of the
// per-thread sums per 16384 counters (1080p: two rounds; the first version looped 8 times with
// four barriers each and took 20 us).
constexpr int SCAN_THREADS = 1024;
__global__ void __launch_bounds__(SCAN_THREADS)
tile_scan_kernel(int T, const int32_t* __restrict__ counts, long long capacity, int32_t* __restrict__ starts,
                 int32_t* __restrict__ offsets, long long* __restrict__ total, int32_t* __restrict__ overflow) {
    constexpr int PER = 16;                                  // 1024 threads x 16 counters = 16384 per round, no spills
    __shared__ long long s_warp[32];
    __shared__ long long s_carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int E = T * COPIES;
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < E; base += SCAN_THREADS * PER) {
        const int e0 = base + tid * PER;
        int c[PER];
#pragma unroll
        for (int v = 0; v < PER / 4; ++v) {
            int4 q = make_int4(0, 0, 0, 0);
            const int e = e0 + 4 * v;                       // E is a multiple of 4 and e a multiple of 4: all-or-nothing
            if (e < E) q = *reinterpret_cast<const int4*>(counts + e);
            c[4 * v] = q.x; c[4 * v + 1] = q.y; c[4 * v + 2] = q.z; c[4 * v + 3] = q.w;
        }
        long long mine = 0;
#pragma unroll
        for (int v = 0; v < PER; ++v) mine += c[v];
        long long x = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) s_warp[warp] = x;
        __syncthreads();
        if (warp == 0) {
            long long w = lane < SCAN_THREADS / 32 ? s_warp[lane] : 0;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const long long y = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += y;
            }
            s_warp[lane] = w;   // inclusive over warps
        }
        __syncthreads();
        const long long carry = s_carry;
        long long excl = carry + (warp ? s_warp[warp - 1] : 0) + x - mine;
#pragma unroll
        for (int v = 0; v < PER / 4; ++v) {
            const int e = e0 + 4 * v;
            int4 st;
            st.x = (int32_t)(excl < capacity ? excl : capacity); excl += c[4 * v];
            st.y = (int32_t)(excl < capacity ? excl : capacity); excl += c[4 * v + 1];
            st.z = (int32_t)(excl < capacity ? excl : capacity); excl += c[4 * v + 2];
            st.w = (int32_t)(excl < capacity ? excl : capacity); excl += c[4 * v + 3];
            if (e < E) {
                *reinterpret_cast<int4*>(starts + e) = st;
                offsets[e / COPIES] = st.x;
            }
        }
        __syncthreads();
        if (tid == SCAN_THREADS - 1) s_carry = carry + s_warp[SCAN_THREADS / 32 - 1];
        __syncthreads();
    }
    if (tid == 0) {
        const long long tot = s_carry;
        offsets[T] = (int32_t)(tot < capacity ? tot : capacity);
        if (total) *total = tot;
        if (overflow && tot > capacity) *overflow = 1;
    }
}

__global__ void __launch_bounds__(256)
tile_scatter_kernel(int N, const int32_t* __restrict__ radii, const float* __restrict__ splats,
                    const int32_t* __restrict__ tiles_per_gauss, int W, int H, int convention,
                    const int32_t* __restrict__ starts, int32_t* __restrict__ tile_counts, long long capacity,
                    unsigned long long* __restrict__ packed) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    if (tiles_per_gauss[i] <= 0) return;
    const int2 r = reinterpret_cast<const int2*>(radii)[i];
    const float2 m = reinterpret_cast<const float2*>(splats + (size_t)i * ADB_SPLAT_STRIDE)[0];
    const float depth = splats[(size_t)i * ADB_SPLAT_STRIDE + 11];
    const int tw = (W + ADB_TILE - 1) / ADB_TILE;
    const int cp = blockIdx.x & (COPIES - 1);
    int x0, x1, y0, y1;
    adb_tile_rect(m.x, m.y, r.x, r.y, W, H, convention, x0, x1, y0, y1);
    const unsigned long long word = ((unsigned long long)__float_as_uint(depth) << 32) | (unsigned)i;
    int tx = x0, ty = y0;
    while (ty < y1) {
        int e[4], a[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {                       // up to four atomics in flight
            e[u] = -1;
            if (ty < y1) {
                e[u] = (ty * tw + tx) * COPIES + cp;
                a[u] = atomicSub(tile_counts + e[u], 1);
                if (++tx == x1) { tx = x0; ++ty; }
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (e[u] >= 0) {
                const long long slot = (long long)starts[e[u]] + (a[u] - 1);
                if (slot < capacity) packed[slot] = word;
            }
    }
}

constexpr int SORT_THREADS = 256;
constexpr int SORT_SMEM_CAP = 4096;    // words sorted in shared memory (32 KB); larger tiles sort in place in global memory
typedef unsigned long long u64;

__device__ __forceinline__ void ce_keep(u64& mine, u64 other, bool keep_min) {
    const bool lt = other < mine;
    mine = (lt == keep_min) ? other : mine;
}

// Bitonic network on one 64-element chunk held by a warp: lane holds positions `lane` (e0) and `lane + 32` (e1).
// Runs the merge levels [lk_first .. 6] when `full`, else only the disperse steps j = 32..1 (tail of a wider merge).
__device__ __forceinline__ void chunk_network(u64& e0, u64& e1, int lane, bool full) {
    if (full) {
#pragma unroll
        for (int lk = 1; lk <= 5; ++lk) {                   // blocks of k = 2^lk <= 32: both halves independently
            const int k = 1 << lk;
            {   // flip: p <-> p ^ (k-1); the lower position keeps the minimum
                const bool low = (lane & (k >> 1)) == 0;
                const u64 y0 = __shfl_xor_sync(0xffffffffu, e0, k - 1), y1 = __shfl_xor_sync(0xffffffffu, e1, k - 1);
                ce_keep(e0, y0, low);
                ce_keep(e1, y1, low);
            }
#pragma unroll
            for (int j = k >> 2; j > 0; j >>= 1) {          // disperse: p <-> p ^ j
                const bool low = (lane & j) == 0;
                const u64 y0 = __shfl_xor_sync(0xffffffffu, e0, j), y1 = __shfl_xor_sync(0xffffffffu, e1, j);
                ce_keep(e0, y0, low);
                ce_keep(e1, y1, low);
            }
        }
        {   // k = 64 flip: position p (e0 of lane p) <-> 63 - p (e1 of lane 31 - p)
            const u64 y = __shfl_sync(0xffffffffu, e1, 31 - lane), z = __shfl_sync(0xffffffffu, e0, 31 - lane);
            ce_keep(e0, y, true);
            ce_keep(e1, z, false);
        }
#pragma unroll
        for (int j = 16; j > 0; j >>= 1) {
            const bool low = (lane & j) == 0;
            const u64 y0 = __shfl_xor_sync(0xffffffffu, e0, j), y1 = __shfl_xor_sync(0xffffffffu, e1, j);
            ce_keep(e0, y0, low);
            ce_keep(e1, y1, low);
        }
    } else {
        {   // j = 32: positions lane and lane + 32 live in the same lane
            const u64 lo = e0 < e1 ? e0 : e1, hi = e0 < e1 ? e1 : e0;
            e0 = lo; e1 = hi;
        }
#pragma unroll
        for (int j = 16; j > 0; j >>= 1) {
            const bool low = (lane & j) == 0;
            const u64 y0 = __shfl_xor_sync(0xffffffffu, e0, j), y1 = __shfl_xor_sync(0xffffffffu, e1, j);
            ce_keep(e0, y0, low);
            ce_keep(e1, y1, low);
        }
    }
}

// Sorts a[0..np2) ascending (np2 a power of two >= 64, padded with ~0 by the caller).  All compare-exchanges ascending
// ("flip" then "disperse" steps).  Exchanges at distance >= 64 go through `a` (shared memory); everything inside aligned
// 64-element chunks runs in registers.
__device__ __forceinline__ void bitonic_sort_shared(u64* a, int np2, int tid) {
    const int lane = tid & 31, warp = tid >> 5, nwarp = SORT_THREADS / 32;
    const int nchunk = np2 >> 6, pairs = np2 >> 1;
    for (int c = warp; c < nchunk; c += nwarp) {            // levels k = 2..64 of every chunk
        u64 e0 = a[c * 64 + lane], e1 = a[c * 64 + 32 + lane];
        chunk_network(e0, e1, lane, true);
        a[c * 64 + lane] = e0; a[c * 64 + 32 + lane] = e1;
    }
    __syncthreads();
    for (int lk = 7; (1 << lk) <= np2; ++lk) {
        const int lh = lk - 1, h = 1 << lh, k = 1 << lk;
        for (int q = tid; q < pairs; q += SORT_THREADS) {  // flip across the block of k
            const int r = q & (h - 1), base = (q >> lh) << lk;
            const int i = base + r, p = base + (k - 1 - r);
            const u64 x = a[i], y = a[p];
            if (x > y) { a[i] = y; a[p] = x; }
        }
        __syncthreads();
        for (int lj = lh - 1; lj >= 6; --lj) {              // disperse at distance j >= 64
            const int j = 1 << lj;
            for (int q = tid; q < pairs; q += SORT_THREADS) {
                const int r = q & (j - 1);
                const int i = ((q >> lj) << (lj + 1)) + r, p = i + j;
                const u64 x = a[i], y = a[p];
                if (x > y) { a[i] = y; a[p] = x; }
            }
            __syncthreads();
        }
        for (int c = warp; c < nchunk; c += nwarp) {        // disperse j = 32..1 inside every chunk
            u64 e0 = a[c * 64 + lane], e1 = a[c * 64 + 32 + lane];
            chunk_network(e0, e1, lane, false);
            a[c * 64 + lane] = e0; a[c * 64 + 32 + lane] = e1;
        }
        __syncthreads();
    }
}

// Fallback for tiles beyond the shared-memory capacity: same network, operands in global memory, any n (indices >= n
// behave as +inf and are skipped).
__device__ __forceinline__ void bitonic_sort_global(volatile u64* a, int n, int tid) {
    int lg = 0;
    while ((1 << lg) < n) ++lg;
    const int pairs = (1 << lg) >> 1;
    for (int lk = 1; lk <= lg; ++lk) {
        const int lh = lk - 1, h = 1 << lh, k = 1 << lk;
        for (int q = tid; q < pairs; q += SORT_THREADS) {
            const int r = q & (h - 1), base = (q >> lh) << lk;
            const int i = base + r, p = base + (k - 1 - r);
            if (p < n) {
                const u64 x = a[i], y = a[p];
                if (x > y) { a[i] = y; a[p] = x; }
            }
        }
        __syncthreads();
        for (int lj = lh - 1; lj >= 0; --lj) {
            const int j = 1 << lj;
            for (int q = tid; q < pairs; q += SORT_THREADS) {
                const int r = q & (j - 1);
                const int i = ((q >> lj) << (lj + 1)) + r, p = i + j;
                if (p < n) {
                    const u64 x = a[i], y = a[p];
                    if (x > y) { a[i] = y; a[p] = x; }
                }
            }
            __syncthreads();
        }
    }
}

__global__ void __launch_bounds__(SORT_THREADS)
tile_sort_kernel(int T, const int32_t* __restrict__ offsets, u64* __restrict__ packed, int cam_id,
                 int n_per_cam, int tile_bits, int64_t* __restrict__ keys, int32_t* __restrict__ vals) {
    __shared__ u64 s_words[SORT_SMEM_CAP];
    const int tile = blockIdx.x;
    const int start = offsets[tile], n = offsets[tile + 1] - start;
    if (n <= 0) return;
    const int tid = threadIdx.x;
    u64* g = packed + start;
    const u64 hi = ((u64)cam_id << (32 + tile_bits)) | ((u64)tile << 32);
    const int vbase = cam_id * n_per_cam;
    if (n <= SORT_SMEM_CAP) {
        int np2 = 64;
        while (np2 < n) np2 <<= 1;
        for (int i = tid; i < np2; i += SORT_THREADS) s_words[i] = i < n ? g[i] : ~0ull;
        __syncthreads();
        if (n > 1) bitonic_sort_shared(s_words, np2, tid);
        for (int i = tid; i < n; i += SORT_THREADS) {
            const u64 w = s_words[i];
            keys[start + i] = (int64_t)(hi | (w >> 32));
            vals[start + i] = vbase + (int32_t)(unsigned)(w & 0xffffffffu);
        }
    } else {
        // rare: a tile with more than SORT_SMEM_CAP splats (L2-resident operands)
        __syncthreads();
        bitonic_sort_global((volatile u64*)g, n, tid);
        __threadfence_block();
        for (int i = tid; i < n; i += SORT_THREADS) {
            const u64 w = g[i];
            keys[start + i] = (int64_t)(hi | (w >> 32));
            vals[start + i] = vbase + (int32_t)(unsigned)(w & 0xffffffffu);
        }
    }
}

}  // namespace

// tile_counts: int32 [2 * ADB_TILE_COUNTER_COPIES * T]: first half = the per-(tile,copy) counters, which must be all-zero
// on entry (they are zero again after adb_raster_tile_scatter_sort: allocate + zero once); second half = segment starts
// written by the scan.  tile_offsets [T+1]; total (int64, device) and overflow (int32, device, only ever SET) may be null.
// `capacity` = number of elements `packed`, `keys` and `vals` can hold; intersections beyond it are dropped (memory-safe)
// and flagged.
static int tile_bucket_impl(int convention, int N, const int32_t* radii, const float* splats,
                            const int32_t* tiles_per_gauss, int W, int H, long long capacity, int32_t* tile_counts,
                            int32_t* tile_offsets, long long* total, int32_t* overflow, int counts_ready, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && W > 0 && H > 0 && capacity >= 0 && capacity < 2147483647LL, "adb_raster_tile_count_scan: bad sizes");
    ADB_REQUIRE(tile_counts && tile_offsets, "adb_raster_tile_count_scan: null pointer");
    const int T = adb_cdiv(W, ADB_TILE) * adb_cdiv(H, ADB_TILE);
    if (N > 0 && !counts_ready) {
        ADB_REQUIRE(radii && splats && tiles_per_gauss, "adb_raster_tile_count_scan: null pointer");
        tile_count_kernel<<<adb_cdiv(N, 256), 256, 0, stream>>>(N, radii, splats, tiles_per_gauss, W, H, convention,
                                                               tile_counts);
        ADB_CHECK_LAUNCH("tile_count_kernel");
    }
    tile_scan_kernel<<<1, SCAN_THREADS, 0, stream>>>(T, tile_counts, capacity, tile_counts + (size_t)T * COPIES, tile_offsets, total,
                                            overflow);
    ADB_CHECK_LAUNCH("tile_scan_kernel");
    return ADB_OK;
}

ADB_API int adb_raster_tile_count_scan(int N, const int32_t* radii, const float* splats, const int32_t* tiles_per_gauss,
                                       int W, int H, int legacy, long long capacity, int32_t* tile_counts,
                                       int32_t* tile_offsets, long long* total, int32_t* overflow, cudaStream_t stream) {
    return tile_bucket_impl(legacy ? ADB_CONV_INRIA : ADB_CONV_GSPLAT, N, radii, splats, tiles_per_gauss, W, H, capacity,
                            tile_counts, tile_offsets, total, overflow, 0, stream);
}

// Scan only: the counters were filled by adb_raster_project_fwd_counts.
ADB_API int adb_raster_tile_scan(int W, int H, long long capacity, int32_t* tile_counts, int32_t* tile_offsets,
                                 long long* total, int32_t* overflow, cudaStream_t stream) {
    return tile_bucket_impl(ADB_CONV_GSPLAT, 0, nullptr, nullptr, nullptr, W, H, capacity, tile_counts, tile_offsets, total,
                            overflow, 1, stream);
}

// Scatter + per-tile sort.  keys [capacity] int64, vals [capacity] int32, packed [capacity] uint64 scratch; tile_counts as
// left by adb_raster_tile_count_scan.
ADB_API int adb_raster_tile_scatter_sort(int N, const int32_t* radii, const float* splats, const int32_t* tiles_per_gauss,
                                         int W, int H, int legacy, int cam_id, int n_cams, long long capacity,
                                         int32_t* tile_counts, const int32_t* tile_offsets, void* packed, int64_t* keys,
                                         int32_t* vals, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && W > 0 && H > 0 && cam_id >= 0 && n_cams > cam_id && capacity >= 0,
                "adb_raster_tile_scatter_sort: bad sizes");
    if (N == 0 || capacity == 0) return ADB_OK;
    ADB_REQUIRE(radii && splats && tiles_per_gauss && tile_counts && tile_offsets && packed && keys && vals,
                "adb_raster_tile_scatter_sort: null pointer");
    const int T = adb_cdiv(W, ADB_TILE) * adb_cdiv(H, ADB_TILE);
    tile_scatter_kernel<<<adb_cdiv(N, 256), 256, 0, stream>>>(N, radii, splats, tiles_per_gauss, W, H,
                                                             legacy ? ADB_CONV_INRIA : ADB_CONV_GSPLAT,
                                                             tile_counts + (size_t)T * COPIES, tile_counts, capacity,
                                                             (unsigned long long*)packed);
    ADB_CHECK_LAUNCH("tile_scatter_kernel");
    tile_sort_kernel<<<T, SORT_THREADS, 0, stream>>>(T, tile_offsets, (unsigned long long*)packed, cam_id, N,
                                                    adb_tile_bits(W, H), keys, vals);
    ADB_CHECK_LAUNCH("tile_sort_kernel");
    return ADB_OK;
}

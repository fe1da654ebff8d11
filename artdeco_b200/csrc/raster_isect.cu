// Tile intersection: for every tile, the depth-sorted list of the splats that touch it.
// Integer / byte work with a BIT-EXACT contract against the oracle (SURVEY.md §8a R2c-R2e, App. B.3):
//   key = (cam << (32+tile_bits)) | (tile << 32) | float_bits(depth),  val = cam*N + gaussian,
//   in the order of a stable ascending sort, over the live bits, of the keys emitted Gaussian-major, then ty outer / tx
//   inner; tile_offsets[t] = the first sorted index of tile t, tile_offsets[T] = the number of intersections.
// Replaces gsplat's isect_tiles / radix sort / isect_offset_encode that the reference reaches through
// Reconstruct/scene/scene_models/h3dgsv3.py:664-680.  No library sort and no host sync:
//
//   count    per Gaussian: one RED.ADD per touched tile into tile_counts[tile][copy]            (16 B read / Gaussian)
//            (fused into the projection by adb_raster_project_fwd_counts / _multi; tile_count_kernel otherwise)
//   scan     one CTA per view: exclusive scan of the T x COPIES counters -> per-(tile,copy) segment starts + tile_offsets[T+1]
//            (clamped to the caller's capacity; the true total and an overflow flag stay on the device)
//   band     per chunk of 2048 Gaussians: one pair (word = depth_bits<<32 | gaussian, x0 | x1 << 16) per tile row the
//            rectangle touches, counted per row in shared memory, one global atomic per (CTA, row) on the row's cursor, pairs
//            grouped by row in shared memory and written as one run per row into the row's region of the scratch (the
//            row's tile segments);
//   expand   one CTA per (row, view): tile cursors in shared memory; per chunk of 1024 pairs the expanded words are
//            grouped by tile in shared memory and written as one run per tile into `packed`; the row's counters are zeroed,
//            so the buffer needs no memset between calls;
//   sort     one CTA per tile: bitonic sort of the tile's 64-bit words — the 64-element sub-networks run in REGISTERS with
//            warp shuffles, only the wider exchanges go through shared memory (global memory for tiles beyond 4096
//            entries) — then keys = cam|tile|depth_bits and vals = cam*N + gaussian are written out.
//
// COPIES = 4 replicas of every tile counter (selected by CTA index) cut the same-address serialisation of the L2 atomics
// that a single counter per tile suffers.  The per-(tile, copy) counters are read only by the scan; the band pass uses one
// cursor per row.  The band and expand passes store runs of consecutive slots: a scatter that stores each word where it
// lands costs one returning L2 atomic and one stray 8-byte store per intersection, and its time follows the number of
// those L2 requests rather than the bytes.
//
// Views: the scan, band, expand and sort take C views at once (one scan CTA per view, a view grid dimension for the
// others).  View c has its own counter block [2*COPIES*T] and tile_offsets row [T+1], and owns the segment
// [base_c, base_c + cap_c) of the one packed/keys/vals buffer, base_c = sum of the previous views' capacities.  Offsets and
// vals are absolute in that buffer, so the blend kernels index it directly; vals follow gsplat's cam*N + gaussian.
//
// Why the order equals the reference's stable radix sort of (tile, depth): the reference emits keys Gaussian-major, so
// inside one (tile, depth) tie the stable sort leaves ascending Gaussian ids — exactly the ascending order of the
// composite word (depth_bits, gaussian).  A Gaussian touches a tile at most once, so the words of a tile are distinct
// and the result does not depend on the order in which the band and expand passes deliver them.  (SURVEY.md App. B.3;
// oracle: adbo_isect_sort.)  A global 45-bit onesweep radix sort of the keys moved 6 x 24 B per intersection and was
// 12.6 % of the round-1 step.
//
// Compiled with -fmad=false like raster_project.cu: it would not matter here (only /16, floor, ceil), but the tile
// rectangle must stay the projection's (adb_tile_rect, raster_common.cuh).
#include "raster_common.cuh"
#include <stdio.h>

namespace {

constexpr int COPIES = ADB_TILE_COUNTER_COPIES;
static_assert(COPIES == 4, "the scan kernel reads one tile's counters as an int4");
constexpr int MAX_VIEWS = 64;

// Per-view segments of the intersection buffer, passed by value (kernel parameters, so a captured graph keeps them).
struct Segments {
    long long base[MAX_VIEWS];
    long long cap[MAX_VIEWS];
};

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

// One CTA of 1024 threads per view, over the view's T*COPIES counters in (tile-major, copy-minor) order.
// starts[e] = base + min(capacity, sum_{f<e} counts[f]);  offsets[t] = starts[t*COPIES];  offsets[T] = base + min(capacity, total).
// offsets_all == NULL: only the totals are computed (nothing else written).
// Each thread owns 16 consecutive counters (4 tiles x 4 copies): four 128-bit loads in flight, one block-wide scan of the
// per-thread sums per 16384 counters (1080p: two rounds; the first version looped 8 times with
// four barriers each and took 20 us).
constexpr int SCAN_THREADS = 1024;
__global__ void __launch_bounds__(SCAN_THREADS)
tile_scan_kernel(int T, int32_t* __restrict__ counts_all, Segments seg, int32_t* __restrict__ offsets_all,
                 long long* __restrict__ total, int32_t* __restrict__ overflow) {
    constexpr int PER = 16;                                  // 1024 threads x 16 counters = 16384 per round, no spills
    __shared__ long long s_warp[32];
    __shared__ long long s_carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int view = blockIdx.x;
    const int32_t* counts = counts_all + (size_t)view * 2 * COPIES * T;
    int32_t* starts = counts_all + (size_t)view * 2 * COPIES * T + (size_t)T * COPIES;
    int32_t* offsets = offsets_all ? offsets_all + (size_t)view * (T + 1) : nullptr;
    const long long capacity = seg.cap[view], seg_base = seg.base[view];
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
            st.x = (int32_t)(seg_base + (excl < capacity ? excl : capacity)); excl += c[4 * v];
            st.y = (int32_t)(seg_base + (excl < capacity ? excl : capacity)); excl += c[4 * v + 1];
            st.z = (int32_t)(seg_base + (excl < capacity ? excl : capacity)); excl += c[4 * v + 2];
            st.w = (int32_t)(seg_base + (excl < capacity ? excl : capacity)); excl += c[4 * v + 3];
            if (offsets && e < E) {
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
        if (offsets) offsets[T] = (int32_t)(seg_base + (tot < capacity ? tot : capacity));
        if (total) total[view] = tot;
        if (overflow && offsets && tot > capacity) overflow[view] = 1;
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
tile_sort_kernel(int T, const int32_t* __restrict__ offsets_all, u64* __restrict__ packed, int cam0,
                 int n_per_cam, int tile_bits, int64_t* __restrict__ keys, int32_t* __restrict__ vals) {
    __shared__ u64 s_words[SORT_SMEM_CAP];
    const int tile = blockIdx.x;
    const int cam_id = cam0 + blockIdx.y;
    const int32_t* offsets = offsets_all + (size_t)blockIdx.y * (T + 1);
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
            if (keys) keys[start + i] = (int64_t)(hi | (w >> 32));
            vals[start + i] = vbase + (int32_t)(unsigned)(w & 0xffffffffu);
        }
    } else {
        // rare: a tile with more than SORT_SMEM_CAP splats (L2-resident operands)
        __syncthreads();
        bitonic_sort_global((volatile u64*)g, n, tid);
        __threadfence_block();
        for (int i = tid; i < n; i += SORT_THREADS) {
            const u64 w = g[i];
            if (keys) keys[start + i] = (int64_t)(hi | (w >> 32));
            vals[start + i] = vbase + (int32_t)(unsigned)(w & 0xffffffffu);
        }
    }
}

// ---- band scatter: (Gaussian, tile row) pairs appended in runs, then expanded into the tiles by one CTA per row ----------
constexpr int BAND_THREADS = 256;
constexpr int BAND_PER = 8;             // Gaussians per thread, held in registers between the counting and the writing pass
constexpr int EXPAND_THREADS = 512;
constexpr int EXPAND_PER = 2;           // pairs per thread per chunk, loaded before any of them is expanded
constexpr int STAGE = 4096;             // entries a CTA stages in shared memory, grouped by row / tile, before writing them
constexpr int MAX_BAND_TILES = 4096;    // tile rows and columns (W, H <= 65536): x0 | x1 << 16 fits a pair's column word

// The splat's tile rectangle and its sort word; false when it has no tiles.  All four loads are issued before any of
// them is tested, so that a thread's Gaussians have their loads in flight together.
__device__ __forceinline__ bool band_splat(size_t vi, int i, const int32_t* __restrict__ radii,
                                           const float* __restrict__ splats, const int32_t* __restrict__ tiles_per_gauss,
                                           int W, int H, int convention, int& x0, int& x1, int& y0, int& y1, u64& word) {
    const int tiles = __ldg(tiles_per_gauss + vi);
    const int2 r = __ldg(reinterpret_cast<const int2*>(radii) + vi);
    const float2 m = __ldg(reinterpret_cast<const float2*>(splats + vi * ADB_SPLAT_STRIDE));
    const float depth = __ldg(splats + vi * ADB_SPLAT_STRIDE + 11);
    adb_tile_rect(m.x, m.y, r.x, r.y, W, H, convention, x0, x1, y0, y1);
    word = ((u64)__float_as_uint(depth) << 32) | (unsigned)i;
    return tiles > 0 && x0 < x1 && y0 < y1;
}

// A warp's runs spread over its lanes: lane p owns the items [lo_p, lo_p + n_p), and f(p, v) runs once for every item v
// of every lane p, 32 items at a time (lane j takes item j of the warp's concatenated runs, found by a binary search of the
// run starts), so that one wide splat does not hold up the other 31 lanes.  All 32 lanes call it with the same `s`.
struct WarpRuns {
    unsigned lo[32], excl[32];
};

template <class F>
__device__ __forceinline__ void warp_runs(WarpRuns& s, int lane, unsigned lo, unsigned n, F&& f) {
    unsigned incl = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    const unsigned total = __shfl_sync(0xffffffffu, incl, 31);
    s.lo[lane] = lo;
    s.excl[lane] = incl - n;
    __syncwarp();
    for (unsigned j = lane; j < total; j += 32) {
        int p = 0;                                  // the last lane whose run starts at or before item j
#pragma unroll
        for (int step = 16; step > 0; step >>= 1)
            if (s.excl[p + step] <= j) p += step;
        f(p, s.lo[p] + (j - s.excl[p]));
    }
    __syncwarp();
}

// Exclusive scan of cnt[0..n) into loc (cnt is zeroed); returns the total.  Each thread owns a contiguous range of entries.
// s_part: THREADS / 32 words.  Ends with a barrier.
template <int THREADS>
__device__ __forceinline__ unsigned block_scan(unsigned* cnt, unsigned* loc, int n, unsigned* s_part) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, per = (n + THREADS - 1) / THREADS;
    const int lo = min(n, tid * per), hi = min(n, lo + per);
    unsigned sum = 0;
    for (int e = lo; e < hi; ++e) sum += cnt[e];
    unsigned incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) s_part[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        unsigned v = lane < THREADS / 32 ? s_part[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned y = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += y;
        }
        if (lane < THREADS / 32) s_part[lane] = v;
    }
    __syncthreads();
    unsigned run = (warp ? s_part[warp - 1] : 0) + incl - sum;
    for (int e = lo; e < hi; ++e) {
        loc[e] = run;
        run += cnt[e];
        cnt[e] = 0;
    }
    const unsigned total = s_part[THREADS / 32 - 1];
    __syncthreads();
    return total;
}

// Band pass.  Grid (Gaussian chunks of BAND_THREADS * BAND_PER, views).  Each CTA counts its pairs per tile row in shared
// memory, reserves one run per row with one global atomic on the row's cursor, then writes its pairs into those runs.
// Row b's region of the pair arrays is its tiles' segment [offsets[b*tw], offsets[(b+1)*tw]): a row has at most as many
// pairs as intersections, so the region holds them unless the capacity cut it (pairs past its end are dropped here and
// rebuilt by the tile pass).  The cursor of row b is the scan's segment start of (tile b*tw, copy 0), which equals
// offsets[b*tw]; it counts every pair of the row, kept or not, and stays below 2^32 (at most N pairs per row).
__global__ void __launch_bounds__(BAND_THREADS)
tile_band_kernel(int N, const int32_t* __restrict__ radii, const float* __restrict__ splats,
                 const int32_t* __restrict__ tiles_per_gauss, int W, int H, int convention, int32_t* __restrict__ counts_all,
                 const int32_t* __restrict__ offsets_all, u64* __restrict__ pair_words, uint32_t* __restrict__ pair_cols) {
    extern __shared__ u64 s_band[];
    __shared__ WarpRuns s_runs[BAND_THREADS / 32];
    __shared__ u64 s_word[BAND_THREADS];
    __shared__ uint32_t s_cols[BAND_THREADS];
    __shared__ unsigned s_part[BAND_THREADS / 32];
    const int tw = (W + ADB_TILE - 1) / ADB_TILE, th = (H + ADB_TILE - 1) / ADB_TILE, T = tw * th;
    u64* s_stage_w = s_band;                                            // [STAGE] the CTA's pairs grouped by row
    uint32_t* s_stage_c = reinterpret_cast<uint32_t*>(s_band + STAGE);  // [STAGE]
    uint16_t* s_stage_b = reinterpret_cast<uint16_t*>(s_stage_c + STAGE);   // [STAGE] their rows
    unsigned* s_cnt = reinterpret_cast<unsigned*>(s_stage_b + STAGE);   // pairs per row, then the rank inside the run
    unsigned* s_base = s_cnt + th;              // the run's first slot
    unsigned* s_end = s_cnt + 2 * th;           // the row region's end
    unsigned* s_loc = s_cnt + 3 * th;           // the run's first entry in the stage
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, view = blockIdx.y;
    unsigned* cursors = reinterpret_cast<unsigned*>(counts_all + (size_t)view * 2 * COPIES * T + (size_t)T * COPIES);
    const int32_t* offsets = offsets_all + (size_t)view * (T + 1);
    for (int b = tid; b < th; b += BAND_THREADS) s_cnt[b] = 0;
    __syncthreads();
    uint32_t cols[BAND_PER], rows[BAND_PER];
    u64 words[BAND_PER];
    const int g0 = blockIdx.x * BAND_THREADS * BAND_PER + tid;
#pragma unroll
    for (int k = 0; k < BAND_PER; ++k) {
        const int i = g0 + k * BAND_THREADS;
        int x0 = 0, x1 = 0, y0 = 0, y1 = 0;
        words[k] = 0;
        if (i >= N || !band_splat((size_t)view * N + i, i, radii, splats, tiles_per_gauss, W, H, convention, x0, x1, y0, y1,
                                  words[k]))
            y0 = y1 = 0;
        rows[k] = (uint32_t)y0 | ((uint32_t)y1 << 16);
        cols[k] = (uint32_t)x0 | ((uint32_t)x1 << 16);
    }
#pragma unroll
    for (int k = 0; k < BAND_PER; ++k) {
        const unsigned y0 = rows[k] & 0xffffu, y1 = rows[k] >> 16;
        warp_runs(s_runs[warp], lane, y0, y1 - y0, [&](int, unsigned b) { atomicAdd(s_cnt + b, 1u); });
    }
    __syncthreads();
    for (int b = tid; b < th; b += BAND_THREADS) {
        const unsigned n = s_cnt[b];
        if (n) {
            s_base[b] = atomicAdd(cursors + (size_t)b * tw * COPIES, n);
            s_end[b] = (unsigned)offsets[(b + 1) * tw];
        }
    }
    const unsigned K = block_scan<BAND_THREADS>(s_cnt, s_loc, th, s_part);
    u64* my_word = s_word + warp * 32;
    uint32_t* my_cols = s_cols + warp * 32;
    const bool staged = K <= STAGE;             // else (many rows per splat) each pair is stored where it lands
#pragma unroll
    for (int k = 0; k < BAND_PER; ++k) {
        const unsigned y0 = rows[k] & 0xffffu, y1 = rows[k] >> 16;
        my_word[lane] = words[k];
        my_cols[lane] = cols[k];
        warp_runs(s_runs[warp], lane, y0, y1 - y0, [&](int p, unsigned b) {
            const unsigned r = atomicAdd(s_cnt + b, 1u);
            if (staged) {
                const unsigned q = s_loc[b] + r;
                s_stage_w[q] = my_word[p];
                s_stage_c[q] = my_cols[p];
                s_stage_b[q] = (uint16_t)b;
            } else if (s_base[b] + r < s_end[b]) {
                pair_words[s_base[b] + r] = my_word[p];
                pair_cols[s_base[b] + r] = my_cols[p];
            }
        });
    }
    if (!staged) return;
    __syncthreads();
    for (unsigned q = tid; q < K; q += BAND_THREADS) {   // consecutive entries of a row go to consecutive slots
        const unsigned b = s_stage_b[q], slot = s_base[b] + (q - s_loc[b]);
        if (slot < s_end[b]) {
            pair_words[slot] = s_stage_w[q];
            pair_cols[slot] = s_stage_c[q];
        }
    }
}

// Tile pass.  Grid (tile rows, views).  The row's tile cursors live in shared memory, seeded from offsets; the CTA streams
// the row's pairs, expands each over its columns [x0, x1) (a shared-memory atomic per tile gives the slot in the tile's
// segment) and so writes each tile's words as runs of consecutive slots.  It also zeroes the row's counters (the first
// half of tile_counts), so they are zero again after the call.  When the capacity cut the row's region below its pair
// count, the kept pairs are not all the row's pairs: the CTA then rebuilds the row's pairs from the splats instead, so
// that every tile the capacity leaves whole is complete and every slot of the region is written.
__global__ void __launch_bounds__(EXPAND_THREADS)
tile_expand_kernel(int N, const int32_t* __restrict__ radii, const float* __restrict__ splats,
                   const int32_t* __restrict__ tiles_per_gauss, int W, int H, int convention,
                   int32_t* __restrict__ counts_all, const int32_t* __restrict__ offsets_all,
                   const u64* __restrict__ pair_words, const uint32_t* __restrict__ pair_cols, u64* __restrict__ packed) {
    extern __shared__ u64 s_tiles[];
    __shared__ WarpRuns s_runs[EXPAND_THREADS / 32];
    __shared__ u64 s_word[EXPAND_THREADS];
    __shared__ unsigned s_part[EXPAND_THREADS / 32];
    const int tw = (W + ADB_TILE - 1) / ADB_TILE, T = tw * ((H + ADB_TILE - 1) / ADB_TILE);
    u64* s_stage_w = s_tiles;                                                       // [STAGE] a chunk's words by tile
    uint16_t* s_stage_x = reinterpret_cast<uint16_t*>(s_tiles + STAGE);             // [STAGE] their tile columns
    unsigned* s_cur = reinterpret_cast<unsigned*>(s_stage_x + STAGE);               // next slot of each tile
    unsigned* s_end = s_cur + tw;                                                   // end of each tile's segment
    unsigned* s_cnt = s_cur + 2 * tw;                                               // a chunk's words per tile
    unsigned* s_loc = s_cur + 3 * tw;                                               // their first entry in the stage
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, band = blockIdx.x, view = blockIdx.y, t0 = band * tw;
    int32_t* counts = counts_all + (size_t)view * 2 * COPIES * T;
    const int32_t* offsets = offsets_all + (size_t)view * (T + 1);
    for (int x = tid; x < tw; x += EXPAND_THREADS) {
        s_cur[x] = (unsigned)offsets[t0 + x];
        s_end[x] = (unsigned)offsets[t0 + x + 1];
        s_cnt[x] = 0;
    }
    for (int e = tid; e < tw * COPIES; e += EXPAND_THREADS) counts[(size_t)t0 * COPIES + e] = 0;
    const unsigned start = (unsigned)offsets[t0], end = (unsigned)offsets[t0 + tw];
    const unsigned pairs_end = reinterpret_cast<const unsigned*>(counts + (size_t)T * COPIES)[(size_t)t0 * COPIES];
    __syncthreads();
    if (start == end) return;
    u64* my_word = s_word + warp * 32;
    auto expand = [&](int p, unsigned x) {
        const unsigned slot = atomicAdd(s_cur + x, 1u);
        if (slot < s_end[x]) packed[slot] = my_word[p];
    };
    if (pairs_end <= end) {
        const int n = (int)(pairs_end - start);
        for (int p0 = 0; p0 < n; p0 += EXPAND_THREADS * EXPAND_PER) {
            u64 w[EXPAND_PER];
            uint32_t c[EXPAND_PER];
#pragma unroll
            for (int k = 0; k < EXPAND_PER; ++k) {
                const int p = p0 + k * EXPAND_THREADS + tid;
                w[k] = 0;
                c[k] = 0;
                if (p < n) {
                    w[k] = pair_words[start + p];
                    c[k] = pair_cols[start + p];
                }
            }
#pragma unroll
            for (int k = 0; k < EXPAND_PER; ++k) {
                const unsigned x0 = c[k] & 0xffffu, x1 = c[k] >> 16;
                warp_runs(s_runs[warp], lane, x0, x1 - x0, [&](int, unsigned x) { atomicAdd(s_cnt + x, 1u); });
            }
            __syncthreads();
            const unsigned K = block_scan<EXPAND_THREADS>(s_cnt, s_loc, tw, s_part);
            if (K > STAGE) {                        // wide pairs: this chunk stores each word where it lands
#pragma unroll
                for (int k = 0; k < EXPAND_PER; ++k) {
                    const unsigned x0 = c[k] & 0xffffu, x1 = c[k] >> 16;
                    my_word[lane] = w[k];
                    warp_runs(s_runs[warp], lane, x0, x1 - x0, expand);
                }
                __syncthreads();
                continue;
            }
#pragma unroll
            for (int k = 0; k < EXPAND_PER; ++k) {
                const unsigned x0 = c[k] & 0xffffu, x1 = c[k] >> 16;
                my_word[lane] = w[k];
                warp_runs(s_runs[warp], lane, x0, x1 - x0, [&](int p, unsigned x) {
                    const unsigned q = s_loc[x] + atomicAdd(s_cnt + x, 1u);
                    s_stage_w[q] = my_word[p];
                    s_stage_x[q] = (uint16_t)x;
                });
            }
            __syncthreads();
            for (unsigned q = tid; q < K; q += EXPAND_THREADS) {   // consecutive entries of a tile: consecutive slots
                const unsigned x = s_stage_x[q], slot = s_cur[x] + (q - s_loc[x]);
                if (slot < s_end[x]) packed[slot] = s_stage_w[q];
            }
            __syncthreads();
            for (int x = tid; x < tw; x += EXPAND_THREADS) {
                s_cur[x] += s_cnt[x];
                s_cnt[x] = 0;
            }
            __syncthreads();
        }
    } else {
        for (int i0 = 0; i0 < N; i0 += EXPAND_THREADS) {
            const int i = i0 + tid;
            int x0 = 0, x1 = 0, y0 = 0, y1 = 0;
            u64 w = 0;
            const bool mine = i < N &&
                band_splat((size_t)view * N + i, i, radii, splats, tiles_per_gauss, W, H, convention, x0, x1, y0, y1, w) &&
                y0 <= band && band < y1;
            my_word[lane] = w;
            warp_runs(s_runs[warp], lane, x0, mine ? x1 - x0 : 0, expand);
        }
    }
}

}  // namespace

// Fills the per-view segments from the host array of capacities; refuses what the int32 offsets cannot address.
static int make_segments(const char* name, int C, const long long* capacities, Segments& seg) {
    char msg[160];
    if (!(C > 0 && C <= MAX_VIEWS)) {
        snprintf(msg, sizeof(msg), "%s: C must be 1..%d", name, MAX_VIEWS);
        adb_set_error_msg(msg);
        return ADB_ERR_INVALID;
    }
    if (!capacities) {
        snprintf(msg, sizeof(msg), "%s: null capacities", name);
        adb_set_error_msg(msg);
        return ADB_ERR_INVALID;
    }
    long long base = 0;
    for (int c = 0; c < C; ++c) {
        if (capacities[c] < 0 || base + capacities[c] >= 2147483647LL) {
            snprintf(msg, sizeof(msg), "%s: capacities must be >= 0 and sum to less than 2^31 - 1", name);
            adb_set_error_msg(msg);
            return ADB_ERR_INVALID;
        }
        seg.base[c] = base;
        seg.cap[c] = capacities[c];
        base += capacities[c];
    }
    return ADB_OK;
}

static int scan_launch(int C, int T, int32_t* tile_counts, const Segments& seg, int32_t* tile_offsets, long long* total,
                       int32_t* overflow, cudaStream_t stream) {
    tile_scan_kernel<<<C, SCAN_THREADS, 0, stream>>>(T, tile_counts, seg, tile_offsets, total, overflow);
    ADB_CHECK_LAUNCH("tile_scan_kernel");
    return ADB_OK;
}

// tile_counts: int32 [2 * ADB_TILE_COUNTER_COPIES * T]: first half = the per-(tile,copy) counters, which must be all-zero
// on entry (the expand pass of adb_raster_tile_band_scatter_sort zeroes them again); second half = segment starts
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
    Segments seg;
    seg.base[0] = 0;
    seg.cap[0] = capacity;
    return scan_launch(1, T, tile_counts, seg, tile_offsets, total, overflow, stream);
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

// C views in one launch (counters filled by adb_raster_project_fwd_multi).  capacities: HOST array [C]; view c's segment
// of the intersection buffer starts at the sum of the previous capacities.  tile_counts [C, 2*4*T], tile_offsets [C, T+1]
// (absolute indices into the buffer), total int64 [C] and overflow int32 [C] on the device (may be NULL).  tile_offsets ==
// NULL computes the totals only (sizing pass: read them, then scan again with capacities = totals).
ADB_API int adb_raster_tile_scan_multi(int C, int W, int H, const long long* capacities, int32_t* tile_counts,
                                       int32_t* tile_offsets, long long* total, int32_t* overflow, cudaStream_t stream) {
    Segments seg;
    const int rc = make_segments("adb_raster_tile_scan_multi", C, capacities, seg);
    if (rc != ADB_OK) return rc;
    ADB_REQUIRE(W > 0 && H > 0, "adb_raster_tile_scan_multi: bad sizes");
    ADB_REQUIRE(tile_counts && (tile_offsets || total), "adb_raster_tile_scan_multi: null pointer");
    const int T = adb_cdiv(W, ADB_TILE) * adb_cdiv(H, ADB_TILE);
    return scan_launch(C, T, tile_counts, seg, tile_offsets, total, overflow, stream);
}

// Pair words (8 B) and pair columns (4 B) per slot of the intersection buffer.
ADB_API int adb_raster_tile_band_scratch_bytes(long long capacity, size_t* bytes) {
    ADB_REQUIRE(bytes && capacity >= 0 && capacity < 2147483647LL, "adb_raster_tile_band_scratch_bytes: bad args");
    *bytes = (size_t)capacity * (sizeof(unsigned long long) + sizeof(uint32_t));
    return ADB_OK;
}

static int band_scatter_sort_launch(const char* name, int N, int C, const int32_t* radii, const float* splats,
                                    const int32_t* tiles_per_gauss, int W, int H, int convention, int cam0,
                                    long long capacity, int32_t* tile_counts, const int32_t* tile_offsets, void* packed,
                                    void* scratch, size_t scratch_bytes, int64_t* keys, int32_t* vals, cudaStream_t stream) {
    const int tw = adb_cdiv(W, ADB_TILE), th = adb_cdiv(H, ADB_TILE), T = tw * th;
    char msg[160];
    if (tw > MAX_BAND_TILES || th > MAX_BAND_TILES) {
        snprintf(msg, sizeof(msg), "%s: W and H must be at most %d", name, MAX_BAND_TILES * ADB_TILE);
        adb_set_error_msg(msg);
        return ADB_ERR_INVALID;
    }
    size_t need = 0;
    adb_raster_tile_band_scratch_bytes(capacity, &need);
    if (scratch_bytes < need) {
        snprintf(msg, sizeof(msg), "%s: scratch too small (%zu < %zu bytes)", name, scratch_bytes, need);
        adb_set_error_msg(msg);
        return ADB_ERR_WORKSPACE;
    }
    u64* pair_words = static_cast<u64*>(scratch);
    uint32_t* pair_cols = reinterpret_cast<uint32_t*>(pair_words + capacity);
    const size_t band_smem = STAGE * (sizeof(u64) + sizeof(uint32_t) + sizeof(uint16_t)) + 4 * th * sizeof(unsigned);
    const size_t expand_smem = STAGE * (sizeof(u64) + sizeof(uint16_t)) + 4 * tw * sizeof(unsigned);
    ADB_CUDA(cudaFuncSetAttribute(tile_band_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)band_smem));
    ADB_CUDA(cudaFuncSetAttribute(tile_expand_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)expand_smem));
    tile_band_kernel<<<dim3(adb_cdiv(N, BAND_THREADS * BAND_PER), C), BAND_THREADS, band_smem, stream>>>(
        N, radii, splats, tiles_per_gauss, W, H, convention, tile_counts, tile_offsets, pair_words, pair_cols);
    ADB_CHECK_LAUNCH("tile_band_kernel");
    tile_expand_kernel<<<dim3(th, C), EXPAND_THREADS, expand_smem, stream>>>(
        N, radii, splats, tiles_per_gauss, W, H, convention, tile_counts, tile_offsets, pair_words, pair_cols,
        (u64*)packed);
    ADB_CHECK_LAUNCH("tile_expand_kernel");
    tile_sort_kernel<<<dim3(T, C), SORT_THREADS, 0, stream>>>(T, tile_offsets, (u64*)packed, cam0, N, adb_tile_bits(W, H),
                                                             keys, vals);
    ADB_CHECK_LAUNCH("tile_sort_kernel");
    return ADB_OK;
}

// Band and expand passes + per-tile sort.  keys [capacity] int64, vals [capacity] int32, packed [capacity] uint64 and
// scratch (adb_raster_tile_band_scratch_bytes(capacity)) scratch; tile_counts as left by adb_raster_tile_count_scan.
ADB_API int adb_raster_tile_band_scatter_sort(int N, const int32_t* radii, const float* splats,
                                              const int32_t* tiles_per_gauss, int W, int H, int legacy, int cam_id,
                                              int n_cams, long long capacity, int32_t* tile_counts,
                                              const int32_t* tile_offsets, void* packed, void* scratch,
                                              size_t scratch_bytes, int64_t* keys, int32_t* vals, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && W > 0 && H > 0 && cam_id >= 0 && n_cams > cam_id && capacity >= 0,
                "adb_raster_tile_band_scatter_sort: bad sizes");
    if (N == 0 || capacity == 0) return ADB_OK;
    ADB_REQUIRE(radii && splats && tiles_per_gauss && tile_counts && tile_offsets && packed && scratch && keys && vals,
                "adb_raster_tile_band_scatter_sort: null pointer");
    ADB_REQUIRE(capacity < 2147483647LL, "adb_raster_tile_band_scatter_sort: bad sizes");
    return band_scatter_sort_launch("adb_raster_tile_band_scatter_sort", N, 1, radii, splats, tiles_per_gauss, W, H,
                                    legacy ? ADB_CONV_INRIA : ADB_CONV_GSPLAT, cam_id, capacity, tile_counts, tile_offsets,
                                    packed, scratch, scratch_bytes, keys, vals, stream);
}

// C views in one launch per pass: radii [C,N,2], splats [C,N,12], tiles_per_gauss [C,N]; tile_counts and tile_offsets as
// left by adb_raster_tile_scan_multi with the SAME host capacities [C].  packed / vals (and keys unless NULL) hold
// sum(capacities) elements, scratch adb_raster_tile_band_scratch_bytes(sum(capacities)) bytes; view c's entries start at
// the sum of the previous capacities, vals = c*N + gaussian.
ADB_API int adb_raster_tile_band_scatter_sort_multi(int N, int C, const int32_t* radii, const float* splats,
                                                    const int32_t* tiles_per_gauss, int W, int H,
                                                    const long long* capacities, int32_t* tile_counts,
                                                    const int32_t* tile_offsets, void* packed, void* scratch,
                                                    size_t scratch_bytes, int64_t* keys, int32_t* vals,
                                                    cudaStream_t stream) {
    Segments seg;
    const int rc = make_segments("adb_raster_tile_band_scatter_sort_multi", C, capacities, seg);
    if (rc != ADB_OK) return rc;
    ADB_REQUIRE(N >= 0 && W > 0 && H > 0 && (long long)C * N < 2147483647LL,
                "adb_raster_tile_band_scatter_sort_multi: bad sizes");
    if (N == 0) return ADB_OK;
    ADB_REQUIRE(radii && splats && tiles_per_gauss && tile_counts && tile_offsets && packed && scratch && vals,
                "adb_raster_tile_band_scatter_sort_multi: null pointer");
    return band_scatter_sort_launch("adb_raster_tile_band_scatter_sort_multi", N, C, radii, splats, tiles_per_gauss, W, H,
                                    ADB_CONV_GSPLAT, 0, seg.base[C - 1] + seg.cap[C - 1], tile_counts, tile_offsets, packed,
                                    scratch, scratch_bytes, keys, vals, stream);
}

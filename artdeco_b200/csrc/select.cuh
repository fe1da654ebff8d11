// Exact order-statistic selection by a two-level 16-bit radix histogram (shared by track.cu and densify.cu).
// A value's order key is split into its high and low 16 bits: level 0 histograms the high halves and hist_find locates the
// bin holding a given rank, level 1 histograms the low halves of the values inside that bin.  Histograms count integers,
// so the result is exact and reproducible run to run.
#pragma once
#include <cuda_runtime.h>

namespace adb_select {

constexpr int HIST_BINS = 65536;
constexpr int SEL_THREADS = 1024;

// float -> uint32 whose unsigned order is the float order; every NaN maps to the largest key (torch.sort puts NaN last)
__device__ __forceinline__ unsigned int order_key(float f) {
    if (f != f) return 0xFFFFFFFFu;
    const unsigned int b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
// hist[bin] += 1 with one atomic per distinct bin of the warp (neighbouring pixels mostly share a bin)
__device__ __forceinline__ void hist_add(unsigned int* hist, unsigned int bin) {
    const unsigned int peers = __match_any_sync(__activemask(), bin);
    if ((threadIdx.x & 31) == (unsigned int)(__ffs(peers) - 1)) atomicAdd(hist + bin, (unsigned int)__popc(peers));
}
__device__ __forceinline__ float key_value(unsigned int k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

// rank r of a histogram -> (bin, rank inside the bin); one CTA of SEL_THREADS threads, each owning HIST_BINS/SEL_THREADS bins.
// The histogram is zeroed on the way out.
__device__ inline void hist_find(unsigned int* __restrict__ hist, const unsigned int* ranks, unsigned int* bins,
                                 unsigned int* in_bin, int n_ranks, unsigned int* s_tot) {
    constexpr int PER = HIST_BINS / SEL_THREADS;
    const int t = threadIdx.x;
    unsigned int loc = 0;
#pragma unroll 8
    for (int b = 0; b < PER; ++b) loc += hist[t * PER + b];
    // inclusive scan of the per-thread totals (Hillis-Steele over shared memory)
    s_tot[t] = loc;
    __syncthreads();
    for (int off = 1; off < SEL_THREADS; off <<= 1) {
        const unsigned int v = t >= off ? s_tot[t - off] : 0u;
        __syncthreads();
        s_tot[t] += v;
        __syncthreads();
    }
    const unsigned int excl = s_tot[t] - loc;
    for (int k = 0; k < n_ranks; ++k) {
        const unsigned int r = ranks[k];
        if (r >= excl && r < excl + loc) {
            unsigned int c = excl;
#pragma unroll 4
            for (int b = 0; b < PER; ++b) {
                const unsigned int h = hist[t * PER + b];
                if (r < c + h) { bins[k] = t * PER + b; in_bin[k] = r - c; break; }
                c += h;
            }
        }
    }
    __syncthreads();
#pragma unroll 8
    for (int b = 0; b < PER; ++b) hist[t * PER + b] = 0u;
}

}  // namespace adb_select

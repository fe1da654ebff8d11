// Key-frame retrieval (VSLAM/mast3r_slam/retrieval_database.py with the trainingfree MASt3R retrieval model and a binary
// ASMK codebook) on the device: whitening + l2 attention, top-nfeat selection, the top-MA merge of the codebook assignment,
// ASMK aggregation + binarisation into a fixed-row inverted file, the inverted-file search and the ranking.  The distance
// GEMM of the assignment runs on the wgmma engine of gemm_tc.cu (adb_retrieval_assign, its top-MA epilogue).
//
// Precision contract (DESIGN.md, "Key-frame retrieval"): the whitening is an fp64 FMA GEMM cast to fp32; the aggregation
// sums d - c_w in fp32 in descriptor order, as numpy's axis-0 reduction does; the search sums float64 in ascending word
// order in one thread with the reference's float32/float64 casts, so the scores are bit-identical to the reference once
// the word ids and signatures are.
#include "common.cuh"
#include <cuda_bf16.h>
#include <float.h>
#include <limits.h>
#include <math.h>

namespace {

// ---- whitening: y = fp32((double(x) - m) @ P) (model.py:55-76), 64x64 output tile per CTA, 4x4 per thread ----
constexpr int WT = 64, WK = 16;

__global__ void __launch_bounds__(256) whiten_kernel(int n, int D, const float* __restrict__ x, const double* __restrict__ m,
                                                     const double* __restrict__ P, float* __restrict__ y) {
    __shared__ double As[WK][WT + 1];
    __shared__ double Bs[WK][WT];
    const int r0 = blockIdx.y * WT, c0 = blockIdx.x * WT;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    double acc[4][4] = {};
    for (int k0 = 0; k0 < D; k0 += WK) {
        for (int e = threadIdx.x; e < WT * WK; e += 256) {
            const int r = e / WK, k = e % WK;
            const int gr = r0 + r, gk = k0 + k;
            As[k][r] = (gr < n && gk < D) ? (double)x[(size_t)gr * D + gk] - m[gk] : 0.0;
            const int kb = e / WT, cb = e % WT;
            Bs[kb][cb] = (k0 + kb < D && c0 + cb < D) ? P[(size_t)(k0 + kb) * D + c0 + cb] : 0.0;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < WK; ++k) {
            double a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { a[i] = As[k][ty + 16 * i]; b[i] = Bs[k][tx + 16 * i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int r = r0 + ty + 16 * i, c = c0 + tx + 16 * j;
            if (r < n && c < D) y[(size_t)r * D + c] = (float)acc[i][j];
        }
}

// attention = ||y||_2 per row from the fp32 values (model.py:88-109 'l2norm'), one warp per row
__global__ void row_norm_kernel(int n, int D, const float* __restrict__ y, float* __restrict__ attn) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= n) return;
    float s = 0.f;
    for (int c = lane; c < D; c += 32) { const float v = y[(size_t)row * D + c]; s = fmaf(v, v, s); }
    s = adb_warp_sum(s);
    if (lane == 0) attn[row] = sqrtf(s);
}

// (key, index) strictly before in the order "larger key first, then smaller index"
__device__ __forceinline__ bool before_desc(float ka, int ia, float kb, int ib) { return ka > kb || (ka == kb && ia < ib); }

// ---- top-nfeat by attention (how_select_local, model.py:113-135): one CTA, bitonic sort of <= 1024 keys ----
__global__ void __launch_bounds__(1024) select_kernel(int n, int nfeat, const float* __restrict__ attn, int* __restrict__ tok) {
    __shared__ float key[1024];
    __shared__ int idx[1024];
    const int t = threadIdx.x;
    key[t] = t < n ? attn[t] : -INFINITY;
    idx[t] = t < n ? t : INT_MAX;
    __syncthreads();
    for (int k = 2; k <= 1024; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            const int p = t ^ j;
            if (p > t) {
                const bool up = (t & k) == 0;   // this pair is sorted into "before" order when up
                const bool sw = up ? before_desc(key[p], idx[p], key[t], idx[t]) : before_desc(key[t], idx[t], key[p], idx[p]);
                if (sw) {
                    const float kk = key[t]; key[t] = key[p]; key[p] = kk;
                    const int ii = idx[t]; idx[t] = idx[p]; idx[p] = ii;
                }
            }
            __syncthreads();
        }
    }
    if (t < nfeat) tok[t] = idx[t];
}

// ---- row gather + bf16 split + squared norm: one CTA per output row ----
__global__ void __launch_bounds__(256) gather_split_kernel(int D, const float* __restrict__ src, const int* __restrict__ tok,
                                                           float* __restrict__ dst, __nv_bfloat16* __restrict__ hi,
                                                           __nv_bfloat16* __restrict__ lo, float* __restrict__ sqn) {
    __shared__ float red[8];
    const long long row = blockIdx.x;
    const long long srow = tok ? tok[row] : row;
    float s = 0.f;
    for (int c = threadIdx.x; c < D; c += 256) {
        const float v = src[srow * D + c];
        if (dst) dst[row * D + c] = v;
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        hi[row * D + c] = h;
        lo[row * D + c] = __float2bfloat16_rn(v - __bfloat162float(h));
        s = fmaf(v, v, s);
    }
    s = adb_warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < 8; ++w) t += red[w];
        sqn[row] = t;
    }
}

// (distance, index) strictly before in the order "smaller distance first, then smaller index"
__device__ __forceinline__ bool before_asc(float da, int ia, float db, int ib) { return da < db || (da == db && ia < ib); }

// ---- merge of the per-tile top-MA candidates of the assignment: one warp per descriptor row ----
__global__ void topma_merge_kernel(int nq, int ntiles, int MA, const float* __restrict__ cd, const int* __restrict__ ci,
                                   int* __restrict__ words) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= nq) return;
    float bd[8];
    int bi[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) { bd[q] = INFINITY; bi[q] = INT_MAX; }
    const long long n = (long long)ntiles * MA;
    for (long long e = lane; e < n; e += 32) {
        const float d = cd[(long long)row * n + e];
        const int i = ci[(long long)row * n + e];
        if (!before_asc(d, i, bd[7], bi[7])) continue;
#pragma unroll
        for (int q = 7; q >= 1; --q) {
            if (before_asc(d, i, bd[q - 1], bi[q - 1])) { bd[q] = bd[q - 1]; bi[q] = bi[q - 1]; }
            else if (before_asc(d, i, bd[q], bi[q])) { bd[q] = d; bi[q] = i; }
        }
        if (before_asc(d, i, bd[0], bi[0])) { bd[0] = d; bi[0] = i; }
    }
    // MA rounds of a warp arg-min over the heads of the 32 sorted lists
    for (int r = 0; r < MA; ++r) {
        float d = bd[0];
        int i = bi[0], src = lane;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float d2 = __shfl_xor_sync(0xffffffffu, d, o);
            const int i2 = __shfl_xor_sync(0xffffffffu, i, o), s2 = __shfl_xor_sync(0xffffffffu, src, o);
            if (before_asc(d2, i2, d, i)) { d = d2; i = i2; src = s2; }
        }
        if (lane == 0) words[(long long)row * MA + r] = i;
        if (lane == src) {
#pragma unroll
            for (int q = 0; q < 7; ++q) { bd[q] = bd[q + 1]; bi[q] = bi[q + 1]; }
            bd[7] = INFINITY; bi[7] = INT_MAX;
        }
    }
}

// ---- aggregation (asmk/kernel.py:26-39) ----
constexpr int AGG_MAX = 8192;   // nfeat * MA

// sorted unique word ids of words[r * ld + c], r < nfeat, c < MA
__global__ void __launch_bounds__(1024) unique_words_kernel(int nfeat, int MA, int ld, const int* __restrict__ words,
                                                            int* __restrict__ out, int* __restrict__ count) {
    __shared__ int v[AGG_MAX];
    __shared__ int wsum[32];
    const int n = nfeat * MA;
    int P = 1;
    while (P < n) P <<= 1;
    for (int e = threadIdx.x; e < P; e += 1024) v[e] = e < n ? words[(e / MA) * ld + e % MA] : INT_MAX;
    __syncthreads();
    for (int k = 2; k <= P; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < P; t += 1024) {
                const int p = t ^ j;
                if (p > t) {
                    const bool up = (t & k) == 0;
                    if (up ? v[t] > v[p] : v[t] < v[p]) { const int a = v[t]; v[t] = v[p]; v[p] = a; }
                }
            }
            __syncthreads();
        }
    // stable compaction of the first element of each run, in chunks of 1024
    int base = 0;
    for (int c0 = 0; c0 < n; c0 += 1024) {
        const int e = c0 + threadIdx.x;
        const bool head = e < n && (e == 0 || v[e] != v[e - 1]);
        const unsigned bal = __ballot_sync(0xffffffffu, head);
        const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
        if (lane == 0) wsum[w] = __popc(bal);
        __syncthreads();
        int off = base;
        for (int q = 0; q < w; ++q) off += wsum[q];
        off += __popc(bal & ((1u << lane) - 1u));
        int tot = 0;
        for (int q = 0; q < 32; ++q) tot += wsum[q];
        __syncthreads();
        if (head) out[off] = v[e];
        base += tot;
    }
    if (threadIdx.x == 0) *count = base;
}

// one warp per unique word; lane j holds dimensions 32 w + j: r_w = sum (d - c_word) over the member descriptors in
// descriptor order, then bit 31 - j of signature word w is (r > 0) (hamming.pyx:24-30,90-117: MSB first)
__global__ void residual_sign_kernel(int nfeat, int MA, int ld, int D, const float* __restrict__ desc,
                                     const int* __restrict__ words, const float* __restrict__ centroids,
                                     const int* __restrict__ uwords, const int* __restrict__ count,
                                     unsigned* __restrict__ sig) {
    const int u = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (u >= *count) return;
    const int word = uwords[u];
    const int nw = D / 32;
    float r[32];
    float c[32];
#pragma unroll
    for (int w = 0; w < 32; ++w) {
        r[w] = 0.f;
        c[w] = w < nw ? centroids[(size_t)word * D + 32 * w + lane] : 0.f;
    }
    for (int i0 = 0; i0 < nfeat; i0 += 32) {
        bool mine = false;
        if (i0 + lane < nfeat)
            for (int q = 0; q < MA; ++q) mine |= words[(i0 + lane) * ld + q] == word;
        unsigned bal = __ballot_sync(0xffffffffu, mine);
        while (bal) {
            const int i = i0 + __ffs(bal) - 1;
            bal &= bal - 1;
            const float* d = desc + (size_t)i * D;
#pragma unroll
            for (int w = 0; w < 32; ++w)
                if (w < nw) r[w] = __fadd_rn(r[w], __fsub_rn(d[32 * w + lane], c[w]));
        }
    }
#pragma unroll
    for (int w = 0; w < 32; ++w) {
        const unsigned b = __brev(__ballot_sync(0xffffffffu, r[w] > 0.f));
        if (w < nw && lane == 0) sig[(size_t)u * nw + w] = b;
    }
}

// ---- inverted-file search (inverted_file.py:86-112, kernel.py:56-70, functional.py:11-15): one CTA per image ----
constexpr int SEARCH_THREADS = 128;

__global__ void __launch_bounds__(SEARCH_THREADS) search_kernel(int nfeat, int nw, const int* __restrict__ q_words,
                                                               const unsigned* __restrict__ q_sig, const int* __restrict__ q_count,
                                                               const int* __restrict__ db_words, const unsigned* __restrict__ db_sig,
                                                               const int* __restrict__ db_count, const float* __restrict__ pow_table,
                                                               double* __restrict__ scores) {
    extern __shared__ float contrib[];   // [nfeat]: the image word's float32 term, NaN when it does not contribute
    const int img = blockIdx.x;
    const int nq = *q_count, nd = db_count[img];
    const int* iw = db_words + (size_t)img * nfeat;
    const unsigned* is = db_sig + (size_t)img * nfeat * nw;
    const double rnf = sqrt((double)nd);
    for (int j = threadIdx.x; j < nd; j += SEARCH_THREADS) {
        const int w = iw[j];
        int lo = 0, hi = nq;   // lower bound of w in the sorted query words
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (q_words[mid] < w) lo = mid + 1; else hi = mid; }
        float v = NAN;
        if (lo < nq && q_words[lo] == w) {
            int p = 0;
            for (int k = 0; k < nw; ++k) p += __popc(q_sig[(size_t)lo * nw + k] ^ is[(size_t)j * nw + k]);
            // s = 1 - 2 p / (32 nw) >= 0  <=>  2 p <= 32 nw; s**alpha from the host-built float32 table,
            // then sim /= sqrt(norm_factor) in float64, stored back into the float32 array
            if (2 * p <= 32 * nw) v = (float)((double)pow_table[p] / rnf);
        }
        contrib[j] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int j = 0; j < nd; ++j)
            if (!isnan(contrib[j])) s += (double)contrib[j];
        // q_norm_factor accumulates float32 idf ones: the divisor is float32 sqrt(float32(|W|))
        scores[img] = s / (double)sqrtf((float)nq);
    }
}

// ---- ranking (retrieval_database.py:224-247,263-267): one CTA ----
// out[0] = n_valid, out[1 .. k] = top-k ids (valid prefix), out[k+1] = oldest valid id (-1: none),
// out[k+2] = n_window, out[k+3 ..] = window ids
constexpr int RANK_THREADS = 1024;

__device__ __forceinline__ bool dbefore(double ka, int ia, double kb, int ib) { return ka > kb || (ka == kb && ia < ib); }

// the element that follows (pk, pi) in the order (key desc, index asc); scale multiplies each score into its key
__device__ void next_best(int n, const double* __restrict__ scores, double scale, double pk, int pi, double* bk, int* bi) {
    __shared__ double sk[32];
    __shared__ int si[32];
    double k = -INFINITY;
    int i = INT_MAX;
    for (int e = threadIdx.x; e < n; e += RANK_THREADS) {
        const double v = scores[e] * scale;
        if (dbefore(pk, pi, v, e) && dbefore(v, e, k, i)) { k = v; i = e; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double k2 = __shfl_xor_sync(0xffffffffu, k, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, i, o);
        if (dbefore(k2, i2, k, i)) { k = k2; i = i2; }
    }
    if ((threadIdx.x & 31) == 0) { sk[threadIdx.x >> 5] = k; si[threadIdx.x >> 5] = i; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < RANK_THREADS / 32; ++w)
            if (dbefore(sk[w], si[w], sk[0], si[0])) { sk[0] = sk[w]; si[0] = si[w]; }
    }
    __syncthreads();
    *bk = sk[0];
    *bi = si[0];
    __syncthreads();
}

__global__ void __launch_bounds__(RANK_THREADS) rank_kernel(int n, const double* __restrict__ scores, int k, double min_thresh,
                                                            int window, long long* __restrict__ out) {
    const int kk = min(k, n), ww = min(window, n);
    double pk = INFINITY, bk;
    int pi = -1, bi;
    int n_valid = 0, oldest = INT_MAX;
    bool valid = true;
    for (int r = 0; r < kk; ++r) {
        next_best(n, scores, 1.0, pk, pi, &bk, &bi);
        valid = valid && bk > min_thresh;
        if (threadIdx.x == 0 && valid) { out[1 + n_valid] = bi; oldest = min(oldest, bi); }
        n_valid += valid;
        pk = bk; pi = bi;
    }
    pk = INFINITY; pi = -1;
    for (int r = 0; r < ww; ++r) {
        next_best(n, scores, 100.0, pk, pi, &bk, &bi);
        if (threadIdx.x == 0) out[k + 3 + r] = bi;
        pk = bk; pi = bi;
    }
    if (threadIdx.x == 0) {
        out[0] = n_valid;
        out[k + 1] = n_valid ? oldest : -1;
        out[k + 2] = ww;
    }
}

bool aligned(const void* p, int a) { return ((uintptr_t)p % a) == 0; }

}  // namespace

ADB_API int adb_retrieval_whiten(int n, int D, const float* x, const double* m, const double* P, float* y, float* attn,
                                 cudaStream_t stream) {
    ADB_REQUIRE(n >= 1 && D >= 1, "adb_retrieval_whiten: bad sizes");
    ADB_REQUIRE(x && m && P && y && attn, "adb_retrieval_whiten: null pointer");
    dim3 grid(adb_cdiv(D, WT), adb_cdiv(n, WT));
    whiten_kernel<<<grid, 256, 0, stream>>>(n, D, x, m, P, y);
    ADB_CHECK_LAUNCH("whiten_kernel");
    row_norm_kernel<<<adb_cdiv(n, 8), 256, 0, stream>>>(n, D, y, attn);
    ADB_CHECK_LAUNCH("row_norm_kernel");
    return ADB_OK;
}

ADB_API int adb_retrieval_select(int n, int nfeat, const float* attn, int* tok, cudaStream_t stream) {
    ADB_REQUIRE(n >= 1 && n <= 1024 && nfeat >= 1 && nfeat <= n, "adb_retrieval_select: need 1 <= nfeat <= n <= 1024");
    ADB_REQUIRE(attn && tok, "adb_retrieval_select: null pointer");
    select_kernel<<<1, 1024, 0, stream>>>(n, nfeat, attn, tok);
    ADB_CHECK_LAUNCH("select_kernel");
    return ADB_OK;
}

ADB_API int adb_retrieval_gather_split(long long rows, int D, const float* src, const int* tok, float* dst, void* hi, void* lo,
                                       float* sqn, cudaStream_t stream) {
    ADB_REQUIRE(rows >= 1 && rows < 2147483647LL && D >= 1, "adb_retrieval_gather_split: bad sizes");
    ADB_REQUIRE(src && hi && lo && sqn, "adb_retrieval_gather_split: null pointer");
    gather_split_kernel<<<(unsigned)rows, 256, 0, stream>>>(D, src, tok, dst, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, sqn);
    ADB_CHECK_LAUNCH("gather_split_kernel");
    return ADB_OK;
}

ADB_API int adb_retrieval_topma_merge(int nq, int ntiles, int MA, const float* cand_d, const int* cand_i, int* words,
                                      cudaStream_t stream) {
    ADB_REQUIRE(nq >= 1 && ntiles >= 1 && MA >= 1 && MA <= 8, "adb_retrieval_topma_merge: bad sizes (MA <= 8)");
    ADB_REQUIRE(cand_d && cand_i && words, "adb_retrieval_topma_merge: null pointer");
    topma_merge_kernel<<<adb_cdiv(nq, 8), 256, 0, stream>>>(nq, ntiles, MA, cand_d, cand_i, words);
    ADB_CHECK_LAUNCH("topma_merge_kernel");
    return ADB_OK;
}

ADB_API int adb_retrieval_aggregate(int nfeat, int D, int MA, int ld, const float* desc, const int* words,
                                    const float* centroids, int* out_words, unsigned* out_sig, int* out_count,
                                    cudaStream_t stream) {
    ADB_REQUIRE(nfeat >= 1 && MA >= 1 && MA <= ld && nfeat * MA <= AGG_MAX, "adb_retrieval_aggregate: need nfeat * MA <= 8192");
    ADB_REQUIRE(D >= 32 && D <= 1024 && D % 32 == 0, "adb_retrieval_aggregate: D must be a multiple of 32, at most 1024");
    ADB_REQUIRE(desc && words && centroids && out_words && out_sig && out_count, "adb_retrieval_aggregate: null pointer");
    ADB_REQUIRE(aligned(out_words, 4) && aligned(out_sig, 4) && aligned(out_count, 4), "adb_retrieval_aggregate: misaligned output");
    unique_words_kernel<<<1, 1024, 0, stream>>>(nfeat, MA, ld, words, out_words, out_count);
    ADB_CHECK_LAUNCH("unique_words_kernel");
    residual_sign_kernel<<<adb_cdiv(nfeat * MA, 8), 256, 0, stream>>>(nfeat, MA, ld, D, desc, words, centroids, out_words,
                                                                      out_count, out_sig);
    ADB_CHECK_LAUNCH("residual_sign_kernel");
    return ADB_OK;
}

ADB_API int adb_retrieval_search(int n_db, int nfeat, int nw, const int* q_words, const unsigned* q_sig, const int* q_count,
                                 const int* db_words, const unsigned* db_sig, const int* db_count, const float* pow_table,
                                 double* scores, cudaStream_t stream) {
    ADB_REQUIRE(n_db >= 0 && nfeat >= 1 && nfeat <= 8192 && nw >= 1 && nw <= 32, "adb_retrieval_search: bad sizes");
    if (n_db == 0) return ADB_OK;
    ADB_REQUIRE(q_words && q_sig && q_count && db_words && db_sig && db_count && pow_table && scores,
                "adb_retrieval_search: null pointer");
    search_kernel<<<n_db, SEARCH_THREADS, nfeat * sizeof(float), stream>>>(nfeat, nw, q_words, q_sig, q_count, db_words,
                                                                           db_sig, db_count, pow_table, scores);
    ADB_CHECK_LAUNCH("search_kernel");
    return ADB_OK;
}

ADB_API int adb_retrieval_rank(int n_db, const double* scores, int k, double min_thresh, int window, long long* out,
                               cudaStream_t stream) {
    ADB_REQUIRE(n_db >= 1 && k >= 1 && window >= 1, "adb_retrieval_rank: bad sizes");
    ADB_REQUIRE(scores && out, "adb_retrieval_rank: null pointer");
    rank_kernel<<<1, RANK_THREADS, 0, stream>>>(n_db, scores, k, min_thresh, window, out);
    ADB_CHECK_LAUNCH("rank_kernel");
    return ADB_OK;
}

// Fused attention on the Hopper tensor cores (wgmma): O = softmax(scale * Q K^T) V for one (batch*head, query group)
// work item at a time, with the score matrix held in registers — S and P never touch HBM or shared memory.
//
// Replaces the reference's materialised attention
//   attn = (q @ k.transpose(-2,-1)) * scale; attn = attn.softmax(-1); x = attn @ v
// (VSLAM/thirdparty/mast3r/dust3r/croco/models/blocks.py:105-109 self-attention, :162-166 cross-attention), which
// the reference runs as three torch kernels with a [B,h,N,N] fp32 tensor written and read twice.
//
// Structure (head_dim = 64, keys processed in blocks of 128):
//   warp 8 (TMA)          the item's Q tiles once; K blocks through a KST-stage ring (read twice: see below)
//   warp 9 (TMA)          V^T blocks through a VST-stage ring (own warp so that a full K ring never delays it)
//   warps 0..7            two consumer warpgroups; warpgroup w owns query rows [64 w, 64 w + 64) of every 128-query tile.
//                         Per key block and query tile: S = Q K^T with wgmma m64n128k16 (bf16x3 = 12 MMAs) into 64
//                         registers; a query row lives in the four threads of one quad, so row max / row sum need two
//                         shuffles.  PASS 1 computes S from the bf16 HI parts only and keeps the row maximum (it only has to
//                         be close to the true one, softmax is invariant to it).  PASS 2 recomputes S in bf16x3, forms
//                         p = exp2((s - max) * scale*log2e), accumulates the row sum, and packs P as bf16 (hi, lo) words
//                         directly in the register A-operand layout of wgmma m64n64k16: O += P V (bf16x3 = 24 MMAs) reads P
//                         from registers and V^T from shared memory.
//   Two passes instead of an online-softmax rescale keep O a pure accumulate chain (no per-block rescale of O).
//   TILES = 1: one 128-query tile per CTA (grid = work items).  TILES = 2: two query tiles share every K / V block
//   (half the K / V traffic per query) in PERSISTENT CTAs looping over the work items; the next item's Q loads while the
//   current one finishes.
// Precision: bf16x3 everywhere (same contract as csrc/gemm_tc.cu); exp via ex2.approx (2 ulp).
#include "common.cuh"
#include "hopper.cuh"
#include <cuda.h>
#include <cuda_bf16.h>
#include <stdio.h>
#include <stdlib.h>
#include <atomic>

namespace {

using namespace hopper;

constexpr int NT = 320;                  // warps 0..7 consumers (two warpgroups), warp 8 TMA (Q, K), warp 9 TMA (V^T)
constexpr int QT = 128, KT = 128, HD = 64;
constexpr int TILE16 = 128 * 64 * 2;     // [128 rows x 64 cols] bf16 = 16 KB
constexpr int TILE8 = 64 * 64 * 2;       // [64 rows x 64 cols] bf16 = 8 KB

struct AttnParams {
    int Nq, Nk, heads, n_groups;         // n_groups: query groups of TILES * 128 per (batch*head)
    float scale_log2e;
    __nv_bfloat16* Ohi; __nv_bfloat16* Olo;   // [B, Nq, heads*64]
    int nterms;
};

// one MUFU.EX2; exp2f() wraps it in a denormal-range rescale (FSETP + 2 predicated FMUL) that softmax weights below 2^-126
// do not need -- they flush to zero
__device__ __forceinline__ float ex2_ftz(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    const __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h2);
}

// Ring depths and shared-memory map (bytes, 1024-aligned tiles) per variant: Q tiles (hi, lo), K stages (hi, lo),
// V^T stages [2 key-chunks x (hi, lo) x 8 KB].  Both variants use 224 KB of the 227 KB a block may have.
template <int TILES>
struct Layout {
    static constexpr int KST = 3, VST = TILES == 1 ? 3 : 2;
    static constexpr int OFF_Q = 0;
    static constexpr int OFF_K = OFF_Q + TILES * 2 * TILE16;
    static constexpr int OFF_V = OFF_K + KST * 2 * TILE16;
    static constexpr int OFF_BAR = OFF_V + VST * 4 * TILE8;
    static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
    enum { B_QFULL = 0, B_QEMPTY = 1, B_KFULL = 2, B_KEMPTY = B_KFULL + KST, B_VFULL = B_KEMPTY + KST,
           B_VEMPTY = B_VFULL + VST, B_COUNT = B_VEMPTY + VST };
};

template <int TILES>
__global__ void __launch_bounds__(NT, 1)
attn_fused_kernel(const __grid_constant__ CUtensorMap mQhi, const __grid_constant__ CUtensorMap mQlo,
                  const __grid_constant__ CUtensorMap mKhi, const __grid_constant__ CUtensorMap mKlo,
                  const __grid_constant__ CUtensorMap mVhi, const __grid_constant__ CUtensorMap mVlo,
                  const AttnParams p, const int n_items) {
    using L = Layout<TILES>;
    constexpr int KST = L::KST, VST = L::VST;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t* bar = (uint64_t*)(smem + L::OFF_BAR);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool x3 = p.nterms == 3;
    const int nb = (p.Nk + KT - 1) / KT;
    const uint32_t kstage_bytes = (x3 ? 2 : 1) * TILE16, v_bytes = (x3 ? 4 : 2) * TILE8;

    if (warp == 8 && lane == 0) {
        mbar_init(bar + L::B_QFULL, 1); mbar_init(bar + L::B_QEMPTY, 8);
        for (int s = 0; s < KST; ++s) { mbar_init(bar + L::B_KFULL + s, 1); mbar_init(bar + L::B_KEMPTY + s, 8); }
        for (int s = 0; s < VST; ++s) { mbar_init(bar + L::B_VFULL + s, 1); mbar_init(bar + L::B_VEMPTY + s, 8); }
        mbar_init_fence();
    }
    __syncthreads();

    if (warp == 8) {
        // ===== TMA producer: the item's Q tiles, then K blocks for both passes =====
        if (lane == 0) {
            uint32_t kc = 0, wi = 0;
            for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++wi) {
                const int bh = item / p.n_groups, q0 = (item % p.n_groups) * TILES * QT;
                mbar_wait(bar + L::B_QEMPTY, (wi & 1) ^ 1);         // every S product of the previous item has retired
                mbar_expect_tx(bar + L::B_QFULL, TILES * kstage_bytes);
                for (int t = 0; t < TILES; ++t) {
                    tma_load_3d(smem + L::OFF_Q + t * 2 * TILE16, &mQhi, bar + L::B_QFULL, 0, q0 + t * QT, bh);
                    if (x3) tma_load_3d(smem + L::OFF_Q + t * 2 * TILE16 + TILE16, &mQlo, bar + L::B_QFULL, 0, q0 + t * QT, bh);
                }
                for (int it = 0; it < 2 * nb; ++it, ++kc) {          // pass 1 then pass 2
                    const int j = it % nb, s = kc % KST;
                    mbar_wait(bar + L::B_KEMPTY + s, ((kc / KST) & 1) ^ 1);
                    uint8_t* st = smem + L::OFF_K + s * 2 * TILE16;
                    const bool lo = x3 && it >= nb;                  // pass 1 multiplies the hi parts only
                    mbar_expect_tx(bar + L::B_KFULL + s, lo ? kstage_bytes : (uint32_t)TILE16);
                    tma_load_3d(st, &mKhi, bar + L::B_KFULL + s, 0, j * KT, bh);
                    if (lo) tma_load_3d(st + TILE16, &mKlo, bar + L::B_KFULL + s, 0, j * KT, bh);
                }
            }
        }
        return;
    }
    if (warp == 9) {
        // ===== TMA producer for V^T (pass 2 only): two 64-key chunks per block =====
        if (lane == 0) {
            uint32_t vc = 0;
            for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
                const int bh = item / p.n_groups;
                for (int j = 0; j < nb; ++j, ++vc) {
                    const int vs = vc % VST;
                    mbar_wait(bar + L::B_VEMPTY + vs, ((vc / VST) & 1) ^ 1);
                    mbar_expect_tx(bar + L::B_VFULL + vs, v_bytes);
                    uint8_t* vt = smem + L::OFF_V + vs * 4 * TILE8;
                    tma_load_3d(vt, &mVhi, bar + L::B_VFULL + vs, j * KT, 0, bh);
                    tma_load_3d(vt + TILE8, &mVhi, bar + L::B_VFULL + vs, j * KT + 64, 0, bh);
                    if (x3) {
                        tma_load_3d(vt + 2 * TILE8, &mVlo, bar + L::B_VFULL + vs, j * KT, 0, bh);
                        tma_load_3d(vt + 3 * TILE8, &mVlo, bar + L::B_VFULL + vs, j * KT + 64, 0, bh);
                    }
                }
            }
        }
        return;
    }

    // ===== consumers =====
    // accumulator element i of this thread: row 16 (warp % 4) + lane / 4 + 8 h with h = (i / 2) % 2 (of the warpgroup's 64),
    // column 8 (i / 4) + 2 (lane % 4) + i % 2
    const int wg = warp >> 2;
    const int rq = (warp & 3) * 16 + (lane >> 2), cq = 2 * (lane & 3);
    const uint32_t qa = smem_u32(smem + L::OFF_Q) + wg * (TILE16 / 2);
    uint32_t kc = 0, vc = 0, wi = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++wi) {
        const int bh = item / p.n_groups, q0 = (item % p.n_groups) * TILES * QT;
        mbar_wait(bar + L::B_QFULL, wi & 1);
        float S[64];
        // S = Q_t K^T of K ring slot ks (full: bf16x3, else hi x hi)
        auto score = [&](int t, int ks, bool full) {
            const uint32_t ka = smem_u32(smem + L::OFF_K + ks * 2 * TILE16);
            const uint64_t dQh = make_smem_desc(qa + t * 2 * TILE16), dQl = make_smem_desc(qa + t * 2 * TILE16 + TILE16);
            const uint64_t dKh = make_smem_desc(ka), dKl = make_smem_desc(ka + TILE16);
#pragma unroll
            for (int i = 0; i < 64; ++i) S[i] = 0.f;
            fence_regs(S);
            wgmma_fence();
            if (full) {
#pragma unroll
                for (int k = 0; k < HD / 16; ++k) {
                    const uint64_t adv = (uint64_t)((k * 32) >> 4);
                    wgmma_m64n128k16_ss(S, dQh + adv, dKh + adv);
                    wgmma_m64n128k16_ss(S, dQh + adv, dKl + adv);
                    wgmma_m64n128k16_ss(S, dQl + adv, dKh + adv);
                }
            } else {
#pragma unroll
                for (int k = 0; k < HD / 16; ++k) {
                    const uint64_t adv = (uint64_t)((k * 32) >> 4);
                    wgmma_m64n128k16_ss(S, dQh + adv, dKh + adv);
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(S);
        };
        // PASS 1: row maxima of the raw hi x hi scores
        float m[TILES][2];
#pragma unroll
        for (int t = 0; t < TILES; ++t) m[t][0] = m[t][1] = -3.0e38f;
        for (int it = 0; it < nb; ++it, ++kc) {
            const int ks = kc % KST;
            mbar_wait(bar + L::B_KFULL + ks, (kc / KST) & 1);
#pragma unroll
            for (int t = 0; t < TILES; ++t) {
                score(t, ks, false);
                const int kbase = it * KT + cq;
#pragma unroll
                for (int i = 0; i < 64; ++i)
                    if (kbase + 8 * (i >> 2) + (i & 1) < p.Nk) m[t][(i >> 1) & 1] = fmaxf(m[t][(i >> 1) & 1], S[i]);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(bar + L::B_KEMPTY + ks);
        }
        float c0[TILES][2], l[TILES][2], O[TILES][32];
        const float c1 = p.scale_log2e;
#pragma unroll
        for (int t = 0; t < TILES; ++t)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float v = m[t][h];
                v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
                v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
                c0[t][h] = -v * c1;
                l[t][h] = 0.f;
            }
#pragma unroll
        for (int t = 0; t < TILES; ++t)
#pragma unroll
            for (int i = 0; i < 32; ++i) O[t][i] = 0.f;
        // PASS 2: p = exp2((s - m) * scale*log2e) packed as bf16 (hi, lo) A fragments; O += P V; row sums
        for (int j = 0; j < nb; ++j, ++kc, ++vc) {
            const int ks = kc % KST, vs = vc % VST;
            mbar_wait(bar + L::B_KFULL + ks, (kc / KST) & 1);
            mbar_wait(bar + L::B_VFULL + vs, (vc / VST) & 1);
            const uint32_t va = smem_u32(smem + L::OFF_V + vs * 4 * TILE8);
            const int kbase = j * KT + cq;
            const bool tail = j * KT + KT > p.Nk;            // only the last key block can hold padded keys
#pragma unroll
            for (int t = 0; t < TILES; ++t) {
                score(t, ks, x3);
                if (t == TILES - 1 && j == nb - 1) {            // the item's last S products have retired: Q may be replaced
                    __syncwarp();
                    if (lane == 0) mbar_arrive(bar + L::B_QEMPTY);
                }
                uint32_t ph[32], pl[32];
#pragma unroll
                for (int i = 0; i < 64; i += 2) {
                    const int h = (i >> 1) & 1;
                    float a = ex2_ftz(fmaf(S[i], c1, c0[t][h]));
                    float b = ex2_ftz(fmaf(S[i + 1], c1, c0[t][h]));
                    if (tail) {
                        const int key = kbase + 8 * (i >> 2);
                        if (key >= p.Nk) a = 0.f;
                        if (key + 1 >= p.Nk) b = 0.f;
                    }
                    l[t][h] += a + b;
                    // packed split: one cvt.rn.bf16x2 for the hi pair, shift/mask to widen it back, one for the lo pair
                    const uint32_t hb = pack_bf16(a, b);
                    ph[i >> 1] = hb;
                    pl[i >> 1] = pack_bf16(a - __uint_as_float(hb << 16), b - __uint_as_float(hb & 0xffff0000u));
                }
                fence_regs(ph);
                fence_regs(pl);
                fence_regs(O[t]);
                wgmma_fence();
                // k-step kk covers keys [16 kk, 16 kk + 16) of the block: A words 4 kk .. 4 kk + 3, V^T chunk kk / 4
                if (x3) {
#pragma unroll
                    for (int kk = 0; kk < KT / 16; ++kk) {
                        const uint32_t vchunk = va + (kk >> 2) * TILE8;
                        const uint64_t adv = (uint64_t)(((kk & 3) * 32) >> 4);
                        const uint64_t dVh = make_smem_desc(vchunk) + adv, dVl = make_smem_desc(vchunk + 2 * TILE8) + adv;
                        wgmma_m64n64k16_rs(O[t], ph + 4 * kk, dVh);
                        wgmma_m64n64k16_rs(O[t], ph + 4 * kk, dVl);
                        wgmma_m64n64k16_rs(O[t], pl + 4 * kk, dVh);
                    }
                } else {
#pragma unroll
                    for (int kk = 0; kk < KT / 16; ++kk) {
                        const uint64_t adv = (uint64_t)(((kk & 3) * 32) >> 4);
                        wgmma_m64n64k16_rs(O[t], ph + 4 * kk, make_smem_desc(va + (kk >> 2) * TILE8) + adv);
                    }
                }
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(O[t]);
                fence_regs(ph);
                fence_regs(pl);
            }
            __syncwarp();
            if (lane == 0) { mbar_arrive(bar + L::B_KEMPTY + ks); mbar_arrive(bar + L::B_VEMPTY + vs); }
        }
        // epilogue: O / l -> bf16 split in [B, Nq, heads*64]
        const int b = bh / p.heads, hh = bh % p.heads;
#pragma unroll
        for (int t = 0; t < TILES; ++t)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float sum = l[t][h];
                sum += __shfl_xor_sync(0xffffffffu, sum, 1);
                sum += __shfl_xor_sync(0xffffffffu, sum, 2);
                const float inv = 1.0f / sum;
                const int qrow = q0 + t * QT + wg * 64 + rq + 8 * h;
                if (qrow >= p.Nq) continue;
                const size_t o = ((size_t)b * p.Nq + qrow) * (size_t)(p.heads * HD) + (size_t)hh * HD + cq;
#pragma unroll
                for (int g = 0; g < 8; ++g) {
                    const float a = O[t][4 * g + 2 * h] * inv, bb = O[t][4 * g + 2 * h + 1] * inv;
                    const uint32_t hb = pack_bf16(a, bb);
                    *reinterpret_cast<uint32_t*>(p.Ohi + o + 8 * g) = hb;
                    if (p.Olo)
                        *reinterpret_cast<uint32_t*>(p.Olo + o + 8 * g) =
                            pack_bf16(a - __uint_as_float(hb << 16), bb - __uint_as_float(hb & 0xffff0000u));
                }
            }
    }
}

// bf16 [batch][rows][cols] (cols contiguous); box = 64 cols x box_rows x 1, SWIZZLE_128B
int make_map(CUtensorMap* map, const void* ptr, long long batch, int rows, int cols, long long ld, int box_rows) {
    hopper::EncodeTiledFn fn = hopper::get_encode_fn();
    if (!fn) { adb_set_error_msg("cuTensorMapEncodeTiled driver entry point unavailable"); return ADB_ERR_CUDA; }
    cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)batch};
    cuuint64_t strides[2] = {(cuuint64_t)ld * 2, (cuuint64_t)rows * ld * 2};
    cuuint32_t box[3] = {64, (cuuint32_t)box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { adb_set_error_msg("adb_attention_bf16: cuTensorMapEncodeTiled failed"); return ADB_ERR_INVALID; }
    return ADB_OK;
}

}  // namespace

// O[b, n, h*64 + d] = sum_k softmax_k(scale * <Q[b,h,n,:], K[b,h,k,:]>) * V[b,h,k,d]   (head_dim 64)
//   Q: bf16 split [B*heads, Nq, 64];  K: [B*heads, Nk, 64];  Vt: [B*heads, 64, Nkpad] (Nkpad % 8 == 0, zero padded);
//   O: bf16 split [B, Nq, heads*64].  *_lo all non-NULL selects bf16x3.
// 0 = automatic (default, currently variant 1; env ADB_ATTN_KERNEL overrides at load), 1 = one query tile per CTA, 2 = two query tiles per
// persistent CTA.  Returns the previous setting.  Both variants produce the same values to rounding (tests/test_gemm.py).
static std::atomic<int> g_attn_variant{getenv("ADB_ATTN_KERNEL") ? atoi(getenv("ADB_ATTN_KERNEL")) : 0};
ADB_API int adb_attention_set_variant(int variant) {
    if (variant < 0 || variant > 2) return -1;
    return g_attn_variant.exchange(variant);
}

ADB_API int adb_attention_bf16(int B, int heads, int Nq, int Nk, int Nkpad, const void* Q_hi, const void* Q_lo,
                               const void* K_hi, const void* K_lo, const void* Vt_hi, const void* Vt_lo, float scale,
                               void* O_hi, void* O_lo, cudaStream_t stream) {
    ADB_REQUIRE(B >= 1 && heads >= 1 && Nq >= 1 && Nk >= 1 && Nkpad >= Nk && Nkpad % 8 == 0, "adb_attention_bf16: bad sizes");
    ADB_REQUIRE(Q_hi && K_hi && Vt_hi && O_hi, "adb_attention_bf16: null pointer");
    const bool x3 = Q_lo && K_lo && Vt_lo;
    ADB_REQUIRE(x3 || (!Q_lo && !K_lo && !Vt_lo), "adb_attention_bf16: give all lo operands or none");
    ADB_REQUIRE((((uintptr_t)O_hi | (uintptr_t)O_lo) % 16) == 0, "adb_attention_bf16: outputs must be 16-byte aligned");
    CUtensorMap mQh, mQl, mKh, mKl, mVh, mVl;
    const long long bh = (long long)B * heads;
    int rc;
    if ((rc = make_map(&mQh, Q_hi, bh, Nq, 64, 64, 128))) return rc;
    if ((rc = make_map(&mKh, K_hi, bh, Nk, 64, 64, 128))) return rc;
    if ((rc = make_map(&mVh, Vt_hi, bh, 64, Nkpad, Nkpad, 64))) return rc;
    mQl = mQh; mKl = mKh; mVl = mVh;
    if (x3) {
        if ((rc = make_map(&mQl, Q_lo, bh, Nq, 64, 64, 128))) return rc;
        if ((rc = make_map(&mKl, K_lo, bh, Nk, 64, 64, 128))) return rc;
        if ((rc = make_map(&mVl, Vt_lo, bh, 64, Nkpad, Nkpad, 64))) return rc;
    }
    AttnParams p;
    p.Nq = Nq; p.Nk = Nk; p.heads = heads;
    p.scale_log2e = scale * 1.4426950408889634f;
    p.Ohi = (__nv_bfloat16*)O_hi; p.Olo = (__nv_bfloat16*)O_lo; p.nterms = x3 ? 3 : 1;
    static AdbDeviceOnce once;
    int num_sms = 0;
    {
        const int rc = once.ensure([]() -> int {
            ADB_CUDA(cudaFuncSetAttribute(attn_fused_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, Layout<1>::SMEM_BYTES));
            ADB_CUDA(cudaFuncSetAttribute(attn_fused_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, Layout<2>::SMEM_BYTES));
            return ADB_OK;
        }, &num_sms);
        if (rc != ADB_OK) return rc;
    }
    // Kernel choice.  Variant 2 (two query tiles per persistent CTA) halves the K/V stream per query, but at 320 threads its
    // two O accumulators exceed the 168-register budget (ptxas serialises part of its wgmma and spills): measured on an H100
    // SXM (400 W), variant 1 is faster at every MASt3R shape (e.g. 16x16 heads x 1024 tokens: 435 vs 537 us; 8x12 x 768:
    // 118 vs 165 us), so the automatic choice is variant 1.
    const long long n1 = bh * adb_cdiv(Nq, QT), n2 = bh * adb_cdiv(Nq, 2 * QT);
    ADB_REQUIRE(n1 < 2147483647LL, "adb_attention_bf16: too many work items");
    int variant = g_attn_variant.load(std::memory_order_relaxed);
    if (variant == 0) variant = 1;
    if (variant == 2) {
        p.n_groups = adb_cdiv(Nq, 2 * QT);
        const int grid = (int)(n2 < num_sms ? n2 : num_sms);
        attn_fused_kernel<2><<<grid, NT, Layout<2>::SMEM_BYTES, stream>>>(mQh, mQl, mKh, mKl, mVh, mVl, p, (int)n2);
        ADB_CHECK_LAUNCH("attn_fused_kernel<2>");
        return ADB_OK;
    }
    p.n_groups = adb_cdiv(Nq, QT);
    attn_fused_kernel<1><<<(unsigned)n1, NT, Layout<1>::SMEM_BYTES, stream>>>(mQh, mQl, mKh, mKl, mVh, mVl, p, (int)n1);
    ADB_CHECK_LAUNCH("attn_fused_kernel<1>");
    return ADB_OK;
}

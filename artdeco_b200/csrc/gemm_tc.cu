// Batched GEMM / implicit-GEMM 3x3 convolution on the Hopper tensor cores (wgmma):
//     D = act(alpha * A * B^T + bias) + residual
//
// This is the one dense-contraction engine of the MASt3R path: every nn.Linear / q@k^T / attn@v of
// VSLAM/thirdparty/mast3r/dust3r/croco/models/blocks.py:58-112,140-169, the patch embedding
// dust3r/dust3r/patch_embed.py:19-29, the local-feature MLP mast3r/catmlp_dpt_head.py:67-69 and the 3x3 / 1x1
// convolutions of the DPT head croco/models/dpt_block.py:79-142,356-410.  The reference runs them as fp32 (TF32)
// cuBLAS / cuDNN calls.
//
// sm_90a structure (hand-written PTX, no CUTLASS):
//   * one CTA per 128x128 output tile; operands are bf16, K-major, staged by TMA (cp.async.bulk.tensor, SWIZZLE_128B)
//     into a multi-stage shared-memory ring guarded by full/empty mbarriers, filled by one producer warp;
//   * two consumer warpgroups, 64 rows each, issue wgmma.mma_async m64n128k16 (bf16 in, fp32 accumulator in registers)
//     straight from the swizzled ring; one k-block's MMAs stay in flight while the next are issued;
//   * the accumulator is PROMOTED to a round-to-nearest fp32 register sum every KCHUNK_KB k-blocks (the tensor core's
//     accumulation error grows linearly with the chain length);
//   * epilogue: the 128x128 fp32 tile is restaged through shared memory (over the drained ring) so that each thread
//     owns 64 consecutive columns of one output row, then alpha / bias / GELU(erf) or ReLU / residual are applied and
//     fp32 and/or a bf16 (hi, lo) split written as full 128 B lines;
//   * "bf16x3": with the lo operands the kernel accumulates A_hi*B_hi + A_hi*B_lo + A_lo*B_hi into the same
//     accumulator (~16 mantissa bits per operand, error ~1e-5): single-pass bf16 or TF32 (the reference's
//     own GPU mode) cannot hold the north-star's 1e-4 pointmap tolerance over 36 layers;
//   * CONV MODE: A is an NHWC activation described by a 4-D tensor map; a tile is a Wb x Hb pixel rectangle
//     and K-block (tap, channel chunk) is ONE shifted TMA box load — out-of-image taps are zero-filled by the
//     TMA unit, which is exactly the conv's zero padding; no im2col buffer exists.
// Warp roles: warps 0..7 = two consumer warpgroups (MMA + epilogue), warp 8 = TMA producer.
#include "common.cuh"
#include "hopper.cuh"
#include <cuda.h>
#include <cuda_bf16.h>
#include <stdio.h>

namespace {

using namespace hopper;

constexpr int BM = 128, BN = 128, BK = 64;    // BK * 2 B = 128 B = one swizzle row
constexpr int TILE_BYTES = BM * BK * 2;       // 16 KB (A and B tiles have the same shape)
constexpr int MMA_K = 16;
constexpr int NCONSUMER = 256;                // two warpgroups
constexpr int NTHREADS = NCONSUMER + 32;      // + the TMA producer warp
constexpr int RING_BYTES = 192 * 1024;        // 6 stages of (A, B) or 3 of (A_hi, B_hi, A_lo, B_lo)
constexpr int KCHUNK_KB = 8;                  // k-blocks (of 64) accumulated by the tensor core before promotion
constexpr int STG_LD = BN + 4;                // fp32 row pitch of the epilogue restaging tile
constexpr int SMEM_BYTES = RING_BYTES + 1024 /*align*/ + 256 /*barriers*/;
static_assert(BM * STG_LD * 4 <= RING_BYTES, "epilogue staging must fit over the ring");

struct GemmParams {
    int M, N, K;
    int batch;
    int nterms;  // 1 or 3
    int stages;
    float* D; long long ldd, sD;
    __nv_bfloat16* Dhi; __nv_bfloat16* Dlo; long long ldo, sO;
    const float* bias;
    const float* residual; long long ldr, sR;
    float alpha;
    int act;          // 0 none, 1 GELU(erf), 2 ReLU
    int split_relu;   // the bf16 split output stores relu(value) (fp32 D keeps the raw value)
    int zdiv;         // z = z_outer * zdiv + z_inner; outputs use (z_outer * s?2 + z_inner * s?)
    long long sD2, sO2, sR2;
    // conv mode (conv_wb > 0): M tile = conv_hb x conv_wb pixel rectangle of an H x W image, K block = (tap, chunk)
    int conv_wb, conv_hb, conv_H, conv_W, conv_chunks, conv_tiles_x, conv_tiles_y;
    // RoPE epilogue (rope_ndst > 0): output columns [0, rope_ndst * rope_C) are attention heads (64 wide); each is rotated
    // with RoPE2D for its token's (y, x) position and written as a bf16 split in head-major layout [B*heads, ntok, 64] to
    // rope_hi/lo[col / rope_C]; the remaining columns take the ordinary D path (D is pre-shifted by the caller).
    int rope_ndst, rope_C, rope_heads, rope_ntok, rope_npos;
    const long long* rope_pos;      // int64 [M, 2] (y, x)
    const float* rope_table;        // [n_pos][16][2] (cos, sin)
    __nv_bfloat16* rope_hi[2]; __nv_bfloat16* rope_lo[2];
};

__device__ __forceinline__ float gelu_erf(float v) { return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f)); }

// 32 B per thread as two 128-bit accesses: one full sector per lane
__device__ __forceinline__ void st_v8(float* p, const float* v) {
    reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
    reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void st_v8_b32(void* p, const uint32_t* w) {
    reinterpret_cast<uint4*>(p)[0] = make_uint4(w[0], w[1], w[2], w[3]);
    reinterpret_cast<uint4*>(p)[1] = make_uint4(w[4], w[5], w[6], w[7]);
}
__device__ __forceinline__ void ld_v8_nc(const float* p, float* v) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

struct TileCoord {
    int bz, mt, nt;
};
__device__ __forceinline__ TileCoord decode_tile(int tile, int tiles_m, int tiles_n) {
    TileCoord c;
    c.nt = tile % tiles_n;
    const int r = tile / tiles_n;
    c.mt = r % tiles_m;
    c.bz = r / tiles_m;
    return c;
}

// Epilogue of one thread: output row `trow` of the tile, columns [n0, n0 + 64) held in acc[2][32].
// ROPE: the epilogue variant of adb_gemm_bf16_rope (own instantiation so that its extra live values do not cost the plain
// GEMM registers); it has no residual / activation / split-output paths.
template <bool ROPE>
__device__ __forceinline__ void store_row(const GemmParams& p, float (&acc)[2][32], int trow, bool conv, int x0, int y0,
                                          int m0, int n0, size_t dbase, size_t obase, size_t rbase, bool vec_ok) {
    long long row;
    if (conv) {
        const int yy = y0 + trow / p.conv_wb, xx = x0 + trow % p.conv_wb;
        row = (yy < p.conv_H && xx < p.conv_W) ? (long long)yy * p.conv_W + xx : -1;
    } else {
        row = m0 + trow < p.M ? m0 + trow : -1;
    }
    if (row < 0) return;
#pragma unroll
    for (int g = 0; g < 2; ++g) {
        const int c0 = n0 + g * 32;
        if (c0 >= p.N) continue;
        float (&v)[32] = acc[g];      // finished accumulators are transformed in place
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            float t = acc[g][j] * p.alpha;
            if (p.bias && c0 + j < p.N) t += __ldg(p.bias + c0 + j);
            if (!ROPE) {
                if (p.act == 1) t = gelu_erf(t);
                else if (p.act == 2) t = fmaxf(t, 0.f);
            }
            v[j] = t;
        }
        if (ROPE && c0 < p.rope_ndst * p.rope_C) {
            // this thread holds dims [d0, d0+32) of one head of token `row`: one RoPE axis (y: d0 = 0, x: d0 = 32),
            // pairs (i, i+16) -- blocks.py:101-103 / pos_embed.py:129-159, fused with the head split
            const int sec = c0 / p.rope_C, cc = c0 - sec * p.rope_C;
            const int hh = cc >> 6, axis = (cc >> 5) & 1;
            long long pz = __ldg(p.rope_pos + row * 2 + axis);
            pz = pz < 0 ? 0 : (pz >= p.rope_npos ? p.rope_npos - 1 : pz);
            const float4* tb = reinterpret_cast<const float4*>(p.rope_table + pz * 32);
#pragma unroll
            for (int i4 = 0; i4 < 8; ++i4) {
                const float4 cs = __ldg(tb + i4);          // (cos, sin) of frequencies 2*i4 and 2*i4+1
                const int i = 2 * i4;
                const float u0 = v[i], w0 = v[i + 16], u1 = v[i + 1], w1 = v[i + 17];
                v[i] = u0 * cs.x - w0 * cs.y;      v[i + 16] = w0 * cs.x + u0 * cs.y;
                v[i + 1] = u1 * cs.z - w1 * cs.w;  v[i + 17] = w1 * cs.z + u1 * cs.w;
            }
            const long long bq = row / p.rope_ntok, nq = row - bq * p.rope_ntok;
            const size_t off = (((size_t)bq * p.rope_heads + hh) * p.rope_ntok + nq) * 64 + axis * 32;
            __nv_bfloat16* hp = p.rope_hi[sec] + off;
            __nv_bfloat16* lp = p.rope_lo[sec] ? p.rope_lo[sec] + off : nullptr;
#pragma unroll
            for (int h8 = 0; h8 < 2; ++h8) {               // 16 values -> one 32-byte store of hi and of lo
                uint32_t hw[8], lw[8];
#pragma unroll
                for (int k2 = 0; k2 < 8; ++k2) {
                    const float a = v[16 * h8 + 2 * k2], b = v[16 * h8 + 2 * k2 + 1];
                    const __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
                    const uint32_t hb = *reinterpret_cast<const uint32_t*>(&h2);
                    const __nv_bfloat162 l2 = __floats2bfloat162_rn(a - __uint_as_float(hb << 16),
                                                                    b - __uint_as_float(hb & 0xffff0000u));
                    hw[k2] = hb;
                    lw[k2] = *reinterpret_cast<const uint32_t*>(&l2);
                }
                st_v8_b32(hp + 16 * h8, hw);
                if (lp) st_v8_b32(lp + 16 * h8, lw);
            }
            continue;
        }
        if (vec_ok && c0 + 32 <= p.N) {
            if (!ROPE && p.residual) {
                const float* rp = p.residual + rbase + (size_t)row * p.ldr + c0;
#pragma unroll
                for (int j8 = 0; j8 < 4; ++j8) {
                    float rs[8];
                    ld_v8_nc(rp + 8 * j8, rs);
#pragma unroll
                    for (int k2 = 0; k2 < 8; ++k2) v[8 * j8 + k2] += rs[k2];
                }
            }
            if (p.D) {
                float* dp = p.D + dbase + (size_t)row * p.ldd + c0;
#pragma unroll
                for (int j8 = 0; j8 < 4; ++j8) st_v8(dp + 8 * j8, v + 8 * j8);
            }
            if (!ROPE && p.Dhi) {
                __nv_bfloat16* hp = p.Dhi + obase + (size_t)row * p.ldo + c0;
                __nv_bfloat16* lp = p.Dlo ? p.Dlo + obase + (size_t)row * p.ldo + c0 : nullptr;
#pragma unroll
                for (int h8 = 0; h8 < 2; ++h8) {
                    uint32_t hw[8], lw[8];
#pragma unroll
                    for (int k2 = 0; k2 < 8; ++k2) {
                        float a = v[16 * h8 + 2 * k2], b = v[16 * h8 + 2 * k2 + 1];
                        if (p.split_relu) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
                        const __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
                        const uint32_t hb = *reinterpret_cast<const uint32_t*>(&h2);
                        const __nv_bfloat162 l2 = __floats2bfloat162_rn(a - __uint_as_float(hb << 16),
                                                                        b - __uint_as_float(hb & 0xffff0000u));
                        hw[k2] = hb;
                        lw[k2] = *reinterpret_cast<const uint32_t*>(&l2);
                    }
                    st_v8_b32(hp + 16 * h8, hw);
                    if (lp) st_v8_b32(lp + 16 * h8, lw);
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                if (c0 + j < p.N) {
                    float t = v[j];
                    if (!ROPE && p.residual) t += __ldg(p.residual + rbase + (size_t)row * p.ldr + c0 + j);
                    if (p.D) p.D[dbase + (size_t)row * p.ldd + c0 + j] = t;
                    if (!ROPE && p.Dhi) {
                        const float ts = p.split_relu ? fmaxf(t, 0.f) : t;
                        const __nv_bfloat16 h = __float2bfloat16_rn(ts);
                        p.Dhi[obase + (size_t)row * p.ldo + c0 + j] = h;
                        if (p.Dlo) p.Dlo[obase + (size_t)row * p.ldo + c0 + j] = __float2bfloat16_rn(ts - __bfloat162float(h));
                    }
                }
            }
        }
    }
}

template <bool ROPE>
__global__ void __launch_bounds__(NTHREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap mapAhi, const __grid_constant__ CUtensorMap mapAlo,
               const __grid_constant__ CUtensorMap mapBhi, const __grid_constant__ CUtensorMap mapBlo,
               const GemmParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    const bool x3 = p.nterms == 3;
    const uint32_t stage_bytes = (x3 ? 4 : 2) * TILE_BYTES;
    uint64_t* full_bar = (uint64_t*)(smem + RING_BYTES);
    uint64_t* empty_bar = full_bar + p.stages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool conv = p.conv_wb > 0;
    const int tiles_m = conv ? p.conv_tiles_x * p.conv_tiles_y : (p.M + BM - 1) / BM;
    const int tiles_n = (p.N + BN - 1) / BN;
    const int num_kb = conv ? 9 * p.conv_chunks : (p.K + BK - 1) / BK;
    const TileCoord tc = decode_tile(blockIdx.x, tiles_m, tiles_n);
    const int m0 = tc.mt * BM, n0 = tc.nt * BN;
    int x0 = 0, y0 = 0;
    if (conv) { x0 = (tc.mt % p.conv_tiles_x) * p.conv_wb; y0 = (tc.mt / p.conv_tiles_x) * p.conv_hb; }

    if (warp == 8 && lane == 0) {
        prefetch_tensormap(&mapAhi);
        prefetch_tensormap(&mapBhi);
        if (x3) { prefetch_tensormap(&mapAlo); prefetch_tensormap(&mapBlo); }
        for (int s = 0; s < p.stages; ++s) { mbar_init(full_bar + s, 1); mbar_init(empty_bar + s, NCONSUMER / 32); }
        mbar_init_fence();
    }
    __syncthreads();

    if (warp == 8) {
        // ===== TMA producer =====
        if (lane == 0) {
            for (int kb = 0; kb < num_kb; ++kb) {
                const int s = kb % p.stages;
                mbar_wait(empty_bar + s, ((kb / p.stages) & 1) ^ 1);
                uint8_t* st = smem + (size_t)s * stage_bytes;
                mbar_expect_tx(full_bar + s, stage_bytes);
                if (conv) {
                    const int tap = kb / p.conv_chunks, ch = kb - tap * p.conv_chunks;
                    const int cx = x0 + (tap % 3) - 1, cy = y0 + (tap / 3) - 1;
                    tma_load_4d(st, &mapAhi, full_bar + s, ch * BK, cx, cy, tc.bz);
                    if (x3) tma_load_4d(st + 2 * TILE_BYTES, &mapAlo, full_bar + s, ch * BK, cx, cy, tc.bz);
                    tma_load_3d(st + TILE_BYTES, &mapBhi, full_bar + s, kb * BK, n0, 0);
                    if (x3) tma_load_3d(st + 3 * TILE_BYTES, &mapBlo, full_bar + s, kb * BK, n0, 0);
                } else {
                    tma_load_3d(st, &mapAhi, full_bar + s, kb * BK, m0, tc.bz);
                    tma_load_3d(st + TILE_BYTES, &mapBhi, full_bar + s, kb * BK, n0, tc.bz);
                    if (x3) {
                        tma_load_3d(st + 2 * TILE_BYTES, &mapAlo, full_bar + s, kb * BK, m0, tc.bz);
                        tma_load_3d(st + 3 * TILE_BYTES, &mapBlo, full_bar + s, kb * BK, n0, tc.bz);
                    }
                }
            }
        }
        return;
    }

    // ===== consumers: warpgroup wg computes rows [64 wg, 64 wg + 64) of the tile =====
    const int wg = warp >> 2;
    float tot[64], acc[64];
    for (int kb0 = 0; kb0 < num_kb; kb0 += KCHUNK_KB) {
        const int kb1 = min(kb0 + KCHUNK_KB, num_kb);
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        for (int kb = kb0; kb < kb1; ++kb) {
            const int s = kb % p.stages;
            mbar_wait(full_bar + s, (kb / p.stages) & 1);
            const uint32_t st = smem_u32(smem + (size_t)s * stage_bytes);
            const uint64_t dAhi = make_smem_desc(st + wg * (TILE_BYTES / 2)), dBhi = make_smem_desc(st + TILE_BYTES);
            const uint64_t dAlo = make_smem_desc(st + 2 * TILE_BYTES + wg * (TILE_BYTES / 2));
            const uint64_t dBlo = make_smem_desc(st + 3 * TILE_BYTES);
            fence_regs(acc);
            wgmma_fence();
            // +32 B per K step, in 16 B descriptor units; the branch stays outside the MMA chains so that no register
            // traffic separates them
            if (x3) {
#pragma unroll
                for (int k = 0; k < BK / MMA_K; ++k) {
                    const uint64_t adv = (uint64_t)((k * MMA_K * 2) >> 4);
                    wgmma_m64n128k16_ss(acc, dAhi + adv, dBhi + adv);
                    wgmma_m64n128k16_ss(acc, dAhi + adv, dBlo + adv);
                    wgmma_m64n128k16_ss(acc, dAlo + adv, dBhi + adv);
                }
            } else {
#pragma unroll
                for (int k = 0; k < BK / MMA_K; ++k) {
                    const uint64_t adv = (uint64_t)((k * MMA_K * 2) >> 4);
                    wgmma_m64n128k16_ss(acc, dAhi + adv, dBhi + adv);
                }
            }
            wgmma_commit();
            wgmma_wait<1>();                       // the previous k-block's MMAs have retired: release its slot
            fence_regs(acc);
            if (kb > kb0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(empty_bar + (kb - 1) % p.stages);
            }
        }
        wgmma_wait<0>();
        fence_regs(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar + (kb1 - 1) % p.stages);
#pragma unroll
        for (int i = 0; i < 64; ++i) tot[i] = kb0 == 0 ? acc[i] : tot[i] + acc[i];
    }

    // ===== epilogue: restage through shared memory so that a thread owns 64 consecutive columns of one row =====
    // Every load of this tile has landed and been consumed, so the ring is free once both warpgroups are past their MMAs.
    float* stg = reinterpret_cast<float*>(smem);
    asm volatile("bar.sync 1, %0;" ::"n"(NCONSUMER) : "memory");
    {
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
            const int r = r0 + 8 * ((i >> 1) & 1), c = c0 + 8 * (i >> 2);
            *reinterpret_cast<float2*>(stg + r * STG_LD + c) = make_float2(tot[i], tot[i + 1]);
        }
    }
    asm volatile("bar.sync 1, %0;" ::"n"(NCONSUMER) : "memory");
    const int trow = threadIdx.x & (BM - 1), half = threadIdx.x >> 7;
    float out[2][32];
#pragma unroll
    for (int g = 0; g < 2; ++g)
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
            const float4 v = *reinterpret_cast<const float4*>(stg + trow * STG_LD + half * 64 + g * 32 + j);
            out[g][j] = v.x; out[g][j + 1] = v.y; out[g][j + 2] = v.z; out[g][j + 3] = v.w;
        }
    const int zo = tc.bz / p.zdiv, zi = tc.bz % p.zdiv;
    const size_t dbase = (size_t)zo * p.sD2 + (size_t)zi * p.sD;
    const size_t obase = (size_t)zo * p.sO2 + (size_t)zi * p.sO;
    const size_t rbase = (size_t)zo * p.sR2 + (size_t)zi * p.sR;
    // 256-bit row segments need 32 B alignment
    const bool vec_ok = (p.ldd % 8 == 0) && (p.ldr % 8 == 0) && (p.ldo % 16 == 0) &&
                        (((uintptr_t)p.D | (uintptr_t)p.residual | (uintptr_t)p.Dhi | (uintptr_t)p.Dlo) % 32 == 0) &&
                        ((dbase | rbase) % 8 == 0) && (obase % 16 == 0);
    store_row<ROPE>(p, out, trow, conv, x0, y0, m0, n0 + half * 64, dbase, obase, rbase, vec_ok);
}

// ---- host side ----
int encode(CUtensorMap* map, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
           const cuuint32_t* box, const char* what) {
    hopper::EncodeTiledFn fn = hopper::get_encode_fn();
    if (!fn) { adb_set_error_msg("cuTensorMapEncodeTiled driver entry point unavailable"); return ADB_ERR_CUDA; }
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        static char msg[200];
        snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled(%s) failed (%d): dims %llu %llu %llu stride0 %llu", what, (int)r,
                 (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2],
                 (unsigned long long)strides[0]);
        adb_set_error_msg(msg);
        return ADB_ERR_INVALID;
    }
    return ADB_OK;
}

// bf16 tensor [batch][rows][K] with element strides (ld, batch_stride); box = 64 (K) x 128 (rows) x 1
int make_map(CUtensorMap* map, const void* ptr, int rows, int K, long long ld, long long bstride, int batch) {
    cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)rows, (cuuint64_t)batch};
    cuuint64_t strides[2] = {(cuuint64_t)ld * 2, (cuuint64_t)(batch > 1 ? bstride : (long long)rows * ld) * 2};
    cuuint32_t box[3] = {(cuuint32_t)BK, (cuuint32_t)BM, 1};
    return encode(map, ptr, 3, dims, strides, box, "matrix");
}

// bf16 NHWC activation [B][H][W][C]; box = 64 channels x Wb x Hb x 1
int make_map_nhwc(CUtensorMap* map, const void* ptr, int B, int H, int W, int C, int Wb, int Hb) {
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
    cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)Wb, (cuuint32_t)Hb, 1};
    return encode(map, ptr, 4, dims, strides, box, "nhwc");
}

int launch(const CUtensorMap& mAhi, const CUtensorMap& mAlo, const CUtensorMap& mBhi, const CUtensorMap& mBlo,
           GemmParams& p, long long num_tiles, cudaStream_t stream) {
    ADB_REQUIRE(num_tiles < 2147483647LL, "adb_gemm_bf16: too many output tiles");
    p.stages = RING_BYTES / ((p.nterms == 3 ? 4 : 2) * TILE_BYTES);
    static AdbDeviceOnce once;
    {
        const int rc = once.ensure([]() -> int {
            ADB_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
            ADB_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
            return ADB_OK;
        });
        if (rc != ADB_OK) return rc;
    }
    if (p.rope_ndst > 0) gemm_tc_kernel<true><<<(unsigned)num_tiles, NTHREADS, SMEM_BYTES, stream>>>(mAhi, mAlo, mBhi, mBlo, p);
    else gemm_tc_kernel<false><<<(unsigned)num_tiles, NTHREADS, SMEM_BYTES, stream>>>(mAhi, mAlo, mBhi, mBlo, p);
    ADB_CHECK_LAUNCH("gemm_tc_kernel");
    return ADB_OK;
}

}  // namespace

// D[z] (fp32, optional) / Dhi,Dlo[z] (bf16 split, optional) = act(alpha * A[z] * B[z]^T + bias) + residual[z]
//   A: bf16 [batch][M][K] (ld = lda elements, batch stride sA), B: bf16 [batch][N][K] (ldb, sB); both K-contiguous,
//   16-byte aligned, lda/ldb multiples of 8.  A_lo and B_lo both non-NULL selects the 3-term bf16x3 product.
//   act: 0 none, 1 GELU (erf), 2 ReLU.  Output batch addressing: z = z_outer * zdiv + z_inner and the
//   output/residual offset is z_outer * s?2 + z_inner * s? (zdiv <= 0: plain z * s?), which lets a [B*h] attention
//   batch write straight into a [B, N, h*64] activation.
ADB_API int adb_gemm_bf16(int batch, int M, int N, int K, const void* A_hi, const void* A_lo, long long lda,
                          long long sA, const void* B_hi, const void* B_lo, long long ldb, long long sB, float* D,
                          long long ldd, long long sD, void* D_hi, void* D_lo, long long ldo, long long sO,
                          const float* bias, const float* residual, long long ldr, long long sR, float alpha, int act,
                          int zdiv, long long sD2, long long sO2, long long sR2, cudaStream_t stream) {
    ADB_REQUIRE(batch >= 1 && M >= 1 && N >= 1 && K >= 1, "adb_gemm_bf16: bad sizes");
    ADB_REQUIRE(A_hi && B_hi && (D || D_hi), "adb_gemm_bf16: null pointer");
    ADB_REQUIRE((A_lo == nullptr) == (B_lo == nullptr), "adb_gemm_bf16: A_lo and B_lo must be given together");
    ADB_REQUIRE(lda % 8 == 0 && ldb % 8 == 0 && sA % 8 == 0 && sB % 8 == 0, "adb_gemm_bf16: strides must be multiples of 8 elements");
    ADB_REQUIRE(((uintptr_t)A_hi % 16 == 0) && ((uintptr_t)B_hi % 16 == 0), "adb_gemm_bf16: operands must be 16-byte aligned");
    ADB_REQUIRE(act >= 0 && act <= 2, "adb_gemm_bf16: unknown activation");
    ADB_REQUIRE(sB != 0 || batch == 1, "adb_gemm_bf16: weight broadcast over batch > 1: fold the batch into M instead");
    GemmParams p{};
    p.nterms = A_lo ? 3 : 1;
    CUtensorMap mAhi, mAlo, mBhi, mBlo;
    int rc;
    if ((rc = make_map(&mAhi, A_hi, M, K, lda, sA, batch))) return rc;
    if ((rc = make_map(&mBhi, B_hi, N, K, ldb, sB, batch))) return rc;
    mAlo = mAhi; mBlo = mBhi;
    if (p.nterms == 3) {
        if ((rc = make_map(&mAlo, A_lo, M, K, lda, sA, batch))) return rc;
        if ((rc = make_map(&mBlo, B_lo, N, K, ldb, sB, batch))) return rc;
    }
    p.M = M; p.N = N; p.K = K; p.batch = batch;
    p.D = D; p.ldd = ldd; p.sD = sD;
    p.Dhi = (__nv_bfloat16*)D_hi; p.Dlo = (__nv_bfloat16*)D_lo; p.ldo = ldo; p.sO = sO;
    p.bias = bias; p.residual = residual; p.ldr = ldr; p.sR = sR;
    p.alpha = alpha; p.act = act; p.split_relu = 0;
    p.zdiv = zdiv > 0 ? zdiv : (1 << 30); p.sD2 = sD2; p.sO2 = sO2; p.sR2 = sR2;
    p.conv_wb = 0;
    const long long tiles = (long long)adb_cdiv(M, BM) * adb_cdiv(N, BN) * batch;
    return launch(mAhi, mAlo, mBhi, mBlo, p, tiles, stream);
}

// Linear layer whose leading output columns are attention heads: y = A W^T + bias with
//   columns [0, n_rope_dst*C)   (C = heads*64)  rotated by RoPE2D (table lookup by the token's (y,x) position), split into
//                               bf16 (hi, lo) and written head-major [B*heads, ntok, 64] to q (section 0) / k (section 1);
//   columns [n_rope_dst*C, N)   written as plain fp32 to D[row * ldd + (col - n_rope_dst*C)]  (the V projection).
// Replaces  qkv = Linear(x); q, k = rope(q), rope(k)  (croco/models/blocks.py:94-103, 150-160) + the head transposes:
// the [rows, 3C] fp32 tensor is never written.  M = B * ntok rows.
ADB_API int adb_gemm_bf16_rope(int M, int N, int K, const void* A_hi, const void* A_lo, long long lda, const void* B_hi,
                               const void* B_lo, long long ldb, const float* bias, int ntok, int heads, int n_rope_dst,
                               const long long* pos, const float* table, int n_pos, void* q_hi, void* q_lo, void* k_hi,
                               void* k_lo, float* D_tail, long long ldd, cudaStream_t stream) {
    ADB_REQUIRE(M >= 1 && N >= 1 && K >= 1 && ntok >= 1 && heads >= 1 && M % ntok == 0, "adb_gemm_bf16_rope: bad sizes");
    ADB_REQUIRE(n_rope_dst == 1 || n_rope_dst == 2, "adb_gemm_bf16_rope: n_rope_dst must be 1 or 2");
    const int C = heads * 64;
    ADB_REQUIRE(N >= n_rope_dst * C, "adb_gemm_bf16_rope: N smaller than the rotated sections");
    ADB_REQUIRE(A_hi && B_hi && pos && table && n_pos >= 1 && q_hi && (n_rope_dst == 1 || k_hi), "adb_gemm_bf16_rope: null pointer");
    ADB_REQUIRE((N == n_rope_dst * C) || D_tail, "adb_gemm_bf16_rope: tail columns need D_tail");
    ADB_REQUIRE((A_lo == nullptr) == (B_lo == nullptr), "adb_gemm_bf16_rope: A_lo and B_lo must be given together");
    ADB_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, "adb_gemm_bf16_rope: strides must be multiples of 8 elements");
    ADB_REQUIRE(((uintptr_t)A_hi % 16 == 0) && ((uintptr_t)B_hi % 16 == 0) && ((uintptr_t)table % 16 == 0) &&
                (((uintptr_t)q_hi | (uintptr_t)q_lo | (uintptr_t)k_hi | (uintptr_t)k_lo) % 32 == 0),
                "adb_gemm_bf16_rope: operands must be 16-byte (outputs 32-byte) aligned");
    GemmParams p{};
    p.nterms = A_lo ? 3 : 1;
    CUtensorMap mAhi, mAlo, mBhi, mBlo;
    int rc;
    if ((rc = make_map(&mAhi, A_hi, M, K, lda, 0, 1))) return rc;
    if ((rc = make_map(&mBhi, B_hi, N, K, ldb, 0, 1))) return rc;
    mAlo = mAhi; mBlo = mBhi;
    if (p.nterms == 3) {
        if ((rc = make_map(&mAlo, A_lo, M, K, lda, 0, 1))) return rc;
        if ((rc = make_map(&mBlo, B_lo, N, K, ldb, 0, 1))) return rc;
    }
    p.M = M; p.N = N; p.K = K; p.batch = 1;
    p.D = D_tail ? D_tail - (long long)n_rope_dst * C : nullptr;   // column c of the GEMM lands at D_tail[c - n_rope_dst*C]
    p.ldd = ldd; p.sD = 0;
    p.Dhi = nullptr; p.Dlo = nullptr; p.ldo = N; p.sO = 0;
    p.bias = bias; p.residual = nullptr; p.ldr = N; p.sR = 0;
    p.alpha = 1.0f; p.act = 0; p.split_relu = 0;
    p.zdiv = 1 << 30; p.sD2 = p.sO2 = p.sR2 = 0;
    p.conv_wb = 0;
    p.rope_ndst = n_rope_dst; p.rope_C = C; p.rope_heads = heads; p.rope_ntok = ntok; p.rope_npos = n_pos;
    p.rope_pos = pos; p.rope_table = table;
    p.rope_hi[0] = (__nv_bfloat16*)q_hi; p.rope_lo[0] = (__nv_bfloat16*)q_lo;
    p.rope_hi[1] = (__nv_bfloat16*)k_hi; p.rope_lo[1] = (__nv_bfloat16*)k_lo;
    const long long tiles = (long long)adb_cdiv(M, BM) * adb_cdiv(N, BN);
    return launch(mAhi, mAlo, mBhi, mBlo, p, tiles, stream);
}

// 3x3 / stride 1 / zero-pad 1 convolution as an implicit GEMM (replaces the nn.Conv2d(k=3) calls of
// croco/models/dpt_block.py:20-77,93-112,368-372):
//   x: bf16 split NHWC [B, H, W, Cin] (Cin % 8 == 0);  w: bf16 split [Cout][9 * Cin_pad], tap-major (ky, kx, ci),
//   Cin_pad = Cin rounded up to 64 with zero fill;  outputs are NHWC [B*H*W, Cout] (fp32 D and/or bf16 split).
//   residual: fp32 NHWC [B*H*W, Cout] or NULL.  act: 0 none, 2 ReLU.  split_relu: split output stores relu(value).
ADB_API int adb_conv3x3_bf16(int B, int H, int W, int Cin, int Cout, const void* x_hi, const void* x_lo,
                             const void* w_hi, const void* w_lo, const float* bias, const float* residual, float* D,
                             void* D_hi, void* D_lo, int act, int split_relu, cudaStream_t stream) {
    ADB_REQUIRE(B >= 1 && H >= 1 && W >= 1 && Cin >= 8 && Cout >= 1, "adb_conv3x3_bf16: bad sizes");
    ADB_REQUIRE(Cin % 8 == 0, "adb_conv3x3_bf16: Cin must be a multiple of 8");
    ADB_REQUIRE(x_hi && w_hi && (D || D_hi), "adb_conv3x3_bf16: null pointer");
    ADB_REQUIRE((x_lo == nullptr) == (w_lo == nullptr), "adb_conv3x3_bf16: x_lo and w_lo must be given together");
    ADB_REQUIRE(act == 0 || act == 2, "adb_conv3x3_bf16: act must be 0 or 2 (ReLU)");
    ADB_REQUIRE((((uintptr_t)x_hi | (uintptr_t)x_lo | (uintptr_t)w_hi | (uintptr_t)w_lo) % 16) == 0,
                "adb_conv3x3_bf16: operands must be 16-byte aligned");
    GemmParams p{};
    p.nterms = x_lo ? 3 : 1;
    int wb = 128;
    while (wb > W && wb > 8) wb >>= 1;          // widest power-of-two row segment that fits the image row
    const int hb = BM / wb;
    const int chunks = (Cin + BK - 1) / BK;
    const int Kpad = 9 * chunks * BK;
    CUtensorMap mAhi, mAlo, mBhi, mBlo;
    int rc;
    if ((rc = make_map_nhwc(&mAhi, x_hi, B, H, W, Cin, wb, hb))) return rc;
    if ((rc = make_map(&mBhi, w_hi, Cout, Kpad, Kpad, 0, 1))) return rc;
    mAlo = mAhi; mBlo = mBhi;
    if (p.nterms == 3) {
        if ((rc = make_map_nhwc(&mAlo, x_lo, B, H, W, Cin, wb, hb))) return rc;
        if ((rc = make_map(&mBlo, w_lo, Cout, Kpad, Kpad, 0, 1))) return rc;
    }
    p.M = H * W; p.N = Cout; p.K = Kpad; p.batch = B;
    p.D = D; p.ldd = Cout; p.sD = (long long)H * W * Cout;
    p.Dhi = (__nv_bfloat16*)D_hi; p.Dlo = (__nv_bfloat16*)D_lo; p.ldo = Cout; p.sO = (long long)H * W * Cout;
    p.bias = bias; p.residual = residual; p.ldr = Cout; p.sR = (long long)H * W * Cout;
    p.alpha = 1.0f; p.act = act; p.split_relu = split_relu;
    p.zdiv = 1 << 30; p.sD2 = p.sO2 = p.sR2 = 0;
    p.conv_wb = wb; p.conv_hb = hb; p.conv_H = H; p.conv_W = W; p.conv_chunks = chunks;
    p.conv_tiles_x = adb_cdiv(W, wb); p.conv_tiles_y = adb_cdiv(H, hb);
    const long long tiles = (long long)p.conv_tiles_x * p.conv_tiles_y * adb_cdiv(Cout, BN) * B;
    return launch(mAhi, mAlo, mBhi, mBlo, p, tiles, stream);
}

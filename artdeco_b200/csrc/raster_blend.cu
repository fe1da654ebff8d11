// Per-tile alpha blending, forward and backward (RGB + depth = 4 channels).
//
// Replaces gsplat's rasterize_to_pixels fwd/bwd that the reference reaches through
// Reconstruct/scene/scene_models/h3dgsv3.py:664-680 (SURVEY.md App. B.4 / B.5):
//   pixel centre (j+0.5, i+0.5); sigma = .5(a dx^2 + c dy^2) + b dx dy; alpha = min(.999, o exp(-sigma));
//   skip if sigma<0 or alpha<1/255; stop when T(1-alpha) <= 1e-4; out += feat*alpha*T; alpha_out = 1-T.
//
// Both kernels are INSTRUCTION-ISSUE bound on this workload (one 48 B record is reused by up to 256 pixels; DRAM
// utilisation is ~2 %), so the design minimises issued instructions per (warp, splat) evaluation:
//  * one CTA per 16x16 tile, 8 warps, each warp owns an 8x4 pixel block (the 32-lane shape with the best lane occupancy
//    on small splats: 51 % of the lanes of an evaluated (warp, splat) pair contribute at the BASELINE workload);
//  * the tile's slice of the depth-sorted list is staged 256 splats at a time as 48 B shared-memory records, the conic
//    pre-scaled by log2(e)/2 so that sigma is 5 FP32 ops and alpha is one MUFU.EX2 without a range-reduction multiply;
//  * CULLING AT STAGING: the thread that stages a record also computes its 8-bit warp mask (which of the tile's eight 8x4
//    blocks the ellipse sigma <= ln(255 o) can reach, intersected with the integer-radius box; see warp_mask).  Each warp
//    then compacts the slots carrying its bit into a private 16-bit hit list with one ballot per 32 slots, padded to a
//    multiple of four with a never-visible dummy record so the evaluation loop is unrolled by four with one LDS.64 of list
//    entries and no remainder code;
//  * the evaluation bodies are branch-free (predicated selects), so the four unrolled bodies interleave;
//  * BACKWARD — the per-splat reduction over the warp's 32 pixels is NOT a shuffle butterfly.  All ten per-Gaussian
//    sums are dot products of two per-(pixel,splat) scalars with weights that do not depend on the splat:
//        raw moments  sum_p vs(p) * {1, lx, ly, lx^2, lx ly, ly^2}   (vs = dL/dsigma, lx/ly = pixel offset in the block)
//        feature grads sum_p fac(p) * v_out[p][0..3]                  (fac = alpha*T)
//    i.e. a [slots x 32 pixels] x [32 x 10] product.  A lane therefore stores just (vs, fac) per evaluation (one STS.64)
//    into a per-warp slot buffer; every SLOTS evaluations the warp transposes roles (lane = slot), streams the slot's row
//    with LDS.128, applies the lane-constant integer weights as immediates (row sums first: 7.75 FMA per pixel
//    instead of 10) and converts the block-origin moments to splat-centred ones once per (warp, splat):
//        sum vs dx = ex S0 - Sx,  sum vs dx^2 = ex (ex S0 - 2 Sx) + Sxx, ...   (ex = mean_x - block origin)
//    About 11 issued instructions per evaluation against ~55 for the packed butterfly + shared atomics it replaces, and
//    the nine moment/feature multiplies leave the per-pixel body as well;
//  * results leave with three 128/64-bit vector REDs per (warp, splat) (red.global.add.v4.f32).
#include "raster_common.cuh"

namespace {

constexpr int BLOCK = ADB_TILE * ADB_TILE;  // 256
constexpr int NWARP = BLOCK / 32;
constexpr unsigned FULL = 0xffffffffu;
constexpr int DUMMY = BLOCK;                // index of the never-visible padding record
constexpr int LIST_STRIDE = BLOCK + 8;      // u16 entries per warp (padding to a multiple of 4 fits)
constexpr float LOG2E = 1.4426950408889634f;

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ float sqrt_approx(float x) {
    float y;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Warp mask of a staged record (A, B as in stage_record) over the tile whose first pixel centre is (tx0, ty0): bit w is set
// when the splat can pass the per-pixel test 0 <= sigma2 <= smax2 somewhere in warp w's 8x4 block, i.e. pixel centres
// x in tx0 + 8 (w & 1) + [0, 7], y in ty0 + 4 (w >> 1) + [0, 3].  Two conservative tests, ANDed:
//  1. the integer-radius box written by the projection (outside it alpha < 1/255 by construction of the radius);
//  2. per 4-pixel row band, the x-interval of the ellipse {sigma2 <= S} over the band's continuous y-range against the two
//     column halves.  For a row offset e = y - my the ellipse's x-range is mx + (-b2 e -+ sqrt(4 ha S - D e^2)) / (2 ha),
//     D = 4 ha hc - b2^2; the right end is concave in e, so its maximum over the band is at its stationary point (the
//     ellipse's rightmost point, e = -b2 xm / (2 hc) with xm the x half-extent) clamped to the band, the left end likewise.
// S is smax2 widened by the rounding error of the per-pixel fp32 sigma2 (terms up to kappa = 4 ha hc / D times sigma2 cancel
// in it) plus relative and absolute slack, and the band and the interval are widened by the rounding of the coordinates, so
// the mask keeps every block that holds a pixel passing the per-pixel test: the image is the same as with no culling.
// A conic that is not positive definite, or too ill-conditioned to bound its rounding, falls back to the box.
// About 110 thread-instructions per record, computed once by the staging thread instead of by every warp.
__device__ __forceinline__ unsigned warp_mask(const float4& A, const float4& B, float tx0, float ty0) {
    const unsigned pr = __float_as_uint(B.w);
    // 65535 is the saturation value written by the projection: treat it as unbounded
    const float rx = (pr & 0xffffu) == 0xffffu ? 3.0e38f : (float)(pr & 0xffffu);
    const float ry = (pr >> 16) == 0xffffu ? 3.0e38f : (float)(pr >> 16);
    const float mx = A.x, my = A.y, ha = A.z, b = A.w, hc = B.x;
    const float D = 4.f * ha * hc - b * b;
    const float kap = __fdividef(4.f * ha * hc, D);
    const bool conic_ok = ha > 0.f && hc > 0.f && D > 0.f && kap < 1.0e6f;
    const float S = fmaxf(0.f, B.z * (1.0002f + 2.0e-6f * kap) + 2.0e-4f);
    const float pad = 1.0e-3f + 2.0e-6f * fmaxf(fabsf(mx), fabsf(my));
    const float rD = rcp_approx(D);
    const float S4a = 4.f * ha * S;
    const float xm = sqrt_approx(4.f * hc * S * rD), ym = sqrt_approx(S4a * rD);
    const float eR = -0.5f * b * xm * rcp_approx(hc);              // row offset of the rightmost point; leftmost at -eR
    const float r2a = rcp_approx(2.f * ha);
    unsigned mask = 0u;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const float xlo = tx0 + 8.f * h, xhi = xlo + 7.f;
        const unsigned cols = (mx + rx >= xlo && mx - rx <= xhi) ? (0x55u << h) : 0u;
        mask |= cols;
    }
    unsigned rows = 0u;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float ylo = ty0 + 4.f * k, yhi = ylo + 3.f;
        if (!(my + ry >= ylo && my - ry <= yhi)) continue;
        if (!conic_ok) { rows |= 3u << (2 * k); continue; }
        const float e0 = ylo - my - pad, e1 = yhi - my + pad;
        if (e0 > ym || e1 < -ym) continue;
        const float cR = fminf(e1, fmaxf(e0, eR)), cL = fminf(e1, fmaxf(e0, -eR));
        const float xR = mx + (sqrt_approx(fmaxf(0.f, S4a - D * cR * cR)) - b * cR) * r2a + pad;
        const float xL = mx - (sqrt_approx(fmaxf(0.f, S4a - D * cL * cL)) + b * cL) * r2a - pad;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const float xlo = tx0 + 8.f * h, xhi = xlo + 7.f;
            if (xL <= xhi && xR >= xlo) rows |= 1u << (2 * k + h);
        }
    }
    return mask & rows;
}

// Shared-memory record (3 x float4, 48 B stride: conflict-free for both the staging stores and the broadcast loads):
//   A = (mx, my, ha, b2)   B = (hc, opacity, smax2, bits rx|ry<<16)   C = (r, g, b, depth | 1/depth for LEGACY)
// with ha = log2e * a/2, b2 = log2e * b, hc = log2e * c/2, smax2 = log2e * ln(255 o) (the projection's margin removed):
//   sigma2 = log2e * sigma = dx (ha dx + b2 dy) + hc dy^2,   alpha = o * 2^(-sigma2),
//   and  alpha >= 1/255  <=>  sigma2 <= smax2  — one compare replaces the alpha test (the two differ only where
//   o 2^(-sigma2) is within an ulp of 1/255, the same measure-zero band in which ex2.approx and the oracle's expf disagree).
// When `mask` is not NULL it receives the record's warp mask over the tile whose first pixel centre is (tx0, ty0).
template <bool LEGACY>
__device__ __forceinline__ void stage_record(float4* __restrict__ rec, const float* __restrict__ splats, int g,
                                             unsigned char* __restrict__ mask, float tx0, float ty0) {
    const float4* p = reinterpret_cast<const float4*>(splats + (size_t)g * ADB_SPLAT_STRIDE);
    float4 A = __ldg(p), B = __ldg(p + 1), C = __ldg(p + 2);
    A.z *= 0.5f * LOG2E;
    A.w *= LOG2E;
    B.x *= 0.5f * LOG2E;
    B.z = (B.z - ADB_SIGMA_MARGIN) * LOG2E;   // exact bound: alpha >= 1/255  <=>  sigma <= ln(255 o)
    if (LEGACY) C.w = 1.0f / C.w;   // Inria: 4th channel blends 1/z (v_splats slot 9 is then dL/d(1/z))
    rec[0] = A;
    rec[1] = B;
    rec[2] = C;
    if (mask) *mask = (unsigned char)warp_mask(A, B, tx0, ty0);
}

__device__ __forceinline__ void write_dummy(float4* __restrict__ rec) {
    rec[0] = make_float4(0.f, 0.f, 0.f, 0.f);
    rec[1] = make_float4(0.f, 0.f, -1.0f, 0.f);  // smax2 = -1: fails "0 <= sigma2 <= smax2" for every pixel
    rec[2] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// A warp's hit list from the staged batch's warp masks (sM[slot], bit w = warp w's block is hit), ascending slot order,
// padded to a multiple of 4 with DUMMY.  `limit`: only slots s >= limit are considered (the backward skips splats behind
// the warp's last contributor).
__device__ __forceinline__ int build_hit_list_from_mask(const unsigned char* __restrict__ sM, unsigned short* __restrict__ list,
                                                        int bsize, int limit, int warp, int lane) {
    const unsigned lt_mask = (1u << lane) - 1u;
    int nhit = 0;
    for (int c0 = (limit > 0 ? (limit & ~31) : 0); c0 < bsize; c0 += 32) {
        const int s = c0 + lane;
        const bool hit = s < bsize && s >= limit && ((sM[s] >> warp) & 1u);
        const unsigned mask = __ballot_sync(FULL, hit);
        if (hit) list[nhit + __popc(mask & lt_mask)] = (unsigned short)s;
        nhit += __popc(mask);
    }
    __syncwarp();
    if (lane < 3) list[nhit + lane] = (unsigned short)DUMMY;
    __syncwarp();
    return nhit;
}

// Record index of a sorted value: the multi-view entry points index the stacked [C,N,12] records with vals (= cam*N + g)
// directly (wrap = 0); the single-view ones pass wrap = N, because their vals may carry a camera offset while `splats` holds
// that one camera's records.
__device__ __forceinline__ int record_index(int v, int wrap) { return wrap ? v % wrap : v; }

// Views: blockIdx.z = view c.  tile_offsets [C][T+1] are absolute indices into vals / hit_mask; colors / alphas / last_ids /
// main_ids are [C,H,W,...] stacks.
// LEGACY = Inria conventions (ADB_CONV_INRIA): alpha <= 0.99, stop when T(1-alpha) < 1e-4 (strict), 4th channel
// accumulates 1/z, and main_ids gets the Gaussian with the largest blending weight alpha*T per pixel (-1: none).
template <bool LEGACY>
__global__ void __launch_bounds__(BLOCK, 4)
blend_fwd_kernel(int W, int H, const float* __restrict__ splats, const int32_t* __restrict__ vals,
                 const int32_t* __restrict__ tile_offsets, int wrap,
                 float* __restrict__ colors, float* __restrict__ alphas, int32_t* __restrict__ last_ids,
                 int32_t* __restrict__ main_ids, unsigned char* __restrict__ hit_mask) {
    constexpr float MAXA = LEGACY ? ADB_MAX_ALPHA_INRIA : ADB_MAX_ALPHA;
    __shared__ __align__(16) float4 sRec[(BLOCK + 1) * 3];
    __shared__ __align__(8) unsigned short sList[NWARP][LIST_STRIDE];
    __shared__ unsigned char sM[BLOCK];         // warp masks of the staged batch

    const int tw = (W + ADB_TILE - 1) / ADB_TILE;
    const int tile = blockIdx.y * tw + blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int x0 = blockIdx.x * ADB_TILE + (warp & 1) * 8, y0 = blockIdx.y * ADB_TILE + (warp >> 1) * 4;
    const int j = x0 + (lane & 7), i = y0 + (lane >> 3);
    const bool inside = (i < H && j < W);
    const float px = (float)j + 0.5f, py = (float)i + 0.5f;
    const float tx0 = (float)(blockIdx.x * ADB_TILE) + 0.5f, ty0 = (float)(blockIdx.y * ADB_TILE) + 0.5f;
    const size_t view_pix = (size_t)blockIdx.z * H * W;
    const int orow = blockIdx.z * (gridDim.x * gridDim.y + 1) + tile;
    const int start = tile_offsets[orow], end = tile_offsets[orow + 1];
    if (tid == 0) write_dummy(sRec + DUMMY * 3);
    const int nb = (end - start + BLOCK - 1) / BLOCK;

    float T = 1.0f;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int cur = 0;
    float best_w = 0.f;
    int best_k = -1;
    bool done = !inside;
    for (int b = 0; b < nb; ++b) {
        const int n_done = __syncthreads_count(done);    // also: every warp has finished reading the previous batch
        const int bstart = start + b * BLOCK;
        const int idx = bstart + tid;
        if (n_done >= BLOCK) break;
        if (idx < end) {
            stage_record<LEGACY>(sRec + tid * 3, splats, record_index(vals[idx], wrap), sM + tid, tx0, ty0);
            if (hit_mask) hit_mask[idx] = sM[tid];
        }
        __syncthreads();
        const int bsize = min(BLOCK, end - bstart);
        if (__all_sync(FULL, done)) continue;
        unsigned short* list = sList[warp];
        const int nhit = build_hit_list_from_mask(sM, list, bsize, 0, warp, lane);
        int cur_t = -1;
        const int nq = (nhit + 3) >> 2;
        for (int q = 0; q < nq; ++q) {
            const uint2 pk = *reinterpret_cast<const uint2*>(list + 4 * q);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const unsigned w32 = (u < 2) ? pk.x : pk.y;
                const int t = (u & 1) ? (int)(w32 >> 16) : (int)(w32 & 0xffffu);
                const float4 A = sRec[t * 3], B = sRec[t * 3 + 1], C = sRec[t * 3 + 2];
                const float dx = A.x - px, dy = A.y - py;
                const float s2 = dx * (A.z * dx + A.w * dy) + (B.x * dy) * dy;
                const float alpha = fminf(MAXA, B.y * ex2_approx(-s2));
                const bool ok = !done && s2 >= 0.f && s2 <= B.z;
                const float nT = fmaf(-T, alpha, T);
                const bool stop = ok && (LEGACY ? (nT < ADB_T_EPS) : (nT <= ADB_T_EPS));
                const bool take = ok && !stop;
                done = done || stop;
                const float w = take ? alpha * T : 0.f;
                acc.x = fmaf(C.x, w, acc.x);
                acc.y = fmaf(C.y, w, acc.y);
                acc.z = fmaf(C.z, w, acc.z);
                acc.w = fmaf(C.w, w, acc.w);
                cur_t = take ? t : cur_t;
                if (LEGACY && w > best_w) { best_w = w; best_k = bstart + t; }
                T = take ? nT : T;
            }
            if ((q & 1) && __all_sync(FULL, done)) break;
        }
        if (cur_t >= 0) cur = bstart + cur_t;
    }
    if (inside) {
        const size_t pix = view_pix + (size_t)i * W + j;
        reinterpret_cast<float4*>(colors)[pix] = acc;
        alphas[pix] = 1.0f - T;
        last_ids[pix] = cur;
        if (LEGACY && main_ids) main_ids[pix] = best_k >= 0 ? record_index(vals[best_k], wrap) : -1;
    }
}

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// Slots per warp in the backward's deferred-reduction buffer: 32 would fit only 2 CTAs/SM.
constexpr int SLOTS = 16;

// Backward shared-memory layout (dynamic).
struct BwdSmem {
    static constexpr int ROW4 = 17;                       // float4 per slot row: 32 x (vs, fac) + 1 pad -> conflict-free
    static constexpr int OFF_REC = 0;                                         // float4 [(BLOCK+1)*3]
    static constexpr int OFF_G = OFF_REC + (BLOCK + 1) * 3 * 16;              // int [BLOCK + 4]
    static constexpr int OFF_M = OFF_G + (BLOCK + 4) * 4;                     // u8 [BLOCK]: the forward's warp masks of the batch
    static constexpr int OFF_LIST = OFF_M + BLOCK;                            // u16 [NWARP][LIST_STRIDE]
    static constexpr int OFF_VO = OFF_LIST + NWARP * LIST_STRIDE * 2;         // float4 [NWARP][32]
    static constexpr int OFF_V = OFF_VO + NWARP * 32 * 16;                    // float4 [NWARP][SLOTS*ROW4]
    static constexpr int BYTES = OFF_V + NWARP * SLOTS * ROW4 * 16;
    static_assert(OFF_G % 16 == 0 && OFF_LIST % 16 == 0 && OFF_VO % 16 == 0 && OFF_V % 16 == 0, "alignment");
};

// The default build fits 4 CTAs/SM (64 registers); the legacy build is bounded for 3.
template <bool LEGACY>
__global__ void __launch_bounds__(BLOCK, LEGACY ? 3 : 4)
blend_bwd_kernel(int W, int H, const float* __restrict__ splats, const int32_t* __restrict__ vals,
                 const int32_t* __restrict__ tile_offsets, int wrap,
                 const float* __restrict__ alphas, const int32_t* __restrict__ last_ids,
                 const float* __restrict__ v_colors, const float* __restrict__ v_alphas,
                 float* __restrict__ v_splats, const unsigned char* __restrict__ hit_mask) {
    constexpr float MAXA = LEGACY ? ADB_MAX_ALPHA_INRIA : ADB_MAX_ALPHA;
    using L = BwdSmem;
    extern __shared__ __align__(16) unsigned char smem[];
    float4* sRec = reinterpret_cast<float4*>(smem + L::OFF_REC);
    int* sG = reinterpret_cast<int*>(smem + L::OFF_G);
    unsigned char* sM = smem + L::OFF_M;

    const int tw = (W + ADB_TILE - 1) / ADB_TILE;
    const int tile = blockIdx.y * tw + blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    unsigned short* list = reinterpret_cast<unsigned short*>(smem + L::OFF_LIST) + warp * LIST_STRIDE;
    float4* sVo = reinterpret_cast<float4*>(smem + L::OFF_VO) + warp * 32;
    float4* sV = reinterpret_cast<float4*>(smem + L::OFF_V) + warp * SLOTS * L::ROW4;
    const int x0 = blockIdx.x * ADB_TILE + (warp & 1) * 8, y0 = blockIdx.y * ADB_TILE + (warp >> 1) * 4;
    const int j = x0 + (lane & 7), i = y0 + (lane >> 3);
    const bool inside = (i < H && j < W);
    const float px = (float)j + 0.5f, py = (float)i + 0.5f;
    const float tx0 = (float)(blockIdx.x * ADB_TILE) + 0.5f, ty0 = (float)(blockIdx.y * ADB_TILE) + 0.5f;
    // view row of tile_offsets by a 32-bit index (a 64-bit pointer bump here costs the 64-register build one more spill slot)
    const int orow = blockIdx.z * (gridDim.x * gridDim.y + 1) + tile;
    const int start = tile_offsets[orow], end = tile_offsets[orow + 1];
    if (end <= start) return;

    const size_t pix = (size_t)blockIdx.z * H * W + (size_t)(inside ? i : 0) * W + (inside ? j : 0);
    const float T_final = inside ? 1.0f - alphas[pix] : 1.0f;
    const int bin_final = inside ? last_ids[pix] : -1;
    const float4 vo = inside ? reinterpret_cast<const float4*>(v_colors)[pix] : make_float4(0.f, 0.f, 0.f, 0.f);
    const float va = inside ? v_alphas[pix] : 0.f;
    float T = T_final;
    float bv = 0.f;
    const float Tva = T_final * va;
    sVo[lane] = vo;
    if (tid == 0) {
        write_dummy(sRec + DUMMY * 3);
        sG[DUMMY] = 0;
    }

    int warp_bin_final = bin_final;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) warp_bin_final = max(warp_bin_final, __shfl_xor_sync(FULL, warp_bin_final, o));

    // reduction-phase role of this lane: slot r_slot, pixel rows [2*r_half, +2) of the warp's 8x4 block
    const int r_slot = lane & (SLOTS - 1), r_half = lane / SLOTS;
    const float4* r_row = sV + r_slot * L::ROW4 + r_half * 8;
    const float4* r_vo = sVo + r_half * 16;
    float2* my_cell = reinterpret_cast<float2*>(sV) + lane;          // + slot * ROW4 * 2 (float2 units)

    const int nb = (end - start + BLOCK - 1) / BLOCK;
    for (int b = 0; b < nb; ++b) {
        __syncthreads();  // previous batch fully consumed
        const int batch_end = end - 1 - b * BLOCK;           // smem slot t <-> sorted index batch_end - t (back to front)
        const int bsize = min(BLOCK, batch_end + 1 - start);
        const int idx = batch_end - tid;
        if (idx >= start) {
            const int g = record_index(vals[idx], wrap);
            sG[tid] = g;
            stage_record<LEGACY>(sRec + tid * 3, splats, g, hit_mask ? nullptr : sM + tid, tx0, ty0);
            if (hit_mask) sM[tid] = hit_mask[idx];
        }
        __syncthreads();
        // a splat at slot s contributes to this warp only if batch_end - s <= warp_bin_final
        const int limit = max(0, batch_end - warp_bin_final);
        if (limit >= bsize) continue;
        const int nhit = build_hit_list_from_mask(sM, list, bsize, limit, warp, lane);
        const int tmin = inside ? batch_end - bin_final : (1 << 30);   // lane-valid iff t >= tmin
        for (int g0 = 0; g0 < nhit; g0 += SLOTS) {
            const int ng = min(SLOTS, nhit - g0);
            const int nq = (ng + 3) >> 2;
            for (int q = 0; q < nq; ++q) {
                const uint2 pk = *reinterpret_cast<const uint2*>(list + g0 + 4 * q);
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const unsigned w32 = (u < 2) ? pk.x : pk.y;
                    const int t = (u & 1) ? (int)(w32 >> 16) : (int)(w32 & 0xffffu);
                    const float4 A = sRec[t * 3], B = sRec[t * 3 + 1], C = sRec[t * 3 + 2];
                    const float dx = A.x - px, dy = A.y - py;
                    const float s2 = dx * (A.z * dx + A.w * dy) + (B.x * dy) * dy;
                    const float ov = B.y * ex2_approx(-s2);
                    const float am = fminf(MAXA, ov);
                    const bool valid = t >= tmin && s2 >= 0.f && s2 <= B.z;
                    // An invalid lane runs with alpha = 0, which leaves T and bv unchanged (ra = 1, fac = 0) and
                    // contributes exact zeros to every sum.
                    const float alpha = valid ? am : 0.f;
                    const float ra = rcp_approx(1.0f - alpha);
                    T *= ra;
                    const float fac = alpha * T;
                    // cv = <feat, v_out>;  bv = sum over later splats of fac*cv  (the scalar the 4-channel "buffer" of
                    // the textbook backward collapses to once it is dotted with v_out)
                    const float cv = fmaf(C.x, vo.x, fmaf(C.y, vo.y, fmaf(C.z, vo.z, C.w * vo.w)));
                    const float v_alpha = fmaf(cv, T, (Tva - bv) * ra);
                    bv = fmaf(fac, cv, bv);
                    // d(alpha)/d(sigma) = -o exp(-sigma); the path is cut where alpha was clamped
                    const float nov = (valid && ov <= MAXA) ? -ov : 0.f;
                    my_cell[(4 * q + u) * (L::ROW4 * 2)] = make_float2(nov * v_alpha, fac);
                }
            }
            __syncwarp();
            // ---- deferred reduction: lane = (slot, pixel-row group) ----
            float S0 = 0.f, Sx = 0.f, Sy = 0.f, Sxx = 0.f, Sxy = 0.f, Syy = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                float R0 = 0.f, R1 = 0.f, R2 = 0.f;
#pragma unroll
                for (int x = 0; x < 8; x += 2) {
                    const float4 v = r_row[r * 4 + x / 2];          // (vs, fac) of pixels (x, r) and (x+1, r)
                    const float4 w0 = r_vo[r * 8 + x], w1 = r_vo[r * 8 + x + 1];
                    R0 += v.x;
                    R1 = fmaf(v.x, (float)x, R1);
                    R2 = fmaf(v.x, (float)(x * x), R2);
                    c0 = fmaf(v.y, w0.x, c0); c1 = fmaf(v.y, w0.y, c1); c2 = fmaf(v.y, w0.z, c2); c3 = fmaf(v.y, w0.w, c3);
                    R0 += v.z;
                    R1 = fmaf(v.z, (float)(x + 1), R1);
                    R2 = fmaf(v.z, (float)((x + 1) * (x + 1)), R2);
                    c0 = fmaf(v.w, w1.x, c0); c1 = fmaf(v.w, w1.y, c1); c2 = fmaf(v.w, w1.z, c2); c3 = fmaf(v.w, w1.w, c3);
                }
                const float ly = (float)(r_half * 2 + r);
                S0 += R0; Sx += R1; Sxx += R2;
                Sy = fmaf(ly, R0, Sy); Sxy = fmaf(ly, R1, Sxy); Syy = fmaf(ly * ly, R0, Syy);
            }
            S0 += __shfl_xor_sync(FULL, S0, 16); Sx += __shfl_xor_sync(FULL, Sx, 16);
            Sy += __shfl_xor_sync(FULL, Sy, 16); Sxx += __shfl_xor_sync(FULL, Sxx, 16);
            Sxy += __shfl_xor_sync(FULL, Sxy, 16); Syy += __shfl_xor_sync(FULL, Syy, 16);
            c0 += __shfl_xor_sync(FULL, c0, 16); c1 += __shfl_xor_sync(FULL, c1, 16);
            c2 += __shfl_xor_sync(FULL, c2, 16); c3 += __shfl_xor_sync(FULL, c3, 16);
            if (r_slot < ng) {
                const int t = list[g0 + r_slot];
                const float4 A = sRec[t * 3];
                float* dst = v_splats + (size_t)sG[t] * ADB_SPLAT_STRIDE;
                // dx = ex - lx, dy = ey - ly with (lx, ly) the integer pixel offset inside the block
                const float ex = A.x - ((float)x0 + 0.5f), ey = A.y - ((float)y0 + 0.5f);
                if (r_half == 0) {
                    if (S0 != 0.f || Sx != 0.f || Sy != 0.f || Sxx != 0.f || Sxy != 0.f) {
                        const float Mx = fmaf(ex, S0, -Sx), My = fmaf(ey, S0, -Sy);
                        const float Mxx = fmaf(ex, fmaf(ex, S0, -2.f * Sx), Sxx);
                        const float Mxy = fmaf(ex, My, fmaf(-ey, Sx, Sxy));
                        red_add_v4(dst, Mx, My, Mxx, Mxy);
                    }
                } else {
                    const float Myy = fmaf(ey, fmaf(ey, S0, -2.f * Sy), Syy);
                    if (Myy != 0.f || S0 != 0.f || c0 != 0.f || c1 != 0.f) red_add_v4(dst + 4, Myy, S0, c0, c1);
                    if (c2 != 0.f || c3 != 0.f) red_add_v2(dst + 8, c2, c3);
                }
            }
            __syncwarp();
        }
    }
}

}  // namespace

// C views (gridDim.z); wrap: see record_index.
static int blend_fwd_impl(bool legacy, int C, int W, int H, int wrap, const float* splats, const int32_t* vals_sorted,
                          const int32_t* tile_offsets, float* colors, float* alphas, int32_t* last_ids,
                          int32_t* main_ids, unsigned char* hit_mask, cudaStream_t stream) {
    // records are read and colours stored as float4: a misaligned view would fault
    ADB_REQUIRE((((uintptr_t)splats | (uintptr_t)colors) % 16) == 0,
                "adb_raster_blend_fwd: splats and colors must be 16-byte aligned");
    dim3 grid(adb_cdiv(W, ADB_TILE), adb_cdiv(H, ADB_TILE), C);
    if (legacy)
        blend_fwd_kernel<true><<<grid, BLOCK, 0, stream>>>(W, H, splats, vals_sorted, tile_offsets, wrap,
                                                           colors, alphas, last_ids, main_ids, hit_mask);
    else
        blend_fwd_kernel<false><<<grid, BLOCK, 0, stream>>>(W, H, splats, vals_sorted, tile_offsets, wrap,
                                                            colors, alphas, last_ids, nullptr, hit_mask);
    ADB_CHECK_LAUNCH("blend_fwd_kernel");
    return ADB_OK;
}

static int blend_fwd_single(bool legacy, int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                            const int32_t* tile_offsets, float* colors, float* alphas, int32_t* last_ids,
                            int32_t* main_ids, unsigned char* hit_mask, cudaStream_t stream) {
    ADB_REQUIRE(W > 0 && H > 0 && n_per_cam >= 0, "adb_raster_blend_fwd: bad sizes");
    ADB_REQUIRE(tile_offsets && colors && alphas && last_ids, "adb_raster_blend_fwd: null pointer");
    return blend_fwd_impl(legacy, 1, W, H, max(n_per_cam, 1), splats, vals_sorted, tile_offsets, colors, alphas, last_ids,
                          main_ids, hit_mask, stream);
}

// `vals` are the sorted values (cam*N + gaussian); n_per_cam = N.  colors [H,W,4], alphas [H,W], last_ids [H,W].
// hit_mask (may be NULL): hit_mask[k] (one byte per sorted intersection, k as in vals_sorted) receives the warps of entry k's
// tile whose 8x4 pixel block the splat can reach — the culling decisions of this pass, which adb_raster_blend_bwd reuses.
// Entries behind the point where a whole tile saturated are left unwritten (the backward never looks at them).
ADB_API int adb_raster_blend_fwd(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                                 const int32_t* tile_offsets, float* colors, float* alphas, int32_t* last_ids,
                                 unsigned char* hit_mask, cudaStream_t stream) {
    return blend_fwd_single(false, W, H, n_per_cam, splats, vals_sorted, tile_offsets, colors, alphas, last_ids, nullptr,
                            hit_mask, stream);
}

// C views in one launch (the multi-view batch): splats [C,N,12] indexed by vals_sorted (= c*N + gaussian) directly,
// tile_offsets [C,T+1] absolute (adb_raster_tile_scan_multi), colors [C,H,W,4], alphas / last_ids [C,H,W]; hit_mask (may be
// NULL) indexed like vals_sorted.  Per view the result of adb_raster_blend_fwd on that view's records, bit for bit;
// last_ids are absolute sorted indices.  N = 0 (no Gaussians: every tile is empty) writes empty images; splats may be NULL.
ADB_API int adb_raster_blend_fwd_multi(int N, int C, int W, int H, const float* splats, const int32_t* vals_sorted,
                                       const int32_t* tile_offsets, float* colors, float* alphas, int32_t* last_ids,
                                       unsigned char* hit_mask, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && C > 0 && C <= 65535 && W > 0 && H > 0, "adb_raster_blend_fwd_multi: bad sizes");
    ADB_REQUIRE(tile_offsets && colors && alphas && last_ids, "adb_raster_blend_fwd_multi: null pointer");
    ADB_REQUIRE(N == 0 || splats, "adb_raster_blend_fwd_multi: null pointer");
    return blend_fwd_impl(false, C, W, H, 0, splats, vals_sorted, tile_offsets, colors, alphas, last_ids, nullptr, hit_mask,
                          stream);
}

// Legacy (Inria) blending: colors[...,3] = sum alpha*T/z (inverse depth); main_ids [H,W] may be NULL.
ADB_API int adb_raster_blend_fwd_legacy(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                                        const int32_t* tile_offsets, float* colors, float* alphas, int32_t* last_ids,
                                        int32_t* main_ids, cudaStream_t stream) {
    return blend_fwd_single(true, W, H, n_per_cam, splats, vals_sorted, tile_offsets, colors, alphas, last_ids, main_ids,
                            nullptr, stream);
}

// C views (gridDim.z); wrap: see record_index.
static int blend_bwd_impl(bool legacy, int C, int W, int H, int wrap, const float* splats, const int32_t* vals_sorted,
                          const int32_t* tile_offsets, const float* alphas, const int32_t* last_ids,
                          const float* v_colors, const float* v_alphas, float* v_splats, const unsigned char* hit_mask,
                          cudaStream_t stream) {
    // float4 record and upstream loads, red.global.add.v4 into the accumulators: a misaligned view would fault
    ADB_REQUIRE((((uintptr_t)splats | (uintptr_t)v_colors | (uintptr_t)v_splats) % 16) == 0,
                "adb_raster_blend_bwd: splats, v_colors and v_splats must be 16-byte aligned");
    dim3 grid(adb_cdiv(W, ADB_TILE), adb_cdiv(H, ADB_TILE), C);
    static AdbDeviceOnce once;
    const int rc = once.ensure([]() -> int {
        ADB_CUDA(cudaFuncSetAttribute(blend_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, BwdSmem::BYTES));
        ADB_CUDA(cudaFuncSetAttribute(blend_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, BwdSmem::BYTES));
        return ADB_OK;
    });
    if (rc != ADB_OK) return rc;
    if (legacy)
        blend_bwd_kernel<true><<<grid, BLOCK, BwdSmem::BYTES, stream>>>(W, H, splats, vals_sorted, tile_offsets, wrap, alphas,
                                                                        last_ids, v_colors, v_alphas, v_splats, hit_mask);
    else
        blend_bwd_kernel<false><<<grid, BLOCK, BwdSmem::BYTES, stream>>>(W, H, splats, vals_sorted, tile_offsets, wrap, alphas,
                                                                         last_ids, v_colors, v_alphas, v_splats, hit_mask);
    ADB_CHECK_LAUNCH("blend_bwd_kernel");
    return ADB_OK;
}

static int blend_bwd_single(bool legacy, int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                            const int32_t* tile_offsets, const float* alphas, const int32_t* last_ids,
                            const float* v_colors, const float* v_alphas, float* v_splats, const unsigned char* hit_mask,
                            cudaStream_t stream) {
    ADB_REQUIRE(W > 0 && H > 0 && n_per_cam >= 0, "adb_raster_blend_bwd: bad sizes");
    ADB_REQUIRE(tile_offsets && alphas && last_ids && v_colors && v_alphas, "adb_raster_blend_bwd: null pointer");
    if (n_per_cam == 0) return ADB_OK;
    ADB_REQUIRE(v_splats, "adb_raster_blend_bwd: null v_splats");
    return blend_bwd_impl(legacy, 1, W, H, n_per_cam, splats, vals_sorted, tile_offsets, alphas, last_ids, v_colors, v_alphas,
                          v_splats, hit_mask, stream);
}

// v_splats [N,12] must be zeroed by the caller; gradients are accumulated into it.  hit_mask (may be NULL): the forward's
// culling decisions (adb_raster_blend_fwd of the SAME splats / vals_sorted / tile_offsets); the per-warp hit lists then come
// from it instead of repeating the box and ellipse tests.  Identical gradients either way.
ADB_API int adb_raster_blend_bwd(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                                 const int32_t* tile_offsets, const float* alphas, const int32_t* last_ids,
                                 const float* v_colors, const float* v_alphas, float* v_splats,
                                 const unsigned char* hit_mask, cudaStream_t stream) {
    return blend_bwd_single(false, W, H, n_per_cam, splats, vals_sorted, tile_offsets, alphas, last_ids, v_colors,
                            v_alphas, v_splats, hit_mask, stream);
}

// C views in one launch: buffers as adb_raster_blend_fwd_multi, v_colors [C,H,W,4], v_alphas [C,H,W], v_splats [C,N,12]
// (zeroed by the caller, accumulated), hit_mask from adb_raster_blend_fwd_multi (may be NULL: the kernel then culls itself).
// N = 0: nothing to accumulate, accepted without a launch.
ADB_API int adb_raster_blend_bwd_multi(int N, int C, int W, int H, const float* splats, const int32_t* vals_sorted,
                                       const int32_t* tile_offsets, const float* alphas, const int32_t* last_ids,
                                       const float* v_colors, const float* v_alphas, float* v_splats,
                                       const unsigned char* hit_mask, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && C > 0 && C <= 65535 && W > 0 && H > 0, "adb_raster_blend_bwd_multi: bad sizes");
    ADB_REQUIRE(tile_offsets && alphas && last_ids && v_colors && v_alphas, "adb_raster_blend_bwd_multi: null pointer");
    if (N == 0) return ADB_OK;
    ADB_REQUIRE(splats && v_splats, "adb_raster_blend_bwd_multi: null pointer");
    return blend_bwd_impl(false, C, W, H, 0, splats, vals_sorted, tile_offsets, alphas, last_ids, v_colors, v_alphas,
                          v_splats, hit_mask, stream);
}

// Legacy (Inria) conventions; v_colors[...,3] is the upstream gradient of the inverse-depth channel and v_splats slot 9
// receives dL/d(1/z) per Gaussian (the caller multiplies by -1/z^2 before adb_raster_project_bwd).
ADB_API int adb_raster_blend_bwd_legacy(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                                        const int32_t* tile_offsets, const float* alphas, const int32_t* last_ids,
                                        const float* v_colors, const float* v_alphas, float* v_splats,
                                        cudaStream_t stream) {
    return blend_bwd_single(true, W, H, n_per_cam, splats, vals_sorted, tile_offsets, alphas, last_ids, v_colors,
                            v_alphas, v_splats, nullptr, stream);
}

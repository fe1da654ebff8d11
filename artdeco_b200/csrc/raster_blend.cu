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
//  * WARP-COOPERATIVE CULLING: lane l tests splat l of a 32-chunk against the warp's block (integer radius box, then the
//    exact minimum of sigma over the block's rectangle against ln(255 o)); a ballot compacts the survivors into the
//    warp's private 16-bit hit list, padded to a multiple of four with a never-visible dummy record so the evaluation
//    loop is unrolled by four with one LDS.64 of list entries and no remainder code;
//  * the evaluation bodies are branch-free (predicated selects), so the four unrolled bodies interleave;
//  * BACKWARD — the per-splat reduction over the warp's 32 pixels is NOT a shuffle butterfly.  All ten per-Gaussian
//    sums are dot products of two per-(pixel,splat) scalars with weights that do not depend on the splat:
//        raw moments  sum_p vs(p) * {1, lx, ly, lx^2, lx ly, ly^2}   (vs = dL/dsigma, lx/ly = pixel offset in the block)
//        feature grads sum_p fac(p) * v_out[p][0..3]                  (fac = alpha*T)
//    i.e. a [slots x 32 pixels] x [32 x 10] product.  A lane therefore stores just (vs, fac) per evaluation (one STS.64)
//    into a per-warp slot buffer; every S evaluations the warp transposes roles (lane = slot), streams the slot's row
//    with LDS.128, applies the lane-constant integer weights as immediates (row sums first: 7.75 FMA per pixel
//    instead of 10) and converts the block-origin moments to splat-centred ones once per (warp, splat):
//        sum vs dx = ex S0 - Sx,  sum vs dx^2 = ex (ex S0 - 2 Sx) + Sxx, ...   (ex = mean_x - block origin)
//    About 11 issued instructions per evaluation against ~55 for the packed butterfly + shared atomics it replaces, and
//    the nine moment/feature multiplies leave the per-pixel body as well;
//  * results leave with three 128/64-bit vector REDs per (warp, splat) (red.global.add.v4.f32).
#include "raster_common.cuh"
#include <stdlib.h>

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

// ---- TMA (bulk async copy) staging: "stage Gaussian attributes into shared memory via TMA" (BASELINE north_star) ----------
// Each thread issues ONE 48-byte cp.async.bulk (global -> shared, SASS UBLKCP) for the record of its list entry of the NEXT
// batch; completion is tracked by an mbarrier per buffer (every thread arrives once; issuing threads add expect_tx 48).
// The copy engine fills buffer (b+1)&1 while the warps evaluate batch b from buffer b&1, so the dependent-load latency of the
// gather (vals[idx] -> splats[g]) no longer sits between two block barriers.  OPT-IN (ADB_BLEND_TMA=1): the blend kernels are
// issue-bound with 3-4 resident CTAs per SM already hiding the gather latency, so the synchronous staging is the default.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred P1;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// Issues this thread's copy of record `g` into `rec` (48 B) or a plain arrival when the thread has no list entry.
__device__ __forceinline__ void issue_record_copy(float4* rec, const float* __restrict__ splats, int g, bool have, uint64_t* bar) {
    if (have) {
        mbar_arrive_expect_tx(bar, ADB_SPLAT_STRIDE * 4);
        bulk_copy_g2s(rec, splats + (size_t)g * ADB_SPLAT_STRIDE, ADB_SPLAT_STRIDE * 4, bar);
    } else {
        mbar_arrive(bar);
    }
}

// In-place version of stage_record's pre-scaling for a record that arrived by bulk copy.
template <bool LEGACY>
__device__ __forceinline__ void prescale_record(float4* __restrict__ rec) {
    float4 A = rec[0], B = rec[1];
    A.z *= 0.5f * LOG2E;
    A.w *= LOG2E;
    B.x *= 0.5f * LOG2E;
    B.z = (B.z - ADB_SIGMA_MARGIN) * LOG2E;
    rec[0] = A;
    rec[1] = B;
    if (LEGACY) rec[2].w = 1.0f / rec[2].w;
}

// warp block geometry: warp w covers pixels x in [bx*16 + (w&1)*8, +8), y in [by*16 + (w>>1)*4, +4)
struct WarpRect {
    float xlo, xhi, ylo, yhi;  // pixel-centre range
};

// Shared-memory record (3 x float4, 48 B stride: conflict-free for both the staging stores and the broadcast loads):
//   A = (mx, my, ha, b2)   B = (hc, opacity, smax2, bits rx|ry<<16)   C = (r, g, b, depth | 1/depth for LEGACY)
// with ha = log2e * a/2, b2 = log2e * b, hc = log2e * c/2, smax2 = log2e * ln(255 o) (the projection's margin removed):
//   sigma2 = log2e * sigma = dx (ha dx + b2 dy) + hc dy^2,   alpha = o * 2^(-sigma2),
//   and  alpha >= 1/255  <=>  sigma2 <= smax2  — one compare replaces the alpha test (the two differ only where
//   o 2^(-sigma2) is within an ulp of 1/255, the same measure-zero band in which ex2.approx and the oracle's expf disagree).
template <bool LEGACY>
__device__ __forceinline__ void stage_record(float4* __restrict__ rec, const float* __restrict__ splats, int g) {
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
}

__device__ __forceinline__ void write_dummy(float4* __restrict__ rec) {
    rec[0] = make_float4(0.f, 0.f, 0.f, 0.f);
    rec[1] = make_float4(0.f, 0.f, -1.0f, 0.f);  // smax2 = -1: fails "0 <= sigma2 <= smax2" for every pixel
    rec[2] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// Can the splat reach alpha >= 1/255 anywhere in the warp's block?  Two conservative tests:
//  1. the integer-radius box written by the projection (outside it alpha < 1/255 by construction of the radius);
//  2. the exact minimum of sigma2(d) = ha dx^2 + hc dy^2 + b2 dx dy over the block's pixel-centre rectangle against smax2 —
//     the same bound the per-pixel pre-test uses, so a culled splat would have failed that pre-test on every pixel of the
//     block and the image is unchanged.  ~1.5 warp-instructions per (warp, splat) because 32 splats are tested per
//     instruction, against ~35 (forward) / ~55 (backward) for the evaluation it avoids.
__device__ __forceinline__ bool splat_box_hits(const float4& A, const float4& B, const WarpRect& r) {
    const unsigned pr = __float_as_uint(B.w);
    // 65535 is the saturation value written by the projection: treat it as unbounded
    const float rx = (pr & 0xffffu) == 0xffffu ? 3.0e38f : (float)(pr & 0xffffu);
    const float ry = (pr >> 16) == 0xffffu ? 3.0e38f : (float)(pr >> 16);
    return (A.x + rx >= r.xlo) && (A.x - rx <= r.xhi) && (A.y + ry >= r.ylo) && (A.y - ry <= r.yhi);
}
__device__ __forceinline__ bool splat_exact_hits(const float4& A, const float4& B, const WarpRect& r) {
    const float x0 = r.xlo - A.x, x1 = r.xhi - A.x, y0 = r.ylo - A.y, y1 = r.yhi - A.y;
    if (x0 <= 0.f && x1 >= 0.f && y0 <= 0.f && y1 >= 0.f) return true;   // centre inside the block
    const float ha = A.z, b = A.w, hc = B.x;
    const float nb_c = -0.5f * __fdividef(b, hc), nb_a = -0.5f * __fdividef(b, ha);
    // minimum over each edge (1-D quadratic, minimiser clamped to the edge); the rectangle's minimum is on its boundary
    float m;
    {
        const float dy0 = fminf(y1, fmaxf(y0, nb_c * x0)), dy1 = fminf(y1, fmaxf(y0, nb_c * x1));
        const float q0 = ha * x0 * x0 + hc * dy0 * dy0 + b * x0 * dy0;
        const float q1 = ha * x1 * x1 + hc * dy1 * dy1 + b * x1 * dy1;
        m = fminf(q0, q1);
    }
    {
        const float dx0 = fminf(x1, fmaxf(x0, nb_a * y0)), dx1 = fminf(x1, fmaxf(x0, nb_a * y1));
        const float q0 = ha * dx0 * dx0 + hc * y0 * y0 + b * dx0 * y0;
        const float q1 = ha * dx1 * dx1 + hc * y1 * y1 + b * dx1 * y1;
        m = fminf(m, fminf(q0, q1));
    }
    // rounding slack: the per-pixel test is sigma2 <= smax2 in the same fp32 arithmetic
    return m <= B.z * 1.0001f + 1e-4f;
}

// Builds the warp's hit list for the staged batch (ascending slot order), padded to a multiple of 4 with DUMMY.
// `limit`: only slots s with s >= limit are considered (the backward skips splats behind the warp's last contributor).
// Two dense phases: (1) the cheap integer-radius box test on all slots, survivors compacted into the list; (2) the exact
// ellipse-vs-rectangle test on the survivors only (46 % of the slots at the bench workload), 32 per instruction, compacted in
// place (the write index never passes the read index).  A single fused test would run the expensive half with most lanes idle.
__device__ __forceinline__ int build_hit_list(const float4* __restrict__ sRec, unsigned short* __restrict__ list,
                                              int bsize, int limit, const WarpRect& rect, int lane) {
    const unsigned lt_mask = (1u << lane) - 1u;
    int nbox = 0;
    for (int c0 = (limit > 0 ? (limit & ~31) : 0); c0 < bsize; c0 += 32) {
        const int s = c0 + lane;
        bool hit = false;
        if (s < bsize && s >= limit) hit = splat_box_hits(sRec[s * 3], sRec[s * 3 + 1], rect);
        const unsigned mask = __ballot_sync(FULL, hit);
        if (hit) list[nbox + __popc(mask & lt_mask)] = (unsigned short)s;
        nbox += __popc(mask);
    }
    __syncwarp();
    int nhit = 0;
    for (int c0 = 0; c0 < nbox; c0 += 32) {
        const int k = c0 + lane;
        int s = 0;
        bool hit = false;
        if (k < nbox) {
            s = list[k];
            hit = splat_exact_hits(sRec[s * 3], sRec[s * 3 + 1], rect);
        }
        const unsigned mask = __ballot_sync(FULL, hit);     // every lane has read its entry before any lane overwrites one
        if (hit) list[nhit + __popc(mask & lt_mask)] = (unsigned short)s;
        nhit += __popc(mask);
        __syncwarp();
    }
    if (lane < 3) list[nhit + lane] = (unsigned short)DUMMY;
    __syncwarp();
    return nhit;
}

// The backward's hit list from the forward's per-entry warp masks (bit w of hit_mask[sorted index] = warp w's block is hit):
// the forward has already run both tests on every entry a warp can need again — the backward only revisits entries up to the
// warp's last contributor, all of which lie in batches that warp went through — so the backward replaces ~150 instructions
// per 32 slots by a table look-up and a compaction.  sM[slot] = mask of the staged batch (slot order = back to front).
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

// LEGACY = Inria conventions (ADB_CONV_INRIA): alpha <= 0.99, stop when T(1-alpha) < 1e-4 (strict), 4th channel
// accumulates 1/z, and main_ids gets the Gaussian with the largest blending weight alpha*T per pixel (-1: none).
template <bool LEGACY, bool ASYNC>
__global__ void __launch_bounds__(BLOCK, 4)
blend_fwd_kernel(int W, int H, const float* __restrict__ splats, const int32_t* __restrict__ vals,
                 const int32_t* __restrict__ tile_offsets, int n_per_cam,
                 float* __restrict__ colors, float* __restrict__ alphas, int32_t* __restrict__ last_ids,
                 int32_t* __restrict__ main_ids, unsigned char* __restrict__ hit_mask) {
    constexpr float MAXA = LEGACY ? ADB_MAX_ALPHA_INRIA : ADB_MAX_ALPHA;
    constexpr int NBUF = ASYNC ? 2 : 1;
    __shared__ __align__(16) float4 sRecBuf[NBUF][(BLOCK + 1) * 3];
    __shared__ __align__(8) unsigned short sList[NWARP][LIST_STRIDE];
    __shared__ __align__(8) uint64_t sBar[2];
    __shared__ unsigned sMask[BLOCK / 4];       // byte s = warp mask of slot s of the current batch (hit_mask != NULL)

    const int tw = (W + ADB_TILE - 1) / ADB_TILE;
    const int tile = blockIdx.y * tw + blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int x0 = blockIdx.x * ADB_TILE + (warp & 1) * 8, y0 = blockIdx.y * ADB_TILE + (warp >> 1) * 4;
    const int j = x0 + (lane & 7), i = y0 + (lane >> 3);
    const bool inside = (i < H && j < W);
    const float px = (float)j + 0.5f, py = (float)i + 0.5f;
    const WarpRect rect{(float)x0 + 0.5f, (float)x0 + 7.5f, (float)y0 + 0.5f, (float)y0 + 3.5f};
    const int start = tile_offsets[tile], end = tile_offsets[tile + 1];
    if (tid < BLOCK / 4) sMask[tid] = 0u;
    // Writes the finished batch's warp masks to hit_mask[start + pb*BLOCK ...] and clears the table (one thread per word, so the
    // clear cannot race with the read; the barrier that follows orders it before the next batch's atomics).
    auto flush_mask = [&](int pb) {
        if (tid < BLOCK / 4) {
            const unsigned w = sMask[tid];
            sMask[tid] = 0u;
            const int i0 = start + pb * BLOCK + tid * 4;
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (i0 + k < end) hit_mask[i0 + k] = (unsigned char)((w >> (8 * k)) & 0xffu);
        }
    };
    int pending = -1;                            // batch whose masks are complete but not written yet (block-uniform)
    if (tid == 0) {
        write_dummy(sRecBuf[0] + DUMMY * 3);
        if (ASYNC) {
            write_dummy(sRecBuf[NBUF - 1] + DUMMY * 3);
            mbar_init(&sBar[0], BLOCK);
            mbar_init(&sBar[1], BLOCK);
            fence_mbar_init();
        }
    }
    const int nb = (end - start + BLOCK - 1) / BLOCK;
    if (ASYNC) {
        __syncthreads();
        if (nb > 0) {       // prologue: batch 0 -> buffer 0
            const int idx0 = start + tid;
            issue_record_copy(sRecBuf[0] + tid * 3, splats, idx0 < end ? vals[idx0] % n_per_cam : 0, idx0 < end, &sBar[0]);
        }
    }

    float T = 1.0f;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int cur = 0;
    float best_w = 0.f;
    int best_k = -1;
    bool done = !inside;
    for (int b = 0; b < nb; ++b) {
        const int n_done = __syncthreads_count(done);    // also: every warp has finished reading the previous batch
        if (hit_mask && pending >= 0) { flush_mask(pending); pending = -1; }
        const int bstart = start + b * BLOCK;
        const int idx = bstart + tid;
        float4* sRec = sRecBuf[ASYNC ? (b & 1) : 0];
        if (ASYNC) {
            if (n_done >= BLOCK) { mbar_wait(&sBar[b & 1], (b >> 1) & 1); break; }   // drain the copy in flight, then leave
            if (b + 1 < nb) {                            // prefetch batch b+1 into the buffer batch b-1 has just released
                const int idx1 = idx + BLOCK;
                fence_proxy_async();
                issue_record_copy(sRecBuf[(b + 1) & 1] + tid * 3, splats, idx1 < end ? vals[idx1] % n_per_cam : 0, idx1 < end,
                                  &sBar[(b + 1) & 1]);
            }
            mbar_wait(&sBar[b & 1], (b >> 1) & 1);
            if (idx < end) prescale_record<LEGACY>(sRec + tid * 3);
        } else {
            if (n_done >= BLOCK) break;
            if (idx < end) stage_record<LEGACY>(sRec + tid * 3, splats, vals[idx] % n_per_cam);
        }
        __syncthreads();
        pending = b;
        const int bsize = min(BLOCK, end - bstart);
        if (__all_sync(FULL, done)) continue;
        unsigned short* list = sList[warp];
        const int nhit = build_hit_list(sRec, list, bsize, 0, rect, lane);
        if (hit_mask) {
            for (int k = lane; k < nhit; k += 32) {
                const unsigned sl = list[k];
                atomicOr(&sMask[sl >> 2], 1u << (((sl & 3u) << 3) + warp));
            }
        }
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
    if (hit_mask && pending >= 0) {              // the loop ran to its end: the last batch's masks are still in shared memory
        __syncthreads();
        flush_mask(pending);
    }
    if (inside) {
        const size_t pix = (size_t)i * W + j;
        reinterpret_cast<float4*>(colors)[pix] = acc;
        alphas[pix] = 1.0f - T;
        last_ids[pix] = cur;
        if (LEGACY && main_ids) main_ids[pix] = best_k >= 0 ? vals[best_k] % n_per_cam : -1;
    }
}

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// Backward shared-memory layout (dynamic): S = slots per warp in the deferred-reduction buffer (16 or 32).
template <int S, bool ASYNC>
struct BwdSmem {
    static constexpr int NBUF = ASYNC ? 2 : 1;
    static constexpr int ROW4 = 17;                       // float4 per slot row: 32 x (vs, fac) + 1 pad -> conflict-free
    static constexpr int REC_BYTES = (BLOCK + 1) * 3 * 16;
    static constexpr int G_BYTES = (BLOCK + 4) * 4;
    static constexpr int OFF_REC = 0;                     // float4 [NBUF][(BLOCK+1)*3]
    static constexpr int OFF_G = OFF_REC + NBUF * REC_BYTES;                  // int [NBUF][BLOCK + 4]
    static constexpr int OFF_BAR = OFF_G + NBUF * G_BYTES;                    // uint64 [2]
    static constexpr int OFF_M = OFF_BAR + 16;                                // u8 [BLOCK]: the forward's warp masks of the batch
    static constexpr int OFF_LIST = OFF_M + BLOCK;                            // u16 [NWARP][LIST_STRIDE]
    static constexpr int OFF_VO = OFF_LIST + NWARP * LIST_STRIDE * 2;         // float4 [NWARP][32]
    static constexpr int OFF_V = OFF_VO + NWARP * 32 * 16;                    // float4 [NWARP][S*ROW4]
    static constexpr int BYTES = OFF_V + NWARP * S * ROW4 * 16;
    static_assert(OFF_G % 16 == 0 && OFF_BAR % 16 == 0 && OFF_LIST % 16 == 0 && OFF_VO % 16 == 0 && OFF_V % 16 == 0, "alignment");
};

template <bool LEGACY, int S, int OCC, bool ASYNC>
__global__ void __launch_bounds__(BLOCK, OCC)
blend_bwd_kernel(int W, int H, const float* __restrict__ splats, const int32_t* __restrict__ vals,
                 const int32_t* __restrict__ tile_offsets, int n_per_cam,
                 const float* __restrict__ alphas, const int32_t* __restrict__ last_ids,
                 const float* __restrict__ v_colors, const float* __restrict__ v_alphas,
                 float* __restrict__ v_splats, const unsigned char* __restrict__ hit_mask) {
    constexpr float MAXA = LEGACY ? ADB_MAX_ALPHA_INRIA : ADB_MAX_ALPHA;
    using L = BwdSmem<S, ASYNC>;
    constexpr int HALVES = 32 / S;          // lanes per slot in the reduction phase
    constexpr int ROWS = 4 / HALVES;        // pixel rows (of 8) each reduction lane walks
    static_assert(S == 16 || S == 32, "S");
    extern __shared__ __align__(16) unsigned char smem[];
    float4* sRec = reinterpret_cast<float4*>(smem + L::OFF_REC);
    int* sG = reinterpret_cast<int*>(smem + L::OFF_G);
    uint64_t* sBar = reinterpret_cast<uint64_t*>(smem + L::OFF_BAR);
    unsigned char* sM = smem + L::OFF_M;

    const int tw = (W + ADB_TILE - 1) / ADB_TILE;
    const int tile = blockIdx.y * tw + blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    unsigned short* list = reinterpret_cast<unsigned short*>(smem + L::OFF_LIST) + warp * LIST_STRIDE;
    float4* sVo = reinterpret_cast<float4*>(smem + L::OFF_VO) + warp * 32;
    float4* sV = reinterpret_cast<float4*>(smem + L::OFF_V) + warp * S * L::ROW4;
    const int x0 = blockIdx.x * ADB_TILE + (warp & 1) * 8, y0 = blockIdx.y * ADB_TILE + (warp >> 1) * 4;
    const int j = x0 + (lane & 7), i = y0 + (lane >> 3);
    const bool inside = (i < H && j < W);
    const float px = (float)j + 0.5f, py = (float)i + 0.5f;
    const WarpRect rect{(float)x0 + 0.5f, (float)x0 + 7.5f, (float)y0 + 0.5f, (float)y0 + 3.5f};
    const int start = tile_offsets[tile], end = tile_offsets[tile + 1];
    if (end <= start) return;

    const size_t pix = (size_t)(inside ? i : 0) * W + (inside ? j : 0);
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
        if (ASYNC) {
            write_dummy(reinterpret_cast<float4*>(smem + L::OFF_REC + L::REC_BYTES) + DUMMY * 3);
            reinterpret_cast<int*>(smem + L::OFF_G + L::G_BYTES)[DUMMY] = 0;
            mbar_init(&sBar[0], BLOCK);
            mbar_init(&sBar[1], BLOCK);
            fence_mbar_init();
        }
    }

    int warp_bin_final = bin_final;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) warp_bin_final = max(warp_bin_final, __shfl_xor_sync(FULL, warp_bin_final, o));

    // reduction-phase role of this lane: slot r_slot, pixel rows [r_half*ROWS, +ROWS) of the warp's 8x4 block
    const int r_slot = lane & (S - 1), r_half = lane / S;
    const float4* r_row = sV + r_slot * L::ROW4 + r_half * (ROWS * 4);
    const float4* r_vo = sVo + r_half * (ROWS * 8);
    float2* my_cell = reinterpret_cast<float2*>(sV) + lane;          // + slot * ROW4 * 2 (float2 units)

    const int nb = (end - start + BLOCK - 1) / BLOCK;
    if (ASYNC) {
        __syncthreads();
        const int idx0 = end - 1 - tid;                      // prologue: batch 0 -> buffer 0
        const int g0 = idx0 >= start ? vals[idx0] % n_per_cam : 0;
        if (idx0 >= start) sG[tid] = g0;
        issue_record_copy(sRec + tid * 3, splats, g0, idx0 >= start, &sBar[0]);
    }
    float4* const sRec0 = sRec;
    int* const sG0 = sG;
    for (int b = 0; b < nb; ++b) {
        __syncthreads();  // previous batch fully consumed
        const int batch_end = end - 1 - b * BLOCK;           // smem slot t <-> sorted index batch_end - t (back to front)
        const int bsize = min(BLOCK, batch_end + 1 - start);
        const int idx = batch_end - tid;
        if (ASYNC) {
            sRec = reinterpret_cast<float4*>(reinterpret_cast<unsigned char*>(sRec0) + (b & 1) * L::REC_BYTES);
            sG = reinterpret_cast<int*>(reinterpret_cast<unsigned char*>(sG0) + (b & 1) * L::G_BYTES);
            if (b + 1 < nb) {                                // prefetch batch b+1 into the buffer batch b-1 has just released
                const int nbuf = (b + 1) & 1;
                const int idx1 = idx - BLOCK;
                const int g1 = idx1 >= start ? vals[idx1] % n_per_cam : 0;
                if (idx1 >= start) reinterpret_cast<int*>(reinterpret_cast<unsigned char*>(sG0) + nbuf * L::G_BYTES)[tid] = g1;
                fence_proxy_async();
                issue_record_copy(reinterpret_cast<float4*>(reinterpret_cast<unsigned char*>(sRec0) + nbuf * L::REC_BYTES) + tid * 3,
                                  splats, g1, idx1 >= start, &sBar[nbuf]);
            }
            mbar_wait(&sBar[b & 1], (b >> 1) & 1);
            if (idx >= start) prescale_record<LEGACY>(sRec + tid * 3);
        } else if (idx >= start) {
            const int g = vals[idx] % n_per_cam;
            sG[tid] = g;
            stage_record<LEGACY>(sRec + tid * 3, splats, g);
        }
        if (hit_mask && idx >= start) sM[tid] = hit_mask[idx];
        __syncthreads();
        // a splat at slot s contributes to this warp only if batch_end - s <= warp_bin_final
        const int limit = max(0, batch_end - warp_bin_final);
        if (limit >= bsize) continue;
        const int nhit = hit_mask ? build_hit_list_from_mask(sM, list, bsize, limit, warp, lane)
                                  : build_hit_list(sRec, list, bsize, limit, rect, lane);
        const int tmin = inside ? batch_end - bin_final : (1 << 30);   // lane-valid iff t >= tmin
        for (int g0 = 0; g0 < nhit; g0 += S) {
            const int ng = min(S, nhit - g0);
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
            for (int r = 0; r < ROWS; ++r) {
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
                const float ly = (float)(r_half * ROWS + r);
                S0 += R0; Sx += R1; Sxx += R2;
                Sy = fmaf(ly, R0, Sy); Sxy = fmaf(ly, R1, Sxy); Syy = fmaf(ly * ly, R0, Syy);
            }
            if (HALVES == 2) {
                S0 += __shfl_xor_sync(FULL, S0, 16); Sx += __shfl_xor_sync(FULL, Sx, 16);
                Sy += __shfl_xor_sync(FULL, Sy, 16); Sxx += __shfl_xor_sync(FULL, Sxx, 16);
                Sxy += __shfl_xor_sync(FULL, Sxy, 16); Syy += __shfl_xor_sync(FULL, Syy, 16);
                c0 += __shfl_xor_sync(FULL, c0, 16); c1 += __shfl_xor_sync(FULL, c1, 16);
                c2 += __shfl_xor_sync(FULL, c2, 16); c3 += __shfl_xor_sync(FULL, c3, 16);
            }
            if (r_slot < ng) {
                const int t = list[g0 + r_slot];
                const float4 A = sRec[t * 3];
                float* dst = v_splats + (size_t)sG[t] * ADB_SPLAT_STRIDE;
                // dx = ex - lx, dy = ey - ly with (lx, ly) the integer pixel offset inside the block
                const float ex = A.x - rect.xlo, ey = A.y - rect.ylo;
                if (r_half == 0) {
                    if (S0 != 0.f || Sx != 0.f || Sy != 0.f || Sxx != 0.f || Sxy != 0.f) {
                        const float Mx = fmaf(ex, S0, -Sx), My = fmaf(ey, S0, -Sy);
                        const float Mxx = fmaf(ex, fmaf(ex, S0, -2.f * Sx), Sxx);
                        const float Mxy = fmaf(ex, My, fmaf(-ey, Sx, Sxy));
                        red_add_v4(dst, Mx, My, Mxx, Mxy);
                    }
                    if (HALVES == 1) {
                        const float Myy = fmaf(ey, fmaf(ey, S0, -2.f * Sy), Syy);
                        if (Myy != 0.f || S0 != 0.f || c0 != 0.f || c1 != 0.f) red_add_v4(dst + 4, Myy, S0, c0, c1);
                        if (c2 != 0.f || c3 != 0.f) red_add_v2(dst + 8, c2, c3);
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

static int blend_fwd_impl(bool legacy, int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                          const int32_t* tile_offsets, float* colors, float* alphas, int32_t* last_ids,
                          int32_t* main_ids, unsigned char* hit_mask, cudaStream_t stream) {
    ADB_REQUIRE(W > 0 && H > 0 && n_per_cam >= 0, "adb_raster_blend_fwd: bad sizes");
    ADB_REQUIRE(tile_offsets && colors && alphas && last_ids, "adb_raster_blend_fwd: null pointer");
    dim3 grid(adb_cdiv(W, ADB_TILE), adb_cdiv(H, ADB_TILE));
    // ADB_BLEND_TMA=1: double-buffered cp.async.bulk (TMA) staging.  Default: synchronous LDG staging (the kernel is
    // issue-bound with 4 CTAs/SM hiding the gather latency, so the extra prescale pass and mbarrier waits buy nothing).
    static const int tma = getenv("ADB_BLEND_TMA") ? atoi(getenv("ADB_BLEND_TMA")) : 0;
    if (legacy)
        blend_fwd_kernel<true, false><<<grid, BLOCK, 0, stream>>>(W, H, splats, vals_sorted, tile_offsets, max(n_per_cam, 1),
                                                                 colors, alphas, last_ids, main_ids, hit_mask);
    else if (tma)
        blend_fwd_kernel<false, true><<<grid, BLOCK, 0, stream>>>(W, H, splats, vals_sorted, tile_offsets, max(n_per_cam, 1),
                                                                 colors, alphas, last_ids, nullptr, hit_mask);
    else
        blend_fwd_kernel<false, false><<<grid, BLOCK, 0, stream>>>(W, H, splats, vals_sorted, tile_offsets, max(n_per_cam, 1),
                                                                  colors, alphas, last_ids, nullptr, hit_mask);
    ADB_CHECK_LAUNCH("blend_fwd_kernel");
    return ADB_OK;
}

// `vals` are the sorted values (cam*N + gaussian); n_per_cam = N.  colors [H,W,4], alphas [H,W], last_ids [H,W].
ADB_API int adb_raster_blend_fwd(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                                 const int32_t* tile_offsets, float* colors, float* alphas, int32_t* last_ids,
                                 cudaStream_t stream) {
    return blend_fwd_impl(false, W, H, n_per_cam, splats, vals_sorted, tile_offsets, colors, alphas, last_ids, nullptr,
                          nullptr, stream);
}

// Same, and hit_mask[k] (one byte per sorted intersection, k as in vals_sorted) receives the warps of entry k's tile whose 8x4
// pixel block the splat can reach — the culling decisions of this pass, which adb_raster_blend_bwd_hits reuses.  Entries behind
// the point where a whole tile saturated are left unwritten (the backward never looks at them).
ADB_API int adb_raster_blend_fwd_hits(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                                      const int32_t* tile_offsets, float* colors, float* alphas, int32_t* last_ids,
                                      unsigned char* hit_mask, cudaStream_t stream) {
    ADB_REQUIRE(hit_mask, "adb_raster_blend_fwd_hits: null hit_mask");
    return blend_fwd_impl(false, W, H, n_per_cam, splats, vals_sorted, tile_offsets, colors, alphas, last_ids, nullptr,
                          hit_mask, stream);
}

// Legacy (Inria) blending: colors[...,3] = sum alpha*T/z (inverse depth); main_ids [H,W] may be NULL.
ADB_API int adb_raster_blend_fwd_legacy(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                                        const int32_t* tile_offsets, float* colors, float* alphas, int32_t* last_ids,
                                        int32_t* main_ids, cudaStream_t stream) {
    return blend_fwd_impl(true, W, H, n_per_cam, splats, vals_sorted, tile_offsets, colors, alphas, last_ids, main_ids,
                          nullptr, stream);
}

template <bool LEGACY, int S, int OCC, bool ASYNC>
static int launch_bwd(dim3 grid, int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                      const int32_t* tile_offsets, const float* alphas, const int32_t* last_ids, const float* v_colors,
                      const float* v_alphas, float* v_splats, const unsigned char* hit_mask, cudaStream_t stream) {
    static AdbDeviceOnce once;
    const int rc = once.ensure([]() -> int {
        ADB_CUDA(cudaFuncSetAttribute(blend_bwd_kernel<LEGACY, S, OCC, ASYNC>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      BwdSmem<S, ASYNC>::BYTES));
        return ADB_OK;
    });
    if (rc != ADB_OK) return rc;
    blend_bwd_kernel<LEGACY, S, OCC, ASYNC><<<grid, BLOCK, BwdSmem<S, ASYNC>::BYTES, stream>>>(
        W, H, splats, vals_sorted, tile_offsets, n_per_cam, alphas, last_ids, v_colors, v_alphas, v_splats, hit_mask);
    return ADB_OK;
}

static int blend_bwd_impl(bool legacy, int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                          const int32_t* tile_offsets, const float* alphas, const int32_t* last_ids,
                          const float* v_colors, const float* v_alphas, float* v_splats, const unsigned char* hit_mask,
                          cudaStream_t stream) {
    ADB_REQUIRE(W > 0 && H > 0 && n_per_cam >= 0, "adb_raster_blend_bwd: bad sizes");
    ADB_REQUIRE(tile_offsets && alphas && last_ids && v_colors && v_alphas, "adb_raster_blend_bwd: null pointer");
    if (n_per_cam == 0) return ADB_OK;
    ADB_REQUIRE(v_splats, "adb_raster_blend_bwd: null v_splats");
    dim3 grid(adb_cdiv(W, ADB_TILE), adb_cdiv(H, ADB_TILE));
    // A/B switches: ADB_BWD_SLOTS=32 -> 32-slot deferred-reduction buffer (2 CTAs/SM);
    // ADB_BWD_OCC=3 -> 79 registers, 3 CTAs/SM instead of the default 64 registers, 4 CTAs/SM.
    static const int slots = getenv("ADB_BWD_SLOTS") ? atoi(getenv("ADB_BWD_SLOTS")) : 16;
    static const int occ = getenv("ADB_BWD_OCC") ? atoi(getenv("ADB_BWD_OCC")) : 4;
    int rc;
#define ADB_BWD_ARGS grid, W, H, n_per_cam, splats, vals_sorted, tile_offsets, alphas, last_ids, v_colors, v_alphas, v_splats, hit_mask, stream
    // ADB_BLEND_TMA=1: double-buffered cp.async.bulk staging (+13 KB of shared memory: 3 CTAs/SM instead of 4); opt-in for
    // the same reason as the forward kernel.
    static const int tma = getenv("ADB_BLEND_TMA") ? atoi(getenv("ADB_BLEND_TMA")) : 0;
    if (legacy) rc = launch_bwd<true, 16, 3, false>(ADB_BWD_ARGS);
    else if (slots == 32) rc = launch_bwd<false, 32, 2, false>(ADB_BWD_ARGS);
    else if (tma) rc = launch_bwd<false, 16, 3, true>(ADB_BWD_ARGS);
    else if (occ == 4) rc = launch_bwd<false, 16, 4, false>(ADB_BWD_ARGS);
    else rc = launch_bwd<false, 16, 3, false>(ADB_BWD_ARGS);
#undef ADB_BWD_ARGS
    if (rc != ADB_OK) return rc;
    ADB_CHECK_LAUNCH("blend_bwd_kernel");
    return ADB_OK;
}

// v_splats [N,12] must be zeroed by the caller; gradients are accumulated into it.
ADB_API int adb_raster_blend_bwd(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                                 const int32_t* tile_offsets, const float* alphas, const int32_t* last_ids,
                                 const float* v_colors, const float* v_alphas, float* v_splats,
                                 cudaStream_t stream) {
    return blend_bwd_impl(false, W, H, n_per_cam, splats, vals_sorted, tile_offsets, alphas, last_ids, v_colors,
                          v_alphas, v_splats, nullptr, stream);
}

// Same with the forward's culling decisions (adb_raster_blend_fwd_hits of the SAME splats / vals_sorted / tile_offsets): the
// per-warp hit lists come from hit_mask instead of repeating the box and ellipse tests.  Identical gradients.
ADB_API int adb_raster_blend_bwd_hits(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                                      const int32_t* tile_offsets, const float* alphas, const int32_t* last_ids,
                                      const float* v_colors, const float* v_alphas, float* v_splats,
                                      const unsigned char* hit_mask, cudaStream_t stream) {
    ADB_REQUIRE(hit_mask, "adb_raster_blend_bwd_hits: null hit_mask");
    return blend_bwd_impl(false, W, H, n_per_cam, splats, vals_sorted, tile_offsets, alphas, last_ids, v_colors,
                          v_alphas, v_splats, hit_mask, stream);
}

// Legacy (Inria) conventions; v_colors[...,3] is the upstream gradient of the inverse-depth channel and v_splats slot 9
// receives dL/d(1/z) per Gaussian (the caller multiplies by -1/z^2 before adb_raster_project_bwd).
ADB_API int adb_raster_blend_bwd_legacy(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                                        const int32_t* tile_offsets, const float* alphas, const int32_t* last_ids,
                                        const float* v_colors, const float* v_alphas, float* v_splats,
                                        cudaStream_t stream) {
    return blend_bwd_impl(true, W, H, n_per_cam, splats, vals_sorted, tile_offsets, alphas, last_ids, v_colors,
                          v_alphas, v_splats, nullptr, stream);
}

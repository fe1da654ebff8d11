// Voxel-hash class assignment: `SceneModel.update_voxel` (Reconstruct/scene/scene_models/h3dgsv3.py:227-316; SURVEY.md §8a R9).
//
// The reference hashes every Gaussian centre to a 0.1 m voxel, then runs THREE full sorts (`torch.unique` over the
// original hashes, over the (voxel, class) pairs and over the unmatched new hashes), a `scatter_max` and a `searchsorted` to
//   (1) give every original point the MAJORITY class of its voxel,
//   (2) give every new point the majority class of the voxel it falls in, or
//   (3) a fresh class id per previously empty voxel: max_cls + 1 + rank of the voxel among the sorted unmatched hashes.
// Here the grouping is done by open-addressing hash tables (one 64-bit CAS per point), the vote by a second table keyed by
// (voxel slot, class) with atomic counters and one packed 64-bit atomicMax per pair, and only the (few) DISTINCT unmatched
// voxels are ever sorted (by the caller) to reproduce the reference's id order.  Integer work with a bit-exact contract.
//
// Voxel key: the reference linearises (vx, vy, vz) with strides (ny*nz, nz, 1); any order-preserving injective packing gives
// the same `unique` order, so key = vx << 42 | vy << 21 | vz (21 bits per axis = 209 km at 0.1 m; larger indices are flagged).
// Tie rule of the vote (equal counts): the SMALLEST class id, which is what scatter_max's first-maximum rule yields on the
// ascending pair list.
#include "common.cuh"

namespace {

typedef unsigned long long u64;
constexpr u64 EMPTY = ~0ull;

__device__ __forceinline__ u64 mix64(u64 x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
    return x;
}

// returns the slot of `key` in the table (inserting it when absent)
__device__ __forceinline__ unsigned table_insert(u64* __restrict__ keys, unsigned mask, u64 key) {
    unsigned s = (unsigned)mix64(key) & mask;
    while (true) {
        const u64 prev = atomicCAS(keys + s, EMPTY, key);
        if (prev == EMPTY || prev == key) return s;
        s = (s + 1) & mask;
    }
}
// returns the slot or 0xffffffff when absent
__device__ __forceinline__ unsigned table_find(const u64* __restrict__ keys, unsigned mask, u64 key) {
    unsigned s = (unsigned)mix64(key) & mask;
    while (true) {
        const u64 k = keys[s];
        if (k == key) return s;
        if (k == EMPTY) return 0xffffffffu;
        s = (s + 1) & mask;
    }
}

// torch: floor((p - min) / voxel_size).long() with a Python-float voxel_size, which PyTorch's CUDA kernel evaluates as
// (p - min) * fl32(1 / voxel_size).  A correctly rounded division puts some points in the neighbouring voxel
// (1.3f / 0.1f = 12.999999, 1.3f * fl32(1 / 0.1f) = 13), so the reciprocal is taken once and multiplied, without contraction.
__device__ __forceinline__ float voxel_inv(float voxel) { return __fdiv_rn(1.0f, voxel); }

__device__ __forceinline__ u64 voxel_key(const float* __restrict__ p, long long i, const float* __restrict__ mn, float inv,
                                         int* __restrict__ overflow) {
    const long long vx = (long long)floorf(__fmul_rn(__fsub_rn(p[3 * i], mn[0]), inv));
    const long long vy = (long long)floorf(__fmul_rn(__fsub_rn(p[3 * i + 1], mn[1]), inv));
    const long long vz = (long long)floorf(__fmul_rn(__fsub_rn(p[3 * i + 2], mn[2]), inv));
    if ((vx | vy | vz) >> 21) *overflow = 1;
    return ((u64)vx << 42) | ((u64)vy << 21) | (u64)vz;
}

__global__ void __launch_bounds__(256)
voxel_insert_orig_kernel(long long N, const float* __restrict__ xyz, const long long* __restrict__ cls, const float* __restrict__ mn,
                         float voxel, u64* __restrict__ vkeys, unsigned vmask, u64* __restrict__ pkeys, int* __restrict__ pcount,
                         unsigned pmask, unsigned* __restrict__ slot_of, int* __restrict__ overflow) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const u64 key = voxel_key(xyz, i, mn, voxel_inv(voxel), overflow);
    const unsigned s = table_insert(vkeys, vmask, key);
    slot_of[i] = s;
    const u64 pair = ((u64)s << 32) | (u64)(unsigned)cls[i];
    const unsigned ps = table_insert(pkeys, pmask, pair);
    atomicAdd(pcount + ps, 1);
}

// one thread per pair-table slot: best[voxel slot] = max over its classes of (count << 32 | ~class)
__global__ void __launch_bounds__(256)
voxel_vote_kernel(unsigned P, const u64* __restrict__ pkeys, const int* __restrict__ pcount, u64* __restrict__ best) {
    const unsigned s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= P) return;
    const u64 pair = pkeys[s];
    if (pair == EMPTY) return;
    const unsigned vslot = (unsigned)(pair >> 32), c = (unsigned)pair;
    atomicMax(best + vslot, ((u64)(unsigned)pcount[s] << 32) | (u64)(0xffffffffu - c));
}

__global__ void __launch_bounds__(256)
voxel_label_orig_kernel(long long N, const unsigned* __restrict__ slot_of, const u64* __restrict__ best, long long* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    out[i] = (long long)(0xffffffffu - (unsigned)best[slot_of[i]]);
}

// new points: label from the voxel table, or insertion of the key into the table of unmatched voxels (uslot_of >= 0)
__global__ void __launch_bounds__(256)
voxel_match_new_kernel(long long M, const float* __restrict__ xyz, const float* __restrict__ mn, float voxel,
                       const u64* __restrict__ vkeys, unsigned vmask, const u64* __restrict__ best, int have_orig,
                       u64* __restrict__ ukeys, unsigned umask, int* __restrict__ uslot_of, long long* __restrict__ out,
                       int* __restrict__ overflow) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M) return;
    const u64 key = voxel_key(xyz, i, mn, voxel_inv(voxel), overflow);
    const unsigned s = have_orig ? table_find(vkeys, vmask, key) : 0xffffffffu;
    if (s != 0xffffffffu) {
        out[i] = (long long)(0xffffffffu - (unsigned)best[s]);
        uslot_of[i] = -1;
    } else {
        uslot_of[i] = (int)table_insert(ukeys, umask, key);
    }
}

// compacts the distinct unmatched keys: list[atomic++] = key
__global__ void __launch_bounds__(256)
voxel_collect_kernel(unsigned U, const u64* __restrict__ ukeys, u64* __restrict__ list, int* __restrict__ count) {
    const unsigned s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= U) return;
    const u64 k = ukeys[s];
    if (k != EMPTY) list[atomicAdd(count, 1)] = k;
}

// sorted[r] -> rank r stored at the key's table slot
__global__ void __launch_bounds__(256)
voxel_rank_kernel(int n, const u64* __restrict__ sorted, const u64* __restrict__ ukeys, unsigned umask, int* __restrict__ urank) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    urank[table_find(ukeys, umask, sorted[r])] = r;
}

__global__ void __launch_bounds__(256)
voxel_label_new_kernel(long long M, const int* __restrict__ uslot_of, const int* __restrict__ urank, long long base,
                       long long* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M) return;
    const int s = uslot_of[i];
    if (s >= 0) out[i] = base + urank[s];
}

}  // namespace

// Stage 1 (original points): tables must be pre-filled by the caller — vkeys[V], pkeys[P] with 0xFF bytes, pcount[P] and
// best[V] with zeros; V and P powers of two >= 2 N.  mn: device float[3] = min over original AND new points.
// Writes slot_of[N] (scratch) and cls_out[N] = majority class of each point's voxel.
ADB_API int adb_voxel_vote(long long N, const float* xyz, const long long* cls, const float* mn, float voxel_size,
                           void* vkeys, long long V, void* pkeys, int* pcount, long long P, void* best, unsigned* slot_of,
                           long long* cls_out, int* overflow, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && voxel_size > 0.f, "adb_voxel_vote: bad sizes");
    if (N == 0) return ADB_OK;
    ADB_REQUIRE(V >= 2 * N && (V & (V - 1)) == 0 && P >= 2 * N && (P & (P - 1)) == 0 && V <= 0x80000000LL && P <= 0x80000000LL,
                "adb_voxel_vote: table sizes must be powers of two >= 2N");
    ADB_REQUIRE(xyz && cls && mn && vkeys && pkeys && pcount && best && slot_of && cls_out && overflow, "adb_voxel_vote: null pointer");
    voxel_insert_orig_kernel<<<adb_cdiv(N, 256), 256, 0, stream>>>(N, xyz, cls, mn, voxel_size, (u64*)vkeys, (unsigned)(V - 1),
                                                                  (u64*)pkeys, pcount, (unsigned)(P - 1), slot_of, overflow);
    ADB_CHECK_LAUNCH("voxel_insert_orig_kernel");
    voxel_vote_kernel<<<adb_cdiv(P, 256), 256, 0, stream>>>((unsigned)P, (const u64*)pkeys, pcount, (u64*)best);
    ADB_CHECK_LAUNCH("voxel_vote_kernel");
    voxel_label_orig_kernel<<<adb_cdiv(N, 256), 256, 0, stream>>>(N, slot_of, (const u64*)best, cls_out);
    ADB_CHECK_LAUNCH("voxel_label_orig_kernel");
    return ADB_OK;
}

// Stage 2 (new points): matched points get their voxel's majority class; the distinct unmatched voxel keys are collected
// into ulist (capacity >= M) with their number in *ucount (device).  ukeys[U] pre-filled with 0xFF, U power of two >= 2 M.
ADB_API int adb_voxel_match_new(long long M, const float* new_xyz, const float* mn, float voxel_size, const void* vkeys,
                                long long V, const void* best, int have_orig, void* ukeys, long long U, int* uslot_of,
                                long long* cls_out, void* ulist, int* ucount, int* overflow, cudaStream_t stream) {
    ADB_REQUIRE(M >= 0 && voxel_size > 0.f, "adb_voxel_match_new: bad sizes");
    if (M == 0) return ADB_OK;
    ADB_REQUIRE(U >= 2 * M && (U & (U - 1)) == 0 && U <= 0x80000000LL, "adb_voxel_match_new: U must be a power of two >= 2M");
    ADB_REQUIRE(new_xyz && mn && ukeys && uslot_of && cls_out && ulist && ucount && overflow && (!have_orig || (vkeys && best)),
                "adb_voxel_match_new: null pointer");
    voxel_match_new_kernel<<<adb_cdiv(M, 256), 256, 0, stream>>>(M, new_xyz, mn, voxel_size, (const u64*)vkeys,
                                                                (unsigned)(have_orig ? V - 1 : 0), (const u64*)best, have_orig,
                                                                (u64*)ukeys, (unsigned)(U - 1), uslot_of, cls_out, overflow);
    ADB_CHECK_LAUNCH("voxel_match_new_kernel");
    voxel_collect_kernel<<<adb_cdiv(U, 256), 256, 0, stream>>>((unsigned)U, (const u64*)ukeys, (u64*)ulist, ucount);
    ADB_CHECK_LAUNCH("voxel_collect_kernel");
    return ADB_OK;
}

// Stage 3: `sorted` = the n distinct unmatched keys in ascending order; unmatched new points get base + rank of their voxel.
ADB_API int adb_voxel_rank_new(long long M, int n, const void* sorted, const void* ukeys, long long U, int* urank,
                               const int* uslot_of, long long base, long long* cls_out, cudaStream_t stream) {
    ADB_REQUIRE(M >= 0 && n >= 0, "adb_voxel_rank_new: bad sizes");
    if (M == 0 || n == 0) return ADB_OK;
    ADB_REQUIRE(sorted && ukeys && urank && uslot_of && cls_out, "adb_voxel_rank_new: null pointer");
    voxel_rank_kernel<<<adb_cdiv(n, 256), 256, 0, stream>>>(n, (const u64*)sorted, (const u64*)ukeys, (unsigned)(U - 1), urank);
    ADB_CHECK_LAUNCH("voxel_rank_kernel");
    voxel_label_new_kernel<<<adb_cdiv(M, 256), 256, 0, stream>>>(M, uslot_of, urank, base, cls_out);
    ADB_CHECK_LAUNCH("voxel_label_new_kernel");
    return ADB_OK;
}

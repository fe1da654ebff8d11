// Gradient exchange of the multi-view optimiser step over NVLink peer memory (BASELINE config 4, SURVEY.md §8e).
//
// One process per GPU; every rank owns ONE peer-visible region (cudaMalloc + CUDA IPC handle, opened by the other ranks with
// lazy peer access), and all inter-GPU traffic is plain stores issued by these kernels through the NVSwitch — no remote
// loads, no library collective:
//
//   all-gather of the colour gradients   peer_push_rgb_kernel: the clamp mask of the SH colour (raster.mask_rgb_grad) fused
//                                        with the broadcast — each rank writes its view's [N,3] row into the table of EVERY
//                                        rank (own included);
//   all-reduce of the [N,11] geometry    peer_scatter_kernel: rank r pushes shard s of its partial sums into slot r of rank s's
//   gradients (reduce-scatter + gather)  staging area;  peer_reduce_bcast_kernel: rank s adds its W slots in rank order (every
//                                        rank therefore receives bit-identical sums) and writes the reduced shard into every
//                                        rank's result buffer.
//
// Ordering between ranks: monotonic step counters in the peer region.  A producer finishes its stores, then
// peer_signal_kernel does fence.sys + st.release.sys of the step number into slot [phase][rank] of every peer; a consumer runs
// peer_wait_kernel (ld.acquire.sys spin, bounded by a wall-clock timeout that sets an error word instead of hanging the GPU)
// before the kernel that reads the data.  The colour table is double-buffered by step parity, so a rank that runs ahead never
// overwrites rows a slower rank is still expanding; the staging and result buffers are protected by the protocol itself
// (nobody can scatter step e+1 before every rank has signalled the end of its step-e reduction).
#include "common.cuh"
#include "raster_common.cuh"
#include <stdlib.h>
#include <string.h>

namespace {

constexpr int MAXW = 8;          // ranks on one NVSwitch domain
struct PeerPtrs { void* p[MAXW]; };

__device__ __forceinline__ void st_release_sys(unsigned* addr, unsigned v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* addr) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(addr) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// flags layout on every rank: unsigned [n_slots][MAXW]; word [slot][r] is written by rank r only.
__global__ void peer_signal_kernel(PeerPtrs flags, int world, int slot, int rank, unsigned value) {
    const int p = threadIdx.x;
    if (p >= world) return;
    __threadfence_system();
    st_release_sys(reinterpret_cast<unsigned*>(flags.p[p]) + slot * MAXW + rank, value);
}

// Waits until flags[slot][r] has reached `value` for every r < world and every slot in [slot_lo, slot_lo + n_slots).
__global__ void peer_wait_kernel(const unsigned* __restrict__ flags, int world, int slot_lo, int n_slots, unsigned value,
                                 unsigned long long timeout_ns, int* __restrict__ err) {
    const int t = threadIdx.x;
    if (t >= world * n_slots) return;
    const unsigned* f = flags + (slot_lo + t / world) * MAXW + (t % world);
    const unsigned long long t0 = globaltimer_ns();
    while ((int)(ld_acquire_sys(f) - value) < 0) {
        if (globaltimer_ns() - t0 > timeout_ns) { atomicExch(err, 1 + slot_lo + t / world); break; }
        __nanosleep(64);
    }
}

// dst_r[row_off + i*3 .. +3] = (splats[i].rgb > 0) ? v_splats[i].v_rgb : 0   for every rank r; campos (3 floats) -> cam_r.
__global__ void __launch_bounds__(256)
peer_push_rgb_kernel(int N, const float* __restrict__ splats, const float* __restrict__ v_splats, PeerPtrs dst, int world,
                     size_t row_off, const float* __restrict__ campos, PeerPtrs cam, size_t cam_off) {
    // 4 Gaussians per thread and iteration: 12 floats = three 128-bit stores per destination
    if (blockIdx.x == 0 && threadIdx.x < 3 && campos) {
        const float v = campos[threadIdx.x];
        for (int r = 0; r < world; ++r) reinterpret_cast<float*>(cam.p[r])[cam_off + threadIdx.x] = v;
    }
    const int nq = (N + 3) / 4;
    for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += gridDim.x * blockDim.x) {
        const int i0 = q * 4;
        float g[12];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int i = i0 + k;
            if (i < N) {
                const float4 C = __ldg(reinterpret_cast<const float4*>(splats + (size_t)i * ADB_SPLAT_STRIDE) + 2);
                const float4 v1 = __ldg(reinterpret_cast<const float4*>(v_splats + (size_t)i * ADB_SPLAT_STRIDE) + 1);
                const float4 v2 = __ldg(reinterpret_cast<const float4*>(v_splats + (size_t)i * ADB_SPLAT_STRIDE) + 2);
                g[3 * k] = C.x > 0.f ? v1.z : 0.f;
                g[3 * k + 1] = C.y > 0.f ? v1.w : 0.f;
                g[3 * k + 2] = C.z > 0.f ? v2.x : 0.f;
            } else {
                g[3 * k] = g[3 * k + 1] = g[3 * k + 2] = 0.f;
            }
        }
        if (i0 + 4 <= N) {
            for (int r = 0; r < world; ++r) {
                float4* d = reinterpret_cast<float4*>(reinterpret_cast<float*>(dst.p[r]) + row_off + (size_t)i0 * 3);
                d[0] = make_float4(g[0], g[1], g[2], g[3]);
                d[1] = make_float4(g[4], g[5], g[6], g[7]);
                d[2] = make_float4(g[8], g[9], g[10], g[11]);
            }
        } else {
            for (int r = 0; r < world; ++r) {
                float* d = reinterpret_cast<float*>(dst.p[r]) + row_off + (size_t)i0 * 3;
                for (int k = 0; k < (N - i0) * 3; ++k) d[k] = g[k];
            }
        }
    }
}

// Plain broadcast of a ready-made [n4] float4 row (the autograd path hands over g_rgb already masked).
__global__ void __launch_bounds__(256)
peer_bcast_kernel(size_t n4, const float4* __restrict__ src, PeerPtrs dst, int world, size_t off4,
                  const float* __restrict__ campos, PeerPtrs cam, size_t cam_off) {
    if (blockIdx.x == 0 && threadIdx.x < 3 && campos) {
        const float v = campos[threadIdx.x];
        for (int r = 0; r < world; ++r) reinterpret_cast<float*>(cam.p[r])[cam_off + threadIdx.x] = v;
    }
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const float4 v = adb_ldg_stream4(src + i);
        for (int r = 0; r < world; ++r) reinterpret_cast<float4*>(dst.p[r])[off4 + i] = v;
    }
}

// Reduce-scatter by push: float4 i of the local partial sums belongs to shard s = i / per and goes to slot `rank` of rank s's
// staging area  stage_s[rank*per + (i - s*per)].
__global__ void __launch_bounds__(256)
peer_scatter_kernel(size_t n4, size_t per, const float4* __restrict__ src, PeerPtrs stage, int rank) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const size_t s = i / per;
        reinterpret_cast<float4*>(stage.p[s])[(size_t)rank * per + (i - s * per)] = adb_ldg_stream4(src + i);
    }
}

// Shard owner: out[rank*per + j] = sum over r (ascending) of stage[r*per + j], written into every rank's result buffer.
__global__ void __launch_bounds__(256)
peer_reduce_bcast_kernel(size_t n_own, size_t per, const float4* __restrict__ stage, PeerPtrs out, int world, int rank) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < n_own; j += stride) {
        float4 v[MAXW];
#pragma unroll
        for (int r = 0; r < MAXW; ++r)
            if (r < world) v[r] = __ldcg(stage + (size_t)r * per + j);
        float4 a = v[0];
#pragma unroll
        for (int r = 1; r < MAXW; ++r)
            if (r < world) { a.x += v[r].x; a.y += v[r].y; a.z += v[r].z; a.w += v[r].w; }
        for (int r = 0; r < world; ++r) reinterpret_cast<float4*>(out.p[r])[(size_t)rank * per + j] = a;
    }
}

int fill_ptrs(PeerPtrs* pp, void* const* ptrs, int world) {
    for (int r = 0; r < MAXW; ++r) pp->p[r] = r < world ? ptrs[r] : nullptr;
    for (int r = 0; r < world; ++r)
        if (!ptrs[r]) return ADB_ERR_INVALID;
    return ADB_OK;
}

// CTAs per exchange kernel (ADB_PEER_CTAS, 1..2112; default: no cap below 16 CTAs per SM of an H100).  The kernels are
// NVLink-bound: grids over every SM give the exchange the most memory parallelism, but their remote stores can stall the
// backward kernels running beside the push on many GPUs; a small cap (e.g. 32 CTAs) avoids that contention at the cost of
// slower copies.  Not tuned on H100.
int peer_ctas() {
    static int n = [] {
        const char* e = getenv("ADB_PEER_CTAS");
        const int v = e ? atoi(e) : 132 * 16;
        return v < 1 ? 1 : (v > 132 * 16 ? 132 * 16 : v);
    }();
    return n;
}

int grid_for(size_t n, int threads) {
    const size_t g = (n + threads - 1) / threads;
    const size_t cap = (size_t)peer_ctas();
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

// ---- peer-visible memory (CUDA IPC) -------------------------------------------------------------------------------------
ADB_API int adb_peer_alloc(size_t bytes, void** ptr) {
    ADB_REQUIRE(ptr && bytes > 0, "adb_peer_alloc: bad arguments");
    ADB_CUDA(cudaMalloc(ptr, bytes));
    ADB_CUDA(cudaMemset(*ptr, 0, bytes));
    ADB_CUDA(cudaDeviceSynchronize());
    return ADB_OK;
}
ADB_API int adb_peer_free(void* ptr) {
    if (ptr) ADB_CUDA(cudaFree(ptr));
    return ADB_OK;
}
ADB_API int adb_peer_export(void* ptr, unsigned char* handle64) {
    ADB_REQUIRE(ptr && handle64, "adb_peer_export: null pointer");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    cudaIpcMemHandle_t h;
    ADB_CUDA(cudaIpcGetMemHandle(&h, ptr));
    memcpy(handle64, &h, 64);
    return ADB_OK;
}
ADB_API int adb_peer_import(const unsigned char* handle64, void** ptr) {
    ADB_REQUIRE(ptr && handle64, "adb_peer_import: null pointer");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    ADB_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return ADB_OK;
}
ADB_API int adb_peer_close(void* ptr) {
    if (ptr) ADB_CUDA(cudaIpcCloseMemHandle(ptr));
    return ADB_OK;
}

// Loads every kernel of this file now.  With lazy module loading (the CUDA 12 default) the FIRST launch of a kernel may have to
// wait for the device to drain — which never happens while a wait kernel spins on a flag that the kernel being loaded is
// supposed to help raise.  Called once per process by peer.PeerExchange before any signal is sent.
ADB_API int adb_peer_warmup(void) {
    cudaFuncAttributes a;
    ADB_CUDA(cudaFuncGetAttributes(&a, peer_signal_kernel));
    ADB_CUDA(cudaFuncGetAttributes(&a, peer_wait_kernel));
    ADB_CUDA(cudaFuncGetAttributes(&a, peer_push_rgb_kernel));
    ADB_CUDA(cudaFuncGetAttributes(&a, peer_bcast_kernel));
    ADB_CUDA(cudaFuncGetAttributes(&a, peer_scatter_kernel));
    ADB_CUDA(cudaFuncGetAttributes(&a, peer_reduce_bcast_kernel));
    return ADB_OK;
}

// ---- ordering -----------------------------------------------------------------------------------------------------------
ADB_API int adb_peer_signal(void* const* flag_ptrs, int world, int slot, int rank, unsigned value, cudaStream_t stream) {
    ADB_REQUIRE(flag_ptrs && world >= 1 && world <= MAXW && slot >= 0 && rank >= 0 && rank < world, "adb_peer_signal: bad arguments");
    PeerPtrs f;
    ADB_REQUIRE(fill_ptrs(&f, flag_ptrs, world) == ADB_OK, "adb_peer_signal: null peer pointer");
    peer_signal_kernel<<<1, 32, 0, stream>>>(f, world, slot, rank, value);
    ADB_CHECK_LAUNCH("peer_signal_kernel");
    return ADB_OK;
}
ADB_API int adb_peer_wait(const void* local_flags, int world, int slot_lo, int n_slots, unsigned value, double timeout_s,
                          int* err, cudaStream_t stream) {
    ADB_REQUIRE(local_flags && err && world >= 1 && world <= MAXW && slot_lo >= 0 && n_slots >= 1 && world * n_slots <= 256,
                "adb_peer_wait: bad arguments");
    const unsigned long long ns = (unsigned long long)((timeout_s > 0 ? timeout_s : 5.0) * 1e9);
    peer_wait_kernel<<<1, 256, 0, stream>>>(reinterpret_cast<const unsigned*>(local_flags), world, slot_lo, n_slots, value, ns, err);
    ADB_CHECK_LAUNCH("peer_wait_kernel");
    return ADB_OK;
}

// ---- data ---------------------------------------------------------------------------------------------------------------
// Row `row_off` (in floats) of every rank's colour table <- masked colour gradient of one local view; cam_ptrs/cam_off (in
// floats): where the view's camera centre goes (campos may be NULL).
ADB_API int adb_peer_push_rgb(int N, const float* splats, const float* v_splats, void* const* dst_ptrs, int world,
                              size_t row_off, const float* campos, void* const* cam_ptrs, size_t cam_off, cudaStream_t stream) {
    ADB_REQUIRE(N >= 0 && splats && v_splats && dst_ptrs && world >= 1 && world <= MAXW && row_off % 4 == 0,
                "adb_peer_push_rgb: bad arguments");
    if (N == 0) return ADB_OK;
    PeerPtrs d, c = {};
    ADB_REQUIRE(fill_ptrs(&d, dst_ptrs, world) == ADB_OK, "adb_peer_push_rgb: null peer pointer");
    if (campos) ADB_REQUIRE(cam_ptrs && fill_ptrs(&c, cam_ptrs, world) == ADB_OK, "adb_peer_push_rgb: null camera pointer");
    peer_push_rgb_kernel<<<grid_for((size_t)adb_cdiv(N, 4), 256), 256, 0, stream>>>(N, splats, v_splats, d, world, row_off, campos, c, cam_off);
    ADB_CHECK_LAUNCH("peer_push_rgb_kernel");
    return ADB_OK;
}
ADB_API int adb_peer_bcast(size_t n_floats, const float* src, void* const* dst_ptrs, int world, size_t off_floats,
                           const float* campos, void* const* cam_ptrs, size_t cam_off, cudaStream_t stream) {
    ADB_REQUIRE(src && dst_ptrs && world >= 1 && world <= MAXW && n_floats % 4 == 0 && off_floats % 4 == 0,
                "adb_peer_bcast: bad arguments (sizes must be multiples of 4 floats)");
    if (n_floats == 0) return ADB_OK;
    PeerPtrs d, c = {};
    ADB_REQUIRE(fill_ptrs(&d, dst_ptrs, world) == ADB_OK, "adb_peer_bcast: null peer pointer");
    if (campos) ADB_REQUIRE(cam_ptrs && fill_ptrs(&c, cam_ptrs, world) == ADB_OK, "adb_peer_bcast: null camera pointer");
    peer_bcast_kernel<<<grid_for(n_floats / 4, 256), 256, 0, stream>>>(n_floats / 4, reinterpret_cast<const float4*>(src), d, world,
                                                                       off_floats / 4, campos, c, cam_off);
    ADB_CHECK_LAUNCH("peer_bcast_kernel");
    return ADB_OK;
}
// n4 float4 of partial sums, shards of `per4` float4 (world * per4 >= n4): push shard s into slot `rank` of stage_ptrs[s].
ADB_API int adb_peer_scatter(size_t n4, size_t per4, const float* src, void* const* stage_ptrs, int world, int rank,
                             cudaStream_t stream) {
    ADB_REQUIRE(src && stage_ptrs && world >= 1 && world <= MAXW && rank >= 0 && rank < world && per4 > 0 && per4 * world >= n4,
                "adb_peer_scatter: bad arguments");
    if (n4 == 0) return ADB_OK;
    PeerPtrs s;
    ADB_REQUIRE(fill_ptrs(&s, stage_ptrs, world) == ADB_OK, "adb_peer_scatter: null peer pointer");
    peer_scatter_kernel<<<grid_for(n4, 256), 256, 0, stream>>>(n4, per4, reinterpret_cast<const float4*>(src), s, rank);
    ADB_CHECK_LAUNCH("peer_scatter_kernel");
    return ADB_OK;
}
// Sum the `world` slots of the local staging area over this rank's shard ([rank*per4, min(n4, (rank+1)*per4))) and write the
// result into every rank's result buffer at the same position.
ADB_API int adb_peer_reduce_bcast(size_t n4, size_t per4, const float* stage, void* const* out_ptrs, int world, int rank,
                                  cudaStream_t stream) {
    ADB_REQUIRE(stage && out_ptrs && world >= 1 && world <= MAXW && rank >= 0 && rank < world && per4 > 0 && per4 * world >= n4,
                "adb_peer_reduce_bcast: bad arguments");
    const size_t lo = (size_t)rank * per4;
    if (lo >= n4) return ADB_OK;
    const size_t n_own = (n4 - lo < per4) ? n4 - lo : per4;
    PeerPtrs o;
    ADB_REQUIRE(fill_ptrs(&o, out_ptrs, world) == ADB_OK, "adb_peer_reduce_bcast: null peer pointer");
    peer_reduce_bcast_kernel<<<grid_for(n_own, 256), 256, 0, stream>>>(n_own, per4, reinterpret_cast<const float4*>(stage), o, world, rank);
    ADB_CHECK_LAUNCH("peer_reduce_bcast_kernel");
    return ADB_OK;
}

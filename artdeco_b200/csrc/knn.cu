// Exact K-nearest-neighbour queries on a uniform grid hash (no host synchronisation, no allocation).
//
// Replaces simple-knn (Reconstruct/submodules/simple-knn):
//   SimpleKNN::knn        simple_knn.cu:188-224  (distCUDA2,  spatial.cu:16-26)  -> adb_knn_mean3
//   SimpleKNN::knn_index2 simple_knn.cu:468-522  (distIndex2, spatial.cu:29-41)  -> adb_knn_index (query_idx = NULL)
//   SimpleKNN::knn_indexQ simple_knn.cu:592-651  (distIndexQ, spatial.cu:44-58)  -> adb_knn_index (query + candidates)
// The reference Morton-sorts the points, boxes them in fixed groups of 1024/128 and makes every thread walk boxes
// with a scalar, uncoalesced gather (points[indices[i]]), after two blocking D2H copies of the bounding box.
// Here: bounding box, grid sizing and cell ids stay on the device; points are radix-sorted by cell id and
// REORDERED into a float4 array (x,y,z,original index), so a row of x-adjacent cells is one contiguous,
// coalesced bucket scan; each query searches Chebyshev shells r = 0,1,2,.. of cells.
//
// Exactness.  A point's cell is floor(fl(fl(x - minx) * fl(1/h))): three roundings, so the computed coordinate
// (in cells) is within 3*2^-24 * n of the true (x - minx)/h, n = the largest cell count of any axis (clamping
// into [0, n-1] only moves a point further from the cells it is clamped away from).  Two points whose cells
// differ by r+1 along an axis are therefore more than (r - slack)*h apart, slack = 2 * 8*2^-24 * n = n*2^-20
// (8 ulps per coordinate, with margin).  The search stops after shell r once the K-th best squared distance is
// <= ((0.99999*r - slack)*h)^2; the factor 0.99999 covers the relative rounding of the fp32 distance (a few
// ulps) and of the bound itself.  Every point not yet visited is then no closer than the K-th best, and the
// result equals the brute force.  On wide grids (hundreds of cells per axis) the fixed 0.99999 alone is not
// enough: a point two cells away can be up to ~4e-5 of a cell closer than 1*h.
// Points with a NaN, an infinite or a coordinate above kFar in magnitude are nobody's neighbour: their squared
// distance to any point near the rest of the cloud overflows fp32, which the brute force never selects.  They
// are left out of the bounding box (one such point would otherwise stretch the grid until every other point
// shares a cell), get a key past the last cell, so they sort to the end and are never scanned, and their own
// row is FLT_MAX / -1 (distCUDA2: inf).  The one difference from the brute force: two such points closer than
// sqrt(FLT_MAX) to each other are not each other's neighbours here.
// Squared distances are evaluated as fma(dz,dz,fma(dx,dx,dy*dy)) — the contraction nvcc applies to the
// reference's `d.x*d.x + d.y*d.y + d.z*d.z` (simple_knn.cu:136,400) — so distCUDA2 is bit-reproducible.
#include "common.cuh"
#include <cfloat>
#include <cub/device/device_radix_sort.cuh>

namespace {

struct Grid {
    float minx, miny, minz, h, inv_h;
    int nx, ny, nz, ncells;
    float slack;  // worst-case error of a cell coordinate difference, in cells (see the header)
};

// |coordinate| above this makes a point unusable (its squared distance to the origin exceeds FLT_MAX)
constexpr float kFar = 1.8e19f;

__device__ __forceinline__ bool usable(float x, float y, float z) {
    return fabsf(x) <= kFar && fabsf(y) <= kFar && fabsf(z) <= kFar;  // false for NaN and +-inf too
}

struct Ws {  // carved out of the caller's workspace
    Grid* grid;
    unsigned* bbox;  // 6 ordered-uint encodings
    unsigned *keys_a, *keys_b;
    int *vals_a, *vals_b;
    float4* sorted;
    int* cell_start;
    int* pos_of;  // original index -> sorted position
    void* cub;
    size_t cub_bytes;
};

__host__ size_t align_up(size_t v) { return (v + 255) & ~(size_t)255; }

__host__ size_t carve(long long P, void* base, size_t cub_bytes, Ws* w) {
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t at = o; o += align_up(bytes); return base ? (char*)base + at : (char*)nullptr; };
    char* g = take(sizeof(Grid));
    char* bb = take(6 * sizeof(unsigned));
    char* ka = take(sizeof(unsigned) * P), *kb = take(sizeof(unsigned) * P);
    char* va = take(sizeof(int) * P), *vb = take(sizeof(int) * P);
    char* so = take(sizeof(float4) * P);
    char* cs = take(sizeof(int) * (2 * P + 66));
    char* po = take(sizeof(int) * P);
    char* cu = take(cub_bytes);
    if (w) {
        w->grid = (Grid*)g; w->bbox = (unsigned*)bb; w->keys_a = (unsigned*)ka; w->keys_b = (unsigned*)kb;
        w->vals_a = (int*)va; w->vals_b = (int*)vb; w->sorted = (float4*)so; w->cell_start = (int*)cs;
        w->pos_of = (int*)po; w->cub = cu; w->cub_bytes = cub_bytes;
    }
    return o;
}

// order-preserving float <-> uint
__device__ __forceinline__ unsigned f2o(float f) {
    unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float o2f(unsigned u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

__global__ void bbox_init_kernel(unsigned* bbox) {
    if (threadIdx.x < 3) bbox[threadIdx.x] = 0xffffffffu;       // mins
    else if (threadIdx.x < 6) bbox[threadIdx.x] = 0u;           // maxs
}

__global__ void __launch_bounds__(256)
bbox_kernel(long long P, const float* __restrict__ pts, unsigned* __restrict__ bbox) {
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x) {
        const float v[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
        if (!usable(v[0], v[1], v[2])) continue;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            mn[a] = fminf(mn[a], v[a]);
            mx[a] = fmaxf(mx[a], v[a]);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
            mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
        }
    if ((threadIdx.x & 31) == 0)
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            atomicMin(bbox + a, f2o(mn[a]));
            atomicMax(bbox + 3 + a, f2o(mx[a]));
        }
}

// single thread: choose the cell size so that a cell holds ~4 points, with at most 2P+64 cells.  The volume is
// formed in double: extents up to 2*kFar would overflow fp32.  With no usable point the box is empty (min > max)
// and the grid is one cell at the origin.
__global__ void grid_setup_kernel(long long P, const unsigned* bbox, Grid* g) {
    float mn[3], e[3];
    float emax = 0.f;
    for (int a = 0; a < 3; ++a) {
        const float lo = o2f(bbox[a]), hi = o2f(bbox[3 + a]);
        const bool empty = !(lo <= hi);
        mn[a] = empty ? 0.f : lo;
        e[a] = empty ? 0.f : hi - lo;
        emax = fmaxf(emax, e[a]);
    }
    if (!(emax > 0.f)) emax = 1.f;
    double vol = 1.0;
    for (int a = 0; a < 3; ++a) vol *= (double)fmaxf(e[a], 1e-3f * emax);
    float h = (float)cbrt(4.0 * vol / (double)P);
    if (!(h > 0.f)) h = emax;
    const long long cap = 2 * P + 64;
    int n[3];
    for (int it = 0; it < 64; ++it) {
        long long tot = 1;
        for (int a = 0; a < 3; ++a) {
            float c = floorf(e[a] / h) + 1.f;
            n[a] = c > 2.0e6f ? 2000000 : (int)c;
            tot *= n[a];
        }
        if (tot <= cap) break;
        h *= 1.26f;
    }
    g->minx = mn[0]; g->miny = mn[1]; g->minz = mn[2];
    g->h = h; g->inv_h = 1.0f / h;
    g->nx = n[0]; g->ny = n[1]; g->nz = n[2];
    g->ncells = n[0] * n[1] * n[2];
    g->slack = (float)max(n[0], max(n[1], n[2])) * 0x1p-20f;
}

__device__ __forceinline__ void cell_of(const Grid& g, float x, float y, float z, int& cx, int& cy, int& cz) {
    cx = min(max((int)floorf((x - g.minx) * g.inv_h), 0), g.nx - 1);
    cy = min(max((int)floorf((y - g.miny) * g.inv_h), 0), g.ny - 1);
    cz = min(max((int)floorf((z - g.minz) * g.inv_h), 0), g.nz - 1);
}

__global__ void __launch_bounds__(256)
cell_id_kernel(long long P, const float* __restrict__ pts, const Grid* __restrict__ gp, unsigned* __restrict__ keys,
               int* __restrict__ vals) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const Grid g = *gp;
    const float x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
    int cx, cy, cz;
    cell_of(g, x, y, z, cx, cy, cz);
    keys[i] = usable(x, y, z) ? (unsigned)((cz * g.ny + cy) * g.nx + cx) : (unsigned)g.ncells;  // past the last cell
    vals[i] = (int)i;
}

__global__ void __launch_bounds__(256)
reorder_kernel(long long P, const float* __restrict__ pts, const unsigned* __restrict__ keys,
               const int* __restrict__ vals, const Grid* __restrict__ gp, float4* __restrict__ sorted,
               int* __restrict__ cell_start, int* __restrict__ pos_of) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int src = vals[i];
    sorted[i] = make_float4(pts[3 * (size_t)src], pts[3 * (size_t)src + 1], pts[3 * (size_t)src + 2], __int_as_float(src));
    pos_of[src] = (int)i;
    const int ncells = gp->ncells;
    const int cur = (int)keys[i];
    if (i == 0) {
        for (int c = 0; c <= cur; ++c) cell_start[c] = 0;
    } else {
        const int prev = (int)keys[i - 1];
        for (int c = prev + 1; c <= cur; ++c) cell_start[c] = (int)i;
    }
    if (i == P - 1)
        for (int c = cur + 1; c <= ncells; ++c) cell_start[c] = (int)P;
}

template <int KMAX>
struct Best {
    float d[KMAX];
    int id[KMAX];
    __device__ __forceinline__ void init() {
#pragma unroll
        for (int k = 0; k < KMAX; ++k) { d[k] = FLT_MAX; id[k] = -1; }
    }
    // ascending insertion, ties keep the earlier-seen entry in front (like updateKBest, simple_knn.cu:134-148)
    __device__ __forceinline__ void push(float dist, int idx) {
#pragma unroll
        for (int k = 0; k < KMAX; ++k)
            if (d[k] > dist) {
                float td = d[k]; int ti = id[k];
                d[k] = dist; id[k] = idx;
                dist = td; idx = ti;
            }
    }
};

// MODE 0: mean of the 3 nearest (distCUDA2).  MODE 1: K nearest ids + distances.
template <int KMAX, int MODE>
__global__ void __launch_bounds__(128)
knn_query_kernel(long long P, long long Q, int K, const Grid* __restrict__ gp, const float4* __restrict__ sorted,
                 const int* __restrict__ cell_start, const int* __restrict__ pos_of,
                 const int* __restrict__ query_idx, const unsigned char* __restrict__ candidate,
                 float* __restrict__ out_d, int* __restrict__ out_i) {
    const long long qi = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (qi >= Q) return;
    const Grid g = *gp;
    // without an explicit query list, thread qi handles the qi-th point in CELL order (spatially coherent warps)
    const int spos = query_idx ? pos_of[query_idx[qi]] : (int)qi;
    const float4 me = sorted[spos];
    const int self = __float_as_int(me.w);
    const long long out_row = query_idx ? qi : (long long)self;
    int cx, cy, cz;
    cell_of(g, me.x, me.y, me.z, cx, cy, cz);
    Best<KMAX> best;
    best.init();
    // an unusable query keeps the empty row
    const int rmax = usable(me.x, me.y, me.z) ? max(g.nx, max(g.ny, g.nz)) : -1;
    for (int r = 0; r <= rmax; ++r) {
        const int z0 = max(cz - r, 0), z1 = min(cz + r, g.nz - 1);
        const int y0 = max(cy - r, 0), y1 = min(cy + r, g.ny - 1);
        for (int z = z0; z <= z1; ++z)
            for (int y = y0; y <= y1; ++y) {
                const bool full_row = (z == cz - r) || (z == cz + r) || (y == cy - r) || (y == cy + r);
                const int row = (z * g.ny + y) * g.nx;
                // the shell's cells in this row: the whole x-range, or just its two end cells
                for (int part = 0; part < 2; ++part) {
                    int xa, xb;
                    if (full_row) {
                        if (part) break;
                        xa = max(cx - r, 0); xb = min(cx + r, g.nx - 1);
                    } else {
                        xa = xb = part ? cx + r : cx - r;
                        if (xa < 0 || xa >= g.nx || (part && r == 0)) continue;
                    }
                    const int s = cell_start[row + xa], e = cell_start[row + xb + 1];
                    for (int j = s; j < e; ++j) {
                        const float4 p = sorted[j];
                        const int pid = __float_as_int(p.w);
                        if (pid == self) continue;
                        if (candidate && !candidate[pid]) continue;
                        const float dx = p.x - me.x, dy = p.y - me.y, dz = p.z - me.z;
                        const float dist = __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
                        if (dist < best.d[KMAX - 1]) best.push(dist, pid);
                    }
                }
            }
        // everything not yet visited is more than (r - slack)*h away (see the header)
        const int kth = (MODE == 0 ? 3 : K) - 1;
        const float bound = fmaxf((float)r * 0.99999f - g.slack, 0.f) * g.h;
        float kth_d = FLT_MAX;
#pragma unroll
        for (int k = 0; k < KMAX; ++k)
            if (k == kth) kth_d = best.d[k];
        if (kth_d <= bound * bound) break;
    }
    if (MODE == 0) {
        out_d[out_row] = (best.d[0] + best.d[1] + best.d[2]) / 3.0f;
    } else {
#pragma unroll
        for (int k = 0; k < KMAX; ++k)
            if (k < K) {
                out_d[out_row * K + k] = best.d[k];
                out_i[out_row * K + k] = best.id[k];
            }
    }
}

int build_grid(long long P, const float* points, const Ws& w, cudaStream_t stream) {
    bbox_init_kernel<<<1, 32, 0, stream>>>(w.bbox);
    const int blocks = (int)((P + 255) / 256 < 132 * 8 ? (P + 255) / 256 : 132 * 8);
    bbox_kernel<<<blocks, 256, 0, stream>>>(P, points, w.bbox);
    grid_setup_kernel<<<1, 1, 0, stream>>>(P, w.bbox, w.grid);
    cell_id_kernel<<<adb_cdiv(P, 256), 256, 0, stream>>>(P, points, w.grid, w.keys_a, w.vals_a);
    ADB_CHECK_LAUNCH("knn grid kernels");
    int bits = 1;  // keys go up to ncells <= 2P+64 (the unusable points' key)
    while (((long long)1 << bits) <= 2 * P + 64) ++bits;
    cub::DoubleBuffer<unsigned> dk(w.keys_a, w.keys_b);
    cub::DoubleBuffer<int> dv(w.vals_a, w.vals_b);
    size_t need = w.cub_bytes;
    ADB_CUDA(cub::DeviceRadixSort::SortPairs(w.cub, need, dk, dv, (int)P, 0, bits, stream));
    reorder_kernel<<<adb_cdiv(P, 256), 256, 0, stream>>>(P, points, dk.Current(), dv.Current(), w.grid, w.sorted,
                                                         w.cell_start, w.pos_of);
    ADB_CHECK_LAUNCH("knn reorder_kernel");
    return ADB_OK;
}

size_t cub_sort_bytes(long long P) {
    size_t b = 0;
    cub::DoubleBuffer<unsigned> dk(nullptr, nullptr);
    cub::DoubleBuffer<int> dv(nullptr, nullptr);
    cub::DeviceRadixSort::SortPairs(nullptr, b, dk, dv, (int)P, 0, 32);
    return b + 256;
}

}  // namespace

ADB_API int adb_knn_workspace_bytes(long long P, size_t* bytes) {
    ADB_REQUIRE(bytes && P >= 0 && P < 1000000000LL, "adb_knn_workspace_bytes: bad args");
    *bytes = carve(P > 0 ? P : 1, nullptr, cub_sort_bytes(P > 0 ? P : 1), nullptr) + 256;
    return ADB_OK;
}

// distCUDA2: mean squared distance to the 3 nearest other points, written in the ORIGINAL point order.
ADB_API int adb_knn_mean3(long long P, const float* points, float* mean_dists, void* ws, size_t ws_bytes,
                          cudaStream_t stream) {
    ADB_REQUIRE(P >= 0 && P < 1000000000LL, "adb_knn_mean3: bad P");
    if (P == 0) return ADB_OK;
    ADB_REQUIRE(points && mean_dists && ws, "adb_knn_mean3: null pointer");
    Ws w;
    const size_t need = carve(P, (void*)(((uintptr_t)ws + 255) & ~(uintptr_t)255), cub_sort_bytes(P), &w);
    if (need + 256 > ws_bytes) { adb_set_error_msg("adb_knn_mean3: workspace too small"); return ADB_ERR_WORKSPACE; }
    int rc = build_grid(P, points, w, stream);
    if (rc) return rc;
    knn_query_kernel<3, 0><<<adb_cdiv(P, 128), 128, 0, stream>>>(P, P, 3, w.grid, w.sorted, w.cell_start, w.pos_of,
                                                                 nullptr, nullptr, mean_dists, nullptr);
    ADB_CHECK_LAUNCH("knn_query_kernel<mean3>");
    return ADB_OK;
}

// distIndex2 (query_idx == NULL: every point queries, Q must equal P, rows in original point order) and
// distIndexQ (query_idx[Q] int32 original ids; candidate[P] uint8 restricts the neighbour set, may be NULL).
// dists/ids are [Q*K]; each row ascending by distance; unfilled slots are FLT_MAX / -1.
ADB_API int adb_knn_index(long long P, const float* points, int K, long long Q, const int32_t* query_idx,
                          const unsigned char* candidate, float* dists, int32_t* ids, void* ws, size_t ws_bytes,
                          cudaStream_t stream) {
    ADB_REQUIRE(P >= 0 && P < 1000000000LL && Q >= 0 && K >= 1, "adb_knn_index: bad sizes");
    ADB_REQUIRE(K <= 32, "adb_knn_index: K must be <= 32");
    ADB_REQUIRE(query_idx || Q == P, "adb_knn_index: Q must equal P when query_idx is NULL");
    if (P == 0 || Q == 0) return ADB_OK;
    ADB_REQUIRE(points && dists && ids && ws, "adb_knn_index: null pointer");
    Ws w;
    const size_t need = carve(P, (void*)(((uintptr_t)ws + 255) & ~(uintptr_t)255), cub_sort_bytes(P), &w);
    if (need + 256 > ws_bytes) { adb_set_error_msg("adb_knn_index: workspace too small"); return ADB_ERR_WORKSPACE; }
    int rc = build_grid(P, points, w, stream);
    if (rc) return rc;
    const int grid = adb_cdiv(Q, 128);
#define ADB_KNN_LAUNCH(KM)                                                                                         \
    knn_query_kernel<KM, 1><<<grid, 128, 0, stream>>>(P, Q, K, w.grid, w.sorted, w.cell_start, w.pos_of, query_idx, \
                                                      candidate, dists, ids)
    if (K <= 4) ADB_KNN_LAUNCH(4);
    else if (K <= 8) ADB_KNN_LAUNCH(8);
    else if (K <= 16) ADB_KNN_LAUNCH(16);
    else ADB_KNN_LAUNCH(32);
#undef ADB_KNN_LAUNCH
    ADB_CHECK_LAUNCH("knn_query_kernel<index>");
    return ADB_OK;
}

/* artdeco_b200 — C ABI of the H100-native (sm_90a) kernels behind ARTDECO's hot-path operators.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the comment says HOST; tensors are dense, row-major, fp32
 *     unless typed otherwise; no allocation happens inside the library (the caller passes outputs and
 *     workspaces); every entry point returns 0 on success, 1 = invalid argument, 2 = CUDA error,
 *     3 = workspace too small, and adb_last_error() (HOST, thread-local) describes the failure;
 *   - every launch goes to the `stream` argument (a cudaStream_t); nothing synchronises the device;
 *   - each declaration cites the reference interface it replaces (paths relative to the ARTDECO tree).
 *   INTEGRATION.md shows the ctypes / pybind binding a reference maintainer would add.
 */
#ifndef ARTDECO_B200_H
#define ARTDECO_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* adb_stream_t; /* == cudaStream_t */

/* ---- library ---- */
const char* adb_last_error(void);
int adb_version(void);
int adb_check_device(void); /* 0 iff the current device is compute capability 9.0 */

/* ---- fused SSIM ----
 * replaces fused_ssim_cuda.fusedssim          Reconstruct/submodules/fused-ssim/ssim.cu:434-478 (ext.cpp:5)
 *          fused_ssim_cuda.fusedssim_backward Reconstruct/submodules/fused-ssim/ssim.cu:480-517 (ext.cpp:6)
 * img1,img2,[maps] are [B,CH,H,W].  ssim_map and ssim_sum may each be NULL (not both); ssim_sum (1 float,
 * caller-zeroed) receives the sum of the map (the mean the Python wrapper returns, __init__.py:41-42).
 * Backward: if dL_dmap is NULL every map element's upstream gradient is (dL_scalar ? *dL_scalar : 1)*dL_scale. */
int adb_ssim_forward(int B, int CH, int H, int W, float C1, float C2, const float* img1, const float* img2,
                     int train, float* ssim_map, float* dm_dmu1, float* dm_dsigma1_sq, float* dm_dsigma12,
                     float* ssim_sum, adb_stream_t stream);
int adb_ssim_backward(int B, int CH, int H, int W, float C1, float C2, const float* img1, const float* img2,
                      const float* dL_dmap, const float* dL_scalar, float dL_scale, const float* dm_dmu1,
                      const float* dm_dsigma1_sq, const float* dm_dsigma12, float* dL_dimg1, adb_stream_t stream);

/* ---- Gaussian-splat rasterizer (one camera per call) ----
 * replaces the stages of gsplat.rendering.rasterization as called at
 * Reconstruct/scene/scene_models/h3dgsv3.py:664-680 (gsplat itself is an un-vendored pip dependency).
 * Layouts: see artdeco_b200/csrc/raster_common.cuh.  viewmat[16], K[9], campos[3] are DEVICE pointers. */
int adb_raster_project_fwd(int N, const float* means, const float* quats, const float* scales,
                           const float* opacities, const float* sh /*[N,16,3] or NULL*/, int sh_degree,
                           const float* viewmat, const float* K, const float* campos, int W, int H, float eps2d,
                           float near_plane, float far_plane, float radius_clip, int32_t* radii /*[N,2]*/,
                           float* splats /*[N,12]*/, int32_t* tiles_per_gauss /*[N]*/, adb_stream_t stream);
/* adb_raster_project_fwd + the first stage of the tile-bucketed intersection fused in (one RED per (Gaussian, touched tile) into
 * tile_counts, see adb_raster_tile_count_scan); follow it with adb_raster_tile_scan instead of adb_raster_tile_count_scan. */
int adb_raster_project_fwd_counts(int N, const float* means, const float* quats, const float* scales,
                                  const float* opacities, const float* sh, int sh_degree, const float* viewmat,
                                  const float* K, const float* campos, int W, int H, float eps2d, float near_plane,
                                  float far_plane, float radius_clip, int32_t* radii, float* splats,
                                  int32_t* tiles_per_gauss, int32_t* tile_counts, adb_stream_t stream);
/* C views of the same Gaussians in one pass: viewmats [C,16], Ks [C,9], camposs [C,3] (device); radii [C,N,2], splats [C,N,12],
 * tiles_per_gauss [C,N], tile_counts [C,2*4*T] (first half of every block zero on entry).  Per view bit-identical to
 * adb_raster_project_fwd_counts; the parameters (and the SH coefficients) are read once. */
int adb_raster_project_fwd_multi(int N, int C, const float* means, const float* quats, const float* scales,
                                 const float* opacities, const float* sh, int sh_degree, const float* viewmats,
                                 const float* Ks, const float* camposs, int W, int H, float eps2d, float near_plane,
                                 float far_plane, float radius_clip, int32_t* radii, float* splats,
                                 int32_t* tiles_per_gauss, int32_t* tile_counts, adb_stream_t stream);
int adb_raster_scan_workspace_bytes(int N, size_t* bytes /*HOST*/);
int adb_raster_isect_scan(int N, const int32_t* tiles_per_gauss, int64_t* cum_tiles /*[N] inclusive*/, void* ws,
                          size_t ws_bytes, adb_stream_t stream);
int adb_raster_isect_emit(int N, const int32_t* radii, const float* splats, const int64_t* cum_tiles, int W, int H,
                          int cam_id, int n_cams, int64_t* keys, int32_t* vals, adb_stream_t stream);
int adb_raster_sort_workspace_bytes(long long n_isect, size_t* bytes /*HOST*/);
int adb_raster_sort(long long n_isect, int W, int H, int n_cams, int64_t* keys_a, int32_t* vals_a, int64_t* keys_b,
                    int32_t* vals_b, void* ws, size_t ws_bytes, int* sorted_in_b /*HOST*/, adb_stream_t stream);
int adb_raster_tile_offsets(long long n_isect, const int64_t* keys_sorted, int W, int H,
                            int32_t* tile_offsets /*[T+1]*/, adb_stream_t stream);
/* Multi-view backward (BASELINE config 4: C views of the same Gaussians per optimiser step; csrc/raster_project_bwd_multi.cu).
 * Same mathematics as C calls of adb_raster_project_bwd summed (gsplat's fully_fused_projection_bwd + spherical_harmonics_bwd
 * under autograd's accumulation, h3dgsv3.py:664-680), with parameters read once and every gradient written once.
 *   adb_raster_project_bwd_multi  radii [C,N,2], splats / v_splats [C,N,12], viewmats [C,16], Ks [C,9] (device).  v_means,
 *       v_quats, v_scales, v_opac are OVERWRITTEN with the sum over cameras (geometry part only); g_rgb [C,N,3] = colour gradient
 *       masked by the SH clamp and visibility (may be NULL); v_viewmats [C,16] ACCUMULATED.
 *   adb_raster_sh_bwd_multi  v_sh [N,48] OVERWRITTEN with sum_c basis(dir_c) (x) g_rgb[c]; v_means += (or =) direction term;
 *       v_campos [C,3] accumulated (may be NULL).  g_rgb / campos may include views rendered on other GPUs. */
int adb_raster_project_bwd_multi(int N, int C, const float* means, const float* quats, const float* scales,
                                 const float* viewmats, const float* Ks, int W, int H, const int32_t* radii,
                                 const float* splats, const float* v_splats, float* v_means, float* v_quats, float* v_scales,
                                 float* v_opac, float* g_rgb, float* v_viewmats, adb_stream_t stream);
int adb_raster_sh_bwd_multi(int N, int C, const float* means, const float* sh, int sh_degree, const float* campos,
                            const float* g_rgb, float* v_sh, float* v_means, int accumulate /* bit0: v_means +=, bit1: v_sh += */,
                            int skip_mod, int skip_val /* skip views c % skip_mod == skip_val when skip_mod > 0 */,
                            float* v_campos, adb_stream_t stream);
/* Split form of adb_raster_sh_bwd_multi for the multi-GPU step: adb_raster_sh_dir_bwd_multi ADDS the direction term of the C
 * LOCAL views to v_means [N,3] (v_campos [C,3] accumulated, may be NULL), taking each view's colour gradient from the blend
 * backward's accumulators with the SH clamp mask (splats[c][i].rgb > 0 ? v_splats[c][i][6:9] : 0; splats / v_splats [C,N,12]) —
 * linear in the views, so the geometry all-reduce sums it over ranks; adb_raster_sh_expand_multi OVERWRITES v_sh [N,48] with
 * sum_c basis(dir_c) (x) g_rgb[c] over all C views of the batch (g_rgb [C,N,3], campos [C,3]: any rank's views). */
int adb_raster_sh_dir_bwd_multi(int N, int C, const float* means, const float* sh, int sh_degree, const float* campos,
                                const float* splats, const float* v_splats, float* v_means, float* v_campos, adb_stream_t stream);
int adb_raster_sh_expand_multi(int N, int C, const float* means, int sh_degree, const float* campos, const float* g_rgb,
                               float* v_sh, adb_stream_t stream);
/* Tile-bucketed intersection (no library sort, no host sync; bit-identical to adb_raster_isect_emit + adb_raster_sort +
 * adb_raster_tile_offsets, i.e. to gsplat's isect_tiles / radix sort / isect_offset_encode behind h3dgsv3.py:664-680):
 *   adb_raster_tile_count_scan   per-tile counts (RED.ADD) + one-CTA exclusive scan -> tile_offsets[T+1] clamped to
 *                                `capacity`; *total (int64, device) = true intersection count, *overflow (int32, device)
 *                                is SET when total > capacity.  tile_counts: int32[2*4*T] (4 replicated counters per tile,
 *                                then their segment starts); the first half must be zero on entry.
 *   adb_raster_tile_scatter_sort scatter depth_bits<<32|gaussian into each tile's segment (counters return to zero), then
 *                                one CTA per tile sorts its segment (bitonic, shared memory; global memory beyond 4096
 *                                entries) and writes keys = cam|tile|depth_bits, vals = cam*N + gaussian.
 * packed: uint64[capacity] scratch.  legacy != 0 selects the Inria tile rectangle. */
int adb_raster_tile_count_scan(int N, const int32_t* radii, const float* splats, const int32_t* tiles_per_gauss, int W, int H,
                               int legacy, long long capacity, int32_t* tile_counts, int32_t* tile_offsets, long long* total,
                               int32_t* overflow, adb_stream_t stream);
int adb_raster_tile_scan(int W, int H, long long capacity, int32_t* tile_counts, int32_t* tile_offsets, long long* total,
                         int32_t* overflow, adb_stream_t stream);
int adb_raster_tile_scatter_sort(int N, const int32_t* radii, const float* splats, const int32_t* tiles_per_gauss, int W, int H,
                                 int legacy, int cam_id, int n_cams, long long capacity, int32_t* tile_counts,
                                 const int32_t* tile_offsets, void* packed, int64_t* keys, int32_t* vals, adb_stream_t stream);
/* View-batched intersection (one launch per stage for C views; 1 <= C <= 64).  capacities: HOST array [C]; view c owns the
 * segment [sum_{c'<c} capacities[c'], +capacities[c]) of one packed / keys / vals buffer (the sum must stay below 2^31 - 1).
 *   adb_raster_tile_scan_multi         one CTA per view: tile_offsets [C,T+1] ABSOLUTE in that buffer, clamped to the view's
 *                                      capacity; total int64 [C] and overflow int32 [C] (SET when total[c] > capacities[c])
 *                                      on the device.  tile_offsets == NULL: totals only (a sizing pass).
 *   adb_raster_tile_scatter_sort_multi scatter (view grid dimension) + per-tile sort over (T, C) CTAs; vals = c*N + gaussian;
 *                                      keys (may be NULL: not written) = c|tile|depth_bits as adb_raster_tile_scatter_sort. */
int adb_raster_tile_scan_multi(int C, int W, int H, const long long* capacities /*HOST [C]*/, int32_t* tile_counts,
                               int32_t* tile_offsets, long long* total, int32_t* overflow, adb_stream_t stream);
int adb_raster_tile_scatter_sort_multi(int N, int C, const int32_t* radii, const float* splats, const int32_t* tiles_per_gauss,
                                       int W, int H, const long long* capacities /*HOST [C]*/, int32_t* tile_counts,
                                       const int32_t* tile_offsets, void* packed, int64_t* keys, int32_t* vals,
                                       adb_stream_t stream);
int adb_raster_blend_fwd(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                         const int32_t* tile_offsets, float* colors /*[H,W,4]*/, float* alphas /*[H,W]*/,
                         int32_t* last_ids /*[H,W]*/, adb_stream_t stream);
int adb_raster_blend_bwd(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                         const int32_t* tile_offsets, const float* alphas, const int32_t* last_ids,
                         const float* v_colors, const float* v_alphas, float* v_splats /*[N,12] zeroed, +=*/,
                         adb_stream_t stream);
/* The same pair sharing the culling decisions: adb_raster_blend_fwd_hits also fills hit_mask — one byte per sorted intersection
 * (index as in vals_sorted): bit w = the splat can reach the 8x4 pixel block of warp w of its tile (entries behind the point
 * where a whole tile saturated are left unwritten) — and adb_raster_blend_bwd_hits builds its per-warp hit lists from it
 * instead of repeating the box and ellipse tests (same splats / vals_sorted / tile_offsets; identical gradients). */
int adb_raster_blend_fwd_hits(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                              const int32_t* tile_offsets, float* colors, float* alphas, int32_t* last_ids,
                              unsigned char* hit_mask, adb_stream_t stream);
int adb_raster_blend_bwd_hits(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                              const int32_t* tile_offsets, const float* alphas, const int32_t* last_ids, const float* v_colors,
                              const float* v_alphas, float* v_splats, const unsigned char* hit_mask, adb_stream_t stream);
/* View-batched blend pair (gridDim.z = C): splats [C,N,12] and v_splats [C,N,12] indexed by vals_sorted (c*N + gaussian)
 * directly, tile_offsets [C,T+1] from adb_raster_tile_scan_multi, colors / v_colors [C,H,W,4], alphas / last_ids / v_alphas
 * [C,H,W]; hit_mask (may be NULL) indexed like vals_sorted.  Per view the same images as the single-view _hits pair; last_ids
 * are absolute sorted indices.  N = 0 (empty scene): the forward writes empty images (splats may be NULL), the backward
 * returns without a launch. */
int adb_raster_blend_fwd_multi(int N, int C, int W, int H, const float* splats, const int32_t* vals_sorted,
                               const int32_t* tile_offsets, float* colors, float* alphas, int32_t* last_ids,
                               unsigned char* hit_mask, adb_stream_t stream);
int adb_raster_blend_bwd_multi(int N, int C, int W, int H, const float* splats, const int32_t* vals_sorted,
                               const int32_t* tile_offsets, const float* alphas, const int32_t* last_ids, const float* v_colors,
                               const float* v_alphas, float* v_splats, const unsigned char* hit_mask, adb_stream_t stream);
int adb_raster_project_bwd(int N, const float* means, const float* quats, const float* scales, const float* sh,
                           int sh_degree, const float* viewmat, const float* K, const float* campos, int W, int H,
                           float eps2d, float near_plane, float far_plane, float radius_clip, const int32_t* radii,
                           const float* splats, const float* v_splats, float* v_means, float* v_quats,
                           float* v_scales, float* v_opac, float* v_sh, float* v_viewmat /*[16] +=*/,
                           float* v_campos /*[3] +=*/, adb_stream_t stream);

/* ---- legacy (Inria / diff_gaussian_rasterization) conventions: GaussianRasterizer / rasterize_gaussians as called at
 * Reconstruct/webviewer/scene_models.py:559-605 (SURVEY.md §8a R3; the fork itself is not vendored, so the constants are
 * the published Inria ones: radius ceil(3 sqrt(lambda_max)), +0.3 px^2 low-pass (pass eps2d = 0.3), near 0.2, alpha <= 0.99,
 * stop at T(1-alpha) < 1e-4, tile rectangle (int)((p-r)/16)..(int)((p+r+15)/16) on pixel-index coordinates).
 * Same buffers and key layout as the gsplat-convention entry points above; scan / sort / tile_offsets / project_bwd are shared. */
int adb_raster_project_fwd_legacy(int N, const float* means, const float* quats, const float* scales,
                                  const float* opacities, const float* sh, int sh_degree, const float* viewmat,
                                  const float* K, const float* campos, int W, int H, float eps2d, float near_plane,
                                  float far_plane, int32_t* radii /*[N,2], both = Inria radius*/, float* splats,
                                  int32_t* tiles_per_gauss, adb_stream_t stream);
int adb_raster_isect_emit_legacy(int N, const int32_t* radii, const float* splats, const int64_t* cum_tiles, int W, int H,
                                 int cam_id, int n_cams, int64_t* keys, int32_t* vals, adb_stream_t stream);
int adb_raster_blend_fwd_legacy(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                                const int32_t* tile_offsets, float* colors /*[H,W,4]: rgb, sum alpha*T/z*/, float* alphas,
                                int32_t* last_ids, int32_t* main_ids /*[H,W] argmax alpha*T, -1 none; may be NULL*/,
                                adb_stream_t stream);
int adb_raster_blend_bwd_legacy(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                                const int32_t* tile_offsets, const float* alphas, const int32_t* last_ids,
                                const float* v_colors, const float* v_alphas, float* v_splats /*slot 9 = dL/d(1/z)*/,
                                adb_stream_t stream);

/* ---- dense matching after a MASt3R pair (SURVEY.md §8f rank 1): mast3r_slam_backends.iter_proj / refine_matches
 * (VSLAM/backend/src/matching_kernels.cu:26-116,119-316; bindings VSLAM/backend/src/gn.cpp:84-112) and the PyTorch glue of
 * VSLAM/utils_matching.py:59-190.  All tensors contiguous, device pointers.
 * adb_match_prep     X11,X21 [B,H,W,3] fp32; idx_init int64 [B,HW] or NULL (identity) -> rays_with_grad [B,H,W,9]
 *                    (unit ray, d/du, d/dv with the [-3,-10,-3]/32 kernels, reflect padding), pts3d_norm [B,HW,3],
 *                    p_init [B,HW,2] (u,v) fp32                                   (utils_matching.py:59-97,120-145)
 * adb_iter_proj      per-point LM on the bilinear ray image -> p_new [B,n,2] fp32, converged u8 [B,n]  (kernels.cu:119-276)
 * adb_match_finalize p1 = trunc(p) int64 [B,HW,2]; valid = converged && ||X11[p1]-X21|| < dist_thresh (utils_matching.py:166-174)
 * adb_refine_matches D11 fp16 [B,H,W,F], D21 fp16 [B,n,F], p1 int64 [B,n,2] -> p1_new int64 [B,n,2] and (optional) the
 *                    linear index u + W v [B,n]; F in {16,24,32}; fp16 score arithmetic as the reference's (kernels.cu:26-83) */
int adb_match_prep(int B, int H, int W, const float* X11, const float* X21, const long long* idx_init,
                   float* rays_with_grad, float* pts3d_norm, float* p_init, adb_stream_t stream);
int adb_iter_proj(int B, int H, int W, int n_pts, const float* rays_with_grad, const float* pts3d_norm,
                  const float* p_init, int max_iter, float lambda_init, float cost_thresh, float* p_new,
                  unsigned char* converged, adb_stream_t stream);
int adb_match_finalize(int B, int H, int W, const float* X11, const float* X21, const float* p,
                       const unsigned char* converged, float dist_thresh, long long* p1, unsigned char* valid,
                       adb_stream_t stream);
int adb_refine_matches(int B, int H, int W, int fdim, int n_pts, const void* D11_f16, const void* D21_f16,
                       int planar /*0: row-major [.,F] as the reference passes them; 1: adb_desc_pack_f16 layout*/,
                       const long long* p1, int radius, int dilation_max, long long* p1_new, long long* lin_idx,
                       adb_stream_t stream);
/* fp32 [B,n_pix,F] -> fp16 (round to nearest even, == Tensor.half()) chunk-planar [B][F/8][n_pix][8]: the layout in which a
 * warp's 128-bit descriptor gathers coalesce (utils_matching.py:178-184 converts with .half() and keeps [.,F] rows). */
int adb_desc_pack_f16(int B, long long n_pix, int fdim, const float* src, void* dst_f16, adb_stream_t stream);

/* ---- optimizer bookkeeping (Reconstruct/scene/optimizers.py) ----
 * adb_adam_update_decay  SparseGaussianAdam.step's update + its per-primitive learning-rate schedule in one pass
 *                        (optimizers.py:116-133,144-161): lr [N,M] is used, then overwritten with max(lr*decay, lr_min) on
 *                        visible rows.
 * adb_compact_*          SparseGaussianAdam.add_and_prune (optimizers.py:163-219; SURVEY.md R6): out = cat(t[mask], ext) for
 *                        every state tensor with one index plan and one gather launch (rows moved as 32-bit words). */
int adb_adam_update_decay(long long N, long long M, float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                          const unsigned char* visible, float* lr /*[N,M] in/out*/, float b1, float b2, float eps,
                          float lr_decay, float lr_min, adb_stream_t stream);
int adb_compact_workspace_bytes(long long N, size_t* bytes);
int adb_compact_plan(long long N, const unsigned char* mask, int32_t* src_of /*[N]*/, int32_t* n_keep_dev /*[1]*/, void* ws,
                     size_t ws_bytes, adb_stream_t stream);
int adb_compact_gather(long long n_keep, long long n_ext, const int32_t* src_of, int n_tensors,
                       const void* const* srcs /*HOST array of device pointers*/, void* const* dsts, const void* const* exts,
                       const int* row_words, const unsigned* fill_words, adb_stream_t stream);

/* ---- covariance-modulation MLP (SceneModel.render, Reconstruct/scene/scene_models/h3dgsv3.py:656-662; mlp_cov :173-177) ----
 * x = cat(global_feat[cls_id], local_feat); o = W2 relu(W1 x + b1) + b2; scale_out = scaling*sigmoid(o[:3]);
 * rot_out = normalize(rotation*o[3:]).  D = Fg+Fl in {32,64}.  Backward ACCUMULATES v_global_feat, v_W1, v_b1, v_W2, v_b2. */
int adb_cov_mlp_forward(long long N, int Fg, int Fl, const float* global_feat, const float* local_feat,
                        const long long* cls_id, const float* W1, const float* b1, const float* W2, const float* b2,
                        const float* scaling, const float* rotation, float* scale_out, float* rot_out, adb_stream_t stream);
int adb_cov_mlp_backward(long long N, int Fg, int Fl, const float* global_feat, const float* local_feat,
                         const long long* cls_id, const float* W1, const float* b1, const float* W2, const float* b2,
                         const float* scaling, const float* rotation, const float* v_scale_out, const float* v_rot_out,
                         float* v_scaling, float* v_rotation, float* v_local_feat, float* v_global_feat, float* v_W1,
                         float* v_b1, float* v_W2, float* v_b2, adb_stream_t stream);

/* ---- sparse Adam (in place, no bias correction) ----
 * replaces diff_gaussian_rasterization.adamUpdate / adamUpdateBasic (on-the-fly-nvs fork, un-vendored); call sites
 * Reconstruct/scene/optimizers.py:48-57 (Basic), 90-99, 116-128, 144-156.  visible: uint8/bool [N] or NULL;
 * lr_dev: NULL (use lr_scalar) or a device tensor of numel 1, N or N*M. */
int adb_adam_update(long long N, long long M, float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                    const unsigned char* visible, const float* lr_dev, long long lr_numel, float lr_scalar, float b1,
                    float b2, float eps, adb_stream_t stream);

/* ---- LoD d_max cull: mask + fade ratio + compacted ascending ids ----
 * replaces the torch block at Reconstruct/scene/scene_models/h3dgsv3.py:626-645 (and the scan at :942-953).
 * count is a DEVICE int32; ids has capacity N; ratio may be NULL. */
int adb_lod_select_workspace_bytes(long long N, size_t* bytes /*HOST*/);
int adb_lod_select(long long N, const float* xyz, const float* d_max, const float* cam /*[3]*/, unsigned char* mask,
                   float* ratio, int32_t* ids, int32_t* count, void* ws, size_t ws_bytes, adb_stream_t stream);
/* Global Gauss-Newton over Sim(3) key-frame poses: mast3r_slam_backends.gauss_newton_rays / gauss_newton_calib
 * (VSLAM/backend/src/gn.cpp:32-82, gn_kernels.cu:813-1637; callers VSLAM/mast3r_slam/global_opt.py:158,208).
 * mode 0 = rays (sigma_a = sigma_ray, sigma_b = sigma_dist), mode 1 = calib (sigma_a = sigma_pixel, sigma_b = sigma_depth; K3x3 =
 * device pointer to the row-major intrinsics).  poses [K,8] (t, q xyzw, s) updated IN PLACE, pose 0 fixed; Xs [K,n,3]; Cs [K,n];
 * ii / jj int64 [E] = positions of the edge's key frames in the pose table; idx_ii2jj int64 [E,n]; valid_match bool [E,n];
 * Q [E,n].  dx_out [K-1,7] = last step; state_out int32[4] on the device = {iterations run, converged, |dx| (float bits),
 * last Cholesky ok}.  The whole solve (normal equations, dense double Cholesky, retraction, termination test) runs on the
 * device: no host sync.  ws from adb_gn_workspace_bytes. */
int adb_gn_workspace_bytes(int n_poses, int n_edges, size_t* bytes /*HOST*/);
int adb_gauss_newton(int mode, int n_poses, int n_pts, int n_edges, float* poses, const float* Xs, const float* Cs,
                     const float* K3x3, const long long* ii, const long long* jj, const long long* idx_ii2jj,
                     const unsigned char* valid_match, const float* Q, int height, int width, int pixel_border, float z_eps,
                     float sigma_a, float sigma_b, float C_thresh, float Q_thresh, int max_iter, float delta_thresh,
                     float* dx_out, int* state_out, void* ws, size_t ws_bytes, adb_stream_t stream);
/* Frame tracking: CameraTracker.track after matching (VSLAM/CameraTracker.py:53-155), calibrated Sim(3) only
 * (optimize_focal is not supported).  N = height * width points in KEY-FRAME pixel order; poses [8] = (t, q xyzw, s).
 * Three calls on one stream share `ws` and the device `state` block; none synchronises the host:
 *   adb_track_prepare  steps 2-5: Qk, the validity masks, constrain_points_to_ray, the 5x5 box-filter covariance and
 *                      meas_k (get_points_poses, :189-219; utils_uncertainty.py:5-50), the match-fraction test (:83-118).
 *   adb_track_solve    opt_pose_calib_sim3 (:296-396): Gauss-Newton with the covariance filter, convergence test
 *                      (nonlinear_optimizer.py:5-25) and T_WCf = quat2unit(T_WCk T_CkCf) (:134).
 *   adb_track_finish   step 6-7: point fusion into the key frame (:136-141, ImageFrame.py:30-48), check_keyframe and
 *                      check_keyframe_map (:144-186). */
enum { ADB_TRACK_OK = 0, ADB_TRACK_LOST_MATCHES = 1, ADB_TRACK_LOST_CHOLESKY = 2, ADB_TRACK_LOST_ZERO_COST = 3 };
typedef struct adb_track_state {
    int32_t lost;            /* ADB_TRACK_*: insufficient matches, non-positive pivot, zero previous cost */
    int32_t iters;           /* Gauss-Newton iterations run */
    int32_t converged;       /* check_convergence stopped the loop */
    int32_t done;            /* the loop has stopped (converged or lost): remaining iterations are no-ops */
    int32_t n_valid_opt, n_valid_kf, n_unique;   /* valid_opt.sum(), valid_kf.sum(), |unique(idx_f2k[valid_match_k])| */
    int32_t is_keyframe, is_keyframe_map;
    float tau_norm;          /* |tau| of the last iteration */
    float cov_threshold;     /* max(quantile(det, 0.9), 1) of the last iteration (covariance filter) */
    float dist_quantile;     /* quantile(|uv_f - uv_k| over valid_opt, thres_keyframe) */
    double cost;             /* 0.5 b^T b of the last iteration (at the pose before its update) */
    double prev_cost;        /* cost of the iteration before */
    double last_dist;        /* last_dist after the key-frame tests */
    double H[49], g[7];      /* normal equations of the last iteration: H = A^T A, g = -A^T b */
    float T_CkCf[8];         /* current relative pose */
    float T_WCk[8];          /* quat2unit(T_WCk) */
} adb_track_state;
/* ws_bytes (HOST) for N points; state_bytes (HOST) = sizeof(adb_track_state). */
int adb_track_workspace_bytes(int n_pts, size_t* ws_bytes /*HOST*/, size_t* state_bytes /*HOST*/);
/* idx_f2k int64 [N] (values in [0, N)), valid_match_k bool [N]; Xff [N,3], Cff [N], Qff [N] in frame order; Qkf [N];
 * kf_X [N,3], kf_C [N], kf_N int32 [1] = the key frame's X_canon, C, N; K3x3 row-major.  Writes Xf, Xf_cov (the diagonal,
 * [N,3]), Qk, meas_k [N,3], valid_meas_k / valid_opt / valid_kf (bool [N]) in key-frame order, and resets `state`
 * (lost = ADB_TRACK_LOST_MATCHES when valid_opt.sum() / N < min_match_frac).  height, width >= 3 (reflect padding). */
int adb_track_prepare(int height, int width, const float* K3x3, const long long* idx_f2k, const unsigned char* valid_match_k,
                      const float* Xff, const float* Cff, const float* Qff, const float* Qkf, const float* kf_X,
                      const float* kf_C, const int32_t* kf_N, float C_conf, float Q_conf, float depth_eps, float min_match_frac,
                      float* Xf, float* Xf_cov, float* Qk, float* meas_k, unsigned char* valid_meas_k, unsigned char* valid_opt,
                      unsigned char* valid_kf, adb_track_state* state, void* ws, size_t ws_bytes, adb_stream_t stream);
/* Inputs as get_points_poses returns them (Xf_cov = diagonal [N,3]); T_WCf / T_WCk as stored (quat2unit is applied here).
 * `state` must come from adb_track_prepare or be zeroed.  A fixed sequence of max_iters iterations, each a no-op once
 * state->done is set.  On success T_WCf_out = quat2unit(T_WCk T_CkCf) and T_CkCf_out = the solution; on a lost outcome
 * T_WCf_out is not written and T_CkCf_out holds the starting pose quat2unit(T_WCk)^-1 quat2unit(T_WCf). */
int adb_track_solve(int n_pts, int height, int width, const float* K3x3, const float* Xf, const float* Xf_cov, const float* Qk,
                    const unsigned char* valid, const float* meas_k, const unsigned char* valid_meas_k, const float* T_WCf,
                    const float* T_WCk, int max_iters, int covariance_filter, int pixel_border, float depth_eps,
                    float sigma_pixel, float sigma_depth, float huber_k, double rel_error, float delta_norm, float* T_WCf_out,
                    float* T_CkCf_out, adb_track_state* state, void* ws, size_t ws_bytes, adb_stream_t stream);
/* After adb_track_solve on the same state.  Unless lost: point fusion when point_fusion != 0 (kf_X, kf_C, kf_N updated in
 * place with Xkf [N,3] and Ckf [N] through state->T_CkCf), then the key-frame tests; last_dist is the caller's value. */
int adb_track_finish(int height, int width, const long long* idx_f2k, const unsigned char* valid_opt, const float* Xkf,
                     const float* Ckf, float* kf_X, float* kf_C, int32_t* kf_N, int point_fusion, double match_frac_thresh,
                     float thres_keyframe, double min_displacement, double last_dist, adb_track_state* state, void* ws,
                     size_t ws_bytes, adb_stream_t stream);
/* update_voxel (Reconstruct/scene/scene_models/h3dgsv3.py:227-316): voxel-hash class ids without the reference's three sorts
 * (csrc/voxel.cu).  Tables are caller-allocated: vkeys[V], pkeys[P], ukeys[U] uint64 pre-filled with 0xFF bytes; pcount[P]
 * int32 and best[V] uint64 zeroed; V, P powers of two >= 2N, U >= 2M.  mn = device float[3] minimum over all points.
 *   adb_voxel_vote       original points -> cls_out[N] = majority class of each point's voxel (ties: smallest id)
 *   adb_voxel_match_new  new points: voxel's class, or their voxel key collected into ulist (count in *ucount, device)
 *   adb_voxel_rank_new   `sorted` = the distinct unmatched keys ascending (caller sorts) -> cls_out = base + rank */
int adb_voxel_vote(long long N, const float* xyz, const long long* cls, const float* mn, float voxel_size, void* vkeys,
                   long long V, void* pkeys, int* pcount, long long P, void* best, unsigned* slot_of, long long* cls_out,
                   int* overflow, adb_stream_t stream);
int adb_voxel_match_new(long long M, const float* new_xyz, const float* mn, float voxel_size, const void* vkeys, long long V,
                        const void* best, int have_orig, void* ukeys, long long U, int* uslot_of, long long* cls_out,
                        void* ulist, int* ucount, int* overflow, adb_stream_t stream);
int adb_voxel_rank_new(long long M, int n, const void* sorted, const void* ukeys, long long U, int* urank,
                       const int* uslot_of, long long base, long long* cls_out, adb_stream_t stream);
/* weed_out_gaussians (Reconstruct/scene/scene_models/h3dgsv3.py:942-953) for ALL key frames in one pass: cams [K,3] camera
 * centres (device); keep[i] = (#{k : |xyz_i - cam_k| < 2 d_max_i} / K > visible_threshold); visible_count [N] may be NULL. */
/* Key-frame densification: the sampler of SceneModel.add_new_gaussians (Reconstruct/scene/scene_models/h3dgsv3.py:766-940,
 * csrc/densify.cu).  One workspace (adb_densify_workspace_bytes for the LoD-1 image, height x width) serves every call.
 *   adb_densify_depth_quantile  out[0] = torch.quantile(values[n], q) (linear, NaN if any value is NaN),
 *                               out[1] = fp32(min(0.01, out[0])) as Python's min evaluates it (a NaN quantile gives 0.01)
 *   adb_densify_sample          one LoD (1, 2, 4 or 8) of an image of height x width: init_proba [h,w] (get_lapla_norm of the
 *                               resized image, x init_proba_scaler), penalty [h,w] (the same of the exposed render; may be NULL;
 *                               0 without a render), flags [h,w] (bit 0 sampled, bit 1 valid) and *n_rows (device) = pixels
 *                               with both bits.  image [3,H,W]; render [3,H,W] raw RGB with element strides render_strides[3]
 *                               (HOST: channel, row, column) or NULL; exposure [3,4]; depth, conf [Hs,Ws]; uniforms [h,w];
 *                               qmin [1] (out[1] above).  h = height / lod, w = width / lod, both >= 2.
 *   adb_densify_emit            after adb_densify_sample on the same workspace: the *n_rows rows in row-major pixel order.
 *                               cam [15] = R [3,3] row-major, t [3], approx_centre [3]; f the focal length in pixels.
 *                               xyz [n,3], f_dc [n,3], scaling [n,3], opacity [n], d_max [n].
 *   adb_densify_prune_mask      mask[i] = sigmoid(opacity[i]) > 0.05 && f max(exp(scaling[i])) / |xyz[i] - approx_centre| < 0.5 width */
int adb_densify_workspace_bytes(int height, int width, size_t* bytes /*HOST*/);
int adb_densify_depth_quantile(long long n, const float* values, float q, float* out /*[2]*/, void* ws, size_t ws_bytes,
                               adb_stream_t stream);
int adb_densify_sample(int height, int width, int lod, const float* image, const float* render,
                       const long long* render_strides /*HOST [3]*/, const float* exposure, int Hs, int Ws, const float* depth,
                       const float* conf, const float* uniforms, const float* qmin, float init_proba_scaler, float gs_add_ratio,
                       float* init_proba, float* penalty, unsigned char* flags, int32_t* n_rows, void* ws, size_t ws_bytes,
                       adb_stream_t stream);
int adb_densify_emit(int height, int width, int lod, const float* image, int Hs, int Ws, const float* depth, const float* conf,
                     const float* init_proba, const unsigned char* flags, const float* cam, double f, float* xyz, float* f_dc,
                     float* scaling, float* opacity, float* d_max, void* ws, size_t ws_bytes, adb_stream_t stream);
int adb_densify_prune_mask(long long N, const float* xyz, const float* opacity, const float* scaling,
                           const float* approx_centre, double f, int width, unsigned char* mask, adb_stream_t stream);
int adb_lod_weed_out(long long N, const float* xyz, const float* d_max, int K, const float* cams, float visible_threshold,
                     int32_t* visible_count, unsigned char* keep, adb_stream_t stream);

/* ---- exact KNN on a grid hash ----
 * replaces SimpleKNN::knn (distCUDA2)        Reconstruct/submodules/simple-knn/simple_knn.cu:188-224, spatial.cu:16-26
 *          SimpleKNN::knn_index2 (distIndex2) simple_knn.cu:468-522, spatial.cu:29-41
 *          SimpleKNN::knn_indexQ (distIndexQ) simple_knn.cu:592-651, spatial.cu:44-58
 * points [P,3]; squared distances; rows sorted ascending; unfilled slots FLT_MAX / -1; K <= 32. */
int adb_knn_workspace_bytes(long long P, size_t* bytes /*HOST*/);
int adb_knn_mean3(long long P, const float* points, float* mean_dists /*[P]*/, void* ws, size_t ws_bytes,
                  adb_stream_t stream);
int adb_knn_index(long long P, const float* points, int K, long long Q, const int32_t* query_idx /*[Q] or NULL*/,
                  const unsigned char* candidate /*[P] or NULL*/, float* dists /*[Q*K]*/, int32_t* ids /*[Q*K]*/,
                  void* ws, size_t ws_bytes, adb_stream_t stream);

/* ---- MASt3R: tensor-core GEMM (wgmma + TMA) and its companions ----
 * adb_gemm_bf16 replaces every nn.Linear / q@k^T / attn@v of the reference model
 *   (VSLAM/thirdparty/mast3r/dust3r/croco/models/blocks.py:58-112,140-169; dust3r/dust3r/patch_embed.py:19-29;
 *    mast3r/catmlp_dpt_head.py:67-69): D[z] = act(alpha * A[z] * B[z]^T + bias) + residual[z],
 *   A bf16 [batch][M][K], B bf16 [batch][N][K], both K-contiguous; *_lo != NULL selects the 3-term bf16x3 product;
 *   outputs fp32 D and/or a bf16 (hi, lo) split; output offset = (z / zdiv) * s?2 + (z % zdiv) * s? (zdiv <= 0: z * s?).
 * adb_layernorm     nn.LayerNorm(eps) rows of C (croco.py:34, blocks.py:127-130,186-191)
 * adb_rope_heads    RoPE2D + head split (pos_embed.py:112-159 / curope/kernels.cu:18-82): x fp32 [B,N,ld] -> bf16 split
 *                   [B,h,N,64] (mode 0 RoPE, 1 plain) or transposed [B,h,64,Npad] (mode 2)
 * adb_softmax_rows  attn.softmax(-1) (blocks.py:106,163), fp32 in, bf16 split out
 * adb_im2col_patch16  operand of the 16x16/s16 patch-embedding conv as a GEMM (patch_embed.py:19-29)
 * adb_split_bf16    x -> (hi = rn(x), lo = rn(x - hi)) */
int adb_gemm_bf16(int batch, int M, int N, int K, const void* A_hi, const void* A_lo, long long lda, long long sA,
                  const void* B_hi, const void* B_lo, long long ldb, long long sB, float* D, long long ldd, long long sD,
                  void* D_hi, void* D_lo, long long ldo, long long sO, const float* bias, const float* residual,
                  long long ldr, long long sR, float alpha, int act /*0 none, 1 GELU(erf)*/, int zdiv, long long sD2,
                  long long sO2, long long sR2, adb_stream_t stream);
/* adb_conv3x3_bf16: 3x3 / stride 1 / pad 1 convolution as an implicit GEMM on the same kernel (4-D TMA boxes, no im2col):
 *   replaces the nn.Conv2d(k=3) calls of croco/models/dpt_block.py:20-77,93-112,368-372.  x NHWC bf16 split, w bf16 split
 *   [Cout][9*Cin_pad] tap-major with Cin padded to 64, x and w 16-byte aligned; outputs NHWC; act 0/2 (ReLU);
 *   split_relu: split stores relu(v).  Any W >= 1 works: the pixel tile's TMA box may be wider than the image. */
int adb_conv3x3_bf16(int B, int H, int W, int Cin, int Cout, const void* x_hi, const void* x_lo, const void* w_hi,
                     const void* w_lo, const float* bias, const float* residual, float* D, void* D_hi, void* D_lo, int act,
                     int split_relu, adb_stream_t stream);
/* adb_attention_bf16: fused softmax(scale * Q K^T) V with the score matrix held in registers; replaces the three
 *   materialised torch ops at croco/models/blocks.py:105-109 (self) and :162-166 (cross).  head_dim 64.
 *   Q [B*heads,Nq,64], K [B*heads,Nk,64], Vt [B*heads,64,Nkpad] bf16 splits, 16-byte aligned; O bf16 split
 *   [B,Nq,heads*64].  Keys >= Nk get weight exactly 0, so Vt's padding columns [Nk, Nkpad) need not be zero, only finite
 *   (0 * Inf would still be NaN).  O_lo may be given in single pass (no Q/K/Vt lo parts) too. */
int adb_attention_bf16(int B, int heads, int Nq, int Nk, int Nkpad, const void* Q_hi, const void* Q_lo, const void* K_hi,
                       const void* K_lo, const void* Vt_hi, const void* Vt_lo, float scale, void* O_hi, void* O_lo,
                       adb_stream_t stream);
/* Attention kernel choice: 0 = automatic by wave count (default), 1 = one 128-query tile per CTA, 2 = two query tiles per
 * persistent CTA sharing every K/V block.  Returns the previous setting (-1: bad argument).  Diagnostic / test switch. */
int adb_attention_set_variant(int variant);
int adb_layernorm(long long rows, int C, const float* x, const float* gamma, const float* beta, float eps, float* y,
                  void* y_hi, void* y_lo, adb_stream_t stream);
int adb_split_bf16(long long n, const float* x, void* hi, void* lo, adb_stream_t stream);
/* Linear layer fused with RoPE2D + head split (croco/models/blocks.py:94-103 self-attention qkv, :150-160 cross-attention
 * projq / projk): y = A W^T + bias, M = B*ntok rows; output columns [0, n_rope_dst*heads*64) are rotated per head with the
 * (cos, sin) table row of the token's (y,x) position and written as bf16 (hi, lo) head-major [B*heads, ntok, 64] to q (first
 * heads*64 columns) and k (next heads*64, n_rope_dst == 2); the remaining columns go to D_tail fp32 [M, ldd] (the V projection).
 * The [M, N] fp32 projection is never written.  table: float [n_pos][16][2] (cos, sin), 16-byte aligned. */
int adb_gemm_bf16_rope(int M, int N, int K, const void* A_hi, const void* A_lo, long long lda, const void* B_hi,
                       const void* B_lo, long long ldb, const float* bias, int ntok, int heads, int n_rope_dst,
                       const long long* pos /*[M,2] int64 (y,x)*/, const float* table, int n_pos, void* q_hi, void* q_lo,
                       void* k_hi, void* k_lo, float* D_tail, long long ldd, adb_stream_t stream);
/* curope.rope_2d(tokens[B,N,H,D] fp32 IN PLACE, positions[B,N,2] int64 (y,x), base, F0) — curope.cpp:49-68, kernels.cu:18-108.
 * tokens: stride(3) == 1 and stride(2) == D as the reference checks (kernels.cu:91); stride_b / stride_n in elements.
 * F0 = -1 applies the inverse rotation (the reference's backward, curope2d.py:25-29). */
int adb_rope2d_inplace(int B, int N, int H, int D, long long stride_b, long long stride_n, float* tokens,
                       const long long* positions, float base, float F0, adb_stream_t stream);
int adb_rope_heads(int B, int N, int h, long long ld, int col0, const float* x, const long long* pos /*[B,N,2] (y,x)*/,
                   const float* table /*[n_pos][16][2] (cos,sin)*/, int n_pos, int mode, int Npad, void* hi, void* lo,
                   adb_stream_t stream);
int adb_softmax_rows(long long rows, int L, long long ld_in, long long ld_out, const float* s, void* hi, void* lo,
                     adb_stream_t stream);
int adb_im2col_patch16(int B, int H, int W, const float* img, void* hi, void* lo, adb_stream_t stream);
/* DPT head companions.  adb_upsample2x_nhwc: F.interpolate(scale_factor=2, mode="bilinear", align_corners=True)
 * (croco/models/dpt_block.py:215-216,320) on NHWC fp32, fused with the FeatureFusionBlock skip add (out = up(x) + addend),
 * the crop of dpt_head.py:57 (Hout <= 2 Hin) and the bf16 split the next conv consumes; y / (hi, lo) may each be NULL.
 * adb_head_postprocess: pixel_shuffle(16) + concat + postprocess of mast3r/catmlp_dpt_head.py:25-39,87-96 and
 * dust3r/heads/postprocess.py:22-58 in one pass: pts [B,H,W,4] (DPT map) + lf [B*(H/16)*(W/16), ld_lf] (local-feature MLP
 * output before the pixel shuffle, 25*256 columns) -> pts3d [B,H,W,3], conf [B,H,W], desc [B,H,W,24], desc_conf [B,H,W]. */
int adb_upsample2x_nhwc(int B, int Hin, int Win, int C, int Hout, int Wout, const float* x, const float* addend, float* y,
                        void* hi, void* lo, adb_stream_t stream);
int adb_head_postprocess(int B, int H, int W, const float* pts, const float* lf, long long ld_lf, int n_desc, float* pts3d,
                         float* conf, float* desc, float* desc_conf, adb_stream_t stream);

/* Gradient exchange of the multi-view step over NVLink peer memory (csrc/peer_exchange.cu; BASELINE config 4 / SURVEY.md 8e; the
 * reference has no multi-GPU step — this replaces the dist.all_gather + dist.all_reduce pair of the NCCL exchange).  One process
 * per GPU: adb_peer_alloc gives a zeroed device region, adb_peer_export its 64-byte CUDA IPC handle (exchanged by the host),
 * adb_peer_import maps another rank's region with peer access.  `*_ptrs` are HOST arrays of `world` (<= 8) device pointers, entry
 * r = the region (plus an offset) of rank r, the caller's own included.  All remote traffic is stores.
 *   adb_peer_signal        fence.sys, then flags_r[slot][rank] = value on every rank r (flags: unsigned [n_slots][8] per rank)
 *   adb_peer_wait          spins until local flags[slot][r] >= value for r < world and slot in [slot_lo, slot_lo+n_slots); after
 *                          timeout_s seconds it sets *err (device int) = 1 + slot instead of hanging the GPU
 *   adb_peer_push_rgb      colour gradient of one view masked by the SH clamp (splats[i].rgb > 0 ? v_splats[i][6:9] : 0) written
 *                          as row `row_off` (floats, multiple of 4) of every rank's table; campos[3] -> cam_ptrs[r] + cam_off
 *   adb_peer_bcast         a ready-made row of n_floats (multiple of 4) to every rank
 *   adb_peer_scatter       reduce-scatter by push: float4 i of src goes to slot `rank` of rank (i / per4)'s staging area
 *   adb_peer_reduce_bcast  the owner sums its shard's `world` slots in rank order and writes the sums to every rank's result */
int adb_peer_warmup(void); /* loads the kernels below (lazy module loading must not happen while a wait kernel spins) */
int adb_peer_alloc(size_t bytes, void** ptr /*HOST out*/);
int adb_peer_free(void* ptr);
int adb_peer_export(void* ptr, unsigned char* handle64 /*HOST out*/);
int adb_peer_import(const unsigned char* handle64 /*HOST*/, void** ptr /*HOST out*/);
int adb_peer_close(void* ptr);
int adb_peer_signal(void* const* flag_ptrs /*HOST*/, int world, int slot, int rank, unsigned value, adb_stream_t stream);
int adb_peer_wait(const void* local_flags, int world, int slot_lo, int n_slots, unsigned value, double timeout_s, int* err,
                  adb_stream_t stream);
int adb_peer_push_rgb(int N, const float* splats, const float* v_splats, void* const* dst_ptrs /*HOST*/, int world, size_t row_off,
                      const float* campos, void* const* cam_ptrs /*HOST*/, size_t cam_off, adb_stream_t stream);
int adb_peer_bcast(size_t n_floats, const float* src, void* const* dst_ptrs /*HOST*/, int world, size_t off_floats,
                   const float* campos, void* const* cam_ptrs /*HOST*/, size_t cam_off, adb_stream_t stream);
int adb_peer_scatter(size_t n4, size_t per4, const float* src, void* const* stage_ptrs /*HOST*/, int world, int rank,
                     adb_stream_t stream);
int adb_peer_reduce_bcast(size_t n4, size_t per4, const float* stage, void* const* out_ptrs /*HOST*/, int world, int rank,
                          adb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif

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

/* ---- mapper training loss (csrc/mapper_loss.cu) ----
 * replaces the pixel loss block of SceneModel.optimization_step, Reconstruct/scene/scene_models/h3dgsv3.py:430-450, with
 * render_from_id's exposure (:611-614) and render's background composite and 1/D (:682-686), and their autograd backward.
 * One view of height h x width w.  colors [h,w,4] (RGB + accumulated depth D) and alphas [h,w] are the rasterizer's raw
 * channels-last outputs (colors and v_colors 16-byte aligned); gt [3,h,w]; mono_idepth [h,w]; exposure [3,4]; bg [3];
 * rdk [h,w] the radial weights (Reconstruct/utils.py:818-826).  Per pixel: c = rgb + (1 - alpha) bg,
 * e = clamp(E[:, :3] c + E[:, 3], 0, 1), inv = 1/D and, when is_important == 0, the mask
 * m = !(rdk|e0-g0| > 0.2 | rdk|e1-g1| > 0.2 | rdk|e1-g1| > 0.2) (as the reference writes it) multiplying e, gt, inv, mono.
 * One workspace (adb_mapper_loss_workspace_bytes) serves a forward and its backward; the forward's partials stay in it
 * until adb_mapper_loss_reduce.
 *   adb_mapper_loss_forward   image [3,h,w] = m e and gt_masked [3,h,w] = m gt (the SSIM operands), invdepth [h,w] = m inv
 *                             (may be NULL), and per-block partial sums of rdk|m e - m gt| and rdk|m inv - m mono|
 *   adb_mapper_loss_reduce    after adb_ssim_forward(image, gt_masked) wrote ssim_map [3,h,w]: terms [4] = loss, l1, mean
 *                             SSIM, depth term, with loss = lambda (1 - ssim) + (1 - lambda) l1 + depth_weight depth.
 *                             Partials are added in a fixed order: bitwise reproducible
 *   adb_mapper_loss_backward  dL [1] the upstream gradient of the loss (device); dssim [3,h,w] = adb_ssim_backward's
 *                             dL/dimage called with dL_scalar = dL and dL_scale = -lambda / (3hw).  Writes v_colors [h,w,4],
 *                             v_alphas [h,w] and v_exposure [3,4] (bg gets no gradient) */
int adb_mapper_loss_workspace_bytes(int height, int width, size_t* bytes /*HOST*/);
int adb_mapper_loss_forward(int height, int width, const float* colors, const float* alphas, const float* gt,
                            const float* mono_idepth, const float* exposure, const float* bg, const float* rdk,
                            int is_important, float* image, float* gt_masked, float* invdepth, void* ws, size_t ws_bytes,
                            adb_stream_t stream);
int adb_mapper_loss_reduce(int height, int width, const float* ssim_map, float lambda_dssim, float depth_weight,
                           float* terms /*[4]*/, void* ws, size_t ws_bytes, adb_stream_t stream);
int adb_mapper_loss_backward(int height, int width, const float* colors, const float* alphas, const float* gt,
                             const float* mono_idepth, const float* exposure, const float* bg, const float* rdk,
                             int is_important, const float* dssim, const float* dL, float lambda_dssim, float depth_weight,
                             float* v_colors, float* v_alphas, float* v_exposure, void* ws, size_t ws_bytes,
                             adb_stream_t stream);

/* ---- held-out key-frame evaluation (csrc/evaluate.cu) ----
 * replaces SceneModel.harmonize_test_exposure, Reconstruct/scene/scene_models/h3dgsv3.py:507-520, and the metric loop of
 * SceneModel.evaluate (:523-558) with psnr (Reconstruct/utils.py:86-87), fused_ssim(train=False) and
 * lpips.LPIPS(net="vgg") (:98; version 0.1, lpips=True, spatial=False, normalize=False).
 *   adb_eval_harmonize       exposure [K,3,4] IN PLACE, is_test [K] uint8: the reference loop in order (a test frame after a
 *                            test frame averages the updated one; idxm = 1 at index 0, idxp = K - 2 at the last index,
 *                            negative indices wrap as Python's do).  An index outside [-K, K) raises IndexError in the
 *                            reference: the loop stops there and *n_bad (device int) = 1, else 0
 * T views of h x w share one evaluation workspace (adb_eval_workspace_bytes; n_gaussians the length of the visibility mask):
 *   adb_eval_count_visible   view t's visibility_filter [n] (uint8) -> per-CTA counts (replaces .sum().item())
 *   adb_eval_image_metrics   colors [T,h,w,4] (16-byte aligned) / alphas [T,h,w] the rasterizer's raw outputs; view t uses
 *                            exposure row view_frame[t] (int32) of the [K,3,4] table.  image [T,3,h,w] = clamp(E[:, :3] rgb +
 *                            E[:, 3], 0, 1) (render_from_id with bg = 0); gt [T,3,h,w]; ssim_map [T,3,h,w] scratch.
 *                            Writes per-CTA partials of the squared error and of the SSIM map (adb_ssim_forward, B = T)
 *   adb_lpips_vgg_forward    frames [frame0, frame0 + n_frames) of img0 = image and img1 = gt, both [T,3,h,w] (h, w >= 16),
 *                            through VGG16 to relu5_3 as a batch of 2 n_frames.  w1 [64,3,3,3] / b1 [64] conv1_1 (fp32),
 *                            shift / scale [3] the ScalingLayer; w_hi / w_lo / bias: HOST arrays of the other 12 convs in
 *                            adb_conv3x3_bf16's weight layout; lin: HOST array of the 5 lin weights [C_l]; taps: NULL or a
 *                            HOST array of 5 device buffers that receive each tap's fp32 NHWC features [2 n_frames,H_l,W_l,C_l]
 *                            (NULL entries allowed).  lws: adb_lpips_workspace_bytes(n_frames, h, w)
 *   adb_eval_reduce          table [T, ADB_EVAL_N_METRICS] (double) per view: PSNR, SSIM, LPIPS (NaN when with_lpips == 0),
 *                            Render, GS, MSE, the five tap means.  PSNR / SSIM / LPIPS are the fp32 values the reference's
 *                            .item() reads; every partial is added in a fixed order in double: bitwise reproducible */
#define ADB_EVAL_N_METRICS 11
int adb_eval_workspace_bytes(int T, int height, int width, long long n_gaussians, size_t* bytes /*HOST*/);
int adb_eval_harmonize(int K, float* exposure, const uint8_t* is_test, int* n_bad, adb_stream_t stream);
int adb_eval_count_visible(int T, int height, int width, long long n_gaussians, int t, const uint8_t* mask, void* ws,
                           size_t ws_bytes, adb_stream_t stream);
int adb_eval_image_metrics(int T, int height, int width, long long n_gaussians, const float* colors, const float* alphas,
                           const float* exposure, const int* view_frame, const float* gt, float* image, float* ssim_map,
                           void* ws, size_t ws_bytes, adb_stream_t stream);
int adb_lpips_workspace_bytes(int n_frames, int height, int width, size_t* bytes /*HOST*/);
int adb_lpips_vgg_forward(int T, int height, int width, long long n_gaussians, int frame0, int n_frames, const float* img0,
                          const float* img1, const float* w1, const float* b1, const float* shift, const float* scale,
                          const void* const* w_hi /*HOST*/, const void* const* w_lo /*HOST*/,
                          const float* const* bias /*HOST*/, const float* const* lin /*HOST*/,
                          float* const* taps /*HOST or NULL*/, void* lws, size_t lws_bytes, void* ews, size_t ews_bytes,
                          adb_stream_t stream);
int adb_eval_reduce(int T, int height, int width, long long n_gaussians, int with_lpips, void* ws, size_t ws_bytes,
                    double* table, adb_stream_t stream);

/* ---- map re-anchoring after the Backend moves its key frames (csrc/reanchor.cu) ----
 *   adb_reanchor_keyframes  replaces the pose loop of run_system.py:194-226 (pypose SE3 / quat2unit / mul / Inv / matrix,
 *                           Keyframe.get_Rt / set_Rt, three torch.linalg.inv per mapper key frame) for all K frames in one
 *                           launch.  slam_T_WC [K_slam,8] the Backend's Sim(3) table (tx ty tz qx qy qz qw s);
 *                           last_keyframe_index [K] int64, is_slam_keyframe [K] uint8, T_CkCf [K,8] (read on non-SLAM rows
 *                           only); rW2C [K,3,2] / tW2C [K,3] updated IN PLACE (set_Rt).  Writes old_c2w / new_c2w [K,4,4]
 *                           (the inverses of get_Rt before and of new_Rt), approx_centres [K,3] = -new_R^T t and
 *                           cam_centres [K,3] = inverse(get_Rt().T)[3,:3] after set_Rt (sixD2mtx's re-orthonormalised R).
 *                           A row whose index is outside [0, K_slam) keeps its pose (new_c2w = old_c2w, both centres its
 *                           current one) and adds 1 to *n_bad (device int32, caller-zeroed)
 *   adb_reanchor_gaussians  replaces SceneModel.rigid_transform_gs (Reconstruct/scene/scene_models/h3dgsv3.py:955-966) and
 *                           update_gaussians (Reconstruct/utils.py:28-60): per Gaussian, with D = new_c2w[id] inv(old_c2w[id]),
 *                           xyz_out = D[:3,:3] xyz + D[:3,3] and rotation_out = mat2quat(D[:3,:3] quat2mat(rotation)) with
 *                           kornia's conversions (wxyz).  ids [N] int64, xyz [N,3], rotation [N,4]; rotation, rotation_out
 *                           and ws 16-byte aligned; outputs must not overlap inputs.  Rows with an id outside [0, K) or a
 *                           singular old_c2w[id] (zero pivot) are copied unchanged and added to *n_bad.  Two launches (one
 *                           over K, one over N); N == 0 launches nothing.  ws: adb_reanchor_workspace_bytes(K) */
int adb_reanchor_workspace_bytes(int K, size_t* bytes /*HOST*/);
int adb_reanchor_keyframes(int K, int K_slam, const float* slam_T_WC, const long long* last_keyframe_index,
                           const unsigned char* is_slam_keyframe, const float* T_CkCf, float* rW2C, float* tW2C,
                           float* old_c2w, float* new_c2w, float* cam_centres, float* approx_centres, int32_t* n_bad,
                           adb_stream_t stream);
int adb_reanchor_gaussians(long long N, int K, const long long* ids, const float* xyz, const float* rotation,
                           const float* old_c2w, const float* new_c2w, float* xyz_out, float* rotation_out, int32_t* n_bad,
                           void* ws, size_t ws_bytes, adb_stream_t stream);

/* ---- key-frame hand-off from the Backend to the mapper (csrc/keyframe.cu) ----
 *   adb_kf_dense_point      replaces Backend.prepare_for_mapper / compute_dense_point (VSLAM/Backend.py:117-193) at SLAM
 *                           resolution H x W.  X_canon [HW,3], K [3,3] row-major, dense_point [HW,4] (16-byte aligned).
 *                           last_T_WC == NULL is the first key frame: points = constrain_points_to_ray(X_canon), channel 3 =
 *                           float(C[p] * fp32(1 / N) > 1.5) with C [HW] and N a device int32 [1]; nothing else is read or
 *                           written.  Otherwise, with T_WC / last_T_WC the Sim(3) poses (tx ty tz qx qy qz qw s) of the key
 *                           frame and of the last key frame and idx_k2l [HW] int64: points = SE3(T_WC[:7]).Inv().Act(
 *                           T_WC.Act(Xc)) in key-frame pixel order, channel 3 = the reprojection confidence of
 *                           Xc[idx_k2l[p]] in the last key frame at its pixel p (1 below 3 px, else 1 / (r - 2)), and
 *                           T_CkC [8] = last_T_WC^-1 T_WC.  A pixel whose idx_k2l is outside [0, HW) is NaN in all four
 *                           channels and adds 1 to *n_bad (device int32, caller-zeroed).  One launch.
 *   adb_kf_pyramid_floats   floats of the packed pyramids of an H x W mapper image with pyr_levels levels (sizes floored
 *                           level by level): idepth_floats = sum of h_l w_l over levels 0.., image_floats = 3 h_l w_l over
 *                           levels 1.. (level 0 of the image pyramid is the image itself).
 *   adb_kf_mapper_inputs    replaces run_system.py:164-192 and Keyframe.__init__'s training branch
 *                           (Reconstruct/scene/keyframe.py:64-127) for an H x W mapper image, 1 <= pyr_levels <= 6.
 *                           image [3,H,W] read through image_strides (HOST [3], elements: channel, row, column);
 *                           dense_point [Hs,Ws,4] as adb_kf_dense_point writes it.  idepth_pyr: levels 0.. packed, level 0 =
 *                           interpolate(where(z != 0, 1 / (z + 1e-4), 1e4), (H, W), bilinear, align_corners=True), level l =
 *                           avg_pool2d(level l-1, 2); image_pyr: levels 1.. packed, [3,h_l,w_l] each (NULL if pyr_levels
 *                           == 1).  From Rt = quat2unit(SE3(T_WC[:7])).Inv().matrix(): rW2C [3,2] = Rt[:3,:2], tW2C [3] =
 *                           Rt[:3,3], approx_centre [3] = -Rt[:3,:3]^T Rt[:3,3] and R [3,3] = sixD2mtx(rW2C).  One launch. */
int adb_kf_dense_point(int height, int width, const float* X_canon, const float* C, const int32_t* N, const float* T_WC,
                       const float* last_T_WC, const long long* idx_k2l, const float* K, float* dense_point, float* T_CkC,
                       int32_t* n_bad, adb_stream_t stream);
int adb_kf_pyramid_floats(int height, int width, int pyr_levels, long long* idepth_floats /*HOST*/,
                          long long* image_floats /*HOST*/);
int adb_kf_mapper_inputs(int height, int width, int Hs, int Ws, int pyr_levels, const float* image,
                         const long long* image_strides /*HOST [3]*/, const float* dense_point, const float* T_WC,
                         float* idepth_pyr, float* image_pyr, float* rW2C, float* tW2C, float* approx_centre, float* R,
                         adb_stream_t stream);

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
/* Tile intersection (no library sort, no host sync; csrc/raster_isect.cu): bit-identical to gsplat's isect_tiles / radix
 * sort / isect_offset_encode behind h3dgsv3.py:664-680 — keys = cam|tile|depth_bits, vals = cam*N + gaussian, in the order
 * of a stable sort of the keys emitted Gaussian-major (oracle/raster_oracle.c, adbo_isect_sort).
 *   adb_raster_tile_count_scan   per-tile counts (RED.ADD) + one-CTA exclusive scan -> tile_offsets[T+1] clamped to
 *                                `capacity`; *total (int64, device) = true intersection count, *overflow (int32, device)
 *                                is SET when total > capacity.  tile_counts: int32[2*4*T] (4 replicated counters per tile,
 *                                then their segment starts); the first half must be zero on entry.
 *   adb_raster_tile_scan         the scan alone, for counters filled by adb_raster_project_fwd_counts.
 *   adb_raster_tile_band_scatter_sort
 *     band pass  one (Gaussian, tile row) pair per tile row a splat touches, appended per CTA in runs to the row's region
 *                of `scratch` (the row's tile segments; pairs of a row cut by the capacity are rebuilt from the splats);
 *     tile pass  one CTA per (tile row, view) expands the row's pairs into its tiles' segments of `packed` and zeroes the
 *                row's counters;
 *     sort       one CTA per tile sorts its segment (bitonic, shared memory; global memory beyond 4096 entries) and writes
 *                keys and vals.
 *     packed: uint64[capacity]; scratch: adb_raster_tile_band_scratch_bytes(capacity) bytes; neither needs initialisation.
 *     tile_counts as left by the scan: its per-tile segment starts are used, and overwritten, as per-row cursors, and its
 *     first half is zero again after a call that launches (N > 0 and capacity > 0).  W and H at most 65536 (4096 tiles).
 * legacy != 0 selects the Inria tile rectangle. */
int adb_raster_tile_count_scan(int N, const int32_t* radii, const float* splats, const int32_t* tiles_per_gauss, int W, int H,
                               int legacy, long long capacity, int32_t* tile_counts, int32_t* tile_offsets, long long* total,
                               int32_t* overflow, adb_stream_t stream);
int adb_raster_tile_scan(int W, int H, long long capacity, int32_t* tile_counts, int32_t* tile_offsets, long long* total,
                         int32_t* overflow, adb_stream_t stream);
/* View-batched intersection (one launch per stage for C views; 1 <= C <= 64).  capacities: HOST array [C]; view c owns the
 * segment [sum_{c'<c} capacities[c'], +capacities[c]) of one packed / keys / vals buffer (the sum must stay below 2^31 - 1).
 *   adb_raster_tile_scan_multi              one CTA per view: tile_offsets [C,T+1] ABSOLUTE in that buffer, clamped to the
 *                                           view's capacity; total int64 [C] and overflow int32 [C] (SET when total[c] >
 *                                           capacities[c]) on the device.  tile_offsets == NULL: totals only (a sizing pass).
 *   adb_raster_tile_band_scatter_sort_multi the three passes above with a view grid dimension; scratch for the sum of the
 *                                           capacities; vals = c*N + gaussian; keys (may be NULL: not written) = c|tile|depth_bits. */
int adb_raster_tile_scan_multi(int C, int W, int H, const long long* capacities /*HOST [C]*/, int32_t* tile_counts,
                               int32_t* tile_offsets, long long* total, int32_t* overflow, adb_stream_t stream);
int adb_raster_tile_band_scratch_bytes(long long capacity, size_t* bytes);
int adb_raster_tile_band_scatter_sort(int N, const int32_t* radii, const float* splats, const int32_t* tiles_per_gauss, int W,
                                      int H, int legacy, int cam_id, int n_cams, long long capacity, int32_t* tile_counts,
                                      const int32_t* tile_offsets, void* packed, void* scratch, size_t scratch_bytes,
                                      int64_t* keys, int32_t* vals, adb_stream_t stream);
int adb_raster_tile_band_scatter_sort_multi(int N, int C, const int32_t* radii, const float* splats,
                                            const int32_t* tiles_per_gauss, int W, int H,
                                            const long long* capacities /*HOST [C]*/, int32_t* tile_counts,
                                            const int32_t* tile_offsets, void* packed, void* scratch, size_t scratch_bytes,
                                            int64_t* keys, int32_t* vals, adb_stream_t stream);
/* Single-view blend pair.  hit_mask (may be NULL) shares the culling decisions: a non-NULL hit_mask makes the forward fill
 * one byte per sorted intersection (index as in vals_sorted): bit w = the splat can reach the 8x4 pixel block of warp w of its
 * tile (entries behind the point where a whole tile saturated are left unwritten).  Given that mask, the backward builds its
 * per-warp hit lists from it instead of repeating the box and ellipse tests (same splats / vals_sorted / tile_offsets;
 * identical gradients).  With NULL the forward writes no mask and the backward culls on its own. */
int adb_raster_blend_fwd(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                         const int32_t* tile_offsets, float* colors /*[H,W,4]*/, float* alphas /*[H,W]*/,
                         int32_t* last_ids /*[H,W]*/, unsigned char* hit_mask /*may be NULL*/, adb_stream_t stream);
int adb_raster_blend_bwd(int W, int H, int n_per_cam, const float* splats, const int32_t* vals_sorted,
                         const int32_t* tile_offsets, const float* alphas, const int32_t* last_ids,
                         const float* v_colors, const float* v_alphas, float* v_splats /*[N,12] zeroed, +=*/,
                         const unsigned char* hit_mask /*may be NULL*/, adb_stream_t stream);
/* View-batched blend pair (gridDim.z = C): splats [C,N,12] and v_splats [C,N,12] indexed by vals_sorted (c*N + gaussian)
 * directly, tile_offsets [C,T+1] from adb_raster_tile_scan_multi, colors / v_colors [C,H,W,4], alphas / last_ids / v_alphas
 * [C,H,W]; hit_mask (may be NULL) indexed like vals_sorted.  Per view the same images as the single-view pair; last_ids
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
 * Same buffers and key layout as the gsplat-convention entry points above; the tile intersection (legacy = 1) and
 * project_bwd are shared. */
int adb_raster_project_fwd_legacy(int N, const float* means, const float* quats, const float* scales,
                                  const float* opacities, const float* sh, int sh_degree, const float* viewmat,
                                  const float* K, const float* campos, int W, int H, float eps2d, float near_plane,
                                  float far_plane, int32_t* radii /*[N,2], both = Inria radius*/, float* splats,
                                  int32_t* tiles_per_gauss, adb_stream_t stream);
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
/* ---- the Backend's factor graph around the global solve (csrc/factor_graph.cu) ----
 * replaces FactorGraph (VSLAM/mast3r_slam/global_opt.py) except the solve, which is adb_gauss_newton.  Two-way edge table
 * of n pixels per row, caller-owned, `capacity` edges = 2 capacity rows: rows_i / rows_j int64 [2 capacity],
 * rows_idx int64 [2 capacity, n], rows_valid uint8 [2 capacity, n], rows_Q [2 capacity, n].  Edge e is row 2e =
 * (i, j, idx_i2j, valid_match_j, Qj) and row 2e+1 = (j, i, idx_j2i, valid_match_i, Qi), the matcher's masks as the
 * reference stores them (the solve applies Q_conf itself): the first 2E rows are adb_gauss_newton's
 * ii / jj (once mapped to pose positions), idx_ii2jj, valid_match and Q.
 *   adb_fg_gate               add_factors after matching (:56-110) for B <= 1024 candidate edges.  cand_ij int64 [B,2]
 *                             (i, j); idx_i2j / idx_j2i int64 [B,n]; valid_match_j / _i uint8 [B,n]; Qii, Qjj, Qji, Qij
 *                             [B,n].  Per pixel Qj = sqrt(Qii[b, idx_i2j] Qji), valid_j = valid_match_j & (Qj > Q_conf),
 *                             and the same for i.  Per edge the valid counts are summed in integers, match_frac =
 *                             count * fp32(1 / n), and the edge is invalid when min(frac_j, frac_i) < min_match_frac
 *                             unless i == j - 1; with is_reloc one invalid edge rejects all B.  Accepted edges are written
 *                             in candidate order at edges n_edges.. of the table (capacity >= n_edges + B: rows up to edge
 *                             n_edges + B - 1 are used as scratch).  accepted int32 [B] (0/1), counts int32 [B,2] (valid_j,
 *                             valid_i).  An index outside [0, n) is not read: its pixel is an invalid match with Q = NaN,
 *                             and it adds 1 to *n_bad (device int32, accumulated).  ws from adb_fg_gate_workspace_bytes.
 *                             Three launches (two when B == 1).
 *   adb_fg_mirror_refresh     the solve's key-frame inputs (get_poses_points, constrain_points_to_ray; :120-126,187-188):
 *                             for each of `rows` rows, mirror row d = ids ? ids[r] : r (rows with d outside
 *                             [0, mirror_rows) are skipped) gets Xm [d] = X (mode 0, rays) or constrain_points_to_ray(X)
 *                             with K [3,3] (mode 1, calib) and Cm [d] = C * fp32(1 / N).  The source row is r when `staged`
 *                             (X [rows,n,3], C [rows,n], N [rows] copied by the caller) and d otherwise (the key-frame store's
 *                             own stacked tensors).  With seen != NULL (int32 [mirror_rows,2]), a row whose (dataset_idx,
 *                             N_updates) equals seen[d] is left as it is, and every row's current pair is written to
 *                             seen_next[d] (another buffer: the caller alternates them).  One launch.
 *   adb_fg_pose_gather        poses [U,8] = quat2unit(T_WC[ids ? ids[r] : r]) for r < U; T_WC [src_rows,8].  One launch.
 *   adb_fg_pose_scatter       update_T_WCs(T_WCs[pin:], unique[pin:]): T_WC[ids ? ids[r] : r] = poses[r] for pin <= r < U;
 *                             nothing when U <= pin.  One launch. */
int adb_fg_gate_workspace_bytes(int B, int n, size_t* bytes /*HOST*/);
int adb_fg_gate(int B, int n, long long n_edges, long long capacity, const long long* cand_ij, const long long* idx_i2j,
                const long long* idx_j2i, const unsigned char* valid_match_j, const unsigned char* valid_match_i,
                const float* Qii, const float* Qjj, const float* Qji, const float* Qij, float Q_conf, float min_match_frac,
                int is_reloc, long long* rows_i, long long* rows_j, long long* rows_idx, unsigned char* rows_valid,
                float* rows_Q, int* accepted, int* counts, int* n_bad, void* ws, size_t ws_bytes, adb_stream_t stream);
int adb_fg_mirror_refresh(int mode, int rows, int height, int width, int mirror_rows, const long long* ids, int staged,
                          const float* X, const float* C, const int32_t* N, const int32_t* dataset_idx,
                          const int32_t* N_updates, const int32_t* seen, int32_t* seen_next, const float* K, float* Xm,
                          float* Cm, adb_stream_t stream);
int adb_fg_pose_gather(int n_unique, int src_rows, const long long* ids, const float* T_WC, float* poses,
                       adb_stream_t stream);
int adb_fg_pose_scatter(int n_unique, int pin, int dst_rows, const long long* ids, const float* poses, float* T_WC,
                        adb_stream_t stream);
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
 * Voxel index floor((p - mn) * fp32(1 / voxel_size)), PyTorch's device arithmetic for the reference's division; class ids
 * are read as 32-bit unsigned values.
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
 * centres (device); keep[i] = (count_i * fp32(1 / K) > visible_threshold) with count_i = #{k : |xyz_i - cam_k| < 2 d_max_i},
 * PyTorch's device arithmetic for the reference's count / K; visible_count [N] may be NULL. */
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
 * adb_layernorm     nn.LayerNorm(eps) rows of C (croco.py:34, blocks.py:127-130,186-191); C a multiple of 8 in [8, 2048];
 *                   x, gamma, beta, y, y_hi, y_lo 16-byte aligned (y or y_hi may be NULL, y_lo NULL gives hi only)
 * adb_rope_heads    RoPE2D + head split (pos_embed.py:112-159 / curope/kernels.cu:18-82): x fp32 [B,N,ld] -> bf16 split
 *                   [B,h,N,64] (mode 0 RoPE, 1 plain) or transposed [B,h,64,Npad] (mode 2, Npad a multiple of 8, pad
 *                   columns written as 0).  ld >= col0 + h*64, ld and col0 multiples of 4; x, hi, lo 16-byte aligned,
 *                   pos and table 8-byte aligned.  Positions outside [0, n_pos) are clamped to the nearest table row.
 * adb_softmax_rows  attn.softmax(-1) (blocks.py:106,163), fp32 in, bf16 split out; columns L..ld_out-1 are not written.
 *                   Any alignment (a misaligned or strided row takes the generic kernel); all -inf or NaN rows give NaN
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
 * output before the pixel shuffle, 25*256 columns) -> pts3d [B,H,W,3], conf [B,H,W], desc [B,H,W,24], desc_conf [B,H,W].
 * Alignment: upsample x, addend, y 16 bytes and hi, lo 8 bytes; head_postprocess pts and desc 16 bytes, the rest 4. */
int adb_upsample2x_nhwc(int B, int Hin, int Win, int C, int Hout, int Wout, const float* x, const float* addend, float* y,
                        void* hi, void* lo, adb_stream_t stream);
int adb_head_postprocess(int B, int H, int W, const float* pts, const float* lf, long long ld_lf, int n_desc, float* pts3d,
                         float* conf, float* desc, float* desc_conf, adb_stream_t stream);

/* ---- Pi3 (the Backend's accurate loop closure) ----
 * Paths under VSLAM/thirdparty/Pi3/pi3/models/ unless stated.  The dense layers run on adb_gemm_bf16 (act 2 = the camera
 * head's ReLU) and adb_attention_bf16; these are the Pi3-specific stages.  H and W must be multiples of 14 and at
 * least 14, every count of frames or views at least 1; misaligned pointers are refused before any launch.
 * adb_pi3_patch14      (imgs - image_mean) / image_std (pi3.py:174) + the 14x14/s14 patch-embedding conv's operand
 *                      (dinov2/layers/patch_embed.py:75): img [BN,3,H,W] in [0,1] -> bf16 split [BN*(H/14)*(W/14), 592],
 *                      columns in (c, ky, kx) order, 588..591 zero.  hi/lo 16-byte aligned, lo may be NULL.
 * adb_pi3_tokens       dinov2/models/vision_transformer.py:215-234: x [BN, 5+n, C] = [cls + pos[0], 4 registers,
 *                      patch + pos[1..n]]; patch [BN*n, C], cls [C], reg [4, C], pos [1+n, C] (the interpolated table).
 * adb_qknorm_rope      layers/attention.py:326-334: q or k of one qkv row block (columns col0 .. col0 + 64h of x fp32
 *                      [B*N, ld]) -> optional per-head LayerNorm(64, eps) (gamma = beta = NULL skips it), RoPE2D base 100
 *                      (layers/pos_embed.py:111-158; table as adb_rope_heads), bf16 split [B, h, N, 64].
 * adb_pi3_point_head   pi3.py:193-209 + transformer_head.py:70-80: pts [BN*hw, 588] and cf [BN*hw, 196] (LinearPts3d GEMM
 *                      outputs; the first `skip` rows of each view are register tokens), pose [BN,4,4] -> points,
 *                      local_points [BN,H,W,3], conf [BN,H,W].
 * adb_pi3_camera_tail  layers/camera_head.py:54-61: average pool of feat [BN*hw, 512] rows skip..hw-1, the more_mlps
 *                      (w0t, w2t transposed [in][out]), fc_t and fc_rot in fp32 -> rot [BN, 9], trans [BN, 3].
 * adb_pi3_svd_pose     layers/camera_head.py:66-93: R = V diag(1,1,det(V U^T)) U^T of the row-normalised rot^T, fp64 Jacobi;
 *                      pose [BN,4,4] = [R t; 0 1] (trans NULL: t = 0).
 * adb_pi3_window_input mast3r_slam/retrieval_database.py:21-41,268-270: img [N,3,Hi,Wi] in [-1,1] -> clamp(x/2 + 1/2, 0, 1)
 *                      bilinearly resized (align_corners=False, no antialias) to out [N,3,Ho,Wo]. */
int adb_pi3_patch14(int BN, int H, int W, const float* img, void* hi, void* lo, adb_stream_t stream);
int adb_pi3_tokens(int BN, int n, int C, const float* patch, const float* cls, const float* reg, const float* pos, float* x,
                   adb_stream_t stream);
int adb_qknorm_rope(int B, int N, int h, long long ld, int col0, const float* x, const float* gamma, const float* beta,
                    float eps, const long long* pos, const float* table, int n_pos, void* hi, void* lo, adb_stream_t stream);
int adb_pi3_point_head(int BN, int H, int W, int hw, int skip, const float* pts, const float* cf, const float* pose,
                       float* points, float* local_points, float* conf, adb_stream_t stream);
int adb_pi3_camera_tail(int BN, int hw, int skip, const float* feat, const float* w0t, const float* b0, const float* w2t,
                        const float* b2, const float* wt, const float* bt, const float* wr, const float* br, float* rot,
                        float* trans, adb_stream_t stream);
int adb_pi3_svd_pose(int BN, const float* rot, const float* trans, float* pose, adb_stream_t stream);
int adb_pi3_window_input(int N, int Hi, int Wi, const float* img, int Ho, int Wo, float* out, adb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif

"""artdeco_b200 — H100-native (sm_90a) kernels behind ARTDECO's hot-path operator surface.

Public operators (same names / argument meaning as the reference's, see each module's docstring):
  ssim.fused_ssim, ssim.FusedSSIMMap, ssim.fusedssim, ssim.fusedssim_backward      (fused_ssim)
  raster.rasterization                                 (gsplat.rendering.rasterization as ARTDECO calls it)
  adam.adamUpdate, adam.adamUpdateBasic                (diff_gaussian_rasterization, on-the-fly-nvs fork)
  knn.distCUDA2, knn.distIndex2, knn.distIndexQ        (simple_knn._C)
  cull.lod_select, cull.lod_cull                       (SceneModel.render's d_max cull)
  covmlp.cov_mlp_modulate                              (SceneModel.render's mlp_cov scale/rotation modulation)
  matching.iter_proj, matching.refine_matches, matching.match   (mast3r_slam_backends + utils_matching)
  optimizers.BaseAdam, optimizers.SparseGaussianAdam   (Reconstruct/scene/optimizers.py: fused step, one-launch add_and_prune)
  legacy.GaussianRasterizer, legacy.rasterize_gaussians  (diff_gaussian_rasterization legacy API, web viewer)
  tracking.track, tracking.opt_pose_calib_sim3         (VSLAM/CameraTracker.py: the Frontend's per-frame Sim(3) tracker)
  densify.add_new_gaussians, densify.sample_lod        (SceneModel.add_new_gaussians: key-frame densification)
  mapper.mapper_loss                                   (SceneModel.optimization_step's pixel loss, forward and backward)
  reanchor.keyframe_poses, reanchor.rigid_transform_gs (run_system.py's map update after the Backend moves its key frames)
  keyframe.dense_point, keyframe.mapper_keyframe       (Backend.prepare_for_mapper + Keyframe.__init__: the key-frame hand-off)
  factor_graph.FactorGraph                             (VSLAM/mast3r_slam/global_opt.py: the Backend's factor graph)
  evaluate.evaluate, lpips.LPIPSVGG                    (SceneModel.evaluate: held-out PSNR, SSIM and LPIPS-VGG)
  pi3.Pi3, pi3.accurate_loop_closure                  (Pi3 and RetrievalDatabase.accurate_loop_closure: the Backend's loop closure)
  retrieval.RetrievalDatabase                          (VSLAM/mast3r_slam/retrieval_database.py: the key-frame retrieval)
There is no CPU implementation: every operator raises unless a CUDA sm_90 device and the C-ABI library
``libartdeco_b200.so`` are available.
"""
from . import _lib  # noqa: F401
from . import adam, covmlp, cull, densify, evaluate, factor_graph, gn, keyframe, knn, legacy, lpips, mapper, mast3r, matching, multiview, optimizers, parallel, pi3, raster, reanchor, retrieval, scene, tracking, voxel  # noqa: F401  (each registers its C signatures)
from .adam import adamUpdate, adamUpdateBasic  # noqa: F401
from .covmlp import cov_mlp_modulate  # noqa: F401
from .cull import lod_cull, lod_select, weed_out_mask  # noqa: F401
from .scene import render_lod  # noqa: F401
from .voxel import update_voxel  # noqa: F401
from .knn import distCUDA2, distIndex2, distIndexQ  # noqa: F401
from .raster import rasterization  # noqa: F401
from .ssim import FusedSSIMMap, fused_ssim, fusedssim, fusedssim_backward  # noqa: F401

__version__ = "0.1.0"

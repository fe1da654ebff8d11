"""Host-side mirror of the hot block of ``SceneModel.render`` (Reconstruct/scene/scene_models/h3dgsv3.py:617-700): the caller
on the optimiser side of the rasterizer path (SURVEY.md §8a R0/R1/R2, BASELINE config 5: "10M Gaussians with LoD dmax cull,
4k render").

    LoD d_max cull  ->  [mlp_cov scale / rotation modulation]  ->  rasterization (RGB+D)  ->  background + inverse depth

What runs differently from the reference's ~30 torch kernels before the rasterizer:
  * the cull is ONE streaming pass (16 B/Gaussian) producing mask, fade ratio and the ascending id list (csrc/lod_cull.cu);
  * the selected rows of EVERY per-Gaussian tensor are gathered by ONE multi-tensor gather launch (csrc/compact.cu, the
    kernel behind ``add_and_prune``) when no gradient is needed (evaluation renders), or by differentiable ``index_select``s
    when it is (training);
  * ``mlp_cov`` is the fused kernel of ``covmlp.cov_mlp_modulate`` (csrc/cov_mlp.cu).
Same return dict as the reference: ``render [3,H,W]``, ``invdepth [1,H,W]``, ``visibility_filter [N0]``,
``global_visibility_filter [n_cls]`` (when class ids are given), ``scale``; plus the raw rasterizer outputs ``colors [1,H,W,4]``
(RGB + accumulated depth) and ``alphas [1,H,W,1]``, which ``mapper.mapper_loss`` consumes (call with ``bg=None`` for that).
"""
from __future__ import annotations

import torch

from . import _lib
from .cull import lod_select
from .raster import rasterization


def render_lod(width: int, height: int, view_matrix: torch.Tensor, *, xyz, opacity, f_dc, f_rest, scaling, rotation, d_max,
               tanfovx: float, tanfovy: float, sh_degree: int = 3, eps2d: float = 0.01, bg: torch.Tensor | None = None,
               cov_mlp=None, local_feat=None, global_feat=None, cls_id=None):
    """``view_matrix``: world->camera [4,4] on the device.  ``opacity`` [N0,1], ``f_dc`` [N0,1,3], ``f_rest`` [N0,15,3],
    ``scaling`` [N0,3], ``rotation`` [N0,4], ``d_max`` [N0,1] — the activated tensors the reference's properties return.
    ``cov_mlp``: optional dict(W1, b1, W2, b2) of ``mlp_cov`` (h3dgsv3.py:173-177) with ``local_feat`` / ``global_feat`` / ``cls_id``."""
    _lib.require_cuda(xyz)
    dev = xyz.device
    N0 = xyz.shape[0]
    need_grad = torch.is_grad_enabled() and any(t is not None and t.requires_grad
                                                for t in (xyz, opacity, f_dc, f_rest, scaling, rotation, local_feat, global_feat))
    cam_centre = torch.inverse(view_matrix.detach())[:3, 3].to(dev)
    selection_mask, ids, ratio = lod_select(xyz, d_max, cam_centre)
    n = int(ids.numel())
    idx = ids.long()
    if need_grad:
        xyz_s = xyz.index_select(0, idx)
        d_s = d_max.reshape(-1, 1).index_select(0, idx)
        dist = (xyz_s - cam_centre.reshape(1, 3)).norm(dim=1, keepdim=True)     # gradient to xyz through the fade ratio
        fade = (dist > d_s) & (dist < 2 * d_s)
        ratio_s = torch.where(fade, (2 * d_s - dist) / d_s, torch.ones_like(dist))
        op_s = (opacity.reshape(N0, 1).index_select(0, idx) * ratio_s).squeeze(-1)
        feats = torch.cat([f_dc.index_select(0, idx), f_rest.index_select(0, idx)], 1)
        sc_s, rot_s = scaling.index_select(0, idx), rotation.index_select(0, idx)
    else:
        from .optimizers import compact_gather
        jobs = [(xyz.detach().float(), None, 0, (3,)), (scaling.detach().float(), None, 0, (3,)),
                (rotation.detach().float(), None, 0, (4,)), (f_dc.detach().float().reshape(N0, 3), None, 0, (3,)),
                (f_rest.detach().float().reshape(N0, -1), None, 0, (int(f_rest.numel() // max(N0, 1)),))]
        with torch.cuda.device(dev):
            xyz_s, sc_s, rot_s, dc_s, rest_s = compact_gather(ids, n, 0, jobs, n_mask=N0)
        feats = torch.cat([dc_s.view(n, 1, 3), rest_s.view(n, -1, 3)], 1)
        op_s = (opacity.detach().reshape(N0) * ratio)[idx]
    if cov_mlp is not None:
        from .covmlp import cov_mlp_modulate
        lf_s = local_feat.index_select(0, idx)
        cid = cls_id.reshape(-1).index_select(0, idx).long()
        sc_s, rot_s = cov_mlp_modulate(sc_s, rot_s, lf_s, global_feat, cid, W1=cov_mlp["W1"], b1=cov_mlp["b1"],
                                       W2=cov_mlp["W2"], b2=cov_mlp["b2"])
    fl_x, fl_y = width / (2 * tanfovx), height / (2 * tanfovy)
    Ks = torch.tensor([[fl_x, 0, width / 2.0], [0, fl_y, height / 2.0], [0, 0, 1]], dtype=torch.float32, device=dev)[None]
    colors, alphas, meta = rasterization(means=xyz_s, quats=rot_s, scales=sc_s, opacities=op_s, colors=feats,
                                         viewmats=view_matrix.unsqueeze(0), Ks=Ks, width=width, height=height,
                                         render_mode="RGB+D", rasterize_mode="classic", absgrad=False, packed=False,
                                         sh_degree=sh_degree, eps2d=eps2d)
    rendered_color = colors[..., 0:3].permute([0, 3, 1, 2])
    rendered_alpha = alphas.permute([0, 3, 1, 2])
    if bg is not None:
        rendered_color = rendered_color + (1.0 - rendered_alpha) * bg.to(dev)[None, :, None, None]
    invdepth = 1.0 / colors[..., 3:4].permute([0, 3, 1, 2])
    visible_mask = torch.zeros(N0, dtype=torch.bool, device=dev)
    visible_mask[idx] = meta["radii"][0].max(dim=1).values > 0
    out = {"render": rendered_color[0], "invdepth": invdepth[0], "visibility_filter": visible_mask, "scale": sc_s,
           "selection_mask": selection_mask, "n_selected": n, "n_isect": int(meta["flatten_ids"].numel()),
           "colors": colors, "alphas": alphas}
    if cls_id is not None and global_feat is not None:
        gv = torch.zeros(len(global_feat), dtype=torch.bool, device=dev)
        gv[cls_id[visible_mask].reshape(-1).long()] = True
        out["global_visibility_filter"] = gv
    return out

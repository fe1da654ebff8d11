"""Host-side mirror of the LEGACY rasterizer API ``diff_gaussian_rasterization.{GaussianRasterizationSettings,
GaussianRasterizer, rasterize_gaussians}`` as the reference's web viewer calls it
(Reconstruct/webviewer/scene_models.py:33-36, 559-605; SURVEY.md §8a R3).

The fork that provides it (on-the-fly-nvs) is not vendored in the reference tree, so the numerical conventions are the
published Inria ones (see include/artdeco_b200.h, "legacy conventions"): positional settings
``(image_height, image_width, tanfovx, tanfovy, bg[3], scale_modifier, projmatrix[4,4] (transposed full projection),
sh_degree, campos[3], prefiltered, debug)`` and the call
``rasterizer(means3D, means2D, opacities[N,1], dc[N,1,3], shs[N,K,3], scales[N,3], rotations[N,4], viewmatrix[4,4]
(transposed world->camera))`` -> ``(color[3,H,W], invdepth[1,H,W], mainGaussID[1,H,W] int32, radii[N] int32)``.
``means2D`` is the usual gradient holder: after backward its ``.grad[:, :2]`` holds dL/d(mean2D) in the Inria NDC scaling
(pixel gradient x 0.5*W, 0.5*H).

All compute goes through the C ABI (adb_raster_*_legacy + the shared tile intersection and project_bwd).
"""
from __future__ import annotations

from typing import NamedTuple

import torch

from . import _lib
from .raster import _f32c, blend_backward, blend_forward, intersect, project, project_backward

EPS2D_INRIA = 0.3
NEAR_INRIA = 0.2


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


class _RasterizeLegacy(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means, means2D, quats, scales, opacities, sh, viewmat, K, campos, W, H, sh_degree):
        _lib.require_cuda(means)
        N = means.shape[0]
        with torch.cuda.device(means.device):
            radii, splats, tpg = project(means, quats, scales, opacities, sh, sh_degree, viewmat, K, campos, W, H,
                                         EPS2D_INRIA, NEAR_INRIA, 1e10, 0.0, legacy=True)
            _, vals, offsets, _ = intersect(radii, splats, tpg, W, H, legacy=True)
            colors, alphas, last_ids, main_ids = blend_forward(W, H, N, splats, vals, offsets, legacy=True)
        ctx.save_for_backward(means, quats, scales, opacities, sh, viewmat, K, campos, radii, splats, vals, offsets,
                              alphas, last_ids)
        ctx.cfg = (W, H, sh_degree)
        r1 = radii[:, 0].contiguous()
        ctx.mark_non_differentiable(main_ids, r1)
        return colors, alphas, main_ids, r1

    @staticmethod
    def backward(ctx, v_colors, v_alphas, *_unused):
        (means, quats, scales, opacities, sh, viewmat, K, campos, radii, splats, vals, offsets, alphas,
         last_ids) = ctx.saved_tensors
        W, H, sh_degree = ctx.cfg
        N = means.shape[0]
        dev = means.device
        v_colors = torch.zeros(H, W, 4, device=dev) if v_colors is None else _f32c(v_colors)
        v_alphas = torch.zeros(H, W, device=dev) if v_alphas is None else _f32c(v_alphas)
        with torch.cuda.device(dev):
            v_splats = blend_backward(W, H, N, splats, vals, offsets, alphas, last_ids, v_colors, v_alphas, legacy=True)
            live = radii[:, 0] > 0
            # slot 9 holds dL/d(1/z); project_bwd expects dL/dz
            z = torch.where(live, splats[:, 11], torch.ones_like(splats[:, 11]))
            v_splats[:, 9] = torch.where(live, -v_splats[:, 9] / (z * z), torch.zeros_like(z))
            # dL/d(mean2D) from the raw moments: d sigma/d mx = a dx + b dy (Inria scales it to NDC units)
            ca, cb, cc = splats[:, 2], splats[:, 3], splats[:, 4]
            gx = torch.where(live, ca * v_splats[:, 0] + cb * v_splats[:, 1], torch.zeros_like(ca))
            gy = torch.where(live, cb * v_splats[:, 0] + cc * v_splats[:, 1], torch.zeros_like(ca))
            v_means2D = torch.stack([gx * (0.5 * W), gy * (0.5 * H), torch.zeros_like(gx)], -1)
            v_means, v_quats, v_scales, v_opac, v_sh, v_view, v_campos = project_backward(
                means, quats, scales, opacities, sh, sh_degree, viewmat, K, campos, W, H, EPS2D_INRIA, NEAR_INRIA, 1e10, 0.0,
                radii, splats, v_splats)
        return (v_means, v_means2D, v_quats, v_scales, v_opac, v_sh, v_view, None, v_campos, None, None, None)


def _intrinsics(s: GaussianRasterizationSettings, dev: torch.device) -> torch.Tensor:
    """K from the settings, built on the device (no host sync).  ``projmatrix`` is the transposed PROJECTION-ONLY matrix,
    exactly what the reference's only call site passes (Reconstruct/webviewer/scene_models.py:549-566,881-887:
    ``getProjectionMatrix2(...).transpose(0,1)``; the view matrix comes per call).  Focal from tanfov as Inria's Jacobian
    uses it; principal point from P[0,2] = (2cx-W)/W, P[1,2] = (2cy-H)/H (Reconstruct/utils.py:133-154)."""
    W, H = int(s.image_width), int(s.image_height)
    P = _f32c(s.projmatrix.to(dev)).t()
    K = torch.zeros(3, 3, dtype=torch.float32, device=dev)
    K[0, 0] = W / (2.0 * float(s.tanfovx))
    K[1, 1] = H / (2.0 * float(s.tanfovy))
    K[0, 2] = (P[0, 2] + 1.0) * (0.5 * W)
    K[1, 2] = (P[1, 2] + 1.0) * (0.5 * H)
    K[2, 2] = 1.0
    return K


def rasterize_gaussians(means3D, means2D, opacities, dc, shs, scales, rotations, viewmatrix,
                        raster_settings: GaussianRasterizationSettings):
    s = raster_settings
    _lib.require_cuda(means3D)
    if s.prefiltered:
        raise NotImplementedError("rasterize_gaussians: prefiltered=True is not supported (the reference passes False)")
    N = means3D.shape[0]
    W, H = int(s.image_width), int(s.image_height)
    dev = means3D.device
    means = _f32c(means3D)
    quats = _f32c(rotations)
    scl = _f32c(scales) * float(s.scale_modifier) if float(s.scale_modifier) != 1.0 else _f32c(scales)
    opac = _f32c(opacities).reshape(N)
    sh = torch.cat([_f32c(dc).reshape(N, -1, 3), _f32c(shs).reshape(N, -1, 3)], 1)
    if (int(s.sh_degree) + 1) ** 2 > sh.shape[1]:
        raise ValueError("sh_degree needs more SH coefficients than dc/shs provide")
    if sh.shape[1] != 16:
        sh = torch.cat([sh, sh.new_zeros(N, 16 - sh.shape[1], 3)], 1) if sh.shape[1] < 16 else sh[:, :16]
    sh = sh.contiguous()
    V = _f32c(viewmatrix).t().contiguous()       # the legacy API passes the transposed world->camera matrix
    K = _intrinsics(s, dev).detach()
    campos = _f32c(s.campos.to(dev)).reshape(3)
    if means2D is None:
        means2D = torch.zeros(N, 3, dtype=torch.float32, device=dev)
    col, alp, main_ids, radii = _RasterizeLegacy.apply(means, means2D, quats, scl, opac, sh, V, K, campos, W, H,
                                                       int(s.sh_degree))
    bg = _f32c(s.bg.to(dev)).reshape(1, 1, 3)
    color = (col[..., :3] + (1.0 - alp[..., None]) * bg).permute(2, 0, 1)
    invdepth = col[..., 3][None]
    return color, invdepth, main_ids[None], radii


class GaussianRasterizer(torch.nn.Module):
    def __init__(self, raster_settings: GaussianRasterizationSettings):
        super().__init__()
        self.raster_settings = raster_settings

    def forward(self, means3D, means2D, opacities, dc, shs, scales, rotations, viewmatrix):
        return rasterize_gaussians(means3D, means2D, opacities, dc, shs, scales, rotations, viewmatrix,
                                   self.raster_settings)

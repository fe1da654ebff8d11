"""Host-side mirror of the pixel loss block of ``SceneModel.optimization_step`` (Reconstruct/scene/scene_models/h3dgsv3.py:430-450,
with ``render_from_id``'s exposure :611-614 and ``render``'s background composite and ``1/D`` :682-686).

    loss = lambda_dssim (1 - SSIM(m e, m gt)) + (1 - lambda_dssim) mean(rdk |m e - m gt|) + depth_weight mean(rdk |m/D - m mono|)

with ``e = clamp(E[:, :3] (rgb + (1 - alpha) bg) + E[:, 3], 0, 1)`` and ``m`` the ``is_important=False`` error mask (all ones
otherwise).  What runs differently from the reference's few dozen eager kernels each way (csrc/mapper_loss.cu):
  * one streaming pass per pixel reads the rasterizer's channels-last ``colors [1,h,w,4]`` / ``alphas [1,h,w,1]`` and writes the
    SSIM operands; the SSIM window work is ``adb_ssim_forward / adb_ssim_backward``; one small launch adds the per-block
    partial sums in a fixed order, so the loss and the exposure gradient are bitwise reproducible;
  * the backward is one pass that writes ``v_colors`` / ``v_alphas`` in the rasterizer's layout (no permutes) and per-block
    partials of ``dL/dE``; the upstream gradient stays on the device (no host sync anywhere);
  * the radial weights ``radial_decay_kernel(h, w, sigma)`` are computed once per ``(h, w, sigma, device)`` with the
    reference's own expression and kept on the device, instead of a CPU build and a pageable upload every step.
``scaling_reg`` is per-Gaussian, not per-pixel, and stays with the caller (``factor * scale.prod(1).mean()``)."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import f32, i32, vp

_lib.register("adb_mapper_loss_workspace_bytes", [i32, i32, C.POINTER(C.c_size_t)])
_lib.register("adb_mapper_loss_forward", [i32, i32, vp, vp, vp, vp, vp, vp, vp, i32, vp, vp, vp, vp, C.c_size_t, vp])
_lib.register("adb_mapper_loss_reduce", [i32, i32, vp, f32, f32, vp, vp, C.c_size_t, vp])
_lib.register("adb_mapper_loss_backward", [i32, i32, vp, vp, vp, vp, vp, vp, vp, i32, vp, vp, f32, f32, vp, vp, vp, vp,
                                           C.c_size_t, vp])

SSIM_C1, SSIM_C2 = 0.01 ** 2, 0.03 ** 2

_RDK: dict = {}


def radial_decay_kernel(H: int, W: int, sigma: float = 0.5) -> torch.Tensor:
    """Reconstruct/utils.py:818-826, the same expression evaluated on the CPU (so the table is bit-identical)."""
    y = torch.linspace(-1, 1, steps=H)
    x = torch.linspace(-1, 1, steps=W)
    yy, xx = torch.meshgrid(y, x, indexing='ij')
    r2 = xx**2 + yy**2
    return torch.exp(-r2 / (2 * sigma**2))


def radial_weights(h: int, w: int, sigma: float, device) -> torch.Tensor:
    """``radial_decay_kernel(h, w, sigma)`` on ``device``, built and uploaded once per key and then reused."""
    device = torch.device(device)
    key = (int(h), int(w), float(sigma), device)
    t = _RDK.get(key)
    if t is None:
        t = radial_decay_kernel(int(h), int(w), sigma).to(device).contiguous()
        _RDK[key] = t
    return t


def workspace(h: int, w: int, device) -> torch.Tensor:
    nb = C.c_size_t(0)
    _lib.call("adb_mapper_loss_workspace_bytes", int(h), int(w), C.byref(nb))
    return torch.empty(nb.value, dtype=torch.uint8, device=device)


def _f32(t: torch.Tensor, shape) -> torch.Tensor:
    t = t.detach()
    if t.dtype != torch.float32:
        raise ValueError(f"mapper_loss expects float32 tensors, got {t.dtype}")
    return t.reshape(shape).contiguous()


class _MapperLoss(torch.autograd.Function):

    @staticmethod
    def forward(ctx, colors, alphas, exposure, gt, mono, bg, rdk, lambda_dssim, depth_weight, is_important):
        h, w = int(colors.shape[1]), int(colors.shape[2])
        dev = colors.device
        cols, alph = _f32(colors, (h, w, 4)), _f32(alphas, (h, w))
        E, gt_, mono_, bg_ = _f32(exposure, (3, 4)), _f32(gt, (3, h, w)), _f32(mono, (h, w)), _f32(bg, (3,))
        ws = workspace(h, w, dev)
        img = torch.empty(3, h, w, dtype=torch.float32, device=dev)
        gtm = torch.empty_like(img)
        inv = torch.empty(1, h, w, dtype=torch.float32, device=dev)
        smap, d1, d2, d3 = (torch.empty_like(img) for _ in range(4))
        terms = torch.empty(4, dtype=torch.float32, device=dev)
        lam, wd = float(lambda_dssim), float(depth_weight)
        s = _lib.stream()
        with torch.cuda.device(dev):
            _lib.call("adb_mapper_loss_forward", h, w, _lib.ptr(cols), _lib.ptr(alph), _lib.ptr(gt_), _lib.ptr(mono_),
                      _lib.ptr(E), _lib.ptr(bg_), _lib.ptr(rdk, torch.float32), int(bool(is_important)), _lib.ptr(img),
                      _lib.ptr(gtm), _lib.ptr(inv), _lib.ptr(ws), ws.numel(), s)
            _lib.call("adb_ssim_forward", 1, 3, h, w, SSIM_C1, SSIM_C2, _lib.ptr(img), _lib.ptr(gtm), 1, _lib.ptr(smap),
                      _lib.ptr(d1), _lib.ptr(d2), _lib.ptr(d3), None, s)
            _lib.call("adb_mapper_loss_reduce", h, w, _lib.ptr(smap), lam, wd, _lib.ptr(terms), _lib.ptr(ws), ws.numel(), s)
        ctx.save_for_backward(cols, alph, E, gt_, mono_, bg_, rdk, img, gtm, d1, d2, d3, ws)
        ctx.args = (h, w, lam, wd, int(bool(is_important)))
        ctx.shapes = (colors.shape, alphas.shape)
        ctx.mark_non_differentiable(img, inv)
        return terms[0].reshape(()), img, inv

    @staticmethod
    def backward(ctx, g_loss, _g_img, _g_inv):
        cols, alph, E, gt_, mono_, bg_, rdk, img, gtm, d1, d2, d3, ws = ctx.saved_tensors
        h, w, lam, wd, important = ctx.args
        dev = cols.device
        g = g_loss.detach().to(torch.float32).reshape(1).contiguous()      # stays on the device: no host sync
        dssim = torch.empty_like(img)
        v_colors = torch.empty(h, w, 4, dtype=torch.float32, device=dev)
        v_alphas = torch.empty(h, w, dtype=torch.float32, device=dev)
        v_E = torch.empty(3, 4, dtype=torch.float32, device=dev)
        s = _lib.stream()
        with torch.cuda.device(dev):
            _lib.call("adb_ssim_backward", 1, 3, h, w, SSIM_C1, SSIM_C2, _lib.ptr(img), _lib.ptr(gtm), None, _lib.ptr(g),
                      -lam / (3 * h * w), _lib.ptr(d1), _lib.ptr(d2), _lib.ptr(d3), _lib.ptr(dssim), s)
            _lib.call("adb_mapper_loss_backward", h, w, _lib.ptr(cols), _lib.ptr(alph), _lib.ptr(gt_), _lib.ptr(mono_),
                      _lib.ptr(E), _lib.ptr(bg_), _lib.ptr(rdk), important, _lib.ptr(dssim), _lib.ptr(g), lam, wd,
                      _lib.ptr(v_colors), _lib.ptr(v_alphas), _lib.ptr(v_E), _lib.ptr(ws), ws.numel(), s)
        cshape, ashape = ctx.shapes
        return (v_colors.reshape(cshape), v_alphas.reshape(ashape), v_E, None, None, None, None, None, None, None)


def mapper_loss(colors: torch.Tensor, alphas: torch.Tensor, gt_image: torch.Tensor, mono_idepth: torch.Tensor,
                exposure: torch.Tensor, bg: torch.Tensor, *, lambda_dssim: float, depth_weight: float, rad_decay: float,
                is_important: bool):
    """The reference's ``lambda (1 - ssim) + (1 - lambda) l1 + depth_weight depth`` for one view.

    ``colors [1,h,w,4]`` / ``alphas [1,h,w,1]``: ``render_lod(..., bg=None)["colors"]`` / ``["alphas"]`` (the raw rasterizer
    outputs, RGB + accumulated depth).  ``gt_image [3,h,w]``, ``mono_idepth [1,h,w]``, ``exposure`` the key frame's
    ``[3,4]`` (or ``[4,4]``, of which rows ``:3`` are used), ``bg [3]``; all float32 on one CUDA device.
    ``depth_weight`` is ``keyframe.depth_loss_weight``, ``rad_decay`` the radial sigma.

    Returns ``(loss, image, invdepth)``: the 0-d loss, differentiable in ``colors``, ``alphas`` and ``exposure`` (``bg``,
    ``gt_image`` and ``mono_idepth`` get no gradient, as in the reference), and the loss's own operands ``image [3,h,w]``
    (exposed, clamped, masked) and ``invdepth [1,h,w]`` (masked ``1/D``), which are not differentiable.  With
    ``is_important=True`` ``invdepth`` equals ``render_lod(...)["invdepth"]``, the value the reference keeps as
    ``keyframe.latest_invdepth``; with ``is_important=False`` that stays ``render_lod``'s unmasked one."""
    _lib.require_cuda(colors)
    if colors.dim() != 4 or colors.shape[0] != 1 or colors.shape[3] != 4:
        raise ValueError(f"colors must be [1,h,w,4], got {tuple(colors.shape)}")
    h, w = int(colors.shape[1]), int(colors.shape[2])
    if alphas.numel() != h * w or gt_image.shape != (3, h, w) or mono_idepth.numel() != h * w:
        raise ValueError(f"alphas [1,h,w,1], gt_image [3,h,w] and mono_idepth [1,h,w] must match colors {tuple(colors.shape)}")
    if exposure.dim() != 2 or exposure.shape[0] < 3 or exposure.shape[1] != 4 or bg.numel() != 3:
        raise ValueError("exposure must be [3,4] (or [4,4]) and bg [3]")
    dev = colors.device
    for name, t in (("alphas", alphas), ("gt_image", gt_image), ("mono_idepth", mono_idepth), ("exposure", exposure),
                    ("bg", bg)):
        if t.device != dev:
            raise ValueError(f"mapper_loss: {name} is on {t.device}, colors on {dev}")
    rdk = radial_weights(h, w, rad_decay, dev)
    loss, image, invdepth = _MapperLoss.apply(colors, alphas, exposure[:3], gt_image, mono_idepth, bg, rdk,
                                              lambda_dssim, depth_weight, is_important)
    return loss, image, invdepth

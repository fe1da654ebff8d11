"""Host-side mirror of ``SceneModel.evaluate`` (Reconstruct/scene/scene_models/h3dgsv3.py:523-558) with
``harmonize_test_exposure`` (:507-520): PSNR, SSIM and LPIPS of every held-out key frame, averaged.

What runs differently from the reference (csrc/evaluate.cu):
  * the harmonisation is one device thread over the stacked ``[K,3,4]`` exposure table, in the reference's order (a test
    frame right after another averages the already updated one; ``idxm = 1`` at index 0, ``idxp = K - 2`` at the last
    index, negative indices wrap as Python's do);
  * every test view is rendered at level 0 through ``render_lod`` into one stacked buffer (the LoD cull is per camera, so
    one view at a time); its visible-Gaussian count stays on the device;
  * one streaming pass applies the exposure and clamp (``render_from_id`` with ``bg = 0``) and takes squared-error partials,
    ``adb_ssim_forward`` runs all views at once, LPIPS-VGG runs on the tensor cores (:mod:`artdeco_b200.lpips`), and one
    launch adds every partial in a fixed order into a ``[T, 11]`` table;
  * the reference's four ``.item()`` per frame become ONE host read at the end (the renders themselves still size their
    buffers on the host, as ``render_lod`` always does).
The mask of the reference's ``evaluate`` is all ones, so nothing is gathered.  ``save_test_frames`` is not mirrored."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import i32, i64, vp
from .scene import render_lod

_lib.register("adb_eval_workspace_bytes", [i32, i32, i32, i64, C.POINTER(C.c_size_t)])
_lib.register("adb_eval_harmonize", [i32, vp, vp, vp, vp])
_lib.register("adb_eval_count_visible", [i32, i32, i32, i64, i32, vp, vp, C.c_size_t, vp])
_lib.register("adb_eval_image_metrics", [i32, i32, i32, i64, vp, vp, vp, vp, vp, vp, vp, vp, C.c_size_t, vp])
_lib.register("adb_eval_reduce", [i32, i32, i32, i64, i32, vp, C.c_size_t, vp, vp])

N_METRICS = 11
COL_PSNR, COL_SSIM, COL_LPIPS, COL_RENDER, COL_GS, COL_MSE, COL_TAPS = 0, 1, 2, 3, 4, 5, 6


def eval_workspace(T: int, h: int, w: int, n_gaussians: int, device) -> torch.Tensor:
    nb = C.c_size_t(0)
    _lib.call("adb_eval_workspace_bytes", int(T), int(h), int(w), int(n_gaussians), C.byref(nb))
    return torch.zeros(nb.value, dtype=torch.uint8, device=device)


def reduce(T: int, h: int, w: int, n_gaussians: int, with_lpips: bool, ews: torch.Tensor) -> torch.Tensor:
    table = torch.empty(T, N_METRICS, dtype=torch.float64, device=ews.device)
    _lib.call("adb_eval_reduce", int(T), int(h), int(w), int(n_gaussians), int(bool(with_lpips)), _lib.ptr(ews),
              ews.numel(), _lib.ptr(table), _lib.stream())
    return table


def harmonize_test_exposure(exposure: torch.Tensor, is_test: torch.Tensor) -> torch.Tensor:
    """``exposure`` [K,3,4] float32 on the device, updated IN PLACE; ``is_test`` [K] bool / uint8 on the same device.
    Returns a device int32 [1]: 1 where the reference's loop raises IndexError (a test frame with K = 1), else 0."""
    _lib.require_cuda(exposure)
    if exposure.dim() != 3 or exposure.shape[1:] != (3, 4) or exposure.dtype != torch.float32 or not exposure.is_contiguous():
        raise ValueError(f"exposure must be a contiguous float32 [K,3,4], got {tuple(exposure.shape)} {exposure.dtype}")
    K = exposure.shape[0]
    if is_test.numel() != K or is_test.device != exposure.device:
        raise ValueError("is_test must be [K] on the exposure's device")
    flags = is_test.reshape(K).to(torch.uint8).contiguous()
    n_bad = torch.empty(1, dtype=torch.int32, device=exposure.device)
    with torch.cuda.device(exposure.device):
        _lib.call("adb_eval_harmonize", K, _lib.ptr(exposure), _lib.ptr(flags), _lib.ptr(n_bad), _lib.stream())
    return n_bad


def metrics_from_renders(colors: torch.Tensor, alphas: torch.Tensor, gt: torch.Tensor, exposure: torch.Tensor,
                         view_frame: torch.Tensor, *, ews: torch.Tensor | None = None, n_gaussians: int = 0,
                         lpips=None, workspace_bytes: int | None = None) -> torch.Tensor:
    """Per-view metrics of T stacked renders, on the device with no host sync.

    ``colors [T,h,w,4]`` / ``alphas [T,h,w(,1)]`` the rasterizer's raw outputs, ``gt [T,3,h,w]``, ``exposure [K,3,4]`` the
    (harmonised) table and ``view_frame [T]`` int32 the key frame of each view.  ``ews``: the evaluation workspace, which
    already holds the visible counts when the caller rendered through :func:`evaluate`.  ``lpips``: an
    :class:`artdeco_b200.lpips.LPIPSVGG` or None.  Returns the [T, 11] float64 table (columns ``COL_*``)."""
    _lib.require_cuda(colors)
    if colors.dim() != 4 or colors.shape[3] != 4:
        raise ValueError(f"colors must be [T,h,w,4], got {tuple(colors.shape)}")
    T, h, w = (int(x) for x in colors.shape[:3])
    if alphas.numel() != T * h * w or tuple(gt.shape) != (T, 3, h, w) or view_frame.numel() != T:
        raise ValueError("alphas [T,h,w], gt [T,3,h,w] and view_frame [T] must match colors")
    if exposure.dim() != 3 or exposure.shape[1:] != (3, 4):
        raise ValueError("exposure must be [K,3,4]")
    dev = colors.device
    for name, t in (("alphas", alphas), ("gt", gt), ("exposure", exposure), ("view_frame", view_frame)):
        if t.device != dev:
            raise ValueError(f"metrics_from_renders: {name} is on {t.device}, colors on {dev}")
    if view_frame.dtype != torch.int32:
        raise ValueError("view_frame must be int32")
    for name, t in (("colors", colors), ("alphas", alphas), ("gt", gt), ("exposure", exposure)):
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError(f"{name} must be a contiguous float32 tensor")
    if lpips is not None and (h < 16 or w < 16):
        raise ValueError("LPIPS needs h and w >= 16 (VGG16 pools four times)")
    if ews is None:
        ews = eval_workspace(T, h, w, n_gaussians, dev)
    image = torch.empty(T, 3, h, w, dtype=torch.float32, device=dev)
    smap = torch.empty_like(image)
    with torch.cuda.device(dev):
        _lib.call("adb_eval_image_metrics", T, h, w, int(n_gaussians), _lib.ptr(colors), _lib.ptr(alphas), _lib.ptr(exposure),
                  _lib.ptr(view_frame), _lib.ptr(gt), _lib.ptr(image), _lib.ptr(smap), _lib.ptr(ews), ews.numel(),
                  _lib.stream())
        del smap
        if lpips is not None:
            from .lpips import DEFAULT_WORKSPACE_BYTES
            lpips.run(T, h, w, n_gaussians, image, gt, ews,
                      DEFAULT_WORKSPACE_BYTES if workspace_bytes is None else int(workspace_bytes))
        return reduce(T, h, w, n_gaussians, lpips is not None, ews)


def evaluate(exposure: torch.Tensor, is_test, view_matrices, gt_images, *, width: int, height: int,
             render_kwargs: dict | None = None, render=None, lpips=None, with_LPIPS: bool = False, all: bool = False,
             first_index: int = 0, workspace_bytes: int | None = None) -> dict:
    """``SceneModel.evaluate(with_LPIPS, all)``.

    ``exposure [K,3,4]`` float32 on the device: the key frames' exposures, harmonised IN PLACE as the reference does.
    ``is_test``: K host booleans (``keyframe.is_test``); ``view_matrices``: K world->camera [4,4] (``keyframe.get_Rt()``);
    ``gt_images``: K images [3,h,w] (``keyframe.image_pyr[0]``; only the test frames' are read); ``render_kwargs``: the
    scene's ``render_lod`` keywords (Gaussians, ``tanfovx`` / ``tanfovy``, ...); or ``render(view_matrix)``: any callable
    returning ``render_lod``'s ``colors``, ``alphas`` and ``visibility_filter`` for one view.  ``first_index`` is
    ``keyframes[0].index``, where the loop starts unless ``all``.  ``lpips``: an :class:`~artdeco_b200.lpips.LPIPSVGG`
    (the reference's ``self.lpips``; None skips the value as a failed ``lpips`` import does).

    Returns the reference's dict: ``PSNR``, ``SSIM``, ``Render``, ``GS`` (and ``LPIPS`` with ``with_LPIPS``) averaged
    over the test frames, and ``n_test_frames``; ``{"n_test_frames": 0}`` without test frames."""
    _lib.require_cuda(exposure)
    dev = exposure.device
    is_test = [bool(x) for x in is_test]
    K = len(is_test)
    if exposure.shape[0] != K or len(view_matrices) != K or len(gt_images) != K:
        raise ValueError("exposure, is_test, view_matrices and gt_images must all have K entries")
    n_bad = harmonize_test_exposure(exposure, torch.tensor(is_test, dtype=torch.uint8).to(dev))
    start = 0 if all else int(first_index)
    views = [i for i in range(start, K) if is_test[i]]
    T = len(views)
    table = None
    if T > 0:
        h, w = int(height), int(width)
        if render is None:
            def render(vm):
                return render_lod(w, h, vm, **render_kwargs)
        ews = n_g = None
        colors = torch.empty(T, h, w, 4, dtype=torch.float32, device=dev)
        alphas = torch.empty(T, h, w, dtype=torch.float32, device=dev)
        gt = torch.empty(T, 3, h, w, dtype=torch.float32, device=dev)
        with torch.no_grad():
            for t, i in enumerate(views):
                out = render(view_matrices[i].to(dev))
                vis = out["visibility_filter"].reshape(-1).contiguous()
                if ews is None:
                    n_g = int(vis.numel())     # GS: len(visibility_filter), the same for every view
                    ews = eval_workspace(T, h, w, n_g, dev)
                colors[t].copy_(out["colors"].reshape(h, w, 4))
                alphas[t].copy_(out["alphas"].reshape(h, w))
                gt[t].copy_(gt_images[i].reshape(3, h, w))
                with torch.cuda.device(dev):
                    _lib.call("adb_eval_count_visible", T, h, w, n_g, t, _lib.ptr(vis.view(torch.uint8)), _lib.ptr(ews),
                              ews.numel(), _lib.stream())
        view_frame = torch.tensor(views, dtype=torch.int32).to(dev)
        table = metrics_from_renders(colors, alphas, gt, exposure, view_frame, ews=ews, n_gaussians=n_g,
                                     lpips=lpips if with_LPIPS else None, workspace_bytes=workspace_bytes)
    # the one host read
    host = torch.cat([n_bad.double(), table.reshape(-1)]) if table is not None else n_bad.double()
    host = host.cpu()
    if host[0] != 0:
        raise IndexError("list index out of range (harmonize_test_exposure: a test key frame without neighbours)")
    return summarise(host[1:].reshape(T, N_METRICS) if T > 0 else None, with_LPIPS, lpips is not None)


def summarise(table, with_LPIPS: bool, have_lpips: bool) -> dict:
    """The reference's accumulation of the per-frame ``.item()`` values, in frame order, from a host table."""
    metrics = {"PSNR": 0.0, "SSIM": 0.0, "Render": 0.0, "GS": 0.0}
    if with_LPIPS:
        metrics["LPIPS"] = 0.0
    n = 0 if table is None else int(table.shape[0])
    for t in range(n):
        row = table[t].tolist()
        metrics["Render"] += int(row[COL_RENDER])
        metrics["GS"] += int(row[COL_GS])
        metrics["PSNR"] += row[COL_PSNR]
        metrics["SSIM"] += row[COL_SSIM]
        if with_LPIPS and have_lpips:
            metrics["LPIPS"] += row[COL_LPIPS]
    if n > 0:
        for k in metrics:
            metrics[k] /= n
    else:
        metrics = {}
    metrics["n_test_frames"] = n
    return metrics

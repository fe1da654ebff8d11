"""Host-side mirror of ``SceneModel.add_new_gaussians`` (Reconstruct/scene/scene_models/h3dgsv3.py:766-940): which pixels of a
new key frame become Gaussians, and with what initial parameters, for each LoD in ``(1, 2, 4, 8)``.

What runs differently from the reference's ~60 small torch kernels and ~5 host syncs per LoD (csrc/densify.cu):
  * one stencil launch per LoD computes the resized image and render, both ``get_lapla_norm`` filters, the Bernoulli decision,
    the depth / confidence samples and the validity test; a scan and one emission launch write the rows in the row-major pixel
    order of the reference's boolean masks.  The host reads one row count per LoD;
  * ``torch.quantile(point_map[:, 2], 0.02)`` and the prune mask are computed once per call instead of once per LoD (the
    reference recomputes the same values in every iteration);
  * the scene does not change inside the LoD loop, so the render is reused while the class ids it was made with are unchanged
    (or when there is no ``mlp_cov``; the rasterizer is deterministic, so reuse is exact).  ``update_voxel`` moves its voxel
    origin with every LoD's new points and may renumber the classes, so with ``mlp_cov`` the render is redone when they change.
The arithmetic is the reference's, including its quirks: ``inverse_sigmoid(0.2 conf)`` is inf or NaN for ``conf >= 5``, new
class ids restart at 0 in every LoD of a cold start, and ``id`` is the given key-frame index."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import f32, i32, i64, vp
from .cull import weed_out_mask
from .scene import render_lod
from .voxel import update_voxel

f64 = C.c_double
_lib.register("adb_densify_workspace_bytes", [i32, i32, C.POINTER(C.c_size_t)])
_lib.register("adb_densify_depth_quantile", [i64, vp, f32, vp, vp, C.c_size_t, vp])
_lib.register("adb_densify_sample", [i32, i32, i32, vp, vp, C.POINTER(C.c_longlong), vp, i32, i32, vp, vp, vp, vp, f32, f32, vp,
                                     vp, vp, vp, vp, C.c_size_t, vp])
_lib.register("adb_densify_emit", [i32, i32, i32, vp, i32, i32, vp, vp, vp, vp, vp, f64, vp, vp, vp, vp, vp, vp, C.c_size_t, vp])
_lib.register("adb_densify_prune_mask", [i64, vp, vp, vp, vp, f64, i32, vp, vp])

LODS = (1, 2, 4, 8)
QUANTILE = 0.02
EXT_KEYS = ("id", "cls_id", "d_max", "xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "local_feat", "global_feat")


def workspace(height: int, width: int, device) -> torch.Tensor:
    nb = C.c_size_t(0)
    _lib.call("adb_densify_workspace_bytes", int(height), int(width), C.byref(nb))
    return torch.empty(nb.value, dtype=torch.uint8, device=device)


def _f32(t: torch.Tensor, shape=None) -> torch.Tensor:
    t = t.detach().float()
    return (t.reshape(shape) if shape is not None else t).contiguous()


def depth_quantile(point_map: torch.Tensor, ws: torch.Tensor | None = None) -> torch.Tensor:
    """``[torch.quantile(point_map[:, 2], 0.02), fp32(min(0.01, that))]`` as a float32 [2] device tensor (no host sync)."""
    _lib.require_cuda(point_map)
    z = _f32(point_map[:, 2]).reshape(-1)
    dev = z.device
    if ws is None:
        ws = workspace(1, 1, dev)
    out = torch.empty(2, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.call("adb_densify_depth_quantile", z.numel(), _lib.ptr(z), QUANTILE, _lib.ptr(out), _lib.ptr(ws), ws.numel(),
                  _lib.stream())
    return out


def prune_mask(xyz: torch.Tensor, opacity: torch.Tensor, scaling: torch.Tensor, approx_centre: torch.Tensor, f: float,
               width: int) -> torch.Tensor:
    """``valid_gs_mask`` of h3dgsv3.py:894-905 from the RAW (pre-activation) opacity [N,1] and scaling [N,3]."""
    _lib.require_cuda(xyz)
    N = int(xyz.shape[0])
    mask = torch.empty(N, dtype=torch.bool, device=xyz.device)
    with torch.cuda.device(xyz.device):
        _lib.call("adb_densify_prune_mask", N, _lib.ptr(_f32(xyz)), _lib.ptr(_f32(opacity)), _lib.ptr(_f32(scaling)),
                  _lib.ptr(_f32(approx_centre, (3,))), float(f), int(width), _lib.ptr(mask.view(torch.uint8)), _lib.stream())
    return mask


def sample_lod(image: torch.Tensor, render: torch.Tensor | None, point_map: torch.Tensor, conf: torch.Tensor, R: torch.Tensor,
               t: torch.Tensor, approx_centre: torch.Tensor, exposure: torch.Tensor, *, lod: int, f: float,
               init_proba_scaler: float, gs_add_ratio: float, uniforms: torch.Tensor, qmin: torch.Tensor,
               ws: torch.Tensor | None = None) -> dict:
    """One LoD of the loop body (h3dgsv3.py:779-891) up to the voxel step.

    ``image`` [3,H,W] (``image_pyr[0]``), ``render`` [3,H,W] raw RGB of the scene from this key frame or None (empty scene),
    ``point_map`` [1,3,Hs,Ws], ``conf`` [1,1,Hs,Ws], ``R`` [3,3] / ``t`` [3] world-to-camera, ``exposure`` [3,4], ``uniforms``
    [H/lod, W/lod] the draw, ``qmin`` the device tensor of ``depth_quantile``.  Returns the maps ``init_proba`` and ``penalty``
    (both x init_proba_scaler; the penalty is 0 without a render), ``flags`` [h,w] uint8 (bit 0 sampled, bit 1 valid), ``n`` and
    the rows ``xyz`` [n,3],
    ``f_dc`` [n,1,3], ``scaling`` [n,3], ``opacity`` [n,1], ``d_max`` [n,1].  One host sync: the row count."""
    _lib.require_cuda(image)
    dev = image.device
    H, W = int(image.shape[-2]), int(image.shape[-1])
    h, w = H // lod, W // lod
    Hs, Ws = int(point_map.shape[-2]), int(point_map.shape[-1])
    img = _f32(image, (3, H, W))
    depth = _f32(point_map[:, 2], (Hs, Ws))
    cf = _f32(conf, (Hs, Ws))
    u = _f32(uniforms, (h, w))
    if ws is None:
        ws = workspace(H, W, dev)
    strides, rptr, eptr = None, None, None
    if render is not None:
        if render.dtype != torch.float32 or tuple(render.shape) != (3, H, W) or render.device != dev:
            raise ValueError(f"render must be a float32 [3,{H},{W}] tensor on {dev}")
        strides = (C.c_longlong * 3)(*render.stride())
        rptr = C.c_void_p(render.data_ptr())
        expo = _f32(exposure, (3, 4))
        eptr = _lib.ptr(expo)
    init_proba = torch.empty(h, w, dtype=torch.float32, device=dev)
    penalty = torch.empty(h, w, dtype=torch.float32, device=dev)
    flags = torch.empty(h, w, dtype=torch.uint8, device=dev)
    n_rows = torch.empty(1, dtype=torch.int32, device=dev)
    qm = qmin.reshape(-1)[-1:].contiguous()
    with torch.cuda.device(dev):
        _lib.call("adb_densify_sample", H, W, int(lod), _lib.ptr(img), rptr, strides, eptr, Hs, Ws, _lib.ptr(depth), _lib.ptr(cf),
                  _lib.ptr(u), _lib.ptr(qm), float(init_proba_scaler), float(gs_add_ratio), _lib.ptr(init_proba),
                  _lib.ptr(penalty), _lib.ptr(flags), _lib.ptr(n_rows), _lib.ptr(ws),
                  ws.numel(), _lib.stream())
        n = int(n_rows.item())
        cam = torch.cat([_f32(R, (9,)), _f32(t, (3,)), _f32(approx_centre, (3,))]).to(dev)
        rows = dict(xyz=torch.empty(n, 3, device=dev), f_dc=torch.empty(n, 1, 3, device=dev),
                    scaling=torch.empty(n, 3, device=dev), opacity=torch.empty(n, 1, device=dev),
                    d_max=torch.empty(n, 1, device=dev))
        if n > 0:
            _lib.call("adb_densify_emit", H, W, int(lod), _lib.ptr(img), Hs, Ws, _lib.ptr(depth), _lib.ptr(cf),
                      _lib.ptr(init_proba), _lib.ptr(flags), _lib.ptr(cam), float(f), _lib.ptr(rows["xyz"]),
                      _lib.ptr(rows["f_dc"]), _lib.ptr(rows["scaling"]), _lib.ptr(rows["opacity"]), _lib.ptr(rows["d_max"]),
                      _lib.ptr(ws), ws.numel(), _lib.stream())
    return dict(init_proba=init_proba, penalty=penalty, flags=flags, n=n, **rows)


def _view_matrix(R: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
    """``keyframe.get_Rt()``: the world-to-camera 4x4."""
    V = torch.eye(4, dtype=torch.float32, device=R.device)
    V[:3, :3] = R.detach().float()
    V[:3, 3] = t.detach().float().reshape(3)
    return V


@torch.no_grad()
def add_new_gaussians(optimizer, frame: dict, *, keyframe_id: int, cam_centres: torch.Tensor, width: int, height: int,
                      f: float, tanfovx: float, tanfovy: float, init_proba_scaler: float, gs_add_ratio: float,
                      voxel_size: float, visible_threshold: float, sh_degree: int = 3, eps2d: float = 0.01,
                      local_feat_dim: int, global_feat_dim: int, cov_mlp=None, uniforms=None) -> dict:
    """``SceneModel.add_new_gaussians(keyframe_id)`` on ``optimizer.params`` (a ``SparseGaussianAdam`` over the reference's
    ``gaussian_params`` keys: raw ``opacity`` / ``scaling``, as the reference stores them).

    ``frame``: ``image`` [3,H,W], ``point_map`` [1,3,Hs,Ws], ``conf`` [1,1,Hs,Ws] (``mono_depth_conf``), ``R`` [3,3], ``t`` [3]
    (``get_R()`` / ``get_t()``), ``approx_centre`` [3], ``exposure`` [3,4], ``is_test``.  ``keyframe_id`` is the index the new
    rows carry (the reference's resolved index), ``cam_centres`` [K,3] the centres of every key frame for
    ``weed_out_gaussians``, ``cov_mlp`` the optional dict(W1, b1, W2, b2) of ``mlp_cov``.  ``uniforms``: optional list of the
    four [H/lod, W/lod] draws; by default they are drawn like the reference's ``torch.rand_like``, in LoD order.

    Returns stats: ``renders`` (renders made), ``rows`` and ``new_voxels`` (per LoD)."""
    stats = dict(renders=0, rows=[], new_voxels=[])
    if frame["is_test"]:
        return stats
    image = frame["image"]
    _lib.require_cuda(image)
    dev = image.device
    if width // LODS[-1] < 2 or height // LODS[-1] < 2:
        raise ValueError("add_new_gaussians needs an image of at least 16x16 (the LoD-8 image must be at least 2x2)")
    if tuple(image.shape[-2:]) != (height, width):
        raise ValueError(f"image is {tuple(image.shape[-2:])}, expected ({height}, {width})")
    P = optimizer.params
    val = lambda k: P[k]["val"]   # noqa: E731
    N = int(val("xyz").shape[0])
    ws = workspace(height, width, dev)
    qmin = depth_quantile(frame["point_map"], ws)
    valid_gs_mask = (prune_mask(val("xyz"), val("opacity"), val("scaling"), frame["approx_centre"], f, width) if N > 0
                     else torch.ones(0, dtype=torch.bool, device=dev))
    if N > 0:
        scene = dict(xyz=val("xyz").detach(), opacity=torch.sigmoid(val("opacity").detach()), f_dc=val("f_dc").detach(),
                     f_rest=val("f_rest").detach(), scaling=torch.exp(val("scaling").detach()),
                     rotation=val("rotation").detach(), d_max=val("d_max").detach())
        view = _view_matrix(frame["R"], frame["t"])
    render, render_cls = None, None
    ext = {k: [] for k in EXT_KEYS}
    n_voxels = 0
    for i, lod in enumerate(LODS):
        h, w = height // lod, width // lod
        if N > 0:
            cls = val("cls_id")
            # reuse is exact when the classes the render read are unchanged; update_voxel has just synchronised the stream,
            # so this comparison's one-byte read does not stall it
            stale = render is None or (cov_mlp is not None and not torch.equal(cls, render_cls))
            if stale:
                mlp = {} if cov_mlp is None else dict(cov_mlp=cov_mlp, local_feat=val("local_feat").detach(),
                                                      global_feat=val("global_feat").detach(), cls_id=cls)
                render = render_lod(width, height, view, tanfovx=tanfovx, tanfovy=tanfovy, sh_degree=sh_degree, eps2d=eps2d,
                                    **scene, **mlp)["render"]
                render_cls = cls.clone()
                stats["renders"] += 1
        u = uniforms[i] if uniforms is not None else torch.rand(h, w, device=dev)
        rows = sample_lod(image, render if N > 0 else None, frame["point_map"], frame["conf"], frame["R"], frame["t"],
                          frame["approx_centre"], frame["exposure"], lod=lod, f=f, init_proba_scaler=init_proba_scaler,
                          gs_add_ratio=gs_add_ratio, uniforms=u, qmin=qmin, ws=ws)
        n = rows["n"]
        if N > 0:
            upd, new_cls, nv = update_voxel(rows["xyz"], val("xyz"), val("cls_id"), voxel_size)
            P["cls_id"]["val"] = upd
        else:
            new_cls, nv = update_voxel(rows["xyz"], val("xyz"), val("cls_id"), voxel_size)
        n_voxels += nv
        stats["rows"].append(n)
        stats["new_voxels"].append(nv)
        ext["id"].append(torch.full((n, 1), int(keyframe_id), dtype=torch.long, device=dev))
        ext["cls_id"].append(new_cls.reshape(n, 1))
        for k in ("d_max", "xyz", "f_dc", "opacity", "scaling"):
            ext[k].append(rows[k])
    L = sum(stats["rows"])
    n_sh = (sh_degree + 1) ** 2 - 1
    cat = {k: torch.cat(ext[k], 0) for k in ("id", "cls_id", "d_max", "xyz", "f_dc", "opacity", "scaling")}
    rotation = torch.zeros(L, 4, device=dev)
    rotation[:, 0] = 1
    cat.update(f_rest=torch.zeros(L, n_sh, 3, device=dev), rotation=rotation,
               local_feat=torch.zeros(L, local_feat_dim, device=dev),
               global_feat=torch.zeros(n_voxels, global_feat_dim, device=dev))
    optimizer.add_and_prune(cat, valid_gs_mask)
    weed = weed_out_mask(val("xyz"), val("d_max"), cam_centres, visible_threshold)
    optimizer.add_and_prune({k: P[k]["val"][:0].detach() for k in EXT_KEYS if k in P}, weed)
    return stats

"""Host-side mirror of the key-frame hand-off from the Backend to the mapper: ``Backend.prepare_for_mapper`` /
``compute_dense_point`` (VSLAM/Backend.py:117-193), the mapper-side lines of run_system.py:161-192 and the training branch of
``Keyframe.__init__`` (Reconstruct/scene/keyframe.py:64-127).

What runs differently from the reference (csrc/keyframe.cu):
  * ``dense_point`` is one launch over the SLAM pixels instead of ~30 torch and pypose kernels; ``mapper_keyframe`` is one
    launch over the mapper image for the 1/z prior, its bilinear resize, both average-pool pyramids and the pose.  Neither
    syncs the host or allocates inside the library, so both can be captured in a CUDA graph;
  * the outputs stay on the device they were made on: the reference's blocking ``.cpu()`` copies of ``densePoint``,
    ``T_WC`` and ``T_CkC`` and their return to the mapper's device are the caller's to make, only when the Backend and the
    mapper use different GPUs;
  * the reference scatters every matched point back to its key-frame pixel; each scattered value is the same function of
    the same input as the value already there, so each point is computed once;
  * an ``idx_k2l`` entry outside ``[0, HW)`` (the reference faults in the gather or raises in ``reshape``) is not read: that
    pixel is NaN in all four channels and counted in ``n_bad``, a device int32;
  * ``idepth_conf_pyr`` is not built: nothing reads it.
Quirks kept: channel 3 of the dense point is the confidence in the LAST key frame's pixel order (the reference returns
``conf_valid[valid_range]``, not the ``conf_valid_sorted`` it also builds); the points use ``SE3(T_WC[:7]).Inv()`` without
``quat2unit``; the first key frame's channel 3 is ``C / N > 1.5`` with ``N`` divided as a Python int (multiplication by its
fp32 reciprocal); the mapper pose does apply ``quat2unit``."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import i32, vp
from .optimizers import BaseAdam

_lib.register("adb_kf_dense_point", [i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp])
_lib.register("adb_kf_pyramid_floats", [i32, i32, i32, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)])
_lib.register("adb_kf_mapper_inputs", [i32, i32, i32, i32, i32, vp, C.POINTER(C.c_longlong), vp, vp, vp, vp, vp, vp, vp, vp,
                                       vp])

BETAS = (0.8, 0.99)
TEST_LR_POSES = 1e-4


def _f32(name: str, t: torch.Tensor, numel: int, dev) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32:
        raise ValueError(f"{name} must be a float32 tensor")
    if t.numel() != numel:
        raise ValueError(f"{name} must have {numel} elements, got {tuple(t.shape)}")
    if t.device != dev:
        raise ValueError(f"{name} is on {t.device}, expected {dev}")
    return t.detach().reshape(-1).contiguous()


@torch.no_grad()
def dense_point(X_canon: torch.Tensor, C: torch.Tensor, N, T_WC: torch.Tensor, K: torch.Tensor, *,
                last_T_WC: torch.Tensor | None = None, idx_k2l: torch.Tensor | None = None):
    """``Backend.prepare_for_mapper``'s ``densePoint`` and ``T_CkC`` for one key frame.

    ``X_canon [Hs,Ws,3]`` (the key frame's canonical points, reshaped to the image), ``C`` its ``Hs*Ws`` summed
    confidences, ``N`` the number of fused frames (the tracker's int32 [1] device tensor, or an int), ``T_WC`` the key
    frame's Sim(3) pose ``[8]`` (``tx ty tz qx qy qz qw s``), ``K [3,3]`` the SLAM intrinsics.  ``last_T_WC [8]`` and
    ``idx_k2l`` (``Hs*Ws`` int64, ``mast3r_match_asymmetric(keyframe, last_keyframe)``'s index) for every key frame but the
    first.  ``C`` and ``N`` are read for the first key frame only.

    Returns ``(densePoint [Hs,Ws,4], T_CkC [8] or None, n_bad)``, with ``n_bad`` a device int32 [1] counting the pixels
    whose ``idx_k2l`` is outside ``[0, Hs*Ws)`` (NaN in all four channels)."""
    if not isinstance(X_canon, torch.Tensor) or X_canon.dim() != 3 or X_canon.shape[2] != 3:
        raise ValueError("X_canon must be an [Hs,Ws,3] tensor")
    H, W = int(X_canon.shape[0]), int(X_canon.shape[1])
    HW = H * W
    dev = X_canon.device
    X = _f32("X_canon", X_canon, 3 * HW, dev)
    k = _f32("K", K, 9, dev)
    first = last_T_WC is None
    if first != (idx_k2l is None):
        raise ValueError("last_T_WC and idx_k2l go together: both for a key frame after the first, neither for the first")
    if first:
        c = _f32("C", C, HW, dev)
        if isinstance(N, torch.Tensor):
            if N.dtype != torch.int32 or N.numel() != 1 or N.device != dev:
                raise ValueError(f"N must be an int32 [1] tensor on {dev} (or an int)")
            n = N.reshape(1).contiguous()
        else:
            n = torch.tensor([int(N)], dtype=torch.int32, device=dev)
        twk = twl = idx = None
    else:
        twk = _f32("T_WC", T_WC, 8, dev)
        twl = _f32("last_T_WC", last_T_WC, 8, dev)
        if not isinstance(idx_k2l, torch.Tensor) or idx_k2l.dtype != torch.int64 or idx_k2l.numel() != HW:
            raise ValueError(f"idx_k2l must be an int64 tensor of {HW} elements")
        if idx_k2l.device != dev:
            raise ValueError(f"idx_k2l is on {idx_k2l.device}, expected {dev}")
        idx = idx_k2l.reshape(-1).contiguous()
        c = n = None
    _lib.require_cuda(X_canon)
    out = torch.empty(H, W, 4, dtype=torch.float32, device=dev)
    T_CkC = None if first else torch.empty(8, dtype=torch.float32, device=dev)
    n_bad = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.call("adb_kf_dense_point", H, W, _lib.ptr(X), _lib.ptr(c), _lib.ptr(n), _lib.ptr(twk), _lib.ptr(twl),
                  _lib.ptr(idx), _lib.ptr(k), _lib.ptr(out), _lib.ptr(T_CkC), _lib.ptr(n_bad), _lib.stream())
    return out, T_CkC, n_bad


def level_sizes(height: int, width: int, pyr_levels: int) -> list:
    """``(h, w)`` of each pyramid level: ``avg_pool2d(., 2)`` floors at every level."""
    return [(height >> l, width >> l) for l in range(pyr_levels)]


@torch.no_grad()
def mapper_keyframe(image: torch.Tensor, densePoint: torch.Tensor, T_WC: torch.Tensor, *, pyr_levels: int, index: int,
                    is_test: bool, lr_poses: float, lr_exposure: float) -> dict:
    """The mapper key frame that run_system.py builds from the Backend's message (``Keyframe(...)`` with no ``prev_kf``).

    ``image [3,H,W]`` float32 (``to_map``'s ``permute(2,0,1)`` of an HWC array is fine: it is read through its strides),
    ``densePoint [Hs,Ws,4]`` as ``dense_point`` returns it, ``T_WC [8]`` the key frame's Sim(3) pose, ``index`` the mapper
    key-frame index (pose lr 0 for index 0), ``is_test`` (pose lr 1e-4 and no exposure group).

    Returns a dict usable as ``densify.add_new_gaussians(frame=...)``: ``image`` (= ``image_pyr[0]``), ``image_pyr`` /
    ``idepth_pyr`` (lists of ``pyr_levels`` tensors ``[3,h,w]`` / ``[1,h,w]``; the mapper trains at the last level),
    ``point_map [1,3,Hs,Ws]`` and ``conf [1,1,Hs,Ws]`` (views of ``densePoint``), ``rW2C [3,2]`` / ``tW2C [3]`` /
    ``exposure [3,4]`` (``nn.Parameter``), ``R [3,3]`` (``sixD2mtx(rW2C)``), ``t`` (= ``tW2C``), ``approx_centre [3]``,
    ``optimizer`` (a ``BaseAdam`` with betas (0.8, 0.99)) and ``is_test``."""
    if not isinstance(image, torch.Tensor) or image.dim() != 3 or image.shape[0] != 3 or image.dtype != torch.float32:
        raise ValueError("image must be a float32 [3,H,W] tensor")
    if not isinstance(densePoint, torch.Tensor) or densePoint.dim() != 3 or densePoint.shape[2] != 4 \
            or densePoint.dtype != torch.float32:
        raise ValueError("densePoint must be a float32 [Hs,Ws,4] tensor")
    dev = densePoint.device
    if image.device != dev:
        raise ValueError(f"image is on {image.device}, densePoint on {dev}")
    pose = _f32("T_WC", T_WC, 8, dev)
    H, W = int(image.shape[1]), int(image.shape[2])
    Hs, Ws = int(densePoint.shape[0]), int(densePoint.shape[1])
    L = int(pyr_levels)
    n_id, n_im = C.c_longlong(0), C.c_longlong(0)
    _lib.call("adb_kf_pyramid_floats", H, W, L, C.byref(n_id), C.byref(n_im))     # validates the sizes on the host
    _lib.require_cuda(densePoint)
    dp = densePoint.detach()
    if not dp.is_contiguous() or dp.data_ptr() % 16:     # one 16-byte row per pixel
        dp = dp.clone()
    id_buf = torch.empty(n_id.value, dtype=torch.float32, device=dev)
    im_buf = torch.empty(n_im.value, dtype=torch.float32, device=dev) if L > 1 else None
    rW2C = torch.empty(3, 2, dtype=torch.float32, device=dev)
    tW2C = torch.empty(3, dtype=torch.float32, device=dev)
    approx = torch.empty(3, dtype=torch.float32, device=dev)
    R = torch.empty(3, 3, dtype=torch.float32, device=dev)
    img = image.detach()
    strides = (C.c_longlong * 3)(*img.stride())
    with torch.cuda.device(dev):
        _lib.call("adb_kf_mapper_inputs", H, W, Hs, Ws, L, C.c_void_p(img.data_ptr()), strides, _lib.ptr(dp), _lib.ptr(pose),
                  _lib.ptr(id_buf), _lib.ptr(im_buf), _lib.ptr(rW2C), _lib.ptr(tW2C), _lib.ptr(approx), _lib.ptr(R),
                  _lib.stream())
    idepth_pyr, image_pyr = [], [image]
    o_id = o_im = 0
    for lvl, (h, w) in enumerate(level_sizes(H, W, L)):
        idepth_pyr.append(id_buf[o_id:o_id + h * w].view(1, h, w))
        o_id += h * w
        if lvl > 0:
            image_pyr.append(im_buf[o_im:o_im + 3 * h * w].view(3, h, w))
            o_im += 3 * h * w
    rW2C, tW2C = torch.nn.Parameter(rW2C), torch.nn.Parameter(tW2C)
    exposure = torch.nn.Parameter(torch.eye(3, 4, device=dev))
    lr = 0 if index == 0 else lr_poses
    if is_test:
        lr = TEST_LR_POSES
    params = {"rW2C": {"val": rW2C, "lr": lr}, "tW2C": {"val": tW2C, "lr": lr}}
    if not is_test:
        params["exposure"] = {"val": exposure, "lr": lr_exposure}
    return dict(image=image, image_pyr=image_pyr, idepth_pyr=idepth_pyr,
                point_map=densePoint[..., :3].permute(2, 0, 1)[None], conf=densePoint[..., 3][None, None],
                rW2C=rW2C, tW2C=tW2C, R=R, t=tW2C, approx_centre=approx, exposure=exposure,
                optimizer=BaseAdam(params, betas=BETAS), is_test=bool(is_test))

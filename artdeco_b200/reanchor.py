"""Host-side mirror of the map update that runs on every SLAM key frame once the Backend's global Gauss-Newton has moved its
Sim(3) key frames (run_system.py:194-227): every mapper key frame's pose is rebuilt from the Backend's table, and every
Gaussian moves rigidly with the key frame that created it (``SceneModel.rigid_transform_gs``, h3dgsv3.py:955-966, and
``update_gaussians``, Reconstruct/utils.py:28-60).

What runs differently from the reference's Python loop over the K mapper key frames (pypose on [1,8] tensors and three
``torch.linalg.inv`` host syncs per frame) and its whole-map ``update_gaussians`` (two gathered [N,4,4] tables, N 4x4
inverses, kornia's four-branch conversion on every row) (csrc/reanchor.cu):
  * ``keyframe_poses`` is one launch over K; nothing is read on the host;
  * ``rigid_transform_gs`` inverts the K distinct ``old_c2w`` once (one launch over K) and moves every Gaussian in one
    streaming launch over N (36 B in, 28 B out per row).
Rows the reference would fault on (``last_keyframe_index`` or ``id`` out of range) or raise on (a singular ``old_c2w``) are
left unchanged and counted in ``n_bad``, a device int32 tensor."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import i32, i64, vp

_lib.register("adb_reanchor_workspace_bytes", [i32, C.POINTER(C.c_size_t)])
_lib.register("adb_reanchor_keyframes", [i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp])
_lib.register("adb_reanchor_gaussians", [i64, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_size_t, vp])


def _check(name: str, t: torch.Tensor, shape: tuple, dtypes: tuple, device) -> None:
    if not isinstance(t, torch.Tensor):
        raise ValueError(f"{name} must be a tensor")
    if t.dtype not in dtypes:
        raise ValueError(f"{name} must be {' or '.join(map(str, dtypes))}, got {t.dtype}")
    if t.dim() != len(shape) or any(s is not None and int(a) != s for a, s in zip(t.shape, shape)):
        raise ValueError(f"{name} must have shape {tuple('*' if s is None else s for s in shape)}, got {tuple(t.shape)}")
    if device is not None and t.device != device:
        raise ValueError(f"{name} is on {t.device}, expected {device}")


def keyframe_poses(rW2C: torch.Tensor, tW2C: torch.Tensor, slam_T_WC: torch.Tensor, last_keyframe_index: torch.Tensor,
                   is_slam_keyframe: torch.Tensor, T_CkCf: torch.Tensor):
    """The pose loop of run_system.py:198-226 for all K mapper key frames at once.

    ``rW2C [K,3,2]`` / ``tW2C [K,3]``: the stacked 6-D rotations and translations of the mapper key frames (float32,
    contiguous), updated IN PLACE as ``set_Rt`` does.  ``slam_T_WC [K_slam,8]``: the Backend's Sim(3) poses (pypose layout
    ``tx ty tz qx qy qz qw s``).  ``last_keyframe_index [K]`` int64, ``is_slam_keyframe [K]`` bool or uint8, ``T_CkCf [K,8]``
    (read on non-SLAM rows only).

    Returns ``(old_c2ws [K,4,4], new_c2ws [K,4,4], cam_centres [K,3], approx_centres [K,3], n_bad)``: the camera-to-world
    matrices before and after, ``inverse(get_Rt().T)[3,:3]`` after ``set_Rt``, ``set_Rt``'s ``approx_centre``, and a device
    int32 [1] counting rows whose ``last_keyframe_index`` is outside ``[0, K_slam)`` (those keep their pose)."""
    if not isinstance(rW2C, torch.Tensor) or rW2C.dim() != 3:
        raise ValueError("rW2C must be a [K,3,2] tensor")
    K = int(rW2C.shape[0])
    dev = rW2C.device
    f32 = (torch.float32,)
    _check("rW2C", rW2C, (K, 3, 2), f32, dev)
    _check("tW2C", tW2C, (K, 3), f32, dev)
    _check("slam_T_WC", slam_T_WC, (None, 8), f32, dev)
    _check("last_keyframe_index", last_keyframe_index, (K,), (torch.int64,), dev)
    _check("is_slam_keyframe", is_slam_keyframe, (K,), (torch.bool, torch.uint8), dev)
    _check("T_CkCf", T_CkCf, (K, 8), f32, dev)
    if not (rW2C.is_contiguous() and tW2C.is_contiguous()):
        raise ValueError("rW2C and tW2C are updated in place and must be contiguous")
    _lib.require_cuda(rW2C)
    slam = slam_T_WC.detach().contiguous()
    idx = last_keyframe_index.contiguous()
    is_slam = is_slam_keyframe.contiguous().view(torch.uint8)
    rel = T_CkCf.detach().contiguous()
    old_c2ws = torch.empty(K, 4, 4, dtype=torch.float32, device=dev)
    new_c2ws = torch.empty_like(old_c2ws)
    cam_centres = torch.empty(K, 3, dtype=torch.float32, device=dev)
    approx_centres = torch.empty_like(cam_centres)
    n_bad = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.call("adb_reanchor_keyframes", K, int(slam.shape[0]), _lib.ptr(slam), _lib.ptr(idx), _lib.ptr(is_slam),
                  _lib.ptr(rel), C.c_void_p(rW2C.data_ptr()), C.c_void_p(tW2C.data_ptr()), _lib.ptr(old_c2ws),
                  _lib.ptr(new_c2ws), _lib.ptr(cam_centres), _lib.ptr(approx_centres), _lib.ptr(n_bad), _lib.stream())
    return old_c2ws, new_c2ws, cam_centres, approx_centres, n_bad


@torch.no_grad()
def rigid_transform_gs(params: dict, old_c2ws: torch.Tensor, new_c2ws: torch.Tensor, cam_centres: torch.Tensor) -> torch.Tensor:
    """``SceneModel.rigid_transform_gs(old_c2ws, new_c2ws, cam_centres)`` with the scene's ``gaussian_params`` dict
    (``SparseGaussianAdam.params``) in place of ``self``.

    ``params["id"]["val"] [N,1]`` int64 is each Gaussian's key frame, ``params["xyz"]["val"] [N,3]`` and
    ``params["rotation"]["val"] [N,4]`` (wxyz, not normalised) float32; ``old_c2ws`` / ``new_c2ws [K,4,4]`` and
    ``cam_centres [K,3]`` as ``keyframe_poses`` returns them.  As in the reference, ``xyz`` and ``rotation`` are REPLACED by new
    tensors made under ``no_grad``: they stop requiring grad, so ``SparseGaussianAdam.step`` skips them until the next
    ``add_and_prune``.  Moments, learning rates and SH coefficients are untouched.  The reference also stores
    ``cam_centres`` on the scene (``self.cam_centres``, the cameras of ``weed_out_gaussians``); that tensor stays with the
    caller, who passes it to ``weed_out_mask``.

    Returns ``n_bad``, a device int32 [1]: rows whose id is outside ``[0, K)`` or whose ``old_c2w`` is singular, copied
    unchanged (the reference would fault or raise)."""
    for key in ("id", "xyz", "rotation"):
        if key not in params or "val" not in params[key]:
            raise ValueError(f"params has no {key!r} value")
    xyz, rot, ids = params["xyz"]["val"], params["rotation"]["val"], params["id"]["val"]
    if not isinstance(xyz, torch.Tensor) or xyz.dim() != 2:
        raise ValueError("params['xyz']['val'] must be an [N,3] tensor")
    N = int(xyz.shape[0])
    dev = xyz.device
    if not isinstance(old_c2ws, torch.Tensor) or old_c2ws.dim() != 3:
        raise ValueError("old_c2ws must be a [K,4,4] tensor")
    K = int(old_c2ws.shape[0])
    f32 = (torch.float32,)
    _check("xyz", xyz, (N, 3), f32, dev)
    _check("rotation", rot, (N, 4), f32, dev)
    _check("id", ids, (N, 1), (torch.int64,), dev)
    _check("old_c2ws", old_c2ws, (K, 4, 4), f32, dev)
    _check("new_c2ws", new_c2ws, (K, 4, 4), f32, dev)
    _check("cam_centres", cam_centres, (K, 3), f32, dev)
    _lib.require_cuda(xyz)
    new_xyz = torch.empty(N, 3, dtype=torch.float32, device=dev)
    new_rot = torch.empty(N, 4, dtype=torch.float32, device=dev)
    n_bad = torch.zeros(1, dtype=torch.int32, device=dev)
    if N > 0:
        r = rot.detach().contiguous()
        if r.data_ptr() % 16:                      # the kernel reads and writes rows as 16-byte vectors
            r = r.clone()
        nb = C.c_size_t(0)
        _lib.call("adb_reanchor_workspace_bytes", K, C.byref(nb))
        ws = torch.empty(max(nb.value, 16), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _lib.call("adb_reanchor_gaussians", N, K, _lib.ptr(ids.contiguous()), _lib.ptr(xyz.detach().contiguous()),
                      _lib.ptr(r), _lib.ptr(old_c2ws.contiguous()),
                      _lib.ptr(new_c2ws.contiguous()), _lib.ptr(new_xyz), _lib.ptr(new_rot), _lib.ptr(n_bad), _lib.ptr(ws),
                      ws.numel(), _lib.stream())
    params["xyz"]["val"] = new_xyz
    params["rotation"]["val"] = new_rot
    return n_bad

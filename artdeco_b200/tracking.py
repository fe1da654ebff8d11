"""The Frontend's per-frame pose tracker: ``CameraTracker.track`` after matching and ``CameraTracker.opt_pose_calib_sim3``
(VSLAM/CameraTracker.py:53-155, :296-396), calibrated Sim(3) only.

``track`` takes what ``mast3r.wrappers.mast3r_match_asymmetric`` returns plus the key frame's ``X_canon`` / ``C`` / ``N`` and
runs steps 2-7 of the reference method in three C-ABI calls (csrc/track.cu): preparation (masks, ray-constrained points,
box-filter covariance, ``meas_k``, the match-fraction test), the Gauss-Newton solve (covariance filter, Huber weights, 7x7
Cholesky, ``Exp(tau) T``, ``check_convergence``) and the finish (point fusion, both key-frame tests).  The reference syncs the
host in every iteration (``cost.item()``) and twice more in the key-frame tests; here the whole frame is one launch sequence
and ``track`` reads the host once, at the end, for ``lost``, the two key-frame flags and ``last_dist``.

Poses are float32 ``[8]`` tensors ``(t, q xyzw, s)``, pypose's Sim3 storage.  ``optimize_focal`` is not supported."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import torch

from . import _lib
from ._lib import f32, i32, vp

f64 = C.c_double
_lib.register("adb_track_workspace_bytes", [i32, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)])
_lib.register("adb_track_prepare", [i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, f32, f32, f32, f32, vp, vp, vp, vp, vp,
                                    vp, vp, vp, vp, C.c_size_t, vp])
_lib.register("adb_track_solve", [i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, f32, f32, f32, f32, f64,
                                  f32, vp, vp, vp, vp, C.c_size_t, vp])
_lib.register("adb_track_finish", [i32, i32, vp, vp, vp, vp, vp, vp, vp, i32, f64, f32, f64, f64, vp, vp, C.c_size_t, vp])

LOST_NONE, LOST_MATCHES, LOST_CHOLESKY, LOST_ZERO_COST = 0, 1, 2, 3


class TrackState(C.Structure):
    """Host view of ``adb_track_state`` (include/artdeco_b200.h)."""
    _fields_ = [("lost", C.c_int32), ("iters", C.c_int32), ("converged", C.c_int32), ("done", C.c_int32),
                ("n_valid_opt", C.c_int32), ("n_valid_kf", C.c_int32), ("n_unique", C.c_int32),
                ("is_keyframe", C.c_int32), ("is_keyframe_map", C.c_int32), ("tau_norm", C.c_float),
                ("cov_threshold", C.c_float), ("dist_quantile", C.c_float), ("cost", C.c_double),
                ("prev_cost", C.c_double), ("last_dist", C.c_double), ("H", C.c_double * 49), ("g", C.c_double * 7),
                ("T_CkCf", C.c_float * 8), ("T_WCk", C.c_float * 8)]

    @classmethod
    def read(cls, state: torch.Tensor) -> "TrackState":
        """Copies the device state block to the host (one sync)."""
        return cls.from_buffer_copy(state.cpu().numpy().tobytes())


@dataclass
class Workspace:
    ws: torch.Tensor
    state: torch.Tensor


def workspace(n: int, device) -> Workspace:
    ws_b, st_b = C.c_size_t(0), C.c_size_t(0)
    _lib.call("adb_track_workspace_bytes", int(n), C.byref(ws_b), C.byref(st_b))
    if st_b.value != C.sizeof(TrackState):
        raise _lib.ArtdecoB200Error("adb_track_state layout differs from tracking.TrackState")
    return Workspace(torch.empty(ws_b.value, dtype=torch.uint8, device=device),
                     torch.zeros(st_b.value, dtype=torch.uint8, device=device))


def _f32(t, shape):
    t = t.detach()
    if t.dtype != torch.float32:
        raise ValueError(f"expected float32, got {t.dtype}")
    return t.reshape(shape).contiguous()


def _u8(mask, n):
    return mask.reshape(n).to(torch.bool).contiguous().view(torch.uint8)


def _pose(T):
    T = T.detach().reshape(-1)
    if T.numel() != 8 or T.dtype != torch.float32:
        raise ValueError("poses are float32 [8] tensors (t, q xyzw, s)")
    return T.contiguous()


def _check_cfg(cfg, optimize_focal):
    if optimize_focal:
        raise NotImplementedError("optimize_focal=True is not supported (its focal-length Jacobian column is not built)")


def prepare(idx_f2k, valid_match_k, Xff, Cff, Qff, Qkf, kf_X, kf_C, kf_N, K, img_size, cfg, ws: Workspace):
    """Steps 2-5 of ``track`` (:65-118) and ``get_points_poses`` (:189-219).  Returns a dict with the key-frame-order
    tensors ``Xf [N,3]``, ``Xf_cov [N,3]`` (the covariance diagonal), ``Qk [N]``, ``meas_k [N,3]`` and the bool masks
    ``valid_meas_k``, ``valid_opt``, ``valid_kf`` [N]; the counts and the match-fraction verdict stay in ``ws.state``."""
    H, W = int(img_size[0]), int(img_size[1])
    n = H * W
    dev = Xff.device
    _lib.require_cuda(Xff)
    if not (kf_N.dtype == torch.int32 and kf_N.numel() == 1 and kf_N.is_cuda):
        raise ValueError("kf_N must be a one-element int32 CUDA tensor")
    out = dict(Xf=torch.empty(n, 3, device=dev), Xf_cov=torch.empty(n, 3, device=dev), Qk=torch.empty(n, device=dev),
               meas_k=torch.empty(n, 3, device=dev), valid_meas_k=torch.empty(n, dtype=torch.bool, device=dev),
               valid_opt=torch.empty(n, dtype=torch.bool, device=dev), valid_kf=torch.empty(n, dtype=torch.bool, device=dev))
    idx = idx_f2k.reshape(n).to(torch.int64).contiguous()
    Kd = _f32(K, (3, 3))
    with torch.cuda.device(dev):
        _lib.call("adb_track_prepare", H, W, _lib.ptr(Kd), _lib.ptr(idx), _lib.ptr(_u8(valid_match_k, n)),
                  _lib.ptr(_f32(Xff, (n, 3))), _lib.ptr(_f32(Cff, (n,))), _lib.ptr(_f32(Qff, (n,))), _lib.ptr(_f32(Qkf, (n,))),
                  _lib.ptr(_f32(kf_X, (n, 3))), _lib.ptr(_f32(kf_C, (n,))), _lib.ptr(kf_N), float(cfg["C_conf"]),
                  float(cfg["Q_conf"]), float(cfg["depth_eps"]), float(cfg["min_match_frac"]), _lib.ptr(out["Xf"]),
                  _lib.ptr(out["Xf_cov"]), _lib.ptr(out["Qk"]), _lib.ptr(out["meas_k"]),
                  _lib.ptr(out["valid_meas_k"].view(torch.uint8)), _lib.ptr(out["valid_opt"].view(torch.uint8)),
                  _lib.ptr(out["valid_kf"].view(torch.uint8)), _lib.ptr(ws.state), _lib.ptr(ws.ws), ws.ws.numel(),
                  _lib.stream())
    return out


def _solve(Xf, Xf_cov, T_WCf, T_WCk, Qk, valid, meas_k, valid_meas_k, img_size, K, cfg, covariance_filter, ws: Workspace):
    H, W = int(img_size[0]), int(img_size[1])
    n = int(Xf.shape[0])
    dev = Xf.device
    cov = Xf_cov.detach()
    if cov.dim() == 3:                                  # the reference's [N,3,3]; only its diagonal is ever non-zero
        cov = cov.diagonal(dim1=-2, dim2=-1)
    T_WCf_out = _pose(T_WCf).clone()
    T_CkCf = torch.empty(8, dtype=torch.float32, device=dev)
    Kd = _f32(K, (3, 3))
    with torch.cuda.device(dev):
        _lib.call("adb_track_solve", n, H, W, _lib.ptr(Kd), _lib.ptr(_f32(Xf, (n, 3))), _lib.ptr(_f32(cov, (n, 3))),
                  _lib.ptr(_f32(Qk, (n,))), _lib.ptr(_u8(valid, n)), _lib.ptr(_f32(meas_k, (n, 3))),
                  _lib.ptr(_u8(valid_meas_k, n)), _lib.ptr(_pose(T_WCf)), _lib.ptr(_pose(T_WCk)), int(cfg["max_iters"]),
                  int(bool(covariance_filter)), int(cfg["pixel_border"]), float(cfg["depth_eps"]), float(cfg["sigma_pixel"]),
                  float(cfg["sigma_depth"]), float(cfg["huber"]), float(cfg["rel_error"]), float(cfg["delta_norm"]),
                  _lib.ptr(T_WCf_out), _lib.ptr(T_CkCf), _lib.ptr(ws.state), _lib.ptr(ws.ws), ws.ws.numel(), _lib.stream())
    return T_WCf_out, T_CkCf


def opt_pose_calib_sim3(Xf, Xf_cov, Xk, Xk_cov, T_WCf, T_WCk, Qk, valid, meas_k, valid_meas_k, idx_f2k, img_size, K, cfg,
                        covariance_filter, optimize_focal=False):
    """CameraTracker.opt_pose_calib_sim3 (:296-396) with the tracker's ``K``, its ``tracking`` config dict and its
    ``covariance_filter`` flag.  Returns ``(T_WCf, T_CkCf, state)``: ``T_WCf = quat2unit(T_WCk T_CkCf)`` and ``state`` the
    device ``adb_track_state`` block (``TrackState.read``).  Where the reference raises (non-positive Cholesky pivot, a zero
    previous cost) ``state.lost`` is set instead, ``T_WCf`` is a copy of the input and ``T_CkCf`` the starting relative
    pose.  ``Xk``, ``Xk_cov`` and ``idx_f2k`` are accepted for the reference's signature; the calibrated solve does not
    read them.  Nothing here syncs the host."""
    _check_cfg(cfg, optimize_focal)
    _lib.require_cuda(Xf)
    ws = workspace(int(Xf.shape[0]), Xf.device)
    T_WCf_out, T_CkCf = _solve(Xf, Xf_cov, T_WCf, T_WCk, Qk, valid, meas_k, valid_meas_k, img_size, K, cfg,
                               covariance_filter, ws)
    return T_WCf_out, T_CkCf, ws.state


def track(idx_f2k, valid_match_k, Xff, Cff, Qff, Xkf, Ckf, Qkf, kf_X, kf_C, kf_N, T_WCf, T_WCk, K, img_size, cfg,
          min_displacement, thres_keyframe, last_dist, covariance_filter=True, point_fusion_frontend=True,
          optimize_focal=False, ws: Workspace | None = None):
    """CameraTracker.track steps 2-7 (:65-155) from the outputs of ``mast3r_match_asymmetric``.

    ``kf_X [N,3]``, ``kf_C [N,1]`` (contiguous float32) and ``kf_N`` (int32 [1]) are the key frame's ``X_canon``, ``C`` and
    ``N``; point fusion updates them in place.  Returns ``(lost, is_keyframe, is_keyframe_map, T_WCf, T_CkCf, last_dist)``;
    on a lost frame ``T_WCf`` equals the input, the key frame is untouched and ``last_dist`` is unchanged.  The one host
    read is at the end, for the three flags and ``last_dist``."""
    _check_cfg(cfg, optimize_focal)
    _lib.require_cuda(Xff)
    H, W = int(img_size[0]), int(img_size[1])
    n = H * W
    if point_fusion_frontend:
        for name, t in (("kf_X", kf_X), ("kf_C", kf_C)):
            if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() != n * (3 if name == "kf_X" else 1):
                raise ValueError(f"{name} must be a contiguous float32 tensor of the key frame's {n} points (updated in place)")
    if ws is None:
        ws = workspace(n, Xff.device)
    prep = prepare(idx_f2k, valid_match_k, Xff, Cff, Qff, Qkf, kf_X, kf_C, kf_N, K, img_size, cfg, ws)
    T_WCf_out, T_CkCf = _solve(prep["Xf"], prep["Xf_cov"], T_WCf, T_WCk, prep["Qk"], prep["valid_opt"], prep["meas_k"],
                               prep["valid_meas_k"], img_size, K, cfg, covariance_filter, ws)
    idx = idx_f2k.reshape(n).to(torch.int64).contiguous()
    Xkf_c = _f32(Xkf, (n, 3)) if point_fusion_frontend else None
    Ckf_c = _f32(Ckf, (n,)) if point_fusion_frontend else None
    with torch.cuda.device(Xff.device):
        _lib.call("adb_track_finish", H, W, _lib.ptr(idx), _lib.ptr(prep["valid_opt"].view(torch.uint8)), _lib.ptr(Xkf_c),
                  _lib.ptr(Ckf_c), _lib.ptr(kf_X if point_fusion_frontend else None),
                  _lib.ptr(kf_C if point_fusion_frontend else None), _lib.ptr(kf_N if point_fusion_frontend else None),
                  int(bool(point_fusion_frontend)), float(cfg["match_frac_thresh"]), float(thres_keyframe),
                  float(min_displacement), float(last_dist), _lib.ptr(ws.state), _lib.ptr(ws.ws), ws.ws.numel(),
                  _lib.stream())
    st = TrackState.read(ws.state)
    if st.lost:
        return True, False, False, T_WCf_out, T_CkCf, last_dist
    return False, bool(st.is_keyframe), bool(st.is_keyframe_map), T_WCf_out, T_CkCf, st.last_dist

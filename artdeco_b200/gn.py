"""Host-side mirror of the reference's global Gauss-Newton entry points ``mast3r_slam_backends.gauss_newton_rays`` and
``gauss_newton_calib`` (VSLAM/backend/src/gn.cpp:32-82, gn_kernels.cu:1141-1229,1546-1637; called from
VSLAM/mast3r_slam/global_opt.py:158,208): same positional arguments, ``Twc`` ([K,8] = t, q xyzw, s) updated IN PLACE, returns
``[dx]`` (the last step, [K-1,7]) like the reference.

What runs differently (csrc/gn.cu): the per-edge normal-equation blocks use the Ji = -Jj structure (35 instead of 119 reduced
values), the system of the free poses is assembled dense in double ON THE DEVICE and solved by an in-kernel Cholesky — the
reference copies the blocks to the host every iteration, factorises with Eigen's SimplicialLLT and syncs again for the
termination test.  Here no iteration touches the host (the convergence flag lives on the device)."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import f32, i32, vp

_lib.register("adb_gn_workspace_bytes", [i32, i32, C.POINTER(C.c_size_t)])
_lib.register("adb_gauss_newton", [i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, f32, f32, f32, f32, f32,
                                   i32, f32, vp, vp, vp, C.c_size_t, vp])


def _solve(mode, Twc, Xs, Cs, K, ii, jj, idx_ii2jj, valid_match, Q, height, width, pixel_border, z_eps, sigma_a, sigma_b,
           C_thresh, Q_thresh, max_iter, delta_thresh, return_state=False, return_workspace=False):
    """Runs the solve.  Returns ``[dx]``, or a tuple that appends the device state [4] (``return_state``) and then the
    uint8 workspace (``return_workspace``) in which the last iteration leaves, in this order: H [D,D] f64 (its strict
    upper triangle still holds the assembled matrix, the lower triangle and the diagonal hold the Cholesky factor), b [D]
    f64 (the solution x, dx = -x), S [E,28] f32 (lower triangle, row-major) and v [E,7] f32; D = 7 (K-1)."""
    _lib.require_cuda(Twc)
    if jj.shape[0] != ii.shape[0]:
        raise ValueError("ii and jj must list the same edges")
    # gn_kernels.cu:160-171: unique sorted key-frame ids; edges address the pose table by their rank in it
    unique = torch.unique(torch.cat([ii, jj]), sorted=True)
    if unique.numel() > int(Xs.shape[0]):
        # a rank >= K would address a pose (and a pointmap) past the end of the tables
        raise ValueError(f"the edges name {unique.numel()} key frames but Twc has {int(Xs.shape[0])} rows")
    ii_pos = torch.searchsorted(unique, ii.contiguous()).long().contiguous()
    jj_pos = torch.searchsorted(unique, jj.contiguous()).long().contiguous()
    return solve_positions(mode, Twc, Xs, Cs, K, ii_pos, jj_pos, idx_ii2jj, valid_match, Q, height, width, pixel_border,
                           z_eps, sigma_a, sigma_b, C_thresh, Q_thresh, max_iter, delta_thresh, return_state,
                           return_workspace)


def solve_positions(mode, Twc, Xs, Cs, K, ii_pos, jj_pos, idx_ii2jj, valid_match, Q, height, width, pixel_border, z_eps,
                    sigma_a, sigma_b, C_thresh, Q_thresh, max_iter, delta_thresh, return_state=False,
                    return_workspace=False):
    """The solve with the edges given as positions in the pose table (int64 [E], each in ``[0, K)``, the caller's to
    guarantee): no ``unique`` and nothing that reads the device from the host, so a caller that keeps its edge list on
    the host (``factor_graph.FactorGraph``) runs the whole solve without a sync.  Same arguments and results as ``_solve``
    otherwise."""
    _lib.require_cuda(Twc)
    dev = Twc.device
    if Twc.dim() != 2 or Twc.shape[1] != 8 or Twc.dtype != torch.float32:
        raise ValueError("Twc must be a float32 [K,8] tensor (t, q xyzw, s)")
    Kp, n = int(Xs.shape[0]), int(Xs.shape[1])
    if Twc.shape[0] != Kp or Cs.shape[0] != Kp:
        raise ValueError("Twc, Xs and Cs must stack the same key frames")
    E = int(ii_pos.shape[0])
    if jj_pos.shape[0] != E:
        raise ValueError("ii and jj must list the same edges")
    for name, t in (("idx_ii2jj", idx_ii2jj), ("valid_match", valid_match), ("Q", Q)):
        if t.numel() != E * n:
            raise ValueError(f"{name} must hold E*n = {E * n} elements, got {t.numel()}")
    if mode == 1 and n != int(height) * int(width):
        raise ValueError(f"calib mode needs one point per pixel: n = {n} but height*width = {int(height) * int(width)}")
    ii_pos = ii_pos.long().contiguous()
    jj_pos = jj_pos.long().contiguous()
    poses = Twc if Twc.is_contiguous() else Twc.contiguous()
    Xc = Xs.detach().float().contiguous()
    Cc = Cs.detach().float().reshape(Kp, n).contiguous()
    idx = idx_ii2jj.long().reshape(E, n).contiguous()
    vm = valid_match.reshape(E, n).to(torch.bool).contiguous()
    Qc = Q.detach().float().reshape(E, n).contiguous()
    Kd = K.detach().float().contiguous() if K is not None else None
    dx = torch.zeros(max(Kp - 1, 0), 7, dtype=torch.float32, device=dev)
    state = torch.zeros(4, dtype=torch.int32, device=dev)
    nb = C.c_size_t(0)
    _lib.call("adb_gn_workspace_bytes", Kp, E, C.byref(nb))
    ws = torch.empty(max(nb.value, 16), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.call("adb_gauss_newton", mode, Kp, n, E, _lib.ptr(poses), _lib.ptr(Xc), _lib.ptr(Cc), _lib.ptr(Kd), _lib.ptr(ii_pos),
                  _lib.ptr(jj_pos), _lib.ptr(idx), _lib.ptr(vm), _lib.ptr(Qc), int(height), int(width), int(pixel_border),
                  float(z_eps), float(sigma_a), float(sigma_b), float(C_thresh), float(Q_thresh), int(max_iter),
                  float(delta_thresh), _lib.ptr(dx), _lib.ptr(state), _lib.ptr(ws), ws.numel(), _lib.stream())
    if poses is not Twc:
        Twc.copy_(poses)
    if not (return_state or return_workspace):
        return [dx]
    return ([dx],) + ((state,) if return_state else ()) + ((ws,) if return_workspace else ())


def gauss_newton_rays(Twc, Xs, Cs, ii, jj, idx_ii2jj, valid_match, Q, sigma_ray, sigma_dist, C_thresh, Q_thresh, max_iter,
                      delta_thresh):
    """gn.cpp:32-56 / gn_kernels.cu:1141-1229."""
    return _solve(0, Twc, Xs, Cs, None, ii, jj, idx_ii2jj, valid_match, Q, 0, 0, 0, 0.0, sigma_ray, sigma_dist, C_thresh,
                  Q_thresh, max_iter, delta_thresh)


def gauss_newton_calib(Twc, Xs, Cs, K, ii, jj, idx_ii2jj, valid_match, Q, height, width, pixel_border, z_eps, sigma_pixel,
                       sigma_depth, C_thresh, Q_thresh, max_iter, delta_thresh):
    """gn.cpp:58-82 / gn_kernels.cu:1546-1637."""
    return _solve(1, Twc, Xs, Cs, K, ii, jj, idx_ii2jj, valid_match, Q, height, width, pixel_border, z_eps, sigma_pixel,
                  sigma_depth, C_thresh, Q_thresh, max_iter, delta_thresh)

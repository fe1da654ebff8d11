"""TEST INFRASTRUCTURE ONLY.  The key-frame hand-off from the Backend to the mapper, restated op for op in PyTorch:
``Backend.prepare_for_mapper`` / ``compute_dense_point`` (VSLAM/Backend.py:117-193, with ``constrain_points_to_ray`` of
mast3r_slam/geometry.py), the mapper-side lines of run_system.py:161-192 and the training branch of ``Keyframe.__init__``
(Reconstruct/scene/keyframe.py:64-127).  Runs on the CPU or the device.

pypose is the ``track_ref`` stand-in on [8] tensors (an SE3 is an [8] tensor with s = 1).  The per-pixel arithmetic of
``compute_dense_point`` (the stand-in's Act, the K matmul and the residual norm) is written out in elementwise operations,
so every step is rounded once and in a fixed order on any device: the confidence 1 / (r - 2) turns one rounding of the
reprojected pixel (|u| ulp) into up to ~1e-4 of the result, so the order has to be pinned.  One addition to the reference:
a pixel whose ``idx_k2l`` is outside ``[0, HW)`` (the reference faults in the gather or raises in ``reshape``) is NaN in all
four channels.  tests/golden/make_keyframe_golden.py pins this module to the reference's own statements; parity of the
stand-in with pypose itself is unpinned (pypose is not vendored or installable)."""
import torch
import torch.nn.functional as F

from oracle import track_ref as pp
from oracle.gn_ref import quat_comp
from oracle.mapper_loss_ref import sixD2mtx


def SE3(x7):
    return torch.cat([x7, torch.ones(1, dtype=x7.dtype, device=x7.device)])


def cross(a, b):
    a0, a1, a2 = a.unbind(-1)
    b0, b1, b2 = b.unbind(-1)
    return torch.stack([a1 * b2 - a2 * b1, a2 * b0 - a0 * b2, a0 * b1 - a1 * b0], -1)


def act(T, X):
    """The stand-in's Sim3 Act s (q X) + t on X [N,3] (gn_ref.act_so3's formula), one rounding per operation."""
    q = T[3:7]
    qv = q[:3].expand(X.shape)
    uv = 2.0 * cross(qv, X)
    return (X + q[3] * uv + cross(qv, uv)) * T[7] + T[:3]


def inv(A):
    qi = A[3:7] * torch.tensor([-1.0, -1.0, -1.0, 1.0], dtype=A.dtype, device=A.device)
    si = 1.0 / A[7]
    return torch.cat([-si * act(torch.cat([A.new_zeros(3), qi, A.new_ones(1)]), A[None, :3])[0], qi, si.reshape(1)])


def mul(A, B):
    return torch.cat([act(A, B[None, :3])[0], quat_comp(A[3:7], B[3:7]), (A[7] * B[7]).reshape(1)])


def compute_dense_point(X_canon, T_WC, last_T_WC, idx_k2l, K, H, W, valid_pixel=3, scatter=True):
    """Backend.compute_dense_point: (points [H,W,3] in key-frame order, conf [H,W] in last-key-frame order, n_bad).
    ``scatter=False`` skips the reference's scatter of the matched points into the key-frame-order points."""
    idx = idx_k2l.reshape(-1)
    HW = H * W
    valid_range = (idx >= 0) & (idx < HW)
    safe = torch.where(valid_range, idx, torch.zeros_like(idx))
    Twk, Twl = T_WC.reshape(8), last_T_WC.reshape(8)
    Tlk = mul(inv(Twl), Twk)
    Xkk_calib = pp.constrain_points_to_ray(X_canon.reshape(HW, 3), H, W, K)
    Xkk_calib_match = Xkk_calib[safe]
    Xkl_calib_match = act(Tlk, Xkk_calib_match).reshape(H, W, 3)
    pkl = Xkl_calib_match / Xkl_calib_match[..., 2:]
    # (K @ pkl)[:2]: all three products of each row, summed left to right, so 0 * inf = NaN propagates as in the matmul
    p0, p1, p2 = pkl.unbind(-1)
    u = K[0, 0] * p0 + K[0, 1] * p1 + K[0, 2] * p2
    v = K[1, 0] * p0 + K[1, 1] * p1 + K[1, 2] * p2
    vk, uk = torch.meshgrid(torch.arange(H, device=X_canon.device), torch.arange(W, device=X_canon.device), indexing="ij")
    du, dv = u - uk, v - vk
    resi = torch.sqrt(du * du + dv * dv).reshape(-1)                  # torch.norm(pkl_es - pll, dim=-1)
    conf_valid = torch.where(resi < valid_pixel, 1., 1 / (resi - valid_pixel + 1))
    Xkw = act(Twk, Xkk_calib_match)
    Tkw_se3 = inv(SE3(Twk[:7]))
    Xkk_calib_match_map = act(Tkw_se3, Xkw)
    Xkk_map_sorted = act(Tkw_se3, act(Twk, Xkk_calib))
    if scatter:
        Xkk_map_sorted[idx[valid_range]] = Xkk_calib_match_map[valid_range]
    conf = conf_valid.clone()
    conf[~valid_range] = float("nan")
    Xkk_map_sorted[~valid_range] = float("nan")
    return Xkk_map_sorted.reshape(H, W, 3), conf.reshape(H, W), int((~valid_range).sum())


def prepare_for_mapper(X_canon, C, N, T_WC, K, H, W, last_T_WC=None, idx_k2l=None, scatter=True):
    """(densePoint [H,W,4], T_CkC [8] or None, n_bad).  ``C`` the summed confidences [HW,1], ``N`` a Python int."""
    if last_T_WC is None:
        point = pp.constrain_points_to_ray(X_canon.reshape(H * W, 3), H, W, K).reshape(H, W, 3)
        point_valid = (C.reshape(-1, 1) / int(N) > 1.5).squeeze(-1).reshape(H, W)
        T_CkC, n_bad = None, 0
    else:
        point, point_valid, n_bad = compute_dense_point(X_canon, T_WC, last_T_WC, idx_k2l, K, H, W, scatter=scatter)
        T_CkC = mul(inv(last_T_WC.reshape(8)), T_WC.reshape(8))
    return torch.cat([point, point_valid[..., None]], dim=-1), T_CkC, n_bad


def mapper_keyframe(image, densePoint, T_WC, pyr_levels):
    """run_system.py:169-173 and Keyframe.__init__ (training branch): a dict of image_pyr, idepth_pyr, point_map, conf,
    rW2C, tW2C, R (= sixD2mtx(rW2C)), approx_centre."""
    point_map = densePoint[..., :3]
    point_conf = densePoint[..., 3]
    Twc = pp.quat2unit(SE3(T_WC.reshape(8)[:7]))
    Rt = pp.matrix(pp.inv(Twc))
    height, width = image.shape[1], image.shape[2]
    pm = point_map.permute(2, 0, 1)[None]
    depth_foundation = pm[:, 2:, ...]
    idepth = torch.where(depth_foundation != 0, 1.0 / (depth_foundation + 1e-4), 1e4)
    idepth_pyr = [F.interpolate(idepth, (height, width), mode="bilinear", align_corners=True)[0]]
    image_pyr = [image]
    for _ in range(pyr_levels - 1):
        idepth_pyr.append(F.avg_pool2d(idepth_pyr[-1], 2))
        image_pyr.append(F.avg_pool2d(image_pyr[-1], 2))
    rW2C = Rt[:3, :2].clone().contiguous()
    tW2C = Rt[:3, 3].clone().contiguous()
    return dict(image_pyr=image_pyr, idepth_pyr=idepth_pyr, point_map=pm, conf=point_conf[None, None].to(torch.float32),
                rW2C=rW2C, tW2C=tW2C, R=sixD2mtx(rW2C), approx_centre=-Rt[:3, :3].T @ Rt[:3, 3])

"""TEST INFRASTRUCTURE ONLY.  Oracle for the frame tracker (csrc/track.cu): ``CameraTracker.track`` steps 2-7,
``get_points_poses``, ``opt_pose_calib_sim3``, ``solve``, ``check_keyframe`` / ``check_keyframe_map``
(VSLAM/CameraTracker.py:53-396), ``constrain_points_to_ray`` / ``project_calib`` / ``act_Sim3`` (mast3r_slam/geometry.py),
``local_diag_cov_from_X1`` (utils_uncertainty.py:5-50), ``check_convergence`` / ``huber`` (nonlinear_optimizer.py) and
``ImageFrame.update_pointmap``, restated in PyTorch operation by operation on any device.  The one deliberate difference:
the normal equations are accumulated and solved in float64 (the reference: float32 under TF32 and cuSOLVER).

pypose is replaced by a small stand-in on ``[8]`` tensors (t, q xyzw, s): ``inv``, ``mul``, ``act``, ``exp``,
``quat2unit``, ``matrix``; ``exp`` is ``gn_ref.exp_sim3``.  PARITY WITH PYPOSE UNPINNED (not vendored, not installable):
the stand-in is pinned by float64 ``matrix_exp`` of the sim(3) generator and the Jacobian by autograd under the left
perturbation ``Exp(d) T`` (tests/test_tracking.py)."""
import math

import torch

from oracle import gn_ref

LOST_NONE, LOST_MATCHES, LOST_CHOLESKY, LOST_ZERO_COST = 0, 1, 2, 3


# ---- pypose stand-in ----
def quat2unit(T):
    q = T[..., 3:7]
    return torch.cat([T[..., :3], q / q.norm(dim=-1, keepdim=True).clamp_min(1e-12), T[..., 7:]], -1)


def act(T, X):
    return gn_ref.act_so3(T[3:7], X) * T[7] + T[:3]


def mul(A, B):
    return torch.cat([act(A, B[:3]), gn_ref.quat_comp(A[3:7], B[3:7]), (A[7] * B[7]).reshape(1)])


def inv(A):
    qi = A[3:7] * torch.tensor([-1.0, -1.0, -1.0, 1.0], dtype=A.dtype, device=A.device)
    si = 1.0 / A[7]
    return torch.cat([-si * gn_ref.act_so3(qi, A[:3]), qi, si.reshape(1)])


def exp(xi):
    t, q, s = gn_ref.exp_sim3(xi)
    return torch.cat([t, q, s.reshape(1)])


def matrix(T):
    """[4,4] with the top-left block s R."""
    q = T[3:7]
    eye = torch.eye(3, dtype=T.dtype, device=T.device)
    R = gn_ref.act_so3(q.expand(3, 4), eye).T                    # columns R e_k
    M = torch.eye(4, dtype=T.dtype, device=T.device)
    M[:3, :3] = T[7] * R
    M[:3, 3] = T[:3]
    return M


# ---- geometry ----
def pixel_grid(H, W, dtype, device):
    v, u = torch.meshgrid(torch.arange(H, device=device), torch.arange(W, device=device), indexing="ij")
    return torch.stack([u, v], -1).reshape(-1, 2).to(dtype)


def backproject(uv, z, K):
    """uv [N,2], z [N,1] -> [N,3]: x, y replaced by the ray through the pixel at depth z."""
    ray = torch.stack([(uv[:, 0] - K[0, 2]) / K[0, 0], (uv[:, 1] - K[1, 2]) / K[1, 1], torch.ones_like(uv[:, 0])], -1)
    return z * ray


def constrain_points_to_ray(X, H, W, K):
    return backproject(pixel_grid(H, W, X.dtype, X.device), X[:, 2:3], K)


def local_diag_cov(X, H, W, win=5, var_floor=1e-12):
    """Diagonal of the local 5x5 covariance, [N,3] (the reference's [N,3,3] has nothing else)."""
    pad = win // 2
    img = X.view(H, W, 3)
    valid = (torch.isfinite(img).all(-1) & (img[..., 2] > 0)).to(X.dtype).unsqueeze(-1)

    def box(a):
        x = torch.nn.functional.pad(a.permute(2, 0, 1).unsqueeze(0), (pad, pad, pad, pad), mode="reflect")
        return torch.nn.functional.avg_pool2d(x, kernel_size=win, stride=1).squeeze(0).permute(1, 2, 0)

    denom = box(valid).clamp_min(1e-9)
    mean = box(img * valid) / denom
    ex2 = box((img * img) * valid) / denom
    return (ex2 - mean * mean).clamp_min(var_floor).reshape(H * W, 3)


def skew(p):
    o = torch.zeros_like(p[:, 0])
    return torch.stack([o, -p[:, 2], p[:, 1], p[:, 2], o, -p[:, 0], -p[:, 1], p[:, 0], o], -1).view(-1, 3, 3)


def project_residual(T, Xf, meas_k, K, H, W, border, z_eps):
    """-> (r [N,3], J [N,3,7] = -dpz/dP [I | -[P]x | P], valid_proj [N], P [N,3])."""
    P = act(T, Xf)
    p = (K.expand(P.shape[0], 3, 3) @ P[..., None]).squeeze(-1)
    p = p / p[:, 2:3]
    u, v = p[:, 0:1], p[:, 1:2]
    x, y, z = P[:, 0:1], P[:, 1:2], P[:, 2:3]
    valid = (u > border) & (u < W - 1 - border) & (v > border) & (v < H - 1 - border) & (z > z_eps)
    logz = torch.log(z)
    logz = torch.where(z > z_eps, logz, torch.zeros_like(logz))
    pz = torch.cat([u, v, logz], -1)
    zi = 1.0 / z[:, 0]
    fx, fy = K[0, 0], K[1, 1]
    d = torch.zeros(P.shape[0], 3, 3, dtype=P.dtype, device=P.device)
    d[:, 0, 0] = fx
    d[:, 1, 1] = fy
    d[:, 0, 2] = -fx * x[:, 0] * zi
    d[:, 1, 2] = -fy * y[:, 0] * zi
    d = d * zi[:, None, None]
    d[:, 2, 2] = zi
    D = torch.cat([torch.eye(3, dtype=P.dtype, device=P.device).expand(P.shape[0], 3, 3), -skew(P), P[..., None]], -1)
    return meas_k - pz, -(d @ D), valid[:, 0], P


def huber(r, k):
    a = r.abs()
    return torch.where(a < k, torch.ones_like(a), k / a)


def cov_det(T, P, var, K):
    """det(JCOV (sR) Sigma (sR)^T JCOV^T) per point, as the reference forms it (:336-345)."""
    R = matrix(T)[:3, :3]
    S = torch.diag_embed(var)
    Sk = R @ S @ R.T
    X, Y, Z = P.unbind(-1)
    o = torch.zeros_like(X)
    JC = torch.stack([K[0, 0] / Z, o, -K[0, 0] * X / (Z ** 2), o, K[1, 1] / Z, -K[1, 1] * Y / (Z ** 2), o, o, 1 / Z],
                     -1).reshape(-1, 3, 3)
    return torch.det(JC @ Sk @ JC.transpose(-1, -2))


# ---- the tracker ----
def get_points_poses(idx_f2k, Xff, Cff, kf_X, kf_C, kf_N, H, W, K, depth_eps):
    """Key-frame-order Xf, Xf_cov diagonal, Cf, Ck, meas_k, valid_meas_k (the frame's update_pointmap with N = 0)."""
    Xf_all = constrain_points_to_ray(Xff, H, W, K)
    Xk = constrain_points_to_ray(kf_X, H, W, K)
    cov = local_diag_cov(Xf_all, H, W)
    Cf, Ck = Cff / 1, kf_C / kf_N
    meas_k = torch.cat([pixel_grid(H, W, Xff.dtype, Xff.device), torch.log(Xk[:, 2:3])], -1)
    valid_meas_k = Xk[:, 2:3] > depth_eps
    meas_k = torch.where(valid_meas_k, meas_k, torch.zeros_like(meas_k))
    return Xf_all[idx_f2k], cov[idx_f2k], Xk, Cf[idx_f2k], Ck, meas_k, valid_meas_k[:, 0]


def prepare(idx_f2k, valid_match_k, Xff, Cff, Qff, Qkf, kf_X, kf_C, kf_N, K, H, W, cfg):
    Xf, cov, Xk, Cf, Ck, meas_k, valid_meas_k = get_points_poses(idx_f2k, Xff, Cff.reshape(-1, 1), kf_X,
                                                                 kf_C.reshape(-1, 1), kf_N, H, W, K, cfg["depth_eps"])
    Qk = torch.sqrt(Qff.reshape(-1, 1)[idx_f2k] * Qkf.reshape(-1, 1))
    vm = valid_match_k.reshape(-1, 1)
    valid_opt = vm & (Cf > cfg["C_conf"]) & (Ck > cfg["C_conf"]) & (Qk > cfg["Q_conf"])
    valid_kf = vm & (Qk > cfg["Q_conf"])
    match_frac = valid_opt.sum() / valid_opt.numel()
    return dict(Xf=Xf, Xf_cov=cov, Xk=Xk, Qk=Qk[:, 0], meas_k=meas_k, valid_meas_k=valid_meas_k, valid_opt=valid_opt[:, 0],
                valid_kf=valid_kf[:, 0], lost=bool(match_frac < cfg["min_match_frac"]))


def opt_pose_calib_sim3(Xf, Xf_cov, T_WCf, T_WCk, Qk, valid, meas_k, valid_meas_k, K, H, W, cfg, covariance_filter,
                        trace=None):
    """Returns (T_WCf, T_CkCf, lost, iterations).  ``trace``, a list, receives per-iteration dicts (H, g, cost,
    threshold, det, valid_cov, tau)."""
    T_WCf, T_WCk = quat2unit(T_WCf), quat2unit(T_WCk)
    Qk, valid, valid_meas_k = Qk.reshape(-1, 1), valid.reshape(-1, 1), valid_meas_k.reshape(-1, 1)
    sq = torch.sqrt(Qk)
    sqrt_info = torch.cat([(1 / cfg["sigma_pixel"] * valid * sq).repeat(1, 2), 1 / cfg["sigma_depth"] * valid * sq], 1)
    T = mul(inv(T_WCk), T_WCf)
    old_cost = float("inf")
    its = 0
    for step in range(cfg["max_iters"]):
        r, J, valid_proj, P = project_residual(T, Xf, meas_k, K, H, W, cfg["pixel_border"], cfg["depth_eps"])
        rec = {}
        if covariance_filter:
            det = cov_det(T, P, Xf_cov, K)
            thr = max(torch.quantile(det, 0.9), 1)
            valid_cov = (det < thr)[:, None]
            rec.update(det=det, threshold=thr, valid_cov=valid_cov[:, 0])
        else:
            valid_cov = torch.ones_like(valid_meas_k)
        s2 = (valid_proj[:, None] & valid_meas_k & valid_cov) * sqrt_info
        rob = s2 * torch.sqrt(huber(s2 * r, cfg["huber"]))
        A = (rob[..., None] * J).view(-1, 7).double()
        b = (rob * r).view(-1, 1).double()
        Hm = A.T @ A
        g = -A.T @ b
        cost = 0.5 * float((b.T @ b).item())
        rec.update(H=Hm, g=g[:, 0], cost=cost)
        if trace is not None:
            trace.append(rec)
        try:
            L = torch.linalg.cholesky(Hm)
        except Exception:  # noqa: BLE001  (the reference's exception path, caught by track as lost)
            return T_WCf, T, LOST_CHOLESKY, its
        tau = torch.cholesky_solve(g, L)[:, 0].float()
        rec["tau"] = tau
        T = quat2unit(mul(exp(tau), T))
        its += 1
        # check_convergence
        if old_cost == 0.0:
            return T_WCf, T, LOST_ZERO_COST, its
        rel = math.fabs((old_cost - cost) / old_cost) if math.isfinite(old_cost) else float("nan")
        if rel < cfg["rel_error"] or torch.linalg.norm(tau) < cfg["delta_norm"]:
            break
        old_cost = cost
    return mul(T_WCk, T), T, LOST_NONE, its


def check_keyframe(idx_f2k, valid_kf, valid_match_k, cfg):
    n = valid_kf.numel()
    match_frac_k = valid_kf.sum() / n
    unique_frac_f = torch.unique(idx_f2k[valid_match_k]).shape[0] / n
    return bool(min(match_frac_k, unique_frac_f) < cfg["match_frac_thresh"])


def check_keyframe_map(idx_f2k, valid_opt, H, W, thres_keyframe, min_displacement, last_dist):
    uvf = torch.stack([idx_f2k % W, idx_f2k // W], -1)
    uvk = pixel_grid(H, W, torch.float32, idx_f2k.device).long()
    dist = torch.norm((uvf - uvk).float(), dim=-1)[valid_opt]
    q = torch.quantile(dist, thres_keyframe).item()
    return (q - last_dist) > min_displacement, q


def update_pointmap(X, C, Xn, Cn):
    return ((C * X) + (Cn * Xn)) / (C + Cn), C + Cn


def track(idx_f2k, valid_match_k, Xff, Cff, Qff, Xkf, Ckf, Qkf, kf_X, kf_C, kf_N, T_WCf, T_WCk, K, H, W, cfg,
          min_displacement, thres_keyframe, last_dist, covariance_filter=True, point_fusion_frontend=True, trace=None):
    """Returns a dict: lost (reason), is_keyframe, is_keyframe_map, T_WCf, T_CkCf, last_dist, kf_X, kf_C, kf_N, iters,
    prep (the prepared tensors)."""
    idx = idx_f2k.reshape(-1)
    vm = valid_match_k.reshape(-1)
    prep = prepare(idx, vm, Xff, Cff, Qff, Qkf, kf_X, kf_C, kf_N, K, H, W, cfg)
    out = dict(lost=LOST_NONE, is_keyframe=False, is_keyframe_map=False, T_WCf=T_WCf, T_CkCf=None, last_dist=last_dist,
               kf_X=kf_X, kf_C=kf_C, kf_N=kf_N, iters=0, prep=prep)
    if prep["lost"]:
        out["lost"] = LOST_MATCHES
        return out
    Tw, Tr, lost, its = opt_pose_calib_sim3(prep["Xf"], prep["Xf_cov"], T_WCf, T_WCk, prep["Qk"], prep["valid_opt"],
                                            prep["meas_k"], prep["valid_meas_k"], K, H, W, cfg, covariance_filter, trace)
    out.update(iters=its, T_CkCf=Tr)
    if lost:
        out["lost"] = lost
        return out
    out["T_WCf"] = quat2unit(Tw)
    if point_fusion_frontend:
        Xkk = act(Tr, Xkf)
        X, Cn = update_pointmap(kf_X, kf_C.reshape(-1, 1), Xkk, Ckf.reshape(-1, 1))
        out.update(kf_X=X, kf_C=Cn.reshape(kf_C.shape), kf_N=kf_N + 1)
    kf = check_keyframe(idx, prep["valid_kf"], vm, cfg)
    out["is_keyframe"] = kf
    if kf:
        out.update(is_keyframe_map=True, last_dist=0)
    else:
        is_map, dq = check_keyframe_map(idx, prep["valid_opt"], H, W, thres_keyframe, min_displacement, last_dist)
        out["is_keyframe_map"] = is_map
        out["dist_quantile"] = dq
        if is_map:
            out["last_dist"] = dq
    return out

"""TEST INFRASTRUCTURE ONLY.  Oracle for the global Gauss-Newton (VSLAM/backend/src/gn_kernels.cu): the reference's kernels
and host loop restated in PyTorch — residuals, Huber weights, Jacobians (gn_kernels.cu:924-1095 rays, :1346-1500 calib),
``apply_Sim3_adj_inv`` (:267-290), the 14x14 block layout and the index bookkeeping of ``SparseBlock`` (:71-113), a double
Cholesky solve (the reference: Eigen SimplicialLLT in double, :136-160), ``expSim3`` / ``retrSim3`` (:316-412) and the
termination rule of the host loop (:1141-1229).  By default everything except the solve runs in float32 like the kernels;
``dtype=torch.float64`` gives the high-precision run the tests compare the kernels' stages with.
PARITY UNPINNED by the reference: its GN extension needs Eigen, which is not vendored, so it cannot be built here; this is a
restatement from the source."""
import torch

EPS = 1e-6


def quat_comp(qi, qj):
    x = qi[..., 3] * qj[..., 0] + qi[..., 0] * qj[..., 3] + qi[..., 1] * qj[..., 2] - qi[..., 2] * qj[..., 1]
    y = qi[..., 3] * qj[..., 1] - qi[..., 0] * qj[..., 2] + qi[..., 1] * qj[..., 3] + qi[..., 2] * qj[..., 0]
    z = qi[..., 3] * qj[..., 2] + qi[..., 0] * qj[..., 1] - qi[..., 1] * qj[..., 0] + qi[..., 2] * qj[..., 3]
    w = qi[..., 3] * qj[..., 3] - qi[..., 0] * qj[..., 0] - qi[..., 1] * qj[..., 1] - qi[..., 2] * qj[..., 2]
    return torch.stack([x, y, z, w], -1)


def act_so3(q, X):
    qv = q[..., :3].expand(X.shape)
    uv = 2.0 * torch.cross(qv, X, dim=-1)
    return X + q[..., 3:4] * uv + torch.cross(qv, uv, dim=-1)


def rel_sim3(ti, qi, si, tj, qj, sj):
    si_inv = 1.0 / si
    qi_inv = qi * torch.tensor([-1.0, -1.0, -1.0, 1.0], dtype=qi.dtype, device=qi.device)
    return act_so3(qi_inv, tj - ti) * si_inv, quat_comp(qi_inv, qj), si_inv * sj


def adj_inv(t, q, s, X):
    """Row vectors X [..., 7] times the inverse adjoint (tau, omega, s)."""
    s_inv = 1.0 / s
    Ra = act_so3(q, X[..., 0:3])
    Y0 = s_inv * Ra
    Y1 = act_so3(q, X[..., 3:6]) + s_inv * torch.cross(t.expand(Ra.shape), Ra, dim=-1)
    Y2 = X[..., 6:7] + s_inv * (t * Ra).sum(-1, keepdim=True)
    return torch.cat([Y0, Y1, Y2], -1)


def huber(r):
    a = r.abs()
    return torch.where(a < 1.345, torch.ones_like(a), 1.345 / a)


def _rows_rays(P, Xi, valid, q, sigma_ray, sigma_dist):
    n1i = Xi.norm(dim=-1, keepdim=True)
    n2j = (P * P).sum(-1, keepdim=True)
    n1j = n2j.sqrt()
    r = P / n1j
    err = torch.cat([r - Xi / n1i, n1j - n1i], -1)                       # [n,4]
    sw_a = torch.where(valid, q.sqrt() / sigma_ray, torch.zeros_like(q))
    sw_b = torch.where(valid, q.sqrt() / sigma_dist, torch.zeros_like(q))
    sw = torch.stack([sw_a, sw_a, sw_a, sw_b], -1)
    w = huber(sw * err) * sw * sw
    n3 = 1.0 / (n1j * n2j)
    eye = torch.eye(3, dtype=P.dtype, device=P.device)
    dr = eye / n1j[..., None] - P[..., :, None] * P[..., None, :] * n3[..., None]   # [n,3,3]
    z = torch.zeros_like(r[..., 0])
    rot = torch.stack([torch.stack([z, r[..., 2], -r[..., 1]], -1), torch.stack([-r[..., 2], z, r[..., 0]], -1),
                       torch.stack([r[..., 1], -r[..., 0], z], -1)], -2)            # rows: (0,z,-y), (-z,0,x), (y,-x,0)
    J3 = torch.cat([dr, rot, torch.zeros_like(r)[..., None]], -1)                   # [n,3,7]
    J4 = torch.cat([r, torch.zeros_like(r), n1j], -1)[..., None, :]                 # [n,1,7]
    return err, w, torch.cat([J3, J4], -2)


def _rows_calib(P, Xi, ind, valid, q, K, height, width, pixel_border, z_eps, sigma_pixel, sigma_depth):
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    u_t, v_t = (ind % width).to(P.dtype), (ind // width).to(P.dtype)
    vz = (P[..., 2] > z_eps) & (Xi[..., 2] > z_eps)
    zj_inv = torch.where(vz, 1.0 / P[..., 2], torch.zeros_like(P[..., 2]))
    zj_log = torch.where(vz, P[..., 2].clamp_min(1e-30).log(), torch.zeros_like(zj_inv))
    zi_log = torch.where(vz, Xi[..., 2].clamp_min(1e-30).log(), torch.zeros_like(zj_inv))
    xz, yz = P[..., 0] * zj_inv, P[..., 1] * zj_inv
    u, v = fx * xz + cx, fy * yz + cy
    vu = (u > pixel_border) & (u < width - 1 - pixel_border)
    vv = (v > pixel_border) & (v < height - 1 - pixel_border)
    valid = valid & vu & vv & vz
    err = torch.stack([u - u_t, v - v_t, zj_log - zi_log], -1)
    sw_a = torch.where(valid, q.sqrt() / sigma_pixel, torch.zeros_like(q))
    sw_b = torch.where(valid, q.sqrt() / sigma_depth, torch.zeros_like(q))
    sw = torch.stack([sw_a, sw_a, sw_b], -1)
    w = huber(sw * err) * sw * sw
    z = torch.zeros_like(xz)
    o = torch.ones_like(xz)
    J = torch.stack([torch.stack([fx * zj_inv, z, -fx * xz * zj_inv, -fx * xz * yz, fx * (1 + xz * xz), -fx * yz, z], -1),
                     torch.stack([z, fy * zj_inv, -fy * yz * zj_inv, -fy * (1 + yz * yz), fy * xz * yz, fy * xz, z], -1),
                     torch.stack([z, z, zj_inv, yz, -xz, z, o], -1)], -2)
    return err, w, J


def exp_so3(phi):
    th2 = (phi * phi).sum()
    if th2 < EPS:
        th4 = th2 * th2
        imag = 0.5 - th2 / 48.0 + th4 / 3840.0
        real = 1.0 - th2 / 8.0 + th4 / 384.0
    else:
        th = th2.sqrt()
        imag = torch.sin(0.5 * th) / th
        real = torch.cos(0.5 * th)
    return torch.cat([imag * phi, real.reshape(1)])


def exp_sim3(xi):
    tau, phi, sigma = xi[0:3], xi[3:6], xi[6]
    scale = torch.exp(sigma)
    q = exp_so3(phi)
    th2 = (phi * phi).sum()
    th = th2.sqrt()
    one = torch.tensor(1.0, dtype=xi.dtype, device=xi.device)
    if sigma.abs() < EPS:
        C = one
        if th.abs() < EPS:
            A, B = 0.5 * one, one / 6.0
        else:
            A, B = (1 - torch.cos(th)) / th2, (th - torch.sin(th)) / (th2 * th)
    else:
        C = (scale - 1) / sigma
        if th.abs() < EPS:
            s2 = sigma * sigma
            A = ((sigma - 1) * scale + 1) / s2
            B = (scale * 0.5 * s2 + scale - 1 - sigma * scale) / (s2 * sigma)
        else:
            a, b, c = scale * torch.sin(th), scale * torch.cos(th), th2 + sigma * sigma
            A = (a * sigma + (1 - b) * th) / (th * c)
            B = (C - ((b - 1) * sigma + a * th) / c) / th2
    c1 = torch.linalg.cross(phi, tau)
    c2 = torch.linalg.cross(phi, c1)
    return C * tau + A * c1 + B * c2, q, scale


HUBER_K = 1.345


def _rel_margin(x, t):
    """|x - t| relative to the larger operand: how far a gated value is from flipping its decision."""
    t = torch.as_tensor(t, dtype=x.dtype, device=x.device)
    return (x - t).abs() / torch.maximum(x.abs(), t.abs()).clamp_min(1e-30)


def edge_ranks(ii, jj):
    """Key-frame ids -> positions in the pose table (the rank of the id among the unique sorted ids, gn_kernels.cu:160-171)."""
    unique = torch.unique(torch.cat([ii, jj]), sorted=True)
    return torch.searchsorted(unique, ii), torch.searchsorted(unique, jj)


def edge_blocks(mode, Twc, Xs, Cs, ii, jj, idx_ii2jj, valid_match, Q, sigma_a, sigma_b, C_thresh, Q_thresh, K=None, height=0,
                width=0, pixel_border=0, z_eps=0.0, dtype=torch.float32, return_rows=False):
    """The per-edge normal-equation blocks of one iteration, computed in ``dtype``.

    Returns a dict:
      S [E,7,7], v [E,7]  the j-side block sum_n w J J^T and gradient sum_n w e J (the i side is the negation: Ji = -Jj);
      A [E,7,7], B [E,7]  magnitude sums  sum w' |J_a||J_b|  and  sum w (|e| + u_e) |J_a|, where u_e is the size of the
                          operands whose difference forms the residual (1 for the unit-ray components, |P| for the distance,
                          the pixel coordinate plus the principal point for u / v, 1 + |log z| for the log depth): rounding
                          in an fp32 evaluation scales with these, so they set the tolerance of a comparison; w' adds
                          w u_e / |e| where huber is active (w = 1.345 sw / |e| inherits the rounding of e);
      margin_pt [E,n]     per point, the smallest relative distance of a gated value to its threshold (Q_thresh, the two
                          confidences against C_thresh, huber's 1.345; calib also z_eps for P_z and Xi_z and the four
                          pixel-border limits); +inf where valid_match is false;
      margin              its minimum;
      err, w, J           (return_rows) the residual rows [E,n,R], their weights and the j-side Jacobian rows [E,n,R,7].
    ``ii`` / ``jj`` are key-frame ids, mapped to pose-table positions as the reference does."""
    E, n, Kp = idx_ii2jj.shape[0], Xs.shape[1], Xs.shape[0]
    ie, je = edge_ranks(ii, jj)
    T, X = Twc.to(dtype), Xs.to(dtype)
    Cs2, Q2 = Cs.reshape(Kp, n).to(dtype), Q.reshape(E, n).to(dtype)
    vm2, idx2 = valid_match.reshape(E, n).bool(), idx_ii2jj.reshape(E, n).long()
    Kd = K.to(dtype) if K is not None else None
    R = 4 if mode == "rays" else 3
    out = {k: [] for k in ("S", "v", "A", "B", "margin_pt", "err", "w", "J")}
    step = max(1, (1 << 17) // max(n, 1))                                  # edges per batch
    for e0 in range(0, E, step):
        sl = slice(e0, min(E, e0 + step))
        ix, jx = ie[sl], je[sl]
        ti, qi, si = T[ix, None, 0:3], T[ix, None, 3:7], T[ix, None, 7:8]     # [e,1,.]
        tj, qj, sj = T[jx, None, 0:3], T[jx, None, 3:7], T[jx, None, 7:8]
        tij, qij, sij = rel_sim3(ti, qi, si, tj, qj, sj)
        vm = vm2[sl]
        ind = torch.where(vm, idx2[sl], torch.zeros_like(idx2[sl]))
        Xi = torch.gather(X[ix], 1, ind[..., None].expand(-1, -1, 3))
        Xj = X[jx]
        P = act_so3(qij.expand(Xj.shape[:-1] + (4,)), Xj) * sij + tij
        q = Q2[sl]
        ci, cj = torch.gather(Cs2[ix], 1, ind), Cs2[jx]
        valid = vm & (q > Q_thresh) & (ci > C_thresh) & (cj > C_thresh)
        gates = [_rel_margin(q, Q_thresh), _rel_margin(ci, C_thresh), _rel_margin(cj, C_thresh)]
        if mode == "rays":
            err, w, Jrow = _rows_rays(P, Xi, valid, q, sigma_a, sigma_b)
            n1 = torch.maximum(P.norm(dim=-1), Xi.norm(dim=-1))
            ue = torch.stack([torch.ones_like(n1)] * 3 + [n1], -1)
            sw = torch.stack([q.sqrt() / sigma_a] * 3 + [q.sqrt() / sigma_b], -1)
        else:
            err, w, Jrow = _rows_calib(P, Xi, ind, valid, q, Kd, height, width, pixel_border, z_eps, sigma_a, sigma_b)
            fx, fy, cx, cy = Kd[0, 0], Kd[1, 1], Kd[0, 2], Kd[1, 2]
            vz = (P[..., 2] > z_eps) & (Xi[..., 2] > z_eps)
            zi = torch.where(vz, 1.0 / P[..., 2], torch.zeros_like(P[..., 2]))
            u, vv = fx * P[..., 0] * zi + cx, fy * P[..., 1] * zi + cy
            u_t, v_t = (ind % width).to(dtype), (ind // width).to(dtype)
            lz = torch.maximum(P[..., 2].abs().clamp_min(1e-30).log().abs(), Xi[..., 2].abs().clamp_min(1e-30).log().abs())
            ue = torch.stack([torch.maximum(u.abs(), u_t) + cx.abs(), torch.maximum(vv.abs(), v_t) + cy.abs(), 1.0 + lz], -1)
            sw = torch.stack([q.sqrt() / sigma_a] * 2 + [q.sqrt() / sigma_b], -1)
            gates += [_rel_margin(P[..., 2], z_eps), _rel_margin(Xi[..., 2], z_eps),
                      _rel_margin(u, pixel_border), _rel_margin(u, width - 1 - pixel_border),
                      _rel_margin(vv, pixel_border), _rel_margin(vv, height - 1 - pixel_border)]
        # huber's switch only matters where the point is used (its weight is continuous there anyway)
        hub = torch.where(valid[..., None], _rel_margin((sw * err).abs(), HUBER_K), torch.full_like(err, float("inf")))
        gates.append(hub.amin(-1))
        m = torch.stack(gates, -1).amin(-1)
        out["margin_pt"].append(torch.where(vm, m, torch.full_like(m, float("inf"))))
        Jj = adj_inv(ti[:, :, None], qi[:, :, None], si[:, :, None], Jrow)      # [e,n,R,7]
        aJ = Jj.abs()
        # where huber is active w = 1.345 sw / |e|: its rounding is that of e, relative u_e / |e|
        active = (sw * err).abs() >= HUBER_K
        wA = w * (1.0 + torch.where(active, ue / err.abs().clamp_min(1e-30), torch.zeros_like(ue)))
        out["S"].append(torch.einsum("enr,enra,enrb->eab", w, Jj, Jj))
        out["v"].append(torch.einsum("enr,enr,enra->ea", w, err, Jj))
        out["A"].append(torch.einsum("enr,enra,enrb->eab", wA, aJ, aJ))
        out["B"].append(torch.einsum("enr,enr,enra->ea", w, err.abs() + ue, aJ))
        if return_rows:
            out["err"].append(err)
            out["w"].append(w)
            out["J"].append(Jj)
    res = {k: torch.cat(vs) if vs else torch.zeros(0) for k, vs in out.items()}
    res["margin"] = float(res["margin_pt"].min()) if res["margin_pt"].numel() else float("inf")
    if not return_rows:
        for k in ("err", "w", "J"):
            res.pop(k)
    return res


def assemble(S, v, ie, je, n_poses, num_fix=1):
    """The dense system of the free poses in float64: block (i,i) += S, (j,j) += S, (i,j) = (j,i) -= S, b_i -= v, b_j += v;
    rows and columns of the fixed poses are dropped (SparseBlock::update_lhs / update_rhs, gn_kernels.cu:71-113)."""
    D = 7 * (n_poses - num_fix)
    H = torch.zeros(D, D, dtype=torch.float64)
    b = torch.zeros(D, dtype=torch.float64)
    S, v = S.double().cpu(), v.double().cpu()
    for e in range(S.shape[0]):
        io, jo = int(ie[e]) - num_fix, int(je[e]) - num_fix
        for (a, sa) in ((io, -1.0), (jo, 1.0)):
            if a < 0:
                continue
            b[a * 7:a * 7 + 7] += sa * v[e]
            for (c, sc) in ((io, -1.0), (jo, 1.0)):
                if c >= 0:
                    H[a * 7:a * 7 + 7, c * 7:c * 7 + 7] += (sa * sc) * S[e]
    return H, b


def retract(Twc, dx, num_fix=1):
    """Twc[k] <- exp(dx[k - num_fix]) Twc[k] for the free poses, in the dtype of ``dx`` (retrSim3, gn_kernels.cu:387-412)."""
    for k in range(num_fix, Twc.shape[0]):
        dt, dq, ds = exp_sim3(dx[k - num_fix])
        t, q, s = Twc[k, 0:3].clone(), Twc[k, 3:7].clone(), Twc[k, 7].clone()
        Twc[k, 3:7] = quat_comp(dq, q)
        Twc[k, 0:3] = act_so3(dq, t) * ds + dt
        Twc[k, 7] = ds * s
    return Twc


def gauss_newton(mode, Twc, Xs, Cs, ii, jj, idx_ii2jj, valid_match, Q, sigma_a, sigma_b, C_thresh, Q_thresh, max_iter,
                 delta_thresh, K=None, height=0, width=0, pixel_border=0, z_eps=0.0, dtype=torch.float32):
    """mode 'rays' | 'calib'.  Twc [K,8] is updated in place; returns (dx_last [K-1,7], iterations run).  The blocks, the
    step and the retraction are evaluated in ``dtype`` (float32 like the kernels, float64 for a high-precision run); the
    system is always assembled and solved in double."""
    num_fix = 1
    Kp = Xs.shape[0]
    ie, je = edge_ranks(ii.cpu(), jj.cpu())
    dx, its = torch.zeros(Kp - num_fix, 7, dtype=dtype, device=Twc.device), 0
    for _ in range(max_iter):
        blk = edge_blocks(mode, Twc, Xs, Cs, ii, jj, idx_ii2jj, valid_match, Q, sigma_a, sigma_b, C_thresh, Q_thresh, K=K,
                          height=height, width=width, pixel_border=pixel_border, z_eps=z_eps, dtype=dtype)
        H, b = assemble(blk["S"], blk["v"], ie, je, Kp, num_fix)
        try:
            L = torch.linalg.cholesky(H)
            x = torch.cholesky_solve(b[:, None], L)[:, 0]
            dx = (-x).to(dtype).reshape(-1, 7).to(Twc.device)
        except Exception:  # noqa: BLE001  (SimplicialLLT failure path returns zeros)
            dx = torch.zeros(Kp - num_fix, 7, dtype=dtype, device=Twc.device)
        retract(Twc, dx, num_fix)
        its += 1
        if float(dx.norm()) < delta_thresh:
            break
    return dx, its

"""The global Gauss-Newton (csrc/gn.cu) stage by stage against float64.

One iteration leaves every stage in the solver's workspace: the per-edge 7x7 blocks S and gradients v, the dense system H
of the free poses (its strict upper triangle), the Cholesky factor L (lower triangle and diagonal), the solution x (in b),
and the retracted poses.  The GPU tests read each stage and compare it with a float64 evaluation of the same operation:
the oracle's blocks (oracle/gn_ref.edge_blocks) at shapes that reach every point split of the edge kernel, the gates
(confidence through idx, Q, z_eps, pixel border) each shown to bite, the assembly of an irregular graph, the solver past
one CTA's row stride (D > 1024) and one warp's substitution stride (D > 32), the failure path, the retraction, and the
benchmark's shape end to end.  The CPU tests pin the oracle itself: its Jacobians against autograd, its exp_sim3 against
the matrix exponential, and its float32 run against its float64 run."""
import ctypes

import pytest
import torch

from oracle import gn_ref
from test_gn import _act_inv, _perturb, _pose_err, _rand_pose, calib_problem, rays_problem

F64 = torch.float64
RAYS = dict(sigma_a=0.003, sigma_b=10.0)
CALIB = dict(sigma_a=1.0, sigma_b=10.0)
TOL_BLOCK = 1e-5           # |S - S64| <= TOL_BLOCK * A,  |v - v64| <= TOL_BLOCK * B
MIN_MARGIN = 1e-4          # every gated value at least this far (relative) from its threshold
WORST = {}                 # largest observed error / tolerance per check, printed with -s


def _note(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), float(ratio))
    print(f"[gn-stages] {key}: worst error/tolerance {WORST[key]:.3g}")


def _kmat(h, w):
    """Non-square intrinsics: fx != fy and an off-centre principal point."""
    return torch.tensor([[0.9 * w, 0.0, 0.47 * w - 0.3], [0.0, 1.1 * w, 0.53 * h + 0.2], [0.0, 0.0, 1.0]])


def _backproject(Kmat, u, v, z):
    return torch.stack([(u - Kmat[0, 2]) / Kmat[0, 0] * z, (v - Kmat[1, 2]) / Kmat[1, 1] * z, z], -1)


def _split(E, n):
    """The edge kernel's point split (adb_gauss_newton): enough CTAs for 8 per SM of a 132-SM H100, at least 1024
    points per CTA."""
    s = min(-(-1056 // E), -(-n // 1024))
    return max(s, 1)


def _ids(ranks):
    return ranks * 3 + 5                  # arbitrary ascending key-frame ids


def block_problem(mode, Kp, E, n, h, w, seed, C_thresh=0.0, Q_thresh=1.0):
    """Random pointmaps on the pixels of an h x w image at depth 2..5, poses near the identity (so that points stay in
    the image), random correspondences, and every frame on some edge.  Q and the confidences keep away from thresholds."""
    g = torch.Generator().manual_seed(seed)
    Kmat = _kmat(h, w)
    T = torch.stack([_rand_pose(g, scale_t=0.1, ang=0.1, s_rng=0.05) for _ in range(Kp)])
    u = torch.rand(Kp, n, generator=g) * (w - 1)
    v = torch.rand(Kp, n, generator=g) * (h - 1)
    Xs = _backproject(Kmat, u, v, 2.0 + 3.0 * torch.rand(Kp, n, generator=g))
    pairs = [(k, (k + 1) % Kp) for k in range(Kp)][:E]
    while len(pairs) < E:
        i, j = torch.randint(0, Kp, (2,), generator=g).tolist()
        if i != j:
            pairs.append((i, j))
    ii = _ids(torch.tensor([p[0] for p in pairs]))
    jj = _ids(torch.tensor([p[1] for p in pairs]))
    idx = torch.randint(0, n, (E, n), generator=g)
    valid = torch.rand(E, n, 1, generator=g) > 0.1
    Q = torch.rand(E, n, 1, generator=g) * 2 + 0.5
    Q = torch.where((Q - Q_thresh).abs() < 0.01, Q + 0.02, Q)
    Cs = torch.rand(Kp, n, 1, generator=g) + 1.0
    Cs = torch.where((Cs - C_thresh).abs() < 0.01, Cs + 0.02, Cs)
    return dict(mode=mode, T=T, Xs=Xs, Cs=Cs, K=Kmat, ii=ii, jj=jj, idx=idx, valid=valid, Q=Q, h=h, w=w, border=-10,
                z_eps=1e-3, C_thresh=C_thresh, Q_thresh=Q_thresh)


def _oracle_blocks(p, dtype=F64, dev=None, **kw):
    """The oracle's blocks of problem ``p``, evaluated on ``dev`` (the float64 reference runs on the GPU where there is
    one: the big shapes take minutes on a CPU), returned on the CPU."""
    sig = RAYS if p["mode"] == "rays" else CALIB
    d = {k: (x.to(dev) if dev is not None and isinstance(x, torch.Tensor) else x) for k, x in p.items()}
    out = gn_ref.edge_blocks(d["mode"], d["T"], d["Xs"], d["Cs"], d["ii"], d["jj"], d["idx"], d["valid"], d["Q"],
                             sig["sigma_a"], sig["sigma_b"], d["C_thresh"], d["Q_thresh"], K=d["K"], height=d["h"],
                             width=d["w"], pixel_border=d["border"], z_eps=d["z_eps"], dtype=dtype, **kw)
    return {k: (x.cpu() if isinstance(x, torch.Tensor) else x) for k, x in out.items()}


def sanitize(p, min_margin=1e-3, dev=None):
    """Drop (valid_match = False) the points whose gated values lie within ``min_margin`` of a threshold, so that float32
    and float64 take the same decisions."""
    m = _oracle_blocks(p, dev=dev)["margin_pt"]
    p["valid"] = p["valid"] & (m >= min_margin).reshape(p["valid"].shape)
    return p


# ----------------------------------------------------------------------------------------------------------------------
# CPU: the oracle against autograd, the matrix exponential and itself
# ----------------------------------------------------------------------------------------------------------------------

def _residual_fn(mode, Ti, Tj, Xi, Xj, ind, Kmat, h, w, side):
    """err(xi) with T_side <- exp(xi) T_side (float64); huber weights play no part."""
    ones = torch.ones(Xj.shape[0], dtype=F64)
    valid = torch.ones(Xj.shape[0], dtype=torch.bool)

    def f(xi):
        dt, dq, ds = gn_ref.exp_sim3(xi)
        T = Tj if side == "j" else Ti
        Tn = torch.cat([gn_ref.act_so3(dq, T[0:3]) * ds + dt, gn_ref.quat_comp(dq, T[3:7]), (ds * T[7]).reshape(1)])
        A, B = (Ti, Tn) if side == "j" else (Tn, Tj)
        tij, qij, sij = gn_ref.rel_sim3(A[0:3], A[3:7], A[7:8], B[0:3], B[3:7], B[7:8])
        P = gn_ref.act_so3(qij, Xj) * sij + tij
        if mode == "rays":
            err, _, _ = gn_ref._rows_rays(P, Xi, valid, ones, 1.0, 1.0)
        else:
            err, _, _ = gn_ref._rows_calib(P, Xi, ind, valid, ones, Kmat, h, w, -1e9, 1e-6, 1.0, 1.0)
        return err
    return f


@pytest.mark.parametrize("mode", ["rays", "calib"])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_jacobians_equal_autograd(mode, seed):
    g = torch.Generator().manual_seed(100 + seed)
    h, w, n = 360, 640, 40
    Kmat = torch.tensor([[500.0, 0.0, 300.5], [0.0, 430.0, 170.2], [0.0, 0.0, 1.0]], dtype=F64)
    Ti = _rand_pose(g, scale_t=0.5, ang=0.8, s_rng=0.3).double()
    Tj = _rand_pose(g, scale_t=0.5, ang=0.8, s_rng=0.3).double()
    for T in (Ti, Tj):
        T[3:7] /= T[3:7].norm()           # exactly unit in float64: act_so3 is only a rotation for a unit quaternion
    # points chosen in camera i (in front of it), carried to frame j so that P is exactly them
    P = _backproject(Kmat, torch.rand(n, generator=g).double() * (w - 1), torch.rand(n, generator=g).double() * (h - 1),
                     2.0 + 3.0 * torch.rand(n, generator=g).double())
    tij, qij, sij = gn_ref.rel_sim3(Ti[0:3], Ti[3:7], Ti[7:8], Tj[0:3], Tj[3:7], Tj[7:8])
    Xj = gn_ref.act_so3(qij * torch.tensor([-1.0, -1, -1, 1], dtype=F64), P - tij) / sij
    Xi = P * (1.0 + 0.05 * torch.randn(n, 1, generator=g).double())
    ind = torch.randperm(n, generator=g)
    Xs = torch.zeros(2, n, 3, dtype=F64)
    Xs[0, ind], Xs[1] = Xi, Xj
    blk = gn_ref.edge_blocks(mode, torch.stack([Ti, Tj]), Xs, torch.ones(2, n), torch.tensor([0]), torch.tensor([1]),
                             ind[None], torch.ones(1, n, dtype=torch.bool), torch.ones(1, n), 1.0, 1.0, 0.0, 0.0, K=Kmat,
                             height=h, width=w, pixel_border=-1e9, z_eps=1e-6, dtype=F64, return_rows=True)
    J = blk["J"][0]                                                   # [n,R,7] j side
    assert torch.isfinite(J).all() and J.abs().amax() > 0
    zero = torch.zeros(7, dtype=F64)
    for side, sign in (("j", 1.0), ("i", -1.0)):
        Jad = torch.autograd.functional.jacobian(_residual_fn(mode, Ti, Tj, Xi, Xj, ind, Kmat, h, w, side), zero)
        scale = J.abs().amax(-1, keepdim=True)                          # per residual row
        err = (sign * J - Jad).abs() / scale
        assert float(err.max()) < 1e-9, (side, float(err.max()))


@pytest.mark.parametrize("sigma,theta", [(1e-9, 1e-8), (1e-9, 0.7), (0.3, 1e-8), (-0.4, 1.1)])
def test_oracle_exp_sim3_equals_matrix_exp(sigma, theta):
    """All four branches of expSim3 (sigma and theta each below / above EPS) in float64."""
    g = torch.Generator().manual_seed(7)
    axis = torch.randn(3, generator=g, dtype=F64)
    phi = axis / axis.norm() * theta
    tau = torch.randn(3, generator=g, dtype=F64)
    xi = torch.cat([tau, phi, torch.tensor([sigma], dtype=F64)])
    assert (abs(sigma) < gn_ref.EPS) == (sigma == 1e-9) and (theta < gn_ref.EPS) == (theta == 1e-8)
    t, q, s = gn_ref.exp_sim3(xi)
    G = torch.zeros(4, 4, dtype=F64)
    G[:3, :3] = torch.tensor([[sigma, -phi[2], phi[1]], [phi[2], sigma, -phi[0]], [-phi[1], phi[0], sigma]], dtype=F64)
    G[:3, 3] = tau
    M = torch.linalg.matrix_exp(G)
    R = gn_ref.act_so3(q.expand(3, 4), torch.eye(3, dtype=F64)).T       # columns R e_k
    assert abs(float(q.norm()) - 1.0) < 1e-14
    assert torch.allclose(s * R, M[:3, :3], rtol=0, atol=1e-12)
    assert torch.allclose(t, M[:3, 3], rtol=0, atol=1e-8 * (1 + float(tau.norm())))


def _agree_32_64(mode, init, args, kw):
    """fp32 and fp64 oracle runs from the same start: blocks within TOL_BLOCK of their magnitudes, the first step within
    what the system's conditioning allows for that block error, and the converged poses."""
    b32 = gn_ref.edge_blocks(mode, init, *args, **kw)
    b64 = gn_ref.edge_blocks(mode, init, *args, dtype=F64, **kw)
    assert float(((b32["S"].double() - b64["S"]) / (TOL_BLOCK * b64["A"])).abs().max()) <= 1.0
    assert float(((b32["v"].double() - b64["v"]) / (TOL_BLOCK * b64["B"])).abs().max()) <= 1.0
    H, _ = gn_ref.assemble(b64["S"], b64["v"], *gn_ref.edge_ranks(args[2], args[3]), init.shape[0])
    cond = float(torch.linalg.cond(H))
    T32, T64 = init.clone(), init.double()
    dx32, _ = gn_ref.gauss_newton(mode, T32, *args, 1, 0.0, **kw)
    dx64, _ = gn_ref.gauss_newton(mode, T64, *args, 1, 0.0, dtype=F64, **kw)
    assert dx64.dtype == F64 and T64.dtype == F64
    assert float((dx32.double() - dx64).abs().max()) <= cond * TOL_BLOCK * float(dx64.abs().max()), cond
    gn_ref.gauss_newton(mode, T32, *args, 9, 1e-6, **kw)
    gn_ref.gauss_newton(mode, T64, *args, 9, 1e-6, dtype=F64, **kw)
    et, eq, es = _pose_err(T32.double(), T64)
    assert et < 1e-5 and eq < 1e-6 and es < 1e-5, (et, eq, es)
    return T64


def test_oracle_float32_and_float64_runs_agree():
    """The fp32 oracle (the kernels' arithmetic) and its float64 run on the problems of test_gn.py."""
    truth, init, Xs, Cs, ii, jj, idx, valid, Q, _ = rays_problem()
    T64 = _agree_32_64("rays", init, (Xs, Cs, ii, jj, idx, valid, Q, RAYS["sigma_a"], RAYS["sigma_b"], 0.0, 1.5), {})
    assert _pose_err(T64, truth.double())[0] < 2e-4
    truth, init, Xs, Cs, Kmat, ii, jj, idx, valid, Q, h, w = calib_problem()
    T64 = _agree_32_64("calib", init, (Xs, Cs, ii, jj, idx, valid, Q, 1.0, 10.0, 0.0, 0.6),
                       dict(K=Kmat, height=h, width=w, pixel_border=-10, z_eps=1e-6))
    assert _pose_err(T64, truth.double())[0] < 5e-4


def test_oracle_blocks_margins_and_magnitudes():
    """edge_blocks' bookkeeping: S symmetric, |S| <= A entrywise, |v| <= B, and the margin finds a planted near-tie."""
    for mode in ("rays", "calib"):
        p = block_problem(mode, 3, 4, 300, 15, 20, seed=3)
        b = _oracle_blocks(p)
        assert ((b["S"] - b["S"].transpose(1, 2)).abs() <= 1e-14 * b["A"]).all()
        assert (b["S"].abs() <= b["A"] * (1 + 1e-12)).all() and (b["v"].abs() <= b["B"]).all()
        k =int(torch.nonzero(p["valid"].reshape(4, 300)[0])[0])
        p["Q"] = p["Q"].clone()
        p["Q"].view(4, 300)[0, k] = p["Q_thresh"] * (1 + 1e-6)
        assert _oracle_blocks(p)["margin"] < 2e-6


# ----------------------------------------------------------------------------------------------------------------------
# GPU
# ----------------------------------------------------------------------------------------------------------------------

_TRI = [(a, c) for a in range(7) for c in range(a + 1)]


def _decode(ws, Kp, E):
    """The workspace layout of adb_gauss_newton: H [D,D] f64, b [D] f64, S [E,28] f32, v [E,7] f32."""
    from artdeco_b200 import _lib
    nb = ctypes.c_size_t(0)
    _lib.call("adb_gn_workspace_bytes", Kp, E, ctypes.byref(nb))
    assert ws.numel() == nb.value
    ws = ws.cpu()
    D = 7 * (Kp - 1)
    out, o = {}, 0
    for name, count, dt in (("H", D * D, F64), ("b", D, F64), ("S28", E * 28, torch.float32), ("v", E * 7, torch.float32)):
        size = count * dt.itemsize
        out[name] = ws[o:o + size].clone().view(dt)
        o += size
    assert o <= nb.value
    out["H"] = out["H"].reshape(D, D)
    S28, out["v"] = out.pop("S28").reshape(E, 28), out["v"].reshape(E, 7)
    S = torch.zeros(E, 7, 7)
    for l, (a, c) in enumerate(_TRI):
        S[:, a, c] = S28[:, l]
        S[:, c, a] = S28[:, l]
    out["S"] = S
    return out


def _run(p, cuda, max_iter=1, delta=0.0, T=None, **over):
    from artdeco_b200 import gn
    q = dict(p, **over)
    sig = RAYS if q["mode"] == "rays" else CALIB
    Td = (q["T"] if T is None else T).clone().to(cuda)
    Kd = q["K"].to(cuda) if q["mode"] == "calib" else None
    (dx,), state, ws = gn._solve(0 if q["mode"] == "rays" else 1, Td, q["Xs"].to(cuda), q["Cs"].to(cuda), Kd,
                                 q["ii"].to(cuda), q["jj"].to(cuda), q["idx"].to(cuda), q["valid"].to(cuda), q["Q"].to(cuda),
                                 q["h"], q["w"], q["border"], q["z_eps"], sig["sigma_a"], sig["sigma_b"], q["C_thresh"],
                                 q["Q_thresh"], max_iter, delta, return_state=True, return_workspace=True)
    out = _decode(ws, q["Xs"].shape[0], q["ii"].shape[0])
    out.update(T=Td.cpu(), dx=dx.cpu(), state=state.cpu())
    return out


def _check_blocks(k, ref, key, tol=TOL_BLOCK):
    rs = float(((k["S"].double() - ref["S"]).abs() / (tol * ref["A"]).clamp_min(1e-300)).max())
    rv = float(((k["v"].double() - ref["v"]).abs() / (tol * ref["B"]).clamp_min(1e-300)).max())
    _note(key + " S", rs)
    _note(key + " v", rv)
    assert rs <= 1.0 and rv <= 1.0, (key, rs, rv)


BLOCK_SHAPES = [  # (E, key frames, n, height, width): the split is 192, 9, 1, 1, 1
    (1, 2, 512 * 384, 384, 512),
    (128, 12, 128 * 96, 96, 128),
    (1200, 40, 2048, 32, 64),
    (6, 4, 37, 1, 37),
    (10, 5, 1000, 25, 40),
]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["rays", "calib"])
@pytest.mark.parametrize("shape", BLOCK_SHAPES, ids=lambda s: f"E{s[0]}-n{s[2]}")
def test_edge_blocks_match_float64(cuda, mode, shape):
    E, Kp, n, h, w = shape
    p = sanitize(block_problem(mode, Kp, E, n, h, w, seed=E + n, C_thresh=0.5), dev=cuda)
    ref = _oracle_blocks(p, dev=cuda)
    assert ref["margin"] >= MIN_MARGIN
    k = _run(p, cuda)
    _check_blocks(k, ref, f"blocks {mode}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["rays", "calib"])
@pytest.mark.parametrize("shape", BLOCK_SHAPES[:2], ids=lambda s: f"E{s[0]}-n{s[2]}")
def test_split_boundaries_exact(cuda, mode, shape):
    """Only the points at the edges of each CTA's range carry weight: a dropped or doubled boundary point shows."""
    E, Kp, n, h, w = shape
    p = block_problem(mode, Kp, E, n, h, w, seed=11)
    split = _split(E, n)
    chunk = -(-n // split)
    keep = {0, n - 1}
    for part in range(1, split):
        keep |= {part * chunk - 1, part * chunk, part * chunk + 1}
    keep = torch.tensor(sorted(k for k in keep if 0 <= k < n))
    vm = torch.zeros(E, n, dtype=torch.bool)
    vm[:, keep] = True
    p["valid"] = vm[..., None]
    p["Q"] = p["Q"].clone().fill_(2.0)
    ref = _oracle_blocks(p, dev=cuda)
    assert ref["margin"] >= MIN_MARGIN
    assert (ref["A"].diagonal(dim1=1, dim2=2) > 0).all()
    k = _run(p, cuda)
    _check_blocks(k, ref, f"split {mode}", tol=1e-6)


GATES = {  # case: (settings of the run, settings that switch the gate off)
    "z_P": (dict(z_eps=0.5), dict(z_eps=0.1)),
    "z_Xi": (dict(z_eps=0.5), dict(z_eps=0.1)),
    "border": (dict(border=2), dict(border=-10)),
    "conf_i": (dict(C_thresh=1.2), dict(C_thresh=0.0)),
    "conf_j": (dict(C_thresh=1.2), dict(C_thresh=0.0)),
    "Q": (dict(Q_thresh=1.0), dict(Q_thresh=0.0)),
}


def gate_problem(case, seed=5):
    """Calib, non-square K, key frames 0,1 on the i side and 2,3 on the j side; points planted where ``case`` gates."""
    h, w = 24, 40
    n = h * w
    p = block_problem("calib", 4, 4, n, h, w, seed=seed, Q_thresh=0.1)
    p.update(ii=_ids(torch.tensor([0, 1, 0, 1])), jj=_ids(torch.tensor([2, 2, 3, 3])), border=2, z_eps=0.5)
    g = torch.Generator().manual_seed(seed + 1)
    Kmat, T, Xs = p["K"], p["T"].double(), p["Xs"].clone()
    Cs, Q, idx, valid = p["Cs"].clone(), p["Q"].clone(), p["idx"].clone(), p["valid"].clone().reshape(4, n)
    # keep every ordinary point comfortably inside the border
    u = torch.rand(4, n, generator=g) * (w - 9) + 4
    v = torch.rand(4, n, generator=g) * (h - 9) + 4
    Xs = _backproject(Kmat, u, v, 2.0 + 3.0 * torch.rand(4, n, generator=g))
    planted = torch.randperm(n, generator=g)[:64].reshape(4, 16)          # 16 points per edge, distinct j-side points
    edges = ((0, 2), (1, 2), (0, 3), (1, 3))
    for e, (i, j) in enumerate(edges):
        ks = planted[e]
        for f, (_, jf) in enumerate(edges):       # a moved j-side point is used by this edge only
            if jf == j and f != e:
                valid[f, ks] = False
        valid[e, ks] = True
        if case in ("z_P", "border"):
            cx, cy = float(Kmat[0, 2]), float(Kmat[1, 2])
            if case == "z_P":
                pix = [(w / 2 + (r % 4) - 2, h / 2 + (r // 4) - 2, 0.3) for r in range(16)]
            else:
                sides = [(1.5, h / 2), (w - 2.5, h / 2), (w / 2, 1.5), (w / 2, h - 2.5)]
                pix = [(sides[r % 4][0] + 0.0, sides[r % 4][1] + 0.0, 2.5 + 0.1 * r) for r in range(16)]
            P = torch.stack([_backproject(Kmat.double(), torch.tensor(a, dtype=F64), torch.tensor(b_, dtype=F64),
                                          torch.tensor(z, dtype=F64)) for a, b_, z in pix])
            tij, qij, sij = gn_ref.rel_sim3(T[i, 0:3], T[i, 3:7], T[i, 7:8], T[j, 0:3], T[j, 3:7], T[j, 7:8])
            Xs[j, ks] = (gn_ref.act_so3(qij * torch.tensor([-1.0, -1, -1, 1], dtype=F64), P - tij) / sij).float()
        elif case == "z_Xi":
            # frames 0 and 1 are never on the j side: a shrunk point only ever acts as an Xi
            m = idx[e, ks]
            Xs[i, m] = Xs[i, m] * (0.25 / Xs[i, m, 2:3])
    if case in ("conf_i", "conf_j"):
        Cs = torch.rand(4, n, 1, generator=g) + 1.3
        frames = (0, 1) if case == "conf_i" else (2, 3)
        low = torch.rand(4, n, 1, generator=g) < 0.25
        for f in frames:
            Cs[f] = torch.where(low[f], torch.full_like(Cs[f], 0.5), Cs[f])
    if case == "Q":
        Q = torch.rand(4, n, 1, generator=g) * 2 + 0.1
        Q = torch.where((Q - 1.0).abs() < 0.01, Q + 0.02, Q)
    p.update(Xs=Xs, Cs=Cs, Q=Q, idx=idx, valid=valid.reshape(4, n, 1))
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(GATES))
def test_gates_match_float64_and_bite(cuda, case):
    on, off = GATES[case]
    p = gate_problem(case)
    p.update(on)
    p = sanitize(p, dev=cuda)
    ref = _oracle_blocks(p, dev=cuda)
    assert ref["margin"] >= MIN_MARGIN
    k = _run(p, cuda)
    _check_blocks(k, ref, f"gate {case}")
    k_off = _run(p, cuda, **off)
    ref_off = _oracle_blocks(dict(p, **off), dev=cuda)
    bite = float(((k_off["S"].double() - k["S"].double()).abs() / ref["A"].clamp_min(1e-300)).max())
    assert bite > 100 * TOL_BLOCK, (case, bite)
    assert float(((k_off["S"].double() - ref_off["S"]).abs() / ref_off["A"].clamp_min(1e-300)).max()) < 1e-3


def _abs_assembly(S, ie, je, n_poses):
    """sum of |S| over every block an edge adds to: the scale of the rounding in H's entries."""
    D = 7 * (n_poses - 1)
    H = torch.zeros(D, D, dtype=F64)
    for e in range(S.shape[0]):
        for a in (int(ie[e]) - 1, int(je[e]) - 1):
            for c in (int(ie[e]) - 1, int(je[e]) - 1):
                if a >= 0 and c >= 0:
                    H[a * 7:a * 7 + 7, c * 7:c * 7 + 7] += S[e].double().abs()
    return H


def assembly_problem():
    """Non-contiguous, unsorted key-frame ids; edges both ways, a duplicate edge, a self-edge; the fixed pose (the
    smallest id, 7) on both sides."""
    ids = [40, 7, 23, 91, 15]
    edges = [(23, 7), (7, 91), (40, 23), (23, 40), (15, 91), (15, 91), (40, 40), (91, 15), (15, 23), (91, 7)]
    order = sorted(ids)
    p = block_problem("rays", 5, len(edges), 500, 20, 25, seed=21)
    p["ii"] = torch.tensor([e[0] for e in edges])
    p["jj"] = torch.tensor([e[1] for e in edges])
    p["ranks"] = {k: order.index(k) for k in ids}
    return sanitize(p)


@pytest.mark.gpu
def test_assembly_of_an_irregular_graph(cuda):
    p = assembly_problem()
    k = _run(p, cuda)
    ie, je = gn_ref.edge_ranks(p["ii"], p["jj"])
    H_ref, b_ref = gn_ref.assemble(k["S"], k["v"], ie, je, 5)
    H_abs = _abs_assembly(k["S"], ie, je, 5)
    up = torch.triu(torch.ones(28, 28, dtype=torch.bool), 1)
    err = ((k["H"] - H_ref).abs() - 1e-12 * H_abs)[up]
    assert float(err.max()) <= 0.0, float(err.max())
    # the self-edge (40, 40) adds S and subtracts it again: H is what the graph without it assembles
    self_e = 6
    assert float(k["S"][self_e].abs().max()) > 0
    keep = torch.tensor([e for e in range(len(ie)) if e != self_e])
    H_wo, b_wo = gn_ref.assemble(k["S"][keep], k["v"][keep], ie[keep], je[keep], 5)
    assert float((((k["H"] - H_wo).abs() - 1e-12 * H_abs)[up]).max()) <= 0.0
    # the fixed pose (rank 0) has no rows: an edge to it only touches the other pose's diagonal block
    for e in (0, 1, 9):                                               # (23, 7), (7, 91), (91, 7)
        one, _ = gn_ref.assemble(k["S"][e:e + 1], k["v"][e:e + 1], ie[e:e + 1], je[e:e + 1], 5)
        r = int(ie[e] if ie[e] > 0 else je[e]) - 1
        blk = torch.zeros(28, 28, dtype=torch.bool)
        blk[r * 7:r * 7 + 7, r * 7:r * 7 + 7] = True
        assert torch.equal(one[blk].reshape(7, 7), k["S"][e].double()) and (one[~blk] == 0).all()
    # the kernel solved this system: b holds x with H x = b (b from its own v, the i side with -v)
    x = torch.linalg.solve(H_ref, b_ref)
    assert torch.allclose(k["b"], x, rtol=1e-6, atol=1e-9 * float(x.abs().max()))
    assert torch.equal(k["T"][0], p["T"][0])


def chain_problem(Kp, n=256, seed=31):
    """A chain of key frames plus loop closures every 4 frames back to frames 0..Kp/4."""
    # the closures from the last frames to frames 0 and 1 put nonzeros (and fill-in) more than 1024 rows below the
    # diagonal at K = 160, where the solver's rows wrap around its CTA
    pairs = [(k, k + 1) for k in range(Kp - 1)] + [(k, k // 2 - 1) for k in range(4, Kp, 4)] + [(Kp - 1, 1), (Kp - 2, 0)]
    p = block_problem("rays", Kp, len(pairs), n, 16, 16, seed=seed)
    p["ii"] = _ids(torch.tensor([a for a, _ in pairs]))
    p["jj"] = _ids(torch.tensor([b for _, b in pairs]))
    return sanitize(p)


@pytest.mark.gpu
@pytest.mark.parametrize("Kp", [6, 160])
def test_dense_cholesky_and_substitution(cuda, Kp):
    """K = 6 (D = 35) crosses the warp stride of the substitutions, K = 160 (D = 1113) the CTA stride of the row loop."""
    p = chain_problem(Kp)
    k = _run(p, cuda)
    D = 7 * (Kp - 1)
    assert int(k["state"][3]) == 1
    ie, je = gn_ref.edge_ranks(p["ii"], p["jj"])
    H, b = gn_ref.assemble(k["S"], k["v"], ie, je, Kp)
    H_abs = _abs_assembly(k["S"], ie, je, Kp)
    up = torch.triu(torch.ones(D, D, dtype=torch.bool), 1)
    assert float((((k["H"] - H).abs() - 1e-12 * H_abs)[up]).max()) <= 0.0
    L = torch.tril(k["H"])
    assert (L.diagonal() > 0).all()
    LL = L @ L.T
    ratio = float(((LL - H).abs() / (1e-12 * (L.abs() @ L.abs().T)).clamp_min(1e-300)).max())
    _note(f"cholesky K={Kp} LL^T", ratio)
    assert ratio <= 1.0
    x = torch.cholesky_solve(b[:, None], torch.linalg.cholesky(H))[:, 0]
    cond = float(torch.linalg.cond(H))
    tol = 1e3 * cond * torch.finfo(F64).eps * float(x.abs().max())
    ratio = float((k["b"] - x).abs().max()) / tol
    _note(f"solve K={Kp} (cond {cond:.3g})", ratio)
    assert ratio <= 1.0
    assert torch.equal(k["dx"].reshape(-1), (-k["b"]).float())


@pytest.mark.gpu
def test_failure_path_zero_pivot(cuda):
    """Every match of the edges of key frame 3 invalid: its rows of H are exactly zero, the first of them a zero pivot."""
    p = block_problem("rays", 5, 8, 400, 20, 20, seed=41)
    dead = 3
    touch = (p["ii"] == _ids(torch.tensor(dead))) | (p["jj"] == _ids(torch.tensor(dead)))
    assert touch.any()
    p["valid"] = p["valid"].clone()
    p["valid"][touch] = False
    k = _run(p, cuda)
    assert torch.equal(k["dx"], torch.zeros_like(k["dx"]))
    assert int(k["state"][3]) == 0 and int(k["state"][0]) == 1
    assert torch.equal(k["T"], p["T"]), "a failed factorisation leaves the poses unchanged"
    k = _run(p, cuda, max_iter=3, delta=1e-3)
    st = k["state"]
    assert int(st[0]) == 1 and int(st[1]) == 1 and int(st[3]) == 0, st
    assert torch.equal(k["T"], p["T"])


def _retraction_ratio(T0, T1, dx):
    """Error of the kernel's retraction against the float64 retraction of the same dx, over 1e-6 (1 + |t|).  The
    translation also gets the rounding of expSim3's float32 C = (e^sigma - 1) / sigma (the reference's arithmetic),
    2^-24 |tau| / |sigma|, which is large when a small scale step comes with a large translation step."""
    ref = gn_ref.retract(T0.double().clone(), dx.double())
    d = dx.double()
    c_err = torch.where(d[:, 6].abs() >= gn_ref.EPS, 2.0 ** -24 * d[:, :3].norm(dim=-1) / d[:, 6].abs(),
                        torch.zeros_like(d[:, 6]))
    t_tol = 1e-6 * (1.0 + ref[1:, 0:3].abs().amax(-1)) + 4 * c_err
    t_tol = torch.cat([torch.full((1,), 1e-6, dtype=F64), t_tol])          # pose 0 is fixed
    tol = torch.cat([t_tol[:, None].expand(-1, 3), torch.full((T0.shape[0], 5), 1e-6, dtype=F64)], -1)
    ratio = float(((T1.double() - ref).abs() / tol).max())
    qn = float((T1[:, 3:7].double().norm(dim=-1) - 1).abs().max())
    return ratio, qn


@pytest.mark.gpu
def test_retraction_matches_float64(cuda):
    truth, init, Xs, Cs, ii, jj, idx, valid, Q, _ = rays_problem(K=5, n=3000, seed=2, mag=0.1)
    p = dict(mode="rays", T=init, Xs=Xs, Cs=Cs, K=None, ii=ii, jj=jj, idx=idx, valid=valid, Q=Q, h=0, w=0, border=0,
             z_eps=0.0, C_thresh=0.0, Q_thresh=1.5)
    T = init.clone()
    small = False
    for it in range(15):
        k = _run(p, cuda, T=T, delta=1e-6)
        ratio, qn = _retraction_ratio(T, k["T"], k["dx"])
        _note("retraction", ratio)
        assert ratio <= 1.0 and qn < 1e-6, (it, ratio, qn)
        dxn = k["dx"].double()
        small = bool((dxn[:, 3:6].norm(dim=-1) < gn_ref.EPS).all() and (dxn[:, 6].abs() < gn_ref.EPS).all())
        T = k["T"]
        if int(k["state"][1]):
            break
    # float32 poses stall at |dx| ~ 3e-7 on this graph; below 1e-6 every component is under EPS
    assert int(k["state"][1]) == 1 and small, "ran to |dx| < 1e-6, whose step takes the small-angle branches"
    assert _pose_err(T, truth)[0] < 2e-4


def bench_problem(seed=0, Kp=32, E=128, n=128 * 96, mag=0.03):
    """A consistent rays graph at the shape bench.py times: every frame sees the same world points."""
    g = torch.Generator().manual_seed(seed)
    truth = torch.stack([_rand_pose(g, scale_t=0.5, ang=0.3, s_rng=0.1) for _ in range(Kp)])
    W = torch.randn(n, 3, generator=g) * 2.0 + torch.tensor([0.0, 0.0, 6.0])
    Xs = torch.stack([_act_inv(truth[k], W) for k in range(Kp)])
    pairs = [(k, k + 1) for k in range(Kp - 1)] + [(k + 1, k) for k in range(Kp - 1)]
    while len(pairs) < E:
        i, j = torch.randint(0, Kp, (2,), generator=g).tolist()
        if i != j:
            pairs += [(i, j), (j, i)]
    pairs = pairs[:E]
    init = truth.clone()
    for k in range(1, Kp):
        init[k] = _perturb(truth[k], g, mag)
    p = dict(mode="rays", T=init, Xs=Xs, Cs=torch.rand(Kp, n, 1, generator=g) + 1.0, K=None,
             ii=_ids(torch.tensor([a for a, _ in pairs])), jj=_ids(torch.tensor([b for _, b in pairs])),
             idx=torch.arange(n)[None].repeat(E, 1), valid=torch.rand(E, n, 1, generator=g) > 0.3,
             Q=torch.rand(E, n, 1, generator=g) + 1.0, h=0, w=0, border=0, z_eps=0.0, C_thresh=0.0, Q_thresh=1.2)
    p["Q"] = torch.where((p["Q"] - 1.2).abs() < 0.01, p["Q"] + 0.02, p["Q"])
    return truth, p


@pytest.mark.gpu
def test_bench_shape_end_to_end(cuda):
    truth, p = bench_problem()
    sanitize(p, dev=cuda)
    d = {k: p[k].to(cuda) for k in ("Xs", "Cs", "ii", "jj", "idx", "valid", "Q")}
    T64 = p["T"].double().to(cuda)
    T = p["T"].clone()
    for it in range(5):
        gn_ref.gauss_newton("rays", T64, d["Xs"], d["Cs"], d["ii"], d["jj"], d["idx"], d["valid"], d["Q"],
                            RAYS["sigma_a"], RAYS["sigma_b"], 0.0, 1.2, 1, 0.0, dtype=F64)
        T = _run(p, cuda, T=T)["T"]
        et, eq, es = _pose_err(T.double(), T64.cpu())
        _note(f"bench-shape iteration {it} (t, 1-|q.q'|, s)", max(et / 1e-4, eq / 1e-6, es / 1e-4))
        assert et < 1e-4 and eq < 1e-6 and es < 1e-4, (it, et, eq, es)
    et, eq, es = _pose_err(T, truth)
    assert et < 2e-4 and eq < 1e-6 and es < 2e-4, (et, eq, es)


@pytest.mark.gpu
def test_wrapper_layouts_and_refusals(cuda, monkeypatch):
    from artdeco_b200 import _lib, gn
    truth, init, Xs, Cs, ii, jj, idx, valid, Q, _ = rays_problem(K=4, n=700, seed=4)
    E, n = idx.shape
    base_args = dict(Xs=Xs, Cs=Cs, ii=ii, jj=jj, idx=idx, valid=valid, Q=Q)

    def call(T, **o):
        a = dict(base_args, **o)
        a = [a[k].to(cuda) for k in ("Xs", "Cs", "ii", "jj", "idx", "valid", "Q")]
        return gn.gauss_newton_rays(T, *a, RAYS["sigma_a"], RAYS["sigma_b"], 0.0, 1.5, 2, 0.0)

    T_ref = init.clone().to(cuda)
    call(T_ref)
    # a non-contiguous view of Twc is updated in place, its neighbours untouched
    base = torch.full((4, 16), 7.0, device=cuda)
    view = base[:, ::2]
    view.copy_(init.to(cuda))
    assert not view.is_contiguous()
    call(view)
    assert torch.allclose(view, T_ref, rtol=0, atol=1e-6) and (base[:, 1::2] == 7.0).all()
    # int32 idx, [E,n] masks and Q, [K,n] confidences
    T2 = init.clone().to(cuda)
    call(T2, idx=idx.int(), valid=valid.reshape(E, n), Q=Q.reshape(E, n), Cs=Cs.reshape(4, n))
    assert torch.allclose(T2, T_ref, rtol=0, atol=1e-6)

    # refusals come before anything is launched
    launched = []
    real_call = _lib.call
    monkeypatch.setattr(_lib, "call", lambda name, *a: (launched.append(name), real_call(name, *a))[1])
    T3 = init.clone().to(cuda)
    bad = [dict(ii=torch.tensor([10, 20, 30, 40]), jj=torch.tensor([20, 30, 40, 50])),     # 5 key frames, 4 poses
           dict(idx=idx[:, :-1]), dict(valid=valid[:-1]), dict(Q=Q[:, :-3])]
    for o in bad:
        if "ii" in o:
            o = dict(o, idx=idx[:4], valid=valid[:4], Q=Q[:4])
        with pytest.raises(ValueError):
            call(T3, **o)
    Kmat = torch.eye(3, device=cuda)
    with pytest.raises(ValueError):
        gn.gauss_newton_calib(T3, Xs.to(cuda), Cs.to(cuda), Kmat, ii.to(cuda), jj.to(cuda), idx.to(cuda), valid.to(cuda),
                              Q.to(cuda), 20, 30, 0, 1e-3, 1.0, 10.0, 0.0, 0.5, 1, 0.0)          # 20*30 != 700
    assert "adb_gauss_newton" not in launched, launched
    assert torch.equal(T3.cpu(), init)

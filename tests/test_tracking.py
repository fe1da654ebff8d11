"""Frame tracker (csrc/track.cu, artdeco_b200/tracking.py) against oracle/track_ref.py.

The reference needs pypose, which is not vendored, so no golden file exists.  The oracle is pinned on the CPU instead: its
Jacobian equals autograd's under the left perturbation Exp(d) T, its Exp equals matrix_exp of the sim(3) generator, and it
drives a perturbed pose back to the truth on a noise-free pair.  Scenes are synthetic: a smooth random key-frame depth map,
a known relative Sim(3), matches by projecting into the frame and rounding to pixels, then noise, outliers and random C / Q."""
import math

import pytest
import torch

from oracle import gn_ref
from oracle import track_ref as ref

CFG = dict(min_match_frac=0.05, max_iters=50, C_conf=0.0, Q_conf=1.5, rel_error=1e-3, delta_norm=1e-3, huber=1.345,
           match_frac_thresh=0.333, sigma_pixel=1.0, sigma_depth=10.0, pixel_border=-10, depth_eps=1e-6)
NO_CONV = dict(CFG, rel_error=0.0, delta_norm=0.0)


def _pose(t, axis, ang, s):
    axis = torch.tensor(axis, dtype=torch.float64)
    axis = axis / axis.norm()
    q = torch.cat([axis * math.sin(ang / 2), torch.tensor([math.cos(ang / 2)], dtype=torch.float64)])
    return torch.cat([torch.tensor(t, dtype=torch.float64), q, torch.tensor([s], dtype=torch.float64)]).float()


def scene(H, W, seed=0, noise=1e-3, outliers=0.05, rel=None, q_lo=1.0, q_hi=3.0, perturb=0.02):
    """Inputs of track() for a frame f and key frame k; `truth` is the true T_CkCf."""
    g = torch.Generator().manual_seed(seed)
    f = 0.8 * W
    K = torch.tensor([[f, 0.0, W / 2 - 0.5], [0.0, f, H / 2 - 0.5], [0.0, 0.0, 1.0]])
    coarse = torch.rand(1, 1, 5, 7, generator=g)
    zk = 2.5 + 1.5 * torch.nn.functional.interpolate(coarse, size=(H, W), mode="bicubic", align_corners=True)[0, 0]
    Xk_true = ref.backproject(ref.pixel_grid(H, W, torch.float32, "cpu"), zk.reshape(-1, 1), K)
    truth = rel if rel is not None else _pose([0.04, -0.03, 0.05], [0.3, 1.0, -0.2], 0.03, 1.02)
    Xf_pts = ref.act(ref.inv(truth), Xk_true)                                # key-frame points in the frame's camera
    p = Xf_pts @ K.T
    uf, vf = torch.round(p[:, 0] / p[:, 2]), torch.round(p[:, 1] / p[:, 2])
    inside = (uf >= 0) & (uf < W) & (vf >= 0) & (vf < H)
    n = H * W
    idx = (vf.clamp(0, H - 1) * W + uf.clamp(0, W - 1)).long()
    n_out = int(outliers * n)
    out_at = torch.randperm(n, generator=g)[:n_out]
    idx[out_at] = torch.randint(0, n, (n_out,), generator=g)
    valid_match = inside & (torch.rand(n, generator=g) > 0.05)
    zf = torch.full((n,), 3.0) + 0.2 * torch.rand(n, generator=g)
    zf[idx[inside]] = Xf_pts[inside, 2]
    zf = zf * (1 + noise * torch.randn(n, generator=g))
    Xff = torch.cat([torch.randn(n, 2, generator=g), zf[:, None]], 1)       # x, y are replaced by the ray constraint
    kf_X = torch.cat([Xk_true[:, :2], (zk.reshape(-1) * (1 + noise * torch.randn(n, generator=g)))[:, None]], 1)
    Xkf = Xf_pts + noise * torch.randn(n, 3, generator=g)
    rnd = lambda lo, hi: (lo + (hi - lo) * torch.rand(n, 1, generator=g))   # noqa: E731
    T_WCk = _pose([0.5, -0.2, 1.0], [1.0, 0.5, 0.2], 0.4, 1.3)
    T_WCf_true = ref.mul(T_WCk, truth)
    xi = perturb * torch.randn(7, generator=g)
    T_WCf = ref.mul(ref.exp(xi), T_WCf_true)
    return dict(idx_f2k=idx[None], valid_match_k=valid_match[None, :, None], Xff=Xff, Cff=rnd(0.5, 2.0), Qff=rnd(q_lo, q_hi),
                Xkf=Xkf, Ckf=rnd(0.5, 2.0), Qkf=rnd(q_lo, q_hi), kf_X=kf_X, kf_C=rnd(0.5, 2.0), kf_N=2, T_WCf=T_WCf,
                T_WCk=T_WCk, K=K, H=H, W=W, truth=truth)


def oracle_track(sc, cfg=CFG, filt=True, fusion=True, min_disp=0.0, thres_kf=0.5, last_dist=0.0, trace=None, dev="cpu"):
    d = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in sc.items()}
    return ref.track(d["idx_f2k"], d["valid_match_k"], d["Xff"], d["Cff"], d["Qff"], d["Xkf"], d["Ckf"], d["Qkf"],
                     d["kf_X"], d["kf_C"], d["kf_N"], d["T_WCf"], d["T_WCk"], d["K"], d["H"], d["W"], cfg, min_disp,
                     thres_kf, last_dist, filt, fusion, trace)


def _rot_err(qa, qb):
    """Angle of qa qb^-1 in radians."""
    qb = qb.double() * torch.tensor([-1.0, -1.0, -1.0, 1.0], dtype=torch.float64)
    d = gn_ref.quat_comp(qa.double(), qb)
    return 2 * math.atan2(float(d[:3].norm()), abs(float(d[3])))


# ============================== CPU ==============================

def test_oracle_jacobian_matches_autograd_left_perturbation():
    sc = scene(12, 16, seed=3)
    X = ref.constrain_points_to_ray(sc["Xff"], 12, 16, sc["K"]).double()
    T = ref.quat2unit(ref.mul(ref.inv(sc["T_WCk"]), sc["T_WCf"]).double())      # unit in float64
    K = sc["K"].double()
    meas = torch.cat([ref.pixel_grid(12, 16, torch.float64, "cpu"), torch.log(X[:, 2:3])], -1)
    r0, J, _, _ = ref.project_residual(T, X, meas, K, 12, 16, -10, 1e-6)

    def res(d):
        return ref.project_residual(ref.mul(ref.exp(d), T), X, meas, K, 12, 16, -10, 1e-6)[0]

    Ja = torch.autograd.functional.jacobian(res, torch.zeros(7, dtype=torch.float64))     # [N,3,7]
    assert torch.allclose(J, Ja, rtol=1e-9, atol=1e-9 * float(Ja.abs().max())), float((J - Ja).abs().max())


@pytest.mark.parametrize("xi", [
    [0.3, -0.2, 0.5, 0.4, -0.3, 0.2, 0.15],        # general
    [0.3, -0.2, 0.5, 0.4, -0.3, 0.2, 1e-8],        # small sigma
    [0.3, -0.2, 0.5, 1e-8, -2e-8, 1e-8, 0.15],     # small angle
    [0.3, -0.2, 0.5, 1e-8, 0.0, 0.0, 0.0],         # both
])
def test_standin_exp_matches_matrix_exp(xi):
    xi = torch.tensor(xi, dtype=torch.float64)
    T = ref.exp(xi)
    G = torch.zeros(4, 4, dtype=torch.float64)
    w = xi[3:6]
    G[:3, :3] = torch.tensor([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]], dtype=torch.float64) + xi[6] * torch.eye(3, dtype=torch.float64)
    G[:3, 3] = xi[:3]
    M = torch.linalg.matrix_exp(G)
    assert torch.allclose(ref.matrix(T), M, rtol=0, atol=2e-6), (ref.matrix(T) - M).abs().max()


def test_oracle_recovers_true_pose_on_noise_free_pair():
    """Matches are rounded to pixels, so the only error left is that quantisation (<= 0.5 px per match at f = 205 px).
    The solve reaches the same fixed point from the true and from the perturbed start; at 192x256 it lies 1.8e-3 from the
    true translation (|t| = 0.07), 3.6e-4 from the true scale and below 1e-4 rad from the true rotation.  Bounds: 1e-3 rad,
    3e-3 in translation, 1e-3 in scale."""
    sc = scene(192, 256, seed=5, noise=0.0, outliers=0.0, perturb=0.03)
    out = oracle_track(sc, cfg=NO_CONV, fusion=False)
    assert out["lost"] == 0
    T, tr = out["T_CkCf"], sc["truth"]
    T0 = ref.quat2unit(ref.mul(ref.inv(sc["T_WCk"]), sc["T_WCf"]))
    assert _rot_err(T0[3:7], tr[3:7]) + float((T0[:3] - tr[:3]).norm()) > 2e-2        # the start is really off
    assert _rot_err(T[3:7], tr[3:7]) < 1e-3
    assert float((T[:3] - tr[:3]).norm()) < 3e-3
    assert abs(float(T[7] / tr[7]) - 1) < 1e-3


@pytest.mark.parametrize("H,W", [(3, 3), (7, 7), (3, 7), (384, 384)])
def test_box_filter_covariance_matches_direct_window(H, W):
    g = torch.Generator().manual_seed(H * 1000 + W)
    X = torch.randn(H * W, 3, generator=g, dtype=torch.float64) + torch.tensor([0.0, 0.0, 3.0], dtype=torch.float64)
    X[::11, 2] = -1.0                                          # invalid (z <= 0)
    got = ref.local_diag_cov(X, H, W)
    refl = lambda i, n: -i if i < 0 else (2 * n - 2 - i if i >= n else i)   # noqa: E731
    img = X.view(H, W, 3)
    rows = [(y, x) for y in range(H) for x in range(W)] if H * W < 400 else \
        [(y, x) for y in (0, 1, 2, H // 2, H - 2, H - 1) for x in (0, 1, W // 3, W - 2, W - 1)]
    for (y, x) in rows:
        pts = torch.stack([img[refl(y + dy, H), refl(x + dx, W)] for dy in range(-2, 3) for dx in range(-2, 3)])
        v = (pts[:, 2] > 0).double()[:, None]
        den = max(float(v.mean()), 1e-9)
        mean = (pts * v).mean(0) / den
        var = ((pts * pts * v).mean(0) / den - mean * mean).clamp_min(1e-12)
        assert torch.allclose(got[y * W + x], var, rtol=1e-9, atol=1e-12), (y, x)


def test_entry_points_refuse_bad_arguments_before_touching_the_device():
    import ctypes as C
    from artdeco_b200 import _lib
    import artdeco_b200  # noqa: F401
    L = _lib.lib()

    def refused(rc, needle):
        msg = L.adb_last_error()
        return rc == 1 and msg is not None and needle in msg.decode()

    a, b = C.c_size_t(0), C.c_size_t(0)
    assert refused(L.adb_track_workspace_bytes(0, C.byref(a), C.byref(b)), "adb_track_workspace_bytes")
    assert refused(L.adb_track_workspace_bytes(16, None, C.byref(b)), "adb_track_workspace_bytes")
    assert L.adb_track_workspace_bytes(12, C.byref(a), C.byref(b)) == 0 and b.value == C.sizeof(
        __import__("artdeco_b200.tracking", fromlist=["TrackState"]).TrackState)
    p = C.c_void_p(16)                                          # never dereferenced: every check comes first
    nul = None
    prep = [p] * 10
    assert refused(L.adb_track_prepare(2, 8, *prep, 0.0, 1.5, 1e-6, 0.05, *[p] * 8, p, a.value, None), ">= 3")
    assert refused(L.adb_track_prepare(4, 8, nul, *prep[1:], 0.0, 1.5, 1e-6, 0.05, *[p] * 8, p, a.value, None), "null input")
    assert refused(L.adb_track_prepare(4, 8, *prep, 0.0, 1.5, 1e-6, 0.05, *[p] * 7, nul, p, a.value, None), "null output")
    solve_ptrs = [p] * 9
    tail = lambda n_ws: [p, p, p, p, C.c_size_t(n_ws), None]   # noqa: E731
    assert refused(L.adb_track_solve(0, 4, 8, *solve_ptrs, 10, 1, -10, C.c_float(1e-6), C.c_float(1.0), C.c_float(10.0),
                                     C.c_float(1.345), C.c_double(1e-3), C.c_float(1e-3), *tail(a.value)), "bad sizes")
    assert refused(L.adb_track_solve(32, 4, 8, *solve_ptrs, -1, 1, -10, C.c_float(1e-6), C.c_float(1.0), C.c_float(10.0),
                                     C.c_float(1.345), C.c_double(1e-3), C.c_float(1e-3), *tail(a.value)), "bad sizes")
    assert refused(L.adb_track_solve(32, 4, 8, p, p, nul, *solve_ptrs[3:], 10, 1, -10, C.c_float(1e-6), C.c_float(1.0),
                                     C.c_float(10.0), C.c_float(1.345), C.c_double(1e-3), C.c_float(1e-3), *tail(a.value)),
                   "null pointer")                              # Xf_cov needed with the covariance filter
    assert refused(L.adb_track_solve(32, 4, 8, *solve_ptrs, 10, 1, -10, C.c_float(1e-6), C.c_float(0.0), C.c_float(10.0),
                                     C.c_float(1.345), C.c_double(1e-3), C.c_float(1e-3), *tail(a.value)), "positive")
    fin = lambda h, w, fuse, thr, ptrs: L.adb_track_finish(h, w, *ptrs, fuse, C.c_double(0.333), C.c_float(thr),  # noqa: E731
                                                          C.c_double(0.1), C.c_double(0.0), p, p, C.c_size_t(1 << 30), None)
    assert refused(fin(0, 8, 1, 0.5, [p] * 7), "bad sizes")
    assert refused(fin(4, 8, 1, 0.5, [p, nul] + [p] * 5), "null pointer")
    assert refused(fin(4, 8, 1, 0.5, [p, p, nul] + [p] * 4), "point fusion")
    assert refused(fin(4, 8, 0, 1.5, [p, p] + [nul] * 5), "thres_keyframe")


def test_optimize_focal_is_refused():
    from artdeco_b200 import tracking
    with pytest.raises(NotImplementedError):
        tracking.track(*([None] * 16), 0.0, 0.5, 0.0, optimize_focal=True)


# ============================== GPU ==============================

def _gpu_track(sc, cuda, cfg=CFG, filt=True, fusion=True, min_disp=0.0, thres_kf=0.5, last_dist=0.0):
    from artdeco_b200 import tracking
    d = {k: (v.to(cuda) if torch.is_tensor(v) else v) for k, v in sc.items()}
    kf_X, kf_C = d["kf_X"].clone(), d["kf_C"].clone()
    kf_N = torch.tensor([sc["kf_N"]], dtype=torch.int32, device=cuda)
    ws = tracking.workspace(sc["H"] * sc["W"], cuda)
    res = tracking.track(d["idx_f2k"], d["valid_match_k"], d["Xff"], d["Cff"], d["Qff"], d["Xkf"], d["Ckf"], d["Qkf"], kf_X,
                         kf_C, kf_N, d["T_WCf"], d["T_WCk"], d["K"], (sc["H"], sc["W"]), cfg, min_disp, thres_kf,
                         last_dist, filt, fusion, ws=ws)
    return res, kf_X, kf_C, kf_N, tracking.TrackState.read(ws.state)


SIZES = [(384, 512), (512, 512), (37, 53)]


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", SIZES)
def test_prepare_matches_oracle(cuda, H, W):
    from artdeco_b200 import tracking
    sc = scene(H, W, seed=11)
    d = {k: (v.to(cuda) if torch.is_tensor(v) else v) for k, v in sc.items()}
    ws = tracking.workspace(H * W, cuda)
    kf_N = torch.tensor([2], dtype=torch.int32, device=cuda)
    got = tracking.prepare(d["idx_f2k"], d["valid_match_k"], d["Xff"], d["Cff"], d["Qff"], d["Qkf"], d["kf_X"], d["kf_C"],
                           kf_N, d["K"], (H, W), CFG, ws)
    st = tracking.TrackState.read(ws.state)
    exp = ref.prepare(d["idx_f2k"].reshape(-1), d["valid_match_k"].reshape(-1), d["Xff"], d["Cff"], d["Qff"], d["Qkf"],
                      d["kf_X"], d["kf_C"], 2, d["K"], H, W, CFG)
    for m in ("valid_meas_k", "valid_opt", "valid_kf"):
        assert torch.equal(got[m], exp[m]), m
    assert st.n_valid_opt == int(exp["valid_opt"].sum()) and st.n_valid_kf == int(exp["valid_kf"].sum())
    vm = d["valid_match_k"].reshape(-1)
    assert st.n_unique == int(torch.unique(d["idx_f2k"].reshape(-1)[vm]).numel())
    assert st.lost == 0
    for k in ("Xf", "Xf_cov", "Qk", "meas_k"):
        e = exp[k].reshape(got[k].shape)
        err = float(((got[k] - e).abs() / e.abs().clamp_min(1e-30)).max())
        assert err <= 1e-5, (k, err)


@pytest.mark.gpu
@pytest.mark.parametrize("filt", [True, False])
def test_one_iteration_matches_oracle(cuda, filt):
    from artdeco_b200 import tracking
    sc = scene(384, 512, seed=21)
    trace = []
    cfg1 = dict(NO_CONV, max_iters=1)
    oracle_track(sc, cfg=cfg1, filt=filt, fusion=False, trace=trace, dev=cuda)
    _, _, _, _, st = _gpu_track(sc, cuda, cfg=cfg1, filt=filt, fusion=False)
    rec = trace[0]
    Hk = torch.tensor(list(st.H), dtype=torch.float64).view(7, 7)
    gk = torch.tensor(list(st.g), dtype=torch.float64)
    He, ge = rec["H"].cpu(), rec["g"].cpu()
    assert float((Hk - He).norm() / He.norm()) < 1e-5, float((Hk - He).norm() / He.norm())
    assert float((gk - ge).norm() / ge.norm()) < 1e-5, float((gk - ge).norm() / ge.norm())
    assert abs(st.cost - rec["cost"]) / rec["cost"] < 1e-5
    if filt:
        # the kernel's threshold is torch.quantile of its own determinants
        d = {k: (v.to(cuda) if torch.is_tensor(v) else v) for k, v in sc.items()}
        ws = tracking.workspace(384 * 512, cuda)
        kf_N = torch.tensor([2], dtype=torch.int32, device=cuda)
        prep = tracking.prepare(d["idx_f2k"], d["valid_match_k"], d["Xff"], d["Cff"], d["Qff"], d["Qkf"], d["kf_X"],
                                d["kf_C"], kf_N, d["K"], (384, 512), CFG, ws)
        tracking._solve(prep["Xf"], prep["Xf_cov"], d["T_WCf"], d["T_WCk"], prep["Qk"], prep["valid_opt"], prep["meas_k"],
                        prep["valid_meas_k"], (384, 512), d["K"], cfg1, True, ws)
        n = 384 * 512
        off = (n * 12 + 255) // 256 * 256                     # the workspace keeps the values it selects after cov_f
        det = ws.ws[off:off + 4 * n].view(torch.float32)
        st2 = tracking.TrackState.read(ws.state)
        q = max(float(torch.quantile(det, 0.9)), 1.0)
        assert st2.cov_threshold == pytest.approx(q, rel=2.5e-7, abs=0), (st2.cov_threshold, q)
        thr_e = float(rec["threshold"])
        vc_k = det < st2.cov_threshold
        vc_e = rec["valid_cov"]
        frac = float((vc_k != vc_e).float().mean())
        assert frac <= 1e-4, frac
        assert abs(st2.cov_threshold - thr_e) / thr_e < 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize("iters", [10, 50])
@pytest.mark.parametrize("filt", [True, False])
def test_full_solve_matches_oracle(cuda, iters, filt):
    sc = scene(384, 512, seed=31)
    cfg = dict(NO_CONV, max_iters=iters)
    exp = oracle_track(sc, cfg=cfg, filt=filt, fusion=False, dev=cuda)
    (lost, _, _, T_WCf, T_CkCf, _), _, _, _, st = _gpu_track(sc, cuda, cfg=cfg, filt=filt, fusion=False)
    assert not lost and exp["lost"] == 0 and st.iters == iters == exp["iters"]
    Te, Tk = exp["T_CkCf"].cpu().double(), T_CkCf.cpu().double()
    et = float((Tk[:3] - Te[:3]).norm() / Te[:3].norm())
    er = _rot_err(Tk[3:7], Te[3:7])
    es = abs(float(Tk[7] / Te[7]) - 1)
    print(f"\n[track solve iters={iters} filter={filt}] rel t {et:.2e}  rot {er:.2e} rad  rel s {es:.2e}")
    assert et < 1e-5 and er < 1e-5 and es < 1e-5, (et, er, es)
    Tw = exp["T_WCf"].cpu().double()
    assert float((T_WCf.cpu().double() - Tw).abs().max()) < 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize("seed,filt", [(41, True), (42, False), (43, True)])
def test_convergence_iteration_count_matches_oracle(cuda, seed, filt):
    sc = scene(384, 512, seed=seed, perturb=0.03)
    exp = oracle_track(sc, cfg=CFG, filt=filt, fusion=False, dev=cuda)
    _, _, _, _, st = _gpu_track(sc, cuda, cfg=CFG, filt=filt, fusion=False)
    print(f"\n[track converge seed={seed}] iters {st.iters} (oracle {exp['iters']}), |tau| {st.tau_norm:.2e}")
    assert st.converged == 1 and st.iters == exp["iters"] < CFG["max_iters"]


def _lost_case(cuda, sc, cfg, reason):
    (lost, kf, kfm, T_WCf, _, ld), kf_X, kf_C, kf_N, st = _gpu_track(sc, cuda, cfg=cfg, last_dist=1.25)
    assert lost and not kf and not kfm and ld == 1.25 and st.lost == reason, (st.lost, reason)
    assert torch.equal(T_WCf.cpu(), sc["T_WCf"])
    assert torch.equal(kf_X.cpu(), sc["kf_X"]) and torch.equal(kf_C.cpu(), sc["kf_C"]) and int(kf_N) == sc["kf_N"]
    exp = oracle_track(sc, cfg=cfg, dev=cuda)
    assert exp["lost"] == reason


@pytest.mark.gpu
def test_lost_insufficient_matches_leaves_state_untouched(cuda):
    sc = scene(64, 96, seed=51)
    sc["Qff"] = sc["Qff"] * 0 + 1.0                            # Qk = sqrt(Qkf) < 1.5 almost everywhere
    sc["Qkf"] = torch.where(torch.rand(sc["Qkf"].shape, generator=torch.Generator().manual_seed(0)) < 0.02,
                            torch.full_like(sc["Qkf"], 4.0), torch.full_like(sc["Qkf"], 1.0))
    _lost_case(cuda, sc, CFG, ref.LOST_MATCHES)


@pytest.mark.gpu
def test_lost_all_rows_invalid_is_a_cholesky_failure(cuda):
    sc = scene(64, 96, seed=52)
    sc["kf_X"][:, 2] = -1.0                                    # every meas_k invalid: H = 0
    _lost_case(cuda, sc, CFG, ref.LOST_CHOLESKY)


@pytest.mark.gpu
def test_lost_nan_in_frame_pointmap(cuda):
    sc = scene(64, 96, seed=53)
    j = int(sc["idx_f2k"][0, 1000])
    sc["Xff"][j, 2] = float("nan")
    _lost_case(cuda, sc, CFG, ref.LOST_CHOLESKY)


@pytest.mark.gpu
def test_keyframe_decisions_match_oracle(cuda):
    """A sweep on both sides of match_frac_thresh (through the outlier and Q mix) and of min_displacement."""
    seen = set()
    # valid_kf fraction about 0.19 with Q ~ U[0.1, 2.2] (a new key frame), above 0.333 with U[1, 3]
    for i, (outl, q_lo, q_hi, min_disp, last) in enumerate([(0.05, 1.0, 3.0, 0.0, 0.0), (0.05, 1.0, 3.0, 50.0, 0.0),
                                                            (0.6, 1.0, 3.0, 0.0, 0.0), (0.05, 0.1, 2.2, 0.0, 0.0),
                                                            (0.05, 1.0, 3.0, 0.5, 3.0), (0.05, 1.0, 3.0, 0.5, 0.0)]):
        sc = scene(96, 128, seed=60 + i, outliers=outl, q_lo=q_lo, q_hi=q_hi,
                   rel=_pose([0.2, 0.0, 0.0], [0, 1, 0], 0.02, 1.0))
        for thres_kf in (0.3, 0.7):
            cfg = dict(CFG, max_iters=5)
            exp = oracle_track(sc, cfg=cfg, min_disp=min_disp, thres_kf=thres_kf, last_dist=last, dev=cuda)
            (lost, kf, kfm, _, _, ld), _, _, _, st = _gpu_track(sc, cuda, cfg=cfg, min_disp=min_disp, thres_kf=thres_kf,
                                                                 last_dist=last)
            assert lost == bool(exp["lost"]) and kf == exp["is_keyframe"] and kfm == exp["is_keyframe_map"], (i, thres_kf)
            assert ld == pytest.approx(exp["last_dist"], abs=0), (i, ld, exp["last_dist"])
            if not kf:
                assert st.dist_quantile == pytest.approx(exp["dist_quantile"], abs=0)
            seen.add((kf, kfm))
    assert seen == {(True, True), (False, True), (False, False)}, seen


@pytest.mark.gpu
def test_point_fusion_matches_oracle(cuda):
    sc = scene(384, 512, seed=71)
    cfg = dict(CFG, max_iters=10)
    exp = oracle_track(sc, cfg=cfg, dev=cuda)
    (lost, _, _, _, T_CkCf, _), kf_X, kf_C, kf_N, _ = _gpu_track(sc, cuda, cfg=cfg)
    assert not lost and int(kf_N) == exp["kf_N"] == 3
    # the fusion itself, through the kernel's own pose (the two solves agree to ~2e-6, see test_full_solve_matches_oracle)
    d = {k: (v.to(cuda) if torch.is_tensor(v) else v) for k, v in sc.items()}
    ex, ec = ref.update_pointmap(d["kf_X"], d["kf_C"], ref.act(T_CkCf, d["Xkf"]), d["Ckf"])
    err = float(((kf_X - ex).norm(dim=-1) / ex.norm(dim=-1)).max())
    print(f"\n[track fusion] max relative error {err:.2e}")
    assert err < 1e-6, err
    assert torch.equal(kf_C, ec)
    assert float(((exp["kf_X"] - ex).norm(dim=-1) / ex.norm(dim=-1)).max()) < 1e-5     # and the oracle's whole frame


@pytest.mark.gpu
def test_solve_is_graph_capturable_and_bitwise_reproducible(cuda):
    from artdeco_b200 import tracking
    sc = scene(384, 512, seed=81)
    d = {k: (v.to(cuda) if torch.is_tensor(v) else v) for k, v in sc.items()}
    n = 384 * 512
    ws = tracking.workspace(n, cuda)
    kf_N = torch.tensor([2], dtype=torch.int32, device=cuda)
    prep = tracking.prepare(d["idx_f2k"], d["valid_match_k"], d["Xff"], d["Cff"], d["Qff"], d["Qkf"], d["kf_X"], d["kf_C"],
                            kf_N, d["K"], (384, 512), CFG, ws)
    args = (prep["Xf"], prep["Xf_cov"], d["T_WCf"], d["T_WCk"], prep["Qk"], prep["valid_opt"], prep["meas_k"],
            prep["valid_meas_k"], (384, 512), d["K"], CFG, True)

    def run():
        ws.state.zero_()
        return tracking._solve(*args, ws)

    a = [t.clone() for t in run()] + [ws.state.clone()]
    b = [t.clone() for t in run()] + [ws.state.clone()]
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = run()
    ws.state.fill_(0xAB)
    graph.replay()
    torch.cuda.synchronize()
    c = [t.clone() for t in outs] + [ws.state.clone()]
    for x, y in zip(a, c):
        assert torch.equal(x, y)
    assert tracking.TrackState.read(ws.state).iters > 1

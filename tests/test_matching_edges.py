"""Dense matching stage by stage at the edges a smooth scene never reaches: image borders and corners, the [1, W-2] x [1, H-2]
clamp, integer positions, NaN / zero / huge points, equal descriptor scores, every descriptor layout and width.

References (oracle/matching_ref.py):
  * match_prep      F.normalize + reflect-padded Scharr convolution in float64; the initial pixel of a linear index as
                    lin_to_pixel computes it, with torch's FLOOR division (a negative index wraps to the previous row).
  * iter_proj       ``iter_proj_exact``: the LM iteration in float64 on the branch sequence of an fp32 trajectory taken
                    in the kernel's operation order, with the margin of every accept/reject decision.
  * match_finalize  truncation and the strict distance test in float64 on inputs built so the fp32 distance is exact.
  * refine_matches  the fp16-emulating search (c10::Half: product and running sum each rounded to half): BIT-EXACT.
  * the reference's own kernels (oracle/_ref/mast3r_matching_ref.so) where they were built.

Bounds.  iter_proj positions agree with float64 within POS_TOL = 1e-4 px: a position below 128 carries an fp32 ulp of at
most 2^-17 px, and each of at most 10 accepted steps rounds it once (<= 10 half-ulps = 3.8e-5 px); the rest covers the
fp32 2x2 solve.  Decision flips: where an accept/reject decision of the float64 run lies within fp32 rounding of its
threshold (mr.cost_rounding_bound), an fp32 evaluation may take the other branch and continue along another trajectory;
such a point is excused only if it ends as good as the float64 one (its float64 cost within that bound of the reference's)
or the float64 run itself had not settled (not converged, or its last step exceeds POS_TOL: points pinned at a clamp
edge oscillate there),
and its flag may differ where ``conv_tie`` says it can.  Nothing else is excused, and every fp64-vs-fp32 disagreement of
the reference itself is shown to lie within the rounding bound.

Each group also builds its nearest plausible bug from oracle outputs and asserts that the comparison rejects it."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import matching_ref as mr

POS_TOL = 1e-4
HALF_MIN = 6.103515625e-05          # smallest normal half: what numeric_limits<Half>::min() would be if it were specialised
LAM0 = 1e-8


# ---- scene builders (CPU) ---------------------------------------------------------------------------------------------------
def _ray(u, v, h, w, ph):
    """A pinhole ray field with a low-frequency bend (per-batch phase ph), float64, unnormalised."""
    f = 0.9 * max(h, w)
    return torch.stack(((u - (w - 1) / 2) / f + 0.03 * torch.sin(0.4 * v + ph),
                        (v - (h - 1) / 2) / f + 0.03 * torch.cos(0.3 * u - ph), torch.ones_like(u)), -1)


def _proj_scene(b, h, w, n_pts, seed, margin=2.5):
    """X11 [b,h,w,3]: the ray field at a varying depth.  X21 [b,n_pts,3]: the field at targets spread over
    [-margin, W-1+margin] x [-margin, H-1+margin], so the optimum of many points is on or beyond a clamp edge.
    p_init [b,n_pts,2]: integer starts (du = dv = 0 at the first evaluation), some outside the image."""
    g = torch.Generator().manual_seed(seed)
    vv, uu = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64), indexing="ij")
    X11, X21, P = [], [], []
    for k in range(b):
        ph = 0.7 * k + 0.1 * seed
        depth = 2.0 + 0.5 * torch.rand(h, w, generator=g, dtype=torch.float64)
        X11.append(_ray(uu, vv, h, w, ph) * depth[..., None])
        tu = torch.rand(n_pts, generator=g, dtype=torch.float64) * (w - 1 + 2 * margin) - margin
        tv = torch.rand(n_pts, generator=g, dtype=torch.float64) * (h - 1 + 2 * margin) - margin
        X21.append(_ray(tu, tv, h, w, ph) * (1.5 + torch.rand(n_pts, generator=g, dtype=torch.float64))[:, None])
        su = torch.clamp(tu.round() + torch.randint(-2, 3, (n_pts,), generator=g), -2, w + 1)
        sv = torch.clamp(tv.round() + torch.randint(-2, 3, (n_pts,), generator=g), -2, h + 1)
        P.append(torch.stack((su, sv), -1))
    return torch.stack(X11).float(), torch.stack(X21).float(), torch.stack(P).float()


def _degenerate(X11, X21):
    """NaN and zero points in X21; NaN pixels in X11 (NaN rays, and NaN gradients around them)."""
    X11, X21 = X11.clone(), X21.clone()
    n = X21.shape[1]
    X21[:, 0:n:7] = float("nan")
    X21[:, 3:n:11] = 0.0
    X21[0, 5:n:13, 1] = float("nan")                 # one NaN component
    h, w = X11.shape[1:3]
    X11[0, h // 2, w // 2] = float("nan")
    X11[-1, 1, w - 2, 2] = float("nan")
    return X11, X21


def _flatten(X11, h0, h1, w0, w1):
    """A constant patch: its rays are equal, so the Scharr gradients inside it are exactly zero."""
    X11 = X11.clone()
    X11[:, h0:h1, w0:w1] = X11[:, h0:h0 + 1, w0:w0 + 1].clone()
    return X11


def _rays_pts(X11, X21):
    """Ray image and unit points from the float64 reference's formulas, rounded to fp32: the inputs both iter_proj
    implementations are fed."""
    rays, pts, _ = _prep64(X11, X21)
    return rays.float(), pts.float()


# ---- match_prep reference ---------------------------------------------------------------------------------------------------
def _unit64(X):
    """F.normalize(dim=-1, eps=1e-12) in float64 on an fp32 input, with the fp32 sum of squares' overflow: a point whose
    |x|^2 exceeds FLT_MAX has norm inf in fp32 (as F.normalize on a CUDA tensor, which accumulates in float) -> ray 0."""
    x = X.double()
    ss = (x * x).sum(-1, keepdim=True)
    n = torch.where(ss > torch.finfo(torch.float32).max, torch.full_like(ss, math.inf), ss.sqrt())
    return x / n.clamp_min(1e-12)


def _prep64(X11, X21):
    b, h, w, _ = X11.shape
    rays = _unit64(X11).permute(0, 3, 1, 2)
    gx, gy = mr.img_gradient(rays)
    return torch.cat((rays, gx, gy), 1).permute(0, 2, 3, 1).contiguous(), _unit64(X21.reshape(b, -1, 3)), None


def _lin_to_pixel_floor(li, w):
    """lin_to_pixel (torch % and //, which floor), as explicit Python integers."""
    return [(x % w, x // w) for x in li]


# ---- refine_matches reference with switchable bugs -----------------------------------------------------------------------------
def _refine(D11, D21, p1, radius, dil, ge=False, reset=False, v_outer=False, fixed_centre=False, fp32_sum=False, start=0.0):
    """mr.refine_matches restated with its visiting order and update rule as switches, so that each plausible bug is one
    flag away from the contract (all False == the reference)."""
    b, h, w, Fd = D11.shape
    n = p1.shape[1]
    bi = torch.arange(b)[:, None].expand(b, n)
    u0, v0 = p1[..., 0].clone(), p1[..., 1].clone()
    un, vn = u0.clone(), v0.clone()
    best = torch.full((b, n), start)
    q = D21.float()
    for d in range(dil, 0, -1):
        rd = radius * d
        if reset:
            best = torch.full((b, n), start)
        steps = range(0, 2 * rd + 1, d)
        order = [(i, j) for j in steps for i in steps] if v_outer else [(i, j) for i in steps for j in steps]
        I = torch.tensor([o[0] for o in order]) - rd
        J = torch.tensor([o[1] for o in order]) - rd
        u, v = u0[..., None] + I, v0[..., None] + J                                  # [b,n,C] in visiting order
        ok = (v >= 0) & (v < h) & (u >= 0) & (u < w)
        prod = q[:, :, None] * D11[bi[..., None], v.clamp(0, h - 1), u.clamp(0, w - 1)].float()
        s = torch.zeros(u.shape)
        for k in range(Fd):                 # the running sum, sequential over the feature dimension
            s = s + prod[..., k] if fp32_sum else (s + prod[..., k].half().float()).half().float()
        for c in range(len(order)):
            upd = ok[..., c] & ((s[..., c] >= best) if ge else (s[..., c] > best))
            best = torch.where(upd, s[..., c], best)
            un, vn = torch.where(upd, u[..., c], un), torch.where(upd, v[..., c], vn)
        if not fixed_centre:
            u0, v0 = un.clone(), vn.clone()
    return torch.stack((un, vn), -1)


def _centres(h, w, reach):
    """Every centre within reach + 2 of the image: each border and corner clips some window, and some centres lie at
    distance reach and beyond, where no candidate is inside."""
    vv, uu = torch.meshgrid(torch.arange(-reach - 2, h + reach + 2), torch.arange(-reach - 2, w + reach + 2), indexing="ij")
    return torch.stack((uu.reshape(-1), vv.reshape(-1)), -1)


def _refine_scene(F_, kind, seed, h=9, w=11, radius=3, dil=4):
    """D11 [2,h,w,F], D21 [2,n,F] fp16 and centres p1 [2,n,2] with n a multiple of 16 and != h*w.
    kind 'random': D21 = a nearby pixel's descriptor + noise.  'ties': D11 drawn from a 3-descriptor palette and D21 a
    palette entry, so equal scores are everywhere.  'floor': batch 0 scores < 0 everywhere; batch 1 scores exactly 0
    everywhere but at one pixel, whose score is the smallest positive half 2^-24: only windows reaching it move."""
    g = torch.Generator().manual_seed(seed)
    c = _centres(h, w, radius * dil)
    n = (c.shape[0] + 15) // 16 * 16
    c = torch.cat((c, c[: n - c.shape[0]]))
    p1 = torch.stack((c, c.flip(0)))
    if kind == "random":
        D11 = F.normalize(torch.randn(2, h, w, F_, generator=g), dim=-1)
        pu = (p1[..., 0] + torch.randint(-2, 3, (2, n), generator=g)).clamp(0, w - 1)
        pv = (p1[..., 1] + torch.randint(-2, 3, (2, n), generator=g)).clamp(0, h - 1)
        D21 = D11[torch.arange(2)[:, None], pv, pu] + 0.3 * torch.randn(2, n, F_, generator=g)
    elif kind == "ties":
        pal = F.normalize(torch.randn(3, F_, generator=g), dim=-1)
        D11 = pal[torch.randint(0, 3, (2, h, w), generator=g)]
        D21 = pal[torch.randint(0, 3, (2, n), generator=g)]
    else:
        D11 = torch.rand(2, h, w, F_, generator=g)
        D21 = torch.zeros(2, n, F_)
        D21[0] = -torch.rand(n, F_, generator=g)
        D11[1] = 0.0
        D11[1, h // 2, w // 2, 0] = 2.0 ** -12
        D21[1, :, 0] = 2.0 ** -12                     # product 2^-24: a subnormal half, > 0 but below HALF_MIN
    return D11.half().contiguous(), D21.half().contiguous(), p1.contiguous()


RD = [(0, 3), (3, 0), (1, 1), (3, 4), (4, 5), (2, 7)]


# ---- CPU: the references pinned ---------------------------------------------------------------------------------------------
def test_p_init_floor_division_pinned():
    """A linear index outside [0, H*W) maps as torch's lin_to_pixel maps it: floor division.  Explicit values for W = 5."""
    li = [-1, -5, -6, -11, 15, 17, 2 ** 40 + 3]
    assert _lin_to_pixel_floor(li, 5) == [(4, -1), (0, -1), (4, -2), (4, -3), (0, 3), (2, 3), (4, 219902325555)]
    X = torch.randn(1, 3, 5, 3)
    _, _, p = mr.prep_for_iter_proj(X, X, torch.tensor([li]))
    assert torch.equal(p[0], torch.tensor(_lin_to_pixel_floor(li, 5), dtype=torch.float32))
    # sensitivity: C's truncating / and % give (-1, 0) for -1 (then clamped to (1, 1), not (W-2, 1))
    neg = [-1, -6, -11]                                # (-5 is a multiple of W: both give (0, -1))
    trunc = [(int(math.fmod(x, 5)), int(x / 5)) for x in neg]
    assert all(a != b for a, b in zip(trunc, _lin_to_pixel_floor(neg, 5)))


def test_oracle_clamp_drops_nan_and_lambda_uses_a_double_literal():
    x = torch.tensor([float("nan"), -3.0, 0.5, 7.0, float("inf"), -float("inf")])
    assert torch.equal(mr._clamp(x, 1, 5), torch.tensor([1.0, 1.0, 1.0, 5.0, 5.0, 1.0]))
    lam = torch.tensor([LAM0, 1e-9, 3e-7, 1.0, 0.7], dtype=torch.float32)
    exact = torch.tensor([float(np.float32(float(np.float32(x)) * 0.1)) for x in lam.tolist()], dtype=torch.float32)
    assert torch.equal(mr.scale_lambda(lam, 0.1), exact)
    # the fp32 decay (lambda * 0.1f) rounds differently somewhere on the sequence the kernel walks from 1e-8
    seq, seq32, differs = torch.tensor([LAM0]), torch.tensor([LAM0]), False
    for _ in range(12):
        seq, seq32 = mr.scale_lambda(seq, 0.1), seq32 * torch.tensor(0.1, dtype=torch.float32)
        differs |= not torch.equal(seq, seq32)
    assert differs, "a planted fp32 lambda decay must be distinguishable"


def test_bilinear_weights_and_lm_step_formula():
    """The reference's bilinear weights (named after the opposite corner) are ordinary bilinear interpolation; one LM step
    is u + (J^T J + lambda I)^-1 J^T (-e) on the interpolated ray and gradients."""
    g = torch.Generator().manual_seed(0)
    img = torch.randn(1, 6, 7, 9, generator=g, dtype=torch.float64)
    u = torch.tensor([[1.0, 2.25, 3.5, 4.999, 5.0]], dtype=torch.float64)
    v = torch.tensor([[1.0, 3.75, 1.5, 2.0, 4.0]], dtype=torch.float64)
    got = mr._bilinear(img, u, v)
    u0, v0 = u.floor().long(), v.floor().long()
    du, dv = (u - u0)[..., None], (v - v0)[..., None]
    I = lambda vv, uu: img[0, vv[0], uu[0]][None]
    want = ((1 - du) * (1 - dv) * I(v0, u0) + du * (1 - dv) * I(v0, u0 + 1) + (1 - du) * dv * I(v0 + 1, u0) +
            du * dv * I(v0 + 1, u0 + 1))
    assert torch.allclose(got, want, rtol=0, atol=1e-12)
    # sensitivity: w12 and w21 swapped differs wherever du != dv
    swapped = ((1 - du) * (1 - dv) * I(v0, u0) + (1 - du) * dv * I(v0, u0 + 1) + du * (1 - dv) * I(v0 + 1, u0) +
               du * dv * I(v0 + 1, u0 + 1))
    assert ((swapped - want).abs().amax(-1) > 1e-3).sum() == 2
    # one step against a direct 2x2 solve
    X11, X21, P = _proj_scene(1, 12, 14, 64, seed=3, margin=-3.0)
    rays, pts = _rays_pts(X11, X21)
    r64, t64 = rays.double(), pts.double()
    uu, vv = mr._clamp(P[..., 0].double(), 1, 12), mr._clamp(P[..., 1].double(), 1, 10)
    lam = torch.full_like(uu, 1e-3)
    cost, un, vn, _ = mr._lm_step(r64, t64, uu, vv, lam, 14, 12)
    s = mr._bilinear(r64, uu, vv)
    e = s[..., 0:3] / s[..., 0:3].norm(dim=-1, keepdim=True) - t64
    J = torch.stack((s[..., 3:6], s[..., 6:9]), -1)                          # [b,n,3,2]
    A = J.transpose(-1, -2) @ J + 1e-3 * torch.eye(2, dtype=torch.float64)
    delta = torch.linalg.solve(A, -(J.transpose(-1, -2) @ e[..., None]))[..., 0]
    want_u = (uu + delta[..., 0]).clamp(1, 12)
    want_v = (vv + delta[..., 1]).clamp(1, 10)
    assert torch.allclose(cost, (e * e).sum(-1), rtol=1e-12, atol=0)
    assert torch.allclose(un, want_u, rtol=0, atol=1e-9) and torch.allclose(vn, want_v, rtol=0, atol=1e-9)


def _iter_proj_check(p, conv, ref, rays, pts):
    """Positions beyond POS_TOL, and flags that differ, that no decision flip explains.  A flip: the point had a decision
    within fp32 rounding (ref["tied"]) and its position is as good as the reference's, its float64 cost within
    cost_rounding_bound of the reference's final cost, or the reference's run was still moving when it
    stopped or had not converged.  A flag may also differ where ref["conv_tie"] says it can go
    either way, or where a flip put the point elsewhere.  Returns (error, bad position mask, bad flag mask)."""
    p = p.double().cpu()
    err = (p - ref["p"]).abs().amax(-1)
    c_ref = mr.cost_at(rays, pts, ref["p"])
    c_got = mr.cost_at(rays, pts, torch.where(torch.isfinite(p), p, ref["p"]))
    # a run still moving when it stops (last step > POS_TOL), or not converged, ends wherever the iteration count leaves
    # it: not a solution to compare
    flip = ref["tied"] & (((c_got - c_ref).abs() <= mr.cost_rounding_bound(torch.maximum(c_got, c_ref))) |
                          (ref["last_step"] > POS_TOL) | ~ref["conv"])
    bad_p = ~(err <= POS_TOL) & ~flip                                 # NaN is bad
    bad_c = (conv.cpu() != ref["conv"]) & ~ref["conv_tie"] & ~(flip & (err > POS_TOL))
    return err, bad_p, bad_c


def _iter_scene(name, seed=0):
    """(X11, X21, p_init) for each named iter_proj scene (n_pts never a multiple of 128)."""
    if name == "clamp":
        return _proj_scene(2, 24, 33, 1000, seed)
    if name == "flat":
        X11, X21, P = _proj_scene(2, 24, 33, 1000, seed, margin=0.0)
        P[:, :200] = torch.stack((torch.arange(200) % 8 + 2.0, torch.arange(200) // 8 % 8 + 2.0), -1)  # inside the patch
        return _flatten(X11, 0, 12, 0, 12), X21, P
    if name == "degenerate":
        X11, X21, P = _proj_scene(2, 24, 33, 1000, seed)
        return (*_degenerate(X11, X21), P)
    if name == "3x3":
        return _proj_scene(2, 3, 3, 200, seed)
    if name == "3xW":
        return _proj_scene(2, 3, 41, 500, seed)
    if name == "Hx3":
        return _proj_scene(2, 37, 3, 500, seed)
    raise KeyError(name)


SCENES = ["clamp", "flat", "degenerate", "3x3", "3xW", "Hx3"]


def _premises(name, X11, P, ref, rays):
    h, w = X11.shape[1:3]
    p = ref["p"]
    assert (P == P.round()).all()                                  # integer starts: du = dv = 0 at the first evaluation
    if name in ("clamp", "degenerate"):
        for k, bound in ((0, 1.0), (0, w - 2.0), (1, 1.0), (1, h - 2.0)):
            assert (p[..., k] == bound).sum() >= 3, f"{name}: no solution pinned at {'uv'[k]} = {bound}"
    if name == "flat":
        assert (rays[:, 1:11, 1:11, 3:] == 0).all(), "the flat patch must have exactly zero gradients"
    if name == "degenerate":
        assert torch.isnan(rays).any()
    if name == "3x3":
        assert (p == 1.0).all()


@pytest.mark.parametrize("name", SCENES)
def test_iter_proj_exact_vs_fp32_oracle(name):
    """The fp32 oracle (legacy op order) against the float64 reference; and every fp64/fp32 decision disagreement of the
    float64 reference itself lies within fp32 rounding of its threshold."""
    X11, X21, P = _iter_scene(name)
    rays, pts = _rays_pts(X11, X21)
    ref = mr.iter_proj_exact(rays, pts, P, 10, LAM0, 1e-6)
    _premises(name, X11, P, ref, rays)
    assert (ref["flip_ratio"] <= 1.0).all(), f"a flip beyond fp32 rounding: ratio {ref['flip_ratio'].max():.3g}"
    p32, c32 = mr.iter_proj(rays, pts, P, 10, LAM0, 1e-6)
    err, bad_p, bad_c = _iter_proj_check(p32, c32, ref, rays, pts)
    assert torch.isfinite(p32).all()
    assert not bad_p.any(), f"{int(bad_p.sum())} positions off, max err {err.max():.3g}"
    assert not bad_c.any(), f"{int(bad_c.sum())} flags off"


def test_iter_proj_sensitivity():
    """Planted bugs in the fp32 iteration are rejected by the comparison: swapped w12/w21, the clamp one pixel low
    ([0, W-2]), and a NaN-propagating clamp."""
    X11, X21, P = _iter_scene("degenerate")
    rays, pts = _rays_pts(X11, X21)
    ref = mr.iter_proj_exact(rays, pts, P, 10, LAM0, 1e-6)

    def run(**patch):
        saved = {k: getattr(mr, k) for k in patch}
        try:
            for k, f in patch.items():
                setattr(mr, k, f)
            return mr.iter_proj(rays, pts, P, 10, LAM0, 1e-6)
        finally:
            for k, f in saved.items():
                setattr(mr, k, f)

    bil, clp = mr._bilinear, mr._clamp

    def swapped(img, u, v):
        u11, v11 = torch.floor(u).long(), torch.floor(v).long()
        du, dv = u - u11.to(u.dtype), v - v11.to(v.dtype)
        bi = torch.arange(img.shape[0])[:, None]
        img = img.to(u.dtype)
        return ((du * dv)[..., None] * img[bi, v11 + 1, u11 + 1] + (du * (1 - dv))[..., None] * img[bi, v11 + 1, u11] +
                ((1 - du) * dv)[..., None] * img[bi, v11, u11 + 1] + ((1 - du) * (1 - dv))[..., None] * img[bi, v11, u11])

    for what, patch in (("swapped w12/w21", dict(_bilinear=swapped)),
                        ("clamp [0, W-2]", dict(_clamp=lambda x, lo, hi: clp(x, lo - 1, hi))),
                        ("NaN-propagating clamp", dict(_clamp=lambda x, lo, hi: x.clamp(lo, hi)))):
        try:
            p, c = run(**patch)
        except (IndexError, RuntimeError):
            continue                       # a NaN position cannot even index the image: rejected
        _, bad_p, bad_c = _iter_proj_check(p, c, ref, rays, pts)
        assert (bad_p | bad_c).sum() >= 10, f"planted bug not caught: {what}"
    assert bil is mr._bilinear and clp is mr._clamp


def test_refine_emulation_matches_oracle_and_each_bug_is_caught():
    """_refine with every switch off is mr.refine_matches; each switch (>= ties, max_score reset per dilation, v outer,
    centre never moved, fp32 running sum) changes the answer on its scene, which also proves the scene reaches the edge:
    equal scores exist where the first-visited candidate wins, and the fp16 running sum rounds away from the fp32 one."""
    for kind in ("random", "ties", "floor"):
        D11, D21, p1 = _refine_scene(24, kind, seed=1)
        assert torch.equal(_refine(D11, D21, p1, 3, 4), mr.refine_matches(D11, D21, p1, 3, 4))
    D11, D21, p1 = _refine_scene(32, "ties", seed=2)
    want = _refine(D11, D21, p1, 3, 4)
    for flag in ("ge", "reset", "v_outer", "fixed_centre"):
        assert not torch.equal(_refine(D11, D21, p1, 3, 4, **{flag: True}), want), f"tie scene misses the {flag} bug"
    D11, D21, p1 = _refine_scene(32, "random", seed=3)
    assert not torch.equal(_refine(D11, D21, p1, 4, 5, fp32_sum=True), _refine(D11, D21, p1, 4, 5)), \
        "no fp16-vs-fp32 rounding difference reached the winner"
    D11, D21, p1 = _refine_scene(16, "floor", seed=4)
    got = _refine(D11, D21, p1, 3, 4)
    assert torch.equal(got[0], p1[0]), "scores <= 0 must keep the input"
    h, w = D11.shape[1:3]
    moved = (got[1] != p1[1]).any(-1)
    assert moved.any() and (got[1][moved] == torch.tensor([w // 2, h // 2])).all(), "the 2^-24 score must win"
    assert not torch.equal(_refine(D11, D21, p1, 3, 4, start=HALF_MIN), got)   # a HALF_MIN start keeps it
    assert not torch.equal(_refine(D11, D21, p1, 3, 4, ge=True), got)          # '>=' moves onto the 0 scores


# ---- GPU -------------------------------------------------------------------------------------------------------------------------
def _ref_module():
    from oracle import build_ref
    try:
        return build_ref.load("mast3r_matching_ref")
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"reference extension unavailable: {e}")


def _ref_call(fn, n_pts, *args):
    """The reference kernels launch 16-thread blocks with no n < n_pts check: only a multiple of 16 stays in bounds."""
    assert n_pts % 16 == 0, f"reference build called with n_pts = {n_pts}"
    out = fn(*args)
    torch.cuda.synchronize()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("hw", [(2, 2), (3, 3), (5, 5), (2, 129), (129, 3), (129, 129)])
def test_match_prep_vs_fp64(cuda, hw):
    from artdeco_b200 import matching as M
    h, w = hw
    g = torch.Generator().manual_seed(h * 1000 + w)
    X11 = torch.randn(3, h, w, 3, generator=g) * torch.tensor([1.0, 10.0, 0.1]).view(3, 1, 1, 1)   # content per batch
    X21 = torch.randn(3, h, w, 3, generator=g)
    mag = [0.0, 1e-30, 1e30, 5e-13, 1e18]
    for k, m in enumerate(mag):                       # exactly zero, 1e-30 (norm < eps), 1e30 (|x|^2 overflows fp32) ...
        X11[k % 3, (k * 7) % h, (k * 5) % w] = m * torch.tensor([0.6, -0.8, 0.0]) if m else 0.0
        X21[k % 3, (k * 3) % h, (k * 2) % w] = m * torch.tensor([0.0, 0.6, 0.8]) if m else 0.0
    n = h * w
    li = torch.randint(-3 * n, 3 * n, (3, n), generator=g)
    li[0, :6] = torch.tensor([-1, -w, -w - 1, n, n + 1, 2 ** 40 + 3])[: min(6, n)]
    rays, pts, p = M.prep_for_iter_proj(X11.to(cuda), X21.to(cuda), li.to(cuda))
    rays_e, pts_e, _ = _prep64(X11, X21)
    # |rays|, |pts| <= 1: a few fp32 roundings of a unit value; gradients sum six of them with weights <= 10/32
    err_r = (rays[..., :3].cpu().double() - rays_e[..., :3]).abs()
    err_g = (rays[..., 3:].cpu().double() - rays_e[..., 3:]).abs()
    assert err_r.max() <= 1e-6 and err_g.max() <= 2e-6, (err_r.max(), err_g.max())
    assert (pts.cpu().double() - pts_e).abs().max() <= 1e-6
    # the border rows and columns (reflect padding) are where the stencil changes, and were compared above: reflection
    # makes the derivative across a border exactly 0, the one along it is not (given 3 or more pixels to difference)
    assert rays[:, [0, -1]][..., 6:].abs().max() <= 2e-6 and rays[:, :, [0, -1]][..., 3:6].abs().max() <= 2e-6
    if w >= 3:
        assert rays_e[:, [0, -1]][..., 3:6].abs().amax() > 0.01
    if h >= 3:
        assert rays_e[:, :, [0, -1]][..., 6:].abs().amax() > 0.01
    # the degenerate magnitudes: 0 -> 0, 1e-30 -> x / 1e-12, 1e30 -> 0 (fp32 overflow), as F.normalize does on the GPU
    assert torch.equal(F.normalize(X11.to(cuda), dim=-1).isnan(), torch.zeros_like(X11, dtype=torch.bool, device=cuda))
    assert (rays[..., :3] - F.normalize(X11.to(cuda), dim=-1)).abs().max() <= 1e-6
    want = torch.tensor([_lin_to_pixel_floor(row, w) for row in li.tolist()], dtype=torch.float32)
    assert torch.equal(p.cpu(), want), "p_init must be lin_to_pixel's floor division, exactly"
    assert (li < 0).any() and (li >= n).any()


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCENES)
@pytest.mark.parametrize("max_iter", [0, 1, 2, 10])
def test_iter_proj_vs_fp64(cuda, name, max_iter):
    from artdeco_b200 import matching as M
    X11, X21, P = _iter_scene(name, seed=max_iter)
    rays, pts = _rays_pts(X11, X21)
    thr = 1e-6
    if name == "clamp" and max_iter == 10:
        # a threshold equal to one point's final cost: its flag hinges on the strict '<' within one ulp
        cc = mr.iter_proj_exact(rays, pts, P, max_iter, LAM0, thr)["cost"]
        fin = cc[torch.isfinite(cc) & (cc > 1e-9)]
        thr = float(np.float32(fin.median()))
    ref = mr.iter_proj_exact(rays, pts, P, max_iter, LAM0, thr)
    if max_iter == 10:
        _premises(name, X11, P, ref, rays)
    if name == "clamp" and max_iter == 10:
        ulp = float(np.spacing(np.float32(thr)))
        assert ((ref["cost"] - thr).abs() <= ulp).any(), "no final cost within one ulp of cost_thresh"
    p, conv = M.iter_proj(rays.to(cuda), pts.to(cuda), P.to(cuda), max_iter, LAM0, thr)
    assert torch.isfinite(p).all(), "a NaN input must end on the clamped position, never NaN"
    err, bad_p, bad_c = _iter_proj_check(p, conv, ref, rays, pts)
    assert not bad_p.any(), f"{int(bad_p.sum())} positions beyond POS_TOL, not flips (max err {err[bad_p].max():.3g})"
    assert not bad_c.any(), f"{int(bad_c.sum())} convergence flags differ outside a rounding tie"
    if max_iter == 0:
        assert torch.equal(p.cpu(), ref["p"].float()) and not conv.any()
    nan_pts = torch.isnan(pts).any(-1)
    if nan_pts.any():                                    # NaN cost: every step is rejected, the start is kept exactly
        assert torch.equal(p.cpu()[nan_pts], ref["p"].float()[nan_pts]) and not conv.cpu()[nan_pts].any()
    print(f"[iter_proj {name} it={max_iter}] max err {err.max():.3g} px, flips over 1e-4 {int((err > POS_TOL).sum())}, "
          f"flag ties {int((conv.cpu() != ref['conv']).sum())}, fp64/fp32 flips {int(ref['flip'].sum())}")


@pytest.mark.gpu
def test_match_finalize_exact(cuda):
    from artdeco_b200 import _lib, matching as M  # noqa: F401
    b, h, w = 2, 6, 7
    n = h * w
    g = torch.Generator().manual_seed(0)
    thr = float(np.float32(0.1))
    up, dn = float(np.nextafter(np.float32(thr), np.float32(1))), float(np.nextafter(np.float32(thr), np.float32(0)))
    k = torch.randint(1, 5, (b, n, 2), generator=g).float()
    up1 = lambda x: float(np.nextafter(np.float32(x), np.float32(np.inf)))
    dn1 = lambda x: float(np.nextafter(np.float32(x), np.float32(-np.inf)))
    p = k.clone()
    for i in range(n):                                  # k, k + 1 ulp, k - 1 ulp, k + 0.5, k + 0.75, k + 1 - 2^-20
        for c in range(2):
            kk = float(k[0, i, c])
            p[:, i, c] = [kk, up1(kk), dn1(kk), kk + 0.5, kk + 0.75, kk + 1 - 2.0 ** -20][(i + 3 * c) % 6]
    p1 = p.double().trunc().long()
    X11 = torch.zeros(b, h, w, 3)
    X11[..., 1:] = torch.randn(b, h, w, 2, generator=g)
    dist = torch.tensor([thr, up, dn, 0.0, 2 * thr, 0.5 * thr])[(torch.arange(n) * 5 // 3) % 6]
    bi = torch.arange(b)[:, None]
    X21 = X11[bi, p1[..., 1], p1[..., 0]].clone()        # [b, n, 3]
    X21[..., 0] = -dist                                  # |X11[p1] - X21| == dist exactly in fp32
    conv = (torch.arange(n) % 2 == 0).expand(b, n).clone()
    conv[1] = ~conv[1]
    d64 = (X11[bi, p1[..., 1], p1[..., 0]].double() - X21.double()).norm(dim=-1)
    want_valid = conv & (d64 < thr)
    # premises: every boundary case is present, with both flag values
    for dd in (thr, up, dn):
        assert ((d64 == dd) & conv).any() and ((d64 == dd) & ~conv).any()
    assert (p == p.floor()).any() and (p - p.floor() == 0.5).any() and (p.frac() > 0.9999).any()
    out_p1 = torch.empty(b, n, 2, dtype=torch.int64, device=cuda)
    valid = torch.empty(b, n, dtype=torch.bool, device=cuda)
    Xa, Xb, pc, cc = (t.to(cuda).contiguous() for t in (X11, X21.reshape(b, h, w, 3), p, conv))
    _lib.call("adb_match_finalize", b, h, w, _lib.ptr(Xa), _lib.ptr(Xb), _lib.ptr(pc), _lib.ptr(cc), thr,
              _lib.ptr(out_p1), _lib.ptr(valid), _lib.stream())
    assert torch.equal(out_p1.cpu(), p1) and torch.equal(valid.cpu(), want_valid)
    # sensitivity: rounding instead of truncation, and '<=' instead of '<'
    assert not torch.equal(p.double().round().long(), p1)
    assert not torch.equal(conv & (d64 <= thr), want_valid)


def _refine_gpu(M, _lib, D11, D21, p1, radius, dil, planar, cuda):
    b, h, w, F_ = D11.shape
    n = p1.shape[1]
    if not planar:
        out, lin = M.refine_matches(D11.to(cuda), D21.to(cuda), p1.to(cuda), radius, dil, return_linear=True)
        return out.cpu(), lin.cpu()
    a, _ = M._pack_f16(D11.float().to(cuda), b, h * w)
    q, _ = M._pack_f16(D21.float().to(cuda), b, n)
    out = torch.empty(b, n, 2, dtype=torch.int64, device=cuda)
    lin = torch.empty(b, n, dtype=torch.int64, device=cuda)
    pc = p1.to(cuda).contiguous()
    _lib.call("adb_refine_matches", b, h, w, F_, n, _lib.ptr(a), _lib.ptr(q), 1, _lib.ptr(pc), radius, dil, _lib.ptr(out),
              _lib.ptr(lin), _lib.stream())
    return out.cpu(), lin.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("F_", [16, 24, 32])
@pytest.mark.parametrize("kind", ["random", "ties", "floor"])
def test_refine_matches_bit_exact_every_layout(cuda, F_, kind):
    from artdeco_b200 import _lib, matching as M
    for radius, dil in RD:
        D11, D21, p1 = _refine_scene(F_, kind, seed=F_ + radius * 10 + dil, radius=max(radius, 1), dil=max(dil, 1))
        assert p1.shape[1] != D11.shape[1] * D11.shape[2]
        want = mr.refine_matches(D11, D21, p1, radius, dil)
        for planar in (0, 1):
            out, lin = _refine_gpu(M, _lib, D11, D21, p1, radius, dil, planar, cuda)
            assert torch.equal(out, want), f"F={F_} {kind} r={radius} d={dil} planar={planar}"
            assert torch.equal(lin, out[..., 0] + D11.shape[2] * out[..., 1])
        if kind == "floor" or dil == 0:
            assert torch.equal(want[0], p1[0])


@pytest.mark.gpu
def test_refine_planar_at_full_image(cuda):
    """The fused flow's call: planar layout with n_pts == H*W (D21 packed over every pixel), at each F."""
    from artdeco_b200 import _lib, matching as M
    for F_ in (16, 24, 32):
        g = torch.Generator().manual_seed(F_)
        h, w = 13, 17
        D11 = F.normalize(torch.randn(2, h, w, F_, generator=g), dim=-1).half()
        D21 = (D11.reshape(2, h * w, F_).float() + 0.4 * torch.randn(2, h * w, F_, generator=g)).half()
        p1 = torch.stack((torch.randint(-3, w + 3, (2, h * w), generator=g), torch.randint(-3, h + 3, (2, h * w), generator=g)), -1)
        want = mr.refine_matches(D11, D21, p1, 2, 3)
        for planar in (0, 1):
            out, _ = _refine_gpu(M, _lib, D11, D21, p1, 2, 3, planar, cuda)
            assert torch.equal(out, want), (F_, planar)


@pytest.mark.gpu
@pytest.mark.parametrize("F_", [16, 24, 32])
def test_desc_pack_f16_bit_equal(cuda, F_):
    from artdeco_b200 import matching as M
    g = torch.Generator().manual_seed(F_)
    b, n = 2, 37
    D = torch.randn(b, n, F_, generator=g) * 100.0
    special = torch.tensor([65504.0, 65519.0, 65520.0, 1e5, -1e5, -65520.0, 2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -26, 1e-6,
                            -1e-7, 6.0e-5, -0.0, 0.0, float("nan"), float("inf"), -float("inf")])
    D.view(-1)[: special.numel()] = special
    D.view(-1)[-special.numel():] = special
    out, fd = M._pack_f16(D.to(cuda), b, n)
    assert fd == F_
    want = D.half().reshape(b, n, F_ // 8, 8).permute(0, 2, 1, 3).reshape(-1)
    got = out.cpu()
    nan = torch.isnan(want)
    assert nan.any() and torch.equal(torch.isnan(got), nan)
    assert torch.equal(got.view(torch.int16)[~nan], want.view(torch.int16)[~nan]), "pack must be bit-equal to .half()"
    assert torch.isinf(want).sum() >= 8 and (want.view(torch.int16) == -32768).any()          # inf and -0.0 present
    assert ((want != 0) & (want.abs() < HALF_MIN)).any()                                      # subnormals present


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["clamp", "flat", "degenerate", "Hx3"])
def test_iter_proj_vs_reference_build(cuda, name):
    """The reference's own iter_proj (--use_fast_math) on the edge scenes, held to the float64 reference's bound."""
    ref_mod = _ref_module()
    X11, X21, P = _iter_scene(name)
    n = P.shape[1] // 16 * 16
    P = P[:, :n].contiguous()
    rays, pts = _rays_pts(X11, X21[:, :n])
    ref = mr.iter_proj_exact(rays, pts, P, 10, LAM0, 1e-6)
    p_r, conv_r = _ref_call(ref_mod.iter_proj, n, rays.to(cuda), pts.to(cuda), P.to(cuda), 10, LAM0, 1e-6)
    err, bad_p, bad_c = _iter_proj_check(p_r, conv_r, ref, rays, pts)
    assert torch.isfinite(p_r).all()
    assert not bad_p.any(), f"reference build: {int(bad_p.sum())} positions off (max err {err.max():.3g})"
    assert not bad_c.any(), f"reference build: {int(bad_c.sum())} flags off"


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["random", "ties", "floor"])
def test_refine_matches_vs_reference_build(cuda, kind):
    from artdeco_b200 import matching as M
    ref_mod = _ref_module()
    for F_ in (16, 24, 32):
        for radius, dil in RD:
            D11, D21, p1 = _refine_scene(F_, kind, seed=7 * F_ + radius + dil, radius=max(radius, 1), dil=max(dil, 1))
            D11, D21, p1 = D11.to(cuda), D21.to(cuda), p1.to(cuda)
            (theirs,) = _ref_call(ref_mod.refine_matches, p1.shape[1], D11, D21, p1, radius, dil)
            (mine,) = M.refine_matches(D11, D21, p1, radius, dil)
            assert torch.equal(mine, theirs), f"F={F_} {kind} r={radius} d={dil}"

"""TEST INFRASTRUCTURE ONLY — never imported by the product path.

CPU/GPU-agnostic PyTorch restatement of the reference's dense matching step:
  * ``prep_for_iter_proj``  VSLAM/utils_matching.py:59-97,120-145 (this is the reference's own PyTorch code path, restated);
  * ``iter_proj``           VSLAM/backend/src/matching_kernels.cu:119-276, vectorised over points (fp32, the reference's
                            operation order; the reference build adds --use_fast_math, VSLAM/setup.py:62-67), with its
                            NaN-dropping clamp and its double-literal lambda update;
  * ``iter_proj_exact``     the same iteration in float64 on the fp32 trajectory's decisions, with the margin of each;
  * ``refine_matches``      matching_kernels.cu:26-83 with c10::Half semantics (product and running sum rounded to fp16,
                            sequential over the feature dimension; max_score starts at ::cuda::std::numeric_limits<c10::Half>::min(),
                            which libcu++ leaves unspecialised: Half() == 0);
  * ``match_iterative_proj``utils_matching.py:148-190.
PINNED on the GPU box against the reference's OWN kernels: oracle/build_ref.py compiles matching_kernels.cu where it lies
into oracle/_ref/mast3r_matching_ref.so (tests/test_matching.py::test_matches_the_reference_cuda_build).  The reference
holds no tests or vectors for this path.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def img_gradient(img):
    b, c, h, w = img.shape
    kx = (1.0 / 32.0) * torch.tensor([[-3.0, 0.0, 3.0], [-10.0, 0.0, 10.0], [-3.0, 0.0, 3.0]], dtype=img.dtype, device=img.device)
    ky = kx.t().contiguous()
    pad = F.pad(img, (1, 1, 1, 1), mode="reflect")
    return (F.conv2d(pad, kx.repeat(c, 1, 1, 1), groups=c), F.conv2d(pad, ky.repeat(c, 1, 1, 1), groups=c))


def prep_for_iter_proj(X11, X21, idx_init=None):
    b, h, w, _ = X11.shape
    rays = F.normalize(X11, dim=-1).permute(0, 3, 1, 2)
    gx, gy = img_gradient(rays)
    rays_grad = torch.cat((rays, gx, gy), 1).permute(0, 2, 3, 1).contiguous()
    pts = F.normalize(X21.reshape(b, -1, 3), dim=-1)
    if idx_init is None:
        idx_init = torch.arange(h * w, device=X11.device)[None].repeat(b, 1)
    p_init = torch.stack((idx_init % w, idx_init // w), -1).to(X11.dtype)
    return rays_grad, pts, p_init


def _bilinear(img, u, v):
    """img [b,h,w,c]; u,v [b,n] -> [b,n,c] with the reference's weights (matching_kernels.cu:153-170): w11 = du dv multiplies
    the pixel at (u11 + 1, v11 + 1), i.e. each weight is named after the corner OPPOSITE the one it multiplies.  Computed
    in u's dtype; an fp32 image is widened when u is float64."""
    b = img.shape[0]
    u11, v11 = torch.floor(u).long(), torch.floor(v).long()
    du, dv = u - u11.to(u.dtype), v - v11.to(v.dtype)
    bi = torch.arange(b, device=img.device)[:, None]
    img = img.to(u.dtype)
    w11, w12, w21, w22 = du * dv, (1 - du) * dv, du * (1 - dv), (1 - du) * (1 - dv)
    return (w11[..., None] * img[bi, v11 + 1, u11 + 1] + w12[..., None] * img[bi, v11 + 1, u11] +
            w21[..., None] * img[bi, v11, u11 + 1] + w22[..., None] * img[bi, v11, u11])


def _clamp(x, lo, hi):
    """fmin(fmax(x, lo), hi), the reference's clamp (matching_kernels.cu:21-23): a NaN lands on lo.  torch.clamp keeps NaN."""
    return torch.where(torch.isnan(x), torch.full_like(x, lo), x.clamp(lo, hi))


def scale_lambda(lam, s):
    """``lambda *= 0.1`` / ``*= 10.0`` on a float lambda: the literal is a double, so the product is formed in double and
    rounded to float once (matching_kernels.cu:262, 266)."""
    return (lam.double() * s).float()


def _dot3(a, b):
    return a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1] + a[..., 2] * b[..., 2]


def _unit(r, recip):
    if recip:      # the kernel's and the reference's r * (1 / sqrt(r.r))
        return r * (1.0 / torch.sqrt(_dot3(r, r)))[..., None]
    return r / r.norm(dim=-1, keepdim=True)


def _lm_step(img, pts, u, v, lam, w, h, recip=True):
    """One LM iteration in u's dtype and, with ``recip``, in the kernel's operation order: (cost at u, candidate un, vn,
    cost at the candidate)."""
    s = _bilinear(img, u, v)
    r, gx, gy = s[..., 0:3], s[..., 3:6], s[..., 6:9]
    e = _unit(r, recip) - pts
    cost = _dot3(e, e)
    A00, A01, A11 = _dot3(gx, gx) + lam, _dot3(gx, gy), _dot3(gy, gy) + lam
    b0, b1 = -_dot3(e, gx), -_dot3(e, gy)
    det_inv = 1.0 / (A00 * A11 - A01 * A01)
    un = _clamp(u + det_inv * (A11 * b0 - A01 * b1), 1, w - 2)
    vn = _clamp(v + det_inv * (-A01 * b0 + A00 * b1), 1, h - 2)
    a = _bilinear(img[..., 0:3], un, vn)
    f = _unit(a, recip) - pts
    return cost, un, vn, _dot3(f, f)


def iter_proj(rays_grad, pts, p_init, max_iter, lambda_init, cost_thresh):
    """fp32.  Rays are renormalised with a division where the kernel multiplies by a reciprocal (<= 1 ulp apart); on an
    exact self-match the division returns each unit ray unchanged, so an integer start stays put."""
    b, h, w, _ = rays_grad.shape
    u = _clamp(p_init[..., 0].float(), 1, w - 2)
    v = _clamp(p_init[..., 1].float(), 1, h - 2)
    lam = torch.full_like(u, lambda_init)
    conv = torch.zeros_like(u, dtype=torch.bool)     # the reference's output starts false and each iteration overwrites it
    for _ in range(max_iter):
        cost, un, vn, new_cost = _lm_step(rays_grad, pts, u, v, lam, w, h, recip=False)
        better = new_cost < cost
        u, v = torch.where(better, un, u), torch.where(better, vn, v)
        lam = torch.where(better, scale_lambda(lam, 0.1), scale_lambda(lam, 10.0))
        conv = torch.where(better, new_cost < cost_thresh, cost < cost_thresh)
    return torch.stack((u, v), -1), conv


def cost_rounding_bound(c):
    """How far an fp32 evaluation of a cost |n(r) - t|^2 (n: normalise) can stray from its exact value.  Each component of
    n(r) - t carries <= 8 units of fp32 roundoff u (four-term bilinear sum, sqrt, divide, multiply, subtract), so the cost
    is off by <= 2 sqrt(3 c) 8u + 4 c u.  A comparison of two costs doubles that; a further 4x covers the approximate sqrt of
    a --use_fast_math build and FMA contraction: 256 u (sqrt(c) + c)."""
    return 256.0 * 2.0 ** -24 * (torch.sqrt(c) + c)


def cost_at(rays_grad, pts, p):
    """float64 cost |n(ray(p)) - t|^2 at positions p [b,n,2]."""
    a = _bilinear(rays_grad[..., 0:3], p[..., 0].double(), p[..., 1].double())
    e = a / a.norm(dim=-1, keepdim=True) - pts.double()
    return (e * e).sum(-1)


def iter_proj_exact(rays_grad, pts, p_init, max_iter, lambda_init, cost_thresh):
    """float64 iter_proj.  Positions, steps and costs are float64; each accept/reject decision is the one an fp32
    trajectory run alongside in the kernel's operation order takes, so both follow the branch sequence the kernel follows.

    Returns a dict:
      p, conv       float64 positions [b,n,2] and the convergence flag (float64 costs against fp32(cost_thresh));
      cost          float64 cost the last flag was decided on;
      p32, conv32   the fp32 trajectory;
      flip          some float64 decision disagreed with the fp32 one;
      flip_ratio    max over those decisions of |cost - new_cost| / cost_rounding_bound (<= 1: within fp32 rounding);
      tied          some decision lay within cost_rounding_bound: an fp32 evaluation may take either branch there and
                    go on along another, equally valid trajectory;
      last_step     float64 length of the last iteration's candidate step: a run still moving when it stops (a point
                    pinned at a clamp edge oscillates there) ends wherever the iteration count leaves it;
      conv_tie      the last iteration's flag can go either way in fp32 (its compared cost is within rounding of
                    cost_thresh, or its decision is a tie whose branches give different flags)."""
    b, h, w, _ = rays_grad.shape
    thr = float(torch.tensor(cost_thresh, dtype=torch.float32))
    img32, img64 = rays_grad.float(), rays_grad.double()
    t32, t64 = pts.float(), pts.double()
    u32 = _clamp(p_init[..., 0].float(), 1, w - 2)
    v32 = _clamp(p_init[..., 1].float(), 1, h - 2)
    u64, v64 = u32.double(), v32.double()
    lam = torch.full_like(u32, lambda_init)
    conv32 = torch.zeros_like(u32, dtype=torch.bool)
    conv64 = torch.zeros_like(conv32)
    conv_tie = torch.zeros_like(conv32)
    flip = torch.zeros_like(conv32)
    flip_ratio = torch.zeros_like(u64)
    tied = torch.zeros_like(conv32)
    last_step = torch.zeros_like(u64)
    cc = torch.full_like(u64, float("nan"))
    for _ in range(max_iter):
        c32, un32, vn32, n32 = _lm_step(img32, t32, u32, v32, lam, w, h)
        c64, un64, vn64, n64 = _lm_step(img64, t64, u64, v64, lam.double(), w, h)
        acc = n32 < c32
        bound = cost_rounding_bound(torch.maximum(c64, n64))
        margin = (c64 - n64).abs()
        tie = margin <= bound
        fl = acc != (n64 < c64)
        flip |= fl
        flip_ratio = torch.where(fl, torch.maximum(flip_ratio, margin / bound), flip_ratio)
        tied |= tie
        last_step = torch.hypot(un64 - u64, vn64 - v64)
        u32, v32 = torch.where(acc, un32, u32), torch.where(acc, vn32, v32)
        u64, v64 = torch.where(acc, un64, u64), torch.where(acc, vn64, v64)
        lam = torch.where(acc, scale_lambda(lam, 0.1), scale_lambda(lam, 10.0))
        conv32 = torch.where(acc, n32 < thr, c32 < thr)
        conv64 = torch.where(acc, n64 < thr, c64 < thr)
        cc = torch.where(acc, n64, c64)
        conv_tie = ((cc - thr).abs() <= cost_rounding_bound(cc)) | (tie & ((n64 < thr) != (c64 < thr)))
    return dict(p=torch.stack((u64, v64), -1), conv=conv64, cost=cc, p32=torch.stack((u32, v32), -1), conv32=conv32, flip=flip,
                flip_ratio=flip_ratio, tied=tied, last_step=last_step, conv_tie=conv_tie)


def refine_matches(D11, D21, p1, radius, dilation_max):
    """D11 [b,h,w,F] fp16, D21 [b,n,F] fp16, p1 int64 [b,n,2].  fp16 arithmetic emulated step by step."""
    b, h, w, Fd = D11.shape
    n = p1.shape[1]
    dev = D11.device
    bi = torch.arange(b, device=dev)[:, None].expand(b, n)
    u0, v0 = p1[..., 0].clone(), p1[..., 1].clone()
    u_new, v_new = u0.clone(), v0.clone()
    max_score = torch.zeros((b, n), dtype=torch.float32, device=dev)   # numeric_limits<c10::Half>::min(): unspecialised, 0
    q = D21.float()
    for d in range(dilation_max, 0, -1):
        rd = radius * d
        for i in range(0, 2 * rd + 1, d):
            for j in range(0, 2 * rd + 1, d):
                u, v = u0 - rd + i, v0 - rd + j
                ok = (v >= 0) & (v < h) & (u >= 0) & (u < w)
                c = D11[bi, v.clamp(0, h - 1), u.clamp(0, w - 1)].float()
                s = torch.zeros(b, n, dtype=torch.float32, device=dev)
                for k in range(Fd):
                    prod = (q[..., k] * c[..., k]).half().float()
                    s = (s + prod).half().float()
                upd = ok & (s > max_score)
                max_score = torch.where(upd, s, max_score)
                u_new, v_new = torch.where(upd, u, u_new), torch.where(upd, v, v_new)
        u0, v0 = u_new.clone(), v_new.clone()
    return torch.stack((u_new, v_new), -1)


def match_iterative_proj(cfg, X11, X21, D11, D21, idx_init=None):
    b, h, w = X21.shape[:3]
    rays_grad, pts, p_init = prep_for_iter_proj(X11, X21, idx_init)
    p, conv = iter_proj(rays_grad, pts, p_init, cfg["max_iter"], cfg["lambda_init"], cfg["convergence_thresh"])
    p1 = p.long()
    bi = torch.arange(b, device=X11.device)[:, None].repeat(1, h * w)
    d = torch.linalg.norm(X11[bi, p1[..., 1], p1[..., 0], :].reshape(b, h, w, 3) - X21, dim=-1)
    valid = conv & (d < cfg["dist_thresh"]).view(b, -1)
    if cfg["radius"] > 0:
        p1 = refine_matches(D11.half(), D21.reshape(b, h * w, -1).half(), p1, cfg["radius"], cfg["dilation_max"])
    return p1[..., 0] + w * p1[..., 1], valid.unsqueeze(-1), p, p1

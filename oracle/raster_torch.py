"""TEST INFRASTRUCTURE ONLY — never imported by the product path.

Pure-PyTorch, differentiable restatement of the renderer the reference calls at
Reconstruct/scene/scene_models/h3dgsv3.py:664-680 (``gsplat.rendering.rasterization`` with
render_mode="RGB+D", rasterize_mode="classic", packed=False, sh_degree=3, eps2d=0.01).

gsplat is a pip dependency that is NOT vendored in /root/reference and not installable offline
(README.md:82, unpinned; >=1.5 inferred from meta['radii'] having two columns, h3dgsv3.py:689), so this
file restates the published algorithm (SURVEY.md Appendix B).  PARITY UNPINNED: no reference test or
golden vector exists for the renderer.  Its only job is to let torch.autograd produce gradients that
pin the analytic backward of the C oracle (oracle/raster_oracle.c) at tiny sizes.
Per-pixel Python loops: use W*H <= ~64*64 and N <= ~200.
"""
from __future__ import annotations

import math

import torch

ALPHA_THRESHOLD = 1.0 / 255.0
MAX_ALPHA = 0.999
T_EPS = 1e-4
TILE = 16

SH_C0 = 0.2820947917738781
SH_C1 = 0.48860251190292


MUTATIONS = ("fxfy_J", "lx_swap", "band_unclamped", "no_dotq", "no_qinv")


def quat_to_rotmat(q: torch.Tensor, mutation: str | None = None) -> torch.Tensor:
    n = q.norm(dim=-1, keepdim=True)
    if mutation == "no_dotq":      # same value; gradient v/|q| instead of (v - <v,q^> q^)/|q|
        q = (q / n).detach() + (q - q.detach()) / n.detach()
    elif mutation == "no_qinv":    # same value; gradient (v - <v,q^> q^) without the 1/|q|
        qn = q / n
        q = qn.detach() + (qn - qn.detach()) * n.detach()
    else:
        q = q / n
    w, x, y, z = q.unbind(-1)
    return torch.stack([
        1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
        2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
        2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], dim=-1).reshape(-1, 3, 3)


def project(means, quats, scales, opacities, viewmat, K, W, H, eps2d=0.01, near=0.01, far=1e10, radius_clip=0.0,
            mutation=None):
    """Returns radii[N,2] (int32), means2d[N,2], depths[N], conics[N,3] (differentiable where defined).

    ``mutation`` (one of MUTATIONS) plants a known bug, so that tests can show they would catch it: fx and fy swapped
    in the Jacobian; the guard-band limits lxp and lxn swapped; the unclamped derivative of the Jacobian used in the
    guard band; the quaternion normalisation backward without its ``- <v,q^> q^`` term or without its ``1/|q|``."""
    assert mutation is None or mutation in MUTATIONS, mutation
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    R, t = viewmat[:3, :3], viewmat[:3, 3]
    p = means @ R.T + t
    x, y, z = p.unbind(-1)
    Rq = quat_to_rotmat(quats, mutation)
    M = Rq * scales[:, None, :]
    Sigma = M @ M.transpose(1, 2)
    Sc = R @ Sigma @ R.T
    tanx, tany = 0.5 * W / fx, 0.5 * H / fy
    lxp, lxn = (W - cx) / fx + 0.3 * tanx, cx / fx + 0.3 * tanx
    lyp, lyn = (H - cy) / fy + 0.3 * tany, cy / fy + 0.3 * tany
    if mutation == "lx_swap":
        lxp, lxn = lxn, lxp
    zs = torch.where(z.abs() > 1e-12, z, torch.full_like(z, 1e-12))
    rz = 1.0 / zs
    tx = zs * torch.minimum(lxp, torch.maximum(-lxn, x * rz))
    ty = zs * torch.minimum(lyp, torch.maximum(-lyn, y * rz))
    if mutation == "band_unclamped":     # clamped value, derivative of the unclamped x and y
        tx = tx.detach() + (x - x.detach())
        ty = ty.detach() + (y - y.detach())
    jx, jy = (fy, fx) if mutation == "fxfy_J" else (fx, fy)
    zero = torch.zeros_like(rz)
    J = torch.stack([jx * rz, zero, -jx * tx * rz * rz, zero, jy * rz, -jy * ty * rz * rz], -1).reshape(-1, 2, 3)
    S2 = J @ Sc @ J.transpose(1, 2)
    means2d = torch.stack([fx * x * rz + cx, fy * y * rz + cy], -1)
    a = S2[:, 0, 0] + eps2d
    b = S2[:, 0, 1]
    c = S2[:, 1, 1] + eps2d
    det = a * c - b * b
    valid = (z >= near) & (z <= far) & (det > 0) & (opacities >= ALPHA_THRESHOLD)
    dets = torch.where(det > 0, det, torch.ones_like(det))
    conics = torch.stack([c / dets, -b / dets, a / dets], -1)
    with torch.no_grad():
        ext = torch.sqrt(2.0 * torch.log(torch.clamp(opacities, min=ALPHA_THRESHOLD) / ALPHA_THRESHOLD)).clamp(max=3.33)
        bb = 0.5 * (a + c)
        lam = bb + torch.sqrt(torch.clamp(bb * bb - det, min=0.01))
        r1 = ext * torch.sqrt(lam)
        rx = torch.ceil(torch.minimum(ext * torch.sqrt(a.clamp(min=0)), r1))
        ry = torch.ceil(torch.minimum(ext * torch.sqrt(c.clamp(min=0)), r1))
        valid = valid & ~((rx <= radius_clip) & (ry <= radius_clip))
        valid = valid & ~((means2d[:, 0] + rx <= 0) | (means2d[:, 0] - rx >= W) |
                          (means2d[:, 1] + ry <= 0) | (means2d[:, 1] - ry >= H))
        radii = torch.stack([rx, ry], -1).to(torch.int32) * valid[:, None].to(torch.int32)
    return radii, means2d, z, conics


def sh_basis(dirs: torch.Tensor, degree: int) -> torch.Tensor:
    """Real SH basis [N,16] (entries above `degree` are zero), standard 3DGS constants
    (Reconstruct/utils.py:119 for C0)."""
    n = dirs / dirs.norm(dim=-1, keepdim=True)
    x, y, z = n.unbind(-1)
    B = [torch.full_like(x, SH_C0)]
    if degree >= 1:
        B += [-SH_C1 * y, SH_C1 * z, -SH_C1 * x]
    if degree >= 2:
        z2 = z * z
        fT0B = -1.092548430592079 * z
        fC1 = x * x - y * y
        fS1 = 2 * x * y
        B += [0.5462742152960395 * fS1, fT0B * y, 0.9461746957575601 * z2 - 0.3153915652525201,
              fT0B * x, 0.5462742152960395 * fC1]
    if degree >= 3:
        fT0C = -2.285228997322329 * z2 + 0.4570457994644658
        fT1B = 1.445305721320277 * z
        fC2 = x * fC1 - y * fS1
        fS2 = x * fS1 + y * fC1
        B += [-0.5900435899266435 * fS2, fT1B * fS1, fT0C * y,
              z * (1.865881662950577 * z2 - 1.119528997770346), fT0C * x, fT1B * fC1,
              -0.5900435899266435 * fC2]
    while len(B) < 16:
        B.append(torch.zeros_like(x))
    return torch.stack(B, -1)


def sh_colors(means, campos, sh, degree):
    basis = sh_basis(means - campos, degree)
    return torch.clamp_min(torch.einsum("nk,nkc->nc", basis, sh) + 0.5, 0.0)


def isect_and_sort(radii, means2d, depths, W, H, cam_id=0, n_cams=1, rect_fn=None):
    """Returns sorted keys (int64), sorted gaussian ids (int32), tile offsets [T_h*T_w] (int32).
    ``rect_fn(i, tw, th) -> (x0, x1, y0, y1) or None`` overrides the gsplat tile rectangle (oracle/legacy_torch.py)."""
    tw, th = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    tile_bits = (tw * th).bit_length()
    keys, vals = [], []
    d_bits = depths.detach().to(torch.float32).contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    for i in range(radii.shape[0]):
        rx, ry = int(radii[i, 0]), int(radii[i, 1])
        if rx <= 0 and ry <= 0:
            continue
        mx, my = float(means2d[i, 0]) / TILE, float(means2d[i, 1]) / TILE
        # float32 arithmetic like the kernels
        f = lambda v: float(torch.tensor(v, dtype=torch.float32))
        if rect_fn is not None:
            rect = rect_fn(i, tw, th)
            if rect is None:
                continue
            x0, x1, y0, y1 = rect
        else:
            x0 = min(max(0, int(math.floor(f(f(mx) - f(rx / TILE))))), tw)
            x1 = min(max(0, int(math.ceil(f(f(mx) + f(rx / TILE))))), tw)
            y0 = min(max(0, int(math.floor(f(f(my) - f(ry / TILE))))), th)
            y1 = min(max(0, int(math.ceil(f(f(my) + f(ry / TILE))))), th)
        for ty in range(y0, y1):
            for tx in range(x0, x1):
                keys.append((cam_id << (32 + tile_bits)) | ((ty * tw + tx) << 32) | int(d_bits[i]))
                vals.append(cam_id * radii.shape[0] + i)
    keys_t = torch.tensor(keys, dtype=torch.int64)
    vals_t = torch.tensor(vals, dtype=torch.int32)
    if len(keys):
        order = torch.sort(keys_t, stable=True).indices
        keys_t, vals_t = keys_t[order], vals_t[order]
    tiles = (keys_t >> 32) & ((1 << tile_bits) - 1)
    offsets = torch.searchsorted(tiles, torch.arange(tw * th, dtype=torch.int64)).to(torch.int32)
    return keys_t, vals_t, offsets


def blend(means2d, conics, opacities, feats, vals, offsets, W, H, max_alpha=MAX_ALPHA, strict_stop=False, main_ids=None):
    """feats [N,CHN]; returns out[H,W,CHN], alpha[H,W], last_ids[H,W] (index into the sorted list).
    ``max_alpha`` / ``strict_stop`` (stop on T(1-a) < eps instead of <=) / ``main_ids`` (int32 [H,W] filled with the
    Gaussian of largest weight alpha*T, -1 none) serve the legacy conventions of oracle/legacy_torch.py."""
    tw = (W + TILE - 1) // TILE
    th = (H + TILE - 1) // TILE
    n_isect = vals.shape[0]
    CH = feats.shape[1]
    out_rows, alpha_rows = [], []
    last = torch.zeros(H, W, dtype=torch.int32)
    for i in range(H):
        row_c, row_a = [], []
        for j in range(W):
            tid = (i // TILE) * tw + (j // TILE)
            start = int(offsets[tid])
            end = int(offsets[tid + 1]) if tid + 1 < tw * th else n_isect
            px, py = j + 0.5, i + 0.5
            T = torch.ones((), dtype=means2d.dtype)
            acc = torch.zeros(CH, dtype=means2d.dtype)
            cur = 0
            best_w = 0.0
            if main_ids is not None:
                main_ids[i, j] = -1
            for k in range(start, end):
                g = int(vals[k])
                dx = means2d[g, 0] - px
                dy = means2d[g, 1] - py
                a, b, c = conics[g]
                sigma = 0.5 * (a * dx * dx + c * dy * dy) + b * dx * dy
                alpha = torch.clamp(opacities[g] * torch.exp(-sigma), max=max_alpha)
                if float(sigma) < 0 or float(alpha) < ALPHA_THRESHOLD:
                    continue
                nT = T * (1 - alpha)
                if (float(nT) < T_EPS) if strict_stop else (float(nT) <= T_EPS):
                    break
                acc = acc + feats[g] * alpha * T
                if main_ids is not None and float(alpha * T) > best_w:
                    best_w = float(alpha * T)
                    main_ids[i, j] = g
                T = nT
                cur = k
            row_c.append(acc)
            row_a.append(1 - T)
            last[i, j] = cur
        out_rows.append(torch.stack(row_c))
        alpha_rows.append(torch.stack(row_a))
    return torch.stack(out_rows), torch.stack(alpha_rows), last


def rasterization(means, quats, scales, opacities, sh, viewmat, K, W, H, sh_degree=3, eps2d=0.01):
    """Single-camera RGB+D render: returns colors[H,W,4], alphas[H,W], radii[N,2]."""
    radii, means2d, depths, conics = project(means, quats, scales, opacities, viewmat, K, W, H, eps2d)
    campos = torch.inverse(viewmat)[:3, 3]
    rgb = sh_colors(means, campos, sh, sh_degree)
    feats = torch.cat([rgb, depths[:, None]], -1)
    _, vals, offsets = isect_and_sort(radii, means2d, depths, W, H)
    out, alpha, _ = blend(means2d, conics, opacities, feats, vals, offsets, W, H)
    return out, alpha, radii

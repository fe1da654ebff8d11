"""TEST INFRASTRUCTURE ONLY.  The pixel loss block of SceneModel.optimization_step restated op for op in PyTorch:
Reconstruct/scene/scene_models/h3dgsv3.py:430-450 (radial-weighted L1, the is_important=False error mask, 1 - SSIM, the
inverse-depth term), render_from_id's exposure (:611-614) and render's background composite and 1/D (:682-686), with
Reconstruct/utils.py:818-826 (radial_decay_kernel) and ``fused_ssim`` replaced by the pinned conv2d SSIM of ssim_ref.
Runs on the CPU or the device; gradients come from autograd.  tests/golden/make_mapper_loss_golden.py pins it to the
reference's own statements."""
import torch

from . import ssim_ref


def radial_decay_kernel(H, W, sigma=0.5):
    y = torch.linspace(-1, 1, steps=H)
    x = torch.linspace(-1, 1, steps=W)
    yy, xx = torch.meshgrid(y, x, indexing='ij')
    r2 = xx**2 + yy**2
    return torch.exp(-r2 / (2 * sigma**2))


def sixD2mtx(r):
    """Reconstruct/utils.py:223-229: the rotation of a key frame's 6-D parameter r [..., 3, 2]."""
    b1 = r[..., 0]
    b1 = b1 / torch.norm(b1, dim=-1, keepdim=True)
    b2 = r[..., 1] - torch.sum(b1 * r[..., 1], dim=-1, keepdim=True) * b1
    b2 = b2 / torch.norm(b2, dim=-1, keepdim=True)
    b3 = torch.cross(b1, b2, dim=-1)
    return torch.stack([b1, b2, b3], dim=-1)


def composite(colors, alphas, bg):
    """render (h3dgsv3.py:682-686) for one view: (render [3,h,w], invdepth [1,h,w])."""
    rendered_color = colors[..., 0:3].permute([0, 3, 1, 2])
    rendered_depth_unnormalized = colors[..., 3:4].permute([0, 3, 1, 2])
    rendered_alpha = alphas.permute([0, 3, 1, 2])
    rendered_color = rendered_color + (1.0 - rendered_alpha) * bg[None, :, None, None]
    invdepth = 1.0 / rendered_depth_unnormalized
    return rendered_color[0], invdepth[0]


def expose(render, exposure):
    """render_from_id (h3dgsv3.py:611-614): (clamped image, the value before the clamp)."""
    c, height, width = render.shape
    pre = (exposure[:3, :3] @ render.reshape(3, -1)) + exposure[:3, 3, None]
    return pre.clamp(0, 1).view(3, height, width), pre.view(3, height, width)


def loss_terms(image, invdepth, gt_image, mono_idepth, rdk, *, lambda_dssim, depth_weight, is_important, ssim_fn=None):
    """h3dgsv3.py:430-450 without scaling_reg.  Returns a dict: loss, l1, ssim (mean), depth, and the masked operands.
    ``ssim_fn(img1, img2)`` (default: the pinned conv2d SSIM) stands for ``fused_ssim``."""
    mask = None
    if not is_important:
        error_map = (rdk * (image - gt_image).abs())
        alpha_mask = torch.bitwise_or(torch.bitwise_or(error_map[0] > 0.2, error_map[1] > 0.2), error_map[1] > 0.2)
        alpha_mask = ~alpha_mask
        mask = alpha_mask
        image = image * alpha_mask
        gt_image = gt_image * alpha_mask
        invdepth = invdepth * alpha_mask
        mono_idepth = mono_idepth * alpha_mask
    l1_loss = (rdk * (image - gt_image).abs()).mean()
    ssim = (ssim_fn or ssim_ref.ssim)(image[None], gt_image[None])
    ssim_loss = 1 - ssim
    depth_loss = (rdk * (invdepth - mono_idepth).abs()).mean()
    loss = lambda_dssim * ssim_loss + (1 - lambda_dssim) * l1_loss + depth_weight * depth_loss
    return dict(loss=loss, l1=l1_loss, ssim=ssim, depth=depth_loss, image=image, gt=gt_image, invdepth=invdepth, mask=mask)


def mapper_loss(colors, alphas, gt_image, mono_idepth, exposure, bg, *, lambda_dssim, depth_weight, rad_decay, is_important,
                ssim_fn=None):
    """The whole block from the rasterizer's raw outputs (colors [1,h,w,4], alphas [1,h,w,1]); same contract as
    artdeco_b200.mapper.mapper_loss plus the intermediates (dict)."""
    render, invdepth = composite(colors, alphas, bg)
    image, pre = expose(render, exposure)
    h, w = image.shape[1:]
    rdk = radial_decay_kernel(h, w, rad_decay).to(image.device)
    out = loss_terms(image, invdepth, gt_image, mono_idepth, rdk, lambda_dssim=lambda_dssim, depth_weight=depth_weight,
                     is_important=is_important, ssim_fn=ssim_fn)
    out["pre_clamp"] = pre
    out["exposed"] = image
    return out


def make_inputs(h, w, seed, *, zero_depth=True):
    """Seeded CPU inputs that reach every branch: pixels with D = 0 (inv = inf), some of them masked (inf * 0 = NaN) when
    ``zero_depth``; channel 0 of the exposure is the identity, so alpha = 1 pixels with rgb 0 or 1 land exactly on the clamp
    bounds (inclusive: the gradient passes) and others beyond them; ground truth equal to the exposed value (e == g ties);
    errors on both sides of the 0.2 mask threshold."""
    g = torch.Generator().manual_seed(seed)
    rgb = -0.1 + 1.2 * torch.rand(1, h, w, 3, generator=g)
    D = 0.5 + 4.0 * torch.rand(1, h, w, 1, generator=g)
    alphas = torch.rand(1, h, w, 1, generator=g)
    n = h * w
    idx = torch.randperm(n, generator=g)
    q = max(n // 40, 1)
    flat_rgb, flat_a, flat_D = rgb.view(n, 3), alphas.view(n), D.view(n)
    flat_a[idx[:4 * q]] = 1.0                                  # no background: c = rgb exactly
    flat_rgb[idx[:q], 0] = 1.0                                 # e0 = 1 on the bound
    flat_rgb[idx[q:2 * q], 0] = 0.0                            # e0 = 0 on the bound
    flat_rgb[idx[2 * q:3 * q], :] = 1.3                        # above: clamped, no gradient
    flat_rgb[idx[3 * q:4 * q], :] = -0.2                       # below: clamped, no gradient
    if zero_depth:
        flat_D[idx[4 * q:5 * q]] = 0.0                         # nothing rendered: inv = inf
    colors = torch.cat([rgb, D], -1).contiguous()
    exposure = torch.tensor([[1.0, 0.0, 0.0, 0.0],
                             [0.05, 1.1, -0.04, 0.02],
                             [-0.03, 0.06, 0.95, -0.01]])
    bg = torch.tensor([0.3, 0.7, 0.45])
    gt = (torch.rand(3, h, w, generator=g) * 0.6 + 0.2)
    gtf = gt.view(3, n)
    # e == g ties: gt equal to the exposed value where it is known exactly (the bounds and the clamped pixels)
    gtf[0, idx[:q // 2]] = 1.0
    gtf[0, idx[q:q + q // 2]] = 0.0
    gtf[:, idx[2 * q:2 * q + q // 2]] = 1.0
    gtf[:, idx[3 * q:3 * q + q // 2]] = 0.0
    mono = 0.2 + 1.5 * torch.rand(1, h, w, generator=g)
    return dict(colors=colors, alphas=alphas.contiguous(), gt=gt.contiguous(), mono=mono, exposure=exposure, bg=bg)

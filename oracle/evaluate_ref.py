"""TEST INFRASTRUCTURE ONLY.  The mapper's quality evaluation restated in PyTorch:
``harmonize_test_exposure`` and ``evaluate`` (Reconstruct/scene/scene_models/h3dgsv3.py:507-558), ``render_from_id``'s
exposure (:611-614) with ``render``'s background composite (:682-686), ``psnr`` (Reconstruct/utils.py:86-87) and
``lpips.LPIPS(net="vgg")`` (version 0.1, lpips=True, spatial=False, normalize=False) with the lpips package's module and
state-dict layout.  ``fused_ssim`` is the pinned conv2d SSIM of ssim_ref.  The lpips package is neither vendored nor
installable here, so the LPIPS head is restated from its published definition (parity with the package is unpinned); the
VGG trunk is torchvision's ``vgg16().features`` cut into lpips's slices.  tests/golden/make_evaluate_golden.py pins the
evaluation loop, the harmonisation and ``psnr`` to the reference's own statements."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ssim_ref
from .mapper_loss_ref import composite

SLICES = ((0, 4), (4, 9), (9, 16), (16, 23), (23, 30))
TAP_CHANNELS = (64, 128, 256, 512, 512)
VGG_CFG = (64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512)


def harmonize_test_exposure(exposures, is_test):
    """h3dgsv3.py:507-520 on a list of per-key-frame exposure tensors (replaced in the list, as the attribute is)."""
    for index in range(len(exposures)):
        if is_test[index]:
            idxm = index - 1 if index != 0 else 1
            idxp = index + 1 if index != len(exposures) - 1 else len(exposures) - 2
            exposures[index] = (exposures[idxm] + exposures[idxp]) / 2
    return exposures


def psnr(img1, img2):
    return 10 * torch.log10(1 / F.mse_loss(img1, img2)).item()


def render_from_colors(colors, alphas, exposure, bg=None):
    """render_from_id at level 0 on the rasterizer's raw colors [1,h,w,4] / alphas [1,h,w,1], bg = 0."""
    h, w = colors.shape[1], colors.shape[2]
    bg = torch.zeros(3, dtype=colors.dtype, device=colors.device) if bg is None else bg
    render, _ = composite(colors, alphas, bg)
    render = (exposure[:3, :3] @ render.reshape(3, -1)) + exposure[:3, 3, None]
    return render.clamp(0, 1).view(3, h, w)


def vgg_features():
    """torchvision.models.vgg16().features[0:30] as a plain Sequential with the same indices (no torchvision needed)."""
    layers, cin = [], 3
    for v in VGG_CFG:
        if v == "M":
            layers.append(nn.MaxPool2d(kernel_size=2, stride=2))
        else:
            layers += [nn.Conv2d(cin, v, kernel_size=3, padding=1), nn.ReLU(inplace=False)]
            cin = v
    return nn.Sequential(*layers)


class ScalingLayer(nn.Module):
    def __init__(self):
        super().__init__()
        self.register_buffer("shift", torch.Tensor([-.030, -.088, -.188])[None, :, None, None])
        self.register_buffer("scale", torch.Tensor([.458, .448, .450])[None, :, None, None])

    def forward(self, inp):
        return (inp - self.shift) / self.scale


class VGGSlices(nn.Module):
    def __init__(self, features=None):
        super().__init__()
        features = vgg_features() if features is None else features
        for k, (a, b) in enumerate(SLICES):
            s = nn.Sequential()
            for x in range(a, b):
                s.add_module(str(x), features[x])
            setattr(self, f"slice{k + 1}", s)

    def forward(self, x):
        outs = []
        for k in range(5):
            x = getattr(self, f"slice{k + 1}")(x)
            outs.append(x)
        return outs


class NetLinLayer(nn.Module):
    def __init__(self, chn_in):
        super().__init__()
        self.model = nn.Sequential(nn.Dropout(), nn.Conv2d(chn_in, 1, 1, stride=1, padding=0, bias=False))

    def forward(self, x):
        return self.model(x)


def normalize_tensor(in_feat, eps=1e-10):
    norm_factor = torch.sqrt(torch.sum(in_feat ** 2, dim=1, keepdim=True))
    return in_feat / (norm_factor + eps)


def head(f0, f1, lin_w):
    """One tap of the LPIPS head: spatial mean of lin(normalize(f0) - normalize(f1))^2, [N,1,1,1]."""
    d = (normalize_tensor(f0) - normalize_tensor(f1)) ** 2
    return F.conv2d(d, lin_w).mean([2, 3], keepdim=True)


class LPIPSRef(nn.Module):
    """lpips.LPIPS(net="vgg") with the package's module names, so its state dict loads unchanged."""

    def __init__(self, features=None):
        super().__init__()
        self.scaling_layer = ScalingLayer()
        self.net = VGGSlices(features)
        for k, c in enumerate(TAP_CHANNELS):
            setattr(self, f"lin{k}", NetLinLayer(c))
        self.eval()

    def taps(self, in0, in1):
        return self.net(self.scaling_layer(in0)), self.net(self.scaling_layer(in1))

    def forward(self, in0, in1):
        outs0, outs1 = self.taps(in0, in1)
        val = 0
        for k in range(5):
            val += head(outs0[k], outs1[k], getattr(self, f"lin{k}").model[1].weight)
        return val


def random_state_dict(seed: int = 0):
    """Seeded random weights: Kaiming-scaled convolutions (activations stay O(1) through 13 layers), small biases and
    non-negative lin weights, as trained lpips weights are."""
    g = torch.Generator().manual_seed(seed)
    m = LPIPSRef()
    sd = {}
    for k, v in m.state_dict().items():
        if k.startswith("net.") and k.endswith("weight"):
            fan_in = v.shape[1] * 9
            sd[k] = torch.randn(v.shape, generator=g) * (2.0 / fan_in) ** 0.5
        elif k.startswith("net.") and k.endswith("bias"):
            sd[k] = torch.randn(v.shape, generator=g) * 0.01
        elif k.startswith("lin"):
            sd[k] = torch.rand(v.shape, generator=g) * (2.0 / v.shape[1])
        else:
            sd[k] = v.clone()
    return sd


def make_lpips(seed: int = 0, device="cpu"):
    m = LPIPSRef()
    m.load_state_dict(random_state_dict(seed))
    return m.to(device).eval()


@torch.no_grad()
def evaluate(exposures, is_test, renders, gt_images, visibility, lpips=None, with_LPIPS=False, all=False, first_index=0):
    """h3dgsv3.py:523-558 with render_from_id on fixed renders.  ``exposures``: K tensors [3,4] (harmonised in the list);
    ``renders[i]`` = (colors [1,h,w,4], alphas [1,h,w,1]) of key frame i; ``visibility[i]`` its visibility_filter."""
    harmonize_test_exposure(exposures, is_test)
    metrics = {"PSNR": 0.0, "SSIM": 0.0, "Render": 0.0, "GS": 0.0}
    if with_LPIPS:
        metrics["LPIPS"] = 0.0
    n_test_frames = 0
    start_index = 0 if all else first_index
    for index in range(start_index, len(is_test)):
        if is_test[index]:
            gt_image = gt_images[index]
            image = render_from_colors(*renders[index], exposures[index])
            mask = torch.ones_like(image[:1] > 0)
            mask = mask.expand_as(image)
            image = image * mask
            gt_image = gt_image * mask
            metrics["Render"] += visibility[index].sum().item()
            metrics["GS"] += len(visibility[index])
            metrics["PSNR"] += psnr(image[mask], gt_image[mask])
            metrics["SSIM"] += ssim_ref.ssim(image[None], gt_image[None]).item()
            if with_LPIPS and lpips is not None:
                metrics["LPIPS"] += lpips(image[None], gt_image[None]).item()
            n_test_frames += 1
    if n_test_frames > 0:
        for metric in metrics:
            metrics[metric] /= n_test_frames
    else:
        metrics = {}
    metrics["n_test_frames"] = n_test_frames
    return metrics

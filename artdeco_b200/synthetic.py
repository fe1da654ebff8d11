"""Seeded synthetic workloads (SURVEY.md §8d).  Everything is generated on the CPU with a
``torch.Generator`` so the same tensors can be fed to the oracle and (after a host->device copy) to the
CUDA path; there is no dataset or checkpoint access."""
from __future__ import annotations

import math

import torch


def raster_scene(N: int, seed: int = 0, z_range=(2.0, 18.0), extent=(8.0, 4.5),
                 scale_range=(0.005, 0.05), dtype=torch.float32):
    """`raster_scene(N, seed)` of SURVEY.md §8d: world == camera-0 frame."""
    g = torch.Generator().manual_seed(seed)
    u = torch.rand(N, 3, generator=g, dtype=dtype)
    means = torch.stack([(u[:, 0] * 2 - 1) * extent[0], (u[:, 1] * 2 - 1) * extent[1],
                         z_range[0] + u[:, 2] * (z_range[1] - z_range[0])], -1)
    ls = math.log(scale_range[0]) + torch.rand(N, 3, generator=g, dtype=dtype) * (
        math.log(scale_range[1]) - math.log(scale_range[0]))
    scales = torch.exp(ls)
    quats = torch.randn(N, 4, generator=g, dtype=dtype)
    quats = quats / quats.norm(dim=-1, keepdim=True)
    opacities = torch.sigmoid(torch.randn(N, generator=g, dtype=dtype) * 1.5)
    sh = torch.cat([torch.randn(N, 1, 3, generator=g, dtype=dtype) * 0.5,
                    torch.randn(N, 15, 3, generator=g, dtype=dtype) * 0.05], 1)
    d_max = 4.0 + torch.rand(N, 1, generator=g, dtype=dtype) * 36.0
    return dict(means=means.contiguous(), quats=quats.contiguous(), scales=scales.contiguous(),
                opacities=opacities.contiguous(), sh=sh.contiguous(), d_max=d_max.contiguous())


def camera(width: int = 1920, height: int = 1080, view: float = 3.5, focal: float | None = None):
    """View v of SURVEY.md §8d: R = rot_y((v-3.5)*2deg), t = (0.2*(v-3.5), 0, 0); fx=fy=1000 at 1080p."""
    f = focal if focal is not None else 1000.0 * width / 1920.0
    K = torch.tensor([[f, 0.0, width / 2.0], [0.0, f, height / 2.0], [0.0, 0.0, 1.0]], dtype=torch.float32)
    ang = math.radians((view - 3.5) * 2.0)
    c, s = math.cos(ang), math.sin(ang)
    V = torch.eye(4, dtype=torch.float32)
    V[:3, :3] = torch.tensor([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])
    V[0, 3] = 0.2 * (view - 3.5)
    return V, K


def upstream_grads(width: int, height: int, seed: int = 1, C: int = 1):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(C, height, width, 4, generator=g), torch.randn(C, height, width, 1, generator=g))


def ssim_pair(B=1, CH=3, H=1080, W=1920, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, CH, H, W, generator=g), torch.rand(B, CH, H, W, generator=g)


def det_weights(shapes: dict, seed: int = 0, device="cpu"):
    """Deterministic per-tensor weights for a {name: shape} table (no checkpoint is available offline): each tensor is
    drawn from its own generator seeded by crc32(name), so any implementation that knows the names and shapes gets
    bit-identical values regardless of construction order.  Scales keep activations O(1) through 36 layers:
    matrices/convs ~ N(0, 1/fan_in), LayerNorm weights 1 + 0.1 N(0,1), biases 0.02 N(0,1)."""
    import zlib
    from concurrent.futures import ThreadPoolExecutor

    def one(item):
        name, shape = item
        g = torch.Generator().manual_seed((zlib.crc32(name.encode()) + 7919 * seed) & 0x7fffffff)
        t = torch.randn(*shape, generator=g, dtype=torch.float32)
        if len(shape) == 1:
            is_norm_w = name.endswith(".weight")
            t = 1.0 + 0.1 * t if is_norm_w else 0.02 * t
        else:
            fan_in = 1
            for d in shape[1:]:
                fan_in *= d
            if ".act_postprocess." in name and name.endswith(".1.weight") and len(shape) == 4 and shape[0] == shape[1] and shape[2] in (2, 4):
                fan_in = shape[0]          # ConvTranspose2d: [in, out, k, k], each output pixel sees `in` taps
            t = t * (1.0 / fan_in) ** 0.5
            if name.endswith(".dpt.head.4.weight") or name.endswith(".head_local_features.fc2.weight"):
                t = t * 0.2                # keeps log-depth d <~ 3.5 (scenes up to ~30 m, like a metric indoor checkpoint);
                                           # pts3d = dir * expm1(d) turns an ABSOLUTE error in d into a relative error in pts3d
        return name, t.to(device)

    # per-tensor generators make the values independent of evaluation order, so the draw can be threaded
    with ThreadPoolExecutor(max_workers=16) as ex:
        return dict(ex.map(one, list(shapes.items())))


def pi3_frames(N: int = 2, H: int = 392, W: int = 518, seed: int = 0):
    """Pi3's input [1, N, 3, H, W] in [0, 1]."""
    g = torch.Generator().manual_seed(seed)
    return torch.rand(1, N, 3, H, W, generator=g)


def mast3r_pair(B: int = 1, H: int = 512, W: int = 512, seed: int = 0):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(B, 3, H, W, generator=g) * 2 - 1, torch.rand(B, 3, H, W, generator=g) * 2 - 1)

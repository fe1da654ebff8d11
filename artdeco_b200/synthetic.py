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


# ---- key-frame retrieval (retrieval.RetrievalDatabase) ----
# Descriptors are built in the whitened space: token t of a place is s_t * normalize(c_w + 0.5 g) for a random visual word
# w, with attention norms s_t = 1 + 1e-3 * rank, so the attention order has 1e-3 relative gaps.  A revisit adds 0.05 of
# fresh noise to every direction of the place.  Margins are measured in float64 on the fp32 encoder tokens; tokens whose
# decision is too close to call in fp32 (attention order, the order of the assignment's MA + 1 nearest distances, the sign
# of an aggregated residual component) are re-drawn until every margin clears its bound.
RETRIEVAL_MARGIN_DIST = 2.0 ** -12      # consecutive gap of the MA + 1 nearest distances / (|d|^2 + |c|^2)
RETRIEVAL_MARGIN_RESID = 2.0 ** -18     # |r_j| / sum |d_j - c_j| over the word's members
RETRIEVAL_MARGIN_ATTN = 1e-5            # relative gap of consecutive attention norms, ranks 0..nfeat


def retrieval_model(K: int, dim: int = 1024, seed: int = 0):
    """(m [1, dim] float64, P [dim, dim] float64 orthogonal, centroids [K, dim] fp32 of unit norm)."""
    g = torch.Generator().manual_seed(seed)
    m = 0.01 * torch.randn(1, dim, generator=g, dtype=torch.float64)
    P, _ = torch.linalg.qr(torch.randn(dim, dim, generator=g, dtype=torch.float64))
    c = torch.randn(K, dim, generator=g, dtype=torch.float64)
    return m, P, (c / c.norm(dim=1, keepdim=True)).float()


def _retrieval_margins(x, m, P, cent, cn, nfeat, ma):
    """float64 margins of one frame's fp32 tokens x [n, dim] -> (offending token ids, (attn, dist, resid) minima)."""
    y = ((x.double() - m) @ P).float().double()
    a = y.norm(dim=1)
    order = torch.argsort(a, descending=True)
    sel = order[:nfeat]
    top = a[order[:nfeat + 1]]
    ag = (top[:-1] - top[1:]) / top[:-1]
    bad = set(order[:nfeat + 1][:-1][ag < RETRIEVAL_MARGIN_ATTN].tolist())
    d = y[sel]
    dist = (d * d).sum(1, keepdim=True) + cn[None, :] - 2.0 * d @ cent.T
    sd, si = torch.sort(dist, dim=1)
    scale = (d * d).sum(1) + cn[si[:, 0]]
    dmin = ((sd[:, 1:ma + 1] - sd[:, :ma]) / scale[:, None]).min(1).values   # the order of the MA words and the MA+1-th
    bad |= set(sel[dmin < RETRIEVAL_MARGIN_DIST].tolist())
    rmin = float("inf")
    for cols in (si[:, :1], si[:, :ma]):
        words = torch.unique(cols)
        for w in words.tolist():
            rows = (cols == w).any(1)
            diff = d[rows] - cent[w]
            ratio = (diff.sum(0).abs() / diff.abs().sum(0).clamp_min(1e-300)).min()
            rmin = min(rmin, float(ratio))
            if ratio < RETRIEVAL_MARGIN_RESID:
                bad |= set(sel[rows].tolist())
    return bad, (float(ag.min()), float(dmin.min()), rmin)


def retrieval_stream(m, P, centroids, schedule, n: int = 768, nfeat: int = 300, ma: int = 5, seed: int = 0):
    """Key-frame encoder features for a schedule of (place, add_after_query) pairs: a place seen before is a revisit.
    Returns a list of dicts {feat [1, n, dim] fp32, place, add, revisit, margins (attn, dist, resid)}."""
    g = torch.Generator().manual_seed(seed + 1)
    dim = P.shape[0]
    cent = centroids.double()
    cn = (cent * cent).sum(1)
    places = {}
    out = []
    for place, add in schedule:
        revisit = place in places
        if not revisit:
            perm = torch.randperm(n, generator=g)
            words = torch.randint(0, cent.shape[0], (n,), generator=g)
            places[place] = (1.0 + 1e-3 * perm.double(), words, torch.randn(n, dim, generator=g, dtype=torch.float64))
        s, words, base = places[place]

        def direction(rows):
            noise = torch.randn(len(rows), dim, generator=g, dtype=torch.float64) / dim ** 0.5
            v = cent[words[rows]] + 0.5 * base[rows] / dim ** 0.5
            v = v / v.norm(dim=1, keepdim=True) + 0.05 * noise if revisit else v + 0.02 * noise
            return v / v.norm(dim=1, keepdim=True) * s[rows, None]

        yd = direction(torch.arange(n))
        for _ in range(100):
            x = ((yd @ P.T) + m).float()
            bad, margins = _retrieval_margins(x, m, P, cent, cn, nfeat, ma)
            if not bad:
                break
            rows = torch.tensor(sorted(bad))
            yd[rows] = direction(rows)
        else:
            raise RuntimeError("retrieval_stream: margins did not clear in 100 re-draws")
        out.append(dict(feat=x[None].contiguous(), place=place, add=add, revisit=revisit, margins=margins))
    return out


# 30 updates: 14 new places (the Pi3 gate is reached at 12), a short-range revisit (retrieval kept), long-range revisits
# (Pi3), a relocalisation query later re-added, never-seen places (empty match) and a second lap.
RETRIEVAL_SCHEDULE = ([(p, True) for p in range(14)] + [(13, True), (1, True), (5, False), (5, True), (100, True),
                      (2, True), (14, True), (15, True), (14, True), (101, False), (3, True), (16, True), (0, True),
                      (17, True), (6, True), (9, True)])

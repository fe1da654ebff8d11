"""The blend forward's per-entry warp masks on the GPU against a brute-force walk over every pixel of every entry's tile.

Bit w of hit_mask[k] must be set wherever warp w's 8x4 block holds a pixel at which entry k passes the per-pixel test
0 <= sigma2 <= smax2 inside the projection's integer-radius box (in float32, with and without FMA contraction): those are
exactly the entries the warp has to evaluate, so a missing bit would drop a splat from the image.  The mask must also stay
well inside the box alone, or the culling does nothing."""
import numpy as np
import pytest
import torch

from artdeco_b200 import synthetic

LOG2E = np.float32(1.4426950408889634)


def _stages(N, W, H, view, dev, **kw):
    from artdeco_b200 import raster as R
    sc = synthetic.raster_scene(N, seed=5, **kw)
    V, K = synthetic.camera(W, H, view=view)
    t = {k: sc[k].to(dev) for k in ("means", "quats", "scales", "opacities", "sh")}
    Vd, Kd = V.to(dev), K.to(dev)
    campos = torch.inverse(Vd)[:3, 3].contiguous()
    radii, splats, tpg = R.project(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], 3, Vd, Kd, campos, W, H,
                                   0.01, 0.01, 1e10, 0.0)
    keys, vals, offs, n = R.intersect(radii, splats, tpg, W, H)
    hits = torch.full((max(1, n),), 0xFF, dtype=torch.uint8, device=dev)     # entries behind a saturated tile stay all-ones
    col, alp, last = R.blend_forward(W, H, N, splats, vals, offs, hits=hits)
    return splats, keys[:n], vals[:n], hits[:n]


def _owed_bits(splats, keys, vals, W):
    """(bits a pixel test needs inside the radius box, bits of the box alone) per entry, by brute force."""
    tw = (W + 15) // 16
    rec = splats.reshape(-1, 12)[vals.long()]
    tile = (keys >> 32).long()
    tx0 = ((tile % tw) * 16).float() + 0.5
    ty0 = ((tile // tw) * 16).float() + 0.5
    mx, my = rec[:, 0], rec[:, 1]
    ha = rec[:, 2] * np.float32(0.5 * LOG2E)
    b2 = rec[:, 3] * LOG2E
    hc = rec[:, 4] * np.float32(0.5 * LOG2E)
    smax2 = (rec[:, 6] - np.float32(0.02)) * LOG2E
    pr = rec[:, 7].contiguous().view(torch.int32).long() & 0xFFFFFFFF
    rx, ry = (pr & 0xFFFF).float(), (pr >> 16).float()
    rx = torch.where(rx == 65535, torch.full_like(rx, 3e38), rx)
    ry = torch.where(ry == 65535, torch.full_like(ry, 3e38), ry)
    need = torch.zeros_like(vals, dtype=torch.int32)
    box = torch.zeros_like(vals, dtype=torch.int32)
    lx = torch.arange(8, device=keys.device).float()
    ly = torch.arange(4, device=keys.device).float()
    for w in range(8):
        xlo = tx0 + 8 * (w & 1)
        ylo = ty0 + 4 * (w >> 1)
        px = (xlo[:, None, None] + lx[None, None, :]).expand(-1, 4, 8).reshape(-1, 32)
        py = (ylo[:, None, None] + ly[None, :, None]).expand(-1, 4, 8).reshape(-1, 32)
        inbox = ((mx + rx >= xlo) & (mx - rx <= xlo + 7) & (my + ry >= ylo) & (my - ry <= ylo + 3))
        dx, dy = mx[:, None] - px, my[:, None] - py
        s_plain = dx * (ha[:, None] * dx + b2[:, None] * dy) + (hc[:, None] * dy) * dy
        inner = (ha[:, None].double() * dx.double() + (b2[:, None] * dy).double()).float()
        s_fma = (dx.double() * inner.double() + ((hc[:, None] * dy) * dy).double()).float()
        hit = torch.zeros_like(inbox)
        for s2 in (s_plain, s_fma):
            hit |= ((s2 >= 0) & (s2 <= smax2[:, None])).any(dim=1)
        need |= (hit & inbox).int() << w
        box |= inbox.int() << w
    return need, box


@pytest.mark.gpu
@pytest.mark.parametrize("N,W,H,view,kw", [(3000, 320, 192, 1.0, {}), (40000, 960, 544, 5.0, dict(scale_range=(0.01, 0.15))),
                                           (20000, 640, 360, 2.0, {})])
def test_forward_hit_mask_keeps_every_block_a_pixel_test_passes(cuda, N, W, H, view, kw):
    splats, keys, vals, hits = _stages(N, W, H, view, cuda, **kw)
    assert vals.numel() > 1000
    need, box = _owed_bits(splats, keys, vals, W)
    h = hits.int()
    missing = need & ~h
    assert int((missing != 0).sum()) == 0, f"{int((missing != 0).sum())} entries lost a bit a passing pixel needs"
    written = hits != 0xFF
    kept = sum(int(((h[written] >> w) & 1).sum()) for w in range(8))
    in_box = sum(int(((box[written] >> w) & 1).sum()) for w in range(8))
    assert kept <= 0.9 * in_box, (kept, in_box)

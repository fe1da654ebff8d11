"""Renders the edge scenes of test_raster_edges.py (both ladder regimes and the frame-sized splats) forward and backward,
single-view and as a C = 3 batch, and saves every output to the file named on the command line.

The blend switches (ADB_BLEND_TMA, ADB_BWD_SLOTS, ADB_BWD_OCC) are read once per process, so test_raster_edges.py runs this
script once per switch and compares its outputs with ``render_all`` computed in its own process on the default path."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

KEYS = ("means", "quats", "scales", "opacities", "sh")


def _views(V):
    """The camera and two shifted copies (0.05 world units in x, 0.03 in y)."""
    out = [V]
    for dx, dy in ((0.05, 0.0), (0.0, 0.03)):
        v = V.copy()
        v[0, 3] += dx
        v[1, 3] += dy
        out.append(v)
    return np.stack(out)


def render_all(dev):
    """{name: CPU tensor}.  fwd_* must be bit-identical across the blend variants, bwd_* equal up to the order of the REDs."""
    import test_raster_edges as E
    from artdeco_b200 import raster as R
    out = {}
    scenes = {k: E.ladder(k)[:5] for k in E.REGIMES}
    scenes["frame"] = E.frame_sized()
    for name, (sc, V, K, W, H) in scenes.items():
        N = len(sc["means"])
        t = {k: torch.from_numpy(sc[k]).to(dev) for k in KEYS}
        g = torch.Generator().manual_seed(4)
        # single view: hit-mask forward, backward from the mask and with the kernel's own culling
        Vd, Kd = torch.from_numpy(V).to(dev), torch.from_numpy(K).to(dev)
        campos = torch.inverse(Vd)[:3, 3].contiguous()
        radii, splats, tpg = R.project(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], 3, Vd, Kd, campos, W, H,
                                       0.01, 0.01, 1e10, 0.0)
        _, vals, offs, n = R.intersect(radii, splats, tpg, W, H)
        hits = torch.zeros(max(1, n), dtype=torch.uint8, device=dev)
        col, alp, last = R.blend_forward(W, H, N, splats, vals, offs, hits=hits)
        vc, va = torch.randn(H, W, 4, generator=g).to(dev), torch.randn(H, W, generator=g).to(dev)
        out[f"fwd_{name}_colors"], out[f"fwd_{name}_alphas"], out[f"fwd_{name}_last"] = col, alp, last
        out[f"fwd_{name}_hits"] = hits
        out[f"bwd_{name}_hits"] = R.blend_backward(W, H, N, splats, vals, offs, alp, last, vc, va, hits=hits)
        out[f"bwd_{name}_own"] = R.blend_backward(W, H, N, splats, vals, offs, alp, last, vc, va)
        # C = 3 through the batched blend
        Vs = torch.from_numpy(_views(V)).to(dev)
        Ks = Kd[None].repeat(3, 1, 1).contiguous()
        P = torch.inverse(Vs)[:, :3, 3].contiguous()
        cnt = R.new_tile_counts(W, H, dev, 3)
        radii, splats, tpg = R.project_multi(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], 3, Vs, Ks, P, W, H,
                                             0.01, 0.01, 1e10, 0.0, cnt)
        _, vals, offs, _, _ = R.intersect_multi(radii, splats, tpg, W, H, cnt, keys=False)
        hits = torch.zeros(max(1, vals.numel()), dtype=torch.uint8, device=dev)
        col, alp, last = R.blend_forward_multi(W, H, splats, vals, offs, hits=hits)
        vc, va = torch.randn(3, H, W, 4, generator=g).to(dev), torch.randn(3, H, W, generator=g).to(dev)
        out[f"fwd_{name}_multi_colors"], out[f"fwd_{name}_multi_alphas"], out[f"fwd_{name}_multi_last"] = col, alp, last
        out[f"fwd_{name}_multi_hits"] = hits
        out[f"bwd_{name}_multi_hits"] = R.blend_backward_multi(W, H, splats, vals, offs, alp, last, vc, va, hits=hits)
        out[f"bwd_{name}_multi_own"] = R.blend_backward_multi(W, H, splats, vals, offs, alp, last, vc, va)
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in out.items()}


if __name__ == "__main__":
    torch.save(render_all(torch.device("cuda:0")), sys.argv[1])

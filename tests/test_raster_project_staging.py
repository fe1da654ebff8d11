"""The projection kernel stages a CTA's parameter rows in shared memory when the view count C divides 8 or is a multiple of 8,
and reads them from global memory otherwise.  Every such C, with a Gaussian count that leaves the last CTA's rows partly
past the end, must reproduce C single-view calls bit for bit: radii, tiles per Gaussian, the records of the visible
(Gaussian, view) pairs and every view's tile counters."""
import pytest
import torch

from artdeco_b200 import synthetic

KEYS = ("means", "quats", "scales", "opacities", "sh")


@pytest.mark.gpu
@pytest.mark.parametrize("C", [2, 4, 6, 16])
def test_project_multi_equals_single_view_calls(cuda, C):
    from artdeco_b200 import raster as R
    N, W, H = 20_000 + 77, 480, 272          # 77 Gaussians past the last full CTA at every C
    sc = synthetic.raster_scene(N, seed=11)
    t = {k: sc[k].to(cuda) for k in KEYS}
    cams = [synthetic.camera(W, H, view=0.5 * v) for v in range(C)]
    Vs = torch.stack([c[0] for c in cams]).to(cuda)
    Ks = torch.stack([c[1] for c in cams]).to(cuda)
    P = torch.inverse(Vs)[:, :3, 3].contiguous()
    cnt = R.new_tile_counts(W, H, cuda, C)
    radii, splats, tpg = R.project_multi(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], 3, Vs, Ks, P, W, H,
                                         0.01, 0.01, 1e10, 0.0, cnt)
    n_vis = 0
    for c in range(C):
        cnt1 = R.new_tile_counts(W, H, cuda)
        r1, s1, tpg1 = R.project(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], 3, Vs[c], Ks[c], P[c], W, H,
                                 0.01, 0.01, 1e10, 0.0, tile_counts=cnt1)
        assert torch.equal(radii[c], r1), f"view {c}: radii"
        assert torch.equal(tpg[c], tpg1), f"view {c}: tiles per Gaussian"
        vis = (r1 != 0).any(-1)
        assert torch.equal(splats[c][vis], s1[vis]), f"view {c}: records"
        assert torch.equal(cnt[c], cnt1), f"view {c}: tile counters"
        n_vis += int(vis.sum())
    assert n_vis > C * N // 10, "the cameras see too little of the scene for the check to mean anything"

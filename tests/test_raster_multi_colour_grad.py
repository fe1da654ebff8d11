"""In one process, multi_view_backward takes the masked colour gradient g_rgb [C,N,3] from the geometry backward kernel instead
of a separate pass over the records: it must equal mask_rgb_grad of the same records bit for bit, for every (view,
Gaussian) pair, visible or not."""
import pytest
import torch

from artdeco_b200 import synthetic

KEYS = ("means", "quats", "scales", "opacities", "sh")


@pytest.mark.gpu
def test_single_process_colour_gradient_equals_mask(cuda):
    from artdeco_b200 import raster as R
    N, W, H, C = 20_000 + 77, 480, 272, 3
    sc = synthetic.raster_scene(N, seed=12)
    t = {k: sc[k].to(cuda) for k in KEYS}
    cams = [synthetic.camera(W, H, view=float(v)) for v in (1.0, 3.0, 5.0)]
    Vs = torch.stack([c[0] for c in cams]).to(cuda)
    Ks = torch.stack([c[1] for c in cams]).to(cuda)
    P = torch.inverse(Vs)[:, :3, 3].contiguous()
    g = torch.Generator().manual_seed(13)
    vc, va = torch.randn(C, H, W, 4, generator=g).to(cuda), torch.randn(C, H, W, generator=g).to(cuda)
    cnt = R.new_tile_counts(W, H, cuda, C)
    radii, splats, tpg = R.project_multi(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], 3, Vs, Ks, P, W, H,
                                         0.01, 0.01, 1e10, 0.0, cnt)
    _, vals, offs, _, _ = R.intersect_multi(radii, splats, tpg, W, H, cnt)
    col, alp, last = R.blend_forward_multi(W, H, splats, vals, offs)
    v_splats = R.blend_backward_multi(W, H, splats, vals, offs, alp, last, vc, va)
    g_rgb = torch.full((C, N, 3), float("nan"), device=cuda)          # poison: every entry must be written
    R.multi_view_backward(t["means"], t["quats"], t["scales"], t["sh"], 3, Vs, Ks, P, W, H, radii, splats, v_splats,
                          out={"g_rgb": g_rgb})
    want = R.mask_rgb_grad(splats, v_splats, torch.empty(C, N, 3, device=cuda))
    assert torch.equal(g_rgb, want)
    assert bool((want != 0).any()), "no visible colour gradient: the check would be vacuous"

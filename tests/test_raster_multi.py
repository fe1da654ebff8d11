"""The multi-view batch stage by stage (raster.project_multi / intersect_multi / blend_forward_multi / blend_backward_multi):
one launch per stage for C views must reproduce C single-view calls — radii, records and tile counts bit for bit, sorted
values and offsets up to the view's segment base, images and last contributors bit for bit, gradients up to the order of
the floating-point REDs."""
import ctypes

import pytest
import torch

from artdeco_b200 import synthetic
from helpers import rel_err

KEYS = ("means", "quats", "scales", "opacities", "sh")


def test_multi_entry_points_refuse_bad_arguments_before_touching_the_device():
    """Status 1 + adb_last_error, no CUDA call: C <= 0, null pointers, capacities that are negative or that the int32 offsets
    cannot address."""
    from artdeco_b200 import _lib
    import artdeco_b200  # noqa: F401  (registers every signature)
    L = _lib.lib()

    def refused(rc, needle):
        msg = L.adb_last_error()
        return rc == 1 and msg is not None and needle in msg.decode()

    caps = (ctypes.c_longlong * 2)(100, 100)
    bad = (ctypes.c_longlong * 2)(100, -1)
    huge = (ctypes.c_longlong * 2)(2_000_000_000, 2_000_000_000)
    dummy = ctypes.c_void_p(16)          # never dereferenced: every call below is refused before a launch
    pf = L.adb_raster_project_fwd_multi
    assert refused(pf(8, 0, dummy, dummy, dummy, dummy, None, 3, dummy, dummy, None, 64, 64, 0.01, 0.01, 1e10, 0.0,
                      dummy, dummy, dummy, dummy, None), "adb_raster_project_fwd_multi")
    assert refused(pf(8, 2, None, dummy, dummy, dummy, None, 3, dummy, dummy, None, 64, 64, 0.01, 0.01, 1e10, 0.0,
                      dummy, dummy, dummy, dummy, None), "adb_raster_project_fwd_multi: null pointer")
    assert refused(pf(8, 2, dummy, dummy, dummy, dummy, None, 3, dummy, dummy, None, 64, 64, 0.01, 0.01, 1e10, 0.0,
                      dummy, dummy, dummy, None, None), "adb_raster_project_fwd_multi: null tile_counts")
    sc = L.adb_raster_tile_scan_multi
    assert refused(sc(0, 64, 64, caps, dummy, dummy, None, None, None), "adb_raster_tile_scan_multi")
    assert refused(sc(65, 64, 64, caps, dummy, dummy, None, None, None), "adb_raster_tile_scan_multi")
    assert refused(sc(2, 64, 64, None, dummy, dummy, None, None, None), "adb_raster_tile_scan_multi: null capacities")
    assert refused(sc(2, 64, 64, bad, dummy, dummy, None, None, None), "adb_raster_tile_scan_multi: capacities")
    assert refused(sc(2, 64, 64, huge, dummy, dummy, None, None, None), "adb_raster_tile_scan_multi: capacities")
    assert refused(sc(2, 64, 64, caps, None, dummy, None, None, None), "adb_raster_tile_scan_multi: null pointer")
    assert refused(sc(2, 64, 64, caps, dummy, None, None, None, None), "adb_raster_tile_scan_multi: null pointer")  # no output
    bf, bb = L.adb_raster_blend_fwd_multi, L.adb_raster_blend_bwd_multi
    assert refused(bf(8, 0, 64, 64, dummy, dummy, dummy, dummy, dummy, dummy, None, None), "adb_raster_blend_fwd_multi")
    assert refused(bf(8, 2, 64, 64, dummy, dummy, dummy, None, dummy, dummy, None, None), "adb_raster_blend_fwd_multi: null pointer")
    assert refused(bf(8, 2, 64, 64, None, dummy, dummy, dummy, dummy, dummy, None, None), "adb_raster_blend_fwd_multi: null pointer")
    assert refused(bb(8, 0, 64, 64, dummy, dummy, dummy, dummy, dummy, dummy, dummy, dummy, None, None),
                   "adb_raster_blend_bwd_multi")
    assert refused(bb(8, 2, 64, 64, dummy, dummy, dummy, dummy, dummy, dummy, dummy, None, None, None),
                   "adb_raster_blend_bwd_multi: null pointer")
    assert refused(bb(-1, 2, 64, 64, dummy, dummy, dummy, dummy, dummy, dummy, dummy, dummy, None, None),
                   "adb_raster_blend_bwd_multi: bad sizes")
    # an empty scene (N = 0): the backward has nothing to accumulate and needs no records
    assert bb(0, 2, 64, 64, None, None, dummy, dummy, dummy, dummy, dummy, None, None, None) == 0
    # an empty problem is accepted without a launch
    assert L.adb_raster_project_fwd_multi(0, 2, None, None, None, None, None, 3, None, None, None, 64, 64, 0.01, 0.01, 1e10,
                                          0.0, None, None, None, dummy, None) == 0


def _setup(N, W, H, views, dev, seed):
    sc = synthetic.raster_scene(N, seed=seed)
    cams = [synthetic.camera(W, H, view=float(v)) for v in views]
    Vs = torch.stack([c[0] for c in cams]).to(dev)
    Ks = torch.stack([c[1] for c in cams]).to(dev)
    P = torch.inverse(Vs)[:, :3, 3].contiguous()
    t = {k: sc[k].to(dev) for k in KEYS}
    g = torch.Generator().manual_seed(seed + 1)
    Cn = len(views)
    vc, va = torch.randn(Cn, H, W, 4, generator=g).to(dev), torch.randn(Cn, H, W, generator=g).to(dev)
    return t, Vs, Ks, P, vc, va


def _single(t, Vs, Ks, P, vc, va, W, H, c):
    from artdeco_b200 import raster as R
    N = t["means"].shape[0]
    cnt = R.new_tile_counts(W, H, t["means"].device)
    radii, splats, tpg = R.project(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], 3, Vs[c], Ks[c], P[c], W, H,
                                   0.01, 0.01, 1e10, 0.0, tile_counts=cnt)
    keys, vals, offs, n = R.intersect(radii, splats, tpg, W, H, counts=cnt)
    hits = torch.full((max(1, n),), 0xAB, dtype=torch.uint8, device=radii.device)        # poison: unwritten entries stay so
    col, alp, last = R.blend_forward(W, H, N, splats, vals, offs, hits=hits)
    v_splats = R.blend_backward(W, H, N, splats, vals, offs, alp, last, vc[c].contiguous(), va[c].contiguous(), hits=hits)
    return dict(radii=radii, splats=splats, tpg=tpg, keys=keys, vals=vals, offs=offs, n=n, hits=hits, col=col, alp=alp,
                last=last, v_splats=v_splats)


def _batched(t, Vs, Ks, P, vc, va, W, H, capacities=None):
    from artdeco_b200 import raster as R
    Cn = Vs.shape[0]
    cnt = R.new_tile_counts(W, H, t["means"].device, Cn)
    radii, splats, tpg = R.project_multi(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], 3, Vs, Ks, P, W, H,
                                         0.01, 0.01, 1e10, 0.0, cnt)
    keys, vals, offs, info, seg = R.intersect_multi(radii, splats, tpg, W, H, cnt, capacities=capacities)
    hits = torch.full((max(1, vals.numel()),), 0xAB, dtype=torch.uint8, device=radii.device)
    col, alp, last = R.blend_forward_multi(W, H, splats, vals, offs, hits=hits)
    v_splats = R.blend_backward_multi(W, H, splats, vals, offs, alp, last, vc, va, hits=hits)
    assert not bool((cnt[:, : cnt.shape[1] // 2] != 0).any()), "the tile counters return to zero"
    return dict(radii=radii, splats=splats, tpg=tpg, keys=keys, vals=vals, offs=offs, info=info, seg=seg, hits=hits, col=col,
                alp=alp, last=last, v_splats=v_splats)


def _check_view(b, s, c, N, tile_bits):
    base = sum(b["seg"][:c])
    n = s["n"]
    assert torch.equal(b["radii"][c], s["radii"]) and torch.equal(b["tpg"][c], s["tpg"]), f"view {c}: radii / tiles"
    vis = (s["radii"] > 0).any(-1)                         # culled Gaussians get no record
    assert torch.equal(b["splats"][c][vis], s["splats"][vis]), f"view {c}: splat records"
    assert torch.equal(b["offs"][c] - base, s["offs"]), f"view {c}: offsets"
    assert torch.equal(b["vals"][base:base + n] - c * N, s["vals"]), f"view {c}: sorted values"
    assert torch.equal(b["keys"][base:base + n], s["keys"] | (c << (32 + tile_bits))), f"view {c}: keys"
    assert torch.equal(b["hits"][base:base + n], s["hits"][:n]), f"view {c}: hit mask"
    assert torch.equal(b["col"][c], s["col"]) and torch.equal(b["alp"][c], s["alp"]), f"view {c}: image"
    last = b["last"][c]
    assert torch.equal(torch.where(last == 0, last, last - base), s["last"]), f"view {c}: last_ids"
    assert rel_err(b["v_splats"][c], s["v_splats"]) < 2e-6, f"view {c}: v_splats"


def _tile_bits(W, H):
    n = ((W + 15) // 16) * ((H + 15) // 16)
    return n.bit_length()


@pytest.mark.gpu
@pytest.mark.parametrize("N,W,H,views", [(20000, 480, 272, (1.0, 3.0, 5.0)),
                                         (1_000_000, 1920, 1080, tuple(range(8)))], ids=["small_C3", "bench_C8_1M_1080p"])
def test_batched_stages_equal_single_view_calls(cuda, N, W, H, views):
    t, Vs, Ks, P, vc, va = _setup(N, W, H, views, cuda, seed=4)
    b = _batched(t, Vs, Ks, P, vc, va, W, H)
    assert b["seg"] == [int(x) for x in b["info"]["n_isect"].tolist()] and not bool(b["info"]["overflow"].any())
    for c in range(len(views)):
        s = _single(t, Vs, Ks, P, vc, va, W, H, c)
        assert s["n"] == b["seg"][c]
        _check_view(b, s, c, N, _tile_bits(W, H))
        del s


@pytest.mark.gpu
def test_capacity_mode_flags_only_the_undersized_view(cuda):
    N, W, H, views = 20000, 480, 272, (0.0, 2.5, 5.0)
    t, Vs, Ks, P, vc, va = _setup(N, W, H, views, cuda, seed=9)
    exact = _batched(t, Vs, Ks, P, vc, va, W, H)
    n = exact["seg"]
    caps = [n[0] + 1000, n[1] // 2, n[2] + 3]
    b = _batched(t, Vs, Ks, P, vc, va, W, H, capacities=caps)
    assert b["seg"] == caps and b["vals"].numel() == sum(caps)
    assert b["info"]["n_isect"].tolist() == n and b["info"]["overflow"].tolist() == [0, 1, 0]
    for c in (0, 2):
        s = _single(t, Vs, Ks, P, vc, va, W, H, c)
        _check_view(b, s, c, N, _tile_bits(W, H))
    assert not torch.equal(b["col"][1], exact["col"][1]), "the undersized view lost intersections"


@pytest.mark.gpu
@pytest.mark.parametrize("capacity", [None, [64, 64]], ids=["sized_by_sync", "capacity_mode"])
def test_empty_scene_renders_and_differentiates_on_the_multi_view_path(cuda, capacity):
    """No Gaussians (after a cull or a prune): rasterization(viewmats[C > 1]) returns empty images and zero-sized gradients,
    forward and backward, as the single-view path does."""
    from artdeco_b200 import raster as R
    W, H = 70, 50                                         # ragged: not a multiple of 16
    cams = [synthetic.camera(W, H, view=v, focal=50.0) for v in (0.0, 3.0)]
    Vs = torch.stack([c[0] for c in cams]).to(cuda).requires_grad_(True)
    Ks = torch.stack([c[1] for c in cams]).to(cuda)
    t = {k: torch.zeros(*s, device=cuda, requires_grad=True)
         for k, s in (("means", (0, 3)), ("quats", (0, 4)), ("scales", (0, 3)), ("opacities", (0,)), ("sh", (0, 16, 3)))}
    c, a, meta = R.rasterization(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], Vs, Ks, W, H,
                                 render_mode="RGB+D", sh_degree=3, eps2d=0.01, isect_capacity=capacity)
    assert c.shape == (2, H, W, 4) and a.shape == (2, H, W, 1) and meta["radii"].shape == (2, 0, 2)
    assert not c.any() and not a.any() and meta["flatten_ids"].numel() == 0 and int(meta["isect_overflow"]) == 0
    (c.sum() + a.sum()).backward()
    torch.cuda.synchronize()
    for k, v in t.items():
        assert v.grad is not None and v.grad.shape == v.shape, k
    assert Vs.grad is not None and not Vs.grad.any()

"""Rasterizer parity (GPU, through the C ABI) against the C oracle, stage by stage and end to end.

Contracts (BASELINE.json north_star):
  * integer work — radii, tile counts, tile keys, sort order (values), tile offsets, last_ids — BIT-EXACT;
  * float work — splat records, colours/depth/alpha, every gradient — within 1e-4 of the tensor's scale.
The blend's discrete decisions (alpha < 1/255 skip, T <= 1e-4 stop) are evaluated with ex2.approx on the GPU and
expf on the CPU, so a handful of pixels may legitimately take the other branch: the image/gradient checks admit
an outlier fraction of 1e-4 and report the count."""
import numpy as np
import pytest
import torch

import oracle
from artdeco_b200 import synthetic
from helpers import assert_close, rel_err

KEYS = ("means", "quats", "scales", "opacities", "sh")


def _scene(N, W, H, seed=0, view=2.0, **kw):
    sc = synthetic.raster_scene(N, seed=seed, **kw)
    V, K = synthetic.camera(W, H, view=view)
    return sc, V, K


def _gpu_stages(sc, V, K, W, H, dev):
    from artdeco_b200 import raster as R
    t = {k: sc[k].to(dev) for k in KEYS}
    Vd, Kd = V.to(dev), K.to(dev)
    campos = torch.inverse(Vd)[:3, 3].contiguous()
    radii, splats, tpg = R.project(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], 3, Vd, Kd, campos, W,
                                   H, 0.01, 0.01, 1e10, 0.0)
    keys, vals, offs, n = R.intersect(radii, splats, tpg, W, H)
    colors, alphas, last = R.blend_forward(W, H, radii.shape[0], splats, vals, offs)
    return dict(radii=radii, splats=splats, tpg=tpg, keys=keys, vals=vals, offs=offs, colors=colors, alphas=alphas,
                last=last, n=n, t=t, V=Vd, K=Kd, campos=campos)


@pytest.mark.gpu
@pytest.mark.parametrize("N,W,H,view", [(3000, 320, 192, 1.0), (20000, 640, 360, 5.0), (100000, 1920, 1080, 3.5)])
def test_forward_stages_match_oracle(cuda, N, W, H, view):
    sc, V, K = _scene(N, W, H, seed=7 if N == 3000 else 0, view=view)
    f = oracle.rasterize_fwd(*[sc[k].numpy() for k in KEYS], V.numpy(), K.numpy(), W, H)
    g = _gpu_stages(sc, V, K, W, H, cuda)
    # --- bit-exact integer contract ---
    assert np.array_equal(g["radii"].cpu().numpy(), f["radii"]), "radii"
    assert np.array_equal(g["tpg"].cpu().numpy(), f["tiles_per_gauss"]), "tiles_per_gauss"
    assert g["n"] == len(f["keys"])
    assert np.array_equal(g["keys"].cpu().numpy(), f["keys"]), "sorted tile keys"
    assert np.array_equal(g["vals"].cpu().numpy(), f["vals"]), "sort indices"
    assert np.array_equal(g["offs"].cpu().numpy()[:-1], f["tile_offsets"]), "tile offsets"
    assert int(g["offs"][-1]) == g["n"]
    # --- float contract on the splat record (visible Gaussians only) ---
    vis = (f["radii"] > 0).any(1)
    sp = g["splats"].cpu().numpy()[vis]
    assert np.array_equal(sp[:, 0:2], f["means2d"][vis]) and np.array_equal(sp[:, 11], f["depths"][vis]), \
        "projection is compiled without FMA contraction and must be bit-identical to the oracle"
    assert np.array_equal(sp[:, 2:5], f["conics"][vis])
    assert_close(sp[:, 8:11], f["rgb"][vis], what="sh colours")
    # --- image ---
    assert_close(g["colors"], f["colors"], what="colors", max_outlier_frac=1e-4)
    assert_close(g["alphas"], f["alphas"], what="alphas", max_outlier_frac=1e-4)
    mism = (g["last"].cpu().numpy() != f["last_ids"]).mean()
    assert mism <= 1e-4, f"last_ids differ on {mism:.2e} of pixels"


@pytest.mark.gpu
def test_golden_fixture_bit_exact(cuda):
    import pathlib
    gf = np.load(pathlib.Path(__file__).parent / "golden" / "raster_small.npz")
    sc, V, K = _scene(int(gf["N"]), int(gf["W"]), int(gf["H"]), seed=int(gf["seed"]), view=float(gf["view"]))
    g = _gpu_stages(sc, V, K, int(gf["W"]), int(gf["H"]), cuda)
    assert np.array_equal(g["radii"].cpu().numpy(), gf["radii"])
    assert np.array_equal(g["keys"].cpu().numpy(), gf["keys"])
    assert np.array_equal(g["vals"].cpu().numpy(), gf["vals"])
    assert np.array_equal(g["offs"].cpu().numpy()[:-1], gf["tile_offsets"])
    assert_close(g["colors"], gf["colors"], what="colors", max_outlier_frac=1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("N,W,H", [(4000, 320, 192), (50000, 960, 540)])
def test_backward_matches_oracle(cuda, N, W, H):
    from artdeco_b200 import raster as R
    sc, V, K = _scene(N, W, H, seed=11, view=5.0, scale_range=(0.01, 0.15))
    args = [sc[k].numpy() for k in KEYS]
    f = oracle.rasterize_fwd(*args, V.numpy(), K.numpy(), W, H)
    vc, va = synthetic.upstream_grads(W, H, seed=1)
    b = oracle.rasterize_bwd(*args, V.numpy(), f, vc[0].numpy(), va[0, ..., 0].numpy())

    t = {k: sc[k].to(cuda).requires_grad_(True) for k in KEYS}
    Vd = V.to(cuda).requires_grad_(True)
    colors, alphas, meta = R.rasterization(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], Vd[None],
                                           K.to(cuda)[None], W, H, render_mode="RGB+D", sh_degree=3, eps2d=0.01)
    ((colors * vc.to(cuda)).sum() + (alphas * va.to(cuda)).sum()).backward()
    fr = 2e-4  # gradient tensors: a flipped blend decision moves a few Gaussians' gradients
    assert_close(t["means"].grad, b["v_means"], what="v_means", max_outlier_frac=fr)
    assert_close(t["quats"].grad, b["v_quats"], what="v_quats", max_outlier_frac=fr)
    assert_close(t["scales"].grad, b["v_scales"], what="v_scales", max_outlier_frac=fr)
    assert_close(t["opacities"].grad, b["v_opac"], what="v_opac", max_outlier_frac=fr)
    assert_close(t["sh"].grad, b["v_sh"], what="v_sh", max_outlier_frac=fr)
    Vt = V.double().requires_grad_(True)
    (torch.inverse(Vt)[:3, 3] * torch.tensor(b["v_campos"], dtype=torch.float64)).sum().backward()
    vV = b["v_viewmat"].astype(np.float64) + Vt.grad.numpy()
    assert rel_err(Vd.grad.cpu().numpy()[:3], vV[:3]) < 1e-3, "viewmat gradient (sum over all Gaussians)"


@pytest.mark.gpu
@pytest.mark.parametrize("N,view", [(100_000, 0.0), (1_000_000, 3.5)], ids=["config2_100k_1080p", "headline_1M_1080p"])
def test_baseline_configs_fwd_bwd_match_oracle(cuda, N, view):
    """BASELINE.json configs[1] (100k Gaussians, 1080p) and the headline workload (1M, 1080p, view 3.5 -- exactly what
    bench.py times): forward AND backward against the C oracle on the same seeded inputs, through the public
    rasterization() + autograd.  Keys / sort indices / offsets / radii bit-exact; image and every gradient within 1e-4
    of scale.  (The oracle needs ~2 s per fwd+bwd at 1M on the GPU box's host cores.)"""
    from artdeco_b200 import raster as R
    W, H = 1920, 1080
    sc, V, K = _scene(N, W, H, seed=0, view=view)
    args = [sc[k].numpy() for k in KEYS]
    f = oracle.rasterize_fwd(*args, V.numpy(), K.numpy(), W, H)
    vc, va = synthetic.upstream_grads(W, H, seed=1)
    b = oracle.rasterize_bwd(*args, V.numpy(), f, vc[0].numpy(), va[0, ..., 0].numpy())

    t = {k: sc[k].to(cuda).requires_grad_(True) for k in KEYS}
    Vd = V.to(cuda).requires_grad_(True)
    colors, alphas, meta = R.rasterization(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], Vd[None],
                                           K.to(cuda)[None], W, H, render_mode="RGB+D", sh_degree=3, eps2d=0.01)
    assert np.array_equal(meta["radii"][0].cpu().numpy(), f["radii"]), "radii"
    assert np.array_equal(meta["isect_ids"].cpu().numpy(), f["keys"]), "sorted tile keys"
    assert np.array_equal(meta["flatten_ids"].cpu().numpy(), f["vals"]), "sort indices"
    assert np.array_equal(meta["isect_offsets"].reshape(-1).cpu().numpy(), f["tile_offsets"]), "tile offsets"
    assert_close(colors[0], f["colors"], what="colors", max_outlier_frac=1e-4)
    assert_close(alphas[0, ..., 0], f["alphas"], what="alphas", max_outlier_frac=1e-4)
    ((colors * vc.to(cuda)).sum() + (alphas * va.to(cuda)).sum()).backward()
    fr = 2e-4
    assert_close(t["means"].grad, b["v_means"], what="v_means", max_outlier_frac=fr)
    assert_close(t["quats"].grad, b["v_quats"], what="v_quats", max_outlier_frac=fr)
    assert_close(t["scales"].grad, b["v_scales"], what="v_scales", max_outlier_frac=fr)
    assert_close(t["opacities"].grad, b["v_opac"], what="v_opac", max_outlier_frac=fr)
    assert_close(t["sh"].grad, b["v_sh"], what="v_sh", max_outlier_frac=fr)
    Vt = V.double().requires_grad_(True)
    (torch.inverse(Vt)[:3, 3] * torch.tensor(b["v_campos"], dtype=torch.float64)).sum().backward()
    vV = b["v_viewmat"].astype(np.float64) + Vt.grad.numpy()
    # a sum over up to 1M Gaussians in fp32 on both sides (different orders): 1e-3 of scale
    assert rel_err(Vd.grad.cpu().numpy()[:3], vV[:3]) < 1e-3, "viewmat gradient"


@pytest.mark.gpu
def test_multi_view_batch_equals_sum_of_single_views(cuda):
    """BASELINE config 4 semantics (SURVEY.md §8e: the step becomes "sum of C view losses"): rasterization() with C=3
    viewmats must return per-view images identical to three C=1 calls, gsplat's concatenated isect ids with the camera bits
    set, and parameter gradients equal to the SUM of the single-view gradients (multi-view projection/SH backward kernels),
    plus per-camera viewmat gradients equal to the single-view ones."""
    from artdeco_b200 import raster as R
    N, W, H = 30000, 640, 352
    sc = synthetic.raster_scene(N, seed=3)
    cams = [synthetic.camera(W, H, view=v) for v in (0.0, 3.5, 7.0)]
    Vs = torch.stack([c[0] for c in cams]).to(cuda)
    Ks = torch.stack([c[1] for c in cams]).to(cuda)
    g = torch.Generator().manual_seed(5)
    vc, va = torch.randn(3, H, W, 4, generator=g).to(cuda), torch.randn(3, H, W, 1, generator=g).to(cuda)
    tm = {k: sc[k].to(cuda).requires_grad_(True) for k in KEYS}
    Vm = Vs.clone().requires_grad_(True)
    cm, am, meta = R.rasterization(tm["means"], tm["quats"], tm["scales"], tm["opacities"], tm["sh"], Vm, Ks, W, H,
                                   render_mode="RGB+D", sh_degree=3, eps2d=0.01)
    assert cm.shape == (3, H, W, 4) and am.shape == (3, H, W, 1) and meta["radii"].shape == (3, N, 2)
    ((cm * vc).sum() + (am * va).sum()).backward()
    ts = {k: sc[k].to(cuda).requires_grad_(True) for k in KEYS}
    tb = oracle.lib().adbo_tile_bits(W, H)
    ids, flat = [], []
    for c in range(3):
        Vc = Vs[c].clone().requires_grad_(True)
        c1, a1, m1 = R.rasterization(ts["means"], ts["quats"], ts["scales"], ts["opacities"], ts["sh"], Vc[None], Ks[c:c + 1], W,
                                     H, render_mode="RGB+D", sh_degree=3, eps2d=0.01)
        assert torch.equal(c1[0], cm[c]) and torch.equal(a1[0], am[c]) and torch.equal(m1["radii"][0], meta["radii"][c])
        ((c1 * vc[c:c + 1]).sum() + (a1 * va[c:c + 1]).sum()).backward()
        assert rel_err(Vm.grad[c], Vc.grad) < 1e-4, "per-camera viewmat gradient"
        ids.append(m1["isect_ids"] | (c << (32 + tb)))
        flat.append(m1["flatten_ids"] + c * N)
    assert torch.equal(meta["isect_ids"], torch.cat(ids)) and torch.equal(meta["flatten_ids"], torch.cat(flat))
    for k in KEYS:
        # same per-pair arithmetic, different summation order over the three views: fp32 rounding only
        assert rel_err(tm[k].grad, ts[k].grad) < 2e-5, k


@pytest.mark.gpu
def test_multi_view_exchange_algebra_matches_single_process(cuda):
    """The multi-GPU exchange (gather of 12 B colour gradients + sum of the 11 geometry floats, SH gradient of every view expanded
    locally, direction term added per rank) emulated in one process: 4 views split over two "ranks" must reproduce the
    single-process 4-view gradients."""
    from artdeco_b200 import raster as R
    N, W, H = 20000, 480, 272
    sc = synthetic.raster_scene(N, seed=8)
    cams = [synthetic.camera(W, H, view=v) for v in (1.0, 3.0, 5.0, 7.0)]
    Vs = torch.stack([c[0] for c in cams]).to(cuda)
    Ks = torch.stack([c[1] for c in cams]).to(cuda)
    P = torch.inverse(Vs)[:, :3, 3].contiguous()
    t = {k: sc[k].to(cuda) for k in KEYS}
    g = torch.Generator().manual_seed(6)
    vc, va = torch.randn(4, H, W, 4, generator=g).to(cuda), torch.randn(4, H, W, generator=g).to(cuda)

    def local(cams_idx):
        Cn = len(cams_idx)
        radii = torch.empty(Cn, N, 2, dtype=torch.int32, device=cuda)
        splats = torch.empty(Cn, N, 12, device=cuda)
        tpg = torch.empty(Cn, N, dtype=torch.int32, device=cuda)
        v_splats = torch.zeros(Cn, N, 12, device=cuda)
        for j, c in enumerate(cams_idx):
            R.project(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], 3, Vs[c], Ks[c], P[c], W, H, 0.01, 0.01,
                      1e10, 0.0, out=(radii[j], splats[j], tpg[j]))
            keys, vals, offs, _ = R.intersect(radii[j], splats[j], tpg[j], W, H)
            col, alp, last = R.blend_forward(W, H, N, splats[j], vals, offs)
            R.blend_backward(W, H, N, splats[j], vals, offs, alp, last, vc[c].contiguous(), va[c].contiguous(), out=v_splats[j])
        return radii, splats, v_splats

    idx_all = [0, 1, 2, 3]
    ra, sa, va_ = local(idx_all)
    full = R.multi_view_backward(t["means"], t["quats"], t["scales"], t["sh"], 3, Vs, Ks, P, W, H, ra, sa, va_)

    class FakeExchange:            # what the exchange does, done by hand: "rank" 0 = views 0,1; "rank" 1 = views 2,3
        def __init__(self, g_all=None, p_all=None):
            self.g, self.p, self.g_all, self.p_all = [], [], g_all, p_all

        def start_gather(self, g_rgb, campos):
            self.g.append(g_rgb.clone()); self.p.append(campos.clone())

        def start_reduce(self):
            pass

        def wait_gather(self):
            return self.g_all, self.p_all

        def wait_reduce(self):
            pass

    # pass 1: what each rank hands to the gather (its local views' masked colour gradients and camera centres)
    loc, rows = [], []
    for ranks_views in ([0, 1], [2, 3]):
        r_, s_, v_ = local(ranks_views)
        loc.append((r_, s_, v_))
        rows.append(R.mask_rgb_grad(s_, v_, torch.empty(2, N, 3, device=cuda)))
    g_all, p_all = torch.cat(rows), torch.cat([P[[0, 1]], P[[2, 3]]])
    # pass 2: every rank's backward with the gathered table; its geometry outputs are PARTIAL sums (local views only, the
    # colour's direction term included) that the reduce adds up
    parts = []
    for k_, ranks_views in enumerate(([0, 1], [2, 3])):
        r_, s_, v_ = loc[k_]
        ex = FakeExchange(g_all, p_all)
        out = R.multi_view_backward(t["means"], t["quats"], t["scales"], t["sh"], 3, Vs[ranks_views], Ks[ranks_views],
                                    P[ranks_views], W, H, r_, s_, v_, exchange=ex)
        assert torch.equal(ex.g[0], rows[k_]), "the backward hands the masked colour gradients of its local views to the gather"
        parts.append([o.clone() for o in out[:5]])
    for k_, name in enumerate(("v_means", "v_quats", "v_scales", "v_opac")):
        assert rel_err(parts[0][k_] + parts[1][k_], full[k_]) < 2e-5, name
    assert rel_err(parts[0][4], full[4]) < 2e-5 and torch.equal(parts[0][4], parts[1][4]), "v_sh expanded from the gathered rows"
    v_sh, v_means_sh = torch.empty(N, 16, 3, device=cuda), torch.empty(N, 3, device=cuda)
    from artdeco_b200 import _lib
    _lib.call("adb_raster_sh_bwd_multi", N, 4, _lib.ptr(t["means"]), _lib.ptr(t["sh"]), 3, _lib.ptr(p_all), _lib.ptr(g_all),
              _lib.ptr(v_sh), _lib.ptr(v_means_sh), 0, 0, 0, None, _lib.stream())
    assert rel_err(v_sh, full[4]) < 2e-5, "fused kernel on the gathered table"
    parts = [(rows[0], P[[0, 1]].contiguous()), (rows[1], P[[2, 3]].contiguous())]
    # accumulate / skip options of the fused kernel: "rank 0" expands its local views (0,1) first, then adds the others from
    # a view-major gathered table [C_local, world] (entry c belongs to rank c % world) with its own entries skipped
    world, rank = 2, 0
    g_vm = torch.stack([torch.stack([parts[r][0][c] for r in range(world)]) for c in range(2)]).reshape(4, N, 3).contiguous()
    p_vm = torch.stack([torch.stack([parts[r][1][c] for r in range(world)]) for c in range(2)]).reshape(4, 3).contiguous()
    v_sh2, v_ms2 = torch.empty(N, 16, 3, device=cuda), torch.empty(N, 3, device=cuda)
    _lib.call("adb_raster_sh_bwd_multi", N, 2, _lib.ptr(t["means"]), _lib.ptr(t["sh"]), 3, _lib.ptr(parts[rank][1].contiguous()),
              _lib.ptr(parts[rank][0].contiguous()), _lib.ptr(v_sh2), _lib.ptr(v_ms2), 0, 0, 0, None, _lib.stream())
    _lib.call("adb_raster_sh_bwd_multi", N, 4, _lib.ptr(t["means"]), _lib.ptr(t["sh"]), 3, _lib.ptr(p_vm), _lib.ptr(g_vm),
              _lib.ptr(v_sh2), _lib.ptr(v_ms2), 3, world, rank, None, _lib.stream())
    assert rel_err(v_sh2, v_sh) < 1e-5 and rel_err(v_ms2, v_means_sh) < 1e-5, "split (local first, then remote) == one pass"


@pytest.mark.gpu
@pytest.mark.parametrize("N,W,H,view,kw", [(3000, 320, 192, 1.0, {}), (50000, 960, 544, 5.0, dict(scale_range=(0.01, 0.15))),
                                           (100000, 1920, 1080, 3.5, {})])
def test_backward_from_the_forward_hit_mask_equals_backward_with_its_own_culling(cuda, N, W, H, view, kw):
    """adb_raster_blend_fwd / adb_raster_blend_bwd with a hit_mask: the forward records which warps each (tile, splat) entry can
    reach and the backward builds its hit lists from that record.  Same images bit for bit; same gradients up to the order of the
    floating-point REDs between tiles."""
    from artdeco_b200 import raster as R
    sc, V, K = _scene(N, W, H, seed=21, view=view, **kw)
    st = _gpu_stages(sc, V, K, W, H, cuda)
    vals, offs, splats = st["vals"], st["offs"], st["splats"]
    hits = torch.full((max(1, vals.numel()),), 0xAB, dtype=torch.uint8, device=cuda)      # poison: unwritten entries stay unused
    col, alp, last = R.blend_forward(W, H, N, splats, vals, offs, hits=hits)
    assert torch.equal(col, st["colors"]) and torch.equal(alp, st["alphas"]) and torch.equal(last, st["last"])
    vc, va = synthetic.upstream_grads(W, H, seed=2)
    vcd, vad = vc[0].contiguous().to(cuda), va[0, ..., 0].contiguous().to(cuda)
    g_own = R.blend_backward(W, H, N, splats, vals, offs, alp, last, vcd, vad)
    g_hit = R.blend_backward(W, H, N, splats, vals, offs, alp, last, vcd, vad, hits=hits)
    assert rel_err(g_hit, g_own) < 2e-6
    # the mask is a pure function of the forward's inputs: the last contributor of every pixel must be marked for its warp
    lastc = last.cpu().numpy()
    hm = hits.cpu().numpy()
    ys, xs = np.nonzero(alp.cpu().numpy() > 0)
    sel = np.random.default_rng(0).choice(len(ys), size=min(2000, len(ys)), replace=False) if len(ys) else []
    for k_ in sel:
        y, x = int(ys[k_]), int(xs[k_])
        warp = ((y % 16) // 4) * 2 + ((x % 16) // 8)
        assert (hm[lastc[y, x]] >> warp) & 1, f"pixel ({x},{y}): its last contributor is not marked for warp {warp}"


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [True, False], ids=["per_view_graphs", "eager"])
def test_multi_gpu_step_path_on_one_rank_matches_the_single_process_step(cuda, graph):
    """multiview.MultiViewStep(world > 1) takes the multi-GPU route — one CUDA graph PER VIEW, per-view gathers, the split SH
    backward, the geometry reduce — which is otherwise only exercised by bench.py --gpus N.  With no process group the exchange
    degenerates to one rank, so the route can run on one GPU and must reproduce the single-graph step."""
    from artdeco_b200.multiview import MultiViewStep
    N, W, H = 20000, 480, 272
    sc = synthetic.raster_scene(N, seed=8)
    cams = [synthetic.camera(W, H, view=v) for v in (1.0, 3.0, 5.0, 7.0)]
    Vs, Ks = torch.stack([c[0] for c in cams]).to(cuda), torch.stack([c[1] for c in cams]).to(cuda)
    t = {k: sc[k].to(cuda) for k in KEYS}
    g = torch.Generator().manual_seed(6)
    vc, va = torch.randn(4, H, W, 4, generator=g).to(cuda), torch.randn(4, H, W, generator=g).to(cuda)
    ref = MultiViewStep(t, Vs, Ks, W, H, world=1)
    eng = MultiViewStep(t, Vs, Ks, W, H, world=2, graph=graph)
    assert ref.exchange is None and eng.exchange is not None
    for e in (ref, eng):
        e.set_upstream(vc, va)
    for step in range(2):                                   # second step = graph replay
        a, b = ref.step(), eng.step()
        torch.cuda.synchronize()
        for k in ("v_means", "v_quats", "v_scales", "v_opac", "v_sh"):
            assert rel_err(b[k], a[k]) < 2e-5, f"step {step}: {k}"
    if graph:
        assert len(eng.graph) == 4 and len(ref.graph) == 1
    assert eng.check_overflow() == ref.check_overflow()


@pytest.mark.gpu
def test_intersect_capacity_mode_has_no_host_sync_and_flags_overflow(cuda):
    """capacity mode of the tile-bucketed intersection: identical keys/vals/offsets without reading the count back, the true
    count and an overflow flag stay on the device, and an undersized capacity is memory-safe and flagged."""
    from artdeco_b200 import raster as R
    N, W, H = 50000, 960, 540
    sc, V, K = _scene(N, W, H, seed=1, view=2.0)
    g = _gpu_stages(sc, V, K, W, H, cuda)
    n = g["n"]
    k2, v2, o2, info = R.intersect(g["radii"], g["splats"], g["tpg"], W, H, capacity=n + 1000)
    assert int(info["n_isect"]) == n and int(info["overflow"]) == 0
    assert torch.equal(k2[:n], g["keys"]) and torch.equal(v2[:n], g["vals"]) and torch.equal(o2, g["offs"])
    sp = g["splats"].cpu().numpy()
    _, kr, vr, orr = oracle.isect(g["radii"].cpu().numpy(), sp[:, 0:2], sp[:, 11], W, H)
    assert len(kr) == n and np.array_equal(g["keys"].cpu().numpy(), kr) and np.array_equal(g["vals"].cpu().numpy(), vr) \
        and np.array_equal(g["offs"].cpu().numpy(), np.append(orr, n)), "the tile-bucketed path must match the C oracle bit for bit"
    k3, v3, o3, info3 = R.intersect(g["radii"], g["splats"], g["tpg"], W, H, capacity=n // 2)
    assert int(info3["overflow"]) == 1 and int(info3["n_isect"]) == n and int(o3[-1]) == n // 2
    m = int(o3[-1])
    full_tiles = int((g["offs"] <= m).sum()) - 1          # tiles that fit entirely are still exact
    assert torch.equal(k3[:int(g["offs"][full_tiles])], g["keys"][:int(g["offs"][full_tiles])])
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_edge_cases(cuda):
    from artdeco_b200 import raster as R
    V, K = synthetic.camera(70, 50, focal=50.0)  # ragged: not a multiple of 16
    z = lambda *s: torch.zeros(*s, device=cuda)
    c, a, meta = R.rasterization(z(0, 3), z(0, 4), z(0, 3), z(0), z(0, 16, 3), V.to(cuda)[None], K.to(cuda)[None], 70, 50,
                                 render_mode="RGB+D", sh_degree=3, eps2d=0.01)
    assert c.shape == (1, 50, 70, 4) and not c.any() and not a.any() and meta["radii"].shape == (1, 0, 2)
    means = torch.tensor([[0, 0, -1.0], [0, 0, 5.0], [500.0, 0, 5.0], [0, 0, 5.0]], device=cuda)
    quats = torch.tensor([[1.0, 0, 0, 0]], device=cuda).repeat(4, 1)
    scales = torch.full((4, 3), 0.1, device=cuda)
    opac = torch.tensor([0.9, 0.001, 0.9, 0.9], device=cuda)
    c, a, meta = R.rasterization(means, quats, scales, opac, z(4, 16, 3), V.to(cuda)[None], K.to(cuda)[None], 70, 50,
                                 render_mode="RGB+D", sh_degree=3, eps2d=0.01)
    assert (meta["radii"][0, :3] == 0).all() and (meta["radii"][0, 3] > 0).all()
    f = oracle.rasterize_fwd(means.cpu().numpy(), quats.cpu().numpy(), scales.cpu().numpy(), opac.cpu().numpy(),
                             np.zeros((4, 16, 3), np.float32), V.numpy(), K.numpy(), 70, 50)
    assert_close(c[0], f["colors"], what="ragged colors")
    assert_close(a[0, ..., 0], f["alphas"], what="ragged alphas")


@pytest.mark.gpu
def test_full_size_properties_1m_1080p(cuda):
    """BASELINE size (1M Gaussians, 1080p): size-independent properties instead of the (slow) oracle."""
    from artdeco_b200 import raster as R
    sc, V, K = _scene(1_000_000, 1920, 1080, seed=0, view=3.5)
    g = _gpu_stages(sc, V, K, 1920, 1080, cuda)
    keys, vals, offs = g["keys"], g["vals"], g["offs"]
    assert g["n"] == int(g["tpg"].sum()) > 1_000_000
    assert bool((keys[1:] >= keys[:-1]).all()), "sortedness"
    same = keys[1:] == keys[:-1]
    assert bool((vals[1:][same] > vals[:-1][same]).all()), "stability"
    tiles = keys >> 32
    T = 120 * 68
    assert bool((offs.long()[:-1] == torch.searchsorted(tiles, torch.arange(T, device=cuda))).all())
    # multiset of values is a permutation of the emission (every Gaussian appears tiles_per_gauss times)
    counts = torch.bincount(vals.long(), minlength=1_000_000)
    assert torch.equal(counts, g["tpg"].long())
    a = g["alphas"]
    assert float(a.min()) >= 0.0 and float(a.max()) <= 1.0 - 1e-4 + 1e-6
    assert torch.isfinite(g["colors"]).all()
    # linearity of the blend in the feature channels: doubling rgb/depth doubles the image
    sp2 = g["splats"].clone()
    sp2[:, 8:12] *= 2
    c2, a2, _ = R.blend_forward(1920, 1080, 1_000_000, sp2, vals, offs)
    assert torch.equal(a2, a) and torch.allclose(c2, 2 * g["colors"], rtol=1e-6, atol=0)


@pytest.mark.gpu
def test_render_lod_matches_oracle_on_the_culled_subset(cuda):
    """BASELINE config 5 at a reduced size: scene.render_lod (LoD d_max cull inside the call, h3dgsv3.py:617-700) must equal
    the oracle's rasterisation of exactly the Gaussians the reference's cull formula keeps, with opacity x fade ratio; the
    no-grad path (one fused gather) and the differentiable path (index_select) must agree to rounding."""
    from artdeco_b200.scene import render_lod
    N, W, H = 120_000, 1280, 720
    sc = synthetic.raster_scene(N, seed=2)
    V, K = synthetic.camera(W, H, view=4.0)
    d_max = sc["d_max"] * 0.25
    cam = torch.inverse(V)[:3, 3]
    dist = (sc["means"] - cam).norm(dim=1, keepdim=True)
    sel = (dist < 2 * d_max).squeeze(-1)
    amask = ((dist > d_max) & (dist < 2 * d_max)).squeeze(-1)
    ratio = (2 * d_max - dist) / d_max
    ratio[~amask] = 1.0
    tanx, tany = W / (2 * float(K[0, 0])), H / (2 * float(K[1, 1]))
    kw = dict(xyz=sc["means"].to(cuda), opacity=sc["opacities"][:, None].to(cuda), f_dc=sc["sh"][:, :1].to(cuda),
              f_rest=sc["sh"][:, 1:].to(cuda), scaling=sc["scales"].to(cuda), rotation=sc["quats"].to(cuda), d_max=d_max.to(cuda),
              tanfovx=tanx, tanfovy=tany, sh_degree=3, eps2d=0.01, bg=torch.tensor([0.1, 0.2, 0.3]))
    with torch.no_grad():
        pkg = render_lod(W, H, V.to(cuda), **kw)
    mism = int((pkg["selection_mask"].cpu() != sel).sum())
    assert mism <= 2, "cull mask (strict '<' on fp32 distances)"
    if mism == 0:
        f = oracle.rasterize_fwd(sc["means"][sel].numpy(), sc["quats"][sel].numpy(), sc["scales"][sel].numpy(),
                                 (sc["opacities"][:, None] * ratio)[sel].squeeze(-1).numpy(), sc["sh"][sel].numpy(), V.numpy(),
                                 K.numpy(), W, H)
        ref = torch.from_numpy(f["colors"][..., :3]).permute(2, 0, 1) + (1 - torch.from_numpy(f["alphas"]))[None] * kw["bg"].view(3, 1, 1)
        assert_close(pkg["render"], ref, what="render", max_outlier_frac=1e-4)
        vis = torch.zeros(N, dtype=torch.bool)
        vis[sel] = torch.from_numpy((f["radii"] > 0).any(1))
        assert torch.equal(pkg["visibility_filter"].cpu(), vis)
        assert pkg["n_isect"] == len(f["keys"])
    kw2 = dict(kw)
    kw2["opacity"] = kw["opacity"].clone().requires_grad_(True)
    pkg2 = render_lod(W, H, V.to(cuda), **kw2)
    # the differentiable path recomputes the fade ratio with torch ops (autograd needs it); the no-grad path takes the kernel's
    assert_close(pkg2["render"], pkg["render"], rtol=1e-5, what="grad path vs no-grad path")
    pkg2["render"].sum().backward()
    assert kw2["opacity"].grad is not None and float(kw2["opacity"].grad.abs().sum()) > 0
    assert float(kw2["opacity"].grad[~pkg["selection_mask"]].abs().sum()) == 0.0

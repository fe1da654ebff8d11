"""Key-frame densification (``SceneModel.add_new_gaussians``, h3dgsv3.py:766-940): ``artdeco_b200.densify`` against the
PyTorch oracle (oracle/densify_ref.py), and the oracle against the golden fixture made by running the reference's own code
(tests/golden/make_densify_golden.py).

Tolerances.  The maps ``init_proba`` and ``penalty`` are compared within 1e-5 absolute against the fp32 oracle on the device
with TF32 off (the oracle's conv2d and exposure matmul).  Sample / valid decisions must be identical except at pixels within
1e-5 of their threshold (|u - (p - q) r| or |depth - qmin|), which are excluded and must be at most 1e-4 of all pixels.  Rows
are compared on the pixels both sides emit: same order and count, float columns within 1e-5 x max(|value|, 1) with
non-finite values at the same places, ids exact.  Integer results of the whole method (class ids, voxel counts, rows kept)
must match exactly; the voxel step of the oracle is evaluated on the implementation's own new points (an ulp of xyz could
move a point across a voxel boundary), after checking those points agree with the oracle's to the row tolerance."""
import math
import os

import pytest
import torch

from oracle import densify_ref as ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "densify_small.pt")
ROW_KEYS = ("xyz", "f_dc", "scaling", "opacity", "d_max")
MARGIN = 1e-5


def golden():
    return torch.load(GOLDEN, weights_only=False)["cases"]


def assert_rows_close(got, want, what):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    fin_g, fin_w = torch.isfinite(got), torch.isfinite(want)
    assert torch.equal(fin_g, fin_w), f"{what}: non-finite values at different positions"
    assert torch.equal(got[~fin_g].nan_to_num(0.0), want[~fin_w].nan_to_num(0.0)), f"{what}: different non-finite values"
    if fin_g.any():
        err = ((got - want).abs() / want.abs().clamp_min(1.0))[fin_g]
        assert float(err.max()) <= 1e-5, f"{what}: max normalised error {float(err.max()):.3e}"


def frame_of(c, dev="cpu"):
    return dict(image=c["image"].to(dev), point_map=c["point_map"].to(dev), conf=c["conf"].to(dev), R=c["R"].to(dev),
                t=c["t"].to(dev), approx_centre=c["approx_centre"].to(dev), exposure=c["exposure"].to(dev), is_test=False)


# ------------------------------------------------------------------ CPU ------------------------------------------------------

def test_oracle_reproduces_the_reference_golden():
    """The golden was computed by the reference's own code on one CPU; PyTorch's CPU kernels (BLAS, conv, vectorised
    reductions) reorder float sums differently on other instruction sets, so float columns agree to the row tolerance, not
    bit for bit.  Everything discrete must be exact: the premises below show every decision of the golden sits far further
    from its threshold than such reordering can move a value, and the voxel step runs on the golden's own new points, so the
    class ids and voxel counts are computed from identical inputs."""
    for c in golden():
        params = {k: v.clone() for k, v in c["params"].items()}
        a = c["args"]
        fr = frame_of(c)
        offset = [0]

        def voxel(new_xyz, xyz, cls_id, vs, lod):
            theirs = c["ext"]["xyz"][offset[0]: offset[0] + new_xyz.shape[0]]
            offset[0] += new_xyz.shape[0]
            assert_rows_close(new_xyz, theirs, f"warm={c['warm']} lod {lod} new xyz")
            return ref._cpu_voxel(theirs, xyz, cls_id, vs)
        out = ref.add_new_gaussians(params, fr, lambda cls: c["raw_render"], keyframe_id=0,
                                    cam_centres=c["approx_centre"][None], width=c["W"], height=c["H"], f=c["f"],
                                    init_proba_scaler=a["init_proba_scaler"], gs_add_ratio=a["gs_add_ratio"],
                                    voxel_size=a["voxel_size"], visible_threshold=0.0, sh_degree=a["sh_degree"],
                                    local_feat_dim=a["local_feat_dim"], global_feat_dim=a["global_feat_dim"],
                                    uniforms=c["uniforms"], update_voxel=voxel)
        # premises: sample, valid and prune decisions are at least 1e-5 from their thresholds
        qmin = ref.depth_threshold(fr["point_map"])
        for i, lod in enumerate(ref.LODS):
            r = out["rows"][i]
            assert float((c["uniforms"][i] - (r["init_proba"] - r["penalty"]) * a["gs_add_ratio"]).abs().min()) > MARGIN
            depth = ref.sample(fr["point_map"][:, 2:], ref.uvs(c["W"], c["H"], lod)[None], c["W"] // lod, c["H"] // lod)[0, 0]
            assert not r["sampled"].any() or float((depth - qmin)[r["sampled"]].abs().min()) > MARGIN
        if c["warm"]:
            p = c["params"]
            sig = torch.sigmoid(p["opacity"])[:, 0]
            screen = c["f"] * torch.exp(p["scaling"]).max(-1)[0] / torch.linalg.vector_norm(p["xyz"] - fr["approx_centre"], dim=-1)
            assert float((sig - 0.05).abs().min()) > MARGIN and float((screen / (0.5 * c["W"]) - 1).abs().min()) > MARGIN
        assert offset[0] == c["ext"]["xyz"].shape[0]
        assert out["renders"] == c["n_renders"]
        assert torch.equal(out["valid_gs_mask"], c["valid_gs_mask"])
        for k, v in c["ext"].items():
            if v.dtype == torch.int64 or k == "rotation":
                assert torch.equal(out["ext"][k], v), k
            else:
                assert_rows_close(out["ext"][k].flatten(1), v.flatten(1), f"golden warm={c['warm']} {k}")
        for k, shape in c["fill_shapes"].items():
            assert tuple(out["ext"][k].shape) == shape and not out["ext"][k].any()
        if c["warm"]:
            assert torch.equal(params["cls_id"][: c["valid_gs_mask"].sum()], c["cls_after"][c["valid_gs_mask"]])


def test_golden_covers_the_reproduced_quirks():
    warm, cold = golden()
    assert warm["warm"] and not cold["warm"]
    # inverse_sigmoid(0.2 conf) for conf >= 5 is NaN, and the rows carry it
    assert any(torch.isnan(c["ext"]["opacity"]).any() for c in (warm, cold))
    # new class ids restart at 0 in every LoD of a cold start
    assert cold["n_renders"] == 0 and int((cold["ext"]["cls_id"] == 0).sum()) >= 2
    assert warm["n_renders"] == 4 and not warm["valid_gs_mask"].all() and warm["valid_gs_mask"].any()


def test_disc_has_37_taps():
    k = ref.disc_kernel()
    assert int((k > 0).sum()) == 37 and torch.equal(k, golden()[0]["disc"])
    assert float(k.max()) == float(torch.tensor(1.0) / torch.tensor(37.0))


def test_cold_start_has_no_render_no_penalty_and_an_empty_prune_mask():
    c = golden()[1]
    fr = frame_of(c)
    params = {k: v.clone() for k, v in c["params"].items()}
    calls = []
    a = c["args"]
    out = ref.add_new_gaussians(params, fr, lambda cls: calls.append(cls), keyframe_id=0, cam_centres=c["approx_centre"][None],
                                width=c["W"], height=c["H"], f=c["f"], init_proba_scaler=a["init_proba_scaler"],
                                gs_add_ratio=a["gs_add_ratio"], voxel_size=a["voxel_size"], visible_threshold=0.0,
                                local_feat_dim=a["local_feat_dim"], global_feat_dim=a["global_feat_dim"], uniforms=c["uniforms"])
    assert not calls and out["renders"] == 0
    assert out["valid_gs_mask"].numel() == 0 and out["valid_gs_mask"].dtype == torch.bool
    assert all(float(r["penalty"].abs().max()) == 0.0 for r in out["rows"])


def test_nan_quantile_gives_the_python_min_default():
    pm = torch.rand(1, 3, 8, 9) + 1.0
    assert ref.depth_threshold(pm) == 1e-2
    pm[0, 2, 3, 4] = float("nan")
    assert math.isnan(torch.quantile(pm[:, 2], 0.02).item())
    assert ref.depth_threshold(pm) == 1e-2                   # min(1e-2, nan) keeps its first argument
    pm = torch.rand(1, 3, 8, 9) * 1e-3
    assert ref.depth_threshold(pm) == torch.quantile(pm[:, 2], 0.02).item() < 1e-2


def test_densify_raises_without_cuda():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from artdeco_b200 import _lib, densify
    with pytest.raises(_lib.ArtdecoB200Error):
        densify.depth_quantile(torch.rand(1, 3, 8, 8))


# ------------------------------------------------------------------ GPU ------------------------------------------------------

@pytest.fixture
def fp32(cuda):
    m, c = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield cuda
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = m, c


def make_frame(H, W, Hs, Ws, seed, dev):
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing="ij")
    image = (0.5 + 0.3 * torch.sin(17 * xx + 5 * yy)[None] * torch.rand(3, 1, 1, generator=g)
             + 0.1 * torch.rand(3, H, W, generator=g)).clamp(0, 1)
    depth = 1.0 + 6.0 * torch.rand(Hs, Ws, generator=g)
    near = torch.rand(Hs, Ws, generator=g) < 0.01                  # ~1% invalid points, below the 2% quantile
    depth[near] = 0.003 * torch.rand(int(near.sum()), generator=g)
    pm = torch.stack([torch.randn(Hs, Ws, generator=g), torch.randn(Hs, Ws, generator=g), depth])[None]
    conf = 4.0 * torch.rand(1, 1, Hs, Ws, generator=g) - 0.5
    conf[0, 0, :2, :3] = 5.5
    ang = 0.15
    R = torch.tensor([[math.cos(ang), 0.0, math.sin(ang)], [0.0, 1.0, 0.0], [-math.sin(ang), 0.0, math.cos(ang)]])
    t = torch.tensor([0.2, -0.1, 0.05])
    expo = torch.eye(3, 4) * 1.05
    expo[:, 3] = torch.tensor([0.01, -0.02, 0.03])
    expo[0, 1] = 0.02
    raw = (0.45 + 0.1 * torch.sin(9 * xx)[None] + 0.005 * torch.rand(3, H, W, generator=g))
    fr = dict(image=image, point_map=pm, conf=conf, R=R, t=t, approx_centre=-R.T @ t, exposure=expo, is_test=False)
    return {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in fr.items()}, raw.to(dev)


def compare_lod(ours, want, u, qmin, fr, lod, what):
    """Maps within 1e-5; decisions equal outside the margin; rows equal on the common pixels.  Returns (excluded, total)."""
    for k in ("init_proba", "penalty"):
        err = float((ours[k] - want[k]).abs().max())
        assert err <= 1e-5, f"{what}: {k} max error {err:.3e}"
    s_o, v_o = (ours["flags"] & 1).bool(), (ours["flags"] & 2).bool()
    H, W = fr["image"].shape[-2:]
    depth = ref.sample(fr["point_map"][:, 2:], ref.uvs(W, H, lod, u.device)[None], W // lod, H // lod)[0, 0]
    excluded = ((u - (want["init_proba"] - want["penalty"]) * RATIO).abs() <= MARGIN) | \
        ((s_o | want["sampled"]) & ((depth - qmin).abs() <= MARGIN))
    assert not ((s_o != want["sampled"]) & ~excluded).any(), f"{what}: sample decisions differ outside the margin"
    both = s_o & want["sampled"]
    assert not ((v_o != want["valid"]) & both & ~excluded).any(), f"{what}: valid flags differ outside the margin"
    keep_o, keep_w = s_o & v_o, want["sampled"] & want["valid"]
    if not excluded.any():
        assert ours["n"] == want["n"], f"{what}: {ours['n']} rows, oracle {want['n']}"
    common = (keep_o & keep_w).reshape(-1)
    io = (torch.cumsum(keep_o.reshape(-1).long(), 0) - 1)[common]
    iw = (torch.cumsum(keep_w.reshape(-1).long(), 0) - 1)[common]
    for k in ROW_KEYS:
        assert_rows_close(ours[k].flatten(1)[io], want[k].flatten(1)[iw], f"{what} {k}")
    return int(excluded.sum()), int(excluded.numel())


RATIO, SCALER = 0.7, 1.5


@pytest.mark.gpu
@pytest.mark.parametrize("H,W,Hs,Ws", [(972, 1296, 384, 512), (45, 61, 23, 31), (50, 70, 37, 29), (16, 17, 9, 11),
                                       (131, 99, 64, 48)])
def test_maps_decisions_and_rows_match_the_oracle(fp32, H, W, Hs, Ws):
    from artdeco_b200 import densify
    dev = fp32
    fr, raw = make_frame(H, W, Hs, Ws, seed=H * 7 + W, dev=dev)
    q = densify.depth_quantile(fr["point_map"])
    qmin = ref.depth_threshold(fr["point_map"])
    assert float(q[1]) == float(torch.tensor(qmin, dtype=torch.float32))
    f = 0.8 * W
    excluded = total = 0
    for lod in ref.LODS:
        for render in (None, raw):
            g = torch.Generator(device=dev).manual_seed(lod)
            u = torch.rand(H // lod, W // lod, device=dev, generator=g)
            # the render as render_lod returns it: a strided view of the [1,H,W,4] colour buffer
            rv = None
            if render is not None:
                buf = torch.zeros(1, H, W, 4, device=dev)
                buf[0, ..., :3] = render.permute(1, 2, 0)
                rv = buf[..., 0:3].permute(0, 3, 1, 2)[0]
            ours = densify.sample_lod(fr["image"], rv, fr["point_map"], fr["conf"], fr["R"], fr["t"], fr["approx_centre"],
                                      fr["exposure"], lod=lod, f=f, init_proba_scaler=SCALER, gs_add_ratio=RATIO, uniforms=u,
                                      qmin=q)
            want = ref.sample_lod(fr["image"], render, fr["point_map"], fr["conf"], fr["R"], fr["t"], fr["approx_centre"],
                                  fr["exposure"], lod=lod, f=f, init_proba_scaler=SCALER, gs_add_ratio=RATIO, uniforms=u,
                                  qmin=qmin)
            e, n = compare_lod(ours, want, u, qmin, fr, lod, f"{H}x{W} lod {lod} render {render is not None}")
            excluded += e
            total += n
            assert want["n"] > 0 or H * W < 2000
    assert excluded <= 1e-4 * total, (excluded, total)


@pytest.mark.gpu
def test_depth_quantile_is_bit_equal_to_torch(cuda):
    from artdeco_b200 import densify
    g = torch.Generator(device=cuda).manual_seed(3)
    for Hs, Ws in ((384, 512), (23, 31), (1, 1), (1, 2), (7, 1)):
        pm = torch.randn(1, 3, Hs, Ws, device=cuda, generator=g) * 3
        pm[0, 2, 0, 0] = -0.0
        if Hs * Ws > 10:
            pm[0, 2, 1:3, :] = 1.25                      # ties
        for nan in (False, True):
            p = pm.clone()
            if nan:
                p[0, 2, -1, -1] = float("nan")
            out = densify.depth_quantile(p)
            want = torch.quantile(p[:, 2], 0.02)
            assert torch.equal(out[0:1].view(torch.int32), want.reshape(1).view(torch.int32)) or \
                (torch.isnan(out[0]) and torch.isnan(want)), (Hs, Ws, nan, float(out[0]), float(want))
            assert float(out[1]) == float(torch.tensor(min(1e-2, want.item()), dtype=torch.float32))


@pytest.mark.gpu
def test_prune_mask_matches_the_oracle(cuda):
    from artdeco_b200 import densify
    g = torch.Generator(device=cuda).manual_seed(5)
    N, W, f = 200_000, 1296, 1000.0
    params = dict(xyz=torch.randn(N, 3, device=cuda, generator=g) * 5, opacity=torch.randn(N, 1, device=cuda, generator=g) * 4,
                  scaling=torch.randn(N, 3, device=cuda, generator=g) - 2)
    centre = torch.tensor([0.3, -0.2, 0.1], device=cuda)
    got = densify.prune_mask(params["xyz"], params["opacity"], params["scaling"], centre, f, W)
    want = ref.prune_mask(params, centre, f, W)
    sig = torch.sigmoid(params["opacity"])[:, 0]
    screen = f * torch.exp(params["scaling"]).max(-1)[0] / torch.linalg.vector_norm(params["xyz"] - centre, dim=-1)
    near = ((sig - 0.05).abs() <= 1e-6) | ((screen / (0.5 * W) - 1).abs() <= MARGIN)
    assert not ((got != want) & ~near).any()
    assert int(near.sum()) <= 1e-4 * N
    assert 0 < int(want.sum()) < N


@pytest.mark.gpu
def test_golden_through_the_device_sampler(cuda):
    from artdeco_b200 import densify
    from artdeco_b200.voxel import update_voxel
    for c in golden():
        fr = frame_of(c, cuda)
        a = c["args"]
        q = densify.depth_quantile(fr["point_map"])
        xyz0 = c["params"]["xyz"].to(cuda)
        cls = c["params"]["cls_id"].to(cuda)
        rows, cls_new, nvox = {k: [] for k in ROW_KEYS}, [], 0
        for i, lod in enumerate(ref.LODS):
            r = densify.sample_lod(fr["image"], c["raw_render"].to(cuda) if c["warm"] else None, fr["point_map"], fr["conf"],
                                   fr["R"], fr["t"], fr["approx_centre"], fr["exposure"], lod=lod, f=c["f"],
                                   init_proba_scaler=a["init_proba_scaler"], gs_add_ratio=a["gs_add_ratio"],
                                   uniforms=c["uniforms"][i].to(cuda), qmin=q)
            for k in ROW_KEYS:
                rows[k].append(r[k])
            if c["warm"]:
                cls, nc, nv = update_voxel(r["xyz"], xyz0, cls, a["voxel_size"])
            else:
                nc, nv = update_voxel(r["xyz"], xyz0, cls, a["voxel_size"])
            cls_new.append(nc)
            nvox += nv
        for k in ROW_KEYS:
            assert_rows_close(torch.cat(rows[k]), c["ext"][k], f"golden warm={c['warm']} {k}")
        assert torch.equal(torch.cat(cls_new).cpu(), c["ext"]["cls_id"])
        assert nvox == c["fill_shapes"]["global_feat"][0]
        if c["warm"]:
            assert torch.equal(cls.cpu(), c["cls_after"])
            m = densify.prune_mask(xyz0, c["params"]["opacity"].to(cuda), c["params"]["scaling"].to(cuda), fr["approx_centre"],
                                   c["f"], c["W"])
            assert torch.equal(m.cpu(), c["valid_gs_mask"])


# ---- end to end ----

def make_scene(N, dev, seed, Fl=20, Fg=12, n_cls=6):
    from artdeco_b200 import synthetic
    sc = synthetic.raster_scene(N, seed=seed, z_range=(2.0, 8.0), extent=(2.5, 2.0))
    g = torch.Generator().manual_seed(seed + 1)
    P = dict(id=torch.zeros(N, 1, dtype=torch.long), cls_id=torch.randint(0, n_cls, (N, 1), generator=g),
             d_max=sc["d_max"], xyz=sc["means"], f_dc=sc["sh"][:, :1].clone(), f_rest=sc["sh"][:, 1:].clone(),
             scaling=torch.log(sc["scales"]), rotation=sc["quats"], opacity=torch.logit(sc["opacities"][:, None]),
             local_feat=torch.randn(N, Fl, generator=g) * 0.3, global_feat=torch.randn(n_cls, Fg, generator=g) * 0.3)
    P["opacity"][: N // 50] = -5.0                                           # pruned: sigmoid < 0.05
    return {k: v.to(dev) for k, v in P.items()}


def mlp(dev, Fl=20, Fg=12, seed=9):
    g = torch.Generator().manual_seed(seed)
    d = Fl + Fg
    return {k: v.to(dev) for k, v in dict(W1=torch.randn(d, d, generator=g) / d ** 0.5, b1=torch.zeros(d),
                                         W2=torch.randn(7, d, generator=g) / d ** 0.5, b2=torch.zeros(7)).items()}


def run_both(dev, P0, fr, *, H, W, cov, voxel_size, monkeypatch, is_test=False):
    from artdeco_b200 import densify
    from artdeco_b200.optimizers import SparseGaussianAdam
    from artdeco_b200.scene import render_lod
    f = 0.9 * W
    tanx, tany = W / (2 * f), H / (2 * f)
    kw = dict(init_proba_scaler=SCALER, gs_add_ratio=RATIO, voxel_size=voxel_size, visible_threshold=0.3,
              local_feat_dim=20, global_feat_dim=12)
    cams = torch.stack([fr["approx_centre"], fr["approx_centre"] + torch.tensor([0.5, 0.0, 0.0], device=dev)])
    fr = dict(fr, is_test=is_test)
    lrs = dict(xyz=1e-3, f_dc=1e-3, f_rest=1e-3, scaling=1e-3, rotation=1e-3, opacity=1e-3, local_feat=1e-3, global_feat=1e-3)
    params = {k: {"val": v.clone(), **({"lr": lrs[k]} if k in lrs else {})} for k, v in P0.items()}
    opt = SparseGaussianAdam(params, (0.5, 0.99), device=dev)
    seen = []
    real = densify.update_voxel

    def spy(new_xyz, xyz, cls_id, voxel_size):
        seen.append(new_xyz.clone())
        return real(new_xyz, xyz, cls_id, voxel_size)
    monkeypatch.setattr(densify, "update_voxel", spy)
    torch.manual_seed(123)
    st = densify.add_new_gaussians(opt, fr, keyframe_id=3, cam_centres=cams, width=W, height=H, f=f, tanfovx=tanx,
                                   tanfovy=tany, cov_mlp=cov, **kw)
    ours = {k: v["val"].detach() for k, v in opt.params.items()}

    refp = {k: v.clone() for k, v in P0.items()}
    V = torch.eye(4, device=dev)
    V[:3, :3], V[:3, 3] = fr["R"], fr["t"]

    def render(cls):
        extra = {} if cov is None else dict(cov_mlp=cov, local_feat=refp["local_feat"], global_feat=refp["global_feat"], cls_id=cls)
        return render_lod(W, H, V, xyz=refp["xyz"], opacity=torch.sigmoid(refp["opacity"]), f_dc=refp["f_dc"],
                          f_rest=refp["f_rest"], scaling=torch.exp(refp["scaling"]), rotation=refp["rotation"],
                          d_max=refp["d_max"], tanfovx=tanx, tanfovy=tany, **extra)["render"].contiguous()

    def voxel(new_xyz, xyz, cls_id, vs, lod):
        i = ref.LODS.index(lod)
        mine = seen[i]
        assert_rows_close(mine, new_xyz, f"new xyz lod {lod}")
        return ref._cpu_voxel(mine, xyz, cls_id, vs)
    torch.manual_seed(123)
    out = ref.add_new_gaussians(refp, fr, render, keyframe_id=3, cam_centres=cams, width=W, height=H, f=f, update_voxel=voxel,
                                **kw)
    return st, ours, out, refp


def assert_params_equal(ours, refp):
    assert set(refp) <= set(ours)
    for k, v in refp.items():
        o = ours[k]
        assert o.shape == v.shape, (k, o.shape, v.shape)
        if v.dtype in (torch.int64, torch.int32):
            assert torch.equal(o.cpu(), v.cpu()), k
        else:
            assert_rows_close(o.flatten(1), v.flatten(1), f"param {k}")


@pytest.mark.gpu
def test_end_to_end_with_mlp_cov_and_changing_classes(fp32, monkeypatch):
    dev = fp32
    H, W = 243, 324
    fr, _ = make_frame(H, W, 96, 128, seed=21, dev=dev)
    P0 = make_scene(20000, dev, seed=4)
    st, ours, out, refp = run_both(dev, P0, fr, H=H, W=W, cov=mlp(dev), voxel_size=0.3, monkeypatch=monkeypatch)
    assert st["rows"] == [r["n"] for r in out["rows"]]
    assert out["renders"] == 4 and 1 < st["renders"] <= 4        # the classes change between LoDs: renders are redone
    assert sum(st["new_voxels"]) == out["ext"]["global_feat"].shape[0]
    assert_params_equal(ours, refp)


@pytest.mark.gpu
def test_end_to_end_cold_start(fp32, monkeypatch):
    dev = fp32
    H, W = 120, 160
    fr, _ = make_frame(H, W, 60, 80, seed=22, dev=dev)
    P0 = {k: v[:0] for k, v in make_scene(10, dev, seed=5).items()}
    st, ours, out, refp = run_both(dev, P0, fr, H=H, W=W, cov=mlp(dev), voxel_size=0.2, monkeypatch=monkeypatch)
    assert st["renders"] == 0 and out["renders"] == 0
    assert min(st["rows"]) > 0
    assert_params_equal(ours, refp)
    # class ids restart at 0 in every LoD
    assert int((out["ext"]["cls_id"] == 0).sum()) >= 4


@pytest.mark.gpu
def test_test_frame_leaves_everything_untouched(fp32, monkeypatch):
    dev = fp32
    fr, _ = make_frame(64, 80, 32, 40, seed=23, dev=dev)
    P0 = make_scene(500, dev, seed=6)
    st, ours, out, refp = run_both(dev, P0, fr, H=64, W=80, cov=mlp(dev), voxel_size=0.3, monkeypatch=monkeypatch, is_test=True)
    assert st == dict(renders=0, rows=[], new_voxels=[])
    for k, v in P0.items():
        assert torch.equal(ours[k], v), k


@pytest.mark.gpu
def test_render_count(fp32, monkeypatch):
    dev = fp32
    H, W = 96, 128
    fr, _ = make_frame(H, W, 48, 64, seed=24, dev=dev)
    P0 = make_scene(3000, dev, seed=7)
    P0["cls_id"].zero_()
    # one huge voxel: every point keeps class 0, so one render serves all four LoDs
    st, ours, out, refp = run_both(dev, P0, fr, H=H, W=W, cov=mlp(dev), voxel_size=1e3, monkeypatch=monkeypatch)
    assert st["renders"] == 1 and out["renders"] == 4
    assert_params_equal(ours, refp)
    # without mlp_cov the class ids are never read by the render
    st, ours, out, refp = run_both(dev, make_scene(3000, dev, seed=8), fr, H=H, W=W, cov=None, voxel_size=0.3,
                                   monkeypatch=monkeypatch)
    assert st["renders"] == 1
    assert_params_equal(ours, refp)

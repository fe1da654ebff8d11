"""Held-out key-frame evaluation (artdeco_b200.evaluate, artdeco_b200.lpips, csrc/evaluate.cu) against the reference's own
statements (tests/golden/evaluate_small.pt, made by make_evaluate_golden.py) and against oracle/evaluate_ref.py."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import evaluate_ref as ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "evaluate_small.pt")
TOL = 1e-5          # PSNR / SSIM, relative
TOL_LPIPS = 1e-4    # LPIPS value (relative) and tap features (of scale): bf16x3 convolutions


def golden():
    return torch.load(GOLDEN, weights_only=False)


def oracle_evaluate(sc, lpips, dev="cpu"):
    K = len(sc["is_test"])
    ex = [sc["exposure"][i].to(dev).clone() for i in range(K)]
    renders = [(sc["colors"][i].to(dev), sc["alphas"][i].to(dev)) for i in range(K)]
    gts = [sc["gt"][i].to(dev) for i in range(K)]
    vis = [sc["visibility"][i].to(dev) for i in range(K)]
    m = ref.evaluate(ex, sc["is_test"].tolist(), renders, gts, vis, lpips=lpips, with_LPIPS=sc["with_LPIPS"],
                     all=sc["all"])
    return m, torch.stack(ex)


def rel(a, b):
    return abs(a - b) / max(abs(b), 1e-30)


def assert_metrics(got, want, what, tol_lpips=TOL_LPIPS):
    assert list(got) == list(want), (what, list(got), list(want))
    for k, v in want.items():
        if k in ("Render", "GS", "n_test_frames"):
            assert got[k] == v, (what, k, got[k], v)
        else:
            tol = tol_lpips if k == "LPIPS" else TOL
            assert rel(got[k], v) <= tol, (what, k, got[k], v, rel(got[k], v))


# ------------------------------------------------------------------ CPU ------------------------------------------------------

def test_oracle_reproduces_the_reference_golden():
    g = golden()
    lp = ref.make_lpips(g["lpips_seed"])
    for name, sc in g["scenes"].items():
        if sc["raises"]:
            with pytest.raises(IndexError):
                oracle_evaluate(sc, lp)
            continue
        m, ex = oracle_evaluate(sc, lp)
        assert torch.equal(ex, sc["exposure_out"]), name
        assert_metrics(m, sc["metrics"], name, tol_lpips=TOL)


def test_golden_covers_the_edge_cases():
    sc = golden()["scenes"]
    t = sc["mixed"]["is_test"].tolist()
    assert t[0] and t[-1] and any(t[i] and t[i + 1] for i in range(len(t) - 1))
    assert len(sc["pair_last"]["is_test"]) == 2 and len(sc["single_test"]["is_test"]) == 1
    assert sc["single_train"]["metrics"] == {"n_test_frames": 0} and sc["single_test"]["raises"] == "IndexError"
    m = sc["mixed"]
    K = len(t)
    # a test frame after a test frame averages the updated one, and the sums are not exactly representable
    e_in, e_out = m["exposure"], m["exposure_out"]
    assert torch.equal(e_out[3], (e_out[2] + e_in[4]) / 2) and not torch.equal(e_out[3], (e_in[2] + e_in[4]) / 2)
    assert torch.equal(e_out[0], (e_in[1] + e_in[1]) / 2) and torch.equal(e_out[K - 1], (e_in[K - 2] + e_in[K - 2]) / 2)
    s = e_in[1].double() + e_in[3].double()
    assert (s.float().double() != s).any()


def test_trunk_matches_torchvision_vgg16():
    tv = pytest.importorskip("torchvision")
    feats = tv.models.vgg16(weights=None).features[:30]
    a, b = ref.LPIPSRef(feats).eval(), ref.LPIPSRef().eval()
    sd = ref.random_state_dict(3)
    a.load_state_dict(sd)
    b.load_state_dict(sd)
    g = torch.Generator().manual_seed(0)
    x0, x1 = torch.rand(1, 3, 40, 36, generator=g), torch.rand(1, 3, 40, 36, generator=g)
    with torch.no_grad():
        ta, tb = a.taps(x0, x1), b.taps(x0, x1)
        for k in range(5):
            assert torch.equal(ta[0][k], tb[0][k]) and torch.equal(ta[1][k], tb[1][k]), k
        assert torch.equal(a(x0, x1), b(x0, x1))


def test_head_against_a_direct_per_pixel_computation():
    g = torch.Generator().manual_seed(1)
    f0, f1 = torch.randn(2, 24, 5, 7, generator=g).double(), torch.randn(2, 24, 5, 7, generator=g).double()
    f0[0, :, 1, 1] = 0.0                     # a zero feature: the 1e-10 keeps it finite
    w = torch.rand(1, 24, 1, 1, generator=g).double()
    got = ref.head(f0, f1, w)
    want = np.zeros(2)
    a, b, wn = f0.numpy(), f1.numpy(), w.numpy().reshape(-1)
    for n in range(2):
        for y in range(5):
            for x in range(7):
                u, v = a[n, :, y, x], b[n, :, y, x]
                d = u / (np.sqrt((u * u).sum()) + 1e-10) - v / (np.sqrt((v * v).sum()) + 1e-10)
                want[n] += (wn * d * d).sum()
    want /= 35
    np.testing.assert_allclose(got.reshape(-1).numpy(), want, rtol=1e-12)


def test_entry_points_refuse_bad_arguments_before_touching_the_device():
    from artdeco_b200 import _lib
    import artdeco_b200  # noqa: F401  (registers every signature)
    L = _lib.lib()

    def refused(rc, needle, status=1):
        msg = L.adb_last_error()
        return rc == status and msg is not None and needle in msg.decode()

    nb = ctypes.c_size_t(0)
    assert refused(L.adb_eval_workspace_bytes(0, 10, 10, 5, ctypes.byref(nb)), "adb_eval_workspace_bytes")
    assert refused(L.adb_eval_workspace_bytes(2, 10, -1, 5, ctypes.byref(nb)), "adb_eval_workspace_bytes")
    assert refused(L.adb_eval_workspace_bytes(2, 10, 10, -1, ctypes.byref(nb)), "adb_eval_workspace_bytes")
    assert refused(L.adb_eval_workspace_bytes(2, 10, 10, 5, None), "null bytes")
    assert L.adb_eval_workspace_bytes(2, 10, 10, 5, ctypes.byref(nb)) == 0 and nb.value > 0
    need = nb.value
    assert refused(L.adb_lpips_workspace_bytes(1, 15, 64, ctypes.byref(nb)), ">= 16")
    assert refused(L.adb_lpips_workspace_bytes(0, 64, 64, ctypes.byref(nb)), "adb_lpips_workspace_bytes")
    assert L.adb_lpips_workspace_bytes(1, 64, 64, ctypes.byref(nb)) == 0 and nb.value > 0
    fake = 1 << 20                                    # never dereferenced: every refusal happens before a launch
    assert refused(L.adb_eval_harmonize(0, fake, fake, fake, None), "K must be")
    assert refused(L.adb_eval_harmonize(3, None, fake, fake, None), "null pointer")
    assert refused(L.adb_eval_count_visible(2, 10, 10, 5, 2, fake, fake, need, None), "view index")
    assert refused(L.adb_eval_count_visible(2, 10, 10, 5, 0, fake, fake, need - 1, None), "workspace too small", 3)
    p = [fake] * 5
    assert refused(L.adb_eval_image_metrics(2, 10, 10, 5, None, *p[1:], fake, fake, fake, need, None), "null pointer")
    assert refused(L.adb_eval_image_metrics(2, 10, 10, 5, fake + 4, *p[1:], fake, fake, fake, need, None), "aligned")
    assert refused(L.adb_eval_image_metrics(2, 10, 10, 5, *p, fake, fake, fake, need - 1, None), "workspace too small", 3)
    assert refused(L.adb_eval_reduce(2, 10, 10, 5, 1, None, need, fake, None), "null pointer")
    assert refused(L.adb_eval_reduce(2, 10, 10, 5, 1, fake, need - 1, fake, None), "workspace too small", 3)
    P12 = ctypes.c_void_p * 12
    arr = P12(*([fake] * 12))
    lin = (ctypes.c_void_p * 5)(*([fake] * 5))
    args = [fake] * 6 + [arr, arr, arr, lin, None, fake, 1 << 40, fake, need, None]
    assert refused(L.adb_lpips_vgg_forward(2, 12, 64, 5, 0, 1, *args), ">= 16")
    assert refused(L.adb_lpips_vgg_forward(2, 64, 64, 5, 1, 2, *args), "frame range")
    bad = P12(*([fake] * 11 + [None]))
    assert refused(L.adb_lpips_vgg_forward(2, 64, 64, 5, 0, 1, *([fake] * 6), arr, bad, arr, lin, None, fake, 1 << 40,
                                           fake, need, None), "null conv weight")
    assert refused(L.adb_lpips_vgg_forward(2, 64, 64, 5, 0, 1, *([fake] * 6), arr, arr, arr, lin, None, fake, 16, fake,
                                           need, None), "workspace too small", 3)


def test_python_wrappers_refuse_without_a_device():
    if torch.cuda.is_available():
        pytest.skip("checks the CPU refusal")
    from artdeco_b200 import _lib, evaluate
    with pytest.raises(_lib.ArtdecoB200Error):
        evaluate.harmonize_test_exposure(torch.zeros(2, 3, 4), torch.zeros(2, dtype=torch.bool))
    with pytest.raises(_lib.ArtdecoB200Error):
        evaluate.metrics_from_renders(torch.zeros(1, 16, 16, 4), torch.zeros(1, 16, 16), torch.zeros(1, 3, 16, 16),
                                      torch.zeros(1, 3, 4), torch.zeros(1, dtype=torch.int32))


# ------------------------------------------------------------------ GPU ------------------------------------------------------

@pytest.fixture
def fp32(cuda):
    m, c = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield cuda
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = m, c


def _ours_on_scene(sc, lp, dev):
    from artdeco_b200 import evaluate
    K = len(sc["is_test"])
    E = sc["exposure"].to(dev).clone()
    renders = {}
    for i in range(K):
        renders[float(i)] = dict(colors=sc["colors"][i].to(dev), alphas=sc["alphas"][i].to(dev),
                                 visibility_filter=sc["visibility"][i].to(dev))
    vms = [torch.full((4, 4), float(i)) for i in range(K)]
    m = evaluate.evaluate(E, sc["is_test"].tolist(), vms, [sc["gt"][i] for i in range(K)], width=sc["gt"].shape[3],
                          height=sc["gt"].shape[2], render=lambda vm: renders[float(vm[0, 0])], lpips=lp,
                          with_LPIPS=sc["with_LPIPS"], all=sc["all"])
    return m, E


@pytest.mark.gpu
def test_kernels_reproduce_the_reference_golden(fp32):
    from artdeco_b200.lpips import LPIPSVGG
    dev = fp32
    g = golden()
    lp = LPIPSVGG(ref.random_state_dict(g["lpips_seed"]), device=dev)
    for name, sc in g["scenes"].items():
        if sc["raises"]:
            with pytest.raises(IndexError):
                _ours_on_scene(sc, lp, dev)
            continue
        m, E = _ours_on_scene(sc, lp, dev)
        assert torch.equal(E.cpu(), sc["exposure_out"]), name          # harmonised exposures bitwise
        assert_metrics(m, sc["metrics"], name)


@pytest.mark.gpu
def test_harmonize_bitwise_against_the_oracle(fp32):
    from artdeco_b200 import evaluate
    dev = fp32
    g = torch.Generator().manual_seed(5)
    for K in (1, 2, 3, 7, 40):
        for trial in range(4):
            is_test = (torch.rand(K, generator=g) < 0.5).tolist()
            if K == 1:
                is_test = [False]
            E = torch.randn(K, 3, 4, generator=g)
            want = ref.harmonize_test_exposure([E[i].clone() for i in range(K)], is_test)
            got = E.to(dev).contiguous()
            n_bad = evaluate.harmonize_test_exposure(got, torch.tensor(is_test, device=dev))
            assert int(n_bad) == 0
            assert torch.equal(got.cpu(), torch.stack(want)), (K, is_test)
    got = torch.randn(1, 3, 4, device=dev)
    before = got.clone()
    assert int(evaluate.harmonize_test_exposure(got, torch.ones(1, dtype=torch.bool, device=dev))) == 1
    assert torch.equal(got, before)


def _random_views(T, h, w, seed, dev):
    g = torch.Generator().manual_seed(seed)
    rgb = torch.rand(T, h, w, 3, generator=g) * 1.2 - 0.1
    colors = torch.cat([rgb, torch.rand(T, h, w, 1, generator=g) + 0.5], -1).contiguous()
    alphas = torch.rand(T, h, w, generator=g)
    # ground truth near the render, so PSNR and LPIPS are in their usual range
    gt = (rgb.permute(0, 3, 1, 2) + 0.05 * torch.randn(T, 3, h, w, generator=g)).clamp(0, 1).contiguous()
    E = (torch.eye(3, 4) + 0.03 * torch.randn(T, 3, 4, generator=g)).contiguous()
    return colors.to(dev), alphas.to(dev), gt.to(dev), E.to(dev)


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,T", [(972, 1296, 2), (486, 648, 3), (37, 53, 2), (16, 16, 2), (31, 45, 3), (17, 33, 1)])
def test_metrics_and_lpips_against_the_oracle(fp32, h, w, T):
    """PSNR / SSIM within 1e-5 relative, each tap's features within 1e-4 of scale, LPIPS within 1e-4 relative.  16x16 makes
    conv5 1x1, 31x45 and 17x33 floor odd sides at the pools."""
    from artdeco_b200 import evaluate
    from artdeco_b200.lpips import LPIPSVGG
    dev = fp32
    colors, alphas, gt, E = _random_views(T, h, w, h * 7 + w, dev)
    sd = ref.random_state_dict(11)
    ours = LPIPSVGG(sd, device=dev)
    oracle = ref.LPIPSRef().to(dev).eval()
    oracle.load_state_dict(sd)
    vf = torch.arange(T, dtype=torch.int32, device=dev)
    table = evaluate.metrics_from_renders(colors, alphas, gt, E, vf, lpips=ours).cpu()
    with torch.no_grad():
        for t in range(T):
            img = ref.render_from_colors(colors[t:t + 1], alphas[t:t + 1, ..., None], E[t])
            p = ref.psnr(img.reshape(-1), gt[t].reshape(-1))
            s = ref.ssim_ref.ssim(img[None], gt[t][None]).item()
            assert rel(table[t, evaluate.COL_PSNR].item(), p) <= TOL, (t, table[t, 0].item(), p)
            assert rel(table[t, evaluate.COL_SSIM].item(), s) <= TOL, (t, table[t, 1].item(), s)
            want = oracle(img[None], gt[t][None]).item()
            assert rel(table[t, evaluate.COL_LPIPS].item(), want) <= TOL_LPIPS, (t, table[t, 2].item(), want)
        # the taps, read through the test hook, on the oracle's own exposed images
        imgs = torch.stack([ref.render_from_colors(colors[t:t + 1], alphas[t:t + 1, ..., None], E[t]) for t in range(T)])
        val, taps = ours.features(imgs, gt)
        o0, o1 = oracle.taps(imgs, gt)
        for k in range(5):
            want = torch.stack([o0[k], o1[k]], 1).reshape(2 * T, *o0[k].shape[1:]).permute(0, 2, 3, 1)
            scale = want.abs().max().item()
            err = (taps[k] - want).abs().max().item()
            assert err <= TOL_LPIPS * scale, (k, err, scale)
        want = oracle(imgs, gt).reshape(-1)
        for t in range(T):
            assert rel(val.reshape(-1)[t].item(), want[t].item()) <= TOL_LPIPS
        assert val.shape == (T, 1, 1, 1)


@pytest.mark.gpu
def test_lpips_call_matches_the_module_and_chunks_by_budget(fp32):
    from artdeco_b200 import lpips as L
    dev = fp32
    sd = ref.random_state_dict(2)
    ours = L.LPIPSVGG(sd, device=dev)
    oracle = ref.LPIPSRef().to(dev).eval()
    oracle.load_state_dict(sd)
    g = torch.Generator().manual_seed(9)
    a, b = torch.rand(5, 3, 70, 90, generator=g).to(dev), torch.rand(5, 3, 70, 90, generator=g).to(dev)
    whole = ours(a, b)
    per = L.workspace_bytes(1, 70, 90)
    chunked = ours(a, b, workspace_bytes_budget=2 * per)
    assert L.frames_per_launch(5, 70, 90, 2 * per) == 2
    assert torch.equal(whole, chunked)                                  # chunking changes no bit
    with torch.no_grad():
        want = oracle(a, b)
    assert whole.shape == want.shape == (5, 1, 1, 1)
    assert ((whole - want).abs() <= TOL_LPIPS * want.abs()).all()


class _FakeLPIPS(torch.nn.Module):
    """A module shaped as lpips.LPIPS(net='vgg') for from_module (its attributes and state-dict names)."""

    def __init__(self, sd):
        super().__init__()
        self.pnet_type, self.version, self.spatial, self.lpips = "vgg", "0.1", False, True
        self.inner = ref.LPIPSRef()
        self.inner.load_state_dict(sd)

    def state_dict(self, *a, **k):
        return self.inner.state_dict()


@pytest.mark.gpu
def test_from_module_copies_the_weights(fp32):
    from artdeco_b200.lpips import LPIPSVGG
    dev = fp32
    sd = ref.random_state_dict(4)
    m = _FakeLPIPS(sd).to(dev)
    a, b = LPIPSVGG.from_module(m), LPIPSVGG(sd, device=dev)
    x0, x1 = torch.rand(2, 3, 32, 48, device=dev), torch.rand(2, 3, 32, 48, device=dev)
    assert torch.equal(a(x0, x1), b(x0, x1))


@pytest.mark.gpu
def test_no_host_sync_before_the_final_read_and_bitwise_repeatable(fp32):
    from artdeco_b200 import evaluate
    from artdeco_b200.lpips import LPIPSVGG
    dev = fp32
    T, h, w = 3, 243, 324
    colors, alphas, gt, E0 = _random_views(T, h, w, 21, dev)
    lp = LPIPSVGG(ref.random_state_dict(5), device=dev)
    flags = torch.tensor([1, 0, 1, 1, 0], dtype=torch.bool, device=dev)
    K = flags.numel()
    vis = (torch.rand(T, 1000, device=dev) < 0.3).to(torch.uint8)
    vf = torch.tensor([0, 2, 3], dtype=torch.int32, device=dev)
    E_full = torch.randn(K, 3, 4, device=dev)
    torch.cuda.synchronize()
    out = []
    for _ in range(2):
        E = E_full.clone()
        ews = evaluate.eval_workspace(T, h, w, 1000, dev)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            n_bad = evaluate.harmonize_test_exposure(E, flags)
            from artdeco_b200 import _lib
            for t in range(T):
                _lib.call("adb_eval_count_visible", T, h, w, 1000, t, _lib.ptr(vis[t]), _lib.ptr(ews), ews.numel(),
                          _lib.stream())
            table = evaluate.metrics_from_renders(colors, alphas, gt, E, vf, ews=ews, n_gaussians=1000, lpips=lp)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        out.append((table.cpu(), int(n_bad), E.cpu()))
    assert out[0][1] == 0
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][2], out[1][2])
    counts = vis.sum(1).cpu()
    assert torch.equal(out[0][0][:, evaluate.COL_RENDER].long(), counts)
    assert (out[0][0][:, evaluate.COL_GS] == 1000).all()


@pytest.mark.gpu
def test_evaluate_through_render_lod_against_the_oracle_fed_the_same_renders(fp32):
    from artdeco_b200 import evaluate, synthetic
    from artdeco_b200.lpips import LPIPSVGG
    from artdeco_b200.scene import render_lod
    dev = fp32
    H, W = 243, 324
    sc = synthetic.raster_scene(50_000, seed=3, z_range=(2.0, 8.0), extent=(2.5, 2.0))
    kw = dict(xyz=sc["means"].to(dev), opacity=sc["opacities"][:, None].to(dev), f_dc=sc["sh"][:, :1].contiguous().to(dev),
              f_rest=sc["sh"][:, 1:].contiguous().to(dev), scaling=sc["scales"].to(dev), rotation=sc["quats"].to(dev),
              d_max=sc["d_max"].to(dev), tanfovx=0.6, tanfovy=0.45)
    K = 5
    is_test = [True, False, True, True, False]
    vms = []
    for i in range(K):
        V = torch.eye(4)
        V[0, 3] = 0.05 * i
        vms.append(V)
    g = torch.Generator().manual_seed(2)
    gts = [torch.rand(3, H, W, generator=g) for _ in range(K)]
    E0 = (torch.eye(3, 4) + 0.03 * torch.randn(K, 3, 4, generator=g)).contiguous()
    sd = ref.random_state_dict(6)
    lp = LPIPSVGG(sd, device=dev)
    oracle = ref.LPIPSRef().to(dev).eval()
    oracle.load_state_dict(sd)
    seen = {}

    def render(vm):
        out = render_lod(W, H, vm, **kw)
        seen[float(vm[0, 3])] = out
        return out

    E = E0.to(dev)
    got = evaluate.evaluate(E, is_test, vms, gts, width=W, height=H, render=render, lpips=lp, with_LPIPS=True, all=True)
    renders, vis = {}, {}
    for i in range(K):
        o = seen.get(float(vms[i][0, 3]))
        if o is not None:
            renders[i] = (o["colors"], o["alphas"])
            vis[i] = o["visibility_filter"]
    ex = [E0[i].to(dev).clone() for i in range(K)]
    want = ref.evaluate(ex, is_test, renders, [x.to(dev) for x in gts], vis, lpips=oracle, with_LPIPS=True, all=True)
    assert torch.equal(E.cpu(), torch.stack(ex).cpu())
    assert_metrics(got, want, "render_lod")
    assert got["n_test_frames"] == 3 and got["Render"] > 0
    no_lpips = evaluate.evaluate(E0.to(dev), is_test, vms, gts, width=W, height=H, render=render, lpips=lp, with_LPIPS=False)
    assert "LPIPS" not in no_lpips and no_lpips["n_test_frames"] == 3

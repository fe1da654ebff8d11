"""The mapper's pixel loss (artdeco_b200.mapper.mapper_loss, csrc/mapper_loss.cu) against the reference's own statements
(tests/golden/mapper_loss_small.pt, made by make_mapper_loss_golden.py) and against oracle/mapper_loss_ref.py."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import mapper_loss_ref as ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mapper_loss_small.pt")
TOL = 1e-5
GRAD_KEYS = ("v_colors", "v_alphas", "v_exposure")


def golden():
    return torch.load(GOLDEN, weights_only=False)["cases"]


def assert_close_nonfinite(got, want, what, tol=TOL, max_outlier_frac=0.0):
    """Non-finite values at the same places with the same value (inf sign, NaN); finite ones within tol x max|finite want|."""
    a = np.asarray(got.detach().cpu(), dtype=np.float64)
    b = np.asarray(want.detach().cpu(), dtype=np.float64)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    fa, fb = np.isfinite(a), np.isfinite(b)
    assert (fa == fb).all(), f"{what}: non-finite at {int((fa != fb).sum())} different places"
    assert (np.isnan(a) == np.isnan(b)).all() and (a[np.isinf(b)] == b[np.isinf(b)]).all(), f"{what}: inf / NaN differ"
    if not fb.any():
        return
    scale = max(np.abs(b[fb]).max(), 1e-20)
    bad = np.abs(a[fb] - b[fb]) > tol * scale
    assert bad.mean() <= max_outlier_frac, (f"{what}: {bad.sum()} of {bad.size} exceed {tol} of scale "
                                            f"(max {np.abs(a[fb] - b[fb]).max() / scale:.3e})")


def run_oracle(inp, c, dev="cpu"):
    colors = inp["colors"].to(dev).clone().requires_grad_(True)
    alphas = inp["alphas"].to(dev).clone().requires_grad_(True)
    exposure = inp["exposure"].to(dev).clone().requires_grad_(True)
    out = ref.mapper_loss(colors, alphas, inp["gt"].to(dev), inp["mono"].to(dev), exposure, inp["bg"].to(dev),
                          lambda_dssim=c["lambda_dssim"], depth_weight=c["depth_weight"], rad_decay=c["rad_decay"],
                          is_important=c["is_important"])
    out["loss"].backward()
    out.update(v_colors=colors.grad, v_alphas=alphas.grad, v_exposure=exposure.grad)
    return out


def run_ours(inp, c, dev):
    from artdeco_b200.mapper import mapper_loss
    colors = inp["colors"].to(dev).clone().requires_grad_(True)
    alphas = inp["alphas"].to(dev).clone().requires_grad_(True)
    exposure = inp["exposure"].to(dev).clone().requires_grad_(True)
    loss, image, invdepth = mapper_loss(colors, alphas, inp["gt"].to(dev), inp["mono"].to(dev), exposure, inp["bg"].to(dev),
                                        lambda_dssim=c["lambda_dssim"], depth_weight=c["depth_weight"],
                                        rad_decay=c["rad_decay"], is_important=c["is_important"])
    loss.backward()
    return dict(loss=loss.detach(), image=image, invdepth=invdepth, v_colors=colors.grad, v_alphas=alphas.grad,
                v_exposure=exposure.grad)


# ------------------------------------------------------------------ CPU ------------------------------------------------------

def test_oracle_reproduces_the_reference_golden():
    """The fixture ran on one CPU; other instruction sets sum the SSIM convolutions in another order, so floats are compared
    within 1e-5 of scale, and every inf / NaN exactly."""
    for c in golden():
        want = c["outputs"]
        got = run_oracle(c["inputs"], c)
        what = f"important={c['is_important']} zero_depth={c['zero_depth']}"
        assert_close_nonfinite(got["loss"], want["loss"], f"{what} loss")
        assert_close_nonfinite(got["image"], want["image"], f"{what} image")
        assert_close_nonfinite(got["invdepth"], want["invdepth"], f"{what} invdepth")
        for k in GRAD_KEYS:
            assert_close_nonfinite(got[k], want[k], f"{what} {k}")


def test_golden_covers_the_edge_cases():
    cases = golden()
    assert {(c["is_important"], c["zero_depth"]) for c in cases} == {(a, b) for a in (True, False) for b in (True, False)}
    for c in cases:
        inp, out = c["inputs"], c["outputs"]
        pre = ref.expose(ref.composite(inp["colors"], inp["alphas"], inp["bg"])[0], inp["exposure"])[1]
        assert (pre == 1).any() and (pre == 0).any() and (pre > 1).any() and (pre < 0).any()   # on and beyond the bounds
        exposed = pre.clamp(0, 1)
        assert (exposed == inp["gt"]).any()                                                     # e == g ties
        zero_d = inp["colors"][0, ..., 3] == 0
        assert bool(zero_d.any()) == c["zero_depth"]
        if c["zero_depth"]:
            if c["is_important"]:
                assert torch.isinf(out["loss"])
            else:
                masked = (out["image"] == 0).all(0) & (inp["gt"] != 0).all(0)
                assert (zero_d & masked).any() and (zero_d & ~masked).any()                     # inf * 0 = NaN and inf
                assert torch.isnan(out["loss"]) and torch.isnan(out["invdepth"]).any()
        else:
            assert torch.isfinite(out["loss"])
        if not c["is_important"]:
            masked = (out["image"] == 0).all(0) & (inp["gt"] != 0).all(0)
            assert 0 < int(masked.sum()) < masked.numel()


def test_radial_table_is_bit_equal_to_the_reference_expression():
    from artdeco_b200 import mapper
    for c in golden():
        t = mapper.radial_weights(c["H"], c["W"], c["rad_decay"], "cpu")
        assert torch.equal(t, c["outputs"]["rdk"])
        assert mapper.radial_weights(c["H"], c["W"], c["rad_decay"], "cpu") is t                # built once per key
        assert torch.equal(ref.radial_decay_kernel(c["H"], c["W"], c["rad_decay"]), c["outputs"]["rdk"])


def test_entry_points_refuse_bad_arguments_before_touching_the_device():
    from artdeco_b200 import _lib
    import artdeco_b200  # noqa: F401  (registers every signature)
    L = _lib.lib()

    def refused(rc, needle, status=1):
        msg = L.adb_last_error()
        return rc == status and msg is not None and needle in msg.decode()

    nb = ctypes.c_size_t(0)
    assert refused(L.adb_mapper_loss_workspace_bytes(0, 5, ctypes.byref(nb)), "adb_mapper_loss_workspace_bytes")
    assert refused(L.adb_mapper_loss_workspace_bytes(5, -1, ctypes.byref(nb)), "adb_mapper_loss_workspace_bytes")
    assert refused(L.adb_mapper_loss_workspace_bytes(5, 5, None), "null bytes")
    assert refused(L.adb_mapper_loss_workspace_bytes(40000, 40000, ctypes.byref(nb)), "3hw")
    assert L.adb_mapper_loss_workspace_bytes(486, 648, ctypes.byref(nb)) == 0 and nb.value > 0
    need = nb.value
    fake = 1 << 20                         # a non-null, 16-byte aligned address that is never dereferenced
    p = [fake] * 7
    ok_out = [fake, fake, fake]
    assert refused(L.adb_mapper_loss_forward(0, 648, *p, 1, *ok_out, fake, need, None), "adb_mapper_loss_forward")
    assert refused(L.adb_mapper_loss_forward(486, 648, None, *p[1:], 1, *ok_out, fake, need, None), "null pointer")
    assert refused(L.adb_mapper_loss_forward(486, 648, *p, 1, *ok_out, None, need, None), "null pointer")
    assert refused(L.adb_mapper_loss_forward(486, 648, fake + 4, *p[1:], 1, *ok_out, fake, need, None), "aligned")
    assert refused(L.adb_mapper_loss_forward(486, 648, *p, 1, *ok_out, fake, need - 1, None), "workspace too small", 3)
    assert refused(L.adb_mapper_loss_reduce(486, 648, None, 0.2, 1.0, fake, fake, need, None), "null pointer")
    assert refused(L.adb_mapper_loss_reduce(486, 0, fake, 0.2, 1.0, fake, fake, need, None), "adb_mapper_loss_reduce")
    assert refused(L.adb_mapper_loss_reduce(486, 648, fake, 0.2, 1.0, fake, fake, 16, None), "workspace too small", 3)
    bw = [fake] * 7
    assert refused(L.adb_mapper_loss_backward(486, 648, *bw, 0, None, fake, 0.2, 1.0, fake, fake, fake, fake, need, None),
                   "null pointer")
    assert refused(L.adb_mapper_loss_backward(486, 648, *bw, 0, fake, fake, 0.2, 1.0, fake + 8, fake, fake, fake, need,
                                              None), "aligned")
    assert refused(L.adb_mapper_loss_backward(-3, 648, *bw, 0, fake, fake, 0.2, 1.0, fake, fake, fake, fake, need, None),
                   "adb_mapper_loss_backward")
    assert refused(L.adb_mapper_loss_backward(486, 648, *bw, 0, fake, fake, 0.2, 1.0, fake, fake, fake, fake, 0, None),
                   "workspace too small", 3)


def test_mapper_loss_raises_without_cuda():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from artdeco_b200 import _lib
    from artdeco_b200.mapper import mapper_loss
    inp = ref.make_inputs(8, 9, 0)
    with pytest.raises(_lib.ArtdecoB200Error):
        mapper_loss(inp["colors"], inp["alphas"], inp["gt"], inp["mono"], inp["exposure"], inp["bg"], lambda_dssim=0.2,
                    depth_weight=1.0, rad_decay=1.0, is_important=True)


# ------------------------------------------------------------------ GPU ------------------------------------------------------

@pytest.fixture
def fp32(cuda):
    m, c = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield cuda
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = m, c


def compare(got, want, inp, c, what):
    """Loss within 1e-5 relative; image, invdepth and gradients within 1e-5 of scale; non-finite values at the same places;
    mask and clamp decisions identical except within 1e-6 of a threshold, at most 1e-4 of the pixels."""
    n_pix = inp["gt"][0].numel()
    pre = want["pre_clamp"].detach()
    near_clamp = ((pre.abs() <= 1e-6) | ((pre - 1).abs() <= 1e-6)).any(0)
    flips = torch.zeros_like(near_clamp)
    # clamp decisions: where the pixel is kept, our image is on a bound exactly where the oracle's is
    kept = want["mask"] if want["mask"] is not None else torch.ones_like(near_clamp)
    on_bound_w = ((want["exposed"] == 0) | (want["exposed"] == 1)).detach()
    on_bound_g = (got["image"] == 0) | (got["image"] == 1)
    flips |= ((on_bound_w != on_bound_g).any(0) & kept & ~near_clamp)
    if want["mask"] is not None:
        # our kept pixels: the masked 1/D is non-zero (finite D) or inf (D = 0) where kept, 0 or NaN (inf * 0) where masked
        inv = got["invdepth"][0]
        ours_kept = (inv != 0) & ~torch.isnan(inv)
        rdk = ref.radial_decay_kernel(*pre.shape[1:], c["rad_decay"]).to(pre.device)
        err = rdk * (want["exposed"].detach() - inp["gt"]).abs()
        near_mask = ((err[:2] - 0.2).abs() <= 1e-6).any(0)
        flips |= (ours_kept != want["mask"]) & ~near_mask
    n_flip = int(flips.sum())
    assert n_flip <= 1e-4 * n_pix, f"{what}: {n_flip} mask / clamp decisions differ"
    frac = 1e-4 if n_pix >= 1e4 else 0.0
    assert_close_nonfinite(got["loss"], want["loss"], f"{what} loss")
    assert_close_nonfinite(got["image"], want["image"], f"{what} image", max_outlier_frac=frac)
    assert_close_nonfinite(got["invdepth"], want["invdepth"], f"{what} invdepth", max_outlier_frac=frac)
    for k in GRAD_KEYS:
        assert_close_nonfinite(got[k], want[k], f"{what} {k}", max_outlier_frac=frac if k != "v_exposure" else 0.0)


@pytest.mark.gpu
def test_golden_through_the_device_kernels(fp32):
    for c in golden():
        inp = {k: v.to(fp32) for k, v in c["inputs"].items()}
        got = run_ours(inp, c, fp32)
        want = c["outputs"]
        what = f"golden important={c['is_important']} zero_depth={c['zero_depth']}"
        assert_close_nonfinite(got["loss"], want["loss"], f"{what} loss")
        assert_close_nonfinite(got["image"], want["image"], f"{what} image")
        assert_close_nonfinite(got["invdepth"], want["invdepth"], f"{what} invdepth")
        for k in GRAD_KEYS:
            assert_close_nonfinite(got[k], want[k], f"{what} {k}")


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(37, 53), (486, 648), (972, 1296)])
@pytest.mark.parametrize("important", [True, False])
@pytest.mark.parametrize("zero_depth", [True, False])
def test_kernels_match_the_oracle_on_the_device(fp32, H, W, important, zero_depth):
    c = dict(lambda_dssim=0.2, depth_weight=0.6, rad_decay=1.0 if important else 0.5, is_important=important)
    inp = {k: v.to(fp32) for k, v in ref.make_inputs(H, W, seed=H + W, zero_depth=zero_depth).items()}
    want = run_oracle(inp, c, fp32)
    got = run_ours(inp, c, fp32)
    compare(got, want, inp, c, f"{H}x{W} important={important} zero_depth={zero_depth}")
    again = run_ours(inp, c, fp32)
    for k in ("loss", "image", "invdepth") + GRAD_KEYS:          # no float atomics anywhere: bitwise reproducible
        assert torch.equal(torch.nan_to_num(got[k], nan=7.0), torch.nan_to_num(again[k], nan=7.0)), k
        assert torch.equal(torch.isnan(got[k]), torch.isnan(again[k])), k


@pytest.mark.gpu
def test_upstream_gradient_scales_every_output(fp32):
    """The upstream gradient of the loss is read on the device and reaches every output: a power-of-two scale of it scales
    every gradient exactly."""
    from artdeco_b200.mapper import mapper_loss
    inp = {k: v.to(fp32) for k, v in ref.make_inputs(64, 80, seed=5, zero_depth=False).items()}
    grads = []
    for scale in (1.0, -2.0):
        colors = inp["colors"].clone().requires_grad_(True)
        alphas = inp["alphas"].clone().requires_grad_(True)
        E = inp["exposure"].clone().requires_grad_(True)
        loss, _, _ = mapper_loss(colors, alphas, inp["gt"], inp["mono"], E, inp["bg"], lambda_dssim=0.2, depth_weight=0.6,
                                 rad_decay=1.0, is_important=False)
        (scale * loss).backward()
        grads.append((colors.grad, alphas.grad, E.grad))
    for a, b in zip(*grads):
        assert a.abs().max() > 0 and torch.equal(b, -2.0 * a)


@pytest.mark.gpu
def test_end_to_end_through_the_rasterizer(fp32):
    """render_lod + mapper_loss + backward against render_lod + the oracle's loss + backward at 100k Gaussians, with the view
    matrix built from a 6-D rotation: every Gaussian parameter, the pose and the exposure within the rasterizer's 1e-4."""
    from helpers import assert_close
    from artdeco_b200 import synthetic
    from artdeco_b200.mapper import mapper_loss
    from artdeco_b200.scene import render_lod
    dev = fp32
    H, W = 486, 648
    sc = synthetic.raster_scene(100_000, seed=3, z_range=(2.0, 8.0), extent=(2.5, 2.0))
    base = dict(xyz=sc["means"], opacity=torch.logit(sc["opacities"][:, None]), f_dc=sc["sh"][:, :1].clone(),
                f_rest=sc["sh"][:, 1:].clone(), scaling=torch.log(sc["scales"]), rotation=sc["quats"])
    base = {k: v.to(dev) for k, v in base.items()}
    d_max = sc["d_max"].to(dev)
    ang = 0.05
    R0 = torch.tensor([[1.0, 0.0, 0.0], [0.0, np.cos(ang), -np.sin(ang)], [0.0, np.sin(ang), np.cos(ang)]],
                      dtype=torch.float32)
    g = torch.Generator().manual_seed(4)
    gt = (0.2 + 0.6 * torch.rand(3, H, W, generator=g)).to(dev)
    mono = (0.1 + 0.4 * torch.rand(1, H, W, generator=g)).to(dev)
    bg = torch.tensor([0.2, 0.5, 0.8], device=dev)
    E0 = torch.tensor([[1.05, 0.02, 0.0, 0.01], [0.0, 0.97, 0.03, -0.02], [0.01, 0.0, 1.02, 0.0]])
    f = 0.8 * W
    res = {}
    for name in ("ours", "oracle"):
        P = {k: v.clone().requires_grad_(True) for k, v in base.items()}
        r6 = R0[:, :2].clone().to(dev).requires_grad_(True)
        t = torch.tensor([0.05, -0.02, 0.1], device=dev, requires_grad=True)
        E = E0.clone().to(dev).requires_grad_(True)
        V = torch.eye(4, device=dev)
        V[:3, :3] = ref.sixD2mtx(r6)
        V[:3, 3] = t
        pkg = render_lod(W, H, V, xyz=P["xyz"], opacity=torch.sigmoid(P["opacity"]), f_dc=P["f_dc"], f_rest=P["f_rest"],
                         scaling=torch.exp(P["scaling"]), rotation=P["rotation"], d_max=d_max, tanfovx=W / (2 * f),
                         tanfovy=H / (2 * f), bg=None)
        kw = dict(lambda_dssim=0.2, depth_weight=0.3, rad_decay=1.0, is_important=False)
        if name == "ours":
            loss = mapper_loss(pkg["colors"], pkg["alphas"], gt, mono, E, bg, **kw)[0]
        else:
            loss = ref.mapper_loss(pkg["colors"], pkg["alphas"], gt, mono, E, bg, **kw)["loss"]
        loss.backward()
        res[name] = dict(loss=loss.detach(), r6=r6.grad, t=t.grad, E=E.grad, **{k: v.grad for k, v in P.items()})
    assert torch.isfinite(res["oracle"]["loss"])
    assert_close(res["ours"]["loss"], res["oracle"]["loss"], rtol=1e-5, what="loss")
    for k in ("xyz", "opacity", "f_dc", "f_rest", "scaling", "rotation", "r6", "t", "E"):
        assert res["oracle"][k] is not None and res["oracle"][k].abs().max() > 0, k
        assert_close(res["ours"][k], res["oracle"][k], what=k)

"""Pi3 on the GPU: the device model against the golden files made by running the reference (tests/golden/make_pi3_golden.py),
against the plain-torch oracle at shapes the golden files do not cover, the SVD orthogonalisation and qk-norm/RoPE
kernels against float64, and the accurate loop closure against the oracle's restatement.

Tolerance: 1e-4 of each tensor's scale (max-abs error over max-abs value) for bf16x3."""
import math
from pathlib import Path

import pytest
import torch

from artdeco_b200 import matching, synthetic
from artdeco_b200.pi3 import Pi3, accurate_loop_closure, param_shapes, score_window, svd_pose, window_input
from artdeco_b200.pi3.model import qknorm_rope
from artdeco_b200.mast3r import ops
from oracle import pi3_torch as pt

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden"
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max())


@pytest.fixture(scope="module")
def weights():
    return synthetic.det_weights(param_shapes())


@pytest.fixture(scope="module")
def model(weights):
    return Pi3().load_state_dict(weights).to(DEV)


@pytest.fixture
def fp32_torch():
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


def check_rotation(R):
    R = R.double().cpu()
    eye = torch.eye(3, dtype=torch.float64).expand_as(R)
    assert (R.transpose(-1, -2) @ R - eye).abs().max() < 1e-6
    assert (torch.linalg.det(R) - 1).abs().max() < 1e-6


@pytest.mark.parametrize("tag", ["small", "full"])
def test_bf16x3_matches_reference_golden(model, tag):
    g = torch.load(GOLDEN / f"pi3_{tag}.pt", weights_only=False)
    sp, tk, ch = g["stride_px"], g["stride_tok"], g["stride_ch"]
    st = {}
    out = model(synthetic.pi3_frames(g["N"], g["H"], g["W"], seed=g["seed"]).to(DEV), stages=st)
    torch.cuda.synchronize()
    for k in ("points", "local_points", "conf"):
        assert rel(out[k][:, :, ::sp, ::sp], g[k]) < 1e-4, (k, rel(out[k][:, :, ::sp, ::sp], g[k]))
    for k in ("encoder", "decoder", "point_hidden", "conf_hidden", "camera_hidden"):
        assert rel(st[k][:, ::tk, ::ch], g["stage." + k]) < 1e-4, (k, rel(st[k][:, ::tk, ::ch], g["stage." + k]))
    assert rel(st["fc_rot"], g["fc_rot"]) < 1e-4 and rel(st["fc_t"], g["fc_t"]) < 1e-4
    pose = out["camera_poses"].reshape(-1, 4, 4)
    ref = g["camera_poses"].reshape(-1, 4, 4)
    s = g["fc_rot_singular_values"]
    gap = torch.stack([s[:, 0] - s[:, 1], s[:, 1] - s[:, 2], s[:, 1] + s[:, 2]], -1).min(-1).values
    err = (pose[:, :3, :3].cpu().double() - ref[:, :3, :3].double()).abs().amax((-1, -2))
    assert bool((err <= 1e-4 * 4 / gap.clamp_min(1e-3)).all()), (err, gap)
    assert rel(pose[:, :3, 3], ref[:, :3, 3]) < 1e-4
    check_rotation(pose[:, :3, :3])


@pytest.mark.parametrize("N,H,W", [(1, 112, 140), (24, 112, 140), (2, 154, 98)], ids=["one_frame", "24_frames", "portrait"])
def test_against_oracle_at_other_shapes(model, weights, fp32_torch, N, H, W):
    imgs = synthetic.pi3_frames(N, H, W, seed=3).to(DEV)
    sd = {k: v.to(DEV) for k, v in weights.items()}
    with torch.inference_mode():
        ref = pt.forward(sd, imgs)
    out = model(imgs)
    torch.cuda.synchronize()
    for k in ("points", "local_points", "conf", "camera_poses"):
        assert out[k].shape == ref[k].shape
        assert rel(out[k], ref[k]) < 1e-4, (k, rel(out[k], ref[k]))
    check_rotation(out["camera_poses"].reshape(-1, 4, 4)[:, :3, :3])


def test_single_pass_bf16_within_stated_bound(model, weights):
    g = torch.load(GOLDEN / "pi3_small.pt", weights_only=False)
    imgs = synthetic.pi3_frames(g["N"], g["H"], g["W"], seed=g["seed"]).to(DEV)
    fast = Pi3(precision="bf16").load_state_dict(weights).to(DEV)
    a, b = fast(imgs), model(imgs)
    torch.cuda.synchronize()
    errs = {k: rel(a[k], b[k]) for k in ("points", "local_points", "conf", "camera_poses")}
    print("bf16 vs bf16x3:", errs)
    assert all(v < 5e-2 for v in errs.values()), errs


def _rot(seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))[0]
    return q * torch.sign(torch.linalg.det(q))


@pytest.mark.parametrize("case", ["identity", "reflection", "equal_singular_values", "rank2", "rank1"])
def test_svd_orthogonalisation_against_float64(case):
    P, Q = _rot(1), _rot(2)
    m = {"identity": torch.eye(3, dtype=torch.float64),
         "reflection": P @ torch.diag(torch.tensor([3.0, 2.0, -1.0], dtype=torch.float64)) @ Q.T,
         "equal_singular_values": P @ torch.diag(torch.tensor([3.0, 1.0, 1.0], dtype=torch.float64)) @ Q.T,
         "rank2": P @ torch.diag(torch.tensor([2.0, 1.0, 0.0], dtype=torch.float64)) @ Q.T,
         "rank1": torch.outer(torch.tensor([1.0, 2.0, 3.0], dtype=torch.float64), torch.tensor([0.3, -0.2, 0.5], dtype=torch.float64)),
         }[case]
    m32 = m.float().reshape(1, 9)
    t = torch.tensor([[0.5, -1.0, 2.0]])
    pose = svd_pose(m32.to(DEV), t.to(DEV)).cpu()
    R = pose[0, :3, :3]
    check_rotation(R[None])
    assert torch.equal(pose[0, :3, 3], t[0]) and torch.equal(pose[0, 3], torch.tensor([0.0, 0.0, 0.0, 1.0]))
    if case != "rank1":     # a rank-1 input has no unique nearest rotation
        ref = pt.svd_orthogonalize(m32.double())[0]
        assert (R.double() - ref).abs().max() < 1e-6, (R, ref)


def test_qknorm_rope_against_float64():
    B, N, h, C = 2, 7, 16, 1024
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(B * N, 3 * C, generator=g) * 3 + 0.5)
    gamma = 1 + 0.1 * torch.randn(64, generator=g)
    beta = 0.05 * torch.randn(64, generator=g)
    top = ops.ROPE_TABLE_POSITIONS - 1
    pos = torch.tensor([[0, 0], [0, top], [top, 0], [top, top], [1, 2], [top - 1, 5], [0, 0]]).repeat(B, 1).view(B, N, 2)
    for col0, norm in ((0, True), (C, True), (C, False)):
        sp = qknorm_rope(x.to(DEV), B, N, h, col0, gamma.to(DEV) if norm else None, beta.to(DEV) if norm else None,
                         pos.to(DEV))
        got = (sp.hi.double() + sp.lo.double()).cpu()
        q = x[:, col0:col0 + C].double().view(B, N, h, 64).transpose(1, 2)
        if norm:
            q = torch.nn.functional.layer_norm(q, (64,), gamma.double(), beta.double(), 1e-5)
        want = pt.rope2d(q, pos)
        # hi + lo carries 16 significant bits: up to 2^-17 (7.6e-6) of each element, the kernel's fp32 arithmetic adds ~1e-7
        assert rel(got, want) < 1e-5, rel(got, want)


def test_every_weight_the_model_passes_is_16_byte_aligned(model):
    """adb_layernorm and adb_pi3_tokens read their parameters with 128-bit loads and refuse misaligned pointers, so every
    fp32 parameter and every bf16 weight split the model holds must start on a 16-byte boundary."""
    bad = [k for k, v in model._sd.items() if v.data_ptr() % 16]
    bad += [k for k, s in model._w.items() for t in (s.hi, s.lo) if t is not None and t.data_ptr() % 16]
    assert len(model._sd) > 100 and not bad, bad


# ---- accurate loop closure --------------------------------------------------------------------------------------
CFG = {"matching": dict(max_iter=10, lambda_init=1e-8, convergence_thresh=1e-6, dist_thresh=1e-1, radius=4, dilation_max=5),
       "retrieval": dict(accurate_min=0.15, k=3)}


def _window(h=56, w=70):
    """A smooth surface seen by the query and by candidates yawed by growing angles (so their overlap, and the match
    fraction, shrinks), plus an exact duplicate for a tie and a candidate of unrelated points."""
    v, u = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    f = 0.9 * w
    d0 = torch.stack(((u - w / 2) / f, (v - h / 2) / f, torch.ones_like(u)), -1)
    d0 = d0 / d0.norm(dim=-1, keepdim=True)

    def view(deg):
        a = math.radians(deg)
        R = torch.tensor([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]])
        d = d0 @ R.T
        return d * (3.0 + 0.6 * torch.sin(3.0 * d[..., 0:1]) * torch.cos(2.0 * d[..., 1:2]))

    g = torch.Generator().manual_seed(5)
    cands = [view(a) for a in (2.0, 12.0, 2.0, 25.0, 5.0, 40.0)] + [torch.rand(h, w, 3, generator=g) * 10]
    return torch.stack(cands + [view(0.0)]).contiguous()


def test_score_window_matches_oracle_restatement():
    pts = _window().to(DEV)
    ids = [10, 11, 12, 13, 14, 15, 16, 30]
    sel, counts = score_window(pts, ids, CFG, chunk=3)
    want, want_counts = pt.score_window(pts, ids, CFG, matching.match_pi3)
    assert sel.tolist() == want and torch.equal(counts, want_counts)
    direct = torch.stack([matching.match_pi3(CFG, pts[i:i + 1].contiguous(), pts[-1:].contiguous())[1].sum() for i in range(7)])
    assert torch.equal(counts, direct)
    frac = counts.double() / pts[0, ..., 0].numel()
    assert (frac > 0.15).any() and (frac <= 0.15).any(), frac      # the gate is exercised on both sides
    assert counts[0] == counts[2]                                     # the duplicate ties


def test_window_input_matches_torch():
    g = torch.Generator().manual_seed(1)
    imgs = (torch.rand(3, 3, 100, 130, generator=g) * 2.4 - 1.2).to(DEV)    # values past [-1, 1] exercise the clamp
    got = window_input(imgs)
    want = pt.prepare_window(imgs)
    assert got.shape == (1, 3, 3, 392, 518) and (got - want).abs().max() < 1e-6


def test_accurate_loop_closure_end_to_end(model):
    g = torch.Generator().manual_seed(2)
    imgs = (torch.rand(4, 3, 96, 128, generator=g) * 2 - 1).to(DEV)
    ids = [3, 7, 8, 9]
    got = accurate_loop_closure(model, imgs, ids, CFG)
    pts = model(window_input(imgs))["points"][0]
    want, _ = pt.score_window(pts, ids, CFG, matching.match_pi3)
    assert got == want

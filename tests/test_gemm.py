"""wgmma GEMM + ViT companion kernels against plain PyTorch fp64 references (floating-point kernels: the torch
reference is the oracle here, per the tier rules)."""
import pytest
import torch

from helpers import rel_err


def _mk(shape, seed, dev):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).to(dev)


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 384, 128), (1024, 3072, 1024), (1000, 200, 136), (77, 64, 1024)])
def test_gemm_bf16x3_matches_fp64(cuda, M, N, K):
    from artdeco_b200.mast3r import ops
    a, w = _mk((M, K), 1, cuda), _mk((N, K), 2, cuda) * 0.05
    bias, res = _mk((N,), 3, cuda), _mk((M, N), 4, cuda)
    ref = a.double() @ w.double().T
    out = torch.empty(M, N, device=cuda)
    ops.gemm(ops.split(a), ops.split(w), M, N, K, out=out)
    assert rel_err(out, ref) < 2e-5, "bf16x3 product must be fp32-class (north-star 1e-4 budget over 36 layers)"
    # fused epilogue: alpha, bias, exact GELU, residual, split output
    sp = ops.Split(torch.empty(M, N, dtype=torch.bfloat16, device=cuda), torch.empty(M, N, dtype=torch.bfloat16, device=cuda))
    ops.gemm(ops.split(a), ops.split(w), M, N, K, out=out, out_split=sp, bias=bias, residual=res, alpha=0.5, act=1)
    ref2 = torch.nn.functional.gelu(0.5 * ref + bias.double()) + res.double()
    assert rel_err(out, ref2) < 2e-5
    assert rel_err(sp.hi.float() + sp.lo.float(), out) < 2e-5   # hi+lo keeps 16 mantissa bits
    # single-pass bf16 (the fast mode) is only bf16-accurate ...
    a1, w1 = ops.split(a, x3=False), ops.split(w, x3=False)
    ops.gemm(a1, w1, M, N, K, out=out)
    e1 = rel_err(out, ref)
    assert 1e-4 < e1 < 2e-2
    # ... but exact for its own bf16 operands up to fp32 accumulation, element by element (tests/test_tensorcore_edges.py)
    ah, wh = a1.hi.double(), w1.hi.double()
    assert ((out.double() - ah @ wh.T).abs() <= 3e-6 * (ah.abs() @ wh.abs().T)).all()


@pytest.mark.gpu
def test_gemm_batched_with_head_addressing(cuda):
    """The attention pattern: batch = B*h, outputs written straight into [B, N, h*64]."""
    from artdeco_b200.mast3r import ops
    B, h, N = 2, 3, 200
    q, k = _mk((B, h, N, 64), 1, cuda), _mk((B, h, N, 64), 2, cuda)
    s = torch.empty(B * h, N, N, device=cuda)
    ops.gemm(ops.split(q), ops.split(k), N, N, 64, batch=B * h, sA=N * 64, sB=N * 64, out=s, sD=N * N, alpha=0.125)
    assert rel_err(s.view(B, h, N, N), 0.125 * q.double() @ k.double().transpose(-1, -2)) < 2e-5
    p = torch.softmax(s, -1)
    v = _mk((B, h, N, 64), 3, cuda)
    Npad = 208
    vt = torch.zeros(B, h, 64, Npad, device=cuda)
    vt[..., :N] = v.transpose(-1, -2)
    pp = torch.zeros(B * h, N, Npad, device=cuda)
    pp[..., :N] = p
    o = torch.empty(B, N, h * 64, device=cuda)
    ops.gemm(ops.split(pp), ops.split(vt), N, 64, Npad, batch=B * h, sA=N * Npad, sB=64 * Npad, out=o, ldd=h * 64,
             zdiv=h, sD=64, sD2=N * h * 64)
    ref = (p.view(B, h, N, N).double() @ v.double()).permute(0, 2, 1, 3).reshape(B, N, h * 64)
    assert rel_err(o, ref) < 2e-5


@pytest.mark.gpu
def test_layernorm_softmax_rope_im2col(cuda):
    from artdeco_b200.mast3r import ops
    x = _mk((3, 50, 768), 5, cuda)
    g, b = _mk((768,), 6, cuda), _mk((768,), 7, cuda)
    y, sp = ops.layernorm(x, g, b, want_fp32=True)
    ref = torch.nn.functional.layer_norm(x.double(), (768,), g.double(), b.double(), 1e-6)
    assert rel_err(y, ref) < 1e-5 and rel_err(sp.hi.float() + sp.lo.float(), ref) < 2e-5
    s = _mk((40, 300), 8, cuda) * 3
    p = ops.softmax_rows(s, 40, 300, 300)
    assert rel_err(p.hi.float() + p.lo.float(), torch.softmax(s.double(), -1)) < 2e-5
    # RoPE2D against the reference formula (croco/models/pos_embed.py:112-159)
    B, N, h = 2, 48, 4
    qkv = _mk((B, N, 3 * h * 64), 9, cuda)
    pos = torch.cartesian_prod(torch.arange(6), torch.arange(8))[None].expand(B, -1, 2).contiguous().to(cuda)
    q = ops.rope_heads(qkv, B, N, h, 3 * h * 64, 0, pos, 0)
    tok = qkv.view(B, N, 3, h, 64)[:, :, 0].permute(0, 2, 1, 3).double()   # B,h,N,64

    def rope1d(t, p1):
        D = 32
        inv = 1.0 / (100.0 ** (torch.arange(0, D, 2, dtype=torch.float64, device=cuda) / D))
        fr = p1[..., None].double() * inv
        fr = torch.cat([fr, fr], -1)[:, None]
        rot = torch.cat([-t[..., 16:], t[..., :16]], -1)
        return t * fr.cos() + rot * fr.sin()
    ref = torch.cat([rope1d(tok[..., :32], pos[..., 0]), rope1d(tok[..., 32:], pos[..., 1])], -1)
    assert rel_err(q.hi.float() + q.lo.float(), ref) < 2e-5
    vt = ops.rope_heads(qkv, B, N, h, 3 * h * 64, 2 * h * 64, None, 2)
    refv = qkv.view(B, N, 3, h, 64)[:, :, 2].permute(0, 2, 3, 1)
    assert rel_err(vt.hi.float() + vt.lo.float(), refv) < 1e-5
    img = _mk((2, 3, 32, 48), 10, cuda)
    a = ops.im2col_patch16(img)
    refa = torch.nn.functional.unfold(img, 16, stride=16).transpose(1, 2).reshape(-1, 768)
    assert rel_err(a.hi.float() + a.lo.float(), refa) < 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [1, 2, 0], ids=["one_qtile_per_cta", "two_qtiles_persistent", "auto"])
@pytest.mark.parametrize("B,h,Nq,Nk", [(1, 2, 128, 128), (2, 3, 200, 200), (1, 16, 1024, 1024), (2, 12, 768, 768), (1, 2, 12, 12), (1, 2, 300, 130),
                                       (8, 16, 1024, 1024)])
def test_fused_attention_matches_fp64(cuda, B, h, Nq, Nk, variant):
    """csrc/attn_tc.cu (both kernel variants, and the automatic choice) against softmax(q k^T / 8) v in fp64
    (blocks.py:105-109,162-166).  (8,16,1024,1024) is the encoder call of the B=4 bench: 512 persistent work items."""
    from artdeco_b200.mast3r import ops
    q, k, v = _mk((B, h, Nq, 64), 1, cuda), _mk((B, h, Nk, 64), 2, cuda), _mk((B, h, Nk, 64), 3, cuda)
    Nkpad = (Nk + 7) // 8 * 8
    vt = torch.zeros(B, h, 64, Nkpad, device=cuda)
    vt[..., :Nk] = v.transpose(-1, -2)
    prev = ops.set_attention_variant(variant)
    try:
        o = ops.attention(ops.split(q), ops.split(k), ops.split(vt), B, h, Nq, Nk, Nkpad, 0.125)
        torch.cuda.synchronize()
    finally:
        ops.set_attention_variant(prev)
    ref = (torch.softmax(0.125 * q.double() @ k.double().transpose(-1, -2), -1) @ v.double()).permute(0, 2, 1, 3).reshape(B * Nq, h * 64)
    assert rel_err(o.hi.float() + o.lo.float(), ref) < 3e-5


@pytest.mark.gpu
@pytest.mark.parametrize("B,N,h,n_dst,tail", [(2, 200, 4, 2, True), (1, 1024, 16, 2, True), (3, 77, 2, 1, False), (2, 130, 12, 1, True)])
def test_gemm_rope_epilogue_matches_separate_kernels(cuda, B, N, h, n_dst, tail):
    """adb_gemm_bf16_rope (Linear + RoPE2D + head split in the epilogue) against Linear (adb_gemm_bf16) followed by the
    standalone adb_rope_heads kernel, and against the fp64 PyTorch formulation (oracle/mast3r_torch.py:rope2d)."""
    from artdeco_b200.mast3r import ops
    from oracle import mast3r_torch as mt
    g = torch.Generator().manual_seed(0)
    C = h * 64
    K = 192
    Nout = n_dst * C + (C if tail else 0)
    x = torch.randn(B * N, K, generator=g)
    w = torch.randn(Nout, K, generator=g) / K ** 0.5
    bias = torch.randn(Nout, generator=g)
    pos = torch.stack([torch.randint(0, 40, (B, N), generator=g), torch.randint(0, 64, (B, N), generator=g)], -1).to(cuda)
    a, ws = ops.split(x.to(cuda)), ops.split(w.to(cuda))
    q, k, v = ops.linear_rope(a, ws, bias.to(cuda), B, N, h, pos, n_dst)
    full, _ = ops.linear(a, ws, bias.to(cuda), B * N)
    q_ref = ops.rope_heads(full, B, N, h, Nout, 0, pos, 0)
    # both sides are 16-bit (hi+lo) roundings of fp32 values that may differ in the last ulp: 2^-16 granularity
    assert rel_err(q.hi.float() + q.lo.float(), q_ref.hi.float() + q_ref.lo.float()) < 2e-5
    if n_dst == 2:
        k_ref = ops.rope_heads(full, B, N, h, Nout, C, pos, 0)
        assert rel_err(k.hi.float() + k.lo.float(), k_ref.hi.float() + k_ref.lo.float()) < 2e-5
    else:
        assert k is None
    if tail:
        assert v.shape == (B * N, C) and rel_err(v, full[:, n_dst * C:]) < 1e-6
    else:
        assert v is None
    # fp64 reference of the whole thing
    y = (x.double() @ w.double().T + bias.double()).view(B, N, -1)
    qd = y[..., :C].reshape(B, N, h, 64).transpose(1, 2)
    assert rel_err(q.hi.float() + q.lo.float(), mt.rope2d(qd, pos.cpu(), base=100.0)) < 3e-5


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,C,crop,add", [(2, 16, 16, 256, None, True), (1, 9, 13, 128, (17, 25), False), (1, 32, 32, 256, None, False),
                                              (2, 8, 8, 256, (16, 16), True)])
def test_upsample2x_matches_torch_interpolate(cuda, B, H, W, C, crop, add):
    """adb_upsample2x_nhwc against F.interpolate(scale_factor=2, mode='bilinear', align_corners=True) exactly as the reference
    calls it (croco/models/dpt_block.py:215-216,320), with the fused skip add, the crop of dpt_head.py:57 and the bf16 split."""
    import torch.nn.functional as F
    from artdeco_b200.mast3r import ops
    x = _mk((B, H, W, C), 21, cuda)
    Ho, Wo = crop if crop else (2 * H, 2 * W)
    addend = _mk((B, Ho, Wo, C), 22, cuda) if add else None
    ref = F.interpolate(x.double().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
    ref = ref[:, :Ho, :Wo]
    if add:
        ref = ref + addend.double()
    y, sp = ops.upsample2x(x, addend=addend, out_hw=crop, want_fp32=True, want_split=True)
    assert y.shape == (B, Ho, Wo, C) and rel_err(y, ref) < 2e-6
    assert rel_err(sp.hi.float() + sp.lo.float(), ref) < 2e-5


@pytest.mark.gpu
def test_head_postprocess_matches_reference_formulas(cuda):
    """adb_head_postprocess against pixel_shuffle(16) + cat + postprocess written out as in mast3r/catmlp_dpt_head.py:25-39,
    87-96 and dust3r/heads/postprocess.py:22-58 (fp64), including a large log-depth range for expm1."""
    import torch.nn.functional as F
    from artdeco_b200.mast3r import ops
    B, H, W = 2, 48, 80
    S = (H // 16) * (W // 16)
    pts = _mk((B, H, W, 4), 31, cuda) * 2.0
    lf = _mk((B * S, 25 * 256), 32, cuda)
    res = ops.head_postprocess(pts, lf, H, W, 24)
    l = F.pixel_shuffle(lf.double().view(B, S, -1).transpose(-1, -2).reshape(B, -1, H // 16, W // 16), 16)
    fmap = torch.cat([pts.double(), l.permute(0, 2, 3, 1)], -1)
    xyz = fmap[..., 0:3]
    d = xyz.norm(dim=-1, keepdim=True)
    assert rel_err(res["pts3d"], xyz / d.clip(min=1e-8) * torch.expm1(d)) < 1e-6
    assert rel_err(res["conf"], 1 + fmap[..., 3].exp()) < 1e-6
    desc = fmap[..., 4:28]
    assert rel_err(res["desc"], desc / desc.norm(dim=-1, keepdim=True)) < 1e-6
    assert rel_err(res["desc_conf"], fmap[..., 28].exp()) < 1e-6

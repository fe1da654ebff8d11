"""The memory-bound companions of the tensor-core kernels on the MASt3R and Pi3 paths, element by element:
csrc/vit_ops.cu (adb_layernorm, adb_softmax_rows, adb_rope_heads, adb_im2col_patch16, adb_upsample2x_nhwc,
adb_head_postprocess, adb_rope2d_inplace) and csrc/pi3.cu (adb_pi3_patch14, adb_pi3_tokens, adb_pi3_point_head,
adb_pi3_camera_tail, adb_pi3_window_input).

* References.  Every arithmetic kernel is compared PER ELEMENT with a float64 restatement of its operation on the very
  fp32 inputs it read.  Pure copies and splits (im2col, head split / transpose, patch normalisation, token assembly) are
  compared bitwise against torch fp32.  Window resizing is compared with F.interpolate on the device.
* Tolerances.  Each bound is derived from the kernel's fp32 operation sequence, with u = 2^-24 the unit roundoff and the
  CUDA maximum ulp errors of the math functions (expf 2, expm1f 1, powf 4, sincosf 2; sqrtf and division are correctly
  rounded).  One ulp of a value v is at most 2u|v|.  The derivation sits in each test's docstring.  Every check prints
  the largest error over its bound; the test fails when that ratio exceeds 1.
* Splits.  A kernel that computes one fp32 value and also writes it as bf16 (hi, lo) must satisfy hi == bf16(y) and
  lo == bf16(y - hi) bitwise.  Run again with lo = NULL, its hi must not change.  hi + lo keeps 16 bits: a split output
  alone is within 2^-16 |y| of the fp32 value y it was made from.
* Canaries.  Pad columns, pad heads and unread NaN columns are pre-filled with sentinels that must come back untouched.
* Bug models (CPU part).  Each models a plausible bug in Python and must land at least 10x the tolerance away.

Which case reaches which code path:
  layernorm_kernel<4> (C <= 1024): C = 8 .. 1024;  <8>: C = 1032 .. 2048.  Lane tails: C = 8, 248, 264, 1016, 1032, 2040.
  softmax_reg_kernel<8>: L = 4, 124, 128, 132, 1020, 1024 with layout "dense" or "ld_pad4";  <16>: L = 1028, 2044,
  2048 in the same layouts;
  softmax_kernel (generic): L = 1, 3, 5, 2052, 5000, and every L with layout "ld_odd" or "offset".
  rope_heads_kernel mode 0 / 1 and heads_transpose_kernel (mode 2): test_rope_heads[mode].
  Grid-stride loops past the launch caps (132 * 32 CTAs of 256 threads in vit_ops.cu, 132 * 16 in pi3.cu):
    rope_heads B=9 N=1035 h=16 (modes 0, 1), im2col B=3 at 512x384, upsample 2x96x128x64, head_postprocess 4x512x544,
    pi3_patch14 24x392x518, pi3_tokens BN=24 n=1036, pi3_point_head 3x392x518, pi3_window_input 2->392x518.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24            # fp32 unit roundoff
SPLIT = 2.0 ** -16        # relative error of hi + lo against the fp32 value they split
TINY = 2.0 ** -126        # absolute floor: values below the smallest normal fp32 may underflow to 0
SENT = -768.0             # canary: finite, exact in fp32 and bf16


def vp(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def call(name, *args):
    from artdeco_b200 import _lib
    import artdeco_b200  # noqa: F401  (registers every signature)
    _lib.call(name, *args, _lib.stream())


def split32(y):
    """The bf16 (hi, lo) split every kernel writes: hi = rn(y), lo = rn(y - hi)."""
    hi = y.to(BF16)
    return hi, (y - hi.float()).to(BF16)


def assert_split(hi, lo, y, what):
    h, l = split32(y)
    assert torch.equal(hi, h), f"{what}: hi != bf16(y)"
    if lo is not None:
        assert torch.equal(lo, l), f"{what}: lo != bf16(y - hi)"


def ratio(err, bnd):
    """Largest err / bound; NaN anywhere in the error counts as infinitely wrong."""
    err, bnd = err.double(), bnd.double()
    if err.numel() == 0:
        return 0.0
    if torch.isnan(err).any():
        return math.inf
    return float((err / bnd).max())


def check(what, err, bnd):
    r = ratio(err, bnd)
    print(f"[companion] {what}: max err / bound = {r:.3e}")
    assert r <= 1.0, f"{what}: error {r:.3e} x the derived bound"
    return r


def gen(seed, dev="cpu"):
    return torch.Generator(device=dev).manual_seed(seed)


# ---- LayerNorm -------------------------------------------------------------------------------------------------------
LN_C = [8, 16, 248, 256, 264, 768, 1016, 1024, 1032, 1536, 2040, 2048]


def ln_rows(C, eps, g):
    """18 rows (two CTAs and a partial third): N(0,1); constant 3 and 0.75 (partial sums exact, so the output is
    exactly beta); one channel 100x the rest; variance comparable to eps; offset rows with mean/std 1e4."""
    rows = [torch.randn(5, C, generator=g), torch.full((2, C), 3.0), torch.full((2, C), 0.75)]
    o = torch.randn(3, C, generator=g)
    o[torch.arange(3), torch.randint(0, C, (3,), generator=g)] = torch.tensor([100.0, -100.0, 100.0])
    rows.append(o)
    rows.append(math.sqrt(eps) * torch.randn(3, C, generator=g))
    rows.append(torch.tensor([[1e4], [-3e3], [50.0]]) + torch.tensor([[1.0], [0.3], [5e-3]]) * torch.randn(3, C, generator=g))
    return torch.cat(rows).float()


def ln_kernel_mean(x):
    """The kernel's fp32 mean, in its order: lane l sums columns k*256 + 8l + e for k, then e (zeros past C), then the
    xor butterfly 16, 8, 4, 2, 1 (every lane ends with the same sum), then one division by C."""
    R, C = x.shape
    CH = 4 if C <= 1024 else 8
    xp = torch.zeros(R, CH * 256, dtype=F32)
    xp[:, :C] = x
    xp = xp.view(R, CH, 32, 8)
    s = torch.zeros(R, 32, dtype=F32)
    for k in range(CH):
        for e in range(8):
            s = s + xp[:, k, :, e]
    lanes = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        s = s + s[:, lanes ^ o]
    return s[:, 0] / torch.tensor(float(C), dtype=F32)


def ln_reference(x, gamma, beta, eps, one_pass=False):
    """float64 LayerNorm of the fp32 rows and the per-element bound of the kernel's fp32 sequence:
      mean: the kernel's fp32 mean mu32 (ln_kernel_mean, its exact order) is off by |mu32 - mu|; half an ulp more allows
            for a compiler that associates the sum differently: dmu = |mu32 - mu| + ulp(mu32) / 2;
      var:  sum of d^2, d = x - mu32: each term 3u, at most 8*ceil(C/256) + 5 additions per lane and butterfly, /C, +eps,
            sqrtf, 1/ -> rstd relative error eps_r = (n_add/2 + 5) u + dmu^2 / (2 (var + eps)) (Sum d^2 = Sum n^2 + C dmu^2);
      out:  (d * rstd) * g + b: |gamma| rstd (dmu + (|n| + dmu)(eps_r + 3u)) + 2u (|y| + |beta|).
    one_pass=True returns the E[x^2] - E[x]^2 bug model in fp32 instead of the reference."""
    x64, g64, b64 = x.double(), gamma.double(), beta.double()
    C = x.shape[1]
    mu = x64.mean(1, keepdim=True)
    n = x64 - mu
    var = (n * n).mean(1, keepdim=True)
    r = 1.0 / torch.sqrt(var + eps)
    y = n * r * g64 + b64
    mu32 = ln_kernel_mean(x)[:, None]
    dmu = (mu32.double() - mu).abs() + 0.5 * 2.0 ** (torch.frexp(mu32).exponent - 24).double()
    n_add = 8 * math.ceil(C / 256) + 5
    eps_r = (n_add / 2 + 5) * U + dmu ** 2 / (2 * (var + eps))
    bnd = g64.abs() * r * (dmu + (n.abs() + dmu) * (eps_r + 3 * U)) + 2 * U * (y.abs() + b64.abs()) + 1e-30
    if one_pass:
        m32 = x.mean(1, keepdim=True)
        v32 = (x * x).mean(1, keepdim=True) - m32 * m32
        y = ((x - m32) / torch.sqrt(v32.clamp(min=0) + eps) * gamma + beta).double()
    return y, bnd


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [1e-6, 1e-5])
@pytest.mark.parametrize("C", LN_C)
def test_layernorm(cuda, C, eps):
    """adb_layernorm per element against float64 (bound: ln_reference), outputs y only, hi only and y + hi + lo."""
    g = gen(C)
    x = ln_rows(C, eps, g)
    gamma = (1.0 + 0.5 * torch.randn(C, generator=g)).float()
    beta = torch.randn(C, generator=g).float()
    ref, bnd = ln_reference(x, gamma, beta, eps)
    xd, gd, bd = x.to(cuda), gamma.to(cuda), beta.to(cuda)
    R = x.shape[0]

    def run(want_y, want_hi, want_lo):
        y = torch.full((R, C), SENT, device=cuda) if want_y else None
        hi = torch.full((R, C), SENT, dtype=BF16, device=cuda) if want_hi else None
        lo = torch.full((R, C), SENT, dtype=BF16, device=cuda) if want_lo else None
        call("adb_layernorm", R, C, vp(xd), vp(gd), vp(bd), float(eps), vp(y), vp(hi), vp(lo))
        return y, hi, lo

    y, hi, lo = run(True, True, True)
    y_only, _, _ = run(True, False, False)
    _, hi_only, _ = run(False, True, False)
    torch.cuda.synchronize()
    y, hi, lo, y_only, hi_only = (t.cpu() for t in (y, hi, lo, y_only, hi_only))
    check(f"layernorm C={C} eps={eps:g}", (y.double() - ref).abs(), bnd)
    assert_split(hi, lo, y, f"layernorm C={C}")
    assert torch.equal(y_only, y) and torch.equal(hi_only, hi)
    # constant rows: the mean is exact, so every output is exactly beta
    assert torch.equal(y[5:9], beta.expand(4, C)) and torch.equal(hi[5:9], beta.to(BF16).expand(4, C))


# ---- softmax ---------------------------------------------------------------------------------------------------------
SM_L = [1, 3, 4, 5, 124, 128, 132, 1020, 1024, 1028, 2044, 2048, 2052, 5000]
# name -> (ld_in - L, ld_out - L, input offset in floats)
SM_LAYOUT = {"dense": (0, 0, 0), "ld_pad4": (4, 8, 0), "ld_odd": (3, 8, 0), "offset": (0, 4, 1)}


def softmax_path(L, ld_in, ld_out, off):
    """adb_softmax_rows' dispatch (hi and lo are fresh allocations, so 8-byte aligned)."""
    fast = L % 4 == 0 and ld_in % 4 == 0 and ld_out % 4 == 0 and off % 4 == 0 and L <= 2048
    return "reg8" if fast and L <= 1024 else ("reg16" if fast else "generic")


def softmax_rows(L, g):
    """Rows: 0-2 N(0,1); 3-5 N(0,30^2); 6 all equal; 7 one dominant entry; 8 -inf next to finite entries;
    9 finfo.min everywhere; 10 all -inf; 11 one NaN.  Rows 10 and 11 must give NaN, as torch.softmax does."""
    x = torch.randn(12, L, generator=g)
    x[3:6] *= 30
    x[6] = 1.5
    x[7] = 0.0
    x[7, (L * 2) // 3] = 200.0
    x[8, ::3] = -math.inf
    if L == 1:
        x[8] = 0.25
    x[9] = torch.finfo(F32).min
    x[10] = -math.inf
    x[11, L // 2] = math.nan
    return x.float()


def softmax_reference(x, drop_tail=None):
    """float64 softmax of the fp32 rows and the bound of the kernel's sequence: e_i = expf(fl(x_i - m)) has relative
    error (|x_i - m| + 4) u (argument rounding, 2 ulp); the row sum S adds ceil(L/32) + 5 positive terms per lane and
    butterfly, so (ceil(L/32) + 5) u + the e-weighted term error; 1/S and e * (1/S) add 2u; the (hi, lo) output adds
    2^-16; values below 2^-126 may underflow (absolute floor).
    drop_tail=c models a kernel that drops columns c.. from the sum and never writes them."""
    x64 = x.double()
    L = x.shape[1]
    m = x64.amax(1, keepdim=True)
    dx = (x64 - m).abs().nan_to_num(1e4, 1e4).clamp(max=1e4)
    e = torch.exp(x64 - m)
    S = e.sum(1, keepdim=True)
    p = e / S
    eps_S = (math.ceil(L / 32) + 5) * U + (e * (dx + 4)).sum(1, keepdim=True) / S * U
    rel = (dx + 4) * U + eps_S + 2 * U
    bnd = p * (rel + SPLIT * (1 + rel)) + TINY
    if drop_tail is not None:
        e2 = e.clone()
        e2[:, drop_tail:] = 0
        p = e2 / e2.sum(1, keepdim=True)
    return p, bnd


@pytest.mark.gpu
@pytest.mark.parametrize("layout", list(SM_LAYOUT))
@pytest.mark.parametrize("L", SM_L)
def test_softmax_rows(cuda, L, layout):
    """adb_softmax_rows per element against float64 (bound: softmax_reference) through all three kernels, with the pad
    columns of ld_out > L left untouched, exact results for equal rows (fp32(1/L)), a dominant entry (1 and 0), -inf
    entries (0) and the finfo.min row (fp32(1/L)), and NaN for all -inf and NaN rows."""
    dli, dlo, off = SM_LAYOUT[layout]
    ld_in, ld_out = L + dli, L + dlo
    x = softmax_rows(L, gen(L + 7 * dli))
    R = x.shape[0]
    buf = torch.full((off + R * ld_in,), 12345.0)
    buf[off:].view(R, ld_in)[:, :L] = x
    s = buf.to(cuda)[off:]
    print(f"[companion] softmax L={L} {layout}: path {softmax_path(L, ld_in, ld_out, off)}")

    def run(with_lo):
        hi = torch.full((R, ld_out), SENT, dtype=BF16, device=cuda)
        lo = torch.full((R, ld_out), SENT, dtype=BF16, device=cuda) if with_lo else None
        call("adb_softmax_rows", R, L, ld_in, ld_out, vp(s), vp(hi), vp(lo))
        return hi, lo

    hi, lo = run(True)
    hi1, _ = run(False)
    torch.cuda.synchronize()
    hi, lo, hi1 = hi.cpu(), lo.cpu(), hi1.cpu()
    assert torch.equal(hi1.view(torch.int16), hi.view(torch.int16))      # bitwise: the NaN rows compare too
    assert (hi[:, L:] == SENT).all() and (lo[:, L:] == SENT).all(), "pad columns were written"
    hi, lo = hi[:, :L], lo[:, :L]
    fin = slice(0, 10)
    p, bnd = softmax_reference(x[fin])
    got = hi[fin].double() + lo[fin].double()
    check(f"softmax L={L} {layout}", (got - p).abs(), bnd)
    uni = (torch.tensor(1.0) / torch.tensor(float(L))).expand(L)     # fp32(1/L): 1 / S with S = L exact, times expf(0) = 1
    for r in (6, 9):
        assert_split(hi[r], lo[r], uni, f"softmax L={L} row {r}")
    one = torch.zeros(L, dtype=F32)
    one[(L * 2) // 3] = 1.0
    assert_split(hi[7], lo[7], one, f"softmax L={L} dominant row")
    if L > 1:
        assert (hi[8, ::3] == 0).all() and (lo[8, ::3] == 0).all(), "-inf logits must give exactly 0"
    assert torch.isnan(hi[10:].float()).all(), "all -inf and NaN rows must give NaN, as torch.softmax does"


# ---- RoPE heads (split, transpose) -----------------------------------------------------------------------------------
def rope_heads_reference(xs, pos, table, partner=16, swap=False):
    """xs float64 [B, h, N, 64] (the head slice), pos [B, N, 2] clamped to the table, table fp32 [n_pos, 16, 2].
    Each 32-dim half (y then x) rotates dim j < 16 with j + 16: (a c - b s, b c + a s) by the table's fp32 (cos, sin).
    Bound: fl(fl(v c) -+ fl(o s)) (or one fma) is within 2u (|v c| + |o s|); the (hi, lo) output adds 2^-16.
    partner=8 / swap=True are bug models (partner dimension j ^ 8; the y and x positions exchanged)."""
    tb = table.double()
    outs, abss = [], []
    for half in (0, 1):
        p = pos[..., 1 - half if swap else half]
        c, s = tb[p][..., 0][:, None], tb[p][..., 1][:, None]     # [B, 1, N, 16]
        t = xs[..., 32 * half:32 * half + 32]
        idx = torch.arange(32, device=xs.device) ^ partner
        o = t[..., idx]
        a, b = t[..., :16], o[..., :16]
        bb, aa = t[..., 16:], o[..., 16:]
        outs += [a * c - b * s, bb * c + aa * s]
        abss += [(a * c).abs() + (b * s).abs(), (bb * c).abs() + (aa * s).abs()]
    out, A = torch.cat(outs, -1), torch.cat(abss, -1)
    return out, 2 * U * A + SPLIT * (out.abs() + 2 * U * A) + 1e-30


def rope_positions(B, N, n_pos, g):
    """(y, x) with y != x, covering 0 and n_pos - 1."""
    y = torch.randint(0, n_pos, (B, N), generator=g)
    y.view(-1)[0] = 0
    y.view(-1)[-1] = n_pos - 1
    x = (y + torch.randint(1, n_pos, (B, N), generator=g)) % n_pos
    return torch.stack([y, x], -1)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("N", [1, 63, 64, 65, 1035])
@pytest.mark.parametrize("h", [1, 12, 16])
def test_rope_heads(cuda, h, N, mode):
    """adb_rope_heads for q (col0 0), k (C) and v (2C) of a qkv row block (ld 3C), for k of a kv block (ld 2C) and for
    rows with extra columns (ld 3C + 12, col0 2C + 8).  Mode 0 against float64 (bound: rope_heads_reference), modes 1
    and 2 bitwise against the split of the input; mode 2's pad columns [N, Npad) exactly 0 in hi and lo."""
    from artdeco_b200.mast3r import ops
    C = h * 64
    B = 9 if (N == 1035 and h == 16 and mode != 2) else 2      # B*N*h*8 = 1.19M threads: past the grid cap
    n_pos = 64
    table = ops.rope_table(n_pos, cuda)
    pos = rope_positions(B, N, n_pos, gen(N + h)).to(cuda)
    Npad = (N + 7) // 8 * 8 + 8
    gd = gen(h * 1000 + N, cuda)
    worst = 0.0
    for ld, col0 in ((3 * C, 0), (3 * C, C), (3 * C, 2 * C), (2 * C, C), (3 * C + 12, 2 * C + 8)):
        x = torch.randn(B, N, ld, generator=gd, device=cuda)
        shape = (B, h, 64, Npad) if mode == 2 else (B, h, N, 64)
        hi = torch.full(shape, SENT, dtype=BF16, device=cuda)
        lo = torch.full(shape, SENT, dtype=BF16, device=cuda)
        hi1 = torch.full(shape, SENT, dtype=BF16, device=cuda)
        for hh, ll in ((hi, lo), (hi1, None)):
            call("adb_rope_heads", B, N, h, ld, col0, vp(x), vp(pos), vp(table), n_pos, mode, Npad, vp(hh), vp(ll))
        assert torch.equal(hi1, hi)
        xs = x[..., col0:col0 + C].reshape(B, N, h, 64).permute(0, 2, 1, 3)
        if mode == 0:
            ref, bnd = rope_heads_reference(xs.double(), pos, table)
            r = ratio((hi.double() + lo.double() - ref).abs(), bnd)
            worst = max(worst, r)
            assert r <= 1.0, (ld, col0, r)
        elif mode == 1:
            assert_split(hi, lo, xs.contiguous(), f"rope_heads mode 1 ld={ld} col0={col0}")
        else:
            assert_split(hi[..., :N], lo[..., :N], xs.transpose(-1, -2).contiguous(), f"rope_heads mode 2 ld={ld}")
            assert not hi[..., N:].any() and not lo[..., N:].any(), "transpose pad columns must be exactly 0"
        del x, hi, lo, hi1
    if mode == 0:
        print(f"[companion] rope_heads h={h} N={N} B={B}: max err / bound = {worst:.3e}")


@pytest.mark.gpu
def test_rope_heads_clamps_positions(cuda):
    """Positions outside [0, n_pos) use the nearest table row: -5 and -1 rotate by row 0 (the identity), 64 and 1000 by
    row 63.  The result equals the kernel's own result for the clamped positions bitwise, and the float64 rotation."""
    from artdeco_b200.mast3r import ops
    B, N, h, n_pos = 1, 6, 2, 64
    table = ops.rope_table(n_pos, cuda)
    pos = torch.tensor([[[-5, 3], [0, -1], [63, 64], [1000, 7], [64, -1000], [5, 63]]], device=cuda)
    x = torch.randn(B, N, h * 64, generator=gen(3, cuda), device=cuda)
    out = []
    for p in (pos, pos.clamp(0, n_pos - 1)):
        hi = torch.empty(B, h, N, 64, dtype=BF16, device=cuda)
        lo = torch.empty_like(hi)
        call("adb_rope_heads", B, N, h, h * 64, 0, vp(x), vp(p.contiguous()), vp(table), n_pos, 0, N, vp(hi), vp(lo))
        out.append((hi, lo))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    ref, bnd = rope_heads_reference(x.view(B, N, h, 64).permute(0, 2, 1, 3).double(), pos.clamp(0, n_pos - 1), table)
    check("rope_heads clamped positions", (out[0][0].double() + out[0][1].double() - ref).abs(), bnd)
    # the identity rows: position -5 / 0 leaves the y half unchanged up to the split
    assert_split(out[0][0][0, :, 0, :32], out[0][1][0, :, 0, :32], x.view(N, h, 64)[0, :, :32], "row 0 is the identity")


# ---- im2col ----------------------------------------------------------------------------------------------------------
def im2col_reference(img, swap=False):
    """F.unfold(16, stride 16) rows [B * patches, 768] in (c, py, px) order; swap=True is the (c, px, py) bug model."""
    a = F.unfold(img, 16, stride=16).transpose(1, 2).reshape(-1, 768)
    if swap:
        a = a.view(-1, 3, 16, 16).transpose(-1, -2).reshape(-1, 768)
    return a


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W", [(1, 16, 16), (2, 32, 48), (3, 512, 384)])
def test_im2col_patch16(cuda, B, H, W):
    """adb_im2col_patch16 bitwise against F.unfold and the split; 3 x 512 x 384 is 1.77M elements, past the grid cap."""
    img = torch.randn(B, 3, H, W, generator=gen(B, cuda), device=cuda)
    n = B * (H // 16) * (W // 16)
    hi, lo, hi1 = (torch.empty(n, 768, dtype=BF16, device=cuda) for _ in range(3))
    call("adb_im2col_patch16", B, H, W, vp(img), vp(hi), vp(lo))
    call("adb_im2col_patch16", B, H, W, vp(img), vp(hi1), None)
    assert_split(hi, lo, im2col_reference(img), f"im2col {B}x{H}x{W}")
    assert torch.equal(hi1, hi)


# ---- bilinear x2 upsampling (align_corners=True) ---------------------------------------------------------------------
def upsample_reference(x, Ho, Wo, addend=None, align_corners=True):
    """float64 bilinear x2 of NHWC x at the kernel's fp32 source coordinates (src = fp32((in-1)/(2in-1)) * dst, as
    torch's upsample_bilinear2d computes them), cropped to Ho x Wo, + addend.
    Bound: hy = 1 - ly and hx = 1 - lx round (u each), three products/fmas per row and per column (3u + 3u) on the
    weighted sum of |v|, the addend add u |out|: 6u M + u |out| + 2u |addend| with M = sum of weight * |v|.
    align_corners=False is the bug model (F.interpolate's half-pixel coordinates)."""
    B, Hin, Win, C = x.shape
    x64 = x.double()
    if not align_corners:
        r = F.interpolate(x64.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=False)
        r = r.permute(0, 2, 3, 1)[:, :Ho, :Wo]
        return (r + addend.double() if addend is not None else r), None

    def axis(n_in, n_out):
        sc = torch.tensor(float(n_in - 1), dtype=F32) / torch.tensor(float(2 * n_in - 1), dtype=F32)
        f = sc * torch.arange(n_out, dtype=F32)
        i0 = f.floor().long()
        i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
        return i0.to(x.device), i1.to(x.device), (f - i0.float()).double().to(x.device)
    y0, y1, ly = axis(Hin, Ho)
    x0, x1, lx = axis(Win, Wo)
    ly, lx = ly[:, None, None], lx[None, :, None]

    def g(yy, xx):
        return x64[:, yy][:, :, xx]
    v00, v01, v10, v11 = g(y0, x0), g(y0, x1), g(y1, x0), g(y1, x1)
    out = (1 - ly) * ((1 - lx) * v00 + lx * v01) + ly * ((1 - lx) * v10 + lx * v11)
    M = (1 - ly) * ((1 - lx) * v00.abs() + lx * v01.abs()) + ly * ((1 - lx) * v10.abs() + lx * v11.abs())
    a = addend.double() if addend is not None else torch.zeros_like(out)
    out = out + a
    return out, 6 * U * M + U * out.abs() + 2 * U * a.abs() + 1e-30


@pytest.mark.gpu
@pytest.mark.parametrize("B,Hin,Win,C,Ho,Wo,add", [
    (2, 1, 5, 4, 2, 10, True), (1, 6, 1, 8, 12, 2, False), (1, 1, 1, 4, 2, 2, True), (2, 9, 13, 4, 17, 25, True),
    (1, 9, 13, 12, 17, 25, False), (2, 8, 6, 256, 16, 12, True), (2, 96, 128, 64, 192, 256, True)])
def test_upsample2x_nhwc(cuda, B, Hin, Win, C, Ho, Wo, add):
    """adb_upsample2x_nhwc per element against float64 (bound: upsample_reference).  Hin = 1 / Win = 1 take the y1 = y0
    branch; 17 x 25 from 9 x 13 is the odd crop; 2 x 192 x 256 x 64 is 1.57M threads, past the grid cap."""
    gd = gen(Hin * 100 + Win, cuda)
    x = torch.randn(B, Hin, Win, C, generator=gd, device=cuda)
    addend = torch.randn(B, Ho, Wo, C, generator=gd, device=cuda) if add else None
    y = torch.full((B, Ho, Wo, C), SENT, device=cuda)
    hi, lo, hi1 = (torch.full((B, Ho, Wo, C), SENT, dtype=BF16, device=cuda) for _ in range(3))
    y1 = torch.full_like(y, SENT)
    call("adb_upsample2x_nhwc", B, Hin, Win, C, Ho, Wo, vp(x), vp(addend), vp(y), vp(hi), vp(lo))
    call("adb_upsample2x_nhwc", B, Hin, Win, C, Ho, Wo, vp(x), vp(addend), None, vp(hi1), None)
    call("adb_upsample2x_nhwc", B, Hin, Win, C, Ho, Wo, vp(x), vp(addend), vp(y1), None, None)
    ref, bnd = upsample_reference(x, Ho, Wo, addend)
    check(f"upsample {B}x{Hin}x{Win}x{C} -> {Ho}x{Wo} add={add}", (y.double() - ref).abs(), bnd)
    assert_split(hi, lo, y, "upsample")
    assert torch.equal(hi1, hi) and torch.equal(y1, y)


# ---- MASt3R head epilogue --------------------------------------------------------------------------------------------
def head_inputs(B, H, W, ld_lf, dev, seed):
    """pts [B,H,W,4]: by pixel index mod 6, xyz = 0, |xyz| = 1e-10, |xyz| = 79.5, |xyz| = 100 (expm1 overflows; every
    component is at least 0.13 |xyz|, so each overflows too), and N(0, 2^2) twice; conf logits +80, -80 or N(0,1).
    lf [B*S, ld_lf]: descriptor norms spread over 1e-3 .. 1e3 per pixel; NaN in the pad columns past 25*256."""
    g = gen(seed, dev)
    S = (H // 16) * (W // 16)
    pts = torch.randn(B, H, W, 4, generator=g, device=dev) * 2
    k = torch.arange(B * H * W, device=dev).view(B, H, W) % 6
    unit = F.normalize(0.3 + torch.rand(B, H, W, 3, generator=g, device=dev), dim=-1) * torch.sign(pts[..., :3] + 1e-3)
    xyz = pts[..., :3]
    xyz[k == 0] = 0.0
    for kk, r in ((1, 1e-10), (2, 79.5), (3, 100.0)):
        xyz[k == kk] = r * unit[k == kk]
    w = pts[..., 3]
    kc = torch.arange(B * H * W, device=dev).view(B, H, W) % 4
    w[kc == 0], w[kc == 1] = 80.0, -80.0
    lf = torch.randn(B * S, ld_lf, generator=g, device=dev)
    lf[:, 25 * 256:] = math.nan
    scale = 10.0 ** (6 * torch.rand(B * S, 1, 256, generator=g, device=dev) - 3)
    lf[:, :24 * 256].view(B * S, 24, 256).mul_(scale)
    return pts, lf


def head_reference(pts, lf, H, W):
    """float64 pixel_shuffle(16) + postprocess.  Bounds:
      pts3d: |xyz| is within 2.5u (3 squares, sqrtf); expm1(d) amplifies that by kappa = d e^d / expm1(d); expm1f 1 ulp
             (2u), max(d, 1e-8) 2.5u, / and * u each: (2.5 kappa + 6.5) u |pts3d|;
      conf, desc_conf: expf 2 ulp (4u), + 1 (u): 4u e^c + u |conf|;
      desc: 24 squares summed (24u), sqrtf (half of it + u), 1/ (u), * (u): 15u |desc|."""
    B = pts.shape[0]
    S = (H // 16) * (W // 16)
    l = F.pixel_shuffle(lf[:, :25 * 256].double().view(B, S, -1).transpose(-1, -2).reshape(B, -1, H // 16, W // 16), 16)
    l = l.permute(0, 2, 3, 1)
    p64 = pts.double()
    xyz = p64[..., :3]
    d = xyz.norm(dim=-1, keepdim=True)
    em = torch.expm1(d)
    p3 = xyz / d.clamp(min=1e-8) * em
    kappa = torch.where(d > 1e-30, d * torch.exp(d) / em.clamp(min=1e-300), torch.ones_like(d))
    e = p64[..., 3].exp()
    desc = l[..., :24]
    desc = desc / desc.norm(dim=-1, keepdim=True)
    q = l[..., 24].exp()
    return dict(pts3d=(p3, (2.5 * kappa + 6.5) * U * p3.abs() + 1e-38), conf=(1 + e, 4 * U * e + U * (1 + e)),
                desc=(desc, 15 * U * desc.abs() + 1e-38), desc_conf=(q, 4 * U * q + 1e-38))


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W", [(2, 48, 80), (1, 64, 32), (4, 512, 544)])
def test_head_postprocess(cuda, B, H, W):
    """adb_head_postprocess per element against float64 (bound: head_reference), H != W so a transposed token index
    fails, ld_lf = 25*256 + 12 with NaN pad columns that must not be read, xyz = 0 giving exactly 0 (not NaN), and the
    overflow pixels giving the same inf as the fp32 reference.  4 x 512 x 544 is 1.11M threads, past the grid cap."""
    from artdeco_b200.mast3r import ops  # noqa: F401  (registers the signature)
    ld_lf = 25 * 256 + 12
    pts, lf = head_inputs(B, H, W, ld_lf, cuda, H + W)
    out = {k: torch.full(s, SENT, device=cuda) for k, s in
           (("pts3d", (B, H, W, 3)), ("conf", (B, H, W)), ("desc", (B, H, W, 24)), ("desc_conf", (B, H, W)))}
    call("adb_head_postprocess", B, H, W, vp(pts), vp(lf), ld_lf, 24, vp(out["pts3d"]), vp(out["conf"]), vp(out["desc"]),
         vp(out["desc_conf"]))
    refs = head_reference(pts, lf, H, W)
    for k, (ref, bnd) in refs.items():
        ref32 = ref.float()
        inf = torch.isinf(ref32)
        got = out[k]
        assert torch.equal(got[inf], ref32[inf]), f"{k}: overflow must give the fp32 reference's inf"
        check(f"head_postprocess {k} {B}x{H}x{W}", (got[~inf].double() - ref[~inf]).abs(), bnd[~inf])
    k6 = torch.arange(B * H * W, device=cuda).view(B, H, W) % 6
    assert (out["pts3d"][k6 == 0] == 0).all(), "xyz = 0 must give 0"
    assert torch.isinf(out["pts3d"][k6 == 3]).all()


# ---- curope in place -------------------------------------------------------------------------------------------------
def rope2d_reference(t, pos, base, F0):
    """float64 curope on tokens [B, N, H, D]: head = [u_y | v_y | u_x | v_x] (Q = D/4 each), pair i rotated by
    pos * F0 / base^(i/Q).  Bound: the fp32 angle is within (ln(base) + 10) u |angle| (i/Q u, powf 4 ulp, / and * u);
    sincosf 2 ulp (4u absolute); u c - v s adds 2u (|u c| + |v s|):
    (|u| + |v|) ((ln base + 10) u |angle| + 4u) + 2u (|u c| + |v s|)."""
    D = t.shape[-1]
    Q = D // 4
    inv = F0 / base ** (torch.arange(Q, dtype=F64, device=t.device) / Q)
    out, bnd = t.clone(), torch.zeros_like(t)
    for ax in (0, 1):
        ang = pos[..., ax].double()[:, :, None, None] * inv          # [B, N, 1, Q]
        c, s = torch.cos(ang), torch.sin(ang)
        u, v = t[..., 2 * Q * ax:2 * Q * ax + Q], t[..., 2 * Q * ax + Q:2 * Q * ax + 2 * Q]
        out[..., 2 * Q * ax:2 * Q * ax + Q] = u * c - v * s
        out[..., 2 * Q * ax + Q:2 * Q * ax + 2 * Q] = v * c + u * s
        e = (u.abs() + v.abs()) * ((math.log(base) + 10) * U * ang.abs() + 4 * U)
        bnd[..., 2 * Q * ax:2 * Q * ax + Q] = e + 2 * U * ((u * c).abs() + (v * s).abs())
        bnd[..., 2 * Q * ax + Q:2 * Q * ax + 2 * Q] = e + 2 * U * ((v * c).abs() + (u * s).abs())
    return out, bnd + 1e-30


@pytest.mark.gpu
@pytest.mark.parametrize("F0", [1.0, -1.0])
@pytest.mark.parametrize("H", [1, 3, 17])
@pytest.mark.parametrize("D", [4, 12, 64, 512])
def test_rope2d_inplace(cuda, D, H, F0):
    """adb_rope2d_inplace per element against float64 (bound: rope2d_reference) on a strided view: tokens
    [B, N, H, D] inside a [B, N, H + 1, D] buffer whose last head is a canary.  D = 64 with H = 17 and D = 512 with
    H = 3 run the per-thread head loop more than once (256 / (D/2) heads per pass)."""
    B, N, base = 2, 7, 100.0
    gd = gen(D * 10 + H, cuda)
    buf = torch.randn(B, N, H + 1, D, generator=gd, device=cuda)
    buf[:, :, H] = SENT
    before = buf.clone()
    pos = torch.randint(0, 200, (B, N, 2), generator=gd, device=cuda)
    tok = buf[:, :, :H]
    call("adb_rope2d_inplace", B, N, H, D, tok.stride(0), tok.stride(1), vp(tok), vp(pos), base, F0)
    ref, bnd = rope2d_reference(before[:, :, :H].double(), pos, base, F0)
    check(f"rope2d D={D} H={H} F0={F0:g}", (tok.double() - ref).abs(), bnd)
    assert (buf[:, :, H] == SENT).all(), "the head past H was written"


# ---- Pi3 -------------------------------------------------------------------------------------------------------------
PI3_MEAN, PI3_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


@pytest.mark.gpu
@pytest.mark.parametrize("BN,H,W", [(1, 14, 28), (2, 42, 70), (24, 392, 518)])
def test_pi3_patch14(cuda, BN, H, W):
    """adb_pi3_patch14 bitwise against torch fp32 (img - mean) / std unfolded 14x14 in (c, ky, kx) order, with columns
    588..591 exactly 0.  24 frames of 392 x 518 are 14.7M elements, past the grid cap."""
    img = torch.rand(BN, 3, H, W, generator=gen(BN, cuda), device=cuda)
    n = BN * (H // 14) * (W // 14)
    hi, lo, hi1 = (torch.full((n, 592), SENT, dtype=BF16, device=cuda) for _ in range(3))
    call("adb_pi3_patch14", BN, H, W, vp(img), vp(hi), vp(lo))
    call("adb_pi3_patch14", BN, H, W, vp(img), vp(hi1), None)
    mean = torch.tensor(PI3_MEAN, device=cuda).view(1, 3, 1, 1)
    std = torch.tensor(PI3_STD, device=cuda).view(1, 3, 1, 1)
    a = torch.zeros(n, 592, device=cuda)
    a[:, :588] = F.unfold((img - mean) / std, 14, stride=14).transpose(1, 2).reshape(n, 588)
    del img
    assert_split(hi, lo, a, f"pi3_patch14 {BN}x{H}x{W}")
    assert torch.equal(hi1, hi)


@pytest.mark.gpu
@pytest.mark.parametrize("BN,n,C", [(2, 1, 4), (2, 1, 1024), (3, 7, 4), (24, 1036, 1024)])
def test_pi3_tokens(cuda, BN, n, C):
    """adb_pi3_tokens bitwise against torch fp32: [cls + pos0, 4 registers, patch + pos[1..n]].  BN = 24, n = 1036,
    C = 1024 is 6.4M float4 threads, past the grid cap."""
    gd = gen(C + n, cuda)
    patch = torch.randn(BN * n, C, generator=gd, device=cuda)
    cls, reg = torch.randn(C, generator=gd, device=cuda), torch.randn(4, C, generator=gd, device=cuda)
    pos = torch.randn(1 + n, C, generator=gd, device=cuda)
    x = torch.full((BN, n + 5, C), SENT, device=cuda)
    call("adb_pi3_tokens", BN, n, C, vp(patch), vp(cls), vp(reg), vp(pos), vp(x))
    ref = torch.cat([(cls + pos[0]).expand(BN, 1, C), reg.expand(BN, 4, C), patch.view(BN, n, C) + pos[1:]], 1)
    assert torch.equal(x, ref)


def pi3_point_reference(pts, cf, pose, BN, H, W, skip, transposed=False):
    """float64 pixel shuffle(14) + local points (x e^z, y e^z, e^z) + pose; conf gathered.  Bound: e^z by expf 2 ulp
    (4u), x e^z one more (5u), the 3x4 pose product at most 3 roundings (3u):
    8u (sum_a |P_a l_a|) + 3u |t|.  transposed=True is the bug model: pixel (Y, X) of a patch read from (X, Y)."""
    gw, hw = W // 14, skip + (H // 14) * (W // 14)
    dev = pts.device
    Y = torch.arange(H, device=dev)[:, None].expand(H, W)
    X = torch.arange(W, device=dev)[None, :].expand(H, W)
    row = (torch.arange(BN, device=dev)[:, None, None] * hw + skip + (Y // 14) * gw + X // 14)
    j = (X % 14) * 14 + Y % 14 if transposed else (Y % 14) * 14 + X % 14
    j = j.expand_as(row)
    f = pts.double()
    z = torch.exp(f[row, 392 + j])
    lp = torch.stack([f[row, j] * z, f[row, 196 + j] * z, z], -1)
    P = pose.double()[:, None, None]
    R, t = P[..., :3, :3], P[..., :3, 3]
    points = (R @ lp[..., None])[..., 0] + t
    bnd_l = torch.stack([5 * U * lp[..., 0].abs(), 5 * U * lp[..., 1].abs(), 4 * U * z], -1)
    bnd_p = 8 * U * (R.abs() @ lp.abs()[..., None])[..., 0] + 3 * U * t.abs()
    return points, bnd_p + 1e-38, lp, bnd_l + 1e-38, cf[row, j]


def pi3_pose(BN, g, dev):
    q, _ = torch.linalg.qr(torch.randn(BN, 3, 3, generator=g, dtype=F64))
    q = q * torch.linalg.det(q)[:, None, None]
    P = torch.eye(4, dtype=F64).repeat(BN, 1, 1)
    P[:, :3, :3] = q
    P[:, :3, 3] = 3 * torch.randn(BN, 3, generator=g, dtype=F64)
    return P.float().to(dev)


@pytest.mark.gpu
@pytest.mark.parametrize("BN,H,W,skip", [(2, 42, 70, 0), (2, 42, 70, 5), (1, 56, 28, 5), (3, 392, 518, 5)])
def test_pi3_point_head(cuda, BN, H, W, skip):
    """adb_pi3_point_head per element against float64 (bound: pi3_point_reference), H != W, a pose with rotation and
    translation, depth logits of +-30, and conf copied bitwise.  3 x 392 x 518 is 609k pixels, past the grid cap."""
    hw = skip + (H // 14) * (W // 14)
    gd = gen(H + skip, cuda)
    pts = torch.randn(BN * hw, 588, generator=gd, device=cuda)
    zl = pts[:, 392:]
    zl[:, ::7] = 30.0
    zl[:, 3::7] = -30.0
    cf = torch.randn(BN * hw, 196, generator=gd, device=cuda)
    pose = pi3_pose(BN, gen(BN + skip), cuda)
    outs = [torch.full((BN, H, W, 3), SENT, device=cuda) for _ in range(2)] + [torch.full((BN, H, W), SENT, device=cuda)]
    call("adb_pi3_point_head", BN, H, W, hw, skip, vp(pts), vp(cf), vp(pose), *(vp(o) for o in outs))
    points, bp, lp, bl, conf = pi3_point_reference(pts, cf, pose, BN, H, W, skip)
    check(f"pi3_point_head local {BN}x{H}x{W} skip={skip}", (outs[1].double() - lp).abs(), bl)
    check(f"pi3_point_head points {BN}x{H}x{W} skip={skip}", (outs[0].double() - points).abs(), bp)
    assert torch.equal(outs[2], conf)


def camera_tail_reference(feat, w, BN, hw, skip):
    """float64 average pool of rows skip..hw-1, relu(W0 f + b0), relu(W2 . + b2), fc_t, fc_rot, with a running error
    bound over the kernel's summation order: a sequential sum rounds each partial sum s_k once (u |s_k|), a product
    that is not fused into it once more (u |x_k w_k|).  The pool sums the n = hw - skip rows in order, then divides (u);
    each layer starts from its bias and adds the 512 products in k order, plus |W| times the bound of its input; relu
    is 1-Lipschitz, and exact where the pre-activation is negative by more than its bound."""
    w = {k: v.double() for k, v in w.items()}
    f32 = feat.double().view(BN, hw, 512)[:, skip:]
    n = hw - skip
    f = f32.mean(1)
    df = U * f32.cumsum(1).abs().sum(1) / n + U * f.abs()

    def layer(x, dx, wt, b):       # wt [in, out]
        terms = x[:, :, None] * wt[None]
        acc = b + terms.cumsum(1)
        return acc[:, -1], U * (acc.abs().sum(1) + terms.abs().sum(1)) + dx @ wt.abs()
    def relu(a, da):
        return a.clamp(min=0), torch.where(a + da < 0, torch.zeros_like(da), da)
    g, dg = relu(*layer(f, df, w["w0t"], w["b0"]))
    h, dh = relu(*layer(g, dg, w["w2t"], w["b2"]))
    t, dt = layer(h, dh, w["wt"].T, w["bt"])
    r, dr = layer(h, dh, w["wr"].T, w["br"])
    return r, dr + 1e-38, t, dt + 1e-38


@pytest.mark.gpu
@pytest.mark.parametrize("BN,hw,skip,dead", [(2, 6, 5, False), (2, 1041, 5, False), (3, 1, 0, False), (2, 40, 5, True)])
def test_pi3_camera_tail(cuda, BN, hw, skip, dead):
    """adb_pi3_camera_tail per element against float64 (bound: camera_tail_reference) with hw - skip = 1 and 1036
    tokens pooled.  Features, MLP weights and biases are non-negative and fc_t / fc_rot rows carry one random sign, so
    every sum adds coherently: the worst-case bound is then within a small factor of the real rounding (about 1e-4 of
    each output), and dropping one input channel or a layer's bias lands far outside it.  dead=True makes every
    first-layer pre-activation negative, so the output is W2-free: relu(b2) through fc_t / fc_rot."""
    gd = gen(hw + BN, cuda)

    def rnd(*shape):
        return torch.rand(*shape, generator=gd, device=cuda)
    feat = rnd(BN * hw, 512)
    w = dict(w0t=rnd(512, 512) / 256, b0=rnd(512), w2t=rnd(512, 512) / 256, b2=rnd(512),
             wt=rnd(3, 512) / 256 * torch.randn(3, 1, generator=gd, device=cuda).sign(), bt=rnd(3) - 0.5,
             wr=rnd(9, 512) / 256 * torch.randn(9, 1, generator=gd, device=cuda).sign(), br=rnd(9) - 0.5)
    if dead:
        w["b0"] = -1e3 - w["b0"]
    rot, trans = torch.full((BN, 9), SENT, device=cuda), torch.full((BN, 3), SENT, device=cuda)
    call("adb_pi3_camera_tail", BN, hw, skip, vp(feat), *(vp(w[k]) for k in ("w0t", "b0", "w2t", "b2", "wt", "bt", "wr", "br")),
         vp(rot), vp(trans))
    r, dr, t, dt = camera_tail_reference(feat, w, BN, hw, skip)
    check(f"pi3_camera_tail rot BN={BN} hw={hw} skip={skip} dead={dead}", (rot.double() - r).abs(), dr)
    check(f"pi3_camera_tail trans BN={BN} hw={hw} skip={skip} dead={dead}", (trans.double() - t).abs(), dt)
    if dead:
        f = feat.double().view(BN, hw, 512)[:, skip:].mean(1)
        assert (f @ w["w0t"].double() + w["b0"].double() < 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("N,Hi,Wi,Ho,Wo", [(2, 100, 150, 392, 518), (2, 600, 900, 392, 518), (1, 1, 37, 28, 56),
                                           (1, 45, 1, 14, 70), (1, 1, 1, 14, 14), (3, 333, 250, 126, 98)])
def test_pi3_window_input(cuda, N, Hi, Wi, Ho, Wo):
    """adb_pi3_window_input against F.interpolate(clamp(img/2 + 1/2, 0, 1), bilinear, align_corners=False) on the
    device, up and down at non-integer ratios and from one row / one column.  Both evaluate the same fp32 expression;
    they may contract the source coordinate differently (u |coord| each, and the output moves at most 1 per unit of
    coordinate since values lie in [0, 1]) and round the blend differently (6u each side):
    bound 12u + 2u (|h_src| + |w_src| + 1).  2 frames at 392 x 518 are 1.2M threads, past the grid cap."""
    img = torch.rand(N, 3, Hi, Wi, generator=gen(Hi * Wi, cuda), device=cuda) * 2.4 - 1.2   # some values clamp
    out = torch.full((N, 3, Ho, Wo), SENT, device=cuda)
    call("adb_pi3_window_input", N, Hi, Wi, vp(img), Ho, Wo, vp(out))
    ref = F.interpolate((img * 0.5 + 0.5).clamp(0, 1), size=(Ho, Wo), mode="bilinear", align_corners=False)
    hs = (Hi / Ho * (torch.arange(Ho, device=cuda, dtype=F64) + 0.5) - 0.5).clamp(min=0)[:, None]
    ws = (Wi / Wo * (torch.arange(Wo, device=cuda, dtype=F64) + 0.5) - 0.5).clamp(min=0)[None, :]
    check(f"pi3_window_input {Hi}x{Wi} -> {Ho}x{Wo}", (out.double() - ref.double()).abs(),
          (12 * U + 2 * U * (hs + ws + 1)).expand(N, 3, Ho, Wo))


# ---- CPU part: refusals and bug models -------------------------------------------------------------------------------
def test_companion_entry_points_refuse_misaligned_pointers_and_short_rows():
    """The checks run before any launch, so fake pointers (never dereferenced) are enough."""
    from artdeco_b200 import _lib
    import artdeco_b200  # noqa: F401  (registers every signature)
    L = _lib.lib()
    f = ctypes.c_float

    def refused(rc, needle):
        msg = L.adb_last_error()
        return rc == 1 and msg is not None and needle in msg.decode()

    p = ctypes.c_void_p(256)            # 256-byte aligned, never dereferenced
    a4 = ctypes.c_void_p(260)           # 4-byte aligned only
    a8 = ctypes.c_void_p(264)           # 8-byte aligned only
    # adb_layernorm: float4 on x, gamma, beta, y; 128-bit stores of y_hi, y_lo
    for args in ((a4, p, p, p, p, p), (p, a4, p, p, p, p), (p, p, a8, p, p, p), (p, p, p, a8, p, p),
                 (p, p, p, None, a8, None), (p, p, p, p, p, a8)):
        x, g, b, y, yh, yl = args
        assert refused(L.adb_layernorm(13, 768, x, g, b, f(1e-6), y, yh, yl, None), "16-byte aligned"), args
    # adb_rope_heads: the row must hold col0 + h*64 columns; 128-bit stores of hi / lo; float2 table reads
    assert refused(L.adb_rope_heads(2, 50, 4, 768, 516, p, p, p, 64, 0, 56, p, p, None), "ld >= col0 + h*64")
    assert refused(L.adb_rope_heads(2, 50, 4, 2 * 256, 300, p, None, None, 64, 2, 56, p, p, None), "ld >= col0 + h*64")
    assert refused(L.adb_rope_heads(2, 50, 4, 768, -4, p, None, None, 64, 1, 56, p, p, None), "ld >= col0 + h*64")
    for mode, (hi, lo, tb) in ((0, (a8, p, p)), (1, (p, a8, p)), (2, (a8, None, p)), (0, (p, p, a4))):
        assert refused(L.adb_rope_heads(2, 50, 4, 768, 0, p, p, tb, 64, mode, 56, hi, lo, None), "aligned"), (mode, hi, lo)
    # adb_upsample2x_nhwc: float4 on x, addend, y; 64-bit stores of hi / lo
    for x, ad, y, hi, lo in ((a8, None, p, None, None), (p, a8, p, None, None), (p, None, a8, None, None),
                             (p, None, None, a4, None), (p, None, None, p, a4)):
        assert refused(L.adb_upsample2x_nhwc(1, 8, 8, 64, 16, 16, x, ad, y, hi, lo, None), "aligned")
    # adb_head_postprocess: float4 on pts and desc
    assert refused(L.adb_head_postprocess(1, 32, 32, a8, p, 6400, 24, p, p, p, p, None), "aligned")
    assert refused(L.adb_head_postprocess(1, 32, 32, p, p, 6400, 24, p, p, a8, p, None), "aligned")
    assert refused(L.adb_head_postprocess(1, 32, 32, p, ctypes.c_void_p(258), 6400, 24, p, p, p, p, None), "aligned")


def test_layernorm_one_pass_variance_bug_is_far_outside_the_bound():
    """E[x^2] - E[x]^2 in fp32 on the offset rows (mean/std 1e4) loses the variance to cancellation."""
    for C in (256, 1032):
        g = gen(C)
        x = ln_rows(C, 1e-6, g)[-3:]
        gamma, beta = torch.ones(C), torch.zeros(C)
        ref, bnd = ln_reference(x, gamma, beta, 1e-6)
        bug, _ = ln_reference(x, gamma, beta, 1e-6, one_pass=True)
        assert ratio((bug - ref).abs(), bnd) >= 10, C


def test_softmax_dropped_partial_chunk_is_far_outside_the_bound():
    """A kernel that drops the last partial 128-column chunk (fast kernels) or 32-column pass (generic kernel)."""
    for L, chunk in ((132, 128), (1028, 128), (2052, 32), (5000, 32)):
        x = softmax_rows(L, gen(L))[:6]
        ref, bnd = softmax_reference(x)
        bug, _ = softmax_reference(x, drop_tail=L // chunk * chunk)
        assert ratio((bug - ref).abs(), bnd) >= 10, L


def test_rope_bug_models_are_far_outside_the_bound():
    """Partner dimension lane ^ 8 instead of ^ 16, and the y and x halves rotated by each other's position."""
    from artdeco_b200.mast3r import ops
    g = gen(5)
    B, N, h, n_pos = 2, 65, 3, 64
    table = ops.rope_table(n_pos, torch.device("cpu"))
    pos = rope_positions(B, N, n_pos, g)
    xs = torch.randn(B, h, N, 64, generator=g, dtype=F64).float().double()
    ref, bnd = rope_heads_reference(xs, pos, table)
    for kw in (dict(partner=8), dict(swap=True)):
        bug, _ = rope_heads_reference(xs, pos, table, **kw)
        assert ratio((bug - ref).abs(), bnd) >= 10, kw


def test_transpose_pad_and_im2col_bug_models_are_caught():
    """An unzeroed transpose pad (the shared tile's stale rows, here the next tokens' values) is not all zero; im2col with
    py and px swapped is not bitwise the unfold order."""
    g = gen(6)
    x = torch.randn(2, 70, 64, generator=g)
    N, Npad = 61, 72
    stale = x[:, :Npad].transpose(-1, -2)                 # what unguarded loads past N would leave in the tile
    assert stale[..., N:].any()
    img = torch.randn(2, 3, 32, 48, generator=g)
    ref = im2col_reference(img)
    bug = im2col_reference(img, swap=True)
    assert (bug != ref).float().mean() > 0.9


def test_point_head_transposed_pixel_shuffle_is_far_outside_the_bound():
    BN, H, W, skip = 2, 42, 70, 5
    hw = skip + (H // 14) * (W // 14)
    g = gen(7)
    pts, cf = torch.randn(BN * hw, 588, generator=g), torch.randn(BN * hw, 196, generator=g)
    pose = pi3_pose(BN, g, "cpu")
    points, bp, lp, bl, _ = pi3_point_reference(pts, cf, pose, BN, H, W, skip)
    bpoints, _, blp, _, _ = pi3_point_reference(pts, cf, pose, BN, H, W, skip, transposed=True)
    assert ratio((blp - lp).abs(), bl) >= 10 and ratio((bpoints - points).abs(), bp) >= 10


def test_upsample_half_pixel_coordinates_are_far_outside_the_bound():
    for B, Hin, Win, C, Ho, Wo in ((2, 9, 13, 4, 17, 25), (1, 6, 1, 8, 12, 2), (1, 16, 16, 4, 32, 32)):
        x = torch.randn(B, Hin, Win, C, generator=gen(Hin))
        ref, bnd = upsample_reference(x, Ho, Wo)
        bug, _ = upsample_reference(x, Ho, Wo, align_corners=False)
        assert ratio((bug - ref).abs(), bnd) >= 10, (Hin, Win)

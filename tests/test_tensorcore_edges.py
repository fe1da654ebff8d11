"""The tensor-core kernels at their edges: csrc/gemm_tc.cu (adb_gemm_bf16, adb_gemm_bf16_rope, adb_conv3x3_bf16) and
csrc/attn_tc.cu (adb_attention_bf16), checked against references built from the very bf16 (hi, lo) operands the
kernels take.

* Exact-operand references: the fp64 sum of the products a kernel documents -- single pass A_hi B_hi^T, bf16x3
  A_hi B_hi^T + A_hi B_lo^T + A_lo B_hi^T (not (A_hi + A_lo)(B_hi + B_lo)^T).  What remains is accumulation error, bounded
  PER ELEMENT by tol * (the same sum over absolute values), so an error confined to a tail tile or a small row is not
  hidden by the largest element.  Operands are non-negative with a random sign per row, so every term of a dot product
  adds coherently: dropping any one of them (a lo term, the last partial k-block, a channel chunk, a border tap) moves
  the result far more than the tolerance.  Every such test computes that bug in Python at its own shape and asserts it
  lands at least 10x the tolerance away ("discrimination").
* Bit-exact structure: selection-matrix GEMMs, one-hot-tap convolutions and one-hot attention rows reduce every dot
  product to one non-zero term, so the result is a gather of the operand that fp32 represents exactly: an addressing
  error shows as a wrong value, not as noise.
* Canaries: outputs live inside larger buffers filled with a finite sentinel (rows past M or the last pixel, padding
  columns when ld > N, elements past the end); everything outside the written region must be untouched.
* True fp64: fp32 inputs -> bf16 split -> kernel against the fp64 result of the fp32 inputs keeps the 2e-5 contract of
  tests/test_gemm.py.

Set ADB_TC_REPORT=<file.json> to write the largest normalised error, the tolerance and the smallest bug margin of each
test group.  The tolerances below were set from a run on an H100 80GB HBM3 (700 W power limit) with at least 2x headroom
over the measured maxima quoted beside them; the whole file takes about 15 s there.
"""
import ctypes
import json
import math
import os

import pytest
import torch
import torch.nn.functional as F

from helpers import rel_err

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
LOG2E = 1.4426950408889634
SENT = -768.0        # canary: finite, exact in fp32 and bf16
GUARD = 256          # sentinel elements before and after every output (1 KB of fp32: keeps 32-byte alignment)
PADV = 1000.0        # finite, non-zero value in Vt's padding columns: the key mask, not zero padding, must hide them
SPLIT = 2.0 ** -16   # hi + lo of an fp32 value: relative rounding of the (hi, lo) output split

# Per-element normalised tolerances (|out - ref| / bound), indexed by x3; "max" is the largest value measured over the
# whole file on an H100 80GB HBM3 (700 W power limit).
TOL_GEMM = {True: 2e-5, False: 3e-6}          # max 8.4e-6 (x3) / 9.9e-7 (single pass): fp32 accumulation in the tensor core
TOL_CONV = {True: 2e-5, False: 3e-6}          # max 8.0e-6 / 8.9e-7 (K up to 9 x 768 at the DPT head's shapes)
# Attention, x3: max 1.8e-5 (output split 2^-17 + P split).  Single pass holds P as bf16 hi only: where the kernel's fp32 p
# and the reference's land on opposite sides of a bf16 rounding boundary that weight differs by 2^-8: max 5.1e-4.
TOL_ATTN = {True: 4e-5, False: 1.5e-3}
TOL_ATTN_LARGE = {8.0: 5e-5, 32.0: 1e-4}      # bf16x3 exact-operand, logit std 8 / 32 after the scale: max 2.2e-5 / 3.3e-5
TOL_ATTN_TRUE = {8.0: 2e-4, 32.0: 6e-4}       # bf16x3 against fp64 of the fp32 inputs, logit std 8 / 32: max 8.1e-5 / 2.5e-4
# One-hot attention rows: p of the addressed key is 1 up to the fp32 rounding of the row shift, so O = V[pi(i)] to the
# (hi, lo) output split in both modes (single pass: pass 1 and pass 2 compute the same hi x hi score).
ONE_HOT_REL = 2.0 ** -14

_REPORT: dict = {}


def _note(group, key, value, pick):
    r = _REPORT.setdefault(group, {})
    r[key] = value if key not in r else pick(r[key], value)


def check(group, err, tol):
    _note(group, "max_err", err, max)
    _note(group, "tol", tol, max)
    assert err <= tol, f"{group}: normalised error {err:.3e} > tolerance {tol:.1e}"


def discriminates(group, bug, bug_err, tol):
    """The Python model of `bug` must land at least 10x the tolerance away from the reference."""
    _note(group, "min_bug_margin", bug_err / tol, min)
    assert bug_err >= 10 * tol, f"{group}: bug model '{bug}' differs by only {bug_err:.3e} (tolerance {tol:.1e})"


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    path = os.environ.get("ADB_TC_REPORT")
    if path and _REPORT:
        with open(path, "w") as f:
            json.dump(_REPORT, f, indent=1, sort_keys=True)


def nerr(out, ref, bound):
    """max |out - ref| / bound over all elements (inf if anything is NaN)."""
    if ref.numel() == 0:
        return 0.0
    d = ((out.to(F64) - ref.to(F64)).abs() / bound.to(F64).clamp_min(1e-300)).max().item()
    return math.inf if math.isnan(d) else d


# ---------------------------------------------------------------------------------------------------------------------
# operands and references (device-agnostic: the CPU tests below run them too)

def gen(dev, seed):
    return torch.Generator(device=dev).manual_seed(seed)


def pos_operand(shape, g, x3, sign_dim=None):
    """bf16 hi in [0.1, 1) and lo in [0, 2^-8 hi), times a random sign per index of `sign_dim`; lo is None unless x3.
    The generator is consumed the same way in both modes, so hi does not depend on x3."""
    dev = g.device
    hi = (0.1 + 0.9 * torch.rand(shape, generator=g, device=dev)).to(BF16)
    lo = (torch.rand(shape, generator=g, device=dev) * 2.0 ** -8 * hi.float()).to(BF16)
    if sign_dim is not None:
        sshape = [1] * len(shape)
        sshape[sign_dim] = shape[sign_dim]
        sg = torch.where(torch.rand(sshape, generator=g, device=dev) < 0.5, -1.0, 1.0).to(BF16)
        hi, lo = hi * sg, lo * sg
    return hi, (lo if x3 else None)


def split(x, x3=True):
    """fp32 -> bf16 (hi, lo) with round-to-nearest, as adb_split_bf16 does."""
    hi = x.to(BF16)
    return hi, ((x - hi.float()).to(BF16) if x3 else None)


def joined(hi, lo):
    """hi + lo in fp32: exact when (hi, lo) is the split of an fp32 value (the pair then spans at most 24 bits)."""
    return hi.float() + lo.float() if lo is not None else hi.float()


def join64(hi, lo):
    """hi + lo in fp64: exact for any pair (pos_operand's lo is not a rounding residual of hi)."""
    return hi.double() + lo.double() if lo is not None else hi.double()


def gemm_exact_ref(ah, al, bh, bl):
    """fp64 sum of the products the kernel forms from these bf16 operands ([.., M, K] x [.., N, K]^T), and the same
    sum over absolute values (the per-element error scale)."""
    ah, bh = ah.to(F64), bh.to(F64)
    r, b = ah @ bh.mT, ah.abs() @ bh.abs().mT
    if al is not None:
        al, bl = al.to(F64), bl.to(F64)
        r = r + ah @ bl.mT + al @ bh.mT
        b = b + ah.abs() @ bl.abs().mT + al.abs() @ bh.abs().mT
    return r, b


def selection_indices(M, K, g):
    """One column index per row of a selection matrix: every k in [0, K) when M >= K, otherwise a random subset that
    holds K - 1 (the last, possibly partial, k-block) and 0."""
    p = torch.randperm(K, generator=g, device=g.device)
    if M >= K:
        return p[torch.arange(M, device=g.device) % K]
    idx = p[:M].clone()
    idx[-1] = K - 1
    if M > 1:
        idx[0] = 0
    return idx


def selection_matrix(idx, K):
    a = torch.zeros(idx.numel(), K, dtype=BF16, device=idx.device)
    a[torch.arange(idx.numel(), device=idx.device), idx] = 1.0
    return a


def conv_tile(W):
    """The kernel's pixel tile: the widest power-of-two row segment wb <= W (at least 8) and hb = 128 / wb rows."""
    wb = 128
    while wb > W and wb > 8:
        wb //= 2
    return wb, 128 // wb


def conv64(x, w, y0=0, y1=None, wrap=False):
    """fp64 3x3 / stride 1 / pad 1 convolution of NHWC x with w [Cout, Cin, 3, 3], output rows [y0, y1) only (NHWC).
    wrap=True pads circularly instead of with zeros (a bug model)."""
    H = x.shape[1]
    y1 = H if y1 is None else y1
    xn = x.to(F64).permute(0, 3, 1, 2)
    xp = F.pad(xn, (1, 1, 1, 1), mode="circular") if wrap else F.pad(xn, (1, 1, 1, 1))
    return F.conv2d(xp[:, :, y0:y1 + 2], w.to(F64)).permute(0, 2, 3, 1)


def conv_exact_ref(xh, xl, wh, wl, y0=0, y1=None, wrap=False):
    r = conv64(xh, wh, y0, y1, wrap)
    b = conv64(xh.abs(), wh.abs(), y0, y1)
    if xl is not None:
        r = r + conv64(xh, wl, y0, y1, wrap) + conv64(xl, wh, y0, y1, wrap)
        b = b + conv64(xh.abs(), wl.abs(), y0, y1) + conv64(xl.abs(), wh.abs(), y0, y1)
    return r, b


def one_hot_tap_weight(Cin, dev):
    """w [9 Cin, Cin, 3, 3]: output channels [t Cin, (t + 1) Cin) are the identity map on tap t = 3 ky + kx."""
    w = torch.zeros(9 * Cin, Cin, 3, 3, dtype=BF16, device=dev)
    c = torch.arange(Cin, device=dev)
    for t in range(9):
        w[t * Cin + c, c, t // 3, t % 3] = 1.0
    return w


def shifted_taps(x):
    """What one_hot_tap_weight computes: channel block t of the output is x shifted by (ky - 1, kx - 1), zero outside."""
    B, H, W, C = x.shape
    xp = F.pad(x.permute(0, 3, 1, 2), (1, 1, 1, 1)).permute(0, 2, 3, 1)
    return torch.cat([xp[:, t // 3:t // 3 + H, t % 3:t % 3 + W] for t in range(9)], -1)


def prep_conv_weight(w):
    """bf16 [Cout, Cin, 3, 3] -> the kernel's layout [Cout, 9 * Cin_pad], tap-major (ky, kx, ci), Cin zero-padded to 64."""
    Cout, Cin = w.shape[:2]
    cpad = (Cin + 63) // 64 * 64
    wp = torch.zeros(Cout, 3, 3, cpad, dtype=w.dtype, device=w.device)
    wp[..., :Cin] = w.permute(0, 2, 3, 1)
    return wp.reshape(Cout, 9 * cpad).contiguous()


def attn_scale_log2e(scale):
    """scale * log2(e) rounded as the kernel's host code rounds it (fp32 product of fp32 operands)."""
    s, l = torch.tensor(scale, dtype=F32), torch.tensor(LOG2E, dtype=F32)
    return float(s * l)


def attn_exact_ref(qh, ql, kh, kl, vh, vl, scale, x3, m_floor=None):
    """Fused attention from the kernel's own operands: scores from the bf16x3 products (hi x hi only when not x3), the
    row shift from the hi x hi scores as pass 1 takes it, p = exp2((s - m) scale log2e) rounded to fp32 and split into
    bf16 (hi, lo) as pass 2 packs it, O = (P_hi V_hi [+ P_hi V_lo + P_lo V_hi]) / sum(p).  q [BH, Nq, 64], k and v
    [BH, Nk, 64] (valid keys only).  Returns (O, bound) in fp64; bound = sum |P||V| / sum(p).
    m_floor (a bug model): the row shift is max(m, m_floor), e.g. 0 for a pass-1 max taken over zero-filled padded keys."""
    qh64, kh64 = qh.to(F64), kh.to(F64)
    s_hi = qh64 @ kh64.mT
    s = s_hi + (qh64 @ kl.to(F64).mT + ql.to(F64) @ kh64.mT) if x3 else s_hi
    c1 = attn_scale_log2e(scale)
    m = s_hi.amax(-1, keepdim=True).to(F32)
    if m_floor is not None:
        m = m.clamp_min(m_floor)
    c0 = (-m * c1).to(F64)
    p = torch.exp2(s * c1 + c0).to(F32)
    p = torch.where(p < 2.0 ** -126, torch.zeros_like(p), p)           # ex2.approx.ftz flushes denormals
    ph = p.to(BF16)
    pl = (p - ph.float()).to(BF16)
    l = p.to(F64).sum(-1, keepdim=True)
    ph64, vh64 = ph.to(F64), vh.to(F64)
    o = ph64 @ vh64
    b = ph64 @ vh64.abs()
    if x3:
        o = o + ph64 @ vl.to(F64) + pl.to(F64) @ vh64
        b = b + ph64 @ vl.to(F64).abs() + pl.to(F64) @ vh64.abs()
    return o / l, b / l


# ---------------------------------------------------------------------------------------------------------------------
# calls with guarded outputs

class Guarded:
    """An output of `n` elements inside a buffer of sentinels (GUARD before, GUARD after); `misalign` shifts the output
    by that many elements."""

    def __init__(self, n, dtype, dev, misalign=0):
        self.front = GUARD + misalign
        self.buf = torch.full((self.front + n + GUARD,), SENT, dtype=dtype, device=dev)
        self.out = self.buf[self.front:self.front + n]
        self.written = torch.zeros(self.buf.shape, dtype=torch.bool, device=dev)

    def take(self, offsets):
        """Values at element offsets (of the output) and mark them as the region the kernel may write."""
        self.written[self.front + offsets] = True
        return self.out[offsets]

    def take_all(self):
        return self.take(torch.arange(self.out.numel(), device=self.out.device))

    def assert_untouched(self, what):
        rest = self.buf[~self.written]
        bad = (rest != SENT).sum().item()
        assert bad == 0, f"{what}: {bad} sentinel elements outside the output were overwritten"


def matrix_offsets(Z, M, N, ld, s=0, zdiv=0, s2=0, dev=None):
    """Element offsets [Z, M, N] of the kernel's batched output addressing: z = z_outer * zdiv + z_inner lands at
    z_outer * s2 + z_inner * s (zdiv <= 0: z * s), row m at + m * ld."""
    z = torch.arange(Z, device=dev)
    zo, zi = (z // zdiv, z % zdiv) if zdiv > 0 else (torch.zeros_like(z), z)
    base = zo * s2 + zi * s
    return base[:, None, None] + torch.arange(M, device=dev)[None, :, None] * ld + torch.arange(N, device=dev)[None, None, :]


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def vector_store_path(ldd, ldr, ldo, ptrs, dbase=0, rbase=0, obase=0):
    """Whether gemm_tc.cu's epilogue may use its 256-bit row stores (its `vec_ok`): ldd and ldr multiples of 8, ldo of
    16 -- each checked even when that output is absent -- and D / residual / D_hi / D_lo (0 when absent) 32-byte
    aligned at every batch offset.  Column groups that end past N take the scalar path either way."""
    return (ldd % 8 == 0 and ldr % 8 == 0 and ldo % 16 == 0 and all(p % 32 == 0 for p in ptrs) and dbase % 8 == 0
            and rbase % 8 == 0 and obase % 16 == 0)


def run_gemm(ah, al, bh, bl, M, N, K, *, want_d=True, want_split=False, ldd=None, ldo=None, misalign=0, bias=None,
             residual=None, ldr=None, alpha=1.0, act=0, vector=None):
    """One unbatched adb_gemm_bf16 call into guarded outputs; returns (D [M, N] or None, (hi, lo) [M, N] or None).
    vector=True / False asserts that the call's layout selects / does not select the 256-bit store path."""
    from artdeco_b200.mast3r import ops
    dev = ah.device
    ldd = N if ldd is None else ldd
    ldo = N if ldo is None else ldo
    ldr = N if ldr is None else ldr
    gd = Guarded(M * ldd, F32, dev, misalign) if want_d else None
    gh = Guarded(M * ldo, BF16, dev, misalign) if want_split else None
    gl = Guarded(M * ldo, BF16, dev, misalign) if want_split else None
    if vector is not None:
        ptrs = [t.out.data_ptr() if t else 0 for t in (gd, gh, gl)]
        ptrs.append(residual.data_ptr() if residual is not None else 0)
        assert vector_store_path(ldd, ldr, ldo, ptrs) == vector, "the layout does not select the intended store path"
    ops.gemm(ops.Split(ah, al), ops.Split(bh, bl), M, N, K, out=gd.out if gd else None, ldd=ldd,
             out_split=ops.Split(gh.out, gl.out) if gh else None, ldo=ldo, bias=bias, residual=residual, ldr=ldr,
             alpha=alpha, act=act)
    torch.cuda.synchronize()
    d = sp = None
    if gd:
        d = gd.take(matrix_offsets(1, M, N, ldd, dev=dev)[0])
        gd.assert_untouched("D")
    if gh:
        off = matrix_offsets(1, M, N, ldo, dev=dev)[0]
        sp = (gh.take(off), gl.take(off))
        gh.assert_untouched("D_hi")
        gl.assert_untouched("D_lo")
    return d, sp


def run_conv(xh, xl, wh, wl, B, H, W, Cin, Cout, *, bias=None, residual=None, act=0, split_relu=0, want_d=True,
             want_split=False):
    """adb_conv3x3_bf16 into guarded NHWC outputs; w is [Cout, Cin, 3, 3] (prepared here)."""
    from artdeco_b200 import _lib
    dev = xh.device
    n = B * H * W * Cout
    wph, wpl = prep_conv_weight(wh), (prep_conv_weight(wl) if wl is not None else None)
    gd = Guarded(n, F32, dev) if want_d else None
    gh = Guarded(n, BF16, dev) if want_split else None
    gl = Guarded(n, BF16, dev) if want_split else None
    _lib.call("adb_conv3x3_bf16", B, H, W, Cin, Cout, _ptr(xh), _ptr(xl), _ptr(wph), _ptr(wpl), _ptr(bias),
              _ptr(residual), _ptr(gd.out) if gd else None, _ptr(gh.out) if gh else None, _ptr(gl.out) if gl else None,
              act, split_relu, _lib.stream())
    torch.cuda.synchronize()
    d = sp = None
    if gd:
        d = gd.take_all().view(B, H, W, Cout)
        gd.assert_untouched("conv D")
    if gh:
        sp = (gh.take_all().view(B, H, W, Cout), gl.take_all().view(B, H, W, Cout))
        gh.assert_untouched("conv D_hi")
        gl.assert_untouched("conv D_lo")
    return d, sp


def run_attention(qh, ql, kh, kl, vth, vtl, B, h, Nq, Nk, Nkpad, scale, variant):
    """adb_attention_bf16 with the given kernel variant into guarded outputs; returns (O_hi, O_lo) [B, Nq, h*64]."""
    from artdeco_b200 import _lib
    from artdeco_b200.mast3r import ops
    dev = qh.device
    n = B * Nq * h * 64
    gh = Guarded(n, BF16, dev)
    gl = Guarded(n, BF16, dev)    # requested in single pass too: measures the kernel, not the bf16 rounding of O
    prev = ops.set_attention_variant(variant)
    try:
        _lib.call("adb_attention_bf16", B, h, Nq, Nk, Nkpad, _ptr(qh), _ptr(ql), _ptr(kh), _ptr(kl), _ptr(vth), _ptr(vtl),
                  float(scale), _ptr(gh.out), _ptr(gl.out), _lib.stream())
        torch.cuda.synchronize()
    finally:
        ops.set_attention_variant(prev)
    oh, ol = gh.take_all().view(B, Nq, h * 64), gl.take_all().view(B, Nq, h * 64)
    gh.assert_untouched("O_hi")
    gl.assert_untouched("O_lo")
    return oh.clone(), ol.clone()


def heads_major(o, B, h, Nq):
    """[B, Nq, h*64] -> [B*h, Nq, 64]"""
    return o.view(B, Nq, h, 64).permute(0, 2, 1, 3).reshape(B * h, Nq, 64)


def make_vt(vh, vl, Nkpad):
    """keys-major V [BH, Nk, 64] -> Vt [BH, 64, Nkpad] with PADV in the padding columns."""
    BH, Nk, _ = vh.shape

    def one(v):
        vt = torch.full((BH, 64, Nkpad), PADV, dtype=BF16, device=v.device)
        vt[..., :Nk] = v.mT
        return vt.contiguous()
    return one(vh), (one(vl) if vl is not None else None)


def attention_all_variants(qh, ql, kh, kl, vth, vtl, B, h, Nq, Nk, Nkpad, scale, group):
    """Runs variants 1, 2 and automatic; asserts they agree bit for bit and returns the fp32 value of (hi + lo)."""
    outs = [run_attention(qh, ql, kh, kl, vth, vtl, B, h, Nq, Nk, Nkpad, scale, v) for v in (1, 2, 0)]
    (h1, l1) = outs[0]
    for v, (hv, lv) in zip((2, 0), outs[1:]):
        same = torch.equal(h1, hv) and torch.equal(l1, lv)
        if not same:
            _note(group, "variant_max_abs_diff", (joined(h1, l1) - joined(hv, lv)).abs().max().item(), max)
        assert same, f"{group}: variant {v} differs from variant 1"
    return joined(h1, l1)


MODES = pytest.mark.parametrize("x3", [True, False], ids=["bf16x3", "bf16"])


# ---------------------------------------------------------------------------------------------------------------------
# adb_gemm_bf16

GEMM_SHAPES = [(1, 129, 8), (4, 1000, 64), (24, 127, 72), (127, 24, 512), (128, 200, 520), (129, 128, 1024),
               (200, 4, 4096), (1000, 129, 4104), (1, 1, 4104)]


def _gemm_bug_models(ah, al, bh, bl, ref, K, x3):
    """(name, fp64 result) of the nearest plausible GEMM bugs."""
    out = []
    kb_last = (K - 1) // 64 * 64
    tail, _ = gemm_exact_ref(ah[:, kb_last:], al[:, kb_last:] if x3 else None, bh[:, kb_last:], bl[:, kb_last:] if x3 else None)
    out.append(("last k-block dropped", ref - tail))
    if K > 512:
        c_last = (K - 1) // 512 * 512
        chunk, _ = gemm_exact_ref(ah[:, c_last:], al[:, c_last:] if x3 else None, bh[:, c_last:], bl[:, c_last:] if x3 else None)
        out.append(("last promotion chunk dropped", ref - chunk))
    if x3:
        out.append(("A_lo B_hi^T dropped", ref - al.to(F64) @ bh.to(F64).mT))
        out.append(("A_hi B_lo^T dropped", ref - ah.to(F64) @ bl.to(F64).mT))
    return out


@pytest.mark.gpu
@MODES
@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_exact_operands_on_vector_and_scalar_paths(cuda, M, N, K, x3):
    """Per-element accumulation error against the exact-operand product; the 256-bit store path (ldd a multiple of 8 and
    ldo of 16, padding columns guarded; full 32-column groups only, so N = 129 / 1000 end in a ragged scalar group), the
    scalar path (ldd = N + 3) and a misaligned output give bit-identical values."""
    group = f"gemm_exact_{'x3' if x3 else 'bf16'}"
    g = gen(cuda, 1000 * M + 10 * N + K)
    ah, al = pos_operand((M, K), g, x3, sign_dim=0)
    bh, bl = pos_operand((N, K), g, x3, sign_dim=0)
    ref, bnd = gemm_exact_ref(ah, al, bh, bl)
    tol = TOL_GEMM[x3]
    ld8, ld16 = (N + 7) // 8 * 8, (N + 15) // 16 * 16
    d_vec, _ = run_gemm(ah, al, bh, bl, M, N, K, ldd=ld8, ldr=ld8, ldo=ld16, vector=True)
    d_sca, _ = run_gemm(ah, al, bh, bl, M, N, K, ldd=N + 3, ldr=ld8, ldo=ld16, vector=False)
    d_mis, _ = run_gemm(ah, al, bh, bl, M, N, K, ldd=ld8, ldr=ld8, ldo=ld16, misalign=1, vector=False)
    check(group, nerr(d_vec, ref, bnd), tol)
    assert torch.equal(d_vec, d_sca) and torch.equal(d_vec, d_mis), "vector and scalar store paths differ"
    if x3:
        # the 2e-5 contract against the fp64 product of the fp32 inputs
        g2 = gen(cuda, 7 + K)
        a = torch.randn(M, K, generator=g2, device=cuda)
        w = torch.randn(N, K, generator=g2, device=cuda) * 0.05
        d, _ = run_gemm(*split(a), *split(w), M, N, K)
        assert rel_err(d, a.double() @ w.double().T) < 2e-5
    for name, bug in _gemm_bug_models(ah, al, bh, bl, ref, K, x3):
        discriminates(group, name, nerr(bug, ref, bnd), tol)


def _gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _act64(x, act):
    return _gelu64(x) if act == 1 else (x.clamp_min(0.0) if act == 2 else x)


@pytest.mark.gpu
@MODES
@pytest.mark.parametrize("outputs", ["D", "split", "both"])
@pytest.mark.parametrize("act", [0, 1, 2], ids=["none", "gelu", "relu"])
def test_gemm_epilogue_order_and_outputs(cuda, act, outputs, x3):
    """D = act(alpha * acc + bias) + residual with alpha != 1, as fp32 D, as the (hi, lo) split (D == NULL) or both;
    the scalar path (ldd, ldr, ldo not multiples of 8) gives the same bits as the vector path (ldd = ldr = 200, ldo = 208:
    six full 32-column groups on the vector path, the last 8 columns scalar)."""
    group = f"gemm_epilogue_{'x3' if x3 else 'bf16'}"
    M, N, K = 129, 200, 520
    g = gen(cuda, 11 + act)
    ah, al = pos_operand((M, K), g, x3, sign_dim=0)
    bh, bl = pos_operand((N, K), g, x3, sign_dim=0)
    ref, bnd = gemm_exact_ref(ah, al, bh, bl)
    alpha = 0.3
    scale = (alpha * ref).abs().mean().item()                 # bias and residual of the accumulator's size: act sees both signs
    bias = torch.randn(N, generator=g, device=cuda) * scale
    res = torch.randn(M, N, generator=g, device=cuda) * scale
    want = _act64(alpha * ref + bias.double(), act) + res.double()
    den = 1.13 * alpha * bnd + bias.double().abs() + res.double().abs()     # GELU's slope is at most 1.13
    tol = TOL_GEMM[x3]
    wd, ws = outputs in ("D", "both"), outputs in ("split", "both")
    results = []
    for ldd, ldr, ldo, vector in ((N, N, (N + 15) // 16 * 16, True), (N + 3, N + 5, N + 1, False)):
        r = res if ldr == N else F.pad(res, (0, ldr - N)).contiguous()
        results.append(run_gemm(ah, al, bh, bl, M, N, K, want_d=wd, want_split=ws, ldd=ldd, ldo=ldo, bias=bias, residual=r,
                                ldr=ldr, alpha=alpha, act=act, vector=vector))
    (d, sp), (d2, sp2) = results
    if wd:
        check(group, nerr(d, want, den), tol)
        assert torch.equal(d, d2), "vector and scalar epilogues differ"
    if ws:
        v = joined(*sp)
        check(group + "_split", nerr(v, want, den), tol + SPLIT)
        assert torch.equal(sp[0], sp2[0]) and torch.equal(sp[1], sp2[1]), "vector and scalar split stores differ"
        if wd:
            hi, lo = split(d)
            assert torch.equal(hi, sp[0]) and torch.equal(lo, sp[1]), "the split is not the rounding of D"
    bugs = [("bias added before alpha", _act64(alpha * (ref + bias.double()), act) + res.double())]
    if act:
        bugs += [("residual added before the activation", _act64(alpha * ref + bias.double() + res.double(), act)),
                 ("activation skipped", alpha * ref + bias.double() + res.double())]
    for name, bug in bugs:
        discriminates(group, name, nerr(bug, want, den), tol)


@pytest.mark.gpu
@MODES
@pytest.mark.parametrize("M,N,K", [(1, 4, 8), (129, 200, 72), (600, 24, 520), (4200, 4, 4104), (1100, 1000, 1024)])
def test_gemm_selection_matrix_is_an_exact_gather(cuda, M, N, K, x3):
    """A = one 1.0 per row (every k addressed when M >= K, and always k = K - 1): D = B[:, idx]^T exactly, hi + lo in
    bf16x3 mode, hi alone in single pass."""
    g = gen(cuda, M + K)
    idx = selection_indices(M, K, g)
    ah = selection_matrix(idx, K)
    al = torch.zeros_like(ah) if x3 else None
    bh, bl = split(torch.randn(N, K, generator=g, device=cuda), x3)
    d, _ = run_gemm(ah, al, bh, bl, M, N, K)
    assert torch.equal(d, joined(bh, bl)[:, idx].T)


@pytest.mark.gpu
@MODES
@pytest.mark.parametrize("layout", ["vector", "scalar"])
def test_gemm_batched_zdiv_addressing_is_exact(cuda, layout, x3):
    """batch = 2 x zdiv 3 with a different selection per batch entry and distinct output / split / residual layouts
    (sD/sD2, sO/sO2, sR/sR2): every value lands at its address bit for bit, nothing else is written."""
    from artdeco_b200.mast3r import ops
    zo_n, zdiv, M, N, K = 2, 3, 600, 72, 520
    Z = zo_n * zdiv
    g = gen(cuda, 5 if x3 else 6)
    idx = [selection_indices(M, K, g) for _ in range(Z)]
    ah = torch.stack([selection_matrix(i, K) for i in idx]).contiguous()
    al = torch.zeros_like(ah) if x3 else None
    bh, bl = split(torch.randn(Z, N, K, generator=g, device=cuda), x3)
    vec = layout == "vector"
    # D: [zo][m][zi][n];  split: [zi][zo][m][ldo];  residual: [zo][zi][m][ldr] with a gap between the z_outer blocks
    ldd = zdiv * N + (8 if vec else 3)
    sD, sD2 = N, M * ldd
    ldo = 80 if vec else 77
    sO, sO2 = zo_n * M * ldo, M * ldo
    ldr = 72 if vec else 75
    sR, sR2 = M * ldr, zdiv * M * ldr + 8
    offD = matrix_offsets(Z, M, N, ldd, sD, zdiv, sD2, cuda)
    offO = matrix_offsets(Z, M, N, ldo, sO, zdiv, sO2, cuda)
    offR = matrix_offsets(Z, M, N, ldr, sR, zdiv, sR2, cuda)
    for off in (offD, offO, offR):
        assert off.unique().numel() == off.numel()
    res_flat = torch.zeros(int(offR.max()) + 1, device=cuda)
    res = torch.randn(Z, M, N, generator=g, device=cuda)
    res_flat[offR] = res
    gd = Guarded(int(offD.max()) + 1, F32, cuda)
    gh = Guarded(int(offO.max()) + 1, BF16, cuda)
    gl = Guarded(int(offO.max()) + 1, BF16, cuda)
    ptrs = [t.out.data_ptr() for t in (gd, gh, gl)] + [res_flat.data_ptr()]
    assert all(vector_store_path(ldd, ldr, ldo, ptrs, (z // zdiv) * sD2 + (z % zdiv) * sD, (z // zdiv) * sR2 + (z % zdiv) * sR,
                                 (z // zdiv) * sO2 + (z % zdiv) * sO) == vec for z in range(Z))
    ops.gemm(ops.Split(ah, al), ops.Split(bh, bl), M, N, K, batch=Z, sA=M * K, sB=N * K, out=gd.out, ldd=ldd, sD=sD,
             out_split=ops.Split(gh.out, gl.out), ldo=ldo, sO=sO, residual=res_flat, ldr=ldr, sR=sR, zdiv=zdiv, sD2=sD2,
             sO2=sO2, sR2=sR2)
    torch.cuda.synchronize()
    want = torch.stack([joined(bh[z], bl[z] if x3 else None)[:, idx[z]].T for z in range(Z)]) + res
    hi, lo = split(want)
    assert torch.equal(gd.take(offD), want)
    assert torch.equal(gh.take(offO), hi) and torch.equal(gl.take(offO), lo)
    gd.assert_untouched("D")
    gh.assert_untouched("D_hi")
    gl.assert_untouched("D_lo")


# ---------------------------------------------------------------------------------------------------------------------
# adb_gemm_bf16_rope

def _rope64(y, bnd, pos, table, heads):
    """RoPE2D of [M, heads*64] fp64 rows with the kernel's (cos, sin) table: dims [0, 32) rotate by the y position,
    [32, 64) by x, pairs (i, i + 16).  Returns ([M, heads, 64] value, bound)."""
    M = y.shape[0]
    y, bnd = y.view(M, heads, 64), bnd.view(M, heads, 64)
    tab = table.to(F64)
    outs, bnds = [], []
    for axis in (0, 1):
        c = tab[pos[:, axis], :, 0][:, None, :]
        s = tab[pos[:, axis], :, 1][:, None, :]
        u, w = y[..., 32 * axis:32 * axis + 16], y[..., 32 * axis + 16:32 * axis + 32]
        bu, bw = bnd[..., 32 * axis:32 * axis + 16], bnd[..., 32 * axis + 16:32 * axis + 32]
        outs += [u * c - w * s, w * c + u * s]
        bnds += [bu * c.abs() + bw * s.abs(), bw * c.abs() + bu * s.abs()]
    return torch.cat(outs, -1), torch.cat(bnds, -1)


@pytest.mark.gpu
@MODES
@pytest.mark.parametrize("B,ntok,h,n_dst,rest", [(2, 200, 4, 2, 40), (1, 77, 2, 1, 13), (3, 130, 2, 2, 0), (2, 129, 12, 1, 100)])
def test_gemm_rope_exact_operands(cuda, B, ntok, h, n_dst, rest, x3):
    """adb_gemm_bf16_rope in both modes against the exact-operand product + bias, rotated in fp64 with the kernel's
    table; tail widths 13 / 40 / 100 are not multiples of 32 (13 not even of 8).  The lo outputs are requested in single
    pass too, so that the GEMM's own error is measured rather than the bf16 rounding of the output."""
    from artdeco_b200 import _lib
    from artdeco_b200.mast3r import ops
    group = f"gemm_rope_{'x3' if x3 else 'bf16'}"
    C, K = h * 64, 520
    N, M = n_dst * C + rest, B * ntok
    g = gen(cuda, M + N)
    ah, al = pos_operand((M, K), g, x3, sign_dim=0)
    wh, wl = pos_operand((N, K), g, x3, sign_dim=0)
    bias = torch.randn(N, generator=g, device=cuda)
    pos = torch.randint(0, 64, (M, 2), generator=g, device=cuda)
    table = ops.rope_table(64, cuda)
    y, bnd = gemm_exact_ref(ah, al, wh, wl)
    y, bnd = y + bias.double(), bnd + bias.double().abs()
    heads = [(Guarded(M * C, BF16, cuda), Guarded(M * C, BF16, cuda)) for _ in range(n_dst)]
    tail = Guarded(M * rest, F32, cuda) if rest else None
    _lib.call("adb_gemm_bf16_rope", M, N, K, _ptr(ah), _ptr(al), K, _ptr(wh), _ptr(wl), K, _ptr(bias), ntok, h, n_dst,
              _ptr(pos), _ptr(table), 64, _ptr(heads[0][0].out), _ptr(heads[0][1].out),
              _ptr(heads[1][0].out) if n_dst == 2 else None, _ptr(heads[1][1].out) if n_dst == 2 else None,
              _ptr(tail.out) if tail else None, max(rest, 1), _lib.stream())
    torch.cuda.synchronize()
    tol = TOL_GEMM[x3]
    for sec, (gh, gl) in enumerate(heads):
        want, wb = _rope64(y[:, sec * C:(sec + 1) * C], bnd[:, sec * C:(sec + 1) * C], pos, table, h)
        got = joined(gh.take_all(), gl.take_all()).view(B, h, ntok, 64).permute(0, 2, 1, 3).reshape(M, h, 64)
        gh.assert_untouched("q/k hi")
        gl.assert_untouched("q/k lo")
        check(group, nerr(got, want, wb), tol + SPLIT)
        swapped, _ = _rope64(y[:, sec * C:(sec + 1) * C], bnd[:, sec * C:(sec + 1) * C], pos.flip(-1), table, h)
        discriminates(group, "y and x positions swapped", nerr(swapped, want, wb), tol + SPLIT)
    if tail:
        got = tail.take_all().view(M, rest)
        tail.assert_untouched("D_tail")
        check(group, nerr(got, y[:, n_dst * C:], bnd[:, n_dst * C:]), tol)


# ---------------------------------------------------------------------------------------------------------------------
# adb_conv3x3_bf16

def _bands(H, W, B):
    """Output row ranges the reference evaluates: the whole image when small, else the first rows, two rows around a
    pixel-tile boundary in the middle and the last rows (every column: the right-hand tiles may be partial)."""
    if B * H * W <= 1 << 14:
        return [(0, H)]
    _, hb = conv_tile(W)
    mid = (H // 2) // hb * hb
    cand = sorted({(0, min(H, 2)), (max(0, mid - 1), min(H, mid + 1)), (max(0, H - 2), H)})
    out = []
    for a, b in cand:
        if out and a <= out[-1][1]:
            out[-1] = (out[-1][0], max(out[-1][1], b))
        else:
            out.append((a, b))
    return out


def _conv_bug_models(xh, xl, wh, wl, Cin, y0, y1, x3):
    out = [("border wrapped instead of zero-filled", conv_exact_ref(xh, xl, wh, wl, y0, y1, wrap=True)[0])]
    if x3:
        out.append(("x_lo w_hi dropped", conv64(xh, wh, y0, y1) + conv64(xh, wl, y0, y1)))
    if Cin > 64:
        keep = torch.ones(Cin, device=wh.device, dtype=BF16)
        keep[(Cin - 1) // 64 * 64:] = 0
        kw = keep[None, :, None, None]
        out.append(("last channel chunk dropped",
                    conv_exact_ref(xh, xl, wh * kw, wl * kw if x3 else None, y0, y1)[0]))
    tap = torch.ones(3, 3, device=wh.device, dtype=BF16)
    tap[1, 1] = 0
    out.append(("centre tap dropped", conv_exact_ref(xh, xl, wh * tap, wl * tap if x3 else None, y0, y1)[0]))
    return out


def _conv_case(cuda, B, H, W, Cin, Cout, x3, group, seed, true_check=True):
    g = gen(cuda, seed)
    xh, xl = pos_operand((B, H, W, Cin), g, x3)
    wh, wl = pos_operand((Cout, Cin, 3, 3), g, x3, sign_dim=0)
    d, _ = run_conv(xh, xl, wh, wl, B, H, W, Cin, Cout)
    tol = TOL_CONV[x3]
    bands = _bands(H, W, B)
    refs = [conv_exact_ref(xh, xl, wh, wl, a, b) for a, b in bands]
    for (a, b), (ref, bnd) in zip(bands, refs):
        check(group, nerr(d[:, a:b], ref, bnd), tol)
    for (a, b), (ref, bnd) in zip(bands, refs):
        for name, bug in _conv_bug_models(xh, xl, wh, wl, Cin, a, b, x3):
            discriminates(group, name, nerr(bug, ref, bnd), tol)
    if x3 and true_check:
        # the 2e-5 contract: fp32 activations and weights against F.conv2d(x, w, padding=1) in fp64
        x = torch.randn(B, H, W, Cin, generator=g, device=cuda)
        w = torch.randn(Cout, Cin, 3, 3, generator=g, device=cuda) / (9 * Cin) ** 0.5
        d, _ = run_conv(*split(x), *split(w), B, H, W, Cin, Cout)
        for a, b in bands:
            assert rel_err(d[:, a:b], conv64(x, w, a, b)) < 2e-5


@pytest.mark.gpu
@MODES
@pytest.mark.parametrize("B,H,W,Cin", [(2, 1, 1, 8), (1, 3, 5, 72), (2, 17, 9, 96), (1, 3, 200, 8), (2, 17, 24, 72),
                                       (1, 1, 200, 96)])
def test_conv3x3_one_hot_taps_are_exact_shifts(cuda, B, H, W, Cin, x3):
    """Nine identity maps, one per tap (Cout = 9 Cin): output block t is the input shifted by (ky - 1, kx - 1) with
    zeros at the border, bit for bit (hi + lo in bf16x3, hi in single pass) -- including W < 8, where the TMA box is
    wider than the image, and partial channel chunks."""
    g = gen(cuda, H * W + Cin)
    xh, xl = split(torch.randn(B, H, W, Cin, generator=g, device=cuda), x3)
    w = one_hot_tap_weight(Cin, cuda)
    d, sp = run_conv(xh, xl, w, torch.zeros_like(w) if x3 else None, B, H, W, Cin, 9 * Cin, want_split=True)
    want = shifted_taps(joined(xh, xl))
    assert torch.equal(d, want)
    hi, lo = split(want)
    assert torch.equal(sp[0], hi) and torch.equal(sp[1], lo)


@pytest.mark.gpu
@MODES
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 1, 1, 8, 4), (1, 3, 5, 72, 130), (2, 17, 9, 96, 4), (1, 17, 24, 8, 130),
                                            (2, 3, 200, 96, 130), (1, 1, 200, 72, 4), (2, 17, 5, 96, 130)])
def test_conv3x3_exact_operands_degenerate_shapes(cuda, B, H, W, Cin, Cout, x3):
    """Widths 1 / 5 / 9 / 24 / 200 (box wider than the image, partial last pixel tile), heights 1 / 3 / 17, Cin 8 / 72 / 96
    (partial channel chunk) and Cout 4 / 130 (partial N tile), B up to 2."""
    _conv_case(cuda, B, H, W, Cin, Cout, x3, f"conv_exact_{'x3' if x3 else 'bf16'}", B * H * W + Cin + Cout)


def dpt_conv3x3_shapes(H, W):
    """(name, h, w, Cin, Cout) of every distinct 3x3 convolution AsymmetricMASt3R._dpt runs for an H x W image: the
    feature-map sizes follow _dpt, the channel counts come from the state-dict shapes."""
    from artdeco_b200.mast3r import FULL_CFG
    from artdeco_b200.mast3r.shapes import param_shapes
    ps = param_shapes(FULL_CFG)
    d = "downstream_head1.dpt."
    nh, nw = H // 16, W // 16
    h3, w3 = (nh + 1) // 2, (nw + 1) // 2        # act_postprocess.3.1 output sampled at even pixels
    sites = [("act_postprocess.3.1", nh, nw), ("scratch.layer1_rn", 4 * nh, 4 * nw), ("scratch.layer2_rn", 2 * nh, 2 * nw),
             ("scratch.layer3_rn", nh, nw), ("scratch.layer4_rn", h3, w3)]
    for r, (fh, fw) in ((4, (h3, w3)), (3, (nh, nw)), (2, (2 * nh, 2 * nw)), (1, (4 * nh, 4 * nw))):
        sites.append((f"scratch.refinenet{r}.resConfUnit2.conv1", fh, fw))
    sites += [("head.0", 8 * nh, 8 * nw), ("head.2", H, W)]
    seen, out = set(), []
    for name, fh, fw in sites:
        cout, cin = ps[d + name + ".weight"][:2]
        if (fh, fw, cin, cout) not in seen:
            seen.add((fh, fw, cin, cout))
            out.append((name, fh, fw, cin, cout))
    return out


@pytest.mark.gpu
@MODES
@pytest.mark.parametrize("H,W", [(512, 512), (384, 512), (512, 384)])
def test_conv3x3_exact_operands_dpt_head_shapes(cuda, H, W, x3):
    """Every 3x3 conv shape of the DPT head at B = 2: at 384 pixels the feature maps are 24 / 48 / 96 / 192 / 384 wide
    (partial pixel tiles), layer1_rn has Cin = 96."""
    for i, (name, fh, fw, cin, cout) in enumerate(dpt_conv3x3_shapes(H, W)):
        _conv_case(cuda, 2, fh, fw, cin, cout, x3, f"conv_dpt_{'x3' if x3 else 'bf16'}", 100 * H + W + i)


@pytest.mark.gpu
@MODES
@pytest.mark.parametrize("bias,residual,act,split_relu,outputs", [
    (False, False, 0, 0, "D"), (True, False, 0, 0, "D"), (True, True, 0, 0, "both"), (True, False, 2, 0, "both"),
    (True, True, 2, 1, "both"), (True, True, 0, 1, "split")])
def test_conv3x3_epilogue(cuda, bias, residual, act, split_relu, outputs, x3):
    """bias, residual (added after the activation), ReLU, split_relu (the split stores relu(v), D keeps v) and a
    split-only output, at a shape with a partial pixel tile, a partial channel chunk and a partial N tile."""
    group = f"conv_epilogue_{'x3' if x3 else 'bf16'}"
    B, H, W, Cin, Cout = 2, 17, 24, 96, 130
    g = gen(cuda, 31 + act + 2 * split_relu)
    xh, xl = pos_operand((B, H, W, Cin), g, x3)
    wh, wl = pos_operand((Cout, Cin, 3, 3), g, x3, sign_dim=0)
    ref, bnd = conv_exact_ref(xh, xl, wh, wl)
    scale = ref.abs().mean().item()
    b = torch.randn(Cout, generator=g, device=cuda) * scale if bias else None
    r = torch.randn(B, H, W, Cout, generator=g, device=cuda) * scale if residual else None
    v = ref + (b.double() if bias else 0.0)
    want = _act64(v, act) + (r.double() if residual else 0.0)
    den = bnd + (b.double().abs() if bias else 0.0) + (r.double().abs() if residual else 0.0)
    wd, ws = outputs in ("D", "both"), outputs in ("split", "both")
    d, sp = run_conv(xh, xl, wh, wl, B, H, W, Cin, Cout, bias=b, residual=r, act=act, split_relu=split_relu,
                     want_d=wd, want_split=ws)
    tol = TOL_CONV[x3]
    if wd:
        check(group, nerr(d, want, den), tol)
    if ws:
        want_s = want.clamp_min(0.0) if split_relu else want
        check(group + "_split", nerr(joined(*sp), want_s, den), tol + SPLIT)
        if wd:
            hi, lo = split(d.clamp_min(0.0) if split_relu else d)
            assert torch.equal(hi, sp[0]) and torch.equal(lo, sp[1])
    bugs = [("bias dropped", _act64(ref, act) + (r.double() if residual else 0.0))] if bias else []
    if residual and act:
        bugs.append(("residual added before the activation", _act64(v + r.double(), act)))
    if act:
        bugs.append(("activation skipped", v + (r.double() if residual else 0.0)))
    for name, bug in bugs:
        discriminates(group, name, nerr(bug, want, den), tol)
    if ws and split_relu:
        discriminates(group + "_split", "split without relu", nerr(want, want.clamp_min(0.0), den), tol + SPLIT)


# ---------------------------------------------------------------------------------------------------------------------
# adb_attention_bf16

ATTN_SHAPES = [(1, 1, 1, 1, 0), (1, 2, 127, 8, 64), (2, 3, 129, 127, 0), (1, 4, 257, 128, 64), (2, 2, 1024, 129, 0),
               (1, 3, 257, 300, 64), (1, 2, 129, 1024, 64), (5, 16, 1024, 300, 0)]


def _attn_inputs(cuda, BH, Nq, Nk, logit_std, x3, seed):
    g = gen(cuda, seed)
    q = torch.randn(BH, Nq, 64, generator=g, device=cuda) * logit_std       # scale 1/8: logits of std logit_std
    k = torch.randn(BH, Nk, 64, generator=g, device=cuda)
    vh, vl = pos_operand((BH, Nk, 64), g, x3, sign_dim=2)
    return q, k, split(q, x3), split(k, x3), (vh, vl)


def _attn_case(cuda, B, h, Nq, Nk, extra, x3, logit_std, group, tol, tol_true=None):
    BH, scale = B * h, 0.125
    Nkpad = (Nk + 7) // 8 * 8 + extra
    q, k, (qh, ql), (kh, kl), (vh, vl) = _attn_inputs(cuda, BH, Nq, Nk, logit_std, x3, BH * Nq + Nk + extra)
    vth, vtl = make_vt(vh, vl, Nkpad)
    o = heads_major(attention_all_variants(qh, ql, kh, kl, vth, vtl, B, h, Nq, Nk, Nkpad, scale, group), B, h, Nq)
    ref, bnd = attn_exact_ref(qh, ql, kh, kl, vh, vl, scale, x3)
    check(group, nerr(o, ref, bnd), tol)
    if tol_true is not None:
        v = join64(vh, vl)
        p = torch.softmax(scale * q.double() @ k.double().mT, -1)
        check(group + "_vs_fp64", nerr(o, p @ v, p @ v.abs()), tol_true)
    if x3:
        bug, _ = attn_exact_ref(qh, ql, kh, kl, vh, torch.zeros_like(vl), scale, x3)
        discriminates(group, "P V_lo dropped", nerr(bug, ref, bnd), tol)
    last = (Nk - 1) // 128 * 128
    if last > 0:
        bug, _ = attn_exact_ref(qh, ql, kh[:, :last], kl[:, :last] if x3 else None, vh[:, :last],
                                vl[:, :last] if x3 else None, scale, x3)
        discriminates(group, "last key block dropped", nerr(bug, ref, bnd), tol)
    return o, ref


@pytest.mark.gpu
@MODES
@pytest.mark.parametrize("B,h,Nq,Nk,extra", ATTN_SHAPES)
def test_attention_exact_operands_all_variants(cuda, B, h, Nq, Nk, extra, x3):
    """Both kernel variants and the automatic choice, bit-identical, against the exact-operand reference; Vt's padding
    columns hold PADV.  (5, 16, 1024, 300): variant 2 has 320 work items on 132 SMs (not a multiple, > 2 per CTA)."""
    mode = "x3" if x3 else "bf16"
    o, _ = _attn_case(cuda, B, h, Nq, Nk, extra, x3, 1.0, f"attn_exact_{mode}", TOL_ATTN[x3])
    if x3:
        # the 3e-5 contract of tests/test_gemm.py against softmax(q k^T / 8) v in fp64 of the fp32 inputs
        BH = B * h
        q, k, _, _, (vh, vl) = _attn_inputs(cuda, BH, Nq, Nk, 1.0, x3, BH * Nq + Nk + extra)
        p = torch.softmax(0.125 * q.double() @ k.double().mT, -1)
        assert rel_err(o, p @ join64(vh, vl)) < 3e-5


@pytest.mark.gpu
@pytest.mark.parametrize("logit_std", [8.0, 32.0])
@pytest.mark.parametrize("B,h,Nq,Nk,extra", [(1, 2, 257, 300, 64), (2, 4, 129, 1024, 0)])
def test_attention_large_logits(cuda, B, h, Nq, Nk, extra, logit_std):
    """Logits of standard deviation 8 and 32 after the scale (bf16x3, every variant).  Pass 1 shifts by the hi x hi
    row maximum, pass 2 exponentiates the bf16x3 scores, so the largest p = exp2((s - m) scale log2e) exceeds 1 by the
    hi-only error of the maximum.  The test computes that exponent from its own operands (report key max_p_log2):
    0.12 at std 8 and 0.47 at std 32, so p <= 2^0.47; it asserts < 16.  The error is at most about
    2^-7 * max_j sum_d |q_d k_jd| * scale; scaled linearly, p would reach fp32 overflow (2^128) only for logits of ~10^4.
    That limit is derived from the bound, not measured: the largest logits run here are those of std 32 (|logit| up to
    ~150) and the -120 rows of test_attention_max_is_taken_over_valid_keys_only."""
    BH, scale = B * h, 0.125
    _, _, (qh, ql), (kh, kl), _ = _attn_inputs(cuda, BH, Nq, Nk, logit_std, True, BH * Nq + Nk + extra)   # _attn_case's operands
    qh64, kh64 = qh.to(F64), kh.to(F64)
    s_hi = qh64 @ kh64.mT
    s3 = s_hi + qh64 @ kl.to(F64).mT + ql.to(F64) @ kh64.mT
    c1 = attn_scale_log2e(scale)
    over = ((s3.amax(-1) - s_hi.amax(-1)) * c1).max().item()       # log2 of the largest p the kernel forms
    _note(f"attn_large_std{int(logit_std)}", "max_p_log2", over, max)
    assert over < 16.0
    _attn_case(cuda, B, h, Nq, Nk, extra, True, logit_std, f"attn_large_std{int(logit_std)}", TOL_ATTN_LARGE[logit_std],
               TOL_ATTN_TRUE[logit_std])


@pytest.mark.gpu
@MODES
@pytest.mark.parametrize("Nq,Nk,extra", [(1, 1, 0), (127, 8, 64), (129, 127, 0), (257, 129, 64), (1024, 300, 0),
                                         (1024, 1024, 64)])
def test_attention_one_hot_rows_address_every_key(cuda, Nq, Nk, extra, x3):
    """q_i = c k_pi(i) with unit keys and c so large that the logit gap x scale x log2e >= 60: softmax is one-hot in
    fp32 and O[i] = V[pi(i)] to the hi + lo rounding.  pi covers every key (Nq >= Nk), the last partial block included;
    each head has its own pi."""
    B, h, scale = 1, 2, 0.125
    BH = B * h
    Nkpad = (Nk + 7) // 8 * 8 + extra
    g = gen(cuda, Nq + Nk)
    k = torch.randn(BH, Nk, 64, generator=g, device=cuda)
    k = k / k.norm(dim=-1, keepdim=True)
    cos = k @ k.mT - 2.0 * torch.eye(Nk, device=cuda)
    maxcos = max(cos.max().item(), 0.0)
    assert maxcos < 0.9
    c = 1.25 * 60.0 / (scale * LOG2E * (1.0 - maxcos))
    idx = torch.stack([selection_indices(Nq, Nk, g) for _ in range(BH)])
    q = c * torch.gather(k, 1, idx[..., None].expand(-1, -1, 64))
    vh, vl = split(torch.randn(BH, Nk, 64, generator=g, device=cuda), x3)
    (qh, ql), (kh, kl) = split(q, x3), split(k, x3)
    vth, vtl = make_vt(vh, vl, Nkpad)
    o = heads_major(attention_all_variants(qh, ql, kh, kl, vth, vtl, B, h, Nq, Nk, Nkpad, scale, "attn_one_hot"), B, h, Nq)
    want = torch.gather(joined(vh, vl), 1, idx[..., None].expand(-1, -1, 64))
    bound = ONE_HOT_REL * want.abs() + 2.0 ** -20 * want.abs().amax(-1, keepdim=True)
    bad = ((o - want).abs() > bound).sum().item()
    assert bad == 0, f"{bad} output values are not the addressed key's value"


@pytest.mark.gpu
@MODES
@pytest.mark.parametrize("Nk,extra", [(1, 64), (8, 64), (127, 0), (129, 64), (300, 64), (1024, 0)])
def test_attention_zero_keys_average_valid_values_only(cuda, Nk, extra, x3):
    """K = 0: every valid key has weight exactly 1, so O is the mean of the Nk valid V rows.  Keys past Nk -- Vt's
    padding columns (PADV) and the zero-filled rest of the last 128-key block -- must get exactly zero weight."""
    group = f"attn_mask_{'x3' if x3 else 'bf16'}"
    B, h, Nq, scale = 2, 2, 129, 0.125
    BH = B * h
    Nkpad = (Nk + 7) // 8 * 8 + extra
    g = gen(cuda, Nk + extra)
    qh, ql = split(torch.randn(BH, Nq, 64, generator=g, device=cuda), x3)
    kh = torch.zeros(BH, Nk, 64, dtype=BF16, device=cuda)
    kl = torch.zeros_like(kh) if x3 else None
    vh, vl = pos_operand((BH, Nk, 64), g, x3, sign_dim=2)
    vth, vtl = make_vt(vh, vl, Nkpad)
    o = heads_major(attention_all_variants(qh, ql, kh, kl, vth, vtl, B, h, Nq, Nk, Nkpad, scale, group), B, h, Nq)
    ref, bnd = attn_exact_ref(qh, ql, kh, kl, vh, vl, scale, x3)
    mean = join64(vh, vl).mean(1, keepdim=True).expand_as(ref)
    assert nerr(ref, mean, bnd) < 1e-12
    tol = TOL_ATTN[x3]
    check(group, nerr(o, ref, bnd), tol)
    # bug model: keys [Nk, end of the last block) not masked -- weight 1 each, V from Vt's padding or the TMA zero fill
    nb_end = (Nk + 127) // 128 * 128
    if nb_end > Nk:
        vpad = torch.zeros(BH, nb_end - Nk, 64, device=cuda, dtype=F64)
        npad = min(Nkpad, nb_end) - Nk
        vpad[:, :npad] = PADV * (2.0 if x3 else 1.0)
        bug = (join64(vh, vl).sum(1, keepdim=True) + vpad.sum(1, keepdim=True)) / nb_end
        discriminates(group, "padded keys not masked", nerr(bug.expand_as(ref), ref, bnd), tol)


@pytest.mark.gpu
@MODES
@pytest.mark.parametrize("Nk", [129, 300])
def test_attention_max_is_taken_over_valid_keys_only(cuda, Nk, x3):
    """Every valid logit is about -120 (keys near one direction u, q = -c u): a row maximum that also saw a padded key
    (score 0) would shift every p below 2^-126, flush them to zero and divide 0 by 0."""
    group = f"attn_negative_{'x3' if x3 else 'bf16'}"
    B, h, Nq, scale = 1, 2, 257, 0.125
    BH = B * h
    Nkpad = (Nk + 7) // 8 * 8
    g = gen(cuda, Nk)
    u = torch.randn(64, generator=g, device=cuda)
    u = u / u.norm()
    k = u + 0.05 * torch.randn(BH, Nk, 64, generator=g, device=cuda)
    k = k / k.norm(dim=-1, keepdim=True)
    q = (-120.0 / scale) * u.expand(BH, Nq, 64) + torch.randn(BH, Nq, 64, generator=g, device=cuda)
    (qh, ql), (kh, kl) = split(q, x3), split(k, x3)
    vh, vl = pos_operand((BH, Nk, 64), g, x3, sign_dim=2)
    vth, vtl = make_vt(vh, vl, Nkpad)
    o = heads_major(attention_all_variants(qh, ql, kh, kl, vth, vtl, B, h, Nq, Nk, Nkpad, scale, group), B, h, Nq)
    ref, bnd = attn_exact_ref(qh, ql, kh, kl, vh, vl, scale, x3)
    tol = TOL_ATTN_LARGE[32.0] if x3 else TOL_ATTN[False]
    check(group, nerr(o, ref, bnd), tol)
    bug, _ = attn_exact_ref(qh, ql, kh, kl, vh, vl, scale, x3, m_floor=0.0)
    discriminates(group, "pass-1 max taken over padded keys", nerr(bug, ref, bnd), tol)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: argument refusal (status 1 + adb_last_error before any CUDA call) and the reference helpers

def _refused(L, rc, needle):
    msg = L.adb_last_error()
    return rc == 1 and msg is not None and needle in msg.decode()


def test_tensorcore_entry_points_refuse_bad_arguments_before_touching_the_device():
    from artdeco_b200 import _lib
    import artdeco_b200  # noqa: F401  (registers every signature)
    L = _lib.lib()
    p16, p8 = ctypes.c_void_p(16), ctypes.c_void_p(24)       # never dereferenced; p8 is only 8-byte aligned

    def gemm(**kw):
        a = dict(batch=1, M=128, N=128, K=64, A_hi=p16, A_lo=None, lda=64, sA=0, B_hi=p16, B_lo=None, ldb=64, sB=0, D=p16,
                 ldd=128, sD=0, D_hi=None, D_lo=None, ldo=128, sO=0, bias=None, residual=None, ldr=128, sR=0, alpha=1.0,
                 act=0, zdiv=0, sD2=0, sO2=0, sR2=0, stream=None)
        a.update(kw)
        return L.adb_gemm_bf16(*a.values())
    for kw in (dict(batch=0), dict(M=0), dict(N=0), dict(K=0), dict(M=-1)):
        assert _refused(L, gemm(**kw), "adb_gemm_bf16: bad sizes"), kw
    assert _refused(L, gemm(A_hi=None), "adb_gemm_bf16: null pointer")
    assert _refused(L, gemm(D=None), "adb_gemm_bf16: null pointer")
    assert _refused(L, gemm(A_lo=p16), "A_lo and B_lo must be given together")
    assert _refused(L, gemm(B_lo=p16), "A_lo and B_lo must be given together")
    for kw in (dict(lda=68), dict(ldb=12), dict(batch=2, sA=4, sB=8192), dict(batch=2, sA=8192, sB=12)):
        assert _refused(L, gemm(**kw), "strides must be multiples of 8"), kw
    assert _refused(L, gemm(A_hi=p8), "16-byte aligned")
    assert _refused(L, gemm(B_hi=p8), "16-byte aligned")
    for act in (-1, 3):
        assert _refused(L, gemm(act=act), "adb_gemm_bf16: unknown activation")
    assert _refused(L, gemm(batch=2, sA=8192, sB=0), "weight broadcast")

    def rope(**kw):
        a = dict(M=256, N=256, K=64, A_hi=p16, A_lo=None, lda=64, B_hi=p16, B_lo=None, ldb=64, bias=None, ntok=128, heads=2,
                 n_rope_dst=2, pos=p16, table=p16, n_pos=64, q_hi=p16, q_lo=None, k_hi=p16, k_lo=None, D_tail=None, ldd=1,
                 stream=None)
        a.update(kw)
        return L.adb_gemm_bf16_rope(*a.values())
    for kw in (dict(M=0), dict(K=0), dict(ntok=0), dict(heads=0), dict(M=200)):
        assert _refused(L, rope(**kw), "adb_gemm_bf16_rope: bad sizes"), kw
    assert _refused(L, rope(n_rope_dst=3), "n_rope_dst must be 1 or 2")
    assert _refused(L, rope(N=192), "N smaller than the rotated sections")
    assert _refused(L, rope(pos=None), "adb_gemm_bf16_rope: null pointer")
    assert _refused(L, rope(k_hi=None), "adb_gemm_bf16_rope: null pointer")
    assert _refused(L, rope(N=300), "tail columns need D_tail")
    assert _refused(L, rope(A_lo=p16), "A_lo and B_lo must be given together")
    assert _refused(L, rope(lda=60), "strides must be multiples of 8")
    assert _refused(L, rope(A_hi=p8), "aligned")
    assert _refused(L, rope(q_hi=ctypes.c_void_p(48)), "outputs 32-byte")

    def conv(**kw):
        a = dict(B=1, H=8, W=8, Cin=64, Cout=64, x_hi=p16, x_lo=None, w_hi=p16, w_lo=None, bias=None, residual=None, D=p16,
                 D_hi=None, D_lo=None, act=0, split_relu=0, stream=None)
        a.update(kw)
        return L.adb_conv3x3_bf16(*a.values())
    for kw in (dict(B=0), dict(H=0), dict(W=0), dict(Cout=0), dict(Cin=0), dict(Cin=4)):
        assert _refused(L, conv(**kw), "adb_conv3x3_bf16: bad sizes"), kw
    for cin in (12, 100):
        assert _refused(L, conv(Cin=cin), "Cin must be a multiple of 8")
    assert _refused(L, conv(x_hi=None), "adb_conv3x3_bf16: null pointer")
    assert _refused(L, conv(D=None), "adb_conv3x3_bf16: null pointer")
    assert _refused(L, conv(x_lo=p16), "x_lo and w_lo must be given together")
    for act in (1, 3, -1):
        assert _refused(L, conv(act=act), "act must be 0 or 2")
    assert _refused(L, conv(x_hi=p8), "adb_conv3x3_bf16: operands must be 16-byte aligned")
    assert _refused(L, conv(x_lo=p8, w_lo=p16), "adb_conv3x3_bf16: operands must be 16-byte aligned")
    assert _refused(L, conv(w_hi=p8), "adb_conv3x3_bf16: operands must be 16-byte aligned")

    def attn(**kw):
        a = dict(B=1, heads=2, Nq=128, Nk=128, Nkpad=128, Q_hi=p16, Q_lo=None, K_hi=p16, K_lo=None, Vt_hi=p16, Vt_lo=None,
                 scale=0.125, O_hi=p16, O_lo=None, stream=None)
        a.update(kw)
        return L.adb_attention_bf16(*a.values())
    for kw in (dict(B=0), dict(heads=0), dict(Nq=0), dict(Nk=0, Nkpad=0), dict(Nkpad=132), dict(Nk=130, Nkpad=128)):
        assert _refused(L, attn(**kw), "adb_attention_bf16: bad sizes"), kw
    assert _refused(L, attn(Vt_hi=None), "adb_attention_bf16: null pointer")
    assert _refused(L, attn(O_hi=None), "adb_attention_bf16: null pointer")
    for kw in (dict(Q_lo=p16), dict(Q_lo=p16, K_lo=p16), dict(Vt_lo=p16), dict(K_lo=p16, Vt_lo=p16)):
        assert _refused(L, attn(**kw), "give all lo operands or none"), kw
    assert _refused(L, attn(O_hi=p8), "outputs must be 16-byte aligned")
    for kw in (dict(Q_hi=p8), dict(K_hi=p8), dict(Vt_hi=p8), dict(Q_lo=p16, K_lo=p16, Vt_lo=p8)):
        assert _refused(L, attn(**kw), "adb_attention_bf16: operands must be 16-byte aligned"), kw

    sv = L.adb_attention_set_variant
    prev = sv(1)
    try:
        assert prev in (0, 1, 2)
        for bad in (3, -1, 100):
            assert sv(bad) == -1
        assert sv(2) == 1, "a refused variant must leave the setting alone"
    finally:
        sv(prev)


def test_exact_operand_reference_is_the_three_documented_terms():
    """bf16x3 reference = A_hi B_hi^T + A_hi B_lo^T + A_lo B_hi^T: it differs from (A_hi + A_lo)(B_hi + B_lo)^T by exactly
    A_lo B_lo^T; the bound is the same sum over absolute values; batched operands broadcast."""
    g = gen("cpu", 0)
    ah, al = pos_operand((3, 5, 40), g, True, sign_dim=1)
    bh, bl = pos_operand((3, 7, 40), g, True, sign_dim=1)
    r, b = gemm_exact_ref(ah, al, bh, bl)
    full = (ah.double() + al.double()) @ (bh.double() + bl.double()).mT
    assert torch.allclose(full - r, al.double() @ bl.double().mT, rtol=0, atol=1e-12)
    assert torch.allclose(b, r.abs(), rtol=1e-12)            # row signs only: the terms of a dot product never cancel
    r1, b1 = gemm_exact_ref(ah, None, bh, None)
    assert torch.equal(r1, ah.double() @ bh.double().mT) and torch.allclose(b1, r1.abs(), rtol=1e-12)
    hi, lo = split(torch.randn(1000, generator=g))
    assert torch.equal(joined(hi, lo).double(), hi.double() + lo.double())     # hi + lo is exact in fp32


def test_selection_builder_addresses_every_column():
    g = gen("cpu", 1)
    for M, K in ((600, 520), (4200, 4104), (1, 8), (129, 72), (5, 4104)):
        idx = selection_indices(M, K, g)
        assert idx.shape == (M,) and int(idx.min()) >= 0 and int(idx.max()) == K - 1
        if M >= K:
            assert idx.unique().numel() == K
        a = selection_matrix(idx, K)
        b = torch.randn(3, K, generator=g).to(BF16)
        r, _ = gemm_exact_ref(a, None, b, None)
        assert torch.equal(r, b.double()[:, idx].T)


def test_batched_offsets_are_the_kernel_addressing():
    off = matrix_offsets(6, 4, 5, 20, s=5, zdiv=3, s2=100)
    assert off[4, 2, 3].item() == 1 * 100 + 1 * 5 + 2 * 20 + 3
    assert off.unique().numel() == off.numel()
    assert matrix_offsets(3, 2, 2, 2, s=4)[2, 1, 1].item() == 2 * 4 + 2 + 1


def test_vector_store_predicate_gates_on_every_leading_dimension():
    """ldo gates the 256-bit path even for a D-only call: ldd = ldr = ldo = 200 is scalar, ldo = 208 vector."""
    assert not vector_store_path(200, 200, 200, [1024, 0, 0, 0])
    assert vector_store_path(200, 200, 208, [1024, 0, 0, 0])
    assert not vector_store_path(203, 200, 208, [1024, 0, 0, 0])
    assert not vector_store_path(200, 200, 208, [1028, 0, 0, 0])             # misaligned D
    assert not vector_store_path(224, 72, 80, [1024, 512, 512, 1024], obase=8)


def test_one_hot_tap_conv_reference_is_a_shift():
    g = gen("cpu", 2)
    for B, H, W, C in ((2, 1, 1, 8), (1, 3, 5, 16), (2, 5, 4, 8)):
        x = torch.randn(B, H, W, C, generator=g).to(BF16)
        got = conv64(x, one_hot_tap_weight(C, "cpu"))
        assert torch.equal(got, shifted_taps(x.double()))
        # tap (1, 1) is the identity; the output blocks differ from the unshifted input everywhere else
        assert torch.equal(got[..., 4 * C:5 * C], x.double())


def test_conv_reference_bands_and_bug_models():
    """A band of the fp64 reference equals the same rows of the whole-image conv; the wrapped border differs only at the
    border; the weight layout is tap-major with zero-padded channels; a positive-operand case discriminates every conv
    bug model by far more than 10x the tolerance."""
    g = gen("cpu", 3)
    B, H, W, Cin, Cout = 2, 9, 7, 72, 5
    xh, xl = pos_operand((B, H, W, Cin), g, True)
    wh, wl = pos_operand((Cout, Cin, 3, 3), g, True, sign_dim=0)
    full, bnd = conv_exact_ref(xh, xl, wh, wl)
    band, _ = conv_exact_ref(xh, xl, wh, wl, 3, 6)
    assert torch.allclose(band, full[:, 3:6], rtol=1e-13, atol=0)
    wrapped, _ = conv_exact_ref(xh, xl, wh, wl, wrap=True)
    assert torch.allclose(wrapped[:, 1:-1, 1:-1], full[:, 1:-1, 1:-1], rtol=1e-13, atol=0)
    for name, bug in _conv_bug_models(xh, xl, wh, wl, Cin, 0, H, True):
        assert nerr(bug, full, bnd) >= 10 * TOL_CONV[True], name
    wp = prep_conv_weight(wh)
    assert wp.shape == (Cout, 9 * 128)
    assert torch.equal(wp.view(Cout, 3, 3, 128)[..., :Cin], wh.permute(0, 2, 3, 1))
    assert not wp.view(Cout, 3, 3, 128)[..., Cin:].any()
    assert conv_tile(1) == (8, 16) and conv_tile(9) == (8, 16) and conv_tile(24) == (16, 8) and conv_tile(200) == (128, 1)
    assert _bands(384, 96, 2) == [(0, 2), (191, 193), (382, 384)] and _bands(3, 5, 1) == [(0, 3)]


def test_gemm_bug_models_are_far_outside_the_tolerance():
    g = gen("cpu", 4)
    for M, N, K in ((4, 6, 72), (3, 5, 520), (2, 3, 4104)):
        for x3 in (True, False):
            ah, al = pos_operand((M, K), g, x3, sign_dim=0)
            bh, bl = pos_operand((N, K), g, x3, sign_dim=0)
            ref, bnd = gemm_exact_ref(ah, al, bh, bl)
            for name, bug in _gemm_bug_models(ah, al, bh, bl, ref, K, x3):
                assert nerr(bug, ref, bnd) >= 10 * TOL_GEMM[x3], (M, N, K, x3, name)


def test_dpt_conv_shapes_follow_the_model():
    s = dpt_conv3x3_shapes(384, 512)
    by_name = {n: (h, w, ci, co) for n, h, w, ci, co in s}
    assert by_name["scratch.layer1_rn"] == (96, 128, 96, 256)
    assert by_name["scratch.layer4_rn"] == (12, 16, 768, 256)
    assert by_name["head.2"] == (384, 512, 128, 128)
    assert {w for _, _, w, _, _ in dpt_conv3x3_shapes(512, 384)} >= {24, 48, 96, 192, 384}


def test_attention_reference_one_hot_mask_and_bug_models():
    """attn_exact_ref: zero keys give the mean of the valid values; a one-hot row gives the addressed value; the
    pass-1-max-over-padded-keys model underflows to NaN where every logit is very negative."""
    g = gen("cpu", 5)
    BH, Nq, Nk = 2, 3, 10
    qh, ql = split(torch.randn(BH, Nq, 64, generator=g))
    kh = torch.zeros(BH, Nk, 64, dtype=BF16)
    vh, vl = pos_operand((BH, Nk, 64), g, True, sign_dim=2)
    o, b = attn_exact_ref(qh, ql, kh, torch.zeros_like(kh), vh, vl, 0.125, True)
    assert torch.allclose(o, join64(vh, vl).mean(1, keepdim=True).expand_as(o), rtol=1e-12, atol=0)
    k = torch.randn(BH, Nk, 64, generator=g)
    k = k / k.norm(dim=-1, keepdim=True)
    q = 2000.0 * k[:, [7, 2, 9]]
    (qh, ql), (kh, kl) = split(q), split(k)
    o, _ = attn_exact_ref(qh, ql, kh, kl, vh, vl, 0.125, True)
    want = join64(vh, vl)[:, [7, 2, 9]]
    assert torch.allclose(o, want, rtol=2.0 ** -14, atol=0)
    qn = -960.0 * k[:, :1].expand(BH, Nq, 64)
    (qh, ql) = split(qn)
    o, _ = attn_exact_ref(qh, ql, kh, kl, vh, vl, 0.125, True)
    assert torch.isfinite(o).all()
    # (keys near one direction, so all logits are near -120: shifting by 0 flushes every p)
    u = k[:, :1]
    kk = u + 0.01 * torch.randn(BH, Nk, 64, generator=g)
    kk = kk / kk.norm(dim=-1, keepdim=True)
    (kh, kl), (qh, ql) = split(kk), split(-960.0 * u.expand(BH, Nq, 64).contiguous())
    ref, bnd = attn_exact_ref(qh, ql, kh, kl, vh, vl, 0.125, True)
    bug, _ = attn_exact_ref(qh, ql, kh, kl, vh, vl, 0.125, True, m_floor=0.0)
    assert torch.isfinite(ref).all() and nerr(bug, ref, bnd) == math.inf

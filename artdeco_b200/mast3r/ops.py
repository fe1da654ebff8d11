"""Thin wrappers over the C ABI for the MASt3R path: tensor-core GEMM (bf16 / bf16x3) and its memory-bound
companions.  A "split" activation is a pair of bf16 tensors (hi, lo) with x ~= hi + lo; every producer kernel writes
the pair directly so GEMM operands never make a separate conversion pass."""
from __future__ import annotations

import ctypes as C

import torch

from .. import _lib
from .._lib import f32, i32, i64, vp

_lib.register("adb_gemm_bf16", [i32, i32, i32, i32, vp, vp, i64, i64, vp, vp, i64, i64, vp, i64, i64, vp, vp, i64, i64,
                                vp, vp, i64, i64, f32, i32, i32, i64, i64, i64, vp])
_lib.register("adb_conv3x3_bf16", [i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, vp])
_lib.register("adb_attention_bf16", [i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, f32, vp, vp, vp])
_lib.register("adb_attention_set_variant", [i32])
_lib.register("adb_layernorm", [i64, i32, vp, vp, vp, f32, vp, vp, vp, vp])
_lib.register("adb_split_bf16", [i64, vp, vp, vp, vp])
_lib.register("adb_rope_heads", [i32, i32, i32, i64, i32, vp, vp, vp, i32, i32, i32, vp, vp, vp])
_lib.register("adb_softmax_rows", [i64, i32, i64, i64, vp, vp, vp, vp])
_lib.register("adb_im2col_patch16", [i32, i32, i32, vp, vp, vp, vp])
_lib.register("adb_upsample2x_nhwc", [i32, i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp])
_lib.register("adb_head_postprocess", [i32, i32, i32, vp, vp, i64, i32, vp, vp, vp, vp, vp])

BF16 = torch.bfloat16


class Split:
    """bf16 (hi, lo) pair; lo is None in single-pass bf16 mode."""
    __slots__ = ("hi", "lo")

    def __init__(self, hi, lo):
        self.hi, self.lo = hi, lo

    @property
    def shape(self):
        return self.hi.shape


def split(x: torch.Tensor, x3: bool = True) -> Split:
    x = x.contiguous()
    hi = torch.empty(x.shape, dtype=BF16, device=x.device)
    lo = torch.empty(x.shape, dtype=BF16, device=x.device) if x3 else None
    _lib.call("adb_split_bf16", x.numel(), _lib.ptr(x, torch.float32), _lib.ptr(hi), _lib.ptr(lo), _lib.stream())
    return Split(hi, lo)


def gemm(a: Split, w: Split, M: int, N: int, K: int, *, batch: int = 1, lda=None, sA=0, ldb=None, sB=0,
         out: torch.Tensor | None = None, ldd=None, sD=0, out_split: Split | None = None, ldo=None, sO=0,
         bias=None, residual=None, ldr=None, sR=0, alpha: float = 1.0, act: int = 0,
         zdiv: int = 0, sD2=0, sO2=0, sR2=0) -> None:
    """D = act(alpha * A @ W^T + bias) + residual, A: [batch, M, K], W: [batch, N, K] (both K-contiguous bf16)."""
    lda = K if lda is None else lda
    ldb = K if ldb is None else ldb
    ldd = N if ldd is None else ldd
    ldo = N if ldo is None else ldo
    ldr = N if ldr is None else ldr
    if batch > 1 and sB == 0:
        raise ValueError("broadcast weights over a batch: fold the batch into M")
    x3 = a.lo is not None and w.lo is not None
    _lib.call("adb_gemm_bf16", batch, M, N, K, _lib.ptr(a.hi), _lib.ptr(a.lo) if x3 else None, lda, sA,
              _lib.ptr(w.hi), _lib.ptr(w.lo) if x3 else None, ldb, sB,
              _lib.ptr(out) if out is not None else None, ldd, sD,
              _lib.ptr(out_split.hi) if out_split is not None else None,
              _lib.ptr(out_split.lo) if (out_split is not None and out_split.lo is not None) else None, ldo, sO,
              _lib.ptr(bias) if bias is not None else None,
              _lib.ptr(residual) if residual is not None else None, ldr, sR, float(alpha), int(act),
              int(zdiv), sD2, sO2, sR2, _lib.stream())


def linear(a: Split, w: Split, bias, rows: int, *, act: int = 0, residual=None, want_fp32=True, want_split=False,
           x3=True):
    """nn.Linear on a [rows, K] split activation; returns (fp32 [rows, N] or None, Split or None)."""
    N, K = w.hi.shape
    dev = a.hi.device
    out = torch.empty(rows, N, dtype=torch.float32, device=dev) if want_fp32 else None
    sp = None
    if want_split:
        sp = Split(torch.empty(rows, N, dtype=BF16, device=dev), torch.empty(rows, N, dtype=BF16, device=dev) if x3 else None)
    gemm(a, w, rows, N, K, out=out, out_split=sp, bias=bias, residual=residual, act=act)
    return out, sp


def layernorm(x: torch.Tensor, gamma, beta, eps: float = 1e-6, want_fp32=False, want_split=True, x3=True):
    C = x.shape[-1]
    rows = x.numel() // C
    x = x.contiguous()
    y = torch.empty_like(x) if want_fp32 else None
    sp = None
    if want_split:
        sp = Split(torch.empty(x.shape, dtype=BF16, device=x.device),
                   torch.empty(x.shape, dtype=BF16, device=x.device) if x3 else None)
    _lib.call("adb_layernorm", rows, C, _lib.ptr(x, torch.float32), _lib.ptr(gamma), _lib.ptr(beta), float(eps),
              _lib.ptr(y) if y is not None else None, _lib.ptr(sp.hi) if sp else None,
              _lib.ptr(sp.lo) if (sp and sp.lo is not None) else None, _lib.stream())
    return y, sp


ROPE_TABLE_POSITIONS = 64      # patch positions per axis in the (cos, sin) table (1024 px at patch 16); n_pos default below
_rope_tables: dict = {}


def rope_table(n_pos: int, device, base: float = 100.0) -> torch.Tensor:
    """(cos, sin) of p * base^(-2i/32), p < n_pos, i < 16 — computed with the reference's own fp32 expressions
    (croco/models/pos_embed.py:118-127) so the rotation angles are the same numbers."""
    key = (n_pos, str(device), base)
    if key not in _rope_tables:
        D = 32
        inv_freq = 1.0 / (base ** (torch.arange(0, D, 2).float().to(device) / D))
        t = torch.arange(n_pos, device=device, dtype=inv_freq.dtype)
        freqs = torch.einsum("i,j->ij", t, inv_freq)
        _rope_tables[key] = torch.stack([freqs.cos(), freqs.sin()], -1).contiguous()
    return _rope_tables[key]


def rope_heads(x: torch.Tensor, B, N, h, ld, col0, pos, mode: int, base: float = 100.0, x3=True, Npad=None, n_pos: int = 64) -> Split:
    dev = x.device
    Npad = N if Npad is None else Npad
    shape = (B, h, 64, Npad) if mode == 2 else (B, h, N, 64)
    hi = torch.empty(shape, dtype=BF16, device=dev)
    lo = torch.empty(shape, dtype=BF16, device=dev) if x3 else None
    table = rope_table(n_pos, dev, base) if mode == 0 else None
    _lib.call("adb_rope_heads", B, N, h, ld, col0, _lib.ptr(x, torch.float32),
              _lib.ptr(pos, torch.int64) if pos is not None else None, _lib.ptr(table) if table is not None else None,
              n_pos, mode, Npad, _lib.ptr(hi), _lib.ptr(lo), _lib.stream())
    return Split(hi, lo)


_lib.register("adb_gemm_bf16_rope", [i32, i32, i32, vp, vp, i64, vp, vp, i64, vp, i32, i32, i32, vp, vp, i32, vp, vp, vp, vp,
                                     vp, i64, vp])


def linear_rope(a: Split, w: Split, bias, B: int, N: int, h: int, pos, n_dst: int, x3=True, base: float = 100.0,
                n_pos: int = 64):
    """Linear + RoPE2D + head split in the GEMM epilogue (adb_gemm_bf16_rope).  The weight's first ``n_dst * h*64`` output
    rows are attention heads (q, then k); returns (q Split [B,h,N,64], k Split | None, tail fp32 [B*N, rest] | None)."""
    Nout, K = w.hi.shape
    C = h * 64
    dev = a.hi.device
    def heads():
        return Split(torch.empty(B, h, N, 64, dtype=BF16, device=dev),
                     torch.empty(B, h, N, 64, dtype=BF16, device=dev) if x3 else None)
    q = heads()
    k = heads() if n_dst == 2 else None
    rest = Nout - n_dst * C
    tail = torch.empty(B * N, rest, dtype=torch.float32, device=dev) if rest > 0 else None
    table = rope_table(n_pos, dev, base)
    use3 = a.lo is not None and w.lo is not None
    _lib.call("adb_gemm_bf16_rope", B * N, Nout, K, _lib.ptr(a.hi), _lib.ptr(a.lo) if use3 else None, K,
              _lib.ptr(w.hi), _lib.ptr(w.lo) if use3 else None, K, _lib.ptr(bias) if bias is not None else None, N, h, n_dst,
              _lib.ptr(pos, torch.int64), _lib.ptr(table), n_pos, _lib.ptr(q.hi), _lib.ptr(q.lo),
              _lib.ptr(k.hi) if k is not None else None, _lib.ptr(k.lo) if k is not None else None,
              _lib.ptr(tail) if tail is not None else None, max(rest, 1), _lib.stream())
    return q, k, tail


def softmax_rows(s: torch.Tensor, rows: int, L: int, ld_in: int, x3=True) -> Split:
    dev = s.device
    hi = torch.empty(rows, L, dtype=BF16, device=dev)
    lo = torch.empty(rows, L, dtype=BF16, device=dev) if x3 else None
    _lib.call("adb_softmax_rows", rows, L, ld_in, L, _lib.ptr(s, torch.float32), _lib.ptr(hi), _lib.ptr(lo), _lib.stream())
    return Split(hi, lo)


def im2col_patch16(img: torch.Tensor, x3=True) -> Split:
    B, C, H, W = img.shape
    assert C == 3
    n = (H // 16) * (W // 16)
    hi = torch.empty(B * n, 768, dtype=BF16, device=img.device)
    lo = torch.empty(B * n, 768, dtype=BF16, device=img.device) if x3 else None
    _lib.call("adb_im2col_patch16", B, H, W, _lib.ptr(img.contiguous(), torch.float32), _lib.ptr(hi), _lib.ptr(lo), _lib.stream())
    return Split(hi, lo)


def prep_conv3x3_weight(w: torch.Tensor, x3=True) -> Split:
    """[Cout, Cin, 3, 3] fp32 -> bf16 split [Cout, 9 * Cin_pad] in (ky, kx, ci) order, Cin zero-padded to 64."""
    Cout, Cin = w.shape[0], w.shape[1]
    cpad = (Cin + 63) // 64 * 64
    wp = torch.zeros(Cout, 3, 3, cpad, dtype=torch.float32, device=w.device)
    wp[..., :Cin] = w.permute(0, 2, 3, 1)
    return split(wp.reshape(Cout, 9 * cpad), x3)


def conv3x3(x: Split, B: int, H: int, W: int, Cin: int, w: Split, bias, Cout: int, *, residual=None, act: int = 0,
            want_fp32=True, want_split=False, split_relu=False, x3=True):
    """NHWC 3x3 conv on the tensor-core kernel.  Returns (fp32 [B,H,W,Cout] or None, Split [B,H,W,Cout] or None)."""
    dev = x.hi.device
    out = torch.empty(B, H, W, Cout, dtype=torch.float32, device=dev) if want_fp32 else None
    sp = None
    if want_split:
        sp = Split(torch.empty(B, H, W, Cout, dtype=BF16, device=dev),
                   torch.empty(B, H, W, Cout, dtype=BF16, device=dev) if x3 else None)
    use3 = x.lo is not None and w.lo is not None
    _lib.call("adb_conv3x3_bf16", B, H, W, Cin, Cout, _lib.ptr(x.hi), _lib.ptr(x.lo) if use3 else None, _lib.ptr(w.hi),
              _lib.ptr(w.lo) if use3 else None, _lib.ptr(bias) if bias is not None else None,
              _lib.ptr(residual) if residual is not None else None, _lib.ptr(out) if out is not None else None,
              _lib.ptr(sp.hi) if sp is not None else None,
              _lib.ptr(sp.lo) if (sp is not None and sp.lo is not None) else None, int(act), int(split_relu), _lib.stream())
    return out, sp


def upsample2x(x: torch.Tensor, addend: torch.Tensor | None = None, out_hw=None, want_fp32=True, want_split=False, x3=True):
    """Bilinear x2 (align_corners=True) of an NHWC fp32 tensor [B,H,W,C], + ``addend`` [B,Ho,Wo,C], cropped to ``out_hw``.
    Returns (fp32 [B,Ho,Wo,C] or None, Split or None)."""
    B, H, W, Cc = x.shape
    Ho, Wo = (2 * H, 2 * W) if out_hw is None else out_hw
    x = x.contiguous()
    if addend is not None:
        addend = addend.contiguous()
        assert addend.shape == (B, Ho, Wo, Cc)
    y = torch.empty(B, Ho, Wo, Cc, dtype=torch.float32, device=x.device) if want_fp32 else None
    sp = None
    if want_split:
        sp = Split(torch.empty(B, Ho, Wo, Cc, dtype=BF16, device=x.device),
                   torch.empty(B, Ho, Wo, Cc, dtype=BF16, device=x.device) if x3 else None)
    _lib.call("adb_upsample2x_nhwc", B, H, W, Cc, Ho, Wo, _lib.ptr(x, torch.float32), _lib.ptr(addend), _lib.ptr(y),
              _lib.ptr(sp.hi) if sp is not None else None, _lib.ptr(sp.lo) if (sp is not None and sp.lo is not None) else None,
              _lib.stream())
    return y, sp


def head_postprocess(pts: torch.Tensor, lf: torch.Tensor, H: int, W: int, n_desc: int = 24):
    """pts [B,H,W,4] fp32 (DPT map), lf [B*S, (n_desc+1)*256] fp32 (local-feature MLP output before pixel_shuffle) ->
    dict(pts3d, conf, desc, desc_conf) as mast3r/catmlp_dpt_head.py:25-39 returns it."""
    B = pts.shape[0]
    dev = pts.device
    pts, lf = pts.contiguous(), lf.contiguous()
    res = dict(pts3d=torch.empty(B, H, W, 3, dtype=torch.float32, device=dev),
               conf=torch.empty(B, H, W, dtype=torch.float32, device=dev),
               desc=torch.empty(B, H, W, n_desc, dtype=torch.float32, device=dev),
               desc_conf=torch.empty(B, H, W, dtype=torch.float32, device=dev))
    _lib.call("adb_head_postprocess", B, H, W, _lib.ptr(pts, torch.float32), _lib.ptr(lf, torch.float32), lf.shape[-1], n_desc,
              _lib.ptr(res["pts3d"]), _lib.ptr(res["conf"]), _lib.ptr(res["desc"]), _lib.ptr(res["desc_conf"]), _lib.stream())
    return res


def set_attention_variant(variant: int) -> int:
    """0 = automatic (default), 1 / 2 force a kernel variant (csrc/attn_tc.cu).  Returns the previous setting."""
    prev = _lib.lib().adb_attention_set_variant(C.c_int(int(variant)))   # returns the previous value, not a status
    if prev < 0:
        raise ValueError("attention variant must be 0, 1 or 2")
    return prev


def attention(q: Split, k: Split, vt: Split, B: int, h: int, Nq: int, Nk: int, Nkpad: int, scale: float, x3=True) -> Split:
    """Fused softmax(scale * q k^T) v on wgmma (S/P stay in registers).  q,k: [B,h,N,64]; vt: [B,h,64,Nkpad];
    returns the bf16 split of the head-merged output [B*Nq, h*64]."""
    dev = q.hi.device
    C = h * 64
    o = Split(torch.empty(B * Nq, C, dtype=BF16, device=dev), torch.empty(B * Nq, C, dtype=BF16, device=dev) if x3 else None)
    use3 = x3 and q.lo is not None and k.lo is not None and vt.lo is not None
    _lib.call("adb_attention_bf16", B, h, Nq, Nk, Nkpad, _lib.ptr(q.hi), _lib.ptr(q.lo) if use3 else None, _lib.ptr(k.hi),
              _lib.ptr(k.lo) if use3 else None, _lib.ptr(vt.hi), _lib.ptr(vt.lo) if use3 else None, float(scale),
              _lib.ptr(o.hi), _lib.ptr(o.lo) if (use3 and o.lo is not None) else None, _lib.stream())
    return o

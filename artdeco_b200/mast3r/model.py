"""Host-side mirror of the reference's ``AsymmetricMASt3R`` for inference
(VSLAM/thirdparty/mast3r/mast3r/model.py:40-68, dust3r/dust3r/model.py:46-211): same constructor defaults as the
checkpoint ARTDECO loads (ViT-L encoder, 12+12 ViT-B decoder blocks, catmlp+dpt heads, pts3d+desc24), same
``state_dict`` key names, and the three internals ARTDECO actually drives — ``_encode_image``, ``_decoder``,
``_downstream_head`` (VSLAM/utils_mast3r.py:30-36,127,132,179) — plus ``forward``.

Every dense contraction of the transformer and of the local-feature MLP runs on the wgmma GEMM
(csrc/gemm_tc.cu) with fused bias/GELU/residual epilogues; LayerNorm, RoPE + head split, softmax and the patch
im2col are hand-written companion kernels (csrc/vit_ops.cu).  ``precision``:
  "bf16x3" (default)  three-term split product, fp32-class accuracy (meets the 1e-4 pointmap tolerance)
  "bf16"              single pass, ~3x less tensor work, ~1e-2 accuracy (NOT within the stated tolerance)
The DPT convolution stack (croco/models/dpt_block.py) runs on the same kernel in its implicit-GEMM conv mode (NHWC
activations, 4-D TMA boxes); torch is left with the bilinear upsampling and a few reshapes.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .. import _lib
from . import ops
from .ops import Split

FULL_CFG = dict(enc_embed_dim=1024, enc_depth=24, enc_num_heads=16, dec_embed_dim=768, dec_depth=12, dec_num_heads=12)


class _PatchEmbedInfo:
    def __init__(self, patch_size=16):
        self.patch_size = (patch_size, patch_size)


def _roundup(v, m):
    return (v + m - 1) // m * m


class AsymmetricMASt3R:
    def __init__(self, precision: str = "bf16x3", **cfg):
        c = dict(FULL_CFG)
        c.update({k: v for k, v in cfg.items() if k in FULL_CFG})
        self.cfg = c
        for k, v in c.items():
            setattr(self, k, v)
        if precision not in ("bf16x3", "bf16"):
            raise ValueError("precision must be 'bf16x3' or 'bf16'")
        self.precision = precision
        self.x3 = precision == "bf16x3"
        import os
        self._fused_attn = os.environ.get("ADB_ATTN", "fused") != "materialized"
        # RoPE + head split in the qkv / projq / projkv GEMM epilogue (ADB_ROPE=separate keeps the standalone kernel for A/B)
        self._fused_rope = os.environ.get("ADB_ROPE", "fused") != "separate"
        self.patch_embed = _PatchEmbedInfo(16)
        self.device = torch.device("cpu")
        self._sd = None          # fp32 tensors (LN params, biases, conv weights)
        self._w = {}             # name -> Split (bf16 hi/lo GEMM weights)
        self._streams = {}
        self.concurrent = True   # run the two decoder sides / two heads on two CUDA streams
        if any(d % 64 for d in (c["enc_embed_dim"] // c["enc_num_heads"], c["dec_embed_dim"] // c["dec_num_heads"])):
            raise ValueError("head_dim must be 64")

    # ---- nn.Module-like surface the callers use -------------------------------------------------
    # The reference hands the model object around: Frontend.py:29-30 (``load_mast3r(...)`` then ``.share_memory()`` before the
    # tracker / backend processes are spawned), retrieval/model.py:123 (``for p in backbone.parameters(): p.requires_grad =
    # False``), :200 (``backbone._encode_image``), mast3r/model.py:21-37 (``load_state_dict(ckpt['model'], strict=False)`` +
    # ``.to(device)``).  This class is not an nn.Module (its weights live as bf16 splits behind a C ABI), so those entry
    # points are provided explicitly with the same semantics.
    def eval(self):
        return self

    def train(self, mode: bool = True):
        if mode:
            raise NotImplementedError("AsymmetricMASt3R (artdeco_b200) is inference-only, as every ARTDECO call site is")
        return self

    def requires_grad_(self, requires_grad: bool = False):
        for p in self.parameters():
            p.requires_grad = requires_grad
        return self

    def share_memory(self):
        """nn.Module.share_memory(): host tensors move to shared memory; CUDA tensors are left alone — exactly torch's
        behaviour (``Tensor.share_memory_`` is a no-op for CUDA storage; they cross process boundaries as CUDA IPC handles
        when the object is pickled by torch.multiprocessing, which ``__getstate__`` below supports)."""
        for v in getattr(self, "_raw", {}).values():
            if not v.is_cuda:
                v.share_memory_()
        return self

    def named_parameters(self, prefix: str = "", recurse: bool = True):
        for k, v in self._param_objs().items():
            yield (prefix + ("." if prefix else "") + k, v)

    def parameters(self, recurse: bool = True):
        for _, v in self.named_parameters():
            yield v

    def state_dict(self, *args, **kwargs):
        """fp32 tensors under the reference's key names (1017 keys for the ViT-L checkpoint, SURVEY.md App. A)."""
        from collections import OrderedDict
        return OrderedDict((k, v) for k, v in getattr(self, "_raw", {}).items())

    def _param_objs(self):
        if getattr(self, "_params", None) is None:
            self._params = {k: torch.nn.Parameter(v, requires_grad=False) for k, v in getattr(self, "_raw", {}).items()}
        return self._params

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_streams"] = {}                 # CUDA streams are per process
        st["_params"] = None
        return st

    def __setstate__(self, st):
        self.__dict__.update(st)

    def to(self, device):
        self.device = torch.device(device)
        if self._sd is not None:
            self._prepare()
        return self

    def cuda(self, index=0):
        return self.to(torch.device("cuda", index))

    @classmethod
    def from_pretrained(cls, path, **kw):
        """Checkpoint layout of mast3r/model.py:21-37: a dict with 'model' (state dict) and 'args' (whose ``.model`` string
        names the constructor call; only the sizes are read from it, the class is always this one)."""
        ckpt = torch.load(path, map_location="cpu", weights_only=False)
        sd = ckpt["model"] if "model" in ckpt else ckpt
        cfg = dict(kw)
        args = ckpt.get("args") if isinstance(ckpt, dict) else None
        spec = getattr(args, "model", args if isinstance(args, str) else None)
        if isinstance(spec, str):
            import re
            for key in FULL_CFG:
                m = re.search(rf"{key}\s*=\s*(\d+)", spec)
                if m and key not in cfg:
                    cfg[key] = int(m.group(1))
        m = cls(**cfg)
        m.load_state_dict(sd, strict=False)
        return m

    def load_state_dict(self, sd, strict: bool = False):
        sd = dict(sd)
        if not any(k.startswith("dec_blocks2") for k in sd):   # dust3r/model.py:90-97
            for k, v in list(sd.items()):
                if k.startswith("dec_blocks."):
                    sd[k.replace("dec_blocks.", "dec_blocks2.", 1)] = v
        self._raw = {k: v.detach().float() for k, v in sd.items()}
        self._params = None
        self._sd = None
        if self.device.type == "cuda":
            self._prepare()
        else:
            self._sd = {}
        return self

    def _prepare(self):
        _lib.require_cuda()
        dev = self.device
        raw = self._raw
        self._sd, self._w = {}, {}
        for k, v in raw.items():
            is_gemm_w = (v.dim() == 2 and k.endswith(".weight")) or k == "patch_embed.proj.weight"
            if is_gemm_w:
                w2 = v.reshape(v.shape[0], -1).contiguous().to(dev)
                self._w[k] = ops.split(w2, self.x3)
            elif v.dim() == 4 and ".dpt." in k and k.endswith(".weight"):
                if ".act_postprocess." in k and k.endswith(".1.weight") and v.shape[-1] in (2, 4):
                    # ConvTranspose2d [Cin, Cout, k, k] -> linear weight [(co, i, j), ci]
                    wt = v.to(dev).permute(1, 2, 3, 0).reshape(-1, v.shape[0]).contiguous()
                    self._w[k] = ops.split(wt, self.x3)
                    bname = k[:-len(".weight")] + ".bias"     # one bias value per (cout, i, j) GEMM column
                    if bname in raw:
                        self._sd[bname + "_cols"] = raw[bname].float().repeat_interleave(v.shape[-1] * v.shape[-2]).contiguous().to(dev)
                elif v.shape[-1] == 3:
                    self._w[k] = ops.prep_conv3x3_weight(v.to(dev), self.x3)
                else:  # 1x1
                    self._w[k] = ops.split(v.to(dev).reshape(v.shape[0], v.shape[1]).contiguous(), self.x3)
            else:
                self._sd[k] = v.contiguous().to(dev)
        # fused projk|projv weights for cross attention
        for blk in ("dec_blocks", "dec_blocks2"):
            for i in range(self.cfg["dec_depth"]):
                p = f"{blk}.{i}.cross_attn"
                if p + ".projk.weight" in raw:
                    wkv = torch.cat([raw[p + ".projk.weight"], raw[p + ".projv.weight"]], 0).contiguous().to(dev)
                    self._w[p + ".projkv.weight"] = ops.split(wkv, self.x3)
                    self._sd[p + ".projkv.bias"] = torch.cat([raw[p + ".projk.bias"], raw[p + ".projv.bias"]]).to(dev)

    def _side_stream(self, device):
        key = torch.device(device).index
        if key not in self._streams:
            self._streams[key] = torch.cuda.Stream(device=device)
        return self._streams[key]

    # ---- building blocks ------------------------------------------------------------------------
    def _linear(self, a: Split, name: str, rows: int, **kw):
        return ops.linear(a, self._w[name + ".weight"], self._sd.get(name + ".bias"), rows, x3=self.x3, **kw)

    def _ln(self, x, name, **kw):
        return ops.layernorm(x, self._sd[name + ".weight"], self._sd[name + ".bias"], 1e-6, x3=self.x3, **kw)

    def _attn_core(self, q: Split, k: Split, vt: Split, B, h, Nq, Nk, Nkpad) -> Split:
        """softmax(q k^T / 8) v, fused (csrc/attn_tc.cu); ADB_ATTN=materialized selects the three-kernel path kept for A/B."""
        if self._fused_attn:
            return ops.attention(q, k, vt, B, h, Nq, Nk, Nkpad, 64 ** -0.5, x3=self.x3)
        dev = q.hi.device
        s = torch.empty(B * h, Nq, Nk, dtype=torch.float32, device=dev)
        ops.gemm(q, k, Nq, Nk, 64, batch=B * h, sA=Nq * 64, sB=Nk * 64, out=s, sD=Nq * Nk, alpha=64 ** -0.5)
        hi = torch.zeros(B * h * Nq, Nkpad, dtype=torch.bfloat16, device=dev) if Nkpad != Nk else \
            torch.empty(B * h * Nq, Nkpad, dtype=torch.bfloat16, device=dev)
        lo = (torch.zeros_like(hi) if Nkpad != Nk else torch.empty_like(hi)) if self.x3 else None
        _lib.call("adb_softmax_rows", B * h * Nq, Nk, Nk, Nkpad, _lib.ptr(s), _lib.ptr(hi), _lib.ptr(lo), _lib.stream())
        p = Split(hi, lo)
        C = h * 64
        o = Split(torch.empty(B * Nq, C, dtype=torch.bfloat16, device=dev),
                  torch.empty(B * Nq, C, dtype=torch.bfloat16, device=dev) if self.x3 else None)
        ops.gemm(p, vt, Nq, 64, Nkpad, batch=B * h, sA=Nq * Nkpad, sB=64 * Nkpad, out_split=o, ldo=C, zdiv=h, sO=64,
                 sO2=Nq * C)
        return o

    def _self_attention(self, x, pos, pre, h):
        """x fp32 [B,N,C] -> x + proj(attn(norm1(x)))  (blocks.py:94-112,128)"""
        B, N, C = x.shape
        _, xn = self._ln(x, pre + ".norm1")
        Npad = _roundup(N, 8)
        if self._fused_rope:
            # q, k leave the qkv GEMM already rotated, head-major and split; only V (fp32 [B*N, C]) is written plainly
            q, k, v = ops.linear_rope(xn, self._w[pre + ".attn.qkv.weight"], self._sd.get(pre + ".attn.qkv.bias"), B, N, h,
                                      pos, 2, x3=self.x3)
            vt = ops.rope_heads(v, B, N, h, C, 0, None, 2, x3=self.x3, Npad=Npad)
        else:
            qkv, _ = self._linear(xn, pre + ".attn.qkv", B * N)
            q = ops.rope_heads(qkv, B, N, h, 3 * C, 0, pos, 0, x3=self.x3)
            k = ops.rope_heads(qkv, B, N, h, 3 * C, C, pos, 0, x3=self.x3)
            vt = ops.rope_heads(qkv, B, N, h, 3 * C, 2 * C, None, 2, x3=self.x3, Npad=Npad)
        o = self._attn_core(q, k, vt, B, h, N, N, Npad)
        out, _ = self._linear(o, pre + ".attn.proj", B * N, residual=x.reshape(B * N, C))
        return out.view(B, N, C)

    def _mlp(self, x, norm, pre):
        B, N, C = x.shape
        _, xn = self._ln(x, norm)
        _, hdn = self._linear(xn, pre + ".fc1", B * N, act=1, want_fp32=False, want_split=True)
        out, _ = self._linear(hdn, pre + ".fc2", B * N, residual=x.reshape(B * N, C))
        return out.view(B, N, C)

    def _block(self, x, pos, pre, h):
        x = self._self_attention(x, pos, pre, h)
        return self._mlp(x, pre + ".norm2", pre + ".mlp")

    def _dec_block(self, x, y, xpos, ypos, pre, h):
        """DecoderBlock.forward (blocks.py:186-191)."""
        B, N, C = x.shape
        Nk = y.shape[1]
        x = self._self_attention(x, xpos, pre, h)
        _, yn = self._ln(y, pre + ".norm_y")
        _, xn = self._ln(x, pre + ".norm2")
        Nkpad = _roundup(Nk, 8)
        if self._fused_rope:
            q, _, _ = ops.linear_rope(xn, self._w[pre + ".cross_attn.projq.weight"],
                                      self._sd.get(pre + ".cross_attn.projq.bias"), B, N, h, xpos, 1, x3=self.x3)
            k, _, v = ops.linear_rope(yn, self._w[pre + ".cross_attn.projkv.weight"],
                                      self._sd.get(pre + ".cross_attn.projkv.bias"), B, Nk, h, ypos, 1, x3=self.x3)
            vt = ops.rope_heads(v, B, Nk, h, C, 0, None, 2, x3=self.x3, Npad=Nkpad)
        else:
            qf, _ = self._linear(xn, pre + ".cross_attn.projq", B * N)
            kv, _ = self._linear(yn, pre + ".cross_attn.projkv", B * Nk)
            q = ops.rope_heads(qf, B, N, h, C, 0, xpos, 0, x3=self.x3)
            k = ops.rope_heads(kv, B, Nk, h, 2 * C, 0, ypos, 0, x3=self.x3)
            vt = ops.rope_heads(kv, B, Nk, h, 2 * C, C, None, 2, x3=self.x3, Npad=Nkpad)
        o = self._attn_core(q, k, vt, B, h, N, Nk, Nkpad)
        x2, _ = self._linear(o, pre + ".cross_attn.proj", B * N, residual=x.reshape(B * N, C))
        return self._mlp(x2.view(B, N, C), pre + ".norm3", pre + ".mlp")

    # ---- the reference surface ----------------------------------------------------------------
    @torch.no_grad()
    def _encode_image(self, image, true_shape=None):
        """dust3r/model.py:127-140 -> (x [B,n,E] fp32, pos [B,n,2] int64, None)."""
        _lib.require_cuda(image)
        B, _, H, W = image.shape
        if H % 16 or W % 16:
            raise AssertionError(f"Input image size ({H}x{W}) is not a multiple of patch size (16).")
        if max(H, W) // 16 > ops.ROPE_TABLE_POSITIONS:
            # the RoPE (cos, sin) table holds this many patch positions per axis; the kernels clamp beyond it, so refuse
            raise ValueError(f"image side {max(H, W)} px exceeds the {ops.ROPE_TABLE_POSITIONS * 16} px the RoPE table covers")
        E = self.cfg["enc_embed_dim"]
        n = (H // 16) * (W // 16)
        with torch.cuda.device(image.device):
            a = ops.im2col_patch16(image.float(), x3=self.x3)
            x, _ = ops.linear(a, self._w["patch_embed.proj.weight"], self._sd["patch_embed.proj.bias"], B * n, x3=self.x3)
            x = x.view(B, n, E)
            yy, xx = torch.arange(H // 16, device=image.device), torch.arange(W // 16, device=image.device)
            pos = torch.cartesian_prod(yy, xx).view(1, n, 2).expand(B, -1, 2).contiguous()
            for i in range(self.cfg["enc_depth"]):
                x = self._block(x, pos, f"enc_blocks.{i}", self.cfg["enc_num_heads"])
            x, _ = self._ln(x, "enc_norm", want_fp32=True, want_split=False)
        return x, pos, None

    @torch.no_grad()
    def _decoder(self, f1, pos1, f2, pos2):
        """dust3r/model.py:172-191 -> two tuples of 13 tensors (encoder output first, dec_norm'd last)."""
        B, N1, E = f1.shape
        N2 = f2.shape[1]
        Dd, h = self.cfg["dec_embed_dim"], self.cfg["dec_num_heads"]
        with torch.cuda.device(f1.device):
            out1, out2 = [f1], [f2]
            g1, _ = self._linear(ops.split(f1.reshape(B * N1, E), self.x3), "decoder_embed", B * N1)
            g2, _ = self._linear(ops.split(f2.reshape(B * N2, E), self.x3), "decoder_embed", B * N2)
            c1, c2 = g1.view(B, N1, Dd), g2.view(B, N2, Dd)
            # The two decoder sides of a layer only depend on the previous layer's pair, so they run concurrently on two
            # CUDA streams (at batch 1 each side's GEMMs fill less than half of the 132 SMs on their own).
            s1 = torch.cuda.current_stream()
            s2 = self._side_stream(f1.device)
            for i in range(self.cfg["dec_depth"]):
                if self.concurrent:
                    s2.wait_stream(s1)
                    with torch.cuda.stream(s2):
                        n2 = self._dec_block(c2, c1, pos2, pos1, f"dec_blocks2.{i}", h)
                    n1 = self._dec_block(c1, c2, pos1, pos2, f"dec_blocks.{i}", h)
                    s1.wait_stream(s2)
                else:
                    n1 = self._dec_block(c1, c2, pos1, pos2, f"dec_blocks.{i}", h)
                    n2 = self._dec_block(c2, c1, pos2, pos1, f"dec_blocks2.{i}", h)
                c1, c2 = n1, n2
                out1.append(c1)
                out2.append(c2)
            out1[-1], _ = self._ln(out1[-1], "dec_norm", want_fp32=True, want_split=False)
            out2[-1], _ = self._ln(out2[-1], "dec_norm", want_fp32=True, want_split=False)
        return tuple(out1), tuple(out2)

    # ---- DPT head (dust3r/heads/dpt_head.py:34-65, croco/models/dpt_block.py:79-218,356-410) ----------------
    # All 3x3 / 1x1 convolutions and both ConvTranspose layers run on the wgmma kernel (implicit GEMM over NHWC
    # activations); only the bilinear x2 upsampling (align_corners=True) and pixel rearrangements stay in torch.
    def _c3(self, x: Split, B, H, W, name, **kw):
        w = self._w[name + ".weight"]
        cin = x.hi.shape[-1]
        return ops.conv3x3(x, B, H, W, cin, w, self._sd.get(name + ".bias"), w.hi.shape[0], x3=self.x3, **kw)

    def _c1(self, x: Split, rows, name, **kw):
        return ops.linear(x, self._w[name + ".weight"], self._sd.get(name + ".bias"), rows, x3=self.x3, **kw)

    def _rcu(self, x_f32, x_relu: Split, B, H, W, pre, residual=None, out_fp32=True, out_relu_split=False,
             out_plain_split=False):
        """ResidualConvUnit: conv2(relu(conv1(relu(x)))) + residual (default: x itself)."""
        _, h = self._c3(x_relu, B, H, W, pre + ".conv1", act=2, want_fp32=False, want_split=True)
        res = x_f32 if residual is None else residual
        return self._c3(h, B, H, W, pre + ".conv2", residual=res.contiguous(), want_fp32=out_fp32,
                        want_split=out_relu_split or out_plain_split, split_relu=out_relu_split)

    def _fusion(self, pre, B, H, W, x0_f32=None, x0_relu: Split = None, x1=None, prev_lowres=None):
        """FeatureFusionBlock: [x0 + RCU1(x1)] -> RCU2 -> up x2 -> out_conv (the 1x1 commutes with the bilinear
        upsampling, so it is applied at the low resolution: a quarter of the FLOPs, same result).  Returns the LOW-resolution
        out_conv output: the x2 upsampling is fused into the consumer (the next block's skip add, or the head's split), see
        ops.upsample2x.  ``prev_lowres``: the previous block's low-resolution output, whose upsampling is this block's x0."""
        if x1 is not None:
            x1_f32, x1_relu = x1
            # x0 + RCU1(x1) = conv2(.) + (x1 + up(prev)): the skip sum is produced by the upsampling kernel itself
            res, _ = ops.upsample2x(prev_lowres, addend=x1_f32, out_hw=(H, W))
            x0_f32, x0_relu = self._rcu(x1_f32, x1_relu, B, H, W, pre + ".resConfUnit1", residual=res, out_relu_split=True)
        _, o = self._rcu(x0_f32, x0_relu, B, H, W, pre + ".resConfUnit2", out_fp32=False, out_plain_split=True)
        y, _ = self._c1(Split(o.hi.view(B * H * W, -1), o.lo.view(B * H * W, -1) if o.lo is not None else None),
                        B * H * W, pre + ".out_conv")
        return y.view(B, H, W, -1)

    def _dpt(self, pre, decout, H, W):
        l2 = self.cfg["dec_depth"]
        hooks = [0, l2 * 2 // 4, l2 * 3 // 4, l2]
        nh, nw = H // 16, W // 16
        B = decout[0].shape[0]
        n = nh * nw
        ap = pre + ".act_postprocess"
        tok = [ops.split(decout[k].float().reshape(B * n, -1), self.x3) for k in hooks]
        # act_postprocess: 1x1 convs are per-token linears; ConvTranspose(k=s) is a linear to (cout, i, j) + rearrangement
        def convT(t, name, k):
            cout = self._sd[name + ".bias"].shape[0]
            # bias folded into the GEMM epilogue (one value per (cout, i, j) column, expanded once in _prepare)
            r, _ = ops.linear(t, self._w[name + ".weight"], self._sd[name + ".bias_cols"], B * n, x3=self.x3)   # [B*n, cout*k*k]
            return r.view(B, nh, nw, cout, k, k).permute(0, 1, 4, 2, 5, 3).reshape(B, nh * k, nw * k, cout)
        _, t0 = self._c1(tok[0], B * n, ap + ".0.0", want_fp32=False, want_split=True)
        _, t1 = self._c1(tok[1], B * n, ap + ".1.0", want_fp32=False, want_split=True)
        l0 = convT(t0, ap + ".0.1", 4)                                                      # [B, 4nh, 4nw, 96]
        l1 = convT(t1, ap + ".1.1", 2)                                                      # [B, 2nh, 2nw, 192]
        _, l2s = self._c1(tok[2], B * n, ap + ".2.0", want_fp32=False, want_split=True)      # [B*n, 384]
        _, t3 = self._c1(tok[3], B * n, ap + ".3.0", want_fp32=False, want_split=True)       # [B*n, 768]
        # 3x3 stride-2 pad-1 conv == the stride-1 conv sampled at even pixels
        t3 = Split(t3.hi.view(B, nh, nw, -1), t3.lo.view(B, nh, nw, -1) if t3.lo is not None else None)
        l3f, _ = self._c3(t3, B, nh, nw, ap + ".3.1")
        l3 = l3f[:, ::2, ::2].contiguous()
        h3, w3 = l3.shape[1], l3.shape[2]
        rn = pre + ".scratch.layer"
        kw = dict(want_fp32=True, want_split=True, split_relu=True)
        f0 = self._c3(ops.split(l0, self.x3), B, 4 * nh, 4 * nw, rn + "1_rn", **kw)
        f1 = self._c3(ops.split(l1, self.x3), B, 2 * nh, 2 * nw, rn + "2_rn", **kw)
        f2 = self._c3(Split(l2s.hi.view(B, nh, nw, -1), l2s.lo.view(B, nh, nw, -1) if l2s.lo is not None else None),
                      B, nh, nw, rn + "3_rn", **kw)
        f3 = self._c3(ops.split(l3, self.x3), B, h3, w3, rn + "4_rn", **kw)
        sc = pre + ".scratch.refinenet"
        # every block hands its LOW-resolution output on; the consumer's kernel upsamples (+ crop of dpt_head.py:57, + skip add)
        q4 = self._fusion(sc + "4", B, h3, w3, f3[0], f3[1])
        q3 = self._fusion(sc + "3", B, nh, nw, x1=f2, prev_lowres=q4)
        q2 = self._fusion(sc + "2", B, 2 * nh, 2 * nw, x1=f1, prev_lowres=q3)
        q1 = self._fusion(sc + "1", B, 4 * nh, 4 * nw, x1=f0, prev_lowres=q2)               # [B, 4nh, 4nw, 256] (low res)
        _, p1 = ops.upsample2x(q1, want_fp32=False, want_split=True, x3=self.x3)           # [B, 8nh, 8nw, 256] split
        o, _ = self._c3(p1, B, 8 * nh, 8 * nw, pre + ".head.0")
        _, o = ops.upsample2x(o, want_fp32=False, want_split=True, x3=self.x3)             # [B, H, W, 128] split
        _, o = self._c3(o, B, H, W, pre + ".head.2", act=2, want_fp32=False, want_split=True)
        out, _ = self._c1(Split(o.hi.view(B * H * W, -1), o.lo.view(B * H * W, -1) if o.lo is not None else None),
                          B * H * W, pre + ".head.4")
        return out.view(B, H, W, -1)                                                        # NHWC, 4 channels

    @torch.no_grad()
    def _downstream_head(self, head_num, decout, img_shape, raw: bool = False):
        """dust3r/model.py:193-197 + mast3r/catmlp_dpt_head.py:71-96.  img_shape: (H, W) or an int tensor [B,2]."""
        if isinstance(img_shape, torch.Tensor):
            hw = img_shape.reshape(-1, 2)
            assert bool((hw == hw[0:1]).all()), "true_shape must be all identical"   # utils/misc.py:56-61
            H, W = (int(v) for v in hw[0].tolist())
        else:
            H, W = int(img_shape[0]), int(img_shape[1])
        decout = list(decout)
        pre = f"downstream_head{head_num}"
        dev = decout[0].device
        with torch.cuda.device(dev):
            pts = self._dpt(pre + ".dpt", decout, H, W)                      # NHWC [B, H, W, 4]
            cat = torch.cat([decout[0].float(), decout[-1].float()], -1)
            B, S, D = cat.shape
            a = ops.split(cat.reshape(B * S, D), self.x3)
            _, hdn = self._linear(a, pre + ".head_local_features.fc1", B * S, act=1, want_fp32=False, want_split=True)
            lf, _ = self._linear(hdn, pre + ".head_local_features.fc2", B * S)
            n_desc = lf.shape[-1] // 256 - 1
            if not raw and n_desc == 24 and H % 16 == 0 and W % 16 == 0:
                # pixel_shuffle + concat + postprocess in one kernel (csrc/vit_ops.cu head_postprocess_kernel)
                return ops.head_postprocess(pts, lf, H, W, n_desc)
            lf = F.pixel_shuffle(lf.view(B, S, -1).transpose(-1, -2).reshape(B, -1, H // 16, W // 16), 16)
            fmap = torch.cat([pts, lf.permute(0, 2, 3, 1)], -1)             # B,H,W,29
            if raw:
                return fmap.permute(0, 3, 1, 2)
            xyz = fmap[..., 0:3]
            d = xyz.norm(dim=-1, keepdim=True)
            res = dict(pts3d=xyz / d.clip(min=1e-8) * torch.expm1(d), conf=1 + fmap[..., 3].exp())
            desc = fmap[..., 4:28]
            res["desc"] = desc / desc.norm(dim=-1, keepdim=True)
            res["desc_conf"] = fmap[..., 28].exp()
        return res

    @torch.no_grad()
    def forward(self, view1, view2):
        """dust3r/model.py:199-211 (symmetrised views are not special-cased: both images are always encoded)."""
        img1, img2 = view1["img"], view2["img"]
        B = img1.shape[0]
        s1 = view1.get("true_shape", torch.tensor(img1.shape[-2:])[None].repeat(B, 1))
        s2 = view2.get("true_shape", torch.tensor(img2.shape[-2:])[None].repeat(B, 1))
        if img1.shape[-2:] == img2.shape[-2:]:
            f, pos, _ = self._encode_image(torch.cat((img1, img2), 0), None)
            (f1, f2), (p1, p2) = f.chunk(2, 0), pos.chunk(2, 0)
        else:
            f1, p1, _ = self._encode_image(img1, s1)
            f2, p2, _ = self._encode_image(img2, s2)
        d1, d2 = self._decoder(f1.contiguous(), p1.contiguous(), f2.contiguous(), p2.contiguous())
        r1 = self._downstream_head(1, [t.float() for t in d1], s1)
        r2 = self._downstream_head(2, [t.float() for t in d2], s2)
        r2["pts3d_in_other_view"] = r2.pop("pts3d")
        return r1, r2

    __call__ = forward


def forward_pair(model: AsymmetricMASt3R, img1, img2):
    """2x _encode_image + _decoder + 2x _downstream_head: the unit BASELINE.json counts as one 'pair' per batch item."""
    H, W = img1.shape[-2:]
    f, pos, _ = model._encode_image(torch.cat((img1, img2), 0), None)
    (f1, f2), (p1, p2) = f.chunk(2, 0), pos.chunk(2, 0)
    d1, d2 = model._decoder(f1.contiguous(), p1.contiguous(), f2.contiguous(), p2.contiguous())
    if not model.concurrent:
        return model._downstream_head(1, d1, (H, W)), model._downstream_head(2, d2, (H, W))
    # the two heads are independent: overlap them on two streams
    s1 = torch.cuda.current_stream()
    s2 = model._side_stream(img1.device)
    s2.wait_stream(s1)
    with torch.cuda.stream(s2):
        r2 = model._downstream_head(2, d2, (H, W))
    r1 = model._downstream_head(1, d1, (H, W))
    s1.wait_stream(s2)
    for v in r2.values():
        v.record_stream(s1)
    return r1, r2

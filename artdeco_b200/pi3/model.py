"""Host-side mirror of the reference's ``Pi3`` for inference (VSLAM/thirdparty/Pi3/pi3/models/pi3.py:17-216): same
``state_dict`` key names, same input ([B, N, 3, H, W] in [0, 1], H and W multiples of 14) and the same output dict
(``points``, ``local_points``, ``conf``, ``camera_poses``, fp32).

Every dense contraction (patch embedding, qkv / proj / MLP, the head projections, the camera head's ReLU blocks) runs on
the wgmma GEMM (csrc/gemm_tc.cu) and every attention on the fused kernel (csrc/attn_tc.cu); the Pi3-specific stages
are in csrc/pi3.cu.  ``precision``:
  "bf16x3" (default)  three-term split product, fp32-class accuracy (meets the 1e-4 tolerance against the reference)
  "bf16"              single pass, about 3x less tensor work, about 1e-2 accuracy (closer to the reference's autocast)
LayerScale (``ls1`` / ``ls2``) is folded into the following projection at load time: W' = diag(ls) W, b' = ls * b,
in fp32 before the split.  Torch is left with the bicubic position-embedding resize (weights only, cached per grid),
the position table, two token copies and a concatenation.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from .. import _lib
from .._lib import f32, i32, i64, vp
from ..mast3r import ops
from ..mast3r.ops import Split
from .shapes import N_SPECIAL, PATCH, param_shapes

_lib.register("adb_pi3_patch14", [i32, i32, i32, vp, vp, vp, vp])
_lib.register("adb_pi3_tokens", [i32, i32, i32, vp, vp, vp, vp, vp, vp])
_lib.register("adb_qknorm_rope", [i32, i32, i32, i64, i32, vp, vp, vp, f32, vp, vp, i32, vp, vp, vp])
_lib.register("adb_pi3_point_head", [i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp])
_lib.register("adb_pi3_camera_tail", [i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp])
_lib.register("adb_pi3_svd_pose", [i32, vp, vp, vp, vp])

E = 1024
HEADS = 16
ENC_DEPTH, DEC_DEPTH, HEAD_DEPTH = 24, 36, 5
K_PATCH = 592                 # 3 * 14 * 14 = 588 taps, padded to a multiple of 8 for the GEMM's row stride
QK_NORM_EPS = 1e-5            # nn.LayerNorm's default: AttentionRope is not given the block's norm_layer (attention.py:248,261)
_FP32_WEIGHTS = ("camera_head.more_mlps.", "camera_head.fc_")


def _roundup(v, m):
    return (v + m - 1) // m * m


def interpolate_pos_embed(pos_embed: torch.Tensor, gh: int, gw: int) -> torch.Tensor:
    """[1, 1 + 37*37, C] -> [1, 1 + gh*gw, C] exactly as dinov2/models/vision_transformer.py:181-213 computes it
    (bicubic, antialias, no offset; the table is returned unchanged at the native 37x37 grid)."""
    N = pos_embed.shape[1] - 1
    M = int(math.sqrt(N))
    if gh == M and gw == M:
        return pos_embed
    pe = pos_embed.float()
    patch = pe[:, 1:].reshape(1, M, M, -1).permute(0, 3, 1, 2)
    patch = F.interpolate(patch, mode="bicubic", antialias=True, size=(gh, gw))
    patch = patch.permute(0, 2, 3, 1).reshape(1, gh * gw, -1)
    return torch.cat((pe[:, 0].unsqueeze(0), patch), dim=1).to(pos_embed.dtype)


def qknorm_rope(x: torch.Tensor, B: int, N: int, h: int, col0: int, gamma, beta, pos, x3=True, eps=QK_NORM_EPS,
                n_pos: int = ops.ROPE_TABLE_POSITIONS) -> Split:
    """Per-head LayerNorm (skipped when gamma is None) + RoPE2D of the heads at columns col0.. of x fp32 [B*N, ld];
    returns the bf16 split [B, h, N, 64] the attention kernel reads."""
    dev = x.device
    hi = torch.empty(B, h, N, 64, dtype=ops.BF16, device=dev)
    lo = torch.empty_like(hi) if x3 else None
    table = ops.rope_table(n_pos, dev)
    _lib.call("adb_qknorm_rope", B, N, h, x.shape[-1], col0, _lib.ptr(x, torch.float32), _lib.ptr(gamma), _lib.ptr(beta),
              float(eps), _lib.ptr(pos, torch.int64), _lib.ptr(table), n_pos, _lib.ptr(hi), _lib.ptr(lo), _lib.stream())
    return Split(hi, lo)


def svd_pose(rot: torch.Tensor, trans: torch.Tensor | None = None) -> torch.Tensor:
    """camera_head.py:66-93 on the device: rot [BN, 9] (fc_rot), trans [BN, 3] -> pose [BN, 4, 4]."""
    rot = rot.float().contiguous()
    pose = torch.empty(rot.shape[0], 4, 4, dtype=torch.float32, device=rot.device)
    _lib.call("adb_pi3_svd_pose", rot.shape[0], _lib.ptr(rot), _lib.ptr(trans.float().contiguous() if trans is not None else None),
              _lib.ptr(pose), _lib.stream())
    return pose


class Pi3:
    """Pi3 (pi3.py:17-216) on the C ABI.  Not an nn.Module: its weights are bf16 (hi, lo) splits held by this object."""

    param_shapes = staticmethod(param_shapes)

    def __init__(self, precision: str = "bf16x3"):
        if precision not in ("bf16x3", "bf16"):
            raise ValueError("precision must be 'bf16x3' or 'bf16'")
        self.precision = precision
        self.x3 = precision == "bf16x3"
        self.patch_size = PATCH
        self.device = torch.device("cpu")
        self._raw = {}
        self._sd = {}            # fp32 device tensors (LayerNorm parameters, biases, tokens, camera MLP)
        self._w = {}             # name -> Split (GEMM weights)
        self._pos_cache = {}

    # ---- nn.Module-like surface ----------------------------------------------------------------
    def eval(self):
        return self

    def train(self, mode: bool = True):
        if mode:
            raise NotImplementedError("Pi3 (artdeco_b200) is inference-only, as ARTDECO's loop closure is")
        return self

    def state_dict(self):
        return dict(self._raw)

    def to(self, device):
        self.device = torch.device(device)
        if self._raw and self.device.type == "cuda":
            self._prepare()
        return self

    def cuda(self, index=0):
        return self.to(torch.device("cuda", index))

    def load_state_dict(self, sd, strict: bool = True):
        """Reference key names; keys inference does not read (``image_mean``, ``image_std``, ``mask_token``) are ignored."""
        shapes = param_shapes()
        missing = [k for k in shapes if k not in sd]
        if strict and missing:
            raise KeyError(f"Pi3.load_state_dict: missing keys {missing[:5]}{'...' if len(missing) > 5 else ''}")
        bad = [k for k in shapes if k in sd and tuple(sd[k].shape) != tuple(shapes[k])]
        if bad:
            raise ValueError(f"Pi3.load_state_dict: wrong shapes for {bad[:5]}")
        self._raw = {k: sd[k].detach().float().cpu() for k in shapes if k in sd}
        self._pos_cache = {}
        if self.device.type == "cuda":
            self._prepare()
        return self

    def _prepare(self):
        _lib.require_cuda()
        dev, raw = self.device, self._raw
        self._sd, self._w, self._pos_cache = {}, {}, {}
        for k, v in raw.items():
            if k == "encoder.patch_embed.proj.weight":
                w = torch.zeros(E, K_PATCH, dtype=torch.float32)
                w[:, :3 * PATCH * PATCH] = v.reshape(E, -1)
                self._w[k] = ops.split(w.to(dev), self.x3)
            elif v.dim() == 2 and k.endswith(".weight") and not k.startswith(_FP32_WEIGHTS):
                pre = k[:-len(".weight")]
                w, b = v, raw.get(pre + ".bias")
                blk = pre.rsplit(".", 2)[0]
                ls = raw.get(blk + ".ls1.gamma") if pre.endswith(".attn.proj") else (
                    raw.get(blk + ".ls2.gamma") if pre.endswith(".mlp.fc2") else None)
                if ls is not None:       # LayerScale folded in fp32 before the split
                    w = ls[:, None] * w
                    self._sd[pre + ".bias"] = (ls * b).to(dev)
                self._w[k] = ops.split(w.contiguous().to(dev), self.x3)
            elif k.startswith("camera_head.more_mlps.") and k.endswith(".weight"):
                self._sd[k[:-len(".weight")] + ".wt"] = v.t().contiguous().to(dev)
            elif k not in self._sd:
                self._sd[k] = v.contiguous().to(dev)
        self._sd["encoder.cls_token"] = self._sd["encoder.cls_token"].reshape(E).contiguous()
        self._sd["encoder.register_tokens"] = self._sd["encoder.register_tokens"].reshape(4, E).contiguous()
        self._sd["register_token"] = self._sd["register_token"].reshape(N_SPECIAL, E).contiguous()

    # ---- building blocks ------------------------------------------------------------------------
    def _linear(self, a: Split, name: str, rows: int, **kw):
        return ops.linear(a, self._w[name + ".weight"], self._sd.get(name + ".bias"), rows, x3=self.x3, **kw)

    def _ln(self, x, name, **kw):
        return ops.layernorm(x, self._sd[name + ".weight"], self._sd[name + ".bias"], 1e-6, x3=self.x3, **kw)

    def _block(self, x, pre, pos, qk_norm):
        """Block (dinov2/layers/block.py:88-113, pos None) or BlockRope (layers/block.py:310-335)."""
        B, N, C = x.shape
        rows = B * N
        _, xn = self._ln(x, pre + ".norm1")
        Npad = _roundup(N, 8)
        if pos is not None and not qk_norm:
            # q, k leave the qkv GEMM already rotated, head-major and split; V is written plainly
            q, k, v = ops.linear_rope(xn, self._w[pre + ".attn.qkv.weight"], self._sd[pre + ".attn.qkv.bias"], B, N, HEADS,
                                      pos, 2, x3=self.x3)
            vt = ops.rope_heads(v, B, N, HEADS, C, 0, None, 2, x3=self.x3, Npad=Npad)
        else:
            qkv, _ = self._linear(xn, pre + ".attn.qkv", rows)
            if pos is None:
                q = ops.rope_heads(qkv, B, N, HEADS, 3 * C, 0, None, 1, x3=self.x3)
                k = ops.rope_heads(qkv, B, N, HEADS, 3 * C, C, None, 1, x3=self.x3)
            else:
                q = qknorm_rope(qkv, B, N, HEADS, 0, self._sd[pre + ".attn.q_norm.weight"],
                                self._sd[pre + ".attn.q_norm.bias"], pos, x3=self.x3)
                k = qknorm_rope(qkv, B, N, HEADS, C, self._sd[pre + ".attn.k_norm.weight"],
                                self._sd[pre + ".attn.k_norm.bias"], pos, x3=self.x3)
            vt = ops.rope_heads(qkv, B, N, HEADS, 3 * C, 2 * C, None, 2, x3=self.x3, Npad=Npad)
        o = ops.attention(q, k, vt, B, HEADS, N, N, Npad, 64 ** -0.5, x3=self.x3)
        x1, _ = self._linear(o, pre + ".attn.proj", rows, residual=x.reshape(rows, C))
        _, xn = self._ln(x1, pre + ".norm2")
        _, hdn = self._linear(xn, pre + ".mlp.fc1", rows, act=1, want_fp32=False, want_split=True)
        x2, _ = self._linear(hdn, pre + ".mlp.fc2", rows, residual=x1)
        return x2.view(B, N, C)

    def _pos_table(self, gh, gw, dev):
        key = (gh, gw, str(dev))
        if key not in self._pos_cache:
            self._pos_cache[key] = interpolate_pos_embed(self._sd["encoder.pos_embed"], gh, gw).reshape(1 + gh * gw, E).contiguous()
        return self._pos_cache[key]

    @staticmethod
    def _positions(BN, gh, gw, dev):
        """pi3.py:147-154: (y, x) + 1 for patches, 0 for the register tokens; [BN, 5 + gh*gw, 2] int64."""
        yy = torch.arange(gh, device=dev).repeat_interleave(gw)
        xx = torch.arange(gw, device=dev).repeat(gh)
        p = torch.cat([torch.zeros(N_SPECIAL, 2, dtype=torch.int64, device=dev), torch.stack([yy, xx], -1) + 1], 0)
        return p[None].expand(BN, -1, -1).contiguous()

    # ---- forward --------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, imgs: torch.Tensor, stages: dict | None = None):
        """imgs [B, N, 3, H, W] in [0, 1] -> dict(points [B,N,H,W,3], local_points [B,N,H,W,3], conf [B,N,H,W,1],
        camera_poses [B,N,4,4]).  ``stages``, when given, receives the intermediate tensors the golden files record."""
        _lib.require_cuda(imgs)
        if imgs.dim() != 5 or imgs.shape[2] != 3:
            raise ValueError(f"Pi3 expects imgs [B, N, 3, H, W], got {tuple(imgs.shape)}")
        B, N, _, H, W = imgs.shape
        if B < 1 or N < 1:
            raise ValueError("Pi3 needs at least one frame")
        if H % PATCH or W % PATCH or H < PATCH or W < PATCH:
            raise ValueError(f"Pi3: image size {H}x{W} is not a multiple of the patch size 14")
        gh, gw = H // PATCH, W // PATCH
        if max(gh, gw) + 1 >= ops.ROPE_TABLE_POSITIONS:
            raise ValueError(f"Pi3: image side {max(H, W)} px exceeds the {(ops.ROPE_TABLE_POSITIONS - 2) * PATCH} px the RoPE table covers")
        if not self._w:
            raise RuntimeError("Pi3: load_state_dict(...) and .to(cuda device) first")
        n, BN, hw = gh * gw, B * N, gh * gw + N_SPECIAL
        dev, x3 = imgs.device, self.x3
        with torch.cuda.device(dev):
            img = imgs.float().contiguous()
            a = Split(torch.empty(BN * n, K_PATCH, dtype=ops.BF16, device=dev),
                      torch.empty(BN * n, K_PATCH, dtype=ops.BF16, device=dev) if x3 else None)
            _lib.call("adb_pi3_patch14", BN, H, W, _lib.ptr(img), _lib.ptr(a.hi), _lib.ptr(a.lo), _lib.stream())
            patch, _ = self._linear(a, "encoder.patch_embed.proj", BN * n)
            x = torch.empty(BN, hw, E, dtype=torch.float32, device=dev)
            _lib.call("adb_pi3_tokens", BN, n, E, _lib.ptr(patch), _lib.ptr(self._sd["encoder.cls_token"]),
                      _lib.ptr(self._sd["encoder.register_tokens"]), _lib.ptr(self._pos_table(gh, gw, dev)), _lib.ptr(x),
                      _lib.stream())
            for i in range(ENC_DEPTH):
                x = self._block(x, f"encoder.blocks.{i}", None, False)
            hidden, _ = self._ln(x, "encoder.norm", want_fp32=True, want_split=False)
            if stages is not None:
                stages["encoder"] = hidden[:, N_SPECIAL:].clone()
            # the encoder's 5 special tokens (cls + 4 registers) are dropped and the decoder's 5 register tokens take
            # their rows (pi3.py:140-143)
            hidden[:, :N_SPECIAL] = self._sd["register_token"]
            pos = self._positions(BN, gh, gw, dev)
            last = []
            for i in range(DEC_DEPTH):
                shape = (BN, hw, E) if i % 2 == 0 else (B, N * hw, E)     # frame attention, then global attention
                hidden = self._block(hidden.view(shape), f"decoder.{i}", pos, True)
                if i >= DEC_DEPTH - 2:
                    last.append(hidden.view(BN, hw, E))
            dec = torch.cat(last, -1)
            if stages is not None:
                stages["decoder"] = dec
            d = ops.split(dec.view(BN * hw, 2 * E), x3)
            heads = {}
            for name in ("point_decoder", "conf_decoder", "camera_decoder"):
                h, _ = self._linear(d, name + ".projects", BN * hw)
                h = h.view(BN, hw, E)
                for j in range(HEAD_DEPTH):
                    h = self._block(h, f"{name}.blocks.{j}", pos, False)
                keep_fp32 = stages is not None or name == "camera_decoder"
                heads[name] = self._linear(ops.split(h.view(BN * hw, E), x3), name + ".linear_out", BN * hw,
                                           want_fp32=keep_fp32, want_split=True)
                if stages is not None:
                    stages[name.replace("_decoder", "_hidden")] = heads[name][0].view(BN, hw, -1)
            pts, _ = self._linear(heads["point_decoder"][1], "point_head.proj", BN * hw)
            cf, _ = self._linear(heads["conf_decoder"][1], "conf_head.proj", BN * hw)
            c32, csp = heads["camera_decoder"]
            for i in range(2):
                pre = f"camera_head.res_conv.{i}.res_conv"
                _, s = self._linear(csp, pre + "1", BN * hw, act=2, want_fp32=False, want_split=True)
                _, s = self._linear(s, pre + "2", BN * hw, act=2, want_fp32=False, want_split=True)
                c32, csp = self._linear(s, pre + "3", BN * hw, act=2, residual=c32, want_split=i == 0)
            rot = torch.empty(BN, 9, dtype=torch.float32, device=dev)
            trans = torch.empty(BN, 3, dtype=torch.float32, device=dev)
            sd = self._sd
            _lib.call("adb_pi3_camera_tail", BN, hw, N_SPECIAL, _lib.ptr(c32), _lib.ptr(sd["camera_head.more_mlps.0.wt"]),
                      _lib.ptr(sd["camera_head.more_mlps.0.bias"]), _lib.ptr(sd["camera_head.more_mlps.2.wt"]),
                      _lib.ptr(sd["camera_head.more_mlps.2.bias"]), _lib.ptr(sd["camera_head.fc_t.weight"]),
                      _lib.ptr(sd["camera_head.fc_t.bias"]), _lib.ptr(sd["camera_head.fc_rot.weight"]),
                      _lib.ptr(sd["camera_head.fc_rot.bias"]), _lib.ptr(rot), _lib.ptr(trans), _lib.stream())
            if stages is not None:
                stages["fc_rot"], stages["fc_t"] = rot, trans
            pose = svd_pose(rot, trans)
            points = torch.empty(B, N, H, W, 3, dtype=torch.float32, device=dev)
            local_points = torch.empty_like(points)
            conf = torch.empty(B, N, H, W, 1, dtype=torch.float32, device=dev)
            _lib.call("adb_pi3_point_head", BN, H, W, hw, N_SPECIAL, _lib.ptr(pts), _lib.ptr(cf), _lib.ptr(pose),
                      _lib.ptr(points), _lib.ptr(local_points), _lib.ptr(conf), _lib.stream())
        return dict(points=points, local_points=local_points, conf=conf, camera_poses=pose.view(B, N, 4, 4))

    __call__ = forward


def flops(N: int, H: int = 392, W: int = 518) -> float:
    """Multiply-adds x 2 of one forward over N frames (dense layers and attention; element-wise work not counted)."""
    n = (H // PATCH) * (W // PATCH)
    T, hw = N * (n + N_SPECIAL), n + N_SPECIAL
    lin_block = 2 * T * E * (3 * E + E + 8 * E)                  # qkv, proj, fc1, fc2
    f = 2 * N * n * E * 3 * PATCH * PATCH                       # patch embedding
    f += ENC_DEPTH * (lin_block + 4 * N * hw * hw * E)          # encoder: frame attention
    f += (DEC_DEPTH // 2) * (2 * lin_block + 4 * N * hw * hw * E + 4 * T * T * E)   # frame + global blocks
    f += 3 * (2 * T * 2 * E * E + HEAD_DEPTH * (lin_block + 4 * N * hw * hw * E))    # head decoders
    f += 2 * T * E * (E + E + 512)                               # linear_out
    f += 2 * T * E * (3 + 1) * PATCH * PATCH                      # LinearPts3d
    f += 2 * 3 * 2 * T * 512 * 512                                # camera head ReLU blocks
    return float(f)

"""LPIPS-VGG on the device: ``lpips.LPIPS(net="vgg")`` (version 0.1, ``lpips=True``, ``spatial=False``) as the mapper's
evaluation uses it (Reconstruct/scene/scene_models/h3dgsv3.py:98, :552).

    LPIPS(x0, x1) = sum_l mean_hw sum_c w_lc (f0_lc / (|f0_l| + 1e-10) - f1_lc / (|f1_l| + 1e-10))^2

with ``f_l`` the VGG16 activations at relu1_2, relu2_2, relu3_3, relu4_3 and relu5_3 of ``(x - shift) / scale``.
What runs (csrc/evaluate.cu, ``adb_lpips_vgg_forward``):
  * conv1_1 (3 -> 64) is a direct fp32 kernel with the ScalingLayer fused in; it writes the NHWC bf16 split;
  * the other twelve convolutions are the wgmma implicit-GEMM ``adb_conv3x3_bf16`` in bf16x3 with the bias and ReLU in the
    epilogue; taps are written in fp32, the rest as the next layer's bf16 split;
  * the 2x2 max-pool reads the fp32 tap and writes the next layer's split; one head kernel per tap writes per-CTA partial
    sums and one single-CTA launch adds them in a fixed order, so the value is bitwise reproducible;
  * both images of a pair go through the network as one batch of 2, and as many pairs per launch as the workspace budget
    holds.
The weights are the lpips package's state dict (``net.slice{1..5}.*``, ``lin{0..4}.model.1.weight``, ``scaling_layer.*``);
lpips loads its trained weights from its own package directory, so :meth:`LPIPSVGG.from_module` copies them from a live
``lpips.LPIPS(net="vgg")`` instead of shadowing the package."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import i32, i64, vp
from .mast3r import ops

_lib.register("adb_lpips_workspace_bytes", [i32, i32, i32, C.POINTER(C.c_size_t)])
_lib.register("adb_lpips_vgg_forward", [i32, i32, i32, i64, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp,
                                        C.c_size_t, vp, C.c_size_t, vp])

# (slice, index in torchvision's vgg16().features) of the 13 convolutions, in order; taps end slices 1..5
VGG_CONVS = ((1, 0), (1, 2), (2, 5), (2, 7), (3, 10), (3, 12), (3, 14), (4, 17), (4, 19), (4, 21), (5, 24), (5, 26), (5, 28))
TAP_CHANNELS = (64, 128, 256, 512, 512)
SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
DEFAULT_WORKSPACE_BYTES = 8 << 30


def workspace_bytes(n_frames: int, h: int, w: int) -> int:
    nb = C.c_size_t(0)
    _lib.call("adb_lpips_workspace_bytes", int(n_frames), int(h), int(w), C.byref(nb))
    return int(nb.value)


def frames_per_launch(T: int, h: int, w: int, budget: int) -> int:
    """The most frames (pairs) whose activations fit ``budget`` bytes, at least one."""
    per = workspace_bytes(1, h, w)
    nf = max(1, min(int(T), int(budget) // per))
    while nf > 1 and workspace_bytes(nf, h, w) > budget:
        nf -= 1
    return nf


class LPIPSVGG:
    """Weights of ``lpips.LPIPS(net="vgg")`` laid out for the device network."""

    def __init__(self, state_dict: dict, device=None):
        sd = {k: v.detach() for k, v in state_dict.items()}
        dev = torch.device(device) if device is not None else sd["net.slice1.0.weight"].device
        if dev.type != "cuda":
            dev = torch.device("cuda", torch.cuda.current_device())
        _lib.require_cuda(torch.empty(0, device=dev))

        def get(k):
            if k not in sd:
                raise KeyError(f"LPIPSVGG: state dict has no {k!r} (expected the lpips package's key names)")
            return sd[k].to(dev, torch.float32).contiguous()

        s0, i0 = VGG_CONVS[0]
        self.w1 = get(f"net.slice{s0}.{i0}.weight")
        self.b1 = get(f"net.slice{s0}.{i0}.bias")
        if self.w1.shape != (64, 3, 3, 3):
            raise ValueError(f"LPIPSVGG: conv1_1 weight must be [64,3,3,3], got {tuple(self.w1.shape)}")
        self.conv_w, self.conv_b = [], []
        cin = 64
        for s, i in VGG_CONVS[1:]:
            w = get(f"net.slice{s}.{i}.weight")
            if w.dim() != 4 or w.shape[1] != cin or w.shape[2:] != (3, 3):
                raise ValueError(f"LPIPSVGG: net.slice{s}.{i}.weight has shape {tuple(w.shape)}")
            self.conv_w.append(ops.prep_conv3x3_weight(w, True))
            self.conv_b.append(get(f"net.slice{s}.{i}.bias"))
            cin = w.shape[0]
        self.lin = []
        for l, c in enumerate(TAP_CHANNELS):
            lw = get(f"lin{l}.model.1.weight").reshape(-1).contiguous()
            if lw.numel() != c:
                raise ValueError(f"LPIPSVGG: lin{l} must have {c} weights, got {lw.numel()}")
            self.lin.append(lw)
        shift = sd.get("scaling_layer.shift")
        scale = sd.get("scaling_layer.scale")
        self.shift = (shift.to(dev, torch.float32).reshape(3).contiguous() if shift is not None
                      else torch.tensor(SHIFT, dtype=torch.float32, device=dev))
        self.scale = (scale.to(dev, torch.float32).reshape(3).contiguous() if scale is not None
                      else torch.tensor(SCALE, dtype=torch.float32, device=dev))
        self.device = dev
        P12, P5 = C.c_void_p * 12, C.c_void_p * 5
        self._w_hi = P12(*[w.hi.data_ptr() for w in self.conv_w])
        self._w_lo = P12(*[w.lo.data_ptr() for w in self.conv_w])
        self._bias = P12(*[b.data_ptr() for b in self.conv_b])
        self._lin = P5(*[l.data_ptr() for l in self.lin])

    @classmethod
    def from_module(cls, m) -> "LPIPSVGG":
        """Copies the weights of a live ``lpips.LPIPS(net="vgg")`` (what ``h3dgsv3.py:98`` builds)."""
        if getattr(m, "pnet_type", "vgg") not in ("vgg", "vgg16") or getattr(m, "version", "0.1") != "0.1":
            raise ValueError("LPIPSVGG.from_module needs lpips.LPIPS(net='vgg', version='0.1')")
        if getattr(m, "spatial", False) or not getattr(m, "lpips", True):
            raise ValueError("LPIPSVGG.from_module needs lpips=True, spatial=False")
        p = next(m.parameters())
        return cls(m.state_dict(), device=p.device if p.is_cuda else None)

    def run(self, T: int, h: int, w: int, n_gaussians: int, img0: torch.Tensor, img1: torch.Tensor, ews: torch.Tensor,
            workspace_bytes_budget: int = DEFAULT_WORKSPACE_BYTES, taps: list | None = None) -> None:
        """Adds every frame's five tap partials to the evaluation workspace ``ews`` (``img0``/``img1`` [T,3,h,w] fp32).
        ``taps``: optional five fp32 buffers [2T,H_l,W_l,C_l] that receive each tap's features (tests read them)."""
        nf = frames_per_launch(T, h, w, workspace_bytes_budget) if taps is None else T
        lws = torch.empty(workspace_bytes(nf, h, w), dtype=torch.uint8, device=self.device)
        s = _lib.stream()
        for f0 in range(0, T, nf):
            n = min(nf, T - f0)
            tp = None
            if taps is not None:
                tp = (C.POINTER(C.c_float) * 5)(*[C.cast(C.c_void_p(t.data_ptr()), C.POINTER(C.c_float)) for t in taps])
            _lib.call("adb_lpips_vgg_forward", T, h, w, int(n_gaussians), f0, n, _lib.ptr(img0, torch.float32),
                      _lib.ptr(img1, torch.float32), _lib.ptr(self.w1), _lib.ptr(self.b1), _lib.ptr(self.shift),
                      _lib.ptr(self.scale), self._w_hi, self._w_lo, self._bias, self._lin, tp, _lib.ptr(lws), lws.numel(),
                      _lib.ptr(ews), ews.numel(), s)

    def _check(self, img0, img1):
        if img0.shape != img1.shape or img0.dim() != 4 or img0.shape[1] != 3:
            raise ValueError(f"LPIPSVGG: images must both be [N,3,h,w], got {tuple(img0.shape)} and {tuple(img1.shape)}")
        if img0.shape[2] < 16 or img0.shape[3] < 16:
            raise ValueError("LPIPSVGG: h and w must be >= 16 (VGG16 pools four times)")
        for t in (img0, img1):
            _lib.require_cuda(t)
            if t.device != self.device:
                raise ValueError(f"LPIPSVGG: images on {t.device}, weights on {self.device}")
        return img0.detach().float().contiguous(), img1.detach().float().contiguous()

    def __call__(self, img0: torch.Tensor, img1: torch.Tensor, workspace_bytes_budget: int = DEFAULT_WORKSPACE_BYTES):
        """``lpips.LPIPS.forward(img0, img1)`` with ``normalize=False``: [N,1,1,1] on the device, no host sync."""
        from . import evaluate as _ev
        a, b = self._check(img0, img1)
        N, _, h, w = a.shape
        ews = _ev.eval_workspace(N, h, w, 0, a.device)
        with torch.cuda.device(a.device):
            self.run(N, h, w, 0, a, b, ews, workspace_bytes_budget)
            table = _ev.reduce(N, h, w, 0, True, ews)
        return table[:, _ev.COL_LPIPS].float().reshape(N, 1, 1, 1)

    def features(self, img0: torch.Tensor, img1: torch.Tensor):
        """Test hook: (value [N,1,1,1], the five taps' fp32 features [2N,H_l,W_l,C_l] with image 2i = img0[i])."""
        from . import evaluate as _ev
        a, b = self._check(img0, img1)
        N, _, h, w = a.shape
        taps, hh, ww = [], h, w
        for c in TAP_CHANNELS:
            taps.append(torch.empty(2 * N, hh, ww, c, dtype=torch.float32, device=a.device))
            hh, ww = hh // 2, ww // 2
        ews = _ev.eval_workspace(N, h, w, 0, a.device)
        with torch.cuda.device(a.device):
            self.run(N, h, w, 0, a, b, ews, taps=taps)
            table = _ev.reduce(N, h, w, 0, True, ews)
        return table[:, _ev.COL_LPIPS].float().reshape(N, 1, 1, 1), taps

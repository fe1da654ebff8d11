"""The Backend's accurate loop closure (VSLAM/mast3r_slam/retrieval_database.py:263-326) without the similarity graph:
the caller picks the window of key frames, as the reference does from its similarity graph, and passes the query last.

  window_input           inverse_normalize + bilinear resize to 392x518 (:21-41,268-270), one kernel (csrc/pi3.cu)
  Pi3 forward            artdeco_b200.pi3.Pi3 (:271-273; bf16x3 here, where the reference uses bf16 autocast)
  score_window           matching.match_pi3 on each (candidate, query) point-map pair in chunks of 32 (:277-290,302-326),
                         per-pair valid-match counts, the fraction, the descending sort, the accurate_min gate and top-k
                         (:292-300)

Ties in the match fraction are ordered exactly as ``torch.argsort(fraction, descending=True)`` orders them on the
device, because that call is made here as the reference makes it.  For the 23 candidates of a full window PyTorch sorts
with a small bitonic network, which is deterministic but not stable: equal fractions need not keep window order.
The selected ids are read back to the host once, at the end, where the reference calls ``.tolist()``."""
from __future__ import annotations

import torch

from .. import _lib, matching
from .._lib import i32, vp

_lib.register("adb_pi3_window_input", [i32, i32, i32, vp, i32, i32, vp, vp])

PI3_H, PI3_W = 392, 518


def window_input(images: torch.Tensor, H: int = PI3_H, W: int = PI3_W) -> torch.Tensor:
    """images [N, 3, h, w] in the SLAM normalisation ([-1, 1]) -> Pi3's input [1, N, 3, H, W] in [0, 1]."""
    _lib.require_cuda(images)
    if images.dim() != 4 or images.shape[1] != 3:
        raise ValueError(f"expected key-frame images [N, 3, h, w], got {tuple(images.shape)}")
    N, _, Hi, Wi = images.shape
    img = images.float().contiguous()
    out = torch.empty(1, N, 3, H, W, dtype=torch.float32, device=images.device)
    with torch.cuda.device(images.device):
        _lib.call("adb_pi3_window_input", N, Hi, Wi, _lib.ptr(img), H, W, _lib.ptr(out), _lib.stream())
    return out


def score_window(points: torch.Tensor, idxs_all, config, chunk: int = 32):
    """points [N, H, W, 3] (Pi3's ``points`` for the window, query last) -> (device tensor of the selected ids, in
    order, and the per-pair valid-match counts [N-1])."""
    ii = list(idxs_all[:-1])
    dev = points.device
    if not ii:
        return torch.empty(0, dtype=torch.int64, device=dev), torch.empty(0, dtype=torch.int64, device=dev)
    valid = []
    for i in range(0, len(ii), chunk):
        e = min(i + chunk, len(ii))
        query = points[-1:].expand(e - i, -1, -1, -1).contiguous()
        _, v = matching.match_pi3(config, points[i:e].contiguous(), query)
        valid.append(v)
    valid = torch.cat(valid, 0)
    counts = valid.sum(-1)
    frac = counts / valid[0].numel()
    order = torch.argsort(frac, descending=True)
    keep = order[frac[order] > config["retrieval"]["accurate_min"]]
    ids = torch.as_tensor(ii, dtype=torch.int64).to(dev, non_blocking=True)
    return ids[keep][:config["retrieval"]["k"]], counts


def accurate_loop_closure(model, images: torch.Tensor, idxs_all, config) -> list:
    """retrieval_database.py:263-300: ``images`` [N, 3, h, w] are the key frames of ``idxs_all`` (query last) in [-1, 1];
    returns the candidate ids whose match fraction with the query exceeds ``retrieval.accurate_min``, best first, at
    most ``retrieval.k`` of them."""
    if len(idxs_all) != images.shape[0] or len(idxs_all) < 1:
        raise ValueError("one image per window id, and at least the query")
    res = model(window_input(images))
    sel, _ = score_window(res["points"][0], idxs_all, config)
    return sel.tolist()

"""Host-side mirror of ``gsplat.rendering.rasterization`` for the exact configuration the reference uses
(Reconstruct/scene/scene_models/h3dgsv3.py:664-680): 3DGS "classic" rasterisation, ``packed=False``,
``absgrad=False``, SH colours, ``render_mode`` "RGB" or "RGB+D".  Same keyword names, same return triple
``(render_colors[C,H,W,ch], render_alphas[C,H,W,1], meta)`` with ``meta['radii']`` of shape [C,N,2]
(h3dgsv3.py:689), and a complete autograd backward (means, quats, scales, opacities, colours, viewmats;
upstream grads for colours AND alphas, h3dgsv3.py:685-686).

All compute goes through the C ABI (adb_raster_*); PyTorch only owns memory, streams and the autograd graph.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
from ._lib import f32, i32, i64, vp

_lib.register("adb_raster_project_fwd", [i32, vp, vp, vp, vp, vp, i32, vp, vp, vp, i32, i32, f32, f32, f32, f32,
                                         vp, vp, vp, vp])
_lib.register("adb_raster_project_fwd_counts", [i32, vp, vp, vp, vp, vp, i32, vp, vp, vp, i32, i32, f32, f32, f32, f32,
                                                vp, vp, vp, vp, vp])
_lib.register("adb_raster_tile_scan", [i32, i32, i64, vp, vp, vp, vp, vp])
_lib.register("adb_raster_tile_count_scan", [i32, vp, vp, vp, i32, i32, i32, i64, vp, vp, vp, vp, vp])
_lib.register("adb_raster_tile_band_scratch_bytes", [i64, C.POINTER(C.c_size_t)])
_lib.register("adb_raster_tile_band_scatter_sort", [i32, vp, vp, vp, i32, i32, i32, i32, i32, i64, vp, vp, vp, vp,
                                                    C.c_size_t, vp, vp, vp])
_lib.register("adb_raster_blend_fwd", [i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp])
_lib.register("adb_raster_blend_bwd", [i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp])
_lib.register("adb_raster_project_bwd", [i32, vp, vp, vp, vp, i32, vp, vp, vp, i32, i32, f32, f32, f32, f32,
                                         vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp])

_lib.register("adb_raster_project_bwd_multi", [i32, i32, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp])
_lib.register("adb_raster_sh_bwd_multi", [i32, i32, vp, vp, i32, vp, vp, vp, vp, i32, i32, i32, vp, vp])
_lib.register("adb_raster_sh_dir_bwd_multi", [i32, i32, vp, vp, i32, vp, vp, vp, vp, vp, vp])
_lib.register("adb_raster_sh_expand_multi", [i32, i32, vp, i32, vp, vp, vp, vp])

_lib.register("adb_raster_project_fwd_legacy", [i32, vp, vp, vp, vp, vp, i32, vp, vp, vp, i32, i32, f32, f32, f32,
                                                vp, vp, vp, vp])
_lib.register("adb_raster_blend_fwd_legacy", [i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp])
_lib.register("adb_raster_blend_bwd_legacy", [i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp])

_caps_t = C.POINTER(C.c_longlong)
_lib.register("adb_raster_project_fwd_multi", [i32, i32, vp, vp, vp, vp, vp, i32, vp, vp, vp, i32, i32, f32, f32, f32, f32,
                                               vp, vp, vp, vp, vp])
_lib.register("adb_raster_tile_scan_multi", [i32, i32, i32, _caps_t, vp, vp, vp, vp, vp])
_lib.register("adb_raster_tile_band_scatter_sort_multi", [i32, i32, vp, vp, vp, i32, i32, _caps_t, vp, vp, vp, vp,
                                                          C.c_size_t, vp, vp, vp])
_lib.register("adb_raster_blend_fwd_multi", [i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp])
_lib.register("adb_raster_blend_bwd_multi", [i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp])


TILE = 16
SPLAT_STRIDE = 12
COUNTER_COPIES = 4      # ADB_TILE_COUNTER_COPIES (csrc/raster_common.cuh)


def _f32c(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def project(means, quats, scales, opacities, sh, sh_degree, viewmat, K, campos, W, H, eps2d, near, far, radius_clip,
            legacy=False, out=None, tile_counts=None):
    """Projection + SH + tile counts for one camera.  Returns radii[N,2] i32, splats[N,12], tiles_per_gauss[N].
    ``legacy``: Inria conventions (see include/artdeco_b200.h, adb_raster_project_fwd_legacy).
    ``out``: optional preallocated (radii, splats, tpg) — slices of per-camera stacks in the multi-view path.
    ``tile_counts``: optional zeroed counter buffer from ``new_tile_counts``: the per-tile counting of the bucketed
    intersection is fused into the projection kernel (pass the same buffer to ``intersect(counts=...)``)."""
    N = means.shape[0]
    dev = means.device
    if out is not None:
        radii, splats, tpg = out
    else:
        radii = torch.empty(N, 2, dtype=torch.int32, device=dev)
        splats = torch.empty(N, SPLAT_STRIDE, dtype=torch.float32, device=dev)
        tpg = torch.empty(N, dtype=torch.int32, device=dev)
    if legacy:
        _lib.call("adb_raster_project_fwd_legacy", N, _lib.ptr(means), _lib.ptr(quats), _lib.ptr(scales),
                  _lib.ptr(opacities), _lib.ptr(sh), int(sh_degree), _lib.ptr(viewmat), _lib.ptr(K), _lib.ptr(campos),
                  W, H, eps2d, near, far, _lib.ptr(radii), _lib.ptr(splats), _lib.ptr(tpg), _lib.stream())
        return radii, splats, tpg
    if tile_counts is not None:
        _lib.call("adb_raster_project_fwd_counts", N, _lib.ptr(means), _lib.ptr(quats), _lib.ptr(scales), _lib.ptr(opacities),
                  _lib.ptr(sh), int(sh_degree), _lib.ptr(viewmat), _lib.ptr(K), _lib.ptr(campos), W, H, eps2d, near, far,
                  radius_clip, _lib.ptr(radii), _lib.ptr(splats), _lib.ptr(tpg), _lib.ptr(tile_counts), _lib.stream())
        return radii, splats, tpg
    _lib.call("adb_raster_project_fwd", N, _lib.ptr(means), _lib.ptr(quats), _lib.ptr(scales), _lib.ptr(opacities),
              _lib.ptr(sh), int(sh_degree), _lib.ptr(viewmat), _lib.ptr(K), _lib.ptr(campos), W, H, eps2d, near, far,
              radius_clip, _lib.ptr(radii), _lib.ptr(splats), _lib.ptr(tpg), _lib.stream())
    return radii, splats, tpg


def project_backward(means, quats, scales, opacities, sh, sh_degree, viewmat, K, campos, W, H, eps2d, near, far,
                     radius_clip, radii, splats, v_splats):
    """Projection + SH backward of one camera (``project``'s arguments, its radii / splats, and the blend backward's
    ``v_splats``).  Returns (v_means, v_quats, v_scales, v_opac, v_sh, v_viewmat[4,4], v_campos[3]); with ``sh=None``
    v_sh and v_campos are None."""
    dev = means.device
    v_means = torch.empty_like(means)
    v_quats = torch.empty_like(quats)
    v_scales = torch.empty_like(scales)
    v_opac = torch.empty_like(opacities)
    v_sh = torch.empty_like(sh) if sh is not None else None
    v_view = torch.zeros(4, 4, dtype=torch.float32, device=dev)
    v_campos = torch.zeros(3, dtype=torch.float32, device=dev) if sh is not None else None
    _lib.call("adb_raster_project_bwd", means.shape[0], _lib.ptr(means), _lib.ptr(quats), _lib.ptr(scales), _lib.ptr(sh),
              int(sh_degree), _lib.ptr(viewmat), _lib.ptr(K), _lib.ptr(campos), W, H, eps2d, near, far, radius_clip,
              _lib.ptr(radii), _lib.ptr(splats), _lib.ptr(v_splats), _lib.ptr(v_means), _lib.ptr(v_quats),
              _lib.ptr(v_scales), _lib.ptr(v_opac), _lib.ptr(v_sh), _lib.ptr(v_view), _lib.ptr(v_campos), _lib.stream())
    return v_means, v_quats, v_scales, v_opac, v_sh, v_view, v_campos


def new_tile_counts(W, H, dev, views=None):
    """Zeroed counter buffer of the tile-bucketed intersection: 4 replicated counters per tile, then their segment starts.
    ``views``: C -> one such block per view, [C, 2*4*T] (``project_multi`` / ``intersect_multi``)."""
    T = ((W + TILE - 1) // TILE) * ((H + TILE - 1) // TILE)
    shape = (2 * COUNTER_COPIES * T,) if views is None else (int(views), 2 * COUNTER_COPIES * T)
    return torch.zeros(shape, dtype=torch.int32, device=dev)


def band_scratch(capacity, dev):
    """Uninitialised scratch of the band scatter (adb_raster_tile_band_scatter_sort*) for ``capacity`` intersections."""
    nb = C.c_size_t(0)
    _lib.call("adb_raster_tile_band_scratch_bytes", int(capacity), C.byref(nb))
    return torch.empty(max(nb.value, 1), dtype=torch.uint8, device=dev)


# ---- the multi-view batch, stage by stage: one launch per stage for C views of the same Gaussians ----------------------------
def project_multi(means, quats, scales, opacities, sh, sh_degree, viewmats, Ks, camposs, W, H, eps2d, near, far, radius_clip,
                  tile_counts, out=None):
    """Projection + SH + fused tile counting of C cameras in one pass (parameters read once).  ``viewmats [C,4,4]``,
    ``Ks [C,3,3]``, ``camposs [C,3]``; ``tile_counts`` from ``new_tile_counts(..., views=C)``.  Returns radii [C,N,2],
    splats [C,N,12], tiles_per_gauss [C,N], per view bit-identical to ``project(..., tile_counts=...)``."""
    N, Cn, dev = means.shape[0], viewmats.shape[0], means.device
    if out is not None:
        radii, splats, tpg = out
    else:
        radii = torch.empty(Cn, N, 2, dtype=torch.int32, device=dev)
        splats = torch.empty(Cn, N, SPLAT_STRIDE, dtype=torch.float32, device=dev)
        tpg = torch.empty(Cn, N, dtype=torch.int32, device=dev)
    _lib.call("adb_raster_project_fwd_multi", N, Cn, _lib.ptr(means), _lib.ptr(quats), _lib.ptr(scales), _lib.ptr(opacities),
              _lib.ptr(sh), int(sh_degree), _lib.ptr(viewmats), _lib.ptr(Ks), _lib.ptr(camposs), W, H, eps2d, near, far,
              radius_clip, _lib.ptr(radii), _lib.ptr(splats), _lib.ptr(tpg), _lib.ptr(tile_counts), _lib.stream())
    return radii, splats, tpg


def intersect_multi(radii, splats, tpg, W, H, counts, capacities=None, keys=True, info=None):
    """Tile-bucketed intersection of C views (``radii [C,N,2]`` ...; ``counts`` filled by ``project_multi``): one scan, the
    two band-scatter passes and one sort launch.  View c owns the segment ``[sum(seg[:c]), +seg[c])`` of one keys / vals
    buffer; offsets [C,T+1] are absolute indices into it and vals = c*N + gaussian (gsplat's concatenated per-camera layout).

    ``capacities=None``: one host sync reads all C counts and the segments are exactly the counts.  ``capacities`` (C ints):
    no host sync; entries of a view beyond its count are undefined, and a view that needed more is flagged in
    ``info["overflow"][c]`` (its image is then incomplete; the other views are unaffected).
    ``keys=False``: the sort writes vals only (keys is then None).  ``info``: optional preallocated
    ``{"n_isect": int64[C], "overflow": int32[C]}``.  Returns ``(keys, vals, offsets, info, seg)``; ``seg`` = the segment
    sizes (all zero when N = 0)."""
    Cn, N = radii.shape[0], radii.shape[1]
    dev = radii.device
    T = ((W + TILE - 1) // TILE) * ((H + TILE - 1) // TILE)
    if info is None:
        info = {"n_isect": torch.zeros(Cn, dtype=torch.int64, device=dev),
                "overflow": torch.zeros(Cn, dtype=torch.int32, device=dev)}
    else:
        info["n_isect"].zero_()
        info["overflow"].zero_()
    offsets = torch.empty(Cn, T + 1, dtype=torch.int32, device=dev)
    if capacities is None:
        zero = (C.c_longlong * Cn)(*([0] * Cn))
        _lib.call("adb_raster_tile_scan_multi", Cn, W, H, zero, _lib.ptr(counts), None, _lib.ptr(info["n_isect"]), None,
                  _lib.stream())
        seg = [int(n) for n in info["n_isect"].tolist()]        # the pipeline's single host sync
        if sum(seg) >= 2147483647:
            raise _lib.ArtdecoB200Error("more than 2^31 tile intersections in the batch")
    else:
        seg = [int(c) for c in capacities]
        if len(seg) != Cn:
            raise ValueError(f"intersect_multi: {len(seg)} capacities for {Cn} views")
        if N == 0:
            seg = [0] * Cn                       # no Gaussians, no intersections: nothing to pad
    caps = (C.c_longlong * Cn)(*seg)
    _lib.call("adb_raster_tile_scan_multi", Cn, W, H, caps, _lib.ptr(counts), _lib.ptr(offsets), _lib.ptr(info["n_isect"]),
              _lib.ptr(info["overflow"]), _lib.stream())
    total = sum(seg)
    vals = torch.empty(max(total, 1), dtype=torch.int32, device=dev)
    keys_t = torch.empty(max(total, 1), dtype=torch.int64, device=dev) if keys else None
    packed = torch.empty(max(total, 1), dtype=torch.int64, device=dev)
    scratch = band_scratch(total, dev)
    _lib.call("adb_raster_tile_band_scatter_sort_multi", N, Cn, _lib.ptr(radii), _lib.ptr(splats), _lib.ptr(tpg), W, H,
              caps, _lib.ptr(counts), _lib.ptr(offsets), _lib.ptr(packed), _lib.ptr(scratch), scratch.numel(),
              _lib.ptr(keys_t), _lib.ptr(vals), _lib.stream())
    return (keys_t[:total] if keys else None), vals[:total], offsets, info, seg


def blend_forward_multi(W, H, splats, vals, offsets, hits=None, out=None):
    """Blend forward of C views in one launch (``splats [C,N,12]``, ``vals`` / ``offsets`` from ``intersect_multi``).
    Returns colors [C,H,W,4], alphas [C,H,W], last_ids [C,H,W] (absolute sorted indices).  ``hits``: ``new_hit_mask(vals)``."""
    Cn, dev = splats.shape[0], splats.device
    if out is not None:
        colors, alphas, last_ids = out
    else:
        colors = torch.empty(Cn, H, W, 4, dtype=torch.float32, device=dev)
        alphas = torch.empty(Cn, H, W, dtype=torch.float32, device=dev)
        last_ids = torch.empty(Cn, H, W, dtype=torch.int32, device=dev)
    if hits is not None and (hits.dtype != torch.uint8 or hits.numel() < vals.numel() or hits.device != dev):
        raise ValueError("blend_forward_multi: hits must be a uint8 tensor with one byte per intersection (new_hit_mask)")
    _lib.call("adb_raster_blend_fwd_multi", splats.shape[1], Cn, W, H, _lib.ptr(splats),
              _lib.ptr(vals) if vals.numel() else None,
              _lib.ptr(offsets), _lib.ptr(colors), _lib.ptr(alphas), _lib.ptr(last_ids), _lib.ptr(hits), _lib.stream())
    return colors, alphas, last_ids


def blend_backward_multi(W, H, splats, vals, offsets, alphas, last_ids, v_colors, v_alphas, out=None, hits=None):
    """Blend backward of C views in one launch.  ``out``: optional ZEROED [C,N,12] accumulator; ``hits``: the mask
    ``blend_forward_multi`` filled for the same buffers."""
    v_splats = out if out is not None else torch.zeros_like(splats)
    if hits is not None and (hits.dtype != torch.uint8 or hits.numel() < vals.numel() or hits.device != splats.device):
        raise ValueError("blend_backward_multi: hits must be the uint8 mask blend_forward_multi filled for these intersections")
    _lib.call("adb_raster_blend_bwd_multi", splats.shape[1], splats.shape[0], W, H, _lib.ptr(splats),
              _lib.ptr(vals) if vals.numel() else None,
              _lib.ptr(offsets), _lib.ptr(alphas), _lib.ptr(last_ids), _lib.ptr(v_colors), _lib.ptr(v_alphas),
              _lib.ptr(v_splats), _lib.ptr(hits), _lib.stream())
    return v_splats


def intersect(radii, splats, tpg, W, H, cam_id=0, n_cams=1, legacy=False, capacity=None, counts=None):
    """Tile keys/values (sorted), tile offsets [T+1] for one camera: count, scan, band scatter, one CTA-local bitonic sort
    per tile (csrc/raster_isect.cu), bit-identical to the stable radix sort of (cam | tile | depth) keys.

    ``capacity=None``: one host sync to size keys/vals exactly (gsplat does the same: ``cum_tiles[-1].item()``);
    returns ``(keys[I], vals[I], offsets, I:int)``.
    ``capacity=int``: NO host sync (CUDA-graph capturable): buffers hold ``capacity`` intersections, the true count and an
    overflow flag stay on the device; returns ``(keys[capacity], vals[capacity], offsets, info)`` with
    ``info = {"n_isect": int64[1] tensor, "overflow": int32[1] tensor}``; entries beyond ``offsets[T]`` are undefined.  On
    overflow the dropped intersections make the image wrong but nothing is written out of bounds.
    ``counts``: the buffer ``project(..., tile_counts=...)`` filled (counting fused into the projection): only the scan runs."""
    N = radii.shape[0]
    dev = radii.device
    T = ((W + TILE - 1) // TILE) * ((H + TILE - 1) // TILE)
    offsets = torch.empty(T + 1, dtype=torch.int32, device=dev)
    if N == 0:
        offsets.zero_()
        e64 = torch.empty(0, dtype=torch.int64, device=dev)
        e32 = torch.empty(0, dtype=torch.int32, device=dev)
        if capacity is None:
            return e64, e32, offsets, 0
        return e64, e32, offsets, {"n_isect": torch.zeros(1, dtype=torch.int64, device=dev),
                                   "overflow": torch.zeros(1, dtype=torch.int32, device=dev)}
    total = torch.zeros(1, dtype=torch.int64, device=dev)
    overflow = torch.zeros(1, dtype=torch.int32, device=dev)
    cap_scan = int(capacity) if capacity is not None else 2147483646
    if counts is not None:
        _lib.call("adb_raster_tile_scan", W, H, cap_scan, _lib.ptr(counts), _lib.ptr(offsets), _lib.ptr(total),
                  _lib.ptr(overflow), _lib.stream())
    else:
        counts = torch.zeros(2 * COUNTER_COPIES * T, dtype=torch.int32, device=dev)   # counters | segment starts
        _lib.call("adb_raster_tile_count_scan", N, _lib.ptr(radii), _lib.ptr(splats), _lib.ptr(tpg), W, H, int(legacy),
                  cap_scan, _lib.ptr(counts), _lib.ptr(offsets), _lib.ptr(total), _lib.ptr(overflow), _lib.stream())
    if capacity is None:
        n_isect = int(total.item())      # the pipeline's single host sync
        if n_isect >= 2147483647:
            raise _lib.ArtdecoB200Error("more than 2^31 tile intersections")
        cap = n_isect
    else:
        cap = int(capacity)
    keys = torch.empty(max(cap, 1), dtype=torch.int64, device=dev)
    vals = torch.empty(max(cap, 1), dtype=torch.int32, device=dev)
    if cap > 0:
        packed = torch.empty(cap, dtype=torch.int64, device=dev)
        scratch = band_scratch(cap, dev)
        _lib.call("adb_raster_tile_band_scatter_sort", N, _lib.ptr(radii), _lib.ptr(splats), _lib.ptr(tpg), W, H,
                  int(legacy), cam_id, n_cams, cap, _lib.ptr(counts), _lib.ptr(offsets), _lib.ptr(packed),
                  _lib.ptr(scratch), scratch.numel(), _lib.ptr(keys), _lib.ptr(vals), _lib.stream())
    else:
        counts.zero_()
    if capacity is None:
        return keys[:n_isect], vals[:n_isect], offsets, n_isect
    return keys[:cap], vals[:cap], offsets, {"n_isect": total, "overflow": overflow}


def new_hit_mask(vals: torch.Tensor):
    """One byte per sorted intersection for ``blend_forward(hits=)`` / ``blend_backward(hits=)``: the forward records which
    warps' pixel blocks each (tile, splat) entry can reach and the backward reuses those culling decisions instead of repeating
    the tests."""
    return torch.empty(max(1, vals.numel()), dtype=torch.uint8, device=vals.device)


def blend_forward(W, H, N, splats, vals, offsets, legacy=False, out=None, hits=None):
    """``legacy`` returns a 4th tensor main_ids[H,W] and accumulates 1/z in colors[...,3].
    ``out``: optional preallocated (colors[H,W,4], alphas[H,W], last_ids[H,W]) — slices of per-camera stacks.
    ``hits``: optional uint8 [len(vals)] (``new_hit_mask``) that receives the culling decisions for ``blend_backward``."""
    dev = splats.device
    if out is not None:
        colors, alphas, last_ids = out
    else:
        colors = torch.empty(H, W, 4, dtype=torch.float32, device=dev)
        alphas = torch.empty(H, W, dtype=torch.float32, device=dev)
        last_ids = torch.empty(H, W, dtype=torch.int32, device=dev)
    if legacy:
        main_ids = torch.empty(H, W, dtype=torch.int32, device=dev)
        _lib.call("adb_raster_blend_fwd_legacy", W, H, N, _lib.ptr(splats), _lib.ptr(vals) if vals.numel() else None,
                  _lib.ptr(offsets), _lib.ptr(colors), _lib.ptr(alphas), _lib.ptr(last_ids), _lib.ptr(main_ids),
                  _lib.stream())
        return colors, alphas, last_ids, main_ids
    if hits is not None:
        if hits.dtype != torch.uint8 or hits.numel() < vals.numel() or hits.device != splats.device:
            raise ValueError("blend_forward: hits must be a uint8 tensor with one byte per intersection (new_hit_mask)")
    _lib.call("adb_raster_blend_fwd", W, H, N, _lib.ptr(splats), _lib.ptr(vals) if vals.numel() else None,
              _lib.ptr(offsets), _lib.ptr(colors), _lib.ptr(alphas), _lib.ptr(last_ids), _lib.ptr(hits), _lib.stream())
    return colors, alphas, last_ids


def blend_backward(W, H, N, splats, vals, offsets, alphas, last_ids, v_colors, v_alphas, legacy=False, out=None, hits=None):
    """``out``: optional ZEROED [N,12] accumulator (a slice of the per-camera stack in the multi-view path).
    ``hits``: the mask ``blend_forward(hits=)`` filled for the SAME splats / vals / offsets."""
    v_splats = out if out is not None else torch.zeros(N, SPLAT_STRIDE, dtype=torch.float32, device=splats.device)
    if legacy:
        _lib.call("adb_raster_blend_bwd_legacy", W, H, N, _lib.ptr(splats), _lib.ptr(vals) if vals.numel() else None,
                  _lib.ptr(offsets), _lib.ptr(alphas), _lib.ptr(last_ids), _lib.ptr(v_colors), _lib.ptr(v_alphas),
                  _lib.ptr(v_splats), _lib.stream())
        return v_splats
    if hits is not None:
        if hits.dtype != torch.uint8 or hits.numel() < vals.numel() or hits.device != splats.device:
            raise ValueError("blend_backward: hits must be the uint8 mask blend_forward filled for these intersections")
    _lib.call("adb_raster_blend_bwd", W, H, N, _lib.ptr(splats), _lib.ptr(vals) if vals.numel() else None,
              _lib.ptr(offsets), _lib.ptr(alphas), _lib.ptr(last_ids), _lib.ptr(v_colors), _lib.ptr(v_alphas),
              _lib.ptr(v_splats), _lib.ptr(hits), _lib.stream())
    return v_splats


class _RasterizeOneCamera(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means, quats, scales, opacities, sh, colors_direct, viewmat, K, campos, W, H, sh_degree, eps2d,
                near, far, radius_clip, cam_id, n_cams):
        _lib.require_cuda(means)
        N = means.shape[0]
        with torch.cuda.device(means.device):
            cnt = new_tile_counts(W, H, means.device) if N > 0 else None
            radii, splats, tpg = project(means, quats, scales, opacities, sh, sh_degree, viewmat, K, campos, W, H,
                                         eps2d, near, far, radius_clip, tile_counts=cnt)
            if colors_direct is not None:
                splats[:, 8:11] = colors_direct
            keys, vals, offsets, n_isect = intersect(radii, splats, tpg, W, H, cam_id, n_cams, counts=cnt)
            hits = new_hit_mask(vals)
            colors, alphas, last_ids = blend_forward(W, H, N, splats, vals, offsets, hits=hits)
        ctx.hits = hits
        ctx.save_for_backward(means, quats, scales, opacities, sh, viewmat, K, campos, radii, splats, vals, offsets,
                              alphas, last_ids)
        ctx.cfg = (W, H, sh_degree, eps2d, near, far, radius_clip, colors_direct is not None)
        ctx.mark_non_differentiable(radii, splats, tpg, keys, vals, offsets)
        return colors, alphas, radii, splats, tpg, keys, vals, offsets

    @staticmethod
    def backward(ctx, v_colors, v_alphas, *_unused):
        (means, quats, scales, opacities, sh, viewmat, K, campos, radii, splats, vals, offsets, alphas,
         last_ids) = ctx.saved_tensors
        W, H, sh_degree, eps2d, near, far, radius_clip, direct = ctx.cfg
        N = means.shape[0]
        dev = means.device
        v_colors = torch.zeros(H, W, 4, device=dev) if v_colors is None else _f32c(v_colors)
        v_alphas = torch.zeros(H, W, device=dev) if v_alphas is None else _f32c(v_alphas)
        with torch.cuda.device(dev):
            v_splats = blend_backward(W, H, N, splats, vals, offsets, alphas, last_ids, v_colors, v_alphas, hits=ctx.hits)
            v_means, v_quats, v_scales, v_opac, v_sh, v_view, v_campos = project_backward(
                means, quats, scales, opacities, sh, sh_degree, viewmat, K, campos, W, H, eps2d, near, far, radius_clip,
                radii, splats, v_splats)
        v_direct = None
        if direct:
            live = (radii > 0).any(-1, keepdim=True)
            v_direct = v_splats[:, 6:9] * live
        return (v_means, v_quats, v_scales, v_opac, v_sh, v_direct, v_view, None, v_campos,
                None, None, None, None, None, None, None, None, None)


class _RasterizeCameras(torch.autograd.Function):
    """C > 1 cameras of the same Gaussians (BASELINE config 4: an 8-view batch per optimiser step), stage by stage: one
    multi-view projection (parameters read once), one view-batched intersection, one blend forward launch for all views.
    Backward: one blend backward launch, then ONE multi-view projection backward (11 geometry gradients summed in registers)
    and ONE multi-view SH backward (v_sh written once) (csrc/raster_project_bwd_multi.cu)."""

    @staticmethod
    def forward(ctx, means, quats, scales, opacities, sh, viewmats, Ks, camposs, W, H, sh_degree, eps2d, near, far,
                radius_clip, exchange=None, capacities=None):
        _lib.require_cuda(means)
        ctx.exchange = exchange
        Cn = viewmats.shape[0]
        dev = means.device
        with torch.cuda.device(dev):
            cnt = new_tile_counts(W, H, dev, Cn)
            radii, splats, tpg = project_multi(means, quats, scales, opacities, sh, sh_degree, viewmats, Ks, camposs, W, H,
                                               eps2d, near, far, radius_clip, cnt)
            caps = None
            if capacities is not None:
                caps = [int(c) for c in capacities] if hasattr(capacities, "__len__") else [int(capacities)] * Cn
            keys, vals, offsets, info, _ = intersect_multi(radii, splats, tpg, W, H, cnt, capacities=caps)
            hits = new_hit_mask(vals)
            colors, alphas, last_ids = blend_forward_multi(W, H, splats, vals, offsets, hits=hits)
        ctx.save_for_backward(means, quats, scales, opacities, sh, viewmats, Ks, camposs, radii, splats, alphas, last_ids,
                              vals, offsets)
        ctx.cfg = (W, H, sh_degree)
        ctx.hits = hits
        # gsplat offsets index the concatenated list (padded per camera in capacity mode): the segment layout of intersect_multi
        isect_offsets = offsets[:, :-1].contiguous()
        if capacities is None:
            overflow = torch.zeros(1, dtype=torch.int32, device=dev)
        else:
            overflow = info["overflow"].amax().reshape(1)
        ctx.mark_non_differentiable(radii, splats, tpg, keys, vals, isect_offsets, overflow)
        return colors, alphas, radii, splats, tpg, keys, vals, isect_offsets, overflow

    @staticmethod
    def backward(ctx, v_colors, v_alphas, *_unused):
        W, H, sh_degree = ctx.cfg
        (means, quats, scales, opacities, sh, viewmats, Ks, camposs, radii, splats, alphas, last_ids, vals,
         offsets) = ctx.saved_tensors
        Cn = viewmats.shape[0]
        dev = means.device
        v_colors = torch.zeros(Cn, H, W, 4, device=dev) if v_colors is None else _f32c(v_colors)
        v_alphas = torch.zeros(Cn, H, W, device=dev) if v_alphas is None else _f32c(v_alphas)
        with torch.cuda.device(dev):
            v_splats = blend_backward_multi(W, H, splats, vals, offsets, alphas, last_ids, v_colors, v_alphas, hits=ctx.hits)
            ex = ctx.exchange
            grads = multi_view_backward(means, quats, scales, sh, sh_degree, viewmats, Ks, camposs, W, H, radii, splats,
                                        v_splats, out=(dict(ex.views) if ex is not None else None), exchange=ex)
        v_means, v_quats, v_scales, v_opac, v_sh, v_views, v_campos = grads
        if ex is not None:      # the bucket is reused by the next step: hand autograd its own copies
            v_means, v_quats, v_scales, v_opac = v_means.clone(), v_quats.clone(), v_scales.clone(), v_opac.clone()
        return (v_means, v_quats, v_scales, v_opac, v_sh, v_views, None, v_campos, None, None, None, None, None, None, None,
                None, None)


def mask_rgb_grad(splats, v_splats, out):
    """Colour gradient masked by the SH clamp (rgb = max(.,0): zero gradient where the record's colour is 0); invisible
    Gaussians have zero accumulators.  ``splats`` / ``v_splats`` [..., N, 12] -> ``out`` [..., N, 3]."""
    return torch.where(splats[..., 8:11] > 0, v_splats[..., 6:9], v_splats.new_zeros(()), out=out)


def multi_view_backward(means, quats, scales, sh, sh_degree, viewmats, Ks, camposs, W, H, radii, splats, v_splats,
                        out=None, exchange=None):
    """Projection + SH backward for C stacked local views (csrc/raster_project_bwd_multi.cu).

    ``out``: optional dict of preallocated gradient tensors (``v_means [N,3], v_quats [N,4], v_scales [N,3], v_opac [N],
    v_sh [N,16,3]``), e.g. views of a flat communication bucket.
    ``exchange`` (multi-GPU; a ``parallel.MultiViewExchange``): the colour gradients of the local views
    are gathered while the geometry kernels run, the 11 geometry floats are summed over ranks while the SH gradient of EVERY
    rank's views is expanded; ``None`` = single process.  Returns (v_means, v_quats, v_scales, v_opac, v_sh, v_viewmats[C,4,4],
    v_campos[C,3] of the local views)."""
    N, Cn = means.shape[0], viewmats.shape[0]
    dev = means.device
    out = out or {}
    v_means = out.get("v_means") if out.get("v_means") is not None else torch.empty_like(means)
    v_quats = out.get("v_quats") if out.get("v_quats") is not None else torch.empty_like(quats)
    v_scales = out.get("v_scales") if out.get("v_scales") is not None else torch.empty_like(scales)
    v_opac = out.get("v_opac") if out.get("v_opac") is not None else torch.empty(N, dtype=torch.float32, device=dev)
    v_sh = out.get("v_sh") if out.get("v_sh") is not None else torch.empty_like(sh)
    v_views = torch.zeros(Cn, 4, 4, dtype=torch.float32, device=dev)
    v_campos = torch.zeros(Cn, 3, dtype=torch.float32, device=dev)
    Vc, Kc, Pc = _f32c(viewmats.detach()), _f32c(Ks.detach()), _f32c(camposs.detach())
    # colour gradient masked by the SH clamp (rgb = max(.,0): zero gradient where the record's colour is 0); invisible
    # Gaussians have zero accumulators.  One process: the geometry kernel writes it as it reads the same two records
    # (bit for bit mask_rgb_grad).  Multi-GPU: produced first so that its all-gather overlaps the geometry kernel.
    g_rgb = out.get("g_rgb")
    if exchange is not None and getattr(exchange, "gather_started", False):
        pass                                      # per-view gathers were issued as each view's blend backward finished
    else:
        if g_rgb is None:
            g_rgb = torch.empty(Cn, N, 3, dtype=torch.float32, device=dev)
        if exchange is not None:
            mask_rgb_grad(splats, v_splats, g_rgb)
            exchange.start_gather(g_rgb, Pc)
    _lib.call("adb_raster_project_bwd_multi", N, Cn, _lib.ptr(means), _lib.ptr(quats), _lib.ptr(scales), _lib.ptr(Vc),
              _lib.ptr(Kc), W, H, _lib.ptr(radii), _lib.ptr(splats), _lib.ptr(v_splats), _lib.ptr(v_means),
              _lib.ptr(v_quats), _lib.ptr(v_scales), _lib.ptr(v_opac), _lib.ptr(g_rgb) if exchange is None else None,
              _lib.ptr(v_views), _lib.stream())
    if exchange is None:
        _lib.call("adb_raster_sh_bwd_multi", N, Cn, _lib.ptr(means), _lib.ptr(sh), int(sh_degree), _lib.ptr(Pc),
                  _lib.ptr(g_rgb), _lib.ptr(v_sh), _lib.ptr(v_means), 1, 0, 0, _lib.ptr(v_campos), _lib.stream())
        return v_means, v_quats, v_scales, v_opac, v_sh, v_views, v_campos
    # Multi-GPU: the SH backward in its split form.  The direction term (gradient of the colour w.r.t. the mean through the view
    # direction) is linear in the views, so each rank adds it for its LOCAL views to its partial geometry sums and the reduce
    # carries it; only the outer product basis(dir) (x) v_rgb needs every rank's colour gradients, and that expansion — the
    # part every rank repeats for all views — then runs without the SH coefficients and the basis gradients.
    _lib.call("adb_raster_sh_dir_bwd_multi", N, Cn, _lib.ptr(means), _lib.ptr(sh), int(sh_degree), _lib.ptr(Pc), _lib.ptr(splats),
              _lib.ptr(v_splats), _lib.ptr(v_means), _lib.ptr(v_campos), _lib.stream())
    exchange.start_reduce()                       # geometry sums (v_means | v_quats | v_scales | v_opac), overlaps the expansion
    g_all, P_all = exchange.wait_gather()
    _lib.call("adb_raster_sh_expand_multi", N, int(g_all.shape[0]), _lib.ptr(means), int(sh_degree), _lib.ptr(P_all),
              _lib.ptr(g_all), _lib.ptr(v_sh), _lib.stream())
    exchange.wait_reduce()
    return v_means, v_quats, v_scales, v_opac, v_sh, v_views, v_campos


def rasterization(means: torch.Tensor, quats: torch.Tensor, scales: torch.Tensor, opacities: torch.Tensor,
                  colors: torch.Tensor, viewmats: torch.Tensor, Ks: torch.Tensor, width: int, height: int,
                  near_plane: float = 0.01, far_plane: float = 1e10, radius_clip: float = 0.0, eps2d: float = 0.3,
                  sh_degree: Optional[int] = None, packed: bool = False, tile_size: int = 16,
                  backgrounds: Optional[torch.Tensor] = None, render_mode: str = "RGB",
                  rasterize_mode: str = "classic", absgrad: bool = False, grad_exchange=None, isect_capacity=None,
                  **unsupported):
    """See module docstring.  ``colors`` is SH [N,K,3] when ``sh_degree`` is given, else RGB [N,3].

    ``grad_exchange`` (not in gsplat; multi-GPU view-parallel training, BASELINE config 4): a
    ``parallel.MultiViewExchange``.  The backward then leaves on every rank the gradients summed over the views of ALL ranks
    (all-gather of the colour gradients + all-reduce of the geometry gradients inside the multi-view backward).

    ``isect_capacity`` (not in gsplat; int or one int per camera): size the intersection buffers by this bound instead of reading
    the count back — the call then has NO host sync (gsplat itself syncs on ``cum_tiles_per_gauss[-1].item()``).
    ``meta["isect_ids"] / ["flatten_ids"]`` are then padded to the capacity per camera and ``meta["isect_overflow"]`` (int32[1] on
    the device) is non-zero when a view needed more: read it together with the loss; the image of that view is then incomplete."""
    if unsupported:
        raise NotImplementedError(f"rasterization(): unsupported arguments {sorted(unsupported)}")
    if packed or absgrad or rasterize_mode != "classic" or tile_size != 16:
        raise NotImplementedError("only packed=False, absgrad=False, rasterize_mode='classic', tile_size=16 "
                                  "(the reference's configuration, h3dgsv3.py:664-680)")
    if render_mode not in ("RGB", "RGB+D"):
        raise NotImplementedError("render_mode must be 'RGB' or 'RGB+D'")
    _lib.require_cuda(means)
    N = means.shape[0]
    C_ = viewmats.shape[0]
    assert means.shape == (N, 3) and quats.shape == (N, 4) and scales.shape == (N, 3) and opacities.shape == (N,)
    assert viewmats.shape == (C_, 4, 4) and Ks.shape == (C_, 3, 3)
    means, quats, scales, opacities = _f32c(means), _f32c(quats), _f32c(scales), _f32c(opacities)
    sh = direct = None
    if sh_degree is not None:
        assert colors.dim() == 3 and colors.shape[0] == N and colors.shape[2] == 3
        if (sh_degree + 1) ** 2 > colors.shape[1]:
            raise ValueError("sh_degree needs more SH coefficients than colors provides")
        sh = _f32c(colors)
        if sh.shape[1] != 16:  # kernel reads a fixed 16x3 block
            sh = torch.cat([sh, sh.new_zeros(N, 16 - sh.shape[1], 3)], 1) if sh.shape[1] < 16 else sh[:, :16].contiguous()
    else:
        assert colors.shape == (N, 3)
        direct = _f32c(colors)
    th, tw = (height + TILE - 1) // TILE, (width + TILE - 1) // TILE
    if grad_exchange is not None and sh is None:
        raise NotImplementedError("grad_exchange needs SH colours (sh_degree given)")
    if isect_capacity is not None and sh is None:
        raise NotImplementedError("isect_capacity needs SH colours (sh_degree given)")
    if (C_ > 1 or grad_exchange is not None or isect_capacity is not None) and sh is not None:
        # multi-view batch: stacked buffers, one multi-view projection/SH backward (see _RasterizeCameras)
        Vs = _f32c(viewmats)
        camposs = torch.inverse(Vs)[:, :3, 3].contiguous()
        col, alp, radii, splats, tpg, isect_ids, flatten_ids, isect_offsets, overflow = _RasterizeCameras.apply(
            means, quats, scales, opacities, sh, Vs, _f32c(Ks).detach(), camposs, int(width), int(height), int(sh_degree),
            float(eps2d), float(near_plane), float(far_plane), float(radius_clip), grad_exchange, isect_capacity)
        if backgrounds is not None:
            col = torch.cat([col[..., :3] + (1.0 - alp[..., None]) * backgrounds.view(C_, 1, 1, 3), col[..., 3:]], -1)
        meta = {
            "radii": radii, "means2d": splats[..., 0:2], "depths": splats[..., 11], "conics": splats[..., 2:5],
            "opacities": opacities, "tiles_per_gauss": tpg, "isect_ids": isect_ids, "flatten_ids": flatten_ids,
            "isect_offsets": isect_offsets.view(C_, th, tw), "isect_overflow": overflow,
            "width": width, "height": height, "tile_size": TILE, "tile_width": tw, "tile_height": th, "n_cameras": C_,
        }
        return (col if render_mode == "RGB+D" else col[..., :3]), alp[..., None], meta
    out_c, out_a, radii_l, metas = [], [], [], []
    base = 0
    for c in range(C_):
        V = _f32c(viewmats[c])
        K = _f32c(Ks[c]).detach()
        campos = torch.inverse(V)[:3, 3].contiguous() if sh is not None else None
        col, alp, radii, splats, tpg, keys, vals, offs = _RasterizeOneCamera.apply(
            means, quats, scales, opacities, sh, direct, V, K, campos, int(width), int(height),
            int(sh_degree) if sh_degree is not None else 0, float(eps2d), float(near_plane), float(far_plane),
            float(radius_clip), c, C_)
        if backgrounds is not None:
            col = torch.cat([col[..., :3] + (1.0 - alp[..., None]) * backgrounds[c].view(1, 1, 3), col[..., 3:]], -1)
        out_c.append(col if render_mode == "RGB+D" else col[..., :3])
        out_a.append(alp[..., None])
        radii_l.append(radii)
        metas.append((splats, tpg, keys, vals, offs + base))  # gsplat offsets index the concatenated list
        base += int(vals.numel())
    meta = {
        "radii": torch.stack(radii_l),
        "means2d": torch.stack([m[0][:, 0:2] for m in metas]),
        "depths": torch.stack([m[0][:, 11] for m in metas]),
        "conics": torch.stack([m[0][:, 2:5] for m in metas]),
        "opacities": opacities,
        "tiles_per_gauss": torch.stack([m[1] for m in metas]),
        "isect_ids": torch.cat([m[2] for m in metas]),
        "flatten_ids": torch.cat([m[3] for m in metas]),
        "isect_offsets": torch.stack([m[4][:-1].view(th, tw) for m in metas]),
        "width": width, "height": height, "tile_size": TILE, "tile_width": tw, "tile_height": th, "n_cameras": C_,
    }
    return torch.stack(out_c), torch.stack(out_a), meta

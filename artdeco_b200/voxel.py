"""Host-side mirror of ``SceneModel.update_voxel`` (Reconstruct/scene/scene_models/h3dgsv3.py:227-316; SURVEY.md §8a R9):
voxel-hash class ids for the LoD / ``mlp_cov`` class embedding.  Same arguments, same return values (a 3-tuple, or the
reference's 2-tuple in the cold-start branch), integer results bit-identical to the reference's sort-based formulation.

What runs differently: three full ``torch.unique`` sorts + ``scatter_max`` + ``searchsorted`` become two hash-table passes and a
vote with packed 64-bit atomics (csrc/voxel.cu); only the DISTINCT previously-empty voxels are sorted (to reproduce the order
in which the reference numbers new classes).  Voxel index arithmetic follows what the reference computes ON THE GPU:
``(p - min) / voxel_size`` with a Python-float divisor is evaluated by PyTorch's CUDA kernel as ``(p - min) * (1 / voxel_size)``
in fp32 (BinaryDivTrueKernel.cu's CPU-scalar fast path)."""
from __future__ import annotations

import torch

from . import _lib
from ._lib import f32, i32, i64, vp

_lib.register("adb_voxel_vote", [i64, vp, vp, vp, f32, vp, i64, vp, vp, i64, vp, vp, vp, vp, vp])
_lib.register("adb_voxel_match_new", [i64, vp, vp, f32, vp, i64, vp, i32, vp, i64, vp, vp, vp, vp, vp, vp])
_lib.register("adb_voxel_rank_new", [i64, i32, vp, vp, i64, vp, vp, i64, vp, vp])


def _pow2(n: int) -> int:
    p = 1024
    while p < n:
        p <<= 1
    return p


def max_class_id(cls: torch.Tensor) -> int:
    """The largest class id (one host sync, like the reference's own ``max().item()``).  The kernels carry class ids as
    32-bit values (the vote packs ``count << 32 | 0xffffffff - id``), so an id at or above 2^32 - 1 is refused."""
    m = int(cls.max().item())
    if m >= 0xFFFFFFFF:
        raise _lib.ArtdecoB200Error(f"update_voxel: class id {m} does not fit the kernels' 32-bit ids (must be < 2^32 - 1)")
    return m


@torch.no_grad()
def update_voxel(new_xyz: torch.Tensor, xyz: torch.Tensor, cls_id: torch.Tensor, voxel_size: float = 0.1):
    """Returns ``(updated_orig_cls_id [N,1] int64, updated_new_cls_id [M,1] int64, new_voxel_count)``; with no original points
    the reference's cold-start pair ``(new_cls_id [M,1], voxel_count)``."""
    _lib.require_cuda(new_xyz)
    dev = new_xyz.device
    M, N = int(new_xyz.shape[0]), int(xyz.shape[0])
    new_c = new_xyz.detach().float().contiguous()
    if M == 0 and N == 0:
        z = torch.zeros(0, 1, dtype=torch.long, device=dev)
        return z, 0
    overflow = torch.zeros(1, dtype=torch.int32, device=dev)
    new_out = torch.zeros(max(M, 1), dtype=torch.long, device=dev)
    # NOTE the reciprocal: this is the arithmetic of the reference on CUDA (see module docstring)
    voxel = float(voxel_size)
    with torch.cuda.device(dev):
        if N > 0:
            xyz_c = xyz.detach().float().contiguous()
            cls = cls_id.detach().reshape(-1).long().contiguous()
            mn = (torch.minimum(xyz_c.amin(0), new_c.amin(0)) if M > 0 else xyz_c.amin(0)).contiguous()
            max_cls = max_class_id(cls)                          # the reference syncs here too (h3dgsv3.py:260)
            V = P = _pow2(2 * N)
            vkeys = torch.full((V,), -1, dtype=torch.int64, device=dev)
            pkeys = torch.full((P,), -1, dtype=torch.int64, device=dev)
            pcount = torch.zeros(P, dtype=torch.int32, device=dev)
            best = torch.zeros(V, dtype=torch.int64, device=dev)
            slot_of = torch.empty(N, dtype=torch.int32, device=dev)
            orig_out = torch.empty(N, dtype=torch.long, device=dev)
            _lib.call("adb_voxel_vote", N, _lib.ptr(xyz_c), _lib.ptr(cls), _lib.ptr(mn), voxel, _lib.ptr(vkeys), V,
                      _lib.ptr(pkeys), _lib.ptr(pcount), P, _lib.ptr(best), _lib.ptr(slot_of), _lib.ptr(orig_out),
                      _lib.ptr(overflow), _lib.stream())
        else:
            mn = new_c.amin(0).contiguous()
            max_cls, V, vkeys, best, orig_out = -1, 0, None, None, None
        n_new_voxels = 0
        if M > 0:
            U = _pow2(2 * M)
            ukeys = torch.full((U,), -1, dtype=torch.int64, device=dev)
            uslot = torch.empty(M, dtype=torch.int32, device=dev)
            ulist = torch.empty(M, dtype=torch.int64, device=dev)
            ucount = torch.zeros(1, dtype=torch.int32, device=dev)
            _lib.call("adb_voxel_match_new", M, _lib.ptr(new_c), _lib.ptr(mn), voxel, _lib.ptr(vkeys), V, _lib.ptr(best),
                      int(N > 0), _lib.ptr(ukeys), U, _lib.ptr(uslot), _lib.ptr(new_out), _lib.ptr(ulist), _lib.ptr(ucount),
                      _lib.ptr(overflow), _lib.stream())
            n_new_voxels = int(ucount.item())
            if n_new_voxels > 0:
                srt = torch.sort(ulist[:n_new_voxels]).values.contiguous()      # only the distinct new voxels are sorted
                urank = torch.empty(U, dtype=torch.int32, device=dev)
                _lib.call("adb_voxel_rank_new", M, n_new_voxels, _lib.ptr(srt), _lib.ptr(ukeys), U, _lib.ptr(urank),
                          _lib.ptr(uslot), max_cls + 1, _lib.ptr(new_out), _lib.stream())
        if int(overflow.item()):
            raise _lib.ArtdecoB200Error("update_voxel: a voxel index exceeds 2^21 per axis (scene extent / voxel_size too large)")
    new_out = new_out[:M].unsqueeze(-1)
    if N == 0:
        return new_out, n_new_voxels
    return orig_out.unsqueeze(-1), new_out, n_new_voxels

"""Host-side multi-GPU plumbing for the two places the hot path shards (SURVEY.md §8e): one process per GPU,
``torch.distributed`` (NCCL on GPUs; gloo in the CPU tests).

* rasterizer, view-parallel: every rank holds a replica of the Gaussians and renders its own views; a step gathers the
  12-byte colour gradients of every view and sums the 11 geometry floats per Gaussian over the ranks
  (``MultiViewExchange``);
* MASt3R: independent pairs are split contiguously across ranks, no collective.
"""
from __future__ import annotations

import torch
import torch.distributed as dist

GRAD_FLOATS = 59    # dense per-Gaussian gradient the exchange replaces: means 3, quats 4, scales 3, opacity 1, SH 48

GEOM_FIELDS = (("v_means", 3), ("v_quats", 4), ("v_scales", 3), ("v_opac", 1))
GEOM_FLOATS = sum(m for _, m in GEOM_FIELDS)  # 11


class MultiViewExchange:
    """Gradient exchange of one multi-view optimiser step split over ranks (BASELINE config 4, SURVEY.md §8e).

    A dense all-reduce of the [N,59] gradient block moves 2(G-1)/G x 236 MB per rank at N = 1M.  48 of the 59 floats are SH
    gradients, and the SH gradient of one view is the outer product basis(dir_view)[16] x v_rgb[3]: it is fully determined by
    12 bytes per (view, Gaussian) plus the view's camera centre.  So the ranks
      * ALL-GATHER the clamp-masked colour gradients ``g_rgb [C_local, N, 3]`` (12 MB per view) and the camera centres, and
        every rank expands the SH gradient of ALL views locally (``adb_raster_sh_expand_multi``);
      * ALL-REDUCE only the 11 geometry floats per Gaussian (44 MB) — one flat bucket the backward kernels write into (the
        colour's gradient through the view direction is added per rank for its local views, ``adb_raster_sh_dir_bwd_multi``).
    Both collectives are asynchronous: the gather overlaps the geometry kernels, the reduce overlaps the expansion
    (``raster.multi_view_backward``).  Result on every rank: exactly the sum over all views of the single-view gradients.
    Works with NCCL (GPU) and gloo (CPU tests)."""

    def __init__(self, n_gaussians: int, views_local: int, device, group=None):
        self.n = n_gaussians
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.views_local = views_local
        self.geom = torch.zeros(n_gaussians * GEOM_FLOATS, dtype=torch.float32, device=device)
        self.views = {}
        o = 0
        for name, m in GEOM_FIELDS:
            v = self.geom[o:o + n_gaussians * m]
            self.views[name] = v.view(n_gaussians, m) if m > 1 else v
            o += n_gaussians * m
        # gathered colour gradients, VIEW-major: g_all[c, r] = view c of rank r (one contiguous all-gather output per local view,
        # so that a view's gather can start as soon as ITS blend backward has finished, while the next view is still rendering)
        self.g_all = torch.empty(views_local, self.world, n_gaussians, 3, dtype=torch.float32, device=device)
        self.campos_all = torch.empty(views_local, self.world, 3, dtype=torch.float32, device=device)
        self._gather, self._reduce = [], None
        self._views_started = 0
        self.bytes_per_step = {"all_gather_recv": (self.world - 1) * views_local * n_gaussians * 12,
                               "all_reduce_payload": n_gaussians * GEOM_FLOATS * 4,
                               "dense_all_reduce_payload_replaced": n_gaussians * GRAD_FLOATS * 4}

    def start_gather_view(self, c: int, g_view: torch.Tensor, campos: torch.Tensor | None = None):
        """Asynchronous all-gather of ONE local view's colour gradients [N,3] (and, with the first view, of the camera centres
        [C_local,3] of the step)."""
        assert g_view.shape == (self.n, 3)
        if self.world == 1:
            self.g_all[c, 0].copy_(g_view)
            if campos is not None:
                self.campos_all[:, 0].copy_(campos)
        else:
            self._gather.append(dist.all_gather_into_tensor(self.g_all[c].view(self.world * self.n, 3), g_view.contiguous(),
                                                            group=self.group, async_op=True))
            if campos is not None:
                # [world, C_local, 3] staging -> transposed into the view-major table after the wait
                self._campos_stage = torch.empty(self.world, self.views_local, 3, dtype=torch.float32, device=g_view.device)
                self._gather.append(dist.all_gather_into_tensor(self._campos_stage.view(self.world * self.views_local, 3),
                                                                campos.contiguous(), group=self.group, async_op=True))
        self._views_started += 1

    def start_gather(self, g_rgb: torch.Tensor, campos: torch.Tensor):
        """All local views at once (used when the views' gradients become available together, e.g. under autograd)."""
        assert g_rgb.shape == (self.views_local, self.n, 3) and campos.shape == (self.views_local, 3)
        for c in range(self.views_local):
            self.start_gather_view(c, g_rgb[c], campos if c == 0 else None)

    @property
    def gather_started(self) -> bool:
        return self._views_started > 0

    def wait_gather(self):
        """Returns (g_all [C_local*world, N, 3], campos_all [C_local*world, 3]) in the same (view-major) order."""
        for w in self._gather:
            w.wait()
        if self._gather and self.world > 1:
            self.campos_all.copy_(self._campos_stage.transpose(0, 1))
        self._gather = []
        self._views_started = 0
        return self.g_all.view(-1, self.n, 3), self.campos_all.view(-1, 3)

    def start_reduce(self):
        self._reduce = dist.all_reduce(self.geom, group=self.group, async_op=True) if self.world > 1 else None

    def wait_reduce(self):
        if self._reduce is not None:
            self._reduce.wait()
            self._reduce = None


def views_for_rank(n_views: int, world: int, rank: int) -> list[int]:
    """GPU g renders views {v : v mod G = g} (SURVEY.md §8e)."""
    return [v for v in range(n_views) if v % world == rank]


def shard_pairs(n_pairs: int, world: int, rank: int) -> range:
    """Contiguous, balanced split of independent MASt3R pairs (sizes differ by at most one)."""
    base, rem = divmod(n_pairs, world)
    start = rank * base + min(rank, rem)
    return range(start, start + base + (1 if rank < rem else 0))

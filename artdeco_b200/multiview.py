"""Multi-view optimiser step engine (BASELINE config 4: "1M-Gaussian scene, 8-view batch optimise, NCCL per-Gaussian grad
allreduce at 2/4/8 GPUs"; SURVEY.md §8e).

One step = forward + backward of every LOCAL view of the batch against the replicated Gaussians, then the gradient
exchange, leaving on every rank the sum over ALL views of the per-view gradients (the step's semantics become "sum of C view
losses"; the reference optimises one view per step, Reconstruct/scene/scene_models/h3dgsv3.py:406-464).

Design:
  * the whole local compute (projection -> tile-bucketed intersection -> blend fwd -> blend bwd) runs stage by stage over
    the batch, one launch per stage for all local views (raster.project_multi / intersect_multi / blend_*_multi); it has no
    host sync (intersection buffers are sized by a capacity measured once) and is captured in ONE CUDA graph;
  * gradients are produced by the multi-view backward kernels (parameters read once, gradients written once);
  * multi-GPU: 12 B colour gradients all-gathered, 11 geometry floats all-reduced, both overlapped with the backward
    kernels, instead of a dense [N,59] all-reduce — by ``parallel.MultiViewExchange`` (NCCL).
"""
from __future__ import annotations

import torch

from . import _lib
from . import raster as R
from .parallel import MultiViewExchange

KEYS = ("means", "quats", "scales", "opacities", "sh")


class MultiViewStep:
    def __init__(self, params: dict, viewmats: torch.Tensor, Ks: torch.Tensor, W: int, H: int, world: int = 1,
                 sh_degree: int = 3, eps2d: float = 0.01, near: float = 0.01, far: float = 1e10, radius_clip: float = 0.0,
                 graph: bool = True, capacity_margin: float = 1.25, overlap_views: bool = False):  # overlap_views: no effect
        """``params``: dict of the five parameter tensors on the device; ``viewmats [C,4,4]``, ``Ks [C,3,3]``: the LOCAL
        views (``parallel.views_for_rank``).  ``world`` > 1 needs an initialised process group, whose ranks then exchange
        gradients through ``parallel.MultiViewExchange``."""
        _lib.require_cuda(params["means"])
        self.p = {k: params[k].detach().contiguous() for k in KEYS}
        self.dev = self.p["means"].device
        self.N = self.p["means"].shape[0]
        self.C = int(viewmats.shape[0])
        self.W, self.H = int(W), int(H)
        self.cfg = (int(sh_degree), float(eps2d), float(near), float(far), float(radius_clip))
        self.V = viewmats.detach().float().contiguous().to(self.dev)
        self.K = Ks.detach().float().contiguous().to(self.dev)
        self.P = torch.inverse(self.V)[:, :3, 3].contiguous()
        N, C, dev = self.N, self.C, self.dev
        self.radii = torch.empty(C, N, 2, dtype=torch.int32, device=dev)
        self.splats = torch.empty(C, N, R.SPLAT_STRIDE, dtype=torch.float32, device=dev)
        self.tpg = torch.empty(C, N, dtype=torch.int32, device=dev)
        self.v_splats = torch.zeros(C, N, R.SPLAT_STRIDE, dtype=torch.float32, device=dev)
        self.v_colors = torch.zeros(C, H, W, 4, dtype=torch.float32, device=dev)     # static upstream-gradient buffers
        self.v_alphas = torch.zeros(C, H, W, dtype=torch.float32, device=dev)
        self.world = world
        self.exchange = MultiViewExchange(N, C, dev) if world > 1 else None
        self.grads = {"v_sh": torch.empty(N, 16, 3, dtype=torch.float32, device=dev)}
        if self.exchange is not None:
            self.grads.update(self.exchange.views)          # geometry gradients live in the all-reduce bucket
        else:
            self.grads.update(v_means=torch.empty(N, 3, device=dev), v_quats=torch.empty(N, 4, device=dev),
                              v_scales=torch.empty(N, 3, device=dev), v_opac=torch.empty(N, device=dev))
        self.grads["g_rgb"] = torch.empty(C, N, 3, dtype=torch.float32, device=dev)
        T = ((W + R.TILE - 1) // R.TILE) * ((H + R.TILE - 1) // R.TILE)
        self.counts = torch.zeros(C, 2 * R.COUNTER_COPIES * T, dtype=torch.int32, device=dev)   # per-view tile counters
        self.n_dev = torch.zeros(C, dtype=torch.int64, device=dev)          # per-view intersection count ...
        self.overflow_dev = torch.zeros(C, dtype=torch.int32, device=dev)   # ... and overflow flag of the last step
        self.capacity = None
        self.margin = capacity_margin
        self.use_graph = graph
        # No effect, kept because callers set it: every stage is one launch for the whole batch, so there are no per-view
        # launches left to overlap on a second stream.
        self.overlap_views = overlap_views
        self.graph = None
        self.render = None          # (colors [C,H,W,4], alphas [C,H,W]) of the last step (world > 1: per-view lists)
        self.info = None            # {"n_isect": int64[C], "overflow": int32[C]} device tensors of the last step
        self.v_views = self.v_campos = None

    # ---- stages -----------------------------------------------------------------------------------------------------
    def _project(self):
        """Projection + SH + tile counting of every local view in one pass over the parameters."""
        sh_degree, eps2d, near, far, rclip = self.cfg
        p = self.p
        self.counts.zero_()
        R.project_multi(p["means"], p["quats"], p["scales"], p["opacities"], p["sh"], sh_degree, self.V, self.K, self.P,
                        self.W, self.H, eps2d, near, far, rclip, self.counts, out=(self.radii, self.splats, self.tpg))

    def _raster(self, views, capacity):
        """intersection -> blend fwd -> blend bwd of the local views ``views`` (a slice), one launch per stage."""
        W, H = self.W, self.H
        caps = None if capacity is None else capacity[views]
        self.v_splats[views].zero_()
        _, vals, offs, _, seg = R.intersect_multi(self.radii[views], self.splats[views], self.tpg[views], W, H,
                                                  self.counts[views], capacities=caps, keys=False,
                                                  info={"n_isect": self.n_dev[views], "overflow": self.overflow_dev[views]})
        hits = R.new_hit_mask(vals)                    # the forward's culling decisions, reused by the backward
        col, alp, last = R.blend_forward_multi(W, H, self.splats[views], vals, offs, hits=hits)
        R.blend_backward_multi(W, H, self.splats[views], vals, offs, alp, last, self.v_colors[views], self.v_alphas[views],
                               out=self.v_splats[views], hits=hits)
        return col, alp, seg

    def _local_views(self, capacity):
        """Every local view as one batch; no host sync when capacity is given."""
        self._project()
        return self._raster(slice(0, self.C), capacity)

    def _view(self, c, capacity):
        """Multi-GPU route: intersection -> blend fwd -> blend bwd -> masked colour gradient of local view c alone, so that its
        gather can start as soon as its blend backward has finished.  The projection of all views runs before view 0."""
        if c == 0:
            self._project()
        col, alp, _ = self._raster(slice(c, c + 1), capacity)
        R.mask_rgb_grad(self.splats[c], self.v_splats[c], self.grads["g_rgb"][c])
        return col[0], alp[0]

    def _gather_view(self, c):
        """Hands local view c's colour gradient to the exchange as soon as its blend backward has been issued."""
        self.exchange.start_gather_view(c, self.grads["g_rgb"][c], self.P if c == 0 else None)

    def _backward(self):
        p = self.p
        out = R.multi_view_backward(p["means"], p["quats"], p["scales"], p["sh"], self.cfg[0], self.V, self.K, self.P, self.W,
                                    self.H, self.radii, self.splats, self.v_splats, out=self.grads, exchange=self.exchange)
        self.v_views, self.v_campos = out[5], out[6]

    def calibrate(self):
        """One eager pass with one host sync: measures the intersection count of every local view and fixes the capacities."""
        with torch.cuda.device(self.dev):
            _, _, counts = self._local_views(None)
            self._backward()
        self.capacity = [int(n * self.margin) + 4096 for n in counts]
        self.n_isect = counts
        return counts

    def _capture(self):
        dev = self.dev
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):                     # warm-up off the capture stream
            if self.exchange is None:
                self._local_views(self.capacity)
                self._backward()
            else:
                for c in range(self.C):
                    self._view(c, self.capacity)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.info = {"n_isect": self.n_dev, "overflow": self.overflow_dev}
        if self.exchange is None:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                col, alp, _ = self._local_views(self.capacity)
                self._backward()
            self.graph, self.render = [g], (col, alp)
            return
        # multi-GPU: one graph PER VIEW, so that view c's colour gradients can be all-gathered (NCCL, outside the graphs)
        # while view c+1 renders; graph 0 also holds the projection of every local view
        graphs, cols, alps = [], [], []
        pool = None
        for c in range(self.C):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=pool):
                col, alp = self._view(c, self.capacity)
            pool = g.pool()
            graphs.append(g)
            cols.append(col)
            alps.append(alp)
        self.graph, self.render = graphs, (cols, alps)

    # ---- public -----------------------------------------------------------------------------------------------------
    def set_upstream(self, v_colors: torch.Tensor, v_alphas: torch.Tensor):
        self.v_colors.copy_(v_colors.reshape(self.v_colors.shape))
        self.v_alphas.copy_(v_alphas.reshape(self.v_alphas.shape))

    @torch.no_grad()
    def step(self):
        """Forward + backward of the local views with the current upstream gradients, then the exchange.  Returns the
        gradient dict (v_means, v_quats, v_scales, v_opac, v_sh); buffers are reused by the next step."""
        with torch.cuda.device(self.dev):
            if self.capacity is None:
                self.calibrate()
            if self.use_graph:
                if self.graph is None:
                    self._capture()
                if self.exchange is None:
                    self.graph[0].replay()
                else:
                    for c, g in enumerate(self.graph):
                        g.replay()
                        self._gather_view(c)
                    self._backward()                    # 2 kernels + the all-reduce, eager (NCCL outside the graphs)
            elif self.exchange is None:
                col, alp, _ = self._local_views(self.capacity)
                self.render, self.info = (col, alp), {"n_isect": self.n_dev, "overflow": self.overflow_dev}
                self._backward()
            else:
                cols, alps = [], []
                for c in range(self.C):
                    col, alp = self._view(c, self.capacity)
                    self._gather_view(c)
                    cols.append(col)
                    alps.append(alp)
                self.render, self.info = (cols, alps), {"n_isect": self.n_dev, "overflow": self.overflow_dev}
                self._backward()
        return self.grads

    def check_overflow(self):
        """Host sync.  Raises if any view's intersection count exceeded its capacity since the last check."""
        if self.info is None:
            return self.n_isect
        counts = [int(n) for n in self.info["n_isect"].tolist()]
        if int(self.info["overflow"].max()):
            raise _lib.ArtdecoB200Error(f"intersection capacity exceeded: counts {counts}, capacities {self.capacity}; "
                                        "call calibrate() again (the scene grew)")
        self.n_isect = counts
        return counts

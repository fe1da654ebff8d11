"""Multi-view optimiser step engine (BASELINE config 4: "1M-Gaussian scene, 8-view batch optimise, NCCL per-Gaussian grad
allreduce at 2/4/8 GPUs"; SURVEY.md §8e).

One step = forward + backward of every LOCAL view of the batch against the replicated Gaussians, then the gradient
exchange, leaving on every rank the sum over ALL views of the per-view gradients (the step's semantics become "sum of C view
losses"; the reference optimises one view per step, Reconstruct/scene/scene_models/h3dgsv3.py:406-464).

Design:
  * the whole local compute (projection -> tile-bucketed intersection -> blend fwd -> blend bwd, per view) has no host
    sync (intersection buffers are sized by a capacity measured once) and is captured in ONE CUDA graph;
  * gradients are produced by the multi-view backward kernels (parameters read once, gradients written once);
  * multi-GPU: 12 B colour gradients all-gathered, 11 geometry floats all-reduced, both overlapped with the backward
    kernels, instead of a dense [N,59] all-reduce — by ``parallel.MultiViewExchange`` (NCCL, default) or ``peer.PeerExchange``
    (this library's kernels storing into the other GPUs' memory over NVLink; ``exchange_kind="peer"`` / ``ADB_EXCHANGE=peer``).
"""
from __future__ import annotations

import torch

from . import _lib
from . import raster as R
from .peer import make_exchange

KEYS = ("means", "quats", "scales", "opacities", "sh")


class MultiViewStep:
    def __init__(self, params: dict, viewmats: torch.Tensor, Ks: torch.Tensor, W: int, H: int, world: int = 1,
                 sh_degree: int = 3, eps2d: float = 0.01, near: float = 0.01, far: float = 1e10, radius_clip: float = 0.0,
                 graph: bool = True, capacity_margin: float = 1.25, overlap_views: bool = False,
                 exchange_kind: str | None = None):
        """``params``: dict of the five parameter tensors on the device; ``viewmats [C,4,4]``, ``Ks [C,3,3]``: the LOCAL
        views (``parallel.views_for_rank``).  ``world`` > 1 needs an initialised process group; ``exchange_kind``: "nccl"
        (library collectives, the default) or "peer" (this library's kernels over NVLink peer memory); ``ADB_EXCHANGE`` sets
        the default (``peer.make_exchange``)."""
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
        self.exchange = make_exchange(N, C, dev, kind=exchange_kind) if world > 1 else None
        self._fused_push = getattr(self.exchange, "fused_mask", False)
        self.grads = {"v_sh": torch.empty(N, 16, 3, dtype=torch.float32, device=dev)}
        if self.exchange is not None:
            self.grads.update(self.exchange.views)          # geometry gradients live in the all-reduce bucket
        else:
            self.grads.update(v_means=torch.empty(N, 3, device=dev), v_quats=torch.empty(N, 4, device=dev),
                              v_scales=torch.empty(N, 3, device=dev), v_opac=torch.empty(N, device=dev))
        self.grads["g_rgb"] = torch.empty(C, N, 3, dtype=torch.float32, device=dev)
        self.capacity = None
        self.margin = capacity_margin
        self.use_graph = graph
        # overlap_views=True runs consecutive views on two CUDA streams (the latency-bound projection / atomics / sort stages of
        # one view could fill the gaps of the other's issue-bound blend kernels; both streams fork from / join the caller's, so
        # the pair is capturable in one graph).  Off by default: co-running issue-bound blend kernels of two views compete for
        # the same issue slots.
        self.overlap_views = overlap_views and self.C > 1
        self._side = torch.cuda.Stream(device=dev) if self.overlap_views else None
        self.graph = None
        self.render = None          # (colors [C,H,W,4], alphas [C,H,W]) of the last step
        self.info = None            # per view: {"n_isect": int64[1], "overflow": int32[1]} device tensors
        self.v_views = self.v_campos = None

    # ---- stages -----------------------------------------------------------------------------------------------------
    def _view(self, c, capacity):
        """projection -> intersection -> blend fwd -> blend bwd -> masked colour gradient of local view c."""
        sh_degree, eps2d, near, far, rclip = self.cfg
        p, W, H, N = self.p, self.W, self.H, self.N
        self.v_splats[c].zero_()
        cnt = R.new_tile_counts(W, H, self.dev)        # per-tile counting is fused into the projection kernel
        R.project(p["means"], p["quats"], p["scales"], p["opacities"], p["sh"], sh_degree, self.V[c], self.K[c], self.P[c],
                  W, H, eps2d, near, far, rclip, out=(self.radii[c], self.splats[c], self.tpg[c]), tile_counts=cnt)
        cap = None if capacity is None else capacity[c]
        keys, vals, offs, info = R.intersect(self.radii[c], self.splats[c], self.tpg[c], W, H, capacity=cap, counts=cnt)
        hits = R.new_hit_mask(vals)                    # the forward's culling decisions, reused by the backward
        col, alp, last = R.blend_forward(W, H, N, self.splats[c], vals, offs, hits=hits)
        R.blend_backward(W, H, N, self.splats[c], vals, offs, alp, last, self.v_colors[c], self.v_alphas[c],
                         out=self.v_splats[c], hits=hits)
        if self.exchange is not None and not self._fused_push:
            R.mask_rgb_grad(self.splats[c], self.v_splats[c], self.grads["g_rgb"][c])
        return col, alp, info, (keys, vals, offs, last)

    def _gather_view(self, c):
        """Hands local view c's colour gradient to the exchange as soon as its blend backward has been issued."""
        campos = self.P if c == 0 else None
        if self._fused_push:
            self.exchange.push_view(c, self.splats[c], self.v_splats[c], campos)       # mask fused with the broadcast
        else:
            self.exchange.start_gather_view(c, self.grads["g_rgb"][c], campos)

    def _local_views(self, capacity):
        """Every local view; no host sync when capacity is given."""
        cols, alps, infos = [None] * self.C, [None] * self.C, [None] * self.C
        cur = torch.cuda.current_stream(self.dev)
        two = self.overlap_views and capacity is not None       # the calibration pass syncs per view: keep it on one stream
        if two:
            self._side.wait_stream(cur)
        for c in range(self.C):
            st = self._side if (two and (c & 1)) else cur
            with torch.cuda.stream(st):
                col, alp, info, tmp = self._view(c, capacity)
                if two and st is not cur:
                    for tns in tmp + (col, alp):
                        tns.record_stream(cur)
            cols[c], alps[c], infos[c] = col, alp, info
        if two:
            cur.wait_stream(self._side)
        return cols, alps, infos

    def _backward(self):
        p = self.p
        out = R.multi_view_backward(p["means"], p["quats"], p["scales"], p["sh"], self.cfg[0], self.V, self.K, self.P, self.W,
                                    self.H, self.radii, self.splats, self.v_splats, out=self.grads, exchange=self.exchange)
        self.v_views, self.v_campos = out[5], out[6]

    def calibrate(self):
        """One eager pass with host syncs: measures the intersection count of every local view and fixes the capacities."""
        with torch.cuda.device(self.dev):
            _, _, infos = self._local_views(None)
            self._backward()
        counts = [int(i) for i in infos]
        self.capacity = [int(n * self.margin) + 4096 for n in counts]
        self.n_isect = counts
        return counts

    def _capture(self):
        dev = self.dev
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):                     # warm-up off the capture stream
            self._local_views(self.capacity)
            if self.exchange is None:
                self._backward()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        if self.exchange is None:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                cols, alps, infos = self._local_views(self.capacity)
                self._backward()
            self.graph, self.render, self.info = [g], (cols, alps), infos
            return
        # multi-GPU: one graph PER VIEW, so that view c's colour gradients can be all-gathered (NCCL, outside the graphs)
        # while view c+1 renders
        graphs, cols, alps, infos = [], [], [], []
        pool = None
        for c in range(self.C):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=pool):
                col, alp, info, _ = self._view(c, self.capacity)
            pool = g.pool()
            graphs.append(g)
            cols.append(col)
            alps.append(alp)
            infos.append(info)
        self.graph, self.render, self.info = graphs, (cols, alps), infos

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
            else:
                cols, alps, infos = [], [], []
                for c in range(self.C):
                    col, alp, info, _ = self._view(c, self.capacity)
                    if self.exchange is not None:
                        self._gather_view(c)
                    cols.append(col)
                    alps.append(alp)
                    infos.append(info)
                self.render, self.info = (cols, alps), infos
                self._backward()
        return self.grads

    def check_overflow(self):
        """Host sync.  Raises if any view's intersection count exceeded its capacity since the last check."""
        if self.info is None:
            return self.n_isect
        counts = [int(i["n_isect"]) for i in self.info]
        if any(int(i["overflow"]) for i in self.info):
            raise _lib.ArtdecoB200Error(f"intersection capacity exceeded: counts {counts}, capacities {self.capacity}; "
                                        "call calibrate() again (the scene grew)")
        self.n_isect = counts
        return counts

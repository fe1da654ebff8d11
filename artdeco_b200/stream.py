"""Synthetic-stream harness for BASELINE config 3 ("PINGPONG stream end-to-end (Frontend+Backend+Mapping), 1 GPU";
SURVEY.md §8d: "100 frames of mast3r_pair + raster_scene growth").  No dataset or checkpoint exists offline, so the stream is
synthetic, but the KERNEL MIX and its contention for one GPU are the reference's (run.sh:15-17 runs Frontend, Backend and the
mapper as processes sharing the device):

  every frame      Frontend: MASt3R asymmetric inference of (frame, last key frame) at batch 1 + dense matching
                   (VSLAM/Frontend.py -> CameraTracker.py:59-61 -> utils_mast3r.py:116-171)
  every k-th frame key frame: the scene grows by M Gaussians (SparseGaussianAdam.add_and_prune, optimizers.py:163-219),
                   distCUDA2 of the new points initialises their scales (h3dgsv3.py uses simple-knn for this)
  every frame      mapper: `mapper_iters` optimiser iterations on the growing scene — render one key-frame view with the
                   LoD cull inside (h3dgsv3.py:617-700), L1 + fused-SSIM loss, backward, SparseGaussianAdam.step
                   (h3dgsv3.py:406-464)

The Frontend runs on its own CUDA stream and the mapper on another, as two processes would interleave on the device.
Reports frames/s and the per-component device time.  This is a harness (measurement + integration check), not a SLAM system:
poses are the synthetic cameras', matches are computed and discarded.
"""
from __future__ import annotations

import time

import torch

from . import synthetic
from .knn import distCUDA2
from .optimizers import SparseGaussianAdam
from .scene import render_lod
from .ssim import fused_ssim


def run(dev, frames: int = 100, keyframe_every: int = 5, grow: int = 20000, mapper_iters: int = 2, W: int = 960, H: int = 544,
        img: int = 512, model=None, seed: int = 0):
    from .mast3r import FULL_CFG, AsymmetricMASt3R, wrappers
    from .mast3r.shapes import random_state_dict
    own_model = model is None
    if own_model:
        sd = random_state_dict(FULL_CFG, dev, seed=0)
        model = AsymmetricMASt3R(precision="bf16x3", **FULL_CFG).load_state_dict(sd).to(dev)
    g = torch.Generator().manual_seed(seed)
    pool = synthetic.raster_scene(grow * (frames // keyframe_every + 2), seed=seed)
    lr = {"xyz": 1e-4, "f_dc": 2.5e-3, "f_rest": 1.25e-4, "opacity": 2.5e-2, "scaling": 5e-3, "rotation": 1e-3}
    z3 = lambda *s: torch.zeros(*s, device=dev)   # noqa: E731
    params = {"xyz": {"val": z3(0, 3), "lr": lr["xyz"]}, "f_dc": {"val": z3(0, 1, 3), "lr": lr["f_dc"]},
              "f_rest": {"val": z3(0, 15, 3), "lr": lr["f_rest"]}, "opacity": {"val": z3(0, 1), "lr": lr["opacity"]},
              "scaling": {"val": z3(0, 3), "lr": lr["scaling"]}, "rotation": {"val": z3(0, 4), "lr": lr["rotation"]},
              "d_max": {"val": z3(0, 1), "lr": 0.0}}
    opt = SparseGaussianAdam(params, betas=(0.5, 0.99), eps=1e-15, lr_dict={}, device=dev)
    s_front, s_map = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
    cfgm = {"matching": dict(max_iter=10, lambda_init=1e-8, convergence_thresh=1e-6, dist_thresh=1e-1, radius=3, dilation_max=5)}
    ev = {k: [] for k in ("frontend", "mapper", "densify")}
    kf_img, n_kf, cursor = None, 0, 0
    gt = torch.rand(3, H, W, generator=g).to(dev)
    V0, K0 = synthetic.camera(W, H, view=3.5)
    tanx, tany = W / (2 * float(K0[0, 0])), H / (2 * float(K0[1, 1]))
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    for f in range(frames):
        frame = type("F", (), {})()
        frame.img = (torch.rand(3, img, img, generator=g) * 2 - 1).to(dev, non_blocking=True)
        if kf_img is None:
            kf_img = frame
        # ---- Frontend stream: MASt3R pair + matching (B = 1 latency path) ----
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(s_front):
            a.record()
            wrappers.mast3r_match_asymmetric(cfgm, model, frame, kf_img)
            b.record()
        ev["frontend"].append((a, b))
        # ---- key frame: grow the scene ----
        if f % keyframe_every == 0:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(s_map):
                a.record()
                sl = slice(cursor, cursor + grow)
                cursor += grow
                new_xyz = pool["means"][sl].to(dev)
                d2 = distCUDA2(new_xyz).clamp_min(1e-7)
                ext = {"xyz": new_xyz, "f_dc": pool["sh"][sl, :1].to(dev), "f_rest": pool["sh"][sl, 1:].to(dev),
                       "opacity": pool["opacities"][sl, None].to(dev), "scaling": torch.sqrt(d2)[:, None].repeat(1, 3).clamp(0.005, 0.05),
                       "rotation": pool["quats"][sl].to(dev), "d_max": pool["d_max"][sl].to(dev)}
                n_old = params["xyz"]["val"].shape[0]
                opt.add_and_prune(ext, torch.ones(n_old, dtype=torch.bool, device=dev))
                b.record()
            ev["densify"].append((a, b))
            kf_img, n_kf = frame, n_kf + 1
        # ---- mapper stream: optimiser iterations on the current scene ----
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(s_map):
            a.record()
            for it in range(mapper_iters):
                V, _ = synthetic.camera(W, H, view=float((f + it) % 8))
                opt.zero_grad()
                P = {k: params[k]["val"] for k in params}
                pkg = render_lod(W, H, V.to(dev), xyz=P["xyz"], opacity=P["opacity"], f_dc=P["f_dc"], f_rest=P["f_rest"],
                                 scaling=P["scaling"], rotation=P["rotation"], d_max=P["d_max"], tanfovx=tanx, tanfovy=tany,
                                 sh_degree=3, eps2d=0.01)
                img_r = pkg["render"]
                loss = 0.8 * (img_r - gt).abs().mean() + 0.2 * (1.0 - fused_ssim(img_r[None], gt[None]))
                loss.backward()
                n_now = P["xyz"].shape[0]
                opt.step(pkg["visibility_filter"], n_now, None, 0)
            b.record()
        ev["mapper"].append((a, b))
    torch.cuda.synchronize(dev)
    wall = time.perf_counter() - t0
    res = {"frames": frames, "fps": frames / wall, "wall_s": wall, "n_gaussians_final": int(params["xyz"]["val"].shape[0]),
           "n_keyframes": n_kf, "image": f"MASt3R {img}x{img}, render {W}x{H}", "mapper_iters_per_frame": mapper_iters,
           "what": "Frontend (MASt3R B=1 pair + dense matching) on one CUDA stream, mapper (LoD cull + rasterize fwd/bwd + "
                   "fused-SSIM + SparseGaussianAdam) and densification (add_and_prune + distCUDA2) on another, one GPU"}
    for k, lst in ev.items():
        if lst:
            ms = [x.elapsed_time(y) for x, y in lst]
            res[f"{k}_ms_mean"] = sum(ms) / len(ms)
            res[f"{k}_calls"] = len(ms)
    if own_model:
        del model
    return res

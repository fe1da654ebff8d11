"""Time one key-frame densification (SceneModel.add_new_gaussians) on CUDA: the oracle's PyTorch restatement
(oracle/densify_ref.py on CUDA tensors, standing in for the reference, with its voxel step on the device kernels so that only
the sampler differs) against artdeco_b200.densify.add_new_gaussians.

    python tests/perf/time_densify.py [--reps 5] [--out /tmp/time_densify.json]

A 1296x972 key frame over a 512x384 point map (PINGPONG at --downsampling 2) on scenes of 100k and 1M Gaussians, with
mlp_cov.  CUDA events around each whole call (both paths end in host reads), after warm-up, the two paths alternated; the
median of --reps.  The split: one render_lod, and the four-LoD sampling alone given a render."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import densify_ref as ref  # noqa: E402
import test_densify as td  # noqa: E402
from artdeco_b200 import densify  # noqa: E402
from artdeco_b200.optimizers import SparseGaussianAdam  # noqa: E402
from artdeco_b200.scene import render_lod  # noqa: E402
from artdeco_b200.voxel import update_voxel  # noqa: E402


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    card = q[0] if q else torch.cuda.get_device_name(0)
    print(f"card: {card}")
    H, W, Hs, Ws = 972, 1296, 384, 512
    f = 0.9 * W
    tanx, tany = W / (2 * f), H / (2 * f)
    fr, _ = td.make_frame(H, W, Hs, Ws, seed=1, dev=dev)
    cov = td.mlp(dev)
    kw = dict(init_proba_scaler=td.SCALER, gs_add_ratio=td.RATIO, voxel_size=0.3, visible_threshold=0.3, local_feat_dim=20,
              global_feat_dim=12)
    cams = fr["approx_centre"][None]
    V = torch.eye(4, device=dev)
    V[:3, :3], V[:3, 3] = fr["R"], fr["t"]
    rows = []
    for N in (100_000, 1_000_000):
        P0 = td.make_scene(N, dev, seed=2)
        scene = lambda P: dict(xyz=P["xyz"], opacity=torch.sigmoid(P["opacity"]), f_dc=P["f_dc"], f_rest=P["f_rest"],  # noqa
                               scaling=torch.exp(P["scaling"]), rotation=P["rotation"], d_max=P["d_max"])

        def render_of(P):
            return lambda cls: render_lod(W, H, V, tanfovx=tanx, tanfovy=tany, cov_mlp=cov, local_feat=P["local_feat"],
                                          global_feat=P["global_feat"], cls_id=cls, **scene(P))["render"].contiguous()

        def dev_voxel(new_xyz, xyz, cls_id, vs, lod):
            return update_voxel(new_xyz, xyz, cls_id, vs)

        stats = {}

        def ours():
            params = {k: {"val": v.clone(), "lr": 1e-3} if k not in ("id", "cls_id", "d_max") else {"val": v.clone()}
                      for k, v in P0.items()}
            opt = SparseGaussianAdam(params, (0.5, 0.99), device=dev)
            stats.update(densify.add_new_gaussians(opt, fr, keyframe_id=1, cam_centres=cams, width=W, height=H, f=f,
                                                   tanfovx=tanx, tanfovy=tany, cov_mlp=cov, **kw))

        def torch_path():
            P = {k: v.clone() for k, v in P0.items()}
            ref.add_new_gaussians(P, fr, render_of(P), keyframe_id=1, cam_centres=cams, width=W, height=H, f=f,
                                  update_voxel=dev_voxel, **kw)

        raw = render_of(P0)(P0["cls_id"])
        us = [torch.rand(H // lod, W // lod, device=dev) for lod in ref.LODS]
        samp = dict(lod=1, f=f, init_proba_scaler=td.SCALER, gs_add_ratio=td.RATIO)

        def ours_sampling():
            q_ = densify.depth_quantile(fr["point_map"])
            for lod, u in zip(ref.LODS, us):
                densify.sample_lod(fr["image"], raw, fr["point_map"], fr["conf"], fr["R"], fr["t"], fr["approx_centre"],
                                   fr["exposure"], **dict(samp, lod=lod), uniforms=u, qmin=q_)

        def torch_sampling():
            for lod, u in zip(ref.LODS, us):
                ref.sample_lod(fr["image"], raw, fr["point_map"], fr["conf"], fr["R"], fr["t"], fr["approx_centre"],
                               fr["exposure"], **dict(samp, lod=lod), uniforms=u, qmin=ref.depth_threshold(fr["point_map"]))

        def one_render():
            render_of(P0)(P0["cls_id"])

        fns = dict(ours=ours, torch=torch_path, ours_sampling=ours_sampling, torch_sampling=torch_sampling, render=one_render)
        for _ in range(2):
            for fn in fns.values():
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in fns}
        for _ in range(a.reps):
            for k, fn in fns.items():
                times[k].append(timed(fn))
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        row = dict(N=N, size=f"{W}x{H}", point_map=f"{Ws}x{Hs}", renders_ours=stats["renders"], renders_torch=4,
                   rows=stats["rows"], ours_ms=round(med["ours"], 2), torch_ms=round(med["torch"], 2),
                   speedup=round(med["torch"] / med["ours"], 2), render_ms=round(med["render"], 2),
                   sampling_ours_ms=round(med["ours_sampling"], 3), sampling_torch_ms=round(med["torch_sampling"], 3))
        rows.append(row)
        print(json.dumps(row))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(dict(card=card, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()

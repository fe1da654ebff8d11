"""Time the mapper's pixel loss (SceneModel.optimization_step's loss block) on CUDA: the oracle's PyTorch glue
(oracle/mapper_loss_ref.py on CUDA tensors with this package's fused_ssim, standing in for the reference: radial table built
on the CPU and uploaded every step, eager composite, exposure, mask and sums, autograd backward) against
artdeco_b200.mapper.mapper_loss, forward + backward.

    python tests/perf/time_mapper_loss.py [--reps 7] [--out /tmp/time_mapper_loss.json]

Sizes 648x486, 1296x972 and 1920x1080, both is_important values.  CUDA events around loss + backward, after warm-up, the
two paths alternated; the median of --reps.  Then one whole training step per path, render_lod (1M Gaussians, 648x486,
bg=None for ours, the composite inside the glue for the oracle's) + loss + backward, so the loss's share of a step is known."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import mapper_loss_ref as ref  # noqa: E402
from artdeco_b200 import synthetic  # noqa: E402
from artdeco_b200.mapper import mapper_loss  # noqa: E402
from artdeco_b200.scene import render_lod  # noqa: E402
from artdeco_b200.ssim import fused_ssim  # noqa: E402

KW = dict(lambda_dssim=0.2, depth_weight=0.6, rad_decay=1.0)


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def bench(fns, reps):
    for _ in range(3):
        for fn in fns.values():
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            times[k].append(timed(fn))
    return {k: sorted(v)[len(v) // 2] for k, v in times.items()}


def torch_loss(colors, alphas, gt, mono, E, bg, important):
    return ref.mapper_loss(colors, alphas, gt, mono, E, bg, is_important=important, ssim_fn=fused_ssim, **KW)["loss"]


def ours_loss(colors, alphas, gt, mono, E, bg, important):
    return mapper_loss(colors, alphas, gt, mono, E, bg, is_important=important, **KW)[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    card = q[0] if q else torch.cuda.get_device_name(0)
    print(f"card: {card}")
    rows = []
    for W, H in ((648, 486), (1296, 972), (1920, 1080)):
        inp = {k: v.to(dev) for k, v in ref.make_inputs(H, W, seed=1, zero_depth=False).items()}
        colors = inp["colors"].requires_grad_(True)
        alphas = inp["alphas"].requires_grad_(True)
        E = inp["exposure"].requires_grad_(True)
        for important in (True, False):
            def step(loss_fn):
                def run():
                    colors.grad = alphas.grad = E.grad = None
                    loss_fn(colors, alphas, inp["gt"], inp["mono"], E, inp["bg"], important).backward()
                return run
            med = bench(dict(ours=step(ours_loss), torch=step(torch_loss)), a.reps)
            row = dict(size=f"{W}x{H}", is_important=important, ours_ms=round(med["ours"], 4),
                       torch_ms=round(med["torch"], 4), speedup=round(med["torch"] / med["ours"], 2))
            rows.append(row)
            print(json.dumps(row))

    # one whole step: render + loss + backward at 1M Gaussians
    W, H = 648, 486
    sc = synthetic.raster_scene(1_000_000, seed=3, z_range=(2.0, 8.0), extent=(2.5, 2.0))
    P = dict(xyz=sc["means"], opacity=torch.logit(sc["opacities"][:, None]), f_dc=sc["sh"][:, :1].clone(),
             f_rest=sc["sh"][:, 1:].clone(), scaling=torch.log(sc["scales"]), rotation=sc["quats"])
    P = {k: v.to(dev).requires_grad_(True) for k, v in P.items()}
    d_max = sc["d_max"].to(dev)
    V = torch.eye(4, device=dev)
    f = 0.8 * W
    g = torch.Generator().manual_seed(4)
    gt = (0.2 + 0.6 * torch.rand(3, H, W, generator=g)).to(dev)
    mono = (0.1 + 0.4 * torch.rand(1, H, W, generator=g)).to(dev)
    bg = torch.rand(3, generator=g).to(dev)
    E = torch.eye(3, 4, device=dev).requires_grad_(True)

    def whole(loss_fn, important):
        def run():
            for t in list(P.values()) + [E]:
                t.grad = None
            pkg = render_lod(W, H, V, xyz=P["xyz"], opacity=torch.sigmoid(P["opacity"]), f_dc=P["f_dc"], f_rest=P["f_rest"],
                             scaling=torch.exp(P["scaling"]), rotation=P["rotation"], d_max=d_max, tanfovx=W / (2 * f),
                             tanfovy=H / (2 * f), bg=None)
            loss_fn(pkg["colors"], pkg["alphas"], gt, mono, E, bg, important).backward()
        return run

    def render_only():
        with torch.no_grad():
            render_lod(W, H, V, xyz=P["xyz"], opacity=torch.sigmoid(P["opacity"]), f_dc=P["f_dc"], f_rest=P["f_rest"],
                       scaling=torch.exp(P["scaling"]), rotation=P["rotation"], d_max=d_max, tanfovx=W / (2 * f),
                       tanfovy=H / (2 * f), bg=None)

    for important in (True, False):
        med = bench(dict(ours=whole(ours_loss, important), torch=whole(torch_loss, important), render_fwd=render_only), a.reps)
        row = dict(whole_step=f"{W}x{H}", gaussians=1_000_000, is_important=important, ours_ms=round(med["ours"], 3),
                   torch_ms=round(med["torch"], 3), saved_ms=round(med["torch"] - med["ours"], 3),
                   render_fwd_ms=round(med["render_fwd"], 3))
        rows.append(row)
        print(json.dumps(row))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(dict(card=card, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()

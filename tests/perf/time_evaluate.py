"""Times one held-out evaluation over T test frames at 1296x972 (the mapper's level-0 resolution) with CUDA events.

Both arms start from the same stacked rasterizer outputs (the rasterizer is shared and not timed) and end with the metrics on
the host:
  ours         artdeco_b200.evaluate: harmonisation, metrics_from_renders with LPIPS-VGG, one host read;
  oracle tf32  oracle/evaluate_ref.py's loop in fp32 on the device with cuDNN TF32 on (the reference's default);
  oracle fp32  the same with TF32 off.
Arms are alternated and medians reported.  The LPIPS pass alone is reported as achieved TFLOP/s against the algorithmic
FLOPs of VGG16 to relu5_3 (2 images per frame, 2 * H * W * 9 * Cin * Cout per conv).

    python tests/perf/time_evaluate.py [--frames 4] [--reps 5]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from artdeco_b200 import evaluate  # noqa: E402
from artdeco_b200.lpips import LPIPSVGG  # noqa: E402
from oracle import evaluate_ref as ref  # noqa: E402

CONVS = ((3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 512), (512, 512),
         (512, 512), (512, 512), (512, 512), (512, 512))
LEVEL_OF = (0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4)


def vgg_flops(h, w):
    f = 0
    for (ci, co), l in zip(CONVS, LEVEL_OF):
        hh, ww = h >> l, w >> l
        f += 2 * hh * ww * 9 * ci * co
    return 2 * f   # two images per frame


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--h", type=int, default=972)
    ap.add_argument("--w", type=int, default=1296)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    T, h, w = args.frames, args.h, args.w
    g = torch.Generator().manual_seed(0)
    rgb = torch.rand(T, h, w, 3, generator=g)
    colors = torch.cat([rgb, torch.rand(T, h, w, 1, generator=g) + 0.5], -1).contiguous().to(dev)
    alphas = torch.rand(T, h, w, generator=g).to(dev)
    gt = (rgb.permute(0, 3, 1, 2) + 0.05 * torch.randn(T, 3, h, w, generator=g)).clamp(0, 1).contiguous().to(dev)
    K = 2 * T
    is_test = [i % 2 == 1 for i in range(K)]
    E0 = (torch.eye(3, 4) + 0.03 * torch.randn(K, 3, 4, generator=g)).contiguous().to(dev)
    sd = ref.random_state_dict(0)
    ours_lp = LPIPSVGG(sd, device=dev)
    oracle_lp = ref.LPIPSRef().to(dev).eval()
    oracle_lp.load_state_dict(sd)
    views = [i for i in range(K) if is_test[i]]
    vf = torch.tensor(views, dtype=torch.int32, device=dev)
    flags = torch.tensor(is_test, device=dev)

    def ours():
        E = E0.clone()
        n_bad = evaluate.harmonize_test_exposure(E, flags)
        table = evaluate.metrics_from_renders(colors, alphas, gt, E, vf, n_gaussians=0, lpips=ours_lp)
        host = torch.cat([n_bad.double(), table.reshape(-1)]).cpu()
        return evaluate.summarise(host[1:].reshape(T, -1), True, True)

    def oracle(tf32):
        def run():
            prev = torch.backends.cudnn.allow_tf32
            torch.backends.cudnn.allow_tf32 = tf32
            try:
                ex = [E0[i].clone() for i in range(K)]
                renders = {i: (colors[t:t + 1], alphas[t:t + 1, ..., None]) for t, i in enumerate(views)}
                gts = {i: gt[t] for t, i in enumerate(views)}
                vis = {i: torch.zeros(0, dtype=torch.bool, device=dev) for i in views}
                with torch.no_grad():
                    return ref.evaluate(ex, is_test, renders, gts, vis, lpips=oracle_lp, with_LPIPS=True, all=True)
            finally:
                torch.backends.cudnn.allow_tf32 = prev
        return run

    ews = evaluate.eval_workspace(T, h, w, 0, dev)
    image = gt.clone()

    def lpips_only():
        ours_lp.run(T, h, w, 0, image, gt, ews)

    arms = {"ours": ours, "oracle_tf32": oracle(True), "oracle_fp32": oracle(False), "lpips_pass": lpips_only}
    for fn in arms.values():   # warm-up (module loads, cuDNN autotuning, allocator)
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(args.reps):
        for k, fn in arms.items():
            times[k].append(timed(fn))
    med = {k: statistics.median(v) for k, v in times.items()}
    m_ours, m_ref = ours(), oracle(False)()
    flops = vgg_flops(h, w) * T
    out = {"gpu": torch.cuda.get_device_name(0), "frames": T, "h": h, "w": w, "median_ms": med,
           "lpips_pass_tflops": flops / (med["lpips_pass"] * 1e-3) / 1e12, "vgg_tflop_per_frame": vgg_flops(h, w) / 1e12,
           "speedup_vs_tf32": med["oracle_tf32"] / med["ours"], "speedup_vs_fp32": med["oracle_fp32"] / med["ours"],
           "ours": m_ours, "oracle_fp32_metrics": m_ref}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

"""Step time and per-stage breakdown of the bench's 8-view optimiser step (artdeco_b200.multiview.MultiViewStep at 1M
Gaussians, 1920x1080, views 0..7, the bench's seeds).  Uses only the engine's public API, so the same script times any
revision of the engine.

Prints one JSON line: the graphed step time (CUDA events over --steps steps after --warmup), then, from one eager step under
_lib.StageTimer, the device time per stage per step and the launches per step; the card's name and power limit are read in
the same process.  The blend stages also get their algorithmic bytes (per view 44 I + 24 P forward, 44 I + 44 P backward,
I = intersections, P = pixels) and the rate they imply."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from artdeco_b200 import _lib, synthetic  # noqa: E402
from artdeco_b200.multiview import MultiViewStep  # noqa: E402

N, W, H, VIEWS = 1_000_000, 1920, 1080, 8


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:  # noqa: BLE001
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--label", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_multiview.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    sc = synthetic.raster_scene(N, seed=0)
    t = {k: sc[k].to(dev) for k in ("means", "quats", "scales", "opacities", "sh")}
    cams = [synthetic.camera(W, H, view=float(v)) for v in range(VIEWS)]
    eng = MultiViewStep(t, torch.stack([c[0] for c in cams]).to(dev), torch.stack([c[1] for c in cams]).to(dev), W, H)
    for j in range(VIEWS):
        vc, va = synthetic.upstream_grads(W, H, seed=1 + j)
        eng.v_colors[j].copy_(vc[0])
        eng.v_alphas[j].copy_(va[0, ..., 0])
    n_isect = eng.calibrate()

    for _ in range(max(args.warmup, 1)):
        eng.step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.steps):
        eng.step()
    b.record()
    torch.cuda.synchronize()
    ms_step = a.elapsed_time(b) / args.steps
    eng.check_overflow()

    eng.use_graph = False
    eng.step()                                  # eager warm-up of the timed pass
    torch.cuda.synchronize()
    _lib.TIMER = _lib.StageTimer()
    eng.step()
    torch.cuda.synchronize()
    stages = {k.replace("adb_raster_", ""): round(ms, 4) for k, (ms, _) in sorted(_lib.TIMER.totals_ms().items())}
    launches = _lib.TIMER.launches
    _lib.TIMER = None
    eng.use_graph = True

    P = W * H
    I_total = float(sum(n_isect))
    blend_bytes = {"blend_fwd": 44 * I_total + VIEWS * 24 * P, "blend_bwd": 44 * I_total + VIEWS * 44 * P}
    blend = {}
    for name, nbytes in blend_bytes.items():
        ms = sum(v for k, v in stages.items() if k.startswith(name))
        blend[name] = {"ms_per_step": ms, "bytes_per_step": nbytes, "GBps": nbytes / (ms * 1e-3) / 1e9 if ms else None}
    print(json.dumps({"label": args.label, "ms_per_step": ms_step, "steps": args.steps, "stage_ms_per_step": stages,
                      "stage_ms_sum": round(sum(stages.values()), 4), "launches_per_step": launches,
                      "n_isect": n_isect, "blend": blend, "device": torch.cuda.get_device_name(dev),
                      "power_limit_w": power_limit_w()}), flush=True)


if __name__ == "__main__":
    main()

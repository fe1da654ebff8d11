"""Time one Pi3 forward of the loop-closure window (24 frames at 392x518) on CUDA: artdeco_b200.pi3.Pi3 in bf16x3 and
in bf16, and oracle/pi3_torch.py under bf16 autocast with SDPA attention, the way the reference runs it
(retrieval_database.py:271-273).  Deterministic weights (synthetic.det_weights); timing does not depend on their values.

    python tests/perf/time_pi3.py [--frames 24] [--reps 5] [--out /tmp/time_pi3.json]

CUDA events around each forward after one warm-up forward per path, the paths alternated; the median of --reps.
Achieved TFLOP/s is artdeco_b200.pi3.model.flops (dense layers and attention, counted from the shapes) over that time.
The activation peak is torch.cuda.max_memory_allocated during a forward minus the memory held before it."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from artdeco_b200 import synthetic  # noqa: E402
from artdeco_b200.pi3 import Pi3, param_shapes  # noqa: E402
from artdeco_b200.pi3.model import flops  # noqa: E402
from oracle import pi3_torch as pt  # noqa: E402


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_pi3 needs a CUDA device")
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    sd = synthetic.det_weights(param_shapes())
    imgs = synthetic.pi3_frames(a.frames, 392, 518, seed=0).to(dev)
    x3 = Pi3("bf16x3").load_state_dict(sd).to(dev)
    b1 = Pi3("bf16").load_state_dict(sd).to(dev)
    weights_gib = {k: torch.cuda.memory_allocated() / 2 ** 30 for k in ("after_load",)}
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    del sd

    def ref():
        with torch.inference_mode(), torch.autocast("cuda", dtype=torch.bfloat16):
            pt.forward(sd_dev, imgs)

    fns = {"artdeco_bf16x3": lambda: x3(imgs), "artdeco_bf16": lambda: b1(imgs), "reference_torch_bf16_autocast": ref}
    peaks = {k: peak(fn) for k, fn in fns.items()}
    times = {k: [] for k in fns}
    for _ in range(a.reps):
        for k, fn in fns.items():
            times[k].append(timed(fn))
    f = flops(a.frames)
    res = dict(gpu=gpu, frames=a.frames, H=392, W=518, flop=f, reps=a.reps, weights_and_inputs_gib=weights_gib,
               activation_peak_gib=peaks,
               ms={k: sorted(v)[len(v) // 2] for k, v in times.items()}, ms_all=times)
    res["tflops"] = {k: f / (v * 1e-3) / 1e12 for k, v in res["ms"].items()}
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()

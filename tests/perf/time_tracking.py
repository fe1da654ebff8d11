"""Time one tracked frame (CameraTracker.track steps 2-7) on CUDA: the oracle's PyTorch restatement (oracle/track_ref.py on
CUDA tensors, standing in for the reference; pypose's own overhead is not included) against artdeco_b200.tracking.track.

  python tests/perf/time_tracking.py [--reps 10] [--out /tmp/time_tracking.json]

Sizes 512x384 and 512x512, covariance filter on and off, convergence disabled at 10 and 50 iterations, plus one converging
scene.  CUDA events around each whole frame (both paths end in a host read), after warm-up, the two paths alternated."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import track_ref as ref  # noqa: E402
import test_tracking as tt  # noqa: E402
from artdeco_b200 import tracking  # noqa: E402

# launches per Gauss-Newton iteration of adb_track_solve (csrc/track.cu)
LAUNCHES_PER_ITER = {True: 6, False: 2}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    card = q[0] if q else torch.cuda.get_device_name(0)
    print(f"card: {card}")
    rows = []
    cases = [(H, W, filt, iters, False) for (H, W) in ((384, 512), (512, 512)) for filt in (True, False) for iters in (10, 50)]
    cases += [(384, 512, True, 50, True)]
    for (H, W, filt, iters, conv) in cases:
        sc = tt.scene(H, W, seed=7, perturb=0.03)
        cfg = dict(tt.CFG if conv else tt.NO_CONV, max_iters=iters)
        d = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in sc.items()}
        ws = tracking.workspace(H * W, dev)

        def run_kernels():
            kf_X, kf_C = d["kf_X"].clone(), d["kf_C"].clone()
            kf_N = torch.tensor([2], dtype=torch.int32, device=dev)
            return tracking.track(d["idx_f2k"], d["valid_match_k"], d["Xff"], d["Cff"], d["Qff"], d["Xkf"], d["Ckf"],
                                  d["Qkf"], kf_X, kf_C, kf_N, d["T_WCf"], d["T_WCk"], d["K"], (H, W), cfg, 0.0, 0.5, 0.0,
                                  filt, True, ws=ws)

        def run_torch():
            out = ref.track(d["idx_f2k"], d["valid_match_k"], d["Xff"], d["Cff"], d["Qff"], d["Xkf"], d["Ckf"], d["Qkf"],
                            d["kf_X"].clone(), d["kf_C"].clone(), 2, d["T_WCf"], d["T_WCk"], d["K"], H, W, cfg, 0.0, 0.5,
                            0.0, filt, True)
            return out["T_WCf"].cpu()

        for _ in range(2):
            run_kernels()
            run_torch()
        torch.cuda.synchronize()
        tk, tt_ = [], []
        for _ in range(a.reps):
            for fn, acc in ((run_kernels, tk), (run_torch, tt_)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                acc.append(e0.elapsed_time(e1))
        st = tracking.TrackState.read(ws.state)
        med = lambda v: sorted(v)[len(v) // 2]   # noqa: E731
        row = dict(size=f"{W}x{H}", filter=filt, max_iters=iters, converging=conv, iters_run=st.iters,
                   torch_ms=round(med(tt_), 3), kernels_ms=round(med(tk), 3), speedup=round(med(tt_) / med(tk), 1),
                   launches_per_iter=LAUNCHES_PER_ITER[filt])
        rows.append(row)
        print(json.dumps(row))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(card=card, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()

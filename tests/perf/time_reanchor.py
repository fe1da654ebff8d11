"""Time the map update of a SLAM key frame on CUDA: the oracle's PyTorch code (oracle/reanchor_ref.py on CUDA tensors, standing
in for the reference: a Python loop over the mapper key frames with three torch.linalg.inv per frame, then update_gaussians on
gathered [N,4,4] tables with N 4x4 inverses and the four-branch quaternion conversion) against artdeco_b200.reanchor's
keyframe_poses + rigid_transform_gs.

    python tests/perf/time_reanchor.py [--reps 5] [--out /tmp/time_reanchor.json]

K in {50, 300} mapper key frames, N in {100k, 1M, 10M} Gaussians.  CUDA events around each whole call (poses + Gaussians),
after warm-up, the two paths alternated; the median of --reps.  Peak memory is torch.cuda.max_memory_allocated above what
was allocated before one call.  The per-Gaussian pass alone (ours: rigid_transform_gs with its two launches) is timed from
CUDA-graph replays of 20 back-to-back calls and reported as bytes/s against the 64 B per Gaussian it needs (36 B read,
28 B written)."""
import argparse
import json
import os
import subprocess
import sys

import torch

REPLAYS = 20
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import reanchor_ref as ref  # noqa: E402
from artdeco_b200 import reanchor  # noqa: E402
from test_reanchor import random_c2ws, random_gaussians, random_pose_inputs  # noqa: E402


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def bench(fns, reps, warmup=2):
    for _ in range(warmup):
        for fn in fns.values():
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            times[k].append(timed(fn))
    return {k: sorted(v)[len(v) // 2] for k, v in times.items()}


def peak_bytes(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    card = q[0] if q else torch.cuda.get_device_name(0)
    print(f"card: {card}")
    rows = []
    for K in (50, 300):
        inp = random_pose_inputs(K, max(K // 3, 1), seed=K, dev=dev)
        last_h, slam_h = inp["last_keyframe_index"].cpu(), inp["is_slam_keyframe"].cpu()   # Python-side frame fields
        old0, new0 = random_c2ws(K, seed=K, dev=dev)
        for N in (100_000, 1_000_000, 10_000_000):
            ids, xyz, rot = random_gaussians(N, K, seed=N, dev=dev)
            cams0 = torch.zeros(K, 3, device=dev)
            P = {"id": {"val": ids}, "xyz": {"val": xyz.clone()}, "rotation": {"val": rot.clone()}}
            T = {"xyz": xyz.clone(), "rotation": rot.clone()}

            def ours():
                old, new, cams, _, _ = reanchor.keyframe_poses(inp["rW2C"], inp["tW2C"], inp["slam_T_WC"],
                                                               inp["last_keyframe_index"], inp["is_slam_keyframe"],
                                                               inp["T_CkCf"])
                reanchor.rigid_transform_gs(P, old, new, cams)

            def torch_path():
                w = ref.keyframe_poses(inp["rW2C"], inp["tW2C"], inp["slam_T_WC"], last_h, slam_h, inp["T_CkCf"])
                T["xyz"], T["rotation"], _ = ref.rigid_transform_gs(ids, T["xyz"], T["rotation"], w["old_c2ws"],
                                                                    w["new_c2ws"])

            # the per-Gaussian pass alone, as device time: REPLAYS captured launches back to back, so the host's
            # per-call Python overhead (larger than the kernels below 1M Gaussians) is not in the window
            G = {"id": {"val": ids}, "xyz": {"val": xyz.clone()}, "rotation": {"val": rot.clone()}}
            reanchor.rigid_transform_gs(G, old0, new0, cams0)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(REPLAYS):
                    reanchor.rigid_transform_gs(G, old0, new0, cams0)

            med = bench(dict(ours=ours, torch=torch_path, ours_gaussians=graph.replay), a.reps)
            med["ours_gaussians"] /= REPLAYS
            mem = dict(ours=peak_bytes(ours), torch=peak_bytes(torch_path))
            row = dict(K=K, N=N, ours_ms=round(med["ours"], 3), torch_ms=round(med["torch"], 3),
                       speedup=round(med["torch"] / med["ours"], 1), ours_gaussian_pass_ms=round(med["ours_gaussians"], 4),
                       gaussian_pass_GBps=round(64 * N / (med["ours_gaussians"] * 1e-3) / 1e9, 1),
                       ours_peak_MB=round(mem["ours"] / 2**20, 1), torch_peak_MB=round(mem["torch"] / 2**20, 1))
            rows.append(row)
            print(json.dumps(row), flush=True)
            del P, T, G, graph
            torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(dict(card=card, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()

"""Time one Backend key frame's factor-graph work on CUDA: gating 4 candidate edges, then ``solve_GN_calib`` with 10
iterations, in artdeco_b200.factor_graph against the oracle's restatement of the reference's glue
(oracle/factor_graph_ref.py on CUDA tensors, with add_factors' copies of the 2B candidate key frames).  Both paths run the
same Gauss-Newton kernel (artdeco_b200.gn), so only the glue differs.

    python tests/perf/time_factor_graph.py [--reps 7] [--warmup 2] [--K 32 128 300] [--out /tmp/time_factor_graph.json]

512x384 key frames, about 3 edges per key frame (the consecutive edge and up to two retrieval edges), the key-frame store
on the host (as ``--device_shared cpu`` runs the reference) and on the device.  Before each timed call one key frame is
fused (its N_updates changes), as the Backend's last key frame is.  CUDA events around each call, the two paths
alternated, the median of --reps after --warmup.  Peak memory is the rise of torch's peak allocation over the
allocation before the call; host-to-device bytes per solve are computed from shapes: the reference copies every key frame
of the graph (image, X and C: 28 B per pixel), this path the refreshed key frames' X and C (16 B per pixel) and the poses."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import factor_graph_ref as ref  # noqa: E402
from oracle import track_ref  # noqa: E402
from artdeco_b200 import factor_graph, gn  # noqa: E402

H, W = 384, 512
CFG = {"local_opt": dict(pin=1, window_size=1000000, C_conf=0.0, Q_conf=1.5, min_match_frac=0.1, pixel_border=-10,
                         depth_eps=1e-6, max_iters=10, sigma_ray=0.003, sigma_dist=10.0, sigma_pixel=1.0, sigma_depth=10.0,
                         delta_norm=1e-8)}
KMAT = torch.tensor([[400.0, 0.0, 255.5], [0.0, 400.0, 191.5], [0.0, 0.0, 1.0]])


class GnKernel:
    """The reference's mast3r_slam_backends interface over artdeco_b200.gn: the same kernel as the product path."""
    gauss_newton_rays = staticmethod(gn.gauss_newton_rays)
    gauss_newton_calib = staticmethod(gn.gauss_newton_calib)


def make_frames(K, device):
    g = torch.Generator().manual_seed(0)
    n = H * W
    Wp = torch.randn(n, 3, generator=g) + torch.tensor([0.0, 0.0, 5.0])
    f = ref.Keyframes(H, W, buffer=K + 1, device="cpu")
    for k in range(K):
        q = torch.randn(4, generator=g) * 0.02 + torch.tensor([0.0, 0.0, 0.0, 1.0])
        T = torch.cat([0.05 * k * torch.ones(3), q / q.norm(), torch.tensor([1.0])])
        X = track_ref.act(track_ref.inv(T), Wp)
        f.append(k, T, X, 1.0 + torch.rand(n, 1, generator=g), N=1, N_updates=1)
    return f.to(device) if device != "cpu" else f


def candidates(k):
    """The consecutive edge and up to two retrieval edges of key frame k."""
    return sorted({k - 1} | ({k // 2, k - 4} - {k - 1}) & set(range(k)))


def matches(B, dev):
    n = H * W
    ar = torch.arange(n, device=dev).repeat(B, 1)
    ones = torch.ones(B, n, 1, dtype=torch.bool, device=dev)
    return [ar, ar.clone(), ones, ones.clone()] + [torch.full((B, n, 1), 2.0, device=dev) for _ in range(4)]


def timed(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), torch.cuda.max_memory_allocated() - base


def run(K, store, dev, reps, warmup):
    frames = make_frames(K, dev if store == "cuda" else "cpu")
    ours = factor_graph.FactorGraph(CFG, None, frames, K=KMAT, device=dev)
    orac = ref.FactorGraphRef(CFG, frames, K=KMAT.to(dev), device=dev, backend=GnKernel)
    m4 = matches(4, dev)
    for k in range(1, K):
        c = candidates(k)
        m = [t[:len(c)] for t in m4]
        ours.add_matches(c, [k] * len(c), 0.1, *m)
        orac.add_matches(c, [k] * len(c), 0.1, *m)
    ours.solve_GN_calib()                      # builds the mirror once, as a running Backend has
    last = K - 1
    cand = sorted({last - 1, last - 2, last - 3, last // 2})[:4]
    while len(cand) < 4:
        cand.append(cand[-1])
    jj = [last] * 4
    g = torch.Generator().manual_seed(1)
    fuse_X = frames.X[last].clone()
    fuse_C = (1.0 + torch.rand(H * W, 1, generator=g)).to(frames.C.device)

    def ours_step():
        ours.add_matches(cand, jj, 0.1, *m4)
        ours.solve_GN_calib()

    def oracle_step():
        [frames[i].to(dev) for i in cand + jj]            # add_factors' copies of the candidate key frames
        orac.add_matches(cand, jj, 0.1, *m4)
        orac.solve_GN_calib()

    t_o, t_r, mem_o, mem_r = [], [], [], []
    for rep in range(warmup + reps):
        frames.update_pointmap(last, fuse_X, fuse_C)
        a, ma = timed(ours_step)
        frames.update_pointmap(last, fuse_X, fuse_C)
        b, mb = timed(oracle_step)
        if rep >= warmup:
            t_o.append(a)
            t_r.append(b)
            mem_o.append(ma)
            mem_r.append(mb)
    U = K
    n = H * W
    h2d_ref = U * n * 28 if store == "cpu" else 0
    h2d_ours = (1 * n * 16 + U * 32) if store == "cpu" else 0
    return dict(K=K, store=store, edges=ours.E, ours_ms=statistics.median(t_o), ref_glue_ms=statistics.median(t_r),
                speedup=statistics.median(t_r) / statistics.median(t_o), ours_peak_bytes=max(mem_o),
                ref_peak_bytes=max(mem_r), ours_h2d_bytes_per_solve=h2d_ours, ref_h2d_bytes_per_solve=h2d_ref)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--K", type=int, nargs="+", default=[32, 128, 300])
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_factor_graph.py needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    card = q[0] if q else torch.cuda.get_device_name(0)
    print(f"card: {card}")
    rows = []
    for K in a.K:
        for store in ("cpu", "cuda"):
            r = run(K, store, dev, a.reps, a.warmup)
            rows.append(r)
            print(f"K={K:4d} store={store:4s} E={r['edges']:4d}  ours {r['ours_ms']:8.2f} ms  reference glue "
                  f"{r['ref_glue_ms']:8.2f} ms  x{r['speedup']:.1f}  peak {r['ours_peak_bytes'] / 2**20:8.1f} / "
                  f"{r['ref_peak_bytes'] / 2**20:8.1f} MiB  H2D/solve {r['ours_h2d_bytes_per_solve'] / 2**20:7.2f} / "
                  f"{r['ref_h2d_bytes_per_solve'] / 2**20:8.1f} MiB", flush=True)
            torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(dict(card=card, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()

"""Time RetrievalDatabase.update on CUDA at ARTDECO's size: n = 768 encoder tokens (512x384), K = 65536 centroids,
nfeat = 300, database sizes 0 / 100 / 1000 / 5000, with the reference-style path in the same run (torch fp32 distance
matrix + torch.topk on the device, then the oracle's numpy ASMK aggregation and inverted-file search on the host).

    python tests/perf/time_retrieval.py [--reps 20] [--sizes 0,100,1000,5000] [--out /tmp/time_retrieval.json]

Per-stage times are CUDA events around each stage's launches (median of --reps); the whole-update time is a host clock
around update(), which ends in its one device-to-host read.  The database is filled by appending 16 synthetic key frames
and repeating their inverted-file rows up to the size (search cost depends on the rows' word counts, not their origin).
Assignment FLOP/s and bytes/s are computed from shapes: 2 * 300 * K * 1024 * 3 (bf16x3) and the bf16 (hi, lo)
centroids read once."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from artdeco_b200 import retrieval as R  # noqa: E402
from artdeco_b200 import synthetic  # noqa: E402
from oracle import retrieval_ref as rr  # noqa: E402


def ev_time(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--sizes", default="0,100,1000,5000")
    ap.add_argument("--K", type=int, default=65536)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_retrieval.py needs a CUDA device")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    K, n, nfeat = args.K, 768, 300
    m, P, cent = synthetic.retrieval_model(K, seed=0)
    frames = synthetic.retrieval_stream(m, P, cent, [(p, True) for p in range(16)] + [(3, True)], n=n, nfeat=nfeat)
    feats = [f["feat"].to(dev) for f in frames]
    db = R.RetrievalDatabase(m, P, cent, nfeat=nfeat, capacity=8192)
    for f in feats[:16]:
        db.update(f, True, 3, 5e-3)
    torch.cuda.synchronize()
    s = db._dev
    q = feats[16]
    cent_dev = cent.to(dev)
    flop = 2.0 * nfeat * K * 1024 * 3
    byts = K * 1024 * 2 * 2.0
    res = dict(device=smi, K=K, n=n, nfeat=nfeat, sizes={})
    desc = db.prep_features(q)
    stages = {
        "prep_features": lambda: db.prep_features(q),
        "quantize_custom(MA=5)": lambda: db.quantize_custom(desc[0], db.params["query_ivf"]),
    }
    codes = db.quantize_custom(desc[0], db.params["query_ivf"])
    stages["aggregate"] = lambda: db._aggregate(desc[0], codes, 5, s["qw"].data_ptr(), s["qsig"].data_ptr(),
                                                s["qcount"].data_ptr())
    for name, fn in stages.items():
        fn()
        res[name + "_ms"] = ev_time(fn, args.reps)
    t = res["quantize_custom(MA=5)_ms"] * 1e-3
    res["assign_tflops"] = flop / t / 1e12
    res["assign_centroid_GBps"] = byts / t / 1e9
    for size in map(int, args.sizes.split(",")):
        rows = db.kf_counter
        if size > 0:
            for k in ("ivf_words", "ivf_sig", "ivf_count"):
                src = s[k][:16].clone()
                reps = (size + 15) // 16
                s[k][:size] = src.repeat((reps,) + (1,) * (src.dim() - 1))[:size]
        db.kf_counter = size
        db.kf_ids = list(range(size))
        r = {}
        if size > 0:
            db._aggregate(desc[0], codes, 5, s["qw"].data_ptr(), s["qsig"].data_ptr(), s["qcount"].data_ptr())
            r["search_ms"] = ev_time(lambda: db._search(size), args.reps)
            sc = db._search(size)
            out = torch.empty(3 + 3 + 23, dtype=torch.int64, device=dev)
            r["rank_ms"] = ev_time(lambda: R._lib.call("adb_retrieval_rank", size, R._lib.ptr(sc), 3, 5e-3, 23,
                                                       R._lib.ptr(out), R._lib.stream()), args.reps)
        ts = []
        for _ in range(args.reps):
            db.kf_counter, db._window = size, None
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            db.update(q, False, 3, 5e-3)
            torch.cuda.synchronize()   # an empty database has no read to wait on
            ts.append((time.perf_counter() - t0) * 1e3)
        r["update_ms"] = float(np.median(ts))
        # reference-style: torch device quantisation, then the host ASMK of the oracle
        ivf = rr.InvertedFile()
        cn = torch.sum(cent_dev ** 2, dim=1)
        if size > 0:
            words_h = [db.ivf_row(i)[0].cpu().numpy() for i in range(min(size, 16))]
            sig_h = [db.ivf_row(i)[1].cpu().numpy().view(np.uint32) for i in range(min(size, 16))]
            for i in range(size):
                ivf.add(sig_h[i % 16], words_h[i % 16])
        ts = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            dq = desc[0]
            l2 = torch.sum(dq ** 2, dim=1)[:, None] + cn[None, :] - 2 * (dq @ cent_dev.mT)
            idx = torch.topk(l2, 5, dim=1, largest=False).indices.cpu().numpy()
            d_np = dq.cpu().numpy()
            if size > 0:
                qsig, qw = rr.aggregate(d_np, idx, cent.numpy())
                ivf.search(qsig, qw)
            ts.append((time.perf_counter() - t0) * 1e3)
        r["reference_style_ms"] = float(np.median(ts))
        res["sizes"][size] = r
        db.kf_counter = rows
        print(size, r, flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()

"""Time the grid-hash KNN (csrc/knn.cu) against another build of the library, for example the parent commit's:

    python tests/perf/time_knn.py --baseline-lib /path/to/other/libartdeco_b200.so [--reps 7] [--out knn.json]

distCUDA2 (adb_knn_mean3) and distIndex2 with K = 8 (adb_knn_index) at 1M points, on the bench scene
(synthetic.raster_scene(1M, seed=0)) and on a flat 200 x 200 plane.  Both builds are loaded into this process and
called through their C ABI on the same inputs and workspace.  Each measurement is CUDA events around 10 back-to-back
calls after warm-up; the two builds alternate, and the median of --reps per call is reported.  The outputs of the two
builds are compared as well: where both are exact they are bit-identical."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from artdeco_b200 import _lib, synthetic  # noqa: E402

CALLS = 10
vp, i32, i64 = C.c_void_p, C.c_int, C.c_longlong


class Build:
    def __init__(self, path):
        self.path = str(path)
        self.h = C.CDLL(self.path)
        for name, args in (("adb_knn_workspace_bytes", [i64, C.POINTER(C.c_size_t)]),
                           ("adb_knn_mean3", [i64, vp, vp, vp, C.c_size_t, vp]),
                           ("adb_knn_index", [i64, vp, i32, i64, vp, vp, vp, vp, vp, C.c_size_t, vp])):
            getattr(self.h, name).argtypes = args
            getattr(self.h, name).restype = C.c_int
        self.h.adb_last_error.restype = C.c_char_p

    def _ok(self, rc):
        if rc:
            raise RuntimeError(f"{self.path}: {self.h.adb_last_error().decode()}")

    def ws_bytes(self, P):
        nb = C.c_size_t(0)
        self._ok(self.h.adb_knn_workspace_bytes(P, C.byref(nb)))
        return nb.value

    def mean3(self, pts, out, ws):
        s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        self._ok(self.h.adb_knn_mean3(pts.shape[0], pts.data_ptr(), out.data_ptr(), ws.data_ptr(), ws.numel(), s))

    def index(self, pts, K, d, ids, ws):
        s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        P = pts.shape[0]
        self._ok(self.h.adb_knn_index(P, pts.data_ptr(), K, P, None, None, d.data_ptr(), ids.data_ptr(),
                                      ws.data_ptr(), ws.numel(), s))


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(CALLS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / CALLS


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-lib", required=True, help="another build of libartdeco_b200.so to compare against")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_knn.py needs a CUDA device")
    _lib.lib()  # builds the tree's library if it is missing
    builds = {"this": Build(_lib.LIB_PATH), "baseline": Build(a.baseline_lib)}
    dev = torch.device("cuda:0")
    P, K = 1_000_000, 8
    g = np.random.default_rng(0)
    scenes = {
        "bench_scene": synthetic.raster_scene(P, seed=0)["means"],
        "flat_plane": torch.from_numpy(np.concatenate([g.uniform(-100, 100, (P, 2)), np.full((P, 1), 2.0)], 1)
                                       .astype(np.float32)),
    }
    ws = torch.empty(max(b.ws_bytes(P) for b in builds.values()), dtype=torch.uint8, device=dev)
    results = {}
    for sname, pts in scenes.items():
        pts = pts.to(dev).contiguous()
        outs = {n: (torch.empty(P, device=dev), torch.empty(P * K, device=dev),
                    torch.empty(P * K, dtype=torch.int32, device=dev)) for n in builds}
        ops = {n: {"distCUDA2": (lambda b=b, o=outs[n]: b.mean3(pts, o[0], ws)),
                   "distIndex2_K8": (lambda b=b, o=outs[n]: b.index(pts, K, o[1], o[2], ws))} for n, b in builds.items()}
        for n in builds:  # warm-up every shape
            for f in ops[n].values():
                f()
                f()
        torch.cuda.synchronize()
        same = {"distCUDA2": torch.equal(outs["this"][0], outs["baseline"][0]),
                "distIndex2_K8_dists": torch.equal(outs["this"][1], outs["baseline"][1]),
                "distIndex2_K8_ids": torch.equal(outs["this"][2], outs["baseline"][2])}
        t = {n: {op: [] for op in ops[n]} for n in builds}
        for _ in range(a.reps):
            for n in builds:
                for op, f in ops[n].items():
                    t[n][op].append(timed(f))
        results[sname] = {"identical_outputs": same}
        for op in ops["this"]:
            m = {n: float(np.median(t[n][op])) for n in builds}
            results[sname][op] = {"this_ms": round(m["this"], 4), "baseline_ms": round(m["baseline"], 4),
                                  "ratio": round(m["this"] / m["baseline"], 4),
                                  "this_all": [round(v, 4) for v in t["this"][op]],
                                  "baseline_all": [round(v, 4) for v in t["baseline"][op]]}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    card = q[0] if q else torch.cuda.get_device_name(0)
    out = {"card": card, "P": P, "K": K, "calls_per_sample": CALLS, "reps": a.reps, "results": results}
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

"""Band scatter and sort of the multi-view tile intersection (adb_raster_tile_band_scatter_sort_multi), timed apart, on the
bench scene (1M Gaussians, 1920x1080, views 0..7, the bench's seeds, capacities from MultiViewStep.calibrate).

Each timed launch is preceded, untimed, by what the step runs before it: counters zeroed, adb_raster_project_fwd_multi,
adb_raster_tile_scan_multi.  It reports:
  * CUDA events around the whole entry point, per launch (--launches launches, after --warmup);
  * the device time of each kernel inside it, from torch.profiler (CUDA activities, a separate run of --launches launches).
Prints one JSON line with the card's name and power limit read in the same process."""
import argparse
import ctypes as C
import json
import os
import re
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from artdeco_b200 import _lib, synthetic  # noqa: E402
from artdeco_b200 import raster as R  # noqa: E402
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
    ap.add_argument("--launches", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--label", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_isect.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    sc = synthetic.raster_scene(N, seed=0)
    t = {k: sc[k].to(dev) for k in ("means", "quats", "scales", "opacities", "sh")}
    cams = [synthetic.camera(W, H, view=float(v)) for v in range(VIEWS)]
    eng = MultiViewStep(t, torch.stack([c[0] for c in cams]).to(dev), torch.stack([c[1] for c in cams]).to(dev), W, H)
    n_isect = eng.calibrate()
    caps = (C.c_longlong * VIEWS)(*eng.capacity)
    total = sum(eng.capacity)
    T = ((W + R.TILE - 1) // R.TILE) * ((H + R.TILE - 1) // R.TILE)
    offsets = torch.empty(VIEWS, T + 1, dtype=torch.int32, device=dev)
    n_dev = torch.zeros(VIEWS, dtype=torch.int64, device=dev)
    ovf = torch.zeros(VIEWS, dtype=torch.int32, device=dev)
    vals = torch.empty(total, dtype=torch.int32, device=dev)
    packed = torch.empty(total, dtype=torch.int64, device=dev)
    st = _lib.stream

    def prepare():
        eng._project()                                  # zeroes the counters, projects and counts every view
        _lib.call("adb_raster_tile_scan_multi", VIEWS, W, H, caps, _lib.ptr(eng.counts), _lib.ptr(offsets),
                  _lib.ptr(n_dev), _lib.ptr(ovf), st())

    args_in = lambda: (N, VIEWS, _lib.ptr(eng.radii), _lib.ptr(eng.splats), _lib.ptr(eng.tpg), W, H, caps,  # noqa: E731
                       _lib.ptr(eng.counts), _lib.ptr(offsets), _lib.ptr(packed))
    nb = C.c_size_t(0)
    _lib.call("adb_raster_tile_band_scratch_bytes", total, C.byref(nb))
    scratch = torch.empty(nb.value, dtype=torch.uint8, device=dev)
    paths = {"band": lambda: _lib.call("adb_raster_tile_band_scatter_sort_multi", *args_in(), _lib.ptr(scratch),
                                       scratch.numel(), None, _lib.ptr(vals), st())}

    res = {}
    for name, fn in paths.items():
        for _ in range(args.warmup):
            prepare()
            fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.launches):
            prepare()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.launches):
                prepare()
                fn()
            torch.cuda.synchronize()
        kernels = {}
        for ev in prof.key_averages():
            if "tile_" in ev.key and "kernel" in ev.key and "scan" not in ev.key and "count" not in ev.key:
                short = re.search(r"(\w+_kernel)", ev.key).group(1)
                kernels[short] = round(ev.device_time_total / 1e3 / args.launches, 4)     # ms per launch
        res[name] = {"ms_per_launch_median": round(statistics.median(ms), 4), "ms_min": round(min(ms), 4),
                     "ms_max": round(max(ms), 4), "kernel_ms_per_launch": kernels}
    print(json.dumps({"label": args.label, "launches": args.launches, "n_isect": n_isect, "capacity": eng.capacity,
                      "paths": res, "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w()}),
          flush=True)


if __name__ == "__main__":
    main()

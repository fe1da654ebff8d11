"""Time the key-frame hand-off on CUDA: the oracle's PyTorch code (oracle/keyframe_ref.py on CUDA tensors, standing in for the
reference: compute_dense_point's torch and pypose kernels, the blocking .cpu() copy of densePoint and its return to the
device, then Keyframe.__init__'s prior, resize and pyramids) against artdeco_b200.keyframe's dense_point + mapper_keyframe.

    python tests/perf/time_keyframe.py [--reps 7] [--out /tmp/time_keyframe.json]

SLAM 512x384 -> mapper 1296x972, pyr_levels = 2.  CUDA events around each whole hand-off, after warm-up, the two paths
alternated; the median of --reps.  The mapper-input kernel alone is timed from CUDA-graph replays of 20 back-to-back launches
and reported as bytes/s against the bytes it must move: the image read once, every pyramid level written once, and the
dense point's z read once."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

REPLAYS = 20
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import keyframe_ref as ref  # noqa: E402
from artdeco_b200 import _lib, keyframe  # noqa: E402
from test_keyframe import make_image, make_inputs  # noqa: E402


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    card = q[0] if q else torch.cuda.get_device_name(0)
    print(f"card: {card}")
    Hs, Ws, H, W, L = 384, 512, 972, 1296, 2
    inp = make_inputs(Hs, Ws, seed=1, dev=dev)
    image = make_image(H, W, seed=2, dev=dev)
    X = inp["X_canon"].reshape(Hs, Ws, 3)
    N = torch.tensor([3], dtype=torch.int32, device=dev)

    def ours():
        dense, _, _ = keyframe.dense_point(X, inp["C"], N, inp["T_WC"], inp["K"], last_T_WC=inp["last_T_WC"],
                                           idx_k2l=inp["idx_k2l"])
        keyframe.mapper_keyframe(image, dense, inp["T_WC"], pyr_levels=L, index=1, is_test=False, lr_poses=1e-3,
                                 lr_exposure=5e-4)

    def torch_path():
        dense, _, _ = ref.prepare_for_mapper(inp["X_canon"], inp["C"], 3, inp["T_WC"], inp["K"], Hs, Ws,
                                             last_T_WC=inp["last_T_WC"], idx_k2l=inp["idx_k2l"])
        dense = dense.cpu().to(dev)                                    # the reference's message round trip
        ref.mapper_keyframe(image, dense, inp["T_WC"], L)

    for _ in range(3):
        ours()
        torch_path()
    torch.cuda.synchronize()
    times = {"ours": [], "torch": []}
    for _ in range(a.reps):
        times["ours"].append(timed(ours))
        times["torch"].append(timed(torch_path))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}

    # the mapper-input kernel alone, on preallocated buffers
    dense, _, _ = keyframe.dense_point(X, inp["C"], N, inp["T_WC"], inp["K"], last_T_WC=inp["last_T_WC"],
                                       idx_k2l=inp["idx_k2l"])
    n_id, n_im = C.c_longlong(0), C.c_longlong(0)
    _lib.call("adb_kf_pyramid_floats", H, W, L, C.byref(n_id), C.byref(n_im))
    id_buf = torch.empty(n_id.value, device=dev)
    im_buf = torch.empty(max(n_im.value, 1), device=dev)
    pose = [torch.empty(n, device=dev) for n in (6, 3, 3, 9)]
    strides = (C.c_longlong * 3)(*image.stride())
    T = inp["T_WC"].contiguous()

    def launch():
        _lib.call("adb_kf_mapper_inputs", H, W, Hs, Ws, L, C.c_void_p(image.data_ptr()), strides, _lib.ptr(dense),
                  _lib.ptr(T), _lib.ptr(id_buf), _lib.ptr(im_buf), *[_lib.ptr(p) for p in pose], _lib.stream())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        launch()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(REPLAYS):
            launch()
    for _ in range(3):
        graph.replay()
    kt = sorted(timed(graph.replay) for _ in range(a.reps))[a.reps // 2] / REPLAYS
    need = 4 * (3 * H * W + n_id.value + n_im.value + Hs * Ws)
    row = dict(slam=f"{Ws}x{Hs}", mapper=f"{W}x{H}", pyr_levels=L, ours_ms=round(med["ours"], 3),
               torch_ms=round(med["torch"], 3), speedup=round(med["torch"] / med["ours"], 1),
               mapper_inputs_kernel_us=round(kt * 1e3, 2), mapper_inputs_MB=round(need / 1e6, 2),
               mapper_inputs_GBps=round(need / (kt * 1e-3) / 1e9, 1))
    print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(dict(card=card, rows=[row]), fh, indent=1)


if __name__ == "__main__":
    main()

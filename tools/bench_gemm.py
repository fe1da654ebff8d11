"""Per-shape timing of the wgmma GEMM on the MASt3R shapes (CUDA events, 20 reps after 3 warm-ups)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from artdeco_b200.mast3r import ops  # noqa: E402

dev = torch.device("cuda:0")
SHAPES = [  # name, batch, M, N, K
    ("enc.qkv", 1, 2048, 3072, 1024), ("enc.proj", 1, 2048, 1024, 1024), ("enc.fc1", 1, 2048, 4096, 1024),
    ("enc.fc2", 1, 2048, 1024, 4096), ("enc.QK^T", 32, 1024, 1024, 64), ("enc.PV", 32, 1024, 64, 1024),
    ("dec.qkv", 1, 1024, 2304, 768), ("dec.proj", 1, 1024, 768, 768), ("dec.fc1", 1, 1024, 3072, 768),
    ("dec.fc2", 1, 1024, 768, 3072), ("dec.QK^T", 12, 1024, 1024, 64), ("dec.PV", 12, 1024, 64, 1024),
    ("head.fc1", 1, 1024, 7168, 1792), ("head.fc2", 1, 1024, 6400, 7168), ("big", 1, 8192, 8192, 4096),
]
for x3 in (True, False):
    for name, b, M, N, K in SHAPES:
        a = ops.split(torch.randn(b * M, K, device=dev), x3)
        w = ops.split(torch.randn(b * N, K, device=dev) * 0.05, x3)
        out = torch.empty(b * M, N, device=dev)
        kw = dict(batch=b, sA=M * K if b > 1 else 0, sB=N * K if b > 1 else 0, sD=M * N if b > 1 else 0, out=out)
        for _ in range(3):
            ops.gemm(a, w, M, N, K, **kw)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(20):
            ops.gemm(a, w, M, N, K, **kw)
        e.record()
        torch.cuda.synchronize()
        us = s.elapsed_time(e) / 20 * 1e3
        fl = 2.0 * b * M * N * K
        print(f"{'x3' if x3 else 'bf16':5s} {name:10s} b={b:2d} {M}x{N}x{K}: {us:8.1f} us  {fl / us / 1e6:7.1f} TFLOP/s algorithmic"
              f"  ({fl * (3 if x3 else 1) / us / 1e6:7.1f} tensor)")

"""Per-stage live timing (CUDA events on the launching stream) of the rasterizer step at the bench workload, without the
e2e / MASt3R / CPU legs."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from artdeco_b200 import _lib, synthetic  # noqa: E402
from artdeco_b200 import raster as R  # noqa: E402

N = int(os.environ.get("ADB_N", "1000000"))
steps = int(os.environ.get("ADB_STEPS", "20"))
W, H = int(os.environ.get("ADB_W", "1920")), int(os.environ.get("ADB_H", "1080"))
view = float(os.environ.get("ADB_VIEW", "3.5"))
dev = torch.device("cuda:0")
sc = synthetic.raster_scene(N, seed=0)
V, K = synthetic.camera(W, H, view=view)
vc, va = synthetic.upstream_grads(W, H, seed=1)
t = {k: sc[k].to(dev) for k in ("means", "quats", "scales", "opacities", "sh")}
Vd, Kd, vcd, vad = V.to(dev), K.to(dev), vc[0].contiguous().to(dev), va[0, ..., 0].contiguous().to(dev)
campos = torch.inverse(Vd)[:3, 3].contiguous()
gm, gq, gs, go, gsh = (torch.empty_like(t[k]) for k in ("means", "quats", "scales", "opacities", "sh"))
vv, vcp = torch.zeros(4, 4, device=dev), torch.zeros(3, device=dev)
info = {}


def step():
    cnt = R.new_tile_counts(W, H, dev) if os.environ.get("ADB_FUSED_COUNT", "1") == "1" else None
    radii, splats, tpg = R.project(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], 3, Vd, Kd, campos, W, H,
                                   0.01, 0.01, 1e10, 0.0, tile_counts=cnt)
    keys, vals, offs, n = R.intersect(radii, splats, tpg, W, H, counts=cnt)
    hits = R.new_hit_mask(vals)
    colors, alphas, last = R.blend_forward(W, H, N, splats, vals, offs, hits=hits)
    v_splats = R.blend_backward(W, H, N, splats, vals, offs, alphas, last, vcd, vad, hits=hits)
    _lib.call("adb_raster_project_bwd", N, _lib.ptr(t["means"]), _lib.ptr(t["quats"]), _lib.ptr(t["scales"]),
              _lib.ptr(t["sh"]), 3, _lib.ptr(Vd), _lib.ptr(Kd), _lib.ptr(campos), W, H, 0.01, 0.01, 1e10, 0.0,
              _lib.ptr(radii), _lib.ptr(splats), _lib.ptr(v_splats), _lib.ptr(gm), _lib.ptr(gq), _lib.ptr(gs),
              _lib.ptr(go), _lib.ptr(gsh), _lib.ptr(vv), _lib.ptr(vcp), _lib.stream())
    info["n_isect"] = n


for _ in range(5):
    step()
torch.cuda.synchronize()
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record()
for _ in range(steps):
    step()
b.record()
torch.cuda.synchronize()
ms = a.elapsed_time(b) / steps
_lib.TIMER = _lib.StageTimer()
for _ in range(steps):
    step()
torch.cuda.synchronize()
tot = _lib.TIMER.totals_ms()
_lib.TIMER = None
print(json.dumps({"N": N, "W": W, "H": H, "ms_per_step": ms, "n_isect": info["n_isect"],
                  "stage_ms": {k.replace("adb_raster_", ""): round(v[0] / v[1], 4) for k, v in tot.items()}}))

"""Runs the REAL reference Pi3 (imported from the reference tree, CPU fp32) on deterministic weights, checks
oracle/pi3_torch.py against it and writes tests/golden/pi3_small.pt (N=3 at 112x140) and tests/golden/pi3_full.pt
(N=2 at 392x518).  Outputs and stage tensors are kept at a pixel / token / channel stride so each file stays at a few
hundred KB; the pixel strides (5, 11) are coprime to the 14-pixel patch, so every position inside a patch is sampled.
Run from the repository root where the reference tree exists:
``python tests/golden/make_pi3_golden.py [small|full] --ref ARTDECO_ROOT``."""
import argparse
import pathlib
import sys
import time

import torch

ROOT = pathlib.Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

from artdeco_b200 import synthetic  # noqa: E402
from artdeco_b200.pi3.shapes import param_shapes  # noqa: E402
from oracle import pi3_torch as pt  # noqa: E402


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-20))


@torch.inference_mode()
def run(ref_root, N, H, W, tag, stride_px, stride_tok, stride_ch):
    sys.path.insert(0, str(ref_root / "VSLAM" / "thirdparty" / "Pi3"))
    from pi3.models.pi3 import Pi3 as RefPi3

    model = RefPi3().eval()
    shapes = param_shapes()
    read_set = {k: tuple(v.shape) for k, v in model.named_parameters()}
    assert read_set == shapes, (set(read_set) ^ set(shapes))
    sd = synthetic.det_weights(shapes)
    res = model.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and set(res.missing_keys) == {"image_mean", "image_std"}, res
    imgs = synthetic.pi3_frames(N, H, W, seed=0)
    st = {}
    hooks = [model.encoder.register_forward_hook(lambda m, i, o: st.__setitem__("encoder", o["x_norm_patchtokens"]))]
    for name in ("point_decoder", "conf_decoder", "camera_decoder"):
        hooks.append(getattr(model, name).register_forward_hook(
            lambda m, i, o, n=name: st.__setitem__(n.replace("_decoder", "_hidden"), o)))
    hooks.append(model.camera_head.fc_rot.register_forward_hook(lambda m, i, o: st.__setitem__("fc_rot", o)))
    hooks.append(model.camera_head.fc_t.register_forward_hook(lambda m, i, o: st.__setitem__("fc_t", o)))
    dec = model.decode
    model.decode = lambda *a: (lambda r: (st.__setitem__("decoder", r[0]), r)[1])(dec(*a))
    t0 = time.time()
    out = model(imgs)
    print(f"[{tag}] reference forward {time.time() - t0:.1f}s")
    gh, gw = H // 14, W // 14
    x_dummy = torch.zeros(1, 1 + gh * gw, 1024)
    pos_table = model.encoder.interpolate_pos_encoding(x_dummy, H, W)

    ost = {}
    t0 = time.time()
    o = pt.forward(sd, imgs, stages=ost)
    print(f"[{tag}] oracle forward {time.time() - t0:.1f}s")
    errs = {k: rel(o[k], out[k]) for k in ("points", "local_points", "conf", "camera_poses")}
    errs.update({"stage." + k: rel(ost[k], st[k]) for k in st})
    errs["pos_table_bits"] = float((pt.interpolate_pos_embed(sd["encoder.pos_embed"], gh, gw) != pos_table).sum())
    print(f"[{tag}] oracle vs reference:", {k: f"{v:.2e}" for k, v in errs.items()})
    assert all(v < 1e-5 for v in errs.values()), errs

    # singular values of the normalised, transposed fc_rot (camera_head.py:85-86): the GPU test scales R's tolerance
    m = torch.nn.functional.normalize(st["fc_rot"].double().reshape(-1, 3, 3), dim=-1).transpose(-1, -2)
    sv = torch.linalg.svdvals(m)
    sp, tk, ch = stride_px, stride_tok, stride_ch
    g = dict(N=N, H=H, W=W, seed=0, stride_px=sp, stride_tok=tk, stride_ch=ch,
             read_set=read_set,
             points=out["points"][:, :, ::sp, ::sp].contiguous(), local_points=out["local_points"][:, :, ::sp, ::sp].contiguous(),
             conf=out["conf"][:, :, ::sp, ::sp].contiguous(), camera_poses=out["camera_poses"].contiguous(),
             fc_rot=st["fc_rot"].contiguous(), fc_t=st["fc_t"].contiguous(), fc_rot_singular_values=sv,
             pos_table=pos_table[:, ::tk, ::ch].contiguous())
    for k in ("encoder", "decoder", "point_hidden", "conf_hidden", "camera_hidden"):
        g["stage." + k] = st[k][:, ::tk, ::ch].contiguous()
    path = ROOT / "tests" / "golden" / f"pi3_{tag}.pt"
    torch.save(g, path)
    print(f"[{tag}] wrote {path} ({path.stat().st_size / 1e6:.2f} MB)")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("which", nargs="*", default=["small", "full"])
    ap.add_argument("--ref", required=True, help="root of the ARTDECO source tree (the directory holding VSLAM/)")
    a = ap.parse_args()
    ref = pathlib.Path(a.ref)
    if "small" in a.which:
        run(ref, 3, 112, 140, "small", 5, 3, 16)
    if "full" in a.which:
        run(ref, 2, 392, 518, "full", 11, 8, 64)

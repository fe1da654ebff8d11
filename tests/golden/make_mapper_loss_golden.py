"""Writes tests/golden/mapper_loss_small.pt by running the reference's OWN loss statements on the CPU.

The reference modules cannot be imported here (gsplat, fused_ssim and the rest of the training stack are not installed), so
the code is extracted with ``ast``:
  * Reconstruct/utils.py: ``radial_decay_kernel``;
  * Reconstruct/scene/scene_models/h3dgsv3.py: ``render_from_id`` (exposure and clamp), the background composite and ``1/D``
    statements of ``render`` (everything after the rasterizer call up to ``invdepth``), and the loss statements of
    ``optimization_step`` (from ``c, h, w = image.shape`` to ``loss = ...``), whose one ``.cuda()`` is dropped;
and executed on the rasterizer outputs of oracle.mapper_loss_ref.make_inputs with ``fused_ssim`` bound to the pinned conv2d
SSIM of oracle.ssim_ref.  ``loss.backward()`` gives the gradients of colors, alphas and the exposure.  Only inputs, outputs and
gradients are saved, no reference source.

    python tests/golden/make_mapper_loss_golden.py [/path/to/reference]
"""
import ast
import os
import sys
import textwrap
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import mapper_loss_ref, ssim_ref  # noqa: E402

H, W = 37, 53
LAMBDA, DEPTH_W = 0.2, 0.6


def _func(src, tree, name):
    node = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == name)
    return node, textwrap.dedent(ast.get_source_segment(src, node))


def _statements(src, stmts, first, last):
    """Source of the statements from the one starting with ``first`` to the one starting with ``last`` (inclusive)."""
    segs = [textwrap.dedent(ast.get_source_segment(src, s)) for s in stmts]
    i = next(k for k, s in enumerate(segs) if s.startswith(first))
    j = next(k for k, s in enumerate(segs) if k >= i and s.startswith(last))
    return "\n".join(segs[i:j + 1])


def extract(ref_dir):
    u_path = os.path.join(ref_dir, "Reconstruct", "utils.py")
    h_path = os.path.join(ref_dir, "Reconstruct", "scene", "scene_models", "h3dgsv3.py")
    u_src, h_src = open(u_path).read(), open(h_path).read()
    u_tree, h_tree = ast.parse(u_src), ast.parse(h_src)
    _, rdk_src = _func(u_src, u_tree, "radial_decay_kernel")
    _, rfi_src = _func(h_src, h_tree, "render_from_id")
    render_node = next(n for n in ast.walk(h_tree) if isinstance(n, ast.FunctionDef) and n.name == "render"
                       and any(a.arg == "view_matrix" for a in n.args.args))
    with_node = next(n for n in render_node.body if isinstance(n, ast.With))
    comp_src = _statements(h_src, with_node.body, "rendered_color = colors", "invdepth = ")
    opt_node, _ = _func(h_src, h_tree, "optimization_step")
    loss_src = _statements(h_src, opt_node.body, "c, h, w = image.shape", "loss = (")
    assert loss_src.count(".cuda()") == 1, "expected the one .cuda() of the radial table"
    loss_src = loss_src.replace(".cuda()", "")
    return rdk_src, rfi_src, comp_src, loss_src


def make_case(code, seed, important, zero_depth, sigma):
    rdk_src, rfi_src, comp_src, loss_src = code
    inp = mapper_loss_ref.make_inputs(H, W, seed, zero_depth=zero_depth)
    colors = inp["colors"].clone().requires_grad_(True)
    alphas = inp["alphas"].clone().requires_grad_(True)
    exposure = inp["exposure"].clone().requires_grad_(True)

    ns = dict(torch=torch)
    exec(rdk_src, ns)
    exec(rfi_src, ns)

    class Stub:
        pass
    self = Stub()
    self.device = "cpu"
    self.width, self.height = W, H
    self.lambda_dssim, self.rad_decay, self.scaling_reg_factor = LAMBDA, sigma, 0.0
    kf = types.SimpleNamespace(exposure=exposure, get_Rt=lambda: torch.eye(4), depth_loss_weight=DEPTH_W)
    self.keyframes = [kf]

    def render(width, height, view_matrix, bg):
        scope = dict(torch=torch, colors=colors, alphas=alphas, bg=bg)
        exec(comp_src, scope)
        return {"render": scope["rendered_color"][0], "invdepth": scope["invdepth"][0]}
    self.render = render
    render_pkg = types.MethodType(ns["render_from_id"], self)(0, pyr_lvl=0, bg=inp["bg"])
    scope = dict(torch=torch, self=self, keyframe=kf, is_important=important, radial_decay_kernel=ns["radial_decay_kernel"],
                 fused_ssim=lambda a, b: ssim_ref.ssim(a, b), image=render_pkg["render"], invdepth=render_pkg["invdepth"],
                 scale=torch.zeros(1, 3), gt_image=inp["gt"], mono_idepth=inp["mono"])
    exec(loss_src, scope)
    scope["loss"].backward()
    out = dict(loss=scope["loss"].detach(), l1=scope["l1_loss"].detach(), ssim_loss=scope["ssim_loss"].detach(),
               depth=scope["depth_loss"].detach(), image=scope["image"].detach(), invdepth=scope["invdepth"].detach(),
               rdk=scope["rdk"].clone(), v_colors=colors.grad.clone(), v_alphas=alphas.grad.clone(),
               v_exposure=exposure.grad.clone())
    return dict(H=H, W=W, seed=seed, is_important=important, zero_depth=zero_depth, rad_decay=sigma, lambda_dssim=LAMBDA,
                depth_weight=DEPTH_W, inputs=inp, outputs=out)


def main():
    ref_dir = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    code = extract(ref_dir)
    cases = [make_case(code, 21, True, True, 1.0), make_case(code, 22, False, True, 1.0),
             make_case(code, 23, True, False, 0.5), make_case(code, 24, False, False, 0.5)]
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mapper_loss_small.pt")
    torch.save(dict(cases=cases), out)
    for c in cases:
        o = c["outputs"]
        print(f"important={c['is_important']} zero_depth={c['zero_depth']}: loss={o['loss'].item():.6g} "
              f"nonfinite v_colors={int((~torch.isfinite(o['v_colors'])).sum())} "
              f"masked={int((o['image'] == 0).all(0).sum()) if not c['is_important'] else 0}")
    print(f"wrote {out} ({os.path.getsize(out) // 1024} KB)")


if __name__ == "__main__":
    main()

"""Writes tests/golden/evaluate_small.pt by running the reference's OWN evaluation code on the CPU.

The reference modules cannot be imported here (gsplat, lpips, fused_ssim and the rest of the training stack are not
installed), so the code is extracted with ``ast``:
  * Reconstruct/utils.py: ``psnr``;
  * Reconstruct/scene/scene_models/h3dgsv3.py: ``SceneModel.harmonize_test_exposure``, ``SceneModel.evaluate`` and
    ``SceneModel.render_from_id``;
and executed as methods of a stub scene whose ``render`` returns fixed rasterizer outputs through the background composite
of oracle.mapper_loss_ref, with ``fused_ssim`` bound to the pinned conv2d SSIM of oracle.ssim_ref and ``self.lpips`` to
oracle.evaluate_ref's LPIPS with seeded random weights (the seed is stored, not the 15M weights).  Scenes cover test frames
at index 0, at the last index and back to back, K = 2, K = 1 without and with a test frame (the reference raises
IndexError there) and exposures that are not exactly representable.  Only inputs and outputs are saved, no reference
source.

    python tests/golden/make_evaluate_golden.py [/path/to/reference]
"""
import ast
import os
import sys
import textwrap

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import evaluate_ref, ssim_ref  # noqa: E402
from oracle.mapper_loss_ref import composite  # noqa: E402

H, W = 20, 28
N_GAUSS = 500
LPIPS_SEED = 7
SCENES = {
    # name: (is_test, with_LPIPS, all)
    "mixed": ([1, 0, 1, 1, 0, 1], True, True),
    "pair_last": ([0, 1], True, False),
    "pair_both": ([1, 1], False, True),
    "single_train": ([0], True, True),
    "single_test": ([1], True, True),
}


def _func(src, tree, name):
    node = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == name)
    return textwrap.dedent(ast.get_source_segment(src, node))


def extract(ref_dir):
    u_path = os.path.join(ref_dir, "Reconstruct", "utils.py")
    h_path = os.path.join(ref_dir, "Reconstruct", "scene", "scene_models", "h3dgsv3.py")
    u_src, h_src = open(u_path).read(), open(h_path).read()
    u_tree, h_tree = ast.parse(u_src), ast.parse(h_src)
    return (_func(u_src, u_tree, "psnr"), _func(h_src, h_tree, "harmonize_test_exposure"),
            _func(h_src, h_tree, "evaluate"), _func(h_src, h_tree, "render_from_id"))


def make_inputs(K, seed):
    g = torch.Generator().manual_seed(seed)
    rgb = torch.rand(K, 1, H, W, 3, generator=g) * 1.2 - 0.1     # exposure and clamp see values outside [0, 1]
    depth = torch.rand(K, 1, H, W, 1, generator=g) + 0.5
    colors = torch.cat([rgb, depth], -1).contiguous()
    alphas = torch.rand(K, 1, H, W, 1, generator=g)
    gt = torch.rand(K, 3, H, W, generator=g)
    base = torch.eye(3, 4).expand(K, 3, 4)
    exposure = (base + 0.05 * torch.randn(K, 3, 4, generator=g)).contiguous()   # not exactly representable sums
    vis = torch.rand(K, N_GAUSS, generator=g) < 0.6
    return colors, alphas, gt, exposure, vis


class _Keyframe:
    def __init__(self, index, is_test, exposure, gt):
        self.index, self.is_test, self.exposure, self.image_pyr = index, bool(is_test), exposure, [gt]

    def get_Rt(self):
        return torch.full((4, 4), float(self.index))


def run_scene(methods, is_test, with_lpips, all_, seed, lpips):
    K = len(is_test)
    colors, alphas, gt, exposure, vis = make_inputs(K, seed)

    class Scene:
        pass

    for name, fn in methods.items():
        setattr(Scene, name, fn)
    sc = Scene()
    sc.device = torch.device("cpu")
    sc.width, sc.height = W, H
    sc.lpips = lpips
    sc.keyframes = [_Keyframe(i, is_test[i], exposure[i].clone(), gt[i]) for i in range(K)]

    def render(width, height, view_matrix, bg):
        i = int(view_matrix[0, 0])
        img, _ = composite(colors[i], alphas[i], bg)
        return {"render": img, "visibility_filter": vis[i]}

    sc.render = render
    out = {"is_test": torch.tensor(is_test, dtype=torch.bool), "with_LPIPS": with_lpips, "all": all_,
           "colors": colors, "alphas": alphas, "gt": gt, "exposure": exposure, "visibility": vis}
    try:
        out["metrics"] = sc.evaluate(with_lpips, all_)
        out["raises"] = None
    except IndexError as e:
        out["metrics"] = None
        out["raises"] = type(e).__name__
    out["exposure_out"] = torch.stack([kf.exposure for kf in sc.keyframes])
    return out


def main(ref_dir):
    psnr_src, harm_src, eval_src, rfi_src = extract(ref_dir)
    ns = {"torch": torch, "F": torch.nn.functional,
          "fused_ssim": lambda a, b, train=True: ssim_ref.ssim(a, b)}
    exec(psnr_src, ns)
    for src in (harm_src, eval_src, rfi_src):
        exec(src, ns)
    methods = {"harmonize_test_exposure": ns["harmonize_test_exposure"], "evaluate": ns["evaluate"],
               "render_from_id": ns["render_from_id"]}
    lpips = evaluate_ref.make_lpips(LPIPS_SEED)
    gold = {"H": H, "W": W, "lpips_seed": LPIPS_SEED, "scenes": {}}
    for k, (name, (is_test, with_lpips, all_)) in enumerate(SCENES.items()):
        gold["scenes"][name] = run_scene(methods, is_test, with_lpips, all_, 100 + k, lpips)
        print(name, gold["scenes"][name]["metrics"], gold["scenes"][name]["raises"])
    path = os.path.join(ROOT, "tests", "golden", "evaluate_small.pt")
    torch.save(gold, path)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")

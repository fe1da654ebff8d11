"""Writes tests/golden/densify_small.pt by running the reference's OWN ``add_new_gaussians`` on the CPU.

The reference modules cannot be imported here (kornia, plyfile, e3nn, gsplat, lpips and torch_scatter are not installed), so
the functions are extracted with ``ast`` from Reconstruct/utils.py (get_lapla_norm, make_torch_sampler, sample,
depth2points, RGB2SH, inverse_sigmoid, C0) and Reconstruct/scene/scene_models/h3dgsv3.py (render_from_id, add_new_gaussians
and the centre / disc / uv lines of __init__) and executed against a stub ``self``:
  * ``self.render`` returns a fixed raw render (``render_from_id`` applies the exposure itself);
  * ``self.update_voxel`` is oracle.voxel_ref.update_voxel; ``optimizer.add_and_prune`` and ``weed_out_gaussians`` record
    their arguments;
  * the two ``device="cuda"`` literals of add_new_gaussians are rewritten to the CPU.
``torch.rand_like`` is wrapped to record the draws.  Only inputs, draws and outputs are saved, no reference source.

    python tests/golden/make_densify_golden.py [/path/to/reference]
"""
import ast
import os
import sys
import types

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import voxel_ref  # noqa: E402

H, W, HS, WS = 45, 61, 23, 31
ARGS = dict(init_proba_scaler=2.0, gs_add_ratio=0.8, voxel_size=0.5, local_feat_dim=4, global_feat_dim=6, sh_degree=3)


def _extract(path, names):
    src = open(path).read()
    tree = ast.parse(src)
    out = {}
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef) and node.name in names and node.name not in out:
            out[node.name] = ast.get_source_segment(src, node)
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id in names for t in node.targets):
            out[node.targets[0].id] = ast.get_source_segment(src, node)
    return out, src, tree


def _dedent(s):
    import textwrap
    return textwrap.dedent(s)


def _init_block(h3_src, h3_tree):
    """The reference's __init__ lines that set self.centre, the disc kernel, self.lods and self.uvs."""
    init = next(n for n in ast.walk(h3_tree) if isinstance(n, ast.FunctionDef) and n.name == "__init__"
                and any(isinstance(a, ast.arg) and a.arg == "width" for a in n.args.args))
    lines = []
    keep = False
    for st in init.body:
        seg = ast.get_source_segment(h3_src, st)
        if "self.centre" in seg:
            lines.append(_dedent(seg))
        if isinstance(st, ast.Assign) and seg.strip().startswith("radius = 3"):
            keep = True
        if keep:
            lines.append(_dedent(seg))
    return "def _init_helpers(self, width, height):\n" + "\n".join("    " + ln for b in lines for ln in b.splitlines()) + "\n"


class Recorder:
    def __init__(self):
        self.calls = []

    def add_and_prune(self, ext, mask):
        self.calls.append(({k: v.clone() for k, v in ext.items()}, mask.clone()))


def make_case(ref_dir, seed, warm):
    utils_path = os.path.join(ref_dir, "Reconstruct", "utils.py")
    h3_path = os.path.join(ref_dir, "Reconstruct", "scene", "scene_models", "h3dgsv3.py")
    u_funcs, _, _ = _extract(utils_path, {"get_lapla_norm", "make_torch_sampler", "sample", "depth2points", "RGB2SH",
                                          "inverse_sigmoid", "C0"})
    h_funcs, h3_src, h3_tree = _extract(h3_path, {"add_new_gaussians", "render_from_id"})
    ns = dict(torch=torch, F=F, math=__import__("math"))
    for name in ("C0", "get_lapla_norm", "make_torch_sampler", "sample", "depth2points", "RGB2SH", "inverse_sigmoid"):
        exec(u_funcs[name], ns)
    anq = _dedent(h_funcs["add_new_gaussians"]).replace('device="cuda"', 'device="cpu"')
    assert anq.count('device="cpu"') == 2, "expected the two device=\"cuda\" literals"
    exec(anq.replace("@torch.no_grad()\n", ""), ns)
    exec(_dedent(h_funcs["render_from_id"]), ns)
    exec(_init_block(h3_src, h3_tree), ns)

    g = torch.Generator().manual_seed(seed)
    image = torch.rand(3, H, W, generator=g)
    image[:, 10:30, 20:40] = 0.5 + 0.4 * torch.rand(3, 1, 1, generator=g)          # flat patch + edges
    depth = 1.0 + 4.0 * torch.rand(HS, WS, generator=g)
    depth[0, :5] = 0.001                                                               # below the 0.02 quantile
    xyzm = torch.stack([torch.randn(HS, WS, generator=g), torch.randn(HS, WS, generator=g), depth])[None]
    conf = 3.0 * torch.rand(1, 1, HS, WS, generator=g) - 0.3                          # some negative
    conf[0, 0, 5:8, 5:8] = 6.0                                                         # inverse_sigmoid -> NaN
    ang = 0.1
    R = torch.tensor([[1.0, 0.0, 0.0], [0.0, torch.cos(torch.tensor(ang)), -torch.sin(torch.tensor(ang))],
                      [0.0, torch.sin(torch.tensor(ang)), torch.cos(torch.tensor(ang))]])
    t = torch.tensor([0.1, -0.2, 0.3])
    Rt = torch.eye(4)
    Rt[:3, :3], Rt[:3, 3] = R, t
    exposure = torch.eye(3, 4) * 1.1
    exposure[:, 3] = torch.tensor([0.02, -0.03, 0.01])
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    raw = 0.45 + 0.1 * torch.sin(xx / 9.0)[None] * torch.tensor([1.0, 0.5, -0.7])[:, None, None] \
        + 0.02 * torch.rand(3, H, W, generator=g)                                   # a smooth scene: a small penalty
    f = 50.0
    N = 300 if warm else 0
    params = dict(
        id=torch.zeros(N, 1, dtype=torch.long), cls_id=torch.randint(0, 5, (N, 1), generator=g),
        d_max=4.0 + 4 * torch.rand(N, 1, generator=g), xyz=torch.randn(N, 3, generator=g) * 2,
        f_dc=torch.randn(N, 1, 3, generator=g), f_rest=torch.zeros(N, 15, 3),
        scaling=torch.log(0.01 + 0.5 * torch.rand(N, 3, generator=g)), rotation=torch.randn(N, 4, generator=g),
        opacity=torch.randn(N, 1, generator=g) * 3, local_feat=torch.zeros(N, ARGS["local_feat_dim"]),
        global_feat=torch.zeros(5 if warm else 0, ARGS["global_feat_dim"]))
    params["scaling"][:5] = 3.0                                                        # huge on screen -> pruned
    init_params = {k: v.clone() for k, v in params.items()}

    kf = types.SimpleNamespace(image_pyr=[image], point_map=xyzm, mono_depth_conf=conf, width=W, height=H,
                               is_test=False, exposure=exposure, approx_centre=-R.T @ t, index=0,
                               get_R=lambda: R, get_t=lambda: t, get_Rt=lambda: Rt.clone())

    class Stub:
        pass
    self = Stub()
    self.device = "cpu"
    self.lock = __import__("threading").Lock()
    self.width, self.height, self.f = W, H, f
    ns["_init_helpers"](self, W, H)
    self.gaussian_params = {k: {"val": v} for k, v in params.items()}
    prop = lambda key, fn=None: property(lambda s: fn(s.gaussian_params[key]["val"]) if fn else s.gaussian_params[key]["val"])  # noqa
    Stub.xyz, Stub.cls_id, Stub.f_dc = prop("xyz"), prop("cls_id"), prop("f_dc")
    Stub.opacity, Stub.scaling = prop("opacity", torch.sigmoid), prop("scaling", torch.exp)
    self.init_proba_scaler = ARGS["init_proba_scaler"]
    self.max_sh_degree = ARGS["sh_degree"]
    self.args = types.SimpleNamespace(gs_add_ratio=ARGS["gs_add_ratio"], voxel_size=ARGS["voxel_size"],
                                      local_feat_dim=ARGS["local_feat_dim"], global_feat_dim=ARGS["global_feat_dim"])
    self.keyframes = [kf]
    renders = []

    def render(width, height, view_matrix, bg):
        renders.append(self.cls_id.clone())
        return {"render": raw.clone(), "invdepth": torch.ones(1, height, width)}
    self.render = render
    self.render_from_id = types.MethodType(ns["render_from_id"], self)
    self.update_voxel = lambda new_xyz, xyz, cls_id, voxel_size=0.1: voxel_ref.update_voxel(new_xyz, xyz, cls_id, voxel_size)
    rec = Recorder()
    self.optimizer = rec
    weeds = []
    self.weed_out_gaussians = lambda: weeds.append(True)

    draws = []
    orig = torch.rand_like

    def rand_like(x, *a, **k):
        r = orig(x, *a, **k)
        draws.append(r.clone())
        return r
    torch.manual_seed(seed)
    torch.rand_like = rand_like
    try:
        ns["add_new_gaussians"](self, 0)
    finally:
        torch.rand_like = orig
    assert len(rec.calls) == 1 and len(weeds) == 1
    ext, mask = rec.calls[0]
    return dict(warm=warm, H=H, W=W, f=f, args=ARGS, image=image, point_map=xyzm, conf=conf, R=R, t=t, Rt=Rt,
                exposure=exposure, approx_centre=-R.T @ t, raw_render=raw, params=init_params, uniforms=draws,
                ext=ext, valid_gs_mask=mask, cls_after=self.cls_id.clone(), n_renders=len(renders),
                disc=self.disc_kernel.clone())


def main():
    ref_dir = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    cases = [make_case(ref_dir, 11, True), make_case(ref_dir, 12, False)]
    for c in cases:                       # plain zero fills: only their shapes are kept
        c["fill_shapes"] = {}
        for k in ("f_rest", "local_feat", "global_feat"):
            assert not c["ext"][k].any()
            c["fill_shapes"][k] = tuple(c["ext"].pop(k).shape)
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "densify_small.pt")
    torch.save(dict(cases=cases), out)
    for c in cases:
        print(f"warm={c['warm']}: rows={c['ext']['xyz'].shape[0]} voxels={c['fill_shapes']['global_feat'][0]} "
              f"renders={c['n_renders']} kept={int(c['valid_gs_mask'].sum())}/{c['valid_gs_mask'].numel()}")
    print(f"wrote {out} ({os.path.getsize(out) // 1024} KB)")


if __name__ == "__main__":
    main()

"""Writes tests/golden/reanchor_small.pt by running the reference's OWN map update of a SLAM key frame on the CPU.

The reference modules cannot be imported here (pypose, kornia, e3nn and plyfile are not installed), so the statements are
extracted with ``ast`` and executed against stubs:
  * run_system.py: the body of ``if is_slam_keyframe and frame_id > 0:`` (the mapper key-frame pose loop);
  * Reconstruct/scene/keyframe.py: ``Keyframe.get_R / get_t / get_Rt / set_Rt``, bound to a stub key frame;
  * Reconstruct/utils.py: ``sixD2mtx`` and ``update_gaussians``;
  * Reconstruct/scene/scene_models/h3dgsv3.py: ``SceneModel.rigid_transform_gs``, bound to a stub scene;
  * ``pp`` is a small LieTensor class over oracle.track_ref's pypose stand-in, and ``kornia.geometry.conversions`` is
    oracle.reanchor_ref's restatement of the two conversions.
Only inputs and outputs are saved, no reference source.

    python tests/golden/make_reanchor_golden.py [/path/to/reference]
"""
import ast
import os
import sys
import textwrap
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import reanchor_ref, track_ref  # noqa: E402

K_SLAM, K_MAP, N_GS = 4, 6, 500


class LieTensor:
    """What the block uses of a pypose Sim3 / SE3 LieTensor of shape [1, 8] / [1, 7]."""

    def __init__(self, x, kind):
        self.kind = kind
        self.x8 = x.reshape(-1)[:7] if kind == "SE3" else x.reshape(8)
        if kind == "SE3":
            self.x8 = reanchor_ref.SE3(self.x8)

    @property
    def data(self):
        return (self.x8[:7] if self.kind == "SE3" else self.x8).reshape(1, -1)

    def to(self, *a, **k):
        return self

    def mul(self, other):
        return LieTensor(track_ref.mul(self.x8, other.x8), self.kind)

    def Inv(self):
        return LieTensor(track_ref.inv(self.x8), self.kind)

    def matrix(self):
        return track_ref.matrix(self.x8)[None]


pp = types.SimpleNamespace(SE3=lambda x: LieTensor(x, "SE3"),
                           quat2unit=lambda T: LieTensor(track_ref.quat2unit(T.x8), T.kind))
kornia = types.SimpleNamespace(geometry=types.SimpleNamespace(conversions=types.SimpleNamespace(
    quaternion_to_rotation_matrix=reanchor_ref.quat2mat, rotation_matrix_to_quaternion=reanchor_ref.mat2quat)))


def _functions(path, names, cls=None):
    src = open(path).read()
    tree = ast.parse(src)
    scope = tree
    if cls is not None:
        scope = next(n for n in ast.walk(tree) if isinstance(n, ast.ClassDef) and n.name == cls)
    out = {}
    for node in ast.walk(scope):
        if isinstance(node, ast.FunctionDef) and node.name in names and node.name not in out:
            out[node.name] = textwrap.dedent(ast.get_source_segment(src, node))
    assert set(out) == set(names), (path, set(names) - set(out))
    return out


def _statements(path):
    """The source lines of the block's body, dedented as one piece."""
    src = open(path).read()
    for node in ast.walk(ast.parse(src)):
        if isinstance(node, ast.If) and ast.get_source_segment(src, node.test) == "is_slam_keyframe and frame_id > 0":
            lines = src.splitlines()
            first, last = node.body[0].lineno, node.body[-1].end_lineno
            return textwrap.dedent("\n".join(lines[first - 1:last]))
    raise AssertionError("the `if is_slam_keyframe and frame_id > 0:` block was not found")


def make_inputs(seed):
    g = torch.Generator().manual_seed(seed)
    # Backend Sim(3) table: scale != 1, quaternions not of unit norm
    slam = torch.zeros(K_SLAM, 8)
    slam[:, :3] = torch.randn(K_SLAM, 3, generator=g)
    q = torch.randn(K_SLAM, 4, generator=g)
    slam[:, 3:7] = q / q.norm(dim=-1, keepdim=True) * (1.0 + 0.05 * torch.randn(K_SLAM, 1, generator=g))
    slam[:, 7] = 0.7 + 0.8 * torch.rand(K_SLAM, generator=g)
    last = torch.tensor([0, 0, 1, 2, 2, 3])
    is_slam = torch.tensor([True, False, True, False, True, False])
    rel = torch.zeros(K_MAP, 8)
    rel[:, :3] = 0.3 * torch.randn(K_MAP, 3, generator=g)
    q = torch.randn(K_MAP, 4, generator=g) * 0.1
    q[:, 3] += 1.0
    rel[:, 3:7] = q / q.norm(dim=-1, keepdim=True) * (1.0 + 0.02 * torch.randn(K_MAP, 1, generator=g))
    rel[:, 7] = 0.9 + 0.2 * torch.rand(K_MAP, generator=g)
    # current mapper poses: slightly non-orthonormal 6-D rotations
    qa = torch.randn(K_MAP, 4, generator=g)
    R = reanchor_ref.quat2mat(qa)
    rW2C = (R[:, :, :2] + 0.01 * torch.randn(K_MAP, 3, 2, generator=g)).contiguous()
    tW2C = torch.randn(K_MAP, 3, generator=g)
    # Gaussians: random rotations reach every mat2quat branch (main() checks it), plus a zero quaternion
    ids = torch.randint(0, K_MAP, (N_GS, 1), generator=g)
    xyz = 2.0 * torch.randn(N_GS, 3, generator=g)
    rot = torch.randn(N_GS, 4, generator=g) * (0.5 + torch.rand(N_GS, 1, generator=g))
    rot[0] = 0.0
    return dict(slam_T_WC=slam, last_keyframe_index=last, is_slam_keyframe=is_slam, T_CkCf=rel, rW2C=rW2C, tW2C=tW2C,
                id=ids, xyz=xyz, rotation=rot)


def run_reference(ref_dir, inp):
    u = _functions(os.path.join(ref_dir, "Reconstruct", "utils.py"), {"sixD2mtx", "update_gaussians"})
    kf = _functions(os.path.join(ref_dir, "Reconstruct", "scene", "keyframe.py"), {"get_R", "get_t", "get_Rt", "set_Rt"},
                    cls="Keyframe")
    h3 = _functions(os.path.join(ref_dir, "Reconstruct", "scene", "scene_models", "h3dgsv3.py"), {"rigid_transform_gs"})
    block = _statements(os.path.join(ref_dir, "run_system.py"))
    ns = dict(torch=torch, kornia=kornia, pp=pp)
    for name in ("sixD2mtx", "update_gaussians"):
        exec(u[name], ns)
    for name in ("get_R", "get_t", "get_Rt", "set_Rt"):
        exec(kf[name], ns)
    exec(h3["rigid_transform_gs"], ns)

    class Frame:
        get_R, get_t, get_Rt, set_Rt = ns["get_R"], ns["get_t"], ns["get_Rt"], ns["set_Rt"]

    frames = []
    for k in range(K_MAP):
        f = Frame()
        f.rW2C = torch.nn.Parameter(inp["rW2C"][k].clone())
        f.tW2C = torch.nn.Parameter(inp["tW2C"][k].clone())
        f.idepth_pyr = [torch.zeros(1)]
        f.is_slam_keyframe = bool(inp["is_slam_keyframe"][k])
        f.last_keyframe_index = int(inp["last_keyframe_index"][k])
        f.T_CkCf = LieTensor(inp["T_CkCf"][k][None], "Sim3")
        frames.append(f)
    backend = [types.SimpleNamespace(T_WC=LieTensor(inp["slam_T_WC"][i][None], "Sim3")) for i in range(K_SLAM)]

    class Scene:
        rigid_transform_gs = ns["rigid_transform_gs"]
        id = property(lambda s: s.gaussian_params["id"]["val"])
        xyz = property(lambda s: s.gaussian_params["xyz"]["val"])
        rotation = property(lambda s: s.gaussian_params["rotation"]["val"])

    scene = Scene()
    scene.keyframes = frames
    scene.gaussian_params = {k: {"val": inp[k].clone()} for k in ("id", "xyz", "rotation")}
    related = {}
    for k in range(K_MAP):
        related.setdefault(int(inp["last_keyframe_index"][k]), []).append(k)
    captured = {}
    orig = Scene.rigid_transform_gs

    def capture(self, old_c2ws, new_c2ws, cam_centres):
        captured.update(old_c2ws=old_c2ws.clone(), new_c2ws=new_c2ws.clone(), cam_centres=cam_centres.clone())
        return orig(self, old_c2ws, new_c2ws, cam_centres)
    Scene.rigid_transform_gs = capture
    env = dict(ns, scene_model=scene, related_frames=related, keyframes=backend, device_mapper="cpu")
    exec(block, env)
    assert captured, "rigid_transform_gs was not called"
    return dict(rW2C=torch.stack([f.rW2C.detach() for f in frames]), tW2C=torch.stack([f.tW2C.detach() for f in frames]),
                approx_centres=torch.stack([f.approx_centre.detach() for f in frames]), **captured,
                xyz=scene.gaussian_params["xyz"]["val"], rotation=scene.gaussian_params["rotation"]["val"],
                cam_centres_scene=scene.cam_centres)


def main():
    ref_dir = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    inp = make_inputs(7)
    out = run_reference(ref_dir, inp)
    _, _, mats = reanchor_ref.rigid_transform_gs(inp["id"], inp["xyz"], inp["rotation"], out["old_c2ws"], out["new_c2ws"])
    branches, _ = reanchor_ref.mat2quat_branch(mats)
    counts = torch.bincount(branches.reshape(-1), minlength=4).tolist()
    assert all(c > 0 for c in counts), counts
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reanchor_small.pt")
    out = {k: v.detach().clone() for k, v in out.items()}
    torch.save(dict(inputs=inp, outputs=out), path)
    print(f"mat2quat branches {counts}; wrote {path} ({os.path.getsize(path) // 1024} KB)")


if __name__ == "__main__":
    main()

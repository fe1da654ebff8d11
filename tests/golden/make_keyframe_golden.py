"""Writes tests/golden/keyframe_small.pt by running the reference's OWN key-frame hand-off on the CPU.

The reference modules cannot be imported here (pypose, lietorch and the MASt3R model are not installed), so the statements
are extracted with ``ast`` and executed against stubs:
  * VSLAM/Backend.py: ``Backend.prepare_for_mapper`` and ``Backend.compute_dense_point``, bound to a stub Backend whose
    ``states.msg2Mapper`` captures the message;
  * VSLAM/mast3r_slam/geometry.py: ``constrain_points_to_ray``, ``backproject`` and ``get_pixel_coords``;
  * run_system.py: the statements from ``T_CkC = keyframe_map_dict["T_CkC"]`` to the ``Keyframe(...)`` construction;
  * Reconstruct/scene/keyframe.py: ``Keyframe.__init__``, with a stub ``BaseAdam`` that records its parameter groups;
  * ``pp`` is a small LieTensor class over oracle.track_ref's pypose stand-in.
Three cases: the first key frame (``C / N`` straddling 1.5), a general key frame (Sim(3) scale != 1, non-unit quaternions,
zero and negative depths, out-of-order matches, odd mapper size) and one whose residuals are exactly 3 px.  Only inputs and
outputs are saved, no reference source.

    python tests/golden/make_keyframe_golden.py [/path/to/reference]
"""
import ast
import os
import sys
import textwrap
import types
from argparse import Namespace

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import track_ref  # noqa: E402

ARGS = dict(pyr_levels=3, depth_loss_weight_init=1.0, depth_loss_weight_decay=0.95, lr_poses=1e-3, lr_exposure=5e-4)


class LieTensor:
    """What the blocks use of a pypose Sim3 / SE3 LieTensor of shape [1, 8] / [1, 7]."""

    def __init__(self, x, kind):
        self.kind = kind
        x = x.reshape(-1)
        self.x8 = torch.cat([x[:7], torch.ones(1, dtype=x.dtype)]) if kind == "SE3" else x[:8].clone()

    @property
    def data(self):
        return (self.x8[:7] if self.kind == "SE3" else self.x8).reshape(1, -1)

    def to(self, *a, **k):
        return self

    def cpu(self):
        return self

    def mul(self, other):
        return LieTensor(track_ref.mul(self.x8, other.x8), self.kind)

    def Inv(self):
        return LieTensor(track_ref.inv(self.x8), self.kind)

    def Act(self, X):
        return track_ref.act(self.x8, X.reshape(-1, 3)).reshape(X.shape)

    def matrix(self):
        return track_ref.matrix(self.x8)[None]


pp = types.SimpleNamespace(Sim3=lambda x: LieTensor(x, "Sim3"), SE3=lambda x: LieTensor(x, "SE3"),
                           quat2unit=lambda T: LieTensor(track_ref.quat2unit(T.x8), T.kind))


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
    # drop decorators (torch.no_grad): the blocks run under no_grad here anyway
    return {k: "\n".join(l for l in v.splitlines() if not l.lstrip().startswith("@")) for k, v in out.items()}


def _statements(path):
    """run_system.py: from ``T_CkC = keyframe_map_dict["T_CkC"]`` to the statement that builds ``keyframe_map``."""
    src = open(path).read()
    for node in ast.walk(ast.parse(src)):
        body = getattr(node, "body", None)
        if not isinstance(body, list):
            continue
        segs = [ast.get_source_segment(src, s) or "" for s in body]
        starts = [i for i, s in enumerate(segs) if s.startswith('T_CkC = keyframe_map_dict["T_CkC"]')]
        ends = [i for i, s in enumerate(segs) if s.startswith("keyframe_map = Keyframe(")]
        if starts and ends:
            lines = src.splitlines()
            return textwrap.dedent("\n".join(lines[body[starts[0]].lineno - 1:body[ends[0]].end_lineno]))
    raise AssertionError("the mapper key-frame construction was not found")


def make_case(kind, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "exact3":
        Hs, Ws, H, W = 6, 8, 12, 16
        K = torch.eye(3)
    else:
        Hs, Ws, H, W = 24, 32, 37, 53
        K = torch.tensor([[30.0, 0.0, 15.3], [0.0, 29.0, 11.7], [0.0, 0.0, 1.0]])
    HW = Hs * Ws
    X = torch.randn(HW, 3, generator=g)
    X[:, 2] = 0.5 + 3.0 * torch.rand(HW, generator=g)
    C = 1.5 * 3 + torch.randn(HW, 1, generator=g)          # N = 3: C / N straddles 1.5
    N = 3
    if kind == "exact3":
        X[:, 2] = 2.0
        T_WC = torch.tensor([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0, 1.0])
        last = T_WC.clone()
        idx = torch.arange(HW)
        cols = idx % Ws
        idx = torch.where(cols >= 3, idx - 3, idx)            # matched 3 px to the left: residual exactly 3
    else:
        X[:5, 2] = 0.0                                        # zero depths
        X[5:9, 2] = -torch.rand(4, generator=g) - 0.1         # negative depths
        q = torch.randn(4, generator=g)
        T_WC = torch.cat([torch.randn(3, generator=g), q / q.norm() * 1.07, torch.tensor([1.3])])
        q = torch.randn(4, generator=g) * 0.05 + torch.tensor([0.0, 0.0, 0.0, 1.0])
        rel = torch.cat([0.2 * torch.randn(3, generator=g), q / q.norm() * 0.98, torch.tensor([0.9])])
        last = track_ref.mul(T_WC, track_ref.inv(rel))
        idx = torch.randperm(HW, generator=g)
    image = torch.rand(H, W, 3, generator=g).permute(2, 0, 1)     # to_map: permute(2,0,1) of an HWC array
    return dict(kind=kind, H_slam=Hs, W_slam=Ws, K=K, X_canon=X, C=C, N=N, T_WC=T_WC, last_T_WC=last,
                idx_k2l=idx[None], image=image, mapper_index=1 if kind != "first" else 0)


def run_reference(ref_dir, inp):
    be = _functions(os.path.join(ref_dir, "VSLAM", "Backend.py"), {"prepare_for_mapper", "compute_dense_point"},
                    cls="Backend")
    geo = _functions(os.path.join(ref_dir, "VSLAM", "mast3r_slam", "geometry.py"),
                     {"constrain_points_to_ray", "backproject", "get_pixel_coords"})
    kf = _functions(os.path.join(ref_dir, "Reconstruct", "scene", "keyframe.py"), {"__init__"}, cls="Keyframe")
    block = _statements(os.path.join(ref_dir, "run_system.py"))
    ns = dict(torch=torch, pp=pp, F=F, Namespace=Namespace, Keyframe=object)   # __init__'s annotations are evaluated
    for src in geo.values():
        exec(src, ns)
    for src in be.values():
        exec(src, ns)
    exec(kf["__init__"], ns)

    class BaseAdam:
        def __init__(self, params, betas):
            self.params, self.betas = params, betas

    ns["BaseAdam"] = BaseAdam

    class Keyframe:
        __init__ = ns["__init__"]
        device = property(lambda s: s.image_pyr[0].device)

    sent = []
    Hs, Ws = inp["H_slam"], inp["W_slam"]
    backend = types.SimpleNamespace(config={"use_calib": True}, K_slam=inp["K"], H_slam=Hs, W_slam=Ws,
                                    states=types.SimpleNamespace(msg2Mapper=sent.append))
    frame = types.SimpleNamespace(X_canon=inp["X_canon"], C=inp["C"], N=inp["N"], img=torch.zeros(3, Hs, Ws), frame_id=5,
                                  T_WC=LieTensor(inp["T_WC"], "Sim3"))
    frame.get_average_conf = lambda: frame.C / frame.N
    last = None if inp["kind"] == "first" else types.SimpleNamespace(T_WC=LieTensor(inp["last_T_WC"], "Sim3"), frame_id=2)
    _bind(backend, ns).prepare_for_mapper(frame, last, 0 if last is None else 1, None if last is None else inp["idx_k2l"])
    msg = sent[0]
    image = inp["image"]
    env = dict(ns, Keyframe=Keyframe, keyframe_map_dict=msg, device_mapper="cpu", frame_id=msg["frame_id"],
               last_keyframe_index=msg["last_keyframe_index"], last_keyframe_frame_id=msg["last_keyframe_frame_id"],
               dataset=_Dataset(image), K_map=torch.tensor([[40.0, 0.0, 26.0], [0.0, 40.0, 18.0], [0.0, 0.0, 1.0]]),
               args=Namespace(**ARGS), mapper_index=inp["mapper_index"])
    exec(block, env)
    k = env["keyframe_map"]
    groups = {name: float(p["lr"]) for name, p in k.optimizer.params.items()}
    return dict(densePoint=msg["densePoint"], T_CkC=msg["T_CkC"].data.reshape(8) if msg["T_CkC"] is not None else None,
                T_WC=msg["T_WC"].reshape(8), image_pyr=[t.contiguous() for t in k.image_pyr], idepth_pyr=k.idepth_pyr,
                point_map=k.point_map.contiguous(), conf=k.mono_depth_conf.contiguous(), rW2C=k.rW2C.detach(),
                tW2C=k.tW2C.detach(), approx_centre=k.approx_centre, exposure=k.exposure.detach(), lr=groups,
                betas=k.optimizer.betas)


def _bind(backend, ns):
    """The stub Backend with the extracted methods bound to it."""
    for name in ("prepare_for_mapper", "compute_dense_point"):
        setattr(backend, name, types.MethodType(ns[name], backend))
    return backend


class _Dataset:
    def __init__(self, image):
        self.transform = types.SimpleNamespace(to_map=lambda img, device: image)

    def __getitem__(self, i):
        return None, {"name": f"frame_{i}.png"}


def main():
    ref_dir = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    cases = []
    for kind, seed in (("first", 1), ("general", 2), ("exact3", 3)):
        inp = make_case(kind, seed)
        cases.append(dict(inputs=inp, outputs=run_reference(ref_dir, inp)))
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "keyframe_small.pt")
    torch.save(dict(args=ARGS, cases=cases), path)
    print(f"wrote {path} ({os.path.getsize(path) // 1024} KB)")


if __name__ == "__main__":
    main()

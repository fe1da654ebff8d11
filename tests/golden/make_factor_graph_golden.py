"""Writes tests/golden/factor_graph_small.pt by running the reference's OWN ``FactorGraph`` on the CPU.

The reference modules cannot be imported here (pypose, lietorch, the MASt3R model and the Gauss-Newton extension are not
installed), so the class is extracted from VSLAM/mast3r_slam/global_opt.py with ``ast`` and executed against stubs:
  * ``constrain_points_to_ray``, ``backproject`` and ``get_pixel_coords``: the reference's own, from geometry.py;
  * ``pp``: a small LieTensor class over oracle.track_ref's pypose stand-in;
  * ``frames``: oracle.factor_graph_ref.Keyframes, 8 key frames of 24x32 with non-unit quaternions and Sim(3) scale != 1;
  * ``mast3r_match_symmetric``: returns seeded matches queued by the script below (recorded in the fixture);
  * ``mast3r_slam_backends``: records its arguments and moves pose rows >= 1 by a fixed delta.
The script covers consecutive and retrieval edges, match counts one above and one below ``min_match_frac``, a low-match
consecutive edge that is kept, a rejected and an accepted relocalisation with ``pop_last``, fusions and pose-only changes
between solves, and both solve modes.  Only inputs and outputs are saved, no reference source.

The file is kept small without losing a bit: the inputs are drawn on grids that small integers hold exactly (points in
1/256, confidences and match scores in 1/64; ``decode`` in tests/test_factor_graph.py restores them), pixel indices are
stored as int16, the graph as the rows each call appended (their indices and match masks as the accepted candidates'
numbers), and each solve's point maps and confidences as the key-frame
rows that differ from the last solve of the same mode.

    python tests/golden/make_factor_graph_golden.py [/path/to/reference]
"""
import ast
import os
import sys
import textwrap
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import track_ref  # noqa: E402
from oracle.factor_graph_ref import Keyframes  # noqa: E402

H, W = 24, 32
N_PIX = H * W
CONFIG = {"local_opt": dict(pin=1, window_size=1000000, C_conf=0.0, Q_conf=1.5, min_match_frac=0.1, pixel_border=-10,
                            depth_eps=1e-6, max_iters=10, sigma_ray=0.003, sigma_dist=10.0, sigma_pixel=1.0, sigma_depth=10.0,
                            delta_norm=1e-8)}
K = torch.tensor([[30.0, 0.0, 15.3], [0.0, 29.0, 11.7], [0.0, 0.0, 1.0]])
GRAPH_KEYS = ("ii", "jj", "idx_ii2jj", "idx_jj2ii", "valid_match_j", "valid_match_i", "Q_ii2jj", "Q_jj2ii")
DELTA = torch.tensor([0.01, -0.02, 0.03, 0.001, -0.002, 0.0015, 0.0005, 0.004])


class LieTensor:
    def __init__(self, x):
        self.data = x

    def __getitem__(self, k):
        return LieTensor(self.data[k])

    def to(self, *a, **k):
        return self


pp = types.SimpleNamespace(Sim3=LieTensor, quat2unit=lambda T: LieTensor(track_ref.quat2unit(T.data)))


class RefFrame:
    def __init__(self, f):
        self.img, self.X_canon, self.C, self.N = f.img, f.X_canon, f.C, f.N
        self.T_WC = LieTensor(f.T_WC)

    def to(self, device):
        return self

    def get_average_conf(self):
        return self.C / self.N


class RefKeyframes(Keyframes):
    def __getitem__(self, idx):
        return RefFrame(super().__getitem__(idx))

    def update_T_WCs(self, T_WCs, idx):
        self.T_WC[idx] = T_WCs.data


class Backend:
    def __init__(self):
        self.calls = []

    def _record(self, mode, args):
        self.calls.append(dict(mode=mode, args=[a.clone() if isinstance(a, torch.Tensor) else a for a in args]))
        args[0][1:] += DELTA

    def gauss_newton_rays(self, *args):
        self._record("rays", args)

    def gauss_newton_calib(self, *args):
        self._record("calib", args)


def _source(path, names, cls=None):
    src = open(path).read()
    tree = ast.parse(src)
    out = {}
    for node in ast.walk(tree):
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)) and node.name in names and node.name not in out:
            out[node.name] = textwrap.dedent(ast.get_source_segment(src, node))
    assert set(out) == set(names), (path, set(names) - set(out))
    return "\n\n".join(out[k] for k in names)


X_SCALE, C_SCALE, Q_SCALE = 256.0, 64.0, 64.0


def points(g):
    """x, y ~ N(0, 1) and z in [0.5, 3.5], in steps of 1/256."""
    X = torch.round(torch.randn(N_PIX, 3, generator=g).clamp(-100, 100) * X_SCALE)
    X[:, 2] = torch.randint(128, 897, (N_PIX,), generator=g).float()
    return X / X_SCALE


def confidences(g):
    """[1, 3] in steps of 1/64."""
    return torch.randint(64, 193, (N_PIX, 1), generator=g).float() / C_SCALE


def make_matches(g, kinds):
    """kinds: "rand" or (count_j, count_i) exact valid counts with every Q = 2 (Qj = Qi = 2 > Q_conf).  Q in [0.5, 3] in
    steps of 1/64."""
    B = len(kinds)
    idx_i2j = torch.stack([torch.randperm(N_PIX, generator=g) for _ in range(B)])
    idx_j2i = torch.stack([torch.randperm(N_PIX, generator=g) for _ in range(B)])
    vj = torch.rand(B, N_PIX, 1, generator=g) < 0.6
    vi = torch.rand(B, N_PIX, 1, generator=g) < 0.6
    Qs = [torch.randint(32, 193, (B, N_PIX, 1), generator=g).float() / Q_SCALE for _ in range(4)]
    for b, k in enumerate(kinds):
        if k == "rand":
            continue
        for q in Qs:
            q[b] = 2.0
        for v, c in ((vj, k[0]), (vi, k[1])):
            v[b] = False
            v[b, torch.randperm(N_PIX, generator=g)[:c]] = True
    return (idx_i2j, idx_j2i, vj, vi, *Qs)


def new_frame(g, k):
    q = torch.randn(4, generator=g)
    T = torch.cat([torch.randn(3, generator=g), q / q.norm() * (0.9 + 0.2 * torch.rand(1, generator=g)),
                   0.8 + 0.4 * torch.rand(1, generator=g)])
    X, C = points(g), confidences(g)
    return dict(dataset_idx=10 * k + 3, T_WC=T, X=X, C=C, N=1 + k % 3, N_updates=1 + k % 3)


def script(g):
    """The event list; the match counts sit one above (77) and one below (76) 0.1 * 768 = 76.8, and 0.3 * 768 = 230.4."""
    ev = []
    for k in range(2):
        ev.append(("append", new_frame(g, k)))
    ev.append(("add", [0], [1], 0.1, False, ["rand"]))
    ev.append(("solve", "calib"))
    ev.append(("append", new_frame(g, 2)))
    ev.append(("add", [1, 0], [2, 2], 0.1, False, [(10, 12), (77, 300)]))       # low-match consecutive kept; 77 kept
    ev.append(("solve", "calib"))
    ev.append(("append", new_frame(g, 3)))
    ev.append(("add", [2, 0, 1], [3, 3, 3], 0.1, False, ["rand", (300, 76), (77, 77)]))   # 76 rejected
    ev.append(("fuse", 1))
    ev.append(("pose", 2))
    ev.append(("solve", "calib"))
    ev.append(("append", new_frame(g, 4)))
    ev.append(("add", [3, 1], [4, 4], 0.1, False, ["rand", "rand"]))
    ev.append(("solve", "rays"))
    ev.append(("append", new_frame(g, 5)))
    ev.append(("add", [1, 2], [5, 5], 0.3, True, [(400, 400), (230, 500)]))     # relocalisation rejected
    ev.append(("pop_last",))
    ev.append(("append", new_frame(g, 6)))
    ev.append(("add", [0, 3], [5, 5], 0.3, True, [(231, 231), (500, 400)]))     # relocalisation accepted
    ev.append(("reloc_pose", 5, 0))
    ev.append(("fuse", 4))
    ev.append(("solve", "calib"))
    ev.append(("append", new_frame(g, 7)))
    ev.append(("add", [5], [6], 0.1, False, ["rand"]))
    ev.append(("append", new_frame(g, 8)))
    ev.append(("add", [6, 2, 0], [7, 7, 7], 0.1, False, ["rand", "rand", (76, 76)]))
    ev.append(("fuse", 6))
    ev.append(("solve", "rays"))
    ev.append(("solve", "calib"))
    return ev


def to_int(t, scale, dtype):
    q = t * scale
    assert torch.equal(q, torch.round(q)) and q.min() >= torch.iinfo(dtype).min and q.max() <= torch.iinfo(dtype).max
    return q.to(dtype)


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    g = torch.Generator().manual_seed(7)
    queue = []
    backend = Backend()
    ns = dict(torch=torch, pp=pp, SharedKeyframes=Keyframes, mast3r_slam_backends=backend,
              mast3r_match_symmetric=lambda *a: queue.pop(0))
    exec(_source(os.path.join(ref, "VSLAM/mast3r_slam/geometry.py"),
                 ["constrain_points_to_ray", "backproject", "get_pixel_coords"]), ns)
    exec(_source(os.path.join(ref, "VSLAM/mast3r_slam/global_opt.py"), ["FactorGraph"]), ns)
    frames = RefKeyframes(H, W, buffer=12)
    fg = ns["FactorGraph"](CONFIG, None, frames, K=K, device="cpu")
    emb = {k: [torch.zeros(1, 2), torch.zeros(1, 2)] for k in range(12)}
    out, n_edges, last_rows = [], 0, {}
    for e in script(g):
        rec = dict(op=e[0])
        if e[0] == "append":
            rec["frame"] = e[1]
            frames.append(**e[1])
        elif e[0] == "pop_last":
            frames.pop_last()
        elif e[0] == "fuse":
            X, C = points(g), confidences(g)
            rec.update(idx=e[1], X=X, C=C)
            frames.update_pointmap(e[1], X, C)
        elif e[0] == "pose":
            T = frames.T_WC[e[1], 0] + 0.05 * torch.randn(8, generator=g)
            rec.update(idx=e[1], T=T)
            frames.T_WC[e[1], 0] = T
        elif e[0] == "reloc_pose":
            rec.update(idx=e[1], src=e[2])
            frames.T_WC[e[1]] = frames.T_WC[e[2]].clone()
        elif e[0] == "add":
            _, ii, jj, frac, reloc, kinds = e
            m = make_matches(g, kinds)
            queue.append(m)
            res = fg.add_factors(ii, jj, frac, emb, is_reloc=reloc)
            rec.update(ii=ii, jj=jj, min_match_frac=frac, is_reloc=reloc, matches=m, result=bool(res))
            # the graph only grows: keep the rows this call appended.  Their indices and match masks are the accepted
            # candidates' rows of the matches: keep which candidates those are
            new = {k: getattr(fg, k)[n_edges:].clone() for k in GRAPH_KEYS}
            picked = [b for b in range(len(ii)) if any(ii[b] == int(a) and jj[b] == int(c) for a, c in zip(new["ii"], new["jj"]))]
            for k, src in (("idx_ii2jj", 0), ("idx_jj2ii", 1), ("valid_match_j", 2), ("valid_match_i", 3)):
                assert torch.equal(new.pop(k), m[src][picked])
            rec["graph"] = dict(new, picked=torch.tensor(picked, dtype=torch.int64))
            n_edges = fg.ii.numel()
        elif e[0] == "solve":
            n0 = len(backend.calls)
            (fg.solve_GN_calib if e[1] == "calib" else fg.solve_GN_rays)()
            call = None
            if len(backend.calls) > n0:
                # the edge arguments are prep_two_way_edges() of the recorded graph: keep the rest
                a = backend.calls[n0]["args"]
                two_way = fg.prep_two_way_edges()
                k = 3 if e[1] == "rays" else 4
                assert all(torch.equal(x, y) for x, y in zip(a[k:k + 5], two_way))
                # point maps and confidences: only the key frames whose rows changed since the last solve of this mode
                unique = torch.unique(torch.cat([fg.ii, fg.jj]), sorted=True).tolist()
                seen = last_rows.setdefault(e[1], {})
                rows = {}
                for r, kf in enumerate(unique):
                    x, c = a[1][r], a[2][r]
                    if kf not in seen or not (torch.equal(seen[kf][0], x) and torch.equal(seen[kf][1], c)):
                        rows[kf] = seen[kf] = (x.clone(), c.clone())
                call = dict(poses=a[0], unique=unique, rows=rows, scalars=a[k + 5:])
            rec.update(mode=e[1], call=call, T_WC=frames.T_WC.clone())
        out.append(rec)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "factor_graph_small.pt")
    for r in out:
        if "frame" in r:
            r["frame"] = dict(r["frame"], X=to_int(r["frame"]["X"], X_SCALE, torch.int16),
                              C=to_int(r["frame"]["C"], C_SCALE, torch.uint8))
        if r["op"] == "fuse":
            r.update(X=to_int(r["X"], X_SCALE, torch.int16), C=to_int(r["C"], C_SCALE, torch.uint8))
        if "matches" in r:
            m = r["matches"]
            r["matches"] = tuple(t.to(torch.int16) for t in m[:2]) + tuple(m[2:4]) + tuple(
                to_int(t, Q_SCALE, torch.uint8) for t in m[4:])
    torch.save(dict(config=CONFIG, K=K, delta=DELTA, h=H, w=W, buffer=12, scales=dict(X=X_SCALE, C=C_SCALE, Q=Q_SCALE),
                    events=out), path)
    print(path, sum(1 for r in out if r["op"] == "solve"), "solves,", [r["result"] for r in out if r["op"] == "add"])


if __name__ == "__main__":
    main()

"""The Backend's factor graph (artdeco_b200.factor_graph, csrc/factor_graph.cu) against the reference's own FactorGraph
(tests/golden/factor_graph_small.pt, made by make_factor_graph_golden.py) and against oracle/factor_graph_ref.py on the
device: gating, the two-way edge table, the key-frame mirror, the pose gather and write-back and the solve."""
import ctypes
import os

import pytest
import torch

from oracle import factor_graph_ref as ref
from oracle import track_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "factor_graph_small.pt")
CFG = {"local_opt": dict(pin=1, window_size=1000000, C_conf=0.0, Q_conf=1.5, min_match_frac=0.1, pixel_border=-10,
                         depth_eps=1e-6, max_iters=10, sigma_ray=0.003, sigma_dist=10.0, sigma_pixel=1.0, sigma_depth=10.0,
                         delta_norm=1e-8)}


def golden():
    """The fixture as the reference saw it (make_factor_graph_golden.py stores it compactly): inputs back in fp32 and
    int64, each call's appended graph rows whole, and each solve's full point maps and confidences."""
    G = torch.load(GOLDEN, weights_only=False)
    sc = G["scales"]
    rows = {}
    for ev in G["events"]:
        if ev["op"] == "append":
            f = ev["frame"]
            ev["frame"] = dict(f, X=f["X"].float() / sc["X"], C=f["C"].float() / sc["C"])
        elif ev["op"] == "fuse":
            ev.update(X=ev["X"].float() / sc["X"], C=ev["C"].float() / sc["C"])
        elif ev["op"] == "add":
            m = ev["matches"]
            ev["matches"] = tuple(t.long() for t in m[:2]) + tuple(m[2:4]) + tuple(t.float() / sc["Q"] for t in m[4:])
            g = ev["graph"]
            p = g.pop("picked")
            for k, src in (("idx_ii2jj", 0), ("idx_jj2ii", 1), ("valid_match_j", 2), ("valid_match_i", 3)):
                g[k] = ev["matches"][src][p]
        elif ev["op"] == "solve" and ev["call"] is not None:
            seen = rows.setdefault(ev["mode"], {})
            seen.update(ev["call"].pop("rows"))
            u = ev["call"].pop("unique")
            ev["call"]["Xs"] = torch.stack([seen[k][0] for k in u])
            ev["call"]["Cs"] = torch.stack([seen[k][1] for k in u])
    return G


def close(a, b, what, tol=1e-6):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    assert a.shape == b.shape, (what, a.shape, b.shape)
    err = ((a - b).abs() / b.abs().clamp_min(1.0)).max().item() if a.numel() else 0.0
    assert err <= tol, f"{what}: max relative error {err:.3e}"


class StubSolve:
    """Records the solve's inputs and moves pose rows >= 1 by the fixture's delta, as the generator's backend does."""

    def __init__(self, delta):
        self.delta, self.calls = delta, []

    def record(self, poses, Xs, Cs, ii, jj, idx, valid, Q, scalars):
        self.calls.append(dict(poses=poses.clone(), Xs=Xs.clone(), Cs=Cs.clone(), ii=ii.clone(), jj=jj.clone(),
                               idx=idx.clone(), valid=valid.clone(), Q=Q.clone(), scalars=list(scalars)))
        poses[1:] += self.delta.to(poses.device)

    # oracle backend interface
    def gauss_newton_rays(self, Twc, Xs, Cs, ii, jj, idx, valid, Q, *s):
        self.record(Twc, Xs, Cs, ii, jj, idx, valid, Q, s)

    def gauss_newton_calib(self, Twc, Xs, Cs, K, ii, jj, idx, valid, Q, *s):
        self.record(Twc, Xs, Cs, ii, jj, idx, valid, Q, s)

    # gn.solve_positions interface (rows interleaved: reordered to the reference's halves)
    def solve_positions(self, mode, Twc, Xs, Cs, K, ii, jj, idx, valid, Q, h, w, border, z_eps, sa, sb, *s):
        order = torch.cat([torch.arange(0, ii.numel(), 2), torch.arange(1, ii.numel(), 2)]).to(ii.device)
        sc = (h, w, border, z_eps, sa, sb) + s if mode == 1 else (sa, sb) + s
        self.record(Twc, Xs, Cs, ii[order], jj[order], idx[order], valid[order], Q[order], sc)


def replay(G, make_graph, frames, solver, check):
    """Runs the fixture's events on `frames` through the graph `make_graph(frames)` and calls check(event, graph, out)."""
    fg = make_graph(frames)
    for ev in G["events"]:
        op, out = ev["op"], None
        if op == "append":
            frames.append(**ev["frame"])
        elif op == "pop_last":
            frames.pop_last()
        elif op == "fuse":
            frames.update_pointmap(ev["idx"], ev["X"], ev["C"])
        elif op == "pose":
            frames.T_WC[ev["idx"], 0] = ev["T"].to(frames.T_WC.device)
        elif op == "reloc_pose":
            frames.T_WC[ev["idx"]] = frames.T_WC[ev["src"]].clone()
        elif op == "add":
            dev = fg.device
            m = [t.to(dev).long() if t.dtype == torch.int16 else t.to(dev) for t in ev["matches"]]
            out = fg.add_matches(ev["ii"], ev["jj"], ev["min_match_frac"], *m, is_reloc=ev["is_reloc"])
        elif op == "solve":
            n0 = len(solver.calls)
            (fg.solve_GN_calib if ev["mode"] == "calib" else fg.solve_GN_rays)()
            out = solver.calls[n0] if len(solver.calls) > n0 else None
        check(ev, fg, out)
    return fg


def check_solve(ev, got, T_WC, graph_edges):
    want = ev["call"]
    assert (got is None) == (want is None)
    if want is not None:
        close(got["poses"], want["poses"], "poses")
        close(got["Xs"], want["Xs"], "Xs")
        close(got["Cs"].reshape(want["Cs"].shape), want["Cs"], "Cs")
        for k, w in zip(("ii", "jj", "idx", "valid"), graph_edges):
            assert torch.equal(got[k].reshape(w.shape).cpu(), w), k
        close(got["Q"].reshape(graph_edges[4].shape), graph_edges[4], "Q")
        assert [float(x) for x in got["scalars"]] == [float(x) for x in want["scalars"]]
    close(T_WC, ev["T_WC"], "T_WC after the write-back")


def accumulate(acc, ev):
    for k, t in ev["graph"].items():
        t = t.long() if k.startswith("idx") else t
        acc[k] = torch.cat([acc[k], t]) if k in acc else t
    return acc


def two_way(acc):
    return (torch.cat((acc["ii"], acc["jj"])), torch.cat((acc["jj"], acc["ii"])),
            torch.cat((acc["idx_ii2jj"], acc["idx_jj2ii"])), torch.cat((acc["valid_match_j"], acc["valid_match_i"])),
            torch.cat((acc["Q_ii2jj"], acc["Q_jj2ii"])))


def test_oracle_reproduces_the_reference_golden():
    G = golden()
    solver = StubSolve(G["delta"])
    acc = {}
    frames = ref.Keyframes(G["h"], G["w"], buffer=G["buffer"])

    def check(ev, fg, out):
        if ev["op"] == "add":
            assert out == ev["result"]
            accumulate(acc, ev)
            for k, w in acc.items():
                got = getattr(fg, k)
                if k.startswith("Q"):
                    close(got, w, k)
                else:
                    assert torch.equal(got, w), k
        elif ev["op"] == "solve":
            check_solve(ev, out, frames.T_WC, two_way(acc))

    replay(G, lambda f: ref.FactorGraphRef(G["config"], f, K=G["K"], backend=solver), frames, solver, check)


def test_golden_covers_the_cases():
    G = golden()
    adds = [e for e in G["events"] if e["op"] == "add"]
    assert [e["result"] for e in adds].count(False) == 1 and any(e["is_reloc"] and e["result"] for e in adds)
    assert {e["mode"] for e in G["events"] if e["op"] == "solve"} == {"calib", "rays"}
    assert any(e["op"] == "pop_last" for e in G["events"]) and any(e["op"] == "fuse" for e in G["events"])
    # one above and one below the threshold, and a kept low-match consecutive edge
    n = G["h"] * G["w"]
    counts = set()
    for e in adds:
        vj, vi = e["matches"][2], e["matches"][3]
        counts |= {int(c) for c in vj.reshape(vj.shape[0], -1).sum(1)} | {int(c) for c in vi.reshape(vi.shape[0], -1).sum(1)}
    assert {76, 77, 10, 230, 231} <= counts and int(0.1 * n) == 76
    assert any(e["graph"]["ii"].numel() and (e["graph"]["ii"] == e["graph"]["jj"] - 1).any() for e in adds)


def test_entry_points_refuse_bad_arguments_before_touching_the_device():
    from artdeco_b200 import _lib
    import artdeco_b200  # noqa: F401  (registers every signature)
    L = _lib.lib()

    def refused(rc, needle):
        msg = L.adb_last_error()
        return rc != 0 and msg is not None and needle in msg.decode()

    fake = 1 << 20
    nb = ctypes.c_size_t(0)
    assert L.adb_fg_gate_workspace_bytes(4, 1000, ctypes.byref(nb)) == 0 and nb.value == 4 * (4 * 4 * 3 + 4)
    assert refused(L.adb_fg_gate_workspace_bytes(0, 1000, ctypes.byref(nb)), "bad size")
    assert refused(L.adb_fg_gate_workspace_bytes(1025, 1000, ctypes.byref(nb)), "bad size")
    assert refused(L.adb_fg_gate_workspace_bytes(4, 1000, None), "null pointer")
    p9 = [fake] * 9
    tail = [fake] * 8

    def gate(B=4, n=1000, E=0, cap=4, ptrs=None, ws=1 << 20, reloc=0, tl=None):
        return L.adb_fg_gate(B, n, E, cap, *(ptrs or p9), 1.5, 0.1, reloc, *(tl or tail), fake, ws, None)

    assert refused(gate(B=0), "bad size")
    assert refused(gate(n=0), "bad size")
    assert refused(gate(E=1, cap=4), "n_edges + B")
    assert refused(gate(E=-1), "bad size")
    assert refused(gate(ptrs=[None] + p9[1:]), "null pointer")
    assert refused(gate(ptrs=p9[:8] + [None]), "null pointer")
    assert refused(gate(tl=tail[:7] + [None]), "null pointer")               # n_bad
    assert L.adb_fg_gate(4, 1000, 0, 4, *p9, 1.5, 0.1, 0, *tail, None, 1 << 20, None) != 0
    assert refused(gate(ws=10), "workspace too small")
    m = [fake] * 6

    def mirror(mode=1, rows=2, h=4, w=5, mrows=8, ids=None, staged=0, X=fake, seen=fake, K=fake):
        return L.adb_fg_mirror_refresh(mode, rows, h, w, mrows, ids, staged, X, fake, fake, fake, fake, seen, fake, K, fake,
                                       fake, None)

    assert refused(mirror(mode=2), "mode")
    assert refused(mirror(h=0), "bad size")
    assert refused(mirror(rows=-1), "bad size")
    assert refused(mirror(X=None), "null pointer")
    assert refused(mirror(K=None), "null pointer")
    assert refused(mirror(rows=9), "more rows than the mirror")
    assert refused(L.adb_fg_mirror_refresh(0, 2, 4, 5, 8, None, 0, *m[:5], fake, None, None, *m[:2], None), "stamps")
    assert L.adb_fg_mirror_refresh(1, 0, 4, 5, 8, None, 0, *m[:5], None, None, fake, fake, fake, None) == 0   # nothing to do
    assert refused(L.adb_fg_pose_gather(5, 4, None, fake, fake, None), "bad size")
    assert refused(L.adb_fg_pose_gather(3, 4, None, None, fake, None), "null pointer")
    assert refused(L.adb_fg_pose_scatter(5, 1, 4, None, fake, fake, None), "bad size")
    assert refused(L.adb_fg_pose_scatter(3, -1, 4, None, fake, fake, None), "bad size")
    assert refused(L.adb_fg_pose_scatter(3, 1, 4, None, fake, None, None), "null pointer")
    assert L.adb_fg_pose_scatter(3, 3, 4, None, fake, fake, None) == 0         # n_unique <= pin: nothing


# ------------------------------------------------------------------ GPU ------------------------------------------------------

@pytest.fixture
def fp32(cuda):
    m, c = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield cuda
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = m, c


@pytest.mark.gpu
@pytest.mark.parametrize("frames_dev", ["cpu", "cuda"])
def test_golden_through_the_device_kernels(fp32, frames_dev, monkeypatch):
    from artdeco_b200 import factor_graph, gn
    G = golden()
    solver = StubSolve(G["delta"])
    monkeypatch.setattr(gn, "solve_positions", solver.solve_positions)
    acc = {}
    frames = ref.Keyframes(G["h"], G["w"], buffer=G["buffer"], device=frames_dev if frames_dev == "cpu" else fp32)

    def check(ev, fg, out):
        if ev["op"] == "add":
            assert out == ev["result"]
            accumulate(acc, ev)
            r = 2 * fg.E
            ii, jj, idx, valid, Q = fg.two_way_edges()
            assert torch.equal(fg.ii.cpu(), acc["ii"]) and torch.equal(fg.jj.cpu(), acc["jj"])
            assert fg.ii_list == acc["ii"].tolist() and fg.jj_list == acc["jj"].tolist()
            assert torch.equal(idx[0:r:2].cpu(), acc["idx_ii2jj"]) and torch.equal(idx[1:r:2].cpu(), acc["idx_jj2ii"])
            assert torch.equal(valid[0:r:2].cpu(), acc["valid_match_j"][..., 0])
            assert torch.equal(valid[1:r:2].cpu(), acc["valid_match_i"][..., 0])
            close(Q[0:r:2], acc["Q_ii2jj"][..., 0], "Qj")
            close(Q[1:r:2], acc["Q_jj2ii"][..., 0], "Qi")
        elif ev["op"] == "solve":
            check_solve(ev, out, frames.T_WC, two_way(acc))

    replay(G, lambda f: factor_graph.FactorGraph(G["config"], None, f, K=G["K"], device=fp32), frames, solver, check)


def matches(B, n, seed, dev, bad=0):
    g = torch.Generator().manual_seed(seed)
    idx_i2j = torch.randint(0, n, (B, n), generator=g)
    idx_j2i = torch.randint(0, n, (B, n), generator=g)
    if bad:
        idx_i2j[0, :bad] = n + torch.arange(bad)
        idx_j2i[-1, -bad:] = -1 - torch.arange(bad)
    vj = torch.rand(B, n, 1, generator=g) < 0.5
    vi = torch.rand(B, n, 1, generator=g) < 0.5
    Q = [0.5 + 2.0 * torch.rand(B, n, 1, generator=g) for _ in range(4)]
    return [t.to(dev) for t in (idx_i2j, idx_j2i, vj, vi, *Q)]


def exact_counts(m, b, cj, ci):
    """Edge b gets exactly cj / ci valid pixels (all Q = 2)."""
    n = m[0].shape[1]
    for q in m[4:]:
        q[b] = 2.0
    for v, c in ((m[2], cj), (m[3], ci)):
        v[b] = False
        v[b, :c] = True


def dev_frames(n_kf, h, w, seed, device):
    g = torch.Generator().manual_seed(seed)
    f = ref.Keyframes(h, w, buffer=n_kf + 2, device=device)
    for k in range(n_kf):
        q = torch.randn(4, generator=g)
        T = torch.cat([torch.randn(3, generator=g), q / q.norm() * 1.05, torch.tensor([1.1])])
        X = torch.randn(h * w, 3, generator=g)
        X[:, 2] = 0.5 + 3.0 * torch.rand(h * w, generator=g)
        f.append(100 + k, T, X, 1.0 + torch.rand(h * w, 1, generator=g), N=1 + k % 3, N_updates=1)
    return f


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 4, 9])
@pytest.mark.parametrize("h,w", [(384, 512), (37, 53)])
def test_gating_matches_the_oracle(fp32, B, h, w):
    from artdeco_b200 import factor_graph
    n = h * w
    thr = int(0.1 * n)                                  # frac(thr) < 0.1 <= frac(thr + 1)
    assert thr / n < 0.1 <= (thr + 1) / n
    frames = dev_frames(2, h, w, 0, fp32)
    for reloc in (False, True):
        for seed in range(3):
            m = matches(B, n, seed + 10 * B, fp32, bad=3 if seed == 1 else 0)
            ii = [3 + b for b in range(B)]
            jj = [20 + b for b in range(B)]
            if B > 1:
                exact_counts(m, 0, thr + 1, thr + 5)     # kept: both at least at the threshold
                exact_counts(m, 1, thr, thr + 50)        # rejected unless consecutive
                if seed == 2:
                    jj[1] = ii[1] + 1                    # consecutive: exempt
            if B == 1 and seed == 2:
                exact_counts(m, 0, thr + 1, thr + 1)
            fg = factor_graph.FactorGraph(CFG, None, frames, device=fp32)
            o = ref.FactorGraphRef(CFG, frames, device=fp32)
            mo = [t.clone() for t in m]
            bad = seed == 1
            if bad:                                      # the oracle cannot read out-of-range indices: give it the pixel
                for t, rows in ((mo[0], (0, slice(0, 3))), (mo[1], (B - 1, slice(n - 3, n)))):
                    t[rows] = 0
                    (mo[2] if t is mo[0] else mo[3])[rows] = False
            got = fg.add_matches(ii, jj, 0.1, *m, is_reloc=reloc)
            want = o.add_matches(ii, jj, 0.1, *mo, is_reloc=reloc)
            assert got == want
            assert torch.equal(fg.last_counts.long(), o.last_counts)
            assert int(fg.n_bad) == (6 if bad else 0)
            assert fg.ii_list == o.ii.tolist() and fg.jj_list == o.jj.tolist()
            r = 2 * fg.E
            _, _, idx, valid, Q = fg.two_way_edges()
            if fg.E:
                keep = o.ii.tolist()
                sel = [ii.index(k) for k in keep]
                for row, src, qa, qb, a in ((0, 0, 4, 6, idx[0:r:2]), (1, 1, 5, 7, idx[1:r:2])):
                    assert torch.equal(a, m[src][sel])
                    gi = m[src][sel].clamp(0, n - 1)
                    Qw = torch.sqrt(torch.gather(m[qa][sel][..., 0], 1, gi) * m[qb][sel][..., 0])
                    inr = (m[src][sel] >= 0) & (m[src][sel] < n)
                    Qg = Q[row:r:2]
                    assert torch.equal(Qg[inr], Qw[inr]) and Qg[~inr].isnan().all()
                    v = m[2 + row][sel][..., 0] & inr                # the matcher's mask, as the reference keeps it
                    assert torch.equal(valid[row:r:2], v)


@pytest.mark.gpu
def test_table_growth_equals_prep_two_way_edges(fp32):
    from artdeco_b200 import factor_graph
    h, w = 24, 40
    n = h * w
    frames = dev_frames(30, h, w, 1, fp32)
    fg = factor_graph.FactorGraph(CFG, None, frames, device=fp32)
    o = ref.FactorGraphRef(CFG, frames, device=fp32)
    caps = set()
    for k in range(1, 30):
        cand_i = sorted({k - 1, max(k - 3, 0), k // 2}) if k > 1 else [0]
        m = matches(len(cand_i), n, 100 + k, fp32)
        if len(cand_i) > 1:
            exact_counts(m, len(cand_i) - 1, 10, 10)        # one rejected retrieval edge now and then
        assert fg.add_matches(cand_i, [k] * len(cand_i), 0.1, *m) == o.add_matches(cand_i, [k] * len(cand_i), 0.1, *m)
        caps.add(fg._cap)
    assert len(caps) >= 4, caps
    ii, jj, idx, valid, Q = fg.two_way_edges()
    want = o.prep_two_way_edges()
    E = fg.E
    order = torch.cat([torch.arange(0, 2 * E, 2), torch.arange(1, 2 * E, 2)]).to(fp32)
    assert torch.equal(ii[order], want[0]) and torch.equal(jj[order], want[1]) and torch.equal(idx[order], want[2])
    assert torch.equal(valid[order], want[3][..., 0]) and torch.equal(Q[order], want[4][..., 0])


def mirror_want(frames, calib, K, n_ids, dev):
    Xs = frames.X[:n_ids].to(dev)
    if calib:
        Xs = torch.stack([track_ref.constrain_points_to_ray(Xs[k], frames.h, frames.w, K.to(dev)) for k in range(n_ids)])
    Cs = torch.stack([frames[k].to(dev).get_average_conf() for k in range(n_ids)])
    return Xs, Cs[..., 0]


@pytest.mark.gpu
@pytest.mark.parametrize("frames_dev", ["cpu", "cuda"])
def test_mirror_follows_the_key_frames(fp32, frames_dev):
    from artdeco_b200 import factor_graph
    h, w = 48, 64
    K = torch.tensor([[50.0, 0.0, 31.7], [0.0, 49.0, 23.2], [0.0, 0.0, 1.0]])
    frames = dev_frames(6, h, w, 2, "cpu")
    if frames_dev == "cuda":
        frames = frames.to(fp32)
    fg = factor_graph.FactorGraph(CFG, None, frames, K=K, device=fp32)
    g = torch.Generator().manual_seed(5)

    def check(calib, n_ids):
        fg.refresh_mirror(factor_graph.CALIB if calib else factor_graph.RAYS, n_ids)
        Xm, Cm = fg.mirror()
        Xw, Cw = mirror_want(frames, calib, K, n_ids, fp32)
        close(Xm[:n_ids], Xw, "Xm")
        close(Cm[:n_ids], Cw, "Cm")

    check(True, 4)
    frames.update_pointmap(1, torch.randn(h * w, 3, generator=g), 1.0 + torch.rand(h * w, 1, generator=g))   # fusion
    check(True, 4)
    frames.T_WC[2, 0, :3] += 1.0                                            # pose only
    check(True, 5)
    frames.pop_last()
    frames.append(999, torch.tensor([0.0, 0, 0, 0, 0, 0, 1, 1]), torch.randn(h * w, 3, generator=g),
                  torch.rand(h * w, 1, generator=g) + 1, N=2, N_updates=1)     # same slot, new dataset_idx
    check(True, 6)
    check(False, 6)                                                          # mode change rebuilds
    frames.update_pointmap(0, torch.randn(h * w, 3, generator=g), 1.0 + torch.rand(h * w, 1, generator=g))
    check(False, 6)
    check(True, 6)


def consistent_frames(n_kf, h, w, seed, device):
    """Key frames that see the same world points at the same pixel index, stored at perturbed poses."""
    g = torch.Generator().manual_seed(seed)
    n = h * w
    Wp = torch.randn(n, 3, generator=g) + torch.tensor([0.0, 0.0, 5.0])
    f = ref.Keyframes(h, w, buffer=n_kf + 2, device=device)
    for k in range(n_kf):
        q = torch.randn(4, generator=g) * 0.05 + torch.tensor([0.0, 0.0, 0.0, 1.0])
        T = torch.cat([0.2 * torch.randn(3, generator=g), q / q.norm(), torch.tensor([1.0 + 0.05 * k])])
        X = track_ref.act(track_ref.inv(T), Wp)
        Ts = T + torch.cat([0.01 * torch.randn(3, generator=g), 0.003 * torch.randn(4, generator=g), torch.zeros(1)])
        f.append(100 + k, T if k == 0 else Ts, X, 1.0 + torch.rand(n, 1, generator=g), N=1, N_updates=1)
    return f


def chain_graph(frames, n_kf, n, seed, dev, skip=None):
    """Consecutive edges plus a retrieval edge to k-2, identity matches; `skip` leaves one key frame out of the graph."""
    from artdeco_b200 import factor_graph
    fg = factor_graph.FactorGraph(CFG, None, frames, K=frames.K_test, device=dev)
    o = ref.FactorGraphRef(CFG, frames, K=frames.K_test.to(dev), device=dev)
    ids = [k for k in range(n_kf) if k != skip]
    for a, b in zip(ids[:-1], ids[1:]):
        cand = [a] + ([b - 2] if b >= 2 and b - 2 != a and b - 2 != skip else [])
        B = len(cand)
        ar = torch.arange(n, device=dev).repeat(B, 1)
        m = [ar, ar.clone(), torch.ones(B, n, 1, dtype=torch.bool, device=dev),
             torch.ones(B, n, 1, dtype=torch.bool, device=dev)] + [torch.full((B, n, 1), 2.0, device=dev) for _ in range(4)]
        assert fg.add_matches(cand, [b] * len(cand), 0.1, *m) == o.add_matches(cand, [b] * len(cand), 0.1, *m)
    return fg, o


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["calib", "rays"])
@pytest.mark.parametrize("skip", [None, 2])
@pytest.mark.parametrize("frames_dev", ["cpu", "cuda"])
def test_solve_matches_gauss_newton_on_the_oracles_inputs(fp32, mode, skip, frames_dev):
    from artdeco_b200 import gn
    h, w = 24, 32
    n = h * w
    frames = consistent_frames(6, h, w, 3, "cpu")
    if frames_dev == "cuda":
        frames = frames.to(fp32)
    frames.K_test = torch.tensor([[30.0, 0.0, 15.3], [0.0, 29.0, 11.7], [0.0, 0.0, 1.0]])
    fg, o = chain_graph(frames, 6, n, 40, fp32, skip)
    calib = mode == "calib"
    unique, Xs, T_WCs, Cs = o.solve_inputs(calib)
    ii, jj, idx, valid, Q = o.prep_two_way_edges()
    Twc = T_WCs[:, 0, :].contiguous().to(fp32)
    c = CFG["local_opt"]
    if calib:
        gn.gauss_newton_calib(Twc, Xs, Cs, frames.K_test.to(fp32), ii, jj, idx, valid, Q, h, w, c["pixel_border"],
                              c["depth_eps"], c["sigma_pixel"], c["sigma_depth"], c["C_conf"], c["Q_conf"], c["max_iters"],
                              c["delta_norm"])
    else:
        gn.gauss_newton_rays(Twc, Xs, Cs, ii, jj, idx, valid, Q, c["sigma_ray"], c["sigma_dist"], c["C_conf"], c["Q_conf"],
                             c["max_iters"], c["delta_norm"])
    before = frames.T_WC.clone()
    (fg.solve_GN_calib if calib else fg.solve_GN_rays)()
    got = frames.T_WC[unique.to(frames.T_WC.device), 0]
    assert torch.equal(got[0].cpu(), before[int(unique[0]), 0].cpu()), "the pinned pose is written"
    untouched = [k for k in range(frames.T_WC.shape[0]) if k not in unique.tolist()]
    assert torch.equal(frames.T_WC[untouched].cpu(), before[untouched].cpu())
    # test_gn.py's device-vs-oracle tolerances: translation and scale 1e-4, quaternion 1e-5
    d = (got[1:].cpu() - Twc[1:].cpu()).abs()
    assert d[:, :3].max() < 1e-4 and d[:, 3:7].max() < 1e-5 and d[:, 7].max() < 1e-4, d.max(0).values
    assert (got[1:].cpu() - before[unique[1:].cpu(), 0].cpu()).abs().max() > 1e-4, "the solve moved nothing"


@pytest.mark.gpu
def test_pin_is_a_no_op(fp32):
    from artdeco_b200 import factor_graph
    frames = dev_frames(2, 16, 16, 4, fp32)
    cfg = {"local_opt": dict(CFG["local_opt"], pin=2)}
    fg = factor_graph.FactorGraph(cfg, None, frames, K=torch.eye(3), device=fp32)
    fg.add_matches([0], [1], 0.1, *matches(1, 256, 1, fp32))
    before = frames.T_WC.clone()
    fg.solve_GN_calib()
    fg.solve_GN_rays()
    assert torch.equal(frames.T_WC, before) and fg.mirror()[0] is None


@pytest.mark.gpu
def test_device_resident_solve_does_not_sync(fp32):
    h, w = 24, 32
    frames = consistent_frames(5, h, w, 6, "cpu").to(fp32)
    frames.K_test = torch.tensor([[30.0, 0.0, 15.3], [0.0, 29.0, 11.7], [0.0, 0.0, 1.0]])
    fg, _ = chain_graph(frames, 5, h * w, 60, fp32)
    fg.solve_GN_calib()                     # first call: library set-up
    torch.cuda.synchronize()
    frames.update_pointmap(3, torch.randn(h * w, 3), torch.rand(h * w, 1) + 1)
    torch.cuda.set_sync_debug_mode("error")
    try:
        fg.solve_GN_calib()
        fg.solve_GN_rays()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()

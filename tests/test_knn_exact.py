"""Grid-hash KNN (csrc/knn.cu) exactness on every query: a constructed shell-boundary case, 1M-point clouds of the
shapes the stream produces against a float64 kd-tree, queries far from their candidates, and non-finite rows.

The squared distance the kernels return is fma(dz,dz,fma(dx,dx,dy*dy)) in fp32; ``dist32`` reproduces it bit for
bit on the host (an exact fp32 fma via round-to-odd in float64), so returned distances are compared exactly."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from artdeco_b200 import synthetic

F32 = np.float32
FLT_MAX = np.finfo(F32).max


# ----------------------------------------------------------------------------- fp32 emulation ----
def fma32(a, b, c):
    """Correctly rounded fp32 fma of float32 arrays: the product is exact in float64, the sum is rounded to odd in
    float64 (53 >= 24 + 2 bits), and rounding that to fp32 gives the single rounding of a*b + c."""
    a64, b64, c64 = (np.asarray(v, F32).astype(np.float64) for v in (a, b, c))
    p = a64 * b64
    s = p + c64
    bp = s - p
    err = (p - (s - bp)) + (c64 - bp)  # TwoSum: s + err == p + c exactly
    fix = (err != 0) & ((s.view(np.int64) & 1) == 0)
    s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(F32)


def dist32(a, b):
    """The kernels' squared distance between float32 points a[..., 3] and b[..., 3]."""
    d = np.asarray(b, F32) - np.asarray(a, F32)
    dx, dy, dz = d[..., 0], d[..., 1], d[..., 2]
    return fma32(dz, dz, fma32(dx, dx, (dy.astype(np.float64) * dy).astype(F32)))


def cell32(x, lo, inv_h, n):
    """cell_of for one axis: floor(fl(fl(x - lo) * inv_h)) clamped to [0, n-1]."""
    t = (np.asarray(x, F32) - F32(lo)) * F32(inv_h)
    return np.clip(np.floor(t).astype(np.int64), 0, n - 1)


def _ord(x):
    """float32 -> int64 key that orders like the floats (and steps by one ulp)."""
    i = np.asarray(x, F32).view(np.int32).astype(np.int64)
    return np.where(i < 0, -(i & 0x7FFFFFFF), i)


def _unord(o):
    o = np.asarray(o, np.int64)
    i = np.where(o < 0, (-o) | 0x80000000, o).astype(np.uint32)
    return i.view(F32)


def first_in_cell(c, lo, h, inv_h, n):
    """Smallest fp32 x whose cell (along one axis) is >= c, for an array of cell numbers c (binary search)."""
    c = np.asarray(c, np.int64)
    a = _ord(F32(lo) + (c - 1).astype(F32) * F32(h))  # cell <= c - 1 at the lower end
    b = _ord(F32(lo) + (c + 1).astype(F32) * F32(h))  # cell >= c at the upper end
    assert (cell32(_unord(a), lo, inv_h, n) < c).all() and (cell32(_unord(b), lo, inv_h, n) >= c).all()
    while (b - a > 1).any():
        m = (a + b) // 2
        ge = cell32(_unord(m), lo, inv_h, n) >= c
        b = np.where(ge, m, b)
        a = np.where(ge, a, m)
    return _unord(b)


def grid_setup(P, lo, hi):
    """grid_setup_kernel on the host (np.cbrt standing in for the device cbrt): (min, h, inv_h, n)."""
    lo, hi = np.asarray(lo, F32), np.asarray(hi, F32)
    e = hi - lo
    emax = F32(e.max()) if e.max() > 0 else F32(1)
    vol = np.prod([float(max(v, F32(1e-3) * emax)) for v in e])
    h = F32(np.cbrt(4.0 * vol / P))
    while True:
        n = [int(np.floor(F32(v) / h)) + 1 for v in e]
        if np.prod(n) <= 2 * P + 64:
            break
        h = F32(h * F32(1.26))
    return lo, h, F32(1) / h, np.array(n)


def boundary_pairs(lo, h, inv_h, n):
    """For every cell k along one axis: xp (last fp32 in cell k), xq (first in cell k+2), their fp32 squared distance
    and the fp32 squared stopping bound after shell 1 of the unpadded rule, fl(h*0.99999)^2.  A pair with
    d < bound is two cells apart yet closer than the shell-1 bound."""
    k = np.arange(1, n - 3)
    xp = np.nextafter(first_in_cell(k + 1, lo, h, inv_h, n), F32(-np.inf))
    xq = first_in_cell(k + 2, lo, h, inv_h, n)
    dx = xq - xp
    d = (dx.astype(np.float64) ** 2).astype(F32)
    b = F32(F32(h) * F32(0.99999))
    bound = F32(b * b)
    shortfall = F32(0.99999) - dx.astype(np.float64) / float(h)  # how much closer than 0.99999*h, in cells
    return k, xp, xq, d, bound, shortfall


# the flat 1M cloud of the constructed case: a 200 x 200 plane at z = 2, bounding box pinned by its corners
PLANE_P, PLANE_LO, PLANE_HI, PLANE_Z = 1_000_000, (-100.0, -100.0, 2.0), (100.0, 100.0, 2.0), 2.0


def test_constructor_finds_pairs_closer_than_the_shell_bound():
    """On the grid the flat 1M plane gets, cells k and k+2 hold fp32 points closer than 0.99999*h: the unpadded
    stopping rule can end a search one shell early.  Runs without a GPU; shows the GPU test below is not vacuous."""
    lo, h, inv_h, n = grid_setup(PLANE_P, PLANE_LO, PLANE_HI)
    assert n.tolist() == [630, 630, 1]
    k, xp, xq, d, bound, short = boundary_pairs(lo[0], h, inv_h, n[0])
    assert (cell32(xp, lo[0], inv_h, n[0]) == k).all() and (cell32(xq, lo[0], inv_h, n[0]) == k + 2).all()
    assert (d < bound).sum() >= 10, f"largest shortfall {short.max():.3g} cells"
    # the padded rule's slack (n * 2^-20 cells, csrc/knn.cu) covers every pair
    assert short.max() < n.max() * 2.0 ** -20


def test_fma32_and_dist32_match_the_oracle():
    g = np.random.default_rng(0)
    a = (g.standard_normal((4000, 3)) * np.array([1e3, 1.0, 1e-3]) + 100).astype(F32)
    # (1 + 2^-12)^2 = 1 + 2^-11 + 2^-24 is halfway between two fp32 values.  Adding 2^-80 puts the exact sum above the
    # midpoint, but float64 rounds it back onto the midpoint: only the round-to-odd step rounds it up.
    t = F32(1 + 2.0 ** -12)
    assert fma32(t, t, F32(2.0 ** -80)) == F32(1 + 2.0 ** -11 + 2.0 ** -23)
    assert fma32(t, t, F32(0)) == F32(1 + 2.0 ** -11)  # the tie itself goes to even
    assert fma32(t, t, F32(-(2.0 ** -80))) == F32(1 + 2.0 ** -11)
    d_ref, i_ref = oracle.knn_index(a, 4)
    assert np.array_equal(dist32(a[:, None, :], a[i_ref]).view(np.uint32), d_ref.view(np.uint32))


# ----------------------------------------------------------------------------- raw calls (GPU) ----
def _knn_index_raw(pts, K, ws):
    """adb_knn_index over every point (distIndex2) into the caller's workspace; returns (d[P,K], ids[P,K], grid)."""
    from artdeco_b200 import _lib
    from artdeco_b200 import knn  # noqa: F401  (registers the signatures)
    P = pts.shape[0]
    d = torch.empty(P * K, dtype=torch.float32, device=pts.device)
    ids = torch.empty(P * K, dtype=torch.int32, device=pts.device)
    _lib.call("adb_knn_index", P, _lib.ptr(pts), K, P, None, None, _lib.ptr(d), _lib.ptr(ids), _lib.ptr(ws),
              ws.numel(), _lib.stream())
    off = (-ws.data_ptr()) % 256  # the Grid struct sits at the 256-aligned start of the workspace
    raw = ws[off:off + 36].cpu()
    f, i = raw[:20].view(torch.float32).numpy(), raw[20:36].view(torch.int32).numpy()
    grid = dict(minx=f[0], miny=f[1], minz=f[2], h=f[3], inv_h=f[4], nx=int(i[0]), ny=int(i[1]), nz=int(i[2]),
                ncells=int(i[3]))
    return d.view(P, K).cpu().numpy(), ids.view(P, K).cpu().numpy(), grid


def _workspace(P, dev):
    from artdeco_b200 import _lib
    from artdeco_b200 import knn  # noqa: F401
    nb = C.c_size_t(0)
    _lib.call("adb_knn_workspace_bytes", P, C.byref(nb))
    return torch.empty(nb.value, dtype=torch.uint8, device=dev)


def _walk_until(base, d_of, lo_d, hi_d, step_dir):
    """Walk fp32 values from ``base`` one ulp at a time until d_of(value) lies in (lo_d, hi_d]."""
    v = F32(base)
    for _ in range(10000):
        d = d_of(v)
        if lo_d < d <= hi_d:
            return v, d
        v = np.nextafter(v, F32(step_dir * np.inf))
    raise AssertionError(f"no fp32 value found near {base} for a distance in ({lo_d}, {hi_d}]")


@pytest.mark.gpu
def test_constructed_shell_boundary_case(cuda):
    """p is the last fp32 point of cell k, q the first of cell k+2, |pq| < 0.99999*h.  Neighbours r in the cells
    shell 1 visits are farther than q but inside the shell-1 bound (placed as close to the bound as fp32 allows), so
    a search that stops after shell 1 returns r instead of q.  distIndex2 (K=1), distCUDA2 (three such r) and distIndexQ are compared with the brute force."""
    from artdeco_b200.knn import distCUDA2, distIndex2, distIndexQ
    g = torch.Generator().manual_seed(11)
    P = PLANE_P
    xy = torch.rand(P, 2, generator=g, dtype=torch.float64) * 200 - 100
    base = np.concatenate([xy.numpy(), np.full((P, 1), PLANE_Z)], 1).astype(F32)
    base[:4, :2] = [[-100, -100], [100, 100], [-100, 100], [100, -100]]  # pin the box
    ws = _workspace(P, cuda)
    _, _, grid = _knn_index_raw(torch.from_numpy(base).to(cuda), 1, ws)
    lo, h, inv_h, nx = grid["minx"], grid["h"], grid["inv_h"], grid["nx"]
    k, xp, xq, d, bound, short = boundary_pairs(lo, h, inv_h, nx)
    good = np.nonzero(d < bound)[0]
    if len(good) < 2:
        pytest.fail(f"the device grid (h={h}, nx={nx}) leaves no pair two cells apart closer than 0.99999*h; "
                    f"largest shortfall {short.max():.3g} cells")
    # two sites in different y rows: site A for K=1 (one r), site B for distCUDA2 (three r).  The rows sit near
    # y = -10 and y = +10, where an fp32 step in y moves a squared distance ~h^2 by less than the window
    # (|pq|^2, bound] is wide; r is placed by stepping its y.
    sites = good[np.argsort(-short[good])[:2]]
    rows = [int((y - grid["miny"]) / h) for y in (-10.0, 10.0)]
    y_rows = [F32(grid["miny"] + F32(h) * F32(j + 0.5)) for j in rows]
    pts = base.copy()
    z0 = F32(PLANE_Z)
    placed = []  # (site, role, index)
    slot = 4
    b = F32(F32(h) * F32(0.99999))
    for site, (s, y0) in enumerate(zip(sites, y_rows)):
        p = np.array([xp[s], y0, z0], F32)
        q = np.array([xq[s], y0, z0], F32)
        d_pq = dist32(p, q)
        # filler within 3h of p moves to the row y = 50, far from both sites (P and the box stay the same)
        near = (np.abs(pts[:, 0] - p[0]) < 3 * h) & (np.abs(pts[:, 1] - p[1]) < 3 * h)
        near[:4] = False
        pts[near, 1] = 50.0
        rs = []
        # (x offset, y direction): straight up, straight down, and half a cell back in x (still p's cell)
        for ox, sign in ([(0.0, 1)] if site == 0 else [(0.0, 1), (0.0, -1), (-0.5, 1)]):
            r = p.copy()
            r[0] = p[0] + F32(ox * h)

            def d_of(v, r=r):
                return dist32(p, np.array([r[0], v, z0], F32))
            oy = np.sqrt(max(float(b) ** 2 - float(r[0] - p[0]) ** 2, 0.0))
            r[1], _ = _walk_until(p[1] + F32(sign * oy), d_of, d_pq, bound, -sign)
            rs.append(r)
        for role, pt in [("p", p), ("q", q)] + [("r", r) for r in rs]:
            pts[slot] = pt
            placed.append((site, role, slot))
            slot += 1
    pts_d = torch.from_numpy(pts).to(cuda)
    d1, i1, grid2 = _knn_index_raw(pts_d, 1, ws)
    assert grid2 == grid, "the grid depends only on the bounding box and P"
    for site, role, idx in placed:
        cx = cell32(pts[idx, 0], lo, inv_h, nx) - k[sites[site]]
        cy = cell32(pts[idx, 1], grid["miny"], inv_h, grid["ny"]) - rows[site]
        want = {"p": (0, 0), "q": (2, 0)}.get(role)
        assert (cx, cy) == want if want else max(abs(cx), abs(cy)) == 1, (role, cx, cy)  # r: in shell 1
    qidx = np.array([idx for _, _, idx in placed], np.int32)
    p_rows = [j for j, (_, role, _) in enumerate(placed) if role == "p"]
    q_of = {site: idx for site, role, idx in placed if role == "q"}

    # distIndex2, K = 1: p's nearest is q
    dr, ir = oracle.knn_index(pts, 1, qidx)
    assert [int(ir[j, 0]) for j in p_rows] == [q_of[0], q_of[1]]
    assert np.array_equal(i1[qidx, 0], ir[:, 0]), f"distIndex2 K=1: kernel {i1[qidx, 0]} vs brute force {ir[:, 0]}"
    assert np.array_equal(d1[qidx, 0].view(np.uint32), dr[:, 0].view(np.uint32))
    d, ids = distIndex2(pts_d, 1)
    assert np.array_equal(ids.cpu().numpy()[qidx], ir[:, 0])

    # distCUDA2: mean of the three nearest, q among them at site B
    d3, _ = oracle.knn_index(pts, 3, qidx)
    m_ref = ((d3[:, 0] + d3[:, 1]) + d3[:, 2]) / F32(3)
    m = distCUDA2(pts_d).cpu().numpy()[qidx]
    assert np.array_equal(m.view(np.uint32), m_ref.view(np.uint32)), f"distCUDA2 {m} vs brute force {m_ref}"

    # distIndexQ: the constructed points query, every other point but a few fillers is a candidate
    cand = np.ones(P, np.uint8)
    cand[np.random.default_rng(1).choice(np.arange(slot, P), 1000, replace=False)] = 0
    dq_ref, iq_ref = oracle.knn_index(pts, 1, qidx, cand)
    dq, iq = distIndexQ(pts_d, torch.from_numpy(qidx).to(cuda), torch.from_numpy(np.nonzero(cand)[0]).to(cuda), 1)
    assert np.array_equal(iq.cpu().numpy(), iq_ref[:, 0])
    assert np.array_equal(dq.cpu().numpy().view(np.uint32), dq_ref[:, 0].view(np.uint32))


# ----------------------------------------------------------------------------- every query at scale (GPU) ----
def _cloud(kind, P, seed):
    g = np.random.default_rng(seed)
    if kind == "plane":
        return np.concatenate([g.uniform(-100, 100, (P, 2)), np.full((P, 1), 2.0)], 1).astype(F32)
    if kind == "slab":
        return (g.uniform(0, 1, (P, 3)) * np.array([40.0, 40.0, 0.5])).astype(F32)
    if kind == "scene":
        return synthetic.raster_scene(P, seed=seed)["means"].numpy()
    if kind == "depth_maps":
        from oracle import track_ref
        H = W = 512
        Kc = torch.tensor([[400.0, 0, 256], [0, 400.0, 256], [0, 0, 1]], dtype=torch.float64)
        uv = track_ref.pixel_grid(H, W, torch.float64, "cpu")
        out = []
        for v in range(-(-P // (H * W))):
            z = 2.0 + 0.004 * uv[:, 0] * (v % 2) + 0.002 * uv[:, 1] + 0.2 * torch.sin(uv[:, 0] / 40.0 + v)
            X = track_ref.backproject(uv, z[:, None], Kc)
            a = 0.4 * v
            R = torch.tensor([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]], dtype=torch.float64)
            out.append(X @ R.T + torch.tensor([0.3 * v, -0.1 * v, 0.5 * v], dtype=torch.float64))
        return torch.cat(out)[:P].numpy().astype(F32)
    if kind == "offset":
        c = np.array([1000.0, -1000.0, 1000.0])
        return (c + g.uniform(-5, 5, (P, 3))).astype(F32)
    if kind == "clusters":
        n_out = P // 1000
        centres = g.uniform(-5, 5, (200, 3))
        pts = centres[g.integers(0, 200, P - n_out)] + g.standard_normal((P - n_out, 3)) * 0.01
        return np.concatenate([pts, g.uniform(-50, 50, (n_out, 3))]).astype(F32)
    if kind == "duplicates":
        u = g.standard_normal((P // 2, 3)).astype(F32)
        reps = np.concatenate([np.ones(P // 4), np.full(P // 8, 2), np.full(P // 8, 4)]).astype(np.int64)
        return np.repeat(u[: len(reps)], reps, 0)[:P]
    raise ValueError(kind)


def _exact_neighbours(pts, M):
    """float64 kd-tree: the M nearest OTHER points of every point, squared distances ascending."""
    from scipy.spatial import cKDTree
    P = pts.shape[0]
    p64 = pts.astype(np.float64)
    dd, ii = cKDTree(p64).query(p64, k=M + 1, workers=-1)
    keep = ii != np.arange(P)[:, None]
    keep[~(~keep).any(1), -1] = False  # self not returned (M+1 duplicates at 0): drop the last instead
    dd, ii = dd[keep].reshape(P, M), ii[keep].reshape(P, M)
    d2 = ((p64[ii] - p64[:, None, :]) ** 2).sum(-1)  # recomputed squared, not the rounded norm squared
    return d2, ii


def _check_rows(pts, K, d, ids, d2, ii, what):
    P = pts.shape[0]
    assert (ids >= 0).all() and (ids < P).all(), f"{what}: -1 or out-of-range ids with {P - 1} other points"
    assert not (ids == np.arange(P)[:, None]).any(), f"{what}: a query is its own neighbour"
    s = np.sort(ids, 1)
    assert (s[:, 1:] != s[:, :-1]).all(), f"{what}: repeated ids in a row"
    # no closer point was missed
    p64 = pts.astype(np.float64)
    got = ((p64[ids] - p64[:, None, :]) ** 2).sum(-1).max(1)
    bad = got > d2[:, K - 1] * (1 + 2.0 ** -21)
    assert not bad.any(), (f"{what}: {bad.sum()} queries missed a closer point, e.g. query {np.nonzero(bad)[0][:5]}: "
                           f"K-th {got[bad][:5]} vs exact {d2[bad, K - 1][:5]}")
    # the returned distances are the kernel's fp32 formula of the returned ids, ascending
    e = dist32(pts[:, None, :], pts[ids])
    assert np.array_equal(d.view(np.uint32), e.view(np.uint32)), f"{what}: distances differ from fp32 fma of the ids"
    assert (d[:, 1:] >= d[:, :-1]).all(), f"{what}: rows not ascending"
    # ids: the brute force's (distance, id) order wherever the K-th and (K+1)-th distances are clearly apart
    ok = d2[:, K - 1] * (1 + 2.0 ** -20) < d2[:, K]
    assert ok.mean() > 0.25, f"{what}: only {ok.mean():.2f} of the rows decide their K-th neighbour"
    cand, dc = ii[ok, :K], dist32(pts[ok, None, :], pts[ii[ok, :K]])
    order = np.lexsort((cand, dc), axis=1)
    ref_ids, ref_d = np.take_along_axis(cand, order, 1), np.take_along_axis(dc, order, 1)
    assert np.array_equal(d[ok].view(np.uint32), ref_d.view(np.uint32)), f"{what}: distances differ from the exact set"
    tie_free = (ref_d[:, 1:] != ref_d[:, :-1]).all(1)
    assert np.array_equal(ids[ok][tie_free], ref_ids[tie_free]), f"{what}: ids differ from the exact neighbours"
    assert np.array_equal(np.sort(ids[ok], 1), np.sort(ref_ids, 1)), f"{what}: id sets differ"


def _mean3_ref(pts, ii):
    """distCUDA2's value from the exact candidates: the three smallest fp32 distances, ((d0+d1)+d2)/3 in fp32."""
    dc = np.sort(dist32(pts[:, None, :], pts[ii]), 1)
    return ((dc[:, 0] + dc[:, 1]) + dc[:, 2]) / F32(3)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,P,K", [
    ("plane", 1_000_000, 8), ("depth_maps", 1_000_000, 8), ("offset", 1_000_000, 8), ("clusters", 1_000_000, 8),
    ("duplicates", 1_000_000, 8), ("scene", 200_000, 17), ("slab", 200_000, 32)])
def test_every_query_exact(cuda, kind, P, K):
    from artdeco_b200.knn import distCUDA2, distIndex2
    pts = _cloud(kind, P, seed=P + K)
    assert pts.shape == (P, 3) and pts.dtype == F32
    d2, ii = _exact_neighbours(pts, K + 2)
    pd = torch.from_numpy(pts).to(cuda)
    d, ids = distIndex2(pd, K)
    _check_rows(pts, K, d.view(P, K).cpu().numpy(), ids.view(P, K).cpu().numpy(), d2, ii, f"{kind} K={K}")
    m = distCUDA2(pd).cpu().numpy()
    ref = _mean3_ref(pts, ii)
    bad = m.view(np.uint32) != ref.view(np.uint32)
    assert not bad.any(), f"distCUDA2 on {kind}: {bad.sum()} rows differ, e.g. {m[bad][:4]} vs {ref[bad][:4]}"


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 8])
def test_distindexq_queries_far_from_the_candidates(cuda, K):
    """1% candidates in a unit box, queries on a shell around it: every query searches many shells."""
    from artdeco_b200.knn import distIndexQ
    g = np.random.default_rng(K)
    P, n_c = 50_000, 500
    c = g.uniform(0, 1, (n_c, 3))
    dirs = g.standard_normal((P - n_c, 3))
    q = dirs / np.linalg.norm(dirs, axis=1, keepdims=True) * g.uniform(3, 20, (P - n_c, 1))
    pts = np.concatenate([q, c]).astype(F32)
    perm = g.permutation(P)
    pts = pts[perm]
    is_c = np.zeros(P, np.uint8)
    is_c[np.argsort(perm)[P - n_c:]] = 1
    qidx = np.nonzero(is_c == 0)[0].astype(np.int32)
    lo, hi = pts[is_c == 1].min(0), pts[is_c == 1].max(0)
    assert (((pts[qidx] < lo) | (pts[qidx] > hi)).any(1)).all(), "every query lies outside the candidates' box"
    d_ref, i_ref = oracle.knn_index(pts, K, qidx, is_c)
    pd = torch.from_numpy(pts).to(cuda)
    d, ids = distIndexQ(pd, torch.from_numpy(qidx).to(cuda), torch.from_numpy(np.nonzero(is_c)[0]).to(cuda), K)
    d, ids = d.view(-1, K).cpu().numpy(), ids.view(-1, K).cpu().numpy()
    assert is_c[ids].all() and (ids >= 0).all(), "neighbours come from the candidate set only"
    assert np.array_equal(d.view(np.uint32), d_ref.view(np.uint32))
    tie_free = (d_ref[:, 1:] != d_ref[:, :-1]).all(1)
    assert np.array_equal(ids[tie_free], i_ref[tie_free])


# ----------------------------------------------------------------------------- non-finite rows (GPU) ----
BAD_ROWS = np.array([
    [np.nan, 0, 0], [np.nan, np.nan, np.nan], [0.5, np.inf, 0], [-np.inf, 0, 0], [0, 0, np.inf],
    [1e30, 0, 0], [0, -1e30, 0], [0, 0, 1e30], [2e19, 0, 0], [np.inf, -np.inf, np.nan]], F32)


def _with_bad_rows(P, seed, extra=()):
    g = np.random.default_rng(seed)
    pts = g.standard_normal((P, 3)).astype(F32)
    bad = np.concatenate([BAD_ROWS, np.asarray(extra, F32).reshape(-1, 3)])
    at = g.choice(P, len(bad), replace=False)
    pts[at] = bad
    return pts, at


@pytest.mark.gpu
@pytest.mark.parametrize("extra", [(), ((0, 1e19, 0),)], ids=["nonfinite", "nonfinite+1e19"])
def test_nonfinite_and_overflowing_rows(cuda, extra):
    """A row whose squared distance to the rest overflows fp32 (non-finite, 1e30, 2e19) is nobody's neighbour and
    has the empty row FLT_MAX / -1 (distCUDA2: inf), as in the brute force; every other row is unchanged.  A 1e19
    row is finite and usable: it stretches the grid, and its distances (~1e38) are still exact."""
    from artdeco_b200.knn import distCUDA2, distIndex2
    P, K = 20_000, 4
    pts, at = _with_bad_rows(P, 5, extra)
    d_ref, i_ref = oracle.knn_index(pts, K)
    m_ref = oracle.knn_mean3(pts)
    n_bad = len(BAD_ROWS)
    assert (i_ref[at[:n_bad]] == -1).all() and (d_ref[at[:n_bad]] == FLT_MAX).all()
    assert not np.isin(i_ref, at[:n_bad]).any() and np.isinf(m_ref[at[:n_bad]]).all()
    pd = torch.from_numpy(pts).to(cuda)
    d, ids = distIndex2(pd, K)
    d, ids = d.view(P, K).cpu().numpy(), ids.view(P, K).cpu().numpy()
    assert np.array_equal(d.view(np.uint32), d_ref.view(np.uint32)), \
        f"{(d.view(np.uint32) != d_ref.view(np.uint32)).any(1).sum()} rows differ from the brute force"
    tie_free = (d_ref[:, 1:] != d_ref[:, :-1]).all(1)
    assert np.array_equal(ids[tie_free], i_ref[tie_free])
    m = distCUDA2(pd).cpu().numpy()
    assert np.array_equal(m.view(np.uint32), m_ref.view(np.uint32))


@pytest.mark.gpu
def test_only_nonfinite_rows(cuda):
    """No usable point at all, and a single finite point among non-finite ones: empty rows, no neighbours."""
    from artdeco_b200.knn import distCUDA2, distIndex2
    for pts in (BAD_ROWS, np.concatenate([BAD_ROWS, [[1, 2, 3]]]).astype(F32)):
        P = pts.shape[0]
        d, ids = distIndex2(torch.from_numpy(pts).to(cuda), 3)
        assert (ids.cpu().numpy() == -1).all() and (d.cpu().numpy() == FLT_MAX).all()
        assert np.isinf(distCUDA2(torch.from_numpy(pts).to(cuda)).cpu().numpy()).all(), P

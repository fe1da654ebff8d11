"""The tile sort and the blend where uniform random scenes never go: tiles of up to 20000 entries (every bitonic level of the
shared-memory sort and the in-place global-memory network), depth ties, tiles that saturate inside a long list, splats larger
than the frame (16-bit cull radii saturated at 65535) and ragged frames.

References: the C oracle (an independent radix sort; a blend that evaluates every entry with expf, without culling).
Integer outputs are bit-exact.  Floating-point outputs are within 1e-4 of the tensor's scale (tests/helpers.py).

Decision flips: the GPU evaluates alpha with ex2.approx, the oracle with expf, so a pixel whose skip (alpha < 1/255) or stop
(T (1 - alpha) <= 1e-4) decision sits on its threshold may take the other branch.  Instead of an outlier fraction, every pixel
where last_ids or the image differs is walked again in fp64 from the oracle's inputs, and one of its decisions must lie within
1e-5 relative of its threshold; gradients are then compared on every Gaussian that such a pixel does not involve.

Each group also builds its nearest plausible bug from oracle outputs and asserts that it would fail the comparison."""
import functools

import numpy as np
import pytest
import torch

import oracle
from helpers import RTOL, rel_err

KEYS = ("means", "quats", "scales", "opacities", "sh")
TILE = 16
BATCH = 256                 # entries the blend stages per batch
SORT_SMEM_CAP = 4096        # largest tile sorted in shared memory (csrc/raster_isect.cu)
FLIP_MARGIN = 1e-5          # a flipped decision must lie this close (relative) to its threshold in fp64
SENSITIVITY = 10.0          # a planted bug must land at least this many tolerances away

LADDER = (1, 2, 63, 64, 65, 255, 256, 257, 1023, 1024, 1025, 2047, 2048, 2049, 4095, 4096, 4097, 8193, 20000)
TIE_N = 5000                # one more tile whose entries all share one depth
REGIMES = {
    # every splat touches one tile and no pixel stops: the whole list is walked, and skips decide
    "walk": dict(screen_scale=1.0, inset=(5.0, 11.0), opacity_range=(0.0045, 0.006)),
    # every pixel of a dense tile stops within its first two batches, long before the end of the list
    "saturate": dict(screen_scale=4.0, inset=(7.0, 9.0), opacity_range=(0.6, 0.99)),
}


# ---- scene builders (CPU) ---------------------------------------------------------------------------------------------------
def _camera(W, H, f):
    K = np.array([[f, 0.0, W / 2.0], [0.0, f, H / 2.0], [0.0, 0.0, 1.0]], np.float32)
    return np.eye(4, dtype=np.float32), K


def _gaussians(u, v, z, screen_scale, opac, W, H, f, rng):
    """Gaussians whose centres project to pixel (u, v) at depth z with a screen-space scale of `screen_scale` px, each axis
    scaled by up to 1.35x either way and randomly rotated (an isotropic Gaussian has no quaternion gradient to compare)."""
    n = len(u)
    means = np.stack([(u - W / 2.0) * z / f, (v - H / 2.0) * z / f, z], 1).astype(np.float32)
    scales = ((np.asarray(screen_scale, np.float64) * z / f)[:, None] * np.exp(rng.uniform(-0.3, 0.3, (n, 3))))
    scales = scales.astype(np.float32)
    quats = rng.normal(size=(n, 4))
    quats = (quats / np.linalg.norm(quats, axis=1, keepdims=True)).astype(np.float32)
    sh = np.zeros((n, 16, 3), np.float32)
    sh[:, 0] = rng.normal(0.0, 0.5, (n, 3))
    sh[:, 1:] = rng.normal(0.0, 0.05, (n, 15, 3))
    return dict(means=means, quats=quats, scales=scales, opacities=np.asarray(opac, np.float32), sh=sh)


def _concat(parts, perm=None):
    out = {k: np.concatenate([p[k] for p in parts]) for k in KEYS}
    if perm is not None:
        out = {k: np.ascontiguousarray(v[perm]) for k, v in out.items()}
    return out


def dense_tiles(W, H, counts, screen_scale, opacity_range, seed, inset=(5.0, 11.0), depths=(2.0, 3.0, 5.0), f=300.0,
                tie_tiles=()):
    """{tile: n}: n Gaussians whose centres lie `inset` px inside `tile` (both axes), depth drawn from `depths` (one depth for
    the tiles in `tie_tiles`), opacity uniform in `opacity_range`; the Gaussian order is shuffled.  Identity viewmat, focal f.
    Returns (scene dict of numpy arrays, viewmat, K)."""
    rng = np.random.default_rng(seed)
    tw = (W + TILE - 1) // TILE
    parts = []
    for tile, n in counts.items():
        tx, ty = tile % tw, tile // tw
        u = tx * TILE + rng.uniform(inset[0], inset[1], n)
        v = ty * TILE + rng.uniform(inset[0], inset[1], n)
        z = np.full(n, depths[1]) if tile in tie_tiles else rng.choice(np.asarray(depths), n)
        parts.append(_gaussians(u, v, z, screen_scale, rng.uniform(*opacity_range, n), W, H, f, rng))
    total = sum(counts.values())
    V, K = _camera(W, H, f)
    return _concat(parts, rng.permutation(total)), V, K


def ladder_layout():
    """The ladder in one frame: every rung (and the tie tile) at the centre of its own 3x3-tile cell, so a splat that spills
    into the neighbouring tiles (the saturating regime) never reaches another rung.  Returns W, H, {tile: n}, tie tile."""
    rungs = list(LADDER) + [TIE_N]
    cols = 5
    rows = (len(rungs) + cols - 1) // cols
    W, H = 3 * cols * TILE, 3 * rows * TILE
    tw = 3 * cols
    counts = {}
    for k, n in enumerate(rungs):
        cx, cy = k % cols, k // cols
        counts[(3 * cy + 1) * tw + 3 * cx + 1] = n
    tie_tile = list(counts)[-1]
    return W, H, counts, tie_tile


@functools.lru_cache(maxsize=None)
def ladder(regime):
    W, H, counts, tie = ladder_layout()
    p = REGIMES[regime]
    sc, V, K = dense_tiles(W, H, counts, p["screen_scale"], p["opacity_range"], seed=11 if regime == "walk" else 12,
                           inset=p["inset"], tie_tiles=(tie,))
    return sc, V, K, W, H, counts, tie


def frame_sized(with_saturated=True):
    """A small random scene (200x120, f = 150) plus splats larger than the frame: a near-plane splat (z = 0.0105, centre
    ~11,400 px off-screen, one radius above 65535), one whose radii are both above 65535, and three of ~300 px at depth 1.5."""
    W, H, f = 200, 120, 150.0
    rng = np.random.default_rng(5)
    n = 1500
    base = _gaussians(rng.uniform(-20, W + 20, n), rng.uniform(-20, H + 20, n), rng.uniform(2.0, 12.0, n),
                      np.exp(rng.uniform(np.log(0.5), np.log(6.0), n)), 1 / (1 + np.exp(-1.5 * rng.normal(size=n))),
                      W, H, f, rng)
    q = rng.normal(size=(n, 4)).astype(np.float32)
    base["quats"] = q / np.linalg.norm(q, axis=1, keepdims=True)
    base["scales"] *= np.exp(rng.uniform(-0.7, 0.7, (n, 3))).astype(np.float32)     # anisotropic
    big = []
    near = dict(means=np.array([[11400 * 0.0105 / f, 0.0, 0.0105]], np.float32), scale=1.3, opac=0.35)
    both = dict(means=np.array([[-0.5, 0.01, 0.0105]], np.float32), scale=2.0, opac=0.3)
    for s in (near, both):
        g = _gaussians(np.zeros(1), np.zeros(1), np.zeros(1), 1.0, [s["opac"]], W, H, f, rng)
        g["means"] = s["means"]
        g["scales"] = np.full((1, 3), s["scale"], np.float32)
        big.append(g)
    for k in range(3):                                   # larger than the frame at moderate depth
        big.append(_gaussians(rng.uniform(0, W, 1), rng.uniform(0, H, 1), np.array([1.5]), rng.uniform(80, 120, 1),
                              rng.uniform(0.3, 0.6, 1), W, H, f, rng))
    sc = _concat([base] + big if with_saturated else [base, big[0]] + big[2:])
    V, K = _camera(W, H, f)
    return sc, V, K, W, H


def ragged(W, H, n_dense=4097, n_sat=300, seed=3):
    """A dense list and saturating splats in the bottom-right (ragged) tile: centres uniform over its visible pixels."""
    rng = np.random.default_rng(seed)
    f = 300.0
    tx, ty = (W - 1) // TILE, (H - 1) // TILE
    x0, x1, y0, y1 = tx * TILE, min(W, tx * TILE + TILE), ty * TILE, min(H, ty * TILE + TILE)
    parts = []
    for n, scale, op in ((n_dense, 1.0, (0.0045, 0.006)), (n_sat, 4.0, (0.6, 0.99))):
        u, v = rng.uniform(x0, x1, n), rng.uniform(y0, y1, n)
        parts.append(_gaussians(u, v, rng.choice(np.array([2.0, 3.0, 5.0]), n), scale, rng.uniform(*op, n), W, H, f, rng))
    V, K = _camera(W, H, f)
    return _concat(parts, rng.permutation(n_dense + n_sat)), V, K, ty * ((W + TILE - 1) // TILE) + tx


@functools.lru_cache(maxsize=None)
def oracle_fwd(key):
    sc, V, K, W, H = _scene(key)
    return oracle.rasterize_fwd(*[sc[k] for k in KEYS], V, K, W, H)


def _scene(key):
    if key in REGIMES:
        sc, V, K, W, H, _, _ = ladder(key)
        return sc, V, K, W, H
    if key == "frame":
        return frame_sized()
    if key == "frame_without_saturated":
        return frame_sized(with_saturated=False)
    W, H = key
    sc, V, K, _ = ragged(W, H)
    return sc, V, K, W, H


def upstream(W, H, seed=1):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(H, W, 4, generator=g), torch.randn(H, W, generator=g)


def tile_counts(f, W, H):
    T = ((W + TILE - 1) // TILE) * ((H + TILE - 1) // TILE)
    o = np.append(f["tile_offsets"].astype(np.int64), len(f["vals"]))
    return np.diff(o)[:T]


# ---- fp64 decision walk -----------------------------------------------------------------------------------------------------
def pixel_walk(f, opac, x, y, W):
    """Walks pixel (x, y) through its tile's list in fp64 from the oracle's inputs.  Returns (smallest relative distance of a
    skip or stop decision to its threshold, Gaussians that contribute in fp64 or lie within FLIP_MARGIN of contributing)."""
    tw = (W + TILE - 1) // TILE
    tl = (y // TILE) * tw + x // TILE
    o = f["tile_offsets"]
    start, end = int(o[tl]), int(o[tl + 1]) if tl + 1 < len(o) else len(f["vals"])
    g = f["vals"][start:end].astype(np.int64)
    if len(g) == 0:
        return np.inf, g
    m2, con = f["means2d"][g].astype(np.float64), f["conics"][g].astype(np.float64)
    dx, dy = m2[:, 0] - (x + 0.5), m2[:, 1] - (y + 0.5)
    sigma = 0.5 * (con[:, 0] * dx * dx + con[:, 2] * dy * dy) + con[:, 1] * dx * dy
    raw = opac[g].astype(np.float64) * np.exp(-sigma)
    alpha = np.minimum(0.999, raw)
    valid = (sigma >= 0) & (alpha >= 1 / 255)
    T_after = np.cumprod(np.where(valid, 1.0 - alpha, 1.0))
    stop = np.nonzero(valid & (T_after <= 1e-4))[0]
    last = int(stop[0]) if len(stop) else len(g) - 1
    seen = slice(0, last + 1)
    skip_m = np.abs(raw[seen] * 255.0 - 1.0)
    stop_m = np.abs(T_after[seen][valid[seen]] / 1e-4 - 1.0)
    margin = min(skip_m.min(initial=np.inf), stop_m.min(initial=np.inf))
    involved = g[seen][raw[seen] * 255.0 >= 1.0 - FLIP_MARGIN]
    return margin, involved


def check_flips(f, opac, colors, alphas, last, W, H, what):
    """Pixels where last_ids or the image (beyond 1e-4 of scale) differ from the oracle must be decision flips.  Returns
    (number of such pixels, largest fp64 margin, Gaussians they involve)."""
    colors, alphas, last = (np.asarray(a.detach().cpu() if isinstance(a, torch.Tensor) else a) for a in (colors, alphas, last))
    sc_c = max(np.abs(f["colors"]).max(), 1e-20)
    sc_a = max(np.abs(f["alphas"]).max(), 1e-20)
    bad = (last != f["last_ids"]) | (np.abs(colors.astype(np.float64) - f["colors"]) > RTOL * sc_c).any(-1) | \
          (np.abs(alphas.astype(np.float64) - f["alphas"]) > RTOL * sc_a)
    ys, xs = np.nonzero(bad)
    assert len(ys) <= max(8, 0.01 * W * H), f"{what}: {len(ys)} of {W * H} pixels differ from the oracle"
    worst, involved = 0.0, [np.zeros(0, np.int64)]
    for y, x in zip(ys.tolist(), xs.tolist()):
        m, g = pixel_walk(f, opac, x, y, W)
        assert m <= FLIP_MARGIN, f"{what}: pixel ({x},{y}) differs but its closest decision is {m:.2e} from its threshold"
        worst = max(worst, m)
        involved.append(g)
    print(f"[{what}] decision-flip pixels: {len(ys)}, largest fp64 margin {worst:.2e}")
    return len(ys), worst, np.unique(np.concatenate(involved))


def close_except(a, b, skip, what, rtol=RTOL):
    """assert_close over the Gaussians (rows) not in `skip`; returns the max error in units of the tolerance."""
    a = np.asarray(a.detach().cpu() if isinstance(a, torch.Tensor) else a, np.float64)
    b = np.asarray(b, np.float64)
    keep = np.ones(a.shape[0], bool)
    keep[skip] = False
    scale = max(np.abs(b).max(), 1e-20)
    err = np.abs(a[keep] - b[keep]).max(initial=0.0) / (rtol * scale)
    assert err <= 1.0, f"{what}: max error {err:.2f} x tolerance on {keep.sum()} Gaussians ({len(skip)} flip-involved skipped)"
    return err


# ---- CPU: builders, premises, coverage ------------------------------------------------------------------------------------
@pytest.mark.parametrize("regime", list(REGIMES))
def test_ladder_builder_gives_the_requested_tile_counts(regime):
    sc, V, K, W, H, counts, tie = ladder(regime)
    f = oracle_fwd(regime)
    tpg = f["tiles_per_gauss"]
    # walk: every splat touches its own tile only; saturate: its 3x3 neighbourhood, which holds no other rung
    assert (tpg == (1 if regime == "walk" else 9)).all()
    cnt = tile_counts(f, W, H)
    for tile, n in counts.items():
        assert cnt[tile] == n, (tile, cnt[tile], n)
    if regime == "walk":
        assert cnt.sum() == sum(counts.values())
    dep = f["depths"][f["vals"][f["tile_offsets"][tie]:f["tile_offsets"][tie] + TIE_N]]
    assert (dep == dep[0]).all(), "the tie tile holds one depth"


def test_ladder_reaches_every_sort_regime():
    """Shared-memory networks padded to every power of two from 64 to 4096, and the global-memory network."""
    W, H, counts, _ = ladder_layout()
    cnt = tile_counts(oracle_fwd("walk"), W, H)
    np2 = {max(64, 1 << int(np.ceil(np.log2(n)))) for n in cnt if 1 < n <= SORT_SMEM_CAP}
    assert np2 >= {64, 128, 256, 512, 1024, 2048, 4096}, sorted(np2)
    assert (cnt > SORT_SMEM_CAP).sum() >= 3 and cnt.max() >= 20000
    assert (cnt > BATCH).sum() >= 10                     # lists of several blend batches


def _tile_alpha64(f, opac, tile, W, n_entries=None):
    """fp64 alpha [256 pixels, entries] of a tile's first `n_entries` entries (0 where skipped)."""
    tw = (W + TILE - 1) // TILE
    o = f["tile_offsets"]
    s = int(o[tile])
    e = int(o[tile + 1]) if tile + 1 < len(o) else len(f["vals"])
    if n_entries is not None:
        e = min(e, s + n_entries)
    g = f["vals"][s:e].astype(np.int64)
    ty, tx = divmod(tile, tw)
    py, px = np.meshgrid(ty * TILE + np.arange(TILE) + 0.5, tx * TILE + np.arange(TILE) + 0.5, indexing="ij")
    px, py = px.reshape(-1, 1), py.reshape(-1, 1)
    m2, con = f["means2d"][g].astype(np.float64), f["conics"][g].astype(np.float64)
    dx, dy = m2[None, :, 0] - px, m2[None, :, 1] - py
    sig = 0.5 * (con[None, :, 0] * dx * dx + con[None, :, 2] * dy * dy) + con[None, :, 1] * dx * dy
    a = np.minimum(0.999, opac[g][None].astype(np.float64) * np.exp(-sig))
    return np.where((sig >= 0) & (a >= 1 / 255), a, 0.0)


def test_regime_premises():
    """walk: no pixel of any rung stops (its transmittance stays above twice the threshold); saturate: every pixel of every
    rung of >= 1024 entries stops within the first two batches (transmittance below half the threshold after 512 entries)."""
    sc, V, K, W, H, counts, _ = ladder("walk")
    f = oracle_fwd("walk")
    for tile in counts:
        T = np.prod(1.0 - _tile_alpha64(f, sc["opacities"], tile, W), axis=1)
        assert T.min() > 2e-4, (tile, T.min())
    sc, V, K, W, H, counts, _ = ladder("saturate")
    f = oracle_fwd("saturate")
    deepest = {}
    for tile, n in counts.items():
        if n < 1024:
            continue
        T = np.prod(1.0 - _tile_alpha64(f, sc["opacities"], tile, W, 2 * BATCH), axis=1)
        assert T.max() < 0.5e-4, (tile, n, T.max())
        ty, tx = divmod(tile, W // TILE)
        block = f["last_ids"][ty * TILE:(ty + 1) * TILE, tx * TILE:(tx + 1) * TILE]
        deepest[n] = int((block - f["tile_offsets"][tile]).max())
    assert max(deepest.values()) < 2 * BATCH, deepest


def test_frame_sized_splats_premise():
    sc, V, K, W, H = frame_sized()
    f = oracle_fwd("frame")
    n = len(sc["means"])
    r = f["radii"][n - 5:]
    T = ((W + TILE - 1) // TILE) * ((H + TILE - 1) // TILE)
    assert r[0, 0] > 65535 and r[0, 1] < 65535 and abs(f["means2d"][n - 5, 0] - W / 2) > 10000, r[0]
    assert (r[1] > 65535).all(), r[1]
    assert (r[2:] > max(W, H)).all(), r[2:]
    assert (f["tiles_per_gauss"][n - 5:] == T).all(), "every frame-sized splat covers every tile"


# ---- CPU: sensitivity -------------------------------------------------------------------------------------------------------
def test_sensitivity_tie_order_and_unsorted_tail():
    f = oracle_fwd("walk")
    W, H, counts, tie = ladder_layout()
    keys, vals = f["keys"], f["vals"]
    # ties of each (tile, depth) run in reverse index order
    rev = vals.copy()
    brk = np.flatnonzero(np.diff(keys)) + 1
    for s, e in zip(np.r_[0, brk], np.r_[brk, len(keys)]):
        rev[s:e] = rev[s:e][::-1]
    n_tied = int((rev != vals).sum())
    assert n_tied > 0.9 * len(vals), "nearly every entry is part of a depth tie"
    o = f["tile_offsets"]
    s = int(o[tie])
    assert not np.array_equal(rev[s:s + TIE_N], vals[s:s + TIE_N])
    # a dense tile whose entries after position 4096 stay in the scatter's (arbitrary) order
    rng = np.random.default_rng(0)
    for tile, n in counts.items():
        if n > SORT_SMEM_CAP + 1:                          # (a tail of one entry is sorted by construction)
            s = int(o[tile])
            bug = vals[s:s + n].copy()
            rng.shuffle(bug[SORT_SMEM_CAP:])
            assert (bug != vals[s:s + n]).sum() > 0.9 * (n - SORT_SMEM_CAP), tile


def _drop_last_batch(f, counts):
    """The oracle's sorted list without the last blend batch of every rung longer than one batch: (vals, tile_offsets)."""
    keep = np.ones(len(f["vals"]), bool)
    o = np.append(f["tile_offsets"].astype(np.int64), len(f["vals"]))
    for tile, n in counts.items():
        if n > BATCH:
            e = int(o[tile + 1])
            keep[e - ((n - 1) % BATCH + 1):e] = False
    offs = np.searchsorted(f["keys"][keep] >> 32, np.arange(len(f["tile_offsets"]))).astype(np.int32)
    return f["vals"][keep], offs


def test_sensitivity_dropping_the_last_batch_of_every_dense_tile():
    sc, V, K, W, H, counts, _ = ladder("walk")
    f = oracle_fwd("walk")
    vals, offs = _drop_last_batch(f, counts)
    col, alp, _ = oracle.blend_fwd(W, H, f["means2d"], f["conics"], sc["opacities"], f["feats"], vals, offs)
    m = np.abs(col - f["colors"]).max() / (RTOL * np.abs(f["colors"]).max())
    print(f"[sensitivity] last batch dropped: {m:.0f} x tolerance")
    assert m >= SENSITIVITY


def test_sensitivity_frame_without_its_saturated_radius_splat():
    f, g = oracle_fwd("frame"), oracle_fwd("frame_without_saturated")
    m = np.abs(f["colors"] - g["colors"]).max() / (RTOL * np.abs(f["colors"]).max())
    print(f"[sensitivity] 65535-radius splat removed: {m:.0f} x tolerance")
    assert m >= SENSITIVITY


# ---- GPU --------------------------------------------------------------------------------------------------------------------
def stages(sc, V, K, W, H, dev, hits=False):
    from artdeco_b200 import raster as R
    t = {k: torch.from_numpy(sc[k]).to(dev) for k in KEYS}
    Vd, Kd = torch.from_numpy(V).to(dev), torch.from_numpy(K).to(dev)
    campos = torch.inverse(Vd)[:3, 3].contiguous()
    radii, splats, tpg = R.project(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], 3, Vd, Kd, campos, W, H,
                                   0.01, 0.01, 1e10, 0.0)
    keys, vals, offs, n = R.intersect(radii, splats, tpg, W, H)
    hm = torch.zeros(max(1, n), dtype=torch.uint8, device=dev) if hits else None
    colors, alphas, last = R.blend_forward(W, H, radii.shape[0], splats, vals, offs, hits=hm)
    return dict(radii=radii, splats=splats, tpg=tpg, keys=keys, vals=vals, offs=offs, n=n, colors=colors, alphas=alphas,
                last=last, hits=hm)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", list(REGIMES))
def test_intersection_ladder_bit_exact(cuda, regime):
    from artdeco_b200 import raster as R
    sc, V, K, W, H, counts, tie = ladder(regime)
    f = oracle_fwd(regime)
    g = stages(sc, V, K, W, H, cuda)
    assert np.array_equal(g["radii"].cpu().numpy(), f["radii"])
    assert np.array_equal(g["tpg"].cpu().numpy(), f["tiles_per_gauss"])
    n = len(f["keys"])
    ref_offs = np.append(f["tile_offsets"], n)

    def same(keys, vals, offs, what, upto=None):
        m = n if upto is None else upto
        assert np.array_equal(keys.cpu().numpy()[:m], f["keys"][:m]), f"{what}: keys"
        assert np.array_equal(vals.cpu().numpy()[:m], f["vals"][:m]), f"{what}: vals"
        if upto is None:
            assert np.array_equal(offs.cpu().numpy(), ref_offs), f"{what}: offsets"

    assert g["n"] == n
    same(g["keys"], g["vals"], g["offs"], "bucketed")
    for cap in (n, n + 4321):
        k2, v2, o2, info = R.intersect(g["radii"], g["splats"], g["tpg"], W, H, capacity=cap)
        assert int(info["n_isect"]) == n and int(info["overflow"]) == 0, cap
        same(k2, v2, o2, f"capacity {cap}")
    # an undersized capacity that cuts the 20000-entry tile after 5000 of its entries
    big = max(counts, key=counts.get)
    cut = int(ref_offs[big]) + 5000
    k3, v3, o3, info = R.intersect(g["radii"], g["splats"], g["tpg"], W, H, capacity=cut)
    assert int(info["overflow"]) == 1 and int(info["n_isect"]) == n and int(o3[-1]) == cut
    o3 = o3.cpu().numpy()
    assert np.array_equal(o3[:big + 1], ref_offs[:big + 1]) and (o3[big + 1:] == cut).all()
    same(k3, v3, None, "undersized capacity", upto=int(ref_offs[big]))
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_intersection_multi_view_dense_tiles_at_a_nonzero_segment_base(cuda):
    """C = 3: view 0 is shifted (its tiles start the buffer), views 1 and 2 see the ladder, so their global-memory sorts run
    at a non-zero base.  Keys, vals and offsets equal the oracle's per-view lists laid end to end; the batched blend equals
    three single-view blends bit for bit."""
    from artdeco_b200 import raster as R
    sc, V, K, W, H, counts, _ = ladder("walk")
    V0 = V.copy()
    V0[0, 3] = 0.37
    Vs = np.stack([V0, V, V])
    N, Cn = len(sc["means"]), 3
    t = {k: torch.from_numpy(sc[k]).to(cuda) for k in KEYS}
    Vd, Kd = torch.from_numpy(Vs).to(cuda), torch.from_numpy(np.stack([K] * Cn)).to(cuda)
    P = torch.inverse(Vd)[:, :3, 3].contiguous()
    cnt = R.new_tile_counts(W, H, cuda, Cn)
    radii, splats, tpg = R.project_multi(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], 3, Vd, Kd, P, W, H,
                                         0.01, 0.01, 1e10, 0.0, cnt)
    keys, vals, offs, info, seg = R.intersect_multi(radii, splats, tpg, W, H, cnt)
    ref_k, ref_v, ref_o, base = [], [], [], 0
    for c in range(Cn):
        r_, m2, d, _ = oracle.project(sc["means"], sc["quats"], sc["scales"], sc["opacities"], Vs[c], oracle.make_cam(K, W, H))
        _, kc, vc, oc = oracle.isect(r_, m2, d, W, H, cam_id=c, n_cams=Cn)
        assert np.array_equal(radii[c].cpu().numpy(), r_)
        ref_k.append(kc)
        ref_v.append(vc)
        ref_o.append(np.append(oc, len(kc)) + base)
        base += len(kc)
    assert seg[0] > 0 and seg[1] == seg[2] == sum(counts.values())
    assert np.array_equal(keys.cpu().numpy(), np.concatenate(ref_k))
    assert np.array_equal(vals.cpu().numpy(), np.concatenate(ref_v))
    assert np.array_equal(offs.cpu().numpy(), np.stack(ref_o))
    hm = torch.zeros(max(1, vals.numel()), dtype=torch.uint8, device=cuda)
    cm, am, lm = R.blend_forward_multi(W, H, splats, vals, offs, hits=hm)
    for c in range(Cn):
        s = int(offs[c, 0])
        h1 = torch.zeros(max(1, seg[c]), dtype=torch.uint8, device=cuda)
        c1, a1, l1 = R.blend_forward(W, H, N, splats[c], vals[s:s + seg[c]] - c * N, offs[c] - s, hits=h1)
        # last_ids are absolute in the batch; a pixel that nothing reaches keeps 0 in both
        assert torch.equal(c1, cm[c]) and torch.equal(a1, am[c]) and torch.equal(torch.where(a1 > 0, l1 + s, 0), lm[c]), c
        assert torch.equal(h1[:seg[c]], hm[s:s + seg[c]]), c


# Gradients in tiles that saturate: the backward recovers each splat's T by dividing T_final by (1 - alpha) back through the
# list, and every factor amplifies alpha's fp32 rounding by alpha / (1 - alpha) (50x at alpha = 0.98) -- in the kernel
# (rcp.approx of an ex2.approx alpha) and in the oracle (expf, exact division) alike.  The measured worst case on the scenes
# below is 1.01e-4 of scale, so scenes with saturating splats compare gradients at 2e-4.
SATURATED_GRAD_RTOL = 2 * RTOL


def _rasterize_and_compare(sc, V, K, W, H, key, cuda, seed=1, grad_rtol=RTOL):
    """rasterization() + autograd against oracle.rasterize_bwd; integer outputs bit-exact, image with decision flips checked
    in fp64, every parameter gradient on the Gaussians no flipped pixel involves.  Returns (stages, report)."""
    from artdeco_b200 import raster as R
    f = oracle_fwd(key)
    vc, va = upstream(W, H, seed)
    b = oracle.rasterize_bwd(*[sc[k] for k in KEYS], V, f, vc.numpy(), va.numpy())
    g = stages(sc, V, K, W, H, cuda)
    assert np.array_equal(g["radii"].cpu().numpy(), f["radii"]), "radii"
    assert np.array_equal(g["keys"].cpu().numpy(), f["keys"]), "keys"
    assert np.array_equal(g["vals"].cpu().numpy(), f["vals"]), "vals"
    flips, worst, involved = check_flips(f, sc["opacities"], g["colors"], g["alphas"], g["last"], W, H, str(key))
    t = {k: torch.from_numpy(sc[k]).to(cuda).requires_grad_(True) for k in KEYS}
    colors, alphas, meta = R.rasterization(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"],
                                           torch.from_numpy(V).to(cuda)[None], torch.from_numpy(K).to(cuda)[None], W, H,
                                           render_mode="RGB+D", sh_degree=3, eps2d=0.01)
    assert torch.equal(colors[0], g["colors"]) and torch.equal(alphas[0, ..., 0], g["alphas"]), \
        "rasterization() renders what the stages render"
    ((colors[0] * vc.to(cuda)).sum() + (alphas[0, ..., 0] * va.to(cuda)).sum()).backward()
    report = dict(flips=flips, margin=worst, involved=len(involved))
    good = np.ones((H, W), bool)
    for name, ref in (("colors", f["colors"]), ("alphas", f["alphas"])):
        a = (g[name].cpu().numpy()).astype(np.float64)
        bad_pix = np.abs(a - ref) > RTOL * np.abs(ref).max()
        good &= ~(bad_pix.any(-1) if bad_pix.ndim == 3 else bad_pix)
    for name, ref in (("colors", f["colors"]), ("alphas", f["alphas"])):
        a = g[name].cpu().numpy().astype(np.float64)
        report[name] = float((np.abs(a - ref)[good]).max(initial=0) / (RTOL * np.abs(ref).max()))
    for k, bk in (("means", "v_means"), ("quats", "v_quats"), ("scales", "v_scales"), ("opacities", "v_opac"),
                  ("sh", "v_sh")):
        report[bk] = close_except(t[k].grad, b[bk], involved, f"{key}: {bk}", rtol=grad_rtol)
    print(f"[{key}] errors in tolerance units (gradients: {grad_rtol:g}): " + ", ".join(f"{k}={v:.3g}" for k, v in report.items()))
    return g, report


@pytest.mark.gpu
@pytest.mark.parametrize("regime", list(REGIMES))
def test_blend_ladder_forward_backward_match_oracle(cuda, regime):
    sc, V, K, W, H, counts, _ = ladder(regime)
    _rasterize_and_compare(sc, V, K, W, H, regime, cuda, grad_rtol=SATURATED_GRAD_RTOL if regime == "saturate" else RTOL)


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(REGIMES) + ["frame"])
def test_blend_ladder_hit_mask_path(cuda, key):
    """blend_forward(hits=) renders the same bits; blend_backward(hits=) matches the kernel's own culling within 2e-6; the
    last contributor of every covered pixel is marked for its warp."""
    from artdeco_b200 import raster as R
    sc, V, K, W, H = _scene(key)
    st = stages(sc, V, K, W, H, cuda)
    N = len(sc["means"])
    hits = torch.full((max(1, st["n"]),), 0xAB, dtype=torch.uint8, device=cuda)
    col, alp, last = R.blend_forward(W, H, N, st["splats"], st["vals"], st["offs"], hits=hits)
    assert torch.equal(col, st["colors"]) and torch.equal(alp, st["alphas"]) and torch.equal(last, st["last"])
    vc, va = upstream(W, H, 2)
    vcd, vad = vc.to(cuda), va.to(cuda)
    g_own = R.blend_backward(W, H, N, st["splats"], st["vals"], st["offs"], alp, last, vcd, vad)
    g_hit = R.blend_backward(W, H, N, st["splats"], st["vals"], st["offs"], alp, last, vcd, vad, hits=hits)
    assert rel_err(g_hit, g_own) < 2e-6
    lastc, hm = last.cpu().numpy(), hits.cpu().numpy()
    ys, xs = np.nonzero(alp.cpu().numpy() > 0)
    warp = ((ys % 16) // 4) * 2 + ((xs % 16) // 8)
    marked = (hm[lastc[ys, xs]] >> warp) & 1
    assert marked.all(), f"{(marked == 0).sum()} pixels' last contributors are not marked for their warp"


@pytest.mark.gpu
def test_frame_sized_splats_match_oracle(cuda):
    sc, V, K, W, H = frame_sized()
    g, _ = _rasterize_and_compare(sc, V, K, W, H, "frame", cuda)
    rec = g["splats"].cpu().numpy()[len(sc["means"]) - 5:, 7].view(np.uint32)
    assert (rec[1] & 0xffff) == 0xffff and (rec[1] >> 16) == 0xffff and (rec[0] & 0xffff) == 0xffff, \
        "radii above 65535 saturate the 16-bit record fields"


RAGGED = [(1, 1), (15, 1), (17, 33), (33, 17), (70, 50)]


@pytest.mark.gpu
@pytest.mark.parametrize("W,H", RAGGED, ids=[f"{w}x{h}" for w, h in RAGGED])
def test_ragged_frames(cuda, W, H):
    """A 4097-entry list and saturating splats in the ragged corner tile: forward and backward against the oracle, and the
    stage outputs written through out= views into buffers whose sentinels must stay untouched."""
    from artdeco_b200 import raster as R
    sc, V, K, corner = ragged(W, H)
    f = oracle_fwd((W, H))
    assert tile_counts(f, W, H)[corner] >= 4097
    g, _ = _rasterize_and_compare(sc, V, K, W, H, (W, H), cuda, grad_rtol=SATURATED_GRAD_RTOL)
    N = len(sc["means"])
    SENT, PAD = 123.25, 16               # 64 bytes: the views keep the 16-byte alignment the blend's vector accesses need

    def boxed(shape, dtype, fill=SENT):
        n = int(np.prod(shape))
        buf = torch.full((PAD + n + PAD,), fill, dtype=dtype, device=cuda)
        return buf, buf[PAD:PAD + n].view(*shape)

    bc, col = boxed((H, W, 4), torch.float32)
    ba, alp = boxed((H, W), torch.float32)
    bl, last = boxed((H, W), torch.int32, 123)
    R.blend_forward(W, H, N, g["splats"], g["vals"], g["offs"], out=(col, alp, last))
    assert torch.equal(col, g["colors"]) and torch.equal(alp, g["alphas"]) and torch.equal(last, g["last"])
    vc, va = upstream(W, H, 3)
    bv, v_spl = boxed((N, 12), torch.float32)
    v_spl.zero_()
    R.blend_backward(W, H, N, g["splats"], g["vals"], g["offs"], alp, last, vc.to(cuda), va.to(cuda), out=v_spl)
    ref = R.blend_backward(W, H, N, g["splats"], g["vals"], g["offs"], alp, last, vc.to(cuda), va.to(cuda))
    assert rel_err(v_spl, ref) < 2e-6
    for buf, fill in ((bc, SENT), (ba, SENT), (bl, 123), (bv, SENT)):
        assert (buf[:PAD] == fill).all() and (buf[-PAD:] == fill).all(), "a sentinel was overwritten"
    # a view one float off the 16-byte grid is refused before any launch
    from artdeco_b200._lib import ArtdecoB200Error
    odd = torch.zeros(H * W * 4 + 1, device=cuda)[1:].view(H, W, 4)
    with pytest.raises(ArtdecoB200Error, match="16-byte aligned"):
        R.blend_forward(W, H, N, g["splats"], g["vals"], g["offs"], out=(odd, alp, last))
    with pytest.raises(ArtdecoB200Error, match="16-byte aligned"):
        R.blend_backward(W, H, N, g["splats"], g["vals"], g["offs"], alp, last, odd, va.to(cuda), out=v_spl)


def test_blend_entry_points_refuse_misaligned_records_and_outputs():
    """The blend kernels read records and upstream colours as float4, store colours as float4 and accumulate with
    red.global.add.v4: each of those buffers off the 16-byte grid is refused with status 1 before any CUDA call."""
    import ctypes
    from artdeco_b200 import _lib
    import artdeco_b200  # noqa: F401  (registers every signature)
    L = _lib.lib()
    ok, odd = ctypes.c_void_p(256), ctypes.c_void_p(256 + 4)     # never dereferenced

    def refused(rc):
        msg = L.adb_last_error()
        return rc == 1 and msg is not None and "16-byte aligned" in msg.decode()

    fwd = lambda sp, col, hm: L.adb_raster_blend_fwd(16, 16, 8, sp, ok, ok, col, ok, ok, hm, None)
    bwd = lambda sp, vc, vs, hm: L.adb_raster_blend_bwd(16, 16, 8, sp, ok, ok, ok, ok, vc, ok, vs, hm, None)
    for hm in (None, ok):
        assert refused(fwd(odd, ok, hm)) and refused(fwd(ok, odd, hm))
        assert refused(bwd(odd, ok, ok, hm)) and refused(bwd(ok, odd, ok, hm)) and refused(bwd(ok, ok, odd, hm))
    assert refused(L.adb_raster_blend_fwd_multi(8, 2, 16, 16, odd, ok, ok, ok, ok, ok, None, None))
    assert refused(L.adb_raster_blend_fwd_multi(8, 2, 16, 16, ok, ok, ok, odd, ok, ok, None, None))
    assert refused(L.adb_raster_blend_bwd_multi(8, 2, 16, 16, ok, ok, ok, ok, ok, ok, ok, odd, None, None))


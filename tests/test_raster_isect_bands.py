"""The band scatter of the tile intersection (adb_raster_tile_band_scatter_sort and its multi-view form): sorted values,
keys, offsets, totals and overflow flags against the C oracle at the edges of its two passes — empty tile rows, views with
nothing visible, N = 0 and 1, a splat covering every tile row, a tile beyond the shared-memory sort, frames that are not a
multiple of the tile, the Inria rectangle (against the PyTorch reference), C = 1 and 8, and capacities cut on and inside
a tile row, with canary words past every buffer.  Also: two runs are bitwise equal, and a graph replay equals the eager
call."""
import ctypes

import numpy as np
import pytest
import torch

import oracle
from artdeco_b200 import synthetic
from oracle import legacy_torch, raster_torch

TILE = 16
CANARY = 0x5A5A5A5A


def _records(N, W, H, seed, rows=None, frame_splat=False, dense=0):
    """Hand-made projection records: radii [N,2], splats [N,12] (mean at 0..1, depth at 11), tiles_per_gauss from the oracle.
    rows = (lo, hi): centres only in those pixel rows (the other tile rows stay empty); dense: Gaussians in one tile."""
    rng = np.random.default_rng(seed)
    lo, hi = rows if rows else (-24.0, H + 24.0)
    means = np.stack([rng.uniform(-24.0, W + 24.0, N), rng.uniform(lo, hi, N)], 1).astype(np.float32)
    radii = rng.integers(0, 40, (N, 2)).astype(np.int32)
    radii[rng.random(N) < 0.1] = 0                                    # culled
    depth = rng.choice(np.float32([1.5, 2.0, 2.0, 3.25]), N) + np.float32(0.125) * rng.integers(0, 3, N)
    if dense:
        k = min(dense, N)
        means[:k] = np.float32([W * 0.5 + 3.0, H * 0.5 + 5.0])
        radii[:k] = 2
    if frame_splat and N:
        means[N // 2] = np.float32([W / 2, H / 2])
        radii[N // 2] = max(W, H)
    splats = np.zeros((N, 12), np.float32)
    splats[:, 0:2] = means
    splats[:, 11] = depth.astype(np.float32)
    tpg, keys, vals, offs = oracle.isect(radii, means, depth.astype(np.float32), W, H)
    return dict(radii=radii, splats=splats, tpg=tpg, keys=keys, vals=vals, offs=np.append(offs, len(keys)))


def _dev(rec, dev):
    return {k: torch.from_numpy(np.ascontiguousarray(rec[k])).to(dev) for k in ("radii", "splats", "tpg")}


def _count(L, d, W, H, counts, legacy=0):
    """Fills one view's tile counters (the projection's counting, done from the records)."""
    from artdeco_b200 import _lib
    T = counts.numel() // 8
    tmp = torch.empty(T + 1, dtype=torch.int32, device=counts.device)
    N = d["radii"].shape[0]
    if N:
        assert L.adb_raster_tile_count_scan(N, _lib.ptr(d["radii"]), _lib.ptr(d["splats"]), _lib.ptr(d["tpg"]), W, H, legacy,
                                            0, _lib.ptr(counts), _lib.ptr(tmp), None, None, _lib.stream()) == 0


def _multi(recs, W, H, dev, capacities=None):
    from artdeco_b200 import _lib
    from artdeco_b200 import raster as R
    L = _lib.lib()
    Cn, N = len(recs), recs[0]["radii"].shape[0]
    ds = [_dev(r, dev) for r in recs]
    radii = torch.stack([d["radii"] for d in ds]).contiguous()
    splats = torch.stack([d["splats"] for d in ds]).contiguous()
    tpg = torch.stack([d["tpg"] for d in ds]).contiguous()
    counts = R.new_tile_counts(W, H, dev, Cn)
    for c in range(Cn):
        _count(L, ds[c], W, H, counts[c])
    keys, vals, offs, info, seg = R.intersect_multi(radii, splats, tpg, W, H, counts, capacities=capacities)
    assert not bool(counts[:, : counts.shape[1] // 2].any()), "the tile counters return to zero"
    return keys, vals, offs, info, seg


def _tile_bits(W, H):
    return (((W + 15) // 16) * ((H + 15) // 16)).bit_length()


def _check_multi(recs, W, H, keys, vals, offs, info, seg):
    N = recs[0]["radii"].shape[0]
    tb = _tile_bits(W, H)
    assert info["overflow"].tolist() == [0] * len(recs)
    assert info["n_isect"].tolist() == [len(r["keys"]) for r in recs]
    for c, r in enumerate(recs):
        base, n = sum(seg[:c]), len(r["keys"])
        assert np.array_equal(offs[c].cpu().numpy() - base, r["offs"]), f"view {c}: offsets"
        assert np.array_equal(vals[base:base + n].cpu().numpy() - c * N, r["vals"]), f"view {c}: vals"
        assert np.array_equal(keys[base:base + n].cpu().numpy(), r["keys"] | (c << (32 + tb))), f"view {c}: keys"


def test_band_entry_points_refuse_bad_arguments_before_touching_the_device():
    from artdeco_b200 import _lib
    import artdeco_b200  # noqa: F401
    L = _lib.lib()

    def refused(rc, needle, status=1):
        msg = L.adb_last_error()
        return rc == status and msg is not None and needle in msg.decode()

    dummy = ctypes.c_void_p(16)
    caps = (ctypes.c_longlong * 2)(100, 100)
    huge = (ctypes.c_longlong * 2)(2_000_000_000, 2_000_000_000)     # the int32 offsets cannot address their sum
    nb = ctypes.c_size_t(0)
    assert L.adb_raster_tile_band_scratch_bytes(100, ctypes.byref(nb)) == 0 and nb.value == 1200
    assert refused(L.adb_raster_tile_band_scratch_bytes(-1, ctypes.byref(nb)), "adb_raster_tile_band_scratch_bytes")
    ss = L.adb_raster_tile_band_scatter_sort
    assert refused(ss(8, dummy, dummy, dummy, 64, 64, 0, 0, 1, 100, dummy, dummy, dummy, None, 1200, dummy, dummy, None),
                   "adb_raster_tile_band_scatter_sort: null pointer")
    assert refused(ss(8, dummy, dummy, dummy, 64, 64, 0, 1, 1, 100, dummy, dummy, dummy, dummy, 1200, dummy, dummy, None),
                   "adb_raster_tile_band_scatter_sort: bad sizes")
    assert refused(ss(8, dummy, dummy, dummy, 64, 64, 0, 0, 1, 100, dummy, dummy, dummy, dummy, 1199, dummy, dummy, None),
                   "scratch too small", status=3)
    assert refused(ss(8, dummy, dummy, dummy, 65552, 64, 0, 0, 1, 100, dummy, dummy, dummy, dummy, 1200, dummy, dummy,
                      None), "W and H must be at most 65536")
    sm = L.adb_raster_tile_band_scatter_sort_multi
    assert refused(sm(8, 0, dummy, dummy, dummy, 64, 64, caps, dummy, dummy, dummy, dummy, 2400, None, dummy, None),
                   "adb_raster_tile_band_scatter_sort_multi")
    assert refused(sm(8, 2, dummy, dummy, dummy, 64, 64, huge, dummy, dummy, dummy, dummy, 2400, None, dummy, None),
                   "adb_raster_tile_band_scatter_sort_multi: capacities")
    assert refused(sm(8, 2, dummy, dummy, dummy, 64, 64, caps, dummy, dummy, dummy, None, 2400, None, dummy, None),
                   "adb_raster_tile_band_scatter_sort_multi: null pointer")
    assert refused(sm(8, 2, dummy, dummy, dummy, 64, 64, caps, dummy, dummy, dummy, dummy, 2400, None, None, None),
                   "adb_raster_tile_band_scatter_sort_multi: null pointer")                      # vals are required
    assert refused(sm(8, 2, dummy, dummy, dummy, 64, 64, caps, dummy, dummy, dummy, dummy, 2399, None, dummy, None),
                   "scratch too small", status=3)
    assert sm(0, 2, None, None, None, 64, 64, caps, None, None, None, None, 0, None, None, None) == 0    # N = 0: no launch


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 8])
@pytest.mark.parametrize("W,H", [(200, 120), (333, 197), (256, 128)])
def test_multi_view_matches_the_oracle(cuda, C, W, H):
    """View 0 random; then (C = 8) empty bottom rows, nothing visible, a frame-sized splat, a tile beyond 4096 entries."""
    N = 6000
    recs = [_records(N, W, H, seed=11)]
    if C == 8:
        recs.append(_records(N, W, H, seed=12, rows=(0.0, H * 0.3)))
        r = _records(N, W, H, seed=13)
        r["radii"][:] = 0
        recs.append(_records_from(r, W, H))
        recs.append(_records(N, W, H, seed=14, frame_splat=True))
        recs.append(_records(N, W, H, seed=15, dense=5000))
        recs += [_records(N, W, H, seed=16 + k) for k in range(3)]
    assert C == len(recs)
    _check_multi(recs, W, H, *_multi(recs, W, H, cuda))
    if C == 8:
        assert len(recs[2]["keys"]) == 0 and np.diff(recs[4]["offs"]).max() > 4096


def _records_from(r, W, H):
    tpg, keys, vals, offs = oracle.isect(r["radii"], r["splats"][:, 0:2], r["splats"][:, 11], W, H)
    return dict(r, tpg=tpg, keys=keys, vals=vals, offs=np.append(offs, len(keys)))


@pytest.mark.gpu
@pytest.mark.parametrize("N", [0, 1])
def test_zero_and_one_gaussian(cuda, N):
    from artdeco_b200 import raster as R
    W, H = 200, 120
    rec = _records(N, W, H, seed=3)
    if N == 1:
        rec["radii"][:] = 20
        rec = _records_from(rec, W, H)
    d = _dev(rec, cuda)
    keys, vals, offs, n = R.intersect(d["radii"], d["splats"], d["tpg"], W, H)
    assert n == len(rec["keys"]) and np.array_equal(offs.cpu().numpy(), rec["offs"])
    assert np.array_equal(keys.cpu().numpy(), rec["keys"]) and np.array_equal(vals.cpu().numpy(), rec["vals"])
    keys, vals, offs, info, seg = _multi([rec, rec], W, H, cuda, capacities=[64, 64])
    if N == 0:
        assert seg == [0, 0] and vals.numel() == 0 and not offs.any()
    else:
        assert info["n_isect"].tolist() == [n, n] and info["overflow"].tolist() == [0, 0]
        for c in range(2):
            o = offs[c].cpu().numpy() - 64 * c
            assert np.array_equal(o, rec["offs"])
            assert np.array_equal(vals[64 * c:64 * c + n].cpu().numpy() - c, rec["vals"])


@pytest.mark.gpu
def test_inria_rectangle_through_the_single_view_entry_point(cuda):
    from artdeco_b200 import raster as R
    N, W, H = 20000, 333, 197
    sc = synthetic.raster_scene(N, seed=4)
    V, K = synthetic.camera(W, H, view=1.0)
    t = {k: sc[k].to(cuda) for k in ("means", "quats", "scales", "opacities", "sh")}
    P = torch.inverse(V.to(cuda))[:3, 3].contiguous()
    radii, splats, tpg = R.project(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], 3, V.to(cuda), K.to(cuda),
                                   P, W, H, 0.01, 0.01, 1e10, 0.0, legacy=True)
    kb, vb, ob, nb = R.intersect(radii, splats, tpg, W, H, cam_id=1, n_cams=2, legacy=True)
    # CPU reference: the gsplat key layout and stable sort over the Inria rectangle; a Gaussian the projection gave no
    # tiles (opacity below 1/255) emits no keys
    r, sp, t = radii.cpu(), splats.cpu(), tpg.cpu()
    rect = lambda i, tw, th: legacy_torch._rect(sp[:, 0:2], r[:, 0], i, tw, th) if t[i] > 0 else None
    kr, vr, orr = raster_torch.isect_and_sort(r, sp[:, 0:2], sp[:, 11], W, H, cam_id=1, n_cams=2, rect_fn=rect)
    assert nb == len(kr) > 0
    assert torch.equal(kb.cpu(), kr) and torch.equal(vb.cpu(), vr)
    assert torch.equal(ob.cpu(), torch.cat([orr, torch.tensor([nb], dtype=torch.int32)]))


def _single_raw(rec, W, H, dev, capacity, tail=64):
    """One view through the C entry points with `tail` canary words past packed, keys, vals and both scratch arrays."""
    from artdeco_b200 import _lib
    L = _lib.lib()
    d = _dev(rec, dev)
    N = d["radii"].shape[0]
    T = ((W + 15) // 16) * ((H + 15) // 16)
    counts = torch.zeros(8 * T, dtype=torch.int32, device=dev)
    offs = torch.empty(T + 1, dtype=torch.int32, device=dev)
    total = torch.zeros(1, dtype=torch.int64, device=dev)
    ovf = torch.zeros(1, dtype=torch.int32, device=dev)
    assert L.adb_raster_tile_count_scan(N, _lib.ptr(d["radii"]), _lib.ptr(d["splats"]), _lib.ptr(d["tpg"]), W, H, 0, capacity,
                                        _lib.ptr(counts), _lib.ptr(offs), _lib.ptr(total), _lib.ptr(ovf), _lib.stream()) == 0
    # one int32 buffer per array: [capacity entries | tail canaries]
    packed = torch.full((2 * (capacity + tail),), CANARY, dtype=torch.int32, device=dev)
    keys = torch.full((2 * (capacity + tail),), CANARY, dtype=torch.int32, device=dev)
    vals = torch.full((capacity + tail,), CANARY, dtype=torch.int32, device=dev)
    # scratch: pair words [capacity] u64 then pair columns [capacity] u32, canaries after both
    nb = ctypes.c_size_t(0)
    assert L.adb_raster_tile_band_scratch_bytes(capacity, ctypes.byref(nb)) == 0 and nb.value == 12 * capacity
    scratch = torch.full((3 * capacity + tail,), CANARY, dtype=torch.int32, device=dev)
    rc = L.adb_raster_tile_band_scatter_sort(N, _lib.ptr(d["radii"]), _lib.ptr(d["splats"]), _lib.ptr(d["tpg"]), W, H, 0, 0, 1,
                                             capacity, _lib.ptr(counts), _lib.ptr(offs), _lib.ptr(packed), _lib.ptr(scratch),
                                             nb.value, _lib.ptr(keys), _lib.ptr(vals), _lib.stream())
    assert rc == 0, L.adb_last_error()
    torch.cuda.synchronize()
    canaries_ok = all(bool((b[-t:] == CANARY).all()) for b, t in ((packed, 2 * tail), (keys, 2 * tail), (vals, tail),
                                                                  (scratch, tail)))
    assert not bool(counts[:4 * T].any()), "the tile counters return to zero"
    return dict(keys=keys[:2 * capacity].view(torch.int64), vals=vals[:capacity], offs=offs, total=int(total),
                overflow=int(ovf), canaries_ok=canaries_ok)


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["exact", "on_row_boundary", "inside_row", "inside_dense_tile"])
def test_capacity_cut_is_memory_safe_flagged_and_leaves_whole_tiles_exact(cuda, where):
    W, H = 333, 197
    tw = (W + 15) // 16
    rec = _records(8000, W, H, seed=21, dense=5000)
    ref = rec["offs"]
    n = len(rec["keys"])
    row = 5
    big = int(np.argmax(np.diff(ref)))
    cap = {"exact": n, "on_row_boundary": int(ref[row * tw]), "inside_row": int(ref[row * tw + tw // 2]) + 3,
           "inside_dense_tile": int(ref[big]) + 3000}[where]
    assert 0 < cap <= n
    g = _single_raw(rec, W, H, cuda, cap)
    assert g["canaries_ok"], "written past the capacity"
    assert g["total"] == n and g["overflow"] == int(cap < n)
    offs = g["offs"].cpu().numpy()
    assert np.array_equal(offs, np.minimum(ref, cap))
    whole = int(ref[np.searchsorted(ref, cap, side="right") - 1])      # entries of the tiles the cut leaves whole
    assert np.array_equal(g["keys"][:whole].cpu().numpy(), rec["keys"][:whole])
    assert np.array_equal(g["vals"][:whole].cpu().numpy(), rec["vals"][:whole])
    v = g["vals"].cpu().numpy()
    assert ((v >= 0) & (v < 8000)).all(), "every slot below the capacity holds a Gaussian of the view"


@pytest.mark.gpu
def test_multi_view_capacity_flags_only_the_cut_view(cuda):
    W, H = 333, 197
    tw = (W + 15) // 16
    recs = [_records(6000, W, H, seed=31 + c) for c in range(3)]
    n = [len(r["keys"]) for r in recs]
    caps = [n[0] + 100, int(recs[1]["offs"][7 * tw]) + 5, n[2]]
    keys, vals, offs, info, seg = _multi(recs, W, H, cuda, capacities=caps)
    assert info["n_isect"].tolist() == n and info["overflow"].tolist() == [0, 1, 0]
    for c in (0, 2):
        base = sum(caps[:c])
        assert np.array_equal(offs[c].cpu().numpy() - base, recs[c]["offs"])
        assert np.array_equal(vals[base:base + n[c]].cpu().numpy() - c * 6000, recs[c]["vals"])
    o1 = offs[1].cpu().numpy() - caps[0]
    assert np.array_equal(o1, np.minimum(recs[1]["offs"], caps[1]))
    v1 = vals[caps[0]:caps[0] + caps[1]].cpu().numpy() - 6000
    assert ((v1 >= 0) & (v1 < 6000)).all()


@pytest.mark.gpu
def test_two_runs_are_bitwise_equal_and_a_graph_replay_equals_the_eager_call(cuda):
    from artdeco_b200 import raster as R
    N, W, H, views = 30000, 480, 272, (0.5, 2.0, 4.5)
    sc = synthetic.raster_scene(N, seed=5)
    cams = [synthetic.camera(W, H, view=v) for v in views]
    Vs = torch.stack([c[0] for c in cams]).to(cuda)
    Ks = torch.stack([c[1] for c in cams]).to(cuda)
    P = torch.inverse(Vs)[:, :3, 3].contiguous()
    t = {k: sc[k].to(cuda) for k in ("means", "quats", "scales", "opacities", "sh")}
    counts = R.new_tile_counts(W, H, cuda, len(views))

    def run(caps):
        counts.zero_()
        radii, splats, tpg = R.project_multi(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], 3, Vs, Ks, P, W, H,
                                             0.01, 0.01, 1e10, 0.0, counts)
        return R.intersect_multi(radii, splats, tpg, W, H, counts, capacities=caps)

    k1, v1, o1, i1, seg = run(None)
    k2, v2, o2, _, _ = run(None)
    assert torch.equal(k1, k2) and torch.equal(v1, v2) and torch.equal(o1, o2)
    caps = [s + 1000 for s in seg]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run(caps)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        kg, vg, og, ig, _ = run(caps)
    eager = [x.clone() for x in run(caps)[:3]]
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(og, eager[2]) and not bool(ig["overflow"].any()) and ig["n_isect"].tolist() == seg
    for c in range(len(views)):                       # entries past a view's count are undefined
        b0, b1 = sum(seg[:c]), sum(caps[:c])
        assert torch.equal(kg[b1:b1 + seg[c]], eager[0][b1:b1 + seg[c]]) and torch.equal(kg[b1:b1 + seg[c]], k1[b0:b0 + seg[c]])
        assert torch.equal(vg[b1:b1 + seg[c]], eager[1][b1:b1 + seg[c]]) and torch.equal(vg[b1:b1 + seg[c]], v1[b0:b0 + seg[c]])
        assert torch.equal(og[c] - b1, o1[c] - b0)

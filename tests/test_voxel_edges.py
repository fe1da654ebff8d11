"""update_voxel where an integer kernel goes wrong: exact voxel boundaries, hash-table load, vote ties, class-id and extent
limits.  Every GPU case is bit-exact against oracle/voxel_ref.py.

The reference computes ``floor((p - min) / voxel_size)`` on CUDA tensors with a Python-float divisor, which PyTorch's CUDA
kernel evaluates as ``(p - min) * fl32(1 / voxel_size)``.  For a few fp32 values per voxel size that lands in a different
voxel than a correctly rounded division (``1.3f / 0.1f = 12.999999`` but ``1.3f * 10 = 13``).  Uniform random clouds hit
such a value a few times per million points, so the boundary finder below enumerates them exhaustively and the GPU cases
put points exactly there, with the classes arranged so that the voxel choice changes the result."""
import functools

import numpy as np
import pytest
import torch

from oracle import voxel_ref

VOXEL_SIZES = (0.1, 0.05, 0.025, 0.3, 0.07)        # 0.3 and 0.07 have inexact fp32 reciprocals
D_RANGE = (1e-3, 7.0)


@functools.lru_cache(maxsize=None)
def boundary_values(voxel_size, lo=D_RANGE[0], hi=D_RANGE[1]):
    """Every fp32 d in [lo, hi] with floor(d / vs) != floor(d * fl32(1 / vs)), vs = fl32(voxel_size); exhaustive over the
    bit patterns (positive floats order like their bits)."""
    v = np.float32(voxel_size)
    inv = np.float32(1.0) / v
    b0, b1 = (int(np.array(x, np.float32).view(np.uint32)) for x in (lo, hi))
    found = []
    for s in range(b0, b1 + 1, 1 << 22):
        d = np.arange(s, min(s + (1 << 22), b1 + 1), dtype=np.uint32).view(np.float32)
        found.append(d[np.floor(d / v) != np.floor(d * inv)])
    return np.concatenate(found)


def div_index(d, voxel_size):
    return np.floor(d / np.float32(voxel_size)).astype(np.int64)


def rcp_index(d, voxel_size):
    return np.floor(d * (np.float32(1.0) / np.float32(voxel_size))).astype(np.int64)


def mid(k, voxel_size):
    """fp32 centre of voxel k along an axis whose minimum is 0: half a voxel from either face under both roundings."""
    return (np.float32(k) + np.float32(0.5)) * np.float32(voxel_size)


def with_ulp_neighbours(b):
    return np.concatenate([b, np.nextafter(b, np.float32(0)), np.nextafter(b, np.float32(np.inf))])


def run(new, xyz, cls, vs, dev):
    from artdeco_b200.voxel import update_voxel
    return update_voxel(new.to(dev), xyz.to(dev), cls.to(dev), vs)


def assert_same(out, ref, what):
    assert len(out) == len(ref), what
    if len(ref) == 2:                                              # cold start: (ids, voxel count)
        got, want = out[0].cpu(), ref[0]
        assert out[1] == ref[1], f"{what}: {out[1]} new voxels, oracle {ref[1]}"
        assert got.dtype == torch.long and got.shape == want.shape
        assert torch.equal(got, want), f"{what}: {int((got != want).sum())} new-point class ids differ"
        return
    assert out[2] == ref[2], f"{what}: {out[2]} new voxels, oracle {ref[2]}"
    for name, got, want in (("original", out[0].cpu(), ref[0]), ("new", out[1].cpu(), ref[1])):
        assert got.dtype == torch.long and got.shape == want.shape, (what, name, got.shape, want.shape)
        bad = (got != want).reshape(-1)
        assert not bad.any(), f"{what}: {int(bad.sum())} {name}-point class ids differ, first at row {int(bad.nonzero()[0])}"


def oracle_by_division(monkeypatch, new, xyz, cls, vs):
    """The oracle with the voxel index taken by a correctly rounded fp32 division: what a kernel that divides computes."""
    with monkeypatch.context() as m:
        m.setattr(voxel_ref, "_vidx", lambda p, mn, v: torch.from_numpy(div_index((p - mn).numpy(), v)))
        return voxel_ref.update_voxel(new, xyz, cls, vs)


# ------------------------------------------------------------------ CPU ------------------------------------------------------

@pytest.mark.parametrize("vs", VOXEL_SIZES)
def test_boundary_finder_finds_values_one_voxel_apart(vs):
    b = boundary_values(vs)
    assert len(b) > 0, "no boundary value: the GPU boundary cases would test nothing"
    assert (np.abs(rcp_index(b, vs) - div_index(b, vs)) == 1).all()
    # the oracle's voxel index is the reciprocal form
    assert torch.equal(voxel_ref._vidx(torch.from_numpy(b), torch.zeros(()), vs), torch.from_numpy(rcp_index(b, vs)))
    if vs == 0.1:
        assert len(b) == 15 and {float(np.float32(x)) for x in (1.3, 5.2, 5.7)} <= set(b.tolist())
    # both directions occur: 0.07's reciprocal rounds down where the division rounds up
    up = rcp_index(b, vs) > div_index(b, vs)
    assert up.all() if vs != 0.07 else not up.any()


def test_class_ids_must_fit_32_bits():
    """The kernels carry class ids as 32-bit values (the vote packs count << 32 | 0xffffffff - id): update_voxel reads
    the largest id anyway (the reference's own max().item()) and refuses one at or above 2^32 - 1."""
    from artdeco_b200 import _lib
    from artdeco_b200.voxel import max_class_id
    assert max_class_id(torch.tensor([[3], [2 ** 32 - 2], [0]])) == 2 ** 32 - 2
    for bad in (2 ** 32 - 1, 2 ** 32, 2 ** 40 + 5):
        with pytest.raises(_lib.ArtdecoB200Error, match="class id"):
            max_class_id(torch.tensor([[1], [bad]]))


# ------------------------------------------------------------------ GPU: the premise --------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("vs", VOXEL_SIZES)
def test_torch_cuda_divides_by_a_python_float_through_the_reciprocal(cuda, vs):
    """The reference's own expression on the device agrees with the oracle's reciprocal form on every boundary value and its
    neighbours, and disagrees with a division on the boundary values themselves."""
    d = with_ulp_neighbours(boundary_values(vs))
    p = torch.from_numpy(np.stack([d, np.zeros_like(d), d], 1))
    p = torch.cat([torch.zeros(1, 3), p])                         # the origin makes min = 0, so p - min = p
    p_dev = p.to(cuda)
    got = torch.floor((p_dev - p_dev.min(dim=0).values) / vs).long().cpu()
    assert torch.equal(got, voxel_ref._vidx(p, p.min(dim=0).values, vs))
    nb = len(boundary_values(vs))
    assert (got[1: nb + 1, 0].numpy() != div_index(d[:nb], vs)).all()


# ------------------------------------------------------------------ GPU: boundaries -----------------------------------------

def boundary_scene(vs, cold):
    """Points on every boundary value b of ``vs`` and on b +- 1 ulp, one row of voxels (y) per value, x carrying the value.
    With lo < hi the two voxels b falls in under division and reciprocal:
      * vote row (warm only): 2 points of class A in the middle of voxel lo, 2 of class B in voxel hi, 3 of class C at x;
        C wins whichever voxel x is counted in, and the other voxel keeps its own class;
      * match row: one point in voxel lo (original, or new when cold) and a new point at x: x is matched or opens voxel hi;
      * a new point far out in x in every match row: unmatched either way, its class id is max_cls + 1 + the rank of its voxel
        among all unmatched voxels, which counts the boundary points that opened one.
    The origin is a point, so min = 0 and p - min = p exactly.  Returns (new, xyz, cls) as CPU tensors."""
    b = boundary_values(vs)
    lo = np.minimum(rcp_index(b, vs), div_index(b, vs))
    xs, los = with_ulp_neighbours(b), np.tile(lo, 3)
    far = mid(int(D_RANGE[1] / vs) + 4, vs)
    z = mid(0, vs)
    xyz, cls, new = [(0.0, 0.0, 0.0)], [0], []
    if cold:
        new.append((0.0, 0.0, 0.0))
    row, c = 0, 1
    for x, k in zip(xs, los):
        if not cold:
            row += 1
            y = mid(row, vs)
            for px, n, cl in ((mid(k, vs), 2, c), (mid(k + 1, vs), 2, c + 1), (x, 3, c + 2)):
                xyz += [(px, y, z)] * n
                cls += [cl] * n
            c += 3
        row += 1
        y = mid(row, vs)
        if cold:
            new.append((mid(k, vs), y, z))
        else:
            xyz.append((mid(k, vs), y, z))
            cls.append(c)
            c += 1
        new += [(x, y, z), (far, y, z)]
    as_f32 = lambda p: torch.from_numpy(np.asarray(p, np.float32).reshape(-1, 3))
    if cold:
        return as_f32(new), as_f32(np.zeros((0, 3))), torch.zeros(0, 1, dtype=torch.long)
    return as_f32(new), as_f32(xyz), torch.tensor(cls, dtype=torch.long)[:, None]


@pytest.mark.gpu
@pytest.mark.parametrize("cold", [False, True], ids=["warm", "cold"])
@pytest.mark.parametrize("vs", VOXEL_SIZES)
def test_update_voxel_at_voxel_boundaries(cuda, monkeypatch, vs, cold):
    new, xyz, cls = boundary_scene(vs, cold)
    ref = voxel_ref.update_voxel(new, xyz, cls, vs)
    div = oracle_by_division(monkeypatch, new, xyz, cls, vs)
    # the scene is built so that dividing changes the result: counts, majorities and matches all flip
    assert ref[-1] != div[-1]
    for r, d in zip(ref[:-1], div[:-1]):
        assert not torch.equal(r, d)
    assert_same(run(new, xyz, cls, vs, cuda), ref, f"voxel {vs} {'cold' if cold else 'warm'} boundaries")


# ------------------------------------------------------------------ GPU: hash tables and the vote ----------------------------

def lattice(nx, ny, nz, vs):
    """One point per voxel centre of an nx x ny x nz block; the first point sits at the origin (same voxel) so min = 0."""
    i = np.arange(nx * ny * nz)
    p = np.stack([mid(i // (ny * nz), vs), mid(i // nz % ny, vs), mid(i % nz, vs)], 1).astype(np.float32)
    p[0] = 0.0
    return torch.from_numpy(p)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(16, 8, 8), (128, 128, 64)], ids=["1024", "1M"])
def test_power_of_two_n_with_every_point_in_its_own_voxel(cuda, shape):
    """N = 2^k distinct voxels: the voxel and pair tables get exactly 2N slots, load factor 0.5."""
    from artdeco_b200.voxel import _pow2
    vs = 0.1
    xyz = lattice(*shape, vs)
    N = xyz.shape[0]
    assert N & (N - 1) == 0 and _pow2(2 * N) == 2 * N
    g = torch.Generator().manual_seed(N)
    cls = torch.randint(0, 1 << 20, (N, 1), generator=g)
    # new points: jittered inside lattice voxels (matched) and beyond the block in x (unmatched, duplicated)
    M = max(N // 4, 8)
    hit = xyz[torch.randint(1, N, (M // 2,), generator=g)] + (torch.rand(M // 2, 3, generator=g) - 0.5) * 0.6 * vs
    out_i = torch.randint(0, 64, (M - M // 2,), generator=g)
    miss = torch.stack([torch.from_numpy(mid(shape[0] + out_i.numpy() % 8, vs)),
                        torch.from_numpy(mid(out_i.numpy() // 8, vs)), torch.full((M - M // 2,), float(mid(1, vs)))], 1)
    new = torch.cat([hit, miss])[torch.randperm(M, generator=g)]
    ref = voxel_ref.update_voxel(new, xyz, cls, vs)
    assert torch.equal(ref[0], cls) and 0 < ref[2] <= 64
    assert_same(run(new, xyz, cls, vs, cuda), ref, f"lattice {shape}")


@pytest.mark.gpu
def test_tied_counts_in_one_voxel_give_the_smallest_id(cuda):
    xyz = torch.rand(10, 3, generator=torch.Generator().manual_seed(0)) * 0.09
    cls = torch.tensor([9, 9, 4, 12, 4, 7, 7, 12, 30, 5])[:, None]   # 9, 4, 7, 12 twice each
    new = xyz[:3] + 0.001
    ref = voxel_ref.update_voxel(new, xyz, cls, 0.1)
    assert ref[0].unique().tolist() == [4] and ref[1].unique().tolist() == [4] and ref[2] == 0
    assert_same(run(new, xyz, cls, 0.1, cuda), ref, "tie")


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["N1_M1_hit", "N1_M1_miss", "N1_M0", "N0_M1"])
def test_single_points(cuda, case):
    xyz = torch.tensor([[0.25, -1.0, 3.0]])
    cls = torch.tensor([[17]])
    new = {"N1_M1_hit": xyz + 0.01, "N1_M1_miss": xyz + 1.0, "N1_M0": xyz[:0], "N0_M1": xyz}[case]
    if case == "N0_M1":
        xyz, cls = xyz[:0], cls[:0]
    ref = voxel_ref.update_voxel(new, xyz, cls, 0.1)
    assert_same(run(new, xyz, cls, 0.1, cuda), ref, case)


@pytest.mark.gpu
def test_all_new_points_matched_skips_the_rank_stage(cuda):
    g = torch.Generator().manual_seed(1)
    xyz = torch.rand(5000, 3, generator=g) * 2
    cls = torch.randint(0, 40, (5000, 1), generator=g)
    new = xyz[torch.randint(0, 5000, (3000,), generator=g)]
    ref = voxel_ref.update_voxel(new, xyz, cls, 0.1)
    assert ref[2] == 0
    assert_same(run(new, xyz, cls, 0.1, cuda), ref, "all matched")


@pytest.mark.gpu
def test_all_new_points_unmatched_and_duplicated(cuda):
    g = torch.Generator().manual_seed(2)
    xyz = torch.rand(4000, 3, generator=g)
    cls = torch.randint(0, 25, (4000, 1), generator=g)
    far = torch.rand(37, 3, generator=g) * 5 + 1.5                 # outside [0, 1]^3
    new = far.repeat(9, 1)[torch.randperm(37 * 9, generator=g)]
    ref = voxel_ref.update_voxel(new, xyz, cls, 0.1)
    assert ref[1].min() > cls.max() and 0 < ref[2] == len(ref[1].unique()) <= 37
    assert_same(run(new, xyz, cls, 0.1, cuda), ref, "all unmatched")


@pytest.mark.gpu
def test_minimum_taken_from_a_new_point(cuda):
    g = torch.Generator().manual_seed(3)
    xyz = torch.rand(20000, 3, generator=g) * 3
    cls = torch.randint(0, 100, (20000, 1), generator=g)
    new = torch.cat([torch.rand(3000, 3, generator=g) * 3.5, torch.tensor([[-0.537, -0.211, -1.013]])])
    ref = voxel_ref.update_voxel(new, xyz, cls, 0.1)
    assert_same(run(new, xyz, cls, 0.1, cuda), ref, "min from a new point")


@pytest.mark.gpu
def test_class_ids_near_2_31_and_2_32(cuda):
    """The vote keys ties by 0xffffffff - id: ids above 2^31 and the largest accepted one, 2^32 - 2, must still lose ties to
    smaller ids and win on counts; new ids start at max + 1 = 2^32 - 1, beyond 32 bits.  Voxel size 1 on half-integer
    coordinates keeps every index exact."""
    t31, t32 = 2 ** 31, 2 ** 32
    voxels = [[t32 - 2, t32 - 2, t31, t31], [t32 - 2, t32 - 2, t32 - 3], [t31 - 1, t31], [0, t32 - 2], [t32 - 2], [t31 + 1]]
    xyz, cls = [], []
    for v, ids in enumerate(voxels):
        xyz += [(v + 0.5, 0.5, 0.5)] * len(ids)
        cls += ids
    xyz = torch.tensor(xyz)
    cls = torch.tensor(cls)[:, None]
    new = torch.cat([xyz + 0.25, torch.tensor([[v + 0.5, 3.5, 0.5] for v in range(6)])])
    ref = voxel_ref.update_voxel(new, xyz, cls, 1.0)
    assert [int(ref[0][sum(map(len, voxels[:v]))]) for v in range(6)] == [t31, t32 - 2, t31 - 1, 0, t32 - 2, t31 + 1]
    assert ref[1][-6:].squeeze(-1).tolist() == list(range(t32 - 1, t32 + 5))
    assert_same(run(new, xyz, cls, 1.0, cuda), ref, "ids near 2^32")


@pytest.mark.gpu
def test_class_id_of_2_32_minus_1_is_refused(cuda):
    from artdeco_b200 import _lib
    xyz = torch.rand(8, 3)
    with pytest.raises(_lib.ArtdecoB200Error, match="class id"):
        run(xyz, xyz, torch.full((8, 1), 2 ** 32 - 1), 0.1, cuda)


@pytest.mark.gpu
@pytest.mark.parametrize("axis", [0, 1, 2, "all"])
@pytest.mark.parametrize("where", ["orig", "new"])
def test_extent_of_2_21_voxels(cuda, axis, where):
    """Keys pack 21 bits per axis: an index of 2^21 - 1 (all three at once gives the largest key, 2^63 - 1) matches the oracle,
    2^21 raises.  Voxel size 1 keeps every index exact."""
    from artdeco_b200 import _lib
    axes = [0, 1, 2] if axis == "all" else [axis]
    base = torch.tensor([[0.0, 0.0, 0.0], [3.5, 2.5, 1.5], [7.5, 0.5, 4.5]])
    for top, ok in ((2 ** 21 - 1, True), (2 ** 21, False)):
        far = torch.tensor([[2.5, 1.5, 0.5]])
        far[0, axes] = top + 0.5
        xyz, new = (torch.cat([base, far]), base + 0.25) if where == "orig" else (base, torch.cat([base + 0.25, far]))
        cls = torch.arange(xyz.shape[0])[:, None] % 2
        if ok:
            assert_same(run(new, xyz, cls, 1.0, cuda), voxel_ref.update_voxel(new, xyz, cls, 1.0), f"extent {axis} {where}")
        else:
            with pytest.raises(_lib.ArtdecoB200Error, match="2\\^21"):
                run(new, xyz, cls, 1.0, cuda)


@pytest.mark.gpu
def test_two_runs_are_bitwise_equal(cuda):
    g = torch.Generator().manual_seed(4)
    xyz = torch.rand(300_000, 3, generator=g) * 4
    cls = torch.randint(0, 3000, (300_000, 1), generator=g)
    new = torch.rand(100_000, 3, generator=g) * 5 - 0.5
    a, b = run(new, xyz, cls, 0.1, cuda), run(new, xyz, cls, 0.1, cuda)
    assert a[2] == b[2] and torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])

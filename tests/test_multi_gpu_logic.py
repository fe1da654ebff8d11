"""N>1 host logic on CPU: world_size-2 gloo processes exercise the gradient bucket all-reduce and the sharding helpers."""
import os
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from artdeco_b200.parallel import GRAD_FLOATS, GradBucket, shard_pairs, views_for_rank
    N = 1000
    b = GradBucket(N, "cpu")
    g = torch.Generator().manual_seed(rank)
    for name, v in b.views.items():
        v.copy_(torch.randn(v.shape, generator=g))
    mine = {k: v.clone() for k, v in b.views.items()}
    b.all_reduce()
    # reference: regenerate both ranks' tensors locally and sum
    ok = True
    tot = {k: torch.zeros_like(v) for k, v in mine.items()}
    for r in range(world):
        gr = torch.Generator().manual_seed(r)
        for name in b.views:
            tot[name] += torch.randn(b.views[name].shape, generator=gr)
    for name in b.views:
        ok &= bool(torch.allclose(b.views[name], tot[name], atol=1e-6))
    ok &= b.flat.numel() == N * GRAD_FLOATS == N * 59
    ok &= views_for_rank(8, world, rank) == [v for v in range(8) if v % world == rank]
    pairs = list(shard_pairs(7, world, rank))
    gathered = [None] * world
    dist.all_gather_object(gathered, pairs)
    ok &= sorted(sum(gathered, [])) == list(range(7)) and max(map(len, gathered)) - min(map(len, gathered)) <= 1
    # --- config-4 exchange: all-gather of per-view colour gradients + all-reduce of the 11 geometry floats ---
    from artdeco_b200.parallel import GEOM_FLOATS, MultiViewExchange
    Cl = 2
    ex = MultiViewExchange(N, Cl, "cpu")
    ok &= ex.geom.numel() == N * GEOM_FLOATS == N * 11 and ex.g_all.shape == (Cl, world, N, 3)
    gr = torch.Generator().manual_seed(100 + rank)
    g_loc, cam_loc = torch.randn(Cl, N, 3, generator=gr), torch.randn(Cl, 3, generator=gr)
    geo_loc = {k: torch.randn(v.shape, generator=gr) for k, v in ex.views.items()}
    for k, v in ex.views.items():
        v.copy_(geo_loc[k])
    ex.start_gather(g_loc, cam_loc)
    ex.start_reduce()
    g_all, cam_all = ex.wait_gather()
    ex.wait_reduce()
    exp_g, exp_c, exp_geo = [], [], {k: torch.zeros_like(v) for k, v in ex.views.items()}
    for r in range(world):
        g2 = torch.Generator().manual_seed(100 + r)
        exp_g.append(torch.randn(Cl, N, 3, generator=g2))
        exp_c.append(torch.randn(Cl, 3, generator=g2))
        for k in exp_geo:
            exp_geo[k] += torch.randn(exp_geo[k].shape, generator=g2)
    # view-major order: entry (c, r) = local view c of rank r, for the gradients and the camera centres alike
    ok &= torch.equal(g_all, torch.stack(exp_g, 1).reshape(-1, N, 3)) and torch.equal(cam_all, torch.stack(exp_c, 1).reshape(-1, 3))
    # a second step through the per-view entry point gives the same result (state is reset by wait_gather)
    for c in range(Cl):
        ex.start_gather_view(c, g_loc[c], cam_loc if c == 0 else None)
    g2, c2 = ex.wait_gather()
    ok &= torch.equal(g2, g_all) and torch.equal(c2, cam_all)
    for k in exp_geo:
        ok &= bool(torch.allclose(ex.views[k], exp_geo[k], atol=1e-6))
    # the exchange factory: on CPU tensors (gloo) both kinds resolve to the library-collective exchange; unknown kinds are refused
    from artdeco_b200.peer import make_exchange
    ok &= type(make_exchange(N, Cl, "cpu")).__name__ == "MultiViewExchange"
    ok &= type(make_exchange(N, Cl, "cpu", kind="peer")).__name__ == "MultiViewExchange"
    try:
        make_exchange(N, Cl, "cpu", kind="mpi")
        ok = False
    except ValueError:
        pass
    q.put((rank, ok))
    dist.destroy_process_group()


def test_gloo_world2_bucket_allreduce_and_sharding():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 1000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, True), (1, True)]


def test_peer_region_layout_is_aligned_and_disjoint():
    """peer.PeerRegion: every block of a rank's peer-visible region starts on a 256-byte boundary, blocks do not overlap, the
    geometry shards cover the [N,11] block and the colour rows keep the [views, N, 3] stride the expansion kernel expects."""
    from artdeco_b200.parallel import GEOM_FLOATS
    from artdeco_b200.peer import MAXW, N_SLOTS, PeerRegion
    for n, cl, world in [(1_000_000, 1, 8), (1_000_000, 4, 2), (20004, 1, 8), (1000, 2, 3), (4, 1, 1)]:
        L = PeerRegion(n, cl, world)
        rows = cl * world
        blocks = [("flags", L.off_flags, N_SLOTS * MAXW), ("cam0", L.off_cam, rows * 3), ("cam1", L.off_cam + L.cam_stride, rows * 3),
                  ("g0", L.off_g, rows * L.row), ("g1", L.off_g + L.g_stride, rows * L.row),
                  ("stage", L.off_stage, world * L.per4 * 4), ("y", L.off_y, world * L.per4 * 4)]
        end = 0
        for name, off, size in blocks:
            assert off % 64 == 0, f"{name} not 256-byte aligned"
            assert off >= end, f"{name} overlaps the previous block"
            end = off + size
        assert end <= L.words
        assert L.row == 3 * n and L.n4 * 4 >= n * GEOM_FLOATS > (L.n4 - 1) * 4
        assert world * L.per4 >= L.n4 > (world - 1) * L.per4 - world          # every float4 has exactly one owner shard
        assert (L.row * 1) % 4 == 0 or n % 4                                   # rows are float4-addressable when N % 4 == 0


def test_new_hit_mask_has_one_byte_per_intersection():
    """raster.new_hit_mask: one byte per sorted intersection, at least one."""
    from artdeco_b200 import raster as R
    vals = torch.zeros(1000, dtype=torch.int32)
    m = R.new_hit_mask(vals)
    assert m.dtype == torch.uint8 and m.numel() == 1000
    assert R.new_hit_mask(vals[:0]).numel() == 1

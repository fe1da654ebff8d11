"""Key-frame retrieval on the H100: the whole golden sequence (made by running the reference's own retrieval and ASMK
code) through RetrievalDatabase.update, and each stage against the oracle."""
import warnings
from pathlib import Path

import numpy as np
import pytest
import torch

from artdeco_b200 import retrieval as R
from artdeco_b200 import synthetic
from oracle import retrieval_ref as rr

from test_retrieval_cpu import pi3_stub

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden" / "retrieval_small.pt"


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, weights_only=False)


@pytest.fixture(scope="module")
def stream(golden):
    m, P, c = synthetic.retrieval_model(golden["K"], seed=golden["seed"])
    return (m, P, c), synthetic.retrieval_stream(m, P, c, golden["schedule"], n=golden["n"], nfeat=golden["nfeat"],
                                                 seed=golden["seed"])


def _db(model, golden, accurate, windows, **kw):
    m, P, c = model
    db = R.RetrievalDatabase(m, P, c, nfeat=golden["nfeat"], config=golden["config"], accurate_loop_closure=accurate, **kw)
    select = pi3_stub(golden["m_frac"], golden["config"])

    def alc(keyframe_id):
        w = db.window(keyframe_id)
        windows.append(w)
        return select(w)
    db.accurate_loop_closure = alc
    return db


@pytest.mark.parametrize("accurate", [True, False])
def test_golden_sequence(cuda, golden, stream, accurate):
    windows = []
    db = _db(stream[0], golden, accurate, windows, capacity=4)   # grows 4 -> 8 -> 16 -> 32 on the way
    cfg = golden["config"]["retrieval"]
    for u, (fr, want) in enumerate(zip(stream[1], golden["updates"])):
        n_before = len(windows)
        out = db.update(fr["feat"].to(cuda), fr["add"], cfg["k"], cfg["min_thresh"])
        if not accurate:
            assert out == golden["plain_out"][u], u
            continue
        assert out == want["out"], (u, out, want["out"])
        assert (len(windows) > n_before) == want["pi3"], u
        if want["pi3"]:
            assert windows[-1] == want["window"], u
        if want["scores"] is not None:
            assert torch.equal(db.topk_codes.cpu(), want["codes"]), u
            got = db.scores.cpu()
            assert torch.equal(got.view(torch.int64), want["scores"].view(torch.int64)), (u, (got - want["scores"]).abs().max())
    if accurate:
        for u, row in golden["ivf_rows"].items():
            words, sig = db.ivf_row(row["image"])
            assert torch.equal(words.cpu(), row["words"]), u
            assert torch.equal(sig.cpu(), row["sig"]), u


def test_whitening_within_one_ulp(cuda, golden, stream):
    (m, P, c), frames = stream
    db = R.RetrievalDatabase(m, P, c, nfeat=golden["nfeat"])
    x = frames[0]["feat"].to(cuda)
    s = db._state()
    y = torch.empty(x.shape[1], 1024, device=cuda)
    attn = torch.empty(x.shape[1], device=cuda)
    R._lib.call("adb_retrieval_whiten", x.shape[1], 1024, R._lib.ptr(x), R._lib.ptr(s["m"]), R._lib.ptr(s["P"]),
                R._lib.ptr(y), R._lib.ptr(attn), R._lib.stream())
    want = ((x[0].double() - s["m"]) @ s["P"]).float()
    ulp = (y.view(torch.int32).long() - want.view(torch.int32).long()).abs()
    print(f"whitening: {int((ulp > 0).sum())} of {ulp.numel()} values differ by 1 ulp from torch float64")
    assert int(ulp.max()) <= 1
    assert torch.allclose(attn, y.norm(dim=1), rtol=1e-6, atol=0)


def test_select_ties_to_lower_index(cuda):
    db = R.RetrievalDatabase(torch.zeros(1, 1024, dtype=torch.float64), torch.eye(1024, dtype=torch.float64),
                             torch.randn(8, 1024), nfeat=300)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 700, 1024, generator=g)
    x[0, 100:400] = x[0, 50]          # 300 equal attention keys straddle the nfeat boundary
    out = db.prep_features(x.to(cuda))[0].cpu()
    a = x[0].norm(dim=1)
    order = sorted(range(700), key=lambda i: (-a[i].item(), i))[:300]
    assert torch.equal(out, x[0, order])


@pytest.mark.parametrize("K", [1, 5, 1000, 4096, 65536])
@pytest.mark.parametrize("ma", [1, 5, 8])
def test_assignment(cuda, K, ma):
    if ma > K:
        pytest.skip("MA > K is refused")
    g = torch.Generator().manual_seed(K * 10 + ma)
    c = torch.randn(K, 1024, generator=g)
    q = torch.randn(300, 1024, generator=g)
    q[7] = c[min(3, K - 1)]                        # an exact hit
    if K >= 5:
        c[4] = c[2]                                # duplicate centroid: equal distances resolve to the lower index
        q[9] = c[2]
    db = R.RetrievalDatabase(torch.zeros(1, 1024, dtype=torch.float64), torch.eye(1024, dtype=torch.float64), c,
                             nfeat=300, query_params={**R.QUERY_PARAMS, "quantize": {"multiple_assignment": max(ma, 1)}},
                             build_params={**R.BUILD_PARAMS, "quantize": {"multiple_assignment": 1}})
    got = db.quantize_custom(q.to(cuda), {"quantize": {"multiple_assignment": ma}}).cpu().long()
    qd, cd = q.double(), c.double()
    dist = (qd * qd).sum(1, keepdim=True) + (cd * cd).sum(1)[None] - 2 * qd @ cd.T
    sd, si = torch.sort(dist, dim=1, stable=True)
    bound = 2.0 ** -13 * ((qd * qd).sum(1, keepdim=True) + (cd * cd).sum(1).max())
    n_checked = 0
    for r in range(300):
        for j in range(ma):
            lo = sd[r, j] - sd[r, j - 1] if j > 0 else torch.tensor(float("inf"))
            hi = sd[r, j + 1] - sd[r, j] if j + 1 < K else torch.tensor(float("inf"))
            if min(lo, hi) > bound[r, 0]:
                assert got[r, j] == si[r, j], (r, j)
                n_checked += 1
    if K >= 5:
        assert got[9, 0] == 2 and (ma == 1 or got[9, 1] == 4)
    print(f"K={K} MA={ma}: {n_checked} of {300 * ma} positions outside the bound, all equal")
    assert n_checked >= 0.5 * 300 * ma   # the duplicated centroid leaves its pair's positions undecided at K = 5


def test_signatures_from_words(cuda):
    g = torch.Generator().manual_seed(5)
    c = torch.randn(4096, 1024, generator=g)
    desc = torch.randn(300, 1024, generator=g)
    words = torch.randint(0, 64, (300, 5), generator=g, dtype=torch.int32)   # many members per word
    db = R.RetrievalDatabase(torch.zeros(1, 1024, dtype=torch.float64), torch.eye(1024, dtype=torch.float64), c)
    s = db._state()
    db._aggregate(desc.to(cuda), words.to(cuda), 5, s["qw"].data_ptr(), s["qsig"].data_ptr(), s["qcount"].data_ptr())
    sig, uw = rr.aggregate(desc.numpy(), words.numpy(), c.numpy())
    n = int(s["qcount"])
    assert n == len(uw)
    assert np.array_equal(s["qw"][:n].cpu().numpy(), uw)
    assert np.array_equal(s["qsig"][:n].cpu().numpy(), sig.view(np.int32))


def test_search_hand_built(cuda):
    """No shared word, all words shared, a one-word image, popcounts 512 and 513 (the s >= 0 edge)."""
    c = torch.randn(64, 1024)
    db = R.RetrievalDatabase(torch.zeros(1, 1024, dtype=torch.float64), torch.eye(1024, dtype=torch.float64), c, nfeat=8)
    s = db._state()
    g = np.random.default_rng(1)
    qwords = np.array([1, 3, 5, 7, 9], dtype=np.int32)
    qsig = g.integers(0, 2 ** 32, (5, 32), dtype=np.uint32)

    def flip(sig, p):
        out = sig.copy()
        for b in range(p):
            out[b // 32] ^= np.uint32(1 << (b % 32))
        return out
    images = [
        (np.array([0, 2, 4], np.int32), g.integers(0, 2 ** 32, (3, 32), dtype=np.uint32)),           # nothing shared
        (qwords.copy(), np.stack([flip(qsig[i], 37 * i) for i in range(5)])),                          # all shared
        (np.array([5], np.int32), flip(qsig[2], 100)[None]),                                           # one word
        (np.array([1, 7, 11], np.int32), np.stack([flip(qsig[0], 512), flip(qsig[3], 513), qsig[0]])),  # s = 0, s < 0
    ]
    ref = rr.InvertedFile()
    for w, sg in images:
        ref.add(sg, w)
    cap = len(images)
    while db._capacity < cap:
        db._grow()
    s = db._dev
    for i, (w, sg) in enumerate(images):
        s["ivf_words"][i, :len(w)] = torch.from_numpy(w).to(cuda)
        s["ivf_sig"][i, :len(w)] = torch.from_numpy(sg.view(np.int32)).to(cuda)
        s["ivf_count"][i] = len(w)
    s["qw"][:5] = torch.from_numpy(qwords).to(cuda)
    s["qsig"][:5] = torch.from_numpy(qsig.view(np.int32)).to(cuda)
    s["qcount"][0] = 5
    got = db._search(cap).cpu().numpy()
    want = ref.search(qsig, qwords)
    assert np.array_equal(got.view(np.int64), want.view(np.int64)), (got, want)
    assert want[0] == 0.0 and want[1] > 0 and want[2] > 0


def test_relocalisation_leaves_ivf_identical(cuda, golden, stream):
    windows = []
    db = _db(stream[0], golden, True, windows)
    cfg = golden["config"]["retrieval"]
    frames = stream[1]
    for fr in frames[:16]:
        db.update(fr["feat"].to(cuda), fr["add"], cfg["k"], cfg["min_thresh"])
    s = db._dev
    before = [s[k].clone() for k in ("ivf_words", "ivf_sig", "ivf_count")]
    n = db.kf_counter
    assert not frames[16]["add"]
    db.update(frames[16]["feat"].to(cuda), False, cfg["k"], cfg["min_thresh"])
    assert db.kf_counter == n
    for a, k in zip(before, ("ivf_words", "ivf_sig", "ivf_count")):
        assert torch.equal(a, s[k]), k


def test_one_sync_per_update(cuda, golden, stream):
    db = _db(stream[0], golden, False, [])
    cfg = golden["config"]["retrieval"]
    frames = stream[1]
    for fr in frames[:3]:
        db.update(fr["feat"].to(cuda), fr["add"], cfg["k"], cfg["min_thresh"])
    feat = frames[3]["feat"].to(cuda)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            db.update(feat, True, cfg["k"], cfg["min_thresh"])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    syncs = [x for x in w if "synchroniz" in str(x.message)]
    assert len(syncs) == 1, [str(x.message) for x in syncs]


class _Frame:
    """A key frame as SharedKeyframes keeps it by default: its image on the host, in [-1, 1], carrying its id."""

    def __init__(self, i):
        self.img = torch.full((3, 8, 8), -1.0 + 2.0 * (i + 1) / 256.0)


class _Pi3StandIn:
    """Called where Pi3 is: records the window's ids from the resized images and returns point maps of one surface seen
    from a yaw that grows with the candidate's id (query at yaw 0), or unrelated points for every fourth id, so match
    fractions fall on both sides of the gate."""

    def __init__(self, h=56, w=70):
        import math
        v, u = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
        d0 = torch.stack(((u - w / 2) / (0.9 * w), (v - h / 2) / (0.9 * w), torch.ones_like(u)), -1)
        self.d0 = d0 / d0.norm(dim=-1, keepdim=True)
        self.math = math
        self.calls = []

    def view(self, deg):
        a = self.math.radians(deg)
        R = torch.tensor([[self.math.cos(a), 0, self.math.sin(a)], [0, 1, 0], [-self.math.sin(a), 0, self.math.cos(a)]])
        d = self.d0 @ R.T
        return d * (3.0 + 0.6 * torch.sin(3.0 * d[..., 0:1]) * torch.cos(2.0 * d[..., 1:2]))

    def candidate(self, i):
        if i % 4 == 3:   # unrelated points: a match fraction near 0
            g = torch.Generator().manual_seed(i)
            return torch.rand(self.d0.shape, generator=g) * 10
        return self.view(3.0 * (i % 11))

    def __call__(self, x):
        assert x.is_cuda and x.shape[:3] == (1, x.shape[1], 3) and x.shape[3:] == (392, 518), x.shape
        ids = [int(round(float(x[0, j].mean()) * 256)) - 1 for j in range(x.shape[1])]
        pts = torch.stack([self.candidate(i) for i in ids[:-1]] + [self.view(0.0)]).to(x.device)
        self.calls.append((ids, pts))
        return {"points": pts[None]}


def test_accurate_loop_closure_reaches_pi3(cuda, golden, stream):
    """The real RetrievalDatabase.accurate_loop_closure over the golden sequence, key-frame images on the host and a Pi3
    stand-in: the window reaches the model on the device, and the result is pi3.score_window's on those point maps."""
    from artdeco_b200.pi3 import loop_closure
    m, P, c = stream[0]
    cfg = {**golden["config"], "matching": dict(max_iter=10, lambda_init=1e-8, convergence_thresh=1e-6, dist_thresh=1e-1,
                                                radius=4, dilation_max=5)}
    pi3 = _Pi3StandIn()
    db = R.RetrievalDatabase(m, P, c, nfeat=golden["nfeat"], config=cfg, accurate_loop_closure=True,
                             keyframes=[_Frame(i) for i in range(len(stream[1]))], model_pi3=pi3)
    n_pi3, fracs = 0, []
    for u, (fr, want) in enumerate(zip(stream[1], golden["updates"])):
        n_before = len(pi3.calls)
        out = db.update(fr["feat"].to(cuda), fr["add"], cfg["retrieval"]["k"], cfg["retrieval"]["min_thresh"])
        assert (len(pi3.calls) > n_before) == want["pi3"], u
        if want["pi3"]:
            ids, pts = pi3.calls[-1]
            assert ids == want["window"], u
            sel, counts = loop_closure.score_window(pts, ids, cfg)
            assert out == sel.tolist(), u
            fracs.append(counts.double() / pts[0, ..., 0].numel())
            n_pi3 += 1
    assert n_pi3 == sum(r["pi3"] for r in golden["updates"])
    fracs = torch.cat(fracs)
    gate = cfg["retrieval"]["accurate_min"]
    assert (fracs > gate).any() and (fracs <= gate).any(), fracs      # the accurate_min gate is met on both sides

"""Key-frame retrieval without a GPU: the oracle against the golden file made by running the reference's own retrieval
and ASMK code (tests/golden/make_retrieval_golden.py), the oracle's packing and Hamming against the compiled reference
module, the similarity-graph window against a restatement of the reference's graph, and the configuration refusals."""
from pathlib import Path

import numpy as np
import pytest
import torch

from artdeco_b200 import synthetic
from artdeco_b200.retrieval import BUILD_PARAMS, QUERY_PARAMS, RetrievalDatabase, pow_table
from oracle import retrieval_ref as rr

GOLDEN = Path(__file__).resolve().parent / "golden" / "retrieval_small.pt"


def pi3_stub(m_frac, config):
    """The golden's Pi3 stand-in: match fraction ((37 i + 11 q) % m_frac) / m_frac, then the reference's selection."""
    def select(window):
        ii, q = window[:-1], window[-1]
        frac = torch.tensor([((37 * i + 11 * q) % m_frac) / m_frac for i in ii], dtype=torch.float32)
        order = torch.argsort(frac, descending=True)
        keep = order[frac[order] > config["retrieval"]["accurate_min"]]
        return [ii[i] for i in keep.tolist()][:config["retrieval"]["k"]]
    return select


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, weights_only=False)


@pytest.fixture(scope="module")
def stream(golden):
    m, P, c = synthetic.retrieval_model(golden["K"], seed=golden["seed"])
    return (m, P, c), synthetic.retrieval_stream(m, P, c, golden["schedule"], n=golden["n"], nfeat=golden["nfeat"],
                                                 seed=golden["seed"])


def test_stream_margins_match_golden(golden, stream):
    for got, want in zip([f["margins"] for f in stream[1]], golden["margins"]):
        assert got == pytest.approx(want, rel=0, abs=0)
    b = golden["bounds"]
    for a, d, r in golden["margins"]:
        assert a >= b["attn"] and d >= b["dist"] and r >= b["resid"]


@pytest.mark.parametrize("accurate", [True, False])
def test_oracle_reproduces_golden(golden, stream, accurate):
    (m, P, c), frames = stream
    cfg = golden["config"]["retrieval"]
    ref = rr.Retrieval(m, P, c, nfeat=golden["nfeat"], accurate=accurate, pi3=pi3_stub(golden["m_frac"], golden["config"]))
    for u, (fr, want) in enumerate(zip(frames, golden["updates"])):
        out = ref.update(fr["feat"], fr["add"], cfg["k"], cfg["min_thresh"])
        if not accurate:
            assert out == golden["plain_out"][u], u
            continue
        rec = ref.log[-1]
        assert out == want["out"], u
        assert rec["pi3"] == want["pi3"], u
        assert rec["window"] == want["window"], u
        if want["scores"] is None:
            assert rec["scores"] is None
        else:
            assert np.array_equal(rec["scores"].view(np.int64), want["scores"].numpy().view(np.int64)), u
            assert np.array_equal(rec["codes"], want["codes"].numpy()), u
    if accurate:
        for u, row in golden["ivf_rows"].items():
            sig, words = ref.ivf.images[row["image"]]
            assert np.array_equal(words, row["words"].numpy())
            assert np.array_equal(sig.view(np.int32), row["sig"].numpy())


def test_pack_and_hamming_match_reference_module():
    from oracle import build_hamming
    try:
        h = build_hamming.load()
    except FileNotFoundError:
        pytest.skip("oracle/_ref/hamming not built")
    g = np.random.default_rng(0)
    for dim in (1024, 40, 31, 64):
        x = g.standard_normal((7, dim)).astype(np.float32)
        x[0, :5] = 0.0
        assert np.array_equal(rr.pack_bits(x), h.binarize_and_pack_2D(x)), dim
        a, b = rr.pack_bits(x), rr.pack_bits(g.standard_normal((5, dim)).astype(np.float32))
        assert np.array_equal(rr.hamming(a, b), h.hamming_cdist_packed(a, b)), dim


def test_pow_table_matches_reference_expressions():
    from oracle import build_hamming
    t = pow_table(3.0)
    assert t.dtype == np.float32 and t.shape == (513,)
    try:
        h = build_hamming.load()
    except FileNotFoundError:
        pytest.skip("oracle/_ref/hamming not built")
    for p in (0, 1, 255, 511, 512):
        a = np.zeros((1, 32), np.uint32)
        b = np.zeros((1, 32), np.uint32)
        for bit in range(p):
            b[0, bit // 32] |= np.uint32(1 << (bit % 32))
        sim = -2 * h.hamming_cdist_packed(a, b).squeeze(0) + 1
        assert np.array_equal(np.power(sim[sim >= 0.0], 3.0), t[p:p + 1]), p


class SimilarityGraph:
    """retrieval_database.py:43-100 as the reference writes it (add, remove, sorted neighbours)."""

    def __init__(self):
        from collections import defaultdict
        self.similarities = defaultdict(dict)

    def add_similarity(self, a, b, s):
        self.similarities[a][b] = s
        self.similarities[b][a] = s

    def remove_frame(self, f):
        if f in self.similarities:
            del self.similarities[f]
        for o in self.similarities:
            if f in self.similarities[o]:
                del self.similarities[o][f]

    def get_similar_frames_sorted(self, f):
        if f not in self.similarities:
            return []
        return [o for o, _ in sorted(self.similarities[f].items(), key=lambda x: x[1], reverse=True)]


def test_window_from_row_equals_similarity_graph(golden):
    graph = SimilarityGraph()
    size = 0
    for rec in golden["updates"]:
        if rec["scores"] is not None:
            scores = rec["scores"]
            for i in range(size):
                graph.add_similarity(size, i, scores[i].item() * 100)
            full = graph.get_similar_frames_sorted(size)[:23] + [size]
            assert full == rr.window_from_row(scores.numpy(), size)
            if rec["window"] is not None:
                assert rec["window"] == full
            if not rec["add"]:
                graph.remove_frame(size)
        if rec["add"]:
            size += 1
    # ties go to the lower id, as Python's stable sort of the ascending row
    assert rr.window_from_row(np.array([0.5, 0.7, 0.5, 0.7]), 4) == [1, 3, 0, 2, 4]


def _tiny():
    return torch.zeros(1, 1024, dtype=torch.float64), torch.eye(1024, dtype=torch.float64), torch.randn(16, 1024)


@pytest.mark.parametrize("kw, msg", [
    (dict(hdims="1024"), "projector"), (dict(residual=True), "projector"), (dict(postwhiten=0), "post-whitening"),
    (dict(featweights="softmax"), "featweights"),
    (dict(build_params={**BUILD_PARAMS, "kernel": {"binary": False}}), "binary"),
    (dict(build_params={**BUILD_PARAMS, "ivf": {"use_idf": True}}), "use_idf"),
    (dict(query_params={**QUERY_PARAMS, "quantize": {"multiple_assignment": 9}}), "multiple_assignment"),
    (dict(build_params={**BUILD_PARAMS, "quantize": {"multiple_assignment": 6}}), "multiple_assignment"),
])
def test_refusals_before_device(kw, msg, monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: (_ for _ in ()).throw(AssertionError("touched the device")))
    with pytest.raises(ValueError, match=msg):
        RetrievalDatabase(*_tiny(), **kw)


def test_ma_above_codebook_size_refused():
    m, P, _ = _tiny()
    with pytest.raises(ValueError, match="multiple_assignment"):
        RetrievalDatabase(m, P, torch.randn(4, 1024))


@pytest.mark.parametrize("feat, msg", [
    (torch.zeros(768, 1024), r"\[1, n, 1024\]"), (torch.zeros(2, 768, 1024), r"\[1, n, 1024\]"),
    (torch.zeros(1, 768, 512), r"\[1, n, 1024\]"), (torch.zeros(1, 768, 1024, dtype=torch.float64), "float32"),
    (torch.zeros(1, 200, 1024), "nfeat"),
])
def test_feat_refusals_before_device(feat, msg, monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: (_ for _ in ()).throw(AssertionError("touched the device")))
    db = RetrievalDatabase(*_tiny(), nfeat=300)
    with pytest.raises(ValueError, match=msg):
        db.update(feat, True, 3, 5e-3)
    assert db._dev is None and db.kf_counter == 0


def _write_checkpoint(tmp_path, K=16, **args):
    """A retrieval checkpoint laid out as Retriever reads it: <prefix>_<suffix>.pth with 'args' and 'model', and
    <prefix>_codebook.pkl with asmk's Codebook.state_dict."""
    import pickle
    from argparse import Namespace
    a = dict(freeze_backbone=1, prewhiten=0, hdims="", residual=0, postwhiten=None, featweights="l2norm", nfeat=300,
             nclusters=K, imsize=512, pretrained="finalmast3r")
    a.update(args)
    g = torch.Generator().manual_seed(0)
    m = torch.randn(1, 1024, generator=g, dtype=torch.float64)
    P = torch.randn(1024, 1024, generator=g, dtype=torch.float64)
    cent = torch.randn(K, 1024, generator=g).numpy()
    path = tmp_path / "retrieval_test_trainingfree.pth"
    torch.save({"args": Namespace(**a), "model": {"prewhiten.m": m, "prewhiten.p": P}}, path)
    with open(tmp_path / "retrieval_test_codebook.pkl", "wb") as fh:
        pickle.dump({"type": "Codebook", "params": {"size": K}, "state": {"centroids": cent}}, fh)
    return path, m, P, cent


def test_from_checkpoint_reads_reference_layout(tmp_path, monkeypatch):
    from argparse import Namespace
    monkeypatch.setattr(torch.cuda, "is_available", lambda: (_ for _ in ()).throw(AssertionError("touched the device")))
    path, m, P, cent = _write_checkpoint(tmp_path)
    db = RetrievalDatabase.from_checkpoint(Namespace(accurate_loop_closure=True), {"retrieval": {}}, str(path), [])
    hm, hP, hc = db._host
    assert torch.equal(hm, m.reshape(-1)) and torch.equal(hP, P) and np.array_equal(hc.numpy(), cent)
    assert db.K == 16 and db.nfeat == 300 and db.is_accurate_loop_closure and db._dev is None
    plain = RetrievalDatabase.from_checkpoint(Namespace(accurate_loop_closure=False), {}, str(path), [])
    assert not plain.is_accurate_loop_closure


def test_codebook_size_parses_asmk_suffixes():
    from artdeco_b200.retrieval import codebook_size
    assert codebook_size("64k") == 65536 and codebook_size("1M") == 1 << 20 and codebook_size(4096) == 4096


@pytest.mark.parametrize("args, model, msg", [
    (dict(hdims="1024"), None, "projector"),
    (dict(postwhiten=0), None, "post-whitening"),
    (dict(featweights="softmax"), None, "featweights"),
    (dict(prewhiten=None), None, "pre-whitening"),
    (dict(), {"prewhiten.m": torch.zeros(1, 1024, dtype=torch.float64)}, "pre-whitening"),
    (dict(nclusters="64k"), None, "nclusters"),
])
def test_from_checkpoint_refusals(tmp_path, monkeypatch, args, model, msg):
    from argparse import Namespace
    monkeypatch.setattr(torch.cuda, "is_available", lambda: (_ for _ in ()).throw(AssertionError("touched the device")))
    path, *_ = _write_checkpoint(tmp_path, **args)
    if model is not None:
        ck = torch.load(path, weights_only=False)
        ck["model"] = model
        torch.save(ck, path)
    with pytest.raises(ValueError, match=msg):
        RetrievalDatabase.from_checkpoint(Namespace(accurate_loop_closure=True), {}, str(path), [])


def test_from_checkpoint_refuses_codebook_of_other_size(tmp_path):
    import pickle
    from argparse import Namespace
    path, *_ = _write_checkpoint(tmp_path)
    with open(tmp_path / "retrieval_test_codebook.pkl", "wb") as fh:
        pickle.dump({"type": "Codebook", "params": {"size": 16}, "state": {"centroids": np.zeros((8, 1024), np.float32)}}, fh)
    with pytest.raises(ValueError, match="centroids"):
        RetrievalDatabase.from_checkpoint(Namespace(accurate_loop_closure=True), {}, str(path), [])

"""Writes tests/golden/retrieval_small.pt by running the reference's OWN key-frame retrieval on the CPU.

The reference package cannot be imported here (faiss, Pi3 weights and the MASt3R backbone are absent), so its code is run
as it lies, against stubs:
  * VSLAM/mast3r_slam/retrieval_database.py: ``RetrievalDatabase``'s update, prep_features, query, add_to_database,
    quantize_custom, accumulate_scores, add_to_ivf_custom and accurate_loop_closure, ``SimilarityGraph``,
    ``inverse_normalize`` and ``resize_image``, extracted with ``ast`` and bound to a stub database;
  * mast3r/retrieval/model.py: ``Whitener`` and ``how_select_local`` (extracted);
  * asmk's kernel.py, inverted_file.py, functional.py and io_helpers.py, loaded by file path under a stub ``asmk``
    package (asmk/__init__ imports faiss), with the reference's hamming.pyx compiled by oracle/build_hamming.py;
  * Pi3: a stub model that records the window it is given (each key frame's image carries its id) and a stub
    ``process_pairs_in_chunks`` whose match fractions are pi3_stub_fraction(id, query) below.
The codebook and features are regenerated from the seed (artdeco_b200.synthetic), not stored.  The sequence runs twice,
with and without --accurate_loop_closure.

    python tests/golden/make_retrieval_golden.py [/path/to/reference]
"""
import ast
import importlib.util
import os
import sys
import textwrap
import types
from argparse import Namespace

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from artdeco_b200 import synthetic  # noqa: E402
from oracle import build_hamming  # noqa: E402

K, N_TOK, NFEAT, SEED = 4096, 768, 300, 0
CONFIG = {"retrieval": {"k": 3, "min_thresh": 5e-3, "accurate_min": 0.15}}
SIG_UPDATES = (0, 14, 17, 29)
M_FRAC = 100


def pi3_stub_fraction(i, q):
    """Match fraction of window frame i against query q (distinct over any 100 consecutive ids)."""
    return ((37 * i + 11 * q) % M_FRAC) / M_FRAC


def _source(path, names, cls=None):
    src = open(path).read()
    tree = ast.parse(src)
    scope = tree if cls is None else next(n for n in ast.walk(tree) if isinstance(n, ast.ClassDef) and n.name == cls)
    out = {}
    for node in scope.body:
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)) and node.name in names:
            out[node.name] = textwrap.dedent(ast.get_source_segment(src, node))
    assert set(out) == set(names), (path, set(names) - set(out))
    return out


def _load_asmk(ref):
    base = os.path.join(ref, "VSLAM/thirdparty/mast3r/asmk/asmk")
    pkg = types.ModuleType("asmk")
    pkg.__path__ = [base]
    sys.modules["asmk"] = pkg
    build_hamming.build()
    sys.modules["asmk.hamming"] = build_hamming.load()
    pkg.hamming = sys.modules["asmk.hamming"]
    for name in ("functional", "io_helpers", "kernel", "inverted_file"):
        spec = importlib.util.spec_from_file_location(f"asmk.{name}", os.path.join(base, f"{name}.py"))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[f"asmk.{name}"] = mod
        spec.loader.exec_module(mod)
        setattr(pkg, name, mod)
    return pkg


def main(ref):
    asmk = _load_asmk(ref)
    rdb_path = os.path.join(ref, "VSLAM/mast3r_slam/retrieval_database.py")
    model_path = os.path.join(ref, "VSLAM/thirdparty/mast3r/mast3r/retrieval/model.py")
    ns = dict(torch=torch, np=np, nn=nn, F=F, io_helpers=asmk.io_helpers, defaultdict=__import__("collections").defaultdict)
    for code in _source(model_path, ["Whitener", "how_select_local"]).values():
        exec(code, ns)
    for code in _source(rdb_path, ["inverse_normalize", "resize_image", "SimilarityGraph"]).values():
        exec(code, ns)
    meths = _source(rdb_path, ["update", "prep_features", "query", "add_to_database", "quantize_custom",
                               "accumulate_scores", "add_to_ivf_custom", "accurate_loop_closure"], cls="RetrievalDatabase")
    for code in meths.values():
        exec(code, ns)

    m, P, cent = synthetic.retrieval_model(K, seed=SEED)
    stream = synthetic.retrieval_stream(m, P, cent, synthetic.RETRIEVAL_SCHEDULE, n=N_TOK, nfeat=NFEAT, seed=SEED)
    build_params = {"kernel": {"binary": True}, "ivf": {"use_idf": False}, "quantize": {"multiple_assignment": 1},
                    "aggregate": {}}
    query_params = {"quantize": {"multiple_assignment": 5}, "aggregate": {}, "search": {"topk": None},
                    "similarity": {"similarity_threshold": 0.0, "alpha": 3.0}}

    def run(accurate):
        db = types.SimpleNamespace()
        for name in meths:
            setattr(db, name, types.MethodType(ns[name], db))
        whitener = ns["Whitener"](1024).requires_grad_(False)   # prewhiten=0: frozen (model.py)
        whitener.m.data.copy_(m)
        whitener.p.data.copy_(P)
        db.model = types.SimpleNamespace(prewhiten=whitener, projector=nn.Identity(), residual=False,
                                         attention=lambda x: x.norm(dim=-1), postwhiten=nn.Identity(), nfeat=NFEAT)
        codebook = types.SimpleNamespace(centroids=cent.numpy(), size=K)
        kern = asmk.kernel.ASMKKernel(codebook, binary=True)
        ivf = asmk.inverted_file.IVF.initialize_empty(codebook_size=K, use_idf=False)
        db.ivf_builder = types.SimpleNamespace(kernel=kern, ivf=ivf, step_params=build_params)
        db.asmk = types.SimpleNamespace(params={"build_ivf": build_params, "query_ivf": query_params}, codebook=codebook)
        db.min_window_number, db.max_window_number, db.accurate_loop_closure_number = 12, 24, 12
        db.is_accurate_loop_closure = accurate
        db.kf_counter, db.kf_ids = 0, []
        db.query_dtype, db.query_device, db.device = torch.float32, "cpu", "cpu"
        db.centroids = cent.clone()
        db.sim_Graph = ns["SimilarityGraph"]()
        db.config = CONFIG
        windows = []

        class Frame:
            def __init__(self, i):
                self.img = torch.full((3, 8, 8), -1.0 + 2.0 * (i + 1) / 256.0)

        def pi3_model(images):
            ids = [int(round(float(images[0, j].mean()) * 256)) - 1 for j in range(images.shape[1])]
            windows.append(ids)
            return {"points": torch.tensor(ids, dtype=torch.float64).reshape(1, -1, 1, 1, 1).expand(1, -1, 2, 2, 3)}

        def process_pairs_in_chunks(pairs, chunk_size=32):
            valid = torch.zeros(pairs.shape[0], M_FRAC, dtype=torch.bool)
            for r in range(pairs.shape[0]):
                i, q = int(pairs[r, 0, 0, 0, 0]), int(pairs[r, 1, 0, 0, 0])
                valid[r, :round(pi3_stub_fraction(i, q) * M_FRAC)] = True
            return None, valid

        db.keyframes = [Frame(i) for i in range(len(stream))]
        db.model_pi3 = pi3_model
        db.process_pairs_in_chunks = process_pairs_in_chunks
        db.args = Namespace(accurate_loop_closure=accurate)
        import builtins
        log = []
        real_print = builtins.print
        builtins.print = lambda *a, **k: None
        real_cap = torch.cuda.get_device_capability
        torch.cuda.get_device_capability = lambda *a: (9, 0)   # accurate_loop_closure picks its autocast dtype
        try:
            for u, fr in enumerate(stream):
                n_before = len(windows)
                scores_seen = {}
                orig_query = db.query

                def query(feat, id, _orig=orig_query):
                    ranks, ranked, codes = _orig(feat, id)
                    sc = np.empty_like(ranked)
                    sc[np.arange(ranked.shape[0])[:, None], ranks] = ranked
                    scores_seen["scores"], scores_seen["codes"] = sc[0], codes
                    return ranks, ranked, codes

                db.query = query
                out = db.update(fr["feat"], fr["add"], CONFIG["retrieval"]["k"], CONFIG["retrieval"]["min_thresh"])
                db.query = orig_query
                rec = dict(out=list(map(int, out)), add=fr["add"], pi3=len(windows) > n_before,
                           window=windows[-1] if len(windows) > n_before else None,
                           scores=torch.from_numpy(scores_seen["scores"].copy()) if "scores" in scores_seen else None,
                           codes=torch.from_numpy(scores_seen["codes"].astype(np.int32)) if "codes" in scores_seen else None)
                log.append(rec)
        finally:
            builtins.print = real_print
            torch.cuda.get_device_capability = real_cap
        return db, log

    db, log = run(True)
    _, log_plain = run(False)
    # the IVF rows of the signature updates: each image's words and packed signatures, as asmk stores them
    ivf = db.ivf_builder.ivf
    kept = {}
    img_of_update, img = {}, 0
    for u, fr in enumerate(stream):
        if fr["add"]:
            img_of_update[u] = img
            img += 1
    for u in SIG_UPDATES:
        i = img_of_update[u]
        words = [w for w in range(K) if ivf.ivf_image_ids[w] is not None and i in ivf.ivf_image_ids[w][:ivf.counts[w]]]
        sig = np.stack([ivf.ivf_vecs[w][list(ivf.ivf_image_ids[w][:ivf.counts[w]]).index(i)] for w in words])
        kept[u] = dict(image=i, words=torch.tensor(words, dtype=torch.int32),
                       sig=torch.from_numpy(sig.astype(np.uint32).view(np.int32)))
    out = dict(K=K, n=N_TOK, nfeat=NFEAT, seed=SEED, config=CONFIG, schedule=synthetic.RETRIEVAL_SCHEDULE,
               margins=[fr["margins"] for fr in stream], bounds=dict(dist=synthetic.RETRIEVAL_MARGIN_DIST,
               resid=synthetic.RETRIEVAL_MARGIN_RESID, attn=synthetic.RETRIEVAL_MARGIN_ATTN),
               updates=log, plain_out=[r["out"] for r in log_plain], ivf_rows=kept, m_frac=M_FRAC)
    path = os.path.join(ROOT, "tests", "golden", "retrieval_small.pt")
    torch.save(out, path)
    print(f"wrote {path} ({os.path.getsize(path)} bytes): outs {[r['out'] for r in log]}")
    print("pi3:", [u for u, r in enumerate(log) if r["pi3"]], "plain:", out["plain_out"])


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")

"""The Backend's key-frame retrieval (VSLAM/mast3r_slam/retrieval_database.py) on the device, for the retrieval
configuration ARTDECO loads (MASt3R_ViTLarge_BaseDecoder_512_catmlpdpt_metric_retrieval_trainingfree.pth): a frozen
whitening, identity projector and post-whitening, l2-norm attention, nfeat local features, and a binary ASMK inverted
file without idf, built with one visual word per feature and queried with ``multiple_assignment`` words, alpha and
similarity threshold 0.

  prep_features     whitening (fp64) + attention + top-nfeat        csrc/retrieval.cu   (:175-196)
  quantize_custom   codebook assignment, bf16x3 wgmma + top-MA      csrc/gemm_tc.cu     (:355-367)
  aggregate         ASMK residual sums + sign packing               csrc/retrieval.cu   (asmk/kernel.py:26-39)
  search            inverted-file scores, float64                   csrc/retrieval.cu   (asmk/inverted_file.py:86-112)
  rank              top-k, min_thresh, oldest candidate, window     csrc/retrieval.cu   (:224-267)

The inverted file is image-major: row i holds image i's sorted word ids, its 32-word signatures and its word count.
``update`` reads the host once, the small rank buffer; everything else stays on the device.

The reference keeps a similarity graph only to sort the current query's row for the Pi3 window
(``accurate_loop_closure``): that row is the score vector of this query, in ascending id order, so the window is
computed on the device from the scores (DESIGN.md, "Key-frame retrieval").  There is no CPU implementation."""
from __future__ import annotations

import ctypes as C
import pickle

import numpy as np
import torch

from . import _lib
from ._lib import i32, i64, vp
from .pi3 import loop_closure

_lib.register("adb_retrieval_whiten", [i32, i32, vp, vp, vp, vp, vp, vp])
_lib.register("adb_retrieval_select", [i32, i32, vp, vp, vp])
_lib.register("adb_retrieval_gather_split", [i64, i32, vp, vp, vp, vp, vp, vp, vp])
_lib.register("adb_retrieval_assign", [i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp])
_lib.register("adb_retrieval_topma_merge", [i32, i32, i32, vp, vp, vp, vp])
_lib.register("adb_retrieval_aggregate", [i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp])
_lib.register("adb_retrieval_search", [i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp])
_lib.register("adb_retrieval_rank", [i32, vp, i32, C.c_double, i32, vp, vp])

DIM = 1024                 # MASt3R ViT-L encoder width
NW = DIM // 32             # uint32 words per binary signature
TILE_N = 128               # centroid columns per assignment tile (gemm_tc.cu BN)
MAX_MA = 8
MAX_TOKENS = 1024          # one CTA sorts the attention keys

# processor.py:98-103
BUILD_PARAMS = {"kernel": {"binary": True}, "ivf": {"use_idf": False}, "quantize": {"multiple_assignment": 1},
                "aggregate": {}}
QUERY_PARAMS = {"quantize": {"multiple_assignment": 5}, "aggregate": {}, "search": {"topk": None},
                "similarity": {"similarity_threshold": 0.0, "alpha": 3.0}}


def pow_table(alpha: float, dim: int = DIM) -> np.ndarray:
    """float32 s**alpha for every popcount p with s = 1 - 2 p / dim >= 0, written with the reference's own float32
    expressions (hamming.pyx:33-42, kernel.py:63-64, functional.py:11-15), so the table equals its values by construction."""
    p = np.arange(dim // 2 + 1, dtype=np.int32)
    h = p.astype(np.float32) / np.float32(dim)
    sim = -2 * h + 1
    return np.power(sim, alpha)


def codebook_size(nclusters) -> int:
    """asmk/codebook.py:15-17: an int, or a string with a 'k' (x 1024) or 'M' (x 1024**2) suffix."""
    if isinstance(nclusters, str) and nclusters[-1] in "kM":
        return int(nclusters[:-1]) * {"k": 1024, "M": 1024 ** 2}[nclusters[-1]]
    return int(nclusters)


class RetrievalDatabase:
    """The reference's ``RetrievalDatabase`` for the trainingfree configuration only.  ``m`` [1, 1024] and ``P``
    [1024, 1024] are the whitening (float64), ``centroids`` [K, 1024] the ASMK codebook.  Configuration checks raise
    ``ValueError`` before anything reaches the device; the device state is built on first use.

    ``update``, ``prep_features``, ``accurate_loop_closure``, ``kf_counter`` and ``kf_ids`` keep the reference's
    arguments and results.  The helpers ``update`` calls keep their names but work on device tensors and differ in
    signature, because the reference's versions move the descriptors and scores to the host:
      * ``quantize_custom(qvecs, params)`` returns int32 word ids on the device (the reference: int64);
      * ``query(feat, k, min_thresh)`` returns (the query's int32 [nfeat, MA] words, the host list read from the rank
        buffer), where the reference's ``query(feat_np, id_np)`` returns numpy (ranks, ranked scores, words); the scores
        stay in ``self.scores``;
      * ``add_to_database(feat, topk_codes)`` takes no image ids: the row is always ``kf_counter``, as the reference's
        ``id_np`` always is."""

    min_window_number = 12
    max_window_number = 24
    accurate_loop_closure_number = 12

    def __init__(self, m, P, centroids, *, nfeat=300, build_params=BUILD_PARAMS, query_params=QUERY_PARAMS,
                 hdims="", residual=False, postwhiten=None, featweights="l2norm", keyframes=None, model_pi3=None,
                 config=None, accurate_loop_closure=False, device="cuda", capacity=64):
        m = torch.as_tensor(m)
        P = torch.as_tensor(P)
        centroids = torch.as_tensor(centroids)
        if hdims not in ("", None) or residual:
            raise ValueError("only the identity projector (hdims='', residual=0) of the trainingfree model is supported")
        if postwhiten is not None:
            raise ValueError("post-whitening is not supported (the trainingfree model has postwhiten=None)")
        if featweights != "l2norm":
            raise ValueError(f"featweights={featweights!r}: only 'l2norm' attention is supported")
        if not build_params["kernel"]["binary"]:
            raise ValueError("binary=False: only the binary ASMK kernel is supported")
        if build_params["ivf"]["use_idf"]:
            raise ValueError("use_idf=True: only the inverted file without idf is supported")
        if query_params["similarity"]["similarity_threshold"] != 0.0:
            raise ValueError("only similarity_threshold=0.0 is supported")
        if query_params["search"].get("topk") is not None:
            raise ValueError("only search topk=None (every database image scored) is supported")
        if tuple(m.shape) != (1, DIM) or tuple(P.shape) != (DIM, DIM):
            raise ValueError(f"whitening must be m [1, {DIM}] and P [{DIM}, {DIM}], got {tuple(m.shape)} and {tuple(P.shape)}")
        if centroids.dim() != 2 or centroids.shape[1] != DIM or centroids.shape[0] < 1:
            raise ValueError(f"centroids must be [K, {DIM}], got {tuple(centroids.shape)}")
        self.K = int(centroids.shape[0])
        self.build_ma = int(build_params["quantize"]["multiple_assignment"])
        self.query_ma = int(query_params["quantize"]["multiple_assignment"])
        for name, ma in (("build", self.build_ma), ("query", self.query_ma)):
            if not 1 <= ma <= min(MAX_MA, self.K):
                raise ValueError(f"{name} multiple_assignment={ma}: must be in [1, min({MAX_MA}, K={self.K})]")
        if self.build_ma > self.query_ma:
            raise ValueError("build multiple_assignment must not exceed the query's (the build reuses the query's words)")
        self.nfeat = int(nfeat)
        if not 1 <= self.nfeat <= MAX_TOKENS:
            raise ValueError(f"nfeat={nfeat}: must be in [1, {MAX_TOKENS}]")
        self.alpha = float(query_params["similarity"]["alpha"])
        self.params = {"build_ivf": build_params, "query_ivf": query_params}

        self.keyframes = keyframes
        self.model_pi3 = model_pi3
        self.config = config
        self.is_accurate_loop_closure = bool(accurate_loop_closure)
        self.device = torch.device(device)
        self.query_device = self.device
        self.kf_counter = 0
        self.kf_ids = []

        self._host = (m.double().reshape(-1), P.double(), centroids.float())
        self._capacity = max(1, int(capacity))
        self._dev = None
        self._window = None      # (query id, device-computed window) of the last query
        self.scores = None       # float64 [database_size] of the last query (device)
        self.topk_codes = None   # int32 [nfeat, query MA] of the last query (device)

    @classmethod
    def from_checkpoint(cls, args, config, modelname, keyframes, model_pi3=None, device="cuda", **kw):
        """Reads what ``Retriever.__init__`` reads (processor.py:72-109): the retrieval ``.pth`` (its args and the
        whitening) and the ``<prefix>_codebook.pkl`` next to it; refuses any configuration but the trainingfree one."""
        import os
        ckpt = torch.load(modelname, "cpu", weights_only=False)
        a = ckpt["args"]
        sd = ckpt["model"]
        if getattr(a, "prewhiten", None) is None or "prewhiten.m" not in sd or "prewhiten.p" not in sd:
            raise ValueError("the checkpoint has no frozen pre-whitening (prewhiten.m / prewhiten.p)")
        dname, bname = os.path.split(modelname)
        cb_path = os.path.join(dname, "_".join(bname.split("_")[:-1]) + "_codebook.pkl")
        with open(cb_path, "rb") as fh:
            cb = pickle.load(fh)
        # asmk_method.py:62 asserts the stored codebook parameters equal the checkpoint's nclusters
        if cb["params"]["size"] != a.nclusters:
            raise ValueError(f"codebook size {cb['params']['size']!r} differs from the checkpoint's nclusters {a.nclusters!r}")
        centroids = torch.from_numpy(np.ascontiguousarray(cb["state"]["centroids"], dtype=np.float32))
        if centroids.dim() != 2 or centroids.shape[0] != codebook_size(a.nclusters):
            raise ValueError(f"the codebook holds {tuple(centroids.shape)} centroids, nclusters={a.nclusters!r}")
        return cls(sd["prewhiten.m"], sd["prewhiten.p"], centroids, nfeat=int(a.nfeat), hdims=a.hdims,
                   residual=getattr(a, "residual", False), postwhiten=a.postwhiten, featweights=a.featweights,
                   keyframes=keyframes, model_pi3=model_pi3, config=config,
                   accurate_loop_closure=getattr(args, "accurate_loop_closure", False), device=device, **kw)

    # ---- device state ----
    def _state(self):
        if self._dev is not None:
            return self._dev
        _lib.require_cuda()
        dev = self.device
        m, P, cent = (t.to(dev).contiguous() for t in self._host)
        nt = (self.K + TILE_N - 1) // TILE_N
        s = dict(m=m, P=P, cent=cent,
                 c_hi=torch.empty(self.K, DIM, dtype=torch.bfloat16, device=dev),
                 c_lo=torch.empty(self.K, DIM, dtype=torch.bfloat16, device=dev),
                 cn=torch.empty(self.K, dtype=torch.float32, device=dev),
                 table=torch.from_numpy(pow_table(self.alpha)).to(dev),
                 q_hi=torch.empty(self.nfeat, DIM, dtype=torch.bfloat16, device=dev),
                 q_lo=torch.empty(self.nfeat, DIM, dtype=torch.bfloat16, device=dev),
                 qn=torch.empty(self.nfeat, dtype=torch.float32, device=dev),
                 cand_d=torch.empty(self.nfeat * nt * self.query_ma, dtype=torch.float32, device=dev),
                 cand_i=torch.empty(self.nfeat * nt * self.query_ma, dtype=torch.int32, device=dev),
                 qw=torch.empty(self.nfeat * self.query_ma, dtype=torch.int32, device=dev),
                 qsig=torch.empty(self.nfeat * self.query_ma, NW, dtype=torch.int32, device=dev),
                 qcount=torch.empty(1, dtype=torch.int32, device=dev),
                 ivf_words=torch.zeros(self._capacity, self.nfeat, dtype=torch.int32, device=dev),
                 ivf_sig=torch.zeros(self._capacity, self.nfeat, NW, dtype=torch.int32, device=dev),
                 ivf_count=torch.zeros(self._capacity, dtype=torch.int32, device=dev))
        with torch.cuda.device(dev):
            _lib.call("adb_retrieval_gather_split", self.K, DIM, _lib.ptr(cent), None, None, _lib.ptr(s["c_hi"]),
                      _lib.ptr(s["c_lo"]), _lib.ptr(s["cn"]), _lib.stream())
        self._dev = s
        return s

    def _grow(self):
        """Doubles the inverted file's rows when the counter reaches them (the host knows the counter: no read)."""
        s = self._dev
        cap = self._capacity * 2
        for key in ("ivf_words", "ivf_sig", "ivf_count"):
            old = s[key]
            new = torch.zeros((cap,) + tuple(old.shape[1:]), dtype=old.dtype, device=old.device)
            new[:self._capacity].copy_(old)
            s[key] = new
        self._capacity = cap

    def _check_feat(self, feat):
        if not isinstance(feat, torch.Tensor) or feat.dim() != 3 or feat.shape[0] != 1 or feat.shape[2] != DIM:
            raise ValueError(f"feat must be [1, n, {DIM}] (one frame's encoder tokens), got "
                             f"{tuple(feat.shape) if isinstance(feat, torch.Tensor) else type(feat)}")
        if feat.dtype != torch.float32:
            raise ValueError(f"feat must be float32, got {feat.dtype}")
        n = feat.shape[1]
        if not self.nfeat <= n <= MAX_TOKENS:
            raise ValueError(f"feat has {n} tokens: need nfeat={self.nfeat} <= n <= {MAX_TOKENS}")

    # ---- the reference's methods ----
    def prep_features(self, backbone_feat):
        """[1, n, 1024] fp32 encoder tokens -> [1, nfeat, 1024] whitened local features, best attention first."""
        self._check_feat(backbone_feat)
        s = self._state()
        x = backbone_feat.to(self.device).contiguous()
        n = x.shape[1]
        y = torch.empty(n, DIM, dtype=torch.float32, device=self.device)
        attn = torch.empty(n, dtype=torch.float32, device=self.device)
        tok = torch.empty(self.nfeat, dtype=torch.int32, device=self.device)
        out = torch.empty(1, self.nfeat, DIM, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            st = _lib.stream()
            _lib.call("adb_retrieval_whiten", n, DIM, _lib.ptr(x), _lib.ptr(s["m"]), _lib.ptr(s["P"]), _lib.ptr(y),
                      _lib.ptr(attn), st)
            _lib.call("adb_retrieval_select", n, self.nfeat, _lib.ptr(attn), _lib.ptr(tok), st)
            _lib.call("adb_retrieval_gather_split", self.nfeat, DIM, _lib.ptr(y), _lib.ptr(tok), _lib.ptr(out),
                      _lib.ptr(s["q_hi"]), _lib.ptr(s["q_lo"]), _lib.ptr(s["qn"]), st)
        return out

    def quantize_custom(self, qvecs, params):
        """qvecs [nfeat, 1024] fp32 (device) -> int32 [nfeat, MA]: the MA nearest centroids, nearest first, ties to the
        lower index."""
        self._split(qvecs)
        return self._quantize(params)

    def _split(self, qvecs):
        """The bf16 (hi, lo) split and squared norms of the descriptors the next assignment reads."""
        s = self._state()
        if qvecs.dim() != 2 or qvecs.shape[0] != self.nfeat or qvecs.shape[1] != DIM or qvecs.dtype != torch.float32:
            raise ValueError(f"qvecs must be [{self.nfeat}, {DIM}] float32")
        q = qvecs.to(self.device).contiguous()
        with torch.cuda.device(self.device):
            _lib.call("adb_retrieval_gather_split", self.nfeat, DIM, _lib.ptr(q), None, None, _lib.ptr(s["q_hi"]),
                      _lib.ptr(s["q_lo"]), _lib.ptr(s["qn"]), _lib.stream())

    def _quantize(self, params):
        """The assignment of the descriptors last split (by prep_features or _split)."""
        s = self._dev
        ma = int(params["quantize"]["multiple_assignment"])
        if not 1 <= ma <= min(MAX_MA, self.K) or ma > self.query_ma:
            raise ValueError(f"multiple_assignment={ma} out of range")
        nt = (self.K + TILE_N - 1) // TILE_N
        words = torch.empty(self.nfeat, ma, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            st = _lib.stream()
            _lib.call("adb_retrieval_assign", self.nfeat, self.K, DIM, ma, _lib.ptr(s["q_hi"]), _lib.ptr(s["q_lo"]),
                      _lib.ptr(s["c_hi"]), _lib.ptr(s["c_lo"]), _lib.ptr(s["qn"]), _lib.ptr(s["cn"]),
                      _lib.ptr(s["cand_d"]), _lib.ptr(s["cand_i"]), st)
            _lib.call("adb_retrieval_topma_merge", self.nfeat, nt, ma, _lib.ptr(s["cand_d"]), _lib.ptr(s["cand_i"]),
                      _lib.ptr(words), st)
        return words

    def _aggregate(self, desc, words, ma, out_words, out_sig, out_count):
        s = self._dev
        with torch.cuda.device(self.device):
            _lib.call("adb_retrieval_aggregate", self.nfeat, DIM, ma, words.shape[1], _lib.ptr(desc), _lib.ptr(words),
                      _lib.ptr(s["cent"]), C.c_void_p(out_words), C.c_void_p(out_sig), C.c_void_p(out_count), _lib.stream())

    def _search(self, n_db):
        s = self._dev
        scores = torch.empty(n_db, dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.call("adb_retrieval_search", n_db, self.nfeat, NW, _lib.ptr(s["qw"]), _lib.ptr(s["qsig"]),
                      _lib.ptr(s["qcount"]), _lib.ptr(s["ivf_words"]), _lib.ptr(s["ivf_sig"]), _lib.ptr(s["ivf_count"]),
                      _lib.ptr(s["table"]), _lib.ptr(scores), _lib.stream())
        return scores

    def query(self, feat, k, min_thresh):
        """feat [1, nfeat, 1024] (prep_features' output) against the database -> (topk_codes [nfeat, MA] on the device,
        the host list read from the rank buffer: [n_valid, top-k ids..., oldest, n_window, window ids...])."""
        self._split(feat[0])
        return self._query(feat, k, min_thresh)

    def _query(self, feat, k, min_thresh):
        s = self._dev
        desc = feat[0]
        codes = self._quantize(self.params["query_ivf"])
        self._aggregate(desc, codes, self.query_ma, s["qw"].data_ptr(), s["qsig"].data_ptr(), s["qcount"].data_ptr())
        n_db = self.kf_counter
        scores = self._search(n_db)
        out = torch.empty(int(k) + 3 + self.max_window_number - 1, dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.call("adb_retrieval_rank", n_db, _lib.ptr(scores), int(k), float(min_thresh),
                      self.max_window_number - 1, _lib.ptr(out), _lib.stream())
        self.scores = scores
        self.topk_codes = codes
        return codes, out.cpu().tolist()   # the one device -> host read of an update

    def add_to_database(self, feat, topk_codes):
        """Appends the frame as inverted-file row ``kf_counter``: its build words are column 0.. of the query's
        assignment, or a fresh assignment for the first frame."""
        if topk_codes is None:
            self._split(feat[0])
        self._add(feat, topk_codes)

    def _add(self, feat, topk_codes):
        desc = feat[0]
        if topk_codes is None:
            topk_codes = self._quantize(self.params["build_ivf"])
        if self.kf_counter == self._capacity:
            self._grow()
        s = self._dev
        r = self.kf_counter
        self._aggregate(desc, topk_codes, self.build_ma, s["ivf_words"][r].data_ptr(), s["ivf_sig"][r].data_ptr(),
                        s["ivf_count"][r:r + 1].data_ptr())
        self.kf_ids.append(self.kf_counter)
        self.kf_counter += 1

    def update(self, feat, add_after_query, k, min_thresh=0.0):
        """retrieval_database.py:200-261: the loop candidates of this key frame (a list of key-frame ids)."""
        self._check_feat(feat)
        feat = self.prep_features(feat)    # also splits the descriptors for the assignment
        database_size = self.kf_counter
        topk_image_inds = []
        topk_codes = None
        self._window = None
        if self.kf_counter > 0:
            topk_codes, out = self._query(feat, k, min_thresh)
            n_valid = out[0]
            retrieved = out[1:1 + n_valid]
            n_win = out[k + 2]
            self._window = (database_size, out[k + 3:k + 3 + n_win])
            if ((database_size < self.min_window_number) and add_after_query) or (not self.is_accurate_loop_closure):
                topk_image_inds = retrieved
            else:
                if n_valid <= 0:
                    need_accurate_loop_closure = True
                else:
                    need_accurate_loop_closure = (database_size - out[k + 1]) > self.accurate_loop_closure_number
                if not add_after_query:
                    need_accurate_loop_closure = True
                if need_accurate_loop_closure:
                    topk_image_inds = self.accurate_loop_closure(database_size)
                else:
                    topk_image_inds = retrieved
        if add_after_query:
            self._add(feat, topk_codes)
        return topk_image_inds

    def window(self, keyframe_id):
        """The Pi3 window of ``accurate_loop_closure(keyframe_id)``: the 23 best-scoring database ids of this query
        (descending score, ties to the lower id), then the query."""
        if self._window is None or self._window[0] != keyframe_id:
            raise ValueError(f"no query of key frame {keyframe_id} in this update")
        return list(self._window[1]) + [keyframe_id]

    def accurate_loop_closure(self, keyframe_id):
        """retrieval_database.py:263-300 through artdeco_b200.pi3.accurate_loop_closure.  The key frames' images may live
        on the host (the reference's SharedKeyframes default) and are gathered onto this database's device."""
        idxs_all = self.window(keyframe_id)
        images = torch.stack([self.keyframes[i].img for i in idxs_all], 0).to(self.device)
        return loop_closure.accurate_loop_closure(self.model_pi3, images, idxs_all, self.config)

    def ivf_row(self, i):
        """Inverted-file row i: (sorted word ids int32 [count], signatures int32 [count, 32] holding the uint32 bits)."""
        if not 0 <= i < self.kf_counter:
            raise IndexError(i)
        s = self._dev
        c = int(s["ivf_count"][i])
        return s["ivf_words"][i, :c], s["ivf_sig"][i, :c]

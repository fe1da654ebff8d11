"""Plain numpy / torch restatement of the Backend's key-frame retrieval (VSLAM/mast3r_slam/retrieval_database.py:175-300
with the trainingfree retrieval model and asmk's binary kernel and inverted file), steps 1-6 of DESIGN.md's retrieval
section.  CPU only; the oracle of artdeco_b200.retrieval and of tests/golden/retrieval_small.pt."""
from __future__ import annotations

import numpy as np
import torch


def prep_features(x, m, P, nfeat):
    """x [1, n, D] fp32 -> [nfeat, D] fp32: y = fp32((double(x) - m) @ P), the nfeat rows of largest fp32 ||y||."""
    y = (x.reshape(-1, x.shape[-1]).double() - m) @ P
    y = y.float()
    attn = y.norm(dim=-1)
    _, idx = torch.topk(attn[None], nfeat, dim=1)
    return y[idx[0]], idx[0]


def quantize(q, centroids, ma):
    """int64 [nq, ma]: indices of the ma smallest fp32 (|q|^2 + |c|^2) - 2 q.c, ascending."""
    d = torch.sum(q ** 2, dim=1)[:, None] + torch.sum(centroids ** 2, dim=1)[None, :] - 2 * (q @ centroids.mT)
    return torch.topk(d, ma, dim=1, largest=False).indices


def pack_bits(r):
    """float32 [n, D] -> uint32 [n, ceil(D/32)]: bit 31 - j of word w is r[:, 32 w + j] > 0, zero padded."""
    b = np.packbits(np.asarray(r) > 0, axis=1, bitorder="big")
    pad = (-b.shape[1]) % 4
    b = np.pad(b, ((0, 0), (0, pad)))
    return b.view(">u4").astype(np.uint32)


def hamming(a, b):
    """Normalised Hamming distance float32 [len(a), len(b)] of packed rows."""
    p = np.bitwise_count(a[:, None, :] ^ b[None, :, :]).sum(-1)
    return p.astype(np.float32) / np.float32(a.shape[1] * 32)


def aggregate(desc, words, centroids):
    """desc [n, D] fp32, words [n, ma] -> (packed residual signs [W, D/32] uint32, sorted unique words [W]).  The
    residual of word w sums (d - c_w) over the descriptors having w, in descriptor order, in fp32."""
    uw = np.unique(words)
    r = np.empty((uw.shape[0], desc.shape[1]), dtype=np.float32)
    for i, w in enumerate(uw):
        sel = desc[(words == w).any(axis=1)] - centroids[w]
        acc = sel[0].copy()
        for row in sel[1:]:
            acc += row
        r[i] = acc
    return pack_bits(r), uw


class InvertedFile:
    """Image-major binary inverted file without idf: image i's (signatures, sorted words)."""

    def __init__(self):
        self.images = []

    def add(self, sig, words):
        self.images.append((sig, words))

    def search(self, qsig, qwords, alpha=3.0):
        """float64 scores [n_images]: sum over shared words, ascending, of float32((s**alpha) / sqrt(n_words(img)))
        for s = 1 - 2 h >= 0 in float32, divided by float32 sqrt(float32 |W_query|)."""
        scores = np.zeros(len(self.images))
        for img, (sig, words) in enumerate(self.images):
            shared, qi, ii = np.intersect1d(qwords, words, assume_unique=True, return_indices=True)
            nf = np.float64(len(words))
            for a, b in zip(qi, ii):
                h = hamming(qsig[a:a + 1], sig[b:b + 1])[0, 0]
                s = np.float32(-2) * h + np.float32(1)
                if s >= 0:
                    s = np.power(np.float32(s), np.float32(alpha))
                    scores[img] += np.float64(np.float32(np.float64(s) / np.sqrt(nf)))
        return scores / np.float64(np.sqrt(np.float32(len(qwords))))


def window_from_row(scores, query_id, max_window=24):
    """The Pi3 window: the ids of the query's similarity row (scores * 100, ids ascending) stably sorted descending,
    the first max_window - 1, then the query."""
    row = [(i, float(scores[i]) * 100) for i in range(len(scores))]
    return [i for i, _ in sorted(row, key=lambda t: t[1], reverse=True)][:max_window - 1] + [query_id]


class Retrieval:
    """retrieval_database.py:200-261 over the functions above.  ``pi3(window)`` stands for accurate_loop_closure's
    Pi3 scoring of a window (query last) and returns its list."""

    def __init__(self, m, P, centroids, *, nfeat=300, build_ma=1, query_ma=5, alpha=3.0, accurate=True, pi3=None):
        self.m, self.P, self.c = m, P, centroids.float()
        self.c_np = self.c.numpy()
        self.nfeat, self.build_ma, self.query_ma, self.alpha = nfeat, build_ma, query_ma, alpha
        self.accurate, self.pi3 = accurate, pi3
        self.ivf = InvertedFile()
        self.kf_counter = 0
        self.log = []

    def update(self, feat, add_after_query, k, min_thresh=0.0):
        desc, _ = prep_features(feat, self.m, self.P, self.nfeat)
        d_np = desc.numpy()
        D = self.kf_counter
        rec = dict(scores=None, codes=None, window=None, pi3=False)
        out, codes = [], None
        if D > 0:
            codes = quantize(desc, self.c, self.query_ma).numpy()
            qsig, qwords = aggregate(d_np, codes, self.c_np)
            scores = self.ivf.search(qsig, qwords, self.alpha)
            rec.update(scores=scores, codes=codes, qwords=qwords, qsig=qsig)
            top = torch.topk(torch.from_numpy(scores), min(k, D))
            retrieved = top.indices[top.values > min_thresh].tolist()
            if ((D < 12) and add_after_query) or not self.accurate:
                out = retrieved
            else:
                need = True if len(retrieved) <= 0 else (D - min(retrieved)) > 12
                if need or not add_after_query:
                    rec["window"] = window_from_row(scores, D)
                    rec["pi3"] = True
                    out = self.pi3(rec["window"])
                else:
                    out = retrieved
        if add_after_query:
            bcodes = quantize(desc, self.c, self.build_ma).numpy() if codes is None else codes[:, :self.build_ma]
            sig, words = aggregate(d_np, bcodes, self.c_np)
            self.ivf.add(sig, words)
            rec.update(build_words=words, build_sig=sig)
            self.kf_counter += 1
        rec["out"] = out
        self.log.append(rec)
        return out

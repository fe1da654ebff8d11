"""weed_out_mask's keep rule at the exact counts where fp32 rounding decides it, and its 1024-camera shared-memory chunks.

The reference computes ``visible_count / len(self.keyframes) > visible_threshold`` on a CUDA int tensor, which PyTorch
evaluates as ``cnt * fl32(1 / K) > fl32(thr)`` (the CPU-scalar fast path of its true-division kernel).  A correctly rounded
``cnt / K`` disagrees at a few (K, cnt) pairs, e.g. K = 500, cnt = 5 at the default threshold 0.01: there the reference keeps
the Gaussian and a division drops it.  The finder below enumerates those pairs; the GPU cases place cameras so that each
Gaussian is seen by an exact, chosen number of them, far from the distance threshold, so that only the keep rule is tested."""
import os

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "densify_small.pt")
THRESHOLDS = (0.01, 0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7)


def keep_rcp(cnt, K, thr):
    """The reference's rule as PyTorch computes it on the device."""
    return np.asarray(cnt, np.float32) * (np.float32(1.0) / np.float32(K)) > np.float32(thr)


def keep_div(cnt, K, thr):
    return np.asarray(cnt, np.float32) / np.float32(K) > np.float32(thr)


def flip_counts(K, thr):
    """Every count 0..K whose keep decision depends on dividing or multiplying by the reciprocal."""
    c = np.arange(K + 1)
    return c[keep_rcp(c, K, thr) != keep_div(c, K, thr)]


def flips(thr, k_max):
    """Every (K, cnt) with 1 <= K <= k_max that flips at ``thr`` (exhaustive)."""
    return [(K, int(c)) for K in range(1, k_max + 1) for c in flip_counts(K, thr)]


# ------------------------------------------------------------------ CPU ------------------------------------------------------

def test_flip_finder():
    at_default = flips(0.01, 5000)
    assert at_default == [(500, 5), (1000, 10), (2000, 20), (2900, 29), (3100, 31), (4000, 40)]
    assert all(keep_rcp(c, K, 0.01) and not keep_div(c, K, 0.01) for K, c in at_default)
    others = {thr: flips(thr, 3000) for thr in THRESHOLDS[1:]}
    assert (30, 3) in others[0.1] and sum(map(len, others.values())) > 50
    assert all(others[thr] for thr in (0.1, 0.2, 0.4, 0.7)), "the GPU flip cases must not test nothing"


def test_densify_golden_has_no_flip_case():
    """tests/golden/densify_small.pt was made on the CPU, where the reference divides; each case has one key frame, whose
    counts (0 or 1) never flip, and a voxel size with an exact reciprocal."""
    for c in torch.load(GOLDEN, weights_only=False)["cases"]:
        K = c["approx_centre"].reshape(-1, 3).shape[0]
        assert K == 1 and not any(len(flip_counts(K, thr)) for thr in (0.0,) + THRESHOLDS)
        vs = np.float32(c["args"]["voxel_size"])
        assert float(np.float32(1.0) / vs) == 1.0 / float(vs)


def test_densify_oracle_weed_out_uses_the_reciprocal():
    """oracle/densify_ref.weed_out gives the device's answer on the CPU too."""
    from oracle import densify_ref as ref
    K, thr = 500, 0.01
    cams = torch.zeros(K, 3)
    cams[:, 0] = torch.arange(1, K + 1, dtype=torch.float32)
    counts = np.array([0, 4, 5, 6, 499, 500])
    params = dict(xyz=torch.zeros(len(counts), 3), d_max=torch.from_numpy((counts + 0.5) / 2).float()[:, None])
    ref.weed_out(params, cams, thr)
    assert torch.equal(params["d_max"][:, 0] * 2 - 0.5, torch.from_numpy(counts[keep_rcp(counts, K, thr)]).float())


# ------------------------------------------------------------------ GPU ------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("thr", THRESHOLDS)
def test_torch_cuda_divides_an_int_count_through_the_reciprocal(cuda, thr):
    """The reference's own expression on the device keeps exactly what cnt * fl32(1/K) > fl32(thr) keeps."""
    for K in sorted({K for K, _ in flips(thr, 3000 if thr > 0.01 else 5000)} | {1, 7, 1025}):
        cnt = torch.arange(K + 1, dtype=torch.int, device=cuda)
        got = ((cnt / K) > thr).cpu().numpy()
        assert (got == keep_rcp(np.arange(K + 1), K, thr)).all(), (K, thr)


def chosen_count_scene(K, seed):
    """K cameras at distances 1..K (shuffled, along three axes) from Gaussians at the origin; Gaussian c has 2 d_max = c + 0.5,
    so exactly c cameras see it, every distance being an integer (to within its rounding) 0.5 away from 2 d_max."""
    g = torch.Generator().manual_seed(seed)
    dirs = torch.tensor([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, -1.0]])
    dist = torch.arange(1, K + 1, dtype=torch.float32)
    cams = dirs[torch.arange(K) % 3] * dist[:, None]
    cams = cams[torch.randperm(K, generator=g)]
    counts = torch.arange(K + 1)
    d_max = (counts.float() + 0.5) / 2
    return torch.zeros(K + 1, 3), d_max, cams, counts


@pytest.mark.gpu
@pytest.mark.parametrize("K,thr", [(500, 0.01), (1000, 0.01), (2000, 0.01), (2900, 0.01), (3100, 0.01), (4000, 0.01),
                                   (30, 0.1), (15, 0.2), (15, 0.4), (30, 0.7), (1025, 0.7), (1025, 0.01), (1024, 0.3), (1, 0.5)])
def test_weed_out_keep_rule_at_exact_counts(cuda, K, thr):
    """Every count 0..K, each by one Gaussian: the visible counts are exact (across the 1024-camera chunks when K > 1024) and
    the keep mask is the reference's rule, including the counts where dividing would decide the other way."""
    from artdeco_b200.cull import weed_out_mask
    xyz, d_max, cams, counts = chosen_count_scene(K, seed=K)
    keep, cnt = weed_out_mask(xyz.to(cuda), d_max.to(cuda), cams.to(cuda), thr, return_count=True)
    assert torch.equal(cnt.cpu().long(), counts), "visible counts"
    want = keep_rcp(counts.numpy(), K, thr)
    flipped = flip_counts(K, thr)
    bad = np.nonzero(keep.cpu().numpy() != want)[0]
    assert not len(bad), f"K={K} thr={thr}: keep differs at counts {bad[:8].tolist()} (division flips at {flipped.tolist()})"

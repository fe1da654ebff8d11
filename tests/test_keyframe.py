"""Key-frame hand-off from the Backend to the mapper (artdeco_b200.keyframe, csrc/keyframe.cu) against the reference's own
statements (tests/golden/keyframe_small.pt, made by make_keyframe_golden.py), against oracle/keyframe_ref.py on the device,
against independent properties, and end to end through densification, the render and the mapper loss."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import keyframe_ref as ref
from oracle import track_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "keyframe_small.pt")
TOL = 1e-5
POSE_KEYS = ("rW2C", "tW2C", "R", "approx_centre")


def golden():
    return torch.load(GOLDEN, weights_only=False)


def assert_rows_close(got, want, what, tol=TOL):
    """Non-finite values at the same places; finite ones within tol x max(|row of want|, 1) per element."""
    a = np.asarray(got.detach().cpu(), dtype=np.float64).reshape(got.shape[0], -1)
    b = np.asarray(want.detach().cpu(), dtype=np.float64).reshape(want.shape[0], -1)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert (np.isnan(a) == np.isnan(b)).all(), f"{what}: NaN at different places"
    fb = np.isfinite(b)
    assert (np.isfinite(a) == fb).all() and (a[np.isinf(b)] == b[np.isinf(b)]).all(), f"{what}: inf differs"
    scale = np.maximum(np.abs(np.where(fb, b, 0)).max(1, keepdims=True), 1.0)
    err = np.abs(np.where(fb, a, 0.0) - np.where(fb, b, 0.0)) / scale
    assert err.max(initial=0.0) <= tol, f"{what}: max error {err.max():.3e} of row scale at row {np.unravel_index(err.argmax(), err.shape)[0]}"


def rows(t, c):
    """[c, h, w] (or [h, w, c] with c last) as one row per pixel."""
    return t.reshape(c, -1).T if t.shape[0] == c else t.reshape(-1, c)


def make_inputs(Hs, Ws, seed, dev="cpu", first=False):
    g = torch.Generator().manual_seed(seed)
    HW = Hs * Ws
    X = torch.randn(HW, 3, generator=g)
    X[:, 2] = 0.5 + 3.0 * torch.rand(HW, generator=g)
    n0 = max(HW // 100, 1)
    X[:n0, 2] = 0.0                                           # zero depths
    X[n0:2 * n0, 2] = -0.1 - torch.rand(n0, generator=g)     # negative depths
    C = 4.5 + torch.randn(HW, 1, generator=g)                 # C / 3 straddles 1.5
    q = torch.randn(4, generator=g)
    T_WC = torch.cat([torch.randn(3, generator=g), q / q.norm() * 1.05, torch.tensor([1.2])])
    q = torch.randn(4, generator=g) * 0.03 + torch.tensor([0.0, 0.0, 0.0, 1.0])
    rel = torch.cat([0.1 * torch.randn(3, generator=g), q / q.norm() * 0.97, torch.tensor([0.9])])
    last = track_ref.mul(T_WC, track_ref.inv(rel))
    # matches: mostly near the same pixel (small residuals), some anywhere
    idx = torch.arange(HW) + torch.randint(-2, 3, (HW,), generator=g)
    far = torch.rand(HW, generator=g) < 0.2
    idx = torch.where(far, torch.randint(0, HW, (HW,), generator=g), idx).clamp(0, HW - 1)
    f = 0.8 * max(Hs, Ws)
    K = torch.tensor([[f, 0.0, (Ws - 1) / 2 + 0.3], [0.0, 1.02 * f, (Hs - 1) / 2 - 0.2], [0.0, 0.0, 1.0]])
    d = dict(X_canon=X, C=C, T_WC=T_WC, last_T_WC=last, idx_k2l=idx, K=K)
    d = {k: v.to(dev) for k, v in d.items()}
    d.update(Hs=Hs, Ws=Ws, N=3)
    if first:
        d["last_T_WC"] = d["idx_k2l"] = None
    return d


def ours_dense(inp):
    from artdeco_b200 import keyframe
    N = torch.tensor([inp["N"]], dtype=torch.int32, device=inp["X_canon"].device)
    return keyframe.dense_point(inp["X_canon"].reshape(inp["Hs"], inp["Ws"], 3), inp["C"], N, inp["T_WC"], inp["K"],
                                last_T_WC=inp["last_T_WC"], idx_k2l=inp["idx_k2l"])


def oracle_dense(inp, scatter=True):
    return ref.prepare_for_mapper(inp["X_canon"], inp["C"], inp["N"], inp["T_WC"], inp["K"], inp["Hs"], inp["Ws"],
                                  last_T_WC=inp["last_T_WC"], idx_k2l=inp["idx_k2l"], scatter=scatter)


def make_image(H, W, seed, dev="cpu"):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(H, W, 3, generator=g).to(dev).permute(2, 0, 1)      # channels-last, as to_map makes it


def ours_mapper(image, dense, T_WC, L, index=1, is_test=False):
    from artdeco_b200 import keyframe
    return keyframe.mapper_keyframe(image, dense, T_WC, pyr_levels=L, index=index, is_test=is_test, lr_poses=1e-3,
                                    lr_exposure=5e-4)


def compare_mapper(got, want, L, what=""):
    assert len(got["idepth_pyr"]) == len(want["idepth_pyr"]) == L and len(got["image_pyr"]) == L
    for lvl in range(L):
        assert got["idepth_pyr"][lvl].shape == want["idepth_pyr"][lvl].shape
        assert got["image_pyr"][lvl].shape == want["image_pyr"][lvl].shape
        assert_rows_close(rows(got["idepth_pyr"][lvl], 1), rows(want["idepth_pyr"][lvl], 1), f"{what} idepth level {lvl}")
        assert_rows_close(rows(got["image_pyr"][lvl], 3), rows(want["image_pyr"][lvl], 3), f"{what} image level {lvl}")
    for k in POSE_KEYS:
        assert_rows_close(got[k].reshape(1, -1), want[k].reshape(1, -1), f"{what} {k}")
    assert got["point_map"].shape == want["point_map"].shape and got["conf"].shape == want["conf"].shape


# ------------------------------------------------------------------ CPU ------------------------------------------------------

def test_oracle_reproduces_the_reference_golden():
    d = golden()
    L = d["args"]["pyr_levels"]
    for case in d["cases"]:
        inp, want = case["inputs"], case["outputs"]
        first = inp["kind"] == "first"
        dense, T_CkC, n_bad = ref.prepare_for_mapper(inp["X_canon"], inp["C"], inp["N"], inp["T_WC"], inp["K"], inp["H_slam"],
                                                     inp["W_slam"], last_T_WC=None if first else inp["last_T_WC"],
                                                     idx_k2l=None if first else inp["idx_k2l"])
        assert n_bad == 0
        assert_rows_close(dense.reshape(-1, 4), want["densePoint"].reshape(-1, 4), f"{inp['kind']} densePoint", tol=1e-6)
        if first:
            assert T_CkC is None and want["T_CkC"] is None
        else:
            assert_rows_close(T_CkC[None], want["T_CkC"][None], f"{inp['kind']} T_CkC", tol=1e-6)
        m = ref.mapper_keyframe(inp["image"], want["densePoint"], want["T_WC"], L)
        for lvl in range(L):
            assert_rows_close(rows(m["idepth_pyr"][lvl], 1), rows(want["idepth_pyr"][lvl], 1), f"idepth {lvl}", tol=1e-6)
            assert_rows_close(rows(m["image_pyr"][lvl], 3), rows(want["image_pyr"][lvl], 3), f"image {lvl}", tol=1e-6)
        for k in ("rW2C", "tW2C", "approx_centre", "point_map", "conf"):
            assert_rows_close(m[k].reshape(1, -1), want[k].reshape(1, -1), k, tol=1e-6)
        assert torch.equal(want["exposure"], torch.eye(3, 4)) and want["betas"] == (0.8, 0.99)
        lr = 0.0 if inp["mapper_index"] == 0 else d["args"]["lr_poses"]
        assert want["lr"] == {"rW2C": lr, "tW2C": lr, "exposure": d["args"]["lr_exposure"]}


def test_golden_covers_the_edge_cases():
    d = golden()
    kinds = {c["inputs"]["kind"]: c for c in d["cases"]}
    assert set(kinds) == {"first", "general", "exact3"}
    first = kinds["first"]
    cn = first["inputs"]["C"] / first["inputs"]["N"]
    assert (cn > 1.5).any() and (cn <= 1.5).any()
    gen = kinds["general"]["inputs"]
    assert abs(float(gen["T_WC"][7]) - 1) > 0.05                                   # Sim(3) scale != 1
    assert abs(float(gen["T_WC"][3:7].norm()) - 1) > 1e-3                          # non-unit quaternion
    z = gen["X_canon"][:, 2]
    assert (z == 0).any() and (z < 0).any()
    H, W = gen["image"].shape[1:]
    assert H % 2 == 1 and W % 2 == 1                                               # odd mapper sizes
    assert not gen["image"].is_contiguous()                                        # channels-last image
    conf = kinds["exact3"]["outputs"]["densePoint"][..., 3]
    assert (conf == 1).all()                                                       # r == 3 exactly: 1 / ((3 - 3) + 1)
    ex = kinds["exact3"]["inputs"]
    idx = ex["idx_k2l"].reshape(-1)
    assert ((torch.arange(idx.numel()) - idx) == 3).any()


def test_oracle_scatter_is_a_no_op_on_the_cpu():
    inp = make_inputs(24, 32, seed=5)
    a, b = oracle_dense(inp, True), oracle_dense(inp, False)
    assert torch.equal(a[0], b[0])


def test_wrappers_refuse_bad_arguments_without_a_device():
    from artdeco_b200 import _lib, keyframe
    inp = make_inputs(6, 8, seed=0)
    X = inp["X_canon"].reshape(6, 8, 3)
    N = torch.tensor([3], dtype=torch.int32)
    good = dict(last_T_WC=inp["last_T_WC"], idx_k2l=inp["idx_k2l"])
    for args, kw in (((X.reshape(-1, 3), inp["C"], N, inp["T_WC"], inp["K"]), good),
                     ((X.double(), inp["C"], N, inp["T_WC"], inp["K"]), good),
                     ((X, inp["C"], N, inp["T_WC"], inp["K"][:2]), good),
                     ((X, inp["C"], N, inp["T_WC"][:7], inp["K"]), good),
                     ((X, inp["C"], N, inp["T_WC"], inp["K"]), dict(last_T_WC=inp["last_T_WC"])),
                     ((X, inp["C"], N, inp["T_WC"], inp["K"]), dict(good, idx_k2l=inp["idx_k2l"].int())),
                     ((X, inp["C"], N, inp["T_WC"], inp["K"]), dict(good, idx_k2l=inp["idx_k2l"][:-1])),
                     ((X, inp["C"][:-1], N, inp["T_WC"], inp["K"]), {}),
                     ((X, inp["C"], N.long(), inp["T_WC"], inp["K"]), {}),
                     ((X, inp["C"], N, inp["T_WC"], inp["K"].to("meta")), good)):
        with pytest.raises(ValueError):
            keyframe.dense_point(*args, **kw)
    dense = torch.zeros(6, 8, 4)
    img = make_image(12, 16, seed=0)
    for a, kw in (((img[:2], dense, inp["T_WC"]), {}), ((img.double(), dense, inp["T_WC"]), {}),
                  ((img, dense[..., :3], inp["T_WC"]), {}), ((img, dense, inp["T_WC"][:6]), {}),
                  ((img, dense.to("meta"), inp["T_WC"]), {})):
        with pytest.raises(ValueError):
            keyframe.mapper_keyframe(*a, pyr_levels=2, index=1, is_test=False, lr_poses=1e-3, lr_exposure=1e-3, **kw)
    for L in (0, 5, 7):                                    # 12 x 16 has no 1x1 level 5; 7 levels are more than supported
        with pytest.raises(_lib.ArtdecoB200Error):
            keyframe.mapper_keyframe(img, dense, inp["T_WC"], pyr_levels=L, index=1, is_test=False, lr_poses=1e-3,
                                     lr_exposure=1e-3)
    if not torch.cuda.is_available():
        with pytest.raises(_lib.ArtdecoB200Error):
            keyframe.dense_point(X, inp["C"], N, inp["T_WC"], inp["K"], **good)
        with pytest.raises(_lib.ArtdecoB200Error):
            ours_mapper(img, dense, inp["T_WC"], 2)


def test_entry_points_refuse_bad_arguments_before_touching_the_device():
    from artdeco_b200 import _lib
    import artdeco_b200  # noqa: F401  (registers every signature)
    L = _lib.lib()

    def refused(rc, needle):
        msg = L.adb_last_error()
        return rc == 1 and msg is not None and needle in msg.decode()

    fake = 1 << 20                          # a non-null, 16-byte aligned address that is never dereferenced
    dp = [fake] * 10
    assert refused(L.adb_kf_dense_point(0, 8, *dp, None), "bad size")
    assert refused(L.adb_kf_dense_point(6, -1, *dp, None), "bad size")
    assert refused(L.adb_kf_dense_point(1 << 15, 1 << 14, *dp, None), "bad size")
    assert refused(L.adb_kf_dense_point(6, 8, None, *dp[1:], None), "null pointer")
    assert refused(L.adb_kf_dense_point(6, 8, *dp[:6], None, *dp[7:], None), "null pointer")       # no K
    assert refused(L.adb_kf_dense_point(6, 8, *dp[:5], None, *dp[6:], None), "null pointer")       # no idx_k2l
    assert refused(L.adb_kf_dense_point(6, 8, *dp[:9], None, None), "null pointer")                # no n_bad
    assert refused(L.adb_kf_dense_point(6, 8, fake, None, fake, None, None, None, fake, fake, None, None, None),
                   "null pointer")                                                                  # first: no C
    assert refused(L.adb_kf_dense_point(6, 8, *dp[:7], fake + 4, *dp[8:], None), "aligned")
    a, b = ctypes.c_longlong(0), ctypes.c_longlong(0)
    assert L.adb_kf_pyramid_floats(5, 7, 3, ctypes.byref(a), ctypes.byref(b)) == 0
    assert (a.value, b.value) == (35 + 6 + 1, 3 * (6 + 1))
    assert refused(L.adb_kf_pyramid_floats(5, 7, 4, ctypes.byref(a), ctypes.byref(b)), "coarsest level")
    assert refused(L.adb_kf_pyramid_floats(5, 7, 0, ctypes.byref(a), ctypes.byref(b)), "pyr_levels")
    assert refused(L.adb_kf_pyramid_floats(5, 7, 1, None, ctypes.byref(b)), "null pointer")
    strides = (ctypes.c_longlong * 3)(1, 48, 3)
    mi = [fake, strides, fake, fake, fake, fake, fake, fake, fake, fake]
    assert refused(L.adb_kf_mapper_inputs(12, 16, 6, 8, 0, *mi, None), "pyr_levels")
    assert refused(L.adb_kf_mapper_inputs(12, 16, 6, 8, 7, *mi, None), "pyr_levels")
    assert refused(L.adb_kf_mapper_inputs(12, 16, 6, 8, 5, *mi, None), "coarsest level")
    assert refused(L.adb_kf_mapper_inputs(12, 16, 0, 8, 2, *mi, None), "bad size")
    assert refused(L.adb_kf_mapper_inputs(0, 16, 6, 8, 1, *mi, None), "bad size")
    assert refused(L.adb_kf_mapper_inputs(12, 16, 6, 8, 2, None, *mi[1:], None), "null pointer")
    assert refused(L.adb_kf_mapper_inputs(12, 16, 6, 8, 2, *mi[:5], None, *mi[6:], None), "null pointer")   # image_pyr
    assert refused(L.adb_kf_mapper_inputs(12, 16, 6, 8, 2, *mi[:9], None, None), "null pointer")          # R
    assert refused(L.adb_kf_mapper_inputs(12, 16, 6, 8, 2, fake, strides, fake + 8, *mi[3:], None), "aligned")


# ------------------------------------------------------------------ GPU ------------------------------------------------------

@pytest.fixture
def fp32(cuda):
    m, c = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield cuda
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = m, c


def check_dense(got, want, inp, what):
    """Rows within tolerance, NaN / inf at the same places, threshold decisions equal except within 1e-6 of them."""
    dense, T_CkC, n_bad = got
    wd, wT, wbad = want
    gc, wc = dense[..., 3].reshape(-1).cpu(), wd[..., 3].reshape(-1).cpu()
    if inp["last_T_WC"] is None:
        cn = inp["C"].reshape(-1).cpu() * (1.0 / inp["N"])
        differ = gc != wc
        assert ((cn[differ] - 1.5).abs() <= 1e-6).all(), f"{what}: C/N decisions differ away from 1.5"
        keep = ~differ
        assert T_CkC is None and wT is None
    else:
        differ = (gc == 1) != (wc == 1)
        assert (torch.minimum(gc[differ], wc[differ]) >= 1 / (1 + 1e-6)).all(), f"{what}: r < 3 decisions differ away from 3"
        keep = ~differ
        assert_rows_close(T_CkC[None], wT[None], f"{what} T_CkC")
    assert int(n_bad) == wbad
    assert_rows_close(dense.reshape(-1, 4)[keep.to(dense.device)], wd.reshape(-1, 4)[keep.to(wd.device)], f"{what} densePoint")


SIZES = [  # (Hs, Ws, H, W, pyr_levels)
    (384, 512, 972, 1296, 2), (384, 512, 486, 648, 3), (37, 53, 77, 101, 4), (48, 64, 17, 31, 2), (48, 64, 17, 31, 1),
    (37, 53, 1, 101, 1), (37, 53, 77, 1, 1), (384, 512, 972, 1296, 4),
]


@pytest.mark.gpu
def test_golden_through_the_device_kernels(fp32):
    d = golden()
    L = d["args"]["pyr_levels"]
    for case in d["cases"]:
        inp = dict(case["inputs"])
        want = case["outputs"]
        first = inp["kind"] == "first"
        dv = {k: inp[k].to(fp32) for k in ("X_canon", "C", "T_WC", "last_T_WC", "idx_k2l", "K")}
        dv.update(Hs=inp["H_slam"], Ws=inp["W_slam"], N=inp["N"])
        if first:
            dv["last_T_WC"] = dv["idx_k2l"] = None
        got = ours_dense(dv)
        check_dense(got, (want["densePoint"], want["T_CkC"], 0), dv, inp["kind"])
        m = ours_mapper(inp["image"].to(fp32), want["densePoint"].to(fp32), want["T_WC"].to(fp32), L,
                        index=inp["mapper_index"])
        want_m = dict(want, R=ref.sixD2mtx(want["rW2C"]))
        compare_mapper(m, want_m, L, inp["kind"])
        lr = 0.0 if inp["mapper_index"] == 0 else 1e-3
        assert {k: p["lr"] for k, p in m["optimizer"].params.items()} == {"rW2C": lr, "tW2C": lr, "exposure": 5e-4}


@pytest.mark.gpu
@pytest.mark.parametrize("first", [False, True])
@pytest.mark.parametrize("Hs,Ws,H,W,L", SIZES)
def test_matches_the_oracle(fp32, Hs, Ws, H, W, L, first):
    inp = make_inputs(Hs, Ws, seed=Hs * 7 + W + L, dev=fp32, first=first)
    got = ours_dense(inp)
    want = oracle_dense(inp)
    check_dense(got, want, inp, f"{Hs}x{Ws}")
    image = make_image(H, W, seed=H + W, dev=fp32)
    m = ours_mapper(image, want[0], inp["T_WC"], L)
    compare_mapper(m, ref.mapper_keyframe(image, want[0], inp["T_WC"], L), L, f"{H}x{W} L={L}")
    assert m["image_pyr"][0] is image and m["image"] is image


@pytest.mark.gpu
def test_scatter_is_a_no_op(fp32):
    inp = make_inputs(384, 512, seed=11, dev=fp32)
    a, b = oracle_dense(inp, True), oracle_dense(inp, False)
    assert torch.equal(a[0], b[0])


@pytest.mark.gpu
def test_out_of_range_matches_are_nan_and_counted(fp32):
    inp = make_inputs(37, 53, seed=12, dev=fp32)
    HW = 37 * 53
    idx = inp["idx_k2l"].clone()
    idx[[0, 5, 100]] = -1
    idx[[7, HW - 1]] = HW
    idx[9] = HW + 1000
    inp["idx_k2l"] = idx
    dense, T_CkC, n_bad = ours_dense(inp)
    assert int(n_bad) == 6
    bad = torch.zeros(HW, dtype=torch.bool)
    bad[[0, 5, 100, 7, HW - 1, 9]] = True
    flat = dense.reshape(-1, 4).cpu()
    assert torch.isnan(flat[bad]).all()
    assert not torch.isnan(flat[~bad]).any()
    check_dense((dense, T_CkC, n_bad), oracle_dense(inp), inp, "bad matches")


@pytest.mark.gpu
def test_deterministic_and_graph_replay(fp32):
    from artdeco_b200 import keyframe
    inp = make_inputs(384, 512, seed=13, dev=fp32)
    image = make_image(972, 1296, seed=3, dev=fp32)
    X = inp["X_canon"].reshape(384, 512, 3)
    N = torch.tensor([3], dtype=torch.int32, device=fp32)

    def run():
        dense, T_CkC, n_bad = keyframe.dense_point(X, inp["C"], N, inp["T_WC"], inp["K"], last_T_WC=inp["last_T_WC"],
                                                   idx_k2l=inp["idx_k2l"])
        m = keyframe.mapper_keyframe(image, dense, inp["T_WC"], pyr_levels=3, index=2, is_test=False, lr_poses=1e-3,
                                     lr_exposure=5e-4)
        out = dict(dense=dense, T_CkC=T_CkC, n_bad=n_bad, **{k: m[k] for k in POSE_KEYS})
        out.update({f"id{i}": t for i, t in enumerate(m["idepth_pyr"])})
        out.update({f"im{i}": t for i, t in enumerate(m["image_pyr"][1:])})
        return out
    e1, e2 = run(), run()
    for k in e1:
        assert torch.equal(e1[k], e2[k]), k
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = run()
    for t in out.values():
        t.detach().fill_(float("nan")) if t.dtype == torch.float32 else t.detach().fill_(-1)
    graph.replay()
    torch.cuda.synchronize()
    for k in out:
        assert torch.equal(out[k].detach(), e1[k].detach()), k


@pytest.mark.gpu
def test_identity_motion_and_constant_depth(fp32):
    """Twl = Twk with s = 1 and idx_k2l = arange: the points are s Xc and every pixel in front of the camera gets conf 1; a
    constant depth gives a constant prior at every level."""
    from artdeco_b200 import keyframe
    dev = fp32
    Hs, Ws = 48, 64
    inp = make_inputs(Hs, Ws, seed=14, dev=dev)
    q = torch.tensor([0.1, -0.2, 0.3, 0.9])
    T = torch.cat([torch.tensor([0.5, -1.0, 2.0]), q / q.norm(), torch.tensor([1.0])]).to(dev)
    idx = torch.arange(Hs * Ws, device=dev)
    dense, T_CkC, n_bad = keyframe.dense_point(inp["X_canon"].reshape(Hs, Ws, 3), inp["C"], 3, T, inp["K"], last_T_WC=T,
                                               idx_k2l=idx)
    Xc = track_ref.constrain_points_to_ray(inp["X_canon"], Hs, Ws, inp["K"])
    assert_rows_close(dense.reshape(-1, 4)[:, :3], Xc, "points", tol=1e-5)
    z = Xc[:, 2]
    assert (dense.reshape(-1, 4)[z > 0, 3] == 1).all()
    assert int(n_bad) == 0
    const = torch.zeros(Hs, Ws, 4, device=dev)
    const[..., 2] = 2.5
    m = keyframe.mapper_keyframe(make_image(77, 101, seed=1, dev=dev), const, T, pyr_levels=4, index=1, is_test=True,
                                 lr_poses=1e-3, lr_exposure=5e-4)
    v = float(1.0 / (torch.tensor(2.5) + 1e-4))                 # the fp32 prior; blends and pools round within an ulp or two
    for lvl in m["idepth_pyr"]:
        assert (lvl - v).abs().max() <= 1e-6 * v
    assert set(m["optimizer"].params) == {"rW2C", "tW2C"} and m["optimizer"].params["rW2C"]["lr"] == 1e-4


@pytest.mark.gpu
def test_end_to_end_densify_render_and_loss(fp32):
    """dense_point -> mapper_keyframe -> densify.add_new_gaussians (fixed draws) and render_lod + mapper_loss at the last
    level, against the same chain fed by the oracle's tensors."""
    from artdeco_b200 import densify, synthetic
    from artdeco_b200.mapper import mapper_loss
    from artdeco_b200.optimizers import SparseGaussianAdam
    from artdeco_b200.scene import render_lod
    dev = fp32
    Hs, Ws, H, W, L = 96, 128, 243, 324, 2
    g = torch.Generator().manual_seed(21)
    inp = make_inputs(Hs, Ws, seed=21, dev=dev)
    inp["X_canon"][:, 2] = (2.0 + 6.0 * torch.rand(Hs * Ws, generator=g)).to(dev)
    q = torch.tensor([0.02, -0.01, 0.01, 1.0])
    inp["T_WC"] = torch.cat([torch.tensor([0.05, -0.02, 0.1]), q, torch.tensor([1.1])]).to(dev)
    image = make_image(H, W, seed=22, dev=dev)
    f = 0.9 * W
    n = 100_000                                                # dense enough to cover every pixel: 1 / D is finite
    sc = synthetic.raster_scene(n, seed=4, z_range=(2.0, 8.0), extent=(2.5, 2.0))
    P0 = dict(id=torch.zeros(n, 1, dtype=torch.long), cls_id=torch.randint(0, 6, (n, 1), generator=g),
              d_max=sc["d_max"], xyz=sc["means"], f_dc=sc["sh"][:, :1].clone(), f_rest=sc["sh"][:, 1:].clone(),
              scaling=torch.log(sc["scales"]), rotation=sc["quats"], opacity=torch.logit(sc["opacities"][:, None]),
              local_feat=torch.zeros(n, 20), global_feat=torch.zeros(6, 12))
    P0 = {k: v.to(dev) for k, v in P0.items()}
    uniforms = [torch.rand(H // lod, W // lod, generator=g).to(dev) for lod in densify.LODS]
    dense_o, _, _ = oracle_dense(inp)
    results = {}
    for name in ("ours", "oracle"):
        if name == "ours":
            dense = ours_dense(inp)[0]
            fr = ours_mapper(image, dense, inp["T_WC"], L)
        else:
            m = ref.mapper_keyframe(image, dense_o, inp["T_WC"], L)
            fr = dict(m, image=image, t=m["tW2C"], exposure=torch.eye(3, 4, device=dev), is_test=False)
        params = {k: {"val": v.clone(), "lr": 1e-3} for k, v in P0.items()}
        opt = SparseGaussianAdam(params, (0.5, 0.99), device=dev)
        cams = fr["approx_centre"].detach()[None]
        st = densify.add_new_gaussians(opt, fr, keyframe_id=1, cam_centres=cams, width=W, height=H, f=f, tanfovx=W / (2 * f),
                                       tanfovy=H / (2 * f), init_proba_scaler=2.0, gs_add_ratio=1.0, voxel_size=0.3,
                                       visible_threshold=0.3, local_feat_dim=20, global_feat_dim=12, uniforms=uniforms)
        P = {k: v["val"].detach() for k, v in opt.params.items()}
        h, w = fr["image_pyr"][-1].shape[1:]
        V = torch.eye(4, device=dev)
        V[:3, :3], V[:3, 3] = fr["R"].detach(), fr["t"].detach()
        pkg = render_lod(w, h, V, xyz=P["xyz"], opacity=torch.sigmoid(P["opacity"]), f_dc=P["f_dc"], f_rest=P["f_rest"],
                         scaling=torch.exp(P["scaling"]), rotation=P["rotation"], d_max=P["d_max"], tanfovx=W / (2 * f),
                         tanfovy=H / (2 * f), bg=None)
        loss = mapper_loss(pkg["colors"], pkg["alphas"], fr["image_pyr"][-1], fr["idepth_pyr"][-1],
                           torch.eye(3, 4, device=dev), torch.tensor([0.2, 0.5, 0.8], device=dev), lambda_dssim=0.2,
                           depth_weight=0.3, rad_decay=1.0, is_important=False)[0]
        results[name] = dict(st=st, P=P, loss=loss.detach())
    a, b = results["ours"], results["oracle"]
    assert a["st"]["rows"] == b["st"]["rows"] and sum(a["st"]["rows"]) > 0
    for k in ("id", "cls_id"):
        assert torch.equal(a["P"][k], b["P"][k]), k
    for k in ("xyz", "f_dc", "scaling", "opacity", "d_max"):
        assert_rows_close(a["P"][k].flatten(1), b["P"][k].flatten(1), k)
    assert torch.isfinite(b["loss"])
    assert abs(float(a["loss"]) - float(b["loss"])) <= 1e-5 * max(abs(float(b["loss"])), 1.0)

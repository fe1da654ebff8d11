"""Map re-anchoring after the Backend moves its key frames (artdeco_b200.reanchor, csrc/reanchor.cu) against the reference's
own statements (tests/golden/reanchor_small.pt, made by make_reanchor_golden.py), against oracle/reanchor_ref.py on the
device, and against an independent property: a rigidly moved map seen from the rigidly moved camera renders the same image."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from oracle import reanchor_ref as ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reanchor_small.pt")
TOL = 1e-5
POSE_KEYS = ("old_c2ws", "new_c2ws", "cam_centres", "approx_centres")


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


def random_pose_inputs(K, K_slam, seed, dev="cpu"):
    g = torch.Generator().manual_seed(seed)
    slam = torch.zeros(K_slam, 8)
    slam[:, :3] = 3.0 * torch.randn(K_slam, 3, generator=g)
    q = torch.randn(K_slam, 4, generator=g)
    slam[:, 3:7] = q / q.norm(dim=-1, keepdim=True) * (1.0 + 0.05 * torch.randn(K_slam, 1, generator=g))
    slam[:, 7] = 0.5 + torch.rand(K_slam, generator=g)
    rel = torch.zeros(K, 8)
    rel[:, :3] = 0.5 * torch.randn(K, 3, generator=g)
    q = 0.2 * torch.randn(K, 4, generator=g)
    q[:, 3] += 1.0
    rel[:, 3:7] = q / q.norm(dim=-1, keepdim=True) * (1.0 + 0.02 * torch.randn(K, 1, generator=g))
    rel[:, 7] = 0.8 + 0.4 * torch.rand(K, generator=g)
    R = ref.quat2mat(torch.randn(K, 4, generator=g))
    rW2C = (R[:, :, :2] + 0.01 * torch.randn(K, 3, 2, generator=g)).contiguous()
    tW2C = 3.0 * torch.randn(K, 3, generator=g)
    last = torch.randint(0, K_slam, (K,), generator=g)
    is_slam = torch.rand(K, generator=g) < 0.5
    d = dict(rW2C=rW2C, tW2C=tW2C, slam_T_WC=slam, last_keyframe_index=last, is_slam_keyframe=is_slam, T_CkCf=rel)
    return {k: v.to(dev) for k, v in d.items()}


def oracle_poses(inp):
    """The oracle on inp's device; the index tensors are read on the host (the reference's own frame objects)."""
    return ref.keyframe_poses(inp["rW2C"], inp["tW2C"], inp["slam_T_WC"], inp["last_keyframe_index"].cpu(),
                              inp["is_slam_keyframe"].cpu(), inp["T_CkCf"])


def random_c2ws(K, seed, dev="cpu"):
    """Rigid old / new camera-to-world tables: 4x4 inverses of get_Rt-style matrices."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(2):
        M = torch.eye(4).repeat(K, 1, 1)
        M[:, :3, :3] = ref.quat2mat(torch.randn(K, 4, generator=g))
        M[:, :3, 3] = 3.0 * torch.randn(K, 3, generator=g)
        out.append(M.to(dev))
    return out


def random_gaussians(N, K, seed, dev="cpu"):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, max(K, 1), (N, 1), generator=g)
    ids = torch.sort(ids, dim=0).values                       # rows are appended per key frame
    xyz = 4.0 * torch.randn(N, 3, generator=g)
    rot = torch.randn(N, 4, generator=g) * torch.exp(torch.randn(N, 1, generator=g))
    return ids.to(dev), xyz.to(dev), rot.to(dev)


# ------------------------------------------------------------------ CPU ------------------------------------------------------

def test_oracle_reproduces_the_reference_golden():
    d = golden()
    inp, want = d["inputs"], d["outputs"]
    got = ref.keyframe_poses(inp["rW2C"], inp["tW2C"], inp["slam_T_WC"], inp["last_keyframe_index"],
                             inp["is_slam_keyframe"], inp["T_CkCf"])
    for k in ("rW2C", "tW2C") + POSE_KEYS:
        assert_rows_close(got[k], want[k], k, tol=1e-6)
    xyz, rot, _ = ref.rigid_transform_gs(inp["id"], inp["xyz"], inp["rotation"], want["old_c2ws"], want["new_c2ws"])
    assert_rows_close(xyz, want["xyz"], "xyz", tol=1e-6)
    assert_rows_close(rot, want["rotation"], "rotation", tol=1e-6)
    assert torch.equal(want["cam_centres_scene"], want["cam_centres"])


def test_golden_covers_the_edge_cases():
    d = golden()
    inp, out = d["inputs"], d["outputs"]
    assert inp["is_slam_keyframe"].any() and (~inp["is_slam_keyframe"]).any()
    assert ((inp["slam_T_WC"][:, 7] - 1).abs() > 0.05).all()                          # Sim(3) scale != 1
    assert ((inp["slam_T_WC"][:, 3:7].norm(dim=-1) - 1).abs() > 1e-3).any()           # non-unit quaternions
    R = ref.sixD2mtx(inp["rW2C"])
    assert ((R[:, :, :2] - inp["rW2C"]).abs().amax() > 1e-3)                          # non-orthonormal 6-D rotations
    assert (inp["rotation"] == 0).all(-1).any()                                       # a zero quaternion
    _, _, mats = ref.rigid_transform_gs(inp["id"], inp["xyz"], inp["rotation"], out["old_c2ws"], out["new_c2ws"])
    b, _ = ref.mat2quat_branch(mats)
    assert set(b.reshape(-1).tolist()) == {0, 1, 2, 3}
    assert not torch.equal(out["cam_centres"], out["approx_centres"])                  # two different R, both used


def test_conversions_round_trip_and_reach_every_branch():
    g = torch.Generator().manual_seed(1)
    q = torch.randn(20000, 4, generator=g, dtype=torch.float64) * torch.exp(torch.randn(20000, 1, generator=g,
                                                                                        dtype=torch.float64))
    m = ref.quat2mat(q)
    eye = torch.eye(3, dtype=torch.float64)
    assert (m @ m.transpose(-1, -2) - eye).abs().max() < 1e-12 and (torch.det(m) - 1).abs().max() < 1e-12
    back = ref.mat2quat(m)
    qn = q / q.norm(dim=-1, keepdim=True)
    assert torch.minimum((back - qn).abs().amax(-1), (back + qn).abs().amax(-1)).max() < 1e-7   # eps 1e-8 in the sqrt
    assert set(ref.mat2quat_branch(m)[0].tolist()) == {0, 1, 2, 3}
    # rotations near pi about x, y and z pick branches 1, 2, 3; a small rotation picks the trace branch
    for axis, branch in ((0, 1), (1, 2), (2, 3)):
        a = math.pi - 0.01
        qa = torch.zeros(1, 4, dtype=torch.float64)
        qa[0, 0], qa[0, 1 + axis] = math.cos(a / 2), math.sin(a / 2)
        assert int(ref.mat2quat_branch(ref.quat2mat(qa))[0]) == branch
    assert int(ref.mat2quat_branch(ref.quat2mat(torch.tensor([[1.0, 0.1, 0.0, 0.0]])))[0]) == 0
    assert torch.equal(ref.quat2mat(torch.zeros(1, 4))[0], torch.eye(3))                  # zero quaternion: identity


def test_pypose_path_agrees_with_float64_matrix_algebra():
    """With unit Sim(3) quaternions, T_WCf is the Sim(3) matrix product with the scale dropped from the rotation only."""
    inp = random_pose_inputs(40, 9, seed=3)
    q = inp["slam_T_WC"][:, 3:7]
    inp["slam_T_WC"][:, 3:7] = q / q.norm(dim=-1, keepdim=True)
    got = oracle_poses(inp)
    D = lambda t: t.double()  # noqa: E731

    def sim3(T):
        M = torch.eye(4, dtype=torch.float64)
        M[:3, :3] = D(T[7]) * ref.quat2mat(D(T[[6, 3, 4, 5]])[None])[0]
        M[:3, 3] = D(T[:3])
        return M
    for k in range(40):
        T = inp["slam_T_WC"][int(inp["last_keyframe_index"][k])]
        if bool(inp["is_slam_keyframe"][k]):
            R, t = ref.quat2mat(D(T[[6, 3, 4, 5]])[None])[0], D(T[:3])
        else:
            B = inp["T_CkCf"][k]
            M = sim3(T) @ sim3(B)
            R = ref.quat2mat(D(T[[6, 3, 4, 5]])[None])[0] @ ref.quat2mat(D(B[[6, 3, 4, 5]])[None])[0]
            t = M[:3, 3]
        c2w = torch.eye(4, dtype=torch.float64)
        c2w[:3, :3], c2w[:3, 3] = R, t
        w2c = torch.linalg.inv(c2w)
        old = torch.eye(4, dtype=torch.float64)
        old[:3, :3], old[:3, 3] = ref.sixD2mtx(D(inp["rW2C"][k])), D(inp["tW2C"][k])
        for name, val in (("new_c2ws", c2w), ("old_c2ws", torch.linalg.inv(old)), ("rW2C", w2c[:3, :2]),
                          ("tW2C", w2c[:3, 3]), ("approx_centres", t), ("cam_centres", t)):
            assert_rows_close(got[name][k][None], val[None], f"frame {k} {name}", tol=2e-5)


def test_wrappers_refuse_bad_arguments_without_a_device():
    from artdeco_b200 import _lib, reanchor
    inp = random_pose_inputs(5, 3, seed=0)
    args = [inp[k] for k in ("rW2C", "tW2C", "slam_T_WC", "last_keyframe_index", "is_slam_keyframe", "T_CkCf")]
    for i, bad in ((0, torch.zeros(5, 2, 3)), (1, torch.zeros(5, 4)), (2, torch.zeros(3, 7)),
                   (3, inp["last_keyframe_index"].int()), (4, torch.zeros(5)), (5, torch.zeros(4, 8)),
                   (1, torch.zeros(5, 3, dtype=torch.float64)), (2, torch.zeros(3, 8, device="meta"))):
        a = list(args)
        a[i] = bad
        with pytest.raises(ValueError):
            reanchor.keyframe_poses(*a)
    with pytest.raises(ValueError):
        reanchor.keyframe_poses(inp["rW2C"].transpose(1, 2).contiguous().transpose(1, 2), *args[1:])
    ids, xyz, rot = random_gaussians(10, 5, seed=0)
    old, new = random_c2ws(5, seed=0)
    cams = torch.zeros(5, 3)

    def params(**over):
        p = dict(id=ids, xyz=xyz, rotation=rot)
        p.update(over)
        return {k: {"val": v} for k, v in p.items()}
    for p, o, n, c in ((params(id=ids.int()), old, new, cams), (params(id=ids[:, 0]), old, new, cams),
                       (params(rotation=rot[:, :3]), old, new, cams), (params(xyz=xyz.double()), old, new, cams),
                       (params(), old[:, :3], new, cams), (params(), old, new[:4], cams), (params(), old, new, cams[:, :2]),
                       (params(), old, new.to("meta"), cams), ({"xyz": {"val": xyz}}, old, new, cams)):
        with pytest.raises(ValueError):
            reanchor.rigid_transform_gs(p, o, n, c)
    if not torch.cuda.is_available():
        with pytest.raises(_lib.ArtdecoB200Error):
            reanchor.keyframe_poses(*args)
        with pytest.raises(_lib.ArtdecoB200Error):
            reanchor.rigid_transform_gs(params(), old, new, cams)


def test_entry_points_refuse_bad_arguments_before_touching_the_device():
    from artdeco_b200 import _lib
    import artdeco_b200  # noqa: F401  (registers every signature)
    L = _lib.lib()

    def refused(rc, needle, status=1):
        msg = L.adb_last_error()
        return rc == status and msg is not None and needle in msg.decode()

    nb = ctypes.c_size_t(0)
    assert refused(L.adb_reanchor_workspace_bytes(-1, ctypes.byref(nb)), "K must be")
    assert refused(L.adb_reanchor_workspace_bytes(4, None), "null bytes")
    assert L.adb_reanchor_workspace_bytes(300, ctypes.byref(nb)) == 0 and nb.value == 300 * 64
    fake = 1 << 20                          # a non-null, 16-byte aligned address that is never dereferenced
    kf = [fake] * 11
    assert refused(L.adb_reanchor_keyframes(-1, 3, *kf, None), "K and K_slam")
    assert refused(L.adb_reanchor_keyframes(4, 3, fake, None, *kf[2:], None), "null pointer")
    assert refused(L.adb_reanchor_keyframes(4, 3, *kf[:-1], None, None), "null pointer")
    assert L.adb_reanchor_keyframes(0, 3, *([None] * 11), None) == 0           # K = 0: nothing to do, nothing read
    g = [fake] * 7
    ws_need = 7 * 64
    assert refused(L.adb_reanchor_gaussians(-1, 7, *g, fake, fake, ws_need, None), "N and K")
    assert refused(L.adb_reanchor_gaussians(100, 7, None, *g[1:], fake, fake, ws_need, None), "null pointer")
    assert refused(L.adb_reanchor_gaussians(100, 7, *g, None, fake, ws_need, None), "null pointer")
    assert refused(L.adb_reanchor_gaussians(100, 7, fake, fake, fake + 4, *g[3:], fake, fake, ws_need, None), "aligned")
    assert refused(L.adb_reanchor_gaussians(100, 7, *g, fake, fake, ws_need - 1, None), "workspace too small", 3)
    assert refused(L.adb_reanchor_gaussians(1 << 31, 7, *g, fake, fake, ws_need, None), "N must be")
    assert L.adb_reanchor_gaussians(0, 7, *([None] * 9), 0, None) == 0         # N = 0 launches nothing


# ------------------------------------------------------------------ GPU ------------------------------------------------------

@pytest.fixture
def fp32(cuda):
    m, c = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield cuda
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = m, c


@pytest.mark.gpu
def test_golden_through_the_device_kernels(fp32):
    from artdeco_b200 import reanchor
    d = golden()
    inp = {k: v.to(fp32) for k, v in d["inputs"].items()}
    want = d["outputs"]
    rW2C, tW2C = inp["rW2C"].clone(), inp["tW2C"].clone()
    out = reanchor.keyframe_poses(rW2C, tW2C, inp["slam_T_WC"], inp["last_keyframe_index"], inp["is_slam_keyframe"],
                                  inp["T_CkCf"])
    for name, got in zip(POSE_KEYS, out[:4]):
        assert_rows_close(got, want[name], name)
    assert_rows_close(rW2C, want["rW2C"], "rW2C")
    assert_rows_close(tW2C, want["tW2C"], "tW2C")
    assert int(out[4]) == 0
    params = {k: {"val": inp[k].clone()} for k in ("id", "xyz", "rotation")}
    n_bad = reanchor.rigid_transform_gs(params, want["old_c2ws"].to(fp32), want["new_c2ws"].to(fp32),
                                        want["cam_centres"].to(fp32))
    assert int(n_bad) == 0
    assert_rows_close(params["xyz"]["val"], want["xyz"], "xyz")
    assert_rows_close(params["rotation"]["val"], want["rotation"], "rotation")


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 7, 300, 2000])
def test_keyframe_poses_match_the_oracle(fp32, K):
    from artdeco_b200 import reanchor
    K_slam = max(K // 3, 1)
    inp = random_pose_inputs(K, K_slam, seed=K, dev=fp32)
    bad = torch.zeros(K, dtype=torch.bool)
    if K >= 7:
        bad[[1, K - 2]] = True
        inp["last_keyframe_index"][1] = -1
        inp["last_keyframe_index"][K - 2] = K_slam
    good = (~bad).nonzero()[:, 0].to(fp32)
    want = oracle_poses({k: v if k == "slam_T_WC" else v[good] for k, v in inp.items()})
    rW2C0, tW2C0 = inp["rW2C"].clone(), inp["tW2C"].clone()
    rW2C, tW2C = inp["rW2C"], inp["tW2C"]
    p_r, p_t = rW2C.data_ptr(), tW2C.data_ptr()
    out = reanchor.keyframe_poses(rW2C, tW2C, inp["slam_T_WC"], inp["last_keyframe_index"], inp["is_slam_keyframe"],
                                  inp["T_CkCf"])
    got = dict(zip(POSE_KEYS, out[:4]))
    assert rW2C.data_ptr() == p_r and tW2C.data_ptr() == p_t                     # updated in place
    assert int(out[4]) == int(bad.sum())
    for k in POSE_KEYS:
        assert_rows_close(got[k][good], want[k], f"K={K} {k}")
    assert_rows_close(rW2C[good], want["rW2C"], f"K={K} rW2C")
    assert_rows_close(tW2C[good], want["tW2C"], f"K={K} tW2C")
    if bad.any():
        b = bad.to(fp32)
        assert torch.equal(rW2C[b], rW2C0[b]) and torch.equal(tW2C[b], tW2C0[b])
        assert torch.equal(got["new_c2ws"][b], got["old_c2ws"][b])
        old = torch.eye(4, device=fp32).repeat(int(bad.sum()), 1, 1)
        old[:, :3, :3], old[:, :3, 3] = ref.sixD2mtx(rW2C0[b]), tW2C0[b]
        assert_rows_close(got["old_c2ws"][b], torch.linalg.inv(old), "unchanged rows old_c2ws")
        assert_rows_close(got["cam_centres"][b], torch.linalg.inv(old)[:, :3, 3], "unchanged rows cam_centres")


def compare_gaussians(got_xyz, got_rot, want_xyz, want_rot, mats, what):
    assert_rows_close(got_xyz, want_xyz, f"{what} xyz")
    a, b = got_rot.double(), want_rot.double()
    assert torch.equal(torch.isnan(a), torch.isnan(b)), f"{what}: rotation NaN at different places"
    fin = torch.isfinite(b).all(-1)
    assert torch.equal(torch.isfinite(a).all(-1), fin), f"{what}: rotation inf at different places"
    diff = (a - b).abs().amax(-1)
    differ = fin & (diff > TOL)
    if differ.any():
        # only where the oracle's own branch decision was within 1e-5 of a tie, and then the same rotation
        _, margin = ref.mat2quat_branch(mats)
        assert (margin.reshape(-1)[differ] <= 1e-5).all(), f"{what}: {int(differ.sum())} rows differ away from a tie"
        assert int(differ.sum()) <= 1e-4 * got_rot.shape[0], f"{what}: {int(differ.sum())} branch flips"
        na, nb = a[differ] / a[differ].norm(dim=-1, keepdim=True), b[differ] / b[differ].norm(dim=-1, keepdim=True)
        assert ((na * nb).sum(-1).abs() >= 1 - 1e-5).all(), f"{what}: a flipped row is not the same rotation"


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 7, 300])
@pytest.mark.parametrize("N", [1, 31, 1000, 100_000, 1_000_000])
def test_rigid_transform_matches_the_oracle(fp32, N, K):
    from artdeco_b200 import reanchor
    dev = fp32
    ids, xyz, rot = random_gaussians(N, K, seed=N + K, dev=dev)
    old, new = random_c2ws(K, seed=K, dev=dev)
    if N >= 31:
        unit = torch.tensor([0.3, -0.5, 0.1, 0.8], device=dev)
        rot[0] = 0.0                                                # zero: the identity
        rot[1] = torch.tensor([1e-20, 0.0, 0.0, 0.0], device=dev)   # tiny norms
        rot[2] = torch.tensor([0.0, 0.0, -1e-20, 1e-20], device=dev)
        rot[3] = unit * 1e18                                        # huge but finite norm
        rot[4] = unit * 1e30                                        # the norm overflows to inf: q / inf = 0
        rot[5, 2] = float("nan")
        rot[6, 0] = float("inf")
        xyz[7, 1] = float("nan")
        xyz[8, 2] = float("-inf")
    params = {"id": {"val": ids}, "xyz": {"val": xyz.clone()}, "rotation": {"val": rot.clone()}}
    n_bad = reanchor.rigid_transform_gs(params, old, new, torch.zeros(K, 3, device=dev))
    want_xyz, want_rot, mats = ref.rigid_transform_gs(ids, xyz, rot, old, new)
    assert int(n_bad) == 0
    compare_gaussians(params["xyz"]["val"], params["rotation"]["val"], want_xyz, want_rot, mats, f"N={N} K={K}")
    # bitwise reproducible
    again = {"id": {"val": ids}, "xyz": {"val": xyz.clone()}, "rotation": {"val": rot.clone()}}
    reanchor.rigid_transform_gs(again, old, new, torch.zeros(K, 3, device=dev))
    for k in ("xyz", "rotation"):
        assert torch.equal(torch.nan_to_num(params[k]["val"], nan=7.0), torch.nan_to_num(again[k]["val"], nan=7.0))


@pytest.mark.gpu
def test_out_of_range_ids_and_singular_frames_are_left_unchanged_and_counted(fp32):
    from artdeco_b200 import reanchor
    dev = fp32
    K, N = 7, 5000
    ids, xyz, rot = random_gaussians(N, K, seed=11, dev=dev)
    old, new = random_c2ws(K, seed=12, dev=dev)
    old[3, :, 1] = 0.0                                              # a zero column: singular
    ids[10:20] = -1
    ids[20:25] = K
    params = {"id": {"val": ids}, "xyz": {"val": xyz.clone()}, "rotation": {"val": rot.clone()}}
    n_bad = reanchor.rigid_transform_gs(params, old, new, torch.zeros(K, 3, device=dev))
    frozen = (ids[:, 0] < 0) | (ids[:, 0] >= K) | (ids[:, 0] == 3)
    assert int(n_bad) == int(frozen.sum()) and int((ids[:, 0] == 3).sum()) > 0
    assert torch.equal(params["xyz"]["val"][frozen], xyz[frozen])
    assert torch.equal(params["rotation"]["val"][frozen], rot[frozen])
    ok = ~frozen
    want_xyz, want_rot, mats = ref.rigid_transform_gs(ids[ok], xyz[ok], rot[ok], old, new)
    compare_gaussians(params["xyz"]["val"][ok], params["rotation"]["val"][ok], want_xyz, want_rot, mats, "valid rows")


@pytest.mark.gpu
def test_empty_map(fp32):
    from artdeco_b200 import reanchor
    old, new = random_c2ws(3, seed=1, dev=fp32)
    params = {"id": {"val": torch.zeros(0, 1, dtype=torch.long, device=fp32)},
              "xyz": {"val": torch.zeros(0, 3, device=fp32)}, "rotation": {"val": torch.zeros(0, 4, device=fp32)}}
    n_bad = reanchor.rigid_transform_gs(params, old, new, torch.zeros(3, 3, device=fp32))
    assert params["xyz"]["val"].shape == (0, 3) and params["rotation"]["val"].shape == (0, 4) and int(n_bad) == 0


@pytest.mark.gpu
def test_scene_level_with_the_optimiser(fp32):
    """Only xyz / rotation change; moments and lr stay bitwise; both stop requiring grad, step skips them, and the next
    add_and_prune makes them trainable again (the reference's own behaviour)."""
    from artdeco_b200 import reanchor
    from artdeco_b200.optimizers import SparseGaussianAdam
    dev = fp32
    K, N = 5, 20000
    g = torch.Generator().manual_seed(2)
    ids, xyz, rot = random_gaussians(N, K, seed=3, dev=dev)
    vals = dict(id=ids, xyz=xyz, rotation=rot, f_dc=torch.randn(N, 1, 3, generator=g).to(dev),
                f_rest=torch.randn(N, 15, 3, generator=g).to(dev), scaling=torch.randn(N, 3, generator=g).to(dev),
                opacity=torch.randn(N, 1, generator=g).to(dev))
    params = {k: {"val": v.clone(), **({} if k == "id" else {"lr": 1e-3})} for k, v in vals.items()}
    opt = SparseGaussianAdam(params, (0.5, 0.99), device=dev)
    keep = torch.ones(N, dtype=torch.bool, device=dev)
    opt.add_and_prune({k: v["val"][:0].detach() for k, v in params.items()}, keep)
    vis = (torch.rand(N, generator=g) > 0.3).to(dev)

    def grads():
        for k, p in params.items():
            if p["val"].requires_grad:
                p["val"].grad = torch.randn(p["val"].shape, generator=g).to(dev)
    grads()
    opt.step(vis, N, None, 0)
    snap = {k: {s: (t.clone() if isinstance(t, torch.Tensor) else t) for s, t in p.items()} for k, p in params.items()}
    old, new = random_c2ws(K, seed=4, dev=dev)
    reanchor.rigid_transform_gs(params, old, new, torch.zeros(K, 3, device=dev))
    for k, p in params.items():
        for s, t in p.items():
            if s == "val" and k in ("xyz", "rotation"):
                assert not torch.equal(t, snap[k][s]) and not t.requires_grad, k
            else:
                assert torch.equal(t, snap[k][s]), (k, s)
    moved = {k: params[k]["val"].clone() for k in ("xyz", "rotation")}
    grads()
    opt.step(vis, N, None, 0)
    for k in ("xyz", "rotation"):
        assert torch.equal(params[k]["val"], moved[k]), k                           # skipped: no grad
        assert torch.equal(params[k]["exp_avg"], snap[k]["exp_avg"]), k
    assert not torch.equal(params["f_dc"]["val"], snap["f_dc"]["val"])
    opt.add_and_prune({k: v["val"][:0].detach() for k, v in params.items()}, keep)
    assert params["xyz"]["val"].requires_grad and params["rotation"]["val"].requires_grad


@pytest.mark.gpu
def test_moved_map_renders_the_same_from_the_moved_camera(fp32):
    """Every Gaussian in key frame 0 with f_rest = 0: rendering the old map from the old pose and the moved map from the new
    pose (keyframe.get_Rt after set_Rt) gives the same image within the rasterizer's 1e-4 of scale."""
    from helpers import assert_close
    from artdeco_b200 import reanchor, synthetic
    from artdeco_b200.scene import render_lod
    dev = fp32
    H, W = 360, 480
    f = 0.8 * W
    sc = synthetic.raster_scene(100_000, seed=5, z_range=(2.0, 8.0), extent=(2.5, 2.0))
    inp = random_pose_inputs(1, 1, seed=6)
    # the current pose is the identity, so the synthetic scene (world == camera 0) is in front of the camera
    inp["rW2C"] = torch.tensor([[[1.0, 0.0], [0.0, 1.0], [0.0, 0.0]]])
    inp["tW2C"] = torch.zeros(1, 3)
    inp["is_slam_keyframe"] = torch.tensor([False])
    inp["slam_T_WC"][0] = torch.tensor([0.3, -0.2, 0.5, 0.05, -0.08, 0.02, 1.0, 1.3])
    inp = {k: v.to(dev) for k, v in inp.items()}
    V_old = torch.eye(4, device=dev)
    V_old[:3, :3], V_old[:3, 3] = ref.sixD2mtx(inp["rW2C"][0]), inp["tW2C"][0]
    old, new, cams, _, _ = reanchor.keyframe_poses(inp["rW2C"], inp["tW2C"], inp["slam_T_WC"], inp["last_keyframe_index"],
                                                   inp["is_slam_keyframe"], inp["T_CkCf"])
    V_new = torch.eye(4, device=dev)
    V_new[:3, :3], V_new[:3, 3] = ref.sixD2mtx(inp["rW2C"][0]), inp["tW2C"][0]
    assert (V_new - V_old).abs().max() > 0.1
    N = sc["means"].shape[0]
    params = {"id": {"val": torch.zeros(N, 1, dtype=torch.long, device=dev)}, "xyz": {"val": sc["means"].to(dev)},
              "rotation": {"val": sc["quats"].to(dev)}}
    common = dict(opacity=sc["opacities"][:, None].to(dev), f_dc=sc["sh"][:, :1].to(dev),
                  f_rest=torch.zeros(N, 15, 3, device=dev), scaling=sc["scales"].to(dev), d_max=sc["d_max"].to(dev),
                  tanfovx=W / (2 * f), tanfovy=H / (2 * f))
    before = render_lod(W, H, V_old, xyz=params["xyz"]["val"], rotation=params["rotation"]["val"], **common)
    reanchor.rigid_transform_gs(params, old, new, cams)
    after = render_lod(W, H, V_new, xyz=params["xyz"]["val"], rotation=params["rotation"]["val"], **common)
    assert before["render"].abs().max() > 0.1
    assert_close(after["render"], before["render"], what="render", max_outlier_frac=1e-3)


@pytest.mark.gpu
def test_both_calls_in_one_cuda_graph(fp32):
    """Captured together, the two calls replay to the eager result: neither reads anything on the host."""
    from artdeco_b200 import reanchor
    dev = fp32
    K, N = 40, 200_000
    inp = random_pose_inputs(K, 12, seed=8, dev=dev)
    ids, xyz, rot = random_gaussians(N, K, seed=9, dev=dev)
    r0, t0 = inp["rW2C"].clone(), inp["tW2C"].clone()

    def run(rW2C, tW2C):
        old, new, cams, approx, nb = reanchor.keyframe_poses(rW2C, tW2C, inp["slam_T_WC"], inp["last_keyframe_index"],
                                                             inp["is_slam_keyframe"], inp["T_CkCf"])
        params = {"id": {"val": ids}, "xyz": {"val": xyz}, "rotation": {"val": rot}}
        nb2 = reanchor.rigid_transform_gs(params, old, new, cams)
        return dict(old=old, new=new, cams=cams, approx=approx, xyz=params["xyz"]["val"],
                    rotation=params["rotation"]["val"], nb=nb + nb2)

    moved = [(r0.clone(), t0.clone()) for _ in range(2)]
    eager = [run(r, t) for r, t in moved]
    assert torch.equal(moved[0][0], moved[1][0]) and torch.equal(moved[0][1], moved[1][1])
    for k in eager[0]:
        assert torch.equal(eager[0][k], eager[1][k]), k                            # bitwise reproducible
    rW2C, tW2C = r0.clone(), t0.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run(rW2C, tW2C)                                                            # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    rW2C.copy_(r0)
    tW2C.copy_(t0)
    with torch.cuda.graph(graph):
        out = run(rW2C, tW2C)
    rW2C.copy_(r0)
    tW2C.copy_(t0)
    graph.replay()
    torch.cuda.synchronize()
    for k in out:
        assert torch.equal(out[k], eager[0][k]), k
    assert torch.equal(rW2C, moved[0][0]) and torch.equal(tW2C, moved[0][1])
    assert int(out["nb"]) == 0

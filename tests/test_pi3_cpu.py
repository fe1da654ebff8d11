"""Pi3 without a GPU: the plain-torch oracle against the golden files made by running the reference, the parameter table,
the position-embedding resize, and the C-ABI refusals of the Pi3 entry points."""
import ctypes
from pathlib import Path

import pytest
import torch

from artdeco_b200 import synthetic
from artdeco_b200.pi3 import interpolate_pos_embed, param_shapes
from oracle import pi3_torch as pt

GOLDEN = Path(__file__).resolve().parent / "golden"


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


@pytest.fixture(scope="module")
def weights():
    return synthetic.det_weights(param_shapes())


@pytest.mark.parametrize("tag", ["small", "full"])
def test_oracle_matches_reference_golden(weights, tag):
    g = torch.load(GOLDEN / f"pi3_{tag}.pt", weights_only=False)
    sp, tk, ch = g["stride_px"], g["stride_tok"], g["stride_ch"]
    st = {}
    with torch.inference_mode():
        out = pt.forward(weights, synthetic.pi3_frames(g["N"], g["H"], g["W"], seed=g["seed"]), stages=st)
    for k in ("points", "local_points", "conf"):
        assert rel(out[k][:, :, ::sp, ::sp], g[k]) < 1e-5, k
    assert rel(out["camera_poses"], g["camera_poses"]) < 1e-5
    assert rel(st["fc_rot"], g["fc_rot"]) < 1e-5 and rel(st["fc_t"], g["fc_t"]) < 1e-5
    for k in ("encoder", "decoder", "point_hidden", "conf_hidden", "camera_hidden"):
        assert rel(st[k][:, ::tk, ::ch], g["stage." + k]) < 1e-5, k


def test_param_shapes_equal_reference_read_set():
    for tag in ("small", "full"):
        g = torch.load(GOLDEN / f"pi3_{tag}.pt", weights_only=False)
        assert {k: tuple(v) for k, v in param_shapes().items()} == g["read_set"]
    assert "encoder.mask_token" not in param_shapes()


@pytest.mark.parametrize("tag", ["small", "full"])
def test_pos_embed_interpolation_is_bit_equal(tag):
    g = torch.load(GOLDEN / f"pi3_{tag}.pt", weights_only=False)
    pe = synthetic.det_weights({"encoder.pos_embed": param_shapes()["encoder.pos_embed"]})["encoder.pos_embed"]
    t = interpolate_pos_embed(pe, g["H"] // 14, g["W"] // 14)[:, ::g["stride_tok"], ::g["stride_ch"]]
    assert t.shape == g["pos_table"].shape and torch.equal(t, g["pos_table"])
    # the native grid returns the table itself, as the reference does
    assert interpolate_pos_embed(pe, 37, 37) is pe


def test_pi3_entry_points_refuse_bad_arguments_before_touching_the_device():
    from artdeco_b200 import _lib
    import artdeco_b200  # noqa: F401  (registers every signature)
    L = _lib.lib()

    def refused(rc, needle):
        msg = L.adb_last_error()
        return rc == 1 and msg is not None and needle in msg.decode()

    p = ctypes.c_void_p(256)            # aligned, never dereferenced
    odd = ctypes.c_void_p(258)          # 2-byte aligned only
    # H or W not a multiple of 14
    assert refused(L.adb_pi3_patch14(1, 100, 140, p, p, p, None), "multiples of 14")
    assert refused(L.adb_pi3_patch14(1, 112, 141, p, p, p, None), "multiples of 14")
    assert refused(L.adb_pi3_point_head(1, 112, 130, 5 + 8 * 9, 5, p, p, p, p, p, p, None), "multiples of 14")
    assert refused(L.adb_pi3_window_input(2, 100, 100, p, 392, 520, p, None), "multiples of 14")
    # N < 1
    assert refused(L.adb_pi3_patch14(0, 112, 140, p, p, p, None), "at least one frame")
    assert refused(L.adb_pi3_point_head(0, 112, 140, 85, 5, p, p, p, p, p, p, None), "at least one frame")
    assert refused(L.adb_pi3_svd_pose(0, p, p, p, None), "at least one view")
    assert refused(L.adb_pi3_window_input(0, 100, 100, p, 392, 518, p, None), "bad input size")
    assert refused(L.adb_pi3_tokens(0, 80, 1024, p, p, p, p, p, None), "bad sizes")
    assert refused(L.adb_pi3_camera_tail(0, 85, 5, p, p, p, p, p, p, p, p, p, p, p, None), "bad sizes")
    assert refused(L.adb_qknorm_rope(0, 85, 16, 3072, 0, p, p, p, ctypes.c_float(1e-5), p, p, 64, p, p, None), "bad sizes")
    # wrong token count for the grid
    assert refused(L.adb_pi3_point_head(1, 112, 140, 80, 5, p, p, p, p, p, p, None), "hw must be")
    # misaligned pointers
    assert refused(L.adb_pi3_patch14(1, 112, 140, p, odd, p, None), "aligned")
    assert refused(L.adb_pi3_tokens(1, 80, 1024, p, p, p, odd, p, None), "aligned")
    assert refused(L.adb_qknorm_rope(1, 85, 16, 3072, 0, odd, p, p, ctypes.c_float(1e-5), p, p, 64, p, p, None), "misaligned")
    assert refused(L.adb_pi3_point_head(1, 112, 140, 85, 5, p, p, p, ctypes.c_void_p(257), p, p, None), "misaligned")
    assert refused(L.adb_pi3_camera_tail(1, 85, 5, ctypes.c_void_p(257), p, p, p, p, p, p, p, p, p, p, None), "misaligned")
    assert refused(L.adb_pi3_svd_pose(1, ctypes.c_void_p(257), p, p, None), "misaligned")
    assert refused(L.adb_pi3_window_input(1, 100, 100, ctypes.c_void_p(257), 392, 518, p, None), "misaligned")
    # null pointers and a lone LayerNorm parameter
    assert refused(L.adb_pi3_patch14(1, 112, 140, None, p, p, None), "null pointer")
    assert refused(L.adb_qknorm_rope(1, 85, 16, 3072, 0, p, p, None, ctypes.c_float(1e-5), p, p, 64, p, p, None),
                   "gamma and beta")


def test_flop_count_of_the_loop_closure_window():
    from artdeco_b200.pi3.model import flops
    f = flops(24)
    assert 90e12 < f < 115e12, f     # about 100 TFLOP for 24 frames at 392x518

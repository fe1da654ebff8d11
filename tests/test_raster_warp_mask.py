"""The blend kernels' per-entry warp mask (csrc/raster_blend.cu warp_mask), restated in numpy.

Bit w of an entry's mask says that warp w's 8x4 pixel block of the tile may hold a pixel where the splat passes the per-pixel
test 0 <= sigma2 <= smax2; a warp evaluates only the entries carrying its bit.  The restatement follows the kernel operation
for operation in float32 and is checked, on random and adversarial records, against a brute-force walk over the tile's 256
pixel centres:
  (a) every block holding a pixel that passes the float32 per-pixel test (with and without FMA contraction) keeps its bit;
  (b) on projection-like splats, the bits kept beyond the float64 exact set stay below a stated fraction of all bits kept.
"""
import numpy as np
import pytest

LOG2E = np.float32(1.4426950408889634)
F = np.float32


def warp_mask(mx, my, ha, b, hc, smax2, rx, ry, tx0, ty0):
    """float32 restatement of warp_mask for arrays of records; rx / ry = 65535 means unbounded."""
    mx, my, ha, b, hc, smax2 = (np.asarray(t, np.float32) for t in (mx, my, ha, b, hc, smax2))
    tx0, ty0 = F(tx0), F(ty0)
    with np.errstate(all="ignore"):
        rxf = np.where(rx == 0xFFFF, F(3.0e38), np.asarray(rx, np.float32)).astype(np.float32)
        ryf = np.where(ry == 0xFFFF, F(3.0e38), np.asarray(ry, np.float32)).astype(np.float32)
        D = F(4) * ha * hc - b * b
        kap = (F(4) * ha * hc) / D
        conic_ok = (ha > 0) & (hc > 0) & (D > 0) & (kap < F(1.0e6))
        S = np.maximum(F(0), smax2 * (F(1.0002) + F(2.0e-6) * kap) + F(2.0e-4))
        pad = F(1.0e-3) + F(2.0e-6) * np.maximum(np.abs(mx), np.abs(my))
        rD = F(1) / D
        S4a = F(4) * ha * S
        xm = np.sqrt(F(4) * hc * S * rD)
        ym = np.sqrt(S4a * rD)
        eR = F(-0.5) * b * xm * (F(1) / hc)
        r2a = F(1) / (F(2) * ha)
        mask = np.zeros(mx.shape, np.uint32)
        for h in range(2):
            xlo = tx0 + F(8 * h)
            xhi = xlo + F(7)
            mask |= np.where((mx + rxf >= xlo) & (mx - rxf <= xhi), np.uint32(0x55 << h), np.uint32(0))
        rows = np.zeros(mx.shape, np.uint32)
        for k in range(4):
            ylo = ty0 + F(4 * k)
            yhi = ylo + F(3)
            box = (my + ryf >= ylo) & (my - ryf <= yhi)
            e0 = ylo - my - pad
            e1 = yhi - my + pad
            band = (e0 <= ym) & (e1 >= -ym)
            cR = np.minimum(e1, np.maximum(e0, eR))
            cL = np.minimum(e1, np.maximum(e0, -eR))
            xR = mx + (np.sqrt(np.maximum(F(0), S4a - D * cR * cR)) - b * cR) * r2a + pad
            xL = mx - (np.sqrt(np.maximum(F(0), S4a - D * cL * cL)) + b * cL) * r2a - pad
            for h in range(2):
                xlo = tx0 + F(8 * h)
                xhi = xlo + F(7)
                hit = box & (~conic_ok | (band & (xL <= xhi) & (xR >= xlo)))
                rows |= np.where(hit, np.uint32(1 << (2 * k + h)), np.uint32(0))
    return (mask & rows).astype(np.uint8)


def pixel_mask(mx, my, ha, b, hc, smax2, tx0, ty0, dtype=np.float32, fma=False):
    """Brute force: bit w set where some pixel centre of warp w's block passes 0 <= sigma2 <= smax2 in `dtype`.
    fma=True contracts the two multiply-adds as the blend kernels' compiled code does (emulated in float64, rounded once)."""
    n = len(mx)
    out = np.zeros(n, np.uint8)
    for w in range(8):
        xs = tx0 + 8 * (w & 1) + np.arange(8)
        ys = ty0 + 4 * (w >> 1) + np.arange(4)
        px, py = (t.astype(dtype) for t in np.meshgrid(xs, ys))
        px, py = px.reshape(1, -1), py.reshape(1, -1)
        c = [np.asarray(t, dtype).reshape(-1, 1) for t in (mx, my, ha, b, hc, smax2)]
        dx, dy = c[0] - px, c[1] - py
        if fma:
            inner = (c[2].astype(np.float64) * dx + (c[3] * dy).astype(np.float64)).astype(dtype)
            s2 = (dx.astype(np.float64) * inner + ((c[4] * dy) * dy).astype(np.float64)).astype(dtype)
        else:
            s2 = dx * (c[2] * dx + c[3] * dy) + (c[4] * dy) * dy
        ok = ((s2 >= 0) & (s2 <= c[5])).any(axis=1)
        out |= (ok.astype(np.uint8) << w)
    return out


def projection_like(n, rng, scale=(0.2, 60.0), aniso=(1.0, 40.0), spread=40.0):
    """Records as stage_record leaves them: 2-D covariances with the 0.3 px^2 dilation, opacity-aware radii."""
    s1 = np.exp(rng.uniform(np.log(scale[0]), np.log(scale[1]), n))
    s2 = s1 / np.exp(rng.uniform(0, np.log(aniso[1]), n))
    th = rng.uniform(0, np.pi, n)
    c, s = np.cos(th), np.sin(th)
    cxx = c * c * s1 ** 2 + s * s * s2 ** 2 + 0.3
    cyy = s * s * s1 ** 2 + c * c * s2 ** 2 + 0.3
    cxy = c * s * (s1 ** 2 - s2 ** 2)
    det = cxx * cyy - cxy ** 2
    a, bb, cc = cyy / det, -cxy / det, cxx / det
    o = rng.uniform(1 / 255 + 1e-4, 0.99, n)
    lg = np.log(o * 255)
    ext = np.minimum(3.33, np.sqrt(2 * lg))
    lam = 0.5 * (cxx + cyy) + np.sqrt(np.maximum(0.01, 0.25 * (cxx + cyy) ** 2 - det))
    rx = np.ceil(np.minimum(ext * np.sqrt(cxx), ext * np.sqrt(lam))).astype(np.int64)
    ry = np.ceil(np.minimum(ext * np.sqrt(cyy), ext * np.sqrt(lam))).astype(np.int64)
    mx = 8.0 + rng.uniform(-spread, spread, n)
    my = 8.0 + rng.uniform(-spread, spread, n)
    rec = dict(mx=F(mx), my=F(my), ha=F(a) * F(0.5) * LOG2E, b=F(bb) * LOG2E, hc=F(cc) * F(0.5) * LOG2E,
               smax2=(F(lg + 0.02) - F(0.02)) * LOG2E)
    return rec, np.minimum(rx, 65535), np.minimum(ry, 65535)


def _adversarial(rng):
    """Needles at every angle, nearly degenerate conics, centres far off the tile, frame-sized splats, zero / huge radii."""
    recs = []
    for spread, scale, aniso in (
        (20.0, (0.3, 3.0), (1.0, 2.0)),         # small round splats near the tile: block edges decide
        (200.0, (50.0, 2000.0), (100.0, 3000.0)),  # needles crossing the tile from far away
        (4000.0, (500.0, 5000.0), (1.0, 30.0)),    # frame-sized splats, centres off-screen
        (30.0, (0.01, 0.5), (1.0, 1.5)),        # splats at the dilation floor
    ):
        recs.append(projection_like(4000, rng, scale=scale, aniso=(1.0, aniso[1]), spread=spread))
    return recs


@pytest.mark.parametrize("tile", [(0, 0), (119, 67), (3, 40)])
def test_mask_keeps_every_block_with_a_passing_pixel(tile):
    rng = np.random.default_rng(7 + tile[0])
    tx0, ty0 = tile[0] * 16 + 0.5, tile[1] * 16 + 0.5
    for rec, rx, ry in [projection_like(20000, rng)] + _adversarial(rng):
        r = dict(rec)
        r["mx"] = F(r["mx"] + tx0 - 8.5)
        r["my"] = F(r["my"] + ty0 - 8.5)
        m = warp_mask(r["mx"], r["my"], r["ha"], r["b"], r["hc"], r["smax2"], rx, ry, tx0, ty0)
        for fma in (False, True):
            need = pixel_mask(r["mx"], r["my"], r["ha"], r["b"], r["hc"], r["smax2"], tx0, ty0, fma=fma)
            # the box bound stays as the projection wrote it: a pixel outside it is left out on purpose (alpha < 1/255
            # there by construction of the radius), so only bits inside the box are owed
            box = warp_mask(r["mx"], r["my"], F(0), F(0), F(0), F(0), rx, ry, tx0, ty0)
            missing = need & box & ~m
            assert not missing.any(), f"{np.count_nonzero(missing)} blocks with a passing pixel lost their bit"


def test_mask_degenerate_conics_fall_back_to_the_box():
    tx0, ty0 = 0.5, 0.5
    mx = np.full(4, 8.0, np.float32)
    ha = F([0.0, -1.0, 1.0, 1.0])
    hc = F([1.0, 1.0, 0.0, 1.0])
    b = F([0.0, 0.0, 0.0, 2.0])                 # last: 4 ha hc - b^2 = 0
    m = warp_mask(mx, mx, ha, b, hc, F([3.0] * 4), np.full(4, 2), np.full(4, 2), tx0, ty0)
    box = warp_mask(mx, mx, F(0), F(0), F(0), F(0), np.full(4, 2), np.full(4, 2), tx0, ty0)
    assert np.array_equal(m, box) and (box == 0x3C).all()     # rows 6..10: bands 1 and 2, both column halves


# Bits kept beyond the float64 exact set, as a fraction of all bits kept: the mask tests the continuous band between pixel
# rows and columns (a splat passing between two rows of centres keeps its bit) and carries rounding slack.  Measured 0.08 %
# on these draws.
EXCESS_BOUND = 0.01


def test_mask_excess_over_the_exact_set_is_small():
    rng = np.random.default_rng(11)
    rec, rx, ry = projection_like(40000, rng, scale=(0.3, 20.0), aniso=(1.0, 8.0), spread=30.0)
    tx0 = ty0 = 0.5
    r = dict(rec)
    m = warp_mask(r["mx"], r["my"], r["ha"], r["b"], r["hc"], r["smax2"], rx, ry, tx0, ty0)
    exact = pixel_mask(r["mx"], r["my"], r["ha"], r["b"], r["hc"], r["smax2"], tx0, ty0, dtype=np.float64)
    box = warp_mask(r["mx"], r["my"], F(0), F(0), F(0), F(0), rx, ry, tx0, ty0)
    kept = np.unpackbits(m).sum()
    extra = np.unpackbits(m & ~(exact & box)).sum()
    assert kept > 10000
    assert extra / kept <= EXCESS_BOUND, extra / kept
    # and the mask is much tighter than the box alone
    assert kept <= 0.8 * np.unpackbits(box).sum()

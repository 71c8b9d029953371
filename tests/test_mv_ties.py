"""CPU checks of the mask voting tie fixtures (tests/mv_ties.py): the float32 emulation is exact on
hand-worked cases, the fixtures put many deciding pixels where the rounding decides, the FMA-free
C oracle gives the FMA-free emulation bit for bit, and the device kernel's two shortcuts for unit
range images (the early exit of agg_exceeds_unit and the covering-weight cut of the search region)
agree with the full candidate-order sum on every deciding pixel."""
from fractions import Fraction

import numpy as np
import pytest

from tests import mv_ties as T

F32 = np.float32
IMAGES = range(len(T.IMAGES))


def _dot(h, w, value):
    """A box covering pixel (h, w) alone at mask coordinate (0, 0): render = value exactly."""
    mask = np.zeros((T.M, T.M), F32)
    mask[0, 0] = value
    return np.array([w, h, w + 0.5, h + 0.5], F32), mask


def test_render_and_aggregate_hand_cases():
    # a one-pixel box at fractions (0.5, 0.25) of mask cell (3, 2)
    box = np.array([10 - 2.5 / 21 * 1.5, 20 - 3.25 / 21 * 1.5, 10 + 0.5 - 2.5 / 21 * 1.5,
                    20 + 0.5 - 3.25 / 21 * 1.5], F32)
    rng = np.random.default_rng(1)
    mask = rng.uniform(0, 1, (T.M, T.M)).astype(F32)
    hh, ww = np.array([20]), np.array([10])
    x1, y1, x2, y2 = box
    px = (F32(10) - x1) * (F32(21) / ((x2 - x1) + F32(1)))
    py = (F32(20) - y1) * (F32(21) / ((y2 - y1) + F32(1)))
    cx, cy = int(np.floor(px)), int(np.floor(py))
    fx, fy = px - F32(cx), py - F32(cy)
    tl, tr = (F32(1) - fx) * (F32(1) - fy), fx * (F32(1) - fy)
    bl, br = (F32(1) - fx) * fy, fx * fy
    m0, m1, m2, m3 = mask[cy, cx], mask[cy, cx + 1], mask[cy + 1, cx], mask[cy + 1, cx + 1]
    fr = lambda v: Fraction(float(v))                                       # noqa: E731
    ref = T.round_f32(fr(br) * fr(m3) + fr(T.round_f32(fr(bl) * fr(m2) + fr(
        T.round_f32(fr(tl) * fr(m0) + fr(tr * m1))))))
    swapped = T.round_f32(fr(br) * fr(m3) + fr(T.round_f32(fr(bl) * fr(m2) + fr(
        T.round_f32(fr(tr) * fr(m1) + fr(tl * m0))))))
    assert T.render(box, mask, hh, ww, "ref")[0] == ref
    assert T.render(box, mask, hh, ww, "swapped")[0] == swapped
    assert T.render(box, mask, hh, ww, "nofma")[0] == ((tl * m0 + tr * m1) + bl * m2) + br * m3
    # outside the box, and the last mask column taken as is
    assert T.render(box, mask, np.array([20]), np.array([11]))[0] == 0
    wide = np.array([10 - 20.1, 20, 10 + 0.0, 20.5], F32)            # px = 20.1 * 21 / 21.1 in [20, 21)
    assert T.render(wide, mask, hh, ww)[0] == mask[0, 20]
    # aggregate: one rounding per term.  z + x*y = 1 + 2^-23 + 2^-24 - 2^-60 lies just below a
    # midpoint; a float64 product and sum land on it and round to even (up): double rounding
    x, y, z = F32(2 ** -12 * (1 + 2 ** -18)), F32(2 ** -12 * (1 - 2 ** -18)), F32(1 + 2 ** -23)
    cands = [(*_dot(5, 5, F32(1)), z), (*_dot(5, 5, x), y)]
    assert F32(float(x) * float(y) + float(z)) == F32(1 + 2 ** -22)
    assert T.aggregate(cands, np.array([5]), np.array([5]))[0] == F32(1 + 2 ** -23)
    # without the fma, x*y rounds to 2^-24 first and the sum is a tie, rounded to even (up)
    assert T.aggregate(cands, np.array([5]), np.array([5]), "nofma")[0] == F32(1 + 2 ** -22)
    # the tiny-tail trap: prev(0.4f) then two terms of 0.51 ulp -> 0.4f -> next(0.4f), on
    prev = np.nextafter(T.THRESH, F32(0))
    t = F32(0.51) * T.ULP
    cands = [(*_dot(5, 5, F32(1)), prev), (*_dot(5, 5, F32(1)), t), (*_dot(5, 5, F32(1)), t)]
    assert T.aggregate(cands, np.array([5]), np.array([5]))[0] == np.nextafter(T.THRESH, F32(1))
    assert not T.early_exit([F32(1)] * 3, [prev, t, t], old=True)
    assert T.early_exit([F32(1)] * 3, [prev, t, t])


def test_resample_hand_case():
    """mask_resize of the aggregate: positions fma(j, ratio, x1), the 4-tap blend, last row / column."""
    H, W = 40, 30
    cands = [(np.array([0, 0, W - 1, H - 1], F32), np.linspace(0, 1, T.M * T.M, dtype=F32).reshape(T.M, T.M),
              F32(0.9))]
    box = (3, 5, W - 1, H - 1)
    out = T.resample(cands, box, H, W)
    j = 20
    ix = T.fma_f32(F32(j), F32(W - 1 - 3 + 1) / F32(21), F32(3))
    iy = T.fma_f32(F32(j), F32(H - 1 - 5 + 1) / F32(21), F32(5))
    sx, sy = int(np.floor(ix)), int(np.floor(iy))
    if sx == W - 1 or sy == H - 1:
        assert out[j, j] == T.aggregate(cands, np.array([sy]), np.array([sx]))[0]
    assert out.dtype == F32 and out.shape == (T.M, T.M)
    a = T.aggregate(cands, np.array([5, 5, 6, 6]), np.array([3, 4, 3, 4]))
    fx, fy = T.fma_f32(F32(0), F32(27) / F32(21), F32(3)) - F32(3), F32(0)
    tl, tr, bl, br = T._weights(fx, fy)
    assert out[0, 0] == T.blend(tl, tr, bl, br, a[0], a[1], a[2], a[3], "ref")


@pytest.mark.parametrize("img", IMAGES)
def test_cases_are_decided_by_one_pixel(img):
    """Each case's deciding pixel is within 30 ulps of 0.4f under `ref`, its decision moves the box,
    and the box is the emulation's with that pixel's own decision."""
    H, W, unit, cases = T.image_cases(img)
    for c in cases:
        assert abs(c["offset"]) <= 30
        on = bool(c["agg"]["ref"] > T.THRESH)
        assert c["boxes_if"][True] != c["boxes_if"][False]
        assert T.emulate(c["cands"], H, W)[0] == c["boxes_if"][on] == c["expect"]["ref"][0]


def test_fixtures_have_teeth():
    cases = [(H, W, c) for i in IMAGES for H, W, _, cs in [T.image_cases(i)] for c in cs]
    dec = lambda c, r: bool(c["agg"][r] > T.THRESH)                       # noqa: E731
    assert sum(dec(c, "ref") != dec(c, "nofma") for _, _, c in cases) >= 50
    assert sum(dec(c, "ref") != dec(c, "swapped") for _, _, c in cases) >= 50
    assert sum(c["offset"] == 0 for _, _, c in cases) >= 20
    plans = [c["plan"] for _, _, c in cases]
    for p in ("interp", "int_edge", "nearest_x", "nearest_y", "nearest_xy", "border", "single",
              "empty", "long", "trap"):
        assert p in plans, p
    assert any(c["expect"]["ref"][0][0] == W // 2 and c["kind"] == "empty" for H, W, c in cases)
    n = [len(c["cands"]) for _, _, c in cases]
    assert {1, 2} <= set(n) and max(n) > 250 and any(3 <= k <= 8 for k in n)
    grid = [T.on_coarse_grid(c, H, W) for H, W, c in cases]
    assert sum(grid) >= 20 and len(grid) - sum(grid) >= 20
    assert {c["side"] for _, _, c in cases} == set(T.SIDES)
    assert any(c["tie"][1] in (0, W - 1) or c["tie"][0] in (0, H - 1) for H, W, c in cases)
    assert not T.IMAGES[2][2] and not T.IMAGES[3][2]        # two images take the full-sum path


@pytest.mark.parametrize("img", IMAGES)
def test_oracle_is_nofma_bit_for_bit(img):
    from oracle import oracle as O
    H, W, _, cases = T.image_cases(img)
    boxes, masks, inds, start, wts = T.pack(cases)
    rm, rb = O.mv(boxes, masks, inds, start, wts, H, W)
    eb, em = T.expected(cases, "nofma")
    assert np.array_equal(rb, eb)
    assert np.array_equal(rm.view(np.int32), em.view(np.int32))


@pytest.mark.parametrize("img", [i for i in IMAGES if T.IMAGES[i][2]])
def test_shortcuts_agree_with_the_full_sum(img):
    """The early exit and the search-region cut, restated, on every deciding pixel of the unit range
    images; with the constants before the fix the early exit fails on every trap case."""
    H, W, _, cases = T.image_cases(img)
    traps = 0
    for c in cases:
        (h, w), cands = c["tie"], c["cands"]
        renders = [T.render(b, m, np.array([h]), np.array([w]))[0] for b, m, _ in cands]
        wts = [wt for _, _, wt in cands]
        full = bool(c["agg"]["ref"] > T.THRESH)
        assert T.early_exit(renders, wts) == full
        if full:
            assert T.covering_cut([b for b, _, _ in cands], wts, h, w)
        if c["plan"] == "trap":
            assert full and not T.early_exit(renders, wts, old=True)
            traps += 1
    assert traps >= 4

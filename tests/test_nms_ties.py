"""CPU checks of the NMS tie fixtures (tests/nms_ties.py): the float32 emulation of devIoU is exact,
the fixtures put many pairs where the rounding of the union decides, the FMA-free C oracle gives
the FMA-free emulation's keep lists, and the block walk of the capped kernels gives greedy NMS
under the reference's rounding."""
from fractions import Fraction

import numpy as np
import pytest

from tests import nms_ties as T
from tests.test_capped_nms_model import capped_nms_blocks

F32 = np.float32
ALL_THRESHOLDS = T.THRESHOLDS + (0.0, -0.5)


def test_round_f32_and_fma_hand_cases():
    one = Fraction(1)
    assert T.round_f32(one + Fraction(1, 2 ** 24)) == F32(1)                     # tie -> even (down)
    assert T.round_f32(one + Fraction(3, 2 ** 24)) == F32(1 + 2 ** -22)          # tie -> even (up)
    assert T.round_f32(one + Fraction(3, 2 ** 24) - Fraction(1, 2 ** 80)) == F32(1 + 2 ** -23)
    assert T.round_f32(-Fraction(7, 10)) == F32(-0.7)
    rng = np.random.default_rng(0)
    for v in rng.uniform(-1e6, 1e6, 200):                   # float64 -> float32 is one rounding
        assert T.round_f32(Fraction(float(v))) == F32(v)
    # x*y + z = 1 + 2^-23 + 2^-24 - 2^-60: just below the midpoint between 1 + 2^-23 and 1 + 2^-22.
    # Through float64 the sum lands ON the midpoint and then rounds to even (up): double rounding.
    x, y, z = F32(2 ** -12 * (1 + 2 ** -18)), F32(2 ** -12 * (1 - 2 ** -18)), F32(1 + 2 ** -23)
    assert F32(float(x) * float(y) + float(z)) == F32(1 + 2 ** -22)
    assert T.fma_f32_exact(x, y, z) == F32(1 + 2 ** -23)
    assert T.fma_f32(x, y, z) == F32(1 + 2 ** -23)
    assert T.fma_f32(-x, y, -z) == F32(-(1 + 2 ** -23))
    assert T.fma_f32(F32(3), F32(5), F32(0.25)) == F32(15.25)


def test_emulated_iou_hand_cases():
    t = 0.7
    # fractional: U differs by an ulp between the roundings, and the decision with it
    a = np.array([20.255356, 219.60185, 216.13614, 257.2605], dtype=F32)
    b = a.copy()
    b[2] = F32(157.07191)
    assert T.quotient(a, b, "ref") == F32(0.7) and not T.suppresses(a, b, t, "ref")
    assert T.quotient(a, b, "swapped") == np.nextafter(F32(0.7), F32(1)) and T.suppresses(a, b, t, "swapped")
    inter, aw, ah, bw, bh = T._terms(a, b)
    sa = aw * ah
    exact_u = T.fma_f32_exact(bw, bh, sa) - inter
    assert T.union(a, b, "ref")[1] == exact_u
    assert T.union(a, b, "swapped")[1] == T.fma_f32_exact(aw, ah, bw * bh) - inter
    # integers: IoU exactly 7/10 is float32(0.7) and does not suppress; one pixel more does
    a = np.array([0, 0, 99, 9], dtype=F32)
    for r in T.ROUNDINGS:
        assert T.quotient(a, np.array([0, 0, 69, 9], dtype=F32), r) == F32(0.7)
        assert not T.suppresses(a, np.array([0, 0, 69, 9], dtype=F32), t, r)
        assert T.suppresses(a, np.array([0, 0, 70, 9], dtype=F32), t, r)
    # touching (+1 width exactly 0), identical, zero width next to a box, two zero-width boxes
    touch = np.array([100, 0, 150, 9], dtype=F32)
    assert T._terms(a, touch)[0] == 0 and not T.suppresses(a, touch, 0.0)
    assert T.suppresses(a, touch, -0.5)
    assert T.suppresses(a, a, 0.7)
    thin = np.array([5, 0, 4, 9], dtype=F32)
    assert T.quotient(a, thin) == 0 and T.suppresses(a, thin, -0.5) and not T.suppresses(a, thin, 0.0)
    assert np.isnan(T.quotient(thin, thin + F32(3))) and not T.suppresses(thin, thin + F32(3), -0.5)


@pytest.mark.parametrize("thresh", T.THRESHOLDS)
def test_vectorized_fma_is_exact_on_the_fixtures(thresh):
    a, b, _ = T.pair_pool(thresh)
    inter, aw, ah, bw, bh = T._terms(a, b)
    for x, y, z in ((bw, bh, aw * ah), (aw, ah, bw * bh)):
        got = T.fma_f32(x, y, z)
        want = np.array([T.fma_f32_exact(*v) for v in zip(x, y, z)], dtype=F32)
        assert np.array_equal(got.view(np.int32), want.view(np.int32))


@pytest.mark.parametrize("thresh", T.THRESHOLDS)
def test_fixtures_have_teeth(thresh):
    a, b, kind = T.pair_pool(thresh)
    ref = T.suppresses(a, b, thresh, "ref")
    assert (ref != T.suppresses(a, b, thresh, "swapped")).sum() >= 50
    assert (ref != T.suppresses(a, b, thresh, "nofma")).sum() >= 50
    band = T.in_fast_band(a, b, thresh)
    assert band.sum() >= 50 and (~band & (kind != "edge")).sum() >= 50   # the fast path decides some
    off = T.ulps_from(T.quotient(a, b), thresh)
    near = (kind == "fractional") | (kind == "integer")
    assert (off[kind == "ratio"] == 0).sum() >= 3
    for k in (0, 1, -1, 17, -17, 30, -30):
        assert (off[near] == k).sum() >= 3, k
    assert np.abs(off[near]).max() <= 30
    for k in ("fractional", "integer", "ratio"):
        assert (kind == k).sum() >= 3, k
    # integer pairs have exact areas: the roundings agree, only the comparison with t is tested
    i = kind != "fractional"
    assert np.array_equal(ref[i], T.suppresses(a[i], b[i], thresh, "swapped"))
    e = np.flatnonzero(kind == "edge").reshape(-1, len(T.EDGE_KINDS))
    inter = T._terms(a, b)[0]
    for col, name in enumerate(T.EDGE_KINDS):
        if name in ("touch_x", "touch_y", "zero_width_inside", "zero_width_both"):
            assert (inter[e[:, col]] == 0).all(), name
        else:
            assert (inter[e[:, col]] > 0).all(), name


@pytest.mark.parametrize("thresh", ALL_THRESHOLDS)
@pytest.mark.parametrize("name", ["small", "big"])
def test_oracle_equals_fma_free_emulation(thresh, name):
    from oracle import oracle as O
    boxes, _, counts, max_keep = T.tie_lists(thresh, name)
    want = T.expected_keep(thresh, name, "nofma")
    for p, c in enumerate(counts):
        got = O.nms_sorted(boxes[p, :c], thresh)
        assert np.array_equal(got[:max_keep] if max_keep else got, want[p]), p


@pytest.mark.parametrize("thresh", ALL_THRESHOLDS)
@pytest.mark.parametrize("block", [64, 256])
def test_block_walk_equals_greedy_on_ties(thresh, block):
    boxes, _, counts, _ = T.tie_lists(thresh, "small")
    for p, c in enumerate(counts):
        b = boxes[p, :c]
        sup = np.stack([T.suppresses(b[i][None], b, thresh, "ref") for i in range(c)])
        for max_keep in (0, c // 4):
            want = T.greedy_keep(b, thresh, "ref", max_keep)
            got = capped_nms_blocks(c, lambda i, j: sup[i, j], max_keep, block)
            assert got == [int(i) for i in want], (p, max_keep)


@pytest.mark.parametrize("thresh", T.THRESHOLDS)
def test_keep_lists_show_every_decision(thresh):
    """Across pairs nothing suppresses: the keep lists of two roundings differ exactly at the later
    boxes of the pairs whose decisions differ."""
    boxes, entries, counts, _ = T.tie_lists(thresh, "small")
    for other in ("swapped", "nofma"):
        want = T.expected_keep(thresh, "small")
        got = T.expected_keep(thresh, "small", other)
        for p in range(len(counts)):
            _, ib, _ = T.observable_pairs(thresh, "small", p, other)
            assert np.array_equal(np.setxor1d(want[p], got[p]), np.sort(ib)), (other, p)


@pytest.mark.parametrize("thresh", T.THRESHOLDS)
def test_ties_reach_every_part_of_each_kernel(thresh):
    """In the capped launch, pairs at a tie (and pairs the swapped rounding decides wrongly) sit with
    a and b in one 64-box block (diagonal words) and in different ones (kept list, off-diagonal
    words), in one 256-box round and in different ones (mode 3), and spread over the 8 CTAs of the
    cluster forms, which split the kept list (mode 2: index / 4 mod 8, mode 3: index mod 8) and the
    diagonal rows (mode 2: 8 of 64 per CTA, mode 3: 32 of 256)."""
    def parts(differ_from):
        ia, ib, ka = (np.concatenate(v) for v in
                      zip(*(T.observable_pairs(thresh, "big", p, differ_from) for p in range(3))))
        return ia, ka, ia // 64 == ib // 64, ia // 256 == ib // 256

    _, _, same64, same256 = parts("swapped")
    for where in (same64, ~same64, same256 & ~same64, ~same256):
        assert where.sum() >= 3
    ia, ka, same64, same256 = parts(None)
    assert set((ka[~same64] // 4) % 8) == set(range(8))
    assert set(ka[~same256] % 8) == set(range(8))
    assert set((ia[same64] % 64) // 8) == set(range(8))
    assert set((ia[same256] % 256) // 32) == set(range(8))
    _, _, _, max_keep = T.tie_lists(thresh, "big")
    nums = [len(k) for k in T.expected_keep(thresh, "big")]
    assert nums[0] == max_keep and nums[2] < max_keep            # max_keep below and above the survivors

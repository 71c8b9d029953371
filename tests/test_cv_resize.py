"""The float32 model of the device's cv2.resize(INTER_LINEAR) rule (tests/cv_resize.py): exact on
hand-worked cases, within an analytic bound of a float64 bilinear sample, its tie fixtures on
0.4f with teeth against every mutant of the rule, and its distance from the live cv2.resize."""
import numpy as np
import pytest

from tests import cv_resize as C

F32 = np.float32


def test_taps_hand_worked():
    # identity: every fraction 0, the last index clamped onto itself
    i0, i1, a0, a1 = C.taps(21, 21, 1.0)
    assert np.array_equal(i0, np.arange(21)) and np.all(a1 == 0) and np.all(a0 == 1)
    assert i1[-1] == 20 and np.array_equal(i1[:-1], np.arange(1, 21))
    # exact 2x and 4x downscales: taps (2d, 2d + 1) and (4d + 1, 4d + 2), both halves
    i0, i1, a0, a1 = C.taps(21, 42, 2.0)
    assert np.array_equal(i0, 2 * np.arange(21)) and np.array_equal(i1, i0 + 1)
    assert np.all(a0 == F32(0.5)) and np.all(a1 == F32(0.5))
    i0, i1, a0, a1 = C.taps(21, 84, 4.0)
    assert np.array_equal(i0, 4 * np.arange(21) + 1) and np.all(a1 == F32(0.5))
    # 1 destination sample from 21: fd = 10 exactly
    assert [int(v[0]) for v in C.taps(1, 21, 21.0)[:2]] == [10, 11]
    # 2 -> 3: fd = -1/6 (clamped to 0), 1/2, 7/6 (s = 1 >= n - 1: both taps 1)
    i0, i1, a0, a1 = C.taps(3, 2, 2 / 3)
    assert list(i0) == [0, 0, 1] and list(i1) == [1, 1, 1]
    assert list(a1) == [0, F32(0.5), 0] and list(a0) == [1, F32(0.5), 1]
    # the fraction is taken from the coordinate in double: 21 -> 37 at d = 36 is
    # fd = 36.5 * 21 / 37 - 0.5 = 20.216..., clamped (s = 20 = n - 1)
    i0, i1, _, a1 = C.taps(37, 21, 21 / 37)
    assert i0[-1] == i1[-1] == 20 and a1[-1] == 0
    assert a1[1] == F32(1.5 * 21 / 37 - 0.5)


def test_resize_hand_worked():
    src = np.array([[0, 1], [2, 3]], F32)
    want = np.array([[0, 0.5, 1], [1, 1.5, 2], [2, 2.5, 3]], F32)
    assert np.array_equal(C.resize(src, 3, 3), want)
    # the rounding order: fl(fl(fl(a a0) + fl(b a1)) b0 + ...) with a1 = fl(f) -- one sample
    # recomputed step by step in float32 scalars
    rng = np.random.default_rng(0)
    src = rng.uniform(0, 1, (21, 21)).astype(F32)
    out = C.resize(src, 37, 29)
    x0, x1, ax0, ax1 = C.taps(37, 21, 21 / 37)
    y0, y1, ay0, ay1 = C.taps(29, 21, 21 / 29)
    for dy, dx in ((3, 5), (17, 30), (28, 36), (0, 0)):
        r0 = F32(F32(src[y0[dy], x0[dx]] * ax0[dx]) + F32(src[y0[dy], x1[dx]] * ax1[dx]))
        r1 = F32(F32(src[y1[dy], x0[dx]] * ax0[dx]) + F32(src[y1[dy], x1[dx]] * ax1[dx]))
        assert out[dy, dx] == F32(F32(r0 * ay0[dy]) + F32(r1 * ay1[dy]))
    # binarisation is >= 0.4f; `gt` is the > mutant
    v = np.array([C.at_ulps(-1), C.THRESH, C.at_ulps(1)])
    assert list(C.binarize(v)) == [False, True, True]
    assert list(C.binarize(v, "gt")) == [False, False, True]


@pytest.mark.parametrize("shape,dst", [((21, 21), (37, 55)), ((21, 21), (300, 200)),
                                       ((42, 42), (21, 21)), ((84, 84), (21, 21)),
                                       ((21, 21), (1, 1)), ((21, 21), (1, 30)),
                                       ((375, 500), (241, 320)), ((60, 80), (96, 128))])
def test_model_within_bound_of_float64(shape, dst):
    """Weights: f rounded to float32 (error <= 2^-25) and 1 - f (one more rounding, <= 2^-25);
    each pass adds 3 roundings of relative 2^-24 on values bounded by A = max|src|, and the
    horizontal pass's error is carried by the vertical weights (sum 1).  In all
    |model - float64| <= A (2 (2^-24 + 3 2^-24)) = A 2^-21."""
    rng = np.random.default_rng(sum(shape) + sum(dst))
    for src in (rng.uniform(0, 1, shape).astype(F32), rng.normal(0, 50, shape).astype(F32)):
        A = float(np.abs(src).max())
        err = np.abs(C.resize(src, dst[1], dst[0]).astype(np.float64) - C.ref64(src, dst[1], dst[0]))
        assert err.max() <= A * 2.0 ** -21


def _placed_values(src, dw, dh, placed):
    v = C.resize(src, dw, dh, src.shape[1] / dw, src.shape[0] / dh)
    return [(int(C.ulps_from(v[dy, dx])), off) for dy, dx, off in placed]


def test_place_ties_hits_its_targets():
    rng = np.random.default_rng(3)
    for (h, w), (dh, dw) in (((21, 21), (37, 55)), ((21, 21), (21, 21)), ((42, 42), (21, 21)),
                             ((21, 21), (1, 30)), ((21, 21), (13, 9))):
        src = rng.uniform(0, 1, (h, w)).astype(F32)
        placed = C.place_ties(rng, src, np.ones((h, w), bool), dw, dh, w / dw, h / dh, max_ties=40)
        assert len(placed) >= min(8, dh * dw // 4), ((h, w), (dh, dw), len(placed))
        got = _placed_values(src, dw, dh, placed)
        assert all(u == off for u, off in got), got
        assert sum(off == 0 for _, off in got) >= len(got) // 3


def _paste_bits(mode):
    fx, H, W = C.paste_fixture(1)
    return np.concatenate([np.stack(C.paste(b, m, c, H, W, mode)[:2]).ravel() for _, b, m, c in fx])


def _binarize_bits(mode):
    return np.concatenate([C.binarize_masks(rb, m, mode)[0] for _, rb, m in C.binarize_fixture(2)])


def _mask_target_bits(mode):
    info, nfg, gm = C.mask_target_fixture(3)
    return C.mask_targets(info, nfg, gm, mode=mode)[0].ravel()


def _mask_layer_bits(mode):
    """The binarised ex-box-sized predictions MaskLayer counts."""
    _, groups = C.mask_layer_fixture(4)
    bits = []
    for M, preds, info in groups:
        for p, mi in zip(preds, info):
            if mi[0] == -1:
                continue
            ex1, ey1, ex2, ey2 = (int(v) for v in mi[4:8])
            ew, eh = ex2 - ex1 + 1, ey2 - ey1 + 1
            v = C.resize(p.reshape(M, M), ew, eh, M / ew, M / eh, mode)
            bits.append(C.binarize(v, mode).ravel())
    return np.concatenate(bits)


FIXTURE_SETS = {"paste": _paste_bits, "binarize": _binarize_bits,
                "mask_target": _mask_target_bits, "mask_layer": _mask_layer_bits}


@pytest.mark.parametrize("name", sorted(FIXTURE_SETS))
def test_every_mutant_flips_bits_in_every_fixture_set(name):
    bits = FIXTURE_SETS[name]
    exact = bits("exact")
    for mode in C.MUTANTS:
        flips = int(np.sum(bits(mode) != exact))
        assert flips >= 3, (name, mode, flips)


def test_mask_layer_labels_sit_on_their_edge():
    """With fg_seg_thresh at a row's IoU the label is kept, one double above it the label is
    dropped: so a single binarised bit more or less in that row flips the label."""
    gm, groups = C.mask_layer_fixture(4)
    for M, preds, info in groups:
        for t in C.iou_thresholds(preds, gm, info)[::2]:
            lab = C.mask_layer(preds, gm, info, t)
            lab_up = C.mask_layer(preds, gm, info, float(np.nextafter(t, np.inf)))
            assert np.sum(lab != lab_up) >= 1


def test_prep_mutants_change_the_blob():
    rng = np.random.default_rng(9)
    im = rng.integers(0, 256, (1, 47, 61, 3), dtype=np.uint8)
    means = (102.9801, 115.9465, 122.7717)
    exact = C.prep(im, 1.7, means)
    assert exact.shape == (1, 3, 80, 104)
    for mode in ("vfma", "hfma", "fcoord", "vfirst"):
        assert np.sum(C.prep(im, 1.7, means, mode) != exact) >= 3, mode


@pytest.mark.parametrize("shape,dst", [((21, 21), (37, 55)), ((21, 21), (300, 200)),
                                       ((42, 42), (21, 21)), ((84, 84), (21, 21)),
                                       ((21, 21), (1, 1)), ((21, 21), (1, 30)),
                                       ((375, 500), (241, 320)), ((375, 500), (600, 800))])
def test_model_against_live_cv2(shape, dst):
    """cv2 is not the exact pin (its bits depend on IPP and the CPU): its distance from the model
    stays within the measured CV2_ULPS, sample by sample."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(sum(shape) * 7 + sum(dst))
    src = rng.uniform(0, 1, shape).astype(F32)
    got = cv2.resize(src, (dst[1], dst[0]))
    d = np.abs(C.ulps_from(got, C.resize(src, dst[1], dst[0])))
    assert d.max() <= C.CV2_ULPS, d.max()

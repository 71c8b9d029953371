"""The numpy restatement of the loss layers (oracle/oracle_loss.py) on hand-computed cases, one per
quirk the device keeps (DESIGN.md "Loss layers"), and its backward against the float64 gradient of
its forward."""
import numpy as np
import pytest

from oracle import oracle_loss as L

F32 = np.float32


# ------------------------------------------------------------------------------ fixed-order sum
def test_fixed_sum_is_the_float64_sum_rounded_once():
    t = np.array([1.0, 2.0 ** -30, -1.0, 3.0], np.float32)
    assert L.fixed_sum(t) == F32(3.0 + 2.0 ** -30)
    big = np.full(5000, 0.1, np.float32)
    assert L.fixed_sum(big) == F32(5000 * float(F32(0.1)))
    assert L.fixed_sum(np.zeros(0, np.float32)) == 0


def test_fixed_sum_order_partials_then_tree():
    """Terms 1024 apart meet first: 2^24 + 1 + 1 in one partial is exact in float64."""
    t = np.zeros(3 * 1024, np.float32)
    t[5], t[5 + 1024], t[5 + 2048] = 2.0 ** 24, 1.0, 1.0
    assert L.fixed_sum(t) == F32(2.0 ** 24 + 2)


# ----------------------------------------------------------------------------- SoftmaxWithLoss
def test_softmax_two_classes_by_hand():
    x = np.array([[0.0, 0.0], [0.0, np.log(3.0)]], np.float32)
    loss, prob = L.softmax_loss(x, np.array([0, 1], np.float32))
    assert np.allclose(prob[:, :, 0], [[0.5, 0.5], [0.25, 0.75]], rtol=0, atol=1e-7)
    want = (np.log(2.0) - np.log(0.75)) / 2
    assert abs(float(loss) - want) < 1e-7


def test_softmax_channel_axis_with_inner():
    """(1, 2, 3) scores: each of the 3 inner positions is its own 2-way softmax."""
    x = np.array([[[0.0, 1.0, 2.0], [0.0, 0.0, 0.0]]], np.float32)
    _, prob = L.softmax_loss(x, np.zeros(3, np.float32))
    e = np.exp([0.0, 1.0, 2.0])
    assert np.allclose(prob[0, 0], e / (e + 1), atol=1e-7)
    assert np.allclose(prob[0].sum(0), 1, atol=1e-7)


@pytest.mark.parametrize("mode,norm", [("FULL", 6), ("VALID", 4), ("BATCH_SIZE", 2), ("NONE", 1)])
def test_softmax_normalization_modes(mode, norm):
    """2 rows x 3 positions, 2 of the 6 labels ignored; uniform scores give log 2 per term."""
    x = np.zeros((2, 2, 3), np.float32)
    lab = np.array([[0, -1, 1], [1, 0, -1]], np.float32)
    loss, prob = L.softmax_loss(x, lab, ignore_label=-1, normalization=mode)
    assert loss == F32(L.fixed_sum(np.full(4, -np.log(F32(0.5)), np.float32)) / F32(norm))
    d = L.softmax_loss_backward(prob, lab, 2.0, ignore_label=-1, normalization=mode)
    assert d[0, :, 1].tolist() == [0, 0] and d[1, :, 2].tolist() == [0, 0]
    assert d[0, 0, 0] == F32(-0.5) * (F32(2) / F32(norm))


def test_softmax_valid_without_ignore_label_counts_every_position():
    x = np.zeros((2, 2, 3), np.float32)
    lab = np.array([[0, -1, 1], [1, 0, -1]], np.float32)
    loss, _ = L.softmax_loss(x, lab, ignore_label=None, normalization="VALID")
    # -1 labels are then out of range: counted, no term
    assert loss == F32(L.fixed_sum(np.full(4, -np.log(F32(0.5)), np.float32)) / F32(6))


def test_softmax_all_ignored_gives_zero_loss_and_zero_diff():
    x = np.random.default_rng(0).standard_normal((4, 21)).astype(np.float32)
    lab = np.full(4, -1, np.float32)
    loss, prob = L.softmax_loss(x, lab, ignore_label=-1)
    assert loss == 0
    d = L.softmax_loss_backward(prob, lab, 1.0, ignore_label=-1)
    assert not d.any()


def test_softmax_loss_floor_at_flt_min():
    x = np.array([[0.0, -200.0]], np.float32)     # p[1] underflows to 0
    loss, _ = L.softmax_loss(x, np.array([1], np.float32))
    assert loss == -L.logf(L.FLT_MIN)


def test_softmax_labels_truncate_toward_zero():
    x = np.array([[0.0, 1.0, 2.0]], np.float32)
    a, _ = L.softmax_loss(x, np.array([1.9], np.float32))
    b, _ = L.softmax_loss(x, np.array([1.0], np.float32))
    assert a == b


def test_softmax_n_valid_equals_trimmed():
    r = np.random.default_rng(1)
    x = r.standard_normal((10, 21)).astype(np.float32)
    lab = r.integers(-1, 21, 10).astype(np.float32)
    a, pa = L.softmax_loss(x, lab, -1, n_valid=6)
    b, pb = L.softmax_loss(x[:6], lab[:6], -1)
    assert a == b and np.array_equal(pa, pb)


# ------------------------------------------------------------------------------- SmoothL1Loss
def test_smooth_l1_branches_by_hand():
    pred = np.array([[0.5, -2.0, 0.0, 1.0]], np.float32)
    loss = L.smooth_l1_loss(pred, np.zeros_like(pred), sigma=1.0)
    assert loss == F32(0.125 + 1.5 + 0.0 + 0.5)          # |x| = 1 is the linear branch
    g = L.smooth_l1_loss_backward(pred, np.zeros_like(pred), sigma=1.0)
    assert g.tolist() == [[0.5, -1.0, 0.0, 1.0]]


def test_smooth_l1_threshold_is_compared_in_double():
    """sigma 0.7: float32(1 / sigma2) lies below 1 / sigma2, so at val = float32(1 / sigma2) the
    double test takes the quadratic branch (a float test would take the linear one): gradient
    sigma2 * val = 0.99999994, not 1."""
    s2 = F32(0.7) * F32(0.7)
    v = F32(1) / s2
    assert float(v) < 1.0 / float(s2)
    pred = np.array([[v, -v]], np.float32)
    g = L.smooth_l1_loss_backward(pred, np.zeros_like(pred), sigma=0.7)
    assert g.tolist() == [[s2 * v, -(s2 * v)]] and g[0, 0] == F32(0.99999994)
    loss = L.smooth_l1_loss(pred, np.zeros_like(pred), sigma=0.7)
    e = F32(0.5 * float(v) * float(v) * float(s2))
    assert loss == F32(2 * float(e))
    # sigma 3: float32(1/9) lies above 1/9 -> linear, value |x| - 0.5/9 in double
    w = F32(1) / F32(9)
    assert float(w) > 1.0 / 9
    g3 = L.smooth_l1_loss_backward(np.array([[w]], np.float32), np.zeros((1, 1), np.float32), sigma=3.0)
    assert g3[0, 0] == 1
    l3 = L.smooth_l1_loss(np.array([[w]], np.float32), np.zeros((1, 1), np.float32), sigma=3.0)
    assert l3 == F32(float(w) - 0.5 / 9.0)


def test_smooth_l1_weights_and_rows_normaliser():
    pred = np.array([[2.0, 2.0], [0.0, 4.0]], np.float32)
    tgt = np.zeros_like(pred)
    wi = np.array([[1.0, 0.0], [1.0, 0.5]], np.float32)
    wo = np.array([[3.0, 3.0], [1.0, 1.0]], np.float32)
    # d = [[2, 0], [0, 2]] -> 1.5, 0, 0, 1.5 -> * wo -> 4.5 + 1.5 = 6, over 2 rows
    assert L.smooth_l1_loss(pred, tgt, wi, wo, sigma=1.0) == F32(3.0)
    g = L.smooth_l1_loss_backward(pred, tgt, wi, wo, sigma=1.0, top_diff=2.0)
    assert g.tolist() == [[3.0, 0.0], [0.0, 0.5]]
    assert L.smooth_l1_loss(pred, tgt, wi, wo, sigma=1.0, n_valid=1) == F32(4.5)


# ---------------------------------------------------------------------- SigmoidCrossEntropyLoss
def test_sigmoid_is_the_double_quotient_of_a_float_exp():
    x = np.linspace(-20, 20, 4001).astype(np.float32)
    e = np.exp(-x.astype(np.float64)).astype(np.float32)
    assert np.array_equal(L.sigmoid(x), (1.0 / (1.0 + e.astype(np.float64))).astype(np.float32))


def test_sigmoid_ce_by_hand():
    x = np.array([[0.0, 2.0, -3.0]], np.float32)
    t = np.array([[1.0, 0.0, 0.0]], np.float32)
    want = np.log(2.0) + (2.0 + np.log1p(np.exp(-2.0))) + np.log1p(np.exp(-3.0))
    assert abs(float(L.sigmoid_ce_loss(x, t)) - want) < 2e-7 * want    # / num = 1
    w = np.array([[1.0, 0.0, 1.0]], np.float32)
    want_w = (np.log(2.0) + np.log1p(np.exp(-3.0))) / 2
    assert abs(float(L.sigmoid_ce_loss(x, t, w)) - want_w) < 2e-7
    d = L.sigmoid_ce_loss_backward(x, t, w, top_diff=2.0)
    assert d[0, 1] == 0 and d[0, 0] == F32(-0.5) * F32(1.0)


def test_sigmoid_ce_zero_weight_sum_leaves_the_top_and_the_diff_unscaled():
    x = np.array([[0.5, -1.0]], np.float32)
    t = np.array([[1.0, 0.0]], np.float32)
    w = np.zeros_like(x)
    assert L.sigmoid_ce_loss(x, t, w, untouched=F32(7.25)) == F32(7.25)
    d = L.sigmoid_ce_loss_backward(x, t, w, top_diff=2.0)
    assert not d.any()


# ------------------------------------------------------------------------------------ Accuracy
def test_accuracy_ties_rank_the_higher_class_first():
    x = np.zeros((3, 4), np.float32)
    assert L.accuracy(x, np.array([3, 3, 3], np.float32)) == 1
    assert L.accuracy(x, np.array([0, 2, 3], np.float32)) == F32(1) / F32(3)
    assert L.accuracy(x, np.array([2, 2, 1], np.float32), top_k=2) == F32(2) / F32(3)


def test_accuracy_minus_one_without_ignore_is_a_miss_and_ignore_skips():
    x = np.array([[0.0, 1.0], [1.0, 0.0]], np.float32)
    lab = np.array([1, -1], np.float32)
    assert L.accuracy(x, lab) == F32(0.5)
    assert L.accuracy(x, lab, ignore_label=-1) == 1
    assert np.isnan(L.accuracy(x, np.full(2, -1, np.float32), ignore_label=-1))


# ---------------------------------------------------------- backward == float64 gradient of forward
def _num_grad(f, x, h=1e-6):
    g = np.zeros(x.shape)
    for i in np.ndindex(x.shape):
        a, b = x.copy(), x.copy()
        a[i] += h
        b[i] -= h
        g[i] = (f(a) - f(b)) / (2 * h)
    return g


def test_softmax_backward_is_the_gradient():
    r = np.random.default_rng(2)
    x = r.standard_normal((5, 3, 4)).astype(np.float32)
    lab = r.integers(-1, 3, (5, 4)).astype(np.float32)
    li = lab.astype(int)

    def f64(z):
        p = np.exp(z - z.max(1, keepdims=True))
        p /= p.sum(1, keepdims=True)
        n, j = np.nonzero(li >= 0)
        return -np.log(p[n, li[n, j], j]).sum() / max(1, (li >= 0).sum())

    _, prob = L.softmax_loss(x, lab, ignore_label=-1)
    d = L.softmax_loss_backward(prob, lab, 1.5, ignore_label=-1)
    assert np.allclose(d, 1.5 * _num_grad(f64, x.astype(np.float64)), rtol=1e-4, atol=1e-6)


def test_smooth_l1_backward_is_the_gradient_away_from_the_kink():
    r = np.random.default_rng(3)
    p = r.standard_normal((6, 8)).astype(np.float32)
    t = r.standard_normal((6, 8)).astype(np.float32)
    wi = r.integers(0, 2, (6, 8)).astype(np.float32)
    wo = r.uniform(0.5, 2, (6, 8)).astype(np.float32)
    s2 = 9.0
    d = wi * (p - t)
    keep = np.abs(np.abs(d) - 1 / s2) > 1e-3                  # away from the kink
    t = np.where(keep, t, t + 0.5).astype(np.float32)

    def f64(z):
        v = wi * (z - t)
        a = np.abs(v)
        return (wo * np.where(a < 1 / s2, 0.5 * v * v * s2, a - 0.5 / s2)).sum() / z.shape[0]

    g = L.smooth_l1_loss_backward(p, t, wi, wo, sigma=3.0, top_diff=0.75)
    assert np.allclose(g, 0.75 * _num_grad(f64, p.astype(np.float64)), rtol=1e-4, atol=1e-6)


def test_sigmoid_ce_backward_is_the_gradient():
    r = np.random.default_rng(4)
    x = (3 * r.standard_normal((4, 9))).astype(np.float32)
    t = r.integers(0, 2, (4, 9)).astype(np.float32)
    w = r.integers(0, 2, (4, 9)).astype(np.float32)

    def f64(z):
        return (w * (np.logaddexp(0, z) - t * z)).sum() / w.sum()

    d = L.sigmoid_ce_loss_backward(x, t, w, top_diff=2.0)
    assert np.allclose(d, 2.0 * _num_grad(f64, x.astype(np.float64)), rtol=1e-4, atol=1e-6)
    assert abs(float(L.sigmoid_ce_loss(x, t, w)) - f64(x.astype(np.float64))) < 1e-5

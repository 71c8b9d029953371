"""numpy restatement of the training net's loss layers, the checker of mnc_b200/csrc/loss.cu:
  SoftmaxWithLoss          caffe-mnc/src/caffe/layers/softmax_loss_layer.cpp:10-86,
                           softmax_loss_layer.cu:11-124, Softmax: softmax_layer.cu:9-120
  SmoothL1Loss             smooth_L1_loss_layer.cpp:13-22, smooth_L1_loss_layer.cu:13-136
  SigmoidCrossEntropyLoss  sigmoid_cross_entropy_loss_layer.cpp:31-97, sigmoid: sigmoid_layer.cu:9-14
  Accuracy                 accuracy_layer.cpp:48-103
Every value keeps the float32 / float64 type the reference gives it, operation by operation.  The
loss sums are the project's fixed-order float64 reduction (`fixed_sum`), not the reference's
unordered cuBLAS or serial float loop (DESIGN.md "Loss layers").  exp / log of a float32 value are
taken in float64 and rounded once (correctly rounded up to the double-rounding corner), so values
they enter are within a few float32 ulp of the device's expf / logf, not bit-equal.

`n_valid` (int or None) keeps only the first n_valid outer rows, as the device's n_valid does."""
import numpy as np

F32 = np.float32
FLT_MIN = np.finfo(np.float32).tiny
FLT_MAX = np.finfo(np.float32).max
NORMALIZATION = {"FULL": 0, "VALID": 1, "BATCH_SIZE": 2, "NONE": 3}
THREADS = 1024   # the one CTA of the device's loss kernels


def fixed_sum(terms):
    """float32(sum of the float32 terms) in the device's order: partial t adds terms t, t + 1024,
    ... in float64; the 1024 partials are added by a halving tree p[t] += p[t + s]."""
    t = np.asarray(terms, np.float32).astype(np.float64).ravel()
    t = np.concatenate([t, np.zeros((-len(t)) % THREADS)]).reshape(-1, THREADS)
    p = np.zeros(THREADS)
    for row in t:
        p = p + row
    s = THREADS // 2
    while s:
        p[:s] = p[:s] + p[s:2 * s]
        s //= 2
    return F32(p[0])


def expf(x):
    return np.exp(np.asarray(x, np.float32).astype(np.float64)).astype(np.float32)


def logf(x):
    return np.log(np.asarray(x, np.float32).astype(np.float64)).astype(np.float32)


def _rows(a, n_valid):
    a = np.asarray(a, np.float32)
    return a if n_valid is None else a[:max(0, min(int(n_valid), a.shape[0]))]


def _onc(x):
    outer = x.shape[0]
    C = x.shape[1] if x.ndim > 1 else 1
    inner = x.size // max(outer * C, 1)
    return x.reshape(outer, C, inner)


# ----------------------------------------------------------------------------- SoftmaxWithLoss
def softmax(x):
    """softmax_layer.cu:86-120 over axis 1 of (outer, C, inner): max from -FLT_MAX, subtract,
    exp, channel sum in channel order, divide -- all float32."""
    x = _onc(np.asarray(x, np.float32))
    m = np.full((x.shape[0], x.shape[2]), -FLT_MAX, np.float32)
    for c in range(x.shape[1]):
        m = np.maximum(x[:, c], m)
    e = expf(x - m[:, None])
    s = np.zeros_like(m)
    for c in range(x.shape[1]):
        s = s + e[:, c]
    return e / s[:, None]


def normalizer(mode, rows, inner, valid_count):
    """get_normalizer (softmax_loss_layer.cpp:58-84): float32 of the count, at least 1."""
    mode = NORMALIZATION.get(mode, mode)
    n = {0: rows * inner, 1: rows * inner if valid_count == -1 else valid_count,
         2: rows, 3: 1}[mode]
    return max(F32(1.0), F32(n))


def _labels(labels, outer, inner):
    """static_cast<int> of the float labels (truncation toward zero)."""
    return np.trunc(np.asarray(labels, np.float32)).astype(np.int64).reshape(outer, inner)


def softmax_loss(scores, labels, ignore_label=None, normalization="VALID", n_valid=None):
    """softmax_loss_layer.cu:11-68 -> (loss float32, prob (rows, C, inner)).  A label outside
    [0, C) that is not ignored counts as valid and adds no term (the reference reads out of
    bounds there)."""
    x = _onc(_rows(scores, n_valid))
    outer, C, inner = x.shape
    lab = _labels(np.asarray(labels, np.float32).reshape(-1)[:outer * inner], outer, inner)
    prob = softmax(x)
    valid = np.ones(lab.shape, bool) if ignore_label is None else lab != ignore_label
    ok = valid & (lab >= 0) & (lab < C)
    pl = np.take_along_axis(prob, np.clip(lab, 0, C - 1)[:, None, :], 1)[:, 0]
    terms = np.where(ok, -logf(np.maximum(pl, FLT_MIN)), F32(0)).astype(np.float32)
    vc = int(valid.sum()) if (NORMALIZATION.get(normalization, normalization) == 1
                              and ignore_label is not None) else -1
    loss = fixed_sum(terms) / normalizer(normalization, outer, inner, vc)
    return F32(loss), prob


def softmax_loss_backward(prob, labels, top_diff=1.0, ignore_label=None, normalization="VALID"):
    """softmax_loss_layer.cu:70-124: prob, -1 at the label, 0 for an ignored position, times
    float32(top_diff / normaliser)."""
    prob = _onc(np.asarray(prob, np.float32))
    outer, C, inner = prob.shape
    lab = _labels(np.asarray(labels, np.float32).reshape(-1)[:outer * inner], outer, inner)
    valid = np.ones(lab.shape, bool) if ignore_label is None else lab != ignore_label
    d = prob.copy()
    for c in range(C):
        d[:, c] = np.where(valid & (lab == c), d[:, c] - F32(1), d[:, c])
        d[:, c] = np.where(valid, d[:, c], F32(0))
    vc = int(valid.sum()) if (NORMALIZATION.get(normalization, normalization) == 1
                              and ignore_label is not None) else -1
    scale = F32(top_diff) / normalizer(normalization, outer, inner, vc)
    return (d * scale).astype(np.float32)


# ------------------------------------------------------------------------------- SmoothL1Loss
def _smooth_l1_d(pred, target, w_in):
    d = np.asarray(pred, np.float32) - np.asarray(target, np.float32)
    return d if w_in is None else np.asarray(w_in, np.float32) * d


def smooth_l1_loss(pred, target, w_in=None, w_out=None, sigma=1.0, n_valid=None):
    """smooth_L1_loss_layer.cu:13-63: d in float32, the branch and its value in float64 stored as
    float32, times w_out; loss = sum / rows."""
    pred, target = _rows(pred, n_valid), _rows(target, n_valid)
    w_in = None if w_in is None else _rows(w_in, n_valid)
    w_out = None if w_out is None else _rows(w_out, n_valid)
    sigma2 = F32(sigma) * F32(sigma)
    val = _smooth_l1_d(pred, target, w_in)
    a = np.abs(val).astype(np.float64)
    s2 = np.float64(sigma2)
    e = np.where(a < 1.0 / s2, 0.5 * val.astype(np.float64) * val.astype(np.float64) * s2,
                 a - 0.5 / s2).astype(np.float32)
    if w_out is not None:
        e = np.asarray(w_out, np.float32) * e
    return F32(fixed_sum(e) / F32(pred.shape[0]))


def smooth_l1_loss_backward(pred, target, w_in=None, w_out=None, sigma=1.0, top_diff=1.0):
    """smooth_L1_loss_layer.cu:67-106, bottom 0: sigma2 * val or sign(val) (threshold in float64),
    * float32(top_diff / num), * w_in, * w_out."""
    pred = np.asarray(pred, np.float32)
    sigma2 = F32(sigma) * F32(sigma)
    val = _smooth_l1_d(pred, target, w_in)
    g = np.where(np.abs(val).astype(np.float64) < 1.0 / np.float64(sigma2), sigma2 * val,
                 np.sign(val)).astype(np.float32)
    d = (F32(top_diff) / F32(pred.shape[0])) * g
    if w_in is not None:
        d = np.asarray(w_in, np.float32) * d
        d = np.asarray(w_out, np.float32) * d
    return d.astype(np.float32)


# ---------------------------------------------------------------------- SigmoidCrossEntropyLoss
def sigmoid(x):
    """SigmoidForward (sigmoid_layer.cu:9-14) as the reference build compiles it: float32 exp of
    -x, then 1. + e and 1. / (...) in float64, rounded once."""
    e = expf(-np.asarray(x, np.float32)).astype(np.float64)
    return (1.0 / (1.0 + e)).astype(np.float32)


def sigmoid_ce_terms(x, t, w=None):
    """The float32 terms w * (x * (t - [x >= 0]) - log(1 + exp(x - 2x[x >= 0]))) of
    sigmoid_cross_entropy_loss_layer.cpp:44-55, all float32: the compiled object calls expf and
    logf (<math.h>, included through mkl_alternate.hpp, brings the float overloads into scope), and
    1 + e, a - l and w * (...) are float operations."""
    x, t = np.asarray(x, np.float32), np.asarray(t, np.float32)
    ge = (x >= 0).astype(np.float32)
    a = x * (t - ge)
    b = x - F32(2) * x * ge
    inner = a - logf(F32(1) + expf(b))
    if w is not None:
        inner = np.asarray(w, np.float32) * inner
    return inner.astype(np.float32)


def sigmoid_ce_loss(x, t, w=None, n_valid=None, untouched=F32(0)):
    """:31-59 -> -sum / sum w (weights), -sum / num (none); with weights summing to 0 the top is
    left as it was (`untouched`)."""
    x, t = _rows(x, n_valid), _rows(t, n_valid)
    w = None if w is None else _rows(w, n_valid)
    s = -fixed_sum(sigmoid_ce_terms(x, t, w))
    if w is None:
        return F32(s / F32(x.shape[0]))
    ws = fixed_sum(w)
    return F32(s / ws) if ws > 0 else F32(untouched)


def sigmoid_ce_loss_backward(x, t, w=None, top_diff=1.0):
    """:62-92: (sigmoid - t) * w, then * float32(top_diff / sum w) when sum w > 0; without
    weights * float32(top_diff / num)."""
    x = np.asarray(x, np.float32)
    d = sigmoid(x) - np.asarray(t, np.float32)
    if w is None:
        return (d * (F32(top_diff) / F32(x.shape[0]))).astype(np.float32)
    d = d * np.asarray(w, np.float32)
    ws = fixed_sum(w)
    return (d * (F32(top_diff) / ws)).astype(np.float32) if ws > 0 else d.astype(np.float32)


# ------------------------------------------------------------------------------------ Accuracy
def accuracy(scores, labels, top_k=1, ignore_label=None, n_valid=None):
    """accuracy_layer.cpp:48-96 literally: rank (score, class) pairs with std::greater (higher
    class first on equal scores), a hit when the label is among the first top_k; accuracy / count
    in float32 (0 / 0 -> nan)."""
    x = _onc(_rows(scores, n_valid))
    outer, C, inner = x.shape
    lab = _labels(np.asarray(labels, np.float32).reshape(-1)[:outer * inner], outer, inner)
    hits, count = 0, 0
    for i in range(outer):
        for j in range(inner):
            lv = int(lab[i, j])
            if ignore_label is not None and lv == ignore_label:
                continue
            ranked = sorted(((float(x[i, k, j]), k) for k in range(C)), reverse=True)
            hits += any(k == lv for _, k in ranked[:top_k])
            count += 1
    with np.errstate(invalid="ignore", divide="ignore"):
        return F32(F32(hits) / F32(count))

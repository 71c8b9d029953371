"""Head layers of the training net on the device: the split-bf16 InnerProduct GEMMs against float64
within the precision contract of tests/fc_bound.py at every MNC layer shape and at tail shapes, the
beta semantics of the backward, determinism and graph replay; max Pooling, ReLU and Sigmoid against
their numpy restatements bit for bit; the box branch through autograd against torch float64; and a
two-stage head step (ROIWarping, pools, shared-weight InnerProducts, ReLU, Sigmoid, losses) in one
CUDA graph against the layer mirrors."""
import zlib

import numpy as np
import pytest
import torch

from tests import fc_bound as F

pytestmark = pytest.mark.gpu
F32 = np.float32
FLT_MAX = np.finfo(np.float32).max


def _np(t):
    return t.detach().cpu().numpy()


def _same(a, b):
    """Bit-equal, except that any NaN equals any NaN (the device's arithmetic returns the canonical
    NaN where numpy propagates an operand's payload)."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32)))


def _within(got, ref64, absprod, extra64):
    """Fraction of the bound used: |got - ref| / (TAU |A||B| + OUT_ROUND (|ref| + |extra|))."""
    err = (got.double() - ref64).abs()
    den = F.TAU * absprod + F.OUT_ROUND * (ref64.abs() + extra64.abs()) + 1e-300
    return float((err / den).max())


def _fc_case(M, N, K, seed):
    from mnc_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) * 0.01
    b = torch.randn(N, device="cuda", generator=g)
    dy = torch.randn(M, N, device="cuda", generator=g)
    dw0 = torch.randn(N, K, device="cuda", generator=g)
    db0 = torch.randn(N, device="cuda", generator=g)
    y = ops.fc_forward(x, w, b)
    dw, db = dw0.clone(), db0.clone()
    dx = ops.fc_backward(x, w, dy, dw=dw, db=db)
    x64, w64, dy64 = x.double(), w.double(), dy.double()
    r = {}
    p = x64 @ w64.T
    r["fwd"] = _within(y, p + b.double(), x64.abs() @ w64.abs().T, p)
    del p
    p = dy64 @ w64
    r["dx"] = _within(dx, p, dy64.abs() @ w64.abs(), p)
    del p
    p = dy64.T @ x64
    r["dw"] = _within(dw, dw0.double() + p, dy64.abs().T @ x64.abs(), p)
    del p
    p = dy64.sum(0)
    r["db"] = _within(db, db0.double() + p, dy64.abs().sum(0), p)
    return r


@pytest.mark.parametrize("name,N,K", F.MNC_FC_SHAPES)
@pytest.mark.parametrize("M", F.BATCHES)
def test_fc_within_bound_at_mnc_shapes(name, N, K, M):
    r = _fc_case(M, N, K, seed=zlib.crc32(name.encode()) + M)
    print("FC_RATIO %s M=%d %s" % (name, M, " ".join("%s=%.3g" % kv for kv in r.items())))
    assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize("M,N,K", F.TAIL_SHAPES)
def test_fc_within_bound_at_tail_shapes(M, N, K):
    r = _fc_case(M, N, K, seed=M * 131 + N * 17 + K)
    print("FC_RATIO tail %dx%dx%d %s" % (M, N, K, " ".join("%s=%.3g" % kv for kv in r.items())))
    assert max(r.values()) <= 1.0, r


def _raw_fc(M, N, K, x, w, b, y, dy, dx, dw, db):
    from mnc_b200._lib import lib, ptr, cur_stream, check
    n = lib.mnc_fc_workspace_bytes(M, N, K)
    ws = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
    if y is not None:
        check(lib.mnc_fc_forward(ptr(x), ptr(w), ptr(b), ptr(y), M, N, K, ptr(ws), n,
                                 cur_stream()), "mnc_fc_forward")
    else:
        check(lib.mnc_fc_backward(ptr(x), ptr(w), ptr(dy), ptr(dx), ptr(dw), ptr(db), M, N, K,
                                  ptr(ws), n, cur_stream()), "mnc_fc_backward")


@pytest.mark.parametrize("M,N,K", [(67, 21, 99), (67, 256, 100352), (300, 84, 8192), (1, 441, 256)])
def test_fc_beta_semantics_and_untouched_memory(M, N, K):
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    x = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g)
    dy = torch.randn(M, N, device="cuda", generator=g)
    pad = 77

    def buf(n, fill):
        return torch.full((n + pad,), fill, dtype=torch.float32, device="cuda")

    # forward: exactly M*N written, nothing past it
    y = buf(M * N, 5.0)
    _raw_fc(M, N, K, x, w, None, y, None, None, None, None)
    assert torch.all(y[M * N:] == 5.0) and torch.isfinite(y[:M * N]).all()
    # dX overwrites (beta 0): a NaN-filled buffer gives the bits of a zero-filled one
    dxa, dxb = buf(M * K, float("nan")), buf(M * K, 0.0)
    _raw_fc(M, N, K, None, w, None, None, dy, dxa, None, None)
    _raw_fc(M, N, K, None, w, None, None, dy, dxb, None, None)
    assert torch.equal(dxa[:M * K], dxb[:M * K]) and torch.isnan(dxa[M * K:]).all()
    # dW / db accumulate (beta 1): from d0 the result is float32(d0 + the result from zeros)
    dw0 = torch.randn(N * K, device="cuda", generator=g)
    db0 = torch.randn(N, device="cuda", generator=g)
    dwa, dba = buf(N * K, 3.0), buf(N, 3.0)
    dwa[:N * K], dba[:N] = dw0, db0
    dwz, dbz = buf(N * K, 0.0), buf(N, 0.0)
    _raw_fc(M, N, K, x, None, None, None, dy, None, dwa, dba)
    _raw_fc(M, N, K, x, None, None, None, dy, None, dwz, dbz)
    assert torch.equal(dwa[:N * K], dw0 + dwz[:N * K]) and torch.equal(dba[:N], db0 + dbz[:N])
    assert torch.all(dwa[N * K:] == 3.0) and torch.all(dba[N:] == 3.0)
    # NULL outputs are neither computed nor touched: a dW-only call gives the dW bits of the full
    # call, and where none of the requested products splits, the workspace is left as it was
    from mnc_b200._lib import lib, ptr, cur_stream, check
    n = lib.mnc_fc_workspace_bytes(M, N, K)
    ws = torch.full((max(n, 1) // 4 + 1,), 9.0, device="cuda")
    s_dw = buf(N * K, 0.0)
    check(lib.mnc_fc_backward(ptr(x), None, ptr(dy), None, ptr(s_dw), None, M, N, K, ptr(ws),
                              ws.numel() * 4, cur_stream()), "mnc_fc_backward")
    full_dw, full_db, full_dx = buf(N * K, 0.0), buf(N, 0.0), buf(M * K, 0.0)
    _raw_fc(M, N, K, x, w, None, None, dy, full_dx, full_dw, full_db)
    assert torch.equal(s_dw, full_dw) and torch.equal(full_dx[:M * K], dxb[:M * K])
    if lib.mnc_fc_split_k(N, K, M) == 1:
        assert torch.all(ws == 9.0)


def test_fc_huge_finite_operands_stay_finite():
    """|x| above the largest bf16 splits into finite parts (hi rounded toward zero)."""
    from mnc_b200 import ops
    x = torch.full((3, 40), 3.4e38, device="cuda")
    x[1] = -3.4e38
    w = torch.full((5, 40), 1e-3, device="cuda")
    y = ops.fc_forward(x, w).double()
    ref = x.double() @ w.double().T
    assert torch.isfinite(y).all()
    assert ((y - ref).abs() <= F.TAU * (x.double().abs() @ w.double().abs().T)).all()


def test_fc_rejects_bad_arguments():
    from mnc_b200._lib import lib
    x = torch.zeros(4, 8, device="cuda")
    y = torch.zeros(4, 4, device="cuda")
    assert lib.mnc_fc_forward(x.data_ptr(), None, None, y.data_ptr(), 4, 4, 8, None, 0, None) == 1
    assert lib.mnc_fc_forward(x.data_ptr(), x.data_ptr(), None, y.data_ptr(), 0, 4, 8, None, 0,
                              None) == 1
    # a split-K shape without its workspace
    assert lib.mnc_fc_split_k(256, 67, 100352) > 1
    big = torch.zeros(67, 100352, device="cuda")
    w = torch.zeros(256, 100352, device="cuda")
    out = torch.zeros(67, 256, device="cuda")
    assert lib.mnc_fc_forward(big.data_ptr(), w.data_ptr(), None, out.data_ptr(), 67, 256, 100352,
                              None, 0, None) == 1
    # dW wanted without x, dX wanted without W
    assert lib.mnc_fc_backward(None, None, y.data_ptr(), None, w.data_ptr(), None, 4, 4, 8, None,
                               0, None) == 1
    assert lib.mnc_fc_backward(None, None, y.data_ptr(), x.data_ptr(), None, None, 4, 4, 8, None,
                               0, None) == 1


def test_fc_deterministic_and_graph_replay():
    from mnc_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(3)
    M, N, K = 67, 256, 100352     # split-K forward
    x = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) * 0.01
    b = torch.randn(N, device="cuda", generator=g)
    dy = torch.randn(M, N, device="cuda", generator=g)

    def step():
        dw = torch.zeros_like(w)
        db = torch.zeros_like(b)
        y = ops.fc_forward(x, w, b)
        dx = ops.fc_backward(x, w, dy, dw=dw, db=db)
        return [y, dx, dw, db]

    a, c = step(), step()
    assert all(torch.equal(u, v) for u, v in zip(a, c))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        out = step()
    gr.replay()
    torch.cuda.synchronize()
    first = [t.clone() for t in out]
    gr.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(u, v) for u, v in zip(first, out))
    assert all(torch.equal(u, v) for u, v in zip(a, out))


# ------------------------------------------------------------------ element-wise layers == numpy
def np_max_pool(x):
    N, C, H, W = x.shape
    PH, PW = (max(H - 2, 0) + 1) // 2 + 1, (max(W - 2, 0) + 1) // 2 + 1
    best = np.full((N, C, PH, PW), -FLT_MAX, F32)
    arg = np.full((N, C, PH, PW), -1, np.int32)
    for dh in (0, 1):
        for dw in (0, 1):
            hh = np.arange(PH) * 2 + dh
            ww = np.arange(PW) * 2 + dw
            ok = (hh[:, None] < H) & (ww[None, :] < W)
            v = x[:, :, np.minimum(hh, H - 1)][:, :, :, np.minimum(ww, W - 1)]
            upd = ok & (v > best)
            best = np.where(upd, v, best)
            arg = np.where(upd, (hh[:, None] * W + ww[None, :]).astype(np.int32), arg)
    return best, arg


def np_max_pool_backward(dy, arg, shape):
    N, C, H, W = shape
    dx = np.zeros((N * C, H * W), F32)
    a = arg.reshape(N * C, -1)
    d = dy.reshape(N * C, -1)
    for p in range(N * C):
        m = a[p] >= 0
        dx[p, a[p][m]] = F32(0) + d[p][m]    # each bottom element is covered by one window
    return dx.reshape(shape)


def _pool_input(rng, shape):
    x = rng.standard_normal(shape).astype(F32)
    x[..., ::3, :] = np.round(x[..., ::3, :])            # ties within windows
    x.reshape(-1)[rng.integers(0, x.size, x.size // 50)] = np.nan
    x[0, 0, :2, :2] = np.nan                             # an all-NaN window
    if shape[2] >= 4 and shape[3] >= 4:                  # windows of signed zeros only
        x[0, 0, 2:4, 0:2] = -0.0
        x[0, 0, 2, 2:4] = 0.0
        x[0, 0, 3, 2:4] = -0.0
    return x


@pytest.mark.parametrize("shape", [(3, 512, 28, 28), (67, 512, 14, 14), (2, 5, 7, 9), (1, 3, 1, 1),
                                   (2, 4, 13, 2)])
def test_max_pool_forward_backward_bitwise(shape):
    from mnc_b200 import ops
    rng = np.random.default_rng(sum(shape))
    x = _pool_input(rng, shape)
    y, m = ops.max_pool_nchw(torch.from_numpy(x).cuda())
    ry, rm = np_max_pool(x)
    assert np.array_equal(_np(m), rm)
    assert _same(_np(y), ry)
    if shape[2] >= 2 and shape[3] >= 2:
        assert _np(y)[0, 0, 0, 0] == -FLT_MAX and _np(m)[0, 0, 0, 0] == -1
    dy = rng.standard_normal(ry.shape).astype(F32)
    sp = np.array([-0.0, np.inf, -np.inf, np.nan, 0.0, -0.0, 1e-45], F32)[:dy.size]
    dy.reshape(-1)[:sp.size] = sp
    dx = ops.max_pool_backward_nchw(torch.from_numpy(dy).cuda(), m, shape)
    assert _same(_np(dx), np_max_pool_backward(dy, rm, shape))


def test_max_pool_rejects_other_parameters():
    from mnc_b200._lib import lib
    x = torch.zeros(1, 1, 4, 4, device="cuda")
    y = torch.zeros(1, 1, 2, 2, device="cuda")
    m = torch.zeros(1, 1, 2, 2, dtype=torch.int32, device="cuda")
    for k, s, p in [(3, 2, 0), (2, 1, 0), (2, 2, 1)]:
        assert lib.mnc_max_pool_nchw(x.data_ptr(), 1, 1, 4, 4, k, s, p, y.data_ptr(), m.data_ptr(),
                                     None) == 1
        assert lib.mnc_max_pool_backward_nchw(y.data_ptr(), m.data_ptr(), 1, 1, 4, 4, k, s, p,
                                              x.data_ptr(), None) == 1


def _special(rng, n):
    x = rng.standard_normal(n).astype(F32) * 4
    sp = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, 88.7, -88.7, 103.0, -104.0],
                  F32)
    x[:sp.size] = sp
    return x


def test_relu_forward_backward_bitwise():
    from mnc_b200 import ops
    rng = np.random.default_rng(5)
    n = 67 * 4096 + 5
    x = _special(rng, n)
    dy = _special(rng, n)
    dy[11:22] = np.array([np.nan, np.inf, -np.inf] * 3 + [1.0, -0.0], F32)   # over special x
    x[11:22] = np.array([-1.0, -2.0, 0.0, -0.0, 3.0, 5.0, np.nan, -3.0, -0.0, np.nan, 2.0], F32)
    y = _np(ops.relu(torch.from_numpy(x).cuda()))
    with np.errstate(invalid="ignore"):
        ry = np.where(x > 0, x, x * F32(0))
        rdx = dy * ((x > 0).astype(F32) + (x <= 0).astype(F32) * F32(0))
    assert _same(y, ry)
    assert np.signbit(y[(x < 0) & np.isfinite(x)]).all()
    dx = _np(ops.relu_backward(torch.from_numpy(x).cuda(), torch.from_numpy(dy).cuda()))
    assert _same(dx, rdx)


def test_sigmoid_forward_backward_bitwise():
    """The forward is the loss layers' sigmoid: SigmoidCrossEntropyLoss's backward at t = 0 and a
    loss weight of `rows` is exactly that sigmoid; the backward equals numpy float32."""
    from mnc_b200 import ops
    from oracle import oracle_loss as L
    rng = np.random.default_rng(6)
    x = _special(rng, 67 * 441)
    xt = torch.from_numpy(x).cuda()
    y = ops.sigmoid(xt)
    finite = np.isfinite(x)
    via_loss = ops.sigmoid_ce_loss_backward(torch.from_numpy(x[finite]).cuda().view(1, -1),
                                            torch.zeros(1, int(finite.sum()), device="cuda"),
                                            top_diff=torch.ones((), device="cuda"))
    assert np.array_equal(_np(y)[finite].view(np.uint32), _np(via_loss).reshape(-1).view(np.uint32))
    ref = L.sigmoid(x)
    assert np.all(np.abs(_np(y)[finite] - ref[finite]) <= 2 * np.spacing(np.abs(ref[finite])))
    assert np.isnan(_np(y)[np.isnan(x)]).all()
    dy = _special(rng, x.size)
    s = _np(y)
    dx = _np(ops.sigmoid_backward(y, torch.from_numpy(dy).cuda()))
    with np.errstate(invalid="ignore", over="ignore"):
        rdx = (dy * s) * (F32(1) - s)
    assert _same(dx, rdx)


# ------------------------------------------------------------------ box branch vs float64 autograd
def test_box_branch_matches_float64_autograd():
    from mnc_b200 import autograd as AG, ops
    g = torch.Generator(device="cuda").manual_seed(11)
    R, C = 67, 512

    def p(*s, scale=1.0):
        return (torch.randn(*s, device="cuda", generator=g) * scale).requires_grad_()

    feat = p(R, C, 14, 14)
    fc7_mask = p(R, 4096, scale=0.5)
    w6, b6 = p(4096, C * 49, scale=0.01), p(4096, scale=0.1)
    w7, b7 = p(4096, 4096, scale=0.02), p(4096, scale=0.1)
    wc, bc = p(21, 8192, scale=0.02), p(21, scale=0.1)
    labels = torch.randint(0, 21, (R,), device="cuda", generator=g).float()
    leaves = [feat, fc7_mask, w6, b6, w7, b7, wc, bc]

    pooled = AG.max_pool(feat)
    h6 = AG.relu(AG.inner_product(pooled, w6, b6))
    h7 = AG.relu(AG.inner_product(h6, w7, b7))
    score = AG.inner_product(torch.cat([fc7_mask, h7], 1), wc, bc)
    loss = AG.softmax_loss(score, labels)
    grads = torch.autograd.grad(loss, leaves)

    # float64 on the same fp32 leaves, with the device's pooling choices and ReLU decisions
    _, mask = ops.max_pool_nchw(feat.detach())
    L64 = [t.detach().double().requires_grad_() for t in leaves]
    f, fm, W6, B6, W7, B7, WC, BC = L64
    pooled64 = f.flatten(2).gather(2, mask.long().flatten(2)).view(R, -1)
    z6 = pooled64 @ W6.T + B6
    a6 = z6 * (h6.detach() > 0)
    z7 = a6 @ W7.T + B7
    a7 = z7 * (h7.detach() > 0)
    s64 = torch.cat([fm, a7], 1) @ WC.T + BC
    loss64 = torch.nn.functional.cross_entropy(s64, labels.long())
    g64 = torch.autograd.grad(loss64, L64)
    assert abs(float(loss.detach()) - float(loss64)) <= 1e-4 * abs(float(loss64))

    # composed bound: the same graph in float64 on |leaves| with the device's decisions, seeded with
    # |dL/dscore| plus what the scores' forward error (3 TAU |score chain|) can move the softmax,
    # gives per element the magnitude S every rounded product along the path is relative to
    A64 = [t.detach().double().abs().requires_grad_() for t in leaves]
    fa, fma, W6a, B6a, W7a, B7a, WCa, BCa = A64
    a6a = (fa.flatten(2).gather(2, mask.long().flatten(2)).view(R, -1) @ W6a.T + B6a) * (h6.detach() > 0)
    a7a = (a6a @ W7a.T + B7a) * (h7.detach() > 0)
    sa = torch.cat([fma, a7a], 1) @ WCa.T + BCa
    p64 = torch.softmax(s64.detach(), 1)
    onehot = torch.nn.functional.one_hot(labels.long(), 21).double()
    seed = (p64 - onehot).abs() / R + p64 * 2 * (3 * F.TAU * sa.detach()).max(1).values[:, None] / R
    S = torch.autograd.grad((sa * seed).sum(), A64)
    for name, a, r, m in zip(["feat", "fc7_mask", "w6", "b6", "w7", "b7", "wc", "bc"], grads, g64, S):
        ratio = float(((a.double() - r).abs() / (8 * F.TAU * m + F.OUT_ROUND * r.abs() + 1e-300)).max())
        print("BOX_BRANCH %s max |err| / composed bound = %.3g" % (name, ratio))
        assert ratio <= 1.0, (name, ratio)


# ------------------------------------------------------------------ two-stage head step
def _head_params(g):
    def p(*s, scale):
        return (torch.randn(*s, device="cuda", generator=g) * scale).requires_grad_()
    P = {}
    for name, N, K in F.MNC_FC_SHAPES:
        P[name + "_w"] = p(N, K, scale=(2.0 / K) ** 0.5)
        P[name + "_b"] = p(N, scale=0.01)
    return P


def _stage(P, conv5, rois, labels, mask_t, mask_w):
    """One stage's heads (train.prototxt, stage 1 or its _ext twin) from conv5_3 and the RoIs."""
    from mnc_b200 import autograd as AG
    premax = AG.roi_warp(conv5, rois, 28, 28, 0.0625)
    r5 = AG.max_pool(premax)                                         # 28 -> 14
    m6 = AG.relu(AG.inner_product(r5, P["fc6_maskest_w"], P["fc6_maskest_b"]))
    mask_pred = AG.inner_product(m6, P["mask_pred_w"], P["mask_pred_b"])
    mask_out = AG.sigmoid(mask_pred)
    box = AG.max_pool(r5)                                            # 14 -> 7
    h7 = AG.relu(AG.inner_product(AG.relu(AG.inner_product(box, P["fc6_w"], P["fc6_b"])),
                                  P["fc7_w"], P["fc7_b"]))
    mfeat = AG.mask_pool(r5, AG.mask_resize(mask_out.view(-1, 1, 21, 21), 14, 14))
    mbox = AG.max_pool(mfeat)
    m7 = AG.relu(AG.inner_product(AG.relu(AG.inner_product(mbox, P["fc6_mask_w"], P["fc6_mask_b"])),
                                  P["fc7_mask_w"], P["fc7_mask_b"]))
    join = torch.cat([m7, h7], 1)
    cls = AG.inner_product(join, P["cls_score_w"], P["cls_score_b"])
    seg = AG.inner_product(join, P["seg_cls_score_w"], P["seg_cls_score_b"])
    bbox = AG.inner_product(join, P["bbox_pred_w"], P["bbox_pred_b"])
    return (AG.softmax_loss(cls, labels) + AG.softmax_loss(seg, labels) +
            AG.sigmoid_ce_loss(mask_pred, mask_t, mask_w) +
            AG.smooth_l1_loss(bbox, torch.zeros_like(bbox))), bbox


def test_two_stage_head_step_graph_replay_and_shared_gradients():
    """Stage 1's heads on ROIWarping of the RoIs, StageBridgeLayer TRAIN on stage 1's bbox_pred,
    stage 2's heads on ROIWarping of the bridged RoIs with the bridge's targets; the whole step,
    forward and backward, in one CUDA graph."""
    from mnc_b200 import autograd as AG
    from oracle import oracle_train as T
    g = torch.Generator(device="cuda").manual_seed(21)
    P = _head_params(g)
    case = T.make_case(3)
    H, W = -(-600 // 16), -(-1000 // 16)
    conv5 = (torch.randn(1, 512, H, W, device="cuda", generator=g).relu()).requires_grad_()
    cu = lambda k: torch.from_numpy(np.ascontiguousarray(case[k])).cuda()
    rois1 = cu("rois").requires_grad_()
    n = rois1.shape[0]
    lab1 = torch.randint(0, 21, (n,), device="cuda", generator=g).float()
    mt1 = (torch.rand(n, 441, device="cuda", generator=g) > 0.5).float()
    mw1 = torch.ones_like(mt1)
    bridge_in = [cu("seg_cls_prob"), cu("gt_boxes"), torch.from_numpy(case["gt_masks"].astype(F32)).cuda(),
                 cu("im_info"), cu("mask_info")]
    leaves = [conv5, rois1] + list(P.values())

    def step():
        l1, bbox1 = _stage(P, conv5, rois1, lab1, mt1, mw1)
        rois2, lab2, mt2, mw2 = AG.stage_bridge_train(
            rois1, bbox1, *bridge_in, means=T.BBOX_NORMALIZE_MEANS, stds=T.BBOX_NORMALIZE_STDS,
            clip_thresh=1.0 / 512)[:4]
        l2, _ = _stage(P, conv5, rois2, lab2, mt2.reshape(-1, 441), mw2.reshape(-1, 441))
        return list(torch.autograd.grad(l1 + l2, leaves + [bbox1]))

    eager = [t.clone() for t in step()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        out = step()
    gr.replay()
    torch.cuda.synchronize()
    first = [t.clone() for t in out]
    gr.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(first, out))
    assert all(torch.equal(a, b) for a, b in zip(eager, out))
    names = ["conv5_3", "rois"] + list(P.keys()) + ["stage-1 bbox_pred"]
    for name, t in zip(names, eager):
        assert torch.isfinite(t).all() and t.abs().sum() > 0, name


def test_inner_product_mirror_accumulates_like_shared_caffe_blobs():
    """The InnerProductLayer mirror, fc6 and fc6_ext sharing blobs_, in Net::Backward order (_ext
    first): the blobs' diffs hold the sum of the two uses, and each bottom diff equals autograd's."""
    from mnc_b200 import autograd as AG
    from mnc_b200.lib.caffe import Blob
    from mnc_b200.lib.caffe.layers import InnerProductLayer
    rng = np.random.default_rng(4)
    N, K = 84, 8192
    x1 = rng.standard_normal((64, K)).astype(F32)
    x2 = rng.standard_normal((67, K)).astype(F32)
    W = (rng.standard_normal((N, K)) * 0.01).astype(F32)
    bias = rng.standard_normal(N).astype(F32)
    d1 = rng.standard_normal((64, N)).astype(F32)
    d2 = rng.standard_normal((67, N)).astype(F32)
    param = {"inner_product_param": {"num_output": N}}

    def blob(a):
        b = Blob()
        b.data = a.copy()
        return b

    b1, b2, t1, t2 = blob(x1), blob(x2), Blob(), Blob()
    L1, L2 = InnerProductLayer(param), InnerProductLayer(param)
    L1.LayerSetUp([b1], [t1])
    L1.blobs_[0].data[...] = W
    L1.blobs_[1].data[...] = bias
    L2.LayerSetUp([b2], [t2])
    L2.blobs_ = L1.blobs_
    L1.Forward([b1], [t1])
    L2.Forward([b2], [t2])
    t1.diff, t2.diff = d1, d2
    L2.Backward([t2], [True], [b2])
    L1.Backward([t1], [True], [b1])

    xt1, xt2 = [torch.from_numpy(a).cuda().requires_grad_() for a in (x1, x2)]
    wt, bt = [torch.from_numpy(a).cuda().requires_grad_() for a in (W, bias)]
    y1, y2 = AG.inner_product(xt1, wt, bt), AG.inner_product(xt2, wt, bt)
    assert np.array_equal(t1.data, _np(y1)) and np.array_equal(t2.data, _np(y2))
    g1 = torch.autograd.grad(y1, [xt1, wt, bt], torch.from_numpy(d1).cuda())
    g2 = torch.autograd.grad(y2, [xt2, wt, bt], torch.from_numpy(d2).cuda())
    assert np.array_equal(b1.diff, _np(g1[0])) and np.array_equal(b2.diff, _np(g2[0]))
    assert np.array_equal(L1.blobs_[0].diff, _np(g1[1] + g2[1]))
    assert np.array_equal(L1.blobs_[1].diff, _np(g1[2] + g2[2]))


def test_head_chains_through_mirrors_in_net_backward_order_equal_autograd():
    """Both stages' chains pool -> fc6 -> ReLU -> fc7 -> ReLU -> cls_score and mask_pred -> Sigmoid
    through the PoolingLayer / InnerProductLayer / ReLULayer (in place, as train.prototxt declares
    them) / SigmoidLayer mirrors, the _ext layers sharing stage 1's blobs_, Backward in
    Net::Backward order (stage 2's layers last to first, then stage 1's): every top, bottom diff and
    parameter diff equals autograd's bit for bit."""
    from mnc_b200 import autograd as AG
    from mnc_b200.lib.caffe import Blob
    from mnc_b200.lib.caffe import layers as LY
    rng = np.random.default_rng(8)
    shapes = {"fc6": (4096, 512 * 49), "fc7": (4096, 4096), "cls_score": (21, 4096),
              "mask_pred": (441, 256)}
    params = {k: ((rng.standard_normal((N, K)) * (2.0 / K) ** 0.5).astype(F32),
                  (rng.standard_normal(N) * 0.01).astype(F32)) for k, (N, K) in shapes.items()}
    stages = []
    for R in (67, 70):
        stages.append({"premax": rng.standard_normal((R, 512, 14, 14)).astype(F32),
                       "xm": rng.standard_normal((R, 256)).astype(F32),
                       "d_cls": rng.standard_normal((R, 21)).astype(F32),
                       "d_mask": rng.standard_normal((R, 441)).astype(F32)})

    def blob(a=None):
        b = Blob()
        if a is not None:
            b.data = a.copy()
        return b

    # ---- mirrors
    shared = {}
    runs = []
    for st in stages:
        B = {k: blob() for k in ("pool", "fc6", "fc7", "cls", "mask_pred", "mask_out")}
        B["premax"], B["xm"] = blob(st["premax"]), blob(st["xm"])
        ip = lambda name: LY.InnerProductLayer({"inner_product_param": {"num_output": shapes[name][0]}})
        seq = [(LY.PoolingLayer({"pooling_param": {"pool": "MAX", "kernel_size": 2, "stride": 2}}),
                "premax", "pool"),
               (ip("fc6"), "pool", "fc6"), (LY.ReLULayer(), "fc6", "fc6"),
               (ip("fc7"), "fc6", "fc7"), (LY.ReLULayer(), "fc7", "fc7"),
               (ip("cls_score"), "fc7", "cls"),
               (ip("mask_pred"), "xm", "mask_pred"), (LY.SigmoidLayer(), "mask_pred", "mask_out")]
        names = {1: "fc6", 3: "fc7", 5: "cls_score", 6: "mask_pred"}
        for i, (layer, bot, top) in enumerate(seq):
            layer.LayerSetUp([B[bot]], [B[top]])
            if i in names:
                n = names[i]
                if n in shared:
                    layer.blobs_ = shared[n]
                else:
                    layer.blobs_[0].data[...] = params[n][0]
                    layer.blobs_[1].data[...] = params[n][1]
                    shared[n] = layer.blobs_
            layer.Forward([B[bot]], [B[top]])
        B["cls"].diff, B["mask_out"].diff = st["d_cls"].copy(), st["d_mask"].copy()
        runs.append((seq, B))
    for seq, B in reversed(runs):
        for layer, bot, top in reversed(seq):
            layer.Backward([B[top]], [True], [B[bot]])

    # ---- autograd
    W = {k: (torch.from_numpy(w).cuda().requires_grad_(), torch.from_numpy(b).cuda().requires_grad_())
         for k, (w, b) in params.items()}
    loss, ins, outs = 0, [], []
    for st in stages:
        pm, xm = (torch.from_numpy(st[k]).cuda().requires_grad_() for k in ("premax", "xm"))
        h7 = AG.relu(AG.inner_product(AG.relu(AG.inner_product(AG.max_pool(pm), *W["fc6"])), *W["fc7"]))
        cls = AG.inner_product(h7, *W["cls_score"])
        mo = AG.sigmoid(AG.inner_product(xm, *W["mask_pred"]))
        loss = loss + (cls * torch.from_numpy(st["d_cls"]).cuda()).sum() + \
            (mo * torch.from_numpy(st["d_mask"]).cuda()).sum()
        ins += [pm, xm]
        outs += [cls, mo]
    leaves = ins + [t for pair in W.values() for t in pair]
    grads = torch.autograd.grad(loss, leaves)

    for (seq, B), cls, mo in zip(runs, outs[0::2], outs[1::2]):
        assert np.array_equal(B["cls"].data, _np(cls)) and np.array_equal(B["mask_out"].data, _np(mo))
    for i, (seq, B) in enumerate(runs):
        assert np.array_equal(B["premax"].diff, _np(grads[2 * i])), i
        assert np.array_equal(B["xm"].diff, _np(grads[2 * i + 1])), i
    for j, name in enumerate(W):
        blobs = shared[name]
        assert np.array_equal(blobs[0].diff, _np(grads[4 + 2 * j])), name
        assert np.array_equal(blobs[1].diff, _np(grads[4 + 2 * j + 1])), name

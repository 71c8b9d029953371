"""Convolution of the training net on the device (mnc_conv_forward / mnc_conv_backward): forward, dX,
dW and db against float64 within the precision contract of tests/conv_bound.py at the 16 layer
shapes of a 600x1000 and a 601x999 image and at tail shapes; the beta semantics and NULL outputs;
argument errors; huge and non-finite operands; determinism and graph replay; the trunk + RPN
training step in one CUDA graph; the RPN branch against float64 autograd; and a chain of
ConvolutionLayer mirrors in Net::Backward order against autograd bit for bit."""
import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from tests import conv_bound as C
from tests import fc_bound as F

pytestmark = pytest.mark.gpu
F32 = np.float32


def _np(t):
    return t.detach().cpu().numpy()


def _within(got, ref64, absprod, extra64):
    """Fraction of the bound used: |got - ref| / (TAU |A||B| + OUT_ROUND (|ref| + |extra|))."""
    err = (got.double() - ref64).abs()
    den = F.TAU * absprod + F.OUT_ROUND * (ref64.abs() + extra64.abs()) + 1e-300
    return float((err / den).max())


def _conv_case(N, Cin, H, W, Cout, k, seed):
    from mnc_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    pad = (k - 1) // 2
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * (2.0 / (Cin * k * k)) ** 0.5
    b = torch.randn(Cout, device="cuda", generator=g)
    dy = torch.randn(N, Cout, H, W, device="cuda", generator=g)
    dw0 = torch.randn(Cout, Cin, k, k, device="cuda", generator=g)
    db0 = torch.randn(Cout, device="cuda", generator=g)
    y = ops.conv_forward(x, w, b)
    dw, db = dw0.clone(), db0.clone()
    dx = ops.conv_backward(x, w, dy, dw=dw, db=db)
    x64, w64, dy64 = x.double(), w.double(), dy.double()
    r = {}
    p = TF.conv2d(x64, w64, padding=pad)
    r["fwd"] = _within(y, p + b.double()[:, None, None], TF.conv2d(x64.abs(), w64.abs(), padding=pad), p)
    del p
    p = torch.nn.grad.conv2d_input(x.shape, w64, dy64, padding=pad)
    r["dx"] = _within(dx, p, torch.nn.grad.conv2d_input(x.shape, w64.abs(), dy64.abs(), padding=pad), p)
    del p
    p = torch.nn.grad.conv2d_weight(x64, w.shape, dy64, padding=pad)
    r["dw"] = _within(dw, dw0.double() + p,
                      torch.nn.grad.conv2d_weight(x64.abs(), w.shape, dy64.abs(), padding=pad), p)
    del p
    p = dy64.sum((0, 2, 3))
    r["db"] = _within(db, db0.double() + p, dy64.abs().sum((0, 2, 3)), p)
    return r


@pytest.mark.parametrize("image", [(600, 1000), (601, 999)])
@pytest.mark.parametrize("name,Cin,Cout,k,level,learns", C.CONV_LAYERS)
def test_conv_within_bound_at_layer_shapes(name, Cin, Cout, k, level, learns, image):
    H, W = C.spatial(*image, level)
    r = _conv_case(1, Cin, H, W, Cout, k, seed=level * 1000 + Cin + Cout + image[1])
    print("CONV_RATIO %s %dx%d (%dx%d) %s" % (name, image[0], image[1], H, W,
                                             " ".join("%s=%.3g" % kv for kv in r.items())))
    assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize("N,Cin,H,W,Cout,k", C.TAIL_SHAPES)
def test_conv_within_bound_at_tail_shapes(N, Cin, H, W, Cout, k):
    r = _conv_case(N, Cin, H, W, Cout, k, seed=N * 7 + Cin * 131 + H * 17 + W + Cout)
    print("CONV_RATIO tail %s %s" % ((N, Cin, H, W, Cout, k), " ".join("%s=%.3g" % kv for kv in r.items())))
    assert max(r.values()) <= 1.0, r


def _raw(N, Cin, H, W, Cout, k, x=None, w=None, b=None, y=None, dy=None, dx=None, dw=None,
         db=None, pad=None, stride=1, ws=None, ws_bytes=None):
    from mnc_b200._lib import lib, ptr, cur_stream
    pad = (k - 1) // 2 if pad is None else pad
    if ws is None:
        n = lib.mnc_conv_workspace_bytes(N, Cin, H, W, Cout, k)
        ws = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
        ws_bytes = n if ws_bytes is None else ws_bytes
    if y is not None:
        return lib.mnc_conv_forward(ptr(x), ptr(w), ptr(b), ptr(y), N, Cin, H, W, Cout, k, pad,
                                    stride, ptr(ws), ws_bytes, cur_stream())
    return lib.mnc_conv_backward(ptr(x), ptr(w), ptr(dy), ptr(dx), ptr(dw), ptr(db), N, Cin, H, W,
                                 Cout, k, pad, stride, ptr(ws), ws_bytes, cur_stream())


@pytest.mark.parametrize("N,Cin,H,W,Cout,k", [(2, 65, 9, 9, 18, 3), (1, 256, 150, 250, 256, 3),
                                              (2, 512, 38, 63, 36, 1), (1, 3, 20, 33, 64, 3)])
def test_conv_beta_semantics_and_untouched_memory(N, Cin, H, W, Cout, k):
    g = torch.Generator(device="cuda").manual_seed(N + Cin + H + W + Cout + k)
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * 0.05
    dy = torch.randn(N, Cout, H, W, device="cuda", generator=g)
    nx, ny, nw = N * Cin * H * W, N * Cout * H * W, Cout * Cin * k * k
    pad = 77

    def buf(n, fill):
        return torch.full((n + pad,), fill, dtype=torch.float32, device="cuda")

    # forward: exactly the output written, nothing past it
    y = buf(ny, 5.0)
    assert _raw(N, Cin, H, W, Cout, k, x=x, w=w, y=y) == 0
    assert torch.all(y[ny:] == 5.0) and torch.isfinite(y[:ny]).all()
    # dX overwrites (beta 0): a NaN-filled buffer gives the bits of a zero-filled one
    dxa, dxb = buf(nx, float("nan")), buf(nx, 0.0)
    assert _raw(N, Cin, H, W, Cout, k, w=w, dy=dy, dx=dxa) == 0
    assert _raw(N, Cin, H, W, Cout, k, w=w, dy=dy, dx=dxb) == 0
    assert torch.equal(dxa[:nx], dxb[:nx]) and torch.isnan(dxa[nx:]).all()
    # dW / db accumulate (beta 1): dW adds each image's product in image order, as Caffe's per-image
    # gemm with beta 1 does; db adds the images' sum once.  From d0 the results are
    # float32(float32(d0 + image 0's dW) + image 1's dW) and float32(d0 + the db from zeros)
    dw0 = torch.randn(nw, device="cuda", generator=g)
    db0 = torch.randn(Cout, device="cuda", generator=g)
    dwa, dba = buf(nw, 3.0), buf(Cout, 3.0)
    dwa[:nw], dba[:Cout] = dw0, db0
    dbz = buf(Cout, 0.0)
    assert _raw(N, Cin, H, W, Cout, k, x=x, dy=dy, dw=dwa, db=dba) == 0
    assert _raw(N, Cin, H, W, Cout, k, dy=dy, db=dbz) == 0
    want = dw0.clone()
    for n in range(N):
        dwn = buf(nw, 0.0)
        assert _raw(1, Cin, H, W, Cout, k, x=x[n:n + 1].contiguous(), dy=dy[n:n + 1].contiguous(),
                    dw=dwn) == 0
        want = want + dwn[:nw]
    assert torch.equal(dwa[:nw], want) and torch.equal(dba[:Cout], db0 + dbz[:Cout])
    assert torch.all(dwa[nw:] == 3.0) and torch.all(dba[Cout:] == 3.0)
    # NULL outputs are neither computed nor touched: a dW-only call gives the dW bits of the full
    # call, a db-only call the db bits
    s_dw, s_db = buf(nw, 0.0), buf(Cout, 0.0)
    assert _raw(N, Cin, H, W, Cout, k, x=x, dy=dy, dw=s_dw) == 0
    assert _raw(N, Cin, H, W, Cout, k, dy=dy, db=s_db) == 0
    full_dw, full_db, full_dx = buf(nw, 0.0), buf(Cout, 0.0), buf(nx, 0.0)
    assert _raw(N, Cin, H, W, Cout, k, x=x, w=w, dy=dy, dx=full_dx, dw=full_dw, db=full_db) == 0
    assert torch.equal(s_dw, full_dw) and torch.equal(s_db, full_db)
    assert torch.equal(full_dx[:nx], dxb[:nx]) and torch.all(full_dx[nx:] == 0.0)


def test_conv_rejects_bad_arguments():
    from mnc_b200 import ops
    from mnc_b200.lib.caffe import Blob
    from mnc_b200.lib.caffe.layers import ConvolutionLayer
    x = torch.zeros(1, 8, 6, 6, device="cuda")
    w3, w1, w5 = (torch.zeros(4, 8, k, k, device="cuda") for k in (3, 1, 5))
    y = torch.zeros(1, 4, 6, 6, device="cuda")
    dy = torch.zeros(1, 4, 6, 6, device="cuda")
    ERR = 1
    # unsupported kernel, pad, stride
    assert _raw(1, 8, 6, 6, 4, 5, x=x, w=w5, y=y, pad=2) == ERR
    assert _raw(1, 8, 6, 6, 4, 3, x=x, w=w3, y=y, pad=0) == ERR
    assert _raw(1, 8, 6, 6, 4, 1, x=x, w=w1, y=y, pad=1) == ERR
    assert _raw(1, 8, 6, 6, 4, 3, x=x, w=w3, y=y, stride=2) == ERR
    assert _raw(1, 8, 6, 6, 4, 3, x=x, w=w3, dy=dy, dw=w3, stride=2) == ERR
    assert _raw(1, 8, 6, 6, 4, 5, x=x, w=w5, dy=dy, dw=w5, pad=2) == ERR
    assert _raw(0, 8, 6, 6, 4, 3, x=x, w=w3, y=y) == ERR
    # a short workspace: the backward needs mnc_conv_workspace_bytes, the forward only the split-K
    # partials of its own product (and succeeds with exactly those)
    from mnc_b200._lib import lib
    for k, w in ((3, w3), (1, w1)):
        n = lib.mnc_conv_workspace_bytes(1, 8, 6, 6, 4, k)
        if n:
            assert _raw(1, 8, 6, 6, 4, k, x=x, w=w, dy=dy, dx=x.clone(), ws_bytes=n - 1) == ERR
            assert _raw(1, 8, 6, 6, 4, k, x=x, dy=dy, dw=w.clone(), ws_bytes=n - 1) == ERR
    xb = torch.zeros(1, 512, 38, 63, device="cuda")
    wb = torch.zeros(512, 512, 3, 3, device="cuda")
    s = lib.mnc_fc_split_k(512, 38 * 63, 512 * 9)
    fwd = s * 512 * 38 * 63 * 4
    assert s > 1 and fwd < lib.mnc_conv_workspace_bytes(1, 512, 38, 63, 512, 3)
    assert _raw(1, 512, 38, 63, 512, 3, x=xb, w=wb, y=xb.clone(), ws_bytes=fwd - 4) == ERR
    assert _raw(1, 512, 38, 63, 512, 3, x=xb, w=wb, y=xb.clone(), ws_bytes=fwd) == 0
    # dW wanted without x, dX wanted without W
    assert _raw(1, 8, 6, 6, 4, 3, dy=dy, dw=w3) == ERR
    assert _raw(1, 8, 6, 6, 4, 3, dy=dy, dx=x) == ERR
    # a grouped weight (Cin / 2 input channels) and a grouped, strided or dilated layer
    with pytest.raises(ValueError):
        ops.conv_forward(x, torch.zeros(4, 4, 3, 3, device="cuda"))
    for extra in ({"group": 2}, {"stride": 2}, {"dilation": 2}, {"pad": 0}, {"kernel_size": 5, "pad": 2}):
        p = dict({"num_output": 4, "kernel_size": 3, "pad": 1}, **extra)
        b, t = Blob(1, 8, 6, 6), Blob()
        with pytest.raises(ValueError):
            ConvolutionLayer({"convolution_param": p}).LayerSetUp([b], [t])


def test_conv_huge_and_non_finite_operands():
    """|x| above the largest bf16 splits into finite parts; a +-Inf or NaN operand makes exactly the
    outputs it enters NaN."""
    from mnc_b200 import ops
    N, Cin, H, W, Cout = 1, 16, 10, 12, 8
    x = torch.full((N, Cin, H, W), 3.4e38, device="cuda")
    x[:, :, ::2] = -3.4e38
    w = torch.full((Cout, Cin, 3, 3), 1e-4, device="cuda")
    y = ops.conv_forward(x, w).double()
    ref = TF.conv2d(x.double(), w.double(), padding=1)
    assert torch.isfinite(y).all()
    assert ((y - ref).abs() <= F.TAU * TF.conv2d(x.double().abs(), w.double().abs(), padding=1)).all()

    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g)
    dy = torch.randn(N, Cout, H, W, device="cuda", generator=g)
    x[0, 3, 4, 5] = float("inf")
    x[0, 7, 2, 2] = float("nan")
    y = ops.conv_forward(x, w)
    want = torch.zeros(H, W, dtype=torch.bool, device="cuda")
    want[3:6, 4:7] = True
    want[1:4, 1:4] = True
    assert torch.equal(torch.isnan(y), want.expand(N, Cout, H, W))
    dw = torch.zeros_like(w)
    ops.conv_backward(x, w, dy, dw=dw, want_dx=False)
    bad = torch.zeros(Cin, dtype=torch.bool, device="cuda")
    bad[[3, 7]] = True
    assert torch.equal(torch.isnan(dw), bad[None, :, None, None].expand_as(dw))
    # a non-finite dY enters the dX of its 3x3 neighbourhood in every channel, and every db it sums
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g)
    dy[0, 2, 6, 0] = float("-inf")
    db = torch.zeros(Cout, device="cuda")
    dx = ops.conv_backward(x, w, dy, db=db)
    want = torch.zeros(H, W, dtype=torch.bool, device="cuda")
    want[5:8, 0:2] = True
    assert torch.equal(torch.isnan(dx), want.expand(N, Cin, H, W))
    assert torch.isinf(db[2]) and torch.isfinite(db[torch.arange(Cout, device="cuda") != 2]).all()


def test_conv_deterministic_and_graph_replay():
    from mnc_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(3)
    # conv5 at 600x1000: split-K forward and dW, N = 2
    N, Cin, H, W, Cout = 2, 512, 38, 63, 512
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) * 0.01
    b = torch.randn(Cout, device="cuda", generator=g)
    dy = torch.randn(N, Cout, H, W, device="cuda", generator=g)
    w1 = torch.randn(36, Cin, 1, 1, device="cuda", generator=g) * 0.01
    dy1 = torch.randn(N, 36, H, W, device="cuda", generator=g)

    def step():
        dw, db = torch.zeros_like(w), torch.zeros_like(b)
        dw1 = torch.zeros_like(w1)
        y = ops.conv_forward(x, w, b)
        dx = ops.conv_backward(x, w, dy, dw=dw, db=db)
        y1 = ops.conv_forward(x, w1)
        dx1 = ops.conv_backward(x, w1, dy1, dw=dw1)
        return [y, dx, dw, db, y1, dx1, dw1]

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


# ------------------------------------------------------------------ trunk + RPN training step
def _trunk_params(g):
    P = {}
    for name, Cin, Cout, k, level, learns in C.CONV_LAYERS:
        w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * (2.0 / (Cin * k * k)) ** 0.5
        b = torch.randn(Cout, device="cuda", generator=g) * 0.01
        P[name] = (w.requires_grad_(learns), b.requires_grad_(learns))
    return P


def _trunk(P, data):
    from mnc_b200 import autograd as AG
    h = data
    for name, *_ in C.CONV_LAYERS[:13]:
        h = AG.relu(AG.convolution(h, *P[name]))
        if name in C.POOL_AFTER:
            h = AG.max_pool(h)
    return h


def _rpn_targets(H, W, g):
    from mnc_b200 import autograd as AG
    gt = torch.tensor([[40., 60., 300., 420., 3.], [500., 100., 900., 560., 7.],
                       [120., 300., 380., 590., 12.]], device="cuda")
    info = torch.tensor([H * 16.0, W * 16.0, 1.0], device="cuda")
    return AG.anchor_target(H, W, gt, info)


def _rpn_loss(P, c5, at):
    from mnc_b200 import autograd as AG
    r = AG.relu(AG.convolution(c5, *P["rpn_conv_3x3"]))
    cls = AG.convolution(r, *P["rpn_cls_score"])
    bbox = AG.convolution(r, *P["rpn_bbox_pred"])
    _, _, H, W = cls.shape
    labels, targets, wi, wo = at
    loss = AG.softmax_loss(cls.view(1, 2, 9 * H, W), labels) + \
        AG.smooth_l1_loss(bbox, targets, wi, wo, sigma=3.0)
    return loss, cls, bbox


def test_trunk_and_rpn_step_in_one_cuda_graph():
    """data -> conv1_1 ... conv5_3 (ReLUs, pools) -> rpn_conv_3x3 -> ReLU -> rpn_cls_score /
    rpn_bbox_pred -> SoftmaxWithLoss (anchor_target labels) + SmoothL1Loss; a seeded head-side diff
    added to conv5_3's diff after the RPN's, as SplitLayer sums its tops; forward and backward in
    one CUDA graph."""
    from mnc_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(17)
    P = _trunk_params(g)
    data = torch.randn(1, 3, 600, 1000, device="cuda", generator=g) * 50
    H5, W5 = C.spatial(600, 1000, 4)
    at = _rpn_targets(H5, W5, g)
    head_diff = torch.randn(1, 512, H5, W5, device="cuda", generator=g) * 1e-3
    learn = [t for name, *_, learns in C.CONV_LAYERS if learns for t in P[name]]

    calls = []
    real = ops.conv_backward

    def spy(x, w, dy, dw=None, db=None, want_dx=True):
        calls.append((tuple(w.shape), want_dx))
        return real(x, w, dy, dw=dw, db=db, want_dx=want_dx)

    def step():
        c5 = _trunk(P, data)
        c5s = c5.detach().requires_grad_()
        loss, _, _ = _rpn_loss(P, c5s, at)
        rpn_params = [t for n in ("rpn_conv_3x3", "rpn_cls_score", "rpn_bbox_pred") for t in P[n]]
        g_rpn = torch.autograd.grad(loss, [c5s] + rpn_params)
        d5 = g_rpn[0] + head_diff          # SplitLayer: top 0 (rpn_conv_3x3) + top 1 (the heads)
        trunk = learn[:-6]
        return list(torch.autograd.grad(c5, trunk, d5)) + list(g_rpn[1:]) + [loss.detach()]

    ops.conv_backward = spy
    try:
        eager = [t.clone() for t in step()]
    finally:
        ops.conv_backward = real
    # 12 learning layers (conv3_1 ... conv5_3 and the RPN's three), one backward each; conv3_1's
    # computes no dX; conv1_x / conv2_x none
    assert len(calls) == 12, calls
    shapes = {(Cout, Cin, k, k): name for name, Cin, Cout, k, *_ in C.CONV_LAYERS}
    assert calls[-1] == ((256, 128, 3, 3), False)
    assert all(want for _, want in calls[:-1])
    assert not any(shapes.get(s, "").startswith(("conv1", "conv2")) for s, _ in calls)

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
    names = [n for n, *_, learns in C.CONV_LAYERS if learns]
    trunk_names = names[:-3]
    order = [(n, k) for n in trunk_names for k in ("w", "b")] + \
        [(n, k) for n in names[-3:] for k in ("w", "b")]
    for (n, kind), t in zip(order, eager[:-1]):
        assert torch.isfinite(t).all() and t.abs().sum() > 0, (n, kind)
    for name in ("conv1_1", "conv1_2", "conv2_1", "conv2_2"):
        assert all(t.grad is None and not t.requires_grad for t in P[name]), name
    print("TRUNK_STEP rpn loss %.6g" % float(eager[-1]))


def test_rpn_branch_matches_float64_autograd():
    """conv5_3 -> rpn_conv_3x3 -> ReLU -> rpn_cls_score / rpn_bbox_pred -> SoftmaxWithLoss +
    SmoothL1Loss, every gradient per element within a composed bound of float64 autograd on the
    same fp32 leaves."""
    g = torch.Generator(device="cuda").manual_seed(23)
    H, W = C.spatial(600, 1000, 4)
    P = _trunk_params(g)
    conv5 = (torch.randn(1, 512, H, W, device="cuda", generator=g).relu()).requires_grad_()
    at = _rpn_targets(H, W, g)
    labels, targets, wi, wo = at
    leaves = [conv5] + [t for n in ("rpn_conv_3x3", "rpn_cls_score", "rpn_bbox_pred") for t in P[n]]
    loss, cls, bbox = _rpn_loss(P, conv5, at)
    grads = torch.autograd.grad(loss, leaves)

    # float64 on the same fp32 leaves with the device's ReLU decisions and smooth-L1 branches
    from mnc_b200 import autograd as AG
    with torch.no_grad():
        relu_on = AG.convolution(conv5, *P["rpn_conv_3x3"]) > 0
        quad = (bbox - targets).abs() * wi < 1.0 / 9.0
    L64 = [t.detach().double().requires_grad_() for t in leaves]
    c, w3, b3, wc, bc, wb, bb = L64

    def heads(c, w3, b3, wc, bc, wb, bb):
        h = (TF.conv2d(c, w3, b3, padding=1)) * relu_on
        return TF.conv2d(h, wc, bc), TF.conv2d(h, wb, bb)

    s64, b64 = heads(*L64)
    lab = labels.view(-1).long()
    valid = lab >= 0
    sc = s64.view(1, 2, -1).permute(0, 2, 1).reshape(-1, 2)
    nv = int(valid.sum())
    loss_cls = TF.cross_entropy(sc[valid], lab[valid], reduction="sum") / nv
    d = (b64 - targets.double()) * wi.double()
    sl1 = torch.where(quad, 0.5 * 9.0 * d * d, d.abs() - 0.5 / 9.0)
    loss64 = loss_cls + (wo.double() * sl1).sum()
    g64 = torch.autograd.grad(loss64, L64)
    assert abs(float(loss.detach()) - float(loss64)) <= 1e-4 * abs(float(loss64))

    # composed bound: the same graph in float64 on |leaves| with the device's decisions, seeded with
    # |dL/dout| plus what each output's forward error (3 TAU |out chain|) can move its loss gradient
    A64 = [t.detach().double().abs().requires_grad_() for t in leaves]
    sa, ba = heads(*A64)
    p64 = torch.softmax(sc.detach(), 1)
    onehot = TF.one_hot(lab.clamp(min=0), 2).double()
    sa2 = sa.detach().view(1, 2, -1).permute(0, 2, 1).reshape(-1, 2)
    seed_s = ((p64 - onehot).abs() + p64 * 2 * (3 * F.TAU * sa2).max(1).values[:, None]) * \
        valid[:, None] / nv
    seed_s = seed_s.view(1, -1, 2).permute(0, 2, 1).reshape(sa.shape)
    seed_b = wo.double() * wi.double() * (torch.where(quad, 9.0 * d.detach().abs(), torch.ones_like(d)) +
                                          9.0 * wi.double() * 3 * F.TAU * ba.detach())
    S = torch.autograd.grad((sa * seed_s).sum() + (ba * seed_b).sum(), A64)
    for name, a, r, m in zip(["conv5_3", "rpn_conv_w", "rpn_conv_b", "cls_w", "cls_b", "bbox_w",
                              "bbox_b"], grads, g64, S):
        ratio = float(((a.double() - r).abs() / (8 * F.TAU * m + F.OUT_ROUND * r.abs() + 1e-300)).max())
        print("RPN_BRANCH %s max |err| / composed bound = %.3g" % (name, ratio))
        assert ratio <= 1.0, (name, ratio)


def test_conv_mirror_chain_in_net_backward_order_equals_autograd():
    """conv2_2 (frozen: param_propagate_down_ false), pool2, conv3_1 ... conv5_3 and the 1x1
    rpn_cls_score through ConvolutionLayer, ReLULayer (in place, as train.prototxt declares them)
    and PoolingLayer mirrors, Backward in Net::Backward order with propagate_down false from conv3_1
    down: every top and parameter diff equals autograd's bit for bit, the frozen layer's blobs'
    diffs are left as they were, and no bottom diff below conv3_1 is written."""
    from mnc_b200 import autograd as AG
    from mnc_b200.lib.caffe import Blob
    from mnc_b200.lib.caffe import layers as LY
    rng = np.random.default_rng(9)
    convs = [l for l in C.CONV_LAYERS
             if l[0] == "conv2_2" or l[0].startswith(("conv3", "conv4", "conv5")) or l[0] == "rpn_cls_score"]
    params = {n: ((rng.standard_normal((Co, Ci, k, k)) * (2.0 / (Ci * k * k)) ** 0.5).astype(F32),
                  (rng.standard_normal(Co) * 0.01).astype(F32)) for n, Ci, Co, k, *_ in convs}
    x0 = np.abs(rng.standard_normal((1, 128, 150, 250))).astype(F32)
    sentinel = {n: [np.full(a.shape, 7.0, F32) for a in params[n]] for n in params}

    def blob(a=None):
        b = Blob()
        if a is not None:
            b.data = a.copy()
        return b

    # ---- mirrors: (layer, bottom, top, propagate_down)
    B = {"conv2_1": blob(x0)}
    seq = []
    prev = "conv2_1"

    def run(L, bot, top, pd):
        L.LayerSetUp([B[bot]], [B[top]])
        if isinstance(L, LY.ConvolutionLayer):
            L.blobs_[0].data[...], L.blobs_[1].data[...] = params[top]
            for blb, sv in zip(L.blobs_, sentinel[top]):
                blb.diff = sv.copy()
            if top == "conv2_2":
                L.param_propagate_down_ = [False, False]
        L.Forward([B[bot]], [B[top]])
        seq.append((L, bot, top, pd))

    learning = False
    for n, Ci, Co, k, *_ in convs:
        B[n] = blob()
        run(LY.ConvolutionLayer({"convolution_param": {"num_output": Co, "kernel_size": k,
                                                        "pad": (k - 1) // 2}}), prev, n, learning)
        learning = True
        if n == "conv2_2":
            learning = False      # conv3_1's bottom: nothing below it learns
        if n == "rpn_cls_score":
            break
        run(LY.ReLULayer(), n, n, n != "conv2_2")
        prev = n
        if n in C.POOL_AFTER:
            pn = "pool" + n[4]
            B[pn] = blob()
            run(LY.PoolingLayer({"pooling_param": {"pool": "MAX", "kernel_size": 2, "stride": 2}}),
                n, pn, n != "conv2_2")
            prev = pn
    seed = rng.standard_normal(B["rpn_cls_score"].shape).astype(F32)
    B["rpn_cls_score"].diff = seed.copy()
    for L, bot, top, pd in reversed(seq):
        L.Backward([B[top]], [pd], [B[bot]])

    # ---- autograd
    W = {n: tuple(torch.from_numpy(a).cuda().requires_grad_(n != "conv2_2") for a in params[n])
         for n in params}
    h = torch.from_numpy(x0).cuda()
    for n, *_ in convs:
        h = AG.convolution(h, *W[n])
        if n == "rpn_cls_score":
            break
        h = AG.relu(h)
        if n in C.POOL_AFTER:
            h = AG.max_pool(h)
    assert np.array_equal(B["rpn_cls_score"].data, _np(h))
    learn = [n for n in W if n != "conv2_2"]
    leaves = [t for n in learn for t in W[n]]
    grads = torch.autograd.grad(h, leaves, torch.from_numpy(seed).cuda())
    assert B["conv2_1"].diff is None and B["pool2"].diff is None
    layers = {top: L for L, _, top, _ in seq if isinstance(L, LY.ConvolutionLayer)}
    for i, n in enumerate(learn):
        # the blobs' diffs held 7.0 before Backward: they accumulate onto it
        assert np.array_equal(layers[n].blobs_[0].diff, _np(grads[2 * i] + 7.0)), n
        assert np.array_equal(layers[n].blobs_[1].diff, _np(grads[2 * i + 1] + 7.0)), n
    assert all(np.array_equal(blb.diff, sv) for blb, sv in zip(layers["conv2_2"].blobs_, sentinel["conv2_2"]))

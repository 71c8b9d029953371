"""Tri-plane conversions, precision modes against each other and against fp64, CUDA-graph replay
vs eager launches, the pipelined host API."""
import numpy as np
import pytest
import torch

from tests import util

pytestmark = pytest.mark.gpu


def test_tri_conversion_device_equals_torch_restatement():
    from mnc_b200 import dense
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(4096, 96, device="cuda", generator=g) * torch.exp2(torch.randint(-8, 6, (4096, 1), device="cuda", generator=g).float())
    x[0, :8] = torch.tensor([0.0, -0.0, 1e-30, -1e-30, 7e4, -7e4, 1.0, -1.0], device="cuda")
    e = dense.exp_for(float(x.abs().max()))
    want = dense.tri_from_f32(x, exp=e)
    got = dense.tri_alloc(x.shape, "cuda")
    amax = torch.zeros(1, dtype=torch.int32, device="cuda")
    dense.f32_to_tri(x.contiguous(), got, e, amax=amax)
    torch.cuda.synchronize()
    assert torch.equal(got.h, want.h) and torch.equal(got.l, want.l) and torch.equal(got.c, want.c)
    assert amax.view(torch.float32).item() == float(x.abs().max())
    back = torch.empty_like(x)
    dense.split_to_f32(got, back)
    assert torch.equal(back, got.float())
    # the two precise planes carry x to ~2^-16 of the tensor maximum
    assert (back - x).abs().max() <= 2.0 ** -15 * x.abs().max()


@pytest.mark.parametrize("M,N,K", [(300, 256, 512), (2400, 192, 4096), (257, 448, 1024)])
def test_both_precision_modes_match_fp64(M, N, K):
    """Inner product in both operand formats: precision mode 1 stays within 3e-5 of fp64 like the
    split-bf16 mode, and a second launch on the same operands returns the same bits."""
    from mnc_b200 import dense
    g = torch.Generator(device="cuda").manual_seed(M + N)
    x = torch.relu(torch.randn(M, K, device="cuda", generator=g))
    w = torch.randn(N, K, device="cuda", generator=g) * (2.0 / K) ** 0.5
    b = torch.randn(N, device="cuda", generator=g) * 0.1
    ref = x.double() @ w.double().T + b.double()
    outs = {}
    for rep in (0, 1):
        xs, ws = dense.split(x), dense.split(w)
        o0 = torch.empty(M, N, device="cuda")
        dense.igemm2(xs.view(2, 1, 1, M, K), 1, 1, M, K, ws, N, 1, bias=b, out_f32=o0)
        xt, wt = dense.tri_from_f32(x), dense.tri_from_f32(w, weight=True)
        o1 = torch.empty(M, N, device="cuda")
        dense.igemm2(xt.view(1, 1, M, K), 1, 1, M, K, wt, N, 1, bias=b, out_f32=o1)
        outs[rep] = (o0, o1)
    torch.cuda.synchronize()
    assert torch.equal(outs[1][0], outs[0][0]) and torch.equal(outs[1][1], outs[0][1])
    for o in outs[0]:
        assert util.rel_err(o.cpu().numpy(), ref.cpu().numpy()) < 3e-5


@pytest.mark.parametrize("B,H,W,Cin,Cout,pool", [(1, 16, 8, 64, 64, False), (3, 37, 53, 64, 64, True),
                                                 (1, 75, 125, 64, 128, False), (2, 30, 21, 128, 128, True),
                                                 (1, 16, 24, 64, 80, False)])
def test_conv3x3_tri_plane_small_cout(B, H, W, Cin, Cout, pool):
    """3x3 convolution in precision mode 1 at the low-Cout shapes of conv1_2 .. conv2_2: ragged
    tiles, Cout tails, fused pooling; all three output planes are reproducible bit for bit and the
    value is within 1e-4 of fp64."""
    from mnc_b200 import dense
    g = torch.Generator(device="cuda").manual_seed(H * W + Cout)
    x = torch.relu(torch.randn(B, H, W, Cin, device="cuda", generator=g))
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / (9 * Cin) ** 0.5
    b = torch.randn(Cout, device="cuda", generator=g) * 0.1
    xt, wt = dense.tri_from_f32(x), dense.conv_weight_to_tri(w)
    Ho, Wo = ((H + 1) // 2, (W + 1) // 2) if pool else (H, W)
    outs = {}
    for rep in (1, 0):
        o = dense.tri_alloc((B, Ho, Wo, Cout), "cuda")
        for t in (o.h, o.l, o.c):
            t.zero_()
        dense.igemm2(xt, B, H, W, Cin, wt, Cout, 9, bias=b, relu=True, out=o, pool=pool, out_exp=9)
        outs[rep] = o
    torch.cuda.synchronize()
    for pl in ("h", "l", "c"):
        assert torch.equal(getattr(outs[1], pl), getattr(outs[0], pl)), pl
    import torch.nn.functional as F
    ref = F.relu(F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), b.double(), padding=1))
    if pool:
        ref = F.max_pool2d(ref, 2, 2, ceil_mode=True)
    assert util.rel_err(outs[1].float().cpu().numpy(), ref.permute(0, 2, 3, 1).cpu().numpy()) < 1e-4


def _engine_outputs(eng, data, im_info):
    out = eng.forward(data, im_info, keep_intermediate=True)
    torch.cuda.synchronize()
    return out


def test_precision_modes_agree_on_full_arch():
    """The fp16 + 2 x FP8 engine against the split-bf16 engine on the same weights and image:
    conv5_3 within 1e-4, identical RoI lists, head outputs within 1e-3."""
    from mnc_b200 import dense, weights as Wt
    from mnc_b200.engine import MNCEngine
    from oracle import oracle as O
    w = Wt.make_weights(Wt.FULL_ARCH)
    im = O.synthetic_image(3, 224, 320)
    blob, info = O.prep_blob(im)
    data, im_info = torch.from_numpy(blob).cuda(), torch.from_numpy(info).cuda()
    a = _engine_outputs(MNCEngine(w, precision="bf16x3"), data, im_info)
    b = _engine_outputs(MNCEngine(w, precision="f16f8"), data, im_info)
    ca, cb = dense.merge(a["_conv5_3"]).cpu().numpy(), dense.merge(b["_conv5_3"]).cpu().numpy()
    assert util.rel_err(cb, ca) < 1e-4
    na, nb = int(a["roi_counts"][0]), int(b["roi_counts"][0])
    assert na == nb and na > 50
    ra, rb = a["rois"][:na].cpu().numpy(), b["rois"][:nb].cpu().numpy()
    # a near-tie may swap or replace a few proposals between the modes (which shifts every later
    # position): pair the lists by coordinates
    d = np.abs(ra[:, None, 1:] - rb[None, :, 1:]).max(axis=2)
    jb = d.argmin(axis=1)
    ia = np.where(d[np.arange(na), jb] < 0.05)[0]
    jb = jb[ia]
    assert len(ia) >= 0.97 * na and len(set(jb)) == len(jb)
    assert (np.diff(jb) <= 0).sum() <= 0.03 * na
    for k in ("mask_proposal", "seg_cls_prob", "cls_prob"):
        assert np.abs(a[k][:na].cpu().numpy()[ia] - b[k][:nb].cpu().numpy()[jb]).max() < 1e-3, k


def test_graph_replay_equals_eager():
    from mnc_b200 import weights as Wt
    from mnc_b200.engine import MNCEngine
    from oracle import oracle as O
    w = Wt.make_weights(Wt.TINY_ARCH)
    eng = MNCEngine(w)
    B, H, W = 2, 224, 320
    blobs = [O.prep_blob(O.synthetic_image(i, H, W)) for i in range(B)]
    data = torch.from_numpy(np.concatenate([b[0] for b in blobs])).cuda()
    info = torch.from_numpy(np.concatenate([b[1] for b in blobs])).cuda()
    hw = torch.tensor([[H, W]] * B, dtype=torch.float32).cuda()
    sc = torch.ones(B).cuda()
    eager = [t.clone() for t in eng.detect(data, info, hw, sc)[:4]]
    for _ in range(3):      # capture, then two replays
        graphed = eng.detect_graphed(data, info, hw, sc)[:4]
    torch.cuda.synchronize()
    for e, g_ in zip(eager, graphed):
        assert torch.equal(e, g_)
    # other inputs of the same shape are copied into the captured buffers
    data2 = torch.from_numpy(np.concatenate([O.prep_blob(O.synthetic_image(7 + i, H, W))[0] for i in range(B)])).cuda()
    want = [t.clone() for t in eng.detect(data2, info, hw, sc)[:4]]
    got = eng.detect_graphed(data2, info, hw, sc)[:4]
    torch.cuda.synchronize()
    for e, g_ in zip(want, got):
        assert torch.equal(e, g_)


def test_two_steps_in_flight_agree():
    """MNCEngine.clone_state: a second engine state over the same weights; two steps issued
    back to back on two streams (graph replays) produce the same record as one alone."""
    from mnc_b200 import weights as Wt
    from mnc_b200.engine import MNCEngine
    from oracle import oracle as O
    w = Wt.make_weights(Wt.TINY_ARCH)
    eng = MNCEngine(w)
    ims = [O.synthetic_image(5 + i, 224, 320) for i in range(2)]
    blobs = [O.prep_blob(im) for im in ims]
    data = torch.from_numpy(np.concatenate([b[0] for b in blobs])).cuda()
    im_info = torch.from_numpy(np.concatenate([b[1] for b in blobs])).cuda()
    im_hw = torch.tensor([[224., 320.]] * 2, device="cuda")
    im_scale = torch.ones(2, device="cuda")
    eng.detect_graphed(data, im_info, im_hw, im_scale)
    torch.cuda.synchronize()
    want = eng.last_record.clone()
    eng2 = eng.clone_state()
    assert eng2.exp is eng.exp and eng2._buf is not eng._buf
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for s, e in ((s1, eng), (s2, eng2)):          # capture the clone's graph, warm both
        with torch.cuda.stream(s):
            e.detect_graphed(data, im_info, im_hw, im_scale)
    torch.cuda.synchronize()
    for _ in range(3):
        for s, e in ((s1, eng), (s2, eng2)):
            with torch.cuda.stream(s):
                e.detect_graphed(data, im_info, im_hw, im_scale)
    torch.cuda.synchronize()
    assert torch.equal(eng.last_record, want) and torch.equal(eng2.last_record, want)


def test_detector_stream_equals_blocking_calls():
    from mnc_b200 import weights as Wt
    from mnc_b200.api import Detector
    from oracle import oracle as O
    det = Detector(Wt.make_weights(Wt.TINY_ARCH), max_batch=2, height=600, width=800)
    batches = [np.stack([O.synthetic_image(10 * k + i, 375, 500) for i in range(2)]) for k in range(4)]
    want = []
    for b in batches:
        bx, mk, sc, vl, s = det.im_detect_images(b)
        want.append((bx.copy(), mk.copy(), sc.copy(), vl.copy(), s))
    n = 0
    for got, w_ in zip(det.im_detect_stream(iter(batches)), want):
        for a, b in zip(got[:4], w_[:4]):
            assert np.array_equal(a, b)
        assert got[4] == w_[4] == 1.6
        n += 1
    assert n == 4


def test_exponent_range_monitor_recalibrates():
    """The tri-plane exponents are frozen on the first forward; an input 200x larger saturates the
    fp16 operands, which range_ok() must detect (the producing kernels keep a running max) and the
    next forward must repair by measuring the exponents again."""
    from mnc_b200 import weights as Wt
    from mnc_b200.engine import MNCEngine
    from oracle import oracle as O
    w = Wt.make_weights(Wt.TINY_ARCH)
    eng = MNCEngine(w)
    blob, info = O.prep_blob(O.synthetic_image(1, 224, 320))
    data, im_info = torch.from_numpy(blob).cuda(), torch.from_numpy(info).cuda()
    eng.forward(data, im_info)
    assert eng.range_ok()
    exp_before = dict(eng.exp)
    big = data * 200.0
    eng.forward(big, im_info)                   # computed with stale exponents: saturated
    assert not eng.range_ok() and eng.last_range_violation
    out = eng.forward(big, im_info, keep_intermediate=True)    # recalibrates first
    assert eng.range_ok()
    assert any(eng.exp[k] < exp_before[k] for k in exp_before)
    # and the result is right again: stage-1 head on the engine's own features vs the oracle
    from mnc_b200 import dense
    n = int(out["roi_counts"][0])
    got14 = dense.merge(out["_feat14"])[:n].permute(0, 3, 1, 2).cpu().numpy()
    with torch.no_grad():
        h = O.head_forward(w, got14)
    # (linear outputs: at 200x the softmax is saturated and amplifies 1e-5 of a logit)
    assert util.rel_err(out["bbox_pred"][:n].cpu().numpy(), h["bbox_pred"]) < 1e-3
    assert util.rel_err(out["_mask_logits"][:n, :441].cpu().numpy(), h["mask_pred"]) < 1e-3

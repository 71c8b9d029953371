"""mnc_igemm_tc2 in precision mode 1 (tri-plane operands, the engine's default) against the fp64
product of the original fp32 operands, element by element:

    |got - ref|_ij  <=  tau(K) * (|X| . |W|^T)_ij  +  the rounding of the output format.

A max-norm relative error hides errors in small columns and separates a correct kernel from one
that drops a correction plane by a small factor only.  The per-element ratio does better: over K
random terms both the format error of a correct kernel and the error of a missing plane shrink as
1/sqrt(K), about 20x apart (a float64 emulation of the format gives max ratio * sqrt(K) =
0.9-1.3e-4 for correct planes and 1.9-2.4e-3 with the activation copy plane zeroed, at every shape
below).  tau(K) = TAU_SQRT_K / sqrt(K) sits between the two; the measured figures are in
DESIGN.md."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import util
from tests.test_gpu_tri_path import _filled

pytestmark = pytest.mark.gpu

TAU_SQRT_K = 4.0e-4


def tau(K):
    return TAU_SQRT_K / math.sqrt(K)


def _linear_case(M, K, N, seed, relu_x=True, bias=True):
    torch.manual_seed(seed)
    x = torch.randn(M, K, device="cuda")
    x = torch.relu(x) if relu_x else x
    w = torch.randn(N, K, device="cuda") / K ** 0.5
    b = torch.randn(N, device="cuda") * 0.5 if bias else None
    ref = x.double() @ w.double().t() + (b.double() if bias else 0.0)
    mag = x.double().abs() @ w.double().abs().t() + (b.double().abs() if bias else 0.0)
    return x, w, b, ref, mag


def _conv_case(B, H, W, Cin, Cout, seed, relu_x=True, bias=True):
    torch.manual_seed(seed)
    x = torch.randn(B, Cin, H, W, device="cuda")
    x = torch.relu(x) if relu_x else x
    w = torch.randn(Cout, Cin, 3, 3, device="cuda") / (9 * Cin) ** 0.5
    b = torch.randn(Cout, device="cuda") * 0.5 if bias else None
    ref = F.conv2d(x.double(), w.double(), b.double() if bias else None, padding=1).permute(0, 2, 3, 1)
    mag = F.conv2d(x.double().abs(), w.double().abs(), b.double().abs() if bias else None,
                   padding=1).permute(0, 2, 3, 1)
    return x.permute(0, 2, 3, 1).contiguous(), w, b, ref, mag


def _ratio(got, ref, mag, out_round):
    """max over elements of (|got - ref| - output rounding)+ / (|X|.|W|^T)."""
    e = ((got.double() - ref).abs() - out_round).clamp_min(0.0)
    return float((e / mag.clamp_min(1e-30)).max())


def _assert_within(got, ref, mag, out_round, K, what):
    r = _ratio(got, ref, mag, out_round)
    print("[tri-gemm] %-44s K=%-6d max|err|/(|X||W|)=%.3e  *sqrt(K)=%.3e  tau=%.3e" % (
        what, K, r, r * math.sqrt(K), tau(K)))
    assert r <= tau(K), "%s: max |err| / (|X||W|) = %.3e > tau = %.3e" % (what, r, tau(K))
    return r


def _relu(t, on):
    return t.clamp_min(0.0) if on else t


# --------------------------------------------------------------------------- split-K, tri operands
@pytest.mark.parametrize("split", [3, 7, 32, 80])
def test_linear_split_k_tri(split):
    """K = 3200 (50 k-steps, a multiple of none of 3, 7, 32); split 80 > k_steps is clamped to 50
    by the host, so the partial planes past the 50th stay as they were (zero)."""
    from mnc_b200 import dense
    M, K, N = 200, 3200, 256
    x, w, b, ref, mag = _linear_case(M, K, N, split)
    xt, wt = dense.tri_from_f32(x), dense.tri_from_f32(w, weight=True)
    part = torch.zeros(split, M, N, device="cuda")
    dense.igemm2(xt.view(1, 1, M, K), 1, 1, M, K, wt, N, 1, out_f32=part, split_k=split, split_stride=M * N)
    if split > K // 64:
        assert float(part[K // 64:].abs().max()) == 0.0
    ref_r = _relu(ref, True)
    exp = dense.exp_for(float(ref_r.abs().max()))
    out = dense.tri_alloc((M, N), "cuda")
    dense.splitk_reduce_tri(part, split, M * N, M, N, out, exp, bias=b, relu=True)
    _assert_within(out.float(), ref_r, mag, util.tri_rounding(ref_r, exp), K, "linear split %d" % split)
    util.check_tri(out, ref_r, exp, tau(K) * mag + util.tri_rounding(ref_r, exp), what="linear split %d" % split)
    # the unsplit launch, tri output, computes the same values up to the order of the fp32 sums
    one = dense.tri_alloc((M, N), "cuda")
    dense.igemm2(xt.view(1, 1, M, K), 1, 1, M, K, wt, N, 1, bias=b, relu=True, out=one, out_exp=exp)
    d = (one.float().double() - out.float().double()).abs()
    assert bool((d <= 2 * tau(K) * mag + 2 * util.tri_rounding(ref_r, exp)).all())


@pytest.mark.parametrize("split", [2, 3, 4])
def test_conv_split_k_tri(split):
    from mnc_b200 import dense
    B, H, W, Cin, Cout = 1, 12, 20, 128, 128
    K = 9 * Cin
    x, w, b, ref, mag = _conv_case(B, H, W, Cin, Cout, 40 + split)
    xt, wt = dense.tri_from_f32(x), dense.conv_weight_to_tri(w)
    M = B * H * W
    part = torch.zeros(split, M, Cout, device="cuda")
    dense.igemm2(xt, B, H, W, Cin, wt, Cout, 9, out_f32=part, split_k=split, split_stride=M * Cout)
    ref_r = _relu(ref, True).reshape(M, Cout)
    exp = dense.exp_for(float(ref_r.max()))
    out = dense.tri_alloc((M, Cout), "cuda")
    dense.splitk_reduce_tri(part, split, M * Cout, M, Cout, out, exp, bias=b, relu=True)
    mag = mag.reshape(M, Cout)
    _assert_within(out.float(), ref_r, mag, util.tri_rounding(ref_r, exp), K, "conv split %d" % split)
    util.check_tri(out, ref_r, exp, tau(K) * mag + util.tri_rounding(ref_r, exp), what="conv split %d" % split)
    one = dense.tri_alloc((B, H, W, Cout), "cuda")
    dense.igemm2(xt, B, H, W, Cin, wt, Cout, 9, bias=b, relu=True, out=one, out_exp=exp)
    d = (one.float().reshape(M, Cout).double() - out.float().double()).abs()
    assert bool((d <= 2 * tau(K) * mag + 2 * util.tri_rounding(ref_r, exp)).all())


# ------------------------------------------------------------------------------------ the fc7 join
def test_fc7_join_two_launches_one_exponent():
    """[fc7_mask | fc7]: two launches write one Tri at out_pix_stride = 2N, out_ch_offset 0 and N,
    with one exponent and one amax slot (engine.py, the 'join' of each stage)."""
    from mnc_b200 import dense
    R, N = 200, 256
    x1, w1, b1, ref1, mag1 = _linear_case(R, N, N, 71)
    x2, w2, b2, ref2, mag2 = _linear_case(R, N, N, 72)
    ref1, ref2 = _relu(ref1, True), _relu(ref2, True)
    exp = dense.exp_for(max(float(ref1.max()), float(ref2.max())))
    join = _filled((R, 2 * N))
    before = join.clone()
    amax = torch.zeros(1, dtype=torch.int32, device="cuda")
    halves = ((x1, w1, b1, N), (x2, w2, b2, 0))
    for i, (x, w, b, off) in enumerate(halves):
        dense.igemm2(dense.tri_from_f32(x).view(1, 1, R, N), 1, 1, R, N, dense.tri_from_f32(w, weight=True), N, 1,
                     bias=b, relu=True, out=join, out_pix_stride=2 * N, out_ch_offset=off, out_exp=exp, amax=amax)
        if i == 0:     # the first launch leaves the other half's bytes alone
            util.check_tri(join, ref1, exp, tau(N) * mag1 + util.tri_rounding(ref1, exp),
                           region=(slice(None), slice(N, 2 * N)), before=before, what="join fc7 only")
    for ref, mag, off, name in ((ref1, mag1, N, "fc7"), (ref2, mag2, 0, "fc7_mask")):
        region = (slice(None), slice(off, off + N))
        _assert_within(join[region].float(), ref, mag, util.tri_rounding(ref, exp), N, "join " + name)
        util.check_tri(join, ref, exp, tau(N) * mag + util.tri_rounding(ref, exp), region=region,
                       what="join " + name)
    got = float(amax.view(torch.float32))
    dec_max = float(join.float().abs().max())
    want = max(float(ref1.abs().max()), float(ref2.abs().max()))
    assert abs(got - want) <= tau(N) * float(torch.cat([mag1, mag2]).max()) + want * 2.0 ** -14
    assert got >= dec_max - dec_max * 2.0 ** -14 - 2.0 ** (-15 - exp)


def test_fc7_join_second_launch_keeps_first_half():
    from mnc_b200 import dense
    R, N = 130, 128
    x, w, b, ref, mag = _linear_case(R, N, N, 81)
    join = _filled((R, 2 * N))
    exp = 6
    dense.igemm2(dense.tri_from_f32(x).view(1, 1, R, N), 1, 1, R, N, dense.tri_from_f32(w, weight=True), N, 1,
                 bias=b, relu=True, out=join, out_pix_stride=2 * N, out_ch_offset=0, out_exp=exp)
    first = join.clone()
    dense.igemm2(dense.tri_from_f32(x).view(1, 1, R, N), 1, 1, R, N, dense.tri_from_f32(w, weight=True), N, 1,
                 bias=b, relu=True, out=join, out_pix_stride=2 * N, out_ch_offset=N, out_exp=exp)
    for a, b_ in ((join.h.view(torch.int16), first.h.view(torch.int16)), (join.l, first.l), (join.c, first.c)):
        assert torch.equal(a[:, :N], b_[:, :N])        # first half unchanged by the second launch
        assert torch.equal(a[:, N:], a[:, :N])         # same operands: same bytes at either offset


# --------------------------------------------------------------------- tri output at Cout tails
@pytest.mark.parametrize("Cout,bias,relu", [(48, True, True), (80, False, True), (144, True, False)])
def test_conv_tri_output_channel_tail(Cout, bias, relu):
    """Cout not a multiple of the tile (BN 64 / 128): TMA clips the channel tail at out_pix_stride
    = Cout + 16, whose 16 padding channels keep their sentinel in all three planes.  relu=False
    with signed inputs gives negative outputs (the sign of the e4m3 planes)."""
    from mnc_b200 import dense
    B, H, W, Cin = 2, 9, 21, 64
    K = 9 * Cin
    x, w, b, ref, mag = _conv_case(B, H, W, Cin, Cout, Cout, relu_x=relu, bias=bias)
    ref = _relu(ref, relu)
    exp = dense.exp_for(float(ref.abs().max()))
    stride = Cout + 16
    out = _filled((B, H, W, stride))
    before = out.clone()
    amax = torch.zeros(1, dtype=torch.int32, device="cuda")
    dense.igemm2(dense.tri_from_f32(x), B, H, W, Cin, dense.conv_weight_to_tri(w), Cout, 9, bias=b, relu=relu,
                 out=out, out_pix_stride=stride, out_exp=exp, amax=amax)
    region = (Ellipsis, slice(0, Cout))
    if not relu:
        assert float(ref.min()) < 0
    _assert_within(out[region].float(), ref, mag, util.tri_rounding(ref, exp), K, "conv tail Cout=%d" % Cout)
    util.check_tri(out, ref, exp, tau(K) * mag + util.tri_rounding(ref, exp), region=region, before=before,
                   what="conv tail Cout=%d" % Cout)
    _check_amax(amax, ref, mag, out[region].float(), exp, K)


@pytest.mark.parametrize("H,W,Cout,relu", [(9, 21, 64, True), (7, 13, 144, False), (1, 1, 128, True)])
def test_conv_tri_pooled_odd(H, W, Cout, relu):
    """Fused 2x2 ceil-mode max pool with tri output (mode 5) on odd H and W: partial windows at the
    edge, into a row wider than Cout."""
    from mnc_b200 import dense
    B, Cin = 2, 64
    K = 9 * Cin
    x, w, b, ref, mag = _conv_case(B, H, W, Cin, Cout, H * W + Cout, relu_x=relu)
    full = _relu(ref, relu).permute(0, 3, 1, 2)
    pooled = F.max_pool2d(full, 2, 2, ceil_mode=True)
    ref_p = pooled.permute(0, 2, 3, 1)
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    stride = Cout + 16
    exp = dense.exp_for(float(ref_p.abs().max()))
    out = _filled((B, Ho, Wo, stride))
    before = out.clone()
    amax = torch.zeros(1, dtype=torch.int32, device="cuda")
    dense.igemm2(dense.tri_from_f32(x), B, H, W, Cin, dense.conv_weight_to_tri(w), Cout, 9, bias=b, relu=relu,
                 out=out, out_pix_stride=stride, pool=True, out_exp=exp, amax=amax)
    region = (Ellipsis, slice(0, Cout))
    # the window maximum of the kernel and of the reference may come from different pixels when two
    # are within the error bound: the bound of every pixel of the window applies
    mag_w = F.max_pool2d(mag.permute(0, 3, 1, 2), 2, 2, ceil_mode=True).permute(0, 2, 3, 1)
    _assert_within(out[region].float(), ref_p, mag_w, util.tri_rounding(ref_p, exp), K, "pooled %dx%d" % (H, W))
    util.check_tri(out, ref_p, exp, tau(K) * mag_w + util.tri_rounding(ref_p, exp), region=region,
                   before=before, what="pooled %dx%d" % (H, W))
    _check_amax(amax, ref_p, mag_w, out[region].float(), exp, K)


def _check_amax(amax, ref, mag, decoded, exp, K, rel_round=2.0 ** -14):
    """amax matches max|ref| within the bound, and is never below max|decoded output| minus one
    output rounding."""
    got = float(amax.view(torch.float32))
    want = float(ref.abs().max())
    assert abs(got - want) <= tau(K) * float(mag.max()) + want * rel_round, (got, want)
    d = float(decoded.abs().max())
    lim = d - d * rel_round - (2.0 ** (-15 - exp) if exp is not None else 0.0)
    assert got >= lim, (got, d)


# ------------------------------------------------------------------------------ amax in all modes
@pytest.mark.parametrize("mode", [0, 1, "1-scalar", 4])
def test_linear_amax_every_output_mode(mode):
    from mnc_b200 import dense
    M, K = 300, 512
    N = 441 if mode == "1-scalar" else 192
    x, w, b, ref, mag = _linear_case(M, K, N, 90 + N, relu_x=False)
    xt, wt = dense.tri_from_f32(x), dense.tri_from_f32(w, weight=True)
    amax = torch.zeros(1, dtype=torch.int32, device="cuda")
    relu = mode == 4
    ref = _relu(ref, relu)
    if mode == 4:
        exp = dense.exp_for(float(ref.abs().max()))
        out = dense.tri_alloc((M, N), "cuda")
        dense.igemm2(xt.view(1, 1, M, K), 1, 1, M, K, wt, N, 1, bias=b, relu=relu, out=out, out_exp=exp, amax=amax)
        got, rnd, e = out.float(), util.tri_rounding(ref, exp), exp
    elif mode == 0:
        # split-bf16 output from tri operands (a valid combination of the general entry point)
        out = torch.zeros(2, M, N, dtype=torch.bfloat16, device="cuda")
        dense.igemm2(xt.view(1, 1, M, K), 1, 1, M, K, wt, N, 1, bias=b, relu=relu, out=out, amax=amax)
        got, rnd, e = dense.merge(out), ref.abs() * 2.0 ** -15, None
    else:
        stride = 448 if N == 441 else N       # 441 at 448: the tail chunk takes scalar stores
        buf = torch.full((M, stride), 7.0, device="cuda")
        dense.igemm2(xt.view(1, 1, M, K), 1, 1, M, K, wt, N, 1, bias=b, relu=relu, out_f32=buf,
                     out_pix_stride=stride, amax=amax)
        assert bool((buf[:, N:] == 7.0).all())
        got, rnd, e = buf[:, :N], ref.abs() * 2.0 ** -23, None
    _assert_within(got, ref, mag, rnd, K, "amax mode %s" % mode)
    _check_amax(amax, ref, mag, got, e, K, rel_round=2.0 ** -14)


# ---------------------------------------------------------------------- the bound finds a defect
@pytest.mark.parametrize("kind", ["linear", "conv"])
def test_bound_detects_zeroed_copy_plane(kind):
    """The same launch with the activation copy plane c zeroed -- a valid input that drops the
    Xc.Wl correction -- must fail the per-element bound that the correct planes pass."""
    from mnc_b200 import dense
    if kind == "linear":
        M, K, N = 256, 1024, 256
        x, w, b, ref, mag = _linear_case(M, K, N, 3)
        xt, wt = dense.tri_from_f32(x), dense.tri_from_f32(w, weight=True)
        shape = (M, N)

        def run(a):
            o = torch.zeros(*shape, device="cuda")
            dense.igemm2(a.view(1, 1, M, K), 1, 1, M, K, wt, N, 1, bias=b, out_f32=o)
            return o
    else:
        B, H, W, Cin, Cout = 1, 16, 32, 128, 128
        K = 9 * Cin
        x, w, b, ref, mag = _conv_case(B, H, W, Cin, Cout, 4)
        xt, wt = dense.tri_from_f32(x), dense.conv_weight_to_tri(w)

        def run(a):
            o = torch.zeros(B, H, W, Cout, device="cuda")
            dense.igemm2(a, B, H, W, Cin, wt, Cout, 9, bias=b, out_f32=o)
            return o
    rnd = ref.abs() * 2.0 ** -23
    good = _assert_within(run(xt), ref, mag, rnd, K, "%s, correct planes" % kind)
    broken = xt.clone()
    broken.c.zero_()
    r = _ratio(run(broken), ref, mag, rnd)
    print("[tri-gemm] %-44s K=%-6d max|err|/(|X||W|)=%.3e  *sqrt(K)=%.3e  tau=%.3e" % (
        kind + ", activation c plane zeroed", K, r, r * math.sqrt(K), tau(K)))
    assert r > tau(K), "zeroed copy plane not detected: %.3e <= tau %.3e" % (r, tau(K))
    assert r > 4 * good

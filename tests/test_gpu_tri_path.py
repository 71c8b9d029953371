"""The tri-plane producers of the default engine (precision mode 1) one by one: every plane of their
outputs against a float64 reference or a bit-exact torch restatement, padding included, and the
head softmax against float64.  An end-to-end comparison cannot see a wrong residual (l) or copy
(c) plane: it costs only ~2^-11 of accuracy in the next GEMM (tests/util.py check_tri)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import util
from tests.test_gpu_roi import _rois

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A


def _filled(shape):
    """Tri buffer whose every byte is SENTINEL."""
    from mnc_b200 import dense
    t = dense.tri_alloc(shape, "cuda")
    for p in (t.h.view(torch.uint8), t.l, t.c):
        p.fill_(SENTINEL)
    return t


def _tri_bits_equal(got, want, what):
    """got / want: Tri; h, l and c bit for bit, except that a zero may carry either sign (fmaxf and
    the ReLU leave the sign of a zero maximum unspecified)."""
    gh, wh = got.h.cpu().view(torch.int16), want.h.cpu().view(torch.int16)
    for name, g, w, zero in (("h", gh, wh, lambda b: (b & 0x7FFF) == 0),
                             ("l", got.l.cpu(), want.l.cpu(), lambda b: (b & 0x7F) == 0),
                             ("c", got.c.cpu(), want.c.cpu(), lambda b: (b & 0x7F) == 0)):
        bad = (g != w) & ~(zero(g) & zero(w))
        assert not bool(bad.any()), "%s: plane %s differs at %d elements, first %s (got %d, want %d)" % (
            what, name, int(bad.sum()), tuple(bad.nonzero()[0].tolist()), int(g[bad][0]), int(w[bad][0]))


# ---------------------------------------------------------------------------------- roi_warp_tri
@pytest.mark.parametrize("sub", [1, 2])
@pytest.mark.parametrize("C,R", [(512, 40), (36, 21)])
def test_roi_warp_tri_planes(sub, C, R):
    """Fused RoI warp (+ 28 -> 14 pool at sub = 2) + 14 -> 7 pool, tri-plane outputs, on the
    edge-case RoIs of test_gpu_roi (whole image, degenerate, off-map, past the edge, round-half,
    malformed) with half of them on batch image 1.  C = 36 (4 mod 8) with odd R puts the 7x7 copy
    plane 4 bytes off an 8-byte boundary: legal for the kernel's 4-byte stores."""
    from oracle import oracle as O
    from mnc_b200 import ops, dense
    rng = np.random.default_rng(C + R + sub)
    H, W = 38, 63
    feat = (np.maximum(rng.normal(size=(2, C, H, W)), 0) * 3).astype(np.float32)
    rois = _rois(R, 5 + sub)
    rois[R // 2:, 0] = 1
    f_nhwc = torch.from_numpy(feat).cuda().permute(0, 2, 3, 1).contiguous()
    exp = dense.exp_for(float(feat.max()))
    o14, o7 = _filled((R + 1, 14, 14, C)), _filled((R + 1, 7, 7, C))
    b14, b7 = o14.clone(), o7.clone()
    ops.roi_warp_tri(f_nhwc, C, H, W, torch.from_numpy(rois).cuda(), sub, o14[:R], o7[:R], exp)
    o14.exp = o7.exp = exp
    want = torch.from_numpy(O.roi_warp(feat, rois, 14 * sub, 14 * sub)).double()
    want14 = F.max_pool2d(want, 2, 2) if sub == 2 else want
    want7 = F.max_pool2d(want14, 2, 2)
    want14, want7 = want14.permute(0, 2, 3, 1), want7.permute(0, 2, 3, 1)
    # the kernel evaluates the bilinear sum with FMAs where the oracle rounds every product: a few
    # fp32 ulp of the largest feature value, on top of the format's own rounding
    fma = 8 * 2.0 ** -24 * float(feat.max())
    for t, w, b, name in ((o14, want14, b14, "out14"), (o7, want7, b7, "out7")):
        util.check_tri(t, w, exp, util.tri_rounding(w, exp) + fma, region=slice(0, R), before=b,
                       what="roi_warp_tri sub=%d %s" % (sub, name))
    assert float(o7.float()[3].abs().max()) == 0.0            # RoI entirely outside the map
    # the split-bf16 instantiation of the same kernel template: both carry the same fp32 value
    s14 = torch.zeros(2, R, 14, 14, C, dtype=torch.bfloat16, device="cuda")
    s7 = torch.zeros(2, R, 7, 7, C, dtype=torch.bfloat16, device="cuda")
    ops.roi_warp_split(f_nhwc, C, H, W, torch.from_numpy(rois).cuda(), sub, s14, s7)
    for t, s in ((o14, s14), (o7, s7)):
        sv = dense.merge(s).double().cpu()
        tv = t.float()[:R].double().cpu()
        assert bool(((tv - sv).abs() <= util.tri_rounding(sv, exp) + sv.abs() * 2.0 ** -16).all())


# --------------------------------------------------------------------------------- mask_pool_tri
def _mask_pool_tri_expected(feat14, mask14):
    """torch float32 restatement: decode h + l/64 (exact), multiply (round to nearest, as
    __fmul_rn), 2x2 max, repack at scale 1 (the input's exponent carries over)."""
    from mnc_b200 import dense
    dec = feat14.h.float() + feat14.l.view(torch.float8_e4m3fn).float() * (1.0 / 64.0)   # [R,14,14,C]
    prod = dec * mask14.view(-1, 14, 14, 1)
    best = F.max_pool2d(prod.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1).contiguous()
    return dense.tri_from_f32(best, exp=0)


@pytest.mark.parametrize("C", [512, 68])
def test_mask_pool_tri_bit_exact(C):
    from mnc_b200 import ops, dense
    torch.manual_seed(C)
    R = 23
    logits = torch.randn(R, 448, device="cuda") * 3
    _, m14 = ops.sigmoid_mask_resize(logits, R)
    m14 = m14.clone()
    m14[0] = 0.0                       # mask exactly 0: every product is a (signed) zero
    m14[1] = 1.0                       # exactly 1: the decoded value itself
    m14[2, :, :7] = 0.0
    m14[2, :, 7:] = 1.0
    x = torch.randn(R, 14, 14, C, device="cuda") * 5          # negative features included
    x[3] = -x[3].abs()                                         # a RoI with no positive value
    exp = dense.exp_for(float(x.abs().max()))
    f14 = dense.tri_from_f32(x, exp=exp)
    out = _filled((R + 1, 7, 7, C))
    before = out.clone()
    written = out[:R]
    ops.mask_pool_tri(f14, m14, R, C, written)
    assert written.exp == exp                 # the output takes the input's exponent
    want = _mask_pool_tri_expected(f14, m14)
    _tri_bits_equal(written, want, "mask_pool_tri")
    for p, q in ((out.h.view(torch.uint8), before.h.view(torch.uint8)), (out.l, before.l), (out.c, before.c)):
        assert torch.equal(p[R:], q[R:])
    # and as a value: the fp64 product of the decoded input, within the format's rounding
    ref = F.max_pool2d((f14.float().double() * m14.view(-1, 14, 14, 1).double()).permute(0, 3, 1, 2), 2, 2)
    ref = ref.permute(0, 2, 3, 1)
    out.exp = exp
    util.check_tri(out, ref, exp, util.tri_rounding(ref, exp) + ref.abs() * 2.0 ** -24, region=slice(0, R),
                   before=before, what="mask_pool_tri")


# ----------------------------------------------------------------------------- splitk_reduce_tri
def _splitk_expected(part, splits, bias, relu):
    acc = torch.zeros_like(part[0])
    for s in range(splits):
        acc = acc + part[s]
    if bias is not None:
        acc = acc + bias
    if relu:
        acc = acc.clamp_min(0.0)
    return acc


@pytest.mark.parametrize("splits", [1, 2, 7, 32])
@pytest.mark.parametrize("bias_on,relu,stride_pad,offset", [(True, True, 0, 0), (False, True, 24, 8),
                                                            (True, False, 40, 16), (False, False, 4, 4)])
def test_splitk_reduce_tri_bit_exact(splits, bias_on, relu, stride_pad, offset):
    """sum over s = 0..splits-1 in fp32, then + bias, then ReLU, packed at 2^exp: every plane bit
    for bit; rows written at out_ch_offset inside a wider row, sentinels around the region."""
    from mnc_b200 import dense
    torch.manual_seed(splits * 100 + stride_pad)
    rows, cols = 77, 96
    part = torch.randn(splits, rows, cols, device="cuda") * 4
    bias = torch.randn(cols, device="cuda") * 3 if bias_on else None
    acc = _splitk_expected(part, splits, bias, relu)
    exp = dense.exp_for(float(acc.abs().max()))
    stride = offset + cols + stride_pad
    out = _filled((rows, stride))
    before = out.clone()
    dense.splitk_reduce_tri(part, splits, rows * cols, rows, cols, out, exp, bias=bias, relu=relu, out_row_stride=stride, out_ch_offset=offset)
    region = (slice(None), slice(offset, offset + cols))
    want = dense.tri_from_f32(acc, exp=exp)
    _tri_bits_equal(out[region], want, "splitk_reduce_tri")
    ref = part.double().sum(0) + (bias.double() if bias_on else 0.0)
    ref = ref.clamp_min(0.0) if relu else ref
    util.check_tri(out, ref, exp, util.tri_rounding(ref, exp) + splits * 2.0 ** -23 * part.abs().sum(0).double()
                   .add(bias.abs().double() if bias_on else 0.0), region=region, before=before,
                   what="splitk_reduce_tri")


@pytest.mark.parametrize("prior", [0.0, "larger"])
def test_splitk_reduce_tri_amax(prior):
    """amax is an atomicMax of |output| as float bits: exact, and a larger prior value stays."""
    from mnc_b200 import dense
    torch.manual_seed(5)
    splits, rows, cols = 3, 129, 64
    part = torch.randn(splits, rows, cols, device="cuda")
    bias = torch.randn(cols, device="cuda")
    acc = _splitk_expected(part, splits, bias, False)
    m = float(acc.abs().max())
    start = 0.0 if prior == 0.0 else 2.0 * m
    amax = torch.tensor([start], dtype=torch.float32, device="cuda").view(torch.int32)
    out = dense.tri_alloc((rows, cols), "cuda")
    dense.splitk_reduce_tri(part, splits, rows * cols, rows, cols, out, 3, bias=bias, relu=False, amax=amax)
    got = float(amax.view(torch.float32))
    assert got == (m if prior == 0.0 else start)


# ---------------------------------------------------------------------------------- softmax_rows
@pytest.mark.parametrize("rows", [1, 7, 130])
@pytest.mark.parametrize("cols", [1, 21, 32, 33, 64])
def test_softmax_rows_against_f64(rows, cols):
    """Row softmax from strided column slices of a 128-wide buffer (the engine's heads[:, 0:21] and
    heads[:, 21:42]) into an output wider than cols.  Bound per element, in fp32 ulp of the
    reference: 2 (expf) + 1 (division) + |x - max| (rounding of the subtraction, amplified by exp)
    + cols (the fp32 sum of the denominator)."""
    from mnc_b200 import ops
    torch.manual_seed(rows * 64 + cols)
    heads = torch.randn(rows, 128, device="cuda") * 4
    if rows >= 7:
        heads[1, :] = 0.0                               # all equal
        heads[2, cols // 2] = 60.0                      # one dominant logit
        heads[3, :] += 1e4
        heads[4, :] -= 1e4
        heads[5, cols // 3:] += 1e4                     # shift inside the row
    for c0 in (0, 21):
        if c0 + cols > 128:
            continue
        x = heads[:, c0:c0 + cols]
        buf = torch.full((rows, cols + 7), -1.0, device="cuda")
        got = ops.softmax_rows(x, cols, out=buf[:, :cols])
        assert got.data_ptr() == buf.data_ptr()
        x64 = x.double().cpu()
        d = x64 - x64.max(1, keepdim=True).values
        ref = torch.exp(d) / torch.exp(d).sum(1, keepdim=True)
        tol = (3.0 + d.abs() + cols) * 2.0 ** -24 * ref + 2.0 ** -126   # (no claim below fp32's normal range)
        err = (buf[:, :cols].double().cpu() - ref).abs()
        assert bool((err <= tol).all()), "cols %d offset %d: worst err/tol %.3g" % (cols, c0, float((err / tol).max()))
        assert bool((buf[:, cols:] == -1.0).all())      # the output row's tail is untouched


def test_softmax_rows_default_output_and_arg_errors():
    from mnc_b200 import ops
    from mnc_b200._lib import lib, ptr, cur_stream
    heads = torch.randn(9, 128, device="cuda")
    got = ops.softmax_rows(heads[:, 21:42], 21)
    assert got.shape == (9, 21) and got.is_contiguous()
    ref = torch.softmax(heads[:, 21:42].double(), 1)
    assert float((got.double() - ref).abs().max()) < 1e-6
    out = torch.empty(9, 128, device="cuda")
    for cols in (0, 65):
        rc = lib.mnc_softmax_rows(ptr(heads), 128, 9, cols, ptr(out), 128, cur_stream())
        assert rc == 1, "cols = %d: rc %d, expected MNC_ERR_ARG" % (cols, rc)


# ------------------------------------------------------------------- plane alignment of the entries
def test_tri_entry_points_reject_misaligned_planes():
    """splitk_reduce_tri, roi_warp_tri and mask_pool_tri store 8 bytes of h and 4 of l / c at a
    time: a plane pointer off that alignment is MNC_ERR_ARG, checked before any launch."""
    from mnc_b200 import ops, dense
    from mnc_b200._lib import MncError

    def shifted(t, plane, nbytes):
        """t with one plane starting nbytes later (same buffer, so the data stay in bounds)."""
        h, l, c = t.h, t.l, t.c
        if plane == "h":
            h = t.h.view(-1).view(torch.uint8)[nbytes:nbytes + 2 * (t.h.numel() - 8)].view(torch.float16)
        elif plane == "l":
            l = t.l.view(-1)[nbytes:nbytes + t.l.numel() - 8]
        else:
            c = t.c.view(-1)[nbytes:nbytes + t.c.numel() - 8]
        return dense.Tri(h, l, c, t.exp)

    rows, cols = 8, 64
    part = torch.randn(2, rows, cols, device="cuda")
    R, C = 3, 64
    feat = torch.rand(1, 10, 12, C, device="cuda")
    rois = torch.tensor([[0, 0, 0, 150, 100]] * R, dtype=torch.float32, device="cuda")
    f14 = dense.tri_from_f32(torch.rand(R, 14, 14, C, device="cuda"))
    m14 = torch.rand(R, 1, 14, 14, device="cuda")
    for plane, nb in (("h", 2), ("h", 4), ("l", 1), ("l", 2), ("c", 1), ("c", 3)):
        out = dense.tri_alloc((rows * cols + 8,), "cuda")
        with pytest.raises(MncError, match="MNC_ERR_ARG"):
            dense.splitk_reduce_tri(part, 2, rows * cols, rows, cols, shifted(out, plane, nb), 0)
        o14 = dense.tri_alloc((R * 196 * C + 8,), "cuda")
        o7 = dense.tri_alloc((R * 49 * C + 8,), "cuda")
        with pytest.raises(MncError, match="MNC_ERR_ARG"):
            ops.roi_warp_tri(feat, C, 10, 12, rois, 1, shifted(o14, plane, nb), o7, 0)
        with pytest.raises(MncError, match="MNC_ERR_ARG"):
            ops.roi_warp_tri(feat, C, 10, 12, rois, 2, o14, shifted(o7, plane, nb), 0)
        with pytest.raises(MncError, match="MNC_ERR_ARG"):
            ops.mask_pool_tri(f14, m14, R, C, shifted(o7, plane, nb))
        if plane != "c":           # mask_pool_tri reads h and l of its input
            with pytest.raises(MncError, match="MNC_ERR_ARG"):
                ops.mask_pool_tri(shifted(dense.tri_from_f32(torch.rand(R * 196 * C + 8, device="cuda")),
                                          plane, nb), m14, R, C, o7)
    # 4-byte aligned e4m3 planes (not 8) are legal: the stores are 4 bytes wide
    out = dense.tri_alloc((rows * cols + 8,), "cuda")
    ok = dense.Tri(out.h, out.l.view(-1)[4:4 + rows * cols], out.c.view(-1)[4:4 + rows * cols], 0)
    dense.splitk_reduce_tri(part, 2, rows * cols, rows, cols, ok, 0)
    torch.cuda.synchronize()

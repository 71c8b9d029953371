"""util.check_tri, the tri-plane format checker of the precision-mode-1 GPU tests, on the CPU: it
accepts the torch restatement dense.tri_from_f32 on adversarial values and rejects every single
defect a producer kernel could have in one of the three planes."""
import pytest
import torch

from mnc_b200 import dense
from tests import util


def _adversarial(exp):
    """fp32 values whose scaled form xs = x * 2^exp covers the format's edge cases."""
    s = 2.0 ** -exp
    vals = [0.0, -0.0, 1.0, -1.0, 4096.0, -4096.0, 3.0, 0.1, -0.7, 65504.0, -65504.0]
    f16_sub = [2.0 ** -24, 3 * 2.0 ** -24, 2.0 ** -15 + 2.0 ** -22, -(2.0 ** -14 - 2.0 ** -24)]
    e4m3_sub = [2.0 ** -10 * 32, 2.0 ** -9 * 32, 5 * 2.0 ** -9 * 32, -(2.0 ** -7) * 32]
    edges = []
    for e in range(-14, 16):                   # fp16 binade edges, from both sides
        p = 2.0 ** e
        edges += [p, -p, p * (1 - 2.0 ** -12), p * (1 + 2.0 ** -11), p * (1 - 2.0 ** -13),
                  p * (1 + 2.0 ** -12)]
    mids = []
    for e in range(-6, 8):                     # exact e4m3 midpoints of xs / 32
        for m in range(8):
            mid = 2.0 ** e * (1 + (2 * m + 1) / 16.0) * 32.0
            mids += [mid, -mid, mid * (1 + 2.0 ** -20)]
    sat = [2.0 ** 14 + 7.5, 2.0 ** 14 * 1.7, 30000.5, 65519.0, 7e4, -1e5]
    rng = torch.Generator().manual_seed(0)
    rnd = torch.randn(4000, generator=rng) * torch.exp2(torch.randint(-12, 14, (4000,), generator=rng).float())
    xs = torch.tensor(vals + f16_sub + e4m3_sub + edges + mids + sat, dtype=torch.float32)
    xs = torch.cat([xs, rnd])
    xs = xs[: xs.numel() // 8 * 8]
    return (xs.double() * s).float()


def _bound(x, t):
    """format rounding, plus the saturation the caller allows for: |x * 2^exp| > 65504 clamps."""
    b = util.tri_rounding(x.double(), t.exp)
    return torch.where(x.double().abs() * 2.0 ** t.exp > 65504.0, torch.full_like(b, float("inf")), b)


@pytest.mark.parametrize("exp", [0, 7, -9])
def test_checker_accepts_restatement(exp):
    x = _adversarial(exp).view(-1, 8)
    t = dense.tri_from_f32(x, exp=exp)
    util.check_tri(t, x.double(), exp, _bound(x, t))


def test_checker_accepts_scaled_random_and_padding():
    torch.manual_seed(1)
    x = torch.relu(torch.randn(37, 48)) * 3
    exp = dense.exp_for(float(x.abs().max()))
    full = dense.tri_alloc((37, 64), "cpu")
    for p in (full.h.view(torch.int16), full.l, full.c):
        p.fill_(0x5A)
    before = full.clone()
    part = dense.tri_from_f32(x, exp=exp)
    full.h[:, 8:56] = part.h
    full.l[:, 8:56] = part.l
    full.c[:, 8:56] = part.c
    full.exp = exp
    util.check_tri(full, x.double(), exp, util.tri_rounding(x.double(), exp), region=(slice(None), slice(8, 56)),
                   before=before)


def _mutations():
    def zero_c(t): t.c.zero_()
    def zero_l(t): t.l.zero_()
    def swap_lc(t): t.l[:], t.c[:] = t.c.clone(), t.l.clone()
    def shift_c(t): t.c[:] = torch.roll(t.c, 1, dims=-1)
    def flip_c(t): t.c ^= 0x80
    def h_ulp(t): t.h.view(torch.int16)[:] += 1
    return [zero_c, zero_l, swap_lc, shift_c, flip_c, h_ulp]


@pytest.mark.parametrize("mutate", _mutations(), ids=lambda f: f.__name__)
@pytest.mark.parametrize("signed", [False, True])
def test_checker_rejects_plane_mutation(mutate, signed):
    torch.manual_seed(2)
    x = torch.randn(64, 96)
    x = x if signed else torch.relu(x)
    exp = dense.exp_for(float(x.abs().max()))
    t = dense.tri_from_f32(x, exp=exp)
    util.check_tri(t, x.double(), exp, util.tri_rounding(x.double(), exp))
    mutate(t)
    with pytest.raises(AssertionError):
        util.check_tri(t, x.double(), exp, util.tri_rounding(x.double(), exp))


@pytest.mark.parametrize("plane", ["h", "l", "c"])
def test_checker_rejects_padding_write(plane):
    torch.manual_seed(3)
    x = torch.randn(16, 32)
    exp = dense.exp_for(float(x.abs().max()))
    full = dense.tri_alloc((16, 48), "cpu")
    for p in (full.h.view(torch.int16), full.l, full.c):
        p.fill_(0x3C)
    before = full.clone()
    part = dense.tri_from_f32(x, exp=exp)
    full.h[:, :32], full.l[:, :32], full.c[:, :32] = part.h, part.l, part.c
    full.exp = exp
    region = (slice(None), slice(0, 32))
    util.check_tri(full, x.double(), exp, util.tri_rounding(x.double(), exp), region=region, before=before)
    getattr(full, plane).view(torch.uint8)[5, -1] ^= 1      # one byte of one padding element
    with pytest.raises(AssertionError, match="padding"):
        util.check_tri(full, x.double(), exp, util.tri_rounding(x.double(), exp), region=region, before=before)


def test_checker_rejects_wrong_exponent_and_single_element_defects():
    torch.manual_seed(4)
    x = torch.relu(torch.randn(32, 64)) + 0.5
    exp = dense.exp_for(float(x.abs().max()))
    bound = util.tri_rounding(x.double(), exp)
    t = dense.tri_from_f32(x, exp=exp)
    with pytest.raises(AssertionError, match="exponent"):
        util.check_tri(t, x.double(), exp + 1, bound)
    # one element at a time: the residual set to 448 (more than half an fp16 ulp below 2^14), the
    # copy one e4m3 step off
    for plane, byte in (("l", 0x7E), ("c", int(t.c[7, 9]) + 1)):
        m = t.clone()
        getattr(m, plane)[7, 9] = byte
        with pytest.raises(AssertionError):
            util.check_tri(m, x.double(), exp, bound)

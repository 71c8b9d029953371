"""The implicit-GEMM persistent scheduler: the output must not depend on how many CTAs share the
tiles.  With max_ctas = 1 one CTA runs every tile, so its operand ring (3 stages at BN = 64, 2 at
BN = 128) wraps at every phase across tile boundaries, with k-step counts of 1, 2, 3 and 5; with 2
and 5 CTAs the tiles interleave.  Every output plane must equal the default grid's bit for bit, in
both precision modes.  Shapes stay small so that the 1-CTA launches take milliseconds."""
import pytest
import torch

pytestmark = pytest.mark.gpu

CTAS = (1, 2, 5)


def _planes(out):
    from mnc_b200 import dense
    if isinstance(out, dense.Tri):
        return [out.h.view(torch.int16), out.l, out.c]
    return [out.view(torch.int16)] if out.dtype == torch.bfloat16 else [out.view(torch.int32)]


def _operands(precision, x, w, conv):
    from mnc_b200 import dense
    if precision == "f16f8":
        return dense.tri_from_f32(x), (dense.conv_weight_to_tri(w) if conv else dense.tri_from_f32(w, weight=True))
    return dense.split(x), (dense.conv_weight_to_split(w) if conv else dense.split(w))


def _out(precision, shape):
    from mnc_b200 import dense
    if precision == "f16f8":
        return dense.tri_alloc(shape, "cuda")
    return torch.zeros((2,) + tuple(shape), dtype=torch.bfloat16, device="cuda")


def _same(runs, what):
    base = _planes(runs[0])
    for n, o in zip(CTAS, runs[1:]):
        for i, (a, b) in enumerate(zip(base, _planes(o))):
            assert torch.equal(a, b), "%s: plane %d differs with max_ctas=%d" % (what, i, n)


@pytest.mark.parametrize("precision", ["f16f8", "bf16x3"])
@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("K", [64, 128, 192, 320])
@pytest.mark.parametrize("M", [100, 257])
def test_linear_tile_loop_invariance(precision, bn, K, M):
    from mnc_b200 import dense
    torch.manual_seed(K + M + bn)
    N = 256
    x = torch.relu(torch.randn(M, K, device="cuda"))
    w = torch.randn(N, K, device="cuda") / K ** 0.5
    b = torch.randn(N, device="cuda")
    a, wt = _operands(precision, x, w, False)
    a4 = a.view(1, 1, M, K) if precision == "f16f8" else a.view(2, 1, 1, M, K)
    runs = []
    for n in (0,) + CTAS:
        o = _out(precision, (M, N))
        dense.igemm2(a4, 1, 1, M, K, wt, N, 1, bias=b, relu=True, out=o, bn=bn, max_ctas=n, out_exp=4)
        runs.append(o)
    _same(runs, "linear M=%d K=%d bn=%d %s" % (M, K, bn, precision))
    # split-K fp32 partials go through the same tile loop (work items = tiles x splits)
    runs = []
    for n in (0,) + CTAS:
        part = torch.zeros(2, M, N, device="cuda")
        dense.igemm2(a4, 1, 1, M, K, wt, N, 1, out_f32=part, split_k=2, split_stride=M * N, bn=bn, max_ctas=n)
        runs.append(part)
    _same(runs, "linear split-K M=%d K=%d bn=%d %s" % (M, K, bn, precision))


@pytest.mark.parametrize("precision", ["f16f8", "bf16x3"])
@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("Cin", [64, 128])
def test_conv_tile_loop_invariance(precision, bn, Cin):
    """9 or 18 k-steps per tile; 2 x 3 spatial tiles (ragged in H and W) x 2 or 1 channel tiles;
    plain and pooled epilogues."""
    from mnc_b200 import dense
    torch.manual_seed(Cin + bn)
    B, H, W, Cout = 1, 11, 37, 128
    x = torch.relu(torch.randn(B, Cin, H, W, device="cuda")).permute(0, 2, 3, 1).contiguous()
    w = torch.randn(Cout, Cin, 3, 3, device="cuda") / (9 * Cin) ** 0.5
    b = torch.randn(Cout, device="cuda")
    a, wt = _operands(precision, x, w, True)
    for pool in (False, True):
        shape = (B, (H + 1) // 2, (W + 1) // 2, Cout) if pool else (B, H, W, Cout)
        runs = []
        for n in (0,) + CTAS:
            o = _out(precision, shape)
            dense.igemm2(a, B, H, W, Cin, wt, Cout, 9, bias=b, relu=True, out=o, bn=bn, max_ctas=n,
                         pool=pool, out_exp=4)
            runs.append(o)
        _same(runs, "conv Cin=%d bn=%d pool=%s %s" % (Cin, bn, pool, precision))

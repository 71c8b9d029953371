"""Edge cases of the implicit-GEMM epilogue not covered elsewhere: conv tiles whose last tile row
holds only 2..4 image rows (H % 8 in 2..4, the rows of the second consumer warpgroup all outside
the image), the fused 2x2 pool on odd W with split-bf16 output (mode 2), and channel tails of the
split-bf16 (mode 0) and fp32 (mode 1) outputs.  Tri-plane operands; every result is
checked against the fp64 product with the tau(K) bound of test_gpu_tri_gemm, and every byte
outside the written region must keep its sentinel."""
import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_tri_gemm import _assert_within, _conv_case, _linear_case, _relu, tau  # noqa: F401

pytestmark = pytest.mark.gpu

SENTINEL_BF16 = -12288.0   # exactly representable in bf16 (-3 * 2^12)


def _split_filled(shape):
    return torch.full((2,) + tuple(shape), SENTINEL_BF16, dtype=torch.bfloat16, device="cuda")


def _split_value(out):
    return out[0].double() + out[1].double()


def _untouched(out, region):
    mask = torch.ones(out.shape[1:], dtype=torch.bool, device=out.device)
    mask[region] = False
    for p in range(out.shape[0]):
        assert bool((out[p][mask].float() == SENTINEL_BF16).all()), "plane %d written outside the region" % p


@pytest.mark.parametrize("H,Cout,bn", [(10, 64, 64), (11, 96, 128), (12, 80, 0), (4, 128, 128)])
def test_conv_split_out_ragged_tile_rows(H, Cout, bn):
    """Mode 0 (split bf16 via TMA store) on H % 8 in {2, 3, 4}: TMA clips the last tile row to the
    image; Cout tails at BN 64 and 128."""
    from mnc_b200 import dense
    B, W, Cin = 2, 19, 64
    K = 9 * Cin
    x, w, b, ref, mag = _conv_case(B, H, W, Cin, Cout, 100 + H)
    ref = _relu(ref, True)
    stride = Cout + 8
    out = _split_filled((B, H, W, stride))
    dense.igemm2(dense.tri_from_f32(x), B, H, W, Cin, dense.conv_weight_to_tri(w), Cout, 9, bias=b, relu=True,
                 out=out, out_pix_stride=stride, bn=bn)
    region = (Ellipsis, slice(0, Cout))
    got = _split_value(out)[region]
    _assert_within(got, ref, mag, ref.abs() * 2.0 ** -16, K, "conv split H=%d Cout=%d" % (H, Cout))
    _untouched(out, region)


@pytest.mark.parametrize("H,W,Cout,relu", [(6, 13, 64, True), (9, 27, 136, False), (3, 17, 128, True)])
def test_conv_split_pooled_odd_width(H, W, Cout, relu):
    """Mode 2 (fused 2x2 ceil-mode max pool, split-bf16 output) on odd W: the right-most window of
    a row has one pixel, its neighbour column lies outside the image."""
    from mnc_b200 import dense
    B, Cin = 2, 64
    K = 9 * Cin
    x, w, b, ref, mag = _conv_case(B, H, W, Cin, Cout, 200 + W, relu_x=relu)
    full = _relu(ref, relu).permute(0, 3, 1, 2)
    ref_p = F.max_pool2d(full, 2, 2, ceil_mode=True).permute(0, 2, 3, 1)
    mag_w = F.max_pool2d(mag.permute(0, 3, 1, 2), 2, 2, ceil_mode=True).permute(0, 2, 3, 1)
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    stride = Cout + 8
    out = _split_filled((B, Ho, Wo, stride))
    dense.igemm2(dense.tri_from_f32(x), B, H, W, Cin, dense.conv_weight_to_tri(w), Cout, 9, bias=b, relu=relu,
                 out=out, out_pix_stride=stride, pool=True)
    region = (Ellipsis, slice(0, Cout))
    _assert_within(_split_value(out)[region], ref_p, mag_w, ref_p.abs() * 2.0 ** -16, K,
                   "pooled split %dx%d" % (H, W))
    _untouched(out, region)


@pytest.mark.parametrize("M,N,bn", [(200, 84, 128), (130, 21, 64), (64, 150, 0)])
def test_linear_fp32_out_channel_tail(M, N, bn):
    """Mode 1 (fp32, stored directly) with N not a multiple of the tile and odd N, into rows wider
    than N (unaligned rows: the per-element stores)."""
    from mnc_b200 import dense
    K = 512
    x, w, b, ref, mag = _linear_case(M, K, N, 300 + N)
    stride = N + 5
    out = torch.full((M, stride), SENTINEL_BF16, dtype=torch.float32, device="cuda")
    dense.igemm2(dense.tri_from_f32(x).view(1, 1, M, K), 1, 1, M, K, dense.tri_from_f32(w, weight=True), N, 1,
                 bias=b, out_f32=out, out_pix_stride=stride, bn=bn)
    _assert_within(out[:, :N], ref, mag, 0.0, K, "linear fp32 N=%d" % N)
    assert bool((out[:, N:] == SENTINEL_BF16).all()), "fp32 row padding written"


@pytest.mark.parametrize("M,N", [(200, 84), (72, 200)])
def test_linear_split_out_channel_tail(M, N):
    """Mode 0 (split bf16) of a linear layer: ragged pixel tile (M not a multiple of 128) and a
    channel tail, through the direct stores (row stride not a multiple of 8, N = 84) and through
    the TMA store (N = 200)."""
    from mnc_b200 import dense
    K = 512
    x, w, b, ref, mag = _linear_case(M, K, N, 400 + N)
    ref = _relu(ref, True)
    stride = N + 8
    out = _split_filled((M, stride))
    dense.igemm2(dense.tri_from_f32(x).view(1, 1, M, K), 1, 1, M, K, dense.tri_from_f32(w, weight=True), N, 1,
                 bias=b, relu=True, out=out, out_pix_stride=stride)
    region = (Ellipsis, slice(0, N))
    _assert_within(_split_value(out)[region], ref, mag, ref.abs() * 2.0 ** -16, K, "linear split N=%d" % N)
    _untouched(out, region)

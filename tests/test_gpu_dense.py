"""Tensor-core implicit GEMM (conv / inner product), conv1_1, pooling vs fp64 / torch references.
Tolerance: the split-bf16 3-product scheme carries ~16 mantissa bits; 1e-4 relative to the output
range is asserted here (north_star allows 1e-3 end to end)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def relerr(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


@pytest.mark.parametrize("M,K,N,bn,split", [(128, 64, 64, 64, 1), (300, 256, 441, 0, 1),
                                            (2394, 512, 54, 64, 1), (300, 12544, 64, 64, 7),
                                            (600, 8192, 126, 128, 4), (1000, 4096, 4096, 128, 1),
                                            (257, 3136, 256, 256, 1), (2400, 1024, 1100, 192, 1),
                                            (300, 512, 441, 192, 1)])
def test_inner_product(M, K, N, bn, split):
    from mnc_b200 import dense
    torch.manual_seed(M + N)
    x = torch.randn(M, K, device="cuda")
    w = torch.randn(N, K, device="cuda") / K ** 0.5
    b = torch.randn(N, device="cuda")
    xs, ws = dense.split(x), dense.split(w)
    # reference from the ORIGINAL fp32 operands (so the 2^-17 operand-split error is inside the
    # tolerance being asserted), and from the split-rounded ones for the exact-arithmetic SIMT check
    ref = (x.double() @ w.double().t() + b.double()).clamp_min(0)
    ref_q = (dense.merge(xs).double() @ dense.merge(ws).double().t() + b.double()).clamp_min(0)
    stride = ((N + 7) // 8) * 8
    if split > 1:
        part = torch.zeros(split, M, N, device="cuda")
        dense.igemm(xs.view(2, 1, 1, M, K), 1, 1, M, K, ws, N, 1, out_f32=part, split_k=split,
                    split_stride=M * N, bn=bn)
        out = torch.zeros(2, M, stride, device="cuda", dtype=torch.bfloat16)
        dense.splitk_reduce(part, split, M * N, M, N, bias=b, relu=True, out=out, out_row_stride=stride)
    else:
        out = torch.zeros(2, M, stride, device="cuda", dtype=torch.bfloat16)
        dense.igemm(xs.view(2, 1, 1, M, K), 1, 1, M, K, ws, N, 1, bias=b, relu=True, out=out,
                    out_pix_stride=stride, bn=bn)
    got = dense.merge(out)[:, :N]
    assert relerr(got, ref) < 1e-4
    if stride > N:
        assert float(dense.merge(out)[:, N:].abs().max()) == 0.0  # padding columns untouched
    # on-device cross-check: SIMT fp32 path on the same operands
    chk = torch.zeros(M, N, device="cuda")
    dense.igemm(xs.view(2, 1, 1, M, K), 1, 1, M, K, ws, N, 1, bias=b, relu=True, out_f32=chk, impl="simt")
    assert relerr(chk, ref_q) < 1e-5
    # precision mode 1 (fp16 + 2 x FP8, tri-plane operands) on the same layer, fp32 out
    if split == 1:
        xt, wt = dense.tri_from_f32(x), dense.tri_from_f32(w, weight=True)
        o1 = torch.zeros(M, N, device="cuda")
        dense.igemm2(xt.view(1, 1, M, K), 1, 1, M, K, wt, N, 1, bias=b, relu=True, out_f32=o1, bn=bn)
        assert relerr(o1, ref) < 1e-4


@pytest.mark.parametrize("B,H,W,Cin,Cout,bn", [(1, 8, 16, 64, 64, 64), (2, 38, 63, 128, 256, 0),
                                               (1, 75, 125, 64, 128, 128), (1, 19, 33, 512, 512, 256),
                                               (3, 5, 7, 64, 64, 64)])
def test_conv3x3(B, H, W, Cin, Cout, bn):
    """vs the naive reference the way Caffe's own conv test does (test_convolution_layer.cpp:231-263,
    1e-4): zero padding, bias, ReLU, ragged tiles (H, W not multiples of the 8x16 pixel tile)."""
    from mnc_b200 import dense
    torch.manual_seed(H * W)
    x = torch.randn(B, Cin, H, W, device="cuda")
    w = torch.randn(Cout, Cin, 3, 3, device="cuda") / (9 * Cin) ** 0.5
    b = torch.randn(Cout, device="cuda")
    xs = dense.split(x.permute(0, 2, 3, 1).contiguous())
    ws = dense.conv_weight_to_split(w)
    # reference from the ORIGINAL fp32 operands: the operand-split error is inside the tolerance
    ref = torch.nn.functional.conv2d(x.double(), w.double(), b.double(), padding=1).clamp_min(0).permute(0, 2, 3, 1)
    out = torch.zeros(2, B, H, W, Cout, device="cuda", dtype=torch.bfloat16)
    dense.igemm(xs, B, H, W, Cin, ws, Cout, 9, bias=b, relu=True, out=out, bn=bn)
    assert relerr(dense.merge(out), ref) < 1e-4
    # precision mode 1 on the same layer tri-plane in and out
    xt, wt = dense.tri_from_f32(x.permute(0, 2, 3, 1).contiguous()), dense.conv_weight_to_tri(w)
    ot = dense.tri_alloc((B, H, W, Cout), "cuda")
    dense.igemm2(xt, B, H, W, Cin, wt, Cout, 9, bias=b, relu=True, out=ot,
                 out_exp=dense.exp_for(float(ref.max())), bn=bn)
    assert relerr(ot.float(), ref) < 1e-4


def test_conv1_1_and_pool_and_layout():
    import torch.nn.functional as F
    from mnc_b200 import dense
    torch.manual_seed(0)
    B, H, W = 2, 37, 53
    data = torch.randn(B, 3, H, W, device="cuda") * 70
    w = torch.randn(64, 3, 3, 3, device="cuda") * 0.01
    b = torch.randn(64, device="cuda")
    out = torch.zeros(2, B, H, W, 64, device="cuda", dtype=torch.bfloat16)
    dense.conv1_1(data, w, b, out)
    ref = F.relu(F.conv2d(data.double(), w.double(), b.double(), padding=1)).permute(0, 2, 3, 1)
    assert relerr(dense.merge(out), ref) < 2e-5
    # ceil-mode 2x2 max pool (pooling_layer.cpp:90-93): 37x53 -> 19x27, partial windows at the edge
    pooled = torch.zeros(2, B, 19, 27, 64, device="cuda", dtype=torch.bfloat16)
    dense.maxpool2x2(out, B, H, W, 64, pooled)
    want = F.max_pool2d(dense.merge(out).permute(0, 3, 1, 2), 2, 2, ceil_mode=True).permute(0, 2, 3, 1)
    assert torch.equal(dense.merge(pooled), want)
    # Caffe's known-answer pooling vector (test_pooling_layer.cpp:60-118, 2x2 stride 1 is not our
    # kernel; the 2x2/2 ceil-mode rule is pinned by the oracle golden test) -- layout round trip:
    nchw = torch.empty(B, 64, 19, 27, device="cuda")
    dense.split_to_nchw(pooled, B, 19, 27, 64, nchw)
    assert torch.equal(nchw, dense.merge(pooled).permute(0, 3, 1, 2))
    back = torch.zeros_like(pooled)
    dense.nchw_to_split(nchw, back)
    assert torch.equal(dense.merge(back), dense.merge(pooled))


@pytest.mark.parametrize("B,H,W", [(2, 37, 53), (1, 5, 128), (3, 20, 300), (1, 600, 1000)])
def test_conv1_1_tensor_core_form(B, H, W):
    """conv1_1 as an MMA (producer warps build the swizzled A tile, K = 27 padded to 32) vs fp64,
    and vs the fp32 FMA kernel; ragged row tiles (W % 128 != 0), image borders, batch > 1."""
    import torch.nn.functional as F
    from mnc_b200 import dense
    torch.manual_seed(B * 1000 + W)
    data = (torch.rand(B, 3, H, W, device="cuda") * 255 - 115).contiguous()   # mean-subtracted pixels
    w = torch.randn(64, 3, 3, 3, device="cuda") * 0.02
    b = torch.randn(64, device="cuda")
    out = torch.zeros(2, B, H, W, 64, device="cuda", dtype=torch.bfloat16)
    dense.conv1_1_tc(data, dense.conv1_1_weight_to_tc(w), b, out)
    ref = F.relu(F.conv2d(data.double(), w.double(), b.double(), padding=1)).permute(0, 2, 3, 1)
    assert relerr(dense.merge(out), ref) < 1e-4
    simt = torch.zeros_like(out)
    dense.conv1_1(data, w, b, simt)
    assert relerr(dense.merge(out), dense.merge(simt).double()) < 1e-4
    # tri-plane output (what the precision-mode-1 convolutions read) + the running max |output|
    ot = dense.tri_alloc((B, H, W, 64), "cuda")
    amax = torch.zeros(1, dtype=torch.int32, device="cuda")
    dense.conv1_1_tc(data, dense.conv1_1_weight_to_tc(w), b, ot, out_exp=dense.exp_for(float(ref.max())),
                     amax=amax)
    assert relerr(ot.float(), ref) < 1e-4
    assert abs(float(amax.view(torch.float32)) - float(ref.max())) < 1e-4 * float(ref.max())


@pytest.mark.parametrize("B,H,W,Cin,Cout,bn", [(1, 75, 125, 64, 128, 128), (2, 37, 53, 64, 64, 64),
                                               (1, 16, 32, 128, 256, 256), (1, 9, 17, 64, 72, 128)])
def test_conv3x3_with_fused_ceil_mode_pool(B, H, W, Cin, Cout, bn):
    """conv + bias + ReLU + 2x2/2 ceil-mode max pool in one epilogue == conv then Caffe pooling
    (pooling_layer.cpp:90-93), including odd H/W (partial windows) and ragged tiles."""
    import torch.nn.functional as F
    from mnc_b200 import dense
    torch.manual_seed(H + W)
    x = torch.randn(B, Cin, H, W, device="cuda")
    w = torch.randn(Cout, Cin, 3, 3, device="cuda") / (9 * Cin) ** 0.5
    b = torch.randn(Cout, device="cuda")
    xs = dense.split(x.permute(0, 2, 3, 1).contiguous())
    ws = dense.conv_weight_to_split(w)
    full = torch.zeros(2, B, H, W, Cout, device="cuda", dtype=torch.bfloat16)
    dense.igemm(xs, B, H, W, Cin, ws, Cout, 9, bias=b, relu=True, out=full, bn=bn)
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    pooled = torch.zeros(2, B, Ho, Wo, Cout, device="cuda", dtype=torch.bfloat16)
    dense.igemm(xs, B, H, W, Cin, ws, Cout, 9, bias=b, relu=True, out=pooled, bn=bn, pool=True)
    want = F.max_pool2d(dense.merge(full).permute(0, 3, 1, 2), 2, 2, ceil_mode=True).permute(0, 2, 3, 1)
    assert torch.equal(dense.merge(pooled), want)
    # precision mode 1 tri-plane in and out
    if Cout % 16 != 0:     # tri-plane rows are 16-byte aligned in every plane: Cout % 16 == 0
        with pytest.raises(Exception, match="MNC_ERR_ARG"):
            dense.igemm2(dense.tri_from_f32(x.permute(0, 2, 3, 1).contiguous()), B, H, W, Cin,
                         dense.conv_weight_to_tri(w), Cout, 9, bias=b, relu=True,
                         out=dense.tri_alloc((B, Ho, Wo, Cout), "cuda"), pool=True, bn=bn)
        return
    ref = F.max_pool2d(F.relu(F.conv2d(x.double(), w.double(), b.double(), padding=1)), 2, 2,
                       ceil_mode=True).permute(0, 2, 3, 1)
    xt, wt = dense.tri_from_f32(x.permute(0, 2, 3, 1).contiguous()), dense.conv_weight_to_tri(w)
    pt = dense.tri_alloc((B, Ho, Wo, Cout), "cuda")
    dense.igemm2(xt, B, H, W, Cin, wt, Cout, 9, bias=b, relu=True, out=pt, pool=True,
                 out_exp=dense.exp_for(float(ref.max())), bn=bn)
    assert relerr(pt.float(), ref) < 1e-4

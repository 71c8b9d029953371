"""Weight container for the MNC 5-stage test net, keyed by Caffe layer names
(models/VGG16/mnc_5stage/test.prototxt), in Caffe layouts: conv (Cout, Cin, kh, kw);
InnerProduct (N, K) with K flattened as (c, h, w) (inner_product_layer.cpp:14-34).
`*_ext` layers share these parameters (test.prototxt:829-834 ...).

No trained weights exist offline (data/scripts/fetch_mnc_model.sh needs the network) and the
prototxt gives fillers only for the three RPN layers (:401-402, 422-423, 436-437), so
`make_weights` is this build's seeded initialiser (SURVEY.md section 8d).
"""
import torch

FULL_ARCH = dict(trunk=[64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512],
                 rpn=512, fc=4096, maskest=256)
# same graph with narrow layers: lets the CPU oracle run end to end in about a second
TINY_ARCH = dict(trunk=[64] * 13, rpn=64, fc=256, maskest=64)
TRUNK_NAMES = ["conv1_1", "conv1_2", "conv2_1", "conv2_2", "conv3_1", "conv3_2", "conv3_3",
               "conv4_1", "conv4_2", "conv4_3", "conv5_1", "conv5_2", "conv5_3"]
POOL_AFTER = {"conv1_2", "conv2_2", "conv3_3", "conv4_3"}


def _train_convs():
    out, cin, level = [], 3, 0
    for name, cout in zip(TRUNK_NAMES, FULL_ARCH["trunk"]):
        out.append((name, cin, cout, 3, level, not name.startswith(("conv1", "conv2"))))
        cin = cout
        level += name in POOL_AFTER
    r = FULL_ARCH["rpn"]
    return out + [("rpn_conv_3x3", cin, r, 3, level, True), ("rpn_cls_score", r, 18, 1, level, True),
                  ("rpn_bbox_pred", r, 36, 1, level, True)]


# The 16 convolutions of models/VGG16/mnc_5stage/train.prototxt: (name, Cin, Cout, kernel, level,
# learns), level = the number of 2x2 ceil-mode pools above the layer, learns = lr_mult > 0
# (conv1_x and conv2_x are frozen)
TRAIN_CONVS = _train_convs()


def train_conv_size(H, W, level):
    """Spatial size of a level of the trunk for an H x W image: `level` max pools of kernel 2,
    stride 2, pad 0, ceil mode (pooling_layer.cpp:90-100)."""
    for _ in range(level):
        H, W = (max(H - 2, 0) + 1) // 2 + 1, (max(W - 2, 0) + 1) // 2 + 1
    return H, W


def make_weights(arch=None, seed=2016):
    """conv & FC weights N(0, sqrt(2/fan_in)), biases 0; RPN weights N(0, 0.01) as the prototxt
    fillers say.  conv1_1 is scaled by 1/64 (mean-subtracted pixels are ~70 RMS) so activations
    are O(1) like a trained net's and softmax / sigmoid outputs are not saturated; bbox_pred by
    0.1 so stage-2 boxes stay near stage-1 boxes.  Returns {name: (weight, bias)} fp32 CPU."""
    arch = arch or FULL_ARCH
    g = torch.Generator().manual_seed(seed)
    w = {}

    def he(shape, fan_in):
        return torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5

    cin = 3
    for name, cout in zip(TRUNK_NAMES, arch["trunk"]):
        wt = he((cout, cin, 3, 3), cin * 9)
        if name == "conv1_1":
            wt = wt / 64.0
        w[name] = (wt, torch.zeros(cout))
        cin = cout
    c5 = cin
    r = arch["rpn"]
    w["rpn_conv_3x3"] = (torch.randn((r, c5, 3, 3), generator=g) * 0.01, torch.zeros(r))
    w["rpn_cls_score"] = (torch.randn((18, r, 1, 1), generator=g) * 0.01, torch.zeros(18))
    w["rpn_bbox_pred"] = (torch.randn((36, r, 1, 1), generator=g) * 0.01, torch.zeros(36))
    fc, me = arch["fc"], arch["maskest"]
    w["fc6_maskest"] = (he((me, c5 * 14 * 14), c5 * 14 * 14), torch.zeros(me))
    w["mask_pred"] = (he((441, me), me), torch.zeros(441))
    w["fc6"] = (he((fc, c5 * 7 * 7), c5 * 7 * 7), torch.zeros(fc))
    w["fc7"] = (he((fc, fc), fc), torch.zeros(fc))
    w["fc6_mask"] = (he((fc, c5 * 7 * 7), c5 * 7 * 7), torch.zeros(fc))
    w["fc7_mask"] = (he((fc, fc), fc), torch.zeros(fc))
    w["cls_score"] = (he((21, 2 * fc), 2 * fc), torch.zeros(21))
    w["seg_cls_score"] = (he((21, 2 * fc), 2 * fc), torch.zeros(21))
    w["bbox_pred"] = (he((84, 2 * fc), 2 * fc) * 0.1, torch.zeros(84))
    return w


def arch_of(weights):
    """Recover the layer widths from a weight dict."""
    return dict(trunk=[weights[n][0].shape[0] for n in TRUNK_NAMES],
                rpn=weights["rpn_conv_3x3"][0].shape[0] if "rpn_conv_3x3" in weights else 0,
                fc=weights["fc7"][0].shape[0],
                maskest=weights["fc6_maskest"][0].shape[0] if "fc6_maskest" in weights else 0)


def make_sibling_weights(graph, arch=None, seed=2016):
    """Seeded weights for the sibling test graphs (mnc_b200/siblings.py), same initialiser:
    "faster_rcnn": no mask layers, cls_score (21, fc) / bbox_pred (84, fc) on fc7 alone
    (faster_rcnn_end2end/test.prototxt:558-616); "cfm": the 5-stage layer set minus the RPN
    (cfm/test.prototxt has no RPN: proposals are inputs)."""
    arch = arch or FULL_ARCH
    w = make_weights(arch, seed)
    fc = arch["fc"]
    if graph == "faster_rcnn":
        g = torch.Generator().manual_seed(seed + 1)
        for n in ("fc6_maskest", "mask_pred", "fc6_mask", "fc7_mask", "seg_cls_score"):
            del w[n]
        w["cls_score"] = (torch.randn((21, fc), generator=g) * (2.0 / fc) ** 0.5, torch.zeros(21))
        w["bbox_pred"] = (torch.randn((84, fc), generator=g) * (2.0 / fc) ** 0.5 * 0.1, torch.zeros(84))
    elif graph == "cfm":
        for n in ("rpn_conv_3x3", "rpn_cls_score", "rpn_bbox_pred"):
            del w[n]
    else:
        raise ValueError(graph)
    return w

"""The proposal stage at batch > 1, every image with its own im_info row [h, w, scale]:

  mnc_rpn_decode          ProposalLayer's decode, clip and min-size filter (proposal_layer.py:95-126)
  ops.proposals_from_rpn  the sort -> gather -> NMS -> write_rois chain behind it
  mnc_stage_bridge        StageBridgeLayer.forward_test (stage_bridge_layer.py:237-255)
  MNCEngine.detect        an image's results do not depend on the rest of its batch

The reference takes one image per call, so the numpy oracle is called once per image with that
image's own im_info row.  Every output buffer the test allocates starts filled with a sentinel, and
what a kernel must not write must still hold it afterwards.

Where the decode's exp(dw), exp(dh) are exact on both sides (dw, dh in {0, +100 -> inf, -200 -> 0,
+inf}) the coordinates are compared bit for bit.  Elsewhere the device's expf and numpy's float32
exp are within 2 ulp of each other (bbox_decode.cuh), so with pw = exp(dw) * width
    |pw_dev - pw_np| <= 2 ulp(exp(dw)) * width + 2 roundings  <= 3 * 2^-23 * pw,
and x1 = pc - 0.5 pw, x2 = pc + 0.5 pw (pc identical on both sides) differ by at most
1.5 * 2^-23 * pw plus one rounding of each result, 2^-23 * |x|.  The test allows twice that,
EXP_BOUND(pc, pw) = 2^-22 * (2 pw + |pc|) per coordinate; the clip can only shrink a difference."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests.test_gpu_detect_tail import SENT_F, SENT_BITS, _bits, _same_bits

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LOSS_LIBS = [os.path.join(ROOT, "oracle", "_ref", n)
                 for n in ("libmnc_ref_loss_nofma.so", "libmnc_ref_loss.so")]
SENT_U8 = 0xAB
PAD = 64                     # spare sentinel elements after every output
A = 9
MIN_SIZE = 16                # cfg.TEST.RPN_MIN_SIZE
F32 = np.float32


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _lib():
    from mnc_b200._lib import lib
    return lib


def _stream():
    from mnc_b200._lib import cur_stream
    return cur_stream()


def _exp_bound(pc, pw):
    """EXP_BOUND of the module docstring, float64."""
    return 2.0 ** -22 * (2.0 * np.abs(pw) + np.abs(pc))


# ============================================================================ 1. rpn_decode
def decode_ref(fg, deltas, row, H, W):
    """proposal_layer.py:95-126 for one image as oracle.proposal_layer_forward runs it: fg (9,H,W)
    scores, deltas (36,H,W), row = that image's im_info.  -> proposals (HWA,4), scores, valid u8."""
    from oracle import oracle as O
    anchors = O.shifted_anchors(H, W)
    d = np.ascontiguousarray(deltas.transpose(1, 2, 0).reshape(-1, 4))
    with np.errstate(over="ignore", invalid="ignore"):
        props = O.bbox_transform_inv(anchors, d)
        props, _ = O.clip_boxes(props, row[:2])
        keep = O.filter_small_boxes(props, MIN_SIZE * row[2])
    valid = np.zeros(H * W * A, np.uint8)
    valid[keep] = 1
    return props.astype(F32), fg.transpose(1, 2, 0).ravel(), valid


def decode_bound(deltas, H, W):
    """EXP_BOUND of every coordinate of the unclipped decode, from float64 pc and pw."""
    from oracle import oracle as O
    anc = O.shifted_anchors(H, W)
    d = deltas.transpose(1, 2, 0).reshape(-1, 4).astype(np.float64)
    w = anc[:, 2] - anc[:, 0] + 1
    h = anc[:, 3] - anc[:, 1] + 1
    with np.errstate(over="ignore", invalid="ignore"):
        bx = _exp_bound(d[:, 0] * w + anc[:, 0] + 0.5 * w, np.exp(d[:, 2]) * w)
        by = _exp_bound(d[:, 1] * h + anc[:, 1] + 0.5 * h, np.exp(d[:, 3]) * h)
    return np.stack([bx, by, bx, by], axis=1)


def side_ok(props, row):
    """filter_small_boxes on given (device) proposals: the valid flag they imply."""
    ws = props[:, 2] - props[:, 0] + F32(1)
    hs = props[:, 3] - props[:, 1] + F32(1)
    ms = MIN_SIZE * row[2]
    with np.errstate(invalid="ignore"):
        return ((ws >= ms) & (hs >= ms)).astype(np.uint8)


def run_rpn_decode(cls, bbox, im_info, H, W, layout, apply_softmax):
    """mnc_rpn_decode on sentinel-filled outputs (PAD spare entries each).  cls / bbox: numpy
    (B,18,H,W) / (B,36,H,W) for 'nchw', cls = one (B,H,W,Cpad) buffer for 'nhwc'.
    -> numpy proposals (B,HWA,4), scores (B,HWA), valid (B,HWA)."""
    from mnc_b200._lib import MNC_OK
    B = im_info.shape[0]
    total = H * W * A
    props = torch.full((B * total * 4 + PAD,), float(SENT_F), dtype=torch.float32, device="cuda")
    scores = torch.full((B * total + PAD,), float(SENT_F), dtype=torch.float32, device="cuda")
    valid = torch.full((B * total + PAD,), SENT_U8, dtype=torch.uint8, device="cuda")
    d_cls, d_info = _dev(cls), _dev(im_info)
    if layout == "nchw":
        d_bbox = _dev(bbox)
        ci, cc, cp, bi, bc, bp = 18 * H * W, H * W, 1, 36 * H * W, H * W, 1
        bptr = d_bbox.data_ptr()
    else:
        cpad = cls.shape[-1]
        ci, cc, cp = H * W * cpad, 1, cpad
        bi, bc, bp = ci, cc, cp
        bptr = d_cls.data_ptr() + 18 * 4
    rc = _lib().mnc_rpn_decode(d_cls.data_ptr(), ci, cc, cp, bptr, bi, bc, bp, d_info.data_ptr(), B, H, W,
                               16, float(MIN_SIZE), int(apply_softmax), props.data_ptr(), scores.data_ptr(),
                               valid.data_ptr(), _stream())
    assert rc == MNC_OK
    torch.cuda.synchronize()
    p, s, v = props.cpu().numpy(), scores.cpu().numpy(), valid.cpu().numpy()
    assert np.all(_bits(p[B * total * 4:]) == SENT_BITS), "proposals written past the batch"
    assert np.all(_bits(s[B * total:]) == SENT_BITS), "scores written past the batch"
    assert np.all(v[B * total:] == SENT_U8), "valid written past the batch"
    return p[:B * total * 4].reshape(B, total, 4), s[:B * total].reshape(B, total), v[:B * total].reshape(B, total)


def im_info_rows(H, W, fracs=((0.9, 0.8), (0.6, 0.95), (0.75, 0.7)), scales=(1.0, 1.6, 0.75)):
    """One [h, w, scale] row per image, h and w strictly inside the (16H, 16W) blob as in a padded
    im_list_to_blob batch."""
    rows = [[max(1, round(fh * 16 * H)), max(1, round(fw * 16 * W)), s] for (fh, fw), s in zip(fracs, scales)]
    rows = np.asarray(rows, F32)
    assert np.all(rows[:, 0] < 16 * H) and np.all(rows[:, 1] < 16 * W)
    return rows


def t_to_nchw(d_t, H, W):
    """(B, H*W*A, k) in anchor order t = (y*W + x)*A + a -> (B, A*k, H, W) NCHW blob."""
    B, _, k = d_t.shape
    return np.ascontiguousarray(d_t.reshape(B, H, W, A * k).transpose(0, 3, 1, 2))


def decode_case(B, H, W, seed):
    """Random RPN outputs with a kind per anchor: 0 = dw = dh = 0, 1 = dw, dh from {+100, -200,
    +inf} (exp exact on both sides), 2 = random dw, dh; a few kind-0/1 anchors get dx = NaN.
    -> fg prob (B,9,H,W), logits (B,18,H,W), deltas (B,36,H,W), kind (B,HWA)."""
    rng = np.random.default_rng(seed)
    total = H * W * A
    kind = rng.integers(0, 3, size=(B, total))
    d = np.zeros((B, total, 4), F32)
    d[:, :, :2] = rng.normal(0, 0.3, size=(B, total, 2))
    special = rng.choice(np.float32([100.0, -200.0, np.inf]), size=(B, total, 2))
    d[:, :, 2:] = np.where((kind == 1)[:, :, None], special,
                           np.where((kind == 2)[:, :, None], rng.normal(0, 0.5, size=(B, total, 2)), 0))
    for img in range(B):
        cand = np.where(kind[img] != 2)[0]
        d[img, rng.choice(cand, size=min(4, len(cand)), replace=False), 0] = np.nan
    fg = rng.uniform(0, 1, size=(B, 9, H, W)).astype(F32)
    logits = rng.normal(0, 2.0, size=(B, 18, H, W)).astype(F32)
    return fg, logits, t_to_nchw(d, H, W), kind


def nhwc_buffer(logits, deltas, cpad):
    """The engine's RPN head buffer: (B,H,W,cpad), channels [0,18) logits, [18,54) deltas, the
    padding NaN (never read)."""
    B, _, H, W = logits.shape
    buf = np.full((B, H, W, cpad), np.nan, F32)
    buf[..., :18] = logits.transpose(0, 2, 3, 1)
    buf[..., 18:54] = deltas.transpose(0, 2, 3, 1)
    return buf


def softmax_fg_bound(logits):
    """fg probability of Caffe's 2-way softmax over (bg = channel a, fg = channel 9 + a) in float64
    from the float32 differences x - max the kernel forms, and the bound on the device's value:
    expf's 2 ulp on eb and ef move ln(ef / (eb + ef)) by at most 4 * 2^-23 * eb / (eb + ef), the
    sum and the division add one rounding each.  -> (fg64 (B,9,H,W), bound)."""
    bg, fg = logits[:, :9].astype(F32), logits[:, 9:].astype(F32)
    m = np.maximum(bg, fg)
    eb = np.exp((bg - m).astype(np.float64))
    ef = np.exp((fg - m).astype(np.float64))
    s = ef / (eb + ef)
    return s, s * (4 * 2.0 ** -23 * eb / (eb + ef) + 2 * 2.0 ** -24) + np.spacing(s.astype(F32)).astype(np.float64)


def check_decode_image(got, fg_want, deltas, kind, row, H, W, img, scores_exact=True):
    """Proposals, valid and scores of one image against decode_ref on that image's slice."""
    props, scores, valid = got
    want_p, want_s, want_v = decode_ref(fg_want, deltas, row, H, W)
    exact = kind != 2
    _same_bits(props[exact], want_p[exact], "proposals image %d (exp exact)" % img)
    bound = decode_bound(deltas, H, W)[~exact]
    diff = np.abs(props[~exact].astype(np.float64) - want_p[~exact])
    assert np.all(diff <= bound), "image %d: decode off by %r > %r" % (img, diff.max(), bound[diff > bound][:3])
    assert np.array_equal(valid[exact], want_v[exact]), "image %d: valid" % img
    # the flag is filter_small_boxes on the device's own proposals, everywhere
    assert np.array_equal(valid, side_ok(props, row)), "image %d: valid vs own proposals" % img
    if scores_exact:
        _same_bits(scores, want_s, "scores image %d" % img)
    return want_p, want_v


SHAPES = [(5, 7), (13, 1), (38, 63)]          # H*W*9 = 315, 117, 21546: none a multiple of 256


@pytest.mark.parametrize("H,W", SHAPES)
@pytest.mark.parametrize("layout,cpad", [("nchw", None), ("nhwc", 54), ("nhwc", 64)])
def test_rpn_decode_batch_per_image(H, W, layout, cpad):
    """Batch of 3 with three different im_info rows (h, w and scale 1.0 / 1.6 / 0.75): each image's
    proposals, scores and valid flags against the oracle on that image alone.  NCHW takes the
    probabilities as they are (scores copied bit for bit; the bg channels hold NaN and must not
    be read); NHWC applies the 2-way softmax to logits in the engine's padded head buffer."""
    B = 3
    fg, logits, deltas, kind = decode_case(B, H, W, seed=H * 100 + W + (cpad or 0))
    info = im_info_rows(H, W)
    if layout == "nchw":
        prob = np.concatenate([np.full((B, 9, H, W), np.nan, F32), fg], axis=1)
        got = run_rpn_decode(prob, deltas, info, H, W, "nchw", 0)
    else:
        got = run_rpn_decode(nhwc_buffer(logits, deltas, cpad), None, info, H, W, "nhwc", 1)
    n_valid = []
    for img in range(B):
        g = tuple(x[img] for x in got)
        if layout == "nchw":
            _, want_v = check_decode_image(g, fg[img], deltas[img], kind[img], info[img], H, W, img)
        else:
            _, want_v = check_decode_image(g, fg[img], deltas[img], kind[img], info[img], H, W, img,
                                           scores_exact=False)
            s64, bound = softmax_fg_bound(logits[img:img + 1])
            s64, bound = s64[0].transpose(1, 2, 0).ravel(), bound[0].transpose(1, 2, 0).ravel()
            err = np.abs(g[1].astype(np.float64) - s64)
            assert np.all(err <= bound), "image %d: softmax off by %r" % (img, (err / bound).max())
        n_valid.append(int(want_v.sum()))
        # dw, dh in {+100, +inf}: the box spans the clipped image
        d_t = deltas[img].transpose(1, 2, 0).reshape(-1, 4)
        span = np.all(d_t[:, 2:] >= 100, axis=1) & ~np.isnan(d_t[:, 0])
        h, w = info[img, 0], info[img, 1]
        assert span.any()
        assert np.all(g[0][span] == np.float32([0, 0, w - 1, h - 1]))
    if (H, W) == (38, 63):
        assert min(n_valid) > 1000                # the filter keeps most; it is not trivially empty


def _ref_softmax_fg(lib, logits_img):
    """The reference's own Softmax (through SoftmaxWithLoss) on the (1, 2, 9H, W) reshape of one
    image's rpn_cls_score, as the test net reshapes it (test.prototxt rpn_cls_score_reshape)."""
    _, H, W = logits_img.shape
    x = np.ascontiguousarray(logits_img.reshape(1, 2, 9 * H, W), dtype=F32)
    lab = np.zeros((1, 9 * H * W), F32)
    loss, prob, diff = np.zeros(1, F32), np.zeros_like(x), np.zeros_like(x)
    P = ctypes.c_void_p
    lib.ref_softmax_loss.argtypes = [P, P] + [ctypes.c_int] * 7 + [ctypes.c_float, P, P, P, P]
    lib.ref_softmax_loss(x.ctypes.data, lab.ctypes.data, 1, 2, 9 * H * W, 0, 0, 1, 0, 1.0,
                         loss.ctypes.data, prob.ctypes.data, diff.ctypes.data, None)
    return prob.reshape(18, H, W)[9:]


@pytest.mark.parametrize("H,W", SHAPES)
@pytest.mark.parametrize("cpad", [54, 64])
def test_rpn_decode_softmax_is_the_reference_softmax(H, W, cpad):
    """The fused softmax of the NHWC form equals the reference's Caffe Softmax bit for bit, image by
    image (both builds of the reference library)."""
    libs = [p for p in REF_LOSS_LIBS if os.path.exists(p)]
    if not libs:
        pytest.skip("reference loss library not built (oracle/loss.mk needs a reference checkout)")
    B = 3
    fg, logits, deltas, kind = decode_case(B, H, W, seed=7 + H * W + cpad)
    logits[0, :, 0, 0] = 0.0                       # bg == fg: exactly 0.5
    logits[1, :9, -1, -1], logits[1, 9:, -1, -1] = 40.0, -40.0
    info = im_info_rows(H, W)
    _, scores, _ = run_rpn_decode(nhwc_buffer(logits, deltas, cpad), None, info, H, W, "nhwc", 1)
    for path in libs:
        lib = ctypes.CDLL(path)
        for img in range(B):
            want = _ref_softmax_fg(lib, logits[img]).transpose(1, 2, 0).ravel()
            _same_bits(scores[img], want, "%s image %d" % (os.path.basename(path), img))


@pytest.mark.parametrize("H,W", SHAPES)
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
def test_rpn_decode_anchor_index_corners(H, W, layout):
    """t = (y*W + x)*9 + a: zero deltas and flat scores everywhere except single marked cells,
    (0, 0, 0) and the far corner (H-1, W-1, 8) among them; the marked values must come out at
    exactly those t, in every image of the batch.  A marked box collapses to a point (dw = dh =
    -200) near its anchor's centre, inside the full-blob image, so it differs from the unmarked
    box however the clip cuts that."""
    B, total = 3, H * W * A
    marks = [[(0, 0, 0), (H - 1, W - 1, 8)], [(H - 1, W - 1, 8), (0, W - 1, 4)], [(0, 0, 0), (H - 1, 0, 5)]]
    d = np.zeros((B, total, 4), F32)
    score_t = np.full((B, total), 0.25, F32)
    logit_t = np.zeros((B, total, 2), F32)              # bg = fg = 0: exactly 0.5
    for img, ms in enumerate(marks):
        for k, (y, x, a) in enumerate(ms):
            t = (y * W + x) * A + a
            u = F32(2.0 ** -10 * (k + 1 + 2 * img))      # |u * anchor side| < 7.5: stays inside
            d[img, t] = [u if x == 0 else -u, u if y == 0 else -u, -200, -200]
            score_t[img, t] = 0.75
            logit_t[img, t, 1] = 50.0                    # fg wins: exactly 1.0
    deltas = t_to_nchw(d, H, W)
    fg = t_to_nchw(score_t[:, :, None], H, W)
    logits = np.concatenate([t_to_nchw(logit_t[:, :, :1], H, W), t_to_nchw(logit_t[:, :, 1:], H, W)], axis=1)
    info = np.array([[16 * H, 16 * W, s] for s in (1.0, 0.5, 0.25)], F32)
    if layout == "nchw":
        prob = np.concatenate([np.full((B, 9, H, W), np.nan, F32), fg], axis=1)
        props, scores, valid = run_rpn_decode(prob, deltas, info, H, W, "nchw", 0)
        marked_score = F32(0.75)
    else:
        props, scores, valid = run_rpn_decode(nhwc_buffer(logits, deltas, 64), None, info, H, W, "nhwc", 1)
        marked_score = F32(1.0)
    kind = np.zeros(total, int)
    for img, ms in enumerate(marks):
        ts = sorted((y * W + x) * A + a for y, x, a in ms)
        check_decode_image((props[img], scores[img], valid[img]), fg[img], deltas[img], kind, info[img],
                           H, W, img, scores_exact=layout == "nchw")
        flat, _, _ = decode_ref(fg[img], np.zeros_like(deltas[img]), info[img], H, W)
        moved = np.where(np.any(_bits(props[img]) != _bits(flat), axis=1))[0]
        assert moved.tolist() == ts, (img, moved.tolist(), ts)
        assert np.where(scores[img] == marked_score)[0].tolist() == ts, img


def _land_side(axis, target, t, anchors, row):
    """dx (axis 0) or dy (axis 1) such that anchor t, with every other delta 0, decodes and clips
    (low side clipped to 0) to a side of exactly `target` under im_info row `row`: a walk over
    float32 values from the estimate, the oracle evaluating each.  None if the side steps over it."""
    from oracle import oracle as O
    box = anchors[t:t + 1]
    size = box[0, axis + 2] - box[0, axis] + 1
    ctr = box[0, axis] + 0.5 * size
    v = F32((float(target) - 1 - 0.5 * size - ctr) / size)
    prev = None
    for _ in range(256):
        dl = np.zeros((1, 4), F32)
        dl[0, axis] = v
        p, _ = O.clip_boxes(O.bbox_transform_inv(box, dl), row[:2])
        side = p[0, axis + 2] - p[0, axis] + F32(1)
        if side == target and p[0, axis] == 0:
            return v
        step = F32(np.inf) if side < target else F32(-np.inf)
        if prev is not None and step != prev:
            return None
        prev = step
        v = np.nextafter(v, step)
    return None


def test_rpn_decode_min_size_boundary_and_special_deltas():
    """filter_small_boxes keeps ws >= 16 * scale and hs >= 16 * scale.  At scale 1.6 the threshold
    is 25.6000004 (non-integer), an odd multiple of its ulp, so only a box side below 32 px can land
    on it: a box at the image's top-left corner (low side clipped to 0) with a searched dx (dy) has
    a clipped width (height) of exactly the threshold, or one float32 ulp below it.  The height
    exactly at the threshold is not reachable that way (dy * 96 skips it), so it comes from
    dh = +inf in an image whose height is the threshold itself (h - 1 + 1 == h, exactly).
    Images: 0 scale 1.6; 1 the next float32 above 1.6 (threshold one ulp higher); 2 scale 0.75;
    3 and 4 scale 1.6 with heights of the threshold and one ulp below.  The same deltas are kept in
    one image and dropped in another.  Also dx = NaN (the clip keeps the NaN: dropped) and
    dw, dh = +inf / +100 (the box spans the clipped image)."""
    from oracle import oracle as O
    H, W = 5, 7
    s = F32(1.6)
    ms = MIN_SIZE * s
    below = np.nextafter(ms, F32(0))
    assert ms == F32(25.6000004) and ms != np.round(ms)
    info = np.array([[70, 100, s], [70, 100, np.nextafter(s, F32(2))], [70, 100, 0.75],
                     [ms, 100, s], [below, 100, s]], F32)
    B = info.shape[0]
    assert MIN_SIZE * info[1, 2] == np.nextafter(ms, F32(100))
    anchors = O.shifted_anchors(H, W)
    total = H * W * A
    d = np.zeros((total, 4), F32)
    marked = []
    for axis, target, cell in [(0, ms, (1, 0)), (0, below, (2, 0)), (1, below, (0, 2))]:
        for a in range(A):
            t = (cell[0] * W + cell[1]) * A + a
            v = _land_side(axis, target, t, anchors, info[0])
            if v is not None:
                break
        assert v is not None, (axis, target)
        d[t, axis] = v
        marked.append(t)
    h_span = (0 * W + 4) * A + 3                   # x in [8, 99]; y spans [0, h - 1]
    d[h_span, 3] = np.inf
    marked.append(h_span)
    # kept? per image: width at the threshold, width below, height below, full height
    want_kept = [[1, 0, 0, 1], [0, 0, 0, 1], [1, 1, 1, 1], [1, 0, 0, 1], [0, 0, 0, 0]]
    # dx = NaN; dw, dh = +inf / +100
    nan_t = [(4 * W + 4) * A + 2, (3 * W + 1) * A + 7]
    d[nan_t[0], 0] = np.nan
    d[nan_t[1], 0] = np.nan
    d[nan_t[1], 2] = np.inf
    span_t = [(3 * W + 3) * A + 0, (3 * W + 4) * A + 4, (3 * W + 5) * A + 8, (4 * W + 6) * A + 3]
    for t, (dw, dh) in zip(span_t, [(np.inf, np.inf), (100, 100), (np.inf, 100), (100, np.inf)]):
        d[t] = [0.3, -0.2, dw, dh]
    deltas = t_to_nchw(np.broadcast_to(d, (B, total, 4)).copy(), H, W)
    fg = np.random.default_rng(3).uniform(0, 1, size=(B, 9, H, W)).astype(F32)
    prob = np.concatenate([np.full((B, 9, H, W), np.nan, F32), fg], axis=1)
    props, scores, valid = run_rpn_decode(prob, deltas, info, H, W, "nchw", 0)
    kind = np.zeros(total, int)
    for img in range(B):
        want_p, want_v = check_decode_image((props[img], scores[img], valid[img]), fg[img], deltas[img], kind,
                                            info[img], H, W, img)
        assert want_v[marked].tolist() == want_kept[img], (img, want_v[marked])
        assert valid[img, marked].tolist() == want_kept[img], (img, valid[img, marked])
        sides = np.stack([want_p[marked, 2] - want_p[marked, 0], want_p[marked, 3] - want_p[marked, 1]]) + F32(1)
        assert sides[0, 0] == ms and sides[0, 1] == below and sides[1, 2] == below
        assert sides[1, 3] == {3: ms, 4: below}.get(img, F32(70))
        assert np.all(valid[img, nan_t] == 0)
        assert np.all(np.isnan(props[img, nan_t][:, [0, 2]])) and not np.isnan(props[img, nan_t][:, [1, 3]]).any()
        assert np.all(props[img, span_t] == np.float32([0, 0, info[img, 1] - 1, info[img, 0] - 1]))
        assert np.all(valid[img, span_t] == (img != 4))


# ============================================================================ 2. the chain at batch 3
def chain_case(H=38, W=63, seed=21):
    """Three images with three outcomes: image 0 a normal map (more than 6000 valid proposals),
    image 1 scale 100 (min size 1600: nothing valid), image 2 valid proposals only in a 5 x 8 cell
    corner (dw = dh = -200 elsewhere: zero-size boxes), so fewer than 6000 valid and fewer than
    300 NMS survivors."""
    rng = np.random.default_rng(seed)
    B = 3
    fg = rng.uniform(0, 1, size=(B, 9, H, W)).astype(F32)
    prob = np.concatenate([np.full((B, 9, H, W), np.nan, F32), fg], axis=1)
    deltas = rng.normal(0, 0.5, size=(B, 36, H, W)).astype(F32)
    mask = np.ones((H, W), bool)
    mask[:5, :8] = False
    for a in range(A):
        deltas[2, 4 * a + 2][mask] = -200
        deltas[2, 4 * a + 3][mask] = -200
    info = np.array([[600, 1000, 1.0], [550, 900, 100.0], [480, 800, 0.75]], F32)
    return prob, deltas, info


@pytest.mark.parametrize("pre_nms_top_n", [6000, 12000, 0])
@pytest.mark.parametrize("batch_index_mode", [True, False])
def test_proposal_chain_batch3(pre_nms_top_n, batch_index_mode):
    """proposals_from_rpn at batch 3, teacher-forced per image on the device's own decode: n_valid,
    counts, order, the sorted boxes, num, roi_counts and the RoIs bit for bit, the padding rows
    [img, 0, 0, 0, 0] in batch-index mode and [0, 0, 0, 0, 0] without.  6000 takes the top-k select,
    12000 (the TRAIN value) and 0 (keep all) the full rank sort at 38 x 63."""
    from mnc_b200 import ops
    from oracle import oracle as O
    H, W, post, thresh = 38, 63, 300, 0.7
    prob, deltas, info = chain_case(H, W)
    B, total = 3, H * W * A
    rois, roi_counts, mid = ops.proposals_from_rpn(_dev(prob), _dev(deltas), _dev(info), B, H, W, "nchw", False,
                                                   pre_nms_top_n=pre_nms_top_n, post_nms_top_n=post,
                                                   nms_thresh=thresh, batch_index_mode=batch_index_mode,
                                                   return_intermediate=True)
    torch.cuda.synchronize()
    rois, roi_counts = rois.cpu().numpy(), roi_counts.cpu().numpy()
    m = {k: v.cpu().numpy() for k, v in mid.items()}
    n_sorted = min(pre_nms_top_n, total) if pre_nms_top_n > 0 else total
    outcome = []
    for img in range(B):
        props, scores, valid = m["proposals"][img], m["scores"][img], m["valid"][img]
        # the decode of this image alone (exactness of the decode itself is section 1's)
        want_p, _, want_v = decode_ref(prob[img, 9:], deltas[img], info[img], H, W)
        assert np.array_equal(valid, side_ok(props, info[img]))
        assert np.allclose(props, want_p, rtol=1e-5, atol=2e-3, equal_nan=True)
        keep_filter = np.where(valid != 0)[0]
        order = keep_filter[O.order_desc(scores[keep_filter])]
        if pre_nms_top_n > 0:
            order = order[:pre_nms_top_n]
        c = len(order)
        # the top-k select reports the valid entries it keeps (at most k), the rank sort all of them
        assert m["order"].shape[1] == (n_sorted if pre_nms_top_n == 6000 else total)
        assert m["n_valid"][img] == min(len(keep_filter), m["order"].shape[1]), img
        assert m["counts"][img] == c == min(len(keep_filter), n_sorted), img
        assert np.array_equal(m["order"][img, :c], order), img
        _same_bits(m["sorted_boxes"][img, :c], props[order], "sorted boxes image %d" % img)
        keep = O.nms_sorted(props[order], thresh)
        k = min(len(keep), post)
        assert m["num"][img] == k and roi_counts[img] == k, (img, m["num"][img], roi_counts[img], len(keep))
        want = np.zeros((post, 5), F32)
        want[:, 0] = img if batch_index_mode else 0
        want[:k, 1:] = props[order[keep[:k]]]
        _same_bits(rois[img], want, "rois image %d" % img)
        outcome.append((len(keep_filter), len(keep)))
    assert outcome[0][0] > 6000 and outcome[0][1] >= post
    assert outcome[1] == (0, 0)
    assert 0 < outcome[2][0] < 6000 and 0 < outcome[2][1] < post and outcome[2][1] < outcome[2][0]


# ============================================================================ 3. stage_bridge
HEAD_W = 128                  # MNCEngine.head: one fp32 row of 128 per RoI
SEG_COLS = slice(21, 42)      # seg_cls_score (the engine softmaxes it into its own 21-wide rows)
BBOX_COLS = slice(42, 126)    # bbox_pred, handed over as this column slice
NCLS = 21


def bridge_case(seed=31):
    """3 images x 300 RoI rows with 217 / 41 / 150 real RoIs, the rest padding [img, 0, 0, 0, 0];
    deltas per (row, class) of kind 0 / 1 / 2 as in section 1; seg_cls_prob rows with the class
    choices that matter (ties, the last column, +inf, NaN in column 0 and later)."""
    from tests import util
    rng = np.random.default_rng(seed)
    B, n = 3, 300
    counts = [217, 41, 150]
    info = np.array([[600, 1000, 1.0], [333, 517, 1.6], [480, 640, 0.75]], F32)
    rois = np.zeros((B * n, 5), F32)
    for img in range(B):
        rois[img * n:(img + 1) * n, 0] = img
        b = util.random_boxes(counts[img], seed + img, width=int(info[img, 1]), height=int(info[img, 0]))
        rois[img * n:img * n + counts[img], 1:] = b
    R = B * n
    kind = rng.integers(0, 3, size=(R, NCLS))
    d = np.zeros((R, NCLS, 4), F32)
    d[:, :, :2] = rng.normal(0, 0.3, size=(R, NCLS, 2))
    special = rng.choice(np.float32([100.0, -200.0, np.inf]), size=(R, NCLS, 2))
    d[:, :, 2:] = np.where((kind == 1)[:, :, None], special,
                           np.where((kind == 2)[:, :, None], rng.normal(0, 0.5, size=(R, NCLS, 2)), 0))
    logits = rng.normal(0, 1, size=(R, NCLS))
    prob = (np.exp(logits) / np.exp(logits).sum(1, keepdims=True)).astype(F32)
    nan, inf = F32(np.nan), F32(np.inf)
    cases = {}
    for img in range(B):
        base = img * n
        for r in [base + 3, base + counts[img] + 5]:                  # a real row and a padding row
            rows = {
                "all equal": np.full(NCLS, F32(1.0 / NCLS)),
                "max in the last column": np.r_[np.full(NCLS - 1, F32(0.01)), F32(0.8)],
                "+inf": np.r_[np.full(7, F32(0.3)), inf, np.full(NCLS - 8, F32(0.5))],
                "+inf twice": np.r_[F32(0.1), F32(0.2), F32(0.1), inf, np.full(5, F32(0.1)), inf, np.full(NCLS - 10, F32(0.9))],
                "NaN in column 0": np.r_[nan, np.full(4, F32(0.2)), F32(0.9), np.full(NCLS - 6, F32(0.01))],
                "NaN later": np.r_[F32(0.05), F32(0.9), np.full(11, F32(0.01)), nan, np.full(NCLS - 14, F32(0.02))],
                "+inf then NaN": np.r_[F32(0.1), F32(0.1), inf, F32(0.1), nan, np.full(12, F32(0.1)), nan, np.full(NCLS - 18, F32(0.1))],
                "NaN in the last column": np.r_[F32(0.3), np.full(NCLS - 2, F32(0.6)), nan],
            }
            for k, (name, row) in enumerate(rows.items()):
                prob[r + k] = row
                kind[r + k] = 0                  # every class exact: a wrong choice shows in the bits
                d[r + k, :, 2:] = 0
                cases.setdefault(name, []).append(r + k)
    return rois, d.reshape(R, 4 * NCLS), kind, prob, info, cases


def bridge_ref(rois, bbox, prob, info, n):
    """StageBridgeLayer.forward_test per image with that image's im_info (the oracle writes batch
    index 0; the kernel copies the RoI's)."""
    from oracle import oracle as O
    out = np.zeros((rois.shape[0], 5), F32)
    for img in range(info.shape[0]):
        sl = slice(img * n, (img + 1) * n)
        with np.errstate(over="ignore", invalid="ignore"):
            out[sl] = O.stage_bridge_forward(rois[sl], bbox[sl], prob[sl], info[img:img + 1])
    out[:, 0] = rois[:, 0]
    return out


@pytest.mark.parametrize("seg_form", ["own rows", "head slice"])
def test_stage_bridge_batch(seg_form):
    """mnc_stage_bridge at batch 3 with the engine's strides: bbox_pred a column slice of the
    128-wide head buffer (the other columns NaN: never read), seg_cls_prob either its own 21-wide
    rows (the engine's softmax output) or a slice of the same buffer.  Bit-exact against the oracle
    per image where the chosen class's exp is exact, EXP_BOUND elsewhere; the class is numpy's
    argmax, which returns the first NaN of a row."""
    from mnc_b200 import ops
    from mnc_b200._lib import MNC_OK
    n = 300
    rois, bbox, kind, prob, info, cases = bridge_case()
    R = rois.shape[0]
    heads = np.full((R, HEAD_W), np.nan, F32)
    heads[:, BBOX_COLS] = bbox
    d_heads = _dev(heads)
    if seg_form == "head slice":
        heads[:, SEG_COLS] = prob
        d_heads = _dev(heads)
        d_seg = d_heads[:, SEG_COLS]
    else:
        d_seg = _dev(prob)
    d_bbox = d_heads[:, BBOX_COLS]
    d_rois, d_info = _dev(rois), _dev(info)
    out = torch.full((R * 5 + PAD,), float(SENT_F), dtype=torch.float32, device="cuda")
    rc = _lib().mnc_stage_bridge(d_rois.data_ptr(), d_bbox.data_ptr(), d_bbox.stride(0), d_seg.data_ptr(),
                                 d_seg.stride(0), NCLS, d_info.data_ptr(), n, R, out.data_ptr(), _stream())
    assert rc == MNC_OK
    got_all = out.cpu().numpy()
    assert np.all(_bits(got_all[R * 5:]) == SENT_BITS), "written past the last RoI"
    got = got_all[:R * 5].reshape(R, 5)
    want = bridge_ref(rois, bbox, prob, info, n)
    best = prob.argmax(axis=1)
    for name, rows in cases.items():
        assert len(rows) == 6
    assert np.all(best[cases["all equal"]] == 0) and np.all(best[cases["max in the last column"]] == NCLS - 1)
    assert np.all(best[cases["+inf"]] == 7) and np.all(best[cases["+inf twice"]] == 3)
    assert np.all(best[cases["NaN in column 0"]] == 0) and np.all(best[cases["NaN later"]] == 13)
    assert np.all(best[cases["+inf then NaN"]] == 4) and np.all(best[cases["NaN in the last column"]] == NCLS - 1)
    # the class choice by name first: a wrong choice decodes another class's deltas
    for name, rows in cases.items():
        exact_rows = [r for r in rows if kind[r, best[r]] != 2]
        _same_bits(got[exact_rows], want[exact_rows], "rows '%s'" % name)
    exact = kind[np.arange(R), best] != 2
    _same_bits(got[exact], want[exact], "stage bridge (exp exact)")
    d = bbox.reshape(R, NCLS, 4)[np.arange(R), best].astype(np.float64)
    w = rois[:, 3].astype(np.float64) - rois[:, 1] + 1
    h = rois[:, 4].astype(np.float64) - rois[:, 2] + 1
    bx = _exp_bound(d[:, 0] * w + rois[:, 1] + 0.5 * w, np.exp(d[:, 2]) * w)
    by = _exp_bound(d[:, 1] * h + rois[:, 2] + 0.5 * h, np.exp(d[:, 3]) * h)
    bound = np.stack([bx, by, bx, by], axis=1)[~exact]
    diff = np.abs(got[~exact, 1:].astype(np.float64) - want[~exact, 1:])
    assert np.all(diff <= bound), diff.max()
    assert np.array_equal(got[:, 0], rois[:, 0])
    # the ops wrapper reads the same strides from the views
    via_ops = ops.stage_bridge(d_rois, d_bbox, d_seg, d_info, n).cpu().numpy()
    _same_bits(via_ops, got, "ops.stage_bridge")


# ============================================================================ 4. images are independent
IMG_H, IMG_W = 224, 320


def _image(i, h, w):
    """Synthetic image i, mean-subtracted, in the top-left corner of a zero (IMG_H, IMG_W) blob
    slot as im_list_to_blob pads a batch."""
    from oracle import oracle as O
    blob, _ = O.prep_blob(O.synthetic_image(i, h, w))
    out = np.zeros((1, 3, IMG_H, IMG_W), F32)
    out[:, :, :h, :w] = blob
    return out


# name -> (synthetic image, h, w, scale): A is in both batches; E's scale makes the min size 1600
IMAGES = {"A": (0, 200, 300, 1.0), "B": (1, 224, 320, 1.0), "C": (2, 180, 256, 0.8),
          "D": (3, 224, 288, 1.2), "E": (4, 224, 320, 100.0)}


def _batch(names):
    data = np.concatenate([_image(i, h, w) for i, h, w, _ in (IMAGES[k] for k in names)])
    info = np.array([[h, w, s] for _, h, w, s in (IMAGES[k] for k in names)], F32)
    hw = np.array([[max(1, round(h / s)), max(1, round(w / s))] for _, h, w, s in (IMAGES[k] for k in names)], F32)
    scale = info[:, 2].copy()
    return data, info, hw, scale


ROW_BLOBS = ["mask_proposal", "seg_cls_prob", "cls_prob", "bbox_pred"]


def _run_engine(eng, names, graphed):
    """detect (or detect_graphed) + mask voting on one batch; every result copied to the host
    before the next call reuses the buffers."""
    from mnc_b200 import ops
    data, info, hw, scale = _batch(names)
    B, n = len(names), 300
    fn = eng.detect_graphed if graphed else eng.detect
    boxes, masks, scores, valid, o = fn(_dev(data), _dev(info), _dev(hw), _dev(scale))
    r = {"boxes": boxes, "masks": masks, "scores": scores, "valid": valid,
         "rec_counts": eng.last_record[:B], "roi_counts": o["roi_counts"],
         "rois": o["rois"].view(B, n, 5), "rois_ext": o["rois_ext"].view(B, n, 5)}
    for k in ROW_BLOBS:
        for suffix in ("", "_ext"):
            r[k + suffix] = o[k + suffix].reshape(B, n, -1)
    vote = ops.mask_voting_checked(boxes, masks, scores, _dev(hw.astype(np.int32)), box_valid=valid)
    for k in ("n_res", "class_bar", "res_score", "res_class", "res_box_idx", "result_mask", "result_box"):
        r["vote_" + k] = vote[k]
    torch.cuda.synchronize()
    return {k: v.cpu().numpy().copy() for k, v in r.items()}


def _same_image(p, q, i, j, what):
    """Image slot i of run p == image slot j of run q, bit for bit."""
    for k in ROW_BLOBS + [b + "_ext" for b in ROW_BLOBS] + ["boxes", "masks", "scores", "valid",
                                                            "rec_counts", "roi_counts", "vote_n_res",
                                                            "vote_class_bar"]:
        assert np.array_equal(_bits(p[k][i]) if p[k].dtype == F32 else p[k][i],
                              _bits(q[k][j]) if q[k].dtype == F32 else q[k][j]), (what, k)
    for k in ("rois", "rois_ext"):
        assert np.array_equal(_bits(p[k][i][:, 1:]), _bits(q[k][j][:, 1:])), (what, k)
        assert np.all(p[k][i][:, 0] == i) and np.all(q[k][j][:, 0] == j), (what, k, "batch index")
    nr = int(p["vote_n_res"][i])
    for k in ("res_score", "res_class", "res_box_idx", "result_mask", "result_box"):
        a, b = p["vote_" + k][i][:nr], q["vote_" + k][j][:nr]
        assert np.array_equal(_bits(a) if a.dtype == F32 else a, _bits(b) if b.dtype == F32 else b), (what, k)


def _check_empty_image(q, j):
    """An image with no proposal: count 0, no valid row, no voted instance, finite record rows, and
    every RoI the padding row [j, 0, 0, 0, 0], so every stage-1 output row is the same."""
    assert q["roi_counts"][j] == 0 and q["rec_counts"][j] == 0
    assert np.all(q["valid"][j] == 0) and q["vote_n_res"][j] == 0
    for k in ("boxes", "scores", "masks"):
        assert np.isfinite(q[k][j]).all(), k
    assert np.all(q["rois"][j] == np.float32([j, 0, 0, 0, 0]))
    for k in ROW_BLOBS:
        assert np.array_equal(_bits(q[k][j]), np.broadcast_to(_bits(q[k][j][:1]), q[k][j].shape)), k


@pytest.mark.parametrize("precision", ["f16f8", "bf16x3"])
def test_engine_image_independent_of_its_batch(precision):
    """With the exponents frozen (measured on the first batch) and B fixed, nothing in a step
    couples images: conv tiles are per image, each FC output row depends on its own inputs,
    split-K is chosen from the shape and reduced in a fixed order, sort / NMS / voting run per
    image.  Image A in slot 0 of [A, B, C] and slot 1 of [D, A, E] gives the same bits in every
    blob, the record and the voting result, eagerly and through a CUDA graph captured on the
    first batch and replayed on the second; E (scale 100: no proposal) comes out empty."""
    from mnc_b200 import weights as Wt
    from mnc_b200.engine import MNCEngine
    eng = MNCEngine(Wt.make_weights(Wt.TINY_ARCH), precision=precision)
    P = _run_engine(eng, ["A", "B", "C"], graphed=False)
    Q = _run_engine(eng, ["D", "A", "E"], graphed=False)
    assert P["roi_counts"][0] > 0 and P["vote_n_res"][0] > 0
    _same_image(P, Q, 0, 1, "eager")
    _check_empty_image(Q, 2)
    Pg = _run_engine(eng, ["A", "B", "C"], graphed=True)
    Qg = _run_engine(eng, ["D", "A", "E"], graphed=True)
    for i in range(3):
        _same_image(P, Pg, i, i, "graph on its capture batch")
    _same_image(P, Qg, 0, 1, "graph replayed on the second batch")
    _check_empty_image(Qg, 2)

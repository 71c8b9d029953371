"""Exact float32 model of the device's cv2.resize(INTER_LINEAR) restatement (`cv_tap` in
mnc_b200/csrc/cv_resize.cuh, `lin_tap` in preprocess.cu) and of the six kernels that use it, the
mutants of its rule, and seeded masks with many samples on the 0.4 threshold.

The rule, per axis of n source samples resized to dst samples, scale = n / dst in double:
  fd = fma(d + 0.5, scale, -0.5) in double (one rounding), s = floor(fd), f = float32(fd - s);
  s < 0 -> s = 0, f = 0;   s >= n - 1 -> both taps n - 1, f = 0;   weights (1 - f, f) in float32;
then per sample the horizontal pass r_k = fl(fl(src[y_k, x0] a0) + fl(src[y_k, x1] a1)) for the two
source rows, and the vertical pass v = fl(fl(r0 b0) + fl(r1 b1)).  numpy's float32 arithmetic
rounds every product and sum once, as __fmul_rn / __fadd_rn do, so the model is plain numpy; the
coordinate's fused multiply-add is taken exactly with fractions.  A binarised sample is v >= 0.4f.

Mutants, for the teeth tests only (each is a plausible slip in a kernel):
  vfma    the vertical blend contracted:   v = fma(r1, b1, fl(r0 b0))
  hfma    the horizontal blends contracted: r_k = fma(src[y_k, x1], a1, fl(src[y_k, x0] a0))
  fcoord  the fraction from a float32 coordinate (OpenCV's own non-IPP path):
          c = float32(fd), s = floor(c), f = fl(c - s)
  vfirst  the vertical pass first, then the horizontal one
  gt      `>` for `>=` in the threshold

Tie fixtures: for a chosen sample, three of its taps keep their values and the fourth (the one of
largest weight) is solved for, then walked over float32 neighbours until the model gives 0.4f
exactly, or 1 or 2 ulps either side.  Every tap of a chosen sample is then locked, so samples placed
later never move it; many samples go into each mask."""
import functools
from fractions import Fraction

import numpy as np

from tests.nms_ties import fma_f32

F32 = np.float32
THRESH = F32(0.4)
MUTANTS = ("vfma", "hfma", "fcoord", "vfirst", "gt")
MODES = ("exact",) + MUTANTS
# target of each solved sample, in ulps of 0.4f (cycled): mostly exactly on it
OFFSETS = (0, 0, 0, 1, -1, 0, 2, -2)

# Largest distance, in float32 ulps (difference of the int32 bit patterns), seen between this model
# and cv2.resize(INTER_LINEAR) on float32 inputs in [0, 1), over the sizes test_cv_resize.py checks
# (21x21 to 1x1 ... 300x200, 42x42 and 84x84 to 21x21, 375x500 to 241x320 and 600x800).  Measured
# with opencv-python 4.13.0 on an Intel Xeon (AVX-512), default path: IPP on, IPP's AVX-512 code
# ("ippIP AVX-512F/CD/BW/DQ/VL (k0) 2022.2.0").  cv2's bits depend on whether IPP runs and on the
# CPU's dispatch level, so this bounds only that build on such a CPU; a binarised cv2 sample may
# differ from the device's only where the model's value lies within this many ulps of 0.4f.
CV2_ULPS = 16


def ulps_from(v, ref=THRESH):
    """Signed float32 ulp distance of v from ref (both positive)."""
    return (np.asarray(v, dtype=F32).view(np.int32).astype(np.int64) -
            np.asarray(ref, dtype=F32).view(np.int32).astype(np.int64))


def at_ulps(k):
    """0.4f moved by k float32 ulps."""
    return (np.array(THRESH).view(np.int32) + np.int32(k)).view(F32)


# ------------------------------------------------------------------------------------------------
# core
@functools.lru_cache(maxsize=4096)
def _coord(dst, scale):
    """fma(d + 0.5, scale, -0.5) for d < dst, correctly rounded to double."""
    s = Fraction(scale)
    return np.array([float(Fraction(2 * d + 1, 2) * s - Fraction(1, 2)) for d in range(dst)])


def taps(dst, n, scale, mode="exact"):
    """cv_tap / lin_tap for destination indices 0..dst-1 of an axis of n source samples
    -> (i0, i1, a0, a1): int64 index arrays and float32 weight arrays."""
    fd = _coord(int(dst), float(scale))
    if mode == "fcoord":
        c = fd.astype(F32)
        s = np.floor(c).astype(np.int64)
        f = (c - s.astype(F32)).astype(F32)
    else:
        s = np.floor(fd).astype(np.int64)
        f = (fd - s).astype(F32)
    neg = s < 0
    s = np.where(neg, 0, s)
    f = np.where(neg, F32(0), f)
    hi = s >= n - 1
    i0 = np.where(hi, n - 1, s)
    i1 = np.where(hi, n - 1, s + 1)
    f = np.where(hi, F32(0), f).astype(F32)
    return i0, i1, (F32(1) - f).astype(F32), f


def blend(p00, p01, p10, p11, ax0, ax1, ay0, ay1, mode="exact"):
    """One sample from its four taps (p_yx) and weights, in the kernels' order."""
    p00, p01, p10, p11 = (np.asarray(p, F32) for p in (p00, p01, p10, p11))
    if mode == "vfirst":
        c0 = p00 * ay0 + p10 * ay1
        c1 = p01 * ay0 + p11 * ay1
        return (c0 * ax0 + c1 * ax1).astype(F32)
    if mode == "hfma":
        r0, r1 = fma_f32(p01, ax1, p00 * ax0), fma_f32(p11, ax1, p10 * ax0)
    else:
        r0, r1 = p00 * ax0 + p01 * ax1, p10 * ax0 + p11 * ax1
    if mode == "vfma":
        return fma_f32(r1, ay1, r0 * ay0)
    return (r0 * ay0 + r1 * ay1).astype(F32)


def binarize(v, mode="exact", thresh=THRESH):
    return v > thresh if mode == "gt" else v >= thresh


def grid_taps(dw, dh, w, h, sx, sy, mode="exact"):
    """Taps of a (dh, dw) destination over an (h, w) source, broadcast to (dh, dw)."""
    x0, x1, ax0, ax1 = taps(dw, w, sx, mode)
    y0, y1, ay0, ay1 = taps(dh, h, sy, mode)
    return (y0[:, None], y1[:, None], x0[None, :], x1[None, :],
            ax0[None, :], ax1[None, :], ay0[:, None], ay1[:, None])


def resize(src, dw, dh, sx=None, sy=None, mode="exact"):
    """src (h, w) float32 -> (dh, dw) float32; sx, sy default to w / dw and h / dh."""
    src = np.asarray(src, F32)
    h, w = src.shape
    sx = w / dw if sx is None else sx
    sy = h / dh if sy is None else sy
    y0, y1, x0, x1, ax0, ax1, ay0, ay1 = grid_taps(dw, dh, w, h, sx, sy, mode)
    return blend(src[y0, x0], src[y0, x1], src[y1, x0], src[y1, x1], ax0, ax1, ay0, ay1, mode)


def ref64(src, dw, dh):
    """The same taps with float64 weights and arithmetic (fractions taken from the rounded
    coordinate in double, clamps as in the rule): a bilinear sample to bound the model against."""
    src = np.asarray(src, np.float64)
    h, w = src.shape

    def ax(dst, n):
        fd = _coord(dst, n / dst)
        s = np.floor(fd)
        f = fd - s
        s = s.astype(np.int64)
        f = np.where(s < 0, 0.0, f)
        s = np.maximum(s, 0)
        hi = s >= n - 1
        return np.where(hi, n - 1, s), np.where(hi, n - 1, s + 1), np.where(hi, 0.0, f)
    x0, x1, fx = ax(dw, w)
    y0, y1, fy = ax(dh, h)
    y0, y1, fy = y0[:, None], y1[:, None], fy[:, None]
    r0 = src[y0, x0] * (1 - fx) + src[y0, x1] * fx
    r1 = src[y1, x0] * (1 - fx) + src[y1, x1] * fx
    return r0 * (1 - fy) + r1 * fy


# ------------------------------------------------------------------------------------------------
# the six consumers
def prep(images, im_scale, means, mode="exact"):
    """prep_image_kernel: images uint8 (B, H, W, 3) BGR -> float32 (B, 3, oh, ow) with
    oh = rint(H * im_scale); pixels float32(double(p) - mean); scale 1 / im_scale in double."""
    B, H, W, _ = images.shape
    oh, ow = int(np.rint(H * im_scale)), int(np.rint(W * im_scale))
    inv = 1.0 / im_scale
    out = np.empty((B, 3, oh, ow), F32)
    for b in range(B):
        for c in range(3):
            plane = (images[b, :, :, c].astype(np.float64) - float(means[c])).astype(F32)
            out[b, c] = resize(plane, ow, oh, inv, inv, mode)
    return out


def round_boxes(boxes, H, W):
    """rintf (half to even) of float32 boxes, clipped to the image -> int64 (n, 4)."""
    r = np.rint(np.asarray(boxes, F32)[:, :4]).astype(np.int64)
    r[:, 0::2] = np.clip(r[:, 0::2], 0, W - 1)
    r[:, 1::2] = np.clip(r[:, 1::2], 0, H - 1)
    return r


def box_resize(mask, x1, y1, x2, y2, mode="exact"):
    """An (M, M) mask resized to the box's size (bh, bw), as paste / binarize do."""
    M = mask.shape[-1]
    bw, bh = x2 - x1 + 1, y2 - y1 + 1
    return resize(mask, bw, bh, M / bw, M / bh, mode)


def voc_color_map():
    """_get_voc_color_map (vis_seg.py:133-148): (256, 3) RGB."""
    cmap = np.zeros((256, 3), np.uint8)
    for i in range(256):
        cid, r, g, b = i, 0, 0, 0
        for j in range(8):
            r |= (cid & 1) << (7 - j)
            g |= ((cid >> 1) & 1) << (7 - j)
            b |= ((cid >> 2) & 1) << (7 - j)
            cid >>= 3
        cmap[i] = (r, g, b)
    return cmap


def paste(boxes, masks, cls, H, W, mode="exact"):
    """paste_instances_kernel for one image: instances painted in list order (later ones win),
    each box outline drawn into the class image with 150 after its mask (the numpy slices
    [a - 1 : a + 1], empty at a = 0).  -> inst int32 (H, W), cls int32 (H, W), bgr uint8 (H, W, 3),
    and close bool (H, W): some instance's resized value there lies within CV2_ULPS of 0.4f."""
    inst = np.zeros((H, W), np.int32)
    clsi = np.zeros((H, W), np.int32)
    close = np.zeros((H, W), bool)
    rb = round_boxes(boxes, H, W)
    for i, (x1, y1, x2, y2) in enumerate(rb):
        if x2 < x1 or y2 < y1:
            continue
        v = box_resize(np.asarray(masks[i], F32), x1, y1, x2, y2, mode)
        on = binarize(v, mode)
        ys, xs = slice(y1, y2 + 1), slice(x1, x2 + 1)
        inst[ys, xs] = np.where(on, i + 1, inst[ys, xs])
        clsi[ys, xs] = np.where(on, int(cls[i]), clsi[ys, xs])
        close[ys, xs] |= in_cv2_band(v)
        for a in (x1, x2):
            if a >= 1:
                clsi[y1:y2 + 1, a - 1:a + 1] = 150
        for a in (y1, y2):
            if a >= 1:
                clsi[a - 1:a + 1, x1:x2 + 1] = 150
    bgr = voc_color_map()[clsi & 255][:, :, ::-1]
    return inst, clsi, np.ascontiguousarray(bgr), close


def binarize_masks(rboxes, masks, mode="exact"):
    """binarize_masks_kernel: the packed uint8 masks and the n + 1 offsets (empty boxes: none)."""
    out, offs = [], [0]
    for (x1, y1, x2, y2), m in zip(np.asarray(rboxes, np.int64), masks):
        if x2 < x1 or y2 < y1:
            offs.append(offs[-1])
            continue
        b = binarize(box_resize(np.asarray(m, F32), x1, y1, x2, y2, mode), mode).astype(np.uint8)
        out.append(b.ravel())
        offs.append(offs[-1] + b.size)
    return (np.concatenate(out) if out else np.zeros(0, np.uint8)), np.array(offs, np.int64)


def _info_ints(mi):
    """The integer fields mask_target_row reads from a 12-float gt_mask_info record (C truncation)."""
    return [int(np.trunc(v)) for v in np.asarray(mi, F32)]


def ex_plane(mi, gt_masks):
    """The ex-box-sized plane of intersect_mask for the record mi, and for each of its pixels the
    (y, x) gt-mask position it reads, -1 where it reads 0 (outside the box intersection or the
    stored mask).  -> (plane float32 (eh, ew), gy (eh, ew), gx (eh, ew))."""
    a, mh, mw, _, ex1, ey1, ex2, ey2, gx1, gy1, gx2, gy2 = _info_ints(mi)
    G, Hm, Wm = gt_masks.shape
    ew, eh = ex2 - ex1 + 1, ey2 - ey1 + 1
    ix1, iy1, ix2, iy2 = max(ex1, gx1), max(ey1, gy1), min(ex2, gx2), min(ey2, gy2)
    yy, xx = np.mgrid[ey1:ey2 + 1, ex1:ex2 + 1]
    gy, gx = yy - gy1, xx - gx1
    live = ((xx >= ix1) & (xx <= ix2) & (yy >= iy1) & (yy <= iy2) & (gx < mw) & (gy < mh) &
            (gx < Wm) & (gy < Hm) & (0 <= a) & (a < G))
    gy, gx = np.where(live, gy, -1), np.where(live, gx, -1)
    plane = np.where(live, gt_masks[min(max(a, 0), G - 1)][np.maximum(gy, 0), np.maximum(gx, 0)],
                     F32(0)).astype(F32)
    return plane, gy, gx


def mask_target(mi, fg, gt_masks, M=21, mode="exact"):
    """mask_target_row: the (M, M) float32 0/1 target and weight of one row."""
    w = np.full((M, M), F32(1) if fg else F32(0))
    a, _, _, _, ex1, ey1, ex2, ey2, gx1, gy1, gx2, gy2 = _info_ints(mi)
    live = (fg and max(ex1, gx1) <= min(ex2, gx2) and max(ey1, gy1) <= min(ey2, gy2) and
            0 <= a < gt_masks.shape[0])
    if not live:
        return np.zeros((M, M), F32), w
    plane, _, _ = ex_plane(mi, gt_masks)
    eh, ew = plane.shape
    return binarize(resize(plane, M, M, ew / M, eh / M, mode), mode).astype(F32), w


def mask_targets(info, nfg, gt_masks, M=21, mode="exact"):
    """Every row of a layer's gt_mask_info; rows < nfg are foreground."""
    t = np.zeros((len(info), 1, M, M), F32)
    w = np.zeros((len(info), 1, M, M), F32)
    for p, mi in enumerate(info):
        t[p, 0], w[p, 0] = mask_target(mi, p < nfg, gt_masks, M, mode)
    return t, w


def in_cv2_band(v, ulps=None):
    """Samples within `ulps` (default CV2_ULPS) of 0.4f: where cv2 may binarise differently."""
    return np.abs(ulps_from(v)) <= (CV2_ULPS if ulps is None else ulps)


def mask_targets_cv2_band(info, nfg, gt_masks, M=21):
    """in_cv2_band() of every foreground row's unthresholded target plane, (K, 1, M, M)."""
    out = np.zeros((len(info), 1, M, M), bool)
    for p, mi in enumerate(info[:nfg]):
        plane, _, _ = ex_plane(mi, gt_masks)
        eh, ew = plane.shape
        if eh > 0 and ew > 0:
            out[p, 0] = in_cv2_band(resize(plane, M, M, ew / M, eh / M))
    return out


def mask_layer_cv2_band(preds, info):
    """Per row: some sample of its prediction resized to the ex box is in_cv2_band()."""
    out = np.zeros(len(info), bool)
    for i, mi in enumerate(np.asarray(info, F32)):
        if mi[0] == F32(-1):
            continue
        M = int(round(np.sqrt(np.size(preds[i]))))
        ex1, ey1, ex2, ey2 = (int(np.rint(v)) for v in mi[4:8])
        ew, eh = ex2 - ex1 + 1, ey2 - ey1 + 1
        if ew > 0 and eh > 0:
            out[i] = in_cv2_band(resize(np.asarray(preds[i], F32).reshape(M, M), ew, eh, M / ew, M / eh)).any()
    return out


def mask_layer_counts(pred, gt_masks, mi, mode="exact"):
    """mask_layer_train_kernel's integers for one RoI: (m1, inter, m2, disjoint).  pred (M*M,)."""
    M = int(round(np.sqrt(np.size(pred))))
    r = [int(np.rint(v)) for v in np.asarray(mi, F32)[4:12]]
    ex1, ey1, ex2, ey2, gx1, gy1, gx2, gy2 = r
    a, mh, mw = (int(np.trunc(v)) for v in np.asarray(mi, F32)[:3])
    G, Hm, Wm = gt_masks.shape
    ew, eh = ex2 - ex1 + 1, ey2 - ey1 + 1
    ix1, iy1, ix2, iy2 = max(ex1, gx1), max(ey1, gy1), min(ex2, gx2), min(ey2, gy2)
    has_gt = 0 <= a < G
    m1 = inter = m2 = 0
    if ew > 0 and eh > 0:
        on = binarize(resize(np.asarray(pred, F32).reshape(M, M), ew, eh, M / ew, M / eh, mode), mode)
        m1 = int(on.sum())
        if has_gt:
            yy, xx = np.mgrid[ey1:ey2 + 1, ex1:ex2 + 1]
            gy, gx = yy - gy1, xx - gx1
            ok = ((xx >= ix1) & (xx <= ix2) & (yy >= iy1) & (yy <= iy2) & (gx < mw) & (gy < mh) &
                  (gx < Wm) & (gy < Hm))
            g = np.zeros(on.shape, bool)
            g[ok] = gt_masks[a][gy[ok], gx[ok]] != 0
            inter = int((on & g).sum())
    if has_gt:
        m2 = int((gt_masks[a][:max(min(mh, Hm), 0), :max(min(mw, Wm), 0)] != 0).sum())
    return m1, inter, m2, not (ix1 <= ix2 and iy1 <= iy2)


def mask_iou(pred, gt_masks, mi, mode="exact"):
    """mask_overlap in double: 0 for disjoint boxes or a union below 1."""
    m1, inter, m2, disjoint = mask_layer_counts(pred, gt_masks, mi, mode)
    uni = float(m1) + m2 - inter
    return 0.0 if disjoint or uni < 1.0 else inter / uni


def mask_layer(preds, gt_masks, info, fg_seg_thresh=0.5, mode="exact"):
    """MaskLayer labels (N,) float32: 0 for rows whose info[0] == -1 or whose IoU < fg_seg_thresh,
    else info[3]."""
    out = np.zeros(len(info), F32)
    for i, mi in enumerate(np.asarray(info, F32)):
        if mi[0] == F32(-1):
            continue
        iou = mask_iou(preds[i], gt_masks, mi, mode)
        out[i] = F32(0) if iou < fg_seg_thresh else mi[3]
    return out


# ------------------------------------------------------------------------------------------------
# tie placement
def place_ties(rng, src, free, dw, dh, sx, sy, lock=None, max_ties=32, lo=-0.5, hi=1.5):
    """Edit src (h, w) float32 in place so that up to max_ties samples of its (dh, dw) resize sit
    on 0.4f or 1-2 ulps from it.  free: bool (h, w), the source pixels that may change (taps
    outside it keep their value).  lock: bool (h, w) updated in place with every tap of a chosen
    sample.  Solved taps stay in [lo, hi].  -> list of (dy, dx, ulps from 0.4f)."""
    h, w = src.shape
    lock = np.zeros((h, w), bool) if lock is None else lock
    y0, y1, x0, x1, ax0, ax1, ay0, ay1 = (np.broadcast_to(t, (dh, dw)) for t in
                                          grid_taps(dw, dh, w, h, sx, sy))
    placed = []
    for flat in rng.permutation(dh * dw):
        if len(placed) >= max_ties:
            break
        dy, dx = divmod(int(flat), dw)
        ys = (y0[dy, dx], y0[dy, dx], y1[dy, dx], y1[dy, dx])
        xs = (x0[dy, dx], x1[dy, dx], x0[dy, dx], x1[dy, dx])
        wts = (ax0[dy, dx], ax1[dy, dx], ay0[dy, dx], ay1[dy, dx])
        wk = [float(wts[0 if q % 2 == 0 else 1]) * float(wts[2 if q < 2 else 3]) for q in range(4)]
        k = int(np.argmax(wk))
        ty, tx = ys[k], xs[k]
        if not free[ty, tx] or lock[ty, tx]:
            continue
        # a tap read twice (clamped axis) must be the solved one in both places
        same = [q for q in range(4) if (ys[q], xs[q]) == (ty, tx)]
        base = [F32(src[ys[q], xs[q]]) for q in range(4)]
        off = OFFSETS[len(placed) % len(OFFSETS)]
        target = at_ulps(off)
        rest = sum(float(base[q]) * wk[q] for q in range(4) if q not in same)
        p = (0.4 - rest) / sum(wk[q] for q in same)
        if not lo <= p <= hi:
            continue
        steps = np.arange(-96, 97, dtype=np.int32)
        cand = (np.array(F32(p)).view(np.int32) + steps).view(F32)
        v = blend(*[cand if q in same else np.full(cand.shape, base[q]) for q in range(4)], *wts)
        hit = np.nonzero(v == target)[0]
        t = cand[hit[np.argmin(np.abs(steps[hit]))]] if hit.size else None
        if t is None or not lo <= float(t) <= hi:
            continue
        src[ty, tx] = t
        for q in range(4):
            lock[ys[q], xs[q]] = True
        placed.append((dy, dx, off))
    return placed


# ------------------------------------------------------------------------------------------------
# fixture sets: one per thresholded consumer, each spanning the geometries where the rule branches
def _masks(rng, n, M):
    return (1.0 / (1.0 + np.exp(-rng.normal(0, 2, (n, M, M))))).astype(F32)


# (M, x1, y1, x2, y2) of the paste / binarize boxes, in a 160 x 120 image: identity 21 -> 21,
# exact 2x and 4x downscales (M = 42, 84 into 21), upscales whose last columns / rows take the
# s >= n - 1 clamp, a 1-pixel box, 1-wide and 1-high boxes, and boxes past the image border
PASTE_BOXES = (
    (21, 2, 2, 22, 22), (42, 30, 2, 50, 22), (84, 60, 2, 80, 22),
    (21, 90, 2, 126, 38), (21, 130, 4, 159, 60), (21, 2, 30, 2, 30), (21, 6, 30, 6, 70),
    (21, 10, 30, 60, 30), (21, 20, 40, 70, 86), (21, 120, 80, 175, 140), (21, -8, 90, 30, 130),
    (21, 76, 44, 83, 119))


def paste_fixture(seed):
    """Instances of several mask sizes (grouped by M: the kernel takes one M per call) with ties.
    -> list of (M, boxes float32 (n, 4), masks (n, M, M), cls int32 (n,)), H, W."""
    rng = np.random.default_rng(seed)
    H, W = 120, 160
    groups = {}
    for M, x1, y1, x2, y2 in PASTE_BOXES:
        groups.setdefault(M, []).append((x1, y1, x2, y2))
    out = []
    for M, bl in sorted(groups.items()):
        boxes = (np.array(bl) + rng.uniform(-0.45, 0.45, (len(bl), 4))).astype(F32)
        masks = _masks(rng, len(bl), M)
        for i, (x1, y1, x2, y2) in enumerate(round_boxes(boxes, H, W)):
            bw, bh = x2 - x1 + 1, y2 - y1 + 1
            place_ties(rng, masks[i], np.ones((M, M), bool), bw, bh, M / bw, M / bh, max_ties=48)
        cls = rng.integers(1, 21, len(bl)).astype(np.int32)
        out.append((M, boxes, masks, cls))
    return out, H, W


def binarize_fixture(seed):
    """Rounded boxes (int32) and masks with ties, grouped by M.  -> list of (M, rboxes, masks)."""
    rng = np.random.default_rng(seed)
    groups = {}
    for M, x1, y1, x2, y2 in PASTE_BOXES:
        x1, y1 = max(x1, 0), max(y1, 0)
        groups.setdefault(M, []).append((x1, y1, x2, y2))
    groups[21] += [(0, 0, 0, 0), (5, 5, 4, 9)]                         # 1 pixel, empty (width 0)
    out = []
    for M, bl in sorted(groups.items()):
        rb = np.array(bl, np.int32)
        masks = _masks(rng, len(bl), M)
        for i, (x1, y1, x2, y2) in enumerate(rb):
            bw, bh = x2 - x1 + 1, y2 - y1 + 1
            if bw > 0 and bh > 0:
                place_ties(rng, masks[i], np.ones((M, M), bool), bw, bh, M / bw, M / bh, max_ties=48)
        out.append((M, rb, masks))
    return out


# gt box (x1, y1, x2, y2) and the ex boxes of the mask-target rows, image 200 x 160, im_scale 1:
# identity (21 wide ex box), 42 and 84 wide (exact 2x / 4x downscales), 1 wide and 1 high, 1 pixel,
# upscales (ex box < 21: the last samples take the clamp), ex boxes only partly covered by the gt
# crop (left / top / right of it), ex boxes that run past the stored mask's extent, and 1-wide /
# 1-high ex boxes on the image's right and bottom edges (x = 199, y = 159)
MT_GT = ((20, 10, 119, 109), (110, 60, 199, 159))
MT_EX = ((0, (30, 20, 50, 40)), (0, (25, 15, 66, 56)), (0, (30, 20, 113, 103)),
         (0, (40, 30, 40, 70)), (0, (40, 30, 80, 30)), (0, (60, 60, 60, 60)),
         (0, (70, 50, 82, 58)), (0, (5, 40, 45, 80)), (0, (60, 0, 100, 40)),
         (0, (90, 70, 130, 100)), (1, (150, 120, 199, 159)), (1, (100, 55, 150, 110)),
         (1, (120, 70, 141, 91)), (1, (112, 62, 195, 145)), (1, (199, 30, 199, 70)),
         (1, (120, 159, 170, 159)))


def mask_target_fixture(seed):
    """gt masks (float32, non-binary values allowed: the kernel reads floats) and 12-float
    gt_mask_info rows with ties in every row.  The second gt mask is stored smaller than its box,
    so part of its box reads 0.  -> (info (K, 12) float32, nfg, gt_masks (G, Hm, Wm) float32)."""
    rng = np.random.default_rng(seed)
    Hm, Wm = 100, 100
    G = len(MT_GT)
    gt_masks = rng.uniform(0, 1, (G, Hm, Wm)).astype(F32)
    gt_masks[rng.uniform(0, 1, gt_masks.shape) < 0.3] = 0
    sizes = ((100, 100), (80, 75))                                  # (mh, mw) stored per gt
    rows = []
    for g, ex in MT_EX:
        mh, mw = sizes[g]
        rows.append([g, mh, mw, 1 + g] + list(ex) + list(MT_GT[g]))
    info = np.array(rows, F32)
    lock = np.zeros((G, Hm, Wm), bool)
    for mi in info:
        mask_target_ties(rng, mi, gt_masks, lock)
    return info, len(info), gt_masks


def mask_target_ties(rng, mi, gt_masks, lock, max_ties=40, M=21):
    """Place ties in the M x M target of record mi by editing the gt mask pixels it reads; lock:
    bool (G, Hm, Wm), the pixels earlier ties read (shared across rows of one gt mask)."""
    plane, gy, gx = ex_plane(mi, gt_masks)
    eh, ew = plane.shape
    a = _info_ints(mi)[0]
    live = gy >= 0
    pl_lock = np.zeros(plane.shape, bool)
    pl_lock[live] = lock[a][gy[live], gx[live]]
    placed = place_ties(rng, plane, live, M, M, ew / M, eh / M, lock=pl_lock, max_ties=max_ties)
    gt_masks[a][gy[live], gx[live]] = plane[live]
    lock[a][gy[live], gx[live]] |= pl_lock[live]
    return placed


# MaskLayer rows: (M of the prediction, ex box, gt index); the ex box is the resize's destination,
# so these are upscales (clamped last samples), identity, 2x / 4x downscales (M = 42, 84 into 21),
# 1-wide / 1-high / 1-pixel boxes, and boxes partly outside the gt box
ML_ROWS = ((21, (30, 20, 50, 40), 0), (21, (25, 15, 66, 56), 0), (21, (30, 20, 113, 103), 0),
           (42, (40, 30, 60, 50), 0), (84, (50, 40, 70, 60), 0), (21, (40, 30, 40, 70), 0),
           (21, (40, 30, 80, 30), 0), (21, (60, 60, 60, 60), 0), (21, (5, 40, 45, 80), 0),
           (21, (100, 55, 150, 110), 1), (21, (112, 62, 195, 145), 1), (21, (120, 70, 127, 77), 1))


def mask_layer_fixture(seed):
    """MaskLayer inputs grouped by prediction size M (one call per M): predictions with ties,
    gt masks (float32 0/1 and other values: the kernel counts != 0) and info rows, one of them -1.
    -> (gt_masks, list of (M, preds (N, M*M), info (N, 12)))."""
    rng = np.random.default_rng(seed)
    _, _, gt_masks = mask_target_fixture(seed)
    sizes = ((100, 100), (80, 75))
    groups = {}
    for M, ex, g in ML_ROWS:
        mh, mw = sizes[g]
        groups.setdefault(M, []).append([g, mh, mw, 1 + g] + list(ex) + list(MT_GT[g]))
    out = []
    for M, rows in sorted(groups.items()):
        info = np.array(rows, F32)
        if M == 21:
            info = np.concatenate([info, np.full((1, 12), -1, F32)])
        preds = _masks(rng, len(info), M)
        for i, mi in enumerate(info):
            if mi[0] == -1:
                continue
            ex1, ey1, ex2, ey2 = (int(v) for v in mi[4:8])
            ew, eh = ex2 - ex1 + 1, ey2 - ey1 + 1
            place_ties(rng, preds[i], np.ones((M, M), bool), ew, eh, M / ew, M / eh, max_ties=48)
        out.append((M, preds.reshape(len(info), M * M), info))
    return gt_masks, out


def iou_thresholds(preds, gt_masks, info):
    """For each live row, its model IoU and the next double above it: as fg_seg_thresh these put
    the row's label on the edge, so one binarised bit more or less in m1 or inter flips it."""
    out = []
    for i, mi in enumerate(np.asarray(info, F32)):
        if mi[0] == F32(-1):
            continue
        iou = mask_iou(preds[i], gt_masks, mi)
        if iou > 0:
            out += [iou, float(np.nextafter(iou, np.inf))]
    return out

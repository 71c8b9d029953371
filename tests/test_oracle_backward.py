"""The C oracle's backward passes (oracle/mnc_oracle_backward.c) against independent numpy
float64 statements: the adjoint identity <fwd(x), g> = <x, bwd(g)> where the reference's backward
is the adjoint of its forward, and the adjoint minus exactly the terms the reference drops where it
is not (ROIWarping's feature window, MaskResize when upsampling).  CPU only."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import oracle_backward as OB

SS = 0.0625
f32 = np.float32


def _roundf(x):
    """C roundf (half away from zero) of float32 values, exactly."""
    x = np.asarray(x, np.float32).astype(np.float64)
    return (np.sign(x) * np.floor(np.abs(x) + 0.5)).astype(np.float32)


def _rois(R, seed, B, H, W, edge=True):
    rng = np.random.default_rng(seed)
    x1, y1 = rng.uniform(0, 16 * W - 17, R), rng.uniform(0, 16 * H - 17, R)
    rois = np.stack([rng.integers(0, B, R), x1, y1, np.minimum(x1 + rng.uniform(16, 400, R), 16 * W - 1),
                     np.minimum(y1 + rng.uniform(16, 400, R), 16 * H - 1)], 1)
    if edge:
        rois = np.vstack([[[0, 0, 0, 16 * W - 1, 16 * H - 1],     # whole map
                           [0, 100, 100, 100, 100],                # degenerate
                           [1, -300, -200, 40, 30],                # partly off the map
                           [1, 16 * W - 20, 16 * H - 20, 16 * W + 300, 16 * H + 300],   # past the edge
                           [0, 8, 8, 23.9, 24.1],                  # round-half cases
                           [0, 500, 300, 400, 200]], rois])        # inverted
    return rois.astype(np.float32)


def _dot(a, b):
    return float(np.sum(a.astype(np.float64) * b.astype(np.float64)))


def _close(a, b, scale, rtol=1e-5):
    assert abs(a - b) <= rtol * scale, (a, b, scale)


def test_mask_pool_adjoint():
    rng = np.random.default_rng(1)
    feat = rng.standard_normal((5, 7, 9, 11)).astype(np.float32)
    mask = rng.uniform(0, 1, (5, 1, 9, 11)).astype(np.float32)
    g = rng.standard_normal(feat.shape).astype(np.float32)
    fd, md = OB.mask_pool_backward(feat, mask, g)
    lhs = _dot(O.mask_pool(feat, mask), g)
    scale = float(np.sum(np.abs(feat.astype(np.float64) * mask * g)))
    _close(lhs, _dot(feat, fd), scale)
    _close(lhs, _dot(mask, md), scale)
    # mask_diff is the serial channel sum c = 0..C-1 in float (mask_pooling_layer.cu:69-72)
    want = np.zeros(mask.shape, np.float32)
    for c in range(feat.shape[1]):
        want[:, 0] = want[:, 0] + g[:, c] * feat[:, c]
    assert np.array_equal(md, want)
    assert np.array_equal(fd, g * mask)


def _resize_matrix(ih_n, iw_n, oh_n, ow_n):
    """Dense float64 matrix of MaskResize's forward (mask_resize_layer.cu:13-73) for one plane, and
    the mask of the (output, input) pairs the reference's backward visits (:146-170)."""
    rh, rw = f32(ih_n) / f32(oh_n), f32(iw_n) / f32(ow_n)

    def taps(x, dim):
        if x < -0.5 or x > dim - 0.5:
            return []
        x = max(x, f32(0))
        lo = int(x)
        if lo >= dim - 1:
            return [(dim - 1, 1.0)]
        lx = float(x) - lo
        return [(lo, 1.0 - lx), (lo + 1, lx)]

    M = np.zeros((oh_n * ow_n, ih_n * iw_n))
    for h in range(oh_n):
        for w in range(ow_n):
            for a, wa in taps(f32(h) * rh, ih_n):
                for b, wb in taps(f32(w) * rw, iw_n):
                    M[h * ow_n + w, a * iw_n + b] += wa * wb
    visit = np.zeros_like(M, dtype=bool)
    for h in range(ih_n):
        for w in range(iw_n):
            hs, ws = int(np.floor(f32(h) / rh)), int(np.floor(f32(w) / rw))
            for ph in (hs, hs + 1):
                for pw in (ws, ws + 1):
                    if ph < oh_n and pw < ow_n and abs(f32(pw) * rw - f32(w)) < 1 and abs(f32(ph) * rh - f32(h)) < 1:
                        visit[ph * ow_n + pw, h * iw_n + w] = True
    return M, visit


@pytest.mark.parametrize("oh,ow", [(14, 14), (7, 9), (21, 21), (28, 28)])
def test_mask_resize_adjoint(oh, ow):
    rng = np.random.default_rng(oh * 100 + ow)
    x = rng.uniform(0, 1, (6, 1, 21, 21)).astype(np.float32)
    g = rng.standard_normal((6, 1, oh, ow)).astype(np.float32)
    bwd = OB.mask_resize_backward(g, 21, 21)
    M, visit = _resize_matrix(21, 21, oh, ow)
    gm = g.reshape(6, -1).astype(np.float64)
    want = (gm @ (M * visit)).reshape(bwd.shape)
    scale = (np.abs(gm) @ np.abs(M)).reshape(bwd.shape)
    assert np.all(np.abs(bwd - want) <= 1e-5 * scale + 1e-30)
    dropped = np.count_nonzero(M * ~visit)
    if oh <= 21:
        # downsampling or identity: the backward is the forward's adjoint
        assert dropped == 0
        _close(_dot(O.mask_resize(x, oh, ow), g), _dot(x, bwd), float(np.sum(np.abs(gm) @ np.abs(M))))
    else:
        # upsampling 21 -> 28: an input row is reached by up to three output rows, the backward
        # visits two (DESIGN.md "Backward semantics")
        assert dropped > 0
        assert not np.allclose(bwd, (gm @ M).reshape(bwd.shape), rtol=1e-3, atol=1e-3)


def test_roi_pool_adjoint():
    rng = np.random.default_rng(3)
    B, C, H, W = 2, 5, 19, 27
    feat = rng.standard_normal((B, C, H, W)).astype(np.float32)
    rois = _rois(40, 4, B, H, W)
    rois = rois[rois[:, 3] >= rois[:, 1]]            # an inverted RoI's gradient is dropped, below
    for P in (7, 6):
        out, arg = O.roi_pool(feat, rois, P, P, return_argmax=True)
        g = rng.standard_normal(out.shape).astype(np.float32)
        fd = OB.roi_pool_backward(g, arg, feat.shape, rois, P, P)
        _close(_dot(out, g), _dot(feat, fd), float(np.sum(np.abs(out.astype(np.float64) * g))))
    # an inverted RoI (end < start) pools row / column `start`, which its in_roi test
    # (roi_pooling_layer.cu:123-124) excludes: no gradient
    inv = np.array([[0, 320, 160, 200, 100]], np.float32)
    out, arg = O.roi_pool(feat, inv, 7, 7, return_argmax=True)
    assert np.all(arg >= 0)
    assert not np.any(OB.roi_pool_backward(np.ones_like(out), arg, feat.shape, inv, 7, 7))


# ---------------------------------------------------------------------------------- ROIWarping
def _warp_geometry(roi, P, H, W):
    """Per axis: the forward's clamped sample coordinate (float32) or None (outside the map), from
    roi_warping_layer.cu:78-99 and :18-47, plus the backward's float32 window pieces (:197-233)."""
    sw, sh, ew, eh = _roundf(roi[1:5] * f32(SS))
    bin_f = (np.maximum(eh - sh, f32(0)) / f32(P), np.maximum(ew - sw, f32(0)) / f32(P))
    bin_b = (np.maximum(eh - sh + f32(1), f32(1)) / f32(P), np.maximum(ew - sw + f32(1), f32(1)) / f32(P))
    samples = []
    for start, b, dim in ((sh, bin_f[0], H), (sw, bin_f[1], W)):
        xs = start + np.arange(P, dtype=np.float32) * b
        ok = ~((xs < -0.5) | (xs > dim - 0.5))
        a = np.maximum(xs, f32(0))
        a = np.where(a.astype(np.int64) >= dim - 1, f32(dim - 1), a)
        samples.append((a, ok))
    return (sh, sw, eh, ew), bin_b, samples


def _warp_feature_adjoint(feat, rois, g, P):
    """float64 adjoint of the forward (all terms) and the same without the terms outside the
    reference's feasible window; also the counts of nonzero-weight terms kept / dropped per axis."""
    B, C, H, W = feat.shape
    full = np.zeros(feat.shape)
    kept = np.zeros(feat.shape)
    mag = np.zeros(feat.shape)
    stats = np.zeros((2, 2), np.int64)     # axis x (kept, dropped) of (tap, sample) pairs
    for r, roi in enumerate(rois):
        n = int(roi[0])
        (sh, sw, eh, ew), bin_b, ((ah, okh), (aw, okw)) = _warp_geometry(roi, P, H, W)
        terms = []                          # per axis: (index, sample, weight, in window)
        for axis, (a, ok, start, end, b, dim) in enumerate(
                ((ah, okh, sh, eh, bin_b[0], H), (aw, okw, sw, ew, bin_b[1], W))):
            t = []
            for p in range(P):
                lo = int(a[p])
                taps = [(lo, 1.0)] if lo >= dim - 1 else [(lo, 1.0 - (float(a[p]) - lo)), (lo + 1, float(a[p]) - lo)]
                for i, wt in taps:
                    if wt == 0:
                        continue
                    hf = f32(i)
                    s = int(np.floor((hf - start - f32(1)) / b - f32(1)))
                    e = int(np.ceil((hf - start + f32(1)) / b))
                    inside = (np.floor(start) <= hf <= np.ceil(end)) and max(min(s, P), 0) <= p < max(min(e, P), 0)
                    if ok[p] and okh.any() and okw.any():
                        stats[axis, 0 if inside else 1] += 1
                    t.append((i, p, wt, inside, ok[p]))
            terms.append(t)
        for (h, ph, wh, inh, okh_) in terms[0]:
            for (w, pw, ww, inw, okw_) in terms[1]:
                if not (okh_ and okw_):
                    continue
                contrib = wh * ww * g[r, :, ph, pw].astype(np.float64)
                full[n, :, h, w] += contrib
                mag[n, :, h, w] += np.abs(contrib)
                if inh and inw:
                    kept[n, :, h, w] += contrib
    return full, kept, mag, stats


@pytest.mark.parametrize("P", [28, 14, 7])
def test_roi_warp_feature_gradient_is_the_windowed_adjoint(P):
    rng = np.random.default_rng(P)
    B, C, H, W = 2, 3, 38, 63
    feat = rng.standard_normal((B, C, H, W)).astype(np.float32)
    rois = _rois(24, P, B, H, W)
    g = rng.standard_normal((rois.shape[0], C, P, P)).astype(np.float32)
    fd, _ = OB.roi_warp_backward(feat, rois, g, P, P)
    full, kept, mag, stats = _warp_feature_adjoint(feat, rois, g, P)
    assert np.all(np.abs(fd - kept) <= 1e-5 * mag + 1e-30)
    share = stats[:, 1] / stats.sum(1)
    print("P=%d dropped share of (tap, sample) pairs: rows %.3f, columns %.3f" % (P, share[0], share[1]))
    assert np.all(share > 0.05)
    # the reference's feature gradient is therefore not the adjoint of its forward
    assert np.abs(fd - full).max() > 1e-2 * np.abs(full).max()


def _coord_terms(feat, roi, g, P, H, W):
    """The reference's coordinate-gradient buffer values (roi_warping_layer.cu:248-359) for one RoI,
    k = 1..4, float32 / float64 exactly as the source promotes them -> (4, C, P, P) float32."""
    n = int(roi[0])
    sw, sh, ew, eh = (int(v) for v in _roundf(roi[1:5] * f32(SS)))
    bin_h = f32(max(eh - sh + 1, 1)) / f32(P)
    bin_w = f32(max(ew - sw + 1, 1)) / f32(P)
    _, _, ((ah, okh), (aw, okw)) = _warp_geometry(roi, P, H, W)
    C = feat.shape[1]
    out = np.zeros((4, C, P, P), np.float32)
    for ph in range(P):
        for pw in range(P):
            if not (okh[ph] and okw[pw]):
                continue                     # outside the map: 0 (the documented deviation)
            h, w = ah[ph], aw[pw]
            ai, aj = int(h), int(w)
            if ai + 1 > H - 1 or aj + 1 > W - 1:
                continue
            mrh = ((h - f32(sh)) / bin_h) / f32(P)
            mrw = ((w - f32(sw)) / bin_w) / f32(P)
            v = [feat[n, :, ai, aj], feat[n, :, ai, aj + 1], feat[n, :, ai + 1, aj], feat[n, :, ai + 1, aj + 1]]
            v = [x.astype(np.float64) for x in v]
            A = (1.0 - np.float64(h)) + ai
            Bh = np.float64(h - f32(ai))
            Aw = (1.0 - np.float64(w)) + aj
            Bw = np.float64(w - f32(aj))

            def acc(terms):
                s = np.zeros(C, np.float32)
                for t in terms:
                    s = (s.astype(np.float64) + t).astype(np.float32)
                return s
            dxc = acc([(-1.0 * A) * v[0], A * v[1], (-1.0 * Bh) * v[2], Bh * v[3]])
            dyc = acc([(-1.0 * Aw) * v[0], (-1.0 * Bw) * v[1], Aw * v[2], Bw * v[3]])
            dw = acc([((0.5 - np.float64(mrw)) * A) * v[0], ((-0.5 + np.float64(mrw)) * A) * v[1],
                      ((0.5 - np.float64(mrw)) * Bh) * v[2], ((-0.5 + np.float64(mrw)) * Bh) * v[3]])
            dh = acc([((0.5 - np.float64(mrh)) * Aw) * v[0], ((0.5 - np.float64(mrh)) * Bw) * v[1],
                      ((-0.5 + np.float64(mrh)) * Aw) * v[2], ((-0.5 + np.float64(mrh)) * Bw) * v[3]])
            ws = [0.5 * dxc.astype(np.float64) - dw, 0.5 * dyc.astype(np.float64) - dh,
                  0.5 * dxc.astype(np.float64) + dw, 0.5 * dyc.astype(np.float64) + dh]
            for k in range(4):
                out[k, :, ph, pw] = (f32(SS) * ws[k].astype(np.float32)) * g[:, ph, pw]
    return out


def test_roi_warp_coordinate_gradient():
    rng = np.random.default_rng(11)
    B, C, H, W = 2, 4, 20, 30
    feat = rng.standard_normal((B, C, H, W)).astype(np.float32)
    rois = _rois(10, 12, B, H, W)
    for P in (7, 14):
        g = rng.standard_normal((rois.shape[0], C, P, P)).astype(np.float32)
        _, rd, ra = OB.roi_warp_backward(feat, rois, g, P, P, want_abs=True)
        assert np.all(rd[:, 0] == 0)
        for r, roi in enumerate(rois):
            t = _coord_terms(feat, roi, g[r], P, H, W).astype(np.float64)
            s = t.reshape(4, -1).sum(1)
            m = np.abs(t).reshape(4, -1).sum(1)
            assert np.allclose(m, ra[r, 1:], rtol=1e-12, atol=0)
            assert np.all(np.abs(rd[r, 1:] - s) <= 1e-6 * m + 1e-30), (r, rd[r], s)
        assert np.abs(rd[:, 1:]).max() > 0

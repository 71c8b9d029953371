"""Exact float32 emulation of mask voting (`_mv`: render, aggregate, tight box, resample), and seeded
voting cases in which one pixel whose aggregate lies on the 0.4 threshold, or a few ulps from it,
decides one side of a result's tight box.

The arithmetic, as nvcc builds the reference (read from `cuobjdump -sass` of `_mv` for sm_90a):
  render     px = fl(fl(w - x1) * fl(M / fl(fl(x2 - x1) + 1))),  cx = floor(px),  fx = px - cx,
             the four bilinear weights tl = fl((1-fx)(1-fy)), tr = fl(fx(1-fy)), bl = fl((1-fx)fy),
             br = fl(fx fy) are plain products, and the blend is
               ref      fma(br, m3, fma(bl, m2, fma(tl, m0, fl(tr * m1))))   top-left tap fused
               swapped  fma(br, m3, fma(bl, m2, fma(tr, m1, fl(tl * m0))))   top-right tap fused
               nofma    fl(fl(fl(tl m0 + tr m1) + bl m2) + br m3)             no contraction
             (a sample in the last mask row or column takes one tap, no arithmetic);
  aggregate  v = fma(r_i, w_i, v) from v = 0 in list order (nofma: v = fl(v + fl(r_i w_i)));
  box        the outermost columns / rows holding a pixel with v > 0.4f, W/2 and H/2 when none does;
  resample   ix = fma(j, fl(fl(x2 - x1 + 1) / M), x1) (nofma: fl(x1 + fl(j * ratio))), the same
             4-tap blend over the aggregate, and the last image row / column taken as is.
`nofma` is the C oracle (-ffp-contract=off) and the reference built with -fmad=false.

Every case is built so that exactly one pixel decides one side: under `ref` its aggregate is
0.4f exactly or 1 to 30 ulps away, every other pixel of the case is far from 0.4, and turning that
pixel on or off moves the box.  The cases sit anywhere in a small image (results do not interact:
each aggregates its own candidates), and many are packed into one call per image."""
import functools

import numpy as np

from tests.nms_ties import fma_f32, round_f32  # noqa: F401  (round_f32: hand-checked cases)

F32 = np.float32
M = 21
THRESH = F32(0.4)
ROUNDINGS = ("ref", "swapped", "nofma")
ULP = F32(2.0 ** -25)                        # ulp of 0.4f
FAR = 1e-5                                   # every pixel but the deciding one is this far from 0.4
OFFSETS = (0,) * 16 + (1,) * 14 + (-1,) * 4 + (2, -2, 3, -3, 5, -5, 8, -8, 13, -13, 21, -21, 30, -30)


def ulps_from(v, ref=THRESH):
    return (np.asarray(v, dtype=F32).view(np.int32).astype(np.int64) -
            int(np.array(ref, dtype=F32).view(np.int32)))


# ------------------------------------------------------------------------------------------------
# emulation
def blend(tl, tr, bl, br, m0, m1, m2, m3, rounding):
    if rounding == "ref":
        return fma_f32(br, m3, fma_f32(bl, m2, fma_f32(tl, m0, tr * m1)))
    if rounding == "swapped":
        return fma_f32(br, m3, fma_f32(bl, m2, fma_f32(tr, m1, tl * m0)))
    if rounding == "nofma":
        return ((tl * m0 + tr * m1) + bl * m2) + br * m3
    raise ValueError(rounding)


def _weights(fx, fy):
    one = F32(1)
    return (one - fx) * (one - fy), fx * (one - fy), (one - fx) * fy, fx * fy


def render(box, mask, hh, ww, rounding="ref"):
    """mask_render of one candidate at pixels (hh, ww) (int arrays) -> float32 array.  mask:
    (M, M), or (n, M, M) with one mask per pixel of the flattened (hh, ww)."""
    x1, y1, x2, y2 = (F32(v) for v in box[:4])
    mask = np.asarray(mask, dtype=F32)
    mask = mask.reshape(-1, M, M) if mask.size > M * M else mask.reshape(1, M, M)
    inside = ~((ww < x1) | (ww > x2) | (hh < y1) | (hh > y2))
    out = np.zeros(np.shape(hh), dtype=F32)
    if not inside.any():
        return out
    h, w = hh[inside], ww[inside]
    k = np.arange(np.size(hh)).reshape(np.shape(hh))[inside] if len(mask) > 1 else np.zeros(len(h), int)
    rw = F32(M) / ((x2 - x1) + F32(1))
    rh = F32(M) / ((y2 - y1) + F32(1))
    px = (w.astype(F32) - x1) * rw
    py = (h.astype(F32) - y1) * rh
    cx, cy = np.floor(px).astype(np.int64), np.floor(py).astype(np.int64)
    assert cx.max() < M and cy.max() < M
    last = M - 1
    v = np.empty(len(h), dtype=F32)
    near = (cx == last) | (cy == last)
    both = (cx == last) & (cy == last)
    v[near] = np.where(both[near], mask[k[near], last, last], mask[k[near], cy[near], cx[near]])
    n = ~near
    if n.any():
        x, y, kk = cx[n], cy[n], k[n]
        tl, tr, bl, br = _weights(px[n] - x.astype(F32), py[n] - y.astype(F32))
        v[n] = blend(tl, tr, bl, br, mask[kk, y, x], mask[kk, y, x + 1], mask[kk, y + 1, x],
                     mask[kk, y + 1, x + 1], rounding)
    out[inside] = v
    return out


def aggregate(cands, hh, ww, rounding="ref"):
    """mask_aggregate: sum_i w_i * render_i in list order.  cands: [(box, mask, weight)]."""
    v = np.zeros(np.shape(hh), dtype=F32)
    for box, mask, wgt in cands:
        r = render(box, mask, hh, ww, rounding)
        v = fma_f32(r, F32(wgt), v) if rounding != "nofma" else v + r * F32(wgt)
    return v


def region(cands, H, W):
    """Union of the candidates' boxes (floor / ceil), clipped: outside it every render is 0."""
    b = np.array([c[0][:4] for c in cands], dtype=F32)
    return (max(int(np.floor(b[:, 0].min())), 0), max(int(np.floor(b[:, 1].min())), 0),
            min(int(np.ceil(b[:, 2].max())), W - 1), min(int(np.ceil(b[:, 3].max())), H - 1))


def tight_box(on, x0, y0, H, W):
    """reduce_mask_col/row + reduce_bounding_x/y over an on-map whose (0, 0) is pixel (y0, x0)."""
    if not on.any():
        return (W // 2, H // 2, W // 2, H // 2)
    yy, xx = np.nonzero(on)
    return (x0 + int(xx.min()), y0 + int(yy.min()), x0 + int(xx.max()), y0 + int(yy.max()))


def resample(cands, box, H, W, rounding="ref"):
    """mask_resize of the aggregate into box -> (M, M) float32."""
    x1, y1, x2, y2 = box
    rw = F32(x2 - x1 + 1) / F32(M)
    rh = F32(y2 - y1 + 1) / F32(M)
    j = np.arange(M, dtype=F32)
    if rounding == "nofma":
        ix, iy = F32(x1) + j * rw, F32(y1) + j * rh
    else:
        ix, iy = fma_f32(j, rw, F32(x1)), fma_f32(j, rh, F32(y1))
    IX, IY = np.meshgrid(ix, iy)                 # [h, w]
    sx, sy = np.floor(IX).astype(np.int64), np.floor(IY).astype(np.int64)
    near = (sx == W - 1) | (sy == H - 1)
    # pixels the output reads: the nearest one, or the 4 of the blend
    px = np.where(near, sx, sx)[..., None] + np.where(near[..., None], 0, np.array([0, 1, 0, 1]))
    py = np.where(near, sy, sy)[..., None] + np.where(near[..., None], 0, np.array([0, 0, 1, 1]))
    both = (sx == W - 1) & (sy == H - 1)
    px[both], py[both] = W - 1, H - 1
    a = aggregate(cands, py.ravel(), px.ravel(), rounding).reshape(py.shape)
    tl, tr, bl, br = _weights(IX - sx.astype(F32), IY - sy.astype(F32))
    v = blend(tl, tr, bl, br, a[..., 0], a[..., 1], a[..., 2], a[..., 3], rounding)
    return np.where(near, a[..., 0], v).astype(F32)


def emulate(cands, H, W, rounding="ref", force=None):
    """`_mv` for one result -> (box, mask).  force = ((h, w), on): that pixel's decision imposed."""
    x0, y0, x1, y1 = region(cands, H, W)
    if x1 < x0 or y1 < y0:
        on = np.zeros((1, 1), bool)
    else:
        hh, ww = np.mgrid[y0:y1 + 1, x0:x1 + 1]
        on = aggregate(cands, hh, ww, rounding) > THRESH
        if force is not None:
            (h, w), val = force
            on[h - y0, w - x0] = val
    box = tight_box(on, x0, y0, H, W)
    return box, resample(cands, box, H, W, rounding)


# ------------------------------------------------------------------------------------------------
# the kernel's two shortcuts for images whose masks lie in [0, 1] and weights are >= 0
def rel_margin(n):
    """mask_voting.cu mv_rel_margin: 1 + (n + 4) 2^-21 for a list of n candidates."""
    return F32(1) + F32(n + 4) * F32(2.0 ** -21)


def early_exit(renders, weights, old=False):
    """agg_exceeds_unit: the predicate `sum > 0.4` walked with its exits.  renders / weights: the
    list's terms at one pixel, float32.  old=True: the exit before the fix, fma(suf, 1.0001, val)."""
    n = len(weights)
    suf = np.zeros(n + 1, dtype=F32)
    for i in range(n - 1, -1, -1):
        suf[i] = suf[i + 1] + weights[i]
    rel = rel_margin(n)
    val = F32(0)
    for i in range(n):
        bound = (fma_f32(suf[i], F32(1.0001), val) if old else fma_f32(suf[i], rel, val) * rel)
        if bound <= THRESH:
            return False
        val = fma_f32(renders[i], weights[i], val)
        if val > THRESH:
            return True
    return bool(val > THRESH)


def covering_cut(boxes, weights, h, w, old=False):
    """The search-region cut: column w and row h are searched iff their covering weight
    u = sum of w_i over the boxes containing them (float32, list order) passes fl(u * rel) > 0.4."""
    boxes = np.asarray(boxes, dtype=F32)
    ux = uy = F32(0)
    for b, wt in zip(boxes, weights):
        if not (w < b[0] or w > b[2]):
            ux = ux + F32(wt)
        if not (h < b[1] or h > b[3]):
            uy = uy + F32(wt)
    m = F32(1.0001) if old else rel_margin(len(weights))
    return bool(ux * m > THRESH) and bool(uy * m > THRESH)


# ------------------------------------------------------------------------------------------------
# cases
SIDES = ("left", "top", "right", "bottom")


def _inward(side):
    return {"left": (0, 1), "right": (0, -1), "top": (1, 0), "bottom": (-1, 0)}[side]


def _body(rng, h0, w0, side, unit):
    """A candidate whose whole box is on, next to the deciding pixel on the inward side."""
    dh, dw = _inward(side)
    lo, hi = rng.integers(1, 8, 2), rng.integers(2, 20)
    if dw:
        xa, xb = (w0 + 1, w0 + hi) if dw > 0 else (w0 - hi, w0 - 1)
        ya, yb = h0 - lo[0], h0 + lo[1]
    else:
        ya, yb = (h0 + 1, h0 + hi) if dh > 0 else (h0 - hi, h0 - 1)
        xa, xb = w0 - lo[0], w0 + lo[1]
    j = rng.uniform(0, 0.9, 4)
    box = np.array([xa - j[0], ya - j[1], xb + j[2], yb + j[3]], dtype=F32)
    mask = rng.uniform(0.8, 1.0, (M, M)).astype(F32)
    if not unit:
        mask[rng.integers(0, M), rng.integers(0, M)] = F32(1.25)
    return box, mask, F32(rng.uniform(0.7, 0.9))


def _pin_box(rng, h0, w0, kind):
    """A box that covers pixel (h0, w0) and, along each thin axis, no other column / row."""
    def thin(p):
        if kind == "int_edge" and rng.random() < 0.5:
            return (F32(p), F32(p) + F32(rng.uniform(0, 0.9))) if rng.random() < 0.5 else \
                   (F32(p) - F32(rng.uniform(0, 0.9)), F32(p))
        a = rng.uniform(0, 0.6)
        return F32(p) - F32(a), F32(p) + F32(rng.uniform(0, 0.95 - a))

    def last_cell(p):
        b = rng.uniform(0, 0.5)
        a = 20 * (1 + b) + rng.uniform(0.02, 0.25) * (1 + b)     # px in [20, 20.3)
        return F32(p) - F32(a), F32(p) + F32(b)

    x = last_cell(w0) if kind in ("nearest_x", "nearest_xy") else thin(w0)
    y = last_cell(h0) if kind in ("nearest_y", "nearest_xy") else thin(h0)
    return np.array([x[0], y[0], x[1], y[1]], dtype=F32)


def _under(rng, h0, w0, n, budget, unit):
    out = []
    wts = rng.dirichlet(np.ones(n)) * budget
    for k in range(n):
        e = rng.uniform(0, 8, 4)
        box = np.array([w0 - e[0], h0 - e[1], w0 + e[2], h0 + e[3]], dtype=F32)
        mask = rng.uniform(0, 1, (M, M)).astype(F32)
        wt = F32(wts[k])
        if not unit and k == 0:
            wt = F32(-0.02)                     # a negative weight: the full-sum path
        out.append((box, mask, wt))
    return out


def _pin_tap(box, h0, w0, finest=False):
    """(row, col) of the pin mask tap with the largest weight at the deciding pixel (finest: with
    the smallest non-zero weight, whose steps move the aggregate by the least)."""
    x1, y1, x2, y2 = box
    px = (F32(w0) - x1) * (F32(M) / ((x2 - x1) + F32(1)))
    py = (F32(h0) - y1) * (F32(M) / ((y2 - y1) + F32(1)))
    cx, cy = int(np.floor(px)), int(np.floor(py))
    if cx == M - 1 or cy == M - 1:
        return (M - 1, M - 1) if cx == cy == M - 1 else (cy, cx)
    tl, tr, bl, br = _weights(px - F32(cx), py - F32(cy))
    wts = np.array([tl, tr, bl, br])
    k = int(np.argmin(np.where(wts > 0, wts, 2))) if finest else int(np.argmax(wts))
    return cy + k // 2, cx + k % 2


def _tune(cands, pin, tap, h0, w0, target, hi):
    """Smallest pin tap value in [0, hi] whose `ref` aggregate at (h0, w0) is >= target."""
    hh, ww = np.array([h0]), np.array([w0])
    mask = cands[pin][1]

    def agg(bits):
        mask[tap] = np.array(bits, dtype=np.int32).view(F32)
        return aggregate(cands, hh, ww)[0]

    lo, top = 0, int(np.array(hi, dtype=F32).view(np.int32))
    if agg(top) < target:
        return None
    while lo < top:
        mid = (lo + top) // 2
        if agg(mid) >= target:
            top = mid
        else:
            lo = mid + 1
    return agg(top)


def _disagree(cands, pin, tap, h0, w0, other, reach=4000):
    """Move the tuned tap by up to `reach` float32 steps to the nearest value where the `ref`
    aggregate is still 0.4f or the next float32 up and `other` decides the other way."""
    mask = cands[pin][1]
    base = int(np.array(mask[tap]).view(np.int32))
    d = np.arange(-reach, reach + 1)
    masks = np.repeat(mask[None], len(d), 0)
    masks[(slice(None),) + tap] = (base + d).astype(np.int32).view(F32)
    var = list(cands)
    var[pin] = (cands[pin][0], masks, cands[pin][2])
    hh, ww = np.full(len(d), h0), np.full(len(d), w0)
    ref, oth = aggregate(var, hh, ww, "ref"), aggregate(var, hh, ww, other)
    ok = np.isin(ulps_from(ref), (0, 1)) & ((ref > THRESH) != (oth > THRESH))
    if ok.any():
        mask[tap] = masks[np.flatnonzero(ok)[np.argmin(np.abs(d[ok]))]][tap]


def _decider(rng, H, W, side, kind, border):
    """Deciding pixel: on the image border for `border`, else with room for the body."""
    m = 24 if kind.startswith("nearest") else 10
    h0, w0 = int(rng.integers(m, H - m)), int(rng.integers(m, W - m))
    if border:
        if side == "left":
            w0 = 0
        elif side == "right":
            w0 = W - 1
        elif side == "top":
            h0 = 0
        else:
            h0 = H - 1
    return h0, w0


def make_case(rng, H, W, kind, unit, n_under, side=None, border=False, spacer=False):
    """One result -> dict(cands, tie, side, kind, ...) or None when the draw fails a check."""
    side = side or SIDES[rng.integers(0, 4)]
    h0, w0 = _decider(rng, H, W, side, kind, border)
    body = [] if kind in ("single", "empty") else [_body(rng, h0, w0, side, unit)]
    under = _under(rng, h0, w0, n_under, 0.22 if kind.startswith("nearest") else 0.3, unit) \
        if kind != "single" else []
    pbox = _pin_box(rng, h0, w0, kind)
    pmask = np.zeros((M, M), dtype=F32) if kind.startswith("nearest") else \
        rng.uniform(0.1, 0.6, (M, M)).astype(F32)
    pin = (pbox, pmask, F32(rng.uniform(0.6, 1.0)))
    items = under + [pin] + body
    perm = rng.permutation(len(items))                     # list order: pin and body anywhere
    cands = [items[i] for i in perm]
    pin_at = int(np.flatnonzero(perm == len(under))[0])
    if spacer:
        q, p = int(rng.integers(2, 4)), int(rng.integers(2, 4))
        if w0 - 6 * q < 0 or h0 - 6 * p < 0:
            return None
        sp = np.array([w0 - 6 * q, h0 - 6 * p, min(w0 + 25, W - 1), min(h0 + 25, H - 1)], dtype=F32)
        cands.append((sp, np.zeros((M, M), dtype=F32), F32(0.45)))     # adds 0 everywhere
    offset = 0 if kind == "empty" and rng.random() < 0.5 else int(rng.choice(OFFSETS))
    if kind == "empty":
        offset = -abs(offset)
    target = (np.array(THRESH).view(np.int32) + np.int32(offset)).view(F32)
    tap = _pin_tap(pbox, h0, w0)
    got = _tune(cands, pin_at, tap, h0, w0, target, F32(1.0) if unit else F32(1.2))
    if got is None or abs(ulps_from(got)) > 30:
        return None
    if offset in (0, 1):
        _disagree(cands, pin_at, _pin_tap(pbox, h0, w0, finest=True), h0, w0, "swapped" if rng.random() < 0.75 else "nofma")
    return _check({"cands": cands, "tie": (h0, w0), "side": side, "kind": kind, "unit": unit,
                   "border": border}, H, W)


def trap_case(rng, H, W, n_tail):
    """The tiny-tail-weight trap of an early exit whose margin is relative to the remaining weight:
    the pin leaves 0.4f - (n_tail - 1) ulps, then n_tail candidates of render 1 and weight
    0.5..0.6 ulp(0.4f) each round the sum up by one ulp, to 0.4f + 1 ulp; their total weight is
    below n_tail - 1 ulps, so a bound of partial + 1.0001 * remaining weight rounds to <= 0.4f."""
    side = SIDES[rng.integers(0, 4)]
    h0, w0 = _decider(rng, H, W, side, "trap", False)
    one = np.ones((M, M), dtype=F32)
    dot = np.array([w0, h0, w0 + 0.5, h0 + 0.5], dtype=F32)       # px = py = 0: render = mask[0, 0]
    start = (np.array(THRESH).view(np.int32) - np.int32(n_tail - 1)).view(F32)
    cands = [_body(rng, h0, w0, side, True), (dot, one, start)]
    cands += [(dot.copy(), one, F32(rng.uniform(0.5, 0.6)) * ULP) for _ in range(n_tail)]
    return _check({"cands": cands, "tie": (h0, w0), "side": side, "kind": "trap", "unit": True,
                   "border": False}, H, W)


def _check(case, H, W):
    """Emulate under every rounding; keep the case if only the deciding pixel is near 0.4, the
    roundings agree elsewhere, and its decision moves the box."""
    cands, (h0, w0) = case["cands"], case["tie"]
    x0, y0, x1, y1 = region(cands, H, W)
    hh, ww = np.mgrid[y0:y1 + 1, x0:x1 + 1]
    aggs = {r: aggregate(cands, hh, ww, r) for r in ROUNDINGS}
    near = np.abs(aggs["ref"].astype(np.float64) - 0.4) < FAR
    near[h0 - y0, w0 - x0] = False
    if near.any():
        return None
    on = aggs["ref"] > THRESH
    on[h0 - y0, w0 - x0] = True
    box_on = tight_box(on, x0, y0, H, W)
    on[h0 - y0, w0 - x0] = False
    box_off = tight_box(on, x0, y0, H, W)
    if box_on == box_off:
        return None
    case["agg"] = {r: F32(aggs[r][h0 - y0, w0 - x0]) for r in ROUNDINGS}
    case["offset"] = int(ulps_from(case["agg"]["ref"]))
    case["boxes_if"] = {True: box_on, False: box_off}
    case["expect"] = {}
    for r in ROUNDINGS:
        box = box_on if case["agg"][r] > THRESH else box_off
        case["expect"][r] = (box, resample(cands, box, H, W, r))
    case["region"] = (x0, y0, x1, y1)
    return case


# images: (H, W, unit range, seed).  Non-unit images hold a mask value 1.25 or a weight -0.02, so
# the device takes the full-sum path for the whole image.
IMAGES = ((150, 200, True, 1), (123, 171, True, 2), (150, 200, False, 3), (97, 131, False, 4))
PLAN = (["interp"] * 46 + ["int_edge"] * 10 + ["nearest_x"] * 5 + ["nearest_y"] * 5 +
        ["nearest_xy"] * 3 + ["border"] * 8 + ["single"] * 3 + ["empty"] * 4 + ["long"] * 2 +
        ["spacer"] * 8)
UNDER_COUNTS = (0, 1, 2, 3, 4, 6, 9)


@functools.lru_cache(maxsize=None)
def image_cases(index):
    """-> (H, W, unit, cases) for IMAGES[index]; traps in the unit images."""
    H, W, unit, seed = IMAGES[index]
    rng = np.random.default_rng([7, seed])
    cases = []
    for what in PLAN:
        for _ in range(200):
            kind = {"border": "interp", "long": "interp", "spacer": "interp"}.get(what, what)
            n_under = int(rng.integers(280, 420)) if what == "long" else int(rng.choice(UNDER_COUNTS))
            c = make_case(rng, H, W, kind, unit, n_under, border=what == "border",
                          spacer=what == "spacer")
            if c is not None:
                c["plan"] = what
                cases.append(c)
                break
        else:
            raise RuntimeError("no case for %s" % what)
    if unit:
        for n_tail in (2, 2, 3, 5):
            for _ in range(50):
                c = trap_case(rng, H, W, n_tail)
                if c is not None:
                    c["plan"] = "trap"
                    cases.append(c)
                    break
            else:
                raise RuntimeError("no trap case")
    return H, W, unit, cases


def pack(cases):
    """-> `_mv` arguments (boxes [nb, 4], masks [nb, 1, M, M], inds, END offsets, weights)."""
    boxes, masks, inds, start, wts = [], [], [], [], []
    for c in cases:
        for box, mask, wt in c["cands"]:
            inds.append(len(boxes))
            boxes.append(box)
            masks.append(mask)
            wts.append(wt)
        start.append(len(inds))
    return (np.array(boxes, dtype=F32), np.array(masks, dtype=F32)[:, None],
            np.array(inds, dtype=np.int32), np.array(start, dtype=np.int32), np.array(wts, dtype=F32))


def expected(cases, rounding="ref"):
    """-> (boxes [k, 4] int32, masks [k, 1, M, M] float32) under `rounding`."""
    return (np.array([c["expect"][rounding][0] for c in cases], dtype=np.int32),
            np.array([c["expect"][rounding][1] for c in cases], dtype=F32)[:, None])


def on_coarse_grid(case, H, W, stride=6):
    """Whether the deciding pixel is on the device's coarse-pass grid, whose origin is the search
    region: the covering-weight cut of the union region in unit images, the union region else."""
    x0, y0, x1, y1 = region(case["cands"], H, W)
    if case["unit"]:
        boxes = [c[0] for c in case["cands"]]
        wts = [c[2] for c in case["cands"]]
        rel = rel_margin(len(wts))
        cols = [w for w in range(x0, x1 + 1)
                if F32(sum_f32(wts, [not (w < b[0] or w > b[2]) for b in boxes])) * rel > THRESH]
        rows = [h for h in range(y0, y1 + 1)
                if F32(sum_f32(wts, [not (h < b[1] or h > b[3]) for b in boxes])) * rel > THRESH]
        x0, y0 = min(cols), min(rows)
    h0, w0 = case["tie"]
    return (h0 - y0) % stride == 0 and (w0 - x0) % stride == 0


def sum_f32(wts, take):
    u = F32(0)
    for wt, t in zip(wts, take):
        if t:
            u = u + F32(wt)
    return u

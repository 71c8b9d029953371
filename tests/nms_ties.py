"""Exact float32 emulation of the NMS suppression test `IoU(a, b) > t`, and score-sorted box lists
whose keep list shows the test's decision at IoUs that round to within a few ulps of `t`.

devIoU (+1 convention, a = the earlier box) is  I / (Sa + Sb - I),  and a compiler may contract one
of the two area products into the sum.  The three roundings of the union U:
  ref      fl(fma(bw, bh, Sa) - I)      the reference `_nms` as nvcc builds it (later box fused)
  swapped  fl(fma(aw, ah, Sb) - I)      the earlier box fused instead
  nofma    fl(fl(Sa + Sb) - I)          no contraction: the C oracle, `-fmad=false` builds
with Sa = fl(aw * ah), Sb = fl(bw * bh), I = fl(w * h) and every other step a float32 operation.
Where the two areas are inexact the three U can differ by an ulp, and so can fl(I / U): at a
ratio within an ulp or two of the threshold that flips the decision.

The pairs are built so that the `ref` quotient lands exactly on t, or a given number of ulps
from it; every pair has its own cell far from all others, so in a list of many pairs a box can
only be suppressed by its partner (or by an identical copy of the partner) and the keep list
shows every pair's decision."""
import functools
from fractions import Fraction

import numpy as np

F32 = np.float32
ROUNDINGS = ("ref", "swapped", "nofma")
THRESHOLDS = (0.7, 0.5, 0.3)
FAST_BAND = 1e-6            # nms_suppresses decides without the division outside I = t*U*(1 +- 1e-6)
CELL = 1024.0


# ------------------------------------------------------------------------------------------------
# float32 arithmetic
def round_f32(x):
    """Fraction -> nearest float32, ties to even (normal range; the boxes here stay in it)."""
    if x == 0:
        return F32(0.0)
    sign = -1 if x < 0 else 1
    x = abs(x)
    e = x.numerator.bit_length() - x.denominator.bit_length()    # 2^e <= x < 2^(e+2)
    if Fraction(2) ** e > x:
        e -= 1
    elif Fraction(2) ** (e + 1) <= x:
        e += 1
    scaled = x * Fraction(2) ** (23 - e)                           # in [2^23, 2^24)
    m, rem = divmod(scaled.numerator, scaled.denominator)
    twice = 2 * rem
    if twice > scaled.denominator or (twice == scaled.denominator and m % 2 == 1):
        m += 1
    return F32(sign * float(Fraction(m) * Fraction(2) ** (e - 23)))


def fma_f32_exact(x, y, z):
    """fmaf(x, y, z): x*y + z rounded once to float32 (scalars)."""
    return round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z)))


def fma_f32(x, y, z):
    """fmaf(x, y, z) over float32 arrays.  x*y is exact in float64 (48 bits); TwoSum gives
    x*y + z = s + err exactly.  Rounding s to float32 is then right unless s sits exactly halfway
    between two float32 values while err != 0, where err decides the direction."""
    x, y, z = (np.asarray(v, dtype=F32) for v in (x, y, z))
    p = x.astype(np.float64) * y.astype(np.float64)
    c = z.astype(np.float64)
    s = p + c
    bv = s - p
    err = (p - (s - bv)) + (c - bv)
    r = s.astype(F32)
    r64 = r.astype(np.float64)
    toward = np.nextafter(r, np.where(s > r64, F32(np.inf), F32(-np.inf)).astype(F32))
    halfway = (s != r64) & (2.0 * (s - r64) == toward.astype(np.float64) - r64)
    flip = halfway & (err != 0) & ((err > 0) == (s > r64))
    return np.where(flip, toward, r).astype(F32)


def _terms(a, b):
    """Widths, heights and the intersection of devIoU, float32; a, b: (..., 4)."""
    a = np.asarray(a, dtype=F32)
    b = np.asarray(b, dtype=F32)
    one, zero = F32(1), F32(0)
    w = np.maximum((np.minimum(a[..., 2], b[..., 2]) - np.maximum(a[..., 0], b[..., 0])) + one, zero)
    h = np.maximum((np.minimum(a[..., 3], b[..., 3]) - np.maximum(a[..., 1], b[..., 1])) + one, zero)
    aw, ah = (a[..., 2] - a[..., 0]) + one, (a[..., 3] - a[..., 1]) + one
    bw, bh = (b[..., 2] - b[..., 0]) + one, (b[..., 3] - b[..., 1]) + one
    return w * h, aw, ah, bw, bh


def union(a, b, rounding="ref"):
    inter, aw, ah, bw, bh = _terms(a, b)
    if rounding == "ref":
        s = fma_f32(bw, bh, aw * ah)
    elif rounding == "swapped":
        s = fma_f32(aw, ah, bw * bh)
    elif rounding == "nofma":
        s = aw * ah + bw * bh
    else:
        raise ValueError(rounding)
    return inter, s - inter


def quotient(a, b, rounding="ref"):
    inter, uni = union(a, b, rounding)
    with np.errstate(divide="ignore", invalid="ignore"):
        return inter / uni


def suppresses(a, b, thresh, rounding="ref"):
    """devIoU(a, b) > thresh, a the earlier box; NaN (0 / 0) compares false as on the device."""
    return quotient(a, b, rounding) > F32(thresh)


def in_fast_band(a, b, thresh):
    """nms_suppresses leaves the decision to the division: U > 0 and I within t*U*(1 +- 1e-6)."""
    inter, uni = union(a, b, "ref")
    tu = F32(thresh) * uni
    return (uni > 0) & ~(inter > tu * F32(1 + FAST_BAND)) & ~(inter < tu * F32(1 - FAST_BAND))


def ulps_from(q, thresh):
    """Signed distance of positive float32 q from float32(thresh), in ulps."""
    return (np.asarray(q, dtype=F32).view(np.int32).astype(np.int64) -
            int(np.array(thresh, dtype=F32).view(np.int32)))


# ------------------------------------------------------------------------------------------------
# pairs
# quotient offsets from t in ulps: mostly t itself and the next float32 up, where one ulp of U
# decides; the wider ones straddle the edge of the +-1e-6 fast-path band (about 12 ulps from t at
# t = 0.7, 10 at t = 0.3)
OFFSETS = (0,) * 12 + (1,) * 12 + (-1, -1, -1, 2, -2, 3, -3, 5, -5, 8, -8, 12, -12, 15, -15, 16, -16,
                                   17, -17, 18, -18, 20, -20, 24, -24, 30, -30)


def _with_x2(b, x2):
    out = b.copy()
    out[:, 2] = x2
    return out


def _search_pairs(a, b, lo, hi, to_f32, target):
    """Per row: the smallest x2 = to_f32(v), v in [lo, hi], whose `ref` quotient with a is >= target
    (IoU grows with b's x2 while b's right edge stays inside a's)."""
    lo, hi = lo.copy(), hi.copy()
    while np.any(lo < hi):
        mid = (lo + hi) // 2
        ge = quotient(a, _with_x2(b, to_f32(mid))) >= target
        hi = np.where(ge, mid, hi)
        lo = np.where(ge, lo, mid + 1)
    return _with_x2(b, to_f32(hi))


def _near_threshold_pairs(rng, thresh, count, origins, integer):
    """`count` tries: b shrinks a's box a little in y and x1, then b's x2 is searched so that the
    `ref` quotient lands on t plus an offset drawn from OFFSETS (ulps)."""
    ox, oy = origins
    lo_side, hi_side = (1000.0, 4000.0) if integer else (20.0, 700.0)
    sw = np.exp(rng.uniform(np.log(lo_side), np.log(hi_side), count))
    sh = np.exp(rng.uniform(np.log(lo_side), np.log(hi_side), count))
    x1 = ox + rng.uniform(0.5, 20, count)
    y1 = oy + rng.uniform(50, 100, count)
    a = np.stack([x1, y1, x1 + sw, y1 + sh], 1)
    b = np.stack([x1 + rng.uniform(0, 0.05, count) * sw, y1 + rng.uniform(-0.05, 0.05, count) * sh,
                  x1 + sw, y1 + sh + rng.uniform(-0.05, 0.05, count) * sh], 1)
    if integer:
        a, b = np.round(a), np.round(b)
    a, b = a.astype(F32), b.astype(F32)
    target = (np.array(thresh, dtype=F32).view(np.int32) +
              rng.choice(OFFSETS, count).astype(np.int32)).view(F32)
    if integer:
        to_f32 = lambda v: v.astype(F32)                                 # noqa: E731
        lo, hi = b[:, 0].astype(np.int64), a[:, 2].astype(np.int64)
    else:
        to_f32 = lambda v: v.astype(np.int32).view(F32)                  # noqa: E731
        lo, hi = b[:, 0].view(np.int32).astype(np.int64), a[:, 2].view(np.int32).astype(np.int64)
    b = _search_pairs(a, b, lo, hi, to_f32, target)
    ok = np.abs(ulps_from(quotient(a, b), thresh)) <= max(OFFSETS)
    return a[ok], b[ok]


def _exact_ratio_pairs(thresh, count, x0, y0):
    """Integer boxes sharing x1 and rows, widths in the ratio t = num / den: IoU is t exactly and
    fl(IoU) == float32(t), which must not suppress; one pixel wider must."""
    num, den = {0.7: (7, 10), 0.5: (1, 2), 0.3: (3, 10)}[thresh]
    pairs = []
    for k in range(count):
        m, rows = 1 + 3 * k, 5 + 7 * k
        x, y = x0 + k * CELL, y0
        a = [x, y, x + den * m - 1, y + rows - 1]
        pairs.append((a, [x, y, x + num * m - 1 + (k % 2), y + rows - 1]))
    return (np.array([p[0] for p in pairs], dtype=F32), np.array([p[1] for p in pairs], dtype=F32))


EDGE_KINDS = ("identical", "touch_x", "touch_y", "overlap_ulp", "zero_width_inside", "zero_width_both")


def edge_pairs(x0, y0):
    """Identical boxes; boxes touching in x or y (+1 intersection width exactly 0) or overlapping
    by one float32 ulp; a zero-width box (x2 = x1 - 1) inside a box, and two zero-width boxes
    (I = U = 0: the quotient is NaN).  Ordered as EDGE_KINDS, repeated for three box shapes."""
    pa, pb = [], []
    one = F32(1)
    for x, y, w, h in ((0.25, 0.5, 99.75, 60.125), (10.0, 20.0, 41.0, 77.0), (3.3, 7.7, 250.9, 130.1)):
        for kind in EDGE_KINDS:
            bx, by = F32(x0 + len(pa) * CELL + x), F32(y0 + y)
            a = np.array([bx, by, bx + F32(w), by + F32(h)], dtype=F32)
            b = a.copy()
            if kind in ("touch_x", "overlap_ulp"):
                b[[0, 2]] = a[2] + one, a[2] + one + F32(w)
                if kind == "overlap_ulp":
                    b[0] = np.nextafter(b[0], F32(-np.inf))
            elif kind == "touch_y":
                b[[1, 3]] = a[3] + one, a[3] + one + F32(h)
            elif kind == "zero_width_inside":
                b[2] = b[0] - one
            elif kind == "zero_width_both":
                a[2] = a[0] - one
                b[[0, 2]] = a[0] + F32(2), a[0] + one
            pa.append(a)
            pb.append(b)
    return np.array(pa, dtype=F32), np.array(pb, dtype=F32)


@functools.lru_cache(maxsize=None)
def pair_pool(thresh, seed=0):
    """(a, b, kind) for one threshold: fractional and integer near-threshold pairs, exact-ratio
    integer ties and the edge pairs, each pair in a cell of its own."""
    rng = np.random.default_rng([seed, int(round(thresh * 1000)) % 1000])
    # stacked along y with x near 0, so that one ulp of b's x2 moves the quotient by a few ulps
    n = 4000
    a1, b1 = _near_threshold_pairs(rng, thresh, n, (np.zeros(n), np.arange(n) * CELL), integer=False)
    a2, b2 = _near_threshold_pairs(rng, thresh, n, (2048.0 + np.arange(n) * 4608.0, np.zeros(n)),
                                   integer=True)
    a3, b3 = _exact_ratio_pairs(thresh, 24, 2048.0, -20000.0)
    a4, b4 = edge_pairs(2048.0, -40000.0)
    kind = (["fractional"] * len(a1) + ["integer"] * len(a2) + ["ratio"] * len(a3) +
            ["edge"] * len(a4))
    return np.concatenate([a1, a2, a3, a4]), np.concatenate([b1, b2, b3, b4]), np.array(kind)


# ------------------------------------------------------------------------------------------------
# lists
def layout(rng, ids, n_dups, dup_ok):
    """Score order of the pairs `ids` plus n_dups extra copies of their first boxes -> rows of
    (pair, role) with role 0 = a, 1 = b, 2 = copy of a.  a always comes before b; the gap is short
    (mostly the same 64-box block), medium (mostly a later block of the same 256-box round) or
    long."""
    n_pairs = len(ids)
    n = 2 * n_pairs + n_dups
    ka = rng.uniform(0, n, n_pairs)
    kind = rng.integers(0, 3, n_pairs)
    gap = np.where(kind == 0, rng.uniform(0.5, 12, n_pairs),
                   np.where(kind == 1, rng.uniform(12, 250, n_pairs), rng.uniform(250, n, n_pairs)))
    dup_src = rng.choice(np.flatnonzero(dup_ok[ids]), n_dups) if n_dups else np.zeros(0, int)
    kd = ka[dup_src] + rng.uniform(0, n, n_dups)
    keys = np.concatenate([ka, ka + gap, kd])
    entries = np.concatenate([np.stack([ids, np.zeros(n_pairs, int)], 1),
                              np.stack([ids, np.ones(n_pairs, int)], 1),
                              np.stack([ids[dup_src], np.full(n_dups, 2)], 1)])
    return entries[np.argsort(keys, kind="stable")]


def boxes_of(entries, pool):
    a, b, _ = pool
    return np.where((entries[:, 1] == 1)[:, None], b[entries[:, 0]], a[entries[:, 0]]).astype(F32)


def greedy_keep(boxes, thresh, rounding="ref", max_keep=0):
    """Greedy NMS over score-sorted boxes with the emulated predicate (the `_nms` keep list)."""
    n = len(boxes)
    removed = np.zeros(n, dtype=bool)
    keep = []
    for i in range(n):
        if removed[i]:
            continue
        keep.append(i)
        if len(keep) == max_keep:
            break
        removed[i + 1:] |= suppresses(boxes[i][None], boxes[i + 1:], thresh, rounding)
    return np.array(keep, dtype=np.int32)


# (t, name) -> one launch's problems.  The list's pairs come from pair_pool(t) for t > 0 and from
# pair_pool(0.3) for t <= 0 (there any overlap, or for t < 0 any box of positive area, suppresses).
# "small": n_max < 1024, the suppression-matrix form; "big": n_max >= 1024 and 4 * max_keep <= n_max,
# the capped forms.  Problem 2 of "big" is mostly copies, so that it has fewer survivors than
# max_keep; problem 1 is the first list cut short by a count.
LISTS = {"small": dict(n_max=1000, counts=(1000, 937, 400), max_keep=0),
         "big": dict(n_max=4096, counts=(4096, 4059, 3000), max_keep=1024)}
LISTS_NONPOSITIVE = {"small": dict(n_max=600, counts=(600, 571, 200), max_keep=0),
                     "big": dict(n_max=1100, counts=(1100, 1063, 900), max_keep=275)}


@functools.lru_cache(maxsize=None)
def tie_lists(thresh, name):
    """-> (boxes float32 [3, n_max, 4] in score order, entries per problem, counts, max_keep)."""
    pool = pair_pool(thresh if thresh > 0 else 0.3)
    a, b, kind = pool
    cfg = (LISTS if thresh > 0 else LISTS_NONPOSITIVE)[name]
    n_max, max_keep = cfg["n_max"], cfg["max_keep"]
    rng = np.random.default_rng([1, int(round(thresh * 1000)) % 1000, n_max])
    # copies of a box must suppress each other: self-IoU > t (positive area)
    dup_ok = (kind != "edge") & suppresses(a, a, max(thresh, 0.0))
    edges = np.flatnonzero(kind == "edge")
    others = np.flatnonzero(kind != "edge")
    boxes = np.zeros((3, n_max, 4), dtype=F32)
    entries = []
    for p in range(3):
        n_pairs = (max_keep or n_max) // 3 if p == 2 else min(len(a), (n_max - 16) // 2)
        ids = np.concatenate([edges, rng.choice(others, n_pairs - len(edges), replace=False)])
        e = layout(rng, ids, n_max - 2 * n_pairs, dup_ok)
        if thresh < 0:
            # a box of zero area first: against it every quotient is 0 / Sb = 0 > t (suppressed)
            # or, for another zero-area box, 0 / 0 = NaN (kept)
            first = np.flatnonzero((e[:, 0] == edges[EDGE_KINDS.index("zero_width_both")]) & (e[:, 1] == 0))
            e = np.concatenate([e[first], np.delete(e, first, 0)])
        entries.append(e)
        boxes[p] = boxes_of(e, pool)
    return boxes, entries, list(cfg["counts"]), max_keep


def expected_keep(thresh, name, rounding="ref"):
    """Per problem: the keep list of greedy NMS over the first counts[p] boxes, cut at max_keep."""
    boxes, _, counts, max_keep = tie_lists(thresh, name)
    return [greedy_keep(boxes[p, :counts[p]], thresh, rounding, max_keep) for p in range(len(counts))]


def observable_pairs(thresh, name, p, differ_from="swapped"):
    """Pairs of problem p whose `ref` decision differs from the `differ_from` rounding (None: whose
    `ref` quotient is t or the next float32 up, where an error of one ulp flips the decision) and
    shows in the keep list (both boxes within the count, b before the walk stops at max_keep)
    -> (position of a, position of b, index of a in the keep list) arrays."""
    boxes, entries, counts, max_keep = tie_lists(thresh, name)
    e = entries[p][:counts[p]]
    keep = expected_keep(thresh, name)[p]
    stop = keep[-1] if max_keep and len(keep) == max_keep else counts[p]
    pos_a = {int(pair): i for i, (pair, role) in enumerate(e) if role == 0}
    ia, ib = [], []
    for j, (pair, role) in enumerate(e):
        if role == 1 and j < stop and int(pair) in pos_a:
            ia.append(pos_a[int(pair)])
            ib.append(j)
    ia, ib = np.array(ia, dtype=int), np.array(ib, dtype=int)
    b = boxes[p]
    if differ_from is None:
        differ = np.isin(ulps_from(quotient(b[ia], b[ib]), thresh), (0, 1))
    else:
        differ = suppresses(b[ia], b[ib], thresh, "ref") != suppresses(b[ia], b[ib], thresh, differ_from)
    ia, ib = ia[differ], ib[differ]
    return ia, ib, np.searchsorted(keep, ia)

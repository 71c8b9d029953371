"""Shapes where the RoI layers' kernels take their shape-dependent branches: one case table shared
by the CPU witness (tests/test_roi_shapes.py), which checks that each case reaches the branch it
was written for, and the GPU tests of ROIWarping / ROIPooling / MaskResize / MaskPooling forward
and backward (tests/test_gpu_roi.py, test_gpu_roi_backward.py, test_gpu_siblings.py).

The GPU tests keep their (2, 40, 38, 63) inputs as one entry each; the table adds:
  training   the ROIWarping of the MNC training net: 512 channels of conv5_3, 64 RoIs clustered on
             3 gt boxes as ProposalTargetLayer emits them -- one 8 x 32 feature tile meets more
             than 2 chunks of 16 RoIs, and the coordinate gradient sums 8 slabs of 64 channels
  tail_c*    channel counts that leave partial channel groups: backward slabs of 8, forward slabs
             of 16 / 32, row-walk plane groups of 8 (28 x 28) and 4 (14 x 14)
  many_rois  ~700 RoIs spread unevenly over 3 images, image 2 with none: tiles meet RoIs in
             several 256-RoI compaction rounds
  generic    pooled sizes that take the generic forward kernel, and a ROIPooling size past the
             backward's 32 limit
  map_*      1 x 1, 3 x 5, 9 x 130 (five tile columns) and portrait 63 x 38 maps at spatial scales
             1/32, 1, 1/8 and 1/32
Every RoI's batch index lies in [0, B): the kernels read the feature blob at it."""
import functools
from dataclasses import dataclass

import numpy as np

F32 = np.float32


@dataclass(frozen=True)
class Case:
    name: str
    B: int
    C: int
    H: int
    W: int
    gen: str              # RoI generator, a key of GENERATORS
    pooled: tuple         # (ph, pw) sizes every layer runs at
    scale: float          # spatial scale
    reaches: tuple        # branches the case is written for (tests/test_roi_shapes.py)
    seed: int = 0
    pool_only: tuple = ()  # ROIPooling forward only: larger than the backward's 32 limit


# ------------------------------------------------------------------------------------------------
# RoI generators: (case, rng) -> float32 (R, 5) in image coordinates (map coordinates / scale)
def _to_image(level, m, scale):
    """Map-coordinate boxes (n, 4) -> RoI rows in image coordinates."""
    return np.hstack([np.asarray(level, F32)[:, None], (np.asarray(m, np.float64) / scale)]).astype(F32)


def edge_rois(B, H, W, scale):
    """The edge RoIs of the layer tests, in map coordinates scaled to the image.  Row 3 lies
    entirely outside the map (every sample is out of range: zero output, zero gradients)."""
    m = np.array([[0, 0, W - 1 / 16, H - 1 / 16],       # whole map
                  [W / 2, H / 2, W / 2, H / 2],         # degenerate: every cell samples one point
                  [-20, -12, 3, 2],                     # partly off the map (negative start)
                  [W + 3, H + 4, W + 15, H + 20],       # entirely outside
                  [W - 2, H - 2, W + 20, H + 20],       # runs past the far edge
                  [0.5, 1.5, W - 1.5, H - 0.5],         # x * scale = k + 0.5: roundf away from zero
                  [0.6 * W, 0.6 * H, 0.3 * W, 0.2 * H]])   # inverted (end < start)
    level = np.arange(len(m)) % B
    return _to_image(level, m, scale)


def _random_rois(rng, n, B, H, W, scale, centre=None, spread=None):
    """Centres uniform over the map (or normal around `centre` with sd `spread`), sizes
    log-uniform from one cell to the map's larger side."""
    if centre is None:
        cx, cy = rng.uniform(-1, W + 1, n), rng.uniform(-1, H + 1, n)
    else:
        cx, cy = rng.normal(centre[0], spread, n), rng.normal(centre[1], spread, n)
    big = max(H, W) * 1.2
    w, h = np.exp(rng.uniform(0, np.log(big), n)), np.exp(rng.uniform(0, np.log(big), n))
    m = np.stack([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2], 1)
    return _to_image(rng.integers(0, B, n), m, scale)


def _gen_random(case, rng):
    return np.vstack([edge_rois(case.B, case.H, case.W, case.scale),
                      _random_rois(rng, 41, case.B, case.H, case.W, case.scale)])


def _gen_training(case, rng):
    """64 RoIs jittered around 3 gt boxes (fg and bg RoIs of ProposalTargetLayer overlap their gt
    box), clipped to the image; two of the boxes share the tile rows 8-15 of tile column 0."""
    Hi, Wi = case.H / case.scale, case.W / case.scale
    gt = np.array([[90, 70, 360, 310], [230, 140, 520, 420], [600, 200, 940, 560]], np.float64)
    k = rng.choice(3, 64, p=[0.4, 0.35, 0.25])
    g = gt[k]
    size = np.repeat(g[:, 2:] - g[:, :2], 2, axis=1)[:, [0, 2, 1, 3]]
    b = g + rng.uniform(-0.3, 0.3, (64, 4)) * size
    b[:, 0::2] = np.clip(b[:, 0::2], 0, Wi - 1)
    b[:, 1::2] = np.clip(b[:, 1::2], 0, Hi - 1)
    return np.hstack([np.zeros((64, 1)), b]).astype(F32)


def _gen_many(case, rng):
    """700 RoIs in random index order: 470 on image 0 (two thirds of them crowded around one
    spot), 230 on image 1, none on image 2."""
    H, W, s = case.H, case.W, case.scale
    parts = [_random_rois(rng, 310, 1, H, W, s, centre=(14, 11), spread=6),
             _random_rois(rng, 153, 1, H, W, s),
             _random_rois(rng, 230, 1, H, W, s)]
    parts[2][:, 0] = 1
    edge = edge_rois(2, H, W, s)
    r = np.vstack(parts)[rng.permutation(693)]
    return np.vstack([edge, r]).astype(F32)


GENERATORS = {"random": _gen_random, "training": _gen_training, "many": _gen_many}

ALL_SIZES = ((28, 28), (14, 14), (7, 7), (9, 5))
GENERIC_SIZES = ((1, 1), (3, 17), (28, 14), (32, 32))

CASES = (
    Case("training", 1, 512, 38, 63, "training", ((28, 28), (14, 14)), 1 / 16,
         ("chunks>2", "coord_slabs>1")),
    Case("tail_c1", 2, 1, 38, 63, "random", ALL_SIZES, 1 / 16,
         ("slab_tail", "fwd_slab_tail", "rowwalk_tail"), seed=1),
    Case("tail_c13", 2, 13, 38, 63, "random", ALL_SIZES, 1 / 16,
         ("slab_tail", "fwd_slab_tail", "rowwalk_tail"), seed=13),
    Case("tail_c42", 2, 42, 38, 63, "random", ALL_SIZES, 1 / 16,
         ("slab_tail", "fwd_slab_tail", "rowwalk_tail"), seed=42),
    Case("tail_c72", 2, 72, 38, 63, "random", ALL_SIZES, 1 / 16,
         ("coord_slabs>1", "fwd_slab_tail", "rowwalk_cta_tail"), seed=72),
    Case("many_rois", 3, 24, 38, 63, "many", ((7, 7), (14, 14)), 1 / 16,
         ("rounds>1", "chunks>2", "empty_image"), seed=700),
    Case("generic", 2, 20, 38, 63, "random", GENERIC_SIZES, 1 / 16,
         ("generic", "slab_tail", "fwd_slab_tail"), seed=5, pool_only=((40, 40),)),
    Case("map_1x1", 2, 9, 1, 1, "random", ((7, 7), (28, 28)), 1 / 32,
         ("partial_tile", "slab_tail"), seed=11),
    Case("map_3x5", 1, 5, 3, 5, "random", ((14, 14), (9, 5)), 1.0,
         ("partial_tile", "slab_tail"), seed=35),
    Case("map_9x130", 2, 16, 9, 130, "random", ((28, 28), (7, 7)), 1 / 8,
         ("tile_cols>=5", "partial_tile"), seed=9),
    Case("map_63x38", 2, 24, 63, 38, "random", ((14, 14), (3, 17)), 1 / 32,
         ("partial_tile", "generic"), seed=63),
)
BY_NAME = {c.name: c for c in CASES}

# MaskResize backward: (N, C, in_h, in_w) <- (out_h, out_w); MaskPooling: (N, C, H, W)
MASK_RESIZE_BWD = {"resize_700": ((700, 1, 21, 21), (14, 14))}
MASK_POOL = {"pool_64x512": (64, 512, 14, 14), "pool_1400": (1400, 2, 14, 14)}


# ------------------------------------------------------------------------------------------------
# inputs (cached: several tests share them; callers must not modify them)
@functools.lru_cache(maxsize=None)
def rois(name):
    c = BY_NAME[name]
    return np.ascontiguousarray(GENERATORS[c.gen](c, np.random.default_rng([c.seed, 1])), dtype=F32)


@functools.lru_cache(maxsize=None)
def feat(name):
    c = BY_NAME[name]
    return np.random.default_rng([c.seed, 2]).standard_normal((c.B, c.C, c.H, c.W)).astype(F32)


def top_diff(name, ph, pw):
    c = BY_NAME[name]
    return np.random.default_rng([c.seed, 3, ph, pw]).standard_normal(
        (rois(name).shape[0], c.C, ph, pw)).astype(F32)


def outside_rows(name):
    """Indices of the RoIs that lie entirely outside the map (row 3 of edge_rois)."""
    return [] if BY_NAME[name].gen == "training" else [3]


def sizes(pool_only=False, max_pooled=32):
    """(case name, ph, pw) over the table, for pytest parametrization."""
    out = []
    for c in CASES:
        for ph, pw in c.pooled + (c.pool_only if pool_only else ()):
            if pool_only or max(ph, pw) <= max_pooled:
                out.append((c.name, ph, pw))
    return out


def size_id(name, ph, pw):
    return "%s-%dx%d" % (name, ph, pw)

"""CPU witness of the RoI case table (tests/roi_shapes.py): with the kernels' launch constants
restated, each case reaches the branch it was written for.  A later edit to a generator that drops
a case back onto the shapes every other test already covers fails here, without a GPU.

Restated from mnc_b200/csrc/roi_backward.cu and roi_ops.cu:
  feature gradients (ROIWarping, ROIPooling): a CTA owns an 8 x 32 tile of one image and 8
    channels; it compacts the RoIs meeting the tile 256 RoI indices at a time (a round) and, for
    ROIWarping, stages them 16 at a time (a chunk)
  coordinate gradient: one CTA per (RoI, 64-channel slab), the slabs summed in a second kernel
  forward: 16 channels per CTA (7 x 7 and generic sizes, ROIPooling), 32 per CTA for the 28 x 28
    and 14 x 14 row walk, whose lanes walk 8 (28 x 28) or 4 (14 x 14) planes together
  grid-stride kernels: blocks = min(ceil(n / threads), cap)."""
import math

import numpy as np
import pytest

from tests import roi_shapes as RS
from tests.test_oracle_backward import _roundf

K_TILE_H, K_TILE_W, K_TILE_THREADS = 8, 32, 256
K_CHUNK, K_SLAB, K_COORD_SLAB = 16, 8, 64
K_WARP_SLAB, K_ROWWALK_CPC = 16, 32
ROWWALK_CH = {28: 8, 14: 4}
K_MAX_POOLED = 32
SMS = 132


def tile_round_hits(case):
    """hits[n, tile row, tile column, round]: RoIs of round `round` (indices 256 * round ...) whose
    rounded rectangle meets the tile -- the compaction test of roi_warp_bwd_feat_kernel
    (floorf / ceilf of the roundf'ed corners) and of roi_pool_bwd_kernel (the same integers)."""
    rois = RS.rois(case.name)
    sw, sh, ew, eh = _roundf(rois[:, 1:5] * np.float32(case.scale)).T
    th, tw = math.ceil(case.H / K_TILE_H), math.ceil(case.W / K_TILE_W)
    rounds = math.ceil(len(rois) / K_TILE_THREADS)
    hits = np.zeros((case.B, th, tw, rounds), np.int64)
    h0 = np.arange(th)[:, None] * K_TILE_H
    w0 = np.arange(tw)[None, :] * K_TILE_W
    for i, roi in enumerate(rois):
        meet = ((np.floor(sw[i]) <= w0 + K_TILE_W - 1) & (np.ceil(ew[i]) >= w0) &
                (np.floor(sh[i]) <= h0 + K_TILE_H - 1) & (np.ceil(eh[i]) >= h0))
        hits[int(roi[0]), :, :, i // K_TILE_THREADS] += meet
    return hits


def warp_dispatch(ph, pw):
    """Which ROIWarping forward kernel mnc_roi_warp_nchw launches."""
    if ph == pw and ph in (28, 14):
        return "rowwalk%d" % ph
    return "nchw7" if (ph, pw) == (7, 7) else "generic"


def rowwalk_partial_group(C, P):
    """Some lane of roi_warp_rowwalk_kernel<P> walks a plane group cut by the CTA's channel count:
    its tail planes re-read plane 0 and must not be stored."""
    return any(min(K_ROWWALK_CPC, C - c0) % ROWWALK_CH[P] for c0 in range(0, C, K_ROWWALK_CPC))


def grid_passes(n, threads, cap):
    blocks = min(max(-(-n // threads), 1), cap)
    return -(-n // (blocks * threads))


def reached(case):
    hits = tile_round_hits(case)
    rois = RS.rois(case.name)
    out = set()
    if hits.max() > 2 * K_CHUNK:
        out.add("chunks>2")
    if ((hits > 0).sum(axis=3) >= 2).any():
        out.add("rounds>1")
    if len(set(rois[:, 0].astype(int))) < case.B:
        out.add("empty_image")
    if case.C % K_SLAB:
        out.add("slab_tail")
    if -(-case.C // K_COORD_SLAB) > 1:
        out.add("coord_slabs>1")
    if case.C % K_WARP_SLAB:
        out.add("fwd_slab_tail")
    if case.C % K_ROWWALK_CPC:
        out.add("rowwalk_cta_tail")
    walks = [p for p, q in case.pooled if warp_dispatch(p, q).startswith("rowwalk")]
    if walks and all(rowwalk_partial_group(case.C, p) for p in walks):
        out.add("rowwalk_tail")
    if any(warp_dispatch(*s) == "generic" for s in case.pooled):
        out.add("generic")
    if case.H % K_TILE_H or case.W % K_TILE_W:
        out.add("partial_tile")
    if math.ceil(case.W / K_TILE_W) >= 5:
        out.add("tile_cols>=5")
    return out


@pytest.mark.parametrize("name", [c.name for c in RS.CASES])
def test_case_reaches_its_branches(name):
    case = RS.BY_NAME[name]
    got = reached(case)
    assert set(case.reaches) <= got, (name, sorted(set(case.reaches) - got))
    rois = RS.rois(name)
    # batch indices are whole numbers in [0, B): the kernels index the blob with them
    assert np.array_equal(rois[:, 0], np.round(rois[:, 0]))
    assert rois[:, 0].min() >= 0 and rois[:, 0].max() < case.B
    assert np.isfinite(rois).all()
    for ph, pw in case.pooled:
        assert 1 <= min(ph, pw) and max(ph, pw) <= K_MAX_POOLED
    for ph, pw in case.pool_only:
        assert max(ph, pw) > K_MAX_POOLED


def test_branch_details():
    C = RS.BY_NAME
    hits = tile_round_hits(C["training"])
    assert hits.max() > 3 * K_CHUNK                       # 4 chunks on the busiest tile
    assert -(-C["training"].C // K_COORD_SLAB) == 8
    many = tile_round_hits(C["many_rois"])
    assert len(RS.rois("many_rois")) > 2 * K_TILE_THREADS   # three rounds
    assert ((many > 0).sum(axis=3) == 3).any()            # a tile meets RoIs of every round
    assert not many[2].any()                              # image 2: no RoI
    # every channel tail at every size, each size on the kernel it is meant for
    tails = [c for c in RS.CASES if c.name.startswith("tail_")]
    assert sorted(c.C for c in tails) == [1, 13, 42, 72]
    for c in tails:
        assert c.pooled == RS.ALL_SIZES
        assert [warp_dispatch(*s) for s in c.pooled] == ["rowwalk28", "rowwalk14", "nchw7", "generic"]
        for P in (28, 14):
            assert rowwalk_partial_group(c.C, P) == (c.C % ROWWALK_CH[P] != 0)
    assert all(warp_dispatch(*s) == "generic" for s in C["generic"].pooled)
    assert sorted(C["generic"].pooled) == sorted(RS.GENERIC_SIZES)
    maps = {(c.H, c.W): c.scale for c in RS.CASES if c.name.startswith("map_")}
    assert maps == {(1, 1): 1 / 32, (3, 5): 1.0, (9, 130): 1 / 8, (63, 38): 1 / 32}
    assert math.ceil(130 / K_TILE_W) == 5


def test_mask_blobs_take_more_than_one_grid_pass():
    (n, c, ih, iw), _ = RS.MASK_RESIZE_BWD["resize_700"]
    assert grid_passes(n * c * ih * iw, 256, SMS * 8) >= 2                 # mask_resize_bwd_kernel
    n, c, h, w = RS.MASK_POOL["pool_64x512"]
    total = n * c * h * w
    assert (h * w) % 4 == 0
    assert grid_passes(total // 4, 256, SMS * 16) >= 2                     # mask_pool_nchw_kernel
    assert grid_passes(total, 256, SMS * 16) >= 2          # ..._scalar_kernel, mask_pool_bwd_feat
    assert grid_passes(n * h * w, 128, SMS * 16) == 1
    n, c, h, w = RS.MASK_POOL["pool_1400"]
    assert grid_passes(n * h * w, 128, SMS * 16) >= 2                      # mask_pool_bwd_mask_kernel

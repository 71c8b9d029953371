"""Every NMS form on IoUs that round to within a few ulps of the threshold (tests/nms_ties.py): the
keep lists must be those of greedy NMS under the reference `_nms`'s rounding of devIoU, where nvcc
fuses the later box's area product into the union:  U = fl(fma(bw, bh, Sa) - I),  q = fl(I / U).
When oracle/_ref holds the reference's own `_nms`, the lists are also run through it."""
import ctypes
import os

import numpy as np
import pytest

from tests import nms_ties as T

pytestmark = pytest.mark.gpu
ALL_THRESHOLDS = T.THRESHOLDS + (0.0, -0.5)
REF_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref",
                      "libmnc_ref.so")


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _dets(boxes):
    """score-sorted (n, 5) dets: descending, tie-free scores."""
    n = len(boxes)
    return np.ascontiguousarray(np.hstack([boxes, np.linspace(1, 0.001, n, dtype=np.float32)[:, None]]),
                                dtype=np.float32)


@pytest.mark.parametrize("thresh", ALL_THRESHOLDS)
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_nms_sorted_ties(thresh, mode):
    """mnc_nms_sorted, batched with ragged counts: the suppression matrix + scan (n < 1024, and mode 0),
    the one-CTA capped walk (1), the 8-CTA cluster (2, the default) and its 256-candidate rounds (3)."""
    import torch
    from mnc_b200 import ops
    from mnc_b200._lib import lib
    prev = ops.nms_set_lazy(mode)
    try:
        for name in ("small", "big"):
            boxes, _, counts, max_keep = T.tie_lists(thresh, name)
            n_max = boxes.shape[1]
            capped = name == "big" and mode > 0
            assert lib.mnc_nms_sorted_launches(n_max, max_keep or n_max) == (1 if capped else 2)
            keep, num = ops.nms_sorted(torch.from_numpy(boxes).cuda(),
                                       torch.tensor(counts, dtype=torch.int32).cuda(), thresh, max_keep)
            keep, num = keep.cpu().numpy(), num.cpu().numpy()
            for p, want in enumerate(T.expected_keep(thresh, name)):
                assert num[p] == len(want) and np.array_equal(keep[p, :num[p]], want), (name, p)
    finally:
        ops.nms_set_lazy(prev)


@pytest.mark.parametrize("thresh", ALL_THRESHOLDS)
def test_nms_host_ties(thresh):
    """mnc_nms_host, the `_nms` drop-in, on every list."""
    from mnc_b200._lib import lib, check
    for name in ("small", "big"):
        boxes, _, counts, _ = T.tie_lists(thresh, name)
        for p, c in enumerate(counts):
            dets = _dets(boxes[p, :c])
            keep = np.zeros(c, dtype=np.int32)
            num = ctypes.c_int(0)
            check(lib.mnc_nms_host(_p(keep), ctypes.byref(num), _p(dets), c, 5, ctypes.c_float(thresh), 0),
                  "mnc_nms_host")
            want = T.greedy_keep(boxes[p, :c], thresh)
            assert np.array_equal(keep[:num.value], want), (name, p)


@pytest.mark.parametrize("thresh", [0.7, 0.3])
def test_gpu_nms_ties(thresh):
    """nms.gpu_nms (mnc_gpu_nms_host: device sort, gather, NMS) on the lists in shuffled row order."""
    import mnc_b200.lib as L
    L.install()
    from nms.gpu_nms import gpu_nms
    rng = np.random.default_rng(5)
    for name in ("small", "big"):
        boxes, _, counts, _ = T.tie_lists(thresh, name)
        dets = _dets(boxes[0])
        perm = rng.permutation(len(dets))                 # row r of the input is sorted row perm[r]
        shuffled = np.empty_like(dets)
        shuffled[perm] = dets
        want = perm[T.greedy_keep(boxes[0], thresh)]
        assert gpu_nms(shuffled, thresh) == [int(i) for i in want], name


@pytest.mark.parametrize("thresh", ALL_THRESHOLDS)
def test_reference_nms_ties(thresh):
    """The reference's `_nms` (lib/nms/nms_kernel.cu compiled unmodified) gives the `ref` emulation's
    keep lists, and the same source built with -fmad=false gives the C oracle's."""
    from oracle import oracle as O
    if not os.path.exists(REF_SO):
        pytest.skip("oracle/_ref/libmnc_ref*.so not built (needs the reference's sources at build time)")
    ref = ctypes.CDLL(REF_SO)
    nofma = ctypes.CDLL(REF_SO.replace(".so", "_nofma.so"))
    for name in ("small", "big"):
        boxes, _, counts, _ = T.tie_lists(thresh, name)
        for p, c in enumerate(counts):
            dets = _dets(boxes[p, :c])
            for lib, want in ((ref, T.greedy_keep(boxes[p, :c], thresh)), (nofma, O.nms_sorted(dets, thresh))):
                keep = np.zeros(c, dtype=np.int32)
                num = ctypes.c_int(0)
                lib._Z4_nmsPiS_PKfiifi(_p(keep), ctypes.byref(num), _p(dets), c, 5, ctypes.c_float(thresh), 0)
                assert np.array_equal(keep[:num.value], want), (name, p, lib is ref)

"""nms.gpu_nms -- reference lib/nms/gpu_nms.pyx:16-31: `gpu_nms(dets, thresh, device_id=0)` ->
list of kept row indices in score order.  One native call (mnc_gpu_nms_host): the
`scores.argsort()[::-1]` sort (ties resolved score descending / index ascending), the gather, the
bitmask NMS and the greedy scan all run on the device -- the .pyx wrapper's host-side sort and fancy
indexing were most of this entry point's time."""
import ctypes

import numpy as np

from mnc_b200._lib import lib, check


def gpu_nms(dets, thresh, device_id=0):
    if dets.dtype != np.float32 or dets.ndim != 2:
        raise ValueError("Buffer dtype mismatch, expected 'float32_t' 2-D")  # cython's check
    boxes_num, boxes_dim = dets.shape
    if boxes_dim < 5:
        raise IndexError("dets needs 5 columns (x1, y1, x2, y2, score)")      # dets[:, 4] in the .pyx
    dets = np.ascontiguousarray(dets)
    keep = np.zeros(boxes_num, dtype=np.int32)
    num_out = ctypes.c_int(0)
    check(lib.mnc_gpu_nms_host(keep.ctypes.data_as(ctypes.c_void_p), ctypes.byref(num_out),
                               dets.ctypes.data_as(ctypes.c_void_p), boxes_num, boxes_dim, thresh,
                               device_id), "mnc_gpu_nms_host")
    return [int(i) for i in keep[:num_out.value]]

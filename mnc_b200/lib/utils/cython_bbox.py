"""utils.cython_bbox -- reference lib/utils/bbox.pyx:15-55 over mnc_bbox_overlaps_host."""
import ctypes

import numpy as np

from mnc_b200._lib import lib, check


def bbox_overlaps(boxes, query_boxes):
    if boxes.dtype != np.float64 or query_boxes.dtype != np.float64:
        raise ValueError("Buffer dtype mismatch, expected 'DTYPE_t' (float64)")
    boxes = np.ascontiguousarray(boxes)
    query_boxes = np.ascontiguousarray(query_boxes)
    N, K = boxes.shape[0], query_boxes.shape[0]
    overlaps = np.zeros((N, K), dtype=np.float64)
    check(lib.mnc_bbox_overlaps_host(boxes.ctypes.data_as(ctypes.c_void_p), N,
                                     query_boxes.ctypes.data_as(ctypes.c_void_p), K,
                                     overlaps.ctypes.data_as(ctypes.c_void_p)),
          "mnc_bbox_overlaps_host")
    return overlaps

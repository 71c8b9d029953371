"""nms.mv -- reference lib/nms/gpu_mv.pyx:13-31 over mnc_mv_host (the `_mv` drop-in)."""
import ctypes

import numpy as np

from mnc_b200._lib import lib, check


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def mv(all_boxes, all_masks, candidate_inds, candidate_start, candidate_weights, image_height,
       image_width, device_id=0):
    for name, arr, dt, nd in (("all_boxes", all_boxes, np.float32, 2),
                              ("all_masks", all_masks, np.float32, 4),
                              ("candidate_inds", candidate_inds, np.int32, 1),
                              ("candidate_start", candidate_start, np.int32, 1),
                              ("candidate_weights", candidate_weights, np.float32, 1)):
        if arr.dtype != dt or arr.ndim != nd:
            raise ValueError("%s: Buffer dtype mismatch, expected %s %d-D" % (name, dt.__name__, nd))
    all_boxes = np.ascontiguousarray(all_boxes)
    all_masks = np.ascontiguousarray(all_masks)
    candidate_inds = np.ascontiguousarray(candidate_inds)
    candidate_start = np.ascontiguousarray(candidate_start)
    candidate_weights = np.ascontiguousarray(candidate_weights)
    all_box_num, boxes_dim = all_boxes.shape
    mask_size = all_masks.shape[3]
    candidate_num = candidate_inds.shape[0]
    result_num = candidate_start.shape[0]
    result_mask = np.zeros((result_num, 1, all_masks.shape[2], all_masks.shape[3]), dtype=np.float32)
    result_box = np.zeros((result_num, boxes_dim), dtype=np.int32)
    check(lib.mnc_mv_host(_p(all_boxes), _p(all_masks), all_box_num, _p(candidate_inds),
                          _p(candidate_start), _p(candidate_weights), candidate_num,
                          int(image_height), int(image_width), boxes_dim, mask_size, result_num,
                          _p(result_mask), _p(result_box), device_id), "mnc_mv_host")
    return result_mask, result_box

"""An MNC_ERR_CUDA names the CUDA error behind it.  Both failures here are refused by the runtime on
the host before any device work is queued, so neither is sticky and the context stays usable."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_cuda_error_is_reported_and_kept():
    import torch
    from mnc_b200 import ops
    from mnc_b200._lib import MncError, check, lib
    # one image past gridDim.y's limit of 65535: the launch is refused with
    # cudaErrorInvalidConfiguration.  n_res = 0 and per-image buffers sized for the whole grid keep
    # even an accepted launch inside its buffers.
    batch, nb, ncls = 65536, 1, 2
    i32 = lambda n: torch.zeros(n, dtype=torch.int32, device="cuda")             # noqa: E731
    boxes = torch.zeros((nb, 4), dtype=torch.float32, device="cuda")
    scores = torch.zeros((nb, ncls), dtype=torch.float32, device="cuda")
    cand_w = torch.zeros(nb, dtype=torch.float32, device="cuda")
    res_idx, res_cls, n_res, cand_inds = i32(1), i32(1), i32(batch), i32(nb)
    cand_begin, cand_end = i32(batch), i32(batch)
    with pytest.raises(MncError, match="invalid configuration argument"):
        check(lib.mnc_vote_candidates(boxes.data_ptr(), scores.data_ptr(), None, nb, ncls,
                                      res_idx.data_ptr(), res_cls.data_ptr(), n_res.data_ptr(), 1,
                                      batch, 0.5, cand_inds.data_ptr(), cand_w.data_ptr(),
                                      cand_begin.data_ptr(), cand_end.data_ptr(), None),
              "mnc_vote_candidates")
    # a later success on the same thread keeps the cause, and the runtime holds no stale error
    x = torch.randn(4, 8, device="cuda")
    assert torch.allclose(ops.softmax_rows(x), torch.softmax(x, 1), atol=1e-5)
    torch.cuda.synchronize()
    assert b"invalid configuration argument" in lib.mnc_last_cuda_error()

    # a host drop-in asked for a device that does not exist
    dets = np.zeros((1, 5), np.float32)
    keep, num = np.zeros(1, np.int32), ctypes.c_int(0)
    rc = lib.mnc_nms_host(keep.ctypes.data_as(ctypes.c_void_p), ctypes.byref(num),
                          dets.ctypes.data_as(ctypes.c_void_p), 1, 5, 0.7, lib.mnc_device_count())
    assert rc == 2
    assert b"invalid device ordinal" in lib.mnc_last_cuda_error()
    torch.zeros(1, device="cuda").add_(1)
    torch.cuda.synchronize()

"""ctypes loader for the C-ABI library (include/mnc_b200.h).

The CUDA library is the product; there is no CPU or PyTorch fallback.  Importing this module
without a built ``libmnc_b200.so`` raises, and every wrapper raises on a non-zero status.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmnc_b200.so")

MNC_OK = 0
_ERR = {1: "MNC_ERR_ARG", 2: "MNC_ERR_CUDA", 3: "MNC_ERR_DRIVER", 4: "MNC_ERR_NOGPU"}


class MncError(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "mnc_b200: %s is missing -- build it with `python -c 'import __graft_entry__ as g; "
            "g.build()'` (there is no CPU fallback)" % LIB_PATH)
    return ctypes.CDLL(LIB_PATH)


lib = _load()
lib.mnc_last_cuda_error.restype = ctypes.c_char_p

c_void_p = ctypes.c_void_p
c_int = ctypes.c_int
c_ll = ctypes.c_longlong
c_float = ctypes.c_float


# kernels launched by each C-ABI entry point (for bench.py's `gpu_launches` claim).  Entry points whose kernel count
# depends on their arguments report it themselves (`launches=`: mnc_nms_sorted_launches,
# mnc_mv_device_launches).
launch_count = 0


def check(rc, what, launches=1):
    global launch_count
    launch_count += launches
    if rc != MNC_OK:
        detail = ""
        if rc == 2:
            detail = " (%s)" % lib.mnc_last_cuda_error().decode()
        raise MncError("%s failed: %s%s" % (what, _ERR.get(rc, rc), detail))


def ptr(t):
    """Device/host pointer of a torch tensor or numpy array (None -> NULL)."""
    if t is None:
        return c_void_p(0)
    if hasattr(t, "data_ptr"):
        return c_void_p(t.data_ptr())
    return c_void_p(t.ctypes.data)


def cur_stream():
    import torch
    return c_void_p(torch.cuda.current_stream().cuda_stream)

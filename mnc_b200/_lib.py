"""ctypes loader for the C-ABI library (include/mnc_b200.h).

The CUDA library is the product; there is no CPU or PyTorch fallback.  Importing this module
without a built ``libmnc_b200.so`` raises, and every wrapper raises on a non-zero status.

Every `mnc_*` function of the header gets its `restype` and `argtypes` from its declaration, so
callers pass plain Python values and ctypes rejects a call with too few arguments or a value of
the wrong kind before it reaches C.  ctypes does not reject extra arguments;
tests/test_abi_bindings.py counts the arguments of every call instead.
"""
import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmnc_b200.so")
HEADER_PATH = os.path.join(_HERE, os.pardir, "include", "mnc_b200.h")

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


_SCALARS = {"int": ctypes.c_int, "unsigned": ctypes.c_uint, "unsigned int": ctypes.c_uint,
            "long long": ctypes.c_longlong, "float": ctypes.c_float, "double": ctypes.c_double}


def _ctype(decl, what, ret=False):
    """ctypes type of a C type as the header writes it.  Any pointer is c_void_p, except a returned
    `const char*` (a C string); a type missing from _SCALARS raises instead of defaulting to int."""
    decl = " ".join(decl.replace("*", " * ").split())
    if ret and decl == "const char *":
        return ctypes.c_char_p
    if "*" in decl:
        return ctypes.c_void_p
    if decl not in _SCALARS:
        raise TypeError("include/mnc_b200.h: %s: no ctypes type for C type %r" % (what, decl))
    return _SCALARS[decl]


def _bind(lib):
    """Set restype and argtypes of every `mnc_*` function the header declares."""
    with open(HEADER_PATH) as f:
        src = re.sub(r"/\*.*?\*/", " ", f.read(), flags=re.S)
    src = re.sub(r"^\s*#.*$", "", src, flags=re.M)
    for ret, name, params in re.findall(r"(\w[\w\s*]*?)\s*\b(mnc_\w+)\s*\(([^)]*)\)\s*;", src):
        params = [] if params.strip() == "void" else params.split(",")
        fn = getattr(lib, name)
        fn.restype = _ctype(ret, name + " return", ret=True)
        fn.argtypes = [_ctype(re.sub(r"\w+\s*$", "", p), "%s parameter %d" % (name, i))
                       for i, p in enumerate(params)]


lib = _load()
_bind(lib)

# Callers written before the bindings wrap scalars by hand (`c_int(n)`, `c_float(x)`); argtypes
# accept an instance of the declared type as well as a plain value, so those calls keep working.
c_int = ctypes.c_int
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
    """Device/host pointer of a torch tensor or numpy array as an int (None -> NULL)."""
    if t is None:
        return None
    if hasattr(t, "data_ptr"):
        return t.data_ptr()
    return t.ctypes.data


def cur_stream():
    import torch
    return torch.cuda.current_stream().cuda_stream

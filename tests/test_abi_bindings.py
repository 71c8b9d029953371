"""ctypes bindings of include/mnc_b200.h (mnc_b200._lib): every declared entry point carries the
restype and argtypes of its declaration, and every call of one in the project passes as many
arguments as the header declares -- ctypes rejects too few arguments but not too many."""
import ast
import ctypes
import glob
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "mnc_b200.h")


def _header_arity():
    """{name: number of parameters} of every `mnc_*` function the header declares."""
    hdr = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    out = {}
    for name, params in re.findall(r"\b(mnc_[a-z0-9_]+)\s*\(([^)]*)\)", hdr):
        params = params.strip()
        out[name] = 0 if params in ("", "void") else params.count(",") + 1
    return out


def test_every_declared_entry_point_is_bound_with_its_parameter_count():
    from mnc_b200._lib import lib
    hdr = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    names = set(re.findall(r"\b(mnc_[a-z0-9_]+)\s*\(", hdr))   # as test_abi_and_host finds them
    bound = {n for n, f in vars(lib).items() if n.startswith("mnc_") and f.argtypes is not None}
    assert bound == names
    arity = _header_arity()
    assert set(arity) == names
    wrong = {n: (len(getattr(lib, n).argtypes), arity[n]) for n in names
             if len(getattr(lib, n).argtypes) != arity[n]}
    assert not wrong, wrong


def test_argtypes_follow_the_declared_types():
    from mnc_b200._lib import lib
    assert lib.mnc_nms_sorted.argtypes[2] is ctypes.c_longlong        # long long problem_stride
    assert lib.mnc_vote_candidates.argtypes[10] is ctypes.c_double    # double iou_thresh
    for i in (12, 13, 15, 17):   # negative_overlap, positive_overlap, fg_fraction, positive_weight
        assert lib.mnc_anchor_target.argtypes[i] is ctypes.c_double, i
    assert lib.mnc_last_cuda_error.restype is ctypes.c_char_p


def test_unknown_c_type_raises_instead_of_defaulting():
    from mnc_b200 import _lib
    assert _lib._ctype("const unsigned int *", "p") is ctypes.c_void_p
    assert _lib._ctype("unsigned", "p") is ctypes.c_uint
    for decl in ("size_t", "long", "short", "int64_t"):
        with pytest.raises(TypeError):
            _lib._ctype(decl, "p")


def test_long_long_result_is_not_truncated_by_the_loader_alone():
    """mnc_nms_workspace_bytes returns long long; its restype must come from mnc_b200._lib, not
    from a module that may not be imported yet."""
    code = ("import sys; from mnc_b200._lib import lib; assert 'mnc_b200.ops' not in sys.modules; "
            "a, b = lib.mnc_nms_workspace_bytes(6000, 500), lib.mnc_nms_workspace_bytes(6000, 1); "
            "assert a == 500 * b and a > 2 ** 31, (a, b)")
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, check=True)


def test_wrong_calls_raise_before_reaching_c():
    from mnc_b200._lib import lib
    workspace_bytes = lib.mnc_nms_workspace_bytes   # host-only; named so the call scan skips it
    with pytest.raises(TypeError):
        workspace_bytes(6000)
    with pytest.raises(ctypes.ArgumentError):
        workspace_bytes(6000.0, 1)


def test_hand_wrapped_scalars_of_the_declared_type_still_work():
    from mnc_b200._lib import lib, c_int
    assert lib.mnc_nms_workspace_bytes(c_int(6000), c_int(500)) == \
        lib.mnc_nms_workspace_bytes(6000, 500)


# ------------------------------------------------------------------ argument count of every call
def _n_args(arg):
    """C arguments one call argument stands for, or None when the source does not say."""
    if not isinstance(arg, ast.Starred):
        return 1
    v = arg.value
    if isinstance(v, (ast.ListComp, ast.GeneratorExp)) and len(v.generators) == 1 \
            and not v.generators[0].ifs:
        v = v.generators[0].iter     # *[ptr(out[k]) for k in ("a", "b")] -> the tuple
    if isinstance(v, (ast.Tuple, ast.List)) and not any(isinstance(e, ast.Starred) for e in v.elts):
        return len(v.elts)
    return None


def _call_errors(source, filename, arity):
    errors = []
    for node in ast.walk(ast.parse(source, filename)):
        if not (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute)
                and node.func.attr.startswith("mnc_")):
            continue
        name = node.func.attr
        where = "%s:%d %s" % (filename, node.lineno, name)
        counts = [_n_args(a) for a in node.args]
        if name not in arity:
            errors.append(where + ": not declared in include/mnc_b200.h")
        elif node.keywords or None in counts:
            errors.append(where + ": cannot count the arguments")
        elif sum(counts) != arity[name]:
            errors.append("%s: %d arguments, the header declares %d" % (where, sum(counts), arity[name]))
    return errors


def test_every_call_passes_the_declared_number_of_arguments():
    arity = _header_arity()
    files = [os.path.join(ROOT, "__graft_entry__.py")]
    files += glob.glob(os.path.join(ROOT, "mnc_b200", "**", "*.py"), recursive=True)
    files += glob.glob(os.path.join(ROOT, "tests", "**", "*.py"), recursive=True)
    errors, n_calls = [], 0
    for path in files:
        src = open(path).read()
        n_calls += len(re.findall(r"\.mnc_\w+\(", src))
        errors += _call_errors(src, os.path.relpath(path, ROOT), arity)
    assert n_calls >= 72
    assert not errors, "\n".join(errors)


def test_call_scan_flags_miscounted_calls():
    arity = _header_arity()
    ok = ("check(lib.mnc_softmax_rows(ptr(x), 8, 2, 3, ptr(y), 8, cur_stream()), 'softmax')\n"
          "lib.mnc_mask_pool_split(ptr(a), *[ptr(b[k]) for k in (0, 1)], 2, 3, *(p, q), s)\n")
    assert _call_errors(ok, "ok.py", arity) == []
    extra = "check(lib.mnc_softmax_rows(ptr(x), 8, 2, 3, ptr(y), 8, 0, cur_stream()), 'softmax')\n"
    assert len(_call_errors(extra, "extra.py", arity)) == 1
    for bad in ("lib.mnc_mask_pool_split(*args)\n", "lib.mnc_abi_version(x=1)\n",
                "lib.mnc_no_such_entry_point()\n"):
        assert len(_call_errors(bad, "bad.py", arity)) == 1, bad

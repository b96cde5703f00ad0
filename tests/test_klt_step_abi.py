"""cosl_klt_group_step / _step_dev on the C-ABI without a GPU: the header declares both calls and
the four ops, the Python constants match them, the library exports the symbols, and a NULL handle
is refused."""
import ctypes as C
import os
import re

from coslam_b200 import api, ctypes_defs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPS = {"COSL_KLT_OP_SKIP": 0, "COSL_KLT_OP_FIRST": 1, "COSL_KLT_OP_TRACK": 2, "COSL_KLT_OP_NEXT": 3}
COSL_E_INVALID = -1


def _header():
    src = open(os.path.join(ROOT, "include", "coslam_b200.h")).read()
    return re.sub(r"/\*.*?\*/", "", src, flags=re.S)


def test_header_declares_the_calls_and_the_ops():
    src = _header()
    for name in ("cosl_klt_group_step", "cosl_klt_group_step_dev"):
        assert re.search(r"\bint\s+" + name + r"\s*\(", src), name
    for name, value in OPS.items():
        m = re.search(r"\b" + name + r"\s*=\s*(\d+)", src)
        assert m and int(m.group(1)) == value, name


def test_python_constants_match_the_header():
    for name, value in OPS.items():
        assert getattr(ctypes_defs, name) == value, name


def test_library_exports_the_calls():
    lib = C.CDLL(api.LIB_PATH)
    assert hasattr(lib, "cosl_klt_group_step") and hasattr(lib, "cosl_klt_group_step_dev")


def test_null_handle_is_invalid():
    ops = (C.c_uint8 * 2)(1, 0)
    assert api.LIB.cosl_klt_group_step(None, ops, None, 0, None, None) == COSL_E_INVALID
    assert api.LIB.cosl_klt_group_step_dev(None, ops, None, 0) == COSL_E_INVALID

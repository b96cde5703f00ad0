"""cosl_klt_group_submit_step on the C-ABI without a GPU: the header declares it, the library exports
it, the binding knows its argument types, and a call that cannot reach a device returns an error
code instead of crashing."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from coslam_b200 import api
from coslam_b200.ctypes_defs import COSL_KLT_OP_NEXT, COSL_KLT_OP_SKIP, KltConfig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSL_E_INVALID, COSL_E_CUDA = -1, -2


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_header_declares_the_call():
    src = open(os.path.join(ROOT, "include", "coslam_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    decl = re.search(r"\bint\s+cosl_klt_group_submit_step\s*\(([^)]*)\)\s*;", src)
    assert decl, "cosl_klt_group_submit_step is not declared"
    args = [a.strip() for a in decl.group(1).split(",")]
    assert args == ["cosl_klt* h", "const uint8_t* ops", "const uint8_t* const* imgs", "size_t pitch"], args


def test_library_exports_the_call_and_the_binding_declares_it():
    lib = C.CDLL(api.LIB_PATH)
    assert hasattr(lib, "cosl_klt_group_submit_step")
    assert api.LIB.cosl_klt_group_submit_step.argtypes == [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    assert callable(getattr(api.KltGroup, "submit_step", None))


def test_null_handle_is_invalid():
    ops = np.array([COSL_KLT_OP_NEXT, COSL_KLT_OP_SKIP], np.uint8)
    img = np.zeros((32, 32), np.uint8)
    imgs = (C.c_void_p * 2)(img.ctypes.data, None)
    assert api.LIB.cosl_klt_group_submit_step(None, ops.ctypes.data, imgs, 32) == COSL_E_INVALID
    assert api.LIB.cosl_klt_group_submit_step(None, None, None, 0) == COSL_E_INVALID
    assert api.LIB.cosl_klt_group_collect(None, None, None) == COSL_E_INVALID


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_no_group_without_a_gpu():
    """Without a device there is no group to submit to: creation reports COSL_E_CUDA and leaves the
    handle NULL, which submit_step refuses."""
    cfg = KltConfig.coslam_live()
    h = C.c_void_p()
    assert api.LIB.cosl_klt_group_create(C.byref(cfg), 2, 64, 64, 3, 8, 8, 0, 0, 0, C.byref(h)) == COSL_E_CUDA
    assert not h.value
    ops = np.array([COSL_KLT_OP_NEXT] * 2, np.uint8)
    img = np.zeros((64, 64), np.uint8)
    imgs = (C.c_void_p * 2)(img.ctypes.data, img.ctypes.data)
    assert api.LIB.cosl_klt_group_submit_step(h, ops.ctypes.data, imgs, 64) == COSL_E_INVALID

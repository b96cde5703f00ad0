"""cosl_klt_group_prefetch / _run_prefetched / _submit_prefetched / _discard_prefetch on the C-ABI
without a GPU: the header declares them, the library exports them, the binding knows their argument
types, and a call that cannot reach a device returns an error code instead of crashing."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from coslam_b200 import api
from coslam_b200.ctypes_defs import COSL_KLT_OP_NEXT, COSL_KLT_OP_SKIP, KltConfig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSL_E_INVALID, COSL_E_CUDA = -1, -2
DECLS = {
    "cosl_klt_group_prefetch": ["cosl_klt* h", "const uint8_t* ops", "const uint8_t* const* imgs", "size_t pitch"],
    "cosl_klt_group_run_prefetched": ["cosl_klt* h", "cosl_klt_feature* const* dest", "int* n"],
    "cosl_klt_group_submit_prefetched": ["cosl_klt* h"],
    "cosl_klt_group_discard_prefetch": ["cosl_klt* h"],
}
ARGTYPES = {
    "cosl_klt_group_prefetch": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t],
    "cosl_klt_group_run_prefetched": [C.c_void_p, C.c_void_p, C.c_void_p],
    "cosl_klt_group_submit_prefetched": [C.c_void_p],
    "cosl_klt_group_discard_prefetch": [C.c_void_p],
}


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.parametrize("name", sorted(DECLS))
def test_header_declares_the_call(name):
    src = open(os.path.join(ROOT, "include", "coslam_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    decl = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", src)
    assert decl, f"{name} is not declared"
    assert [a.strip() for a in decl.group(1).split(",")] == DECLS[name]


@pytest.mark.parametrize("name", sorted(DECLS))
def test_library_exports_the_call_and_the_binding_declares_it(name):
    assert hasattr(C.CDLL(api.LIB_PATH), name)
    assert getattr(api.LIB, name).argtypes == ARGTYPES[name]


def test_group_has_the_methods():
    for m in ("prefetch", "run_prefetched", "submit_prefetched", "discard_prefetch"):
        assert callable(getattr(api.KltGroup, m, None)), m


def test_null_handle_is_invalid():
    ops = np.array([COSL_KLT_OP_NEXT, COSL_KLT_OP_SKIP], np.uint8)
    img = np.zeros((32, 32), np.uint8)
    imgs = (C.c_void_p * 2)(img.ctypes.data, img.ctypes.data)
    assert api.LIB.cosl_klt_group_prefetch(None, ops.ctypes.data, imgs, 32) == COSL_E_INVALID
    assert api.LIB.cosl_klt_group_prefetch(None, None, None, 0) == COSL_E_INVALID
    assert api.LIB.cosl_klt_group_run_prefetched(None, None, None) == COSL_E_INVALID
    assert api.LIB.cosl_klt_group_submit_prefetched(None) == COSL_E_INVALID
    assert api.LIB.cosl_klt_group_discard_prefetch(None) == COSL_E_INVALID


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_no_group_without_a_gpu():
    """Without a device there is no group to prefetch into: creation reports COSL_E_CUDA and leaves
    the handle NULL, which every prefetch call refuses (no CPU fallback)."""
    cfg = KltConfig.coslam_live()
    h = C.c_void_p()
    assert api.LIB.cosl_klt_group_create(C.byref(cfg), 2, 64, 64, 3, 8, 8, 0, 0, 0, C.byref(h)) == COSL_E_CUDA
    assert not h.value
    img = np.zeros((64, 64), np.uint8)
    imgs = (C.c_void_p * 2)(img.ctypes.data, img.ctypes.data)
    assert api.LIB.cosl_klt_group_prefetch(h, None, imgs, 64) == COSL_E_INVALID
    assert api.LIB.cosl_klt_group_run_prefetched(h, None, None) == COSL_E_INVALID
    assert api.LIB.cosl_klt_group_submit_prefetched(h) == COSL_E_INVALID
    assert api.LIB.cosl_klt_group_discard_prefetch(h) == COSL_E_INVALID

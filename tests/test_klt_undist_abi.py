"""cosl_klt_set_undistortion and cosl_klt_group_download_undistorted on the C-ABI without a GPU: the header
declares them with these argument lists, the library exports them, the binding knows their argument types and
KltGroup has the methods, and a call that cannot reach a device returns an error code instead of crashing."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from coslam_b200 import api
from coslam_b200.ctypes_defs import KltConfig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSL_E_INVALID, COSL_E_CUDA = -1, -2
DECLS = {
    "cosl_klt_set_undistortion": ["cosl_klt* h", "const double* K", "const double* kc"],
    "cosl_klt_group_download_undistorted": ["cosl_klt* h", "double* const* pos", "float* const* cov"],
}
ARGTYPES = {
    "cosl_klt_set_undistortion": [C.c_void_p, C.c_void_p, C.c_void_p],
    "cosl_klt_group_download_undistorted": [C.c_void_p, C.c_void_p, C.c_void_p],
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
    assert [" ".join(a.split()) for a in decl.group(1).split(",")] == DECLS[name]


@pytest.mark.parametrize("name", sorted(DECLS))
def test_library_exports_the_call_and_the_binding_declares_it(name):
    assert hasattr(C.CDLL(api.LIB_PATH), name)
    assert getattr(api.LIB, name).argtypes == ARGTYPES[name]


def test_group_has_the_methods():
    for m in ("set_undistortion", "download_undistorted"):
        assert callable(getattr(api.KltGroup, m, None)), m


def test_null_handle_is_invalid():
    K = np.eye(3)
    kc = np.zeros(5)
    pos, cov = np.zeros((4, 2)), np.zeros((4, 3), np.float32)
    pp, cp = (C.c_void_p * 1)(pos.ctypes.data), (C.c_void_p * 1)(cov.ctypes.data)
    assert api.LIB.cosl_klt_set_undistortion(None, K.ctypes.data, kc.ctypes.data) == COSL_E_INVALID
    assert api.LIB.cosl_klt_set_undistortion(None, None, None) == COSL_E_INVALID
    for a, b in ((pp, cp), (pp, None), (None, cp), (None, None)):
        assert api.LIB.cosl_klt_group_download_undistorted(None, a, b) == COSL_E_INVALID
    assert np.all(pos == 0) and np.all(cov == 0)


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_no_group_without_a_gpu():
    """Without a device a group cannot be made (COSL_E_CUDA, handle left NULL), so there is nothing to arm
    or download from: both calls refuse the NULL handle (no CPU fallback)."""
    cfg = KltConfig.coslam_live()
    h = C.c_void_p()
    assert api.LIB.cosl_klt_group_create(C.byref(cfg), 2, 64, 64, 3, 8, 8, 0, 0, 0, C.byref(h)) == COSL_E_CUDA
    assert not h.value
    K = np.tile(np.eye(3), (2, 1, 1))
    kc = np.zeros((2, 5))
    assert api.LIB.cosl_klt_set_undistortion(h, K.ctypes.data, kc.ctypes.data) == COSL_E_INVALID
    pos = np.zeros((2, 64, 2))
    pp = (C.c_void_p * 2)(pos[0].ctypes.data, pos[1].ctypes.data)
    assert api.LIB.cosl_klt_group_download_undistorted(h, pp, None) == COSL_E_INVALID

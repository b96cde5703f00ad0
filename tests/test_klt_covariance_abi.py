"""cosl_klt_set_covariance and cosl_klt_group_download_covariance on the C-ABI without a GPU: the header
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
    "cosl_klt_set_covariance": ["cosl_klt* h", "float noise_var"],
    "cosl_klt_group_download_covariance": ["cosl_klt* h", "float* const* cov"],
}
ARGTYPES = {
    "cosl_klt_set_covariance": [C.c_void_p, C.c_float],
    "cosl_klt_group_download_covariance": [C.c_void_p, C.c_void_p],
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
    for m in ("set_covariance", "download_covariance"):
        assert callable(getattr(api.KltGroup, m, None)), m


def test_null_handle_is_invalid():
    out = np.zeros((4, 3), np.float32)
    cov = (C.c_void_p * 1)(out.ctypes.data)
    for v in (0.0, 1.0, -1.0, float("nan")):
        assert api.LIB.cosl_klt_set_covariance(None, v) == COSL_E_INVALID
    assert api.LIB.cosl_klt_group_download_covariance(None, cov) == COSL_E_INVALID
    assert api.LIB.cosl_klt_group_download_covariance(None, None) == COSL_E_INVALID
    assert np.all(out == 0)


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_no_group_without_a_gpu():
    """Without a device a group cannot be made (COSL_E_CUDA, handle left NULL), so there is nothing to arm
    or download from: both calls refuse the NULL handle (no CPU fallback)."""
    cfg = KltConfig.coslam_live()
    h = C.c_void_p()
    assert api.LIB.cosl_klt_group_create(C.byref(cfg), 2, 64, 64, 3, 8, 8, 0, 0, 0, C.byref(h)) == COSL_E_CUDA
    assert not h.value
    assert api.LIB.cosl_klt_set_covariance(h, 0.0) == COSL_E_INVALID
    out = np.zeros((2, 64, 3), np.float32)
    cov = (C.c_void_p * 2)(out[0].ctypes.data, out[1].ctypes.data)
    assert api.LIB.cosl_klt_group_download_covariance(h, cov) == COSL_E_INVALID

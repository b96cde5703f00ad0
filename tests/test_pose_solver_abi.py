"""The pose solver handle's C-ABI without a GPU: declared and exported, bad arguments refused with
COSL_E_INVALID before any device is touched, and no CPU fallback when there is no device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from coslam_b200 import api
from coslam_b200.ctypes_defs import PoseOpt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("cosl_pose_solver_create", "cosl_pose_solver_destroy", "cosl_pose_solver_submit",
           "cosl_pose_solver_query", "cosl_pose_solver_collect", "cosl_pose_solver_stream")
E_INVALID, E_CUDA = -1, -2


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_symbols_declared_and_exported():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coslam_b200.h")).read(), flags=re.S)
    assert "typedef struct cosl_pose_solver cosl_pose_solver;" in src
    declared = set(re.findall(r"\b(cosl_pose_solver_[a-z]+)\s*\(", src))
    assert declared == set(SYMBOLS)
    lib = C.CDLL(api.LIB_PATH)
    for s in SYMBOLS:
        assert hasattr(lib, s), s


def test_create_refuses_bad_arguments():
    L = api.LIB
    h = C.c_void_p()
    assert L.cosl_pose_solver_create(0, 4, 100, None) == E_INVALID
    for dev, cams, pts in ((-1, 4, 100), (0, 0, 100), (0, -3, 100), (0, 4, -1)):
        h.value = None
        assert L.cosl_pose_solver_create(dev, cams, pts, C.byref(h)) == E_INVALID, (dev, cams, pts)
        assert not h.value
        assert b"bad argument" in L.cosl_last_error()


def test_null_handle_is_refused():
    L = api.LIB
    one = np.ones(9)
    n = np.array([1], np.int32)
    M, m = (C.c_void_p * 1)(one.ctypes.data), (C.c_void_p * 1)(one.ctypes.data)
    opts = (PoseOpt * 1)(PoseOpt.defaults())
    out = np.empty(9)
    done, ok, ms = C.c_int(7), C.c_int(0), C.c_double(0)
    assert L.cosl_pose_solver_destroy(None) == E_INVALID
    assert L.cosl_pose_solver_submit(None, 1, one.ctypes.data, one.ctypes.data, one.ctypes.data, n.ctypes.data,
                                     M, m, None, 10.0, opts) == E_INVALID
    assert L.cosl_pose_solver_query(None, C.byref(done)) == E_INVALID and done.value == 7
    assert L.cosl_pose_solver_collect(None, out.ctypes.data, out.ctypes.data, opts, C.byref(ok),
                                      C.byref(ms)) == E_INVALID
    assert L.cosl_pose_solver_stream(None) is None


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_create_without_a_device_is_a_cuda_error():
    h = C.c_void_p()
    assert api.LIB.cosl_pose_solver_create(0, 4, 100, C.byref(h)) == E_CUDA
    assert not h.value
    with pytest.raises(api.CoslError, match="error -2"):
        api.PoseSolver(0, 13, 2000)

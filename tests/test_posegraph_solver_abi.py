"""The pose-graph solver handle's C-ABI without a GPU: declared and exported, NULL handles and arguments refused
with COSL_E_INVALID before any device is touched, and no CPU fallback when there is no device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from coslam_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("cosl_posegraph_solver_create", "cosl_posegraph_solver_destroy", "cosl_posegraph_solver_submit_chains",
           "cosl_posegraph_solver_submit", "cosl_posegraph_solver_query", "cosl_posegraph_solver_collect",
           "cosl_posegraph_solver_stream")
E_INVALID, E_CUDA = -1, -2


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_symbols_declared_and_exported():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coslam_b200.h")).read(), flags=re.S)
    assert "typedef struct cosl_posegraph_solver cosl_posegraph_solver;" in src
    declared = set(re.findall(r"\b(cosl_posegraph_solver_[a-z_]+)\s*\(", src))
    assert declared == set(SYMBOLS)
    lib = C.CDLL(api.LIB_PATH)
    for s in SYMBOLS:
        assert hasattr(lib, s), s


def test_create_refuses_bad_arguments():
    L = api.LIB
    h = C.c_void_p()
    assert L.cosl_posegraph_solver_create(0, None) == E_INVALID
    assert L.cosl_posegraph_solver_create(-1, C.byref(h)) == E_INVALID
    assert not h.value
    assert b"bad argument" in L.cosl_last_error()


def test_null_handle_is_refused():
    L = api.LIB
    off = np.array([0, 2], np.int32)
    fx = np.array([1, 0], np.uint8)
    one = np.ones(18)
    ids = np.array([0], np.int32)
    out = np.empty(18)
    done, ms = C.c_int(7), C.c_double(0)
    p = one.ctypes.data
    assert L.cosl_posegraph_solver_destroy(None) == E_INVALID
    assert b"null pose-graph solver handle" in L.cosl_last_error()
    assert L.cosl_posegraph_solver_submit_chains(None, 1, off.ctypes.data, fx.ctypes.data, p, p, p, p) == E_INVALID
    assert L.cosl_posegraph_solver_submit(None, 2, fx.ctypes.data, p, p, 1, ids.ctypes.data, ids.ctypes.data, p, p,
                                          None, 0) == E_INVALID
    assert L.cosl_posegraph_solver_query(None, C.byref(done)) == E_INVALID and done.value == 7
    assert L.cosl_posegraph_solver_collect(None, out.ctypes.data, out.ctypes.data, None, C.byref(ms)) == E_INVALID
    assert L.cosl_posegraph_solver_stream(None) is None


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_create_without_a_device_is_a_cuda_error():
    h = C.c_void_p()
    assert api.LIB.cosl_posegraph_solver_create(0, C.byref(h)) == E_CUDA
    assert not h.value
    with pytest.raises(api.CoslError, match="error -2"):
        api.PoseGraphSolver(0)

"""The registration handle at the C-ABI without a GPU: the header declares cosl_assoc_solver_create, _destroy, _submit,
_query, _collect and _stream with these argument lists, the library exports them, the binding declares them, a NULL
handle is refused, and without a device create fails with COSL_E_CUDA (no CPU fallback)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSL_E_INVALID = -1
COSL_E_CUDA = -2

ARGS = {
    "cosl_assoc_solver_create": ["int device", "int maxCams", "int maxPts", "int maxQueries", "int maxFeats",
                                 "int maxTrackObs", "cosl_assoc_solver** out"],
    "cosl_assoc_solver_destroy": ["cosl_assoc_solver* s"],
    "cosl_assoc_solver_submit": ["cosl_assoc_solver* s", "int nCams", "const double* K9", "const double* R",
                                 "const double* t", "const double* const* camCov", "const int* wh",
                                 "const int* featOff", "const double* mf", "const double* covf", "const int* owned",
                                 "const int* trkOff", "const int* trkCam", "const double* trkM", "int nPts",
                                 "const double* X", "const double* PX", "const int* qOff", "const int* qCam",
                                 "double pixel_var", "double gate", "double track_gate"],
    "cosl_assoc_solver_query": ["cosl_assoc_solver* s", "int* done"],
    "cosl_assoc_solver_collect": ["cosl_assoc_solver* s", "int* status", "int* feat", "double* d2", "double* pred",
                                  "double* device_ms"],
}


def _header():
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coslam_b200.h")).read(), flags=re.S)


@pytest.mark.parametrize("fn", sorted(ARGS))
def test_header_declares_it(fn):
    decl = re.search(rf"\bint\s+{fn}\s*\(([^)]*)\)\s*;", _header())
    assert decl
    assert [" ".join(a.split()) for a in decl.group(1).split(",")] == ARGS[fn]


def test_header_declares_the_stream():
    assert re.search(r"\bvoid\*\s+cosl_assoc_solver_stream\s*\(\s*cosl_assoc_solver\*\s+s\s*\)\s*;", _header())


def test_library_exports_and_binding_declares_them(api):
    lib = C.CDLL(api.LIB_PATH)
    vp, ci, cd = C.c_void_p, C.c_int, C.c_double
    want = {"cosl_assoc_solver_create": [ci] * 6 + [C.POINTER(vp)],
            "cosl_assoc_solver_destroy": [vp],
            "cosl_assoc_solver_submit": [vp, ci] + [vp] * 12 + [ci] + [vp] * 4 + [cd] * 3,
            "cosl_assoc_solver_query": [vp, C.POINTER(ci)],
            "cosl_assoc_solver_collect": [vp] * 6,
            "cosl_assoc_solver_stream": [vp]}
    for fn, types in want.items():
        assert hasattr(lib, fn), fn
        assert getattr(api.LIB, fn).argtypes == types, fn
    assert api.LIB.cosl_assoc_solver_stream.restype == vp
    assert {"feat_off", "q_off", "q_cam", "covf", "owned", "trk_off", "trk_cam", "trk_m", "cam_cov", "pixel_var", "gate",
            "track_gate"} <= set(api.AssocSolver.submit.__code__.co_varnames)
    assert api.AssocSolver._prefix == "cosl_assoc_solver" and callable(api.AssocSolver.collect)


def test_null_handle_is_invalid(api):
    L = api.LIB
    K = np.eye(3).ravel()
    wh = (C.c_int * 2)(640, 480)
    off = (C.c_int * 2)(0, 0)
    q = (C.c_int * 2)(0, 1)
    assert L.cosl_assoc_solver_destroy(None) == COSL_E_INVALID
    assert b"null registration handle" in L.cosl_last_error()
    assert L.cosl_assoc_solver_submit(None, 1, K.ctypes.data, K.ctypes.data, K.ctypes.data, None, wh, off, None, None,
                                      None, None, None, None, 1, K.ctypes.data, K.ctypes.data, q, q, 1.0, 9.21,
                                      9.21) == COSL_E_INVALID
    assert b"null registration handle" in L.cosl_last_error()
    done = C.c_int(0)
    assert L.cosl_assoc_solver_query(None, C.byref(done)) == COSL_E_INVALID
    assert L.cosl_assoc_solver_collect(None, None, None, None, None, None) == COSL_E_INVALID
    assert b"null registration handle" in L.cosl_last_error()
    assert L.cosl_assoc_solver_stream(None) is None
    h = C.c_void_p()
    assert L.cosl_assoc_solver_create(0, 0, 10, 20, 30, 0, C.byref(h)) == COSL_E_INVALID
    assert L.cosl_assoc_solver_create(0, 4, 10, 20, 0, 0, C.byref(h)) == COSL_E_INVALID
    assert L.cosl_assoc_solver_create(0, 4, 10, 20, 30, -1, C.byref(h)) == COSL_E_INVALID


def test_no_cpu_fallback_without_a_gpu(api):
    """Without a usable device, create fails with COSL_E_CUDA and leaves the handle NULL; there is no CPU path."""
    import torch

    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    h = C.c_void_p()
    assert api.LIB.cosl_assoc_solver_create(0, 4, 10, 20, 30, 0, C.byref(h)) == COSL_E_CUDA
    assert not h.value
    with pytest.raises(api.CoslError):
        api.AssocSolver(0, 4, 10, 20, 30)

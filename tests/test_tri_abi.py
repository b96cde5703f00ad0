"""The triangulation handle at the C-ABI without a GPU: the header declares cosl_tri_solver_create, _destroy, _submit,
_query, _collect and _stream with these argument lists, the library exports them, the binding declares them, and a NULL
handle is refused."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSL_E_INVALID = -1

ARGS = {
    "cosl_tri_solver_create": ["int device", "int maxCams", "int maxPts", "int maxViews", "cosl_tri_solver** out"],
    "cosl_tri_solver_destroy": ["cosl_tri_solver* s"],
    "cosl_tri_solver_submit": ["cosl_tri_solver* s", "int nCams", "const double* K9", "const double* R",
                               "const double* t", "const double* const* camCov", "int nPts", "const int* viewOff",
                               "const int* viewCam", "const double* m", "const double* covm", "double pixel_var",
                               "double max_err"],
    "cosl_tri_solver_query": ["cosl_tri_solver* s", "int* done"],
    "cosl_tri_solver_collect": ["cosl_tri_solver* s", "double* X", "double* P", "double* stat", "int* status",
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
    assert re.search(r"\bvoid\*\s+cosl_tri_solver_stream\s*\(\s*cosl_tri_solver\*\s+s\s*\)\s*;", _header())


def test_library_exports_and_binding_declares_them(api):
    lib = C.CDLL(api.LIB_PATH)
    vp, ci, cd = C.c_void_p, C.c_int, C.c_double
    want = {"cosl_tri_solver_create": [ci, ci, ci, ci, C.POINTER(vp)],
            "cosl_tri_solver_destroy": [vp],
            "cosl_tri_solver_submit": [vp, ci, vp, vp, vp, vp, ci, vp, vp, vp, vp, cd, cd],
            "cosl_tri_solver_query": [vp, C.POINTER(ci)],
            "cosl_tri_solver_collect": [vp] * 6,
            "cosl_tri_solver_stream": [vp]}
    for fn, types in want.items():
        assert hasattr(lib, fn), fn
        assert getattr(api.LIB, fn).argtypes == types, fn
    assert api.LIB.cosl_tri_solver_stream.restype == vp
    assert {"view_off", "view_cam", "covm", "cam_cov", "pixel_var", "max_err"} <= set(
        api.TriSolver.submit.__code__.co_varnames)
    assert api.TriSolver._prefix == "cosl_tri_solver" and callable(api.TriSolver.collect)


def test_null_handle_is_invalid(api):
    L = api.LIB
    K = np.eye(3).ravel()
    off = (C.c_int * 2)(0, 2)
    cam = (C.c_int * 2)(0, 0)
    m = np.zeros(4)
    assert L.cosl_tri_solver_destroy(None) == COSL_E_INVALID
    assert b"null triangulation handle" in L.cosl_last_error()
    assert L.cosl_tri_solver_submit(None, 1, K.ctypes.data, K.ctypes.data, K.ctypes.data, None, 1, off, cam,
                                    m.ctypes.data, None, 1.0, 5.0) == COSL_E_INVALID
    assert b"null triangulation handle" in L.cosl_last_error()
    done = C.c_int(0)
    assert L.cosl_tri_solver_query(None, C.byref(done)) == COSL_E_INVALID
    assert L.cosl_tri_solver_collect(None, None, None, None, None, None) == COSL_E_INVALID
    assert b"null triangulation handle" in L.cosl_last_error()
    assert L.cosl_tri_solver_stream(None) is None
    h = C.c_void_p()
    assert L.cosl_tri_solver_create(0, 0, 10, 20, C.byref(h)) == COSL_E_INVALID
    assert L.cosl_tri_solver_create(0, 4, 10, 1, C.byref(h)) == COSL_E_INVALID

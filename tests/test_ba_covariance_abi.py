"""cosl_ba_solver_set_covariance / _download_covariance and cosl_ba_debug_tile_selinv at the C-ABI without a GPU:
the header declares them with these argument lists, the library exports them, the binding declares them, and a
NULL handle is refused."""
import ctypes as C
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSL_E_INVALID = -1

DECLS = {
    "cosl_ba_solver_set_covariance": ["cosl_ba_solver* s", "double pixel_var"],
    "cosl_ba_solver_download_covariance": ["cosl_ba_solver* s", "double* camCov", "double* ptCov", "double out[8]"],
    "cosl_ba_debug_tile_selinv": ["int mf", "const uint8_t* adj", "int nd_depth", "const double* S", "double* Z",
                                  "int* fail", "int out[8]"],
}


def test_header_declares_the_covariance_calls():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coslam_b200.h")).read(), flags=re.S)
    for name, args in DECLS.items():
        decl = re.search(r"\bint\s+%s\s*\(([^)]*)\)\s*;" % name, src)
        assert decl, name
        assert [" ".join(a.split()) for a in decl.group(1).split(",")] == args


def test_library_exports_and_binding_declares_them(api):
    lib = C.CDLL(api.LIB_PATH)
    for name in DECLS:
        assert hasattr(lib, name)
    for meth in ("set_covariance", "download_covariance"):
        assert callable(getattr(api.BaSolver, meth, None))
    assert callable(api.ba_debug_tile_selinv)
    vp = C.c_void_p
    assert api.LIB.cosl_ba_solver_set_covariance.argtypes == [vp, C.c_double]
    assert api.LIB.cosl_ba_solver_download_covariance.argtypes == [vp, vp, vp, C.POINTER(C.c_double)]
    assert api.LIB.cosl_ba_debug_tile_selinv.argtypes == [C.c_int, vp, C.c_int, vp, vp, C.POINTER(C.c_int),
                                                          C.POINTER(C.c_int)]


def test_null_handle_and_bad_arguments_are_invalid(api):
    out = (C.c_double * 8)()
    assert api.LIB.cosl_ba_solver_set_covariance(None, 1.0) == COSL_E_INVALID
    assert api.LIB.cosl_ba_solver_download_covariance(None, None, None, out) == COSL_E_INVALID
    Z = np.zeros((6, 6))
    fail, o = C.c_int(0), (C.c_int * 8)()
    assert api.LIB.cosl_ba_debug_tile_selinv(0, None, -1, None, Z.ctypes.data_as(C.c_void_p), C.byref(fail),
                                             o) == COSL_E_INVALID

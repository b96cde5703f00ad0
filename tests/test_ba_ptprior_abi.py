"""cosl_ba_solver_set_pt_prior at the C-ABI without a GPU: the header declares it with this argument list, the library
exports it, the binding declares it, and a NULL handle is refused (with priors, when clearing and with nPrior < 0)."""
import ctypes as C
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSL_E_INVALID = -1
ARGS = ["cosl_ba_solver* s", "int nPrior", "const int32_t* pts", "const double* X", "const double* cov"]


def test_header_declares_the_call():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coslam_b200.h")).read(), flags=re.S)
    decl = re.search(r"\bint\s+cosl_ba_solver_set_pt_prior\s*\(([^)]*)\)\s*;", src)
    assert decl
    assert [" ".join(a.split()) for a in decl.group(1).split(",")] == ARGS


def test_library_exports_and_binding_declares_it(api):
    assert hasattr(C.CDLL(api.LIB_PATH), "cosl_ba_solver_set_pt_prior")
    assert callable(getattr(api.BaSolver, "set_pt_prior", None))
    vp, ci = C.c_void_p, C.c_int
    assert api.LIB.cosl_ba_solver_set_pt_prior.argtypes == [vp, ci, vp, vp, vp]


def test_null_handle_is_invalid(api):
    vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    pts = np.array([1], np.int32)
    X, cov = np.zeros(3), np.eye(3)
    f = api.LIB.cosl_ba_solver_set_pt_prior
    assert f(None, 1, vp(pts), vp(X), vp(cov)) == COSL_E_INVALID
    assert "null solver handle" in api.LIB.cosl_last_error().decode()
    assert f(None, 0, None, None, None) == COSL_E_INVALID
    assert f(None, -1, None, None, None) == COSL_E_INVALID

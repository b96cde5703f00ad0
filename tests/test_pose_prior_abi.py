"""cosl_pose_solver_submit_prior at the C-ABI without a GPU: the header declares it with this argument list, the
library exports it, the binding declares it, and a NULL handle is refused."""
import ctypes as C
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSL_E_INVALID = -1

ARGS = ["cosl_pose_solver* s", "int C", "const double* K9", "const double* R0", "const double* t0", "const int* npts",
        "const double* const* Ms", "const double* const* ms", "const double* const* covx",
        "const double* const* prior", "const double* const* prevErrs", "double tau", "const cosl_pose_opt* opts"]


def test_header_declares_submit_prior():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coslam_b200.h")).read(), flags=re.S)
    decl = re.search(r"\bint\s+cosl_pose_solver_submit_prior\s*\(([^)]*)\)\s*;", src)
    assert decl
    assert [" ".join(a.split()) for a in decl.group(1).split(",")] == ARGS


def test_library_exports_and_binding_declares_it(api):
    lib = C.CDLL(api.LIB_PATH)
    assert hasattr(lib, "cosl_pose_solver_submit_prior")
    vp, ci, cd = C.c_void_p, C.c_int, C.c_double
    assert api.LIB.cosl_pose_solver_submit_prior.argtypes == [vp, ci, vp, vp, vp, vp, vp, vp, vp, vp, vp, cd, vp]
    assert "prior" in api.PoseSolver.submit.__code__.co_varnames


def test_null_handle_is_invalid(api):
    L = api.LIB
    K = np.eye(3).ravel()
    n = (C.c_int * 1)(0)
    p = (C.c_void_p * 1)(None)
    opts = (api.PoseOpt * 1)(api.PoseOpt.defaults())
    assert L.cosl_pose_solver_submit_prior(None, 1, K.ctypes.data, K.ctypes.data, K.ctypes.data, n, p, p, None, p,
                                           None, 10.0, opts) == COSL_E_INVALID
    assert L.cosl_pose_solver_submit_prior(None, 1, None, None, None, None, None, None, None, None, None, 10.0,
                                           None) == COSL_E_INVALID
    assert b"null pose solver handle" in L.cosl_last_error()

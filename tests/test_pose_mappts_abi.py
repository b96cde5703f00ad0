"""The map-point update of the pose solver at the C-ABI without a GPU: the header declares cosl_pose_solver_reserve_mappts,
_submit_mappts and _download_mappts with these argument lists, the library exports them, the binding declares them,
and a NULL handle is refused."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSL_E_INVALID = -1

PRIOR_ARGS = ["cosl_pose_solver* s", "int C", "const double* K9", "const double* R0", "const double* t0",
              "const int* npts", "const double* const* Ms", "const double* const* ms", "const double* const* covx",
              "const double* const* prior", "const double* const* prevErrs", "double tau", "const cosl_pose_opt* opts"]
ARGS = {
    "cosl_pose_solver_reserve_mappts": ["cosl_pose_solver* s", "int maxMapPts"],
    "cosl_pose_solver_submit_mappts": PRIOR_ARGS + ["const int* nmap", "const double* const* Xmap",
                                                    "const double* const* Pmap", "const double* const* mmap",
                                                    "const double* const* covm", "double gate"],
    "cosl_pose_solver_download_mappts": ["cosl_pose_solver* s", "double* X", "double* P", "double* stat",
                                         "int* status"],
}


@pytest.mark.parametrize("fn", sorted(ARGS))
def test_header_declares_it(fn):
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coslam_b200.h")).read(), flags=re.S)
    decl = re.search(rf"\bint\s+{fn}\s*\(([^)]*)\)\s*;", src)
    assert decl
    assert [" ".join(a.split()) for a in decl.group(1).split(",")] == ARGS[fn]


def test_library_exports_and_binding_declares_them(api):
    lib = C.CDLL(api.LIB_PATH)
    vp, ci, cd = C.c_void_p, C.c_int, C.c_double
    want = {"cosl_pose_solver_reserve_mappts": [vp, ci],
            "cosl_pose_solver_submit_mappts": [vp, ci] + [vp] * 9 + [cd, vp] + [vp] * 5 + [cd],
            "cosl_pose_solver_download_mappts": [vp] * 5}
    for fn, types in want.items():
        assert hasattr(lib, fn), fn
        assert getattr(api.LIB, fn).argtypes == types, fn
    assert {"mappts", "gate"} <= set(api.PoseSolver.submit.__code__.co_varnames)
    assert callable(api.PoseSolver.reserve_mappts) and callable(api.PoseSolver.download_mappts)


def test_null_handle_is_invalid(api):
    L = api.LIB
    K = np.eye(3).ravel()
    n = (C.c_int * 1)(0)
    p = (C.c_void_p * 1)(None)
    opts = (api.PoseOpt * 1)(api.PoseOpt.defaults())
    assert L.cosl_pose_solver_reserve_mappts(None, 10) == COSL_E_INVALID
    assert b"null pose solver handle" in L.cosl_last_error()
    assert L.cosl_pose_solver_submit_mappts(None, 1, K.ctypes.data, K.ctypes.data, K.ctypes.data, n, p, p, None, None,
                                            None, 10.0, opts, n, p, p, p, None, 5.99) == COSL_E_INVALID
    assert b"null pose solver handle" in L.cosl_last_error()
    assert L.cosl_pose_solver_download_mappts(None, None, None, None, None) == COSL_E_INVALID
    assert b"null pose solver handle" in L.cosl_last_error()

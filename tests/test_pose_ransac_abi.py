"""PnP RANSAC of the pose solver at the C-ABI without a GPU: the header declares cosl_pose_solver_set_ransac,
_download_ransac and _download_ransac_hyps with these argument lists, the library exports them, the binding declares
them, a NULL handle is refused, and without a device a handle cannot be made (COSL_E_CUDA): there is no CPU path."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSL_E_INVALID = -1
COSL_E_CUDA = -2

ARGS = {
    "cosl_pose_solver_set_ransac": ["cosl_pose_solver* s", "int C", "const uint8_t* use", "int nHyp",
                                    "double err_thres", "int min_inliers", "uint64_t seed"],
    "cosl_pose_solver_download_ransac": ["cosl_pose_solver* s", "double* R", "double* t", "double* stat",
                                         "uint8_t* inl"],
    "cosl_pose_solver_download_ransac_hyps": ["cosl_pose_solver* s", "int maxHyp", "int* nHyp", "int* idx",
                                              "double* pose", "int* inliers", "double* sse"],
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
    want = {"cosl_pose_solver_set_ransac": [vp, ci, vp, ci, cd, ci, C.c_uint64],
            "cosl_pose_solver_download_ransac": [vp] * 5,
            "cosl_pose_solver_download_ransac_hyps": [vp, ci] + [vp] * 5}
    for fn, types in want.items():
        assert hasattr(lib, fn), fn
        assert getattr(api.LIB, fn).argtypes == types, fn
    for name in ("set_ransac", "download_ransac", "download_ransac_hyps"):
        assert callable(getattr(api.PoseSolver, name))
    assert {"use", "n_hyp", "err_thres", "min_inliers", "seed"} <= set(api.PoseSolver.set_ransac.__code__.co_varnames)


def test_null_handle_is_invalid(api):
    L = api.LIB
    use = np.ones(2, np.uint8)
    assert L.cosl_pose_solver_set_ransac(None, 2, use.ctypes.data, 64, 2.0, 6, 0) == COSL_E_INVALID
    assert b"null pose solver handle" in L.cosl_last_error()
    assert L.cosl_pose_solver_download_ransac(None, None, None, None, None) == COSL_E_INVALID
    assert b"null pose solver handle" in L.cosl_last_error()
    assert L.cosl_pose_solver_download_ransac_hyps(None, 0, None, None, None, None, None) == COSL_E_INVALID
    assert b"null pose solver handle" in L.cosl_last_error()


def test_no_device_no_handle(api):
    import torch

    if torch.cuda.is_available():
        pytest.skip("a device is present")
    h = C.c_void_p()
    assert api.LIB.cosl_pose_solver_create(0, 2, 100, C.byref(h)) == COSL_E_CUDA
    assert not h.value

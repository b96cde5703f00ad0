"""cosl_pose_solver_set_covariance / _download_covariance at the C-ABI without a GPU: the header declares them with
these argument lists, the library exports them, the binding declares them, and a NULL handle is refused."""
import ctypes as C
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSL_E_INVALID = -1

DECLS = {
    "cosl_pose_solver_set_covariance": ["cosl_pose_solver* s", "double pixel_var"],
    "cosl_pose_solver_download_covariance": ["cosl_pose_solver* s", "double* cov", "double* err", "double* out"],
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
        assert callable(getattr(api.PoseSolver, meth, None))
    vp = C.c_void_p
    assert api.LIB.cosl_pose_solver_set_covariance.argtypes == [vp, C.c_double]
    assert api.LIB.cosl_pose_solver_download_covariance.argtypes == [vp, vp, vp, vp]


def test_null_handle_is_invalid(api):
    out = (C.c_double * 4)()
    assert api.LIB.cosl_pose_solver_set_covariance(None, 1.0) == COSL_E_INVALID
    assert api.LIB.cosl_pose_solver_set_covariance(None, -1.0) == COSL_E_INVALID
    assert api.LIB.cosl_pose_solver_download_covariance(None, None, None, out) == COSL_E_INVALID

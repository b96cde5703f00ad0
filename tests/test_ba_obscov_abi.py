"""cosl_ba_solver_set_obs_cov and cosl_sba_motstr_levmar_x_cov at the C-ABI without a GPU: the header declares them
with these argument lists, the library exports them, the binding declares them, a NULL handle is refused, a
measurement covariance that is not finite, not symmetric or not positive definite is refused with the index of the
observation before any device work, and valid ones reach the device (COSL_E_CUDA without one)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import ba_dense as D
from test_gpu_ba_async import _torch_cuda

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSL_E_INVALID, COSL_E_CUDA = -1, -2

DECLS = {
    "cosl_ba_solver_set_obs_cov": ["cosl_ba_solver* s", "const double* covx"],
    "cosl_sba_motstr_levmar_x_cov": ["int n", "int ncon", "int m", "int mcon", "const char* vmask", "double* p",
                                     "int cnp", "int pnp", "const double* x", "const double* covx", "int mnp",
                                     "const double* rot0params", "int itmax", "int verbose", "const double opts[5]",
                                     "double info[10]", "int device"],
}


def test_header_declares_the_calls():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coslam_b200.h")).read(), flags=re.S)
    for name, args in DECLS.items():
        decl = re.search(r"\bint\s+%s\s*\(([^)]*)\)\s*;" % name, src)
        assert decl, name
        assert [" ".join(a.split()) for a in decl.group(1).split(",")] == args


def test_library_exports_and_binding_declares_them(api):
    lib = C.CDLL(api.LIB_PATH)
    for name in DECLS:
        assert hasattr(lib, name)
    assert callable(getattr(api.BaSolver, "set_obs_cov", None)) and callable(api.sba_motstr_levmar_x)
    vp, ci = C.c_void_p, C.c_int
    assert api.LIB.cosl_ba_solver_set_obs_cov.argtypes == [vp, vp]
    assert api.LIB.cosl_sba_motstr_levmar_x_cov.argtypes == [ci] * 4 + [vp, vp, ci, ci, vp, vp, ci, vp, ci, ci, vp,
                                                                       vp, ci]


def test_null_handle_is_invalid(api):
    cov = np.eye(2).reshape(1, 4)
    assert api.LIB.cosl_ba_solver_set_obs_cov(None, cov.ctypes.data_as(C.c_void_p)) == COSL_E_INVALID
    assert api.LIB.cosl_ba_solver_set_obs_cov(None, None) == COSL_E_INVALID


def _sba(api, covx):
    """cosl_sba_motstr_levmar_x_cov on a small rig scene: (rc, message, p before, p after)"""
    prob = D.rig_intrinsics(n=12)
    p, rot0, vmask = D.pack_sba(prob)
    p0 = p.copy()
    vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None  # noqa: E731
    opts = np.array([1e-7, 1e-12, 1e-12, 0.0, 1e-16])
    info = np.zeros(10)
    c = None if covx is None else np.ascontiguousarray(covx(prob.nobs), np.float64)
    rc = api.LIB.cosl_sba_motstr_levmar_x_cov(prob.n, prob.n_con, prob.m, prob.m_con, vp(vmask), vp(p), 11, 3,
                                              vp(prob.xy), vp(c), 2, vp(rot0), 5, 0, vp(opts), vp(info), 0)
    return rc, api.LIB.cosl_last_error().decode(), p0, p


def _spd(N):
    c = np.tile([2.0, 0.3, 0.3, 1.0], (N, 1))
    c[::3] = [0.25, -0.1, -0.1, 0.5]
    return c


BAD = {  # name -> (what to write into observation 7's [s00, s01, s10, s11], the word the message carries)
    "nan": ([np.nan, 0.0, 0.0, 1.0], "not finite"),
    "inf": ([1.0, 0.0, 0.0, np.inf], "not finite"),
    "asymmetric": ([1.0, 0.2, 0.2 + 1e-9, 1.0], "not symmetric"),
    "indefinite": ([1.0, 2.0, 2.0, 1.0], "not positive definite"),
    "negative": ([-1.0, 0.0, 0.0, 1.0], "not positive definite"),
    "zero": ([0.0, 0.0, 0.0, 0.0], "not positive definite"),
    "singular": ([1.0, 1.0, 1.0, 1.0], "not positive definite"),
}


@pytest.mark.parametrize("name", sorted(BAD))
def test_bad_covariances_are_invalid_and_named(api, name):
    entry, word = BAD[name]

    def covx(N):
        c = _spd(N)
        c[7] = entry
        c[11] = entry  # a later bad one: the first is named
        return c

    rc, msg, p0, p = _sba(api, covx)
    assert rc == COSL_E_INVALID, (rc, msg)
    assert "observation 7 " in msg and word in msg, msg
    assert np.array_equal(p, p0)


@pytest.mark.skipif(_torch_cuda() is not None, reason="checks the no-GPU failure mode")
@pytest.mark.parametrize("covx", [None, _spd, lambda N: _spd(N) * 1e4 + [0, 1e-10, 0, 0]], ids=["null", "spd", "scaled"])
def test_valid_covariances_reach_the_device(api, covx):
    rc, msg, p0, p = _sba(api, covx)
    assert rc == COSL_E_CUDA, (rc, msg)
    assert np.array_equal(p, p0)


def test_wrapper_checks_the_count(api):
    prob = D.rig_intrinsics(n=12)
    p, rot0, vmask = D.pack_sba(prob)
    with pytest.raises(ValueError):
        api.sba_motstr_levmar_x(p, rot0, vmask, prob.xy, 5, [1e-7, 1e-12, 1e-12, 0.0, 1e-16],
                                covx=np.tile(np.eye(2), (prob.nobs - 1, 1, 1)))

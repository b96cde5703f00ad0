"""ctypes access to oracle/_ref/libintracam_cov_ref.so = the UNMODIFIED reference file
/root/reference/src/slam/SL_IntraCamPose.cpp compiled against the stand-ins of oracle/ref_stubs/ with the working
covariance primitives of oracle/ref_stubs_cov/primitives_cov.cpp (recipe: `make -C oracle -f Makefile.obscov`, needs
/root/reference).  TEST INFRASTRUCTURE: used only by tests/ to pin the whitened pose restatement
(tests/pose_obscov_dense.py) to the reference's own intraCamCovEstimate."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "_ref", "libintracam_cov_ref.so")
_lib = None


def available():
    return os.path.exists(PATH)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(PATH)
        vp = C.c_void_p
        L.ref_intraCamCovEstimate.argtypes = [vp, vp, vp, C.c_int, vp, vp, vp, vp, C.c_double, vp, vp, vp, vp]
        L.ref_intraCamCovEstimate.restype = C.c_int
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def intracam_cov_estimate(K, R0, t0, Ms, ms, covx, tau, prev_errs=None, opt_in=None):
    """intraCamCovEstimate of the reference (slam/SL_IntraCamPose.cpp:711-795) with the image-plane covariances covx
    [n, 2, 2] or [n, 4] (px^2) that the harness's getProjectionCovMat hands back per point.  opt_in as
    ref.intracam_estimate's.  Returns ok, R, t, dict of the option block after the call."""
    K = np.ascontiguousarray(K, np.float64).ravel()
    R0 = np.ascontiguousarray(R0, np.float64).ravel()
    t0 = np.ascontiguousarray(t0, np.float64).ravel()
    Ms = np.ascontiguousarray(Ms, np.float64).reshape(-1, 3)
    ms = np.ascontiguousarray(ms, np.float64).reshape(-1, 2)
    cv = np.ascontiguousarray(covx, np.float64).reshape(-1, 4)
    assert len(cv) == len(Ms)
    pe = None if prev_errs is None else np.ascontiguousarray(prev_errs, np.float64)
    oi = None if opt_in is None else np.ascontiguousarray(opt_in, np.float64)
    R, t, oo = np.empty(9), np.empty(3), np.zeros(8)
    ok = lib().ref_intraCamCovEstimate(_p(K), _p(R0), _p(t0), len(Ms), _p(pe), _p(cv), _p(Ms), _p(ms), float(tau),
                                       _p(R), _p(t), _p(oi), _p(oo))
    keys = ("lambda", "lambda0", "err0", "err", "errRW", "retTypeLM", "nIterLM", "nIterRW")
    return bool(ok), R.reshape(3, 3), t, dict(zip(keys, oo))

"""ctypes access to oracle/liboracle_pg_general.so = posegraph_general_oracle.cpp, the CPU restatement of
the camera-group merge's pose-graph solve (built by oracle/Makefile.pg_general).  TEST INFRASTRUCTURE:
used by tests/, tests/golden/ and tools/ only."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is not None:
        return _LIB
    path = os.path.join(_HERE, "liboracle_pg_general.so")
    if not os.path.exists(path):
        subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "Makefile.pg_general", "liboracle_pg_general.so"])
    L = C.CDLL(path)
    L.orc_posegraph_solve.argtypes = ([C.c_int] + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 5 + [C.c_int]
                                      + [C.c_void_p] * 3)
    _LIB = L
    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def posegraph_solve(fixed, R, t, id1, id2, eR, et, scale_col=None, n_scale=0):
    """General pose graph with shared unknown scales (posegraph_oracle.cpp: computeNewCameraRotations +
    computeNewCameraTranslations4).  scale_col[e] = scale column of edge e, -1 = known scale; None:
    all known.  Returns newR (n,3,3), newt (n,3), scale (n_scale,); raises on a rank-deficient system
    or bad indices."""
    fx = np.ascontiguousarray(fixed, np.int32)
    n = fx.size
    R = np.ascontiguousarray(R, np.float64).reshape(n, 3, 3)
    t = np.ascontiguousarray(t, np.float64).reshape(n, 3)
    id1 = np.ascontiguousarray(id1, np.int32)
    id2 = np.ascontiguousarray(id2, np.int32)
    ne = id1.size
    eR = np.ascontiguousarray(eR, np.float64).reshape(ne, 3, 3)
    et = np.ascontiguousarray(et, np.float64).reshape(ne, 3)
    sc = None if scale_col is None else np.ascontiguousarray(scale_col, np.int32)
    nR, nt, s = np.empty((n, 3, 3)), np.empty((n, 3)), np.empty(max(1, int(n_scale)))
    rc = lib().orc_posegraph_solve(n, _ptr(fx), _ptr(R), _ptr(t), ne, _ptr(id1), _ptr(id2), _ptr(eR), _ptr(et),
                                   _ptr(sc), int(n_scale), _ptr(nR), _ptr(nt), _ptr(s))
    if rc != 0:
        raise RuntimeError("orc_posegraph_solve: " + ("rank-deficient system" if rc == 1 else "bad index"))
    return nR, nt, s[:int(n_scale)]

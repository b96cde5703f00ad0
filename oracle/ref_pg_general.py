"""ctypes access to oracle/_ref/libposegraph_merge_ref.so = the UNMODIFIED reference file
slam/SL_GlobalPoseEstimation.cpp compiled against the stand-ins of oracle/ref_stubs_pg/ with the C entry
of oracle/ref_stubs_pg/merge_entry.cpp (recipe: oracle/Makefile.pg_general, target `ref`; needs the
reference tree).  TEST INFRASTRUCTURE: pins oracle/posegraph_general_oracle.cpp and generates
tests/golden/posegraph_merge_ref.npz."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "_ref", "libposegraph_merge_ref.so")
_lib = None


def available():
    return os.path.exists(PATH)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def posegraph_merge(fixed, R, t, id1, id2, eR, et, scale_id):
    """MergeCameraGroup::recomputeKeyCamPoses of the reference on a graph built the way
    _constructGraphForKeyFrms does (app/SL_MergeCameraGroup.cpp:907-1035, :1083-1086): scale_id[e] >= 0
    marks a constraint edge with uncertain scale and that scale id.  Runs computeNewCameraRotations +
    computeNewCameraTranslations4 (slam/SL_GlobalPoseEstimation.cpp:52-218, :361-525).  Returns newR,
    newt, s (CamPoseEdge::s per edge)."""
    global _lib
    if _lib is None:
        _lib = C.CDLL(PATH)
        _lib.ref_posegraph_merge.argtypes = [C.c_int] + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 8
        _lib.ref_posegraph_merge.restype = None
    fx = np.ascontiguousarray(fixed, np.int32)
    n = fx.size
    R = np.ascontiguousarray(R, np.float64).reshape(n, 3, 3)
    t = np.ascontiguousarray(t, np.float64).reshape(n, 3)
    id1 = np.ascontiguousarray(id1, np.int32)
    id2 = np.ascontiguousarray(id2, np.int32)
    ne = id1.size
    eR = np.ascontiguousarray(eR, np.float64).reshape(ne, 3, 3)
    et = np.ascontiguousarray(et, np.float64).reshape(ne, 3)
    sid = np.ascontiguousarray(scale_id, np.int32)
    nR, nt, s = np.empty((n, 3, 3)), np.empty((n, 3)), np.zeros(max(1, ne))
    _lib.ref_posegraph_merge(n, _p(fx), _p(R), _p(t), ne, _p(id1), _p(id2), _p(eR), _p(et), _p(sid),
                                _p(nR), _p(nt), _p(s))
    return nR, nt, s[:ne]

"""BA problems the C-ABI refuses before it touches a device (no GPU needed): a (point, camera) pair
observed twice, and observation lists that do not start at 0 -- in the library and in the oracle."""
import ctypes as C
import os
import re

import numpy as np

from coslam_b200 import api
from coslam_b200.ctypes_defs import BaOptions
from coslam_b200.problem import BAProblem

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSL_E_INVALID = -1


def problem(cams_per_point, m=4, m_con=1):
    n = len(cams_per_point)
    cam = np.concatenate([np.asarray(c, np.int32) for c in cams_per_point])
    ptr = np.concatenate([[0], np.cumsum([len(c) for c in cams_per_point])]).astype(np.int64)
    K = np.tile([500.0, 0, 320, 0, 500, 240, 0, 0, 1], (m, 1))
    R = np.tile(np.eye(3).ravel(), (m, 1))
    t = np.zeros((m, 3))
    X = np.column_stack([np.zeros(n), np.zeros(n), np.full(n, 5.0)])
    return BAProblem(K, R, t, X, ptr, cam, np.full((len(cam), 2), 300.0), m_con, 0)


def create(prob):
    h = C.c_void_p()
    s = prob.struct()
    rc = api.LIB.cosl_ba_solver_create(C.byref(s), C.byref(BaOptions.defaults()), None, C.byref(h))
    if rc == 0:
        api.LIB.cosl_ba_solver_destroy(h)
    return rc, api.LIB.cosl_last_error().decode()


def test_header_states_one_observation_per_pair():
    src = open(os.path.join(ROOT, "include", "coslam_b200.h")).read()
    doc = src[:src.index("} cosl_ba_problem;")]
    assert re.search(r"a camera observes a point at most once", doc)


def test_duplicate_observation_is_invalid():
    rc, err = create(problem([[0, 1, 2], [1, 2, 2, 3], [0, 3]]))
    assert rc == COSL_E_INVALID and "twice" in err
    # the same camera twice, not next to each other (the lists need not be sorted for the check)
    rc, err = create(problem([[0, 1], [2, 3, 2]]))
    assert rc == COSL_E_INVALID and "twice" in err


def test_ptr_must_start_at_zero():
    prob = problem([[0, 1], [1, 2]])
    prob.ptr = np.array([1, 2, 4], np.int64)
    prob.cam = np.array([0, 1, 1, 2], np.int32)
    prob.xy = np.full((4, 2), 300.0)
    assert create(prob)[0] == COSL_E_INVALID


def test_valid_problem_passes_the_checks():
    """A problem without repeated pairs gets past validation: COSL_OK with a device, COSL_E_CUDA
    (no device) without one -- never COSL_E_INVALID."""
    rc, _ = create(problem([[0, 1, 2], [1, 2, 3], [0, 3]]))
    assert rc != COSL_E_INVALID


def test_oracle_refuses_duplicates(orc):
    prob = problem([[0, 1, 2], [1, 2, 2, 3], [0, 3]])
    s = prob.struct()
    info = np.zeros(16)
    rc = orc.lib().orc_ba_run_fixed(C.byref(s), C.byref(BaOptions.defaults()), 1, info.ctypes.data_as(C.c_void_p))
    assert rc == COSL_E_INVALID

"""cosl_ba_solver_stop / _progress at the C-ABI without a GPU: the header declares both calls, the library
exports them, the binding declares them, and a NULL handle is refused."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from coslam_b200 import synth
from coslam_b200.ctypes_defs import BaOptions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COSL_E_INVALID, COSL_E_CUDA = -1, -2


def _torch_cuda():
    try:
        import torch
        return torch if torch.cuda.is_available() else None
    except Exception:
        return None


def test_header_declares_stop_and_progress():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coslam_b200.h")).read(), flags=re.S)
    for name, args in (("stop", ["cosl_ba_solver* s"]), ("progress", ["cosl_ba_solver* s", "double out[8]"])):
        decl = re.search(r"\bint\s+cosl_ba_solver_%s\s*\(([^)]*)\)\s*;" % name, src)
        assert decl, name
        assert [a.strip() for a in decl.group(1).split(",")] == args


def test_library_exports_and_binding_declares_stop_and_progress(api):
    lib = C.CDLL(api.LIB_PATH)
    for name in ("stop", "progress"):
        assert hasattr(lib, "cosl_ba_solver_" + name)
        assert callable(getattr(api.BaSolver, name, None))
    assert api.LIB.cosl_ba_solver_stop.argtypes == [C.c_void_p]
    assert api.LIB.cosl_ba_solver_progress.argtypes == [C.c_void_p, C.POINTER(C.c_double)]


def test_null_handle_is_invalid_for_stop_and_progress(api):
    out = (C.c_double * 8)()
    assert api.LIB.cosl_ba_solver_stop(None) == COSL_E_INVALID
    assert api.LIB.cosl_ba_solver_progress(None, out) == COSL_E_INVALID


@pytest.mark.skipif(_torch_cuda() is not None, reason="checks the no-GPU failure mode")
def test_no_solver_to_stop_without_a_gpu(api):
    """Without a device creation reports COSL_E_CUDA and leaves the handle NULL, which stop and progress
    refuse (no CPU fallback)."""
    prob = synth.make_ba_scene(2, 3, 200, 320, 240, seed=6, m_con=2, n_con=2)[0]
    h = C.c_void_p()
    opt = BaOptions.defaults()
    assert api.LIB.cosl_ba_solver_create(C.byref(prob.struct()), C.byref(opt), None, C.byref(h)) == COSL_E_CUDA
    assert not h.value
    assert api.LIB.cosl_ba_solver_stop(h) == COSL_E_INVALID
    out = np.zeros(8)
    assert api.LIB.cosl_ba_solver_progress(h, out.ctypes.data_as(C.POINTER(C.c_double))) == COSL_E_INVALID

"""Static checks on the compiled gain trackers (no GPU needed): the SASS of klt_gain_fused and
klt_gain_pass in the built library holds no select between scalar kernel parameters, and the
kernels keep their register budget without spilling.

A kernel-parameter struct can only be read with constant loads at fixed offsets.  Code that picks
a field from one of two by-value parameter structs (a reference bound to `cond ? A : B`) compiles
to chains of predicated 32-bit LDCs over every candidate offset, once per field read; a plain
select between two scalar parameters still leaves one predicated LDC per field.  The tracker runs
that code on every pass, so any predicated 32-bit LDC is a regression.  ptxas also predicates
the 64-bit load of a pointer parameter that only a predicated access uses (one such load each in
the fused and the per-pass kernel); those are not selects and are allowed.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "coslam_b200", "libcoslam_b200.so")
KERNELS = ["klt_gain_fusedILi3E", "klt_gain_fusedILi0E", "klt_gain_passILi3E", "klt_gain_passILi0E"]
MAX_REGS = 128  # 4 CTAs of 128 threads per SM for the fused kernel


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    if exe is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip(f"{LIB} is not built")
    return exe


def _by_function(text, header):
    """{mangled name: text of its section} for the kernels under test"""
    out = {}
    for part in re.split(header, text)[1:]:
        name = part.split(None, 1)[0].rstrip(":")
        for k in KERNELS:
            if k in name:
                out[k] = part
    missing = [k for k in KERNELS if k not in out]
    assert not missing, f"kernels not found in {LIB}: {missing}"
    return out


def test_gain_trackers_have_no_predicated_scalar_constant_loads():
    exe = _cuobjdump()
    sass = subprocess.run([exe, "-sass", LIB], check=True, capture_output=True, text=True).stdout
    bad = {}
    for k, body in _by_function(sass, r"\n\s*Function : ").items():
        loads = re.findall(r"@!?U?P[0-6T]\s+LDC(?:\.(?:U8|S8|U16|S16|32))?\s+[^;]*;", body)
        if loads:
            bad[k] = (len(loads), loads[:4])
    assert not bad, f"predicated 32-bit constant loads (selects between kernel parameters): {bad}"


def test_gain_trackers_register_budget_and_no_spills():
    exe = _cuobjdump()
    res = subprocess.run([exe, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    for k, body in _by_function(res, r"\n\s*Function ").items():
        m = re.search(r"REG:(\d+)\s+STACK:(\d+)\s+SHARED:\d+\s+LOCAL:(\d+)", body)
        assert m, f"no resource usage for {k}"
        regs, stack, local = map(int, m.groups())
        assert regs <= MAX_REGS, f"{k}: {regs} registers > {MAX_REGS}"
        assert stack == 0 and local == 0, f"{k}: spills (stack {stack} B, local {local} B)"

"""Static checks on the KLT detector link's programmatic dependent launches (no GPU needed).

klt_nm_verify and klt_select_refill are launched with programmatic stream serialization.  In the
built library every instance of both executes griddepcontrol.wait (SASS ACQBULK) exactly once and
griddepcontrol.launch_dependents (PREEXIT) after it; klt_select_refill reads the feature table for
its dead-slot scan before the wait, and the candidate keys only after it.  Both keep a small
register count and use no local memory.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "coslam_b200", "libcoslam_b200.so")
KERNELS = ["klt_nm_verifyILb0EE", "klt_nm_verifyILb1EE", "klt_select_refillILb0EE", "klt_select_refillILb1EE"]
MAX_REGS = {"klt_nm_verify": 40, "klt_select_refill": 64}  # select: 1024 threads per CTA


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
    out = {}
    for part in re.split(header, text)[1:]:
        name = part.split(None, 1)[0].rstrip(":")
        for k in KERNELS:
            if k in name:
                out[k] = part
    missing = [k for k in KERNELS if k not in out]
    assert not missing, f"kernels not found in {LIB}: {missing}"
    return out


def _offsets(body, opcode):
    pat = r"/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P[0-7T]\s+)?" + re.escape(opcode) + r"\b"
    return [int(a, 16) for a in re.findall(pat, body)]


def test_detector_kernels_wait_once_and_trigger_after_the_wait():
    exe = _cuobjdump()
    text = subprocess.run([exe, "-sass", LIB], check=True, capture_output=True, text=True).stdout
    for k, body in _by_function(text, r"\n\s*Function : ").items():
        wait, trig = _offsets(body, "ACQBULK"), _offsets(body, "PREEXIT")
        assert len(wait) == 1, f"{k}: griddepcontrol.wait at {wait}"
        assert len(trig) == 1 and wait[0] < trig[0], f"{k}: launch_dependents {trig} not after the wait {wait}"


def test_detector_kernels_keep_registers_without_local_memory():
    exe = _cuobjdump()
    res = subprocess.run([exe, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    for k, body in _by_function(res, r"\n\s*Function ").items():
        m = re.search(r"REG:(\d+)\s+STACK:(\d+)\s+SHARED:\d+\s+LOCAL:(\d+)", body)
        assert m, f"no resource usage for {k}"
        regs, stack, local = map(int, m.groups())
        assert regs <= MAX_REGS[k.split("ILb")[0]], f"{k}: {regs} registers"
        assert stack == 0 and local == 0, f"{k}: stack {stack} B, local {local} B"

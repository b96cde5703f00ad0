"""Static checks on the programmatic dependent launches of the KLT pyramid chain (no GPU needed).

Levels >= 2 of the pyramid (klt_pyr_down_tma) are launched with programmatic stream serialization,
so their CTAs may start while the kernel that writes their source level (klt_front or the level
above) still runs.  In the built library:
  * every klt_pyr_down_tma instance executes griddepcontrol.wait (SASS ACQBULK) after its
    tensor-map prefetches and before its TMA load (UTMALDG), and griddepcontrol.launch_dependents
    (PREEXIT) after the wait;
  * every klt_front instance executes launch_dependents after the last of its global stores, not at
    kernel start;
  * no instance uses more registers or stack than it did before the change.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "coslam_b200", "libcoslam_b200.so")
PYR = ["klt_pyr_down_tmaILb0EE", "klt_pyr_down_tmaILb1EE"]
FRONT = ["klt_frontILb0ELb0EE", "klt_frontILb0ELb1EE", "klt_frontILb1ELb0EE", "klt_frontILb1ELb1EE"]
# (registers, stack bytes) per instance; the STORE_L0 front passes already spilled a few bytes
BUDGET = {"klt_pyr_down_tmaILb0EE": (30, 0), "klt_pyr_down_tmaILb1EE": (30, 0),
          "klt_frontILb0ELb0EE": (128, 0), "klt_frontILb0ELb1EE": (128, 0),
          "klt_frontILb1ELb0EE": (128, 8), "klt_frontILb1ELb1EE": (128, 16)}


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


def _by_function(text, header, kernels):
    """{kernel: text of its section}"""
    out = {}
    for part in re.split(header, text)[1:]:
        name = part.split(None, 1)[0].rstrip(":")
        for k in kernels:
            if k in name:
                out[k] = part
    missing = [k for k in kernels if k not in out]
    assert not missing, f"kernels not found in {LIB}: {missing}"
    return out


def _offsets(body, opcode):
    """addresses of the instructions whose opcode (after an optional predicate) starts with `opcode`"""
    pat = r"/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P[0-7T]\s+)?" + re.escape(opcode) + r"\b"
    return [int(a, 16) for a in re.findall(pat, body)]


@pytest.fixture(scope="module")
def sass():
    exe = _cuobjdump()
    text = subprocess.run([exe, "-sass", LIB], check=True, capture_output=True, text=True).stdout
    return _by_function(text, r"\n\s*Function : ", PYR + FRONT)


def test_pyramid_levels_wait_for_their_source_before_the_tma_load(sass):
    for k in PYR:
        body = sass[k]
        wait, load, pf = _offsets(body, "ACQBULK"), _offsets(body, "UTMALDG"), _offsets(body, "UTMACCTL.PF")
        trig = _offsets(body, "PREEXIT")
        assert len(wait) == 1 and len(load) == 1, f"{k}: griddepcontrol.wait {wait}, TMA loads {load}"
        assert wait[0] < load[0], f"{k}: the TMA load at {load[0]:#x} precedes the wait at {wait[0]:#x}"
        assert len(pf) == 2 and max(pf) < wait[0], f"{k}: tensor-map prefetches {pf} not ahead of the wait"
        assert len(trig) == 1 and wait[0] < trig[0], f"{k}: launch_dependents {trig} not after the wait"


def test_front_pass_triggers_its_dependents_after_its_stores(sass):
    for k in FRONT:
        body = sass[k]
        trig, stores = _offsets(body, "PREEXIT"), _offsets(body, "STG")
        assert len(trig) == 1, f"{k}: {len(trig)} launch_dependents"
        assert stores and max(stores) < trig[0], f"{k}: a global store follows launch_dependents"
        assert not _offsets(body, "ACQBULK"), f"{k}: the front pass waits on a grid dependency"


def test_pdl_kernels_keep_their_register_budget():
    exe = _cuobjdump()
    res = subprocess.run([exe, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    for k, body in _by_function(res, r"\n\s*Function ", PYR + FRONT).items():
        m = re.search(r"REG:(\d+)\s+STACK:(\d+)\s+SHARED:\d+\s+LOCAL:(\d+)", body)
        assert m, f"no resource usage for {k}"
        regs, stack, local = map(int, m.groups())
        max_regs, max_stack = BUDGET[k]
        assert regs <= max_regs, f"{k}: {regs} registers > {max_regs}"
        assert stack <= max_stack and local == 0, f"{k}: stack {stack} B (budget {max_stack}), local {local} B"

"""Static checks on the window walk of the hw = 3 gain trackers (no GPU needed).

Lane gl < 7 of a lane group owns window column gl and reads tap rows 0..7 of columns gl and gl + 1:
16 LDS.128 per window instead of 4 per pixel (28 per lane), both for the I0 samples staged once per
level and for the I1 samples of every pass.  The build before the column walk issued 56 LDS.128 in
each klt_gain_fused<3, *> instance; the column walk issues 32.  The pixel coordinates are constants
plus the lane index, so no division by the window width (a multiply-high by the reciprocal of 7)
is left in either driver.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "coslam_b200", "libcoslam_b200.so")
FUSED = ["klt_gain_fusedILi3ELb0E", "klt_gain_fusedILi3ELb1E"]
PASS = ["klt_gain_passILi3ELb0E", "klt_gain_passILi3ELb1E"]
LDS128_BEFORE = 56  # per klt_gain_fused<3, *> instance, row-major walk
LDS128_COLUMN_WALK = 2 * 16  # I0 staging + one pass
# x / 7 and x % 7 compile to a multiply-high by 0x92492493 (signed, shown as -0x6db6db6d) or by
# 0x24924925 (unsigned)
DIV7 = re.compile(r"IMAD\.HI(?:\.U32)?\s[^;]*(?:0x6db6db6d|0x92492493|0x24924925|0x24924924)")


def _sass():
    exe = shutil.which("cuobjdump")
    if exe is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    if exe is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip(f"{LIB} is not built")
    text = subprocess.run([exe, "-sass", LIB], check=True, capture_output=True, text=True).stdout
    out = {}
    for part in re.split(r"\n\s*Function : ", text)[1:]:
        name = part.split(None, 1)[0]
        for k in FUSED + PASS:
            if k in name:
                out[k] = part
    missing = [k for k in FUSED + PASS if k not in out]
    assert not missing, f"kernels not found in {LIB}: {missing}"
    return out


def test_fused_hw3_tracker_shares_the_bilinear_taps():
    bodies = _sass()
    for k in FUSED:
        n = len(re.findall(r"\bLDS\.128\b", bodies[k]))
        assert n < LDS128_BEFORE, f"{k}: {n} LDS.128, the row-major walk issued {LDS128_BEFORE}"
        assert n <= LDS128_COLUMN_WALK, f"{k}: {n} LDS.128 > {LDS128_COLUMN_WALK} of the column walk"


def test_hw3_trackers_do_not_divide_by_the_window_width():
    bodies = _sass()
    for k in FUSED + PASS:
        hits = DIV7.findall(bodies[k])
        assert not hits, f"{k}: division by 7 in the window walk: {hits[:3]}"

"""Generates tests/golden/posegraph_merge_ref.npz from the UNMODIFIED reference file
slam/SL_GlobalPoseEstimation.cpp (compiled by `make -C oracle -f Makefile.pg_general ref` into
oracle/_ref/libposegraph_merge_ref.so; needs the reference tree, so it runs where that is present).  Cases: key-frame graphs of a camera-group
merge as MergeCameraGroup::_constructGraphForKeyFrms builds them, solved by computeNewCameraRotations +
computeNewCameraTranslations4 -- 2, 4 and 13 cameras, 1 and 3 constraint edges, two scale ids, noisy
measurements."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from coslam_b200.synth import make_merge_graph  # noqa: E402
from oracle import ref_pg_general as ref  # noqa: E402

SPECS = [
    dict(n_key=6, n_cams=2, seed=1, n_constraints=1),
    dict(n_key=8, n_cams=4, seed=2, n_constraints=1),
    dict(n_key=8, n_cams=4, seed=3, n_constraints=3),
    dict(n_key=5, n_cams=13, seed=4, n_constraints=3),
    dict(n_key=6, n_cams=4, seed=5, n_constraints=3, n_scale_ids=2),
    dict(n_key=7, n_cams=4, seed=6, n_constraints=2, noise=0.01),
    dict(n_key=4, n_cams=13, seed=7, n_constraints=1, noise=0.02),
]
KEYS = ("fixed", "R", "t", "id1", "id2", "eR", "et", "scale_id")

if __name__ == "__main__":
    cases = {}
    for i, sp in enumerate(SPECS):
        g = make_merge_graph(**sp)
        nR, nt, s = ref.posegraph_merge(*(g[k] for k in KEYS))
        for k in KEYS:
            cases[f"c{i}_{k}"] = g[k]
        cases[f"c{i}_newR"], cases[f"c{i}_newt"], cases[f"c{i}_s"] = nR, nt, s
    cases["n_cases"] = np.int32(len(SPECS))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "posegraph_merge_ref.npz"), **cases)
    print("wrote", len(SPECS), "cases")

"""Worker for tests/test_flow_lm_boundaries.py: runs flow-LM cases on the single-CTA kernel.  The parent sets VDO_FLOW_SINGLE_CTA=1,
which the library reads once per process, hence a process of its own.  argv: output .npz, then cases as n:mode:quirk."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run(out_path, cases):
    from vdo_slam_b200 import capi
    from tests.test_flow_lm_boundaries import single_cta_problem
    assert os.environ.get("VDO_FLOW_SINGLE_CTA"), "run with VDO_FLOW_SINGLE_CTA=1"
    ctx = capi.Context(0)
    out = {}
    for n, mode, quirk in cases:
        g = capi.pose_opt_flow2(ctx, [single_cta_problem(n, mode, quirk)], quirk=quirk, modes=[mode], trace=True)[0]
        key = f"{n}_{mode}_{quirk}_"
        for k in ("T", "flow", "inlier", "stats"):
            out[key + k] = g[k]
        for k, v in g["trace"].items():
            out[key + "trace_" + k] = np.asarray(v)
    np.savez(out_path, **out)


if __name__ == "__main__":
    run(sys.argv[1], [tuple(int(v) for v in c.split(":")) for c in sys.argv[2:]])

#!/usr/bin/env python
"""Generate tests/golden/lm_solve_pins.npz on a machine with an H100 (the library built):

    python tests/golden/make_lm_golden.py [OUT]

lm_solve_pins.npz  the outputs of the device Levenberg-Marquardt solves and of the log-det greedy selection on the cases of
                   lm_pins_lib (ODOM, RIG, GD), as computed before the solvers shared one trust-region policy and one Cholesky
                   (csrc/lm.cuh).  mloam_odom_solve (free_mask 1, 2, 3; converged, capped at max_iterations, a far start, a single
                   plane): pose_i, ext, lm_iterations, termination, final_cost and H.  mloam_calib_rig on three LiDARs with and without
                   priors: the same, with every extrinsic and the rows per LiDAR.  good_features (gd): the selected indices.  Each case
                   also holds inputs_sha256, the checksum of the seeded inputs the outputs belong to.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402
import lm_pins_lib as lpl  # noqa: E402


def main(out):
    m = ge._load()
    ctx = m.Context(0)
    try:
        rec = lpl.run_all(ctx)
    finally:
        ctx.close()
    np.savez(out, **rec)
    for k in sorted(rec):
        if k.endswith((".termination", ".lm_iterations")):
            print(k, int(rec[k]))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "lm_solve_pins.npz"))

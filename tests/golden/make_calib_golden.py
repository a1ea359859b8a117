#!/usr/bin/env python
"""Generate tests/golden/calib_frame_12dof.npz on a machine with an H100 (the library built):

    python tests/golden/make_calib_golden.py [OUT]

calib_frame_12dof.npz  mloam_calib_frame's outputs on the cases of calib_rig_lib.CALIB_GOLDEN, as computed by its own 12-DoF
                       implementation ([pose_i | ext_cal] in one 12x12 system, two matcher passes per outer iteration), before
                       that implementation was replaced by the rig solver's two-LiDAR case.  Per case: pose_i, ext_cal, the stats
                       termination, lm_iterations, n_surf, final_cost, n_surf_in, n_corner_in and H, and inputs_sha256, the
                       checksum of the seeded inputs the outputs belong to.  Two runs in fresh processes gave identical bytes.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402
import calib_rig_lib as crl  # noqa: E402


def main(out):
    m = ge._load()
    ctx = m.Context(0)
    rec = {}
    try:
        for name, (kind, outer, inner, groups, own) in crl.CALIB_GOLDEN.items():
            cs = crl.calib_golden_inputs(kind)
            crl.calib_golden_maps(ctx, cs, own)
            pi, ec, st = ctx.calib_frame(*crl.calib_golden_groups(cs, groups), cs["pivot"], cs["pose_i_init"], cs["ext_ref"], cs["ext_cal_init"],
                                         outer, inner, own_cal_maps=own)
            rec[f"{name}.inputs_sha256"] = np.array(cs["sha256"])
            rec[f"{name}.pose_i"], rec[f"{name}.ext_cal"] = pi, ec
            for k in crl.CALIB_GOLDEN_STATS:
                rec[f"{name}.{k}"] = np.array(st[k])
            rec[f"{name}.H"] = np.asarray(st["H"], np.float64)
    finally:
        ctx.close()
    np.savez(out, **rec)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "calib_frame_12dof.npz"))

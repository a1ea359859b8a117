"""The online-calibration step over the whole rig on one GPU: python tools/bench_calib_rig.py [--steps 100] [--repeats 5].

bench.py's C4 rig: 4 LiDARs x 64 rings x 2048 columns, the RV extrinsics (tests/synthetic.py rig_extrinsics) with LiDARs 1-3 off by 2 deg /
5 cm, seeded synthetic sweeps (frame i for LiDAR 0, the pivot frame for the others), leaf 0.4 / 0.2 features.  The local maps are
buildCalibMap's: the reference LiDAR's features of the window's five frames (pivot .. pivot + 4), moved into the pivot frame and filtered
with leaf 0.2 by mloam_local_map_build into map slots 0 / 1.  max_outer 2, max_inner 4, no prior.  Arms, alternated `--repeats` times in
one process, `--steps` calls each:
  rig       mloam_calib_rig over the four LiDARs (one problem, one trust region)
  chained   three mloam_calib_frame calls, one per calibrated LiDAR, each solving pose_i again — a different problem, for cost only
and once the CPU oracle (orc_calib_rig, serial) on the same inputs and maps.  Reported: calls/s and ms per call of each arm (host clock
around calls that end in a device synchronise), launches per call, the oracle's ms, the largest pose difference between the GPU and the
oracle, and the command's steps and repeats.  The card name and power limit are read in the same run.  Writes nothing into the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import __graft_entry__ as ge  # noqa: E402
import calib_rig_lib as crl  # noqa: E402
import oracle_lib as orc  # noqa: E402
import synthetic as syn  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    m = ge._load()
    scene = syn.make_scene()
    tiny = syn.make_submap(scene, 1000)  # make_rig_case's own map is replaced by the window's local map below
    rc = crl.make_rig_case(scene, 4, 64, 2048, 0, submap=tiny)
    ctx = m.Context(0)
    traj, ext0 = syn.trajectory(10), syn.rig_extrinsics(4)[0]
    surf_stack, corner_stack, pose_local = [], [], []
    for k in range(3, 8):  # the window: pivot (frame 3) .. frame 7 = frame i
        cloud, ss, se = syn.make_sweep(scene, traj[k], 64, 2048, seed=500 + k, lidar_id=0, ext=ext0)
        f = orc.extract_cloud(cloud, ss, se)
        surf_stack.append(orc.voxel_grid(f["surf_points_less_flat"], 0.4, False)[0])
        corner_stack.append(orc.voxel_grid(f["corner_points_less_sharp"], 0.2, False)[0])
        pose_local.append(syn.pose_mul(syn.pose_inv(rc["pivot"]), syn.pose_mul(traj[k], ext0)))
    rc["corner_map"] = ctx.local_map_build(0, corner_stack, pose_local, 0.2)  # buildCalibMap's leaf, estimator.cpp:1103-1109
    rc["surf_map"] = ctx.local_map_build(1, surf_stack, pose_local, 0.2)
    outer, inner = 2, 4

    def rig():
        return ctx.calib_rig(rc["surf"], rc["corner"], rc["pivot"], rc["pose_i_init"], rc["ext_init"], 0, max_outer=outer, max_inner=inner)

    def chained():
        pi = rc["pose_i_init"]
        for n in (1, 2, 3):
            pi, _, _ = ctx.calib_frame(rc["surf"][0], rc["corner"][0], rc["surf"][n], rc["corner"][n], rc["pivot"], pi, rc["ext_init"][0],
                                       rc["ext_init"][n], outer, inner)

    arms = {"rig": rig, "chained": chained}
    res = {k: {"ms": [], "launches": None} for k in arms}
    for f in arms.values():  # warm-up: module load, first allocations
        f()
        f()
    for _ in range(a.repeats):
        for k, f in arms.items():
            l0 = ctx.launch_count()
            t0 = time.perf_counter()
            for _ in range(a.steps):
                f()
            res[k]["ms"].append(1e3 * (time.perf_counter() - t0) / a.steps)  # every call ends in a synchronise (its read-back)
            res[k]["launches"] = (ctx.launch_count() - l0) / a.steps
    pi, ex, st, rows = rig()
    t0 = time.perf_counter()
    rpi, rex, rst, rrows = crl.calib_rig(rc["surf_map"], rc["corner_map"], rc["surf"], rc["corner"], rc["pivot"], rc["pose_i_init"], rc["ext_init"], 0,
                                         max_outer=outer, max_inner=inner)
    orc_ms = 1e3 * (time.perf_counter() - t0)
    diff = max(max(syn.pose_err(pi, rpi)), max(max(syn.pose_err(ex[n], rex[n])) for n in range(4)))
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = {"config": "C4 rig 4 x 64 x 2048", "steps": a.steps, "repeats": a.repeats,
           "map_points": {"surf": int(rc["surf_map"].shape[0]), "corner": int(rc["corner_map"].shape[0])}, "features": int(sum(len(x) for x in rc["surf"] + rc["corner"])),
           "max_outer": outer, "max_inner": inner, "gpu": smi.splitlines()[0] if smi else None, "oracle_ms": round(orc_ms, 1),
           "rows_equal_oracle": bool(np.array_equal(rows, rrows)), "termination_equal_oracle": st["termination"] == rst["termination"],
           "max_pose_diff_vs_oracle": diff}
    for k, v in res.items():
        ms = float(np.median(v["ms"]))
        out[k] = {"ms_per_call_median": round(ms, 3), "ms_runs": [round(x, 3) for x in v["ms"]], "calls_per_s": round(1e3 / ms, 1),
                  "launches_per_call": v["launches"]}
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()

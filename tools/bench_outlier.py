"""Per-frame cost of the outlier cloud (mloam_set_outlier) in the closed mapper loop on one GPU:
python tools/bench_outlier.py [--frames 60] [--repeats 3].

tools/bench_mapper.py's device loop (mloam_keyframe_submap -> mloam_frame(rebuild_maps = 0) -> mloam_keyframe_save, C2-sized sweeps of one
64 x 2048 LiDAR through the rig merge, config_handheld's keyframe parameters) with the outlier cloud off and on (MAP_OUTLIER_RES 0.8 m),
the two arms alternated `--repeats` times in one process, plain and with_ua.  Reported per arm and run: the median ms of the frame call
and of the whole step, the launches per frame, and the largest pose difference between the arms (the outlier cloud does not touch the
solve) next to the one between the runs of the off arm, with the card name and power limit read in the same run.  Writes nothing into the tree."""
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
import bench_mapper as bm  # noqa: E402
import mapper_lib as ml  # noqa: E402
import synthetic as syn  # noqa: E402

LEAF = 0.8  # MAP_OUTLIER_RES of the KITTI / Oxford / UTBM configurations


def run(m, wl, with_ua, leaf):
    sweeps, odom, ext, ext_cov, thr = wl
    p = m.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = 64, 10, 1, 0.0, 2048
    ctx = m.Context(0, p)
    ctx.set_lidars(1, ext)
    ctx.set_uncertainty(with_ua, ext_cov if with_ua else None, bm.COV_MEAS, thr)
    ctx.set_outlier(leaf)
    ctx.keyframes_init(bm.KF["dist"], bm.KF["orient"], bm.KF["radius"], bm.KF["res"], thr)
    n = max(s[0].shape[0] for s in sweeps)
    buf = np.zeros((n, 4), np.float32)  # one sweep buffer: frames replay their graph
    wmap_wodom = np.array([0, 0, 0, 0, 0, 0, 1.0])
    ms_frame, ms_step, launches, poses = [], [], [], []
    for k, (cloud, ss, se, _) in enumerate(sweeps):
        buf[:] = 0
        buf[:cloud.shape[0]] = cloud
        pred = ml.pose_mul(wmap_wodom, odom[k])
        t0 = time.perf_counter()
        ctx.keyframe_submap(pred)
        l0 = ctx.launch_count()
        t1 = time.perf_counter()
        pose, _ = ctx.frame(buf, ss, se, None, None, pred, False)
        t2 = time.perf_counter()
        l1 = ctx.launch_count()
        ctx.keyframe_save()
        t3 = time.perf_counter()
        wmap_wodom = ml.pose_mul(pose, ml.pose_inv(odom[k]))
        poses.append(pose)
        if k > 1:  # the first steps also load modules and capture
            ms_frame.append((t2 - t1) * 1e3), ms_step.append((t3 - t0) * 1e3), launches.append(l1 - l0)
    ctx.close()
    return dict(ms_frame=float(np.median(ms_frame)), ms_step=float(np.median(ms_step)), launches_per_frame=float(np.median(launches)),
                poses=np.stack(poses))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 2
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    m = bench.load_mloam()
    wl = bm.workload(args.frames)
    out = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi.splitlines()[0] if smi else None, "frames": args.frames, "leaf": LEAF}
    for with_ua in (False, True):
        runs = {"off": [], "on": []}
        for _ in range(args.repeats):
            for arm in ("off", "on"):
                runs[arm].append(run(m, wl, with_ua, LEAF if arm == "on" else 0.0))
        res = {arm: {k: [round(r[k], 4) for r in v] for k in ("ms_frame", "ms_step", "launches_per_frame")} for arm, v in runs.items()}
        diff = lambda x, y: max(max(syn.pose_err(a, b)) for a, b in zip(x["poses"], y["poses"]))  # noqa: E731
        res["max_pose_diff_on_vs_off"] = max(diff(a, b) for a, b in zip(runs["on"], runs["off"]))
        res["max_pose_diff_between_off_runs"] = max(diff(runs["off"][0], b) for b in runs["off"][1:])
        out["with_ua" if with_ua else "plain"] = res
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())

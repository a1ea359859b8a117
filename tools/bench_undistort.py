"""Cost of the undistortion (mloam_set_distortion) in the frame path on one GPU, with the look-ahead on:
python tools/bench_undistort.py [--frames 60] [--warmup 10] [--repeats 3] [--configs C2,C4].

C2 (one 64 x 2048 LiDAR, 1M-point submap) and C4 (four of them, 5M points) as bench.py sizes them, 10 GN iterations, the submaps built once
(mloam_map_build) and frames with rebuild_maps = 0, every frame announcing the next sweep (mloam_frame_set_next).  Three arms:
  off        the undistortion off
  on         on, each sweep's poses given with its call (mloam_frame_undistort, a new pose every frame so that graph replays take it): the
             undistortion, the merge and both scan filters leave the look-ahead branch for the main stream of the call
  announced  on, each sweep's poses announced with the sweep (mloam_frame_set_next_undistort): the branch runs them again
The arms alternate `--repeats` times in one process.  Reported per arm and run: frames/s over the timed frames (host clock around calls that
end in a device synchronise), the median frame, launches per frame and graph captures in the timed window; per configuration the median
frame time the on and announced arms add over off, and whether the two on-arms' outputs (every timed pose and the last frame's scans) are
byte-identical.  The split of the on arm's added time: one more on-arm run with stage profiling (the stream path, event scopes around each
stage, serial filters, no look-ahead) reports the event-timed ms per frame of `k_undistort` ("undistort") and of the two scan filters
("voxel").  The card name and power limit are read in the same run.  Writes nothing into the tree."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
import synthetic as syn  # noqa: E402


def workload(cfg, n_sweeps=4):
    scene = syn.make_scene()
    traj = syn.trajectory(n_sweeps + 2)
    surf_map, corner_map = syn.make_submap(scene, cfg["map_points"])
    sweeps = [syn.make_multi_sweep(scene, traj[1 + k], cfg["lidars"], cfg["rings"], cfg["horizon"], seed=70 + k) for k in range(n_sweeps)]
    return traj, surf_map, corner_map, sweeps


def rlt(k):
    """The odometry's relative pose of sweep k (a new one every frame, so that graph replays take it)."""
    return np.array([0.5 + 0.001 * (k % 7), 0.01, 0.0, 0.0, 0.0, np.sin(0.01 + 0.001 * (k % 5)), np.cos(0.01 + 0.001 * (k % 5))])


def run(m, cfg, wl, arm, frames, warmup, profile=False):
    traj, surf_map, corner_map, sweeps = wl
    L = cfg["lidars"]
    p = m.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = cfg["rings"] * L, cfg["gn_iters"], 1, 0.0, cfg["horizon"]
    ctx = m.Context(0, p)
    try:
        ext = sweeps[0][3]
        ctx.set_lidars(L, ext)
        ctx.map_build(m.MAP_SURF, surf_map)
        ctx.map_build(m.MAP_CORNER, corner_map)
        if arm != "off":
            ctx.set_distortion(True, 0.1)
        if profile:
            ctx.profile(True)
        times, launches, poses = [], [], []
        captures0 = 0
        for k in range(warmup + frames):
            cloud, ss, se, _ = sweeps[k % len(sweeps)]
            nx = sweeps[(k + 1) % len(sweeps)]
            ctx.frame_set_next(nx[0], nx[1], nx[2])
            if arm == "announced":
                ctx.frame_set_next_undistort(m.undistort_poses(rlt(k + 1), 0, ext, 0))
            if arm == "on" or (arm == "announced" and k == 0):
                ctx.frame_undistort(m.undistort_poses(rlt(k), 0, ext, 0))
            if k == warmup:
                captures0 = ctx.profile_get("graph_captures")[1]
            l0 = ctx.launch_count()
            t0 = time.perf_counter()
            pose, _ = ctx.frame(cloud, ss, se, None, None, traj[1 + k % len(sweeps)], False)
            t1 = time.perf_counter()
            if k >= warmup:
                times.append(t1 - t0), launches.append(ctx.launch_count() - l0), poses.append(pose)
            if profile and k + 1 == warmup:
                ctx.profile_reset()
        if profile:
            return {name: ctx.profile_get(name)[0] / len(times) for name in ("undistort", "voxel", "extract")}
        out = np.concatenate([np.ravel(poses)] + [np.ravel(a).view(np.uint8) for a in ctx.frame_scan()]).tobytes()
        return dict(fps=len(times) / sum(times), median_ms=1e3 * float(np.median(times)), launches=float(np.mean(launches)),
                    captures=ctx.profile_get("graph_captures")[1] - captures0, undistort_ahead=ctx.profile_get("undistort_ahead")[1],
                    out=hashlib.sha256(out).hexdigest()[:16])
    finally:
        ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--configs", default="C2,C4")
    a = ap.parse_args()
    m = bench.load_mloam()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = {"gpu": smi, "configs": {}}
    for name in a.configs.split(","):
        cfg = dict(bench.CONFIGS[name])
        wl = workload(cfg)
        arms = {"off": [], "on": [], "announced": []}
        for _ in range(a.repeats):
            for arm in arms:
                arms[arm].append(run(m, cfg, wl, arm, a.frames, a.warmup))
        added = {arm: float(np.median([b["median_ms"] - o["median_ms"] for o, b in zip(arms["off"], arms[arm])])) for arm in ("on", "announced")}
        same = len({r["out"] for r in arms["on"] + arms["announced"]}) == 1
        split = run(m, cfg, wl, "on", a.frames, a.warmup, profile=True)
        out["configs"][name] = dict(arms, added_ms_per_frame=added, on_arms_identical=same, profiled_ms_per_frame=split)
        print(name, json.dumps(out["configs"][name]), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

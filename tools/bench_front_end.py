"""Raw driver sweeps into the frame path on one GPU: python tools/bench_front_end.py [--steps 30] [--repeats 3].

At the KITTI (1 x 64 rings, horizon 4000, ROI 1 m) and Oxford (2 x 32 rings, horizon 1800, timestamp overload) shapes, three variants
alternate `--repeats` times in one process on the same synthetic raw sweeps (firing order, tests/front_end_lib.py) and submap:
  chain       the path without a device front end: calTimestamp on the CPU (libm restatement), mloam_project_cloud per LiDAR (one H2D -> D2H
              round trip each), concatenation of clouds and ScanInfo on the host, then mloam_frame
  raw         mloam_frame_raw: removeNaN + calTimestamp + projection batched over the rig on the device
  raw_ahead   mloam_frame_raw with the next sweep announced (mloam_frame_set_next_raw): its front end and extraction run in the look-ahead
The line reports frames/s of each run, kernel launches per frame (mloam_launch_count), host-to-device bytes per frame of the sweep inputs
(exact; submaps excluded: every variant uploads the same ones), and the card name and power limit read in the same run.  Writes nothing into the tree."""
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

import front_end_lib as fel  # noqa: E402
import synthetic as syn  # noqa: E402

SHAPES = {"kitti": dict(n_lidars=1, rings=64, horizon=4000, roi=1.0, time_field=False),
          "oxford": dict(n_lidars=2, rings=32, horizon=1800, roi=0.5, time_field=True)}


def load_mloam():
    import importlib.util
    spec = importlib.util.spec_from_file_location("mloam_b200", os.path.join(ROOT, "m-loam_b200", "__init__.py"))
    m = importlib.util.module_from_spec(spec)
    sys.modules["mloam_b200"] = m
    spec.loader.exec_module(m)
    return m


def exts(n):
    return np.array([[0.3 * np.cos(2 * np.pi * l / n), 0.3 * np.sin(2 * np.pi * l / n), 0.0, 0.0, 0.0, np.sin(np.pi * l / (2 * n)),
                      np.cos(np.pi * l / (2 * n))] for l in range(n)])


def workload(s, n_frames, scene, traj):
    ext = exts(s["n_lidars"])
    frames = []
    for k in range(n_frames):
        parts = [fel.raw_sweep(scene, traj[k], s["rings"], s["horizon"], seed=100 * k + l, time_field=s["time_field"],
                               ext=ext[l] if s["n_lidars"] > 1 else None) for l in range(s["n_lidars"])]
        init = syn.perturb_pose(traj[k], np.random.Generator(np.random.PCG64(k)))
        timed = sum(fel.cal_timestamp(pp, s["time_field"], 0.1).nbytes for pp in parts)
        proj, _, _ = fel.front_end(np.concatenate(parts), [p.shape[0] for p in parts], s["rings"], s["horizon"], s["roi"], 0.1, s["time_field"])
        chain_h2d = timed + proj.nbytes + 8 * s["n_lidars"] * s["rings"]  # exact: the per-LiDAR uploads, the sweep and its ScanInfo
        frames.append(dict(raw=np.ascontiguousarray(np.concatenate(parts)), counts=np.array([p.shape[0] for p in parts], np.int32),
                           parts=parts, init=init, chain_h2d=chain_h2d))
    return ext, frames


def run(m, s, ext, frames, surf_map, corner_map, variant, steps):
    p = m.default_params()
    p.n_scans, p.max_inner, p.max_ring_points = s["n_lidars"] * s["rings"], 1, s["horizon"]
    ctx = m.Context(0, p)
    if s["n_lidars"] > 1:
        ctx.set_lidars(s["n_lidars"], ext)
    ctx.set_front_end(s["rings"], s["horizon"], s["roi"], 0.1, s["time_field"])
    n = len(frames)

    def step(k):
        f = frames[k % n]
        if variant == "chain":
            outs, ss, se, base = [], [], [], 0
            for part in f["parts"]:
                timed = fel.cal_timestamp(part, s["time_field"], 0.1)
                c, a, b = ctx.project_cloud(timed, s["rings"], s["horizon"], s["roi"])
                outs.append(c), ss.append(a + base), se.append(b + base)
                base += c.shape[0]
            return ctx.frame(np.concatenate(outs), np.concatenate(ss), np.concatenate(se), surf_map, corner_map, f["init"])
        if variant == "raw_ahead":
            g = frames[(k + 1) % n]
            ctx.frame_set_next_raw(g["raw"], g["counts"])
        return ctx.frame_raw(f["raw"], f["counts"], surf_map, corner_map, f["init"])

    for k in range(2 * n):  # warm-up: allocations, graph capture
        step(k)
    ctx.sync()
    l0 = ctx.launch_count()
    t0 = time.perf_counter()
    for k in range(steps):
        step(k)
    ctx.sync()
    dt = time.perf_counter() - t0
    launches = (ctx.launch_count() - l0) / steps
    if variant == "chain":  # each LiDAR's timed cloud up, its projection down, then the projected sweep + its ScanInfo up again
        h2d = float(np.mean([f["chain_h2d"] for f in frames]))
    else:
        h2d = float(np.mean([f["raw"].nbytes for f in frames]))
    ctx.close()
    return dict(fps=steps / dt, launches_per_frame=launches, h2d_bytes_per_frame=h2d)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--frames", type=int, default=4)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        sys.exit(1)
    m = load_mloam()
    scene = syn.make_scene()
    traj = syn.trajectory(args.frames)
    surf_map, corner_map = syn.make_submap(scene, 100000)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi.splitlines()[0] if smi else None, "steps": args.steps, "repeats": args.repeats,
           "frames": args.frames, "shapes": {}}
    for name, s in SHAPES.items():
        ext, frames = workload(s, args.frames, scene, traj)
        res = {v: [] for v in ("chain", "raw", "raw_ahead")}
        for _ in range(args.repeats):
            for v in res:
                res[v].append(run(m, s, ext, frames, surf_map, corner_map, v, args.steps))
        out["shapes"][name] = {v: {"fps": [round(r["fps"], 1) for r in rs], "launches_per_frame": rs[-1]["launches_per_frame"],
                                   "h2d_bytes_per_frame": int(rs[-1]["h2d_bytes_per_frame"])} for v, rs in res.items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

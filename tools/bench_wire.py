"""PointCloud2 messages into the frame path on one GPU: python tools/bench_wire.py [--steps 30] [--repeats 3].

bench.py's seeded sweeps of C2 (1 x 64 x 2048) and C4 on one GPU (4 x 64 x 2048), one message per LiDAR, packed (tests/wire_lib.py) into
three layouts: pcl::toROSMsg's PointXYZI (32 B), a Velodyne-style packed x y z intensity ring time (22 B, unaligned floats) and FLOAT64
big-endian (48 B).  Maps are built once; frames run with graphs on (max_inner 1, bench.py's GN iterations).  Arms, alternated `--repeats`
times in one process:
  host          unpackPointCloud2 (m-loam_b200/host/mloam_io.hpp) per LiDAR on the host, then mloam_frame_raw (16 B per point over PCIe)
  msg           mloam_frame_msg: the messages' bytes go up as they are (point_step B per point) and one launch unpacks the rig
each with and without the look-ahead (+_ahead: the next frame's sweep announced, unpacked on the host at announcement in the host arm).
Reported per configuration and layout: frames/s of each run, wall ms per frame, host unpack ms per frame, PCIe bytes per frame of the
sweep, launches per frame, and — from a separate profiled run of the msg arm — the unpack kernel's event time and its bytes (point_step
read + 16 written per point) over 3.35 TB/s.  Every run's poses are compared across the arms (bit for bit); a mismatch exits non-zero.
The card name and power limit are read in the same run.  Writes nothing into the tree."""
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

import bench  # noqa: E402
import synthetic as syn  # noqa: E402
import wire_lib as wl  # noqa: E402

LAYOUTS = ["xyzi32", "velodyne22", "f64be48"]
ARMS = ["host", "host_ahead", "msg", "msg_ahead"]
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def workload(cfg, n_frames):
    """bench.make_workload's submap, initial poses and extrinsics, and its sweeps per LiDAR (the same syn.make_sweep calls)."""
    w = bench.make_workload(syn, cfg, 1, 0, n_frames)
    scene = syn.make_scene()
    traj = syn.trajectory(n_frames + 2)
    frames = []
    for k in range(n_frames):
        parts = [syn.make_sweep(scene, traj[k + 1], cfg["rings"], cfg["horizon"], seed=100 + k, lidar_id=l, ext=w["ext_all"][l])[0]
                 for l in range(cfg["lidars"])]
        frames.append(dict(parts=parts, init=w["frames"][k]["init"]))
    return w, frames


def make_ctx(m, cfg, w, msgs):
    p = m.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.max_ring_points = cfg["lidars"] * cfg["rings"], cfg["gn_iters"], 1, cfg["horizon"]
    ctx = m.Context(0, p)
    if cfg["lidars"] > 1:
        ctx.set_lidars(cfg["lidars"], w["ext_all"])
    ctx.set_front_end(cfg["rings"], cfg["horizon"], 0.5, 0.1, False)
    ctx.set_front_end_layout([wl.layout(m, g, None) for g in msgs[0]])
    ctx.map_build(m.MAP_SURF, w["surf_map"])
    ctx.map_build(m.MAP_CORNER, w["corner_map"])
    return ctx


def run(m, cfg, w, frames, msgs, arm, steps):
    ctx = make_ctx(m, cfg, w, msgs)
    n = len(frames)
    args = [[wl.as_arg(g) for g in ms] for ms in msgs]
    unpacked, t_unpack = {}, [0.0]
    # the host arm's sweeps go into one buffer per frame slot, as a caller reuses its buffers: the same pointers come back every n frames
    slots = [np.empty((sum(g["width"] * g["height"] for g in ms), 4), np.float32) for ms in msgs]
    counts = [np.array([g["width"] * g["height"] for g in ms], np.int32) for ms in msgs]

    def host_sweep(k):  # the host arm's unpack, timed
        if k not in unpacked:
            t = time.perf_counter()
            np.concatenate([wl.unpack(g) for g in msgs[k % n]], out=slots[k % n])
            t_unpack[0] += time.perf_counter() - t
            unpacked[k] = (slots[k % n], counts[k % n])
            unpacked.pop(k - 2, None)
        return unpacked[k]

    def step(k):
        ahead = arm.endswith("_ahead")
        if arm.startswith("host"):
            raw, counts = host_sweep(k)
            if ahead:
                ctx.frame_set_next_raw(*host_sweep(k + 1))
            return ctx.frame_raw(raw, counts, None, None, frames[k % n]["init"], rebuild_maps=False)
        if ahead:
            ctx.frame_set_next_msg(args[(k + 1) % n])
        return ctx.frame_msg(args[k % n], None, None, frames[k % n]["init"], rebuild_maps=False)

    for k in range(2 * n):  # warm-up: allocations, graph capture
        step(k)
    ctx.sync()
    unpacked.clear()
    t_unpack[0] = 0.0
    l0 = ctx.launch_count()
    poses = []
    t0 = time.perf_counter()
    for k in range(2 * n, 2 * n + steps):
        poses.append(step(k)[0])
    ctx.sync()
    dt = time.perf_counter() - t0
    launches = (ctx.launch_count() - l0) / steps
    ctx.close()
    h2d = [sum(16 * g["width"] * g["height"] for g in ms) if arm.startswith("host") else sum(g["height"] * g["row_step"] for g in ms) for ms in msgs]
    return dict(fps=steps / dt, ms_per_frame=1e3 * dt / steps, host_unpack_ms=1e3 * t_unpack[0] / steps, launches=launches,
                h2d=float(np.mean(h2d)), poses=np.array(poses))


def profile_unpack(m, cfg, w, frames, msgs, steps):
    """The unpack kernel's event time per frame, from a run with stage profiling on (stream path)."""
    ctx = make_ctx(m, cfg, w, msgs)
    ctx.profile(True)
    args = [[wl.as_arg(g) for g in ms] for ms in msgs]
    for k in range(len(frames)):
        ctx.frame_msg(args[k], None, None, frames[k]["init"], rebuild_maps=False)
    ctx.profile_reset()
    for k in range(steps):
        ctx.frame_msg(args[k % len(frames)], None, None, frames[k % len(frames)]["init"], rebuild_maps=False)
    ms, launches = ctx.profile_get("wire_unpack")
    ctx.close()
    return ms / max(launches, 1), launches / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--frames", type=int, default=4)
    ap.add_argument("--configs", default="C2,C4")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        sys.exit(1)
    m = bench.load_mloam()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    out = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi.strip().splitlines()[0] if smi.strip() else None, "steps": args.steps,
           "repeats": args.repeats, "frames": args.frames, "results": {}}
    identical = True
    for name in args.configs.split(","):
        cfg = bench.CONFIGS[name]
        w, frames = workload(cfg, args.frames)
        n_pts = float(np.mean([sum(q.shape[0] for q in f["parts"]) for f in frames]))
        for lay in LAYOUTS:
            rng = np.random.default_rng(7)
            msgs = [[wl.pack(q, lay, rng=rng) for q in f["parts"]] for f in frames]
            res = {a: [] for a in ARMS}
            same = True
            for _ in range(args.repeats):
                for a in ARMS:
                    res[a].append(run(m, cfg, w, frames, msgs, a, args.steps))
                ref = res["host"][-1]["poses"]
                same &= all(np.array_equal(res[a][-1]["poses"], ref) for a in ARMS)
            identical &= same
            k_ms, k_launches = profile_unpack(m, cfg, w, frames, msgs, args.steps)
            step = wl.LAYOUTS[lay][0]
            k_bytes = n_pts * (step + 16)
            out["results"][f"{name}/{lay}"] = {
                "points_per_frame": int(n_pts), "point_step": step, "outputs_identical": bool(same),
                "unpack_kernel": {"ms": round(k_ms, 4), "launches_per_frame": k_launches, "bytes": int(k_bytes),
                                  "share_of_3.35TB/s": round(k_bytes / (k_ms * 1e-3) / HBM_BYTES_PER_S, 3)},
                **{a: {"fps": [round(r["fps"], 1) for r in rs], "ms_per_frame": [round(r["ms_per_frame"], 3) for r in rs],
                       "host_unpack_ms_per_frame": round(float(np.median([r["host_unpack_ms"] for r in rs])), 3),
                       "h2d_bytes_per_frame": int(rs[-1]["h2d"]), "launches_per_frame": rs[-1]["launches"]} for a, rs in res.items()}}
    out["outputs_identical"] = identical
    print(json.dumps(out))
    sys.exit(0 if identical else 1)


if __name__ == "__main__":
    main()

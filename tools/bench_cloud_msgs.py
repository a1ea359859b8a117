"""The registered clouds as PointCloud2 data on one GPU: python tools/bench_cloud_msgs.py [--steps 30] [--repeats 3].

bench.py's seeded sweeps of C2 (1 x 64 x 2048) and C4 on one GPU (4 x 64 x 2048), ring-ordered, through mloam_frame with graphs on
(max_inner 1, bench.py's GN iterations) and the registered clouds on (mloam_set_registered).  After every frame the mapper publishes
pubPointCloud's three clouds (full_res, surf_last, corner_last) as PointXYZI messages.  Arms, alternated `--repeats` times in one process:
  host       three mloam_frame_registered reads (16 B per point over PCIe) + packPointCloud2 (m-loam_b200/host/mloam_io.hpp) on the host
  pageable   mloam_cloud_msgs of the three clouds into pageable memory (32 B per point over PCIe, one launch)
  pinned     the same into pinned memory
Reported per configuration and arm: frames/s and ms per frame (frame call + messages), host ms per frame spent on the messages, PCIe bytes
per frame, launches per frame, and — from a separate profiled run — k_wire_pack's event time and its bytes (16 read + 32 written per
point) over 3.35 TB/s.  Every timed frame's messages are hashed and compared across the arms; a mismatch exits non-zero.  The card name
and power limit are read in the same run.  Writes nothing into the tree."""
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
import cloud_msgs_lib as cml  # noqa: E402
import synthetic as syn  # noqa: E402

ARMS = ["host", "pageable", "pinned"]
REG = [0, 1, 2]
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def make_ctx(m, cfg, w):
    p = m.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.max_ring_points = cfg["lidars"] * cfg["rings"], cfg["gn_iters"], 1, cfg["horizon"]
    ctx = m.Context(0, p)
    if cfg["lidars"] > 1:
        ctx.set_lidars(cfg["lidars"], w["ext_all"])
    ctx.set_registered(True)
    ctx.map_build(m.MAP_SURF, w["surf_map"])
    ctx.map_build(m.MAP_CORNER, w["corner_map"])
    return ctx


def frame(ctx, fr):
    g = fr["groups"][0]
    return ctx.frame(g["cloud"], g["ss"], g["se"], None, None, fr["init"], False)


def run(m, cfg, w, arm, steps, torch):
    ctx = make_ctx(m, cfg, w)
    frames = w["frames"]
    n = len(frames)
    cap = max(fr["groups"][0]["cloud"].shape[0] for fr in frames) + 16
    if arm == "pageable":
        bufs = [np.empty(32 * cap, np.uint8) for _ in REG]
    elif arm == "pinned":
        bufs = [torch.empty(32 * cap, dtype=torch.uint8).pin_memory().numpy() for _ in REG]

    def messages():
        if arm == "host":
            return [cml.pack(ctx.frame_registered(t)) for t in REG]
        return ctx.cloud_msgs(REG, out=bufs)

    for k in range(2 * n):  # warm-up: allocations, graph capture
        frame(ctx, frames[k % n])
        messages()
    ctx.sync()
    l0 = ctx.launch_count()
    t_frame = t_msg = 0.0
    digests, widths = [], []
    for k in range(steps):
        t0 = time.perf_counter()
        frame(ctx, frames[k % n])  # returns with the pose on the host: the frame's work is done
        t1 = time.perf_counter()
        msgs = messages()
        t2 = time.perf_counter()
        t_frame += t1 - t0
        t_msg += t2 - t1
        digests.append([hashlib.sha256(b).hexdigest() for b in msgs])
        widths.append([len(b) // 32 for b in msgs])
    launches = (ctx.launch_count() - l0) / steps
    ctx.close()
    pts = float(np.mean([sum(x) for x in widths]))
    return dict(fps=steps / (t_frame + t_msg), ms_per_frame=1e3 * (t_frame + t_msg) / steps, host_ms=1e3 * t_msg / steps, launches=launches,
                pcie=(16 if arm == "host" else 32) * pts, points=pts, digests=digests)


def profile_pack(m, cfg, w, steps):
    """k_wire_pack's event time per call, from a run with stage profiling on (stream path)."""
    ctx = make_ctx(m, cfg, w)
    ctx.profile(True)
    frames = w["frames"]
    for fr in frames:
        frame(ctx, fr)
        ctx.cloud_msgs(REG)
    ctx.profile_reset()
    for k in range(steps):
        frame(ctx, frames[k % len(frames)])
        ctx.cloud_msgs_device(REG)
    ms, launches = ctx.profile_get("wire_pack")
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
        w = bench.make_workload(syn, cfg, 1, 0, args.frames)
        res = {a: [] for a in ARMS}
        same = True
        for _ in range(args.repeats):
            for a in ARMS:
                res[a].append(run(m, cfg, w, a, args.steps, torch))
            same &= all(res[a][-1]["digests"] == res["host"][-1]["digests"] for a in ARMS)
        identical &= same
        k_ms, k_launches = profile_pack(m, cfg, w, args.steps)
        pts = res["host"][-1]["points"]
        k_bytes = pts * (16 + 32)
        out["results"][name] = {
            "points_per_frame": int(pts), "outputs_identical": bool(same),
            "pack_kernel": {"ms": round(k_ms, 4), "launches_per_call": k_launches, "bytes": int(k_bytes),
                            "share_of_3.35TB/s": round(k_bytes / (k_ms * 1e-3) / HBM_BYTES_PER_S, 3)},
            **{a: {"fps": [round(r["fps"], 1) for r in rs], "ms_per_frame": [round(r["ms_per_frame"], 3) for r in rs],
                   "host_ms_per_frame": round(float(np.median([r["host_ms"] for r in rs])), 3),
                   "pcie_bytes_per_frame": int(rs[-1]["pcie"]), "launches_per_frame": rs[-1]["launches"]} for a, rs in res.items()}}
    out["outputs_identical"] = identical
    print(json.dumps(out))
    sys.exit(0 if identical else 1)


if __name__ == "__main__":
    main()

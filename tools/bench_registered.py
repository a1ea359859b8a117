"""The registered clouds (mloam_set_registered, pubPointCloud) off against on, on one GPU: python tools/bench_registered.py [--steps 200] [--repeats 3].

bench.py's C2 (1 x 64 x 2048 sweep, keyframe-built 1M-point submap) and C4 (4 x 64 x 2048, all four LiDARs batched in one context, 5M-point
submap) frames from device memory, with the sweep look-ahead, CUDA graphs, the keyframe cadence and an L2 flush between timed steps, as
bench.py runs them.  The two arms alternate `--repeats` times in one process; every run first plays the schedule long enough that each frame
graph is captured and replayed before timing, and fails if a graph is captured in the timed window.  Per arm: frames/s and launches per frame;
the on arm's poses and statistics must equal the off arm's byte for byte.  A separate pass with stage profiling on gives k_registered's time
(CUDA events around the launch, stream path); the bytes it moves are computed from the clouds' counts (16 B read + 16 B written per point),
and the extraction-time copy of the sweep (16 B read + 16 B written per sweep point) is reported beside them.  The host read-back of each
cloud is timed with a host clock around the synchronous call.  Prints one JSON line; writes nothing into the tree.  Fails without a GPU."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
import synthetic as syn  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
N_FRAMES = 8
WARM = 3 * 4 * bench.KEYFRAME_EVERY  # three periods of the (sweep, rebuild) schedule: the frame after the first sighting of a
                                      # key may still differ in its look-ahead state, so every key is captured before timing


def make_ctx(m, torch, cfg, wl, reg):
    p = m.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = cfg["rings"] * cfg["lidars"], cfg["gn_iters"], 1, 0.0, cfg["horizon"]
    ctx = m.Context(0, p)
    my = [f["groups"][0] for f in wl["frames"]]
    if cfg["lidars"] > 1:
        ctx.set_lidars(cfg["lidars"], my[0]["ext"])
    ctx.set_registered(reg)
    dev = torch.device("cuda", 0)
    d_surf, d_corner = torch.from_numpy(wl["surf_map"]).to(dev), torch.from_numpy(wl["corner_map"]).to(dev)
    d = [dict(cloud=torch.from_numpy(g["cloud"]).to(dev), ss=torch.from_numpy(g["ss"]).to(dev), se=torch.from_numpy(g["se"]).to(dev)) for g in my]
    stream = torch.cuda.Stream(device=dev)
    ctx.set_stream(stream.cuda_stream)
    n_scans = p.n_scans

    def step(k):
        g, dk, dn = my[k % N_FRAMES], d[k % N_FRAMES], d[(k + 1) % N_FRAMES]
        ctx.frame_set_next_device(dn["cloud"].data_ptr(), my[(k + 1) % N_FRAMES]["cloud"].shape[0], dn["ss"].data_ptr(), dn["se"].data_ptr(), n_scans)
        return ctx.frame_device(dk["cloud"].data_ptr(), g["cloud"].shape[0], dk["ss"].data_ptr(), dk["se"].data_ptr(), n_scans, d_surf.data_ptr(),
                                wl["surf_map"].shape[0], d_corner.data_ptr(), wl["corner_map"].shape[0], wl["frames"][k % N_FRAMES]["init"],
                                k % bench.KEYFRAME_EVERY == 0)

    return ctx, stream, step, (d_surf, d_corner, d)


def measure(m, torch, cfg, wl, steps, reg):
    ctx, stream, step, keep = make_ctx(m, torch, cfg, wl, reg)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=torch.device("cuda", 0))
    with torch.cuda.stream(stream):
        for k in range(WARM):
            step(k)
    torch.cuda.synchronize()
    cap0 = ctx.profile_get("graph_captures")[1]
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    launches, results = [], []
    with torch.cuda.stream(stream):
        for k in range(steps):
            flush.fill_(k & 0xFF)
            l0 = ctx.launch_count()
            evs[k][0].record(stream)
            pose, st = step(WARM + k)
            evs[k][1].record(stream)
            launches.append(ctx.launch_count() - l0)
            scalars = tuple(sorted(dict(st).items()))  # before "H" and "eig" are materialised into the dict
            results.append((pose.tobytes(), scalars, st["H"].tobytes(), st["eig"].tobytes()))
    torch.cuda.synchronize()
    res = dict(frames_per_s=steps / (sum(a.elapsed_time(b) for a, b in evs) / 1e3), launches=sorted(set(launches)),
               captures_in_window=int(ctx.profile_get("graph_captures")[1] - cap0), results=results)
    if reg:  # the clouds of the last frame: sizes and the host read-back of each
        res["points"] = [int(ctx.frame_registered(w).shape[0]) for w in range(3)]
        rb = []
        for w in range(3):
            ts = []
            for _ in range(5):
                t0 = time.perf_counter()
                ctx.frame_registered(w)
                ts.append(time.perf_counter() - t0)
            rb.append(statistics.median(ts) * 1e3)
        res["readback_ms"] = rb
        ts = []
        for _ in range(5):
            t0 = time.perf_counter()
            ctx.frame_registered_device(m.REGISTERED_FULL_RES)
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        res["device_copy_ms_full_res"] = statistics.median(ts) * 1e3
    ctx.close()
    return res


def kernel_time(m, torch, cfg, wl):
    """k_registered between CUDA events with stage profiling on (stream path, the look-ahead off)."""
    ctx, stream, step, keep = make_ctx(m, torch, cfg, wl, True)
    with torch.cuda.stream(stream):
        for k in range(4):
            step(k)
        ctx.profile(True)
        ctx.profile_reset()
        for k in range(4, 24):
            step(k)
    ms, n = ctx.profile_get("registered")
    ctx.close()
    return ms / n, n


def run_config(m, torch, name, steps, repeats):
    cfg = dict(bench.CONFIGS[name])
    wl = bench.make_workload(syn, cfg, 1, 0, N_FRAMES)
    runs = {"off": [], "on": []}
    for _ in range(repeats):
        runs["off"].append(measure(m, torch, cfg, wl, steps, False))
        runs["on"].append(measure(m, torch, cfg, wl, steps, True))
    identical = all(a["results"] == b["results"] for a, b in zip(runs["off"], runs["on"]))
    k_ms, k_n = kernel_time(m, torch, cfg, wl)
    pts = runs["on"][-1]["points"]
    n_sweep = wl["frames"][0]["groups"][0]["cloud"].shape[0]
    kernel_bytes = 32 * sum(pts)
    copy_bytes = 32 * n_sweep
    fps_off = statistics.median(r["frames_per_s"] for r in runs["off"])
    fps_on = statistics.median(r["frames_per_s"] for r in runs["on"])
    return {"config": name, "workload": f"{cfg['lidars']} x {cfg['rings']} x {cfg['horizon']}, {cfg['map_points']} map points, look-ahead, graphs",
            "frames_per_s": {k: [round(r["frames_per_s"], 1) for r in v] for k, v in runs.items()},
            "median_frame_ms": {"off": round(1e3 / fps_off, 4), "on": round(1e3 / fps_on, 4)},
            "on_cost_share_of_frame": round(fps_off / fps_on - 1.0, 4),
            "launches_per_frame": {k: v[-1]["launches"] for k, v in runs.items()},
            "graph_captures_in_timed_window": {k: [r["captures_in_window"] for r in v] for k, v in runs.items()},
            "poses_and_stats_identical": identical,
            "points": dict(zip(("full_res", "surf_last", "corner_last"), pts)), "sweep_points": n_sweep,
            "k_registered_ms": round(k_ms, 5), "k_registered_launches_timed": k_n,
            "k_registered_bytes": kernel_bytes, "k_registered_bytes_per_s": round(kernel_bytes / (k_ms * 1e-3), 1),
            "k_registered_share_of_3_35_TBps": round(kernel_bytes / (k_ms * 1e-3) / HBM_BYTES_PER_S, 4),
            "extraction_copy_bytes": copy_bytes,
            "host_readback_ms": dict(zip(("full_res", "surf_last", "corner_last"), [round(x, 4) for x in runs["on"][-1]["readback_ms"]])),
            "device_copy_ms_full_res": round(runs["on"][-1]["device_copy_ms_full_res"], 4)}, identical and not any(
                r["captures_in_window"] for v in runs.values() for r in v)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--configs", default="C2,C4")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 2
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    m = bench.load_mloam()
    out, ok = [], True
    for name in args.configs.split(","):
        r, good = run_config(m, torch, name, args.steps, args.repeats)
        out.append(r)
        ok = ok and good
    print(json.dumps({"gpu_and_power_limit": card, "steps": args.steps, "repeats": args.repeats, "configs": out}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())

"""gd_float (mloam_set_gf_float) against gd_fix on one GPU: python tools/bench_gf_float.py [--steps 200] [--repeats 3].

bench.py's C2 frames (64 x 2048 sweep, keyframe-built 1M-point submap, keyframe cadence, sweep look-ahead, L2 flush between timed
steps) with the good-feature configuration the reference runs: gf_method 3, gf_ratio 0.4, and the reference's max_outer = 2 (not
bench.py's 10 iterations — the reference never selects features over ten).  Arm A leaves the mode off (gd_fix); arm B turns it on with a
MAP_DEG_THRE at the median of the factors a first pass records, so the ratio goes back and forth between 0.4 and 0.8 during the run.  The
arms alternate `--repeats` times in one process.  Every run first plays four periods of the timed schedule (40 frames: 8 sweeps, every
10th frame rebuilds the maps, every 10th evaluates), so that each frame graph is captured and replayed before timing, and fails if a
graph is captured in the timed window.  The kernel's own time comes from a separate pass with stage profiling on (CUDA events around
k_gf_full_hessian, stream path).  Prints one JSON line; writes nothing into the tree.  Fails without a GPU."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
import synthetic as syn  # noqa: E402

GF_RATIO, MAX_OUTER, PERIOD = 0.4, 2, 40


def make_ctx(m, torch, cfg, wl, n_frames):
    p = m.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = cfg["rings"], MAX_OUTER, 1, 0.0, cfg["horizon"]
    p.gf_method, p.gf_ratio, p.gf_seed = 3, GF_RATIO, 5
    ctx = m.Context(0, p)
    my = [f["groups"][0] for f in wl["frames"]]
    dev = torch.device("cuda", 0)
    d_surf, d_corner = torch.from_numpy(wl["surf_map"]).to(dev), torch.from_numpy(wl["corner_map"]).to(dev)
    d = [dict(cloud=torch.from_numpy(g["cloud"]).to(dev), ss=torch.from_numpy(g["ss"]).to(dev), se=torch.from_numpy(g["se"]).to(dev)) for g in my]
    stream = torch.cuda.Stream(device=dev)
    ctx.set_stream(stream.cuda_stream)
    n_scans = cfg["rings"]

    def step(k):
        g, dk, dn = my[k % n_frames], d[k % n_frames], d[(k + 1) % n_frames]
        ctx.frame_set_next_device(dn["cloud"].data_ptr(), my[(k + 1) % n_frames]["cloud"].shape[0], dn["ss"].data_ptr(), dn["se"].data_ptr(), n_scans)
        return ctx.frame_device(dk["cloud"].data_ptr(), g["cloud"].shape[0], dk["ss"].data_ptr(), dk["se"].data_ptr(), n_scans, d_surf.data_ptr(),
                                wl["surf_map"].shape[0], d_corner.data_ptr(), wl["corner_map"].shape[0], wl["frames"][k % n_frames]["init"],
                                k % bench.KEYFRAME_EVERY == 0)

    return ctx, stream, step, (d_surf, d_corner, d)


def factors(m, torch, cfg, wl, n_frames):
    """gf_deg_factor of the schedule's evaluation frames (threshold far below: the ratio stays gf_ratio), and the kernel's event time."""
    ctx, stream, step, keep = make_ctx(m, torch, cfg, wl, n_frames)
    ctx.set_gf_float(True, -1e30)
    ctx.profile(True)
    out = []
    for k in range(2 * PERIOD):
        step(k)
        r = ctx.gf_float_report()
        if r["evaluated"]:
            out.append(r["deg_factor"])
    ms, n = ctx.profile_get("gf_full_hessian")
    ctx.close()
    return out, (ms / n if n else None), n


def measure(m, torch, cfg, wl, n_frames, steps, thre):
    ctx, stream, step, keep = make_ctx(m, torch, cfg, wl, n_frames)
    if thre is not None:
        ctx.set_gf_float(True, thre)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=torch.device("cuda", 0))
    for k in range(4 * PERIOD):
        step(k)
    torch.cuda.synchronize()
    cap0 = ctx.profile_get("graph_captures")[1]
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    kinds, launches, ratios, from_graph = [], [], [], 0
    with torch.cuda.stream(stream):
        for k in range(steps):
            flush.fill_(k & 0xFF)
            l0 = ctx.launch_count()
            evs[k][0].record(stream)
            step(4 * PERIOD + k)
            evs[k][1].record(stream)
            launches.append(ctx.launch_count() - l0)
            r = ctx.gf_float_report() if thre is not None else {"evaluated": False, "ratio_cur": GF_RATIO}
            kinds.append(r["evaluated"]), ratios.append(r["ratio_cur"])
    torch.cuda.synchronize()
    captures = ctx.profile_get("graph_captures")[1] - cap0
    ms = [a.elapsed_time(b) for a, b in evs]
    ev = [t for t, e in zip(ms, kinds) if e]
    ot = [t for t, e in zip(ms, kinds) if not e]
    res = dict(frames_per_s=steps / (sum(ms) / 1e3), captures_in_window=int(captures), eval_frames=len(ev),
               median_ms_eval=statistics.median(ev) if ev else None, median_ms_other=statistics.median(ot),
               launches_eval=sorted({n for n, e in zip(launches, kinds) if e}), launches_other=sorted({n for n, e in zip(launches, kinds) if not e}),
               ratio_switches=sum(1 for a, b in zip(ratios, ratios[1:]) if a != b), ratios_seen=sorted(set(ratios)))
    ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 2
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    m = bench.load_mloam()
    cfg = bench.CONFIGS["C2"]
    n_frames = 8
    wl = bench.make_workload(syn, cfg, 1, 0, n_frames)
    fs, kernel_ms, kernel_n = factors(m, torch, cfg, wl, n_frames)
    thre = statistics.median(fs)
    runs = {"gd_fix": [], "gd_float": []}
    for _ in range(args.repeats):
        runs["gd_fix"].append(measure(m, torch, cfg, wl, n_frames, args.steps, None))
        runs["gd_float"].append(measure(m, torch, cfg, wl, n_frames, args.steps, thre))
    b = runs["gd_float"]
    line = {"workload": f"C2 frames, gf_method 3, gf_ratio {GF_RATIO}, max_outer {MAX_OUTER}", "gpu_and_power_limit": card, "steps": args.steps,
            "map_deg_thre": thre, "factors_seen": [round(f, 3) for f in sorted(set(fs))],
            "frames_per_s": {k: [round(r["frames_per_s"], 1) for r in v] for k, v in runs.items()},
            "gd_float_median_ms": {"evaluation_frames": [round(r["median_ms_eval"], 4) for r in b], "other_frames": [round(r["median_ms_other"], 4) for r in b]},
            "gd_fix_median_ms": [round(r["median_ms_other"], 4) for r in runs["gd_fix"]],
            "evaluation_frames_per_run": b[-1]["eval_frames"], "ratio_switches_per_run": b[-1]["ratio_switches"], "ratios_seen": b[-1]["ratios_seen"],
            "launches_per_frame": {"gd_fix": runs["gd_fix"][-1]["launches_other"], "gd_float_other": b[-1]["launches_other"],
                                   "gd_float_evaluation": b[-1]["launches_eval"]},
            "graph_captures_in_timed_window": {k: [r["captures_in_window"] for r in v] for k, v in runs.items()},
            "k_gf_full_hessian_ms": None if kernel_ms is None else round(kernel_ms, 5), "k_gf_full_hessian_launches_timed": kernel_n}
    print(json.dumps(line))
    if any(r["captures_in_window"] for v in runs.values() for r in v):
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())

#!/usr/bin/env python
"""Kernel timeline of graph-replayed C2 frames (64 x 2048 sweep, 1M-point keyframe submap, 10 GN iterations, inputs resident on
the device as in bench.py) with torch.profiler: device time per kernel and frame, and how much of each candidate evaluation
(k_eval_candidate) runs while the speculative matcher (k_match_knn) of the next GN iteration is running.
  python tools/trace_replay.py OUT_DIR [frames]      (writes OUT_DIR/replay.pt.trace.json)"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import synthetic as syn  # noqa: E402


def main():
    out = sys.argv[1]
    n_frames = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    import torch
    from torch.profiler import ProfilerActivity, profile

    m = bench.load_mloam()
    cfg = bench.CONFIGS["C2"]
    p = m.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = cfg["rings"], cfg["gn_iters"], 1, 0.0, cfg["horizon"]
    ctx = m.Context(0, p)
    wl = bench.make_workload(syn, cfg, 1, 0, 1, "keyframes")
    fr = wl["frames"][0]
    g = fr["groups"][0]
    dev = torch.device("cuda", 0)
    d = {k: torch.from_numpy(v).to(dev) for k, v in (("cloud", g["cloud"]), ("ss", g["ss"]), ("se", g["se"]),
                                                      ("surf", wl["surf_map"]), ("corner", wl["corner_map"]))}

    def step(rebuild):
        return ctx.frame_device(d["cloud"].data_ptr(), g["cloud"].shape[0], d["ss"].data_ptr(), d["se"].data_ptr(), cfg["rings"],
                                d["surf"].data_ptr(), wl["surf_map"].shape[0], d["corner"].data_ptr(), wl["corner_map"].shape[0],
                                fr["init"], rebuild)

    step(True)
    for _ in range(4):  # stream path, capture, replays
        step(False)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n_frames):
            step(False)
        torch.cuda.synchronize()
    os.makedirs(out, exist_ok=True)
    path = os.path.join(out, "replay.pt.trace.json")
    prof.export_chrome_trace(path)
    ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"]

    def short(name):
        return name.split("(")[0].replace("void ", "").replace("mloam::", "")

    per = {}
    for e in ev:
        s = per.setdefault(short(e["name"]), [0, 0.0])
        s[0] += 1
        s[1] += e["dur"]
    print(f"{len(ev)} kernels in {n_frames} replayed frames; device time per frame (us) and launches per frame:")
    for k, (cnt, dur) in sorted(per.items(), key=lambda kv: -kv[1][1]):
        print(f"  {dur / n_frames:9.1f}  {cnt / n_frames:5.1f}  {k}")
    knn = [(e["ts"], e["ts"] + e["dur"]) for e in ev if "k_match_knn" in e["name"]]
    cand = [(e["ts"], e["ts"] + e["dur"]) for e in ev if "k_eval_candidate" in e["name"]]
    lin = [(e["ts"], e["ts"] + e["dur"]) for e in ev if "k_linearize" in e["name"]]
    both = sum(max(0.0, min(b, d1) - max(a, c0)) for a, b in cand for c0, d1 in knn)
    tc = sum(b - a for a, b in cand)
    print(f"k_eval_candidate: {len(cand) / n_frames:.1f} per frame, {tc / max(1, len(cand)):.1f} us each, "
          f"{100.0 * both / tc if tc else 0.0:.1f} % of its time next to a running k_match_knn")
    print(f"k_match_knn: {sum(b - a for a, b in knn) / max(1, len(knn)):.1f} us each; "
          f"k_linearize: {sum(b - a for a, b in lin) / max(1, len(lin)):.1f} us each")
    starts = sorted(e["ts"] for e in ev)
    ends = sorted(e["ts"] + e["dur"] for e in ev)
    print(f"first kernel to last kernel: {(ends[-1] - starts[0]) / n_frames:.1f} us per frame")
    ctx.close()


if __name__ == "__main__":
    main()

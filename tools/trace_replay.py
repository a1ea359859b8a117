#!/usr/bin/env python
"""Kernel timeline of graph-replayed C2 frames (64 x 2048 sweep, 1M-point keyframe submap, 10 GN iterations, inputs resident on
the device as in bench.py) with torch.profiler: device time per kernel and frame, and how much of each candidate evaluation
(k_eval_candidate) runs while the speculative matcher (k_match_knn) of the next GN iteration is running.
  python tools/trace_replay.py OUT_DIR [frames] [--phases]      (writes OUT_DIR/replay.pt.trace.json)
--phases: afterwards, the same frames on a second context with MLOAM_LIN_TRACE=1 and MLOAM_KNN_TRACE=1 (no profiler): the phase
split of k_linearize's pass 0 per GN iteration from %globaltimer / clock64 stamps inside the kernel (feature loop = fit + evaluation,
block reduction, ticket, LM tail), and the GN chain's kernel boundaries from those stamps and k_match_knn's per-warp timelines.
MLOAM_PDL is passed through (read at context creation)."""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import synthetic as syn  # noqa: E402


LIN_TRACE_BLOCK, LIN_TRACE_SLOT = 64, 64 * 64  # solve_kernels.cu


def phases(tr):
    """One traced k_linearize pass 0 (LIN_TRACE_SLOT words) -> phase boundaries [us] from the first warp's entry."""
    blk = tr.reshape(64, LIN_TRACE_BLOCK)
    blk = blk[blk[:, 0] != 0]
    warps = blk[:, :32].reshape(-1, 4).astype(np.int64)  # [entry, loop ns, fit cycles, loop cycles] per warp
    t0 = int(warps[:, 0].min())
    loop_end = int((warps[:, 0] + warps[:, 1]).max())
    fit_share = float(np.mean(warps[:, 2] / np.maximum(warps[:, 3], 1)))  # of a warp's feature-loop cycles
    last = blk[blk[:, 34] != 0]
    us = lambda t: (int(t) - t0) / 1000.0  # noqa: E731
    return {"blocks": len(blk), "loop_end": us(loop_end), "fit_share": fit_share, "reduced": us(blk[:, 32].max()),
            "ticket": us(last[0, 33]) if len(last) else float("nan"), "tail_start": us(last[0, 34]) if len(last) else float("nan"),
            "tail_end": us(last[0, 35]) if len(last) else float("nan"), "t_entry": t0, "t_tail_end": int(last[0, 35]) if len(last) else 0}


def chain_gaps(lin, knn):
    """The GN chain's kernel boundaries of one frame [us], from the k_linearize slots (phases()) and the k_match_knn timelines
    ([enter, exit] per warp, enter taken after the grid-dependency wait): per GN iteration i, (a) the tail end of k_linearize i ->
    the first warp of matcher i + 1, (b) the last warp of matcher i -> the first block of k_linearize i."""
    spans = []
    for tl in knn:
        tl = tl[tl[:, 0] != 0].astype(np.int64)
        spans.append((int(tl[:, 0].min()), int(tl[:, 1].max())))
    n = min(len(lin), len(spans))
    b = [(lin[i]["t_entry"] - spans[i][1]) / 1000.0 for i in range(n)]
    a = [(spans[i + 1][0] - lin[i]["t_tail_end"]) / 1000.0 for i in range(n - 1)]
    return a, b


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    out = args[0]
    n_frames = int(args[1]) if len(args) > 1 else 5
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
    knn_pf = len(knn) // n_frames  # a frame's first matcher launch searches blind, the later ones are seeded
    if knn_pf > 1:
        knn.sort()
        first = [b - a for k, (a, b) in enumerate(knn) if k % knn_pf == 0]
        seeded = [b - a for k, (a, b) in enumerate(knn) if k % knn_pf != 0]
        print(f"k_match_knn per frame: {knn_pf} launches; first (blind) {np.mean(first):.1f} us, seeded {np.mean(seeded):.1f} us "
              f"(min {np.min(seeded):.1f}, max {np.max(seeded):.1f})")
    per_frame = len(lin) // n_frames  # the last k_linearize of a frame runs both passes, the others pass 0 only
    if per_frame > 1:
        lin.sort()
        two = [lin[f * per_frame + per_frame - 1] for f in range(n_frames)]
        one = [x for k, x in enumerate(lin) if k % per_frame != per_frame - 1]
        print(f"k_linearize pass 0 only: {sum(b - a for a, b in one) / len(one):.1f} us each; "
              f"two-pass (last GN iteration): {sum(b - a for a, b in two) / len(two):.1f} us each")
    starts = sorted(e["ts"] for e in ev)
    ends = sorted(e["ts"] + e["dur"] for e in ev)
    print(f"first kernel to last kernel: {(ends[-1] - starts[0]) / n_frames:.1f} us per frame")
    ctx.close()
    if "--phases" not in sys.argv:
        return
    os.environ["MLOAM_LIN_TRACE"] = "1"  # read at context creation
    os.environ["MLOAM_KNN_TRACE"] = "1"
    ctx = m.Context(0, p)
    step(True)
    for _ in range(4):
        step(False)
    rows, gaps = [], []
    buf = np.zeros(16 * LIN_TRACE_SLOT, dtype=np.uint64)
    n_pairs = 8 * 4 * torch.cuda.get_device_properties(0).multi_processor_count  # k_match_knn: MWARPS x up to 4 CTAs per SM
    tl = np.zeros((n_pairs, 2), dtype=np.uint64)
    for _ in range(n_frames):
        step(False)
        n_slots = C.c_int(0)
        rc = m.lib().mloam_debug_lin_trace(ctx._h, buf.ctypes.data_as(C.c_void_p), buf.size, C.byref(n_slots))
        assert rc == 0, rc
        rows.append([phases(buf[s * LIN_TRACE_SLOT:(s + 1) * LIN_TRACE_SLOT]) for s in range(n_slots.value)])
        knn, s, n_knn = [], 0, C.c_int(1)
        while s < n_knn.value:
            rc = m.lib().mloam_debug_knn_timeline(ctx._h, s, tl.ctypes.data_as(C.c_void_p), n_pairs, C.byref(n_knn))
            assert rc == 0, rc
            knn.append(tl.copy())
            s += 1
        gaps.append(chain_gaps(rows[-1], knn))
    ctx.close()
    keys = ["loop_end", "reduced", "ticket", "tail_start", "tail_end"]
    print(f"k_linearize pass 0 phase boundaries, us from the first warp's entry, mean of {n_frames} replayed frames "
          f"({rows[0][0]['blocks']} blocks); fit = share of the feature loop's cycles spent in fit_one")
    print(f"  {'GN it':>5s} " + " ".join(f"{k:>10s}" for k in keys) + f" {'fit share':>10s}")
    for s in range(len(rows[0])):
        mean = {k: float(np.mean([r[s][k] for r in rows])) for k in keys + ["fit_share"]}
        print(f"  {s:5d} " + " ".join(f"{mean[k]:10.2f}" for k in keys) + f" {mean['fit_share']:10.2f}")
    spec = [r[s] for r in rows for s in range(len(r) - 1)]
    if spec:
        mean = {k: float(np.mean([x[k] for x in spec])) for k in keys + ["fit_share"]}
        print("  speculative iterations (all but the last): " + ", ".join(f"{k} {mean[k]:.2f}" for k in keys) +
              f", fit share {mean['fit_share']:.2f}")
    ga = np.array([g[0] for g in gaps])
    gb = np.array([g[1] for g in gaps])
    print(f"GN chain boundaries, us, mean of {n_frames} replayed frames: (a) k_linearize tail end -> first k_match_knn warp of the "
          f"next iteration, (b) last k_match_knn warp -> first k_linearize block (negative: the next kernel was already running)")
    print(f"  {'GN it':>5s} {'(a)':>8s} {'(b)':>8s}")
    for i in range(gb.shape[1]):
        a_i = f"{ga[:, i].mean():8.2f}" if i < ga.shape[1] else f"{'':8s}"
        print(f"  {i:5d} {a_i} {gb[:, i].mean():8.2f}")
    per = ga.sum(axis=1) + gb.sum(axis=1)
    print(f"  per frame: sum (a) {ga.sum(axis=1).mean():.1f}, sum (b) {gb.sum(axis=1).mean():.1f}, total {per.mean():.1f} "
          f"(min {per.min():.1f}, max {per.max():.1f})")
    # queries and SM cycles per search path from stage profiling (stream path, instrumented matcher), per frame
    os.environ["MLOAM_KNN_TRACE"] = "0"
    ctx = m.Context(0, p)
    step(True)
    ctx.profile(True)
    ctx.profile_reset()
    for _ in range(n_frames):
        step(False)
    torch.cuda.synchronize()
    print(f"k_match_knn per search path, stage profiling, per frame (mean of {n_frames}): queries, mean SM cycles per query")
    for path in ("keep_matched", "keep_rejected", "ball", "blind"):
        q = ctx.profile_get(f"knn_{path}")[1] / n_frames
        cyc = ctx.profile_get(f"knn_cycles_{path}")[1] / n_frames
        print(f"  {path:>13s} {q:9.1f} {cyc / max(q, 1e-9):9.0f}")
    print(f"  slowest query {ctx.profile_get('knn_max_query_cycles')[1]:.0f} cycles; "
          f"{ctx.profile_get('knn_queries_over_32k_cycles')[1] / n_frames:.1f} queries over 32k cycles per frame")
    ctx.close()


if __name__ == "__main__":
    main()

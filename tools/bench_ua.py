"""The uncertainty-aware mapper (with_ua) against the plain frame on one GPU: python tools/bench_ua.py [--config C2] [--steps 50].

The workload of bench.py (same sweeps, submap, keyframe cadence, sweep look-ahead, L2 flush between timed steps).  with_ua runs
with seeded extrinsic covariances (tests/uncertainty_lib.py ext_covariances, scale 1.6) and a TRACE_THRESHOLD_MAPPING at the 80th
percentile of the first frame's point traces, so that the gate drops part of the scan.  The two variants alternate `--repeats` times
in one process; the line reports frames/s of each run, launches and features per step, and the last with_ua frame's pose and pose
covariance against the oracle (orc_ua_frame_multi).  Writes nothing into the tree."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
import oracle_lib as orc  # noqa: E402
import synthetic as syn  # noqa: E402
import uncertainty_lib as ua  # noqa: E402

COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])


def ua_setup(wl):
    g, fr = wl["frames"][0]["groups"][0], wl["frames"][0]
    ext_cov = ua.ext_covariances(g["ext"].shape[0], seed=5, scale=1.6)
    _, _, _, sc = ua.frame_multi_ua(g["cloud"], g["ss"], g["se"], g["ext"].shape[0], g["ext"], ext_cov, COV_MEAS, 1e30, wl["surf_map"][:10],
                                    wl["corner_map"][:10], fr["init"])  # a 10-point map: only the uncertainty, no solve
    c6 = np.concatenate([sc["surf_cov6"], sc["corner_cov6"]]).astype(np.float64)
    tr = np.sort(c6[:, 0] + c6[:, 3] + c6[:, 5])
    k = int(0.8 * tr.shape[0])
    return ext_cov, float(0.5 * (tr[k - 1] + tr[k]))


def measure(m, torch, cfg, wl, n_frames, steps, ext_cov, thr, with_ua):
    L = cfg["lidars"]
    p = m.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = cfg["rings"], cfg["gn_iters"], 1, 0.0, cfg["horizon"]
    ctx = m.Context(0, p)
    my = [f["groups"][0] for f in wl["frames"]]
    if L > 1:
        ctx.set_lidars(L, my[0]["ext"])
    if with_ua:
        ctx.set_uncertainty(True, ext_cov, COV_MEAS, thr)
    n_scans = cfg["rings"] * L
    dev = torch.device("cuda", 0)
    d_surf, d_corner = torch.from_numpy(wl["surf_map"]).to(dev), torch.from_numpy(wl["corner_map"]).to(dev)
    d = [dict(cloud=torch.from_numpy(g["cloud"]).to(dev), ss=torch.from_numpy(g["ss"]).to(dev), se=torch.from_numpy(g["se"]).to(dev)) for g in my]
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    stream = torch.cuda.Stream(device=dev)
    ctx.set_stream(stream.cuda_stream)

    def step(k, rebuild):
        g, dk, dn = my[k % n_frames], d[k % n_frames], d[(k + 1) % n_frames]
        ctx.frame_set_next_device(dn["cloud"].data_ptr(), my[(k + 1) % n_frames]["cloud"].shape[0], dn["ss"].data_ptr(), dn["se"].data_ptr(), n_scans)
        return ctx.frame_device(dk["cloud"].data_ptr(), g["cloud"].shape[0], dk["ss"].data_ptr(), dk["se"].data_ptr(), n_scans, d_surf.data_ptr(),
                                wl["surf_map"].shape[0], d_corner.data_ptr(), wl["corner_map"].shape[0], wl["frames"][k % n_frames]["init"], rebuild)

    for rb in (True, False):  # as bench.py: every (frame, rebuild) combination allocates, captures, then replays before timing
        for _ in range(4):
            for k in range(n_frames):
                step(k, rb)
    for k in range(n_frames):
        step(k, k == n_frames - 1)
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    l0, feats, last = ctx.launch_count(), 0, None
    with torch.cuda.stream(stream):
        for k in range(steps):
            flush.fill_(k & 0xFF)
            evs[k][0].record(stream)
            last = step(k, k % bench.KEYFRAME_EVERY == 0)
            evs[k][1].record(stream)
            feats += last[1]["n_surf_in"] + last[1]["n_corner_in"]
    torch.cuda.synchronize()
    ms = [a.elapsed_time(b) for a, b in evs]
    res = dict(value=L * steps / (sum(ms) / 1e3), ms_per_step=sum(ms) / steps, launches_per_step=(ctx.launch_count() - l0) / steps,
               features_per_step=feats / steps, last_pose=last[0], last_stats=last[1], last_cov=ctx.pose_covariance(), k_last=(steps - 1) % n_frames)
    ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2", choices=["C2", "C4"])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 2
    m = bench.load_mloam()
    cfg = bench.CONFIGS[args.config]
    n_frames = 8 if cfg["lidars"] == 1 else 4
    wl = bench.make_workload(syn, cfg, 1, 0, n_frames)
    ext_cov, thr = ua_setup(wl)
    runs = {"plain": [], "with_ua": []}
    last = None
    for _ in range(args.repeats):
        for name in ("plain", "with_ua"):
            r = measure(m, torch, cfg, wl, n_frames, args.steps, ext_cov, thr, name == "with_ua")
            runs[name].append(r)
            if name == "with_ua":
                last = r
    fr = wl["frames"][last["k_last"]]
    g = fr["groups"][0]
    o = bench.oracle_opts(orc, cfg)
    rpose, rst, rcov, _ = ua.frame_multi_ua(g["cloud"], g["ss"], g["se"], g["ext"].shape[0], g["ext"], ext_cov, COV_MEAS, thr, wl["surf_map"],
                                            wl["corner_map"], fr["init"], o)
    dt, dr = syn.pose_err(last["last_pose"], rpose)
    line = {"config": args.config, "gpu": torch.cuda.get_device_name(0), "steps": args.steps, "trace_threshold": thr,
            "frames_per_s": {k: [round(r["value"], 1) for r in v] for k, v in runs.items()},
            "ms_per_step": {k: [round(r["ms_per_step"], 4) for r in v] for k, v in runs.items()},
            "launches_per_step": {k: v[-1]["launches_per_step"] for k, v in runs.items()},
            "features_per_step": {k: v[-1]["features_per_step"] for k, v in runs.items()},
            "with_ua_vs_oracle": {"pose_m": dt, "pose_rad": dr, "features_in_gpu": [last["last_stats"]["n_surf_in"], last["last_stats"]["n_corner_in"]],
                                  "features_in_oracle": [rst["n_surf_in"], rst["n_corner_in"]],
                                  "pose_cov_rel_err": float(np.linalg.norm(last["last_cov"] - rcov) / np.linalg.norm(rcov))}}
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    sys.exit(main())

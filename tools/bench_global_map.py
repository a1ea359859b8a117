"""The global map of the device keyframe store (mloam_global_map) against the oracle's CPU restatement of pubGlobalMap / saveGlobalMap:
python tools/bench_global_map.py [--keyframes 200 1000 2000] [--repeats 5] [--oracle-max 1000].

For each store size N: N keyframes 2.5 m apart on a 40-wide grid, each holding the with_ua-gated, down-sampled scans of one of 8 synthetic
32 x 1800 sweeps (what mloam_frame leaves for mloam_keyframe_save), with a small random pose covariance.  Both modes run with the reference's
parameters: SURROUND (pubGlobalMap) with GLOBALMAP_KF_RADIUS 1000 m around the last keyframe, kf_leaf 10 m, leaf MAP_SURF_RES 0.4 m; SAVE
(saveGlobalMap) over every keyframe with leaf 0.8 m.  Device: one warm-up call, then the median of `--repeats` mloam_global_map calls timed
on the host around the call (it ends in a stream synchronise, because the map sizes come back to the host; reading the maps back is not
timed), and the call's launch count.  Oracle: the
same store in the oracle's single-threaded restatement, one timed call per mode for N <= --oracle-max (not measured above it), and whether
the device result is bit-identical to it.  Prints one JSON line with the card's name and power limit, read in the same run.  Writes
nothing into the tree."""
import argparse
import ctypes as C
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
import global_map_lib as gl  # noqa: E402
import mapper_lib as ml  # noqa: E402
import synthetic as syn  # noqa: E402
import uncertainty_lib as ua  # noqa: E402

COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])
TRACE = 0.3  # TRACE_THRESHOLD_MAPPING of the store


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True, timeout=30)
        name, power = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})", "unknown"


def build(m, n_kf, sweeps, ext, ext_cov):
    """The device store and the oracle store of n_kf keyframes."""
    p = m.default_params()
    p.n_scans, p.max_ring_points = 32, 2048
    cx = m.Context(0, p)
    cx.set_lidars(1, ext)
    cx.set_uncertainty(True, ext_cov, COV_MEAS, 1e3)
    cx.keyframes_init(2.0, 10.0, 50.0, 1.0, TRACE)
    om = ml.Mapper(2.0, 10.0, 50.0, 1.0, TRACE)
    om.set_lidars(ext, ext_cov, COV_MEAS, True)
    rng = np.random.default_rng(1)
    scans = {}
    pose = None
    for k in range(n_kf):
        s = k % len(sweeps)
        cloud, ss, se, _, _ = sweeps[s]
        cx.frame(cloud, ss, se, None, None, sweeps[s][4], False)
        if s not in scans:
            sp, _, cp, _ = cx.frame_scan()
            scans[s] = (sp, cp)
        pose = syn.pose7([2.5 * (k % 40), 2.5 * (k // 40), 0.0], syn.quat_from_rpy(0.0, 0.0, 0.01 * k))
        cov = np.diag(rng.uniform(1e-6, 1e-5, 6))
        assert cx.keyframe_save(pose, cov)
        om.save(pose, cov, *scans[s])
    return cx, om, pose


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keyframes", type=int, nargs="+", default=[200, 1000, 2000])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--oracle-max", type=int, default=1000)
    args = ap.parse_args()
    m = bench.load_mloam()
    name, power = gpu_info()
    scene = syn.make_scene()
    traj = syn.trajectory(8)
    sweeps = [syn.make_multi_sweep(scene, traj[k], 1, 32, 1800, seed=300 + k) + (traj[k],) for k in range(8)]
    ext = sweeps[0][3]
    ext_cov = ua.ext_covariances(1, seed=5)
    rows = []
    for n_kf in args.keyframes:
        cx, om, last = build(m, n_kf, sweeps, ext, ext_cov)
        try:
            stored = sum(sum(x.shape[0] for x in (cx.keyframe_scan(i)[2], cx.keyframe_scan(i)[4])) for i in range(min(n_kf, 8)))
            stored_pts = int(round(stored / min(n_kf, 8) * n_kf))
            for mode, mode_name, leaf in ((m.GLOBAL_MAP_SURROUND, "surround", 0.4), (m.GLOBAL_MAP_SAVE, "save", 0.8)):
                g = cx.global_map(mode, None, 1000.0, 10.0, leaf)
                ts = []
                for _ in range(args.repeats):
                    l0 = cx.launch_count()
                    t0 = time.perf_counter()
                    rc = m.lib().mloam_global_map(cx._h, mode, None, C.c_double(1000.0), C.c_double(10.0), C.c_float(leaf), None, None, None)
                    ts.append(time.perf_counter() - t0)
                    launches = cx.launch_count() - l0
                    assert rc == 0, rc
                row = dict(keyframes=n_kf, mode=mode_name, stored_points=stored_pts, chosen=len(cx.global_map_chosen()),
                           map_points=[int(x.shape[0]) for x in g[::2]], gpu_ms_median=round(1e3 * float(np.median(ts)), 3),
                           gpu_ms_min=round(1e3 * min(ts), 3), launches=launches, oracle_ms=None, bit_identical=None)
                if n_kf <= args.oracle_max:
                    t0 = time.perf_counter()
                    o_ch, o = gl.global_map(om, mode, last, 1000.0, 10.0, leaf)
                    row["oracle_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
                    row["bit_identical"] = bool(o_ch == cx.global_map_chosen() and all(np.array_equal(a, b) for a, b in zip(g, o)))
                rows.append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
        finally:
            cx.close()
            om.close()
    print(json.dumps(dict(bench="global_map", gpu=name, power_limit=power, repeats=args.repeats, rows=rows)))


if __name__ == "__main__":
    main()

"""The mapper's saved maps and a caller's sweep as ASCII PCD files (mloam_cloud_pcd*, mloam_pcd_encode) against the caller path of today:
python tools/bench_pcd_write.py [--keyframes 200 1000 2000] [--repeats 5].

Stores: N keyframes 2.5 m apart on a 40-wide grid, each holding the with_ua-gated scans of one of 8 synthetic 32 x 1800 sweeps (as
tools/bench_global_map.py builds them), and the SAVE global map (saveGlobalMap: every keyframe, kf_leaf 10 m, leaf 0.8 m).  The three
files of saveGlobalMap (pose_keyframes_3d, maps 0 and 1) are written by
  (a) the caller path: mloam_global_map_read of both maps, the keyframe positions from mloam_keyframe_scan, cov_trace summed on the host,
      and host/mloam_io.hpp writePCDASCII (PCL's writer restated with iostreams);
  (b) mloam_cloud_pcd into pinned memory;
  (c) mloam_cloud_pcd_device.
The sweep: test_parse_bag's savePCDFileASCII of a 4 x 64 x 2048 rig, four pcl::PointXYZ files, by
  (d) mloam_pcd_encode, against writePCDASCII on the host.
Each arm: one warm-up, then the median of --repeats host-clock timings (every call ends in a stream synchronise), output MB/s and the
launch count; whether every arm's bytes are identical.  Prints one JSON line with the card's name and power limit, read in the same run.
Writes nothing into the tree."""
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
import pcd_write_lib as pw  # noqa: E402
import synthetic as syn  # noqa: E402
import uncertainty_lib as ua  # noqa: E402

COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])
TRACE = 0.3  # TRACE_THRESHOLD_MAPPING of the store


def gpu_info():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True, timeout=30)
    name, power = [s.strip() for s in out.strip().splitlines()[0].split(",")]
    return name, power


def build(m, n_kf, sweeps, ext, ext_cov):
    p = m.default_params()
    p.n_scans, p.max_ring_points = 32, 2048
    cx = m.Context(0, p)
    cx.set_lidars(1, ext)
    cx.set_uncertainty(True, ext_cov, COV_MEAS, 1e3)
    cx.keyframes_init(2.0, 10.0, 50.0, 1.0, TRACE)
    rng = np.random.default_rng(1)
    for k in range(n_kf):
        s = k % len(sweeps)
        cloud, ss, se, _, pose_s = sweeps[s]
        cx.frame(cloud, ss, se, None, None, pose_s, False)
        pose = syn.pose7([2.5 * (k % 40), 2.5 * (k // 40), 0.0], syn.quat_from_rpy(0.0, 0.0, 0.01 * k))
        assert cx.keyframe_save(pose, np.diag(rng.uniform(1e-6, 1e-5, 6)))
    return cx


def timed(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return out, float(np.median(ts))


def caller_path(m, cx):
    """The three files as a caller writes them today."""
    lib = m.lib()
    files = []
    n_kf = cx.keyframe_query()[0]
    kf = np.zeros((n_kf, 4), np.float32)
    pose, ns, nc = np.zeros(7), C.c_int(0), C.c_int(0)
    for i in range(n_kf):
        lib.mloam_keyframe_scan(cx._h, i, pose.ctypes.data_as(C.c_void_p), None, None, None, 0, C.byref(ns), None, None, 0, C.byref(nc))
        kf[i, :3], kf[i, 3] = pose[:3].astype(np.float32), i
    files.append(pw.write_ascii(pw.XYZI, kf))
    for which in (0, 1):
        n = C.c_int(0)
        lib.mloam_global_map_read(cx._h, which, None, None, 0, C.byref(n))
        pts, cov6 = np.zeros((max(n.value, 1), 4), np.float32), np.zeros((max(n.value, 1), 6), np.float32)
        assert lib.mloam_global_map_read(cx._h, which, pts.ctypes.data_as(C.c_void_p), cov6.ctypes.data_as(C.c_void_p), pts.shape[0],
                                         C.byref(n)) == 0
        pts, cov6 = pts[:n.value], cov6[:n.value]
        trace = ((cov6[:, 0] + cov6[:, 3]) + cov6[:, 5]).astype(np.float32)
        files.append(pw.write_ascii(pw.XYZI_COV, pts, cov6, trace))
    return files


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--keyframes", type=int, nargs="+", default=[200, 1000, 2000])
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    m = bench.load_mloam()
    name, power = gpu_info()
    lib = m.lib()
    scene = syn.make_scene()
    traj = syn.trajectory(8)
    sweeps = [syn.make_multi_sweep(scene, traj[k], 1, 32, 1800, seed=300 + k) + (traj[k],) for k in range(8)]
    ext = sweeps[0][3]
    ext_cov = ua.ext_covariances(1, seed=5)
    src = [m.PCD_KEYFRAMES, m.MSG_GLOBAL_MAP0, m.MSG_GLOBAL_MAP1]
    rows = []

    def arm(cx, fn, out_bytes):
        l0 = cx.launch_count()
        fn()
        launches = cx.launch_count() - l0
        res, sec = timed(fn, args.repeats)
        return res, dict(ms=round(1e3 * sec, 3), mb_per_s=round(out_bytes / sec / 1e6, 1), launches=launches)

    for n_kf in args.keyframes:
        cx = build(m, n_kf, sweeps, ext, ext_cov)
        try:
            cx.global_map(m.GLOBAL_MAP_SAVE, None, 1000.0, 10.0, 0.8)
            ref = caller_path(m, cx)
            total = sum(len(f) for f in ref)
            pinned = [torch.zeros(len(f) + 64, dtype=torch.uint8).pin_memory().numpy() for f in ref]
            a_files, a = arm(cx, lambda: caller_path(m, cx), total)
            b_files, b = arm(cx, lambda: cx.cloud_pcd(src, out=pinned), total)
            srcs, ptrs, nb = (C.c_int * 3)(*src), (C.c_void_p * 3)(), (C.c_size_t * 3)()
            _, c = arm(cx, lambda: lib.mloam_cloud_pcd_device(cx._h, 3, srcs, ptrs, nb), total)
            c_files = [t.cpu().numpy().tobytes() for t in cx.cloud_pcd_device(src)]
            row = dict(keyframes=n_kf, map_points=[f.count(b"\n") - 11 for f in ref[1:]], file_mb=round(total / 1e6, 2),
                       caller=a, cloud_pcd_pinned=b, cloud_pcd_device=c, identical=bool(a_files == ref and b_files == ref and c_files == ref))
        finally:
            cx.close()
        rows.append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)

    # the sweep: four PointXYZ files of 64 x 2048 points
    ext4 = syn.rig_extrinsics(4)
    cloud = syn.make_multi_sweep(scene, traj[1], 4, 64, 2048, seed=77, ext=ext4)[0]
    parts = np.array_split(cloud[: 4 * 64 * 2048], 4)
    clouds = [(m.PCD_XYZ, np.ascontiguousarray(p)) for p in parts]
    cx = m.Context(0)
    try:
        host_files, host_s = timed(lambda: [pw.write_ascii(pw.XYZ, p) for _, p in clouds], args.repeats)
        total = sum(len(f) for f in host_files)
        pinned = [torch.zeros(len(f) + 64, dtype=torch.uint8).pin_memory().numpy() for f in host_files]
        d_files, d = arm(cx, lambda: cx.pcd_encode(clouds, out=pinned), total)
        sweep = dict(points=int(sum(p.shape[0] for p in parts)), file_mb=round(total / 1e6, 2),
                     host_writer=dict(ms=round(1e3 * host_s, 3), mb_per_s=round(total / host_s / 1e6, 1)), pcd_encode=d,
                     identical=bool(d_files == host_files))
    finally:
        cx.close()
    print(json.dumps(sweep), file=sys.stderr, flush=True)
    print(json.dumps(dict(bench="pcd_write", gpu=name, power_limit=power, repeats=args.repeats, save_global_map=rows, sweep=sweep)))


if __name__ == "__main__":
    main()

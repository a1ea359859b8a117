"""The closed mapper loop on one GPU with the keyframes kept on the device, against the host path it replaces:
python tools/bench_mapper.py [--frames 60] [--repeats 2].

Both paths run process() (lidar_mapper_keyframe.cpp:1062-1101) over the same C2-sized sweeps (one 64 x 2048 LiDAR through the rig
merge, 0.1 m and 0.11 deg per frame, odometry drifting 2 mm / 0.02 deg per frame) with the keyframe parameters of config_handheld:
DISTANCE_KEYFRAMES 1 m, ORIENTATION_KEYFRAMES 1 deg, SURROUNDING_KF_RADIUS 50 m, MAP_SUR_KF_RES 1.0 m.
  device: mloam_keyframe_submap -> mloam_frame(rebuild_maps = 0) -> mloam_keyframe_save; no keyframe point crosses PCIe.
  host:   the loop a caller wrote before: saveKeyframe's test, the radius search and the surrounding-set bookkeeping in numpy, every
          keyframe's scans copied device -> host (mloam_frame_scan), the keyframe-position filter (mloam_voxel_downsample),
          mloam_compound_pose_cov per (keyframe, LiDAR) and mloam_submap_assemble (host -> device) of every chosen keyframe per map.
Plain (with_ua = 0) and with_ua; the two paths alternate `--repeats` times in one process.  Reported per path: ms per keyframe step
(a step that saved or rebuilt) and per regular step, the frame call's share of each, frames whose graph capture failed, frames/s, PCIe bytes per keyframe step computed from the sizes, the largest pose
difference between the paths, and the card name and power limit read in the same run.  Writes nothing into the tree."""
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
import mapper_lib as ml  # noqa: E402
import synthetic as syn  # noqa: E402
import uncertainty_lib as ua  # noqa: E402

COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])
KF = dict(dist=1.0, orient=1.0, radius=50.0, res=1.0)


def trajectory(n_frames, seed=syn.SEED):
    """syn.trajectory's drive (1 m/s at 10 Hz, 1 cm / 0.2 deg jitter) turning 0.002 rad per frame: a keyframe about every 10 frames."""
    rng = np.random.Generator(np.random.PCG64(seed + 1))
    poses, x, y, yaw = [], -12.0, 0.0, 0.0
    for _ in range(n_frames):
        jt, jr = rng.normal(0, 0.01, 3), rng.normal(0, np.radians(0.2), 3)
        poses.append(syn.pose7([x + jt[0], y + jt[1], 1.8 + jt[2]], syn.quat_from_rpy(jr[0], jr[1], yaw + jr[2])))
        x, y, yaw = x + 0.1 * np.cos(yaw), y + 0.1 * np.sin(yaw), yaw + 0.002
    return np.stack(poses)


def workload(n_frames):
    scene = syn.make_scene()
    traj = trajectory(n_frames)
    sweeps = [syn.make_multi_sweep(scene, traj[k], 1, 64, 2048, seed=200 + k) for k in range(n_frames)]
    odom = np.stack([syn.pose_mul(traj[k], syn.pose7([0.002 * k, -0.001 * k, 0.0], syn.quat_from_rpy(0.0, 0.0, np.radians(0.02 * k))))
                     for k in range(n_frames)])
    ext = sweeps[0][3]
    ext_cov = ua.ext_covariances(1, seed=5, scale=1.6)
    _, _, _, sc = ua.frame_multi_ua(sweeps[0][0], sweeps[0][1], sweeps[0][2], 1, ext, ext_cov, COV_MEAS, 1e30, np.zeros((10, 4), np.float32),
                                    np.zeros((10, 4), np.float32), traj[0])
    c6 = np.concatenate([sc["surf_cov6"], sc["corner_cov6"]]).astype(np.float64)
    tr = np.sort(c6[:, 0] + c6[:, 3] + c6[:, 5])
    k = int(0.9 * tr.shape[0])
    return sweeps, odom, ext, ext_cov, float(0.5 * (tr[k - 1] + tr[k]))


class HostStore:
    """The caller-side keyframe loop the device store replaces (state of saveKeyframe / extractSurroundingKeyFrames on the host)."""

    def __init__(self, ctx, ext, ext_cov, with_ua, thr):
        self.ctx, self.ext, self.ext_cov, self.with_ua, self.thr = ctx, ext, ext_cov, with_ua, thr
        self.poses, self.covs, self.surf, self.corner = [], [], [], []
        self.prev_pt, self.prev_q = np.zeros(3, np.float32), np.array([0, 0, 0, 1.0])
        self.sur, self.stale = [], True
        self.bytes = 0

    def save(self, pose, cov):
        if not ml.np_keyframe_due(pose, self.prev_pt, self.prev_q, len(self.poses), KF["dist"], KF["orient"]):
            return False
        sp, sc6, cp, cc6 = self.ctx.frame_scan()  # device -> host: points + cov_vec of both scans
        self.bytes += sp.nbytes + sc6.nbytes + cp.nbytes + cc6.nbytes
        self.poses.append(pose.copy()), self.covs.append(np.zeros((6, 6)) if len(self.poses) <= 11 else cov.copy())
        self.surf.append(sp), self.corner.append(cp)
        self.prev_pt, self.prev_q = pose[:3].astype(np.float32), pose[3:].copy()
        self.stale = True
        return True

    def submap(self, pred):
        if not self.poses or not self.stale:
            return False
        pos = np.stack([p[:3] for p in self.poses]).astype(np.float32)
        found, _ = ml.np_radius_search(pos, pred[:3].astype(np.float32), KF["radius"])
        self.sur, _ = ml.np_bookkeeping(self.sur, found)
        pts = np.concatenate([pos[self.sur], np.arange(len(self.sur), dtype=np.float32)[:, None]], 1)
        ds = self.ctx.voxel_downsample(pts, KF["res"], True)
        chosen = [self.sur[int(p[3])] for p in ds]
        L = self.ext.shape[0]
        pc, cc = np.zeros((len(chosen), L, 7)), np.zeros((len(chosen), L, 36))
        for i, k in enumerate(chosen):
            for l in range(L):
                a, b = self.ctx.compound_pose_cov(self.poses[k], self.covs[k], self.ext[l], self.ext_cov[l] if self.with_ua else np.zeros((6, 6)))
                pc[i, l], cc[i, l] = a, b.reshape(36)
        poses = np.stack([self.poses[k] for k in chosen])
        n = []
        for slot, clouds, leaf in ((1, [self.surf[k] for k in chosen], self.ctx.params.surf_leaf), (0, [self.corner[k] for k in chosen], self.ctx.params.corner_leaf)):
            self.bytes += sum(c.nbytes for c in clouds)  # host -> device: every chosen keyframe, every rebuild
            n.append(self.ctx.submap_assemble(slot, clouds, poses, self.ext, pc, cc, COV_MEAS, leaf, self.with_ua, self.thr, self.thr, 0.0,
                                              want_output=False))
        self.stale = not (n[0] > 0 and n[1] > 0)
        return True


def run(m, wl, with_ua, device):
    sweeps, odom, ext, ext_cov, thr = wl
    p = m.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = 64, 10, 1, 0.0, 2048
    ctx = m.Context(0, p)
    ctx.set_lidars(1, ext)
    ctx.set_uncertainty(with_ua, ext_cov if with_ua else None, COV_MEAS, thr)
    if device:
        ctx.keyframes_init(KF["dist"], KF["orient"], KF["radius"], KF["res"], thr)
    else:
        hs = HostStore(ctx, ext, ext_cov, with_ua, thr)
        ctx.map_build(1, np.zeros((0, 4), np.float32)), ctx.map_build(0, np.zeros((0, 4), np.float32))
    n = max(s[0].shape[0] for s in sweeps)
    buf = np.zeros((n, 4), np.float32)  # one sweep buffer: frames replay their graph
    wmap_wodom = np.array([0, 0, 0, 0, 0, 0, 1.0])
    ms_kf, ms_reg, fr_kf, fr_reg, poses, kf_bytes, n_kf_steps = [], [], [], [], [], 0, 0
    for k, (cloud, ss, se, _) in enumerate(sweeps):
        buf[:] = 0
        buf[:cloud.shape[0]] = cloud
        pred = ml.pose_mul(wmap_wodom, odom[k])
        t0 = time.perf_counter()
        if device:
            rebuilt = ctx.keyframe_submap(pred)[0]
        else:
            b0 = hs.bytes
            rebuilt = hs.submap(pred)
        t1 = time.perf_counter()
        pose, st = ctx.frame(buf, ss, se, None, None, pred, False)
        t2 = time.perf_counter()
        if device:
            saved = ctx.keyframe_save()
        else:
            saved = hs.save(pose, ctx.pose_covariance())
        dt = (time.perf_counter() - t0) * 1e3  # frame and save end in a device synchronisation
        wmap_wodom = ml.pose_mul(pose, ml.pose_inv(odom[k]))
        poses.append(pose)
        if k > 1:  # the first steps also load modules and capture
            (ms_kf if (saved or rebuilt) else ms_reg).append(dt)
            (fr_kf if (saved or rebuilt) else fr_reg).append((t2 - t1) * 1e3)
        if saved or rebuilt:
            n_kf_steps += 1
            if not device:
                kf_bytes += hs.bytes - b0
    n_kf = ctx.keyframe_query()[0] if device else len(hs.poses)
    capture_failures = ctx.profile_get("graph_capture_failures")[1]
    ctx.close()
    total = sum(ms_kf) + sum(ms_reg)
    med = lambda v: float(np.median(v)) if v else None  # noqa: E731
    return dict(ms_keyframe_step=med(ms_kf), ms_regular_step=med(ms_reg), ms_frame_in_keyframe_step=med(fr_kf), ms_frame_in_regular_step=med(fr_reg),
                regular_steps=len(ms_reg), graph_capture_failures=capture_failures, frames_per_s=(len(ms_kf) + len(ms_reg)) / (total / 1e3), keyframes=n_kf, keyframe_steps=n_kf_steps,
                pcie_point_bytes_per_keyframe_step=(kf_bytes / max(n_kf_steps, 1)) if not device else 0, poses=np.stack(poses))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 2
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    m = bench.load_mloam()
    wl = workload(args.frames)
    out = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi.splitlines()[0] if smi else None, "frames": args.frames,
           "keyframe_params": KF, "trace_threshold": wl[4]}
    for with_ua in (False, True):
        runs = {"device": [], "host": []}
        for _ in range(args.repeats):
            for path in ("device", "host"):
                runs[path].append(run(m, wl, with_ua, path == "device"))
        d, h = runs["device"][-1], runs["host"][-1]
        dpose = max(max(syn.pose_err(a, b)) for a, b in zip(d["poses"], h["poses"]))
        out["with_ua" if with_ua else "plain"] = {
            path: {k: ([None if r[k] is None else round(r[k], 3) for r in v] if k.startswith("ms_") or k == "frames_per_s" else v[-1][k])
                   for k in ("ms_keyframe_step", "ms_regular_step", "ms_frame_in_keyframe_step", "ms_frame_in_regular_step", "frames_per_s", "keyframes",
                             "keyframe_steps", "regular_steps", "graph_capture_failures", "pcie_point_bytes_per_keyframe_step")}
            for path, v in runs.items()}
        out["with_ua" if with_ua else "plain"]["max_pose_diff_device_vs_host"] = dpose
    print(json.dumps(out))
    return 0


if __name__ == "__main__":
    sys.exit(main())

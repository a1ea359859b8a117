"""Test infrastructure of the outlier cloud (mloam_set_outlier / mloam_frame_outlier / mloam_keyframe_outlier and the outlier appends of
mloam_global_map): the binding of the oracle's frame_outlier (oracle/orc_ua.cpp in oracle_lib's library; the keyframe store and the global
map with outliers are mapper_lib.Mapper and global_map_lib.global_map), and an independent composition of the same steps in numpy from the
oracle's single-step entry points."""
from __future__ import annotations

import ctypes as C

import numpy as np

import global_map_lib as gml
import oracle_lib as orc
import uncertainty_lib as ua

SURROUND, SAVE = gml.SURROUND, gml.SAVE
_p = orc._p


def frame_outlier(cloud, scan_start, n_lidars, ext7, ext_cov, cov_meas, with_ua, trace_threshold, leaf):
    """The oracle's laser_cloud_outlier_cov of a rig frame (mloam_frame's inputs): (points [m,4], cov6 [m,6])."""
    pts = orc.cloud(cloud)
    ss = np.ascontiguousarray(scan_start, np.int32)
    e = np.ascontiguousarray(ext7, np.float64).reshape(-1)
    ec = np.ascontiguousarray(ext_cov if ext_cov is not None else np.zeros((n_lidars, 6, 6)), np.float64).reshape(-1)
    cm = np.ascontiguousarray(cov_meas, np.float64).reshape(9)
    out, c6, n = np.zeros((n_lidars, 4), np.float32), np.zeros((n_lidars, 6), np.float32), C.c_int(0)
    orc.lib().orc_outlier_frame(_p(pts), pts.shape[0], _p(ss), ss.shape[0], n_lidars, _p(e), _p(ec), _p(cm), int(with_ua),
                                C.c_double(trace_threshold), C.c_float(leaf), _p(out), _p(c6), C.byref(n))
    return out[:n.value].copy(), c6[:n.value].copy()


# ---------------------------------------------------------------------------------------- independent composition
def np_rig_matrix(ext7):
    """Pose(q, t).T_.cast<float>(): the float 3x4 matrix of a normalised quaternion and a translation."""
    e = np.asarray(ext7, np.float64)
    x, y, z, w = e[3:7] / np.linalg.norm(e[3:7])
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    return np.concatenate([R, e[:3, None]], axis=1).astype(np.float32)


def np_first_points(cloud, scan_start, n_lidars):
    """laser_cloud_out.points[0] of each LiDAR's part of the concatenation, (laser id, point) for the non-empty parts."""
    cloud = np.asarray(cloud, np.float32)
    R = len(scan_start) // n_lidars
    out = []
    for l in range(n_lidars):
        lo = int(scan_start[l * R]) - 5
        hi = int(scan_start[(l + 1) * R]) - 5 if l + 1 < n_lidars else cloud.shape[0]
        if lo < hi:
            out.append((l, cloud[lo]))
    return out


def np_transform(p, m):
    """pcl::transformPointCloud of one point: x' = m00 x + m01 y + m02 z + m03 in float, left to right."""
    f = np.float32
    return np.array([f(f(f(m[r, 0] * p[0]) + f(m[r, 1] * p[1])) + f(m[r, 2] * p[2])) + m[r, 3] for r in range(3)], np.float32)


def compose_frame(cloud, scan_start, n_lidars, ext7, ext_cov, cov_meas, with_ua, trace_threshold, leaf):
    """The four steps one by one: first points, float transform with intensity = id, VoxelGridCovarianceMLOAM<PointI>, the trace gate.
    Returns (points, cov6, traces of the filtered points) — the traces let a caller keep its cases away from the threshold."""
    ext7 = np.asarray(ext7, np.float64).reshape(-1, 7)
    raw = []
    for l, p in np_first_points(cloud, scan_start, n_lidars):
        raw.append(np.concatenate([np_transform(p, np_rig_matrix(ext7[l])), [np.float32(l)]]).astype(np.float32))
    if not raw:
        return np.zeros((0, 4), np.float32), np.zeros((0, 6), np.float32), np.zeros(0)
    ds, _ = orc.voxel_grid(np.stack(raw), leaf, intensity_last=True)
    pts, cov, traces = [], [], []
    for p in ds:
        c6 = np.zeros(6, np.float32)
        if with_ua:
            idx = int(p[3])
            sel = orc.associate(p[None], ua.pose_inv(ext7[idx]))
            c6 = orc.point_uncertainty(sel, ext7[idx], ext_cov[idx], cov_meas)[0]
            tr = float(c6[0]) + float(c6[3]) + float(c6[5])
            traces.append(tr)
            if tr > trace_threshold:
                continue
        pts.append(p), cov.append(c6)
    if not pts:
        return np.zeros((0, 4), np.float32), np.zeros((0, 6), np.float32), np.array(traces)
    return np.stack(pts).astype(np.float32), np.stack(cov).astype(np.float32), np.array(traces)


def compose_global(keyframes, ext7, ext_cov, cov_meas, with_ua, trace_thr, mode, chosen, leaf):
    """keyframes[id] = (pose7, cov 6x6, surf, corner, outlier).  Each chosen keyframe's clouds through cloudUCTAssociateToMap, concatenated in
    the reference's orders — SURROUND surf, corner, outlier into map 0; SAVE surf, outlier into map 0 and corner into map 1 — then
    VoxelGridCovarianceMLOAM<PointIWithCov>(leaf)."""
    ext7 = np.asarray(ext7, np.float64).reshape(-1, 7)
    L = ext7.shape[0]
    raw = [[], []]
    order = [(0, 0), (1, 0), (2, 0)] if mode == SURROUND else [(0, 0), (2, 0), (1, 1)]
    for i in chosen:
        pose, cov = keyframes[i][:2]
        pc, cc = [], []
        for l in range(L):
            ec = ext_cov[l] if with_ua else np.zeros((6, 6))
            a, b = orc.compound_pose_cov(pose, cov, ext7[l], ec)
            pc.append(a), cc.append(b)
        for t, m in order:
            cl = keyframes[i][2 + t]
            if cl.shape[0] == 0:
                continue
            raw[m].append(orc.cloud_uct_associate(cl, pose, ext7, np.stack(pc), np.stack(cc), cov_meas, with_ua, trace_thr))
    out = []
    for parts in raw[:1 if mode == SURROUND else 2]:
        if not parts:
            out += [np.zeros((0, 4), np.float32), np.zeros((0, 6), np.float32)]
            continue
        p, c6, _, _ = orc.voxel_grid_cov(np.concatenate([x[0] for x in parts]), np.concatenate([x[1] for x in parts]),
                                         np.concatenate([x[2] for x in parts]), leaf, trace_thr)
        out += [p, c6]
    return out

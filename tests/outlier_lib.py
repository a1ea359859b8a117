"""Test infrastructure of the outlier cloud (mloam_set_outlier / mloam_frame_outlier / mloam_keyframe_outlier and the outlier appends of
mloam_global_map): ctypes binding of the oracle's restatement (tests/host/orc_outlier.cpp over oracle/orc_mapper.cpp), compiled on first use
into a temporary directory keyed by the sources' hash (the tree is never written), and an independent composition of the same steps in
numpy from the oracle's single-step entry points."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import global_map_lib as gml
import oracle_lib as orc
import uncertainty_lib as ua

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host", "orc_outlier.cpp")
SURROUND, SAVE = gml.SURROUND, gml.SAVE
_p = orc._p
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for f in sorted(f for f in os.listdir(orc.ORC_DIR) if f.endswith((".hpp", ".cpp"))):
            h.update(f.encode())
            with open(os.path.join(orc.ORC_DIR, f), "rb") as fh:
                h.update(fh.read())
        with open(SRC, "rb") as fh:
            h.update(fh.read())
        h.update(" ".join(ua.CXXFLAGS).encode())
        so = os.path.join(tempfile.gettempdir(), f"mloam_orc_outlier_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["/usr/bin/g++", *ua.CXXFLAGS, "-shared", "-o", tmp, SRC])
            os.replace(tmp, so)
        _lib = C.CDLL(so)
        _lib.orc_outlier_mapper_create.restype = C.c_void_p
        _lib.orc_outlier_mapper_create.argtypes = [C.c_double] * 5 + [C.c_float] * 2
        _lib.orc_outlier_global_map.restype = C.c_void_p
        _lib.orc_outlier_global_map.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_double, C.c_float, C.c_void_p]
        _lib.orc_outlier_global_map_read.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.orc_outlier_global_map_free.argtypes = [C.c_void_p]
        for f in ("orc_outlier_mapper_destroy", "orc_outlier_mapper_set_lidars", "orc_outlier_mapper_save", "orc_outlier_frame"):
            getattr(_lib, f).argtypes = None
    return _lib


def frame_outlier(cloud, scan_start, n_lidars, ext7, ext_cov, cov_meas, with_ua, trace_threshold, leaf):
    """The oracle's laser_cloud_outlier_cov of a rig frame (mloam_frame's inputs): (points [m,4], cov6 [m,6])."""
    pts = orc.cloud(cloud)
    ss = np.ascontiguousarray(scan_start, np.int32)
    e = np.ascontiguousarray(ext7, np.float64).reshape(-1)
    ec = np.ascontiguousarray(ext_cov if ext_cov is not None else np.zeros((n_lidars, 6, 6)), np.float64).reshape(-1)
    cm = np.ascontiguousarray(cov_meas, np.float64).reshape(9)
    out, c6, n = np.zeros((n_lidars, 4), np.float32), np.zeros((n_lidars, 6), np.float32), C.c_int(0)
    lib().orc_outlier_frame(_p(pts), pts.shape[0], _p(ss), ss.shape[0], n_lidars, _p(e), _p(ec), _p(cm), int(with_ua),
                            C.c_double(trace_threshold), C.c_float(leaf), _p(out), _p(c6), C.byref(n))
    return out[:n.value].copy(), c6[:n.value].copy()


class Mapper:
    """The oracle's keyframe store with an outlier cloud per keyframe, made and used by this module's library."""

    def __init__(self, distance_keyframes, orientation_keyframes_deg, radius, sur_kf_res, trace_threshold, surf_leaf=0.4, corner_leaf=0.2):
        self._h = C.c_void_p(lib().orc_outlier_mapper_create(distance_keyframes, orientation_keyframes_deg, radius, sur_kf_res, trace_threshold,
                                                             surf_leaf, corner_leaf))

    def close(self):
        if self._h:
            lib().orc_outlier_mapper_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_lidars(self, ext7, ext_cov, cov_meas, with_ua: bool):
        e = np.ascontiguousarray(ext7, np.float64).reshape(-1)
        ec = None if ext_cov is None else np.ascontiguousarray(ext_cov, np.float64).reshape(-1)
        cm = None if cov_meas is None else np.ascontiguousarray(cov_meas, np.float64).reshape(9)
        lib().orc_outlier_mapper_set_lidars(self._h, e.shape[0] // 7, _p(e), _p(ec), _p(cm), int(with_ua))

    def save(self, pose7, cov, surf, corner, outlier):
        """saveKeyframe with the three clouds: (saved, (distance margin [m], angle margin [deg]))."""
        s, c, o = orc.cloud(surf), orc.cloud(corner), orc.cloud(np.asarray(outlier, np.float32).reshape(-1, 4))
        m = np.zeros(2)
        r = lib().orc_outlier_mapper_save(self._h, _p(np.ascontiguousarray(pose7, np.float64)), _p(np.ascontiguousarray(cov, np.float64).reshape(36)),
                                          _p(s), s.shape[0], _p(c), c.shape[0], _p(o), o.shape[0], _p(m))
        return bool(r), (m[0], m[1])


def global_map(mapper: Mapper, mode: int, center7, radius: float, kf_leaf: float, leaf: float):
    """The oracle's global map with the outlier appends: (chosen ids, [map 0 points, map 0 cov6, map 1 points, map 1 cov6])."""
    ct = None if center7 is None else np.ascontiguousarray(center7, np.float64)
    cnt = np.zeros(3, np.int32)
    r = lib().orc_outlier_global_map(mapper._h.value, int(mode), _p(ct), float(radius), float(kf_leaf), float(leaf), _p(cnt))
    try:
        ch = np.zeros(max(cnt[0], 1), np.int32)
        out = []
        for which in (0, 1):
            n = int(cnt[1 + which])
            p, c6 = np.zeros((max(n, 1), 4), np.float32), np.zeros((max(n, 1), 6), np.float32)
            lib().orc_outlier_global_map_read(r, which, _p(ch), _p(p), _p(c6))
            out += [p[:n], c6[:n]]
        return ch[:cnt[0]].tolist(), out
    finally:
        lib().orc_outlier_global_map_free(r)


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

"""Test infrastructure of the registered clouds (mloam_set_registered / mloam_frame_registered): the binding of the oracle's pubPointCloud at a
given pose (oracle/orc_registered.cpp, built by oracle/registered.mk), and an independent composition of the same steps in numpy from the
single-step pieces (TransformToEnd of undistort_lib, the float rig matrix of outlier_lib, extractCloud of oracle_lib)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib as orc
import outlier_lib as ol
import undistort_lib as udl

_p = orc._p
FULL_RES, SURF, CORNER = 0, 1, 2
_lib = None


def lib():
    """oracle/liborc_registered.so (oracle/registered.mk), rebuilt when a source is newer."""
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-C", orc.ORC_DIR, "-f", "registered.mk"], stdout=subprocess.DEVNULL)
        _lib = C.CDLL(os.path.join(orc.ORC_DIR, "liborc_registered.so"))
    return _lib


def _f64(a):
    return None if a is None else np.ascontiguousarray(a, np.float64).reshape(-1)


def registered(cloud, scan_start, scan_end, pose7, ext7=None, single_ext7=None, poses7=None, scan_period=0.1, outlier=False):
    """The oracle's three clouds [full_res, surf_last, corner_last] at pose7.  ext7 [L, 7]: the rig merge; None: one LiDAR, moved with
    single_ext7 (None: not moved).  poses7 [L, 7]: the undistortion.  outlier: append laser_cloud_outlier to the full-resolution cloud."""
    pts = orc.cloud(cloud)
    ss, se = np.ascontiguousarray(scan_start, np.int32), np.ascontiguousarray(scan_end, np.int32)
    n = pts.shape[0]
    L = 1 if ext7 is None else np.asarray(ext7).reshape(-1, 7).shape[0]
    full, surf, corner = np.zeros((n + L, 4), np.float32), np.zeros((max(n, 1), 4), np.float32), np.zeros((max(n, 1), 4), np.float32)
    nf, ns, nc = C.c_int(0), C.c_int(0), C.c_int(0)
    lib().orc_frame_registered(_p(pts), n, _p(ss), _p(se), ss.shape[0], L, _p(_f64(ext7)), _p(_f64(single_ext7)), _p(_f64(poses7)),
                               C.c_float(scan_period), int(bool(outlier)), _p(np.ascontiguousarray(pose7, np.float64)), _p(full), C.byref(nf),
                               _p(surf), C.byref(ns), _p(corner), C.byref(nc))
    return [full[:nf.value].copy(), surf[:ns.value].copy(), corner[:nc.value].copy()]


# ---------------------------------------------------------------------------------------- independent composition
def np_associate(pts, pose7):
    """pointAssociateToMap: q * p + t as Eigen evaluates it (v + w (2 u x v) + u x (2 u x v)) in double, stored to float, intensity kept."""
    p = np.asarray(pts, np.float32)
    out = p.copy()
    if p.shape[0] == 0:
        return out
    x = np.asarray(pose7, np.float64)
    ux, uy, uz, w = x[3], x[4], x[5], x[6]
    vx, vy, vz = (p[:, k].astype(np.float64) for k in range(3))
    with np.errstate(invalid="ignore", over="ignore"):  # non-finite points are transformed like the others
        cx, cy, cz = uy * vz - uz * vy, uz * vx - ux * vz, ux * vy - uy * vx
        cx, cy, cz = cx + cx, cy + cy, cz + cz
        dx, dy, dz = uy * cz - uz * cy, uz * cx - ux * cz, ux * cy - uy * cx
        out[:, 0] = ((vx + w * cx + dx) + x[0]).astype(np.float32)
        out[:, 1] = ((vy + w * cy + dy) + x[1]).astype(np.float32)
        out[:, 2] = ((vz + w * cz + dz) + x[2]).astype(np.float32)
    return out


def np_rig(pts, ext7, laser_id):
    """transformCloudFeature: the float 3x4 matrix of ext7, PCL's order, intensity = laser id."""
    m = ol.np_rig_matrix(ext7)
    p = np.asarray(pts, np.float32)
    out = np.zeros_like(p)
    with np.errstate(invalid="ignore", over="ignore"):  # non-finite points are transformed like the others
        for r in range(3):  # float32 ufuncs: one rounding per multiply and add, left to right (outlier_lib.np_transform, vectorised)
            out[:, r] = ((m[r, 0] * p[:, 0] + m[r, 1] * p[:, 1]) + m[r, 2] * p[:, 2]) + m[r, 3]
    out[:, 3] = np.float32(laser_id)
    return out


def parts(n, scan_start, n_lidars):
    """LiDAR l's part [scan_start[l R] - 5, scan_start[(l + 1) R] - 5) of the concatenation, the last one ending at n."""
    R = len(scan_start) // n_lidars
    return [(int(scan_start[l * R]) - 5, int(scan_start[(l + 1) * R]) - 5 if l + 1 < n_lidars else n) for l in range(n_lidars)]


def compose(cloud, scan_start, scan_end, pose7, ext7=None, single_ext7=None, poses7=None, scan_period=0.1, outlier=False):
    """registered() step by step: per LiDAR part [TransformToEnd] -> base frame, the features of its own extractCloud the same way, the outlier
    points after the sweep, pointAssociateToMap with pose7 last."""
    cloud = orc.cloud(cloud)
    ss, se = np.asarray(scan_start, np.int32), np.asarray(scan_end, np.int32)
    L = 1 if ext7 is None else np.asarray(ext7).reshape(-1, 7).shape[0]
    R = len(ss) // L
    full, surf, corner, outl = [], [], [], []
    cuts = parts(cloud.shape[0], ss, L) if ext7 is not None else [(0, cloud.shape[0])]
    for l, (lo, hi) in enumerate(cuts):
        part = cloud[lo:hi] if hi > lo else np.zeros((0, 4), np.float32)
        f = orc.extract_cloud(part, ss[l * R:(l + 1) * R] - lo, se[l * R:(l + 1) * R] - lo) if part.shape[0] else None
        clouds = [part] + ([f["surf_points_less_flat"], f["corner_points_less_sharp"]] if f else [part[:0], part[:0]])
        for k, c in enumerate(clouds):
            if poses7 is not None and c.shape[0]:
                c = udl.points(c, np.asarray(poses7).reshape(-1, 7)[l], scan_period)
            if ext7 is not None:
                c = np_rig(c, np.asarray(ext7).reshape(-1, 7)[l], l)
            elif single_ext7 is not None:
                c = np_associate(c, single_ext7)
            (full, surf, corner)[k].append(c)
        if outlier and lo < hi and 0 <= lo < cloud.shape[0]:
            e = np.asarray(ext7).reshape(-1, 7)[l] if ext7 is not None else (single_ext7 if single_ext7 is not None else [0, 0, 0, 0, 0, 0, 1.0])
            outl.append(np_rig(cloud[lo:lo + 1], e, l))
    cat = lambda cs: np.concatenate(cs) if cs else np.zeros((0, 4), np.float32)  # noqa: E731
    return [np_associate(cat(full + outl), pose7), np_associate(cat(surf), pose7), np_associate(cat(corner), pose7)]


def bits_equal(a, b):
    """Bit identity with NaN and inf compared by class and position, finite values by their int32 views."""
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    if a.shape != b.shape:
        return False
    fa, fb = np.isfinite(a), np.isfinite(b)
    if not np.array_equal(fa, fb) or not np.array_equal(np.isnan(a), np.isnan(b)) or not np.array_equal(np.isposinf(a), np.isposinf(b)):
        return False
    return np.array_equal(a[fa].view(np.int32), b[fb].view(np.int32))

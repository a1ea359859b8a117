"""Test infrastructure of the undistortion (mloam_set_distortion / mloam_frame_undistort / mloam_undistort_poses): bindings of the
oracle's restatement (oracle/orc_ua.cpp in oracle_lib's library) and of the device header compiled for the host
(tests/host/undistort_header.cpp over m-loam_b200/csrc/undistort.cuh, host_build); and a sweep seen by a sensor that moves during it, with
its exact answer."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

import host_build
import oracle_lib as orc

_p = orc._p


def header():
    return host_build.load("undistort_header")


def points(pts, pose7, scan_period=0.1):
    """The oracle's TransformToEnd of points [n,4] with one pose [t q]."""
    p = orc.cloud(pts)
    out = np.zeros_like(p)
    orc.lib().orc_undist_points(_p(p), p.shape[0], _p(np.ascontiguousarray(pose7, np.float64)), C.c_float(scan_period), _p(out))
    return out


def header_points(pts, pose7s, scan_period=0.1, use_libm=False):
    """The device header's TransformToEnd on the host: (points, double sines that differ from the C library's); point i takes pose
    i % len(pose7s)."""
    p = orc.cloud(pts)
    poses = np.ascontiguousarray(pose7s, np.float64).reshape(-1, 7)
    out, diff = np.zeros_like(p), C.c_longlong(0)
    header().ud_transform(_p(p), p.shape[0], _p(poses), poses.shape[0], C.c_float(scan_period), int(use_libm), _p(out), C.byref(diff))
    return out, diff.value


def poses(pose_rlt7, idx_ref, ext7, estimate_extrinsic):
    e = np.ascontiguousarray(ext7, np.float64).reshape(-1, 7)
    out = np.zeros_like(e)
    orc.lib().orc_undist_poses(_p(np.ascontiguousarray(pose_rlt7, np.float64)), int(idx_ref), e.shape[0], _p(e), int(estimate_extrinsic), _p(out))
    return out


def frame(cloud, scan_start, scan_end, n_lidars, ext7, pose7s, surf_map, corner_map, pose_init, scan_period=0.1, single_ext7=None,
          ext_cov=None, cov_meas=None, trace_threshold=0.0, opts=None, corner_leaf=0.2, surf_leaf=0.4):
    """The oracle's frame with the undistortion (pose7s None: without it).  ext7 None: the single-LiDAR path (single_ext7: the extrinsic of
    mloam_set_extrinsic).  ext_cov: with_ua.  Returns (pose, stats, cov 6x6, dict(surf, surf_cov6, corner, corner_cov6))."""
    pts, sm, cm = orc.cloud(cloud), orc.cloud(surf_map), orc.cloud(corner_map)
    ss, se = np.ascontiguousarray(scan_start, np.int32), np.ascontiguousarray(scan_end, np.int32)
    f64 = lambda a: None if a is None else np.ascontiguousarray(a, np.float64).reshape(-1)  # noqa: E731
    opts = orc.default_opts() if opts is None else np.ascontiguousarray(opts, np.float64)
    out, stats, cov = np.empty(7), np.zeros(20), np.zeros(36)
    n = pts.shape[0]
    so, sc, co, cc = np.zeros((n, 4), np.float32), np.zeros((n, 6), np.float32), np.zeros((n, 4), np.float32), np.zeros((n, 6), np.float32)
    ns, nc = C.c_int(0), C.c_int(0)
    cmeas = f64(cov_meas if cov_meas is not None else np.zeros((3, 3)))
    orc.lib().orc_frame_ua(_p(pts), n, _p(ss), _p(se), ss.shape[0], n_lidars, _p(f64(ext7)), _p(f64(single_ext7)), _p(f64(pose7s)),
                           C.c_float(scan_period), _p(f64(ext_cov)), _p(cmeas), C.c_double(trace_threshold), _p(sm), sm.shape[0], _p(cm),
                           cm.shape[0], C.c_float(corner_leaf), C.c_float(surf_leaf), _p(np.ascontiguousarray(pose_init, np.float64)),
                           _p(opts), _p(out), _p(stats), _p(cov), None, _p(so), _p(sc), C.byref(ns), _p(co), _p(cc), C.byref(nc))
    names = ["ran", "n_surf", "n_corner", "lm_iterations", "final_cost", "degenerate"]
    st = {k: stats[i] for i, k in enumerate(names)}
    st.update(n_surf_in=int(stats[18]), n_corner_in=int(stats[19]))
    return out, st, cov.reshape(6, 6), dict(surf=so[:ns.value].copy(), surf_cov6=sc[:ns.value].copy(), corner=co[:nc.value].copy(),
                                           corner_cov6=cc[:nc.value].copy())


# ---------------------------------------------------------------------------------------- numpy helpers
def qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz])


def qrot(q, v):
    u, w = np.asarray(q[:3]), q[3]
    uv = 2 * np.cross(u, v)
    return v + w * uv + np.cross(u, uv)


def pose_mul(a, b):
    q = qmul(a[3:], b[3:])
    return np.concatenate([qrot(a[3:], b[:3]) + a[:3], q / np.linalg.norm(q)])


def pose_inv(a):
    q = np.array([-a[3], -a[4], -a[5], a[6]]) / np.linalg.norm(a[3:])
    return np.concatenate([-qrot(q, a[:3]), q])


def rot_pose(axis, angle, t):
    """[t q] of a rotation by angle about axis."""
    ax = np.asarray(axis, np.float64)
    ax = ax / np.linalg.norm(ax)
    return np.concatenate([np.asarray(t, np.float64), ax * math.sin(angle / 2), [math.cos(angle / 2)]])


def moving_sweep(rng, n, pose_end7, scan_period=0.1, rings=16, r_min=0.5, r_max=100.0):
    """A sweep of a sensor that moves from the identity at its start to pose_end7 at its end with constant angular and linear velocity (the
    interpolation TransformToStart assumes: rotation slerp(s), translation s t).  Point k is a static world point X_k seen at the sweep
    fraction s_k: p = R(s)^T (X - s t), intensity = ring + s scan_period.  Returns (points [n,4] float32, X seen from the end pose [n,3])."""
    q = np.asarray(pose_end7[3:], np.float64)
    t = np.asarray(pose_end7[:3], np.float64)
    ang = 2 * math.atan2(np.linalg.norm(q[:3]), q[3])
    axis = q[:3] / max(np.linalg.norm(q[:3]), 1e-300)
    s = rng.uniform(0.0, 1.0, n)
    ring = rng.integers(0, rings, n)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    p_local = d * rng.uniform(r_min, r_max, n)[:, None]
    pts = np.zeros((n, 4), np.float32)
    end = np.zeros((n, 3))
    for k in range(n):
        qs = np.concatenate([axis * math.sin(s[k] * ang / 2), [math.cos(s[k] * ang / 2)]])
        X = qrot(qs, p_local[k]) + s[k] * t  # world point (the sweep-start frame)
        pts[k, :3] = p_local[k]
        pts[k, 3] = np.float32(ring[k]) + np.float32(s[k] * scan_period)
        end[k] = qrot(np.array([-q[0], -q[1], -q[2], q[3]]), X - t)
    return pts, end

"""Test infrastructure of the uncertainty-aware mapper (with_ua): ctypes binding of the oracle's with_ua entry points
(oracle/orc_ua.cpp, compiled on first use into a temporary directory, keyed by the sources' hash, so that the tree is never
written) and a seeded generator of extrinsic covariances."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import oracle_lib as orc

ORC_DIR = orc.ORC_DIR
CXXFLAGS = ["-O3", "-march=x86-64-v3", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-Wall", "-Wno-unused-function",
            "-Wno-array-bounds"]  # the flags of oracle/Makefile's liborc.so
_p = orc._p
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = sorted(f for f in os.listdir(ORC_DIR) if f.endswith(".hpp")) + ["orc_ua.cpp"]
        h = hashlib.sha256()
        for f in srcs:
            h.update(f.encode())
            with open(os.path.join(ORC_DIR, f), "rb") as fh:
                h.update(fh.read())
        h.update(" ".join(CXXFLAGS).encode())
        so = os.path.join(tempfile.gettempdir(), f"mloam_orc_ua_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["/usr/bin/g++", *CXXFLAGS, "-shared", "-o", tmp, os.path.join(ORC_DIR, "orc_ua.cpp")])
            os.replace(tmp, so)
        _lib = C.CDLL(so)
    return _lib


def frame_multi_ua(cloud_, scan_start, scan_end, n_lidars, ext7, ext_cov, cov_meas, trace_threshold, surf_map, corner_map, pose_init, opts=None,
                   corner_leaf=0.2, surf_leaf=0.4):
    """orc.frame_multi with with_ua = true: per-point uncertainty + trace gate after the scan filters, sqrt_info weights, cov_mapping.
    Returns (pose, stats, cov 6x6, dict(surf, surf_cov6, corner, corner_cov6, H))."""
    pts, sm, cm = orc.cloud(cloud_), orc.cloud(surf_map), orc.cloud(corner_map)
    ss = np.ascontiguousarray(scan_start, np.int32)
    se = np.ascontiguousarray(scan_end, np.int32)
    ext = np.ascontiguousarray(ext7, np.float64).reshape(-1)
    ec = np.ascontiguousarray(ext_cov, np.float64).reshape(-1)
    cmeas = np.ascontiguousarray(cov_meas, np.float64).reshape(9)
    opts = orc.default_opts() if opts is None else np.ascontiguousarray(opts, np.float64)
    pose_init = np.ascontiguousarray(pose_init, np.float64)
    out, stats, cov, H = np.empty(7), np.zeros(20), np.zeros(36), np.zeros(36)
    n = pts.shape[0]
    so, sc, co, cc = np.zeros((n, 4), np.float32), np.zeros((n, 6), np.float32), np.zeros((n, 4), np.float32), np.zeros((n, 6), np.float32)
    ns, nc = C.c_int(0), C.c_int(0)
    lib().orc_ua_frame_multi(_p(pts), n, _p(ss), _p(se), ss.shape[0], n_lidars, _p(ext), _p(ec), _p(cmeas), C.c_double(trace_threshold), _p(sm),
                             sm.shape[0], _p(cm), cm.shape[0], C.c_float(corner_leaf), C.c_float(surf_leaf), _p(pose_init), _p(opts), _p(out),
                             _p(stats), _p(cov), _p(H), _p(so), _p(sc), C.byref(ns), _p(co), _p(cc), C.byref(nc))
    names = ["ran", "n_surf", "n_corner", "lm_iterations", "final_cost", "degenerate"]
    st = {k: stats[i] for i, k in enumerate(names)}
    st.update(n_surf_in=int(stats[18]), n_corner_in=int(stats[19]))
    scans = dict(surf=so[:ns.value].copy(), surf_cov6=sc[:ns.value].copy(), corner=co[:nc.value].copy(), corner_cov6=cc[:nc.value].copy(),
                 H=H.reshape(6, 6))
    return out, st, cov.reshape(6, 6), scans


def scan2map_ua_cov(surf_map, corner_map, surf_scan, surf_cov6, corner_scan, corner_cov6, pose_init, opts=None):
    """orc.scan2map_ua that also returns cov_mapping = H^-1 at the returned pose and that H: (pose, stats, cov 6x6, H 6x6)."""
    sm, cm, ss, cs = orc.cloud(surf_map), orc.cloud(corner_map), orc.cloud(surf_scan), orc.cloud(corner_scan)
    sc = np.ascontiguousarray(surf_cov6, np.float32)
    cc = np.ascontiguousarray(corner_cov6, np.float32)
    opts = orc.default_opts() if opts is None else np.ascontiguousarray(opts, np.float64)
    pose_init = np.ascontiguousarray(pose_init, np.float64)
    out, stats, cov, H = np.empty(7), np.zeros(8), np.zeros(36), np.zeros(36)
    lib().orc_ua_scan2map(_p(sm), sm.shape[0], _p(cm), cm.shape[0], _p(ss), ss.shape[0], _p(sc), _p(cs), cs.shape[0], _p(cc), _p(pose_init), _p(opts),
                          _p(out), _p(stats), _p(cov), _p(H))
    return out, {"ran": stats[0], "n_surf": int(stats[1]), "n_corner": int(stats[2]), "lm_iterations": int(stats[3]),
                 "final_cost": stats[4]}, cov.reshape(6, 6), H.reshape(6, 6)


def pose_inv(x7):
    """Pose::inverse of a [t q] parameter block (liborc's orc_pose_inv)."""
    a = np.ascontiguousarray(x7, np.float64)
    out = np.zeros(7)
    orc.lib().orc_pose_inv(_p(a), _p(out))
    return out


def ext_covariances(n_lidars: int, seed: int = 0, scale: float = 1.0) -> np.ndarray:
    """[n_lidars, 6, 6] seeded extrinsic covariances [translation | rotation] (pose_ext[l].cov_ of the /extrinsics message):
    standard deviations of 5-10 cm and 0.6-1.2 deg times `scale`, correlated, symmetric positive definite."""
    rng = np.random.Generator(np.random.PCG64(seed))
    out = []
    for _ in range(n_lidars):
        sig = np.concatenate([0.05 * (1.0 + rng.random(3)), 0.01 * (1.0 + rng.random(3))]) * scale
        M = rng.normal(size=(6, 6))
        corr = 0.7 * np.eye(6) + 0.3 * (M @ M.T) / 6.0
        d = 1.0 / np.sqrt(np.diag(corr))
        out.append((sig * d)[:, None] * corr * (sig * d)[None, :])
    return np.stack(out)

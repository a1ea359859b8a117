"""ctypes bindings of the oracle's gd_float pieces (oracle/orc_gf_float.hpp: eval_full_hessian and the policy of
lidar_mapper_keyframe.cpp:456-495 in front of orc::scan2map) and the numpy restatement of evalFullHessian's serial sum the tests compare both sides against."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_lib as orc

_lib = None


def lib():
    """oracle/liborc_gf_float.so (oracle/gf_float.mk), rebuilt when a source is newer."""
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-C", orc.ORC_DIR, "-f", "gf_float.mk"], stdout=subprocess.DEVNULL)
        _lib = C.CDLL(os.path.join(orc.ORC_DIR, "liborc_gf_float.so"))
    return _lib


def full_hessian(kind, map_pts, scan, pose7, cov6=None, default_trace=0.0075, H=None, feat_num=0, opts=None):
    """ActiveFeatureSelection::evalFullHessian for one feature set: (H + sum J^T J, feat_num + matched); H None = 1e-6 I."""
    mp, sc = orc.cloud(map_pts), orc.cloud(scan)
    pose7 = np.ascontiguousarray(pose7, np.float64)
    cv = None if cov6 is None else np.ascontiguousarray(cov6, np.float32)
    op = None if opts is None else np.ascontiguousarray(opts, np.float64)
    Hm = (np.eye(6) * 1e-6 if H is None else np.array(H, np.float64)).reshape(36).copy()
    fn = C.c_int(feat_num)
    lib().orc_full_hessian(ord(kind), orc._p(mp), mp.shape[0], orc._p(sc), sc.shape[0], orc._p(cv), C.c_double(default_trace), orc._p(pose7),
                           orc._p(op), orc._p(Hm), C.byref(fn))
    return Hm.reshape(6, 6), fn.value


def scan2map(surf_map, corner_map, surf_scan, corner_scan, pose_init, opts, surf_cov6=None, corner_cov6=None):
    """One mapper frame from its down-sampled scans on, under the mode gf_float_set left (off: orc.scan2map / orc.scan2map_ua)."""
    sm, cm, ss, cs = orc.cloud(surf_map), orc.cloud(corner_map), orc.cloud(surf_scan), orc.cloud(corner_scan)
    sc = None if surf_cov6 is None else np.ascontiguousarray(surf_cov6, np.float32)
    cc = None if corner_cov6 is None else np.ascontiguousarray(corner_cov6, np.float32)
    opts = np.ascontiguousarray(opts, np.float64)
    pose_init = np.ascontiguousarray(pose_init, np.float64)
    out, stats, H = np.empty(7), np.zeros(16), np.zeros((6, 6))
    lib().orc_gf_float_scan2map(orc._p(sm), sm.shape[0], orc._p(cm), cm.shape[0], orc._p(ss), ss.shape[0], orc._p(sc), orc._p(cs), cs.shape[0],
                                orc._p(cc), orc._p(pose_init), orc._p(opts), orc._p(out), orc._p(stats), orc._p(H))
    return out, {"ran": int(stats[0]), "n_surf": int(stats[1]), "n_corner": int(stats[2]), "lm_iterations": int(stats[3]),
                 "final_cost": stats[4], "H": H}


def gf_float_set(on, map_deg_thre=0.0, gf_ratio_ini=1.0):
    """Start (frame_cnt 0, ratio min(1, ini)) or end gd_float for the scan2map calls of this module."""
    lib().orc_gf_float_set(int(bool(on)), C.c_float(map_deg_thre), C.c_double(gf_ratio_ini))


def gf_float_threshold(map_deg_thre):
    lib().orc_gf_float_threshold(C.c_float(map_deg_thre))


def gf_float_get():
    out = np.zeros(5)
    lib().orc_gf_float_get(orc._p(out))
    return {"frame_cnt": int(out[0]), "ratio_cur": out[1], "deg_factor": out[2], "total_feat_num": int(out[3]), "evaluated": bool(out[4])}


def serial_hessian(jaco, matched, H=None):
    """mat_H = mat_H + jaco^T jaco, matched feature by matched feature in index order: one multiply and one add per element, in double."""
    Hm = np.eye(6) * 1e-6 if H is None else np.array(H, np.float64)
    for j in np.asarray(jaco, np.float64)[np.asarray(matched, bool)]:
        Hm = Hm + np.outer(j, j)
    return Hm


def float_at_or_above(x):
    """The smallest float32 >= x, and the float32 just below it: MAP_DEG_THRE values on the two sides of `factor > threshold`."""
    f = np.float32(x)
    if float(f) < x:
        f = np.nextafter(f, np.float32(np.inf))
    return f, np.nextafter(f, np.float32(-np.inf))

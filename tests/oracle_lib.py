"""ctypes binding of the CPU oracle (oracle/liborc.so) and of oracle/_ref/libref_knn.so.  lib() is the one place that loads the
oracle; uncertainty_lib, mapper_lib, global_map_lib, outlier_lib and undistort_lib bind their entry points through it.

Test infrastructure: imported only by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs.  The product package never imports this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORC_DIR = os.path.join(ROOT, "oracle")

F_PLANE, F_EDGE, F_EDGE_VEC, F_ODOM_PLANE, F_ODOM_EDGE = 0, 1, 2, 3, 4
(O_MAX_OUTER, O_MAX_INNER, O_HUBER, O_EIG_THRE, O_N_NEIGH, O_CHECK_FOV, O_POINT_PLANE, O_POINT_EDGE, O_COV_TRACE,
 O_DIST_SQ_THR, O_NEARBY_SCAN, O_MIN_MATCH_SQ, O_MIN_PLANE_DIS, O_GF_METHOD, O_GF_RATIO, O_GF_SEED) = range(16)

_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_f64p = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
_u8p = np.ctypeslib.ndpointer(dtype=np.uint8, flags="C_CONTIGUOUS")


def build(force: bool = False) -> None:
    so = os.path.join(ORC_DIR, "liborc.so")
    srcs = [os.path.join(ORC_DIR, f) for f in os.listdir(ORC_DIR) if f.endswith((".hpp", ".cpp"))]
    stale = (not os.path.exists(so)) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)
    if force or stale:
        subprocess.check_call(["make", "-C", ORC_DIR, "liborc.so"], stdout=subprocess.DEVNULL)
    if os.path.isdir("/root/reference") and (force or not os.path.exists(os.path.join(ORC_DIR, "_ref", "libref_knn.so"))):
        subprocess.check_call(["make", "-C", ORC_DIR, "ref"], stdout=subprocess.DEVNULL)


_lib = None
_ref = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(os.path.join(ORC_DIR, "liborc.so"))
        _lib.orc_logdet.restype = C.c_double
        _lib.orc_map_sqrt_info.restype = C.c_double
        _lib.orc_map_sqrt_info.argtypes = [C.c_double]
        _lib.orc_use_ref_tree.restype = C.c_int
        _lib.orc_use_ref_tree.argtypes = [C.c_char_p]
        # the keyframe store (mapper_lib.Mapper) and the global map hand out handles
        _lib.orc_mapper_create.restype = C.c_void_p
        _lib.orc_mapper_create.argtypes = [C.c_double] * 5 + [C.c_float] * 2
        _lib.orc_global_map.restype = C.c_void_p
        _lib.orc_global_map.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_double, C.c_float, C.c_void_p]
        _lib.orc_global_map_read.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.orc_global_map_free.argtypes = [C.c_void_p]
        _lib.orc_set_threads(1)  # serial, like the reference's mapper; bench's all-cores arm raises it explicitly
    return _lib


def ref_lib():
    """oracle/_ref/libref_knn.so — the reference's own nanoflann, or None when not built."""
    global _ref
    if _ref is None:
        p = os.path.join(ORC_DIR, "_ref", "libref_knn.so")
        if not os.path.exists(p):
            return None
        _ref = C.CDLL(p)
    return _ref


def set_threads(n: int) -> None:
    lib().orc_set_threads(int(n))


def cloud(a) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.float32)
    assert a.ndim == 2 and a.shape[1] == 4
    return a


def default_opts() -> np.ndarray:
    o = np.zeros(lib().orc_num_opts(), dtype=np.float64)
    lib().orc_default_opts(o.ctypes.data_as(C.c_void_p))
    return o


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def map_sqrt_info(cov_trace: float) -> float:
    return float(lib().orc_map_sqrt_info(C.c_double(cov_trace)))


def knn(map_, q, k, brute=False):
    map_, q = cloud(map_), cloud(q)
    idx = np.empty((q.shape[0], k), np.int32)
    sqd = np.empty((q.shape[0], k), np.float32)
    lib().orc_knn(_p(map_), map_.shape[0], _p(q), q.shape[0], k, _p(idx), _p(sqd), int(brute))
    return idx, sqd


def ref_knn(map_, q, k):
    r = ref_lib()
    assert r is not None
    map_, q = cloud(map_), cloud(q)
    idx = np.empty((q.shape[0], k), np.int32)
    sqd = np.empty((q.shape[0], k), np.float32)
    r.ref_knn(_p(map_), map_.shape[0], _p(q), q.shape[0], k, _p(idx), _p(sqd))
    return idx, sqd


def eig3f(A):
    A = np.ascontiguousarray(A, np.float32).reshape(9)
    w = np.empty(3, np.float32)
    V = np.empty(9, np.float32)
    lib().orc_eig3f(_p(A), _p(w), _p(V))
    return w, V.reshape(3, 3)


def lsq_plane(A):
    A = np.ascontiguousarray(A, np.float32)
    n = np.empty(3, np.float32)
    ok = lib().orc_lsq_plane(_p(A), A.shape[0], _p(n))
    return bool(ok), n


def eig_sym(A):
    A = np.ascontiguousarray(A, np.float64)
    N = A.shape[0]
    w = np.empty(N)
    V = np.empty((N, N))
    lib().orc_eig_sym(N, _p(A), _p(w), _p(V))
    return w, V


def huber(a, s):
    out = np.empty(2)
    lib().orc_huber(C.c_double(a), C.c_double(s), _p(out))
    return out


def associate(pts, pose7):
    pts = cloud(pts)
    out = np.empty_like(pts)
    pose7 = np.ascontiguousarray(pose7, np.float64)
    lib().orc_associate(_p(pts), pts.shape[0], _p(pose7), _p(out))
    return out


def plus(x7, d6, V=None):
    x7 = np.ascontiguousarray(x7, np.float64)
    d6 = np.ascontiguousarray(d6, np.float64)
    out = np.empty(7)
    Vp = None if V is None else _p(np.ascontiguousarray(V, np.float64))
    lib().orc_plus(_p(x7), _p(d6), Vp, _p(out))
    return out


def eval_degeneracy(H, thre):
    H = np.ascontiguousarray(H, np.float64)
    V = np.empty((6, 6))
    eig = np.empty(6)
    flag = C.c_int(0)
    lib().orc_eval_degeneracy(_p(H), C.c_double(thre), _p(V), _p(eig), C.byref(flag))
    return V, eig, bool(flag.value)


def voxel_grid(pts, leaf, intensity_last=False):
    pts = cloud(pts)
    out = np.empty_like(pts)
    n = C.c_int(0)
    ok = lib().orc_voxel_grid(_p(pts), pts.shape[0], C.c_float(leaf), int(intensity_last), _p(out), C.byref(n))
    return out[: n.value].copy(), bool(ok)


def extract_cloud(pts, scan_start, scan_end):
    pts = cloud(pts)
    n = pts.shape[0]
    ss = np.ascontiguousarray(scan_start, np.int32)
    se = np.ascontiguousarray(scan_end, np.int32)
    bufs = [np.empty((n, 4), np.float32) for _ in range(4)]
    counts = np.zeros(4, np.int32)
    curv = np.zeros(n, np.float32)
    label = np.zeros(n, np.int32)
    lib().orc_extract_cloud(_p(pts), n, _p(ss), _p(se), ss.shape[0], _p(bufs[0]), _p(bufs[1]), _p(bufs[2]), _p(bufs[3]),
                            _p(counts), _p(curv), _p(label))
    keys = ["corner_points_sharp", "corner_points_less_sharp", "surf_points_flat", "surf_points_less_flat"]
    out = {k: bufs[i][: counts[i]].copy() for i, k in enumerate(keys)}
    out["laser_cloud"] = pts
    out["curvature"] = curv
    out["label"] = label
    return out


def match_from_map(kind, map_, data, pose7, n_neigh=5, check_fov=False, opts=None):
    map_, data = cloud(map_), cloud(data)
    opts = default_opts() if opts is None else np.ascontiguousarray(opts, np.float64)
    pose7 = np.ascontiguousarray(pose7, np.float64)
    n = data.shape[0]
    valid = np.zeros(n, np.uint8)
    coeffs = np.zeros((n, 6))
    nn = np.zeros((n, n_neigh), np.int32)
    lib().orc_match_from_map(ord(kind), _p(map_), map_.shape[0], _p(data), n, _p(pose7), n_neigh, int(check_fov), _p(opts),
                             _p(valid), _p(coeffs), _p(nn))
    return valid.astype(bool), coeffs, nn


def match_from_scan(kind, scan, data, pose7, opts=None, with_nn3=False):
    """Features in query order: (query index [cnt], coeffs [cnt, 6]) and, with_nn3, [closest, ind2, ind3] [cnt, 3]
    (ind3 = -1 for 'c')."""
    scan, data = cloud(scan), cloud(data)
    opts = default_opts() if opts is None else np.ascontiguousarray(opts, np.float64)
    pose7 = np.ascontiguousarray(pose7, np.float64)
    n = data.shape[0]
    fidx = np.zeros(max(n, 1), np.int32)
    coeffs = np.zeros((max(n, 1), 6))
    nn3 = np.zeros((max(n, 1), 3), np.int32)
    cnt = lib().orc_match_from_scan_nn3(ord(kind), _p(scan), scan.shape[0], _p(data), n, _p(pose7), _p(opts), _p(fidx),
                                        _p(coeffs), _p(nn3))
    if with_nn3:
        return fidx[:cnt].copy(), coeffs[:cnt].copy(), nn3[:cnt].copy()
    return fidx[:cnt].copy(), coeffs[:cnt].copy()


def factor_eval(kind, point, coeffs, sqrt_info, x, want_jac=True):
    point = np.ascontiguousarray(point, np.float64)
    c6 = np.zeros(6)
    c6[: len(coeffs)] = coeffs
    x21 = np.zeros(21)
    xx = np.ascontiguousarray(x, np.float64).reshape(-1)
    x21[: xx.shape[0]] = xx
    r = np.zeros(3)
    J = np.zeros(63)
    lib().orc_factor_eval(kind, _p(point), _p(c6), C.c_double(sqrt_info), _p(x21), _p(r), _p(J) if want_jac else None)
    return r, J


def normal_eq(types, points, coeffs, sqrt_info, huber_a, x7):
    types = np.ascontiguousarray(types, np.uint8)
    points = np.ascontiguousarray(points, np.float64)
    coeffs = np.ascontiguousarray(coeffs, np.float64)
    x7 = np.ascontiguousarray(x7, np.float64)
    H = np.empty((6, 6))
    g = np.empty(6)
    cost = C.c_double(0)
    lib().orc_normal_eq(_p(types), _p(points), _p(coeffs), types.shape[0], C.c_double(sqrt_info), C.c_double(huber_a), _p(x7),
                        _p(H), _p(g), C.byref(cost))
    return H, g, cost.value


def scan2map(surf_map, corner_map, surf_scan, corner_scan, pose_init, opts=None):
    sm, cm, ss, cs = cloud(surf_map), cloud(corner_map), cloud(surf_scan), cloud(corner_scan)
    opts = default_opts() if opts is None else np.ascontiguousarray(opts, np.float64)
    pose_init = np.ascontiguousarray(pose_init, np.float64)
    out = np.empty(7)
    stats = np.zeros(16)
    H = np.zeros((6, 6))
    lib().orc_scan2map(_p(sm), sm.shape[0], _p(cm), cm.shape[0], _p(ss), ss.shape[0], _p(cs), cs.shape[0], _p(pose_init),
                       _p(opts), _p(out), _p(stats), _p(H))
    names = ["ran", "n_surf", "n_corner", "lm_iterations", "final_cost", "degenerate", "t_kdtree", "t_match", "t_solver"]
    st = {k: stats[i] for i, k in enumerate(names)}
    st["eig"] = stats[9:15].copy()
    st["H"] = H
    return out, st


def frame(cloud_, scan_start, scan_end, surf_map, corner_map, pose_init, opts=None, corner_leaf=0.2, surf_leaf=0.4):
    """extractCloud -> downsampleCurrentScan -> scan2MapOptimization on the CPU (one LiDAR sweep)."""
    pts, sm, cm = cloud(cloud_), cloud(surf_map), cloud(corner_map)
    ss = np.ascontiguousarray(scan_start, np.int32)
    se = np.ascontiguousarray(scan_end, np.int32)
    opts = default_opts() if opts is None else np.ascontiguousarray(opts, np.float64)
    pose_init = np.ascontiguousarray(pose_init, np.float64)
    out = np.empty(7)
    stats = np.zeros(20)
    lib().orc_frame(_p(pts), pts.shape[0], _p(ss), _p(se), ss.shape[0], _p(sm), sm.shape[0], _p(cm), cm.shape[0],
                    C.c_float(corner_leaf), C.c_float(surf_leaf), _p(pose_init), _p(opts), _p(out), _p(stats))
    names = ["ran", "n_surf", "n_corner", "lm_iterations", "final_cost", "degenerate", "t_kdtree", "t_match", "t_solver"]
    st = {k: stats[i] for i, k in enumerate(names)}
    st.update(t_extract=stats[16], t_downsample=stats[17], n_surf_in=int(stats[18]), n_corner_in=int(stats[19]))
    return out, st


def frame_multi(cloud_, scan_start, scan_end, n_lidars, ext7, surf_map, corner_map, pose_init, opts=None, corner_leaf=0.2, surf_leaf=0.4):
    """Multi-LiDAR frame: per-LiDAR extractCloud -> transformCloudFeature -> merged downsample -> scan2MapOptimization."""
    pts, sm, cm = cloud(cloud_), cloud(surf_map), cloud(corner_map)
    ss = np.ascontiguousarray(scan_start, np.int32)
    se = np.ascontiguousarray(scan_end, np.int32)
    ext = np.ascontiguousarray(ext7, np.float64).reshape(-1)
    opts = default_opts() if opts is None else np.ascontiguousarray(opts, np.float64)
    pose_init = np.ascontiguousarray(pose_init, np.float64)
    out = np.empty(7)
    stats = np.zeros(20)
    lib().orc_frame_multi(_p(pts), pts.shape[0], _p(ss), _p(se), ss.shape[0], n_lidars, _p(ext), _p(sm), sm.shape[0], _p(cm), cm.shape[0],
                          C.c_float(corner_leaf), C.c_float(surf_leaf), _p(pose_init), _p(opts), _p(out), _p(stats))
    names = ["ran", "n_surf", "n_corner", "lm_iterations", "final_cost", "degenerate", "t_kdtree", "t_match", "t_solver"]
    st = {k: stats[i] for i, k in enumerate(names)}
    st.update(t_extract=stats[16], t_downsample=stats[17], n_surf_in=int(stats[18]), n_corner_in=int(stats[19]))
    return out, st


def prepare_multi(cloud_, scan_start, scan_end, n_lidars, ext7, corner_leaf=0.2, surf_leaf=0.4):
    """(corner_ds, surf_ds) of one LiDAR group as they enter scan2MapOptimization."""
    pts = cloud(cloud_)
    ss = np.ascontiguousarray(scan_start, np.int32)
    se = np.ascontiguousarray(scan_end, np.int32)
    ext = np.ascontiguousarray(ext7, np.float64).reshape(-1)
    co, so = np.empty((pts.shape[0], 4), np.float32), np.empty((pts.shape[0], 4), np.float32)
    nc, ns = C.c_int(0), C.c_int(0)
    lib().orc_prepare_multi(_p(pts), pts.shape[0], _p(ss), _p(se), ss.shape[0], n_lidars, _p(ext), C.c_float(corner_leaf), C.c_float(surf_leaf),
                            _p(co), C.byref(nc), _p(so), C.byref(ns))
    return co[:nc.value].copy(), so[:ns.value].copy()


def set_gf_groups(surf_sizes=None, corner_sizes=None):
    """Per-group good-feature selection for the next scan2map calls (None: one selection over the whole scan)."""
    s = np.ascontiguousarray(surf_sizes if surf_sizes is not None else [], np.int32)
    c = np.ascontiguousarray(corner_sizes if corner_sizes is not None else [], np.int32)
    lib().orc_set_gf_groups(int(s.shape[0]), _p(s), _p(c))


def calib_frame(surf_map, corner_map, surf_ref, corner_ref, surf_cal, corner_cal, pivot, pose_i, ext_ref, ext_cal, max_outer=2, max_inner=4,
                huber_a=1.0, surf_map_cal=None, corner_map_cal=None, opts=None):
    """Online extrinsic calibration step (orc_calib_frame).  Returns (pose_i, ext_cal, stats)."""
    e4 = np.zeros((0, 4), np.float32)
    arrs = [cloud(x) if x is not None and len(x) else e4 for x in (surf_map, corner_map, surf_map_cal, corner_map_cal, surf_ref, corner_ref, surf_cal, corner_cal)]
    opts = default_opts() if opts is None else np.ascontiguousarray(opts, np.float64)
    pv = np.ascontiguousarray(pivot, np.float64)
    pi = np.array(pose_i, np.float64)
    er = np.ascontiguousarray(ext_ref, np.float64)
    ec = np.array(ext_cal, np.float64)
    st = np.zeros(4)
    args = []
    for a in arrs:
        args += [_p(a), a.shape[0]]
    lib().orc_calib_frame(*args, _p(pv), _p(pi), _p(er), _p(ec), max_outer, max_inner, C.c_double(huber_a), _p(opts), _p(st))
    return pi, ec, {"lm_iterations": int(st[0]), "final_cost": st[1], "rows": int(st[2]), "termination": int(st[3])}


def good_features_odom(kind, map_pts, scan, pivot, pose_i, ext, gf_ratio, seed, opts=None):
    mp, sc = cloud(map_pts), cloud(scan)
    n = sc.shape[0]
    a, b, e = (np.ascontiguousarray(x, np.float64) for x in (pivot, pose_i, ext))
    opts = default_opts() if opts is None else np.ascontiguousarray(opts, np.float64)
    matched, jaco, sel, H = np.zeros(max(n, 1), np.uint8), np.zeros((max(n, 1), 6)), np.zeros(max(n, 1), np.int32), np.zeros(36)
    ns = C.c_int(0)
    lib().orc_good_features_odom(ord(kind), _p(mp), mp.shape[0], _p(sc), n, _p(a), _p(b), _p(e), C.c_double(gf_ratio), C.c_ulonglong(seed), _p(opts),
                                 _p(matched), _p(jaco), _p(sel), C.byref(ns), _p(H))
    return {"sel": sel[:ns.value].copy(), "H": H.reshape(6, 6), "matched": matched[:n].astype(bool), "jaco": jaco[:n]}


def local_map_build(clouds, pose_local7, leaf):
    clouds = [cloud(x) for x in clouds]
    counts = np.ascontiguousarray([x.shape[0] for x in clouds], np.int32)
    allp = cloud(np.concatenate(clouds))
    pl = np.ascontiguousarray(pose_local7, np.float64).reshape(-1, 7)
    out = np.zeros((allp.shape[0], 4), np.float32)
    no = C.c_int(0)
    lib().orc_local_map_build(len(clouds), _p(allp), _p(counts), _p(pl), C.c_float(leaf), _p(out), C.byref(no))
    return out[:no.value].copy()


def project_cloud(cloud_, vertical_scans, horizon_scans, roi_range=0.5):
    """ImageSegmenter::segmentCloud with segment_flag false: (ring-ordered cloud, scan_start, scan_end)."""
    pts = cloud(cloud_)
    n = pts.shape[0]
    out = np.zeros((max(n, 1), 4), np.float32)
    ss, se = np.zeros(vertical_scans, np.int32), np.zeros(vertical_scans, np.int32)
    no = C.c_int(0)
    lib().orc_project_cloud(_p(pts), n, vertical_scans, horizon_scans, C.c_double(roi_range), _p(out), C.byref(no), _p(ss), _p(se))
    return out[:no.value].copy(), ss, se


def project_pixels(cloud_, vertical_scans, horizon_scans, roi_range=0.5):
    pts = cloud(cloud_)
    pix = np.zeros(max(pts.shape[0], 1), np.int32)
    lib().orc_project_pixels(_p(pts), pts.shape[0], vertical_scans, horizon_scans, C.c_double(roi_range), _p(pix))
    return pix[:pts.shape[0]]


def compound_pose_cov(p1, cov1, p2, cov2):
    """compoundPoseWithCov (method 2): returns (pose7, cov 6x6) of p1 * p2."""
    a, b = np.ascontiguousarray(p1, np.float64), np.ascontiguousarray(p2, np.float64)
    c1, c2 = np.ascontiguousarray(cov1, np.float64).reshape(36), np.ascontiguousarray(cov2, np.float64).reshape(36)
    po, co = np.zeros(7), np.zeros(36)
    lib().orc_compound_pose_cov(_p(a), _p(c1), _p(b), _p(c2), _p(po), _p(co))
    return po, co.reshape(6, 6)


def cloud_uct_associate(cloud_, pose_global, ext, pose_compound, cov_compound, cov_meas, with_ua=True, trace_threshold=200.0):
    """cloudUCTAssociateToMap: returns (points [m,4], cov6 [m,6], trace [m])."""
    pts = cloud(cloud_)
    n = pts.shape[0]
    ext = np.ascontiguousarray(ext, np.float64).reshape(-1, 7)
    pc = np.ascontiguousarray(pose_compound, np.float64).reshape(-1, 7)
    cc = np.ascontiguousarray(cov_compound, np.float64).reshape(-1, 36)
    cm = np.ascontiguousarray(cov_meas, np.float64).reshape(9)
    pg = np.ascontiguousarray(pose_global, np.float64)
    op, oc, ot = np.zeros((n, 4), np.float32), np.zeros((n, 6), np.float32), np.zeros(n, np.float32)
    no = C.c_int(0)
    lib().orc_cloud_uct_associate(_p(pts), n, _p(pg), ext.shape[0], _p(ext), _p(pc), _p(cc), _p(cm), int(with_ua), C.c_double(trace_threshold),
                                  _p(op), _p(oc), _p(ot), C.byref(no))
    return op[:no.value].copy(), oc[:no.value].copy(), ot[:no.value].copy()


def voxel_grid_cov(pts, cov6, trace, leaf, trace_threshold):
    """VoxelGridCovarianceMLOAM<PointIWithCov>::filter: returns (points, cov6, trace, ok)."""
    p = cloud(pts)
    n = p.shape[0]
    c6 = np.ascontiguousarray(cov6, np.float32).reshape(-1, 6)
    tr = np.ascontiguousarray(trace, np.float32)
    op, oc, ot = np.zeros((max(n, 1), 4), np.float32), np.zeros((max(n, 1), 6), np.float32), np.zeros(max(n, 1), np.float32)
    no = C.c_int(0)
    ok = lib().orc_voxel_grid_cov(_p(p), _p(c6), _p(tr), n, C.c_float(leaf), C.c_float(trace_threshold), _p(op), _p(oc), _p(ot), C.byref(no))
    return op[:no.value].copy(), oc[:no.value].copy(), ot[:no.value].copy(), bool(ok)


def use_ref_tree(on: bool = True) -> bool:
    """Timed CPU arm only: build / search the kd-trees with the reference's nanoflann (oracle/_ref/libref_knn.so)."""
    path = os.path.join(ORC_DIR, "_ref", "libref_knn.so")
    L = lib()
    if on and os.path.exists(path):
        return bool(L.orc_use_ref_tree(path.encode()))
    L.orc_use_ref_tree(None)
    return False


def point_uncertainty(pts, pose7, cov_pose, cov_meas):
    pts = cloud(pts)
    pose7 = np.ascontiguousarray(pose7, np.float64)
    cp = np.ascontiguousarray(cov_pose, np.float64).reshape(36)
    cm = np.ascontiguousarray(cov_meas, np.float64).reshape(9)
    out = np.zeros((pts.shape[0], 6), np.float32)
    lib().orc_point_uncertainty(_p(pts), pts.shape[0], _p(pose7), _p(cp), _p(cm), _p(out))
    return out


def scan2map_ua(surf_map, corner_map, surf_scan, surf_cov6, corner_scan, corner_cov6, pose_init, opts=None):
    sm, cm, ss, cs = cloud(surf_map), cloud(corner_map), cloud(surf_scan), cloud(corner_scan)
    sc = np.ascontiguousarray(surf_cov6, np.float32)
    cc = np.ascontiguousarray(corner_cov6, np.float32)
    opts = default_opts() if opts is None else np.ascontiguousarray(opts, np.float64)
    pose_init = np.ascontiguousarray(pose_init, np.float64)
    out = np.empty(7)
    stats = np.zeros(8)
    lib().orc_scan2map_ua(_p(sm), sm.shape[0], _p(cm), cm.shape[0], _p(ss), ss.shape[0], _p(sc), _p(cs), cs.shape[0], _p(cc),
                          _p(pose_init), _p(opts), _p(out), _p(stats))
    return out, {"ran": stats[0], "n_surf": int(stats[1]), "n_corner": int(stats[2]), "lm_iterations": int(stats[3]),
                 "final_cost": stats[4]}


def odom_solve(types, points, coeffs, pivot, pose_i, ext, free_mask, max_it=4, huber_a=1.0, sqrt_info=1.0):
    types = np.ascontiguousarray(types, np.uint8)
    points = np.ascontiguousarray(points, np.float64)
    coeffs = np.ascontiguousarray(coeffs, np.float64)
    pivot = np.ascontiguousarray(pivot, np.float64)
    xi = np.array(pose_i, np.float64)
    xe = np.array(ext, np.float64)
    stats = np.zeros(3)
    lib().orc_odom_solve(types.shape[0], _p(types), _p(points), _p(coeffs), _p(pivot), _p(xi), _p(xe), int(free_mask), int(max_it),
                         C.c_double(huber_a), C.c_double(sqrt_info), _p(stats))
    return xi, xe, {"lm_iterations": int(stats[0]), "final_cost": stats[1], "termination": int(stats[2])}


def track_cloud(prev_less_sharp, prev_less_flat, cur_sharp, cur_flat, pose_ini, opts=None):
    a, b, c, d = cloud(prev_less_sharp), cloud(prev_less_flat), cloud(cur_sharp), cloud(cur_flat)
    if opts is None:
        opts = default_opts()
        opts[O_MAX_OUTER], opts[O_MAX_INNER] = 2, 4
    opts = np.ascontiguousarray(opts, np.float64)
    pose_ini = np.ascontiguousarray(pose_ini, np.float64)
    out = np.empty(7)
    stats = np.zeros(3)
    lib().orc_track_cloud(_p(a), a.shape[0], _p(b), b.shape[0], _p(c), c.shape[0], _p(d), d.shape[0], _p(pose_ini), _p(opts),
                          _p(out), _p(stats))
    return out, {"n_corner": int(stats[0]), "n_surf": int(stats[1]), "lm_iterations": int(stats[2])}


GF_WO, GF_RND, GF_FPS, GF_GD = 0, 1, 2, 3


def good_features(kind, map_pts, scan, pose7, method, gf_ratio, seed, cov6=None, default_trace=0.0075, n_neigh=5, opts=None):
    """ActiveFeatureSelection::goodFeatureMatching for one feature set (explicit seed).  Returns a dict with
    matched (bool[n]), jaco (n,6), sel (int[], selection order), H (6,6)."""
    import ctypes as C

    mp, sc = cloud(map_pts), cloud(scan)
    n = sc.shape[0]
    pose7 = np.ascontiguousarray(pose7, np.float64)
    cv = None if cov6 is None else np.ascontiguousarray(cov6, np.float32)
    op = None if opts is None else np.ascontiguousarray(opts, np.float64)
    matched = np.zeros(max(n, 1), np.uint8)
    jaco = np.zeros((max(n, 1), 6))
    sel = np.zeros(max(n, 1), np.int32)
    n_sel = C.c_int(0)
    H = np.zeros((6, 6))
    lib().orc_good_features(ord(kind), _p(mp), mp.shape[0], _p(sc), n, _p(cv), C.c_double(default_trace), _p(pose7), int(method),
                            C.c_double(gf_ratio), C.c_ulonglong(seed), int(n_neigh), _p(op), _p(matched), _p(jaco), _p(sel),
                            C.byref(n_sel), _p(H))
    return {"matched": matched[:n].astype(bool), "jaco": jaco[:n], "sel": sel[: n_sel.value].copy(), "H": H}


def gf_select(method, gf_ratio, seed, matched, jaco, xyz4):
    import ctypes as C

    matched = np.ascontiguousarray(matched, np.uint8)
    jaco = np.ascontiguousarray(jaco, np.float64)
    xyz4 = cloud(xyz4)
    n = matched.shape[0]
    sel = np.zeros(max(n, 1), np.int32)
    n_sel = C.c_int(0)
    H = np.zeros((6, 6))
    lib().orc_gf_select(int(method), C.c_double(gf_ratio), C.c_ulonglong(seed), n, _p(matched), _p(jaco), _p(xyz4), _p(sel), C.byref(n_sel), _p(H))
    return sel[: n_sel.value].copy(), H

"""ctypes binding of libmloam_b200.so (C ABI: include/mloam_b200.h).

Plumbing for tests/ and bench.py only — the product is the shared library and the C++ host shim under
m-loam_b200/host/.  There is NO CPU fallback: importing works anywhere (so the symbol table can be checked
on a CPU box), but creating a Context without an H100 raises.

The directory name carries a hyphen, so load it with tests/conftest.py's `load_mloam()` (importlib) or
    importlib.util.spec_from_file_location("mloam_b200", ".../m-loam_b200/__init__.py")
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.environ.get("MLOAM_LIB", os.path.join(HERE, "libmloam_b200.so"))

MAP_CORNER, MAP_SURF, MAP_SCAN_CORNER, MAP_SCAN_SURF = 0, 1, 2, 3
E_NO_DEVICE = -2

# every entry point include/mloam_b200.h declares
ABI_SYMBOLS = [
    "mloam_default_params", "mloam_ctx_create", "mloam_ctx_destroy", "mloam_set_params", "mloam_set_stream", "mloam_sync",
    "mloam_last_error", "mloam_version", "mloam_launch_count", "mloam_profile_enable", "mloam_profile_get",
    "mloam_profile_reset", "mloam_project_cloud", "mloam_frame_set_next", "mloam_frame_set_next_device", "mloam_extract_features", "mloam_extract_debug", "mloam_voxel_downsample", "mloam_map_build",
    "mloam_map_build_device", "mloam_map_size", "mloam_knn", "mloam_match_from_map", "mloam_factor_evaluate",
    "mloam_normal_equations", "mloam_pose_plus", "mloam_scan2map", "mloam_scan2map_device", "mloam_frame",
    "mloam_frame_device", "mloam_set_extrinsic", "mloam_set_lidars", "mloam_calib_frame", "mloam_compound_pose_cov", "mloam_cloud_uct_associate", "mloam_voxel_downsample_cov", "mloam_submap_assemble", "mloam_good_features_odom", "mloam_local_map_build", "mloam_match_from_scan", "mloam_track_cloud", "mloam_odom_solve", "mloam_point_uncertainty", "mloam_scan2map_ua", "mloam_good_features", "mloam_comm_unique_id", "mloam_comm_init", "mloam_comm_destroy", "mloam_comm_p2p_export", "mloam_comm_p2p_init", "mloam_comm_p2p_reset",
    "mloam_set_uncertainty", "mloam_pose_covariance", "mloam_frame_scan",
    "mloam_keyframes_init", "mloam_keyframe_save", "mloam_keyframe_submap", "mloam_keyframe_query", "mloam_keyframe_scan",
    "mloam_cal_timestamp", "mloam_set_front_end", "mloam_front_end", "mloam_frame_raw", "mloam_frame_raw_device", "mloam_frame_set_next_raw",
    "mloam_frame_set_next_raw_device",
]


class Params(C.Structure):
    _fields_ = [
        ("n_scans", C.c_int), ("distance_sq_threshold", C.c_float), ("nearby_scan", C.c_float),
        ("min_match_sq_dis", C.c_float), ("min_plane_dis", C.c_float), ("n_neigh", C.c_int), ("check_fov", C.c_int),
        ("point_plane_factor", C.c_int), ("point_edge_factor", C.c_int), ("huber_a", C.c_double), ("eig_thre", C.c_double),
        ("cov_trace", C.c_double), ("max_outer", C.c_int), ("max_inner", C.c_int), ("map_cell", C.c_float),
        ("corner_leaf", C.c_float), ("surf_leaf", C.c_float), ("gf_method", C.c_int), ("gf_ratio", C.c_float), ("gf_seed", C.c_uint),
        ("max_ring_points", C.c_int), ("reserved", C.c_int * 4),
    ]


class SolveStats(C.Structure):
    _fields_ = [
        ("ran", C.c_int), ("n_surf", C.c_int), ("n_corner", C.c_int), ("lm_iterations", C.c_int), ("degenerate", C.c_int),
        ("termination", C.c_int), ("final_cost", C.c_double), ("eig", C.c_double * 6), ("H", C.c_double * 36),
        ("n_surf_in", C.c_int), ("n_corner_in", C.c_int), ("reserved", C.c_int * 6),
    ]

    def as_dict(self):
        return _Stats(self)


class _Stats(dict):
    """Solve statistics as a dict; the two array entries ("eig", "H") are materialised on first access (a per-frame call
    should not pay for arrays nobody reads)."""

    def __init__(self, st: "SolveStats"):
        super().__init__(ran=st.ran, n_surf=st.n_surf, n_corner=st.n_corner, lm_iterations=st.lm_iterations, degenerate=st.degenerate,
                         termination=st.termination, final_cost=st.final_cost, n_surf_in=st.n_surf_in, n_corner_in=st.n_corner_in)
        self._st = st

    def __missing__(self, key):
        if key == "eig":
            v = np.array(self._st.eig[:])
        elif key == "H":
            v = np.array(self._st.H[:]).reshape(6, 6)
        else:
            raise KeyError(key)
        self[key] = v
        return v

    def __contains__(self, key):
        return key in ("eig", "H") or dict.__contains__(self, key)


class Features(C.Structure):
    _fields_ = [
        ("corner_points_sharp", C.c_void_p), ("corner_points_less_sharp", C.c_void_p), ("surf_points_flat", C.c_void_p),
        ("surf_points_less_flat", C.c_void_p), ("n_sharp", C.c_int), ("n_less_sharp", C.c_int), ("n_flat", C.c_int),
        ("n_less_flat", C.c_int), ("cap", C.c_int),
    ]


def build(force: bool = False) -> str:
    """Compile libmloam_b200.so for sm_90a in-tree (nvcc cross-compiles without a GPU)."""
    srcs = []
    for d in (os.path.join(HERE, "csrc"), os.path.join(ROOT, "include")):
        srcs += [os.path.join(d, f) for f in os.listdir(d) if f.endswith((".cu", ".cuh", ".h"))]
    stale = (not os.path.exists(LIB_PATH)) or any(os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in srcs)
    if force or stale:
        if not os.path.exists("/usr/local/cuda/bin/nvcc"):
            raise RuntimeError("libmloam_b200.so is missing/stale and nvcc is not available to build it")
        subprocess.check_call(["make", "-C", HERE, "-j8"], stdout=subprocess.DEVNULL)
    return LIB_PATH


_lib = None


def lib():
    """Load the shared library (RuntimeError if it has not been built — there is no fallback path)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'`")
        _lib = C.CDLL(LIB_PATH)
        _lib.mloam_last_error.restype = C.c_char_p
        _lib.mloam_version.restype = C.c_char_p
        _lib.mloam_launch_count.restype = C.c_longlong
    return _lib


def default_params() -> Params:
    p = Params()
    lib().mloam_default_params(C.byref(p))
    return p


def _cloud(a) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.float32)
    assert a.ndim == 2 and a.shape[1] == 4, a.shape
    return a


def _p(a):
    # c_void_p built from the buffer address: several times cheaper than ndarray.ctypes.data_as on a per-frame call path
    return None if a is None else C.c_void_p(a.__array_interface__["data"][0])


class MloamError(RuntimeError):
    pass


class Context:
    """One CUDA device + stream + arenas (mloam_ctx_t)."""

    def __init__(self, device: int = 0, params: Params | None = None):
        self._h = C.c_void_p()
        self.params = params if params is not None else default_params()
        rc = lib().mloam_ctx_create(device, C.byref(self.params), C.byref(self._h))
        if rc != 0:
            raise MloamError(f"mloam_ctx_create failed ({rc}): an H100 (sm_90a) device is required, there is no CPU path")

    def close(self):
        if self._h:
            lib().mloam_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise MloamError(f"mloam error {rc}: {lib().mloam_last_error(self._h).decode()}")

    def set_params(self, **kw):
        for k, v in kw.items():
            setattr(self.params, k, v)
        self._ck(lib().mloam_set_params(self._h, C.byref(self.params)))

    def set_stream(self, cuda_stream_ptr: int):
        self._ck(lib().mloam_set_stream(self._h, C.c_void_p(cuda_stream_ptr)))

    def sync(self):
        self._ck(lib().mloam_sync(self._h))

    def launch_count(self) -> int:
        return int(lib().mloam_launch_count(self._h))

    def profile(self, on: bool):
        self._ck(lib().mloam_profile_enable(self._h, int(on)))

    def profile_reset(self):
        self._ck(lib().mloam_profile_reset(self._h))

    def profile_get(self, name: str):
        ms, cnt = C.c_double(0), C.c_longlong(0)
        self._ck(lib().mloam_profile_get(self._h, name.encode(), C.byref(ms), C.byref(cnt)))
        return ms.value, cnt.value

    # ---- maps / kNN
    def map_build(self, slot: int, pts, cell: float = 0.0):
        pts = _cloud(pts)
        self._ck(lib().mloam_map_build(self._h, slot, _p(pts), pts.shape[0], C.c_float(cell)))

    def map_build_device(self, slot: int, d_ptr: int, m: int, cell: float = 0.0):
        self._ck(lib().mloam_map_build_device(self._h, slot, C.c_void_p(d_ptr), m, C.c_float(cell)))

    def map_size(self, slot: int) -> int:
        return int(lib().mloam_map_size(self._h, slot))

    def knn(self, slot: int, q, k: int, max_sqdist: float, pose7=None):
        q = _cloud(q)
        idx = np.empty((q.shape[0], k), np.int32)
        sqd = np.empty((q.shape[0], k), np.float32)
        pose = None if pose7 is None else np.ascontiguousarray(pose7, np.float64)
        self._ck(lib().mloam_knn(self._h, slot, _p(q), q.shape[0], _p(pose), k, C.c_float(max_sqdist), _p(idx), _p(sqd)))
        return idx, sqd

    def match_from_map(self, slot: int, kind: str, pts, pose7, want_nn: bool = True):
        pts = _cloud(pts)
        n = pts.shape[0]
        pose = np.ascontiguousarray(pose7, np.float64)
        valid = np.zeros(n, np.uint8)
        coeffs = np.zeros((n, 6), np.float64)
        nn = np.zeros((n, self.params.n_neigh), np.int32) if want_nn else None
        self._ck(lib().mloam_match_from_map(self._h, slot, ord(kind), _p(pts), n, _p(pose), _p(valid), _p(coeffs), _p(nn)))
        return valid.astype(bool), coeffs, nn

    # ---- factors / normal equations
    def factor_evaluate(self, kind: int, points, coeffs, params, sqrt_info=None, want_jac: bool = True):
        points = np.ascontiguousarray(points, np.float64).reshape(-1, 3)
        n = points.shape[0]
        cf = np.zeros((n, 6))
        coeffs = np.asarray(coeffs, np.float64).reshape(n, -1)
        cf[:, : coeffs.shape[1]] = coeffs
        rows = 3 if kind == 2 else 1
        cols = 21 if kind >= 3 else 7
        x = np.zeros(21)
        xx = np.ascontiguousarray(params, np.float64).reshape(-1)
        x[: xx.shape[0]] = xx
        si = None if sqrt_info is None else np.ascontiguousarray(np.broadcast_to(sqrt_info, (n,)), np.float64)
        res = np.zeros((n, rows))
        jac = np.zeros((n, rows, cols)) if want_jac else None
        self._ck(lib().mloam_factor_evaluate(self._h, kind, n, _p(points), _p(cf), _p(si), _p(x), _p(res), _p(jac)))
        return res, jac

    def normal_equations(self, types, points, coeffs, sqrt_info, huber_a, pose7):
        types = np.ascontiguousarray(types, np.uint8)
        points = np.ascontiguousarray(points, np.float64)
        coeffs = np.ascontiguousarray(coeffs, np.float64)
        pose = np.ascontiguousarray(pose7, np.float64)
        H, g, cost = np.zeros((6, 6)), np.zeros(6), C.c_double(0)
        self._ck(lib().mloam_normal_equations(self._h, types.shape[0], _p(types), _p(points), _p(coeffs), C.c_double(sqrt_info),
                                              C.c_double(huber_a), _p(pose), _p(H), _p(g), C.byref(cost)))
        return H, g, cost.value

    def pose_plus(self, x7, d6, V=None):
        x7 = np.ascontiguousarray(x7, np.float64)
        d6 = np.ascontiguousarray(d6, np.float64)
        Vp = None if V is None else np.ascontiguousarray(V, np.float64)
        out = np.zeros(7)
        self._ck(lib().mloam_pose_plus(self._h, _p(x7), _p(d6), _p(Vp), _p(out)))
        return out

    # ---- extraction / voxel grid
    def extract_features(self, cloud, scan_start, scan_end):
        cloud = _cloud(cloud)
        n = cloud.shape[0]
        ss = np.ascontiguousarray(scan_start, np.int32)
        se = np.ascontiguousarray(scan_end, np.int32)
        bufs = [np.empty((max(n, 1), 4), np.float32) for _ in range(4)]
        f = Features()
        f.corner_points_sharp, f.corner_points_less_sharp = _p(bufs[0]), _p(bufs[1])
        f.surf_points_flat, f.surf_points_less_flat = _p(bufs[2]), _p(bufs[3])
        f.cap = n
        self._ck(lib().mloam_extract_features(self._h, _p(cloud), n, _p(ss), _p(se), ss.shape[0], C.byref(f)))
        return {"corner_points_sharp": bufs[0][: f.n_sharp].copy(), "corner_points_less_sharp": bufs[1][: f.n_less_sharp].copy(),
                "surf_points_flat": bufs[2][: f.n_flat].copy(), "surf_points_less_flat": bufs[3][: f.n_less_flat].copy(),
                "laser_cloud": cloud}

    def extract_debug(self, n: int):
        curv = np.zeros(n, np.float32)
        label = np.zeros(n, np.int32)
        self._ck(lib().mloam_extract_debug(self._h, _p(curv), _p(label), n))
        return curv, label

    def voxel_downsample(self, pts, leaf: float, intensity_last: bool = False):
        pts = _cloud(pts)
        out = np.empty((max(pts.shape[0], 1), 4), np.float32)
        n = C.c_int(0)
        self._ck(lib().mloam_voxel_downsample(self._h, _p(pts), pts.shape[0], C.c_float(leaf), int(intensity_last), _p(out), C.byref(n)))
        return out[: n.value].copy()

    def debug_stamps(self):
        """MLOAM_STAMP=1: [(label, ns since the frame's first stamp)] of the last frame (graph replay included)."""
        buf = (C.c_ulonglong * 256)()
        n = C.c_int(0)
        self._ck(lib().mloam_debug_stamps(self._h, buf, 256, C.byref(n)))
        lib().mloam_debug_stamp_label.restype = C.c_char_p
        return [(lib().mloam_debug_stamp_label(self._h, i).decode(), int(buf[i]) - int(buf[0])) for i in range(n.value)]

    def project_cloud(self, cloud, vertical_scans: int, horizon_scans: int, roi_range: float = 0.5):
        """ImageSegmenter::segmentCloud with segment_cloud: 0 -> (ring-ordered cloud, scan_start, scan_end)."""
        pts = _cloud(cloud)
        out = np.empty((max(pts.shape[0], 1), 4), np.float32)
        ss, se = np.zeros(max(vertical_scans, 1), np.int32), np.zeros(max(vertical_scans, 1), np.int32)
        n = C.c_int(0)
        self._ck(lib().mloam_project_cloud(self._h, _p(pts), pts.shape[0], int(vertical_scans), int(horizon_scans), C.c_double(roi_range), _p(out),
                                           C.byref(n), _p(ss), _p(se)))
        return out[: n.value].copy(), ss, se

    # ---- raw driver sweeps (removeNaN + calTimestamp + projection on the device)
    def cal_timestamp(self, cloud, time_field: bool = False, scan_period: float = 0.1):
        """removeNaNFromPointCloud + FeatureExtract::calTimestamp of one LiDAR's sweep -> the finite points, intensity = relative time.
        time_field: the timestamp [us] is in the intensity column (PointITimeCloud overload)."""
        pts = _cloud(cloud)
        out = np.empty((max(pts.shape[0], 1), 4), np.float32)
        n = C.c_int(0)
        self._ck(lib().mloam_cal_timestamp(self._h, _p(pts), pts.shape[0], int(time_field), C.c_float(scan_period), _p(out), C.byref(n)))
        return out[: n.value].copy()

    def set_front_end(self, vertical_scans: int, horizon_scans: int, roi_range: float = 0.5, scan_period: float = 0.1, time_field: bool = False):
        self._ck(lib().mloam_set_front_end(self._h, int(vertical_scans), int(horizon_scans), C.c_double(roi_range), C.c_float(scan_period),
                                           int(time_field)))

    def front_end(self, raw, counts):
        """The front end of frame_raw() alone -> (ring-ordered sweep, scan_start, scan_end); the first n_lidars x vertical_scans entries
        of scan_start / scan_end are the sweep's ScanInfo."""
        raw = _cloud(raw)
        cnt = np.ascontiguousarray(counts, np.int32)
        out = np.empty((max(raw.shape[0], 1), 4), np.float32)
        n_rings = 1024
        ss, se = np.zeros(n_rings, np.int32), np.zeros(n_rings, np.int32)
        n = C.c_int(0)
        self._ck(lib().mloam_front_end(self._h, _p(raw), _p(cnt), _p(out), C.byref(n), _p(ss), _p(se)))
        return out[: n.value].copy(), ss, se

    def frame_raw(self, raw, counts, surf_map, corner_map, pose_init7, rebuild_maps: bool = True):
        """mloam_frame on the rig's raw sweeps (concatenated LiDAR-major, counts[l] points of LiDAR l)."""
        raw = _cloud(raw)
        cnt = np.ascontiguousarray(counts, np.int32)
        sm = None if surf_map is None else _cloud(surf_map)
        cm = None if corner_map is None else _cloud(corner_map)
        pi = np.ascontiguousarray(pose_init7, np.float64)
        out = np.zeros(7)
        st = SolveStats()
        self._ck(lib().mloam_frame_raw(self._h, _p(raw), _p(cnt), _p(sm), 0 if sm is None else sm.shape[0], _p(cm),
                                       0 if cm is None else cm.shape[0], int(rebuild_maps), _p(pi), _p(out), C.byref(st)))
        return out, st.as_dict()

    def frame_raw_device(self, d_raw: int, counts, d_surf_map: int, n_surf_map: int, d_corner_map: int, n_corner_map: int, pose_init7,
                         rebuild_maps: bool = True):
        cnt = np.ascontiguousarray(counts, np.int32)
        pi = np.ascontiguousarray(pose_init7, np.float64)
        out = np.zeros(7)
        st = SolveStats()
        self._ck(lib().mloam_frame_raw_device(self._h, C.c_void_p(d_raw), _p(cnt), C.c_void_p(d_surf_map), n_surf_map, C.c_void_p(d_corner_map),
                                              n_corner_map, int(rebuild_maps), _p(pi), _p(out), C.byref(st)))
        return out, st.as_dict()

    def frame_set_next_raw(self, raw, counts):
        """Announce the raw sweeps of the next frame_raw() call (pass the SAME array to it).  None withdraws."""
        if raw is None:
            self._next_keep = None
            self._ck(lib().mloam_frame_set_next_raw(self._h, None, None))
            return
        raw = _cloud(raw)
        cnt = np.ascontiguousarray(counts, np.int32)
        self._next_keep = (raw, cnt)  # must outlive the coming frame call
        self._ck(lib().mloam_frame_set_next_raw(self._h, _p(raw), _p(cnt)))

    def frame_set_next_raw_device(self, d_raw: int, counts):
        cnt = None if d_raw is None else np.ascontiguousarray(counts, np.int32)
        self._ck(lib().mloam_frame_set_next_raw_device(self._h, None if d_raw is None else C.c_void_p(d_raw), _p(cnt)))

    # ---- orchestrators
    def scan2map(self, surf_scan, corner_scan, pose_init7):
        ss, cs = _cloud(surf_scan), _cloud(corner_scan)
        pi = np.ascontiguousarray(pose_init7, np.float64)
        out = np.zeros(7)
        st = SolveStats()
        self._ck(lib().mloam_scan2map(self._h, _p(ss), ss.shape[0], _p(cs), cs.shape[0], _p(pi), _p(out), C.byref(st)))
        return out, st.as_dict()

    def scan2map_device(self, d_surf: int, n_surf: int, d_corner: int, n_corner: int, pose_init7):
        pi = np.ascontiguousarray(pose_init7, np.float64)
        out = np.zeros(7)
        st = SolveStats()
        self._ck(lib().mloam_scan2map_device(self._h, C.c_void_p(d_surf), n_surf, C.c_void_p(d_corner), n_corner, _p(pi), _p(out),
                                             C.byref(st)))
        return out, st.as_dict()

    def frame(self, cloud, scan_start, scan_end, surf_map, corner_map, pose_init7, rebuild_maps: bool = True):
        cloud = _cloud(cloud)
        ss = np.ascontiguousarray(scan_start, np.int32)
        se = np.ascontiguousarray(scan_end, np.int32)
        sm = None if surf_map is None else _cloud(surf_map)
        cm = None if corner_map is None else _cloud(corner_map)
        pi = np.ascontiguousarray(pose_init7, np.float64)
        out = np.zeros(7)
        st = SolveStats()
        self._ck(lib().mloam_frame(self._h, _p(cloud), cloud.shape[0], _p(ss), _p(se), ss.shape[0], _p(sm),
                                   0 if sm is None else sm.shape[0], _p(cm), 0 if cm is None else cm.shape[0], int(rebuild_maps),
                                   _p(pi), _p(out), C.byref(st)))
        return out, st.as_dict()

    def frame_set_next(self, cloud, scan_start, scan_end):
        """Announce the sweep of the next frame() call (host arrays; pass the SAME arrays to that call): it is extracted on a side
        stream while the coming frame is solved.  None withdraws."""
        if cloud is None:
            self._next_keep = None
            self._ck(lib().mloam_frame_set_next(self._h, None, 0, None, None, 0))
            return
        cloud = _cloud(cloud)
        ss = np.ascontiguousarray(scan_start, np.int32)
        se = np.ascontiguousarray(scan_end, np.int32)
        self._next_keep = (cloud, ss, se)  # must outlive the coming frame call
        self._ck(lib().mloam_frame_set_next(self._h, _p(cloud), cloud.shape[0], _p(ss), _p(se), ss.shape[0]))

    def frame_set_next_device(self, d_cloud: int, n: int, d_scan_start: int, d_scan_end: int, n_scans: int):
        self._ck(lib().mloam_frame_set_next_device(self._h, C.c_void_p(d_cloud), n, C.c_void_p(d_scan_start), C.c_void_p(d_scan_end), n_scans))

    def frame_device(self, d_cloud: int, n: int, d_scan_start: int, d_scan_end: int, n_scans: int, d_surf_map: int, n_surf_map: int,
                     d_corner_map: int, n_corner_map: int, pose_init7, rebuild_maps: bool = True):
        pi = np.ascontiguousarray(pose_init7, np.float64)
        out = np.zeros(7)
        st = SolveStats()
        self._ck(lib().mloam_frame_device(self._h, C.c_void_p(d_cloud), n, C.c_void_p(d_scan_start), C.c_void_p(d_scan_end), n_scans,
                                          C.c_void_p(d_surf_map), n_surf_map, C.c_void_p(d_corner_map), n_corner_map,
                                          int(rebuild_maps), _p(pi), _p(out), C.byref(st)))
        return out, st.as_dict()

    def match_from_scan(self, slot: int, kind: str, pts, pose7):
        pts = _cloud(pts)
        n = pts.shape[0]
        pose = np.ascontiguousarray(pose7, np.float64)
        valid = np.zeros(n, np.uint8)
        coeffs = np.zeros((n, 6), np.float64)
        nn3 = np.zeros((n, 3), np.int32)
        self._ck(lib().mloam_match_from_scan(self._h, slot, ord(kind), _p(pts), n, _p(pose), _p(valid), _p(coeffs), _p(nn3)))
        return valid.astype(bool), coeffs, nn3

    def track_cloud(self, prev_less_sharp, prev_less_flat, cur_sharp, cur_flat, pose_ini7):
        a, b, c, d = _cloud(prev_less_sharp), _cloud(prev_less_flat), _cloud(cur_sharp), _cloud(cur_flat)
        pi = np.ascontiguousarray(pose_ini7, np.float64)
        out = np.zeros(7)
        st = SolveStats()
        self._ck(lib().mloam_track_cloud(self._h, _p(a), a.shape[0], _p(b), b.shape[0], _p(c), c.shape[0], _p(d), d.shape[0], _p(pi),
                                         _p(out), C.byref(st)))
        return out, st.as_dict()

    def point_uncertainty(self, pts, pose7, cov_pose, cov_meas):
        pts = _cloud(pts)
        pose = np.ascontiguousarray(pose7, np.float64)
        cp = np.ascontiguousarray(cov_pose, np.float64).reshape(36)
        cm = np.ascontiguousarray(cov_meas, np.float64).reshape(9)
        out = np.zeros((pts.shape[0], 6), np.float32)
        self._ck(lib().mloam_point_uncertainty(self._h, _p(pts), pts.shape[0], _p(pose), _p(cp), _p(cm), _p(out)))
        return out

    def scan2map_ua(self, surf_scan, surf_cov6, corner_scan, corner_cov6, pose_init7):
        ss, cs = _cloud(surf_scan), _cloud(corner_scan)
        sc = np.ascontiguousarray(surf_cov6, np.float32)
        cc = np.ascontiguousarray(corner_cov6, np.float32)
        pi = np.ascontiguousarray(pose_init7, np.float64)
        out = np.zeros(7)
        st = SolveStats()
        self._ck(lib().mloam_scan2map_ua(self._h, _p(ss), ss.shape[0], _p(sc), _p(cs), cs.shape[0], _p(cc), _p(pi), _p(out), C.byref(st)))
        return out, st.as_dict()

    def calib_frame(self, surf_ref, corner_ref, surf_cal, corner_cal, pivot7, pose_i7, ext_ref7, ext_cal7, max_outer: int = 2, max_inner: int = 4,
                    huber_a: float = 1.0, own_cal_maps: bool = False):
        sr, cr, sc, cc = (None if x is None or len(x) == 0 else _cloud(x) for x in (surf_ref, corner_ref, surf_cal, corner_cal))
        n = [0 if x is None else x.shape[0] for x in (sr, cr, sc, cc)]
        pv = np.ascontiguousarray(pivot7, np.float64)
        pi = np.array(pose_i7, np.float64)
        er = np.ascontiguousarray(ext_ref7, np.float64)
        ec = np.array(ext_cal7, np.float64)
        st = SolveStats()
        self._ck(lib().mloam_calib_frame(self._h, _p(sr), n[0], _p(cr), n[1], _p(sc), n[2], _p(cc), n[3], _p(pv), _p(pi), _p(er), _p(ec),
                                         max_outer, max_inner, C.c_double(huber_a), int(own_cal_maps), C.byref(st)))
        return pi, ec, st.as_dict()

    def local_map_build(self, slot: int, clouds, pose_local7, leaf: float, map_cell: float = 0.0):
        clouds = [_cloud(x) for x in clouds]
        counts = np.ascontiguousarray([x.shape[0] for x in clouds], np.int32)
        allp = _cloud(np.concatenate(clouds)) if clouds else np.zeros((0, 4), np.float32)
        pl = np.ascontiguousarray(pose_local7, np.float64).reshape(-1, 7)
        out = np.zeros((max(allp.shape[0], 1), 4), np.float32)
        no = C.c_int(0)
        self._ck(lib().mloam_local_map_build(self._h, slot, len(clouds), _p(allp), _p(counts), _p(pl), C.c_float(leaf), C.c_float(map_cell), _p(out),
                                             C.byref(no)))
        return out[:no.value].copy()

    def good_features_odom(self, slot: int, kind: str, pts, pivot7, pose_i7, ext7, gf_ratio: float, seed: int):
        pts = _cloud(pts)
        n = pts.shape[0]
        a, b, e = (np.ascontiguousarray(x, np.float64) for x in (pivot7, pose_i7, ext7))
        sel = np.zeros(max(n, 1), np.int32)
        n_sel = C.c_int(0)
        H = np.zeros(36)
        matched = np.zeros(max(n, 1), np.uint8)
        jaco = np.zeros((max(n, 1), 6))
        self._ck(lib().mloam_good_features_odom(self._h, slot, ord(kind), _p(pts), n, _p(a), _p(b), _p(e), C.c_double(gf_ratio), C.c_ulonglong(seed),
                                                _p(sel), C.byref(n_sel), _p(H), _p(matched), _p(jaco)))
        return {"sel": sel[:n_sel.value].copy(), "H": H.reshape(6, 6), "matched": matched[:n].astype(bool), "jaco": jaco[:n]}

    # ---- submap assembly with uncertainty
    @staticmethod
    def compound_pose_cov(p1, cov1, p2, cov2):
        a, b = np.ascontiguousarray(p1, np.float64), np.ascontiguousarray(p2, np.float64)
        c1, c2 = np.ascontiguousarray(cov1, np.float64).reshape(36), np.ascontiguousarray(cov2, np.float64).reshape(36)
        po, co = np.zeros(7), np.zeros(36)
        rc = lib().mloam_compound_pose_cov(_p(a), _p(c1), _p(b), _p(c2), _p(po), _p(co))
        if rc != 0:
            raise MloamError(f"mloam_compound_pose_cov: {rc}")
        return po, co.reshape(6, 6)

    def cloud_uct_associate(self, pts, pose_global, ext, pose_compound, cov_compound, cov_meas, with_ua: bool = True, trace_threshold: float = 200.0):
        pts = _cloud(pts)
        n = pts.shape[0]
        ext = np.ascontiguousarray(ext, np.float64).reshape(-1, 7)
        pc = np.ascontiguousarray(pose_compound, np.float64).reshape(-1, 7)
        cc = np.ascontiguousarray(cov_compound, np.float64).reshape(-1, 36)
        cm = np.ascontiguousarray(cov_meas, np.float64).reshape(9)
        pg = np.ascontiguousarray(pose_global, np.float64)
        op, oc, ot = np.zeros((max(n, 1), 4), np.float32), np.zeros((max(n, 1), 6), np.float32), np.zeros(max(n, 1), np.float32)
        no = C.c_int(0)
        self._ck(lib().mloam_cloud_uct_associate(self._h, _p(pts), n, _p(pg), ext.shape[0], _p(ext), _p(pc), _p(cc), _p(cm), int(with_ua),
                                                 C.c_double(trace_threshold), _p(op), _p(oc), _p(ot), C.byref(no)))
        return op[:no.value].copy(), oc[:no.value].copy(), ot[:no.value].copy()

    def voxel_downsample_cov(self, pts, cov6, trace, leaf: float, trace_threshold: float):
        pts = _cloud(pts)
        n = pts.shape[0]
        c6 = np.ascontiguousarray(cov6, np.float32).reshape(-1, 6)
        tr = np.ascontiguousarray(trace, np.float32)
        op, oc, ot = np.zeros((max(n, 1), 4), np.float32), np.zeros((max(n, 1), 6), np.float32), np.zeros(max(n, 1), np.float32)
        no = C.c_int(0)
        self._ck(lib().mloam_voxel_downsample_cov(self._h, _p(pts), _p(c6), _p(tr), n, C.c_float(leaf), C.c_float(trace_threshold), _p(op), _p(oc),
                                                  _p(ot), C.byref(no)))
        return op[:no.value].copy(), oc[:no.value].copy(), ot[:no.value].copy()

    def submap_assemble(self, slot: int, clouds, poses7, ext, pose_compound, cov_compound, cov_meas, leaf: float, with_ua: bool = True,
                        trace_threshold_assoc: float = 200.0, trace_threshold_filter: float = 200.0, map_cell: float = 0.0, want_output: bool = True):
        """clouds: list of [n_k,4] keyframe clouds; poses7 [K,7]; pose_compound [K,L,7]; cov_compound [K,L,36]."""
        clouds = [_cloud(x) for x in clouds]
        counts = np.ascontiguousarray([x.shape[0] for x in clouds], np.int32)
        allp = _cloud(np.concatenate(clouds)) if clouds else np.zeros((0, 4), np.float32)
        n = allp.shape[0]
        poses = np.ascontiguousarray(poses7, np.float64).reshape(-1, 7)
        ext = np.ascontiguousarray(ext, np.float64).reshape(-1, 7)
        pc = np.ascontiguousarray(pose_compound, np.float64).reshape(-1, 7)
        cc = np.ascontiguousarray(cov_compound, np.float64).reshape(-1, 36)
        cm = np.ascontiguousarray(cov_meas, np.float64).reshape(9)
        op = np.zeros((max(n, 1), 4), np.float32) if want_output else None
        oc = np.zeros((max(n, 1), 6), np.float32) if want_output else None
        no = C.c_int(0)
        self._ck(lib().mloam_submap_assemble(self._h, slot, len(clouds), _p(allp), _p(counts), _p(poses), ext.shape[0], _p(ext), _p(pc), _p(cc), _p(cm),
                                             int(with_ua), C.c_double(trace_threshold_assoc), C.c_float(leaf), C.c_float(trace_threshold_filter),
                                             C.c_float(map_cell), _p(op), _p(oc), C.byref(no)))
        if not want_output:
            return no.value
        return op[:no.value].copy(), oc[:no.value].copy()

    def odom_solve(self, types, points, coeffs, pivot7, pose_i7, ext7, free_mask: int, max_iterations: int = 4, huber_a: float = 1.0,
                   sqrt_info: float = 1.0):
        types = np.ascontiguousarray(types, np.uint8)
        points = np.ascontiguousarray(points, np.float64)
        coeffs = np.ascontiguousarray(coeffs, np.float64)
        pv = np.ascontiguousarray(pivot7, np.float64)
        xi, xe = np.array(pose_i7, np.float64), np.array(ext7, np.float64)
        st = SolveStats()
        self._ck(lib().mloam_odom_solve(self._h, types.shape[0], _p(types), _p(points), _p(coeffs), _p(pv), _p(xi), _p(xe), int(free_mask),
                                        int(max_iterations), C.c_double(huber_a), C.c_double(sqrt_info), C.byref(st)))
        return xi, xe, st.as_dict()

    def set_lidars(self, n_lidars: int, ext7=None):
        e = None if ext7 is None else np.ascontiguousarray(ext7, np.float64).reshape(-1)
        self._ck(lib().mloam_set_lidars(self._h, n_lidars, _p(e)))

    def set_uncertainty(self, with_ua: bool, ext_cov=None, cov_meas=None, trace_threshold: float = 0.0):
        """with_ua frames (mloam_set_uncertainty): ext_cov [n_lidars, 6, 6] extrinsic covariances [translation | rotation],
        cov_meas 3x3 COV_MEASUREMENT, trace_threshold TRACE_THRESHOLD_MAPPING.  Call after set_lidars; may be called before every frame."""
        if not with_ua:
            self._ck(lib().mloam_set_uncertainty(self._h, 0, None, None, C.c_double(0.0)))
            return
        ec = np.ascontiguousarray(ext_cov, np.float64).reshape(-1)
        cm = np.ascontiguousarray(cov_meas, np.float64).reshape(9)
        self._ck(lib().mloam_set_uncertainty(self._h, 1, _p(ec), _p(cm), C.c_double(trace_threshold)))

    def pose_covariance(self) -> np.ndarray:
        """pose_wmap_curr.cov_ of the last frame / scan2map solve (6x6, [translation | rotation]; zeros without with_ua)."""
        out = np.zeros(36)
        self._ck(lib().mloam_pose_covariance(self._h, _p(out)))
        return out.reshape(6, 6)

    def frame_scan(self):
        """The down-sampled (with with_ua: gated) scans of the last frame with cov_vec: (surf [n,4], surf_cov6 [n,6], corner, corner_cov6)."""
        ns, nc = C.c_int(0), C.c_int(0)
        self._ck(lib().mloam_frame_scan(self._h, None, None, 0, C.byref(ns), None, None, 0, C.byref(nc)))
        sp, sc = np.zeros((max(ns.value, 1), 4), np.float32), np.zeros((max(ns.value, 1), 6), np.float32)
        cp, cc = np.zeros((max(nc.value, 1), 4), np.float32), np.zeros((max(nc.value, 1), 6), np.float32)
        self._ck(lib().mloam_frame_scan(self._h, _p(sp), _p(sc), sp.shape[0], C.byref(ns), _p(cp), _p(cc), cp.shape[0], C.byref(nc)))
        return sp[:ns.value].copy(), sc[:ns.value].copy(), cp[:nc.value].copy(), cc[:nc.value].copy()

    # ---- keyframe store (saveKeyframe / extractSurroundingKeyFrames on the device)
    def keyframes_init(self, distance_keyframes: float, orientation_keyframes_deg: float, surrounding_kf_radius: float, map_sur_kf_res: float,
                       trace_threshold: float):
        """Empty keyframe store and empty map slots (the first frames fail the map gate)."""
        self._ck(lib().mloam_keyframes_init(self._h, C.c_double(distance_keyframes), C.c_double(orientation_keyframes_deg),
                                            C.c_double(surrounding_kf_radius), C.c_double(map_sur_kf_res), C.c_double(trace_threshold)))

    def keyframe_save(self, pose7=None, cov=None) -> bool:
        """saveKeyframe for the last frame; None: the frame's pose / covariance (zero while <= 10 keyframes).  True when saved."""
        p = None if pose7 is None else np.ascontiguousarray(pose7, np.float64)
        cv = None if cov is None else np.ascontiguousarray(cov, np.float64).reshape(36)
        saved = C.c_int(0)
        self._ck(lib().mloam_keyframe_save(self._h, _p(p), _p(cv), C.byref(saved)))
        return bool(saved.value)

    def keyframe_submap(self, pose_pred7, want_output: bool = False):
        """extractSurroundingKeyFrames at the prediction.  Returns (rebuilt, n_surf, n_corner), plus
        (surf [n,4], surf_cov6, corner, corner_cov6) with want_output."""
        pp = np.ascontiguousarray(pose_pred7, np.float64)
        rb, ns, nc = C.c_int(0), C.c_int(0), C.c_int(0)
        if not want_output:
            self._ck(lib().mloam_keyframe_submap(self._h, _p(pp), C.byref(rb), None, None, 0, C.byref(ns), None, None, 0, C.byref(nc)))
            return bool(rb.value), ns.value, nc.value
        # a filtered map holds at most as many points as all stored keyframes together
        cap = [1, 1]
        for k in range(self.keyframe_query()[0]):
            a, b = C.c_int(0), C.c_int(0)
            self._ck(lib().mloam_keyframe_scan(self._h, k, None, None, None, None, 0, C.byref(a), None, None, 0, C.byref(b)))
            cap[0] += a.value
            cap[1] += b.value
        sp, sc = np.zeros((cap[0], 4), np.float32), np.zeros((cap[0], 6), np.float32)
        cp, cc = np.zeros((cap[1], 4), np.float32), np.zeros((cap[1], 6), np.float32)
        self._ck(lib().mloam_keyframe_submap(self._h, _p(pp), C.byref(rb), _p(sp), _p(sc), cap[0], C.byref(ns), _p(cp), _p(cc), cap[1], C.byref(nc)))
        return bool(rb.value), sp[:ns.value].copy(), sc[:ns.value].copy(), cp[:nc.value].copy(), cc[:nc.value].copy()

    def keyframe_query(self):
        """(keyframe count, surrounding ids in order, ids chosen by the last rebuild's position filter)."""
        nk, ns, nch = C.c_int(0), C.c_int(0), C.c_int(0)
        self._ck(lib().mloam_keyframe_query(self._h, C.byref(nk), None, 0, C.byref(ns), None, 0, C.byref(nch)))
        sur, ch = np.zeros(max(ns.value, 1), np.int32), np.zeros(max(nch.value, 1), np.int32)
        self._ck(lib().mloam_keyframe_query(self._h, C.byref(nk), _p(sur), sur.shape[0], C.byref(ns), _p(ch), ch.shape[0], C.byref(nch)))
        return nk.value, sur[:ns.value].tolist(), ch[:nch.value].tolist()

    def keyframe_scan(self, kf_id: int):
        """Keyframe kf_id as stored: (pose7, cov 6x6, surf [n,4], surf_cov6, corner, corner_cov6)."""
        pose, cov = np.zeros(7), np.zeros(36)
        ns, nc = C.c_int(0), C.c_int(0)
        self._ck(lib().mloam_keyframe_scan(self._h, int(kf_id), None, None, None, None, 0, C.byref(ns), None, None, 0, C.byref(nc)))
        sp, sc = np.zeros((max(ns.value, 1), 4), np.float32), np.zeros((max(ns.value, 1), 6), np.float32)
        cp, cc = np.zeros((max(nc.value, 1), 4), np.float32), np.zeros((max(nc.value, 1), 6), np.float32)
        self._ck(lib().mloam_keyframe_scan(self._h, int(kf_id), _p(pose), _p(cov), _p(sp), _p(sc), sp.shape[0], C.byref(ns), _p(cp), _p(cc),
                                           cp.shape[0], C.byref(nc)))
        return pose, cov.reshape(6, 6), sp[:ns.value].copy(), sc[:ns.value].copy(), cp[:nc.value].copy(), cc[:nc.value].copy()

    def set_extrinsic(self, ext7=None):
        e = None if ext7 is None else np.ascontiguousarray(ext7, np.float64)
        self._ck(lib().mloam_set_extrinsic(self._h, _p(e)))

    # ---- good-feature selection
    def good_features(self, slot: int, kind: str, pts, pose7, method: int, gf_ratio: float, seed: int, cov6=None):
        pts = _cloud(pts)
        n = pts.shape[0]
        pose = np.ascontiguousarray(pose7, np.float64)
        cv = None if cov6 is None else np.ascontiguousarray(cov6, np.float32)
        sel = np.zeros(max(n, 1), np.int32)
        n_sel = C.c_int(0)
        H = np.zeros((6, 6))
        matched = np.zeros(max(n, 1), np.uint8)
        jaco = np.zeros((max(n, 1), 6))
        self._ck(lib().mloam_good_features(self._h, slot, ord(kind), _p(pts), n, _p(cv), _p(pose), int(method), C.c_double(gf_ratio),
                                           C.c_ulonglong(seed), _p(sel), C.byref(n_sel), _p(H), _p(matched), _p(jaco)))
        return {"sel": sel[: n_sel.value].copy(), "H": H, "matched": matched[:n].astype(bool), "jaco": jaco[:n]}

    # ---- multi-GPU
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        rc = lib().mloam_comm_unique_id(buf)
        if rc != 0:
            raise MloamError(f"mloam_comm_unique_id failed ({rc})")
        return buf.raw

    def comm_init(self, nranks: int, rank: int, uid: bytes):
        self._ck(lib().mloam_comm_init(self._h, nranks, rank, C.c_char_p(uid)))

    def comm_p2p_export(self) -> bytes:
        buf = C.create_string_buffer(64)
        self._ck(lib().mloam_comm_p2p_export(self._h, buf))
        return buf.raw

    def comm_p2p_reset(self):
        self._ck(lib().mloam_comm_p2p_reset(self._h))

    def comm_p2p_init(self, nranks: int, rank: int, handles):
        blob = b"".join(handles)
        assert len(blob) == 64 * nranks
        self._ck(lib().mloam_comm_p2p_init(self._h, nranks, rank, C.c_char_p(blob)))

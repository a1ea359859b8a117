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
GLOBAL_MAP_SURROUND, GLOBAL_MAP_SAVE = 0, 1  # mloam_global_map modes: pubGlobalMap, saveGlobalMap
REGISTERED_FULL_RES, REGISTERED_SURF, REGISTERED_CORNER = 0, 1, 2  # mloam_frame_registered clouds (pubPointCloud)
# mloam_cloud_msgs sources: PointXYZI messages (32 B per point), then PointXYZIWithCov messages (48 B per point)
MSG_FULL_RES, MSG_SURF_LAST, MSG_CORNER_LAST, MSG_SURROUND, MSG_GLOBAL_MAP0, MSG_GLOBAL_MAP1 = 0, 1, 2, 3, 4, 5
PCD_KEYFRAMES = 6  # mloam_cloud_pcd's seventh source: pose_keyframes_3d (PointXYZI)
PCD_XYZ, PCD_XYZI, PCD_XYZI_COV = 0, 1, 2  # mloam_pcd_encode layouts
E_NO_DEVICE = -2

# every entry point include/mloam_b200.h declares
ABI_SYMBOLS = [
    "mloam_default_params", "mloam_ctx_create", "mloam_ctx_destroy", "mloam_set_params", "mloam_set_stream", "mloam_sync",
    "mloam_last_error", "mloam_version", "mloam_launch_count", "mloam_profile_enable", "mloam_profile_get",
    "mloam_profile_reset", "mloam_project_cloud", "mloam_frame_set_next", "mloam_frame_set_next_device", "mloam_extract_features", "mloam_extract_debug", "mloam_voxel_downsample", "mloam_map_build",
    "mloam_map_build_device", "mloam_map_size", "mloam_knn", "mloam_match_from_map", "mloam_factor_evaluate",
    "mloam_normal_equations", "mloam_pose_plus", "mloam_scan2map", "mloam_scan2map_device", "mloam_frame",
    "mloam_frame_device", "mloam_set_extrinsic", "mloam_set_lidars", "mloam_calib_frame", "mloam_calib_rig", "mloam_compound_pose_cov", "mloam_cloud_uct_associate", "mloam_voxel_downsample_cov", "mloam_submap_assemble", "mloam_good_features_odom", "mloam_local_map_build", "mloam_match_from_scan", "mloam_track_cloud", "mloam_odom_solve", "mloam_point_uncertainty", "mloam_scan2map_ua", "mloam_good_features", "mloam_comm_unique_id", "mloam_comm_init", "mloam_comm_destroy", "mloam_comm_p2p_export", "mloam_comm_p2p_init", "mloam_comm_p2p_reset",
    "mloam_set_uncertainty", "mloam_pose_covariance", "mloam_frame_scan",
    "mloam_keyframes_init", "mloam_keyframe_save", "mloam_keyframe_submap", "mloam_keyframe_query", "mloam_keyframe_scan",
    "mloam_global_map", "mloam_global_map_read", "mloam_global_map_chosen",
    "mloam_cal_timestamp", "mloam_set_front_end", "mloam_front_end", "mloam_frame_raw", "mloam_frame_raw_device", "mloam_frame_set_next_raw",
    "mloam_frame_set_next_raw_device", "mloam_set_outlier", "mloam_frame_outlier", "mloam_keyframe_outlier",
    "mloam_undistort_poses", "mloam_set_distortion", "mloam_frame_undistort", "mloam_frame_set_next_undistort",
    "mloam_full_hessian", "mloam_set_gf_float", "mloam_set_gf_float_threshold", "mloam_gf_float_report",
    "mloam_set_registered", "mloam_frame_registered", "mloam_frame_registered_device",
    "mloam_set_front_end_layout", "mloam_front_end_msg", "mloam_frame_msg", "mloam_frame_msg_device", "mloam_frame_set_next_msg",
    "mloam_frame_set_next_msg_device", "mloam_cloud_msgs", "mloam_cloud_msgs_device",
    "mloam_pcd_decode", "mloam_pcd_decode_device", "mloam_front_end_pcd", "mloam_frame_pcd", "mloam_frame_pcd_device",
    "mloam_frame_set_next_pcd", "mloam_frame_set_next_pcd_device", "mloam_cloud_pcd", "mloam_cloud_pcd_device", "mloam_pcd_encode",
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


class Pc2Layout(C.Structure):
    """mloam_pc2_layout_t: one driver's PointCloud2 point layout (offset / datatype per lane x, y, z, lane 3; datatype 0: no lane 3)."""
    _fields_ = [("point_step", C.c_int), ("offset", C.c_int * 4), ("datatype", C.c_int * 4), ("is_bigendian", C.c_int)]


class Pc2Msg(C.Structure):
    """mloam_pc2_msg_t: one LiDAR's message (data: host or device bytes)."""
    _fields_ = [("data", C.c_void_p), ("size", C.c_size_t), ("width", C.c_int), ("height", C.c_int), ("row_step", C.c_size_t)]


def pc2_layout(point_step: int, fields, is_bigendian: bool = False) -> Pc2Layout:
    """fields: [(offset, datatype)] of x, y, z and optionally lane 3 (datatype 7 FLOAT32, 8 FLOAT64)."""
    lay = Pc2Layout()
    lay.point_step, lay.is_bigendian = int(point_step), int(bool(is_bigendian))
    for k, (off, dt) in enumerate(fields):
        lay.offset[k], lay.datatype[k] = int(off), int(dt)
    return lay


def _msgs(msgs):
    """msgs: per LiDAR (data, width, height, row_step) with data a host uint8 array, or (ptr, size, width, height, row_step) with a
    device pointer -> a Pc2Msg array."""
    arr = (Pc2Msg * len(msgs))()
    for l, m in enumerate(msgs):
        if len(m) == 4:
            data, width, height, row_step = m
            arr[l].data, arr[l].size = data.__array_interface__["data"][0], data.nbytes
        else:
            ptr, size, width, height, row_step = m
            arr[l].data, arr[l].size = ptr, size
        arr[l].width, arr[l].height, arr[l].row_step = int(width), int(height), int(row_step)
    return arr


class PcdBody(C.Structure):
    """mloam_pcd_t: one PCD file's ASCII body (data: host or device bytes after the DATA line), POINTS, tokens per line, x / y / z token index."""
    _fields_ = [("data", C.c_void_p), ("size", C.c_size_t), ("points", C.c_int), ("tokens", C.c_int), ("index", C.c_int * 3),
                ("reserved", C.c_int)]


def _pcds(bodies):
    """bodies: per file (data, points, tokens, (ix, iy, iz)) with data a host uint8 array or bytes, or (ptr, size, points, tokens, index)
    with a device pointer -> a PcdBody array (host data must outlive the call)."""
    arr = (PcdBody * len(bodies))()
    for f, b in enumerate(bodies):
        if len(b) == 4:
            data, points, tokens, index = b
            if isinstance(data, (bytes, bytearray)):
                data = np.frombuffer(data, np.uint8)
            arr[f].data, arr[f].size = (data.__array_interface__["data"][0] if data.nbytes else None), data.nbytes
        else:
            ptr, size, points, tokens, index = b
            arr[f].data, arr[f].size = ptr, size
        arr[f].points, arr[f].tokens = int(points), int(tokens)
        for k in range(3):
            arr[f].index[k] = int(index[k])
    return arr


class PcdCloud(C.Structure):
    """mloam_pcd_cloud_t: one host cloud for mloam_pcd_encode (pts [count, 4]; cov6 [count, 6] and trace [count] for PCD_XYZI_COV)."""
    _fields_ = [("pts", C.c_void_p), ("cov6", C.c_void_p), ("trace", C.c_void_p), ("count", C.c_int), ("layout", C.c_int)]


def msg_step(source: int) -> int:
    """point_step of a cloud_msgs source: 32 (PointXYZI) or 48 (PointXYZIWithCov)."""
    return 32 if source <= MSG_CORNER_LAST else 48


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


def undistort_poses(pose_rlt7, idx_ref: int, ext7s, estimate_extrinsic: int = 0) -> np.ndarray:
    """mloam_undistort_poses: the pose each LiDAR's features are undistorted with, [n_lidars, 7] ([t q]), from the odometry's relative pose
    of LiDAR idx_ref and the extrinsics [n_lidars, 7] (every LiDAR takes idx_ref's unless estimate_extrinsic == 2)."""
    r = np.ascontiguousarray(pose_rlt7, np.float64).reshape(7)
    e = np.ascontiguousarray(ext7s, np.float64).reshape(-1, 7)
    out = np.zeros_like(e)
    rc = lib().mloam_undistort_poses(_p(r), int(idx_ref), e.shape[0], _p(e), int(estimate_extrinsic), _p(out))
    if rc != 0:
        raise ValueError(f"mloam_undistort_poses: {rc}")
    return out


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
        self.device = device
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
        old = {k: getattr(self.params, k) for k in kw}
        for k, v in kw.items():
            setattr(self.params, k, v)
        rc = lib().mloam_set_params(self._h, C.byref(self.params))
        if rc != 0:  # refused: the context keeps its parameters, and so does this copy of them
            for k, v in old.items():
                setattr(self.params, k, v)
        self._ck(rc)

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

    # ---- the frame entry points: one sweep kind each, from host or device memory
    def _frame(self, fn, sweep, maps, pose_init7, rebuild_maps):
        """fn(ctx, *sweep, *maps, rebuild_maps, pose_init7, pose_out7, stats) -> (pose, stats)."""
        pi = np.ascontiguousarray(pose_init7, np.float64)
        out = np.zeros(7)
        st = SolveStats()
        self._ck(fn(self._h, *sweep, *maps, int(rebuild_maps), _p(pi), _p(out), C.byref(st)))
        return out, st.as_dict()

    def _frame_host(self, fn, sweep, surf_map, corner_map, pose_init7, rebuild_maps):
        sm = None if surf_map is None else _cloud(surf_map)
        cm = None if corner_map is None else _cloud(corner_map)
        maps = (_p(sm), 0 if sm is None else sm.shape[0], _p(cm), 0 if cm is None else cm.shape[0])
        return self._frame(fn, sweep, maps, pose_init7, rebuild_maps)

    def _frame_device(self, fn, sweep, d_surf_map, n_surf_map, d_corner_map, n_corner_map, pose_init7, rebuild_maps):
        return self._frame(fn, sweep, (C.c_void_p(d_surf_map), n_surf_map, C.c_void_p(d_corner_map), n_corner_map), pose_init7, rebuild_maps)

    def _announce(self, fn, keep, *args):
        """A frame_set_next* call.  keep: its host inputs, which the coming frame call reads; held until the next announcement or
        withdrawal (None)."""
        self._next_keep = keep
        self._ck(fn(self._h, *args))

    def _front_end(self, fn, n_pts, *sweep):
        """fn(ctx, *sweep, out, n_out, scan_start, scan_end) -> (ring-ordered sweep, scan_start, scan_end)."""
        out = np.empty((max(n_pts, 1), 4), np.float32)
        ss, se = np.zeros(1024, np.int32), np.zeros(1024, np.int32)
        n = C.c_int(0)
        self._ck(fn(self._h, *sweep, _p(out), C.byref(n), _p(ss), _p(se)))
        return out[: n.value].copy(), ss, se

    def front_end(self, raw, counts):
        """The front end of frame_raw() alone -> (ring-ordered sweep, scan_start, scan_end); the first n_lidars x vertical_scans entries
        of scan_start / scan_end are the sweep's ScanInfo."""
        raw = _cloud(raw)
        cnt = np.ascontiguousarray(counts, np.int32)
        return self._front_end(lib().mloam_front_end, raw.shape[0], _p(raw), _p(cnt))

    def frame_raw(self, raw, counts, surf_map, corner_map, pose_init7, rebuild_maps: bool = True):
        """mloam_frame on the rig's raw sweeps (concatenated LiDAR-major, counts[l] points of LiDAR l)."""
        raw = _cloud(raw)
        cnt = np.ascontiguousarray(counts, np.int32)
        return self._frame_host(lib().mloam_frame_raw, (_p(raw), _p(cnt)), surf_map, corner_map, pose_init7, rebuild_maps)

    def frame_raw_device(self, d_raw: int, counts, d_surf_map: int, n_surf_map: int, d_corner_map: int, n_corner_map: int, pose_init7,
                         rebuild_maps: bool = True):
        cnt = np.ascontiguousarray(counts, np.int32)
        return self._frame_device(lib().mloam_frame_raw_device, (C.c_void_p(d_raw), _p(cnt)), d_surf_map, n_surf_map, d_corner_map,
                                  n_corner_map, pose_init7, rebuild_maps)

    def frame_set_next_raw(self, raw, counts):
        """Announce the raw sweeps of the next frame_raw() call (pass the SAME array to it).  None withdraws."""
        raw = None if raw is None else _cloud(raw)
        cnt = None if raw is None else np.ascontiguousarray(counts, np.int32)
        self._announce(lib().mloam_frame_set_next_raw, (raw, cnt), _p(raw), _p(cnt))

    def frame_set_next_raw_device(self, d_raw: int, counts):
        cnt = None if d_raw is None else np.ascontiguousarray(counts, np.int32)
        self._ck(lib().mloam_frame_set_next_raw_device(self._h, None if d_raw is None else C.c_void_p(d_raw), _p(cnt)))

    # ---- PointCloud2 messages (unpacked on the device, then the raw front end)
    def set_front_end_layout(self, layouts):
        """One Pc2Layout (pc2_layout) per LiDAR of set_lidars."""
        arr = (Pc2Layout * len(layouts))(*layouts)
        self._ck(lib().mloam_set_front_end_layout(self._h, len(layouts), arr))

    def front_end_msg(self, msgs):
        """front_end() on the rig's messages (host bytes, see _msgs) -> (ring-ordered sweep, scan_start, scan_end)."""
        arr = _msgs(msgs)
        return self._front_end(lib().mloam_front_end_msg, sum(int(m.width) * int(m.height) for m in arr), arr)

    def frame_msg(self, msgs, surf_map, corner_map, pose_init7, rebuild_maps: bool = True):
        """frame_raw() on the rig's messages in host memory (see _msgs)."""
        return self._frame_host(lib().mloam_frame_msg, (_msgs(msgs),), surf_map, corner_map, pose_init7, rebuild_maps)

    def frame_msg_device(self, msgs, d_surf_map: int, n_surf_map: int, d_corner_map: int, n_corner_map: int, pose_init7, rebuild_maps: bool = True):
        """frame_raw_device() on the rig's messages in device memory: msgs per LiDAR (ptr, size, width, height, row_step)."""
        return self._frame_device(lib().mloam_frame_msg_device, (_msgs(msgs),), d_surf_map, n_surf_map, d_corner_map, n_corner_map, pose_init7,
                                  rebuild_maps)

    def frame_set_next_msg(self, msgs):
        """Announce the messages of the next frame_msg() call (pass the SAME arrays to it).  None withdraws."""
        self._announce(lib().mloam_frame_set_next_msg, msgs, None if msgs is None else _msgs(msgs))

    def frame_set_next_msg_device(self, msgs):
        self._ck(lib().mloam_frame_set_next_msg_device(self._h, None if msgs is None else _msgs(msgs)))

    # ---- PCD files (ASCII bodies decoded on the device)
    def pcd_decode(self, bodies) -> np.ndarray:
        """mloam_pcd_decode: the files' points (x, y, z, 0) in file order, file after file (bodies: host bytes, see _pcds)."""
        arr = _pcds(bodies)
        out = np.empty((max(sum(max(0, b.points) for b in arr), 1), 4), np.float32)
        self._ck(lib().mloam_pcd_decode(self._h, len(arr), arr, _p(out)))
        return out[: sum(b.points for b in arr)]

    def pcd_decode_device(self, bodies, d_out: int):
        """mloam_pcd_decode_device: bodies in device memory (ptr, size, points, tokens, index) -> d_out (device float4s)."""
        arr = _pcds(bodies)
        self._ck(lib().mloam_pcd_decode_device(self._h, len(arr), arr, C.c_void_p(d_out)))

    def front_end_pcd(self, bodies):
        """front_end() on the rig's ASCII PCD bodies (host bytes, see _pcds) -> (ring-ordered sweep, scan_start, scan_end)."""
        arr = _pcds(bodies)
        return self._front_end(lib().mloam_front_end_pcd, sum(max(0, b.points) for b in arr), arr)

    def frame_pcd(self, bodies, surf_map, corner_map, pose_init7, rebuild_maps: bool = True):
        """frame_raw() on the rig's ASCII PCD bodies in host memory (see _pcds)."""
        return self._frame_host(lib().mloam_frame_pcd, (_pcds(bodies),), surf_map, corner_map, pose_init7, rebuild_maps)

    def frame_pcd_device(self, bodies, d_surf_map: int, n_surf_map: int, d_corner_map: int, n_corner_map: int, pose_init7, rebuild_maps: bool = True):
        """frame_raw_device() on the rig's bodies in device memory: per LiDAR (ptr, size, points, tokens, index)."""
        return self._frame_device(lib().mloam_frame_pcd_device, (_pcds(bodies),), d_surf_map, n_surf_map, d_corner_map, n_corner_map, pose_init7,
                                  rebuild_maps)

    def frame_set_next_pcd(self, bodies):
        """Announce the bodies of the next frame_pcd() call (pass the SAME arrays to it).  None withdraws."""
        self._announce(lib().mloam_frame_set_next_pcd, bodies, None if bodies is None else _pcds(bodies))

    def frame_set_next_pcd_device(self, bodies):
        self._ck(lib().mloam_frame_set_next_pcd_device(self._h, None if bodies is None else _pcds(bodies)))

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
        return self._frame_host(lib().mloam_frame, (_p(cloud), cloud.shape[0], _p(ss), _p(se), ss.shape[0]), surf_map, corner_map, pose_init7,
                                rebuild_maps)

    def frame_set_next(self, cloud, scan_start, scan_end):
        """Announce the sweep of the next frame() call (host arrays; pass the SAME arrays to that call): it is extracted on a side
        stream while the coming frame is solved.  None withdraws."""
        if cloud is None:
            self._announce(lib().mloam_frame_set_next, None, None, 0, None, None, 0)
            return
        cloud = _cloud(cloud)
        ss = np.ascontiguousarray(scan_start, np.int32)
        se = np.ascontiguousarray(scan_end, np.int32)
        self._announce(lib().mloam_frame_set_next, (cloud, ss, se), _p(cloud), cloud.shape[0], _p(ss), _p(se), ss.shape[0])

    def frame_set_next_device(self, d_cloud: int, n: int, d_scan_start: int, d_scan_end: int, n_scans: int):
        self._ck(lib().mloam_frame_set_next_device(self._h, C.c_void_p(d_cloud), n, C.c_void_p(d_scan_start), C.c_void_p(d_scan_end), n_scans))

    def frame_device(self, d_cloud: int, n: int, d_scan_start: int, d_scan_end: int, n_scans: int, d_surf_map: int, n_surf_map: int,
                     d_corner_map: int, n_corner_map: int, pose_init7, rebuild_maps: bool = True):
        sweep = (C.c_void_p(d_cloud), n, C.c_void_p(d_scan_start), C.c_void_p(d_scan_end), n_scans)
        return self._frame_device(lib().mloam_frame_device, sweep, d_surf_map, n_surf_map, d_corner_map, n_corner_map, pose_init7, rebuild_maps)

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

    def calib_rig(self, surf, corner, pivot7, pose_i7, ext7s, idx_ref: int = 0, prior7s=None, prior_pos: float = 0.0, prior_rot: float = 0.0,
                  max_outer: int = 2, max_inner: int = 4, huber_a: float = 1.0, own_cal_maps: bool = False):
        """mloam_calib_rig: surf / corner are per-LiDAR clouds (None or empty: no features).  Returns (pose_i, ext7s [L, 7], stats, rows [L])."""
        L = len(surf)
        if len(corner) != L:
            raise ValueError(f"calib_rig: {L} surf clouds but {len(corner)} corner clouds")
        sc = [np.zeros((0, 4), np.float32) if x is None or len(x) == 0 else _cloud(x) for x in surf]
        cc = [np.zeros((0, 4), np.float32) if x is None or len(x) == 0 else _cloud(x) for x in corner]
        ns = np.array([x.shape[0] for x in sc], np.int32)
        nc = np.array([x.shape[0] for x in cc], np.int32)
        hs = np.ascontiguousarray(np.concatenate(sc), np.float32) if ns.sum() else None
        hc = np.ascontiguousarray(np.concatenate(cc), np.float32) if nc.sum() else None
        pv = np.ascontiguousarray(pivot7, np.float64)
        pi = np.array(pose_i7, np.float64)
        ex = np.array(ext7s, np.float64)
        pr = None if prior7s is None else np.ascontiguousarray(prior7s, np.float64)
        if ex.shape != (L, 7) or (pr is not None and pr.shape != (L, 7)) or pv.shape != (7,) or pi.shape != (7,):
            raise ValueError(f"calib_rig: {L} LiDARs need ext7s / prior7s of shape ({L}, 7) and 7-vector poses")
        rows = np.zeros(L, np.int32)
        st = SolveStats()
        self._ck(lib().mloam_calib_rig(self._h, L, idx_ref, _p(hs), _p(ns), _p(hc), _p(nc), _p(pv), _p(pi), _p(ex), _p(pr), C.c_double(prior_pos),
                                       C.c_double(prior_rot), max_outer, max_inner, C.c_double(huber_a), int(own_cal_maps), C.byref(st), _p(rows)))
        return pi, ex, st.as_dict(), rows

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

    def full_hessian(self, slot: int, kind: str, pts, pose7, cov6=None, H=None, feat_num: int = 0):
        """evalFullHessian for one feature set: returns (H + sum J^T J over the matched features, feat_num + their count).  H None: 1e-6 I."""
        pts = _cloud(pts)
        n = pts.shape[0]
        x = np.ascontiguousarray(pose7, np.float64)
        Hm = (np.eye(6) * 1e-6 if H is None else np.array(H, np.float64)).reshape(36).copy()
        cv = None if cov6 is None else np.ascontiguousarray(cov6, np.float32)
        fn = C.c_int(feat_num)
        self._ck(lib().mloam_full_hessian(self._h, slot, ord(kind), _p(pts), n, _p(cv), _p(x), _p(Hm), C.byref(fn)))
        return Hm.reshape(6, 6), fn.value

    def set_gf_float(self, on: bool, map_deg_thre: float = 0.0):
        """gd_float (needs params.gf_method = 3): the ratio is adapted on the device every 10th solve call."""
        self._ck(lib().mloam_set_gf_float(self._h, int(bool(on)), C.c_float(map_deg_thre)))

    def set_gf_float_threshold(self, map_deg_thre: float):
        self._ck(lib().mloam_set_gf_float_threshold(self._h, C.c_float(map_deg_thre)))

    def gf_float_report(self):
        r, f = C.c_double(0), C.c_double(0)
        t, e, k = C.c_int(0), C.c_int(0), C.c_longlong(0)
        self._ck(lib().mloam_gf_float_report(self._h, C.byref(r), C.byref(f), C.byref(t), C.byref(e), C.byref(k)))
        return {"ratio_cur": r.value, "deg_factor": f.value, "total_feat_num": t.value, "evaluated": bool(e.value), "frame_cnt": k.value}

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

    def set_distortion(self, on: bool, scan_period: float = 0.1):
        """DISTORTION (mloam_set_distortion): motion-compensate each sweep's less-sharp and less-flat features with the pose given by
        frame_undistort before every frame call.  Call after set_lidars."""
        self._ck(lib().mloam_set_distortion(self._h, int(bool(on)), C.c_float(scan_period)))

    def frame_undistort(self, pose7s):
        """The per-LiDAR pose_undist [n_lidars, 7] ([t q], as undistort_poses returns it) of the sweep of the next frame call."""
        p = np.ascontiguousarray(pose7s, np.float64).reshape(-1, 7)
        self._ck(lib().mloam_frame_undistort(self._h, p.shape[0], _p(p)))

    def frame_set_next_undistort(self, pose7s):
        """The per-LiDAR pose_undist [n_lidars, 7] of the sweep announced by the last frame_set_next* call: the look-ahead then undistorts,
        merges and down-samples it while the coming frame is solved, and the call that takes it needs no frame_undistort."""
        p = np.ascontiguousarray(pose7s, np.float64).reshape(-1, 7)
        self._ck(lib().mloam_frame_set_next_undistort(self._h, p.shape[0], _p(p)))

    def set_outlier(self, map_outlier_res: float):
        """The outlier cloud of segment_cloud: 0 (mloam_set_outlier): leaf MAP_OUTLIER_RES > 0 turns it on, 0 off.  Call after set_lidars."""
        self._ck(lib().mloam_set_outlier(self._h, C.c_float(map_outlier_res)))

    def _outlier(self, fn, *lead):
        n = C.c_int(0)
        self._ck(fn(self._h, *lead, None, None, 0, C.byref(n)))
        p, c6 = np.zeros((max(n.value, 1), 4), np.float32), np.zeros((max(n.value, 1), 6), np.float32)
        self._ck(fn(self._h, *lead, _p(p), _p(c6), p.shape[0], C.byref(n)))
        return p[:n.value].copy(), c6[:n.value].copy()

    def frame_outlier(self):
        """laser_cloud_outlier_cov of the last frame: (points [n,4] in the base frame, intensity = laser id; cov6 [n,6])."""
        return self._outlier(lib().mloam_frame_outlier)

    def keyframe_outlier(self, kf_id: int):
        """Keyframe kf_id's stored outlier cloud: (points [n,4], cov6 [n,6])."""
        return self._outlier(lib().mloam_keyframe_outlier, C.c_int(int(kf_id)))

    def set_registered(self, on: bool):
        """pubPointCloud's clouds (mloam_set_registered): every frame call also moves the full-resolution sweep (with the outlier points when
        set_outlier is on), surf_last and corner_last into the map frame with the returned pose."""
        self._ck(lib().mloam_set_registered(self._h, int(bool(on))))

    def frame_registered(self, which: int) -> np.ndarray:
        """Registered cloud `which` (REGISTERED_FULL_RES / _SURF / _CORNER) of the last frame call: [n, 4] float32, intensity as documented."""
        n = C.c_int(0)
        self._ck(lib().mloam_frame_registered(self._h, int(which), None, 0, C.byref(n)))
        p = np.zeros((max(n.value, 1), 4), np.float32)
        self._ck(lib().mloam_frame_registered(self._h, int(which), _p(p), p.shape[0], C.byref(n)))
        return p[:n.value].copy()

    def frame_registered_device(self, which: int):
        """The same cloud as a CUDA tensor [n, 4] float32: a device-to-device copy of the context's buffer, which the next frame call reuses."""
        import torch

        ptr, n = C.c_void_p(), C.c_int(0)
        self._ck(lib().mloam_frame_registered_device(self._h, int(which), C.byref(ptr), C.byref(n)))
        if n.value == 0:
            return torch.zeros((0, 4), dtype=torch.float32, device=f"cuda:{self.device}")

        class _View:  # the context's buffer as a CUDA array, viewed without a copy
            __cuda_array_interface__ = {"shape": (n.value, 4), "typestr": "<f4", "data": (ptr.value, False), "version": 3, "strides": None}

        return torch.as_tensor(_View(), device=f"cuda:{self.device}").clone()

    # ---- the published clouds as sensor_msgs/PointCloud2 data (pcl::toROSMsg on the device)
    @staticmethod
    def _sources(sources):
        src = (C.c_int * len(sources))(*[int(s) for s in sources])
        return src, (C.c_int * len(sources))()

    def cloud_msgs(self, sources, out=None):
        """The PointCloud2 data of each source (MSG_*) as bytes, packed by one launch per call: width x 32 bytes (PointXYZI) or
        width x 48 (PointXYZIWithCov).  out (optional): per source a writable uint8 array (pageable or pinned) the library copies into;
        without it a size query runs first."""
        src, width = self._sources(sources)
        n = len(sources)
        if out is None:
            self._ck(lib().mloam_cloud_msgs(self._h, n, src, (C.c_void_p * n)(), (C.c_size_t * n)(), width))
            out = [np.empty(width[k] * msg_step(s), np.uint8) for k, s in enumerate(sources)]
        ptrs = (C.c_void_p * n)(*[a.__array_interface__["data"][0] if a.nbytes else None for a in out])
        self._ck(lib().mloam_cloud_msgs(self._h, n, src, ptrs, (C.c_size_t * n)(*[a.nbytes for a in out]), width))
        return [out[k][: width[k] * msg_step(s)].tobytes() for k, s in enumerate(sources)]

    def cloud_msgs_device(self, sources):
        """The same messages as CUDA uint8 tensors, cloned from the context's buffer (which the next cloud_msgs* call reuses)."""
        import torch

        src, width = self._sources(sources)
        n = len(sources)
        ptrs = (C.c_void_p * n)()
        self._ck(lib().mloam_cloud_msgs_device(self._h, n, src, ptrs, width))
        res = []
        for k, s in enumerate(sources):
            nb = width[k] * msg_step(s)
            if nb == 0:
                res.append(torch.zeros(0, dtype=torch.uint8, device=f"cuda:{self.device}"))
                continue

            class _View:  # the context's buffer as a CUDA array, viewed without a copy
                __cuda_array_interface__ = {"shape": (nb,), "typestr": "|u1", "data": (ptrs[k], False), "version": 3, "strides": None}

            res.append(torch.as_tensor(_View(), device=f"cuda:{self.device}").clone())
        return res

    # ---- the mapper's clouds and caller clouds as ASCII PCD files (PCDWriter::write on the device)
    def _pcd_host(self, call, n, out):
        """call(h_data, cap_bytes, bytes) with a size query first unless out (per file a writable uint8 array) is given."""
        nb = (C.c_size_t * n)()
        if out is None:
            self._ck(call((C.c_void_p * n)(), (C.c_size_t * n)(), nb))
            out = [np.empty(nb[k], np.uint8) for k in range(n)]
        ptrs = (C.c_void_p * n)(*[a.__array_interface__["data"][0] if a.nbytes else None for a in out])
        self._ck(call(ptrs, (C.c_size_t * n)(*[a.nbytes for a in out]), nb))
        return [out[k][:nb[k]].tobytes() for k in range(n)]

    def cloud_pcd(self, sources, out=None):
        """The ASCII PCD file of each source (MSG_* or PCD_KEYFRAMES) as bytes, written by one launch per call (b"" for an empty
        cloud).  out (optional): per source a writable uint8 array (pageable or pinned) the library copies into."""
        src = (C.c_int * len(sources))(*[int(s) for s in sources])
        return self._pcd_host(lambda h, cap, nb: lib().mloam_cloud_pcd(self._h, len(sources), src, h, cap, nb), len(sources), out)

    def cloud_pcd_device(self, sources):
        """The same files as CUDA uint8 tensors, cloned from the context's buffer (which the next PCD write reuses)."""
        import torch

        n = len(sources)
        src, nb, ptrs = (C.c_int * n)(*[int(s) for s in sources]), (C.c_size_t * n)(), (C.c_void_p * n)()
        self._ck(lib().mloam_cloud_pcd_device(self._h, n, src, ptrs, nb))
        res = []
        for k in range(n):
            if nb[k] == 0:
                res.append(torch.zeros(0, dtype=torch.uint8, device=f"cuda:{self.device}"))
                continue

            class _View:  # the context's buffer as a CUDA array, viewed without a copy
                __cuda_array_interface__ = {"shape": (nb[k],), "typestr": "|u1", "data": (ptrs[k], False), "version": 3, "strides": None}

            res.append(torch.as_tensor(_View(), device=f"cuda:{self.device}").clone())
        return res

    def pcd_encode(self, clouds, out=None):
        """savePCDFileASCII of host clouds: each (layout, pts [n,4]) or (PCD_XYZI_COV, pts, cov6 [n,6], trace [n]) -> the files as bytes."""
        n = len(clouds)
        arr, keep = (PcdCloud * n)(), []
        for k, c in enumerate(clouds):
            layout, pts = int(c[0]), np.ascontiguousarray(c[1], np.float32).reshape(-1, 4)
            keep.append(pts)
            arr[k].pts, arr[k].count, arr[k].layout = _p(pts).value if pts.size else None, pts.shape[0], layout
            if len(c) > 2:
                c6, tr = np.ascontiguousarray(c[2], np.float32).reshape(-1, 6), np.ascontiguousarray(c[3], np.float32).reshape(-1)
                keep += [c6, tr]
                arr[k].cov6, arr[k].trace = _p(c6).value if c6.size else None, _p(tr).value if tr.size else None
        return self._pcd_host(lambda h, cap, nb: lib().mloam_pcd_encode(self._h, n, arr, h, cap, nb), n, out)

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

    # ---- global map of the keyframe store (pubGlobalMap / saveGlobalMap on the device)
    def global_map(self, mode: int, center=None, radius: float = 1000.0, kf_leaf: float = 10.0, leaf: float | None = None):
        """GLOBAL_MAP_SURROUND: (map [n,4], cov6) of the keyframes within `radius` of center (None: the last tested frame position),
        leaf default params.surf_leaf.  GLOBAL_MAP_SAVE: (surf [n,4], surf_cov6, corner [m,4], corner_cov6) of every keyframe, leaf
        default 2 * params.surf_leaf.  The chosen keyframe ids: global_map_chosen()."""
        if leaf is None:
            leaf = self.params.surf_leaf * (2.0 if mode == GLOBAL_MAP_SAVE else 1.0)
        ct = None if center is None else np.ascontiguousarray(center, np.float64)
        nch, n0, n1 = C.c_int(0), C.c_int(0), C.c_int(0)
        self._ck(lib().mloam_global_map(self._h, int(mode), _p(ct), C.c_double(radius), C.c_double(kf_leaf), C.c_float(leaf), C.byref(nch),
                                        C.byref(n0), C.byref(n1)))
        out = []
        for which, n in enumerate((n0.value, n1.value)[:1 if mode == GLOBAL_MAP_SURROUND else 2]):
            p, c6, got = np.zeros((max(n, 1), 4), np.float32), np.zeros((max(n, 1), 6), np.float32), C.c_int(0)
            self._ck(lib().mloam_global_map_read(self._h, which, _p(p), _p(c6), p.shape[0], C.byref(got)))
            out += [p[:got.value], c6[:got.value]]
        return tuple(out)

    def global_map_chosen(self):
        """Keyframe ids the last global_map's position filter chose, in filter order."""
        n = C.c_int(0)
        self._ck(lib().mloam_global_map_chosen(self._h, None, 0, C.byref(n)))
        ids = np.zeros(max(n.value, 1), np.int32)
        self._ck(lib().mloam_global_map_chosen(self._h, _p(ids), ids.shape[0], C.byref(n)))
        return ids[:n.value].tolist()

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

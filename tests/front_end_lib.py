"""Raw driver sweeps for the front-end tests: synthetic sweeps in firing order, the host builds of tests/host/front_end_host.cpp
(the libm restatement of removeNaNFromPointCloud + FeatureExtract::calTimestamp, and csrc/cal_timestamp.cuh compiled for the host),
and the front-end chain the reference runs per LiDAR (estimator.cpp:249-261): calTimestamp -> segmentCloud (segment_cloud: 0)."""
import ctypes as C
import math

import numpy as np

import host_build
import oracle_lib as orc
import synthetic as syn


def host_lib():
    """tests/host/front_end_host.cpp built for the host (host_build)."""
    return host_build.load("front_end_host")


def _run(fn, cloud, time_field, scan_period):
    pts = np.ascontiguousarray(cloud, np.float32).reshape(-1, 4)
    out = np.zeros((max(pts.shape[0], 1), 4), np.float32)
    n = fn(pts.ctypes.data_as(C.c_void_p), pts.shape[0], int(time_field), C.c_float(scan_period), out.ctypes.data_as(C.c_void_p))
    return out[:n].copy()


def cal_timestamp(cloud, time_field=False, scan_period=0.1):
    """The reference loop with libm atan2f: removeNaN + calTimestamp of one LiDAR."""
    return _run(host_lib().ref_cal_timestamp, cloud, time_field, scan_period)


def cal_timestamp_header(cloud, time_field=False, scan_period=0.1):
    """csrc/cal_timestamp.cuh built for the host (the kernels' arithmetic and flip-index formulation)."""
    return _run(host_lib().host_cal_timestamp, cloud, time_field, scan_period)


def front_end(raw, counts, vertical_scans, horizon_scans, roi_range, scan_period=0.1, time_field=False):
    """Per LiDAR calTimestamp + project_cloud, concatenated LiDAR-major with the ScanInfo offset by each LiDAR's start."""
    outs, ss_all, se_all = [], [], []
    base, off = 0, 0
    for c in counts:
        timed = cal_timestamp(raw[off:off + c], time_field, scan_period)
        off += c
        p, ss, se = orc.project_cloud(timed, vertical_scans, horizon_scans, roi_range)
        outs.append(p)
        ss_all.append(np.asarray(ss, np.int32) + base)
        se_all.append(np.asarray(se, np.int32) + base)
        base += p.shape[0]
    return np.concatenate(outs).astype(np.float32), np.concatenate(ss_all), np.concatenate(se_all)


def ring_elevations(vertical_scans):
    """Elevations [rad] at the centres of the projection's rows (image_segmenter.cpp:18-63)."""
    if vertical_scans == 16:
        return np.radians(np.arange(16) * 2.0 - 15.0)
    if vertical_scans == 32:
        res = 41.33 / 31
        return np.radians(-30.67 + (np.arange(32) + 0.5) * res)
    return syn.ring_elevations(64)


def raw_sweep(scene, pose, vertical_scans, horizon, seed, az0=None, time_field=False, ext=None, n_nan=0, max_range=100.0):
    """One LiDAR's raw sweep in FIRING order: column after column (all rings of one azimuth), the azimuth atan2(y, x) decreasing from
    az0 over one revolution (the direction in which calTimestamp's -atan2 grows), driver intensities in [0, 255) — or, with time_field,
    the firing time in microseconds in the intensity column.  n_nan points get a non-finite coordinate."""
    rng = np.random.default_rng(seed)
    if az0 is None:
        az0 = rng.uniform(-math.pi, math.pi)
    T = pose if ext is None else syn.pose_mul(pose, ext)
    R = syn.quat_to_mat(T[3:])
    el = ring_elevations(vertical_scans)
    az = az0 - 2.0 * math.pi * np.arange(horizon) / horizon
    ce, se_ = np.cos(el)[None, :], np.sin(el)[None, :]
    Ds = np.stack([ce * np.cos(az)[:, None], ce * np.sin(az)[:, None], np.broadcast_to(se_, (horizon, vertical_scans))], axis=2).reshape(-1, 3)
    t = syn._cast(scene, T[:3], Ds @ R.T) + rng.normal(0, 0.02, Ds.shape[0])
    keep = (t > 0.5) & (t < max_range)
    P = (Ds * t[:, None]).astype(np.float32)
    col = np.repeat(np.arange(horizon), vertical_scans)
    w = (col * (1e5 / horizon)).astype(np.float32) if time_field else rng.uniform(0, 255, col.shape[0]).astype(np.float32)
    cloud = np.concatenate([P, w[:, None]], 1)[keep]
    if n_nan:
        idx = rng.choice(np.arange(1, cloud.shape[0] - 1), n_nan, replace=False)
        bad = np.array([np.nan, np.inf, -np.inf], np.float32)
        cloud[idx, rng.integers(0, 3, n_nan)] = bad[rng.integers(0, 3, n_nan)]
    return np.ascontiguousarray(cloud, np.float32)

"""Test infrastructure of the keyframe store: bindings of the oracle's mapper state machine (oracle/orc_mapper.cpp in oracle_lib's library:
saveKeyframe with the optional outlier cloud, clearCloud, extractSurroundingKeyFrames and the process() driver), and independent numpy
restatements of the keyframe decision, the radius search, the surrounding-set bookkeeping and the keyframe-position filter."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_lib as orc
import uncertainty_lib as ua  # noqa: F401  (tests reach the covariance generator as ml.ua)

_p = orc._p


def _f64(a, n=None):
    a = np.ascontiguousarray(a, np.float64)
    return a if n is None else a.reshape(n)


class Mapper:
    """The oracle's keyframe store (one per mapper)."""

    def __init__(self, distance_keyframes, orientation_keyframes_deg, radius, sur_kf_res, trace_threshold, surf_leaf=0.4, corner_leaf=0.2):
        self._h = C.c_void_p(orc.lib().orc_mapper_create(distance_keyframes, orientation_keyframes_deg, radius, sur_kf_res, trace_threshold,
                                                     surf_leaf, corner_leaf))

    def close(self):
        if self._h:
            orc.lib().orc_mapper_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_lidars(self, ext7, ext_cov, cov_meas, with_ua: bool):
        e = _f64(ext7).reshape(-1)
        ec = None if ext_cov is None else _f64(ext_cov).reshape(-1)
        cm = None if cov_meas is None else _f64(cov_meas, 9)
        orc.lib().orc_mapper_set_lidars(self._h, e.shape[0] // 7, _p(e), _p(ec), _p(cm), int(with_ua))

    def save(self, pose7, cov, surf, corner, outlier=None):
        """saveKeyframe, with the keyframe's outlier cloud when given: (saved, (distance margin [m], angle margin [deg]))."""
        s, c = orc.cloud(surf), orc.cloud(corner)
        o = None if outlier is None else orc.cloud(np.asarray(outlier, np.float32).reshape(-1, 4))
        m = np.zeros(2)
        r = orc.lib().orc_mapper_save_outlier(self._h, _p(_f64(pose7)), _p(_f64(cov, 36)), _p(s), s.shape[0], _p(c), c.shape[0], _p(o),
                                          0 if o is None else o.shape[0], _p(m))
        return bool(r), (m[0], m[1])

    def submap(self, pred7):
        """extractSurroundingKeyFrames: (rebuilt, min |d2 - radius^2|)."""
        rm = np.zeros(1)
        r = orc.lib().orc_mapper_submap(self._h, _p(_f64(pred7)), _p(rm))
        return bool(r), float(rm[0])

    def query(self):
        """(keyframe count, surrounding ids, chosen ids, surf map size, corner map size)."""
        cnt = np.zeros(5, np.int32)
        orc.lib().orc_mapper_query(self._h, _p(cnt), None, None)
        sur, ch = np.zeros(max(cnt[1], 1), np.int32), np.zeros(max(cnt[2], 1), np.int32)
        orc.lib().orc_mapper_query(self._h, _p(cnt), _p(sur), _p(ch))
        return int(cnt[0]), sur[:cnt[1]].tolist(), ch[:cnt[2]].tolist(), int(cnt[3]), int(cnt[4])

    def maps(self):
        """(surf [n,4], surf_cov6, corner [m,4], corner_cov6)."""
        _, _, _, ns, nc = self.query()
        out = []
        for t, n in ((0, ns), (1, nc)):
            p, c6 = np.zeros((max(n, 1), 4), np.float32), np.zeros((max(n, 1), 6), np.float32)
            orc.lib().orc_mapper_map(self._h, t, _p(p), _p(c6))
            out += [p[:n], c6[:n]]
        return tuple(out)

    def keyframe(self, kf_id: int):
        """pose_keyframes_6d[kf_id]: (pose7, cov 6x6) as saveKeyframe stored them."""
        pose, cov = np.zeros(7), np.zeros(36)
        orc.lib().orc_mapper_keyframe(self._h, int(kf_id), _p(pose), _p(cov))
        return pose, cov.reshape(6, 6)

    def reassoc_differs(self) -> int:
        return int(orc.lib().orc_mapper_reassoc_differs(self._h))

    def process(self, cloud, scan_start, scan_end, odom7, frame_trace_threshold, opts):
        """One process() pass: (pose, cov 6x6, info dict)."""
        pts = orc.cloud(cloud)
        ss, se = np.ascontiguousarray(scan_start, np.int32), np.ascontiguousarray(scan_end, np.int32)
        out, cov, info = np.zeros(7), np.zeros(36), np.zeros(8)
        orc.lib().orc_mapper_process(self._h, _p(pts), pts.shape[0], _p(ss), _p(se), ss.shape[0], _p(_f64(odom7)), C.c_double(frame_trace_threshold),
                                 _p(np.ascontiguousarray(opts, np.float64)), _p(out), _p(cov), _p(info))
        keys = ("rebuilt", "ran", "saved", "dist_margin", "angle_margin", "radius_margin", "n_surf_in", "n_corner_in")
        return out, cov.reshape(6, 6), dict(zip(keys, info.tolist()))


def pose_mul(a, b):
    """Pose::operator* (pose.cpp:110-113) as the oracle's driver evaluates it."""
    out = np.zeros(7)
    orc.lib().orc_mapper_pose_mul(_p(_f64(a)), _p(_f64(b)), _p(out))
    return out


def pose_inv(a):
    out = np.zeros(7)
    orc.lib().orc_mapper_pose_inv(_p(_f64(a)), _p(out))
    return out


# ---------------------------------------------------------------------------------------- independent numpy restatements
def np_keyframe_due(pose7, prev_pt, prev_q, n_keyframes, dist_kf, orient_deg):
    """saveKeyframe's test (:649-653): float PointI distance, Eigen's angularDistance in degrees."""
    if n_keyframes == 0:
        return True
    cur = np.asarray(pose7[:3], np.float64).astype(np.float32)
    d = (cur - np.asarray(prev_pt, np.float32)).astype(np.float32)
    s = np.float32(d[0] * d[0]) + np.float32(d[1] * d[1])
    s = np.float32(s + np.float32(d[2] * d[2]))
    dist = np.sqrt(np.float32(s))
    ax, ay, az, aw = (float(v) for v in pose7[3:])
    bx, by, bz, bw = -prev_q[0], -prev_q[1], -prev_q[2], prev_q[3]
    x = aw * bx + ax * bw + ay * bz - az * by
    y = aw * by + ay * bw + az * bx - ax * bz
    z = aw * bz + az * bw + ax * by - ay * bx
    w = aw * bw - ax * bx - ay * by - az * bz
    ang = 2.0 * np.arctan2(np.sqrt(x * x + y * y + z * z), abs(w)) / np.pi * 180.0
    return bool(float(dist) > dist_kf or ang > orient_deg)


def np_radius_search(pos_f32, q_f32, radius):
    """pcl::KdTreeFLANN::radiusSearch with L2_Simple in float: ids with d2 < (float)radius^2, ascending (d2, id)."""
    p = np.asarray(pos_f32, np.float32)
    q = np.asarray(q_f32, np.float32)
    dd = (p - q[None, :]).astype(np.float32)
    d2 = np.zeros(p.shape[0], np.float32)
    for k in range(3):
        d2 = (d2 + (dd[:, k] * dd[:, k]).astype(np.float32)).astype(np.float32)
    r2 = np.float32(radius * radius)
    ids = np.nonzero(d2 < r2)[0]
    order = np.lexsort((ids, d2[ids]))
    return ids[order].tolist(), d2


def np_bookkeeping(existing, found):
    """:274-323: drop the ids that left (survivors keep their order), append the new ids in search order; returns (set, new ids)."""
    fs = set(found)
    sur = [i for i in existing if i in fs]
    new = [i for i in found if i not in set(sur)]
    return sur + new, new


def np_position_filter(pos_f32, leaf):
    """VoxelGridCovarianceMLOAM<PointI> over the set's positions (intensity = position): one output per voxel in pcl's voxel-index order,
    carrying the LAST listed position of the voxel."""
    p = np.asarray(pos_f32, np.float32)
    inv = np.float32(1.0) / np.float32(leaf)
    mn, mx = p.min(0), p.max(0)
    minb = np.floor(mn * inv).astype(np.int64)
    maxb = np.floor(mx * inv).astype(np.int64)
    div = maxb - minb + 1
    ijk = (np.floor(p * inv) - minb.astype(np.float32)).astype(np.int64)
    idx = ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * div[0] * div[1]
    out = []
    for v in np.unique(idx):
        out.append(int(np.nonzero(idx == v)[0][-1]))
    return out

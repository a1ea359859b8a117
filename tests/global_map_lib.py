"""Test infrastructure of the global map (mloam_global_map): ctypes binding of the oracle's pubGlobalMap / saveGlobalMap restatement
(tests/host/orc_global_map.cpp over oracle/orc_mapper.cpp's keyframe store), compiled on first use into a temporary directory keyed by
the sources' hash (the tree is never written), and an independent composition of the same steps from the oracle's single-step entry
points (radius search, position filter, cloudUCTAssociateToMap, VoxelGridCovarianceMLOAM) in numpy.

The library carries the whole keyframe-store oracle (orc_mapper.cpp is included), and `Mapper` here creates, fills and frees its store
through that same library: a store never crosses from one shared library into another."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import mapper_lib as ml
import oracle_lib as orc
import uncertainty_lib as ua

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host", "orc_global_map.cpp")
SURROUND, SAVE = 0, 1
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
        so = os.path.join(tempfile.gettempdir(), f"mloam_orc_global_map_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["/usr/bin/g++", *ua.CXXFLAGS, "-shared", "-o", tmp, SRC])
            os.replace(tmp, so)
        _lib = C.CDLL(so)
        _lib.orc_global_map.restype = C.c_void_p
        _lib.orc_global_map.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_double, C.c_float, C.c_void_p]
        _lib.orc_global_map_read.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.orc_global_map_free.argtypes = [C.c_void_p]
        _lib.orc_mapper_create.restype = C.c_void_p
        _lib.orc_mapper_create.argtypes = [C.c_double] * 5 + [C.c_float] * 2
        for f in ("orc_mapper_destroy", "orc_mapper_set_lidars", "orc_mapper_save"):
            getattr(_lib, f).argtypes = None
    return _lib


class Mapper:
    """The oracle's keyframe store with saveKeyframe (what mapper_lib.Mapper offers for it), made and used by this module's library, so
    that global_map() runs on it in the library that made it."""

    def __init__(self, distance_keyframes, orientation_keyframes_deg, radius, sur_kf_res, trace_threshold, surf_leaf=0.4, corner_leaf=0.2):
        self._h = C.c_void_p(lib().orc_mapper_create(distance_keyframes, orientation_keyframes_deg, radius, sur_kf_res, trace_threshold,
                                                     surf_leaf, corner_leaf))

    def close(self):
        if self._h:
            lib().orc_mapper_destroy(self._h)
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
        lib().orc_mapper_set_lidars(self._h, e.shape[0] // 7, _p(e), _p(ec), _p(cm), int(with_ua))

    def save(self, pose7, cov, surf, corner):
        """saveKeyframe: (saved, (distance margin [m], angle margin [deg]))."""
        s, c = orc.cloud(surf), orc.cloud(corner)
        m = np.zeros(2)
        r = lib().orc_mapper_save(self._h, _p(np.ascontiguousarray(pose7, np.float64)), _p(np.ascontiguousarray(cov, np.float64).reshape(36)),
                                  _p(s), s.shape[0], _p(c), c.shape[0], _p(m))
        return bool(r), (m[0], m[1])


def global_map(mapper: Mapper, mode: int, center7, radius: float, kf_leaf: float, leaf: float):
    """The oracle's global map of a Mapper's keyframes: (chosen ids, [map 0 points, map 0 cov6, map 1 points, map 1 cov6]).  center7:
    the pose whose float position is the centre (SURROUND; the position the last save tested when the device call passes NULL)."""
    if not isinstance(mapper, Mapper):
        raise TypeError("global_map needs a global_map_lib.Mapper (a store made by this module's library)")
    ct = None if center7 is None else np.ascontiguousarray(center7, np.float64)
    cnt = np.zeros(3, np.int32)
    r = lib().orc_global_map(mapper._h.value, int(mode), _p(ct), float(radius), float(kf_leaf), float(leaf), _p(cnt))
    try:
        ch = np.zeros(max(cnt[0], 1), np.int32)
        out = []
        for which in (0, 1):
            n = int(cnt[1 + which])
            p, c6 = np.zeros((max(n, 1), 4), np.float32), np.zeros((max(n, 1), 6), np.float32)
            lib().orc_global_map_read(r, which, _p(ch), _p(p), _p(c6))
            out += [p[:n], c6[:n]]
        return ch[:cnt[0]].tolist(), out
    finally:
        lib().orc_global_map_free(r)


# ---------------------------------------------------------------------------------------- independent composition
def np_candidates(pos_f32, mode, center_f32=None, radius=None):
    """The keyframes offered to the position filter: radius search order (SURROUND) or id order (SAVE)."""
    if mode == SURROUND:
        return ml.np_radius_search(pos_f32, center_f32, radius)[0]
    return list(range(len(pos_f32)))


def np_chosen(pos_f32, cand, kf_leaf):
    """The position filter over the candidates' positions with intensity = id: the last-listed id of each voxel, in voxel order."""
    if not cand:
        return []
    p = np.asarray(pos_f32, np.float32)[cand]
    return [cand[i] for i in ml.np_position_filter(p, kf_leaf)]


def compose(keyframes, ext7, ext_cov, cov_meas, with_ua, trace_thr, mode, chosen, leaf):
    """keyframes[id] = (pose7, cov 6x6, surf [n,4], corner [m,4]).  Each chosen keyframe's clouds through cloudUCTAssociateToMap with the
    compound of its pose and each extrinsic, concatenated in the mode's order, then VoxelGridCovarianceMLOAM<PointIWithCov>(leaf)."""
    ext7 = np.asarray(ext7, np.float64).reshape(-1, 7)
    L = ext7.shape[0]
    raw = [[], []]
    for i in chosen:
        pose, cov, surf, corner = keyframes[i]
        pc, cc = [], []
        for l in range(L):
            ec = ext_cov[l] if with_ua else np.zeros((6, 6))
            a, b = orc.compound_pose_cov(pose, cov, ext7[l], ec)
            pc.append(a), cc.append(b)
        for t, cl in ((0, surf), (1, corner)):
            if cl.shape[0] == 0:
                continue
            got = orc.cloud_uct_associate(cl, pose, ext7, np.stack(pc), np.stack(cc), cov_meas, with_ua, trace_thr)
            raw[0 if mode == SURROUND else t].append(got)
    out = []
    for parts in raw[:1 if mode == SURROUND else 2]:
        if not parts:
            out += [np.zeros((0, 4), np.float32), np.zeros((0, 6), np.float32)]
            continue
        p, c6, tr, _ = orc.voxel_grid_cov(np.concatenate([x[0] for x in parts]), np.concatenate([x[1] for x in parts]),
                                          np.concatenate([x[2] for x in parts]), leaf, trace_thr)
        out += [p, c6]
    return out

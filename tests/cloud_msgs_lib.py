"""The published clouds as PointCloud2 data (mloam_cloud_msgs*) for the tests and tools/bench_cloud_msgs.py: the host build of
tests/host/cloud_msgs_host.cpp (m-loam_b200/host/mloam_io.hpp packPointCloud2 / packPointCloud2Cov / cloudMsgView), and the cov_trace of
the covariance clouds composed from the oracle's single steps (cloudUCTAssociateToMap, VoxelGridCovarianceMLOAM)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import oracle_lib as orc

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_lib = None


def host_lib():
    """tests/host/cloud_msgs_host.cpp built with g++ into the temporary directory, keyed by the hash of its sources (the tree is never written)."""
    global _lib
    if _lib is None:
        src = os.path.join(HERE, "host", "cloud_msgs_host.cpp")
        io = os.path.join(ROOT, "m-loam_b200", "host")
        h = hashlib.sha256()
        for f in (src, os.path.join(io, "mloam_io.hpp"), os.path.join(ROOT, "include", "mloam_b200.h")):
            with open(f, "rb") as fh:
                h.update(fh.read())
        so = os.path.join(tempfile.gettempdir(), f"mloam_cloud_msgs_host_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            out = subprocess.run(["g++", "-std=c++14", "-O2", "-Wall", "-shared", "-fPIC", "-I" + io, src, "-o", tmp], capture_output=True, text=True)
            assert out.returncode == 0, out.stderr[-3000:]
            os.replace(tmp, so)
        _lib = C.CDLL(so)
    return _lib


def _ptr(a):
    return C.c_void_p(a.__array_interface__["data"][0])


def pack(pts) -> bytes:
    """packPointCloud2 of float4 points [n, 4]: the PointXYZI message data."""
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
    out = np.zeros(32 * p.shape[0], np.uint8)
    host_lib().cm_pack(_ptr(p), C.c_size_t(p.shape[0]), _ptr(out))
    return out.tobytes()


def pack_cov(pts, cov6, trace) -> bytes:
    """packPointCloud2Cov of points [n, 4], cov_vec [n, 6] and cov_trace [n]: the PointXYZIWithCov message data."""
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
    c = np.ascontiguousarray(cov6, np.float32).reshape(-1, 6)
    t = np.ascontiguousarray(trace, np.float32).reshape(-1)
    assert c.shape[0] == t.shape[0] == p.shape[0]
    out = np.zeros(48 * p.shape[0], np.uint8)
    host_lib().cm_pack_cov(_ptr(p), _ptr(c), _ptr(t), C.c_size_t(p.shape[0]), _ptr(out))
    return out.tobytes()


def view(source: int, width: int):
    """cloudMsgView(source, width): (header dict, [(name, offset, datatype, count)])."""
    hdr = np.zeros(7, np.int32)
    names = C.create_string_buffer(16 * 11)
    offs, dts, cnts = np.zeros(11, np.int32), np.zeros(11, np.int32), np.zeros(11, np.int32)
    nf = host_lib().cm_view(int(source), C.c_size_t(width), _ptr(hdr), names, _ptr(offs), _ptr(dts), _ptr(cnts))
    keys = ("height", "width", "point_step", "row_step", "is_bigendian", "is_dense", "n_fields")
    fields = [(names.raw[16 * k:16 * k + 16].split(b"\0")[0].decode(), int(offs[k]), int(dts[k]), int(cnts[k])) for k in range(nf)]
    return dict(zip(keys, hdr.tolist())), fields


def associate(pose7, cov, pts, ext7, ext_cov, cov_meas, with_ua: bool, trace_thr: float):
    """cloudUCTAssociateToMap of one keyframe cloud (the oracle's single step) with the compound of the keyframe's pose and covariance and
    each extrinsic, as the keyframe store associates it: (points, cov_vec, cov_trace)."""
    ext7 = np.asarray(ext7, np.float64).reshape(-1, 7)
    pc, cc = [], []
    for l in range(ext7.shape[0]):
        a, b = orc.compound_pose_cov(pose7, cov, ext7[l], ext_cov[l] if with_ua else np.zeros((6, 6)))
        pc.append(a), cc.append(b)
    return orc.cloud_uct_associate(pts, pose7, ext7, np.stack(pc), np.stack(cc), cov_meas, with_ua, trace_thr)[:3]


def voxel_cov(parts, leaf: float, trace_thr: float):
    """VoxelGridCovarianceMLOAM<PointIWithCov>(leaf) of the concatenated (points, cov_vec, cov_trace) parts, with the cov_trace it stores
    (the input's on the int32-overflow pass-through): (points, cov_vec, cov_trace)."""
    parts = [q for q in parts if q[0].shape[0] > 0]
    if not parts:
        return np.zeros((0, 4), np.float32), np.zeros((0, 6), np.float32), np.zeros(0, np.float32)
    return orc.voxel_grid_cov(np.concatenate([q[0] for q in parts]), np.concatenate([q[1] for q in parts]),
                              np.concatenate([q[2] for q in parts]), leaf, trace_thr)[:3]

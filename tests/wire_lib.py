"""PointCloud2 messages for the message-frame tests and tools/bench_wire.py: driver layouts, packing of a raw sweep into a message with
numpy structured arrays, and the host build of tests/host/wire_host.cpp (m-loam_b200/host/mloam_io.hpp: unpackPointCloud2 and
resolvePointCloud2Layout), the host statement of the rules the device unpack follows."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FLOAT32, FLOAT64 = 7, 8

# name -> (point_step, big endian, [(field, offset, numpy type)]); "timestamp" is lane 3 with time_field 1 ([us], PointITimeCloud)
LAYOUTS = {
    # pcl::toROSMsg of a PointXYZI cloud (x y z at 0 4 8, intensity at 16, 32-byte points), the timestamp in the padding
    "xyzi32": (32, False, [("x", 0, "f4"), ("y", 4, "f4"), ("z", 8, "f4"), ("intensity", 16, "f4"), ("timestamp", 20, "f4")]),
    # Velodyne-style x y z intensity ring time, packed: the time field at an unaligned offset
    "velodyne22": (22, False, [("x", 0, "f4"), ("y", 4, "f4"), ("z", 8, "f4"), ("intensity", 12, "f4"), ("ring", 16, "u2"),
                               ("timestamp", 18, "f4")]),
    # FLOAT64 coordinates and timestamp, big-endian, 48-byte points
    "f64be48": (48, True, [("x", 0, "f8"), ("y", 8, "f8"), ("z", 16, "f8"), ("intensity", 24, "f4"), ("timestamp", 32, "f8")]),
    # 16-byte points: x y z timestamp, aligned like the float4 sweep itself
    "xyzt16": (16, False, [("x", 0, "f4"), ("y", 4, "f4"), ("z", 8, "f4"), ("timestamp", 12, "f4")]),
    # 48-byte points with the fields out of order at odd offsets, FLOAT64 timestamp first
    "odd48": (48, False, [("timestamp", 0, "f8"), ("z", 9, "f4"), ("x", 13, "f4"), ("y", 17, "f4"), ("intensity", 40, "f4")]),
}


def _datatype(t):
    return FLOAT64 if t == "f8" else FLOAT32 if t == "f4" else 4  # 4: UINT16


def pack(points, layout, height=1, row_pad=0, rng=None):
    """One LiDAR's raw sweep (n x 4 float32, w = the timestamp [us] or the intensity) as a PointCloud2 message of `layout`: height rows of
    width = ceil(n / height) points (the tail filled with NaN points), row_pad bytes of filler after each row.  FLOAT64 fields carry
    values with bits below float precision, so that the unpack's rounding is exercised.  Returns a dict (data: uint8 array, width,
    height, row_step, point_step, big, fields [(name, offset, datatype)])."""
    rng = rng if rng is not None else np.random.default_rng(0)
    step, big, fields = LAYOUTS[layout]
    pts = np.asarray(points, np.float32)
    n = pts.shape[0]
    width = -(-n // height)
    full = np.full((width * height, 4), np.nan, np.float32)
    full[:n] = pts
    end = ">" if big else "<"
    dt = np.dtype({"names": [f[0] for f in fields], "formats": [end + f[2] for f in fields], "offsets": [f[1] for f in fields], "itemsize": step})
    rec = np.zeros(width * height, dt)
    vals = {"x": full[:, 0], "y": full[:, 1], "z": full[:, 2], "timestamp": full[:, 3], "intensity": rng.uniform(0, 255, width * height),
            "ring": rng.integers(0, 64, width * height)}
    for name, _, t in fields:
        v = vals[name]
        if t == "f8" and name in ("x", "y", "z"):
            v = v.astype(np.float64) * (1.0 + rng.uniform(-1e-9, 1e-9, v.shape[0]))
        rec[name] = v
    row_step = width * step + row_pad
    buf = np.full((height, row_step), 0xAB, np.uint8)
    buf[:, : width * step] = rec.view(np.uint8).reshape(height, width * step)
    return dict(data=buf.reshape(-1), width=width, height=height, row_step=row_step, point_step=step, big=big,
                fields=[(f[0], f[1], _datatype(f[2])) for f in fields])


def host_lib():
    """tests/host/wire_host.cpp built with g++ into the temporary directory, keyed by the hash of its sources (the tree is never written)."""
    global _lib
    if _lib is None:
        src = os.path.join(HERE, "host", "wire_host.cpp")
        io = os.path.join(ROOT, "m-loam_b200", "host")
        h = hashlib.sha256()
        for f in (src, os.path.join(io, "mloam_io.hpp"), os.path.join(ROOT, "include", "mloam_b200.h")):
            with open(f, "rb") as fh:
                h.update(fh.read())
        so = os.path.join(tempfile.gettempdir(), f"mloam_wire_host_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            out = subprocess.run(["g++", "-std=c++14", "-O2", "-Wall", "-shared", "-fPIC", "-I" + io, src, "-o", tmp], capture_output=True, text=True)
            assert out.returncode == 0, out.stderr[-3000:]
            os.replace(tmp, so)
        _lib = C.CDLL(so)
    return _lib


_lib = None


def _field_arrays(fields):
    names = (C.c_char_p * len(fields))(*[f[0].encode() for f in fields])
    offs = (C.c_int * len(fields))(*[f[1] for f in fields])
    dts = (C.c_int * len(fields))(*[f[2] for f in fields])
    return names, offs, dts


def unpack(msg, lane3=None, size=None):
    """unpackPointCloud2 of msg with lane 3 = the field lane3 (None: the default, "intensity") -> n x 4 float32, or None when refused."""
    names, offs, dts = _field_arrays(msg["fields"])
    out = np.zeros((msg["width"] * msg["height"], 4), np.float32)
    data = msg["data"]
    ok = host_lib().wire_unpack(C.c_void_p(data.ctypes.data), C.c_size_t(data.nbytes if size is None else size), msg["width"], msg["height"],
                                C.c_size_t(msg["row_step"]), msg["point_step"], int(msg["big"]), len(msg["fields"]), names, offs, dts,
                                None if lane3 is None else lane3.encode(), C.c_void_p(out.ctypes.data))
    return out if ok else None


def layout(mloam, msg, lane3):
    """resolvePointCloud2Layout of msg's fields (lane3: the lane-3 field name or None) -> mloam.Pc2Layout, or None when refused."""
    names, offs, dts = _field_arrays(msg["fields"])
    lay = mloam.Pc2Layout()
    ok = host_lib().wire_layout(msg["point_step"], int(msg["big"]), len(msg["fields"]), names, offs, dts, None if lane3 is None else lane3.encode(),
                                C.byref(lay))
    return lay if ok else None


def as_arg(msg):
    """The (data, width, height, row_step) tuple the binding's message entry points take."""
    return (msg["data"], msg["width"], msg["height"], msg["row_step"])

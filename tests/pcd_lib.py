"""PCD helpers shared by the PCD tests and tools/bench_pcd.py: the host build of csrc/pcd_ascii.cuh and the PCD rules of
m-loam_b200/host/mloam_io.hpp (tests/host/pcd_host.cpp), token packing, and PCD files as pcl::io::savePCDFileASCII writes them."""
import ctypes as C

import numpy as np

import host_build

_P = C.c_void_p


def lib():
    return host_build.load("pcd_host")


def pack(tokens):
    """[bytes] -> (buffer, offsets int64[n + 1])."""
    off = np.zeros(len(tokens) + 1, np.int64)
    off[1:] = np.cumsum([len(t) for t in tokens])
    return np.frombuffer(b"".join(tokens) or b"\0", np.uint8).copy(), off


def _ptr(a):
    return _P(a.__array_interface__["data"][0])


def parse(buf, off):
    """The device parser on the host: (status int32[n], bits uint32[n])."""
    n = off.size - 1
    st, bits = np.zeros(n, np.int32), np.zeros(n, np.uint32)
    lib().pcd_parse(_ptr(buf), _ptr(off), C.c_longlong(n), _ptr(st), _ptr(bits))
    return st, bits


def stream(buf, off):
    """libstdc++'s istringstream >> float (+ atof fallback, "nan"), as PCL's copyStringValue<float>: bits uint32[n]."""
    n = off.size - 1
    bits = np.zeros(n, np.uint32)
    lib().pcd_stream(_ptr(buf), _ptr(off), C.c_longlong(n), _ptr(bits))
    return bits


def fmt(bits, prec):
    """%.<prec>g of float bits -> (buffer, offsets), by the C library's printf."""
    bits = np.ascontiguousarray(bits, np.uint32)
    n = bits.size
    cap = n * (prec + 16) + 16
    buf, off = np.zeros(cap, np.uint8), np.zeros(n + 1, np.int64)
    w = lib().pcd_format(_ptr(bits), C.c_longlong(n), int(prec), _ptr(buf), C.c_longlong(cap), _ptr(off))
    assert w >= 0
    return buf[:w].copy() if w else np.zeros(1, np.uint8), off


def header(data: bytes):
    """resolvePCDHeader -> dict, or None when refused."""
    out = np.zeros(11, np.int64)
    if not lib().pcd_header(C.c_char_p(data), C.c_size_t(len(data)), _ptr(out)):
        return None
    k = ["points", "body", "tokens", "ix", "iy", "iz", "binary", "point_step", "ox", "oy", "oz"]
    return dict(zip(k, (int(v) for v in out)))


def decode_ascii(body: bytes, points: int, tokens: int, index):
    """decodePCDASCII -> (rc, float32[points, 4])."""
    out = np.zeros((max(points, 1), 4), np.float32)
    idx = np.ascontiguousarray(index, np.int32)
    rc = lib().pcd_decode_ascii(C.c_char_p(body), C.c_size_t(len(body)), int(points), int(tokens), _ptr(idx), _ptr(out))
    return rc, out[:points]


def fields_header(fields, points, data="ascii"):
    """The v0.7 header savePCDFileASCII / savePCDFileBinary write; fields: [(name, size, type, count)]."""
    names = " ".join(f[0] for f in fields)
    return ("# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\n"
            f"FIELDS {names}\nSIZE {' '.join(str(f[1]) for f in fields)}\nTYPE {' '.join(f[2] for f in fields)}\n"
            f"COUNT {' '.join(str(f[3]) for f in fields)}\nWIDTH {points}\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {points}\n"
            f"DATA {data}\n").encode()


XYZ = [("x", 4, "F", 1), ("y", 4, "F", 1), ("z", 4, "F", 1)]
XYZI = XYZ + [("intensity", 4, "F", 1)]


def ascii_body(cols, prec=8, sep=" ", eol="\n"):
    """Rows of columns (float32 arrays of one length) as %.<prec>g lines (PCL's writer uses %.8g)."""
    cols = [np.ascontiguousarray(c, np.float32) for c in cols]
    txt = [fmt(c.view(np.uint32), prec) for c in cols]
    strs = [[bytes(b[o[k]:o[k + 1]]) for k in range(o.size - 1)] for b, o in txt]
    return b"".join(sep.encode().join(r) + eol.encode() for r in zip(*strs))

"""PCD writer helpers shared by the PCD writer tests and tools/bench_pcd_write.py: the host build of csrc/pcd_format.cuh and of
m-loam_b200/host/mloam_io.hpp writePCDASCII (tests/host/pcd_write_host.cpp), and the float bit patterns the tests push through both."""
import ctypes as C

import numpy as np

import host_build
import pcd_lib as pl

_P = C.c_void_p
XYZ, XYZI, XYZI_COV = 0, 1, 2  # MLOAM_PCD_*
FIELDS = {XYZ: pl.XYZ, XYZI: pl.XYZI,
          XYZI_COV: pl.XYZI + [(n, 4, "F", 1) for n in ("cov_xx", "cov_xy", "cov_xz", "cov_yy", "cov_yz", "cov_zz", "cov_trace")]}


def lib():
    return host_build.load("pcd_write_host")


def _ptr(a):
    return None if a is None else _P(a.__array_interface__["data"][0])


def fmt8(bits):
    """pcd::format_float of float bits -> (buffer, offsets)."""
    bits = np.ascontiguousarray(bits, np.uint32)
    n = bits.size
    cap = n * 14 + 16
    buf, off = np.zeros(cap, np.uint8), np.zeros(n + 1, np.int64)
    w = lib().pcd_format8(_ptr(bits), C.c_longlong(n), _ptr(buf), C.c_longlong(cap), _ptr(off))
    assert w >= 0
    return buf[:w].copy() if w else np.zeros(1, np.uint8), off


def printf8(bits):
    """What PCL writes for float bits by the C library's printf: %.8g, with "nan" for every NaN -> (buffer, offsets)."""
    bits = np.ascontiguousarray(bits, np.uint32)
    buf, off = pl.fmt(bits, 8)
    nan = np.isnan(bits.view(np.float32))
    if not nan.any():
        return buf, off
    toks = [b"nan" if nan[k] else bytes(buf[off[k]:off[k + 1]]) for k in range(bits.size)]
    return pl.pack(toks)


def write_ascii(layout, pts, cov6=None, trace=None) -> bytes:
    """writePCDASCII of a cloud: pts [n, 4] float32, cov6 [n, 6] and trace [n] for XYZI_COV."""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 4)
    n = pts.shape[0]
    c6 = None if cov6 is None else np.ascontiguousarray(cov6, np.float32).reshape(-1, 6)
    tr = None if trace is None else np.ascontiguousarray(trace, np.float32).reshape(-1)
    cap = 512 + n * 165
    buf = np.zeros(cap, np.uint8)
    w = lib().pcd_write_ascii(int(layout), _ptr(pts), _ptr(c6), _ptr(tr), C.c_longlong(n), _ptr(buf), C.c_longlong(cap))
    assert w >= 0
    return buf[:w].tobytes()


def cov_cloud(rng, n):
    """n random PointXYZIWithCov points: (pts [n,4], cov6 [n,6], trace [n]), float32, spread over many magnitudes."""
    pts = (rng.standard_normal((n, 4)) * 10.0 ** rng.integers(-3, 4, (n, 4))).astype(np.float32)
    cov6 = (rng.standard_normal((n, 6)) * 10.0 ** rng.integers(-6, 0, (n, 6))).astype(np.float32)
    trace = (cov6[:, 0] + cov6[:, 3]) + cov6[:, 5]
    return pts, cov6, trace.astype(np.float32)


def targeted_bits():
    """The targeted float sets: every exponent x the first and last 4096 mantissas, both signs; exact ties of %.8g (all of them, both
    signs); powers of ten +-4 ulp; the %f / %e boundaries; subnormals, zeros, infinities, NaNs."""
    m = np.concatenate([np.arange(4096), np.arange((1 << 23) - 4096, 1 << 23)]).astype(np.uint32)
    e = np.arange(256, dtype=np.uint32)
    grid = (e[:, None] << np.uint32(23) | m[None, :]).ravel()
    t = ties()
    sets = [grid, grid | np.uint32(0x80000000), t, t | np.uint32(0x80000000)]
    p10 = np.array([10.0 ** k for k in range(-45, 39)], np.float32).view(np.uint32).astype(np.int64)
    sets.append(np.clip((p10[:, None] + np.arange(-4, 5)[None, :]).ravel(), 1, 0x7f7fffff).astype(np.uint32))
    for edge in (1e-5, 1e-4, 1e7, 1e8, 99999999.5, 9.9999995e-5, 9.99999995e7, 9.99999995e-5):
        b = np.array([edge], np.float32).view(np.uint32).astype(np.int64)[0]
        sets.append(np.arange(b - 64, b + 65, dtype=np.int64).astype(np.uint32))
    sets.append(np.array([0, 0x80000000, 1, 0x80000001, 0x7fffff, 0x800000, 0x7f7fffff, 0xff7fffff, 0x7f800000, 0xff800000,
                          0x7fc00000, 0xffc00000, 0x7f800001, 0xff800001, 0x7fbfffff, 0xffffffff, 0x7fc12345, 0xfff00000], np.uint32))
    return np.concatenate(sets)


def ties():
    """Every float whose exact value has nine significant digits ending in 5: the exact ties of %.8g.  Such a value is N / 2^f with N odd
    and f >= 1, whose decimal expansion has f fractional digits, the last a 5; nine significant digits put it in [10^(8 - f), 10^(9 - f)),
    and N < 2^24 makes it a float.  That leaves f = 2 .. 12: every tie in [1, 2^24) and the few hundred below 1."""
    out = []
    for f in range(1, 13):
        lo = -(-(10 ** 8) * 2 ** f // 10 ** f)  # ceil(10^(8 - f) 2^f)
        hi = min(-(-(10 ** 9) * 2 ** f // 10 ** f), 1 << 24)  # N < 10^(9 - f) 2^f, N < 2^24
        N = np.arange(lo | 1, hi, 2, dtype=np.int64)
        if N.size:
            out.append(np.ldexp(N.astype(np.float64), -f).astype(np.float32).view(np.uint32))
    return np.concatenate(out)

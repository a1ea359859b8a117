"""CPU tests of the PCD writer: csrc/pcd_format.cuh built for the host prints every float as the C library's %.8g does (with "nan" for
every NaN, as PCL writes it), on every exponent's first and last mantissas, a million random bit patterns, every exact tie, powers of
ten, the %f / %e boundaries and the special values; host/mloam_io.hpp writePCDASCII writes pcd_lib's header and that body for all
three layouts and the known answers; the PCD reader reads a written file back to strtof of its tokens; the new entry points are
declared, exported and bound, and the adapter's wrappers compile against the stub headers."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import pcd_lib as pl
import pcd_write_lib as pw

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["mloam_cloud_pcd", "mloam_cloud_pcd_device", "mloam_pcd_encode"]


def _same(bits):
    got_b, got_o = pw.fmt8(bits)
    want_b, want_o = pw.printf8(bits)
    if np.array_equal(got_o, want_o) and np.array_equal(got_b[:got_o[-1]], want_b[:want_o[-1]]):
        return
    for k in range(bits.size):
        g, w = bytes(got_b[got_o[k]:got_o[k + 1]]), bytes(want_b[want_o[k]:want_o[k + 1]])
        assert g == w, (hex(int(bits[k])), g, w)


def test_targeted_sets_match_printf():
    bits = pw.targeted_bits()
    assert bits.size > 2 * 256 * 8192 + 2 * 10 ** 7
    _same(bits)


def test_random_bit_patterns_match_printf():
    rng = np.random.default_rng(20261018)
    _same(rng.integers(0, 1 << 32, size=10 ** 6, dtype=np.uint64).astype(np.uint32))


def test_ties_are_exact_and_round_to_even():
    t = pw.ties().view(np.float32).astype(np.float64)
    # nine significant digits, the last a 5, exactly
    for v in t[:: max(1, t.size // 2000)]:
        s = repr(float(v))
        digits = re.sub(r"[^0-9]", "", s.split("e")[0]).lstrip("0")
        assert len(digits) == 9 and digits[-1] == "5", s


@pytest.mark.parametrize("value,text", [(1234567.25, "1234567.2"), (1234567.75, "1234567.8"), (1e-4, "9.9999997e-05"),
                                        (16777215.0, "16777215"), (1e8, "1e+08"), (0.1, "0.1"), (1.4e-45, "1.4012985e-45"),
                                        (3.4028234663852886e38, "3.4028235e+38"), (-0.0, "-0"), (float("inf"), "inf"),
                                        (float("-inf"), "-inf")])
def test_known_answers(value, text):
    b, o = pw.fmt8(np.array([value], np.float32).view(np.uint32))
    assert bytes(b[:o[1]]).decode() == text
    assert pw.write_ascii(pw.XYZ, np.array([[value, 0, 0, 0]], np.float32)).endswith(f"\n{text} 0 0\n".encode())


def test_nans_of_either_sign_and_any_payload_are_nan():
    nans = np.array([0x7fc00000, 0xffc00000, 0x7f800001, 0xff800001, 0x7fffffff, 0xffffffff, 0x7fa5a5a5], np.uint32)
    b, o = pw.fmt8(nans)
    assert bytes(b[:o[-1]]) == b"nan" * nans.size
    pts = np.zeros((nans.size, 4), np.uint32)
    pts[:, 0] = pts[:, 3] = nans
    body = pw.write_ascii(pw.XYZI, pts.view(np.float32)).split(b"DATA ascii\n")[1]
    assert body == b"nan 0 0 nan\n" * nans.size


@pytest.mark.parametrize("layout", [pw.XYZ, pw.XYZI, pw.XYZI_COV])
@pytest.mark.parametrize("n", [1, 7, 1000])
def test_write_ascii_is_header_and_printf_body(layout, n):
    rng = np.random.default_rng(n + 10 * layout)
    pts, cov6, trace = pw.cov_cloud(rng, n)
    pts.view(np.uint32)[:: 7, 1] = 0xffc00000  # NaNs of both signs, infinities and signed zeros in the rows
    pts.view(np.uint32)[3:: 11, 2] = 0x80000000
    pts[5:: 13, 0] = -np.inf
    cols = [pts[:, k] for k in range(3 if layout == pw.XYZ else 4)]
    if layout == pw.XYZI_COV:
        cols += [cov6[:, k] for k in range(6)] + [trace]
        got = pw.write_ascii(layout, pts, cov6, trace)
    else:
        got = pw.write_ascii(layout, pts)
    body = pl.ascii_body(cols).replace(b"-nan", b"nan")
    assert got == pl.fields_header(pw.FIELDS[layout], n) + body


def test_empty_cloud_writes_nothing():
    assert pw.write_ascii(pw.XYZI, np.zeros((0, 4), np.float32)) == b""


def test_written_file_reads_back_to_strtof_of_its_tokens():
    rng = np.random.default_rng(5)
    bits = rng.integers(0, 1 << 32, size=3 * 20000, dtype=np.uint64).astype(np.uint32)
    pts = np.zeros((20000, 4), np.uint32)
    pts[:, :3] = bits.reshape(-1, 3)
    data = pw.write_ascii(pw.XYZ, pts.view(np.float32))
    h = pl.header(data)
    assert h is not None and h["points"] == 20000 and h["tokens"] == 3 and not h["binary"]
    rc, out = pl.decode_ascii(data[h["body"]:], h["points"], h["tokens"], (h["ix"], h["iy"], h["iz"]))
    assert rc == 0
    toks = data[h["body"]:].split()
    buf, off = pl.pack(toks)
    want = pl.stream(buf, off).reshape(-1, 3)
    assert np.array_equal(out[:, :3].view(np.uint32), want)
    finite = np.isfinite(pts[:, :3].view(np.float32))
    # %.8g keeps 8 of the 9 digits a float needs: within one unit of the 8th digit
    a, b = pts[:, :3].view(np.float32)[finite].astype(np.float64), out[:, :3][finite].astype(np.float64)
    assert (np.abs(a - b) <= np.abs(a) * 1e-7 + 1e-45).all()


def test_symbols_in_header_library_and_binding(mloam):
    mloam.build()
    hdr = open(os.path.join(ROOT, "include", "mloam_b200.h")).read()
    declared = set(re.findall(r"\b(mloam_[a-z0-9_]+)\s*\(", hdr))
    for s in NEW:
        assert s in declared and s in mloam.ABI_SYMBOLS and hasattr(mloam.lib(), s), s
    for m in ("cloud_pcd", "cloud_pcd_device", "pcd_encode"):
        assert callable(getattr(mloam.Context, m)), m
    assert (mloam.PCD_KEYFRAMES, mloam.PCD_XYZ, mloam.PCD_XYZI, mloam.PCD_XYZI_COV) == (6, 0, 1, 2)


def test_struct_layout_matches_binding(mloam):
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "sz.c")
        with open(src, "w") as f:
            f.write('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(){printf("%%zu %%zu %%zu %%zu %%zu %%zu",'
                    "sizeof(mloam_pcd_cloud_t), offsetof(mloam_pcd_cloud_t, pts), offsetof(mloam_pcd_cloud_t, cov6),"
                    "offsetof(mloam_pcd_cloud_t, trace), offsetof(mloam_pcd_cloud_t, count), offsetof(mloam_pcd_cloud_t, layout));"
                    "return 0;}\n" % os.path.join(ROOT, "include", "mloam_b200.h"))
        subprocess.check_call(["gcc", src, "-o", os.path.join(d, "sz")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "sz")]).split()]
    P = mloam.PcdCloud
    assert got == [C.sizeof(P), P.pts.offset, P.cov6.offset, P.trace.offset, P.count.offset, P.layout.offset]


def test_adapter_wrappers_compile_against_stub_headers(mloam):
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "pcd_write.o")
        out = subprocess.run(["g++", "-std=c++14", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "tests", "stubs"),
                              "-I" + os.path.join(ROOT, "m-loam_b200", "host"), "-I" + os.path.join(ROOT, "include"), "-c",
                              os.path.join(ROOT, "tests", "stubs", "pcd_write_compile_test.cpp"), "-o", obj], capture_output=True, text=True)
        assert out.returncode == 0, out.stderr[-3000:]
        syms = subprocess.run(["nm", "-C", obj], capture_output=True, text=True).stdout
    needed = set(re.findall(r"U (mloam_[a-z0-9_]+)", syms))
    assert {"mloam_cloud_pcd", "mloam_pcd_encode", "mloam_global_map"} <= needed
    for s in needed:
        assert hasattr(mloam.lib(), s), s

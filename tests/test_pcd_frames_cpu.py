"""CPU tests of the PCD decode: csrc/pcd_ascii.cuh built for the host reads every token as libstdc++'s istringstream >> float (+ atof
fallback) does, the float PCL's copyStringValue<float> stores, bit for bit; it refuses every token outside its grammar or over 19
significant digits; host/mloam_io.hpp resolves PCD headers and decodes ASCII bodies by its rules; the new entry points are declared,
exported and bound, and mloam_pcd_t matches the binding."""
import ctypes as C
import os
import re
import subprocess
import tempfile
from decimal import Decimal, getcontext

import numpy as np
import pytest

import pcd_lib as pl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["mloam_pcd_decode", "mloam_pcd_decode_device", "mloam_front_end_pcd", "mloam_frame_pcd", "mloam_frame_pcd_device",
       "mloam_frame_set_next_pcd", "mloam_frame_set_next_pcd_device"]


def _check_same(tokens):
    buf, off = pl.pack(tokens)
    st, got = pl.parse(buf, off)
    assert (st == 0).all(), [tokens[k] for k in np.flatnonzero(st)[:5]]
    want = pl.stream(buf, off)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, [(tokens[k], hex(got[k]), hex(want[k])) for k in bad[:5]]
    return got


def _tokens(buf, off):
    return [bytes(buf[off[k]:off[k + 1]]) for k in range(off.size - 1)]


def test_printf_forms_of_2_24_floats_match_libstdcxx_and_round_trip():
    """%.8g, %.9g and %.17g of 2^24 floats spread over every exponent (random bits, NaN left out), in batches."""
    rng = np.random.default_rng(20261018)
    total = 0
    for _ in range(17):
        bits = rng.integers(0, 1 << 32, size=1 << 20, dtype=np.uint64).astype(np.uint32)
        bits = bits[~np.isnan(bits.view(np.float32))]
        for prec in (8, 9, 17):
            buf, off = pl.fmt(bits, prec)
            st, got = pl.parse(buf, off)
            assert (st == 0).all()
            want = pl.stream(buf, off)
            bad = np.flatnonzero(got != want)
            assert bad.size == 0, [(bytes(buf[off[k]:off[k + 1]]), hex(got[k]), hex(want[k])) for k in bad[:5]]
            if prec >= 9:  # %.9g and %.17g name their float
                assert (got == bits).all()
        total += bits.size
    assert total >= 1 << 24


def test_subnormal_and_normal_boundaries():
    ks = np.concatenate([np.arange(0, 4096), np.arange((1 << 23) - 4096, (1 << 23) + 4096)]).astype(np.uint32)
    bits = np.concatenate([ks, ks | np.uint32(0x80000000)])
    for prec in (6, 8, 9, 12, 17):
        buf, off = pl.fmt(bits, prec)
        got = _check_same(_tokens(buf, off))
        if prec >= 9:
            assert (got == bits).all()
    # the rounding boundary between 0 and the smallest subnormal (2^-150) and around it, in the last digit
    getcontext().prec = 60
    half = Decimal(2) ** -150
    toks = []
    for digits in range(1, 20):
        s = f"{half:.{digits - 1}e}"
        m, e = s.split("e")
        last = int(m.replace(".", ""))
        for d in (-1, 0, 1):
            v = str(last + d)
            toks.append(f"{v[0]}.{v[1:]}e{int(e) - (len(v) - len(str(last)))}".encode() if len(v) > 1 else f"{v}e{e}".encode())
    toks += [b"1e-46", b"7e-46", b"7.1e-46", b"1.4e-45", b"1.401298464324817e-45", b"-7e-46", b"1e-45", b"1e-300"]
    _check_same(toks)


def test_ties_to_even_with_at_most_19_digits():
    """Decimals exactly halfway between two floats: ties-to-even decides."""
    getcontext().prec = 80
    rng = np.random.default_rng(5)
    toks = [b"16777217", b"16777219", b"2345678.125", b"33554434", b"33554438", b"-16777217", b"0.500000029802322387695312"[:20]]
    for _ in range(20000):
        k = int(rng.integers(-30, 40))
        m = int(rng.integers(1 << 23, 1 << 24))
        mid = (Decimal(2 * m + 1) * Decimal(2) ** (k - 1)).normalize()
        digits = mid.as_tuple().digits
        if len(digits) <= 19:
            toks.append(format(mid, "f").encode() if abs(mid.as_tuple().exponent) < 30 else f"{mid:e}".encode())
    assert len(toks) > 5000
    got = _check_same(toks)
    assert got[0] == np.float32(16777216).view(np.uint32) and got[1] == np.float32(16777220).view(np.uint32)
    assert got[2] == np.float32(2345678.0).view(np.uint32)


def test_flt_max_overflow_threshold_and_special_forms():
    toks = [b"3.40282347e38", b"3.40282346e38", b"3.40282348e38", b"3.4028235e38", b"3.4028236e38", b"-3.4028236e38",
            b"3.402823567797336616e38", b"3.402823567797336617e38", b"3.402823567797336615e38", b"3.40282356779733661e38",
            b"1e39", b"-1e39", b"1e38", b"1E+05", b"1e+05", b"+.5", b"5.", b"-0", b"-0.0", b"+0", b"0e99999999999", b"1e-99999999999",
            b"inf", b"-inf", b"+inf", b"nan", b"0.0000000000000000000000000000001234567890123456789",
            b"1234567890123456789000000000000000", b"000000000000000000000001.5", b"1.500000000000000000000000000",
            b"12345678901234567.89", b".1234567890123456789e-3"]
    got = _check_same(toks)
    f = got.view(np.float32)
    assert np.isposinf(f[toks.index(b"1e39")]) and np.isneginf(f[toks.index(b"-1e39")])
    assert got[toks.index(b"-0")] == 0x80000000 and got[toks.index(b"+0")] == 0
    assert got[toks.index(b"nan")] == 0x7fc00000
    assert got[toks.index(b"3.402823567797336617e38")] == 0x7f800000
    assert got[toks.index(b"3.402823567797336616e38")] == 0x7f7fffff


def test_refuses_tokens_outside_the_grammar_and_over_19_digits():
    bad = [b"", b"+", b"-", b".", b"e5", b"1e", b"1e+", b"1.2.3", b"1x", b"0x10", b"NaN", b"-nan", b"+nan", b"Inf", b"infinity", b"1,5",
           b"--1", b"+-1", b"1e5.0", b"..5", b"1d5", b"+.", b"-.e1", b"1e 5", b"nan0", b"in", b"\x00"]
    buf, off = pl.pack(bad)
    st, _ = pl.parse(buf, off)
    assert (st == 1).all(), [bad[k] for k in np.flatnonzero(st != 1)]
    long = [b"12345678901234567891", b"1.2345678901234567891", b"0.000123456789012345678901", b"-98765432109876543211e-5",
            b"10000000000000000001", b"1.0000000000000000001"]
    buf, off = pl.pack(long)
    st, _ = pl.parse(buf, off)
    assert (st == 2).all(), [long[k] for k in np.flatnonzero(st != 2)]
    # trailing zeros are not significant: 19 digits each
    ok = [b"1234567890123456789", b"1234567890123456789000", b"0.0001234567890123456789", b"100000000000000000000000000000",
          b"12345678901234567890", b"1.2345678901234567890", b"-98765432109876543210e-5"]
    _check_same(ok)


def _xyz(n, seed=1):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((n, 3)) * 20).astype(np.float32)


def test_headers_pcl_writes_and_the_ones_refused():
    h = pl.header(pl.fields_header(pl.XYZ, 10) + b"1 2 3\n")
    assert h and h["points"] == 10 and h["tokens"] == 3 and (h["ix"], h["iy"], h["iz"]) == (0, 1, 2) and h["binary"] == 0
    hdr = pl.fields_header(pl.XYZI, 7)
    h = pl.header(hdr + b"rest")
    assert h["tokens"] == 4 and h["body"] == len(hdr) and h["point_step"] == 16
    padded = [("_", 1, "U", 4), ("x", 4, "F", 1), ("rgb", 4, "U", 1), ("y", 4, "F", 1), ("_", 4, "F", 3), ("z", 4, "F", 1), ("t", 8, "F", 1)]
    h = pl.header(pl.fields_header(padded, 3))
    assert (h["ix"], h["iy"], h["iz"], h["tokens"]) == (4, 6, 10, 12) and (h["ox"], h["oy"], h["oz"]) == (4, 12, 28)
    assert h["point_step"] == 40
    assert pl.header(pl.fields_header(pl.XYZ, 3, "binary"))["binary"] == 1
    assert pl.header(pl.fields_header(pl.XYZ, 3, "binary_compressed")) is None
    assert pl.header(pl.fields_header([("x", 4, "F", 1), ("y", 4, "F", 1)], 3)) is None
    assert pl.header(pl.fields_header([("x", 8, "F", 1), ("y", 4, "F", 1), ("z", 4, "F", 1)], 3)) is None
    assert pl.header(pl.fields_header([("x", 4, "F", 1), ("y", 4, "F", 2), ("z", 4, "F", 1)], 3)) is None
    assert pl.header(pl.fields_header([("x", 4, "I", 1), ("y", 4, "F", 1), ("z", 4, "F", 1)], 3)) is None
    assert pl.header(pl.fields_header(pl.XYZ, 3).replace(b"DATA ascii\n", b"")) is None


def test_binary_helper_equals_resolve_pointcloud2_layout(mloam):
    import wire_lib as wl

    padded = [("x", 4, "F", 1), ("_", 1, "U", 4), ("y", 4, "F", 1), ("z", 4, "F", 1), ("intensity", 4, "F", 1)]
    hdr = pl.fields_header(padded, 5, "binary")
    data = hdr + bytes(5 * 20)
    L, M = mloam.Pc2Layout(), mloam.Pc2Msg()
    assert pl.lib().pcd_binary_msg(C.c_char_p(data), C.c_size_t(len(data)), C.byref(L), C.byref(M)) == 1
    msg = {"point_step": 20, "big": False, "fields": [("x", 0, 7), ("_", 4, 2), ("y", 8, 7), ("z", 12, 7), ("intensity", 16, 7)]}
    ref = wl.layout(mloam, msg, None)
    assert ref is not None and bytes(L) == bytes(ref)
    assert M.width == 5 and M.height == 1 and M.row_step == 100 and M.size == 100
    short = hdr + bytes(99)
    assert pl.lib().pcd_binary_msg(C.c_char_p(short), C.c_size_t(len(short)), C.byref(L), C.byref(M)) == 0


def test_decode_ascii_lines_crlf_tabs_blank_extra():
    p = _xyz(6)
    body = pl.ascii_body([p[:, 0], p[:, 1], p[:, 2]])
    rc, out = pl.decode_ascii(body, 6, 3, (0, 1, 2))
    assert rc == 0 and np.array_equal(out[:, :3].view(np.uint32), p.view(np.uint32)) and (out[:, 3] == 0).all()
    lines = body.split(b"\n")[:-1]
    messy = (b"\n  \t\r\n" + b"\r\n".join(l.replace(b" ", b" \t  ") + b" 7 8 extra" for l in lines) + b"\r\n\n1 2 3\n9 9\n")
    rc, out2 = pl.decode_ascii(messy, 6, 3, (0, 1, 2))
    assert rc == 0 and np.array_equal(out2, out)
    rc, out3 = pl.decode_ascii(b"  " + body.replace(b"\n", b"  \n"), 6, 3, (0, 1, 2))
    assert rc == 0 and np.array_equal(out3, out)
    # token indices other than 0, 1, 2 and a tab-separated layout
    body4 = pl.ascii_body([p[:, 2], p[:, 0], np.zeros(6), p[:, 1]], sep="\t")
    rc, out4 = pl.decode_ascii(body4, 6, 4, (1, 3, 0))
    assert rc == 0 and np.array_equal(out4, out)
    assert pl.decode_ascii(body, 7, 3, (0, 1, 2))[0] == 8            # fewer lines than POINTS
    assert pl.decode_ascii(b"1 2\n", 1, 3, (0, 1, 2))[0] == 1        # a short line
    assert pl.decode_ascii(b"1 2 3\n4 5\n", 2, 3, (0, 1, 2))[0] == 1
    assert pl.decode_ascii(b"1 2 x\n", 1, 3, (0, 1, 2))[0] == 2      # a bad token
    assert pl.decode_ascii(b"1 2 3 x\n", 1, 4, (0, 1, 2))[0] == 0    # not x / y / z: not read
    assert pl.decode_ascii(b"1 2 12345678901234567891\n", 1, 3, (0, 1, 2))[0] == 4
    rc, o = pl.decode_ascii(b"nan inf -inf\n-0 1e39 1e-46\n", 2, 3, (0, 1, 2))
    assert rc == 0 and np.isnan(o[0, 0]) and np.isposinf(o[0, 1]) and np.isneginf(o[0, 2])
    assert o[1, :3].view(np.uint32).tolist() == [0x80000000, 0x7f800000, 0]


def test_symbols_in_header_library_and_binding(mloam):
    mloam.build()
    hdr = open(os.path.join(ROOT, "include", "mloam_b200.h")).read()
    declared = set(re.findall(r"\b(mloam_[a-z0-9_]+)\s*\(", hdr))
    for s in NEW:
        assert s in declared and s in mloam.ABI_SYMBOLS and hasattr(mloam.lib(), s), s
    for m in ("pcd_decode", "pcd_decode_device", "front_end_pcd", "frame_pcd", "frame_pcd_device", "frame_set_next_pcd",
              "frame_set_next_pcd_device"):
        assert callable(getattr(mloam.Context, m)), m


def test_struct_layout_matches_binding(mloam):
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "sz.c")
        with open(src, "w") as f:
            f.write('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(){printf("%%zu %%zu %%zu %%zu %%zu %%zu",'
                    "sizeof(mloam_pcd_t), offsetof(mloam_pcd_t, size), offsetof(mloam_pcd_t, points), offsetof(mloam_pcd_t, tokens),"
                    "offsetof(mloam_pcd_t, index), offsetof(mloam_pcd_t, reserved));return 0;}\n" % os.path.join(ROOT, "include", "mloam_b200.h"))
        subprocess.check_call(["gcc", src, "-o", os.path.join(d, "sz")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "sz")]).split()]
    P = mloam.PcdBody
    assert got == [C.sizeof(P), P.size.offset, P.points.offset, P.tokens.offset, P.index.offset, P.reserved.offset]


@pytest.mark.parametrize("src", ["pcd_compile_test.cpp", "pcd_shim_compile_test.cpp"])
def test_adapter_and_shim_wrappers_compile_against_stub_headers(mloam, src):
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "pcd.o")
        out = subprocess.run(["g++", "-std=c++14", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "tests", "stubs"),
                              "-I" + os.path.join(ROOT, "m-loam_b200", "host"), "-I" + os.path.join(ROOT, "include"), "-c",
                              os.path.join(ROOT, "tests", "stubs", src), "-o", obj], capture_output=True, text=True)
        assert out.returncode == 0, out.stderr[-3000:]
        syms = subprocess.run(["nm", "-C", obj], capture_output=True, text=True).stdout
    needed = set(re.findall(r"U (mloam_[a-z0-9_]+)", syms))
    assert "mloam_pcd_decode" in needed
    for s in needed:
        assert hasattr(mloam.lib(), s), s

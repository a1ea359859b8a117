"""CPU tests of the published clouds as PointCloud2 data (mloam_cloud_msgs*): the entry points and source constants are declared,
exported and bound; m-loam_b200/host/mloam_io.hpp's packPointCloud2Cov writes the PointXYZIWithCov layout a numpy structured dtype
describes, with zero padding, and its messages (and packPointCloud2's) unpack through unpackPointCloud2; cloudMsgView gives each source's
fields, steps and is_dense; the adapter's toROSMsg and the shim's cloudMsgs wrappers compile against the stub headers."""
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import cloud_msgs_lib as cml
import wire_lib as wl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["mloam_cloud_msgs", "mloam_cloud_msgs_device"]
SOURCES = {"MLOAM_MSG_FULL_RES": 0, "MLOAM_MSG_SURF_LAST": 1, "MLOAM_MSG_CORNER_LAST": 2, "MLOAM_MSG_SURROUND": 3, "MLOAM_MSG_GLOBAL_MAP0": 4,
           "MLOAM_MSG_GLOBAL_MAP1": 5}
XYZI = np.dtype({"names": ["x", "y", "z", "intensity"], "formats": ["<f4"] * 4, "offsets": [0, 4, 8, 16], "itemsize": 32})
COV_NAMES = ["x", "y", "z", "intensity", "cov_xx", "cov_xy", "cov_xz", "cov_yy", "cov_yz", "cov_zz", "cov_trace"]
COV_OFFS = [0, 4, 8, 16, 20, 24, 28, 32, 36, 40, 44]
XYZI_COV = np.dtype({"names": COV_NAMES, "formats": ["<f4"] * 11, "offsets": COV_OFFS, "itemsize": 48})


def _cloud(n, seed=0):
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-80, 80, (n, 4)).astype(np.float32)
    cov6 = rng.uniform(-1e-3, 1e-2, (n, 6)).astype(np.float32)
    tr = rng.uniform(0, 0.1, n).astype(np.float32)
    return pts, cov6, tr


def test_symbols_in_header_library_and_binding(mloam):
    mloam.build()
    hdr = open(os.path.join(ROOT, "include", "mloam_b200.h")).read()
    declared = set(re.findall(r"\b(mloam_[a-z0-9_]+)\s*\(", hdr))
    for s in NEW:
        assert s in declared and s in mloam.ABI_SYMBOLS and hasattr(mloam.lib(), s), s
    for name, v in SOURCES.items():
        assert re.search(r"#define %s %d\b" % (name, v), hdr), name
        assert getattr(mloam, name[len("MLOAM_"):]) == v, name
    assert callable(mloam.Context.cloud_msgs) and callable(mloam.Context.cloud_msgs_device)
    assert [mloam.msg_step(s) for s in range(6)] == [32, 32, 32, 48, 48, 48]


def test_pack_cov_matches_structured_dtype_with_zero_padding():
    pts, cov6, tr = _cloud(1001, seed=3)
    pts[5, 0], pts[6, 1], pts[7, 2] = np.nan, np.inf, -np.inf
    got = np.frombuffer(cml.pack_cov(pts, cov6, tr), np.uint8)
    assert got.size == 48 * 1001
    rec = got.view(XYZI_COV)
    for k, name in enumerate(("x", "y", "z", "intensity")):
        assert np.array_equal(rec[name].view(np.uint32), pts[:, k].view(np.uint32)), name
    for k, name in enumerate(COV_NAMES[4:10]):
        assert np.array_equal(rec[name].view(np.uint32), cov6[:, k].view(np.uint32)), name
    assert np.array_equal(rec["cov_trace"].view(np.uint32), tr.view(np.uint32))
    assert not got.reshape(-1, 48)[:, 12:16].any()  # the only padding of the 48-byte layout
    want = np.zeros(1001, XYZI_COV)
    for k, name in enumerate(("x", "y", "z", "intensity")):
        want[name] = pts[:, k]
    for k, name in enumerate(COV_NAMES[4:10]):
        want[name] = cov6[:, k]
    want["cov_trace"] = tr
    assert got.tobytes() == want.tobytes()  # numpy's structured array zero-fills its padding too
    assert cml.pack_cov(pts[:0], cov6[:0], tr[:0]) == b""


def test_pack_xyzi_zero_padding():
    pts, _, _ = _cloud(257, seed=4)
    got = np.frombuffer(cml.pack(pts), np.uint8)
    want = np.zeros(257, XYZI)
    for k, name in enumerate(("x", "y", "z", "intensity")):
        want[name] = pts[:, k]
    assert got.tobytes() == want.tobytes()
    assert not got.reshape(-1, 32)[:, 12:16].any() and not got.reshape(-1, 32)[:, 20:].any()


@pytest.mark.parametrize("source", range(6))
def test_view_fields_steps_and_round_trip(source):
    n = 333
    pts, cov6, tr = _cloud(n, seed=10 + source)
    hdr, fields = cml.view(source, n)
    step = 32 if source < 3 else 48
    assert hdr == dict(height=1, width=n, point_step=step, row_step=step * n, is_bigendian=0, is_dense=int(source != 0),
                       n_fields=4 if source < 3 else 11)
    names = ["x", "y", "z", "intensity"] if source < 3 else COV_NAMES
    offs = [0, 4, 8, 16] if source < 3 else COV_OFFS
    assert fields == [(nm, o, 7, 1) for nm, o in zip(names, offs)]
    data = cml.pack(pts) if source < 3 else cml.pack_cov(pts, cov6, tr)
    msg = dict(data=np.frombuffer(data, np.uint8).copy(), width=n, height=1, row_step=step * n, point_step=step, big=False,
               fields=[(nm, o, dt) for nm, o, dt, _ in fields])
    back = wl.unpack(msg)
    assert back is not None and np.array_equal(back.view(np.uint32), pts.view(np.uint32))
    if source >= 3:  # the covariance fields read back by name, as a subscriber's fromROSMsg does
        for k, name in enumerate(COV_NAMES[4:]):
            want = cov6[:, k] if k < 6 else tr
            assert np.array_equal(wl.unpack(msg, lane3=name)[:, 3].view(np.uint32), want.view(np.uint32)), name


def test_wrappers_compile_against_stub_headers(mloam):
    stubs = os.path.join(ROOT, "tests", "stubs")
    needed = set()
    with tempfile.TemporaryDirectory() as td:
        for src, inc in (("cloud_msgs_adapter_compile_test.cpp", ["-I" + stubs]),
                         ("cloud_msgs_shim_compile_test.cpp", ["-I" + os.path.join(ROOT, "m-loam_b200", "host"), "-I" + os.path.join(ROOT, "include")])):
            obj = os.path.join(td, src + ".o")
            out = subprocess.run(["g++", "-std=c++14", "-Wall", "-Werror", *inc, "-c", os.path.join(stubs, src), "-o", obj], capture_output=True,
                                 text=True)
            assert out.returncode == 0, (src, out.stderr[-3000:])
            syms = subprocess.run(["nm", "-C", obj], capture_output=True, text=True).stdout
            got = set(re.findall(r"U (mloam_[a-z0-9_]+)", syms))
            assert "mloam_cloud_msgs" in got, src
            needed |= got
    mloam.build()
    for s in needed:
        assert hasattr(mloam.lib(), s), s

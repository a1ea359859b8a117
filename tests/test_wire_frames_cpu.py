"""CPU tests of the PointCloud2 message frames: the new entry points are declared, exported and bound; mloam_pc2_layout_t / mloam_pc2_msg_t
match the binding; the shim's message wrappers compile; m-loam_b200/host/mloam_io.hpp resolves layouts and unpacks messages (lane 3 =
the timestamp field) as a numpy structured-array decode does, and refuses a field that does not lie inside the point."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import wire_lib as wl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["mloam_set_front_end_layout", "mloam_front_end_msg", "mloam_frame_msg", "mloam_frame_msg_device", "mloam_frame_set_next_msg",
       "mloam_frame_set_next_msg_device"]


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def test_symbols_in_header_library_and_binding(mloam):
    mloam.build()
    hdr = open(os.path.join(ROOT, "include", "mloam_b200.h")).read()
    declared = set(re.findall(r"\b(mloam_[a-z0-9_]+)\s*\(", hdr))
    for s in NEW:
        assert s in declared and s in mloam.ABI_SYMBOLS and hasattr(mloam.lib(), s), s
    for m in ("set_front_end_layout", "front_end_msg", "frame_msg", "frame_msg_device", "frame_set_next_msg", "frame_set_next_msg_device"):
        assert callable(getattr(mloam.Context, m)), m


def test_struct_layouts_match_binding(mloam):
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "sz.c")
        with open(src, "w") as f:
            f.write('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(){printf("%%zu %%zu %%zu %%zu %%zu %%zu %%zu %%zu %%zu %%zu",'
                    "sizeof(mloam_pc2_layout_t), offsetof(mloam_pc2_layout_t, offset), offsetof(mloam_pc2_layout_t, datatype),"
                    "offsetof(mloam_pc2_layout_t, is_bigendian), sizeof(mloam_pc2_msg_t), offsetof(mloam_pc2_msg_t, size),"
                    "offsetof(mloam_pc2_msg_t, width), offsetof(mloam_pc2_msg_t, height), offsetof(mloam_pc2_msg_t, row_step), 0ul);return 0;}\n"
                    % os.path.join(ROOT, "include", "mloam_b200.h"))
        subprocess.check_call(["gcc", src, "-o", os.path.join(d, "sz")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "sz")]).split()][:9]
    L, M = mloam.Pc2Layout, mloam.Pc2Msg
    want = [C.sizeof(L), L.offset.offset, L.datatype.offset, L.is_bigendian.offset, C.sizeof(M), M.size.offset, M.width.offset,
            M.height.offset, M.row_step.offset]
    assert got == want, (got, want)


def test_shim_wrappers_compile_against_stub_headers(mloam):
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "wire_shim_compile_test.o")
        out = subprocess.run(["g++", "-std=c++14", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "tests", "stubs"),
                              "-I" + os.path.join(ROOT, "m-loam_b200", "host"), "-I" + os.path.join(ROOT, "include"), "-c",
                              os.path.join(ROOT, "tests", "stubs", "wire_shim_compile_test.cpp"), "-o", obj], capture_output=True, text=True)
        assert out.returncode == 0, out.stderr[-3000:]
        syms = subprocess.run(["nm", "-C", obj], capture_output=True, text=True).stdout
    needed = set(re.findall(r"U (mloam_[a-z0-9_]+)", syms))
    assert {"mloam_set_front_end_layout", "mloam_frame_msg"} <= needed
    mloam.build()
    for s in needed:
        assert hasattr(mloam.lib(), s), s


def _msg(layout, n=100, **kw):
    rng = np.random.default_rng(1)
    pts = np.concatenate([rng.uniform(-50, 50, (n, 3)), rng.uniform(0, 1e5, (n, 1))], 1).astype(np.float32)
    return wl.pack(pts, layout, rng=rng, **kw), pts


def test_layout_helper_accepts_and_rejects(mloam):
    for name, (step, big, fields) in wl.LAYOUTS.items():
        msg, _ = _msg(name)
        lay = wl.layout(mloam, msg, "timestamp")
        off = {f[0]: f[1] for f in fields}
        typ = {f[0]: wl._datatype(f[2]) for f in fields}
        assert lay is not None and lay.point_step == step and lay.is_bigendian == int(big), name
        assert list(lay.offset) == [off["x"], off["y"], off["z"], off["timestamp"]], name
        assert list(lay.datatype) == [typ["x"], typ["y"], typ["z"], typ["timestamp"]], name
        lay0 = wl.layout(mloam, msg, None)  # time_field 0: no lane 3
        assert lay0 is not None and lay0.datatype[3] == 0 and lay0.offset[3] == 0 and list(lay0.offset)[:3] == list(lay.offset)[:3]
    msg, _ = _msg("velodyne22")
    base = msg["fields"]
    for bad in ([f for f in base if f[0] != "y"],                                      # y missing
                [f if f[0] != "z" else ("z", 8, 4) for f in base],                     # UINT16 z
                [f if f[0] != "x" else ("x", 19, 7) for f in base]):                   # x at 19..23 of a 22-byte point
        assert wl.layout(mloam, dict(msg, fields=bad), None) is None, bad
    assert wl.layout(mloam, dict(msg, fields=[f for f in base if f[0] != "timestamp"]), "timestamp") is None  # lane 3 asked, missing
    assert wl.layout(mloam, dict(msg, fields=[f if f[0] != "timestamp" else ("timestamp", 18, 8) for f in base]), "timestamp") is None  # 18 + 8 > 22
    assert wl.layout(mloam, dict(msg, fields=[f if f[0] != "timestamp" else ("timestamp", 18, 1) for f in base]), "timestamp") is None  # INT8
    assert wl.layout(mloam, dict(msg, fields=[f if f[0] != "x" else ("x", 18, 7) for f in base]), None) is not None  # 18 + 4 == 22: inside


@pytest.mark.parametrize("layout", sorted(wl.LAYOUTS))
@pytest.mark.parametrize("height,row_pad", [(1, 0), (4, 0), (4, 13)])
def test_unpack_lane3_timestamp_equals_structured_decode(layout, height, row_pad):
    msg, _ = _msg(layout, n=1001, height=height, row_pad=row_pad)
    step, big, fields = wl.LAYOUTS[layout]
    end = ">" if big else "<"
    dt = np.dtype({"names": [f[0] for f in fields], "formats": [end + f[2] for f in fields], "offsets": [f[1] for f in fields], "itemsize": step})
    rows = msg["data"].reshape(msg["height"], msg["row_step"])[:, : msg["width"] * step]
    rec = np.ascontiguousarray(rows).reshape(-1).view(dt)
    want = np.stack([rec["x"], rec["y"], rec["z"], rec["timestamp"]], 1).astype(np.float32)  # float64 -> float32: round to nearest
    got = wl.unpack(msg, "timestamp")
    assert got is not None and np.array_equal(_bits(got), _bits(want))
    if "intensity" in rec.dtype.names:  # the default lane 3 stays the intensity field
        assert np.array_equal(_bits(wl.unpack(msg)[:, 3]), _bits(rec["intensity"].astype(np.float32)))
    assert wl.unpack(msg, "timestamp", size=msg["data"].nbytes - 1) is None  # shorter than height x row_step


def test_unpack_rejects_field_past_point_step():
    """A field with offset + size > point_step: with row_step == width x point_step the last point's field would be read past
    height x row_step bytes.  unpackPointCloud2 refuses the message as it refuses a short buffer.  Built from the two-argument call
    only, as any existing caller makes it."""
    src = r'''
#include <cstdio>
#include "mloam_io.hpp"
using namespace mloam::io;
int main() {
  std::vector<uint8_t> bytes(3 * 16, 0);
  PointCloud2View m;
  m.width = 3, m.height = 1, m.point_step = 16, m.row_step = 48;
  const char *names[4] = {"x", "y", "z", "intensity"};
  const uint32_t offs[4] = {0, 4, 8, 14};  // intensity at 14..18 of a 16-byte point
  for (int k = 0; k < 4; k++) { PointField f; f.name = names[k], f.offset = offs[k], f.datatype = FLOAT32; m.fields.push_back(f); }
  m.data = bytes.data(), m.data_size = bytes.size();
  std::vector<mloam_point_t> out;
  const bool bad_ok = unpackPointCloud2(m, out);
  m.fields[3].offset = 12;  // 12..16: inside
  const bool good_ok = unpackPointCloud2(m, out);
  m.fields[2].datatype = FLOAT64, m.fields[2].offset = 12, m.fields.pop_back();  // a FLOAT64 z at 12..20
  const bool bad64_ok = unpackPointCloud2(m, out);
  std::printf("%d %d %d\n", bad_ok, good_ok, bad64_ok);
  return 0;
}
'''
    with tempfile.TemporaryDirectory() as td:
        cpp, exe = os.path.join(td, "bounds.cpp"), os.path.join(td, "bounds")
        with open(cpp, "w") as f:
            f.write(src)
        out = subprocess.run(["g++", "-std=c++14", "-Wall", "-I" + os.path.join(ROOT, "m-loam_b200", "host"), cpp, "-o", exe], capture_output=True, text=True)
        assert out.returncode == 0, out.stderr[-3000:]
        res = subprocess.run([exe], capture_output=True, text=True).stdout.split()
    assert res == ["0", "1", "0"], res

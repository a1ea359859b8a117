"""CPU tests: the C-ABI library builds for sm_90a, loads, and exports every symbol include/mloam_b200.h declares;
without a device, context creation fails loudly (no CPU fallback)."""
import os
import re

import pytest


def test_library_loads_and_exports_header_symbols(mloam):
    mloam.build()
    lib = mloam.lib()
    hdr = open(os.path.join(mloam.ROOT, "include", "mloam_b200.h")).read()
    declared = sorted(set(re.findall(r"\b(mloam_[a-z0-9_]+)\s*\(", hdr)))
    assert declared, "no declarations found"
    for sym in declared:
        assert hasattr(lib, sym), f"{sym} declared in include/mloam_b200.h but not exported"
    assert set(declared) == set(mloam.ABI_SYMBOLS)
    assert b"sm_90a" in lib.mloam_version()


def test_struct_layouts_match_defaults(mloam):
    p = mloam.default_params()
    assert p.n_neigh == 5 and p.max_outer == 2 and p.max_inner == 30
    assert abs(p.min_match_sq_dis - 1.0) < 1e-7 and abs(p.min_plane_dis - 0.2) < 1e-7
    assert abs(p.huber_a - 0.1) < 1e-15 and p.eig_thre == 100.0 and abs(p.cov_trace - 0.0075) < 1e-15
    assert abs(p.corner_leaf - 0.2) < 1e-7 and abs(p.surf_leaf - 0.4) < 1e-7
    # the fields carved out of the reserved tail sit where the C struct puts them (a shifted layout would scramble these)
    assert p.gf_method == 0 and abs(p.gf_ratio - 1.0) < 1e-7 and p.gf_seed == 0 and all(v == 0 for v in p.reserved)
    import ctypes

    # sizes of the C structs (gcc, include/mloam_b200.h): the ctypes mirrors must agree byte for byte
    import subprocess
    import tempfile

    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "sz.c")
        with open(src, "w") as f:
            f.write('#include <stdio.h>\n#include "%s"\nint main(){printf("%%zu %%zu %%zu", sizeof(mloam_params_t), sizeof(mloam_solve_stats_t), '
                    'sizeof(mloam_features_t));return 0;}\n' % os.path.join(mloam.ROOT, "include", "mloam_b200.h"))
        subprocess.check_call(["gcc", src, "-o", os.path.join(d, "sz")])
        sizes = [int(x) for x in subprocess.check_output([os.path.join(d, "sz")]).split()]
    assert sizes == [ctypes.sizeof(mloam.Params), ctypes.sizeof(mloam.SolveStats), ctypes.sizeof(mloam.Features)]


def test_no_device_fails_loudly(mloam):
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(mloam.MloamError):
        mloam.Context(0)


def test_only_sm90a_sass_is_embedded(mloam):
    import subprocess

    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-lelf", mloam.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_cpp_host_shim_compiles_links_and_refuses_to_run_without_gpu(mloam):
    """m-loam_b200/host/mloam_shim.hpp mirrors the reference's class surface over the C ABI; its self-test must build
    with plain g++ (no CUDA, PCL, Eigen or Ceres headers) and, with no device, fail loudly instead of falling back."""
    import subprocess

    import torch

    mloam.build()
    exe = os.path.join(mloam.HERE, "host", "shim_selftest")
    subprocess.check_call(["make", "-C", mloam.HERE, "host/shim_selftest"], stdout=subprocess.DEVNULL)
    assert os.path.exists(exe)
    if torch.cuda.is_available():
        pytest.skip("a GPU is present (the gpu-marked test runs the binary)")
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 2 and "no CPU path" in out.stdout


def test_wire_format_helpers_selftest():
    """m-loam_b200/host/mloam_io.hpp (PointCloud2 <-> float4, mloam_msgs PODs, TUM dump): host-only, checked by its own self-test."""
    import subprocess
    ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(ROOT, "m-loam_b200", "host", "io_selftest")
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "m-loam_b200"), "host/io_selftest"], stdout=subprocess.DEVNULL)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "io_selftest OK" in out.stdout, out.stdout + out.stderr


def test_adapter_compiles_against_stub_headers(mloam):
    """m-loam_b200/host/mloam_adapter.hpp — the hot-path classes with the reference's own PCL / Eigen / Ceres types — is compiled
    against the minimal stand-in headers of tests/stubs/ with the reference's call shapes, and every C-ABI symbol it needs is exported."""
    import subprocess
    import tempfile
    ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "adapter_compile_test.o")
        out = subprocess.run(["g++", "-std=c++14", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "tests", "stubs"), "-c",
                              os.path.join(ROOT, "tests", "stubs", "adapter_compile_test.cpp"), "-o", obj], capture_output=True, text=True)
        assert out.returncode == 0, out.stderr[-3000:]
        syms = subprocess.run(["nm", "-C", obj], capture_output=True, text=True).stdout
    needed = sorted(set(re.findall(r"U (mloam_[a-z0-9_]+)", syms)))
    assert len(needed) >= 10
    lib = mloam.lib()
    for s in needed:
        assert hasattr(lib, s), s


def _host_projection_lib(td):
    import ctypes
    import subprocess
    ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    so = os.path.join(td, "libproject_host.so")
    out = subprocess.run(["g++", "-std=c++14", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "m-loam_b200", "csrc"),
                          os.path.join(ROOT, "tests", "stubs", "project_host.cpp"), "-o", so], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-3000:]
    return ctypes.CDLL(so)


def test_projection_arithmetic_matches_oracle_on_the_host():
    """csrc/project.cuh + csrc/fd_atan.cuh (what k_project_pixels evaluates) built for the host: (a) fd::atanf / fd::atan2f return the C
    library's bits (the reference's pixel assignment depends on them: image_segmenter.hpp:103,119), (b) every point lands in the oracle's
    pixel — random clouds, points on pixel borders, degenerate points — for the 16-, 32- and 64-ring parameter sets."""
    import ctypes as C
    import tempfile
    import numpy as np
    import oracle_lib as orc
    with tempfile.TemporaryDirectory() as td:
        h = _host_projection_lib(td)
        h.host_fd_atan_mismatches.restype = C.c_long
        rng = np.random.default_rng(5)
        n = 2_000_000
        x = (rng.uniform(-80, 80, n) * np.exp2(rng.integers(-40, 40, n) * (rng.random(n) < 0.3))).astype(np.float32)
        y = (rng.uniform(-80, 80, n) * np.exp2(rng.integers(-40, 40, n) * (rng.random(n) < 0.3))).astype(np.float32)
        sp = np.array([0, -0.0, 1, -1, np.inf, -np.inf, np.nan, 1e-38, -1e-38, 1e38, 1e-45, 0.4375, 0.6875, 1.1875, 2.4375, 2.0 ** 25, 2.0 ** 26], np.float32)
        x = np.concatenate([x, np.repeat(sp, sp.size)]).astype(np.float32)
        y = np.concatenate([y, np.tile(sp, sp.size)]).astype(np.float32)
        ok = ~(np.isnan(x) | np.isnan(y))  # NaN payloads are not compared
        xs, ys = np.ascontiguousarray(x[ok]), np.ascontiguousarray(y[ok])
        bad = h.host_fd_atan_mismatches(xs.ctypes.data_as(C.c_void_p), ys.ctypes.data_as(C.c_void_p), C.c_long(xs.size))
        assert bad == 0, bad
        for rings, hs in ((16, 1800), (32, 2169), (64, 2048)):
            n = 400_000
            az, el = rng.uniform(-np.pi, np.pi, n), np.deg2rad(rng.uniform(-35, 20, n))
            # a third of the azimuths / elevations sit (almost) on pixel borders
            k = n // 3
            az[:k] = np.deg2rad((rng.integers(0, hs, k) + 0.5) * 360.0 / hs - 180.0) + rng.normal(0, 1e-7, k)
            if rings == 16:
                el[k:2 * k] = np.deg2rad(rng.integers(-1, 17, k) * 2.0 - 15.1) + rng.normal(0, 1e-7, k)
            r = rng.uniform(0.1, 90, n)
            pts = np.stack([r * np.cos(el) * np.sin(az), r * np.cos(el) * np.cos(az), r * np.sin(el), rng.random(n)], 1).astype(np.float32)
            pts[:8] = [[0, 0, 0, 0], [0, 0, 1, 0], [0, 0, -1, 0], [1, 0, 0, 0], [0, 1, 0, 0], [-1, 0, 0, 0], [0, -1, 0, 0], [np.nan, 1, 1, 0]]
            for roi in (0.5, 0.0):
                want = orc.project_pixels(pts, rings, hs, roi)
                got = np.zeros(n, np.int32)
                h.host_project_pixels(pts.ctypes.data_as(C.c_void_p), n, rings, hs, C.c_double(roi), got.ctypes.data_as(C.c_void_p))
                assert np.array_equal(got, want), (rings, roi, int((got != want).sum()))
                assert (want >= 0).sum() > n // 4


def test_bench_contract_on_a_cpu_box():
    """bench.py without a GPU: the reference arm (CPU restatement, the one leg that may execute oracle/) prints ONE JSON line with the
    contract's keys; our arm refuses to run (no CPU fallback) with a JSON error and a non-zero exit code."""
    import json
    import subprocess
    import sys
    import torch
    ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [ln for ln in out.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "scan_to_map_lidar_frames_per_sec" and d["unit"] == "frames/s"
    assert d["value"] > 0 and d["higher_is_better"] is True and d["n_gpus"] == 1 and d["gpu_launches"] == 0
    assert d["config"]["workload"].startswith("C2") and d["data"] == "synthetic"
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and "rig frame" in cb["sample"]
    assert d["e2e"] == {"value": d["value"], "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    if not torch.cuda.is_available():
        ours = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "0"], capture_output=True, text=True, timeout=300)
        assert ours.returncode != 0 and "no CUDA device" in ours.stdout

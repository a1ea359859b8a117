"""CPU tests of the raw-sweep front end: csrc/cal_timestamp.cuh built for the host equals the libm restatement of removeNaNFromPointCloud +
FeatureExtract::calTimestamp (feature_extract.cpp:25-114) bit for bit, the restatement gives the known answers, and the adapter's calTimestamp
overloads compile against the stub headers."""
import math
import os
import re
import subprocess
import tempfile

import numpy as np

import front_end_lib as fel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sweep_xy(rng, n, az0, revs=1.0, jitter=0.0):
    """n points in firing order: atan2 decreasing from az0 over `revs` revolutions."""
    az = az0 - 2 * math.pi * revs * np.arange(n) / max(n, 1) + rng.normal(0, jitter, n)
    r = rng.uniform(1, 60, n)
    return np.stack([r * np.cos(az), r * np.sin(az), rng.uniform(-3, 3, n), rng.uniform(0, 255, n)], 1).astype(np.float32)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def _same(a, b):
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


def test_header_matches_libm_restatement_bit_for_bit():
    rng = np.random.default_rng(17)
    clouds = []
    # sweeps starting in every quadrant and exactly on +-pi / the axes, single and partial revolutions, both directions
    starts = [math.pi, -math.pi, 0.0, math.pi / 2, -math.pi / 2, 3.0, -3.0, 2.0, -2.0, 1.0, -1.0] + list(rng.uniform(-math.pi, math.pi, 60))
    for k, a0 in enumerate(starts):
        for revs in (1.0, 0.999, 0.6, 1.3, -1.0):
            c = _sweep_xy(rng, 4000, a0, revs, jitter=0.002 * (k % 3))
            if a0 in (math.pi, -math.pi):  # exactly on the negative x axis: y = +0 / -0
                c[0, 1] = 0.0 if a0 > 0 else -0.0
                c[0, 0] = -abs(c[0, 0])
            clouds.append(c)
    # random clouds (no firing order): points on both sides of the flip everywhere
    for _ in range(110):
        clouds.append(_sweep_xy(rng, 5000, 0.0)[rng.permutation(5000)])
    # one- and two-point clouds, empty
    for _ in range(200):
        clouds.append(_sweep_xy(rng, 1, rng.uniform(-4, 4)))
        clouds.append(_sweep_xy(rng, 2, rng.uniform(-4, 4), revs=rng.uniform(-1.5, 1.5)))
    clouds.append(np.zeros((0, 4), np.float32))
    # non-finite x, y, z — as the first, the last and interior points
    bad = [np.nan, np.inf, -np.inf]
    for k in range(90):
        c = _sweep_xy(rng, 600, rng.uniform(-math.pi, math.pi))
        lane, val = k % 3, bad[(k // 3) % 3]
        where = [0, c.shape[0] - 1] if k % 2 else list(rng.integers(0, 600, 20))
        for i in where:
            c[i, lane] = val
        if k % 5 == 0:
            c[:3, :3] = np.nan  # the first three points dropped: the sweep starts at the fourth
        clouds.append(c)
    clouds.append(np.full((4, 4), np.nan, np.float32))
    total = sum(c.shape[0] for c in clouds)
    assert total >= 2_000_000, total
    for i, c in enumerate(clouds):
        for tf in (False, True):
            want = fel.cal_timestamp(c, tf, 0.1)
            got = fel.cal_timestamp_header(c, tf, 0.1)
            assert _same(got, want), (i, tf, c.shape)


def test_known_answers():
    rng = np.random.default_rng(3)
    for a0 in (math.pi, 2.5, 0.3, -0.7, -2.9):
        c = _sweep_xy(rng, 3601, a0)
        c[-1, :2] = c[0, :2]  # the last point closes the revolution: same direction as the first
        t = fel.cal_timestamp(c, False, 0.1)[:, 3]
        assert t[0] == 0.0
        assert np.all(np.diff(t) >= 0), a0
        assert t[-1] == np.float32(0.1), (a0, t[-1])
    # the first FINITE point is the time origin
    c = _sweep_xy(rng, 100, 1.0)
    c[:2, 0] = np.nan
    out = fel.cal_timestamp(c, False, 0.1)
    assert out.shape[0] == 98 and out[0, 3] == 0.0 and np.array_equal(_bits(out[:, :3]), _bits(c[2:, :3]))
    # timestamp mode: (float)(t * 1e-6) of the timestamp in the intensity lane
    c = _sweep_xy(rng, 1000, 0.0)
    c[:, 3] = rng.uniform(0, 1e5, 1000).astype(np.float32)
    out = fel.cal_timestamp(c, True, 0.1)
    assert np.array_equal(_bits(out[:, 3]), _bits((c[:, 3].astype(np.float64) * 1e-6).astype(np.float32)))


def test_adapter_cal_timestamp_compiles_against_stub_headers(mloam):
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "adapter_cal_timestamp_test.o")
        out = subprocess.run(["g++", "-std=c++14", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "tests", "stubs"), "-c",
                              os.path.join(ROOT, "tests", "stubs", "adapter_cal_timestamp_test.cpp"), "-o", obj], capture_output=True, text=True)
        assert out.returncode == 0, out.stderr[-3000:]
        syms = subprocess.run(["nm", "-C", obj], capture_output=True, text=True).stdout
    needed = set(re.findall(r"U (mloam_[a-z0-9_]+)", syms))
    assert "mloam_cal_timestamp" in needed
    mloam.build()
    for s in needed:
        assert hasattr(mloam.lib(), s), s

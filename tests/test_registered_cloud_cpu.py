"""CPU tests of the registered clouds (pubPointCloud, lidar_mapper_keyframe.cpp:690-714): the oracle's entry (oracle/orc_registered.cpp) against
a numpy composition of its single steps (TransformToEnd, the float rig matrix, pointAssociateToMap in double with float stores, the order of
the parts and of the outlier points) on 1, 3 and 16 LiDARs and at the edges; a known answer; the new entry points at the boundary; the adapter
and shim wrappers compiled against the stubs."""
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import registered_lib as rl
import synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("mloam_set_registered", "mloam_frame_registered", "mloam_frame_registered_device")
POSE = syn.pose7([3.0, -1.5, 0.4], syn.quat_from_rpy(0.02, -0.01, 0.7))


def _undist(n_lidars):
    return np.stack([syn.pose7([0.08 + 0.01 * l, -0.02, 0.004], syn.quat_from_rpy(0.001, -0.002, 0.03 + 0.002 * l)) for l in range(n_lidars)])


def _rig(rng, counts):
    """A ring-ordered concatenation from per-LiDAR, per-ring point counts, with the reference's ScanInfo (start = size + 5, end = size - 6);
    intensity = ring + relative time."""
    pts, ss, se, size = [], [], [], 0
    for lidar in counts:
        for r, c in enumerate(lidar):
            ss.append(size + 5)
            p = np.zeros((c, 4), np.float32)
            p[:, :3] = rng.normal(0.0, 6.0, (c, 3))
            p[:, 3] = r + 0.1 * rng.random(c)
            pts.append(p)
            size += c
            se.append(size - 6)
    return np.concatenate(pts), np.array(ss, np.int32), np.array(se, np.int32)


def _check(cloud, ss, se, **kw):
    got = rl.registered(cloud, ss, se, POSE, **kw)
    want = rl.compose(cloud, ss, se, POSE, **kw)
    for t in range(3):
        assert rl.bits_equal(got[t], want[t]), (t, got[t].shape, want[t].shape)
    return got


@pytest.mark.parametrize("outlier", [False, True])
@pytest.mark.parametrize("distortion", [False, True])
@pytest.mark.parametrize("n_lidars", [1, 3, 16])
def test_rig_matches_composition(n_lidars, distortion, outlier):
    """Ray-cast rig sweeps: the parts LiDAR by LiDAR with intensity = laser id, then one outlier point per LiDAR when on."""
    cloud, ss, se, ext = syn.make_multi_sweep(syn.make_scene(), syn.trajectory(3)[1], n_lidars, 16, 256 if n_lidars == 16 else 512, seed=9)
    got = _check(cloud, ss, se, ext7=ext, poses7=_undist(n_lidars) if distortion else None, outlier=outlier)
    assert got[0].shape[0] == cloud.shape[0] + (n_lidars if outlier else 0)
    assert got[1].shape[0] > 0 and got[2].shape[0] > 0
    ids = got[0][:cloud.shape[0], 3]
    assert np.all(np.diff(ids) >= 0) and ids[-1] == n_lidars - 1
    if outlier:
        assert got[0][cloud.shape[0]:, 3].tolist() == list(range(n_lidars))


@pytest.mark.parametrize("distortion", [False, True])
@pytest.mark.parametrize("ext", [False, True])
def test_single_lidar_matches_composition(ext, distortion):
    """Without the rig merge: pointAssociateToMap with the single extrinsic (intensity kept), or no move at all; the outlier point takes the
    extrinsic's float matrix and intensity 0."""
    cloud, ss, se = syn.make_sweep(syn.make_scene(), syn.trajectory(3)[1], 16, 512, seed=4)
    single = syn.pose7([0.5, 0.1, 1.2], syn.quat_from_rpy(0.0, 0.05, 0.2)) if ext else None
    for outlier in (False, True):
        got = _check(cloud, ss, se, single_ext7=single, poses7=_undist(1) if distortion else None, outlier=outlier)
        assert got[0].shape[0] == cloud.shape[0] + int(outlier)
        assert np.array_equal(got[0][:cloud.shape[0], 3], cloud[:, 3])


@pytest.mark.parametrize("distortion", [False, True])
def test_edges(distortion):
    """An empty LiDAR part (no outlier point for it), a LiDAR whose ring 0 is empty, NaN and inf coordinates in the sweep (moved like the others)."""
    rng = np.random.Generator(np.random.PCG64(5))
    counts = [[40] * 4, [0] * 4, [0, 30, 30, 30]]
    cloud, ss, se = _rig(rng, counts)
    cloud[3, 0], cloud[50, 1], cloud[-7, 2] = np.nan, np.inf, -np.inf
    ext = np.stack([syn.pose7([0.1 * l, 0.2, -0.1 * l], syn.quat_from_rpy(0.01 * l, 0.0, 0.5 * l)) for l in range(3)])
    got = _check(cloud, ss, se, ext7=ext, poses7=_undist(3) if distortion else None, outlier=True)
    n = cloud.shape[0]
    assert got[0][n:, 3].tolist() == [0.0, 2.0]  # LiDAR 1's part is empty; LiDAR 2's first point is its ring 1's
    assert not np.isfinite(got[0][3, :3]).all() and not np.isfinite(got[0][50, :3]).all() and not np.isfinite(got[0][n - 7, :3]).all()
    assert np.isfinite(got[0][4]).all()
    got = _check(cloud, ss, se, ext7=ext, outlier=False)
    assert got[0].shape[0] == n


def test_known_answer():
    """LiDAR 1 of a two-LiDAR rig sits at (1, 2, 0) turned 180 deg about z; its first point (3, 0, 0) is (-2, 2, 0) in the base frame, and the
    pose (10, 20, 30) turned 180 deg about x puts it at (8, 18, 30), intensity 1."""
    rng = np.random.Generator(np.random.PCG64(6))
    cloud, ss, se = _rig(rng, [[8, 8], [8, 8]])
    cloud[16] = [3.0, 0.0, 0.0, 0.25]
    ext = np.array([[0, 0, 0, 0, 0, 0, 1.0], [1.0, 2.0, 0.0, 0, 0, 1.0, 0]])
    pose = np.array([10.0, 20.0, 30.0, 1.0, 0, 0, 0])
    for outlier in (False, True):
        full = rl.registered(cloud, ss, se, pose, ext7=ext, outlier=outlier)[0]
        assert full[16].tolist() == [8.0, 18.0, 30.0, 1.0]
        if outlier:
            assert full[-1].tolist() == [8.0, 18.0, 30.0, 1.0] and full.shape[0] == 34
    cloud[0] = [3.0, 0.0, 0.0, 0.25]  # one LiDAR with the same extrinsic: pointAssociateToMap twice, intensity kept
    single = rl.registered(cloud[:16], ss[:2], se[:2], pose, single_ext7=ext[1])[0]
    assert single[0].tolist() == [8.0, 18.0, 30.0, 0.25]


def test_entry_points_at_the_boundary(mloam):
    hdr = open(os.path.join(ROOT, "include", "mloam_b200.h")).read()
    lib = mloam.lib()
    for n in NAMES:
        assert re.search(r"\bint " + n + r"\(", hdr), n
        assert n in mloam.ABI_SYMBOLS and hasattr(lib, n), n
    for k, name in enumerate(("FULL_RES", "SURF", "CORNER")):
        assert re.search(r"#define MLOAM_REGISTERED_%s %d\b" % (name, k), hdr), name
        assert getattr(mloam, "REGISTERED_" + name) == k


def test_adapter_and_shim_wrap_the_entry_points(mloam):
    """The reference-shaped wrappers: the adapter against the stand-in PCL / Eigen headers, the shim with plain g++; both need only exported
    symbols."""
    with tempfile.TemporaryDirectory() as td:
        for src, inc in (("registered_adapter_compile_test.cpp", ["-I" + os.path.join(ROOT, "tests", "stubs")]),
                         ("registered_shim_compile_test.cpp", ["-I" + os.path.join(ROOT, "m-loam_b200", "host"), "-I" + os.path.join(ROOT, "include")])):
            obj = os.path.join(td, src + ".o")
            out = subprocess.run(["g++", "-std=c++14", "-Wall", "-Werror", *inc, "-c", os.path.join(ROOT, "tests", "stubs", src), "-o", obj],
                                 capture_output=True, text=True)
            assert out.returncode == 0, out.stderr[-3000:]
            syms = subprocess.run(["nm", "-C", obj], capture_output=True, text=True).stdout
            needed = set(re.findall(r"U (mloam_[a-z0-9_]+)", syms))
            assert {"mloam_set_registered", "mloam_frame_registered"} <= needed, src
            for s in needed:
                getattr(mloam.lib(), s)

"""CPU tests of the undistortion (DISTORTION: TransformToEnd with the odometry's relative pose): the device header's restated sine against
the C library's at the float output, a known answer from a sweep seen by a moving sensor, the oracle's slerp branches, the pose helper
against numpy compositions (the library's mloam_undistort_poses and the oracle's), the oracle's frame with the step off against
orc_frame_multi, and the new entry points in the header and the library."""
import math
import os
import re
import sys

import numpy as np
import pytest

import oracle_lib as orc
import synthetic as syn
import undistort_lib as udl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["mloam_undistort_poses", "mloam_set_distortion", "mloam_frame_undistort"]


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def _random_poses(rng, n, max_angle=0.3, max_t=3.0):
    out = []
    for _ in range(n):
        out.append(udl.rot_pose(rng.normal(size=3), rng.uniform(0.0, max_angle), rng.uniform(-max_t, max_t, 3)))
    return np.array(out)


def _random_points(rng, n, scan_period=0.1, rings=64):
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    p = np.zeros((n, 4), np.float32)
    p[:, :3] = d * rng.uniform(0.5, 100.0, n)[:, None]
    p[:, 3] = rng.integers(0, rings, n).astype(np.float32) + (rng.uniform(0.0, 1.0, n) * scan_period).astype(np.float32)
    return p


def test_restated_sine_gives_the_float_points_of_the_c_library():
    """2.4 M seeded points (ranges 0.5-100 m, s in [0, 1)) under 4096 poses (rotation up to 0.3 rad per sweep) plus the edge poses:
    |w| at 1 - eps and one ulp below, w < 0, the identity.  The header's TransformToEnd with fdlibm's sine equals it with the C library's
    sine to the float; the double sines that differ are counted and reported."""
    rng = np.random.Generator(np.random.PCG64(11))
    one = 1.0 - np.finfo(np.float64).eps
    w_edge = [one, np.nextafter(one, 0.0)]
    edge = [np.array([0.1, -0.2, 0.3, 0.0, 0.0, math.sqrt(1 - w * w), w]) for w in w_edge]
    edge += [np.concatenate([[0.5, 0.1, 0.0], -udl.rot_pose([1, 2, 3], 0.25, [0, 0, 0])[3:]]), np.array([0, 0, 0, 0, 0, 0, 1.0])]
    poses = np.concatenate([_random_poses(rng, 4096), np.array(edge)])
    total, diff_sines = 0, 0
    for chunk in range(6):
        pts = _random_points(rng, 400_000)
        a, d = udl.header_points(pts, poses, use_libm=True)
        b, _ = udl.header_points(pts, poses, use_libm=False)
        assert np.array_equal(_bits(a), _bits(b)), int(np.sum(np.any(_bits(a) != _bits(b), axis=1)))
        total += pts.shape[0]
        diff_sines += d
    print(f"{total} points: {diff_sines} of {2 * total} double sines differ from the C library's by an ulp; the float points agree")
    # the oracle (C library sine, independent restatement) agrees with the header on a slice of them, pose by pose
    pts = _random_points(rng, 20_000)
    for k in (0, 1, 4096, 4097, 4098, 4099):
        got, _ = udl.header_points(pts, poses[k:k + 1])
        assert np.array_equal(_bits(got), _bits(udl.points(pts, poses[k]))), k


@pytest.mark.parametrize("angle", [0.05, 0.3])
def test_known_answer_moving_sensor(angle):
    """A sweep seen by a sensor moving at constant angular and linear velocity from the identity to pose_end, rel_time in the intensity,
    undistorted with that relative pose, lands on the static scene seen from the sweep-end pose (float noise: the intensity's float fraction
    and the float stores)."""
    rng = np.random.Generator(np.random.PCG64(5))
    pose_end = udl.rot_pose([0.2, 0.3, 1.0], angle, [1.2, -0.4, 0.1])
    pts, want = udl.moving_sweep(rng, 20_000, pose_end)
    got = udl.points(pts, pose_end)
    dev, _ = udl.header_points(pts, pose_end)
    assert np.array_equal(_bits(got), _bits(dev))
    assert np.array_equal(got[:, 3], pts[:, 3])
    rng_m = np.linalg.norm(pts[:, :3].astype(np.float64), axis=1)
    err = np.linalg.norm(got[:, :3].astype(np.float64) - want, axis=1)
    # s carries the float intensity's quantisation, ulp(ring) / scan_period <= 2e-5 (rings < 16): that much of the motion
    tol = 2e-5 * (angle * rng_m + np.linalg.norm(pose_end[:3])) + 2e-7 * rng_m + 1e-6
    assert np.all(err <= tol), float(np.max(err / tol))
    # without the step the points are off by the motion
    raw_err = np.linalg.norm(pts[:, :3].astype(np.float64) - want, axis=1)
    assert np.median(raw_err) > 100 * np.median(err)


def test_oracle_slerp_branches():
    """The identity rotation takes slerp's linear weights (end = (float)((float)(p + s t) - t)); w < 0 negates the second weight, so -q moves
    the points as q does (to rounding); the identity pose is applied, not skipped, and s = 0 moves a point by the rotation's inverse only."""
    rng = np.random.Generator(np.random.PCG64(2))
    pts = _random_points(rng, 5000)
    t = np.array([0.7, -0.3, 0.2])
    got = udl.points(pts, np.concatenate([t, [0, 0, 0, 1.0]]))
    s = ((pts[:, 3] - pts[:, 3].astype(np.int32).astype(np.float32)) / np.float32(0.1)).astype(np.float64)
    un = (pts[:, :3].astype(np.float64) + s[:, None] * t).astype(np.float32)
    want = (un.astype(np.float64) - t).astype(np.float32)
    assert np.array_equal(_bits(got[:, :3]), _bits(want))
    q = udl.rot_pose([1, -1, 0.5], 0.2, t)
    qn = q.copy()
    qn[3:] = -qn[3:]
    a, b = udl.points(pts, q), udl.points(pts, qn)
    assert np.max(np.abs(a[:, :3] - b[:, :3])) < 1e-4
    ident = udl.points(pts, np.array([0, 0, 0, 0, 0, 0, 1.0]))
    assert np.allclose(ident, pts, atol=0, rtol=1e-6)
    p0 = pts.copy()
    p0[:, 3] = np.floor(p0[:, 3])  # s = 0: TransformToStart is the identity, TransformToEnd q^-1 (p - t)
    z = udl.points(p0, q)
    want0 = np.stack([udl.qrot(np.array([-q[3], -q[4], -q[5], q[6]]), p.astype(np.float64) - q[:3]) for p in p0[:50, :3]])
    assert np.allclose(z[:50, :3], want0, atol=2e-5)


@pytest.mark.parametrize("estimate_extrinsic", [0, 2])
def test_pose_helper_against_numpy(mloam, estimate_extrinsic):
    """pose_undist[n] = ext_n^-1 pose_rlt ext_n; every LiDAR takes IDX_REF's unless ESTIMATE_EXTRINSIC == 2.  IDX_REF's extrinsic is not the
    identity.  The library's host helper equals the oracle's bit for bit and numpy's composition to rounding."""
    ext = np.array([udl.rot_pose([0, 0, 1], 0.4, [0.3, 0.1, 0.05]), udl.rot_pose([1, 0, 0], -0.2, [-0.4, 0.2, 0.0]),
                    udl.rot_pose([0, 1, 1], 1.1, [0.0, -0.5, 0.3])])
    rlt = udl.rot_pose([0.1, 0.2, 1.0], 0.08, [1.5, 0.05, -0.02])
    for idx_ref in (0, 1):
        got = mloam.undistort_poses(rlt, idx_ref, ext, estimate_extrinsic)
        assert np.array_equal(got, udl.poses(rlt, idx_ref, ext, estimate_extrinsic))
        und = [udl.pose_mul(udl.pose_mul(udl.pose_inv(e), rlt), e) for e in ext]
        for n in range(3):
            want = und[n if estimate_extrinsic == 2 else idx_ref]
            assert np.allclose(got[n], want, atol=1e-14), (idx_ref, n)
    with pytest.raises(ValueError):
        mloam.undistort_poses(rlt, 3, ext, 0)


def test_oracle_off_equals_frame_multi():
    """With the step off (no poses) the oracle's frame is orc_frame_multi's, bit for bit; with the identity-rotation pose and a w < 0 pose it
    runs and changes the scans."""
    scene = syn.make_scene()
    traj = syn.trajectory(3)
    surf_map, corner_map = syn.make_submap(scene, 30000)
    cloud, ss, se, ext = syn.make_multi_sweep(scene, traj[1], 2, 16, 512, seed=3)
    o = orc.default_opts()
    o[orc.O_MAX_OUTER], o[orc.O_MAX_INNER] = 3, 1
    ref, rst = orc.frame_multi(cloud, ss, se, 2, ext, surf_map, corner_map, traj[1], o)
    got, gst, _, scans = udl.frame(cloud, ss, se, 2, ext, None, surf_map, corner_map, traj[1], opts=o)
    assert np.array_equal(got, ref)
    for k in ("ran", "n_surf", "n_corner", "lm_iterations", "final_cost", "n_surf_in", "n_corner_in"):
        assert gst[k] == rst[k], k
    cs, sf = orc.prepare_multi(cloud, ss, se, 2, ext)
    assert np.array_equal(_bits(scans["surf"]), _bits(sf)) and np.array_equal(_bits(scans["corner"]), _bits(cs))
    for pose in (np.array([0.2, 0.0, 0.0, 0, 0, 0, 1.0]), np.concatenate([[0.1, 0.1, 0], -udl.rot_pose([0, 0, 1], 0.05, [0, 0, 0])[3:]])):
        _, st, _, sc = udl.frame(cloud, ss, se, 2, ext, np.stack([pose, pose]), surf_map, corner_map, traj[1], opts=o)
        assert st["ran"] == 1 and not np.array_equal(_bits(sc["surf"][:100]), _bits(scans["surf"][:100]))


def test_header_declares_and_library_exports_the_new_entry_points(mloam):
    with open(os.path.join(ROOT, "include", "mloam_b200.h")) as f:
        declared = set(re.findall(r"^int (mloam_\w+)\(", f.read(), re.M))
    for s in NEW_SYMBOLS:
        assert s in declared and s in mloam.ABI_SYMBOLS, s
        getattr(mloam.lib(), s)


def test_adapter_and_shim_wrap_the_entry_points(mloam):
    """mloam_adapter.hpp's setDistortion / undistortPoses / undistortMeasurements compile against the stub headers with the calls of
    Estimator::process and need only exported symbols; mloam_shim.hpp's wrappers compile."""
    import subprocess
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        obj = os.path.join(td, "adapter_undistort_test.o")
        out = subprocess.run(["g++", "-std=c++14", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "tests", "stubs"), "-c",
                              os.path.join(ROOT, "tests", "stubs", "adapter_undistort_test.cpp"), "-o", obj], capture_output=True, text=True)
        assert out.returncode == 0, out.stderr[-3000:]
        syms = subprocess.run(["nm", "-C", obj], capture_output=True, text=True).stdout
        needed = set(re.findall(r"U (mloam_[a-z0-9_]+)", syms))
        assert set(NEW_SYMBOLS) <= needed
        for s in needed:
            getattr(mloam.lib(), s)
        src = os.path.join(td, "shim_use.cpp")
        with open(src, "w") as f:
            f.write('#include "' + os.path.join(ROOT, "m-loam_b200", "host", "mloam_shim.hpp") + '"\n'
                    "int shim_use(mloam_ctx_t *ctx) {\n"
                    "  mloam::setDistortion(ctx, true, 0.1f);\n"
                    "  std::vector<Pose> p = mloam::undistortPoses(Pose(), 0, std::vector<Pose>(2), 2);\n"
                    "  mloam::undistortMeasurements(ctx, p);\n"
                    "  return (int)p.size();\n}\n")
        out = subprocess.run(["g++", "-std=c++14", "-Wall", "-Werror", "-c", src, "-o", os.path.join(td, "shim_use.o")], capture_output=True,
                             text=True)
        assert out.returncode == 0, out.stderr[-3000:]

"""GPU tests (-m gpu) of the undistortion (DISTORTION: mloam_set_distortion / mloam_frame_undistort) through the C ABI: the scans entering
the solve (mloam_frame_scan) bit-identical to the oracle's (oracle/orc_ua.cpp) — mloam_frame and mloam_frame_raw, 1 and 3
LiDARs, with_ua on and off, the single-LiDAR paths —, pose and statistics within the frame parity tolerance of the oracle and bit-identical
across the stream path, graph capture and replays with a new pose every call, with and without the look-ahead and a broken announcement;
the outlier cloud untouched; the keyframe store and both global maps; the launch count; the edges; and the feature off exactly as before."""
import math
import os

import numpy as np
import pytest

import front_end_lib as fel
import global_map_lib as gl
import mapper_lib as ml
import oracle_lib as orc
import synthetic as syn
import uncertainty_lib as ua
import undistort_lib as udl

pytestmark = pytest.mark.gpu

E_INVALID, E_STATE = -1, -4
COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])
RINGS, HORIZON, OUTER = 16, 512, 4
POSE_TOL = 1e-4  # metres / radians, as tests/test_gpu_parity.py
SP = 0.1


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def _same(a, b):
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


def _exts(n):
    out = []
    for l in range(n):
        a = 2 * math.pi * l / n
        out.append([0.3 * math.cos(a), 0.3 * math.sin(a), 0.05 * l, 0.0, 0.0, math.sin(a / 4 + 0.2), math.cos(a / 4 + 0.2)])
    return np.array(out, np.float64)


def _rlt(k):
    """The odometry's relative pose of call k: a new one every call (replays must take it)."""
    return udl.rot_pose([0.1, 0.2 * (-1) ** k, 1.0], 0.02 + 0.01 * k, [0.4 + 0.05 * k, 0.03 * k, -0.01])


@pytest.fixture(scope="module")
def scene():
    sc = syn.make_scene()
    surf_map, corner_map = syn.make_submap(sc, 60000)
    return dict(scene=sc, traj=syn.trajectory(6), surf_map=surf_map, corner_map=corner_map)


def _ctx(mloam, n_lidars, env=None):
    env = env or {}
    for k, v in env.items():
        os.environ[k] = v
    try:
        p = mloam.default_params()
        p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = RINGS * n_lidars, OUTER, 1, 0.5, 1024
        return mloam.Context(0, p)
    finally:
        for k in env:
            os.environ.pop(k)


def _frames(sc, n_lidars, raw, nan_lidar=None, drop_ring0=None):
    ext = _exts(n_lidars)
    out = []
    for k in (1, 2):
        pose = sc["traj"][k]
        if raw:
            parts = [fel.raw_sweep(sc["scene"], pose, RINGS, HORIZON, 40 + 31 * k + l, ext=ext[l]) for l in range(n_lidars)]
            if nan_lidar is not None:
                parts[nan_lidar][:, 0] = np.nan
            out.append((np.ascontiguousarray(np.concatenate(parts)), np.array([p.shape[0] for p in parts], np.int32)))
        else:
            cloud, ss, se, _ = syn.make_multi_sweep(sc["scene"], pose, n_lidars, RINGS, HORIZON, seed=40 + k, ext=ext)
            if drop_ring0 is not None:
                r = drop_ring0 * RINGS
                lo, hi = ss[r] - 5, se[r] + 6
                cloud = np.ascontiguousarray(np.concatenate([cloud[:lo], cloud[hi:]]))
                d = hi - lo
                ss, se = ss.copy(), se.copy()
                ss[r], se[r] = lo + 5, lo - 6
                ss[r + 1:] -= d
                se[r + 1:] -= d
            out.append((cloud, ss, se))
    return out, ext


def _ring_ordered(mloam, frames, n_lidars):
    cx = _ctx(mloam, n_lidars)
    try:
        cx.set_lidars(n_lidars, _exts(n_lidars))
        cx.set_front_end(RINGS, HORIZON)
        out = []
        for raw, counts in frames:
            cloud, ss, se = cx.front_end(raw, counts)
            out.append((cloud, ss[:n_lidars * RINGS], se[:n_lidars * RINGS]))
        return out
    finally:
        cx.close()


def _poses(k, ext, fixed=None):
    """The poses of call k: mloam_undistort_poses's with ESTIMATE_EXTRINSIC == 2, so that every LiDAR of the rig has its own (the oracle's
    restatement, bit-identical to the library's: tests/test_undistort_cpu.py)."""
    return fixed if fixed is not None else udl.poses(_rlt(k), 0, ext, 2)


def _fixed(w, n):
    """Per LiDAR its own pose with the same rotation |w|: translations differ by LiDAR."""
    return np.array([[0.3 + 0.25 * l, -0.1 - 0.1 * l, 0.05, 0.0, 0.0, math.sqrt(1.0 - w * w), w] for l in range(n)])


def _run(mloam, sc, frames, ext, raw, with_ua, on=True, lookahead=False, graphs=True, n_rounds=3, outlier=0.0, fixed=None, broken=False,
         toggle=False, profile=False):
    """Frames A, B, A, B, ... (the same arrays, so that graphs capture and replay), a new pose every call: per frame (pose, stats, scan,
    outlier) and the launch count of each frame."""
    L = ext.shape[0]
    cx = _ctx(mloam, L, None if graphs else {"MLOAM_DISABLE_GRAPHS": "1"})
    ext_cov = ua.ext_covariances(L, seed=3)
    out, launches = [], []
    try:
        cx.set_lidars(L, ext)
        cx.set_uncertainty(with_ua, ext_cov if with_ua else None, COV_MEAS, 1e3)
        if outlier:
            cx.set_outlier(outlier)
        if on or toggle:
            cx.set_distortion(True, SP)
        if toggle:
            cx.set_distortion(False)
        if raw:
            cx.set_front_end(RINGS, HORIZON)
        if profile:  # stage profiling: the stream path with event scopes, serial scan filters, no look-ahead
            cx.profile(True)
        seq = [frames[k % 2] for k in range(2 * n_rounds)]
        for k, fr in enumerate(seq):
            if lookahead and k + 1 < len(seq):
                nx = seq[k] if broken else seq[k + 1]  # broken: announces this sweep again, the next call passes the other one
                (cx.frame_set_next_raw if raw else cx.frame_set_next)(*nx)
            if on:
                cx.frame_undistort(_poses(k, ext, fixed))
            l0 = cx.launch_count()
            if raw:
                pose, st = cx.frame_raw(fr[0], fr[1], sc["surf_map"], sc["corner_map"], sc["traj"][1 + k % 2])
            else:
                pose, st = cx.frame(fr[0], fr[1], fr[2], sc["surf_map"], sc["corner_map"], sc["traj"][1 + k % 2])
            launches.append(cx.launch_count() - l0)
            out.append((pose, dict(st), cx.frame_scan(), cx.frame_outlier() if outlier else None))
    finally:
        cx.close()
    return out, launches


def _oracle(inputs, ext, with_ua, k, fixed=None):
    L = ext.shape[0]
    c, ss, se = inputs[k % 2]
    o = orc.default_opts()
    o[orc.O_MAX_OUTER], o[orc.O_MAX_INNER] = OUTER, 1
    return udl.frame(c, ss, se, L, ext, _poses(k, ext, fixed), SCENE["surf_map"], SCENE["corner_map"], SCENE["traj"][1 + k % 2], SP,
                     ext_cov=ua.ext_covariances(L, seed=3) if with_ua else None, cov_meas=COV_MEAS, trace_threshold=1e3, opts=o)


SCENE = {}


def _check(got, inputs, ext, with_ua, fixed=None):
    for k, g in enumerate(got):
        pose, st, _, sc = _oracle(inputs, ext, with_ua, k, fixed)
        sp, sc6, cp, cc6 = g[2]
        assert _same(sp, sc["surf"]) and _same(cp, sc["corner"]), k
        assert _same(sc6, sc["surf_cov6"]) and _same(cc6, sc["corner_cov6"]), k
        assert g[1]["n_surf_in"] == st["n_surf_in"] and g[1]["n_corner_in"] == st["n_corner_in"], k
        dt, dr = syn.pose_err(g[0], pose)
        assert dt <= POSE_TOL and dr <= POSE_TOL, (k, dt, dr)


@pytest.mark.parametrize("with_ua", [False, True])
@pytest.mark.parametrize("path", ["frame", "raw"])
@pytest.mark.parametrize("n_lidars", [1, 3])
def test_frame_matches_oracle(mloam, scene, n_lidars, path, with_ua):
    """The scans bit-identical to the oracle's and the pose within the parity tolerance; poses, statistics and scans bit-identical across
    the stream path, capture and replays (a new pose every call), with and without the look-ahead, and with stage profiling; every LiDAR of
    the rig has its own pose; one launch more than with it off."""
    SCENE.update(scene)
    raw = path == "raw"
    frames, ext = _frames(scene, n_lidars, raw)
    inputs = _ring_ordered(mloam, frames, n_lidars) if raw else frames
    off, off_launches = _run(mloam, scene, frames, ext, raw, with_ua, on=False)
    if n_lidars > 1:  # every LiDAR its own pose, so that the pose a point takes depends on its LiDAR
        p0 = _poses(0, ext)
        assert all(not np.array_equal(p0[a], p0[b]) for a in range(n_lidars) for b in range(a))
    first = None
    for graphs, lookahead, profile in [(g, la, False) for g in (True, False) for la in (False, True)] + [(True, True, True)]:
        got, launches = _run(mloam, scene, frames, ext, raw, with_ua, lookahead=lookahead, graphs=graphs, profile=profile)
        if first is None:
            first = got
            _check(got, inputs, ext, with_ua)
            assert not _same(got[0][2][0], off[0][2][0])  # the step moved the scans
        for k, (g, f) in enumerate(zip(got, first)):
            assert np.array_equal(g[0], f[0]) and g[1] == f[1], (graphs, lookahead, profile, k)
            assert all(_same(a, b) for a, b in zip(g[2], f[2])), (graphs, lookahead, profile, k)
        if not lookahead and not profile:
            assert launches == [n + 1 for n in off_launches], (launches, off_launches)


@pytest.mark.parametrize("raw", [False, True])
def test_broken_announcement_and_outlier_cloud(mloam, scene, raw):
    """An announcement of the wrong sweep gives the results of no announcement; the outlier cloud is the one of the frame without the step."""
    SCENE.update(scene)
    frames, ext = _frames(scene, 3, raw)
    want, _ = _run(mloam, scene, frames, ext, raw, False, n_rounds=2)
    got, _ = _run(mloam, scene, frames, ext, raw, False, lookahead=True, broken=True, n_rounds=2)
    for g, w in zip(got, want):
        assert np.array_equal(g[0], w[0]) and g[1] == w[1] and all(_same(a, b) for a, b in zip(g[2], w[2]))
    on, _ = _run(mloam, scene, frames, ext, raw, True, n_rounds=2, outlier=0.8, lookahead=True)
    off, _ = _run(mloam, scene, frames, ext, raw, True, on=False, n_rounds=2, outlier=0.8)
    for a, b in zip(on, off):
        assert _same(a[3][0], b[3][0]) and _same(a[3][1], b[3][1])


def test_feature_off_unchanged(mloam, scene):
    """Turned on and off again, a context gives the launch counts, poses and statistics of one that never turned it on."""
    frames, ext = _frames(scene, 3, False)
    never, nl = _run(mloam, scene, frames, ext, False, False, on=False, lookahead=True)
    toggled, tl = _run(mloam, scene, frames, ext, False, False, on=False, toggle=True, lookahead=True)
    assert nl == tl
    for a, b in zip(never, toggled):
        assert np.array_equal(a[0], b[0]) and a[1] == b[1] and all(_same(x, y) for x, y in zip(a[2], b[2]))


@pytest.mark.parametrize("with_ext", [False, True])
def test_single_lidar_paths(mloam, scene, with_ext):
    """Without the rig merge (no extrinsics in mloam_set_lidars): the whole sweep is LiDAR 0's, undistorted before mloam_set_extrinsic's
    transform (or none)."""
    cloud, ss, se = syn.make_sweep(scene["scene"], scene["traj"][2], RINGS, HORIZON, seed=5)
    ext1 = np.array([0.2, -0.1, 0.3, 0.0, 0.0, math.sin(0.15), math.cos(0.15)])
    cx = _ctx(mloam, 1)
    o = orc.default_opts()
    o[orc.O_MAX_OUTER], o[orc.O_MAX_INNER] = OUTER, 1
    try:
        if with_ext:
            cx.set_extrinsic(ext1)
        cx.set_distortion(True, SP)
        for k in range(3):
            pu = mloam.undistort_poses(_rlt(k), 0, ext1[None], 0)
            cx.frame_undistort(pu)
            pose, st = cx.frame(cloud, ss, se, scene["surf_map"], scene["corner_map"], scene["traj"][2])
            sp, _, cp, _ = cx.frame_scan()
            wp, wst, _, wsc = udl.frame(cloud, ss, se, 1, None, pu, scene["surf_map"], scene["corner_map"], scene["traj"][2], SP,
                                        single_ext7=ext1 if with_ext else None, opts=o)
            assert _same(sp, wsc["surf"]) and _same(cp, wsc["corner"]), k
            dt, dr = syn.pose_err(pose, wp)
            assert dt <= POSE_TOL and dr <= POSE_TOL, (k, dt, dr)
    finally:
        cx.close()


def test_edges(mloam, scene):
    """An empty ring 0 and an empty LiDAR; s = 0 and the last rel_time below scan_period; |w| at 1 - eps and one ulp below; the identity."""
    SCENE.update(scene)
    frames, ext = _frames(scene, 3, False, drop_ring0=1)
    got, _ = _run(mloam, scene, frames, ext, False, False, n_rounds=1)
    _check(got, frames, ext, False)
    frames, ext = _frames(scene, 3, True, nan_lidar=1)
    inputs = _ring_ordered(mloam, frames, 3)
    got, _ = _run(mloam, scene, frames, ext, True, False, n_rounds=1)
    _check(got, inputs, ext, False)
    frames, ext = _frames(scene, 3, False)
    for c, _, _ in frames:  # s = 0 on every other point, the largest float fraction below scan_period on the rest
        ring = np.floor(c[:, 3])
        c[0::2, 3] = ring[0::2]
        c[1::2, 3] = np.nextafter((ring[1::2] + np.float32(SP)).astype(np.float32), np.float32(0))
    one = 1.0 - np.finfo(np.float64).eps
    for w in (one, np.nextafter(one, 0.0), 1.0):
        fixed = _fixed(w, 3)
        got, _ = _run(mloam, scene, frames, ext, False, False, n_rounds=1, fixed=fixed)
        _check(got, frames, ext, False, fixed=fixed)
    fixed = np.tile([0, 0, 0, 0, 0, 0, 1.0], (3, 1))
    got, _ = _run(mloam, scene, frames, ext, False, False, n_rounds=1, fixed=fixed)
    _check(got, frames, ext, False, fixed=fixed)
    # an empty LiDAR between two others, each with its own pose: the offsets of the empty one must not shift the others' poses
    frames, ext = _frames(scene, 3, True, nan_lidar=1)
    inputs = _ring_ordered(mloam, frames, 3)
    fixed = _fixed(math.cos(0.02), 3)
    got, _ = _run(mloam, scene, frames, ext, True, False, n_rounds=1, fixed=fixed, lookahead=True)
    _check(got, inputs, ext, False, fixed=fixed)


def test_missing_pose_count_and_communicator(mloam, scene):
    frames, ext = _frames(scene, 3, False)
    cx = _ctx(mloam, 3)
    try:
        cx.set_lidars(3, ext)
        c, ss, se = frames[0]
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
            cx.frame_undistort(np.tile([0, 0, 0, 0, 0, 0, 1.0], (3, 1)))  # off
        cx.set_distortion(True, SP)
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
            cx.frame(c, ss, se, scene["surf_map"], scene["corner_map"], scene["traj"][1])
        cx.frame_undistort(np.tile([0, 0, 0, 0, 0, 0, 1.0], (2, 1)))
        with pytest.raises(mloam.MloamError, match=f"error {E_INVALID}"):
            cx.frame(c, ss, se, scene["surf_map"], scene["corner_map"], scene["traj"][1])
        cx.frame_undistort(np.tile([0, 0, 0, 0, 0, 0, 1.0], (3, 1)))
        cx.frame(c, ss, se, scene["surf_map"], scene["corner_map"], scene["traj"][1])
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):  # consumed
            cx.frame(c, ss, se, scene["surf_map"], scene["corner_map"], scene["traj"][1])
        with pytest.raises(mloam.MloamError, match=f"error {E_INVALID}"):
            cx.set_distortion(True, 0.0)
    finally:
        cx.close()
    import torch  # noqa: F401  (torch's NCCL first, as test_keyframe_mapper.py explains)
    cx = _ctx(mloam, 1)
    try:
        try:
            cx.comm_init(1, 0, mloam.Context.comm_unique_id())
        except mloam.MloamError as e:
            pytest.skip(f"no NCCL on this machine: {e}")
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
            cx.set_distortion(True, SP)
    finally:
        cx.close()


@pytest.mark.parametrize("with_ua", [False, True])
def test_keyframe_loop_and_global_maps(mloam, with_ua):
    """The mapper loop with the keyframe store and the undistortion: each frame's scans are the oracle's, every keyframe stores them, and both
    global maps after every keyframe equal the oracle's bit for bit."""
    n_lidars, n_loop = 3, 16
    kf = dict(dist=0.3, orient=2.0, radius=6.0, res=1.0, thr=1e3)
    sc = syn.make_scene()
    traj = syn.trajectory(n_loop)
    ext = syn.rig_extrinsics(n_lidars)
    ext_cov = ua.ext_covariances(n_lidars, seed=7)
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = 16 * n_lidars, 10, 1, 0.5, 1024
    cx = mloam.Context(0, p)
    om = ml.Mapper(kf["dist"], kf["orient"], kf["radius"], kf["res"], kf["thr"])
    n_kf = 0
    try:
        cx.set_lidars(n_lidars, ext)
        cx.set_distortion(True, SP)
        cx.keyframes_init(kf["dist"], kf["orient"], kf["radius"], kf["res"], kf["thr"])
        om.set_lidars(ext, ext_cov, COV_MEAS, with_ua)
        for k in range(n_loop):
            cloud, ss, se, _ = syn.make_multi_sweep(sc, traj[k], n_lidars, 16, 1024, seed=60 + k, ext=ext)
            cx.set_uncertainty(with_ua, ext_cov if with_ua else None, COV_MEAS, 1e3)
            cx.keyframe_submap(traj[k])
            pu = mloam.undistort_poses(_rlt(k), 0, ext, 2)
            cx.frame_undistort(pu)
            pose, _ = cx.frame(cloud, ss, se, None, None, traj[k], False)
            sp, sc6, cp, cc6 = cx.frame_scan()
            _, _, _, want = udl.frame(cloud, ss, se, n_lidars, ext, pu, np.zeros((0, 4), np.float32), np.zeros((0, 4), np.float32), traj[k], SP,
                                      ext_cov=ext_cov if with_ua else None, cov_meas=COV_MEAS, trace_threshold=1e3)
            assert _same(sp, want["surf"]) and _same(cp, want["corner"]) and _same(sc6, want["surf_cov6"]), k
            if not cx.keyframe_save():
                continue
            n_kf += 1
            kid = cx.keyframe_query()[0] - 1
            kpose, kcov, ksp, _, kcp, _ = cx.keyframe_scan(kid)
            assert _same(ksp, sp) and _same(kcp, cp), k
            assert om.save(kpose, kcov, ksp, kcp, outlier=np.zeros((0, 4), np.float32))[0], k
            for mode in (mloam.GLOBAL_MAP_SURROUND, mloam.GLOBAL_MAP_SAVE):
                g = cx.global_map(mode, center=pose)
                leaf_m = p.surf_leaf * (2.0 if mode == mloam.GLOBAL_MAP_SAVE else 1.0)
                ids, want_g = gl.global_map(om, mode, pose, 1000.0, 10.0, leaf_m)
                assert cx.global_map_chosen() == ids, (k, mode)
                for a, b in zip(g, want_g):
                    assert _same(a, b), (k, mode)
    finally:
        om.close()
        cx.close()
    assert n_kf >= 3

"""GPU tests (-m gpu) of the undistortion in the look-ahead (mloam_frame_set_next_undistort): a sweep announced with its poses is
undistorted, merged and down-sampled in the look-ahead branch, and every result is the one of the same frames without any announcement —
poses, statistics, the scans (also equal to the oracle's, oracle/orc_ua.cpp), the outlier cloud and the three registered clouds; graph
replay and the stream path agree; "undistort_ahead" counts the sweeps whose undistortion moved to the branch; the mapper loop keeps the
same keyframe store and global maps; the edges where the branch's work must not be taken; the error paths; and a context that never calls
the entry point keeps its launches and graph captures."""
import math
import os

import numpy as np
import pytest

import front_end_lib as fel
import oracle_lib as orc
import synthetic as syn
import uncertainty_lib as ua
import undistort_lib as udl

pytestmark = pytest.mark.gpu

E_INVALID, E_STATE = -1, -4
COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])
RINGS, HORIZON, OUTER = 16, 512, 4
SP = 0.1
STATS = ("ran", "n_surf", "n_corner", "n_surf_in", "n_corner_in", "lm_iterations", "termination", "degenerate", "final_cost")


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


def _poses(k, ext):
    """The poses of sweep k: a new odometry pose every sweep, every LiDAR of the rig its own (ESTIMATE_EXTRINSIC == 2)."""
    rlt = udl.rot_pose([0.1, 0.2 * (-1) ** k, 1.0], 0.02 + 0.01 * k, [0.4 + 0.05 * k, 0.03 * k, -0.01])
    return udl.poses(rlt, 0, ext, 2)


@pytest.fixture(scope="module")
def scene():
    sc = syn.make_scene()
    surf_map, corner_map = syn.make_submap(sc, 60000)
    return dict(scene=sc, traj=syn.trajectory(6), surf_map=surf_map, corner_map=corner_map)


def _ctx(mloam, n_lidars, graphs=True):
    if not graphs:
        os.environ["MLOAM_DISABLE_GRAPHS"] = "1"
    try:
        p = mloam.default_params()
        p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = RINGS * n_lidars, OUTER, 1, 0.5, 1024
        return mloam.Context(0, p)
    finally:
        os.environ.pop("MLOAM_DISABLE_GRAPHS", None)


def _frames(sc, n_lidars, raw):
    ext = _exts(n_lidars)
    out = []
    for k in (1, 2):
        pose = sc["traj"][k]
        if raw:
            parts = [fel.raw_sweep(sc["scene"], pose, RINGS, HORIZON, 40 + 31 * k + l, ext=ext[l]) for l in range(n_lidars)]
            out.append((np.ascontiguousarray(np.concatenate(parts)), np.array([p.shape[0] for p in parts], np.int32)))
        else:
            cloud, ss, se, _ = syn.make_multi_sweep(sc["scene"], pose, n_lidars, RINGS, HORIZON, seed=40 + k, ext=ext)
            out.append((cloud, ss, se))
    return out, ext


def _setup(cx, L, ext, raw, with_ua):
    cx.set_lidars(L, ext)
    cx.set_uncertainty(with_ua, ua.ext_covariances(L, seed=3) if with_ua else None, COV_MEAS, 1e3)
    cx.set_outlier(0.8)
    cx.set_registered(True)
    cx.set_distortion(True, SP)
    if raw:
        cx.set_front_end(RINGS, HORIZON)


def _announce(cx, raw, fr):
    (cx.frame_set_next_raw if raw else cx.frame_set_next)(*fr)


def _call(mloam, cx, sc, raw, fr, init):
    if raw:
        pose, st = cx.frame_raw(fr[0], fr[1], sc["surf_map"], sc["corner_map"], init)
    else:
        pose, st = cx.frame(fr[0], fr[1], fr[2], sc["surf_map"], sc["corner_map"], init)
    scan = cx.frame_scan()
    out = dict(pose=pose, stats=[st[f] for f in STATS], scan=scan, outlier=cx.frame_outlier(),
               registered=[cx.frame_registered(w) for w in (mloam.REGISTERED_FULL_RES, mloam.REGISTERED_SURF, mloam.REGISTERED_CORNER)])
    return out


def _equal(a, b):
    return (np.array_equal(a["pose"], b["pose"]) and a["stats"] == b["stats"] and all(_same(x, y) for x, y in zip(a["scan"], b["scan"]))
            and all(_same(x, y) for x, y in zip(a["outlier"], b["outlier"]))
            and all(_same(x, y) for x, y in zip(a["registered"], b["registered"])))


def _run(mloam, sc, frames, ext, raw, with_ua, mode, graphs=True, n_rounds=4):
    """Frames A, B, A, B, ... (the same arrays, so that graphs capture and replay; from the sixth frame on a call replays a graph captured
    by an earlier call, whose look-ahead undistorted with other poses), each sweep with its own poses.  mode: "none" no
    announcement; "plain" the next sweep announced without poses (extracted ahead only); "ahead" announced with its poses, which the call
    that takes it does not repeat; "again" announced with them and given again, with the same bits, at the call.  Returns per frame the
    outputs and launches, the "undistort_ahead" count and the graph captures of the run."""
    L = ext.shape[0]
    cx = _ctx(mloam, L, graphs)
    out, launches = [], []
    try:
        _setup(cx, L, ext, raw, with_ua)
        seq = [frames[k % 2] for k in range(2 * n_rounds)]
        for k, fr in enumerate(seq):
            if mode != "none" and k + 1 < len(seq):
                _announce(cx, raw, seq[k + 1])
                if mode in ("ahead", "again"):
                    cx.frame_set_next_undistort(_poses(k + 1, ext))
            if mode in ("none", "plain", "again") or k == 0:
                cx.frame_undistort(_poses(k, ext))
            l0 = cx.launch_count()
            out.append(_call(mloam, cx, sc, raw, fr, sc["traj"][1 + k % 2]))
            launches.append(cx.launch_count() - l0)
        return out, launches, cx.profile_get("undistort_ahead")[1], cx.profile_get("graph_captures")[1]
    finally:
        cx.close()


def _check_oracle(got, inputs, ext, with_ua, sc):
    L = ext.shape[0]
    o = orc.default_opts()
    o[orc.O_MAX_OUTER], o[orc.O_MAX_INNER] = OUTER, 1
    for k, g in enumerate(got):
        c, ss, se = inputs[k % 2]
        _, st, _, want = udl.frame(c, ss, se, L, ext, _poses(k, ext), sc["surf_map"], sc["corner_map"], sc["traj"][1 + k % 2], SP,
                                   ext_cov=ua.ext_covariances(L, seed=3) if with_ua else None, cov_meas=COV_MEAS, trace_threshold=1e3,
                                   opts=o)
        sp, sc6, cp, cc6 = g["scan"]
        assert _same(sp, want["surf"]) and _same(cp, want["corner"]), k
        assert _same(sc6, want["surf_cov6"]) and _same(cc6, want["corner_cov6"]), k


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


@pytest.mark.parametrize("with_ua", [False, True])
@pytest.mark.parametrize("path", ["frame", "raw"])
@pytest.mark.parametrize("n_lidars", [1, 3])
def test_same_results_as_no_announcement(mloam, scene, n_lidars, path, with_ua):
    """Frames whose next sweep is announced with its poses are bit-identical to the same frames without any announcement, on graph replay
    and on the stream path; the scans are the oracle's; every announced sweep a call took was undistorted in the branch; in steady state a
    frame launches what it launches without the poses announced, and captures as many graphs."""
    raw = path == "raw"
    frames, ext = _frames(scene, n_lidars, raw)
    none, none_l, none_ahead, _ = _run(mloam, scene, frames, ext, raw, with_ua, "none")
    plain, plain_l, plain_ahead, plain_caps = _run(mloam, scene, frames, ext, raw, with_ua, "plain")
    n = len(none)
    for mode, graphs in (("ahead", True), ("ahead", False), ("again", True)):
        got, got_l, ahead, caps = _run(mloam, scene, frames, ext, raw, with_ua, mode, graphs=graphs)
        for k in range(n):
            assert _equal(got[k], none[k]), (mode, graphs, k)
        assert ahead == n - 1, (mode, graphs, ahead)
        assert got_l[1:n - 1] == plain_l[1:n - 1] == none_l[1:n - 1], (mode, graphs, got_l, plain_l, none_l)
        if graphs:
            assert caps == plain_caps, (mode, caps, plain_caps)
    for k in range(n):
        assert _equal(plain[k], none[k]), k
    assert none_ahead == 0 and plain_ahead == 0
    _check_oracle(got, _ring_ordered(mloam, frames, n_lidars) if raw else frames, ext, with_ua, scene)


def _pair(mloam, sc, frames, ext, announce_pose=True, before_first=(), between=(), call_pose=None):
    """Frame A, then frame B, B announced with frame A (with its poses when announce_pose); `before_first` runs after the announcement and
    before frame A, `between` between the two calls; frame B gives `call_pose` with mloam_frame_undistort (None: no call).  With
    announce_pose False the poses of B are given at its call.  Returns both frames' outputs and the "undistort_ahead" count."""
    L = ext.shape[0]
    cx = _ctx(mloam, L)
    try:
        _setup(cx, L, ext, False, False)
        p0, p1 = _poses(0, ext), _poses(1, ext)
        if announce_pose is not None:
            _announce(cx, False, frames[1])
            if announce_pose:
                cx.frame_set_next_undistort(p1)
        for f in before_first:
            f(cx)
        cx.frame_undistort(p0)
        a = _call(mloam, cx, sc, False, frames[0], sc["traj"][1])
        for f in between:
            f(cx)
        if call_pose is not None:
            cx.frame_undistort(call_pose)
        b = _call(mloam, cx, sc, False, frames[1], sc["traj"][2])
        return [a, b], cx.profile_get("undistort_ahead")[1]
    finally:
        cx.close()


def test_edges(mloam, scene):
    """Each edge gives the results of no announcement with the poses the call used, and "undistort_ahead" says whether the branch's work
    was taken: other bits at the call (one ulp away, or a pose that moves the scans) are not taken, the same bits and no pose at the call
    are; a new announcement of the sweep, mloam_set_lidars and DISTORTION turned off and on withdraw the poses and their work."""
    frames, ext = _frames(scene, 3, False)
    p1 = _poses(1, ext)
    p1u = p1.copy()
    p1u[0, 0] = np.nextafter(p1u[0, 0], np.inf)  # one ulp away: rarely visible in the float scans, but other bits
    p1x = p1.copy()
    p1x[:, 0] += 0.05  # a pose that moves the scans
    lidars = lambda cx: cx.set_lidars(3, ext)  # noqa: E731
    renew = lambda cx: cx.frame_set_next(*frames[1])  # noqa: E731
    cases = [
        ("one ulp away at the call", dict(call_pose=p1u), p1u, 0),
        ("another pose at the call", dict(call_pose=p1x), p1x, 0),
        ("same bits at the call", dict(call_pose=p1), p1, 1),
        ("no pose at the call", dict(), p1, 1),
        ("withdrawn by a new announcement", dict(before_first=[renew], call_pose=p1), p1, 0),
        ("set_lidars before frame A", dict(before_first=[lidars], call_pose=p1), p1, 0),
        ("set_lidars between the calls", dict(between=[lidars], call_pose=p1), p1, 0),
        ("DISTORTION off and on between the calls", dict(between=[lambda cx: cx.set_distortion(False), lambda cx: cx.set_distortion(True, SP)],
                                                         call_pose=p1), p1, 0),
    ]
    refs = {}
    for label, kw, used, want_ahead in cases:
        key = used.tobytes()
        if key not in refs:
            refs[key], _ = _pair(mloam, scene, frames, ext, announce_pose=None, call_pose=used)
        got, ahead = _pair(mloam, scene, frames, ext, **kw)
        assert ahead == want_ahead, (label, ahead)
        for k in range(2):
            assert _equal(got[k], refs[key][k]), (label, k)
    assert not _equal(refs[p1.tobytes()][1], refs[p1x.tobytes()][1])  # the comparison sees a pose taken from the wrong place


def test_errors(mloam, scene):
    frames, ext = _frames(scene, 3, False)
    (ca, sa, ea), (cb, sb, eb) = frames
    p0, p1 = _poses(0, ext), _poses(1, ext)

    def refused(code, f, *a):
        with pytest.raises(mloam.MloamError, match=f"error {code}"):
            f(*a)

    cx = _ctx(mloam, 3)
    try:
        cx.set_lidars(3, ext)
        cx.frame_set_next(cb, sb, eb)
        refused(E_STATE, cx.frame_set_next_undistort, p1)  # DISTORTION off
        cx.set_distortion(True, SP)
        refused(E_STATE, cx.frame_set_next_undistort, p1)  # withdrawn by mloam_set_distortion
        cx.frame_set_next(None, None, None)
        refused(E_STATE, cx.frame_set_next_undistort, p1)  # no sweep announced
        for setter in (lambda: cx.set_lidars(3, ext), lambda: cx.set_params(), lambda: cx.set_front_end(RINGS, HORIZON)):
            cx.frame_set_next(cb, sb, eb)
            setter()
            refused(E_STATE, cx.frame_set_next_undistort, p1)  # withdrawn
        cx.frame_set_next(cb, sb, eb)
        refused(E_INVALID, cx.frame_set_next_undistort, p1[:2])
        refused(E_INVALID, cx.frame_set_next_undistort, np.concatenate([p1, p1[:1]]))
        for bad in (np.nan, np.inf):
            q = p1.copy()
            q[2, 4] = bad
            refused(E_INVALID, cx.frame_set_next_undistort, q)
        cx.frame_set_next_undistort(p1)
        cx.frame_undistort(p0)
        cx.frame(ca, sa, ea, scene["surf_map"], scene["corner_map"], scene["traj"][1])
        refused(E_STATE, cx.frame_set_next_undistort, p1)  # the call consumed the announcement
        # the announced poses serve the call that takes the announced sweep only
        cx.frame_set_next(cb, sb, eb)
        cx.frame_set_next_undistort(p1)
        cx.frame_undistort(p0)
        cx.frame(ca, sa, ea, scene["surf_map"], scene["corner_map"], scene["traj"][1])
        refused(E_STATE, cx.frame, ca, sa, ea, scene["surf_map"], scene["corner_map"], scene["traj"][1])
    finally:
        cx.close()
    import torch  # noqa: F401  (torch's NCCL first, as test_keyframe_mapper.py explains)
    cx = _ctx(mloam, 3)
    try:
        cx.set_lidars(3, ext)
        cx.set_distortion(True, SP)
        try:
            cx.comm_init(1, 0, mloam.Context.comm_unique_id())
        except mloam.MloamError as e:
            pytest.skip(f"no NCCL on this machine: {e}")
        cx.frame_set_next(cb, sb, eb)
        refused(E_STATE, cx.frame_set_next_undistort, p1)  # a communicator is attached
    finally:
        cx.close()


def _loop(mloam, announce, with_ua, n_loop=14):
    """The mapper loop with the keyframe store, DISTORTION, the outlier cloud and the registered clouds: per frame the outputs, per saved
    keyframe what the store holds and both global maps."""
    n_lidars = 3
    kf = dict(dist=0.3, orient=2.0, radius=6.0, res=1.0, thr=1e3)
    sc = syn.make_scene()
    traj = syn.trajectory(n_loop)
    ext = syn.rig_extrinsics(n_lidars)
    ext_cov = ua.ext_covariances(n_lidars, seed=7)
    sweeps = [syn.make_multi_sweep(sc, traj[k], n_lidars, 16, 1024, seed=60 + k, ext=ext)[:3] for k in range(n_loop)]
    pu = [mloam.undistort_poses(udl.rot_pose([0.1, 0.2 * (-1) ** k, 1.0], 0.02 + 0.01 * k, [0.4, 0.03 * k, -0.01]), 0, ext, 2)
          for k in range(n_loop)]
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = 16 * n_lidars, 10, 1, 0.5, 1024
    cx = mloam.Context(0, p)
    frames, stored = [], []
    try:
        cx.set_lidars(n_lidars, ext)
        cx.set_uncertainty(with_ua, ext_cov if with_ua else None, COV_MEAS, 1e3)
        cx.set_outlier(0.8)
        cx.set_registered(True)
        cx.set_distortion(True, SP)
        cx.keyframes_init(kf["dist"], kf["orient"], kf["radius"], kf["res"], kf["thr"])
        for k in range(n_loop):
            cx.keyframe_submap(traj[k])
            if announce and k + 1 < n_loop:
                cx.frame_set_next(*sweeps[k + 1])
                cx.frame_set_next_undistort(pu[k + 1])
            if not announce or k == 0:
                cx.frame_undistort(pu[k])
            cloud, ss, se = sweeps[k]
            pose, st = cx.frame(cloud, ss, se, None, None, traj[k], False)
            frames.append(dict(pose=pose, stats=[st[f] for f in STATS], scan=cx.frame_scan(), outlier=cx.frame_outlier(),
                               registered=[cx.frame_registered(w) for w in (mloam.REGISTERED_FULL_RES, mloam.REGISTERED_SURF,
                                                                            mloam.REGISTERED_CORNER)]))
            if not cx.keyframe_save():
                continue
            kid = cx.keyframe_query()[0] - 1
            kpose, kcov, *kscan = cx.keyframe_scan(kid)
            maps = [cx.global_map(mode, center=pose) for mode in (mloam.GLOBAL_MAP_SURROUND, mloam.GLOBAL_MAP_SAVE)]
            stored.append(dict(k=k, pose=kpose, cov=kcov, scan=kscan, outlier=cx.keyframe_outlier(kid), maps=maps, chosen=cx.global_map_chosen()))
        return frames, stored, cx.profile_get("undistort_ahead")[1]
    finally:
        cx.close()


@pytest.mark.parametrize("with_ua", [False, True])
def test_mapper_loop(mloam, with_ua):
    """With the poses announced the loop gives the same frames, the same keyframe store and both global maps bit for bit."""
    want_f, want_s, _ = _loop(mloam, False, with_ua)
    got_f, got_s, ahead = _loop(mloam, True, with_ua)
    assert ahead == len(got_f) - 1
    for k, (a, b) in enumerate(zip(got_f, want_f)):
        assert _equal(a, b), k
    assert len(got_s) == len(want_s) >= 3
    for a, b in zip(got_s, want_s):
        assert a["k"] == b["k"] and np.array_equal(a["pose"], b["pose"]) and np.array_equal(a["cov"], b["cov"]), a["k"]
        assert all(_same(x, y) for x, y in zip(a["scan"], b["scan"])), a["k"]
        assert all(_same(x, y) for x, y in zip(a["outlier"], b["outlier"])), a["k"]
        assert a["chosen"] == b["chosen"], a["k"]
        for ma, mb in zip(a["maps"], b["maps"]):
            assert all(_same(x, y) for x, y in zip(ma, mb)), a["k"]

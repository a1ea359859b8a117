"""GPU tests (-m gpu) of the outlier cloud of segment_cloud: 0 (mloam_set_outlier): the frame's laser_cloud_outlier_cov through the C ABI
against the oracle (oracle/orc_ua.cpp, oracle/orc_mapper.cpp) bit for bit — mloam_frame and mloam_frame_raw, 1 and 3 LiDARs, with_ua on and off, the
look-ahead, graph replay and the stream path, its edges and the trace gate's boundary —, the frame's other results unchanged by it, the
keyframe store's third cloud and the global maps with the outlier appends in the closed mapper loop, and the feature off exactly as before."""
import math
import os

import numpy as np
import pytest

import front_end_lib as fel
import global_map_lib as gl
import mapper_lib as ml
import outlier_lib as ol
import synthetic as syn
import uncertainty_lib as ua

pytestmark = pytest.mark.gpu

E_INVALID, E_STATE = -1, -4
COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])
LEAF = 0.8
RINGS, HORIZON = 16, 512


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def _same(a, b):
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


def _exts(n):
    out = []
    for l in range(n):
        a = 2 * math.pi * l / n
        out.append([0.3 * math.cos(a), 0.3 * math.sin(a), 0.05 * l, 0.0, 0.0, math.sin(a / 4), math.cos(a / 4)])
    return np.array(out, np.float64)


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
        p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = RINGS * n_lidars, 4, 1, 0.5, 1024
        return mloam.Context(0, p)
    finally:
        for k in env:
            os.environ.pop(k)


def _frames(sc, n_lidars, raw, nan_lidar=None, drop_ring0=None):
    """Two sweeps (A, B) of the rig.  ring-ordered: (cloud, scan_start, scan_end); raw: (raw, counts).  nan_lidar: that LiDAR's raw sweep is
    all non-finite (an empty part); drop_ring0: that LiDAR's ring 0 is removed from the ring-ordered sweep."""
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
    """The oracle's inputs of raw frames: the ring-ordered sweep and its ScanInfo (mloam_front_end, on a context of its own)."""
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


def _run(mloam, sc, frames, ext, raw, with_ua, lookahead=False, graphs=True, leaf=LEAF, thr=1e3, n_rounds=3, call_off=False):
    """Frames A, B, A, B, ... (the same arrays, so that graphs capture and replay): per frame (pose, stats, outlier or None, frame_scan) and
    the launch count of each frame."""
    L = ext.shape[0]
    cx = _ctx(mloam, L, None if graphs else {"MLOAM_DISABLE_GRAPHS": "1"})
    ext_cov = ua.ext_covariances(L, seed=3)
    out, launches = [], []
    try:
        cx.set_lidars(L, ext)
        cx.set_uncertainty(with_ua, ext_cov if with_ua else None, COV_MEAS, thr)
        if leaf or call_off:
            cx.set_outlier(leaf)
        if raw:
            cx.set_front_end(RINGS, HORIZON)
        seq = [frames[k % 2] for k in range(2 * n_rounds)]
        for k, fr in enumerate(seq):
            if lookahead and k + 1 < len(seq):
                (cx.frame_set_next_raw if raw else cx.frame_set_next)(*seq[k + 1])
            l0 = cx.launch_count()
            if raw:
                pose, st = cx.frame_raw(fr[0], fr[1], sc["surf_map"], sc["corner_map"], sc["traj"][1 + k % 2])
            else:
                pose, st = cx.frame(fr[0], fr[1], fr[2], sc["surf_map"], sc["corner_map"], sc["traj"][1 + k % 2])
            launches.append(cx.launch_count() - l0)
            out.append((pose, dict(st), cx.frame_outlier() if leaf else None, cx.frame_scan()))
    finally:
        cx.close()
    return out, launches


def _oracle(inputs, ext, with_ua, thr=1e3, leaf=LEAF):
    L = ext.shape[0]
    return [ol.frame_outlier(c, ss, L, ext, ua.ext_covariances(L, seed=3), COV_MEAS, with_ua, thr, leaf) for c, ss, _ in inputs]


@pytest.mark.parametrize("with_ua", [False, True])
@pytest.mark.parametrize("path", ["frame", "raw"])
@pytest.mark.parametrize("n_lidars", [1, 3])
def test_frame_outlier_matches_oracle(mloam, scene, n_lidars, path, with_ua):
    """Bit-identical points, cov_vec and count, on the stream path and from graph replays, with and without the look-ahead; and the
    frame's other results (pose, statistics, mloam_frame_scan) bit-identical to the run without the outlier cloud."""
    raw = path == "raw"
    frames, ext = _frames(scene, n_lidars, raw)
    want = _oracle(_ring_ordered(mloam, frames, n_lidars) if raw else frames, ext, with_ua)
    assert all(w[0].shape[0] >= 1 for w in want)
    off, off_launches = _run(mloam, scene, frames, ext, raw, with_ua, leaf=0.0)
    for graphs in (True, False):
        for lookahead in (False, True):
            got, launches = _run(mloam, scene, frames, ext, raw, with_ua, lookahead=lookahead, graphs=graphs)
            for k, (g, o) in enumerate(zip(got, off)):
                wp, wc = want[k % 2]
                assert _same(g[2][0], wp) and _same(g[2][1], wc), (graphs, lookahead, k)
                assert np.array_equal(g[0], o[0]) and g[1] == o[1], (graphs, lookahead, k)
                assert all(_same(a, b) for a, b in zip(g[3], o[3])), (graphs, lookahead, k)
            if not lookahead:  # one launch more per frame, replayed or not
                assert launches == [n + 1 for n in off_launches], (launches, off_launches)


@pytest.mark.parametrize("with_ua", [False, True])
def test_frame_outlier_edges(mloam, scene, with_ua):
    """A LiDAR whose ring 0 is empty (its first point is ring 1's), an empty LiDAR (all points non-finite), two LiDARs whose first points
    share a 0.8 m voxel."""
    frames, ext = _frames(scene, 3, False, drop_ring0=1)
    want = _oracle(frames, ext, with_ua)
    got, _ = _run(mloam, scene, frames, ext, False, with_ua, n_rounds=2)
    for k, g in enumerate(got):
        assert _same(g[2][0], want[k % 2][0]) and _same(g[2][1], want[k % 2][1]), k
    frames, ext = _frames(scene, 3, True, nan_lidar=1)
    inputs = _ring_ordered(mloam, frames, 3)
    assert [l for l, _ in ol.np_first_points(inputs[0][0], inputs[0][1], 3)] == [0, 2]
    want = _oracle(inputs, ext, with_ua)
    got, _ = _run(mloam, scene, frames, ext, True, with_ua, n_rounds=2)
    for k, g in enumerate(got):
        assert _same(g[2][0], want[k % 2][0]) and _same(g[2][1], want[k % 2][1]), k
        assert 1 not in g[2][0][:, 3].tolist()
    # LiDARs 0 and 1 at one place with one orientation: their first points lie in one voxel and merge
    frames, _ = _frames(scene, 3, False)
    ext = _exts(3)
    ext[1] = ext[0]
    for c, ss, _ in frames:
        c[ss[RINGS] - 5, :3] = c[ss[0] - 5, :3]
    want = _oracle(frames, ext, with_ua)
    got, _ = _run(mloam, scene, frames, ext, False, with_ua, n_rounds=2)
    for k, g in enumerate(got):
        assert want[k % 2][0].shape[0] == 2 and 0.0 not in want[k % 2][0][:, 3].tolist()
        assert _same(g[2][0], want[k % 2][0]) and _same(g[2][1], want[k % 2][1]), k


def _exact_trace(frames, ext, idx):
    """The double trace of the filtered outlier point with the idx-th smallest trace: the smallest threshold that keeps it, found by
    bisection over the doubles with the oracle."""
    L = ext.shape[0]
    _, _, tr = ol.compose_frame(frames[0][0], frames[0][1], L, ext, ua.ext_covariances(L, seed=3), COV_MEAS, True, 1e3, LEAF)
    target = np.sort(tr)[idx]

    def kept(t):
        return ol.frame_outlier(frames[0][0], frames[0][1], L, ext, ua.ext_covariances(L, seed=3), COV_MEAS, True, t, LEAF)[0].shape[0] > idx

    lo, hi = np.float64(target * 0.999).view(np.int64), np.float64(target * 1.001).view(np.int64)
    assert not kept(lo.view(np.float64)) and kept(hi.view(np.float64))
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if kept(np.int64(mid).view(np.float64)):
            hi = mid
        else:
            lo = mid
    return float(np.int64(hi).view(np.float64))


def test_frame_outlier_trace_boundary(mloam, scene):
    """with_ua: a trace exactly at TRACE_THRESHOLD_MAPPING keeps the point, one ulp above it drops the point."""
    frames, ext = _frames(scene, 3, False)
    frames = [frames[0], frames[0]]
    t = _exact_trace(frames, ext, 0)
    for thr, n_kept in ((t, 1), (np.nextafter(t, -np.inf), 0)):
        want = _oracle(frames, ext, True, thr=thr)
        assert want[0][0].shape[0] == n_kept
        got, _ = _run(mloam, scene, frames, ext, False, True, thr=thr, n_rounds=2)
        for g in got:
            assert _same(g[2][0], want[0][0]) and _same(g[2][1], want[0][1])


def test_off_means_off(mloam, scene):
    """mloam_set_outlier(ctx, 0) and never calling it give the same poses, statistics, frame launch counts; frame_outlier then refuses."""
    frames, ext = _frames(scene, 3, False)
    a, la = _run(mloam, scene, frames, ext, False, True, leaf=0.0)
    b, lb = _run(mloam, scene, frames, ext, False, True, leaf=0.0, call_off=True)
    assert la == lb
    for x, y in zip(a, b):
        assert np.array_equal(x[0], y[0]) and x[1] == y[1] and all(_same(p, q) for p, q in zip(x[3], y[3]))


def test_error_paths(mloam, scene):
    frames, ext = _frames(scene, 3, False)
    cx = _ctx(mloam, 3)
    try:
        cx.set_lidars(3, ext)
        for bad in (-0.1, float("nan"), float("inf")):
            with pytest.raises(mloam.MloamError, match=f"error {E_INVALID}"):
                cx.set_outlier(bad)
        cx.set_outlier(LEAF)
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):  # before any frame
            cx.frame_outlier()
        cx.set_outlier(0.0)
        c, ss, se = frames[0]
        cx.frame(c, ss, se, scene["surf_map"], scene["corner_map"], scene["traj"][1])
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):  # the frame ran with it off
            cx.frame_outlier()
        cx.set_outlier(LEAF)
        cx.frame(c, ss, se, scene["surf_map"], scene["corner_map"], scene["traj"][1])
        lib = mloam.lib()
        import ctypes as C

        n = C.c_int(-1)
        assert lib.mloam_frame_outlier(cx._h, None, None, 0, C.byref(n)) == 0 and n.value >= 2
        buf, cov = np.zeros((n.value, 4), np.float32), np.zeros((n.value, 6), np.float32)
        m = C.c_int(-1)  # the capacity rule: too small -> MLOAM_E_INVALID with the size in *n
        assert lib.mloam_frame_outlier(cx._h, mloam._p(buf), None, n.value - 1, C.byref(m)) == E_INVALID and m.value == n.value
        assert lib.mloam_frame_outlier(cx._h, None, mloam._p(cov), n.value - 1, C.byref(m)) == E_INVALID and m.value == n.value
        assert lib.mloam_frame_outlier(cx._h, mloam._p(buf), mloam._p(cov), n.value, C.byref(m)) == 0 and m.value == n.value
        assert _same(buf, cx.frame_outlier()[0])
        cx.keyframes_init(1.0, 10.0, 50.0, 1.0, 1e3)
        with pytest.raises(mloam.MloamError, match=f"error {E_INVALID}"):
            cx.keyframe_outlier(0)
        cx.frame(c, ss, se, None, None, scene["traj"][1], False)
        assert cx.keyframe_save()
        k = C.c_int(-1)
        assert lib.mloam_keyframe_outlier(cx._h, 0, mloam._p(buf), None, 0, C.byref(k)) == E_INVALID and k.value >= 1
    finally:
        cx.close()


def test_communicator_rejected(mloam):
    import torch  # noqa: F401  (torch's NCCL first, as test_keyframe_mapper.py explains)
    cx = _ctx(mloam, 1)
    try:
        try:
            cx.comm_init(1, 0, mloam.Context.comm_unique_id())
        except mloam.MloamError as e:
            pytest.skip(f"no NCCL on this machine: {e}")
        for leaf in (LEAF, 0.0):
            with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
                cx.set_outlier(leaf)
    finally:
        cx.close()


# ---------------------------------------------------------------------------------------------------- closed mapper loop
N_LOOP = 26
KF = dict(dist=0.3, orient=2.0, radius=6.0, res=1.0, thr=1e3)


def _loop(mloam, n_lidars, with_ua, leaf, om=None):
    """The mapper loop of process() on the device (frames with the keyframe store, as test_keyframe_mapper.py runs it) with the outlier cloud
    at `leaf`.  om (a mapper_lib.Mapper): every saved keyframe goes into it as stored on the device, and both global map modes are
    compared with it after every keyframe.  Returns per frame (pose, saved) and the launch count of every mloam_global_map call."""
    sc = syn.make_scene()
    traj = syn.trajectory(N_LOOP)
    ext = syn.rig_extrinsics(n_lidars)
    sweeps = [syn.make_multi_sweep(sc, traj[k], n_lidars, 16, 1024, seed=60 + k, ext=ext) for k in range(N_LOOP)]
    odom = [syn.pose_mul(traj[k], syn.pose7([0.002 * k, -0.001 * k, 0.0], syn.quat_from_rpy(0.0, 0.0, np.radians(0.02 * k)))) for k in range(N_LOOP)]
    ext_cov = ua.ext_covariances(n_lidars, seed=7)
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = 16 * n_lidars, 10, 1, 0.5, 1024
    cx = mloam.Context(0, p)
    out, gm_launches, n_outlier_kf = [], [], 0
    try:
        cx.set_lidars(n_lidars, ext)
        cx.set_outlier(leaf)
        cx.keyframes_init(KF["dist"], KF["orient"], KF["radius"], KF["res"], KF["thr"])
        if om is not None:
            om.set_lidars(ext, ext_cov, COV_MEAS, with_ua)
        wmap_wodom = np.array([0, 0, 0, 0, 0, 0, 1.0])
        for k in range(N_LOOP):
            cloud, ss, se, _ = sweeps[k]
            cx.set_uncertainty(with_ua, ext_cov if with_ua else None, COV_MEAS, 1e3)
            pred = ml.pose_mul(wmap_wodom, odom[k])
            cx.keyframe_submap(pred)
            pose, st = cx.frame(cloud, ss, se, None, None, pred, False)
            wmap_wodom = ml.pose_mul(pose, ml.pose_inv(odom[k]))
            fo = cx.frame_outlier() if leaf else None
            saved = cx.keyframe_save()
            out.append((pose, saved))
            if not saved:
                continue
            kid = cx.keyframe_query()[0] - 1
            ko = cx.keyframe_outlier(kid)
            if leaf:
                want = ol.frame_outlier(cloud, ss, n_lidars, ext, ext_cov, COV_MEAS, with_ua, 1e3, leaf)
                assert _same(fo[0], want[0]) and _same(fo[1], want[1]), k
                assert _same(ko[0], fo[0]) and _same(ko[1], fo[1]), k
                n_outlier_kf += ko[0].shape[0] > 0
            else:
                assert ko[0].shape == (0, 4)
            for mode in (mloam.GLOBAL_MAP_SURROUND, mloam.GLOBAL_MAP_SAVE):
                l0 = cx.launch_count()
                g = cx.global_map(mode, center=pose)
                gm_launches.append(cx.launch_count() - l0)
                if om is None:
                    continue
                if mode == mloam.GLOBAL_MAP_SURROUND:
                    kpose, kcov, sp, _, cp, _ = cx.keyframe_scan(kid)
                    assert om.save(kpose, kcov, sp, cp, outlier=ko[0])[0], k
                leaf_m = p.surf_leaf * (2.0 if mode == mloam.GLOBAL_MAP_SAVE else 1.0)
                ids, want = gl.global_map(om, mode, pose, 1000.0, 10.0, leaf_m)
                assert cx.global_map_chosen() == ids, (k, mode)
                for a, b in zip(g, want):
                    assert _same(a, b), (k, mode)
    finally:
        cx.close()
    return out, gm_launches, n_outlier_kf


@pytest.mark.parametrize("with_ua", [False, True])
@pytest.mark.parametrize("n_lidars", [1, 3])
def test_closed_loop_keyframes_and_global_maps(mloam, n_lidars, with_ua):
    """Every keyframe's stored outlier cloud is its frame's; both global maps after every keyframe equal the oracle's bit for bit; the
    poses and keyframe decisions and the global map launch counts equal those of the run without the outlier cloud."""
    om = ml.Mapper(KF["dist"], KF["orient"], KF["radius"], KF["res"], KF["thr"])
    try:
        on, on_launches, n_kf = _loop(mloam, n_lidars, with_ua, LEAF, om)
    finally:
        om.close()
    off, off_launches, _ = _loop(mloam, n_lidars, with_ua, 0.0)
    assert n_kf >= 4
    assert all(np.array_equal(a[0], b[0]) and a[1] == b[1] for a, b in zip(on, off))
    assert on_launches == off_launches

"""GPU tests (-m gpu) of the PointCloud2 message frames: mloam_front_end_msg / mloam_frame_msg* against mloam_front_end / mloam_frame_raw on
the sweep host/mloam_io.hpp unpackPointCloud2 gives for the same messages — bit for bit, for driver layouts of 16 to 48 bytes, FLOAT64 and
big-endian data, organised clouds with padded rows, non-finite points, both time_field modes; on the stream path and from captured graphs,
with and without the look-ahead, from host and from device bytes — and every error the message entry points return."""
import math

import numpy as np
import pytest

import front_end_lib as fel
import synthetic as syn
import wire_lib as wl

pytestmark = pytest.mark.gpu

E_INVALID, E_STATE = -1, -4
RINGS, HORIZON = 16, 1800
COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def _same(a, b):
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


@pytest.fixture(scope="module")
def scene():
    sc = syn.make_scene()
    surf_map, corner_map = syn.make_submap(sc, 60000)
    return dict(scene=sc, traj=syn.trajectory(6), surf_map=surf_map, corner_map=corner_map)


def _exts(n):
    out = []
    for l in range(n):
        a = 2 * math.pi * l / n
        out.append([0.3 * math.cos(a), 0.3 * math.sin(a), 0.05 * l, 0.0, 0.0, math.sin(a / 4), math.cos(a / 4)])
    return np.array(out, np.float64)


# per LiDAR: (layout, height, row padding)
RIGS = {
    "one": [("xyzi32", 1, 0)],
    "three": [("velodyne22", 1, 0), ("f64be48", 4, 8), ("odd48", 2, 3)],
    "two16": [("xyzt16", 3, 16), ("xyzi32", 1, 0)],
}


def _sweep(sc, pose, rig, seed, time_field, n_nan=20, all_nan=None):
    """One sweep of the rig as messages, and the raw sweep + counts unpackPointCloud2 gives for them (lane 3 = timestamp with time_field)."""
    spec = RIGS[rig]
    ext = _exts(len(spec))
    rng = np.random.default_rng(seed)
    msgs, parts = [], []
    for l, (lay, h, pad) in enumerate(spec):
        raw = fel.raw_sweep(sc, pose, RINGS, HORIZON, seed * 31 + l, time_field=time_field, ext=ext[l] if len(spec) > 1 else None, n_nan=n_nan)
        if all_nan == l:
            raw[:, :3] = np.nan
        m = wl.pack(raw, lay, height=h, row_pad=pad, rng=rng)
        msgs.append(m)
        parts.append(wl.unpack(m, "timestamp" if time_field else None))
    raw = np.ascontiguousarray(np.concatenate(parts))
    counts = np.array([p.shape[0] for p in parts], np.int32)
    return dict(msgs=msgs, raw=raw, counts=counts, ext=ext)


def _layouts(mloam, sw, time_field):
    return [wl.layout(mloam, m, "timestamp" if time_field else None) for m in sw["msgs"]]


def _ctx(mloam, n_lidars, max_inner):
    p = mloam.default_params()
    p.n_scans = n_lidars * RINGS
    p.max_inner = max_inner
    return mloam.Context(0, p)


# ------------------------------------------------------------------------------------------------ front end
@pytest.mark.parametrize("rig", sorted(RIGS))
@pytest.mark.parametrize("time_field", [False, True])
def test_front_end_msg_bit_identical(mloam, scene, rig, time_field):
    n = len(RIGS[rig])
    cx = _ctx(mloam, n, 30)
    try:
        if n > 1:
            cx.set_lidars(n, _exts(n))
        cx.set_front_end(RINGS, HORIZON, 0.5, 0.1, time_field)
        for k, all_nan in enumerate([None, n - 1]):  # the second sweep: one LiDAR's points all non-finite
            sw = _sweep(scene["scene"], scene["traj"][2 + k], rig, 50 + k, time_field, n_nan=30, all_nan=all_nan)
            cx.set_front_end_layout(_layouts(mloam, sw, time_field))
            got, gs, ge = cx.front_end_msg([wl.as_arg(m) for m in sw["msgs"]])
            want, ws, we = cx.front_end(sw["raw"], sw["counts"])
            R = n * RINGS
            assert _same(got, want), (rig, k, got.shape, want.shape)
            assert got.shape[0] > (1000 if n > 1 or k == 0 else -1)  # a one-LiDAR rig whose points are all non-finite: empty
            assert np.array_equal(gs[:R], ws[:R]) and np.array_equal(ge[:R], we[:R])
    finally:
        cx.close()


# ------------------------------------------------------------------------------------------------ frames
def _setup(mloam, cx, rig, sw, time_field, full, undist):
    n = len(RIGS[rig])
    if n > 1:
        cx.set_lidars(n, sw["ext"])
    cx.set_front_end(RINGS, HORIZON, 0.5, 0.1, time_field)
    cx.set_front_end_layout(_layouts(mloam, sw, time_field))  # a raw context keeps its results with layouts set
    if full:
        cx.set_uncertainty(True, np.stack([np.diag([1e-4, 1e-4, 1e-4, 1e-5, 1e-5, 1e-5])] * n), COV_MEAS, 10.0)
        cx.set_outlier(0.8)
        cx.set_registered(True)
    if undist:
        cx.set_distortion(True, 0.1)


def _undist_poses(n, k):
    a = 0.004 * (k + 1)
    return np.array([[0.4 + 0.05 * k, 0.02, 0.01, 0.0, 0.0, math.sin(a), math.cos(a)]] * n)


def _run(mloam, scene, rig, sweeps, inits, time_field, kind, ahead, graph, full=False, undist=False):
    """Frames over the sweeps (twice with graphs: the second pass replays) -> per frame (pose, stats, scan, cov, outlier, registered),
    and the context's launches per frame, "undistort_ahead" and "graph_captures" counts.  kind: raw | msg | msg_dev."""
    import torch
    n = len(RIGS[rig])
    cx = _ctx(mloam, n, 1 if graph else 30)
    try:
        _setup(mloam, cx, rig, sweeps[0], time_field, full, undist)
        sm, cm = scene["surf_map"], scene["corner_map"]
        dev = kind == "msg_dev"
        if dev:
            keep = [[torch.from_numpy(m["data"]).cuda() for m in s["msgs"]] for s in sweeps]
            d_msgs = [[(t.data_ptr(), t.numel(), m["width"], m["height"], m["row_step"]) for t, m in zip(ts, s["msgs"])] for ts, s in zip(keep, sweeps)]
            d_sm, d_cm = torch.from_numpy(sm).cuda(), torch.from_numpy(cm).cuda()
            torch.cuda.synchronize()
        h_msgs = [[wl.as_arg(m) for m in s["msgs"]] for s in sweeps]
        seq = list(range(len(sweeps))) * (2 if graph else 1)
        out, launches = [], []
        announced = False
        for i, k in enumerate(seq):
            if undist and not announced:
                cx.frame_undistort(_undist_poses(n, k))
            nxt = seq[i + 1] if ahead and i + 1 < len(seq) else None
            if nxt is not None:
                if kind == "raw":
                    cx.frame_set_next_raw(sweeps[nxt]["raw"], sweeps[nxt]["counts"])
                elif dev:
                    cx.frame_set_next_msg_device(d_msgs[nxt])
                else:
                    cx.frame_set_next_msg(h_msgs[nxt])
                if undist:
                    cx.frame_set_next_undistort(_undist_poses(n, nxt))
            announced = nxt is not None and undist
            l0 = cx.launch_count()
            if kind == "raw":
                res = cx.frame_raw(sweeps[k]["raw"], sweeps[k]["counts"], sm, cm, inits[k])
            elif dev:
                res = cx.frame_msg_device(d_msgs[k], d_sm.data_ptr(), d_sm.shape[0], d_cm.data_ptr(), d_cm.shape[0], inits[k])
            else:
                res = cx.frame_msg(h_msgs[k], sm, cm, inits[k])
            launches.append(cx.launch_count() - l0)
            pose, st = res
            r = [pose, {x: st[x] for x in ("ran", "n_surf", "n_corner", "lm_iterations", "degenerate", "termination", "final_cost", "n_surf_in",
                                           "n_corner_in")}, cx.frame_scan(), cx.pose_covariance()]
            if full:
                r += [cx.frame_outlier(), [cx.frame_registered(w) for w in range(3)]]
            out.append(r)
        return out, launches, cx.profile_get("undistort_ahead")[1], cx.profile_get("graph_captures")[1]
    finally:
        cx.close()


def _assert_same(a, b):
    assert np.array_equal(a[0], b[0]), (a[0], b[0])
    assert a[1] == b[1], (a[1], b[1])
    assert a[1]["ran"] == 1
    for x, y in zip(a[2], b[2]):
        assert _same(x, y)
    assert np.array_equal(a[3], b[3])
    if len(a) > 4:
        for x, y in zip(a[4], b[4]):
            assert _same(x, y)
        for x, y in zip(a[5], b[5]):
            assert x.shape[0] > 0 and _same(x, y)


def _assert_one_more(got_l, ref_l, ahead):
    """One more launch per frame; with the look-ahead the first frame also unpacks the announced sweep and the last frame takes its
    sweep unpacked, so the run holds one more launch per frame."""
    d = [a - b for a, b in zip(got_l, ref_l)]
    assert sum(d) == len(d) and (ahead or d == [1] * len(d)), (d, got_l, ref_l)
    if ahead:
        assert d[1:-1] == [1] * (len(d) - 2), d


def _sweeps(scene, rig, time_field, k0=2, n=3):
    sweeps = [_sweep(scene["scene"], scene["traj"][k], rig, 10 + k, time_field) for k in range(k0, k0 + n)]
    inits = [syn.perturb_pose(scene["traj"][k], np.random.Generator(np.random.PCG64(7 + k))) for k in range(k0, k0 + n)]
    return sweeps, inits


@pytest.mark.parametrize("rig,time_field,full", [("one", False, False), ("three", True, False), ("three", True, True)])
@pytest.mark.parametrize("graph", [False, True])
def test_frame_msg_bit_identical_to_frame_raw(mloam, scene, rig, time_field, full, graph):
    sweeps, inits = _sweeps(scene, rig, time_field)
    base, base_l, _, base_g = _run(mloam, scene, rig, sweeps, inits, time_field, "raw", False, graph, full)
    raw_ahead, raw_ahead_l, _, raw_ahead_g = _run(mloam, scene, rig, sweeps, inits, time_field, "raw", True, graph, full)
    for kind in ("msg", "msg_dev"):
        for ahead in (False, True):
            got, got_l, _, got_g = _run(mloam, scene, rig, sweeps, inits, time_field, kind, ahead, graph, full)
            for x, y in zip(got, base):
                _assert_same(x, y)
            # one launch more per sweep (the unpack; with the look-ahead it runs in the frame before), as many graph captures as raw frames
            ref_l, ref_g = (raw_ahead_l, raw_ahead_g) if ahead else (base_l, base_g)
            _assert_one_more(got_l, ref_l, ahead)
            assert got_g == ref_g, (kind, ahead, got_g, ref_g)


@pytest.mark.parametrize("graph", [False, True])
def test_distortion_with_announced_poses(mloam, scene, graph):
    rig = "two16"
    sweeps, inits = _sweeps(scene, rig, True)
    base, _, _, _ = _run(mloam, scene, rig, sweeps, inits, True, "raw", False, graph, undist=True)
    raw_ahead, raw_l, raw_ua, raw_g = _run(mloam, scene, rig, sweeps, inits, True, "raw", True, graph, undist=True)
    assert raw_ua > 0
    for kind in ("msg", "msg_dev"):
        got, got_l, got_ua, got_g = _run(mloam, scene, rig, sweeps, inits, True, kind, True, graph, undist=True)
        for x, y in zip(got, base):
            _assert_same(x, y)
        assert got_ua == raw_ua and got_g == raw_g, (kind, got_ua, raw_ua, got_g, raw_g)
        _assert_one_more(got_l, raw_l, True)


def test_lookahead_of_other_bytes_is_not_taken(mloam, scene):
    """The look-ahead matches on the messages' pointers and shapes: the same bytes at another address are unpacked at their call."""
    rig = "three"
    sweeps, inits = _sweeps(scene, rig, True, n=2)
    base, _, _, _ = _run(mloam, scene, rig, sweeps, inits, True, "raw", False, False)
    cx = _ctx(mloam, 3, 30)
    try:
        _setup(mloam, cx, rig, sweeps[0], True, False, False)
        h = [[wl.as_arg(m) for m in s["msgs"]] for s in sweeps]
        copy = [(a[0].copy(),) + tuple(a[1:]) for a in h[1]]
        for announced, taken in ((h[1], h[1]), (h[1], copy), (copy, h[1])):
            cx.frame_set_next_msg(announced)
            r0 = cx.frame_msg(h[0], scene["surf_map"], scene["corner_map"], inits[0])
            r1 = cx.frame_msg(taken, scene["surf_map"], scene["corner_map"], inits[1])
            for got, want in ((r0, base[0]), (r1, base[1])):
                assert np.array_equal(got[0], want[0]) and got[1]["lm_iterations"] == want[1]["lm_iterations"]
    finally:
        cx.close()


# ------------------------------------------------------------------------------------------------ errors
def test_error_paths(mloam, scene):
    rig = "three"
    sw = _sweep(scene["scene"], scene["traj"][2], rig, 3, True)
    sm, cm = scene["surf_map"], scene["corner_map"]
    init = scene["traj"][2]
    h = [wl.as_arg(m) for m in sw["msgs"]]
    lays = _layouts(mloam, sw, True)

    def rc(expect, fn, *a):
        with pytest.raises(mloam.MloamError, match=f"error {expect}"):
            fn(*a)

    cx = _ctx(mloam, 3, 30)
    try:
        cx.set_lidars(3, sw["ext"])
        rc(E_STATE, cx.frame_msg, h, sm, cm, init)  # no front end
        cx.set_front_end(RINGS, HORIZON, 0.5, 0.1, True)
        rc(E_STATE, cx.frame_msg, h, sm, cm, init)  # no layout
        rc(E_STATE, cx.front_end_msg, h)
        cx.set_front_end_layout(lays[:2])
        rc(E_STATE, cx.frame_msg, h, sm, cm, init)  # layouts for 2 LiDARs, the rig has 3
        rc(E_STATE, cx.frame_set_next_msg, h)
        # bad layouts
        bad = [mloam.pc2_layout(22, [(0, 7), (4, 7), (8, 7), (18, 8)]), mloam.pc2_layout(22, [(0, 7), (4, 5), (8, 7)]),
               mloam.pc2_layout(22, [(0, 7), (4, 7), (-1, 7)]), mloam.pc2_layout(0, [(0, 7), (4, 7), (8, 7)]),
               mloam.pc2_layout(2048, [(0, 7), (4, 7), (8, 7)])]
        for b in bad:
            rc(E_INVALID, cx.set_front_end_layout, [b] * 3)
        cx.set_front_end_layout(lays)
        # time_field 1 without a lane-3 field
        cx.set_front_end_layout(_layouts(mloam, sw, False))
        rc(E_INVALID, cx.frame_msg, h, sm, cm, init)
        rc(E_INVALID, cx.front_end_msg, h)
        cx.set_front_end_layout(lays)
        # messages: zero points, row_step < width x point_step, size < height x row_step
        m1 = sw["msgs"][1]
        cases = [(m1["data"], 0, m1["height"], m1["row_step"]), (m1["data"], m1["width"], 0, m1["row_step"]),
                 (m1["data"], m1["width"], m1["height"], m1["width"] * m1["point_step"] - 1),
                 (m1["data"][:-1], m1["width"], m1["height"], m1["row_step"])]
        for case in cases:
            hh = list(h)
            hh[1] = case
            rc(E_INVALID, cx.frame_msg, hh, sm, cm, init)
            rc(E_INVALID, cx.frame_set_next_msg, hh)
            rc(E_INVALID, cx.front_end_msg, hh)
            rc(E_INVALID, cx.frame_msg_device, [(1 << 40, a[0].nbytes, a[1], a[2], a[3]) for a in hh], 0, 0, 0, 0, init)
        rc(E_INVALID, cx.frame_msg_device, [(0, a[0].nbytes, a[1], a[2], a[3]) for a in h], 0, 0, 0, 0, init)  # NULL data
        # the same calls pass once the messages are right
        pose, st = cx.frame_msg(h, sm, cm, init)
        assert st["ran"] == 1
    finally:
        cx.close()


def test_communicator_rejected(mloam, scene):
    import torch  # noqa: F401  (torch's NCCL first, see test_keyframe_mapper.py)
    sw = _sweep(scene["scene"], scene["traj"][2], "one", 3, False)
    cx = _ctx(mloam, 1, 30)
    try:
        try:
            cx.comm_init(1, 0, mloam.Context.comm_unique_id())
        except mloam.MloamError as e:
            pytest.skip(f"no NCCL on this machine: {e}")
        cx.set_front_end(RINGS, HORIZON)
        cx.set_front_end_layout(_layouts(mloam, sw, False))
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
            cx.frame_msg([wl.as_arg(m) for m in sw["msgs"]], scene["surf_map"], scene["corner_map"], scene["traj"][2])
    finally:
        cx.close()

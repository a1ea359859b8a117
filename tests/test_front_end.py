"""GPU tests (-m gpu) of the raw-sweep front end: removeNaN + calTimestamp (mloam_cal_timestamp) and the rig-batched range-image projection
(mloam_front_end) against the host restatements, and mloam_frame_raw* against mloam_frame fed with the same front end computed on the host —
bit for bit, on the stream path and under graph capture / replay, with and without the raw look-ahead."""
import math

import numpy as np
import pytest

import front_end_lib as fel
import synthetic as syn

pytestmark = pytest.mark.gpu

E_INVALID, E_STATE = -1, -4
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
    """Sensor -> base extrinsics of an n-LiDAR rig: spread around the base, yawed."""
    out = []
    for l in range(n):
        a = 2 * math.pi * l / n
        out.append([0.3 * math.cos(a), 0.3 * math.sin(a), 0.05 * l, 0.0, 0.0, math.sin(a / 4), math.cos(a / 4)])
    return np.array(out, np.float64)


def _rig_sweep(sc, pose, n_lidars, rings, horizon, seed, time_field=False, n_nan=0):
    ext = _exts(n_lidars)
    parts = [fel.raw_sweep(sc, pose, rings, horizon, seed * 31 + l, time_field=time_field, ext=ext[l] if n_lidars > 1 else None, n_nan=n_nan)
             for l in range(n_lidars)]
    return np.ascontiguousarray(np.concatenate(parts)), np.array([p.shape[0] for p in parts], np.int32), ext


def _ctx(mloam, rings_total, max_inner=30):
    p = mloam.default_params()
    p.n_scans = rings_total
    p.max_inner = max_inner
    return mloam.Context(0, p)


# ------------------------------------------------------------------------------------------------ calTimestamp
@pytest.mark.parametrize("time_field", [False, True])
def test_cal_timestamp_bit_exact(ctx, scene, time_field):
    rng = np.random.default_rng(4)
    for k in range(6):
        raw = fel.raw_sweep(scene["scene"], scene["traj"][k % 6], 32, 1800, seed=k, az0=rng.uniform(-math.pi, math.pi), time_field=time_field,
                            n_nan=40 * k)
        if k == 5:
            raw[0, 1] = np.nan  # first and last points dropped
            raw[-1, 2] = np.inf
        got = ctx.cal_timestamp(raw, time_field, 0.1)
        want = fel.cal_timestamp(raw, time_field, 0.1)
        assert _same(got, want), (k, got.shape, want.shape)
    for raw in (raw[:1], raw[1:3], np.full((3, 4), np.nan, np.float32)):
        assert _same(ctx.cal_timestamp(raw, time_field, 0.1), fel.cal_timestamp(raw, time_field, 0.1))


# ------------------------------------------------------------------------------------------------ batched projection
@pytest.mark.parametrize("n_lidars,rings", [(2, 32), (4, 16), (16, 16)])
def test_batched_projection_equals_per_lidar_oracle(mloam, scene, n_lidars, rings):
    raw, counts, ext = _rig_sweep(scene["scene"], scene["traj"][2], n_lidars, rings, 1800, seed=n_lidars, n_nan=25)
    cx = _ctx(mloam, n_lidars * rings)
    try:
        cx.set_lidars(n_lidars, ext)
        for tf in (False, True):
            cx.set_front_end(rings, 1800, 0.5, 0.1, tf)
            got, gs, ge = cx.front_end(raw, counts)
            want, ws, we = fel.front_end(raw, counts, rings, 1800, 0.5, 0.1, tf)
            R = n_lidars * rings
            assert _same(got, want), (tf, got.shape, want.shape)
            assert np.array_equal(gs[:R], ws) and np.array_equal(ge[:R], we)
    finally:
        cx.close()


# ------------------------------------------------------------------------------------------------ mloam_frame_raw vs mloam_frame
SHAPES = {  # KITTI: 1 x 64, horizon 4000, ROI 1 m; Oxford: 2 x 32, horizon 1800, timestamp overload
    "kitti": dict(n_lidars=1, rings=64, horizon=4000, roi=1.0, time_field=False),
    "oxford": dict(n_lidars=2, rings=32, horizon=1800, roi=0.5, time_field=True),
}


def _setup(cx, s, ext, with_ua):
    if s["n_lidars"] > 1:
        cx.set_lidars(s["n_lidars"], ext)
    cx.set_front_end(s["rings"], s["horizon"], s["roi"], 0.1, s["time_field"])
    if with_ua:
        ec = np.stack([np.diag([1e-4, 1e-4, 1e-4, 1e-5, 1e-5, 1e-5])] * s["n_lidars"])
        cx.set_uncertainty(True, ec, COV_MEAS, 10.0)


def _results(cx, out):
    pose, st = out
    return pose, {k: st[k] for k in ("ran", "n_surf", "n_corner", "lm_iterations", "degenerate", "termination", "final_cost", "n_surf_in",
                                     "n_corner_in")}, cx.frame_scan(), cx.pose_covariance()


def _assert_same(a, b):
    assert np.array_equal(a[0], b[0]), (a[0], b[0])
    assert a[1] == b[1], (a[1], b[1])
    for x, y in zip(a[2], b[2]):
        assert _same(x, y)
    assert np.array_equal(a[3], b[3])


@pytest.mark.parametrize("shape", ["kitti", "oxford"])
@pytest.mark.parametrize("rebuild", [True, False])
@pytest.mark.parametrize("graph", [False, True])
def test_frame_raw_bit_identical_to_frame(mloam, scene, shape, rebuild, graph):
    s = SHAPES[shape]
    R = s["n_lidars"] * s["rings"]
    sweeps = [_rig_sweep(scene["scene"], scene["traj"][k], s["n_lidars"], s["rings"], s["horizon"], seed=10 + k, time_field=s["time_field"], n_nan=15)
              for k in (2, 3)]
    ext = sweeps[0][2]
    sm, cm = scene["surf_map"], scene["corner_map"]
    a, b = _ctx(mloam, R, 1 if graph else 30), _ctx(mloam, R, 1 if graph else 30)
    try:
        for with_ua in (False, True):
            for cx in (a, b):
                _setup(cx, s, ext, with_ua)
                if not rebuild:
                    cx.map_build(mloam.MAP_SURF, sm)
                    cx.map_build(mloam.MAP_CORNER, cm)
            # four frames per sweep: stream path, then (graph) capture and replays
            for k, (raw, counts, _) in enumerate(sweeps):
                ref_cloud, ss, se = fel.front_end(raw, counts, s["rings"], s["horizon"], s["roi"], 0.1, s["time_field"])
                init = syn.perturb_pose(scene["traj"][2 + k], np.random.Generator(np.random.PCG64(7 + k)))
                for rep in range(4 if graph else 1):
                    got = _results(a, a.frame_raw(raw, counts, sm, cm, init, rebuild_maps=rebuild))
                    want = _results(b, b.frame(ref_cloud, ss, se, sm, cm, init, rebuild_maps=rebuild))
                    assert got[1]["ran"] == 1
                    _assert_same(got, want)
                    if with_ua:
                        assert np.any(got[3] != 0)
    finally:
        a.close()
        b.close()


def test_frame_raw_device_matches_host(mloam, scene):
    import torch
    s = SHAPES["oxford"]
    raw, counts, ext = _rig_sweep(scene["scene"], scene["traj"][3], 2, 32, 1800, seed=5, time_field=True, n_nan=10)
    init = syn.perturb_pose(scene["traj"][3], np.random.Generator(np.random.PCG64(1)))
    a, b = _ctx(mloam, 64, 1), _ctx(mloam, 64, 1)
    try:
        for cx in (a, b):
            _setup(cx, s, ext, False)
        d_raw = torch.from_numpy(raw).cuda()
        d_sm, d_cm = torch.from_numpy(scene["surf_map"]).cuda(), torch.from_numpy(scene["corner_map"]).cuda()
        torch.cuda.synchronize()
        for _ in range(3):
            got = a.frame_raw_device(d_raw.data_ptr(), counts, d_sm.data_ptr(), d_sm.shape[0], d_cm.data_ptr(), d_cm.shape[0], init)
            want = b.frame_raw(raw, counts, scene["surf_map"], scene["corner_map"], init)
            assert np.array_equal(got[0], want[0]) and got[1]["lm_iterations"] == want[1]["lm_iterations"]
    finally:
        a.close()
        b.close()


# ------------------------------------------------------------------------------------------------ raw look-ahead
def test_raw_lookahead_same_results(mloam, scene):
    import torch
    s = SHAPES["oxford"]
    sweeps = [_rig_sweep(scene["scene"], scene["traj"][k], 2, 32, 1800, seed=20 + k, time_field=True) for k in range(1, 6)]
    ext = sweeps[0][2]
    inits = [syn.perturb_pose(scene["traj"][k], np.random.Generator(np.random.PCG64(30 + k))) for k in range(1, 6)]
    sm, cm = scene["surf_map"], scene["corner_map"]

    def run(announce, device=False):
        cx = _ctx(mloam, 64, 1)
        try:
            _setup(cx, s, ext, True)
            d = [torch.from_numpy(r).cuda() for r, _, _ in sweeps] if device else None
            d_sm, d_cm = (torch.from_numpy(sm).cuda(), torch.from_numpy(cm).cuda()) if device else (None, None)
            torch.cuda.synchronize()
            out = []
            for rep in range(2):  # the second pass replays captured graphs
                for k in range(len(sweeps)):
                    nxt = announce(k)
                    if nxt is not None:
                        r, c, _ = sweeps[nxt]
                        if device:
                            cx.frame_set_next_raw_device(d[nxt].data_ptr(), c)
                        else:
                            cx.frame_set_next_raw(r, c)
                    raw, counts, _ = sweeps[k]
                    if device:
                        res = cx.frame_raw_device(d[k].data_ptr(), counts, d_sm.data_ptr(), d_sm.shape[0], d_cm.data_ptr(), d_cm.shape[0], inits[k])
                    else:
                        res = cx.frame_raw(raw, counts, sm, cm, inits[k])
                    out.append(_results(cx, res))
            return out
        finally:
            cx.close()

    base = run(lambda k: None)
    in_order = run(lambda k: k + 1 if k + 1 < len(sweeps) else None)
    broken = run(lambda k: (k + 2) % len(sweeps) if k % 2 else k)  # announces a later sweep, or the current one again
    dev = run(lambda k: k + 1 if k + 1 < len(sweeps) else None, device=True)
    for o in (in_order, broken, dev):
        for x, y in zip(o, base):
            _assert_same(x, y)


# ------------------------------------------------------------------------------------------------ launches
def test_front_end_launches_batched(mloam, scene):
    """mloam_frame_raw launches a constant number of kernels more than mloam_frame on the same rig, for 1, 2 and 4 LiDARs."""
    diffs = []
    for n in (1, 2, 4):
        raw, counts, ext = _rig_sweep(scene["scene"], scene["traj"][2], n, 16, 1800, seed=40 + n)
        ref_cloud, ss, se = fel.front_end(raw, counts, 16, 1800, 0.5, 0.1, False)
        init = syn.perturb_pose(scene["traj"][2], np.random.Generator(np.random.PCG64(2)))
        a, b = _ctx(mloam, 16 * n), _ctx(mloam, 16 * n)
        try:
            for cx in (a, b):
                cx.set_lidars(n, ext)
                cx.set_front_end(16, 1800, 0.5, 0.1, False)
            la, lb = a.launch_count(), b.launch_count()
            pa, _ = a.frame_raw(raw, counts, scene["surf_map"], scene["corner_map"], init)
            pb, _ = b.frame(ref_cloud, ss, se, scene["surf_map"], scene["corner_map"], init)
            assert np.array_equal(pa, pb)
            diffs.append((a.launch_count() - la) - (b.launch_count() - lb))
        finally:
            a.close()
            b.close()
    assert diffs[0] > 0 and diffs == [diffs[0]] * 3, diffs


# ------------------------------------------------------------------------------------------------ errors
def test_error_paths(mloam, scene):
    raw, counts, ext = _rig_sweep(scene["scene"], scene["traj"][2], 2, 16, 1800, seed=3)
    sm, cm = scene["surf_map"], scene["corner_map"]
    init = scene["traj"][2]
    cx = _ctx(mloam, 32)
    try:
        cx.set_lidars(2, ext)
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):  # no front end configured
            cx.frame_raw(raw, counts, sm, cm, init)
        with pytest.raises(mloam.MloamError, match=f"error {E_INVALID}"):
            cx.set_front_end(40, 1800)
        cx.set_front_end(16, 1800)
        with pytest.raises(mloam.MloamError, match=f"error {E_INVALID}"):  # an empty sweep (the node's empty_check)
            cx.frame_raw(raw, np.array([counts.sum(), 0], np.int32), sm, cm, init)
        with pytest.raises(mloam.MloamError, match=f"error {E_INVALID}"):
            cx.frame_set_next_raw(raw, np.array([0, counts.sum()], np.int32))
        cx.set_params(max_ring_points=1024)  # below horizon_scans
        with pytest.raises(mloam.MloamError, match=f"error {E_INVALID}"):
            cx.frame_raw(raw, counts, sm, cm, init)
        with pytest.raises(mloam.MloamError, match=f"error {E_INVALID}"):
            cx.set_front_end(16, 1800)
        cx.set_params(max_ring_points=2048)
        pose, st = cx.frame_raw(raw, counts, sm, cm, init)
        assert st["ran"] == 1
    finally:
        cx.close()


def test_communicator_rejected(mloam, scene):
    import torch  # noqa: F401  (torch's NCCL first, see test_keyframe_mapper.py)
    raw, counts, _ = _rig_sweep(scene["scene"], scene["traj"][2], 1, 16, 1800, seed=3)
    cx = _ctx(mloam, 16)
    try:
        try:
            cx.comm_init(1, 0, mloam.Context.comm_unique_id())
        except mloam.MloamError as e:
            pytest.skip(f"no NCCL on this machine: {e}")
        cx.set_front_end(16, 1800)
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
            cx.frame_raw(raw, counts, scene["surf_map"], scene["corner_map"], scene["traj"][2])
    finally:
        cx.close()

"""One context, the solves and frames of the library interleaved on it: every result is bit-identical to the same call on a fresh context
given the same map builds.  A call's settings — the tracker's minimum correspondences and degeneracy threshold, the speculative
schedule's deferred fit, the pose covariance request of the with_ua solves, a raw sweep's layout, the look-ahead state of a frame graph —
must not leak into the next call."""
import numpy as np
import pytest

import front_end_lib as fel
import oracle_lib as orc
import synthetic as syn

pytestmark = pytest.mark.gpu

COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])


@pytest.fixture(scope="module")
def data():
    scene = syn.make_scene()
    traj = syn.trajectory(6)
    surf_map, corner_map = syn.make_submap(scene, 50000)
    sweeps = [syn.make_sweep(scene, traj[k], 16, 1024, seed=k) for k in (3, 4)]
    feats = [orc.extract_cloud(*s) for s in sweeps]
    cs, _ = orc.voxel_grid(feats[1]["corner_points_less_sharp"], 0.2, True)
    sf, _ = orc.voxel_grid(feats[1]["surf_points_less_flat"], 0.4, True)
    init = syn.perturb_pose(traj[4], np.random.Generator(np.random.PCG64(11)))
    # normal-equation rows: the scan's features matched against the submaps at the initial pose
    vs, cfs, _ = orc.match_from_map("s", surf_map, sf, init)
    vc, cfc, _ = orc.match_from_map("c", corner_map, cs, init)
    rows = (np.array([ord("s")] * int(vs.sum()) + [ord("c")] * int(vc.sum()), np.uint8),
            np.concatenate([sf[vs][:, :3], cs[vc][:, :3]]).astype(np.float64),
            np.concatenate([cfs[vs], cfc[vc]]).astype(np.float32).astype(np.float64))
    rng = np.random.default_rng(5)
    cov6 = [np.abs(rng.normal(0, 1e-3, (x.shape[0], 6))).astype(np.float32) for x in (sf, cs)]
    raw = fel.raw_sweep(scene, traj[4], 16, 1800, seed=6, n_nan=10)
    return dict(surf_map=surf_map, corner_map=corner_map, sweep=sweeps[1], prev=feats[0], cur=feats[1], surf_scan=sf, corner_scan=cs,
                init=np.asarray(init, np.float64), rows=rows, cov6=cov6, raw=raw)


def _ctx(mloam):
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = 16, 10, 1, 0.5, 0
    cx = mloam.Context(0, p)
    cx.set_front_end(16, 1800, 0.5, 0.1, False)
    return cx


def _maps(cx, d):
    cx.map_build(1, d["surf_map"], 0.5)
    cx.map_build(0, d["corner_map"], 0.5)


def _solve(cx, out):
    pose, st = out
    return [pose, {k: st[k] for k in ("ran", "n_surf", "n_corner", "lm_iterations", "degenerate", "termination", "final_cost", "n_surf_in",
                                      "n_corner_in")}, st["eig"], st["H"], cx.pose_covariance()]


def _scan2map(cx, d):
    return _solve(cx, cx.scan2map(d["surf_scan"], d["corner_scan"], d["init"]))


def _track(cx, d):
    p, c = d["prev"], d["cur"]
    init = np.array([0.02, -0.01, 0.0, 0.0, 0.0, 0.0, 1.0])
    return _solve(cx, cx.track_cloud(p["corner_points_less_sharp"], p["surf_points_less_flat"], c["corner_points_sharp"], c["surf_points_flat"],
                                     init))


def _normal_equations(cx, d):
    return list(cx.normal_equations(*d["rows"], 1.0, 0.1, d["init"]))


def _scan2map_ua(cx, d):
    return _solve(cx, cx.scan2map_ua(d["surf_scan"], d["cov6"][0], d["corner_scan"], d["cov6"][1], d["init"]))


def _frame(cx, d):
    cloud, ss, se = d["sweep"]
    return _solve(cx, cx.frame(cloud, ss, se, d["surf_map"], d["corner_map"], d["init"]))


def _frame_raw(cx, d):
    return _solve(cx, cx.frame_raw(d["raw"], [d["raw"].shape[0]], d["surf_map"], d["corner_map"], d["init"]))


def _assert_same(got, want, what):
    for a, b in zip(got, want):
        if isinstance(a, dict):
            assert a == b, (what, a, b)
        else:
            assert np.array_equal(np.asarray(a), np.asarray(b)), (what, a, b)


def test_calls_leave_no_settings_behind(mloam, data):
    """scan2map (speculative schedule: max_inner 1), track_cloud (min_corr 10, eig_thre 0), normal_equations, scan2map_ua (reports a
    covariance), five frames, a raw frame and track_cloud again.  A frame's look-ahead parity is part of its graph key and alternates,
    so frames 3 and 4 capture graphs and frame 5 replays the graph of frame 3."""
    steps = [("scan2map", _scan2map, True), ("track_cloud", _track, False), ("normal_equations", _normal_equations, False),
             ("scan2map_ua", _scan2map_ua, True)] + [(f"frame {k}", _frame, False) for k in range(1, 6)] + \
            [("frame_raw", _frame_raw, False), ("track_cloud again", _track, False)]
    shared = _ctx(mloam)
    try:
        _maps(shared, data)
        got = [(name, run(shared, data)) for name, run, _ in steps]
    finally:
        shared.close()
    for (name, run, needs_maps), (_, res) in zip(steps, got):
        fresh = _ctx(mloam)
        try:
            if needs_maps:
                _maps(fresh, data)
            want = run(fresh, data)
        finally:
            fresh.close()
        _assert_same(res, want, name)
    assert got[0][1][1]["ran"] == 1 and got[0][1][1]["n_surf"] > 500
    assert got[1][1][1]["ran"] == 1 and got[1][1][1]["n_surf"] > 0
    assert np.any(got[3][1][4] != 0)  # scan2map_ua reports H^-1
    assert not np.any(got[4][1][4])  # ... and the frame after it does not
    assert all(r[1]["ran"] == 1 for _, r in got[4:10])

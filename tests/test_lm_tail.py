"""The LM step of every solve runs on one warp of the tail block (lm_advance_warp, solve_kernels.cu); MLOAM_LM_TAIL=serial keeps the
single-thread state machine it replaces.  Both do the same floating-point operations in the same order, so every result must be
bit-identical: pose, H / H0, eigenvalues, termination, iteration and match counts, cost and the with_ua pose covariance.  The cases
cover the fused tail (stream path and graph replay), the speculative schedule's candidate tail, a degenerate solve (eigen-solver and
remapped V_update), the tracker (several LM iterations per solve), a solve skipped under min_corr and with_ua."""
import os

import numpy as np
import pytest

import bench
import oracle_lib as orc
import synthetic as syn

pytestmark = pytest.mark.gpu

KEYS = ("ran", "n_surf", "n_corner", "lm_iterations", "degenerate", "termination", "final_cost", "n_surf_in", "n_corner_in")


def _context(mloam, p, tail):
    if tail:
        os.environ["MLOAM_LM_TAIL"] = tail
    try:
        return mloam.Context(0, p)
    finally:
        os.environ.pop("MLOAM_LM_TAIL", None)


def _result(cx, out):
    pose, st = out
    return [pose, {k: st[k] for k in KEYS}, st["eig"], st["H"], cx.pose_covariance()]


def _assert_same(got, want):
    for a, b in zip(got, want):
        if isinstance(a, dict):
            assert a == b, (a, b)
        else:
            assert np.array_equal(np.asarray(a), np.asarray(b)), (a, b)


def _both(mloam, p, run):
    """run(cx) -> list of results, on a context with the serial tail and on one with the warp tail."""
    res = []
    for tail in ("serial", None):
        cx = _context(mloam, p, tail)
        try:
            res.append(run(cx))
        finally:
            cx.close()
    return res


@pytest.fixture(scope="module")
def c1():
    scene = syn.make_scene()
    traj = syn.trajectory(6)
    surf_map, corner_map = syn.make_submap(scene, 50000)
    sweeps = [syn.make_sweep(scene, traj[k], 16, 1024, seed=k) for k in (3, 4)]
    feats = [orc.extract_cloud(*s) for s in sweeps]
    cs, _ = orc.voxel_grid(feats[1]["corner_points_less_sharp"], 0.2, True)
    sf, _ = orc.voxel_grid(feats[1]["surf_points_less_flat"], 0.4, True)
    init = np.asarray(syn.perturb_pose(traj[4], np.random.Generator(np.random.PCG64(11))), np.float64)
    rng = np.random.default_rng(5)
    cov6 = [np.abs(rng.normal(0, 1e-3, (x.shape[0], 6))).astype(np.float32) for x in (sf, cs)]
    return dict(surf_map=surf_map, corner_map=corner_map, sweep=sweeps[1], prev=feats[0], cur=feats[1], surf_scan=sf, corner_scan=cs,
                init=init, cov6=cov6)


def _c1_params(mloam, inner=1):
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = 16, 10, inner, 0.5, 0
    return p


def _maps(cx, surf_map, corner_map):
    cx.map_build(1, surf_map, 0.5)
    cx.map_build(0, corner_map, 0.5)


def test_full_size_frames_stream_and_replay(mloam):
    """C2 (64 x 2048 sweep, 1M-point keyframe submap, 10 GN iterations): the first frame runs on the stream and is captured, the
    next ones replay the graph."""
    cfg = bench.CONFIGS["C2"]
    wl = bench.make_workload(syn, cfg, 1, 0, 1)
    fr = wl["frames"][0]
    g = fr["groups"][0]
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = cfg["rings"], cfg["gn_iters"], 1, 0.0, cfg["horizon"]
    serial, warp = _both(mloam, p, lambda cx: [_result(cx, cx.frame(g["cloud"], g["ss"], g["se"], wl["surf_map"], wl["corner_map"],
                                                                       fr["init"], rebuild)) for rebuild in (True, False, False)])
    for a, b in zip(serial, warp):
        assert a[1]["ran"] == 1 and a[1]["n_surf"] > 1000
        _assert_same(b, a)


@pytest.mark.parametrize("inner", [1, 3])
def test_c1_frames_and_scan2map(mloam, c1, inner):
    """C1 frames (the speculative schedule with one LM iteration, the serial one with three) and scan2map with a poor guess, whose
    last GN iterations reject their step."""
    def run(cx):
        cloud, ss, se = c1["sweep"]
        out = [_result(cx, cx.frame(cloud, ss, se, c1["surf_map"], c1["corner_map"], c1["init"], rebuild)) for rebuild in (True, False)]
        init = c1["init"].copy()
        init[:3] += 0.6
        out.append(_result(cx, cx.scan2map(c1["surf_scan"], c1["corner_scan"], init)))
        return out
    serial, warp = _both(mloam, _c1_params(mloam, inner), run)
    for a, b in zip(serial, warp):
        assert a[1]["ran"] == 1
        _assert_same(b, a)


def test_degenerate_map(mloam):
    """A floor plane and one line along x: translation along x is unconstrained, so the Cholesky test of H - eig_thre I fails, the
    eigen-solver runs and the step goes through the remapped V_update."""
    g = np.arange(-10.0, 10.0, 0.2)
    xx, yy = np.meshgrid(g, g)
    plane = np.stack([xx.ravel(), yy.ravel(), np.zeros(xx.size), np.zeros(xx.size)], 1).astype(np.float32)
    line = np.stack([np.arange(-10.0, 10.0, 0.05), np.full(400, 2.0), np.full(400, 1.0), np.zeros(400)], 1).astype(np.float32)
    rng = np.random.default_rng(3)
    surf_scan = plane[rng.choice(plane.shape[0], 800, replace=False)].copy()
    surf_scan[:, :2] += rng.uniform(-0.05, 0.05, (800, 2)).astype(np.float32)
    corner_scan = line[rng.choice(line.shape[0], 60, replace=False)].copy()
    corner_scan[:, 0] += rng.uniform(-0.02, 0.02, 60).astype(np.float32)
    init = np.array([0.05, -0.03, 0.04, 0.004, -0.003, 0.002, 1.0])
    init[3:] /= np.linalg.norm(init[3:])

    def run(cx):
        _maps(cx, plane, line)
        return [_result(cx, cx.scan2map(surf_scan, corner_scan, init))]
    serial, warp = _both(mloam, _c1_params(mloam), run)
    assert serial[0][1]["ran"] == 1 and serial[0][1]["degenerate"] == 1, serial[0][1]
    _assert_same(warp[0], serial[0])


def test_tracker_and_min_corr(mloam, c1):
    """track_cloud runs several LM iterations per solve (rejected steps shrink the radius); a tracker solve with a handful of features
    falls under min_corr and is skipped with the pose untouched."""
    p, c = c1["prev"], c1["cur"]
    init = np.array([0.02, -0.01, 0.0, 0.0, 0.0, 0.0, 1.0])

    def run(cx):
        out = [_result(cx, cx.track_cloud(p["corner_points_less_sharp"], p["surf_points_less_flat"], c["corner_points_sharp"],
                                          c["surf_points_flat"], init))]
        out.append(_result(cx, cx.track_cloud(p["corner_points_less_sharp"], p["surf_points_less_flat"], c["corner_points_sharp"][:2],
                                               c["surf_points_flat"][:3], init)))
        return out
    serial, warp = _both(mloam, _c1_params(mloam), run)
    assert serial[0][1]["ran"] == 1 and serial[0][1]["lm_iterations"] > 2, serial[0][1]
    assert serial[1][1]["termination"] == 5, serial[1][1]
    for a, b in zip(serial, warp):
        _assert_same(b, a)


def test_with_ua_pose_covariance(mloam, c1):
    """scan2map_ua reports the pose covariance H^-1 of the last evaluation (LMState::H of the two-pass tail)."""
    def run(cx):
        _maps(cx, c1["surf_map"], c1["corner_map"])
        return [_result(cx, cx.scan2map_ua(c1["surf_scan"], c1["cov6"][0], c1["corner_scan"], c1["cov6"][1], c1["init"]))]
    serial, warp = _both(mloam, _c1_params(mloam), run)
    assert serial[0][1]["ran"] == 1 and np.abs(serial[0][4]).sum() > 0
    _assert_same(warp[0], serial[0])

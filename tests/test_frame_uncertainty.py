"""Uncertainty-aware frames (with_ua = true, the configuration of every mapper launch file of the reference) through
mloam_frame: per-point uncertainty + trace gate after the scan filters, sqrt_info-weighted solve, pose covariance H^-1 at the
returned pose (lidar_mapper_keyframe.cpp:356-421, :541-560, :600-632) and the gated keyframe scans — against the oracle's
orc_ua_frame_multi (oracle/orc_ua.cpp), across schedules, graph capture / replay, speculation and look-ahead, and into the submap assembly."""
import os

import numpy as np
import pytest

import bench
import oracle_lib as orc
import uncertainty_lib as ua
import synthetic as syn

pytestmark = pytest.mark.gpu

POSE_TOL_T = 1e-4  # metres   (as tests/test_gpu_parity.py)
POSE_TOL_R = 1e-4  # radians
COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])
SCHEDULES = {"bench": (10, 1), "reference": (2, 30)}  # (max_outer, max_inner): graph + speculation | stream path


def _case(name):
    """C1: 16 x 1024 sweep, 50k-point submap; C2: 64 x 2048, 1M-point keyframe submap (bench workload); C4: 4 x 64 x 2048 RV rig,
    5M-point submap.  ua_scale: of the extrinsic covariances, so that >= 20 % of the gated features get sqrt_info < 1.  `merged`: the context gets the rig extrinsics (intensity = laser id); otherwise intensity keeps the ring."""
    scene = syn.make_scene()
    if name == "C1":
        traj = syn.trajectory(6)
        surf_map, corner_map = syn.make_submap(scene, 50000)
        cloud, ss, se = syn.make_sweep(scene, traj[4], 16, 1024, seed=4)
        init = syn.perturb_pose(traj[4], np.random.Generator(np.random.PCG64(11)))
        return dict(surf_map=surf_map, corner_map=corner_map, cloud=cloud, ss=ss, se=se, ext=syn.rig_extrinsics(1), init=init, rings=16,
                    horizon=1024, merged=False, cell=0.5, ua_scale=1.0)
    if name == "C2":
        wl = bench.make_workload(syn, bench.CONFIGS["C2"], 1, 0, 1)
        fr = wl["frames"][0]
        g = fr["groups"][0]
        return dict(surf_map=wl["surf_map"], corner_map=wl["corner_map"], cloud=g["cloud"], ss=g["ss"], se=g["se"], ext=g["ext"], init=fr["init"],
                    rings=64, horizon=2048, merged=False, cell=0.0, ua_scale=1.6)
    traj = syn.trajectory(8)
    surf_map, corner_map = syn.make_submap(scene, 5_000_000)
    cloud, ss, se, ext = syn.make_multi_sweep(scene, traj[6], 4, 64, 2048, seed=21)
    init = syn.perturb_pose(traj[6], np.random.Generator(np.random.PCG64(23)))
    return dict(surf_map=surf_map, corner_map=corner_map, cloud=cloud, ss=ss, se=se, ext=ext, init=init, rings=64, horizon=2048, merged=True,
                cell=0.25, ua_scale=1.3)


_CASES = {}


def case(name):
    if name not in _CASES:
        _CASES[name] = _case(name)
    return _CASES[name]


def _trace(c6):
    return c6[:, 0].astype(np.float64) + c6[:, 3].astype(np.float64) + c6[:, 5].astype(np.float64)


def _sqrt_info(c6):
    return np.minimum(np.sqrt(1.0 / _trace(c6)) / 3.0, 1.0)


def _threshold(c, ext_cov, q=0.8):
    """A TRACE_THRESHOLD_MAPPING between two traces at the q-quantile of the oracle's (ungated) scan covariances."""
    L = c["ext"].shape[0]
    _, _, _, sc = ua.frame_multi_ua(c["cloud"], c["ss"], c["se"], L, c["ext"], ext_cov, COV_MEAS, 1e30, c["surf_map"][:10], c["corner_map"][:10],
                                     c["init"])
    tr = np.sort(np.concatenate([_trace(sc["surf_cov6"]), _trace(sc["corner_cov6"])]))
    k = int(q * tr.shape[0])
    return 0.5 * (tr[k - 1] + tr[k]), tr.shape[0]


def _params(mloam, c, outer, inner, **kw):
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = c["rings"], outer, inner, c["cell"], c["horizon"]
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _context(mloam, p, c, env=None):
    env = env or {}
    for k, v in env.items():
        os.environ[k] = v
    try:
        cx = mloam.Context(0, p)
    finally:
        for k in env:
            os.environ.pop(k)
    if c["merged"]:
        cx.set_lidars(c["ext"].shape[0], c["ext"])
    return cx


def _run(cx, c, ext_cov, thr, rebuild=True, with_ua=True):
    if with_ua:
        cx.set_uncertainty(True, ext_cov, COV_MEAS, thr)
    else:
        cx.set_uncertainty(False)
    pose, st = cx.frame(c["cloud"], c["ss"], c["se"], c["surf_map"], c["corner_map"], c["init"], rebuild)
    return pose, st, cx.pose_covariance(), cx.frame_scan()


def _oracle(c, ext_cov, thr, outer, inner, gf=None):
    o = orc.default_opts()
    o[orc.O_MAX_OUTER], o[orc.O_MAX_INNER] = outer, inner
    if gf:
        o[orc.O_GF_METHOD], o[orc.O_GF_RATIO], o[orc.O_GF_SEED] = gf[0], gf[1], 0
    return ua.frame_multi_ua(c["cloud"], c["ss"], c["se"], c["ext"].shape[0], c["ext"], ext_cov, COV_MEAS, thr, c["surf_map"], c["corner_map"],
                              c["init"], o)


def _same(a, b):
    (pa, sa, ca, _), (pb, sb, cb, _) = a, b
    assert np.array_equal(pa, pb) and np.array_equal(ca, cb)
    for k in ("ran", "n_surf", "n_corner", "lm_iterations", "termination", "degenerate", "n_surf_in", "n_corner_in", "final_cost"):
        assert sa[k] == sb[k], k
    assert np.array_equal(np.asarray(sa["H"]), np.asarray(sb["H"]))


def _check_vs_oracle(g, r, c, n_pre):
    pose, st, cov, (sp, sc6, cp, cc6) = g
    rpose, rst, rcov, rs = r
    assert st["ran"] == 1 and rst["ran"] == 1
    # not vacuous: a real share of the features is down-weighted, and the gate drops 5-30 % of the scan
    n_kept = rst["n_surf_in"] + rst["n_corner_in"]
    assert 0.05 <= 1.0 - n_kept / n_pre <= 0.30, (n_kept, n_pre)
    assert (_sqrt_info(np.concatenate([rs["surf_cov6"], rs["corner_cov6"]])) < 1.0).mean() >= 0.2
    assert st["n_surf_in"] == rst["n_surf_in"] and st["n_corner_in"] == rst["n_corner_in"]
    assert st["n_surf"] == int(rst["n_surf"]) and st["n_corner"] == int(rst["n_corner"])
    dt, dr = syn.pose_err(pose, rpose)
    assert dt <= POSE_TOL_T and dr <= POSE_TOL_R, (dt, dr)
    # the gated scans (saveKeyframe's laser_cloud_*_cov): points bit-identical, cov_vec to float rounding
    cols = slice(0, 4) if c["merged"] else slice(0, 3)  # without the rig merge intensity keeps the ring (the oracle's is the laser id 0)
    assert np.array_equal(sp[:, cols], rs["surf"][:, cols]) and np.array_equal(cp[:, cols], rs["corner"][:, cols])
    assert np.allclose(sc6, rs["surf_cov6"], rtol=2e-6, atol=1e-12) and np.allclose(cc6, rs["corner_cov6"], rtol=2e-6, atol=1e-12)
    # pose_wmap_curr.cov_ = H^-1 at the returned pose
    assert np.linalg.norm(cov - rcov) <= 1e-9 * np.linalg.norm(rcov), np.linalg.norm(cov - rcov) / np.linalg.norm(rcov)
    assert np.linalg.norm(cov - cov.T) <= 1e-9 * np.linalg.norm(cov)
    assert np.all(np.linalg.eigvalsh(0.5 * (cov + cov.T)) > 0)


@pytest.mark.parametrize("sched", ["bench", "reference"])
@pytest.mark.parametrize("name", ["C1", "C2", "C4"])
def test_frame_ua_matches_oracle(mloam, name, sched):
    """Each configuration and schedule against the oracle; with the bench schedule the stream path, the graph capture and the
    replay give bit-identical pose, statistics and covariance."""
    c = case(name)
    outer, inner = SCHEDULES[sched]
    ext_cov = ua.ext_covariances(c["ext"].shape[0], seed=5, scale=c["ua_scale"])
    thr, n_pre = _threshold(c, ext_cov)
    cx = _context(mloam, _params(mloam, c, outer, inner), c)
    try:
        runs = [_run(cx, c, ext_cov, thr, rebuild) for rebuild in ((True, True, True) if inner == 1 else (True,))]
    finally:
        cx.close()
    for r in runs[1:]:
        _same(runs[0], r)
    _check_vs_oracle(runs[0], _oracle(c, ext_cov, thr, outer, inner), c, n_pre)


def test_frame_ua_fuse_and_lookahead_bit_identical(mloam):
    """C2 with the bench schedule: the serial schedule (MLOAM_FUSE_ITER=0) and the speculative one, with and without the sweep
    look-ahead, give the same pose, statistics, covariance and gated scans bit for bit."""
    c = case("C2")
    ext_cov = ua.ext_covariances(1, seed=5, scale=c["ua_scale"])
    thr, _ = _threshold(c, ext_cov)
    res = []
    for fuse in ("0", "1"):
        cx = _context(mloam, _params(mloam, c, 10, 1), c, {"MLOAM_FUSE_ITER": fuse})
        try:
            plain = [_run(cx, c, ext_cov, thr, rb) for rb in (True, False, False)]
            ahead = []
            for rb in (True, False, False):  # the same sweep announced as the next one: the next call takes the prefetched features
                cx.frame_set_next(c["cloud"], c["ss"], c["se"])
                ahead.append(_run(cx, c, ext_cov, thr, rb))
        finally:
            cx.close()
        res.append(plain + ahead)
    ref = res[0][0]
    for r in res[0] + res[1]:
        _same(ref, r)
        for a, b in zip(ref[3], r[3]):
            assert np.array_equal(a, b)


def test_scan2map_ua_covariance_with_rejected_last_step(mloam):
    """The C1 poor-guess case whose last GN iterations leave the pose unchanged (a rejected step): cov = H^-1 at x, not at the
    candidate; serial and speculative schedules bit-identical, and equal to the oracle's covariance."""
    scene = syn.make_scene()
    traj = syn.trajectory(6)
    surf_map, corner_map = syn.make_submap(scene, 50000)
    cloud, ss, se = syn.make_sweep(scene, traj[4], 16, 1024, seed=4)
    f = orc.extract_cloud(cloud, ss, se)
    cs, _ = orc.voxel_grid(f["corner_points_less_sharp"], 0.2, True)
    sf, _ = orc.voxel_grid(f["surf_points_less_flat"], 0.4, True)
    init = np.array(syn.perturb_pose(traj[4], np.random.Generator(np.random.PCG64(11))), dtype=np.float64)
    init[:3] += 0.6
    ident = np.array([0, 0, 0, 0, 0, 0, 1.0])
    ext_cov = ua.ext_covariances(1, seed=3)[0]
    sc6, cc6 = orc.point_uncertainty(sf, ident, ext_cov, COV_MEAS), orc.point_uncertainty(cs, ident, ext_cov, COV_MEAS)
    p = mloam.default_params()
    p.max_outer, p.max_inner, p.map_cell = 10, 1, 0.5
    res = []
    for fuse in ("0", "1"):
        os.environ["MLOAM_FUSE_ITER"] = fuse
        try:
            cx = mloam.Context(0, p)
        finally:
            os.environ.pop("MLOAM_FUSE_ITER")
        try:
            cx.map_build(1, surf_map, 0.5)
            cx.map_build(0, corner_map, 0.5)
            pose, st = cx.scan2map_ua(sf, sc6, cs, cc6, init)
            res.append((pose, st, cx.pose_covariance(), None))
            pose0, _ = cx.scan2map(sf, cs, init)
            assert not cx.pose_covariance().any()  # with_ua = false: zero (:621)
        finally:
            cx.close()
    _same(*res)
    pose, st, cov, _ = res[1]
    assert st["termination"] in (0, 1), st["termination"]  # the last step was not taken
    o = orc.default_opts()
    o[orc.O_MAX_OUTER], o[orc.O_MAX_INNER] = 10, 1
    rpose, rst, rcov, rH = ua.scan2map_ua_cov(surf_map, corner_map, sf, sc6, cs, cc6, init, o)
    assert max(syn.pose_err(pose, rpose)) <= POSE_TOL_T
    assert np.linalg.norm(cov - rcov) <= 1e-9 * np.linalg.norm(rcov), np.linalg.norm(cov - rcov) / np.linalg.norm(rcov)


def test_covariances_changed_between_replays(mloam):
    """New covariances and threshold between two replays of the captured frame: the replay reads the staged values — its result
    equals a fresh context without graphs given the same inputs, and differs from the previous covariances' result."""
    c = case("C1")
    p = _params(mloam, c, 10, 1)
    cov_a, cov_b = ua.ext_covariances(1, seed=5), ua.ext_covariances(1, seed=9, scale=1.3)
    thr_a, _ = _threshold(c, cov_a)
    thr_b, _ = _threshold(c, cov_b, 0.85)
    cx = _context(mloam, p, c)
    try:
        a = [_run(cx, c, cov_a, thr_a, rb) for rb in (True, True, True)]  # stream path, capture, replay
        b = _run(cx, c, cov_b, thr_b, True)  # replays the same graph with the new staged values
        b2 = _run(cx, c, cov_b, thr_b, True)
    finally:
        cx.close()
    _same(a[1], a[2])
    _same(b, b2)
    fresh = _context(mloam, p, c, {"MLOAM_DISABLE_GRAPHS": "1"})
    try:
        ref_b = _run(fresh, c, cov_b, thr_b, True)
    finally:
        fresh.close()
    _same(b, ref_b)
    for x, y in zip(b[3], ref_b[3]):
        assert np.array_equal(x, y)
    assert not np.array_equal(a[2][2], b[2]) and a[2][1]["n_surf_in"] != b[1]["n_surf_in"]


def test_zero_covariance_matches_plain_frame_and_zero_cases(mloam):
    """Zero extrinsic covariances and a threshold above every trace: every weight clamps to 1 as with with_ua = false, so pose and
    statistics are bit-identical to the plain frame.  The pose covariance is zero without with_ua and for a map-gated frame."""
    c = case("C1")
    for outer, inner in SCHEDULES.values():
        cx = _context(mloam, _params(mloam, c, outer, inner), c)
        try:
            plain = [_run(cx, c, None, 0.0, True, with_ua=False) for _ in range(3 if inner == 1 else 1)]
            assert not plain[-1][2].any() and not plain[-1][3][1].any()
            ua_runs = [_run(cx, c, np.zeros((1, 6, 6)), 1e30, True) for _ in range(3 if inner == 1 else 1)]
            # map gate (:429): a submap with <= 50 surf points -> the frame does not run, covariance zero (:637)
            cx.set_uncertainty(True, ua.ext_covariances(1, seed=5), COV_MEAS, 1e30)
            _, st_g = cx.frame(c["cloud"], c["ss"], c["se"], c["surf_map"][:40], c["corner_map"], c["init"], True)
            assert st_g["ran"] == 0 and not cx.pose_covariance().any()
        finally:
            cx.close()
        pp, sp_, _, _ = plain[-1]
        pu, su, cu, _ = ua_runs[-1]
        assert np.array_equal(pp, pu)
        for k in ("ran", "n_surf", "n_corner", "lm_iterations", "termination", "degenerate", "n_surf_in", "n_corner_in", "final_cost"):
            assert sp_[k] == su[k], k
        assert np.array_equal(np.asarray(sp_["H"]), np.asarray(su["H"]))
        assert cu.any()


def test_frame_ua_good_feature_selection(mloam):
    """gd_fix with ratio 0.2 sees the per-point covariances (lidar_mapper.h:130-174): the same selections as the oracle."""
    c = case("C1")
    ext_cov = ua.ext_covariances(1, seed=5)
    thr, n_pre = _threshold(c, ext_cov)
    cx = _context(mloam, _params(mloam, c, 5, 1, gf_method=3, gf_ratio=0.2, gf_seed=0), c)
    try:
        g = _run(cx, c, ext_cov, thr, True)
    finally:
        cx.close()
    r = _oracle(c, ext_cov, thr, 5, 1, gf=(3, 0.2))
    _check_vs_oracle(g, r, c, n_pre)


def test_frame_scan_and_pose_covariance_feed_submap_assembly(mloam, ctx):
    """Loop closure of the uncertainty-aware mapper: a frame's gated scan with its pose and covariance (saveKeyframe) ->
    compoundPoseWithCov with each extrinsic -> mloam_submap_assemble, bit-identical to the oracle's submap from the same inputs."""
    c = case("C4")
    L = c["ext"].shape[0]
    ext_cov = ua.ext_covariances(L, seed=5, scale=c["ua_scale"])
    thr, _ = _threshold(c, ext_cov)
    cx = _context(mloam, _params(mloam, c, 10, 1), c)
    try:
        pose, st, cov, (sp, sc6, cp, cc6) = _run(cx, c, ext_cov, thr, True)
    finally:
        cx.close()
    assert st["ran"] == 1 and cov.any() and sp.shape[0] > 1000
    pcs, ccs = [], []
    for l in range(L):
        pc, cc = mloam.Context.compound_pose_cov(pose, cov, c["ext"][l], ext_cov[l])
        pcs.append(pc), ccs.append(cc)
    pcs, ccs = np.array(pcs), np.array(ccs)
    keyframe = sp  # stored as the frame left it: base frame, laser id in the intensity
    thr_a, leaf, thr_f = 50.0, 0.4, 50.0
    gp, gc = ctx.submap_assemble(1, [keyframe], pose[None], c["ext"], pcs[None], ccs[None], COV_MEAS, leaf, True, thr_a, thr_f, 0.5)
    p, c6, tr = orc.cloud_uct_associate(keyframe, pose, c["ext"], pcs, ccs, COV_MEAS, True, thr_a)
    rp, rc, rt, ok = orc.voxel_grid_cov(p, c6, tr, leaf, thr_f)
    assert ok and 0 < rp.shape[0] < keyframe.shape[0]
    assert gp.shape == rp.shape and np.array_equal(gp, rp)
    assert np.allclose(gc, rc, rtol=1e-5, atol=1e-12)

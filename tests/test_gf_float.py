"""gd_float on the GPU (-m gpu), through the C ABI: mloam_full_hessian against the serial sum and the oracle, and sequences of
solve calls with mloam_set_gf_float against the oracle's policy (lidar_mapper_keyframe.cpp:456-495) frame by frame."""
import os

import numpy as np
import pytest

import gf_float_lib as gfl
import oracle_lib as orc
import synthetic as syn

pytestmark = pytest.mark.gpu

POSE_TOL_T = 1e-4  # metres, the parity tolerance of tests/test_gpu_parity.py
POSE_TOL_R = 1e-4  # radians
# gf_deg_factor against the oracle's: the device's Jacobian rows agree with the oracle's to 1e-9 (test_gpu_parity.py), and so does their sum
FACTOR_TOL = 1e-7
N_FRAMES = 35
RATIO = 0.375  # exact in the float of params.gf_ratio, so the oracle (double) and the device see one number


@pytest.fixture(scope="module")
def c1():
    """Config C1: 16-ring x 1024 sweep, 50k-point submap."""
    scene = syn.make_scene()
    traj = syn.trajectory(6)
    surf_map, corner_map = syn.make_submap(scene, 50000)
    cloud, ss, se = syn.make_sweep(scene, traj[4], 16, 1024, seed=4)
    f = orc.extract_cloud(cloud, ss, se)
    cs, _ = orc.voxel_grid(f["corner_points_less_sharp"], 0.2, True)
    sf, _ = orc.voxel_grid(f["surf_points_less_flat"], 0.4, True)
    init = syn.perturb_pose(traj[4], np.random.Generator(np.random.PCG64(11)))
    return dict(scene=scene, truth=traj[4], surf_map=surf_map, corner_map=corner_map, cloud=np.ascontiguousarray(cloud, np.float32),
                ss=np.ascontiguousarray(ss, np.int32), se=np.ascontiguousarray(se, np.int32), corner_scan=cs, surf_scan=sf, init=init)


def _inits(truth, n):
    """Pose guesses of n frames: near the truth, except frames 15..24, which start 1.5 m off (fewer matches: a smaller factor)."""
    rng = np.random.Generator(np.random.PCG64(3))
    out = []
    for k in range(1, n + 1):
        x = syn.perturb_pose(truth, rng)
        if 15 <= k <= 24:
            x[0] += 1.5
        out.append(x)
    return out


def _opts(max_outer=2, max_inner=1):
    o = orc.default_opts()
    o[orc.O_MAX_OUTER], o[orc.O_MAX_INNER] = max_outer, max_inner
    o[orc.O_GF_METHOD], o[orc.O_GF_RATIO], o[orc.O_GF_SEED] = orc.GF_GD, RATIO, 7
    return o


def _params(mloam, max_outer=2, max_inner=1):
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = 16, max_outer, max_inner, 0.5, 1024
    p.gf_method, p.gf_ratio, p.gf_seed = 3, RATIO, 7
    return p


def _oracle_run(call, inits, thre):
    """call(x) -> (pose, stats) runs one oracle frame; returns the per-frame log with the policy's state after each."""
    gfl.gf_float_set(True, thre, RATIO)
    log = []
    try:
        for x in inits:
            pose, st = call(x)
            log.append(dict(gfl.gf_float_get(), pose=pose, n_surf=int(st["n_surf"]), n_corner=int(st["n_corner"])))
    finally:
        gfl.gf_float_set(False)
    return log


def _gpu_run(c, call, inits, thre):
    c.set_gf_float(True, thre)
    log = []
    for x in inits:
        l0 = c.launch_count()
        pose, st = call(x)
        log.append(dict(c.gf_float_report(), pose=pose, n_surf=st["n_surf"], n_corner=st["n_corner"], launches=c.launch_count() - l0))
    return log


def _check(got, ref, want_ratios=None):
    for k, (g, r) in enumerate(zip(got, ref), 1):
        assert g["frame_cnt"] == r["frame_cnt"] == k
        assert g["evaluated"] == r["evaluated"] == (k % 10 == 0), k
        assert g["ratio_cur"] == r["ratio_cur"], (k, g["ratio_cur"], r["ratio_cur"])
        assert g["total_feat_num"] == r["total_feat_num"], k
        assert abs(g["deg_factor"] - r["deg_factor"]) <= FACTOR_TOL * max(1.0, abs(r["deg_factor"])), (k, g["deg_factor"], r["deg_factor"])
        assert (g["n_surf"], g["n_corner"]) == (r["n_surf"], r["n_corner"]), k
        dt, dr = syn.pose_err(g["pose"], r["pose"])
        assert dt <= POSE_TOL_T and dr <= POSE_TOL_R, (k, dt, dr)
    if want_ratios is not None:
        assert [g["ratio_cur"] for g in got] == want_ratios


def _threshold_between(ref):
    f10, f20, f30 = (ref[k - 1]["deg_factor"] for k in (10, 20, 30))
    assert f20 < min(f10, f30)
    return 0.5 * (f20 + min(f10, f30))


SWITCH = [RATIO] * 19 + [0.8] * 10 + [RATIO] * 6  # ini -> 0.8 at frame 20 -> ini at frame 30


# ------------------------------------------------------------------------------------------------ evalFullHessian
@pytest.mark.parametrize("with_cov", [False, True])
def test_full_hessian_is_the_serial_sum(ctx, c1, with_cov):
    ctx.map_build(1, c1["surf_map"], 0.5)
    ctx.map_build(0, c1["corner_map"], 0.5)
    rng = np.random.default_rng(9)
    H, n = None, 0
    Hn, Ho, no = None, None, 0
    for kind, slot, mp, scan in (("s", 1, c1["surf_map"], c1["surf_scan"]), ("c", 0, c1["corner_map"], c1["corner_scan"])):
        cov6 = None
        if with_cov:  # point covariances with traces on both sides of the sqrt_info clamp
            d = rng.uniform(0.001, 0.2, (scan.shape[0], 3))
            cov6 = np.zeros((scan.shape[0], 6), np.float32)
            cov6[:, [0, 3, 5]] = d
        rows = ctx.good_features(slot, kind, scan, c1["init"], orc.GF_WO, 1.0, 0, cov6=cov6)  # the device's rows and matched flags
        one, n_one = ctx.full_hessian(slot, kind, scan, c1["init"], cov6=cov6)
        assert n_one == int(rows["matched"].sum()) > 50
        assert one.tobytes() == gfl.serial_hessian(rows["jaco"], rows["matched"]).tobytes()  # index order, one product and one add each
        ref, n_ref = gfl.full_hessian(kind, mp, scan, c1["init"], cov6=cov6)
        assert n_one == n_ref and np.allclose(one, ref, rtol=1e-9, atol=1e-12)
        H, n = ctx.full_hessian(slot, kind, scan, c1["init"], cov6=cov6, H=H, feat_num=n)  # the chain of :463-467
        Hn = gfl.serial_hessian(rows["jaco"], rows["matched"], Hn)
        Ho, no = gfl.full_hessian(kind, mp, scan, c1["init"], cov6=cov6, H=Ho, feat_num=no)
    assert H.tobytes() == Hn.tobytes() and n == no
    assert np.allclose(H, Ho, rtol=1e-9, atol=1e-12) and np.array_equal(H, H.T)
    # nothing to add: an empty set, and a set without any map support
    H0, n0 = ctx.full_hessian(1, "s", np.zeros((0, 4), np.float32), c1["init"], H=H, feat_num=n)
    far = c1["surf_scan"].copy()
    far[:, :3] += 1000.0
    H1, n1 = ctx.full_hessian(1, "s", far, c1["init"], H=H, feat_num=n)
    assert H0.tobytes() == H.tobytes() == H1.tobytes() and n0 == n1 == n


def test_full_hessian_far_from_the_origin(ctx, c1):
    off = np.array([4096.0, -2048.0, 512.0], np.float32)
    sm = c1["surf_map"].copy()
    sm[:, :3] += off
    x = c1["init"].copy()
    x[:3] += off
    ctx.map_build(1, sm, 0.5)
    rows = ctx.good_features(1, "s", c1["surf_scan"], x, orc.GF_WO, 1.0, 0)
    H, n = ctx.full_hessian(1, "s", c1["surf_scan"], x)
    assert n == int(rows["matched"].sum()) > 50 and H.tobytes() == gfl.serial_hessian(rows["jaco"], rows["matched"]).tobytes()
    ref, n_ref = gfl.full_hessian("s", sm, c1["surf_scan"], x)
    assert n == n_ref and np.allclose(H, ref, rtol=1e-7, atol=1e-9)


# ------------------------------------------------------------------------------------------------ the policy over a run of frames
def test_frames_follow_the_oracle_policy(mloam, c1):
    """mloam_frame, one LiDAR: 35 frames on the same sweep and maps, the pose guess moving; the ratio goes ini -> 0.8 -> ini."""
    inits = _inits(c1["truth"], N_FRAMES)
    # the oracle's frame: extractCloud and downsampleCurrentScan (the fixture's scans), then the gd_float scan2MapOptimization
    ocall = lambda x: gfl.scan2map(c1["surf_map"], c1["corner_map"], c1["surf_scan"], c1["corner_scan"], x, _opts())
    thre = _threshold_between(_oracle_run(ocall, inits, -1e30))
    ref = _oracle_run(ocall, inits, thre)
    c = mloam.Context(0, _params(mloam))
    got = _gpu_run(c, lambda x: c.frame(c1["cloud"], c1["ss"], c1["se"], c1["surf_map"], c1["corner_map"], x), inits, thre)
    _check(got, ref, SWITCH)
    # the frames ran from two kinds of graph; a third and fourth exist only for the halves of the feature double buffer
    assert c.profile_get("graph_captures")[1] <= 4 and c.profile_get("graph_capture_failures")[1] == 0
    other = {g["launches"] for k, g in enumerate(got, 1) if k % 10 and k > 4}
    evalf = {g["launches"] for k, g in enumerate(got, 1) if k % 10 == 0}
    assert len(other) == 1 and evalf == {next(iter(other)) + 1}  # an evaluation frame is one launch more: k_gf_full_hessian
    # a changed threshold re-captures nothing (checked before any other context allocates: the allocation epoch is shared)
    caps = c.profile_get("graph_captures")[1]
    c.set_gf_float_threshold(1e30)  # every evaluation from here on is "degenerate": 0.8
    more = [c.frame(c1["cloud"], c1["ss"], c1["se"], c1["surf_map"], c1["corner_map"], x) for x in inits[:5]]
    assert c.gf_float_report()["frame_cnt"] == 40 and c.gf_float_report()["ratio_cur"] == 0.8 and more[4][1]["ran"] == 1
    assert c.profile_get("graph_captures")[1] == caps
    c.close()
    # the same frames with gd_float off: the launches of a non-evaluation frame, and gd_fix's results
    off = mloam.Context(0, _params(mloam))
    l0 = off.launch_count()
    pose_off, st_off = off.frame(c1["cloud"], c1["ss"], c1["se"], c1["surf_map"], c1["corner_map"], inits[0])
    assert off.launch_count() - l0 == got[0]["launches"]
    assert pose_off.tobytes() == got[0]["pose"].tobytes()  # before the first evaluation the ratio is ini: gd_fix bit for bit
    off.close()
    # the stream path gives the same bits as the graphs
    os.environ["MLOAM_DISABLE_GRAPHS"] = "1"
    try:
        plain = mloam.Context(0, _params(mloam))
    finally:
        os.environ.pop("MLOAM_DISABLE_GRAPHS")
    ref_plain = _gpu_run(plain, lambda x: plain.frame(c1["cloud"], c1["ss"], c1["se"], c1["surf_map"], c1["corner_map"], x), inits, thre)
    plain.close()
    for g, r in zip(got, ref_plain):
        assert g["pose"].tobytes() == r["pose"].tobytes() and g["deg_factor"] == r["deg_factor"] and g["ratio_cur"] == r["ratio_cur"]


def test_threshold_boundary_on_the_device(mloam, c1):
    """`gf_deg_factor > MAP_DEG_THRE` with the threshold a float: at the float at or above the device's own factor the ratio is 0.8, one
    float ulp below it is ini."""
    inits = _inits(c1["truth"], 10)
    out = {}
    for name in ("free", "at", "below"):
        c = mloam.Context(0, _params(mloam))
        c.map_build(1, c1["surf_map"], 0.5)
        c.map_build(0, c1["corner_map"], 0.5)
        thre = -1e30 if name == "free" else out["thresholds"][name]
        log = _gpu_run(c, lambda x: c.scan2map(c1["surf_scan"], c1["corner_scan"], x), inits, thre)
        c.close()
        out[name] = log[9]
        if name == "free":
            at, below = gfl.float_at_or_above(log[9]["deg_factor"])
            out["thresholds"] = {"at": float(at), "below": float(below)}
    assert out["free"]["evaluated"] and out["free"]["ratio_cur"] == RATIO
    assert out["at"]["deg_factor"] == out["below"]["deg_factor"] == out["free"]["deg_factor"]
    assert out["at"]["ratio_cur"] == 0.8 and out["below"]["ratio_cur"] == RATIO


def test_rig_frames_follow_the_oracle_policy(mloam):
    """mloam_frame on a 3-LiDAR rig (the merge of the three sweeps feeds one selection and one evaluation)."""
    scene = syn.make_scene()
    traj = syn.trajectory(6)
    surf_map, corner_map = syn.make_submap(scene, 50000)
    cloud, ss, se, ext = syn.make_multi_sweep(scene, traj[4], 3, 16, 1024, seed=41)
    cloud, ss, se = np.ascontiguousarray(cloud, np.float32), np.ascontiguousarray(ss, np.int32), np.ascontiguousarray(se, np.int32)
    inits = _inits(traj[4], N_FRAMES)
    corner_scan, surf_scan = orc.prepare_multi(cloud, ss, se, 3, ext)  # per-LiDAR extraction, merge, the two scan filters
    ocall = lambda x: gfl.scan2map(surf_map, corner_map, surf_scan, corner_scan, x, _opts())
    thre = _threshold_between(_oracle_run(ocall, inits, -1e30))
    ref = _oracle_run(ocall, inits, thre)
    c = mloam.Context(0, _params(mloam))
    c.set_lidars(3, ext)
    got = _gpu_run(c, lambda x: c.frame(cloud, ss, se, surf_map, corner_map, x), inits, thre)
    c.close()
    _check(got, ref, SWITCH)


def test_scan2map_ua_follows_the_oracle_policy(mloam, c1):
    """with_ua: the rows carry sqrt_info of each point's covariance (mloam_scan2map_ua), LM iterations polled by the host (max_inner 4)."""
    rng = np.random.default_rng(2)
    cov = []
    for scan in (c1["surf_scan"], c1["corner_scan"]):
        c6 = np.zeros((scan.shape[0], 6), np.float32)
        c6[:, [0, 3, 5]] = rng.uniform(0.001, 0.2, (scan.shape[0], 3))
        cov.append(c6)
    inits = _inits(c1["truth"], N_FRAMES)
    ocall = lambda x: gfl.scan2map(c1["surf_map"], c1["corner_map"], c1["surf_scan"], c1["corner_scan"], x, _opts(2, 4), cov[0], cov[1])
    thre = _threshold_between(_oracle_run(ocall, inits, -1e30))
    ref = _oracle_run(ocall, inits, thre)
    c = mloam.Context(0, _params(mloam, 2, 4))
    c.map_build(1, c1["surf_map"], 0.5)
    c.map_build(0, c1["corner_map"], 0.5)
    got = _gpu_run(c, lambda x: c.scan2map_ua(c1["surf_scan"], cov[0], c1["corner_scan"], cov[1], x), inits, thre)
    c.close()
    _check(got, ref, SWITCH)


def test_lookahead_and_map_gate(mloam, c1):
    """Announcing the next sweep changes nothing; a frame that fails the map gate advances frame_cnt without evaluating."""
    inits = _inits(c1["truth"], 12)
    frame = lambda c, x, cm: c.frame(c1["cloud"], c1["ss"], c1["se"], c1["surf_map"], cm, x)
    tiny = np.ascontiguousarray(c1["corner_map"][:5])
    logs = []
    for announce in (False, True):
        c = mloam.Context(0, _params(mloam))
        c.set_gf_float(True, -1e30)
        log = []
        for k, x in enumerate(inits, 1):
            if announce:
                c.frame_set_next(c1["cloud"], c1["ss"], c1["se"])
            pose, st = frame(c, x, tiny if k == 10 else c1["corner_map"])
            log.append(dict(c.gf_float_report(), pose=pose, ran=st["ran"]))
        c.close()
        logs.append(log)
    for a, b in zip(*logs):
        assert a["pose"].tobytes() == b["pose"].tobytes() and a["frame_cnt"] == b["frame_cnt"] and a["evaluated"] == b["evaluated"]
    assert [g["frame_cnt"] for g in logs[0]] == list(range(1, 13))
    assert logs[0][9]["ran"] == 0 and not any(g["evaluated"] for g in logs[0])
    assert all(g["ratio_cur"] == RATIO and g["deg_factor"] == 0.0 for g in logs[0])


def test_errors(mloam, c1):
    p = _params(mloam)
    p.gf_method = 1
    c = mloam.Context(0, p)
    with pytest.raises(Exception):
        c.set_gf_float(True, 0.0)  # gd_float is gd_fix with an adaptive ratio: gf_method must be 3
    with pytest.raises(Exception):
        c.gf_float_report()        # the mode is off
    c.set_gf_float(False)
    c.set_params(gf_method=3)
    c.set_gf_float(True, 0.0)
    with pytest.raises(Exception):
        c.gf_float_report()        # no solve call yet
    c.set_params(gf_method=1)
    with pytest.raises(Exception):
        c.frame(c1["cloud"], c1["ss"], c1["se"], c1["surf_map"], c1["corner_map"], c1["init"])  # the method changed under the mode
    c.set_gf_float(False)
    pose, st = c.frame(c1["cloud"], c1["ss"], c1["se"], c1["surf_map"], c1["corner_map"], c1["init"])
    assert st["ran"] == 1
    c.close()

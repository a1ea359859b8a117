"""The device keyframe store (mloam_keyframes_init / _save / _submap / _query) against the oracle's mapper state machine
(oracle/orc_mapper.cpp): saveKeyframe, clearCloud and extractSurroundingKeyFrames (lidar_mapper_keyframe.cpp:641-683, :921-927,
:254-354) in an open loop (bit-identical submaps), in the closed mapper loop of process() (:1062-1101), across schedules, and on edges."""
import os

import numpy as np
import pytest

import mapper_lib as ml
import oracle_lib as orc
import synthetic as syn
import uncertainty_lib as ua

pytestmark = pytest.mark.gpu

COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])
E_STATE = -4


def _traj_out_and_back(n, step=0.25, seed=5):
    """Along the free corridor (y ~ 0) out and back: every place is passed twice, so keyframes leave the set and re-enter it."""
    rng = np.random.Generator(np.random.PCG64(seed))
    half = n // 2
    xs = [-12.0 + step * min(k, n - 1 - k) * (2 * half / max(n - 1, 1)) for k in range(n)]
    out = []
    for k, x in enumerate(xs):
        jt = rng.normal(0, 0.01, 3)
        yaw = 0.02 * np.sin(0.3 * k)
        out.append(syn.pose7([x + jt[0], 0.3 * np.sin(0.2 * k) + jt[1], 1.8 + jt[2]], syn.quat_from_rpy(0.0, 0.0, yaw)))
    return np.stack(out)


def _params(mloam, n_scans, outer=10, inner=1):
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = n_scans, outer, inner, 0.5, 1024
    return p


def _sweeps(scene, traj, n_lidars, seed=40):
    return [syn.make_multi_sweep(scene, traj[k], n_lidars, 16, 1024, seed=seed + k) for k in range(len(traj))]


_SWEEPS = {}


def _cached_sweeps(key, scene, traj, n_lidars):
    if key not in _SWEEPS:
        _SWEEPS[key] = _sweeps(scene, traj, n_lidars)
    return _SWEEPS[key]


@pytest.mark.parametrize("with_ua", [True, False])
@pytest.mark.parametrize("n_lidars", [1, 3])
def test_open_loop_bit_identical(mloam, n_lidars, with_ua):
    """Frames on the GPU, keyframe poses and covariances given to both sides: at every step the saved flag, the surrounding ids and
    their order, the chosen ids and both submaps (points and cov_vec) are bit-identical to the oracle's.  The extrinsic covariances
    change between keyframes; the case evicts, re-enters and merges keyframes in position-filter voxels."""
    scene = syn.make_scene()
    traj = _traj_out_and_back(48, step=0.3)
    sweeps = _cached_sweeps(("ol", n_lidars), scene, traj, n_lidars)
    ext = sweeps[0][3]
    L = ext.shape[0]
    dist_kf, orient, radius, res, thr = 0.9, 5.0, 2.6, 1.5, 0.05
    cx = mloam.Context(0, _params(mloam, 16 * L))
    om = ml.Mapper(dist_kf, orient, radius, res, thr)
    rng = np.random.default_rng(11)
    n_evict = n_reenter = n_multi = n_cached_decides = n_rebuilt = 0
    seen, prev_sur = set(), []
    first_scan = None
    try:
        cx.set_lidars(L, ext)
        cx.keyframes_init(dist_kf, orient, radius, res, thr)
        ext_cov = ua.ext_covariances(L, seed=1)
        for k, (cloud, ss, se, _) in enumerate(sweeps):
            pred = traj[k]
            cx.set_uncertainty(with_ua, ext_cov if with_ua else None, COV_MEAS, 1e3)
            om.set_lidars(ext, ext_cov, COV_MEAS, with_ua)
            g = cx.keyframe_submap(pred, want_output=True)
            o_rb, _ = om.submap(pred)
            assert g[0] == o_rb, k
            n_kf, sur, chosen = cx.keyframe_query()
            o_n, o_sur, o_chosen, _, _ = om.query()
            assert (n_kf, sur) == (o_n, o_sur), k
            if o_rb:
                n_rebuilt += 1
                assert chosen == o_chosen, k
                osp, osc, ocp, occ = om.maps()
                assert np.array_equal(g[1], osp) and np.array_equal(g[2], osc), k
                assert np.array_equal(g[3], ocp) and np.array_equal(g[4], occ), k
                n_evict += len(set(prev_sur) - set(sur))
                n_reenter += len((set(sur) - set(prev_sur)) & seen)
                seen |= set(sur)
                n_multi += len(chosen) < len(sur)
                if with_ua:
                    n_cached_decides += om.reassoc_differs() > 0
                prev_sur = sur
            cx.frame(cloud, ss, se, None, None, pred, False)
            sp, sc6, cp, cc6 = cx.frame_scan()
            cov = np.diag(rng.uniform(1e-5, 1e-4, 6))
            saved = cx.keyframe_save(traj[k], cov)
            o_saved, _ = om.save(traj[k], cov, sp, cp)
            assert saved == o_saved, k
            if saved and first_scan is None:
                first_scan = (sp, sc6, cp, cc6)
            if saved and with_ua:  # the /extrinsics message changes between keyframes
                ext_cov = ua.ext_covariances(L, seed=100 + k, scale=1.0 + 0.5 * rng.random())
        # the arena grew (chunks double) while keyframes were cached: the first keyframe is unchanged
        _, _, ksp, ksc, kcp, kcc = cx.keyframe_scan(0)
        assert all(np.array_equal(a, b) for a, b in zip((ksp, ksc, kcp, kcc), first_scan))
        assert cx.keyframe_query()[0] >= 8
    finally:
        cx.close()
        om.close()
    assert n_rebuilt >= 8 and n_evict >= 3 and n_reenter >= 1 and n_multi >= 1, (n_rebuilt, n_evict, n_reenter, n_multi)
    if with_ua:
        assert n_cached_decides >= 1


# ---------------------------------------------------------------------------------------------------- closed loop
N_CLOSED = 60
RESTART = 44  # the store is initialised again here: empty maps in slots whose buffers are already grown (no re-allocation)
KF = dict(dist=0.3, orient=2.0, radius=6.0, res=1.0, thr=1e3)


def _closed_case():
    scene = syn.make_scene()
    traj = syn.trajectory(N_CLOSED)
    sweeps = _cached_sweeps("closed", scene, traj, 1)
    # odometry drifts away from the truth: 2 mm + 0.02 deg per frame
    odom = []
    for k in range(N_CLOSED):
        odom.append(syn.pose_mul(traj[k], syn.pose7([0.002 * k, -0.001 * k, 0.0], syn.quat_from_rpy(0.0, 0.0, np.radians(0.02 * k)))))
    n = max(c[0].shape[0] for c in sweeps) + 64  # one padded size: the padding lies after the last ring window, extraction ignores it
    padded = []
    for cloud, ss, se, ext in sweeps:
        buf = np.zeros((n, 4), np.float32)
        buf[:cloud.shape[0]] = cloud
        padded.append((buf, ss, se))
    # frames 0-3 gate their scans with TRACE_THRESHOLD 0 (no point kept): the first keyframe holds no point, its submap fails the map gate
    thr = [0.0 if k < 4 else 1e3 for k in range(N_CLOSED)]
    return padded, sweeps[0][3], np.stack(odom), thr


def _gpu_closed_loop(mloam, env=None, lookahead=False):
    padded, ext, odom, thr = _closed_case()
    env = env or {}
    for k, v in env.items():
        os.environ[k] = v
    try:
        cx = mloam.Context(0, _params(mloam, 16))
    finally:
        for k in env:
            os.environ.pop(k)
    bufs = [np.zeros_like(padded[0][0]), np.zeros_like(padded[0][0])]
    ext_cov = ua.ext_covariances(1, seed=7)
    out, kf_stored = [], []
    try:
        cx.set_lidars(1, ext)
        cx.keyframes_init(KF["dist"], KF["orient"], KF["radius"], KF["res"], KF["thr"])
        wmap_wodom = np.array([0, 0, 0, 0, 0, 0, 1.0])
        for k in range(N_CLOSED):
            cloud, ss, se = padded[k]
            b = bufs[k % 2] if lookahead else bufs[0]
            if not lookahead or k == 0:
                np.copyto(b, cloud)
            if lookahead and k + 1 < N_CLOSED:
                np.copyto(bufs[(k + 1) % 2], padded[k + 1][0])
            if k == RESTART:
                kf_stored = [cx.keyframe_scan(i)[:2] for i in range(cx.keyframe_query()[0])]  # the store's pose_keyframes_6d
                cx.keyframes_init(KF["dist"], KF["orient"], KF["radius"], KF["res"], KF["thr"])
                wmap_wodom = np.array([0, 0, 0, 0, 0, 0, 1.0])
            cx.set_uncertainty(True, ext_cov, COV_MEAS, thr[k])                          # this frame's /extrinsics (:1028-1046)
            pred = ml.pose_mul(wmap_wodom, odom[k])                                      # transformAssociateToMap
            rebuilt, _, _ = cx.keyframe_submap(pred)                                     # extractSurroundingKeyFrames
            if lookahead and k + 1 < N_CLOSED:
                cx.frame_set_next(bufs[(k + 1) % 2], padded[k + 1][1], padded[k + 1][2])
            pose, st = cx.frame(b, ss, se, None, None, pred, False)                      # downsampleCurrentScan + scan2MapOptimization
            cov = cx.pose_covariance()
            wmap_wodom = ml.pose_mul(pose, ml.pose_inv(odom[k]))                         # transformUpdate
            saved = cx.keyframe_save()                                                   # saveKeyframe (-> clearCloud)
            n_kf, sur, chosen = cx.keyframe_query()
            out.append(dict(pose=pose, cov=cov, ran=st["ran"], saved=saved, rebuilt=rebuilt, sur=sur, chosen=chosen, n_kf=n_kf))
    finally:
        cx.close()
    return out, kf_stored


_GPU_CLOSED = {}


def _gpu_closed(mloam):
    if "ref" not in _GPU_CLOSED:
        _GPU_CLOSED["ref"] = _gpu_closed_loop(mloam)
    return _GPU_CLOSED["ref"]


def test_closed_loop_matches_oracle(mloam):
    """~60 frames of the mapper loop from an empty store, with_ua: the same keyframe decisions and surrounding lists as the oracle's
    process() driver, pose within 1e-4, covariance within 1e-9 relative, and every decision and radius test at least 1e-6 away from its
    threshold.  The keyframes the store recorded (mloam_keyframe_save with the frame's pose and covariance) equal the oracle's: at
    least 12, so that keyframes are stored both under and past the zero-covariance rule (zero while <= 10 keyframes, :607-608)."""
    g, g_kfs = _gpu_closed(mloam)
    padded, ext, odom, thr = _closed_case()
    om = ml.Mapper(KF["dist"], KF["orient"], KF["radius"], KF["res"], KF["thr"])
    om.set_lidars(ext, ua.ext_covariances(1, seed=7), COV_MEAS, True)
    o = orc.default_opts()
    o[orc.O_MAX_OUTER], o[orc.O_MAX_INNER] = 10, 1
    n_gated, n_kf_before_restart = 0, 0
    try:
        for k in range(N_CLOSED):
            cloud, ss, se = padded[k]
            if k == RESTART:
                n_kf_before_restart = om.query()[0]
                o_kfs = [om.keyframe(i) for i in range(n_kf_before_restart)]
                om.close()
                om = ml.Mapper(KF["dist"], KF["orient"], KF["radius"], KF["res"], KF["thr"])
                om.set_lidars(ext, ua.ext_covariances(1, seed=7), COV_MEAS, True)
            pose, cov, info = om.process(cloud, ss, se, odom[k], thr[k], o)
            r = g[k]
            _, sur, chosen, _, _ = om.query()
            assert r["saved"] == bool(info["saved"]) and r["rebuilt"] == bool(info["rebuilt"]) and r["ran"] == int(info["ran"]), k
            assert r["sur"] == sur, k
            if info["rebuilt"]:
                assert r["chosen"] == chosen, k
            dt, dr = syn.pose_err(r["pose"], pose)
            assert dt <= 1e-4 and dr <= 1e-4, (k, dt, dr)
            if info["ran"]:  # the frame's H^-1 (mloam_pose_covariance), before the <= 10 keyframes rule
                assert np.any(cov) and np.linalg.norm(r["cov"] - cov) <= 1e-9 * np.linalg.norm(cov), k
            else:  # map gate (:637)
                assert not np.any(r["cov"]) and not np.any(cov), k
            n_gated += info["ran"] == 0
            # margins: the decision that decided (distance, else angle) and every radius test are >= 1e-6 away from their thresholds
            if k > 0:
                assert abs(info["dist_margin"]) >= 1e-6, k
                if info["dist_margin"] <= 0:
                    assert abs(info["angle_margin"]) >= 1e-6, k
            if info["rebuilt"]:
                assert info["radius_margin"] >= 1e-6, k
        assert n_kf_before_restart >= 12 and g[RESTART - 1]["n_kf"] == n_kf_before_restart and g[-1]["n_kf"] == om.query()[0]
        assert len(g_kfs) == len(o_kfs)
        for i, ((gp, gc), (op, oc)) in enumerate(zip(g_kfs, o_kfs)):
            assert max(syn.pose_err(gp, op)) <= 1e-4, i
            if i <= 10:  # saved while the store held <= 10 keyframes: zero
                assert not gc.any() and not oc.any(), i
            else:
                assert oc.any() and np.linalg.norm(gc - oc) <= 1e-9 * np.linalg.norm(oc), i
        assert n_gated >= 3 and any(r["ran"] for r in g)
    finally:
        om.close()


@pytest.mark.parametrize("variant", ["no_graphs", "lookahead", "fuse0"])
def test_closed_loop_schedules_bit_identical(mloam, variant):
    """The closed loop replays its frames (one reused sweep buffer) and flips the map gate (an empty store, then a keyframe whose scans
    are gated to nothing, then full keyframes, then the store initialised again on the warm context): graphs vs MLOAM_DISABLE_GRAPHS=1, the sweep look-ahead, MLOAM_FUSE_ITER=0 give the
    same poses, covariances and keyframe decisions bit for bit."""
    ref, ref_kfs = _gpu_closed(mloam)
    env = {"no_graphs": {"MLOAM_DISABLE_GRAPHS": "1"}, "lookahead": {}, "fuse0": {"MLOAM_FUSE_ITER": "0"}}[variant]
    got, got_kfs = _gpu_closed_loop(mloam, env, lookahead=variant == "lookahead")
    assert len(ref_kfs) == len(got_kfs) and all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) for a, b in zip(ref_kfs, got_kfs))
    flips = sum(a["ran"] != b["ran"] for a, b in zip(ref[:-1], ref[1:]))
    assert flips >= 3 and not ref[0]["ran"] and ref[RESTART - 1]["ran"] and not ref[RESTART]["ran"]
    for k, (a, b) in enumerate(zip(ref, got)):
        assert np.array_equal(a["pose"], b["pose"]) and np.array_equal(a["cov"], b["cov"]), (variant, k)
        assert (a["ran"], a["saved"], a["rebuilt"], a["sur"], a["chosen"]) == (b["ran"], b["saved"], b["rebuilt"], b["sur"], b["chosen"]), (variant, k)


# ---------------------------------------------------------------------------------------------------- edges
def test_edges_state_errors(mloam):
    """Save before any frame, and a second save for the same frame: MLOAM_E_STATE.  A keyframe with zero kept points is stored and
    extracted as an empty cloud."""
    scene = syn.make_scene()
    traj = syn.trajectory(3)
    cloud, ss, se, ext = syn.make_multi_sweep(scene, traj[1], 1, 16, 1024, seed=3)
    cx = mloam.Context(0, _params(mloam, 16))
    try:
        with pytest.raises(mloam.MloamError, match="keyframes_init"):
            cx.keyframe_save()
        cx.set_lidars(1, ext)
        cx.keyframes_init(1.0, 1.0, 30.0, 1.0, 10.0)
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
            cx.keyframe_save()
        cx.set_uncertainty(True, ua.ext_covariances(1, seed=1), COV_MEAS, 0.0)  # every point gated out
        _, st = cx.frame(cloud, ss, se, None, None, traj[1], False)
        assert st["ran"] == 0  # empty map slots after init: the map gate (:429)
        assert cx.keyframe_save()
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
            cx.keyframe_save()
        _, _, sp, _, cp, _ = cx.keyframe_scan(0)
        assert sp.shape[0] == 0 and cp.shape[0] == 0
        rebuilt, ns, nc = cx.keyframe_submap(traj[1])
        assert rebuilt and ns == 0 and nc == 0
        assert cx.keyframe_query()[1:] == ([0], [0])
    finally:
        cx.close()


def test_edges_exact_thresholds(mloam):
    """Explicit keyframe poses exactly at the thresholds: a float distance equal to DISTANCE_KEYFRAMES or an angle below
    ORIENTATION_KEYFRAMES is not a keyframe (`>`), the next float up / a larger angle is."""
    scene = syn.make_scene()
    traj = syn.trajectory(2)
    cloud, ss, se, ext = syn.make_multi_sweep(scene, traj[1], 1, 16, 1024, seed=3)
    cx = mloam.Context(0, _params(mloam, 16))
    one = np.float32(1.0)
    seq = [([0.0, 0.0, 0.0], 0.0, True), ([1.0, 0.0, 0.0], 0.0, False), ([0.0, 1.0, 0.0], 0.0, False),
           ([float(np.nextafter(one, np.float32(2))), 0.0, 0.0], 0.0, True), ([1.0, 0.0, 0.0], 0.9, False), ([1.0, 0.0, 0.0], 1.1, True)]
    try:
        cx.set_lidars(1, ext)
        cx.keyframes_init(1.0, 1.0, 30.0, 1.0, 10.0)
        for t, yaw, want in seq:
            cx.frame(cloud, ss, se, None, None, traj[1], False)
            pose = syn.pose7(t, syn.quat_from_rpy(0.0, 0.0, np.radians(yaw)))
            assert cx.keyframe_save(pose, np.zeros((6, 6))) == want, (t, yaw)
    finally:
        cx.close()


def test_edges_communicator_rejected(mloam):
    """A context with a communicator attached: the keyframe store is single-GPU, MLOAM_E_STATE."""
    # torch ships its own NCCL: a process that loads the system libnccl through mloam_comm_init first can no longer import torch, so
    # this test imports it first, as every torch program that attaches a communicator does (and later tests of the session can)
    import torch  # noqa: F401
    cx = mloam.Context(0, _params(mloam, 16))
    try:
        try:
            cx.comm_init(1, 0, mloam.Context.comm_unique_id())
        except mloam.MloamError as e:
            pytest.skip(f"no NCCL on this machine: {e}")
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
            cx.keyframes_init(1.0, 1.0, 30.0, 1.0, 10.0)
    finally:
        cx.close()


@pytest.mark.parametrize("with_ua", [True, False])
def test_prediction_outside_every_keyframe_radius(mloam, with_ua):
    """After a save, a prediction farther than SURROUNDING_KF_RADIUS from every keyframe (a pose jump, a relocalisation): the rebuild
    runs with an empty surrounding set and yields empty maps, so the frame fails the map gate (:429) — as the oracle.  Back within the
    radius, the next call rebuilds and the maps are bit-identical to the oracle's again."""
    scene = syn.make_scene()
    traj = syn.trajectory(4)
    sweeps = [syn.make_multi_sweep(scene, traj[k], 1, 16, 1024, seed=60 + k) for k in range(4)]
    ext = sweeps[0][3]
    ext_cov = ua.ext_covariances(1, seed=2)
    jump = np.array([100.0, 0.0, 0.0, 0, 0, 0, 0])
    cx = mloam.Context(0, _params(mloam, 16))
    om = ml.Mapper(1.0, 1.0, 30.0, 1.0, 10.0)
    om.set_lidars(ext, ext_cov, COV_MEAS, with_ua)
    cov = np.diag(np.full(6, 1e-4))

    def step(k, pred, save_pose):
        g = cx.keyframe_submap(pred, want_output=True)
        o_rb, _ = om.submap(pred)
        assert g[0] == o_rb and cx.keyframe_query()[1:] == tuple(om.query()[1:3])
        osp, osc, ocp, occ = om.maps()
        assert all(np.array_equal(a, b) for a, b in zip(g[1:], (osp, osc, ocp, occ)))
        cloud, ss, se, _ = sweeps[k]
        _, st = cx.frame(cloud, ss, se, None, None, pred, False)
        sp, _, cp, _ = cx.frame_scan()
        assert cx.keyframe_save(save_pose, cov) == om.save(save_pose, cov, sp, cp)[0]
        return g, st

    try:
        cx.set_lidars(1, ext)
        cx.set_uncertainty(with_ua, ext_cov if with_ua else None, COV_MEAS, 1e3)
        cx.keyframes_init(1.0, 1.0, 30.0, 1.0, 10.0)
        step(0, traj[0], traj[0])                                # keyframe 0 (empty maps: gated)
        g, st = step(1, traj[1], traj[1] + jump)                 # submap from keyframe 0; keyframe 1 saved 100 m away (clearCloud)
        assert g[0] and g[1].shape[0] > 50 and st["ran"] == 1
        g, st = step(2, traj[2] + 2 * jump, traj[2] + 2 * jump)  # no keyframe within 30 m of the prediction
        assert g[0] and g[1].shape[0] == 0 and g[3].shape[0] == 0 and cx.keyframe_query()[1:] == ([], [])
        assert st["ran"] == 0 and not cx.pose_covariance().any()
        g, st = step(3, traj[3], traj[3])                        # keyframe 2 was saved 200 m away; back near keyframe 0
        assert g[0] and cx.keyframe_query()[1] == [0] and g[1].shape[0] > 50 and st["ran"] == 1
    finally:
        cx.close()
        om.close()

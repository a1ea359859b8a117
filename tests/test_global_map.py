"""The global map of the device keyframe store (mloam_global_map / _read / _chosen) against the oracle's pubGlobalMap / saveGlobalMap
(oracle/orc_mapper.cpp over its keyframe store): bit-identical chosen ids, points, cov_vec and sizes in both modes,
1 and 3 LiDARs, with_ua on and off; a mapper loop that computes a global map after every keyframe is bit-identical to one that does not;
the launch count does not grow with the keyframes; edges."""
import ctypes as C

import numpy as np
import pytest

import global_map_lib as gl
import mapper_lib as ml
import synthetic as syn
import uncertainty_lib as ua

pytestmark = pytest.mark.gpu

COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])
E_INVALID, E_STATE = -1, -4


def _params(mloam, n_scans):
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = n_scans, 10, 1, 0.5, 1024
    return p


def _traj(n, step=0.35, seed=5):
    rng = np.random.Generator(np.random.PCG64(seed))
    out = []
    for k in range(n):
        jt = rng.normal(0, 0.01, 3)
        out.append(syn.pose7([-12.0 + step * k + jt[0], 0.3 * np.sin(0.2 * k) + jt[1], 1.8 + jt[2]], syn.quat_from_rpy(0.0, 0.0, 0.02 * np.sin(0.3 * k))))
    return np.stack(out)


def _compare(cx, om, mode, center, radius, kf_leaf, leaf, ctx="", last_tested=None):
    """One global map on both sides: chosen ids, sizes, points and cov_vec bit-identical.  center None: the device takes the position the
    last keyframe_save tested, the oracle `last_tested` (that pose).  Returns the device maps."""
    g = cx.global_map(mode, center, radius, kf_leaf, leaf)
    g_ch = cx.global_map_chosen()
    o_ch, o = gl.global_map(om, mode, center if center is not None else last_tested, radius, kf_leaf, leaf)
    assert g_ch == o_ch, (ctx, mode)
    n_maps = 1 if mode == gl.SURROUND else 2
    for t in range(n_maps):
        assert g[2 * t].shape == o[2 * t].shape, (ctx, mode, t, g[2 * t].shape, o[2 * t].shape)
        assert np.array_equal(g[2 * t], o[2 * t]) and np.array_equal(g[2 * t + 1], o[2 * t + 1]), (ctx, mode, t)
    return g


@pytest.mark.parametrize("with_ua", [True, False])
@pytest.mark.parametrize("n_lidars", [1, 3])
def test_global_map_bit_identical(mloam, n_lidars, with_ua):
    """Frames on the GPU, each frame's gated scans saved as keyframes on both sides (the extrinsic covariances change between
    keyframes).  After every keyframe, and at the end with several radii and leaves, both modes are bit-identical to the oracle's:
    chosen ids, sizes, points and cov_vec.  The centre is the last tested position (NULL) or explicit."""
    scene = syn.make_scene()
    traj = _traj(36)
    sweeps = [syn.make_multi_sweep(scene, traj[k], n_lidars, 16, 1024, seed=40 + k) for k in range(len(traj))]
    ext = sweeps[0][3]
    L = ext.shape[0]
    thr = 0.08 if with_ua else 10.0
    cx = mloam.Context(0, _params(mloam, 16 * L))
    om = ml.Mapper(0.9, 5.0, 2.6, 1.5, thr)
    rng = np.random.default_rng(11)
    n_saved = n_multi = 0
    try:
        cx.set_lidars(L, ext)
        cx.keyframes_init(0.9, 5.0, 2.6, 1.5, thr)
        ext_cov = ua.ext_covariances(L, seed=1)
        for k, (cloud, ss, se, _) in enumerate(sweeps):
            cx.set_uncertainty(with_ua, ext_cov if with_ua else None, COV_MEAS, 1e3)
            om.set_lidars(ext, ext_cov, COV_MEAS, with_ua)
            cx.frame(cloud, ss, se, None, None, traj[k], False)
            sp, _, cp, _ = cx.frame_scan()
            cov = np.diag(rng.uniform(1e-5, 1e-4, 6))
            saved = cx.keyframe_save(traj[k], cov)
            assert saved == om.save(traj[k], cov, sp, cp)[0], k
            if saved:
                n_saved += 1
                g = _compare(cx, om, gl.SURROUND, None, 1000.0, 2.5, 0.4, k, last_tested=traj[k])
                _compare(cx, om, gl.SAVE, None, 1000.0, 2.5, 0.8, k)
                n_multi += len(cx.global_map_chosen()) < n_saved
                if with_ua:
                    ext_cov = ua.ext_covariances(L, seed=100 + k, scale=1.0 + 0.5 * rng.random())
        assert n_saved >= 10 and g[0].shape[0] > 200
        for radius, kf_leaf, leaf in ((3.0, 1.0, 0.4), (6.0, 10.0, 0.3), (1000.0, 2.5, 0.5)):
            _compare(cx, om, gl.SURROUND, traj[20], radius, kf_leaf, leaf, (radius, kf_leaf))
        _compare(cx, om, gl.SAVE, None, 1000.0, 10.0, 0.8, "save kf_leaf 10")
        assert n_multi >= 1
    finally:
        cx.close()
        om.close()


# ---------------------------------------------------------------------------------------------------- non-interference
N_LOOP = 40


def _loop(mloam, with_global_map):
    """The mapper loop of process() (with_ua) with optional global maps (both modes) after every saved keyframe: per frame the pose,
    covariance, stats, keyframe decisions, keyframe_query and the frame's launch count."""
    scene = syn.make_scene()
    traj = syn.trajectory(N_LOOP)
    sweeps = [syn.make_multi_sweep(scene, traj[k], 1, 16, 1024, seed=80 + k) for k in range(N_LOOP)]
    ext = sweeps[0][3]
    cx = mloam.Context(0, _params(mloam, 16))
    out = []
    try:
        cx.set_lidars(1, ext)
        cx.keyframes_init(0.3, 2.0, 6.0, 1.0, 1e3)
        cx.set_uncertainty(True, ua.ext_covariances(1, seed=7), COV_MEAS, 1e3)
        wmap_wodom = np.array([0, 0, 0, 0, 0, 0, 1.0])
        for k in range(N_LOOP):
            cloud, ss, se, _ = sweeps[k]
            pred = ml.pose_mul(wmap_wodom, traj[k])
            rebuilt, _, _ = cx.keyframe_submap(pred)
            l0 = cx.launch_count()
            pose, st = cx.frame(cloud, ss, se, None, None, pred, False)
            launches = cx.launch_count() - l0
            cov = cx.pose_covariance()
            wmap_wodom = ml.pose_mul(pose, ml.pose_inv(traj[k]))
            saved = cx.keyframe_save()
            if saved and with_global_map:
                cx.global_map(mloam.GLOBAL_MAP_SURROUND)
                cx.global_map(mloam.GLOBAL_MAP_SAVE)
            out.append(dict(pose=pose, cov=cov, stats={k2: v for k2, v in st.items()}, eig=st["eig"], H=st["H"], saved=saved, rebuilt=rebuilt,
                            query=cx.keyframe_query(), launches=launches))
    finally:
        cx.close()
    return out


def test_global_map_does_not_interfere(mloam):
    """The same loop with a global map after every keyframe and without: bit-identical poses, covariances, stats, keyframe decisions,
    keyframe_query results and per-frame launch counts."""
    a, b = _loop(mloam, False), _loop(mloam, True)
    assert sum(r["saved"] for r in a) >= 5 and any(r["stats"]["ran"] for r in a)
    for k, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x["pose"], y["pose"]) and np.array_equal(x["cov"], y["cov"]), k
        assert x["stats"] == y["stats"] and np.array_equal(x["eig"], y["eig"]) and np.array_equal(x["H"], y["H"]), k
        assert (x["saved"], x["rebuilt"], x["query"], x["launches"]) == (y["saved"], y["rebuilt"], y["query"], y["launches"]), k


# ---------------------------------------------------------------------------------------------------- batching
def _store_with(mloam, n_kf):
    """A store of n_kf keyframes 3 m apart, each holding the gated scans of the same sweep."""
    scene = syn.make_scene()
    traj = syn.trajectory(2)
    cloud, ss, se, ext = syn.make_multi_sweep(scene, traj[1], 1, 16, 1024, seed=3)
    cx = mloam.Context(0, _params(mloam, 16))
    cx.set_lidars(1, ext)
    cx.keyframes_init(1.0, 1.0, 30.0, 1.0, 10.0)
    for k in range(n_kf):
        cx.frame(cloud, ss, se, None, None, traj[1], False)
        assert cx.keyframe_save(syn.pose7([3.0 * (k % 40), 3.0 * (k // 40), 0.0], [0, 0, 0, 1.0]), np.zeros((6, 6)))
    return cx


def test_launch_count_does_not_grow_with_keyframes(mloam):
    """A global map of 10 keyframes and one of 400 take the same number of launches, in both modes."""
    counts = {}
    for n_kf in (10, 400):
        cx = _store_with(mloam, n_kf)
        try:
            for mode in (mloam.GLOBAL_MAP_SURROUND, mloam.GLOBAL_MAP_SAVE):
                l0 = cx.launch_count()
                g = cx.global_map(mode, radius=1e4, kf_leaf=1.0)
                counts[(n_kf, mode)] = cx.launch_count() - l0
                assert len(cx.global_map_chosen()) == n_kf and g[0].shape[0] > 0
        finally:
            cx.close()
    for mode in (mloam.GLOBAL_MAP_SURROUND, mloam.GLOBAL_MAP_SAVE):
        assert counts[(10, mode)] == counts[(400, mode)] > 0, counts


# ---------------------------------------------------------------------------------------------------- edges
def test_edges(mloam):
    """Without mloam_keyframes_init: MLOAM_E_STATE.  An empty store: empty result, no launch.  A keyframe whose scans were gated to
    nothing, a radius excluding every keyframe, a filter whose voxel index overflows int32 (the input passes through), and a read with
    too small a capacity (MLOAM_E_INVALID, the size reported) followed by a successful one — all against the oracle."""
    scene = syn.make_scene()
    traj = syn.trajectory(4)
    sw = [syn.make_multi_sweep(scene, traj[k], 1, 16, 1024, seed=60 + k) for k in range(4)]
    ext = sw[0][3]
    lib = mloam.lib()
    cx = mloam.Context(0, _params(mloam, 16))
    om = ml.Mapper(1.0, 1.0, 30.0, 1.0, 10.0)
    try:
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
            cx.global_map(mloam.GLOBAL_MAP_SAVE)
        cx.set_lidars(1, ext)
        ext_cov = ua.ext_covariances(1, seed=2)
        om.set_lidars(ext, ext_cov, COV_MEAS, True)
        cx.keyframes_init(1.0, 1.0, 30.0, 1.0, 10.0)
        l0 = cx.launch_count()
        assert cx.global_map(mloam.GLOBAL_MAP_SURROUND, center=traj[0])[0].shape[0] == 0 and cx.global_map_chosen() == []
        assert cx.global_map(mloam.GLOBAL_MAP_SAVE)[2].shape[0] == 0 and cx.launch_count() == l0
        cov = np.diag(np.full(6, 1e-4))
        for k in range(4):
            cx.set_uncertainty(True, ext_cov, COV_MEAS, 0.0 if k == 0 else 1e3)  # keyframe 0: every point gated out
            cloud, ss, se, _ = sw[k]
            cx.frame(cloud, ss, se, None, None, traj[k], False)
            sp, _, cp, _ = cx.frame_scan()
            pose = traj[k] + np.array([2.0 * k, 0, 0, 0, 0, 0, 0])
            assert cx.keyframe_save(pose, cov) and om.save(pose, cov, sp, cp)[0]
            if k == 0:
                assert sp.shape[0] == 0 and cp.shape[0] == 0
        _compare(cx, om, gl.SURROUND, None, 1000.0, 1.0, 0.4, "gated keyframe", last_tested=pose)
        _compare(cx, om, gl.SAVE, None, 1000.0, 1.0, 0.8, "gated keyframe")
        g = _compare(cx, om, gl.SURROUND, traj[0] + np.array([500.0, 0, 0, 0, 0, 0, 0]), 30.0, 1.0, 0.4, "outside")
        assert g[0].shape[0] == 0 and cx.global_map_chosen() == []
        g = _compare(cx, om, gl.SAVE, None, 1.0, 1.0, 1e-4, "int32 overflow")  # ~40 m at 0.1 mm: 4e5^3 voxels, the input passes through
        assert g[0].shape[0] > 1000
        n = C.c_int(0)
        small = np.zeros((10, 4), np.float32)
        assert lib.mloam_global_map_read(cx._h, 0, mloam._p(small), None, 10, C.byref(n)) == E_INVALID and n.value == g[0].shape[0]
        big, big6 = np.zeros((n.value, 4), np.float32), np.zeros((n.value, 6), np.float32)
        assert lib.mloam_global_map_read(cx._h, 0, mloam._p(big), mloam._p(big6), n.value, C.byref(n)) == 0
        assert np.array_equal(big, g[0]) and np.array_equal(big6, g[1])
        ids = np.zeros(1, np.int32)
        assert lib.mloam_global_map_chosen(cx._h, mloam._p(ids), 1, C.byref(n)) == E_INVALID and n.value == 4
    finally:
        cx.close()
        om.close()


def _identity_store(mloam, positions, trace_threshold):
    """A device and an oracle store with one keyframe per position (identity rotations, zero covariances, one LiDAR with the identity
    extrinsic and COV_MEASUREMENT diag(0.25, 0.25, 0.5)): every associated point's covariance is COV_MEASUREMENT exactly, trace 1.0."""
    scene = syn.make_scene()
    traj = syn.trajectory(2)
    cloud, ss, se, _ = syn.make_multi_sweep(scene, traj[1], 1, 16, 1024, seed=9)
    ident = np.array([[0, 0, 0, 0, 0, 0, 1.0]])
    cm = np.diag([0.25, 0.25, 0.5])
    cx = mloam.Context(0, _params(mloam, 16))
    om = ml.Mapper(0.5, 1.0, 30.0, 1.0, trace_threshold)
    cx.set_lidars(1, ident)
    cx.set_uncertainty(True, np.zeros((1, 6, 6)), cm, 1e3)
    om.set_lidars(ident, np.zeros((1, 6, 6)), cm, True)
    cx.keyframes_init(0.5, 1.0, 30.0, 1.0, trace_threshold)
    for p in positions:
        cx.frame(cloud, ss, se, None, None, traj[1], False)
        sp, _, cp, _ = cx.frame_scan()
        pose = syn.pose7(np.asarray(p, np.float64), [0, 0, 0, 1.0])
        assert cx.keyframe_save(pose, np.zeros((6, 6))) and om.save(pose, np.zeros((6, 6)), sp, cp)[0]
    return cx, om


def test_radius_edges_on_device(mloam):
    """The device radius search around an explicit centre: a keyframe at float d2 == (float)r^2 exactly is excluded, one a float ulp
    inside is included, as the oracle."""
    r = 4.0
    inside = float(np.nextafter(np.float32(r), np.float32(0)))
    pos = np.array([[-10.0, 0, 0], [0, 0, 0], [0, r, 0], [inside, 0, 0]], np.float32)
    cx, om = _identity_store(mloam, pos, 10.0)
    try:
        d2 = ml.np_radius_search(pos, pos[1], r)[1]
        assert d2[2] == np.float32(r * r) and d2[3] < np.float32(r * r)
        centre = syn.pose7([0.0, 0.0, 0.0], [0, 0, 0, 1.0])
        g = _compare(cx, om, gl.SURROUND, centre, r, 0.5, 0.4, "radius edge")
        assert sorted(cx.global_map_chosen()) == [1, 3] and g[0].shape[0] > 0
    finally:
        cx.close()
        om.close()


def test_trace_exactly_at_threshold(mloam):
    """Every associated point has trace exactly 1.0: with TRACE_THRESHOLD_MAPPING 1.0 the association keeps them (the gate is
    `trace > threshold`), one double ulp below it drops them all; both bit-identical to the oracle."""
    pos = [[0.0, 0.0, 0.0], [2.0, 0.0, 0.0]]
    for thr, kept in ((1.0, True), (float(np.nextafter(1.0, 0.0)), False)):
        cx, om = _identity_store(mloam, pos, thr)
        try:
            g = _compare(cx, om, gl.SAVE, None, 1000.0, 0.5, 0.05, ("trace", thr))
            assert (g[0].shape[0] > 100) == kept and (g[2].shape[0] > 10) == kept, (thr, g[0].shape, g[2].shape)
        finally:
            cx.close()
            om.close()


def test_communicator_rejected(mloam):
    """A context with a communicator attached: the global map is single-GPU, MLOAM_E_STATE."""
    import torch  # noqa: F401  (torch's NCCL first, as test_keyframe_mapper.py explains)
    cx = mloam.Context(0, _params(mloam, 16))
    try:
        try:
            cx.comm_init(1, 0, mloam.Context.comm_unique_id())
        except mloam.MloamError as e:
            pytest.skip(f"no NCCL on this machine: {e}")
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
            cx.global_map(mloam.GLOBAL_MAP_SURROUND)
    finally:
        cx.close()

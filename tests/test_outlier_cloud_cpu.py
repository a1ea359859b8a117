"""CPU tests of the oracle's outlier cloud (segment_cloud: 0; oracle/orc_ua.cpp, oracle/orc_mapper.cpp): laser_cloud_outlier_cov of a frame against a
numpy composition of its four steps (the first point of each LiDAR's part of the sweep, the float 3x4 extrinsic in PCL's order with
intensity = laser id, VoxelGridCovarianceMLOAM<PointI>(MAP_OUTLIER_RES), the with_ua trace gate), and the global maps with the outlier
appends against the single steps concatenated in the reference's two orders (lidar_mapper_keyframe.cpp:818-827, :873-882)."""
import numpy as np
import pytest

import global_map_lib as gl
import mapper_lib as ml
import outlier_lib as ol
import synthetic as syn
import uncertainty_lib as ua

COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])
LEAF = 0.8  # MAP_OUTLIER_RES of the KITTI / Oxford / UTBM configurations
EMPTY = np.zeros((0, 4), np.float32)


def _ext(n_lidars):
    ext = [syn.pose7([0.0, 0.0, 0.0], [0, 0, 0, 1.0])]
    for l in range(1, n_lidars):
        ext.append(syn.pose7([0.3 * l, -0.2 * l, 0.05 * l], syn.quat_from_rpy(0.01 * l, -0.02 * l, 0.3 * l)))
    return np.stack(ext)


def _rig(rng, counts):
    """A ring-ordered concatenation from per-LiDAR, per-ring point counts, with the reference's ScanInfo (start = size + 5, end = size - 6)."""
    pts, ss, se, size = [], [], [], 0
    for lidar in counts:
        for c in lidar:
            ss.append(size + 5)
            p = np.zeros((c, 4), np.float32)
            p[:, :3] = rng.normal(0.0, 6.0, (c, 3))
            p[:, 3] = len(ss) - 1 + rng.random(c)
            pts.append(p)
            size += c
            se.append(size - 6)
    return np.concatenate(pts) if pts else EMPTY, np.array(ss, np.int32), np.array(se, np.int32)


def _check(cloud, ss, n_lidars, ext, with_ua, thr=1e3, ext_cov=None):
    ext_cov = ua.ext_covariances(n_lidars, seed=3) if ext_cov is None else ext_cov
    got_p, got_c = ol.frame_outlier(cloud, ss, n_lidars, ext, ext_cov, COV_MEAS, with_ua, thr, LEAF)
    want_p, want_c, traces = ol.compose_frame(cloud, ss, n_lidars, ext, ext_cov, COV_MEAS, with_ua, thr, LEAF)
    # the composition's trace is a sum of float cov_vec entries, the oracle's the double one: keep the cases clear of the threshold
    assert all(abs(t - thr) > 1e-6 * max(thr, 1.0) for t in traces)
    assert np.array_equal(got_p, want_p) and np.array_equal(got_c, want_c)
    return got_p, got_c


@pytest.mark.parametrize("with_ua", [False, True])
@pytest.mark.parametrize("n_lidars", [1, 3, 16])
def test_frame_outlier_matches_composition(n_lidars, with_ua):
    """Ray-cast rig sweeps: one point per LiDAR before the filter, laser ids in order, cov_vec zero without with_ua."""
    scene = syn.make_scene()
    cloud, ss, _, ext = syn.make_multi_sweep(scene, syn.trajectory(3)[1], n_lidars, 16, 512, seed=9)
    p, c = _check(cloud, ss, n_lidars, ext, with_ua)
    assert 1 <= p.shape[0] <= n_lidars and np.all(np.diff(p[:, 3]) != 0) | (p.shape[0] == 1)
    assert with_ua == bool(np.any(c))


@pytest.mark.parametrize("with_ua", [False, True])
def test_frame_outlier_edges(with_ua):
    rng = np.random.default_rng(4)
    ext = _ext(3)
    # a LiDAR whose ring 0 is empty: its first point is ring 1's first
    cloud, ss, _ = _rig(rng, [[30, 30], [0, 25], [20, 0]])
    p, _ = _check(cloud, ss, 3, ext, with_ua)
    firsts = ol.np_first_points(cloud, ss, 3)
    assert [l for l, _ in firsts] == [0, 1, 2] and np.array_equal(firsts[1][1], cloud[60])
    # an empty LiDAR (the middle one, and the last one) contributes no point
    for counts, ids in (([[12, 12], [0, 0], [15, 9]], [0, 2]), ([[12, 12], [7, 9], [0, 0]], [0, 1])):
        cloud, ss, _ = _rig(rng, counts)
        assert [l for l, _ in ol.np_first_points(cloud, ss, 3)] == ids
        p, _ = _check(cloud, ss, 3, ext, with_ua)
        assert sorted(set(p[:, 3].astype(int).tolist())) <= ids
    # every LiDAR empty: an empty cloud
    cloud, ss, _ = _rig(rng, [[0, 0], [0, 0]])
    cloud = np.zeros((1, 4), np.float32)  # the sweep buffer is never read
    p, c = ol.frame_outlier(cloud[:0], ss, 2, ext[:2], None, COV_MEAS, with_ua, 1e3, LEAF)
    assert p.shape == (0, 4) and c.shape == (0, 6)


def test_frame_outlier_shared_voxel():
    """Two LiDARs whose first points fall into one 0.8 m voxel merge into one point: the float mean of x, y, z, the LAST point's id."""
    rng = np.random.default_rng(5)
    cloud, ss, _ = _rig(rng, [[10, 10], [10, 10], [10, 10]])
    ext = np.stack([syn.pose7([0, 0, 0], [0, 0, 0, 1.0])] * 3)
    cloud[0, :3] = [1.10, 2.20, 0.30]
    cloud[20, :3] = [1.30, 2.05, 0.45]   # same voxel as LiDAR 0's
    cloud[40, :3] = [9.00, -3.0, 1.00]
    for with_ua in (False, True):
        p, _ = _check(cloud, ss, 3, ext, with_ua)
        assert p.shape[0] == 2
        merged = p[np.argmin(np.abs(p[:, 0] - 1.2))]
        f = np.float32
        assert merged[3] == 1.0 and merged[0] == f(f(f(0) + f(1.10)) + f(1.30)) / f(2)


def test_frame_outlier_trace_gate():
    """with_ua: a point whose trace exceeds TRACE_THRESHOLD_MAPPING is dropped, a point under it kept."""
    scene = syn.make_scene()
    cloud, ss, _, ext = syn.make_multi_sweep(scene, syn.trajectory(3)[1], 3, 16, 512, seed=9)
    ext_cov = ua.ext_covariances(3, seed=3)
    _, _, tr = ol.compose_frame(cloud, ss, 3, ext, ext_cov, COV_MEAS, True, 1e3, LEAF)
    tr = np.sort(tr)
    assert tr.shape[0] >= 2
    thr = 0.5 * (tr[0] + tr[1])
    p, _ = _check(cloud, ss, 3, ext, True, thr=thr, ext_cov=ext_cov)
    assert p.shape[0] == 1
    p, _ = _check(cloud, ss, 3, ext, True, thr=0.5 * tr[0], ext_cov=ext_cov)
    assert p.shape[0] == 0


def _stores(rng, n_kf, n_lidars, with_ua, outliers=True):
    """The same keyframes saved into one store with their outlier clouds and into another without them: keyframes[id] = (pose, cov, surf,
    corner, outlier)."""
    ext, ext_cov = _ext(n_lidars), ua.ext_covariances(n_lidars, seed=4)
    thr = 0.12 if with_ua else 10.0
    mo, mg = ml.Mapper(0.5, 1.0, 10.0, 1.0, thr), ml.Mapper(0.5, 1.0, 10.0, 1.0, thr)
    for m in (mo, mg):
        m.set_lidars(ext, ext_cov, COV_MEAS, with_ua)
    kfs = []
    for k in range(n_kf):
        t = np.array([2.0 * k, 1.5, 1.5]) + rng.uniform(-1.0, 1.0, 3) * [0.2, 0.2, 0.1]
        pose = syn.pose7(t, syn.quat_from_rpy(0.0, 0.0, 0.1 * k))
        cov = np.diag(rng.uniform(1e-5, 1e-4, 6)) if k > 2 else np.zeros((6, 6))
        cl = []
        for n in (int(rng.integers(20, 60)), int(rng.integers(10, 30)), int(rng.integers(1, n_lidars + 1)) if outliers else 0):
            p = np.zeros((n, 4), np.float32)
            p[:, :3] = rng.normal(0.0, 4.0, (n, 3)) + t
            p[:, 3] = rng.integers(0, n_lidars, n)
            cl.append(p)
        assert mo.save(pose, cov, cl[0], cl[1], outlier=cl[2])[0] and mg.save(pose, cov, cl[0], cl[1])[0]
        kfs.append((pose, cov, *cl))
    return mo, mg, kfs, ext, ext_cov, thr


@pytest.mark.parametrize("with_ua", [False, True])
@pytest.mark.parametrize("n_lidars", [1, 3])
def test_global_map_outlier_orders(n_lidars, with_ua):
    rng = np.random.default_rng(10 + n_lidars)
    mo, mg, kfs, ext, ext_cov, thr = _stores(rng, 14, n_lidars, with_ua)
    assert sum(k[4].shape[0] for k in kfs) > 0
    pos = np.array([k[0][:3] for k in kfs], np.float32)
    try:
        for mode, leaf in ((ol.SURROUND, 0.4), (ol.SAVE, 0.8)):
            centre = kfs[6][0]
            cand = gl.np_candidates(pos, mode, pos[6], 12.0)
            chosen = gl.np_chosen(pos, cand, 10.0)
            ids, maps = gl.global_map(mo, mode, centre, 12.0, 10.0, leaf)
            assert ids == chosen and len(chosen) >= 2
            want = ol.compose_global(kfs, ext, ext_cov, COV_MEAS, with_ua, thr, mode, chosen, leaf)
            for a, b in zip(maps, want):
                assert np.array_equal(a, b)
            # without the gate every outlier point reaches the maps: they differ from the maps of surf and corner alone
            _, plain = gl.global_map(mg, mode, centre, 12.0, 10.0, leaf)
            if not with_ua:
                assert not all(np.array_equal(a, b) for a, b in zip(maps, plain))
    finally:
        mo.close(), mg.close()


@pytest.mark.parametrize("with_ua", [False, True])
def test_global_map_without_outliers_is_unchanged(with_ua):
    """A store whose keyframes hold empty outlier clouds, and one saved without them, give exactly the composition of surf and corner
    alone over the same chosen ids."""
    rng = np.random.default_rng(21)
    mo, mg, kfs, ext, ext_cov, thr = _stores(rng, 12, 3, with_ua, outliers=False)
    pos = np.array([k[0][:3] for k in kfs], np.float32)
    try:
        for mode, leaf in ((ol.SURROUND, 0.4), (ol.SAVE, 0.8)):
            chosen = gl.np_chosen(pos, gl.np_candidates(pos, mode, pos[5], 1000.0), 10.0)
            want = gl.compose([k[:4] for k in kfs], ext, ext_cov, COV_MEAS, with_ua, thr, mode, chosen, leaf)
            for m in (mo, mg):
                ids, maps = gl.global_map(m, mode, kfs[5][0], 1000.0, 10.0, leaf)
                assert ids == chosen and all(np.array_equal(x, y) for x, y in zip(maps, want))
    finally:
        mo.close(), mg.close()

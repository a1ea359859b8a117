"""CPU tests of the oracle's global map (pubGlobalMap / saveGlobalMap, oracle/orc_mapper.cpp) against an independent composition
of its steps: the radius selection and its order (with a keyframe exactly on the radius and one a float ulp inside), the keyframe-position
filter with the last id of a voxel winning, the concatenation order of each mode, and the leaf each mode filters at."""
import numpy as np
import pytest

import global_map_lib as gl
import mapper_lib as ml
import synthetic as syn
import uncertainty_lib as ua

COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])
EMPTY = np.zeros((0, 4), np.float32)


def _ext(n_lidars):
    ext = [syn.pose7([0.0, 0.0, 0.0], [0, 0, 0, 1.0])]
    for l in range(1, n_lidars):
        ext.append(syn.pose7([0.3 * l, -0.2 * l, 0.05 * l], syn.quat_from_rpy(0.01 * l, -0.02 * l, 0.3 * l)))
    return np.stack(ext)


def _cloud(rng, n, n_lidars, centre):
    p = np.zeros((n, 4), np.float32)
    p[:, :3] = rng.normal(0.0, 4.0, (n, 3)) + centre
    p[:, 3] = rng.integers(0, n_lidars, n)
    return p


def _store(rng, n_kf, n_lidars, with_ua, spread=6.0, empty_surf=()):
    """An oracle store of n_kf keyframes (every save forced by a 2 m step) and what it holds: keyframes[id] = (pose, cov, surf, corner)."""
    ext, ext_cov = _ext(n_lidars), ua.ext_covariances(n_lidars, seed=4)
    m = ml.Mapper(0.5, 1.0, 10.0, 1.0, 0.12 if with_ua else 10.0)
    m.set_lidars(ext, ext_cov, COV_MEAS, with_ua)
    kfs = []
    for k in range(n_kf):
        t = np.array([2.0 * k, 1.5, 1.5]) + rng.uniform(-spread, spread, 3) * [0.2, 0.2, 0.1]
        pose = syn.pose7(t, syn.quat_from_rpy(0.0, 0.0, 0.1 * k))
        cov = np.diag(rng.uniform(1e-5, 1e-4, 6)) if k > 2 else np.zeros((6, 6))
        surf = EMPTY if k in empty_surf else _cloud(rng, int(rng.integers(20, 60)), n_lidars, t)
        corner = _cloud(rng, int(rng.integers(5, 30)), n_lidars, t)
        saved, _ = m.save(pose, cov, surf, corner)
        assert saved
        kfs.append((pose, cov, surf, corner))
    return m, kfs, ext, ext_cov


def _pos(kfs):
    return np.array([k[0][:3] for k in kfs]).astype(np.float32)


@pytest.mark.parametrize("with_ua", [True, False])
@pytest.mark.parametrize("n_lidars", [1, 3])
def test_both_modes_match_composition(n_lidars, with_ua):
    """Both modes: the chosen ids equal the radius search / id order followed by the last-wins position filter, and the maps equal the
    chosen keyframes' associated clouds concatenated in the mode's order and filtered at the given leaf, bit for bit."""
    rng = np.random.default_rng(7 + n_lidars)
    m, kfs, ext, ext_cov = _store(rng, 24, n_lidars, with_ua, empty_surf=(5,))
    thr = 0.12 if with_ua else 10.0
    pos = _pos(kfs)
    n_points = 0
    try:
        for mode, leaf, kf_leaf in ((gl.SURROUND, 0.4, 3.0), (gl.SURROUND, 0.7, 10.0), (gl.SAVE, 0.8, 3.0), (gl.SAVE, 1.1, 10.0)):
            centre = kfs[11][0]
            chosen, maps = gl.global_map(m, mode, centre, 15.0, kf_leaf, leaf)
            cand = gl.np_candidates(pos, mode, centre[:3].astype(np.float32), 15.0)
            assert chosen == gl.np_chosen(pos, cand, kf_leaf), mode
            assert len(chosen) < len(cand) and len(chosen) >= 3, (mode, len(chosen), len(cand))  # voxels with several keyframes
            want = gl.compose(kfs, ext, ext_cov, COV_MEAS, with_ua, thr, mode, chosen, leaf)
            for a, b in zip(maps, want):
                assert a.shape == b.shape and np.array_equal(a, b), mode
            if mode == gl.SURROUND:
                assert maps[2].shape[0] == 0
            n_points += maps[0].shape[0] + maps[2].shape[0]
        assert n_points > 100
    finally:
        m.close()


def test_save_concatenation_order_differs_from_surround():
    """SAVE puts corner into a map of its own; SURROUND appends each keyframe's corner after its surf.  With one keyframe and a leaf
    that keeps every point apart, SURROUND's map is SAVE's surf map followed by its corner map (filter order is voxel order, so compare
    as sets) and a leaf twice as large merges points."""
    rng = np.random.default_rng(3)
    m, kfs, _, _ = _store(rng, 1, 1, False)
    try:
        _, s = gl.global_map(m, gl.SURROUND, kfs[0][0], 5.0, 10.0, 1e-3)
        _, v = gl.global_map(m, gl.SAVE, None, 0.0, 10.0, 1e-3)
        n_s, n_c = kfs[0][2].shape[0], kfs[0][3].shape[0]
        assert s[0].shape[0] == n_s + n_c and v[0].shape[0] == n_s and v[2].shape[0] == n_c
        key = lambda a: sorted(map(tuple, a.tolist()))  # noqa: E731
        assert key(s[0]) == key(np.concatenate([v[0], v[2]]))
        _, big = gl.global_map(m, gl.SURROUND, kfs[0][0], 5.0, 10.0, 8.0)
        assert big[0].shape[0] < s[0].shape[0]
    finally:
        m.close()


def test_radius_edges_and_empty():
    """No keyframe: nothing chosen.  A keyframe at float d2 == (float)r^2 exactly is excluded, one a float ulp inside is included; a
    radius excluding every keyframe chooses nothing and yields empty maps."""
    m = ml.Mapper(0.5, 1.0, 10.0, 1.0, 10.0)
    m.set_lidars(_ext(1), None, None, False)
    try:
        assert gl.global_map(m, gl.SURROUND, syn.pose7([0, 0, 0], [0, 0, 0, 1.0]), 5.0, 1.0, 0.4)[0] == []
        assert gl.global_map(m, gl.SAVE, None, 0.0, 1.0, 0.4)[0] == []
        r = 4.0
        inside = float(np.nextafter(np.float32(r), np.float32(0)))
        pos = np.array([[-10.0, 0, 0], [0, 0, 0], [0, r, 0], [inside, 0, 0]], np.float32)  # centre at keyframe 1
        for p in pos:
            pts = np.array([[p[0], p[1], 0.0, 0.0], [p[0] + 0.01, p[1] + 0.5, 0.0, 0.0]], np.float32)
            assert m.save(syn.pose7(p.astype(np.float64), [0, 0, 0, 1.0]), np.zeros((6, 6)), pts, EMPTY)[0]
        c = syn.pose7([0.0, 0.0, 0.0], [0, 0, 0, 1.0])
        cand, d2 = ml.np_radius_search(pos, pos[1], r)
        assert d2[2] == np.float32(r * r) and d2[3] < np.float32(r * r) and cand == [1, 3]
        chosen, maps = gl.global_map(m, gl.SURROUND, c, r, 0.5, 0.01)
        assert sorted(chosen) == [1, 3] and maps[0].shape[0] == 4
        chosen, maps = gl.global_map(m, gl.SURROUND, syn.pose7([500.0, 0, 0], [0, 0, 0, 1.0]), r, 0.5, 0.01)
        assert chosen == [] and maps[0].shape[0] == 0
    finally:
        m.close()


def test_position_filter_last_id_wins():
    """Several keyframes in one kf_leaf voxel: the filter keeps the id listed last (radius order for SURROUND, id order for SAVE), not the
    nearest one; the chosen ids follow voxel order."""
    m = ml.Mapper(0.05, 1.0, 10.0, 1.0, 10.0)
    m.set_lidars(_ext(1), None, None, False)
    xs = [1.0, 1.2, 1.1, 1.3, 25.0, 25.5]  # ids 0-3 in one 10 m voxel, 4-5 in another
    try:
        for x in xs:
            m.save(syn.pose7([x, 0.0, 0.0], [0, 0, 0, 1.0]), np.zeros((6, 6)), np.array([[x, 0, 0, 0]], np.float32), EMPTY)
        assert gl.global_map(m, gl.SAVE, None, 0.0, 10.0, 0.4)[0] == [3, 5]
        # around x = 0: radius order is 0, 2, 1, 3 (then 4, 5): the farthest of the first voxel, id 3, is listed last
        assert gl.global_map(m, gl.SURROUND, syn.pose7([0.0, 0, 0], [0, 0, 0, 1.0]), 100.0, 10.0, 0.4)[0] == [3, 5]
        # around x = 1.35: radius order 3, 1, 2, 0 -> id 0 wins
        assert gl.global_map(m, gl.SURROUND, syn.pose7([1.35, 0, 0], [0, 0, 0, 1.0]), 100.0, 10.0, 0.4)[0] == [0, 5]
    finally:
        m.close()

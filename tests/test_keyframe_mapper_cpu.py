"""CPU tests of the oracle's keyframe state machine (oracle/orc_mapper.cpp) against independent numpy restatements: the saveKeyframe
decision at and around both thresholds, the surrounding-set bookkeeping of extractSurroundingKeyFrames (:274-323) on random enter /
leave sequences, the radius-search order with exact distance ties, and the keyframe-position filter choosing the last-listed keyframe
of each voxel."""
import numpy as np

import mapper_lib as ml
import synthetic as syn

EMPTY = np.zeros((0, 4), np.float32)
ZERO_COV = np.zeros((6, 6))
IDENT_EXT = np.array([[0, 0, 0, 0, 0, 0, 1.0]])


def _pose(t, yaw_deg=0.0):
    return syn.pose7(t, syn.quat_from_rpy(0.0, 0.0, np.radians(yaw_deg)))


def _mapper(dist=1.0, orient=1.0, radius=5.0, res=1.0):
    m = ml.Mapper(dist, orient, radius, res, 10.0)
    m.set_lidars(IDENT_EXT, None, None, False)
    return m


def _one_point(x, y, z):
    return np.array([[x, y, z, 0.0]], np.float32)


def test_save_decision_first_and_thresholds():
    """The first keyframe is always saved; then a save exactly when the float distance > DISTANCE_KEYFRAMES or the angle >
    ORIENTATION_KEYFRAMES.  Steps straddle both thresholds by a few ulps and by 1e-6."""
    rng = np.random.default_rng(3)
    m = _mapper(dist=1.0, orient=1.0)
    prev_pt, prev_q, n = np.zeros(3, np.float32), np.array([0, 0, 0, 1.0]), 0
    base = np.array([2.5, -1.25, 0.5])
    steps = [0.0]
    for d in (1.0, 1.0 + 1e-6, 1.0 - 1e-6):
        steps += [d, np.nextafter(d, 2.0), np.nextafter(d, 0.0)]
    angles = [0.0, 1.0, 1.0 + 1e-6, 1.0 - 1e-6, np.nextafter(1.0, 2.0), 0.5, 1.5]
    decisions = []
    cur = base.copy()
    yaw = 10.0
    for i in range(160):
        if i % 2 == 0:
            d = steps[rng.integers(len(steps))]
            u = rng.normal(size=3)
            cur = cur + d * u / np.linalg.norm(u)
            dyaw = 0.0
        else:
            dyaw = angles[rng.integers(len(angles))]
        pose = _pose(cur, yaw + dyaw)
        want = ml.np_keyframe_due(pose, prev_pt, prev_q, n, 1.0, 1.0)
        got, _ = m.save(pose, ZERO_COV, EMPTY, EMPTY)
        assert got == want, (i, pose)
        decisions.append(got)
        if got:
            prev_pt, prev_q, n = pose[:3].astype(np.float32), pose[3:].copy(), n + 1
            yaw = yaw + dyaw
    assert decisions[0] and 20 <= sum(decisions) <= 140
    assert m.query()[0] == sum(decisions)


def test_save_decision_exact_distance_boundary():
    """A displacement whose float distance is exactly DISTANCE_KEYFRAMES is not a keyframe (`>`), the next float up is."""
    m = _mapper(dist=1.0, orient=1.0)
    assert m.save(_pose([0.0, 0.0, 0.0]), ZERO_COV, EMPTY, EMPTY)[0]
    assert not m.save(_pose([1.0, 0.0, 0.0]), ZERO_COV, EMPTY, EMPTY)[0]
    assert m.save(_pose([np.nextafter(np.float32(1.0), np.float32(2.0)), 0.0, 0.0]), ZERO_COV, EMPTY, EMPTY)[0]
    assert ml.np_keyframe_due(_pose([1.0, 0, 0]), np.zeros(3, np.float32), np.array([0, 0, 0, 1.0]), 1, 1.0, 1.0) is False


def _positions_mapper(pos, radius, res):
    """A store whose keyframes sit at `pos` (one tiny cloud each, so that a map is never empty unless no keyframe is chosen)."""
    m = _mapper(dist=0.0, orient=0.0, radius=radius, res=res)
    for i, p in enumerate(pos):
        saved, _ = m.save(_pose(p, 0.01 * i), ZERO_COV, _one_point(*p), _one_point(*p))
        assert saved
    return m


def test_bookkeeping_random_enter_leave_sequences():
    """Random keyframe layouts and query walks: the surrounding list after each rebuild equals the numpy bookkeeping (survivors in their
    order, new ids appended in radius order) and the chosen ids equal the numpy position filter's choice."""
    rng = np.random.default_rng(7)
    n_evict = n_reenter = n_multi = 0
    for trial in range(12):
        pos = rng.uniform(-8, 8, size=(40, 3)).astype(np.float32).astype(np.float64)
        pos[:, 2] *= 0.1
        m = _positions_mapper(pos, 4.0, 1.5)
        pos32 = pos.astype(np.float32)
        existing, seen = [], set()
        for step in range(25):
            q = rng.uniform(-8, 8, 3)
            q[2] = 0.0
            # a save empties the maps; a rebuild needs them empty, so every query follows a (non-)save of a far pose: use a fresh
            # clearCloud by saving a keyframe far away (outside every radius)
            far = np.array([1000.0 + 10 * step + 100 * trial, 0, 0])
            assert m.save(_pose(far), ZERO_COV, EMPTY, EMPTY)[0]
            pos32 = np.vstack([pos32, far.astype(np.float32)])
            rebuilt, _ = m.submap(_pose(q))
            assert rebuilt
            found, _ = ml.np_radius_search(pos32, q.astype(np.float32), 4.0)
            want, new = ml.np_bookkeeping(existing, found)
            n_evict += len(set(existing) - set(found))
            n_reenter += len(set(new) & seen)
            seen |= set(new)
            _, sur, chosen, _, _ = m.query()
            assert sur == want, (trial, step)
            if sur:
                pick = ml.np_position_filter(pos32[sur], 1.5)
                assert chosen == [sur[j] for j in pick]
                n_multi += len(sur) > len(pick)
            existing = want
    assert n_evict >= 50 and n_reenter >= 10 and n_multi >= 10, (n_evict, n_reenter, n_multi)


def test_radius_search_exact_ties_order_by_id():
    """Keyframes at exactly equal float distances (a lattice around the query): ordered by id within a tie; a keyframe at exactly the
    radius is outside (`<`)."""
    pts = []
    for x in (-2.0, -1.0, 1.0, 2.0):
        for y in (-2.0, -1.0, 1.0, 2.0):
            pts.append([x, y, 0.0])
    pts.append([3.0, 0.0, 0.0])  # d2 == radius^2
    pts = np.array(pts)
    perm = np.random.default_rng(1).permutation(len(pts))
    pts = pts[perm]
    m = _positions_mapper(pts, 3.0, 0.25)
    assert m.save(_pose([100.0, 0, 0]), ZERO_COV, EMPTY, EMPTY)[0]  # clearCloud
    rebuilt, margin = m.submap(_pose([0.0, 0.0, 0.0]))
    assert rebuilt and margin == 0.0
    _, sur, _, _, _ = m.query()
    want, d2 = ml.np_radius_search(np.vstack([pts, [[100.0, 0, 0]]]).astype(np.float32), np.zeros(3, np.float32), 3.0)
    assert sur == want
    far_id = int(np.nonzero(perm == len(pts) - 1)[0][0])
    assert far_id not in sur and len(sur) == 16
    ties = [d2[i] for i in sur]
    assert ties == sorted(ties) and len(set(ties)) < len(ties)


def test_position_filter_takes_last_listed_keyframe():
    """Several keyframes per MAP_SUR_KF_RES voxel: the filter's output carries the highest set position of each voxel, so the cloud of
    the LAST listed keyframe of a voxel enters the map (and only it)."""
    pos = np.array([[0.1, 0.1, 0.0], [0.2, 0.3, 0.0], [0.15, 0.7, 0.0], [1.4, 0.2, 0.0], [1.6, 0.1, 0.0], [0.3, 0.2, 0.0]])
    m = _positions_mapper(pos, 10.0, 1.0)
    assert m.save(_pose([100.0, 0, 0]), ZERO_COV, EMPTY, EMPTY)[0]
    assert m.submap(_pose([0.0, 0.0, 0.0]))[0]
    _, sur, chosen, _, _ = m.query()
    pick = ml.np_position_filter(pos[sur].astype(np.float32), 1.0)
    assert chosen == [sur[j] for j in pick] and len(chosen) == 2
    # the voxel [0,1)^2 holds keyframes 0, 1, 2, 5: the last listed one is chosen
    in_v0 = [j for j, s in enumerate(sur) if s in (0, 1, 2, 5)]
    assert sur[max(in_v0)] in chosen
    sp, _, _, _ = m.maps()
    assert sp.shape[0] == 2


def test_cache_keeps_association_under_changed_covariances():
    """with_ua: a keyframe that stays in the set keeps the association it got when it entered; after the extrinsic covariances change
    its re-association would differ — the cache decides the map."""
    rng = np.random.default_rng(4)
    cloud = np.concatenate([rng.uniform(-10, 10, (400, 3)), np.zeros((400, 1))], 1).astype(np.float32)
    m = ml.Mapper(0.5, 5.0, 20.0, 1.0, 1e6)
    ext = np.array([[0.1, 0, 0.2, 0, 0, 0, 1.0]])
    cov_a = ml.ua.ext_covariances(1, seed=1)
    m.set_lidars(ext, cov_a, np.eye(3) * 0.0025, True)
    assert m.save(_pose([0, 0, 0]), np.eye(6) * 1e-4, cloud, cloud)[0]
    assert m.submap(_pose([0, 0, 0]))[0]
    assert m.reassoc_differs() == 0
    m.set_lidars(ext, ml.ua.ext_covariances(1, seed=2, scale=2.0), np.eye(3) * 0.0025, True)
    assert m.reassoc_differs() == 1

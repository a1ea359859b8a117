"""GPU tests (-m gpu) at the edges where the kernels' exactness claims matter: distance ties, duplicated, collinear and
exactly coplanar neighbourhoods, cell and voxel faces, coarsened grids, kilometre-scale coordinates, path boundaries of
the voxel filters and of extractCloud's in-CTA sort.  Every case is compared with a CPU reference (the oracle, or a
plain numpy / math.fsum statement of the operation) and counts the edge it claims to hit, so that it cannot pass
vacuously.  Discrete results are compared bit for bit; floating-point reductions within an error bound."""
import os

import numpy as np
import pytest

import edges as E
import oracle_lib as orc
import synthetic as syn

pytestmark = pytest.mark.gpu

POSE_TOL = 1e-4  # metres / radians (BASELINE.json north_star)
FAR = np.array([2731.3, -1873.9, 41.7])


def _rand_cloud(rng, n, lo, hi):
    return E.cloud(rng.uniform(lo, hi, (n, 3)))


def _check_knn(ctx, slot, m, q, k, max_sqdist, pose=None, brute_oracle=True):
    """ctx.knn against the numpy brute force (and the oracle's brute force when the map is finite), bit for bit."""
    idx, sqd = ctx.knn(slot, q, k, max_sqdist, pose7=pose)
    qq = q if pose is None else orc.associate(q, pose)
    ridx, rsqd = E.knn_brute(m, qq, k, max_sqdist)
    assert np.array_equal(idx, ridx), np.argwhere(idx != ridx)[:5]
    assert np.array_equal(sqd.view(np.uint32), rsqd.view(np.uint32))
    if brute_oracle:
        oidx, osqd = orc.knn(m, qq, k, brute=True)
        inside = osqd < np.float32(max_sqdist)
        assert np.array_equal(np.where(inside, oidx, -1), ridx)
        assert np.array_equal(np.where(inside, osqd, np.inf).astype(np.float32), rsqd)
    return ridx, rsqd


# ------------------------------------------------------------------------------------------------ 1. exact kNN
@pytest.mark.parametrize("k", [1, 5, 10])
@pytest.mark.parametrize("cell", [0.25, 0.5])
def test_knn_lattice_ties(ctx, k, cell):
    """Lattice map (spacing 0.125): queries at lattice points, body and face centres have several neighbours at exactly
    the same distance, so the index decides the K-set at its boundary."""
    shape = (24, 20, 12)
    m = E.lattice(shape, 0.125, (-1.5, -1.25, -0.75))
    q = E.lattice_queries(shape, 0.125, (-1.5, -1.25, -0.75), np.random.default_rng(k), 900)
    ctx.map_build(2, m, cell)
    _check_knn(ctx, 2, m, q, k, 1.0)
    _, s1 = E.knn_brute(m, q, k, 1.0, extra=1)
    assert E.boundary_ties(s1, k).mean() >= 0.3


@pytest.mark.parametrize("k", [1, 5, 10])
def test_knn_exact_duplicates(ctx, k):
    rng = np.random.default_rng(30 + k)
    base = _rand_cloud(rng, 1500, -2, 2)
    m, reps = E.duplicated(base, rng)
    q = np.concatenate([E.near(base, rng, 300, 0.0), _rand_cloud(rng, 300, -2.5, 2.5)])
    ctx.map_build(2, m, 0.5)
    ridx, _ = _check_knn(ctx, 2, m, q, k, 1.0)
    if k > 1:
        _, s1 = E.knn_brute(m, q, k, 1.0, extra=1)
        assert E.boundary_ties(s1, k).sum() >= 100


@pytest.mark.parametrize("k", [1, 5, 10])
def test_knn_dense_cell_many_tiles(ctx, k):
    """3200 points in one 0.5 m cell: a ring-1 run of > 10 TMA tiles (256 points), split between the lanes' runs."""
    rng = np.random.default_rng(50 + k)
    m = E.dense_cell(rng, 3200, 0.5)
    assert E.cell_counts(m, 0.5).max() >= 3000
    q = np.concatenate([_rand_cloud(rng, 200, -0.2, 0.7), _rand_cloud(rng, 56, -5, 5)])
    ctx.map_build(2, m, 0.5)
    _check_knn(ctx, 2, m, q, k, 1.0)


@pytest.mark.parametrize("k", [1, 5, 10])
def test_knn_plane_and_line_grids(ctx, k):
    """Degenerate grid shapes: a plane of exactly constant z (nz = 1) and a line along y (nx = nz = 1)."""
    rng = np.random.default_rng(60 + k)
    xy = rng.uniform(-10, 10, (20000, 2))
    plane = E.cloud(np.stack([xy[:, 0], xy[:, 1], np.full(20000, 1.5)], 1))
    line = E.cloud(np.stack([np.full(5000, 0.75), rng.uniform(-20, 20, 5000), np.full(5000, -2.25)], 1))
    for m, lo, hi in ((plane, (-11, -11, 0.5), (11, 11, 2.5)), (line, (-0.5, -21, -3.5), (2.0, 21, -1.0))):
        q = E.cloud(rng.uniform(lo, hi, (400, 3)))
        ctx.map_build(2, m, 0.5)
        _check_knn(ctx, 2, m, q, k, 2.0)


@pytest.mark.parametrize("k", [1, 10])
def test_knn_coarsened_grid(ctx, k):
    """50k points plus one outlier 1e5 m away at cell 0.25: the cell edge doubles until the grid fits, and then the whole
    cloud falls into one cell."""
    rng = np.random.default_rng(70 + k)
    m = np.concatenate([_rand_cloud(rng, 50000, 1, 20), E.cloud([[1e5, 1e5, 1e5]])])
    level, cell = E.grid_level(m, 0.25)
    assert level >= 8 and E.cell_counts(m, cell).max() >= 45000
    q = np.concatenate([_rand_cloud(rng, 60, 0, 21), E.cloud([[1e5 - 0.5, 1e5, 1e5]])])
    ctx.map_build(2, m, 0.25)
    _check_knn(ctx, 2, m, q, k, 1.0)


@pytest.mark.parametrize("offset", [FAR, np.array([2e4, -2e4, 2e4 / 3])])
@pytest.mark.parametrize("k", [1, 5, 10])
def test_knn_far_from_origin(ctx, k, offset):
    """test_knn_index_exact's random map, moved thousands of metres away; queries in a sensor frame through pose7."""
    rng = np.random.default_rng(100 + k)
    m = _rand_cloud(rng, 200000, -10, 10)[:40000]
    m = E.cloud(m[:, :3].astype(np.float64) + offset)
    q = _rand_cloud(rng, 800, -11, 11)
    pose = syn.pose7(offset, syn.quat_from_rpy(0.1, -0.2, 0.3))
    ctx.map_build(2, m, 0.5)
    ridx, _ = _check_knn(ctx, 2, m, q, k, 1.0, pose=pose)
    assert (ridx[:, k - 1] >= 0).sum() >= 100


@pytest.mark.parametrize("k", [1, 5, 10])
def test_knn_cell_faces(ctx, k):
    """Map points and queries whose coordinates are exact multiples of the cell (negative ones included), and queries
    outside the bounding box."""
    rng = np.random.default_rng(80 + k)
    cell = 0.5
    m = E.cloud(rng.integers(-8, 9, (6000, 3)) * cell)
    m = np.concatenate([m, E.cloud(rng.integers(-16, 17, (6000, 3)) * (cell / 2))])
    q = np.concatenate([E.cloud(rng.integers(-8, 9, (300, 3)) * cell), E.cloud(rng.integers(-11, 12, (300, 3)) * cell)])
    assert (np.abs(q[:, :3]) > 4.0).any(axis=1).sum() >= 50  # outside the bounding box
    ctx.map_build(2, m, cell)
    _check_knn(ctx, 2, m, q, k, 4.0)


def test_knn_radius_boundary(ctx):
    """A neighbour at exactly max_sqdist is excluded (d2 < max_sqdist); at nextafter(d2, +inf) it is included."""
    base = np.array([2731.25, -1873.875, 41.75])
    offs = np.array([[1, 0, 0], [0, -2, 0], [0, 0, 3], [-4, 0, 0]], np.float64)
    centres = [np.zeros(3), base, -base, np.array([-0.5, 0.25, 8.0])]
    m = E.cloud(np.concatenate([c + offs for c in centres]))
    q = E.cloud(np.array(centres))
    ctx.map_build(2, m, 0.5)
    for k in (1, 5):
        for j, d2 in enumerate((1.0, 4.0, 9.0, 16.0)):
            for r2, n_in in ((np.float32(d2), j), (np.nextafter(np.float32(d2), np.float32(np.inf)), j + 1)):
                idx, sqd = ctx.knn(2, q, k, float(r2))
                ridx, rsqd = E.knn_brute(m, q, k, float(r2))
                assert np.array_equal(idx, ridx) and np.array_equal(sqd, rsqd)
                assert np.all((idx >= 0).sum(1) == min(n_in, k))


def test_knn_non_finite(ctx):
    """NaN / Inf queries return -1 / inf; NaN / Inf map points are never returned and the others keep their indices."""
    rng = np.random.default_rng(90)
    m = _rand_cloud(rng, 20000, -5, 5)
    bad = rng.choice(20000, 600, replace=False)
    m[bad[:200], 0] = np.nan
    m[bad[200:400], 1] = np.inf
    m[bad[400:], 2] = -np.inf
    q = _rand_cloud(rng, 600, -5.5, 5.5)
    q[::7, 0] = np.nan
    q[1::11, 2] = np.inf
    q[2::13, 1] = -np.inf
    ctx.map_build(2, m, 0.5)
    for k in (1, 5, 10):
        idx, sqd = _check_knn(ctx, 2, m, q, k, 1.0, brute_oracle=False)
        assert not np.isin(idx, bad).any()
        nonfin = ~np.all(np.isfinite(q[:, :3]), axis=1)
        assert nonfin.sum() >= 100 and np.all(idx[nonfin] == -1) and np.all(np.isinf(sqd[nonfin]))


def test_knn_wide_ball(ctx):
    """A 20 m line of points every 2 mm, cell 0.002 (1 x 10001 x 1 cells), k = 1 within 5 m (DISTANCE_SQ_THRESHOLD):
    the ball of a query 0.3-4 m off the line spans more than 4096 cell rows, and its nearest point must still be found."""
    m = E.wide_ball_line(0.002)
    q = E.wide_ball_queries(np.random.default_rng(5), 256)
    ctx.map_build(2, m, 0.002)
    ridx, _ = _check_knn(ctx, 2, m, q, 1, 25.0, brute_oracle=False)
    assert np.all(ridx[:, 0] >= 0)
    assert (2 * np.sqrt(25.0) / 0.002 > 4096) and np.all(np.abs(q[:, 1] - 10) <= 4)


# ------------------------------------------------------------------------------------------------ 2. matcher decisions
def _far_c1():
    scene = syn.make_scene()
    traj = syn.trajectory(6)
    surf_map, corner_map = syn.make_submap(scene, 50000)
    cloud, ss, se = syn.make_sweep(scene, traj[4], 16, 1024, seed=4)
    f = orc.extract_cloud(cloud, ss, se)
    cs, _ = orc.voxel_grid(f["corner_points_less_sharp"], 0.2, True)
    sf, _ = orc.voxel_grid(f["surf_points_less_flat"], 0.4, True)
    init = np.array(syn.perturb_pose(traj[4], np.random.Generator(np.random.PCG64(11))))
    init[:3] += FAR
    move = lambda a: E.cloud(a[:, :3].astype(np.float64) + FAR, a[:, 3])
    return dict(surf_map=move(surf_map), corner_map=move(corner_map), surf_scan=sf, corner_scan=cs, init=init, cloud=cloud, ss=ss, se=se)


@pytest.fixture(scope="module")
def far_c1():
    return _far_c1()


def _matcher_maps(rng):
    """name -> (map, scan points in the sensor frame, pose7) for the degenerate neighbourhoods."""
    pose = syn.pose7([0.0625, -0.125, 0.25], [0, 0, 0, 1])
    inv = lambda w: E.cloud(w[:, :3].astype(np.float64) - pose[:3])
    out = {}
    for name, m in (("plane_axis", E.coplanar_patches(False)), ("plane_rot", E.coplanar_patches(True)), ("rods", E.rods())):
        out[name] = (m, inv(E.near(m, rng, 3000, 0.06)), pose)
    base = np.concatenate([E.coplanar_patches(False)[::3], E.rods()[::2]])
    dup = np.ascontiguousarray(np.repeat(base, 5, axis=0)[rng.permutation(base.shape[0] * 5)])
    out["dup5"] = (dup, inv(E.near(base, rng, 3000, 0.06)), pose)
    return out


@pytest.fixture(scope="module")
def matcher_maps():
    return _matcher_maps(np.random.default_rng(7))


def _compare_match(ctx, kind, m, data, pose, n_neigh, fov):
    slot = 0 if kind == "c" else 1
    ctx.set_params(n_neigh=n_neigh, check_fov=int(fov))
    try:
        ctx.map_build(slot, m, 0.5)
        valid, coeffs, nn = ctx.match_from_map(slot, kind, data, pose)
    finally:
        ctx.set_params(n_neigh=5, check_fov=0)
    rvalid, rcoeffs, rnn = orc.match_from_map(kind, m, data, pose, n_neigh=n_neigh, check_fov=fov)
    assert np.array_equal(valid, rvalid)
    assert np.array_equal(nn[valid], rnn[rvalid])
    if kind == "s":
        assert np.array_equal(coeffs[valid], rcoeffs[rvalid])
    else:
        a, b = coeffs[valid], rcoeffs[rvalid]
        same = np.all(a == b, axis=1)
        swapped = np.all(a[:, [3, 4, 5, 0, 1, 2]] == b, axis=1)
        assert np.all(same | swapped)
    return rvalid, rcoeffs, rnn


def degeneracy_counts(kind, m, data, pose, n_neigh, rvalid, rcoeffs, rnn, counts):
    """Adds to counts the queries whose K-set (within MIN_MATCH_SQ_DIS, as the matcher searches it) is rank 1 / rank 2,
    has an exactly diagonal scatter matrix, and (planes) the accepted fits with exactly zero residuals.  The oracle
    reports neighbours of accepted queries only, so the K-sets come from the brute force, which equals them there."""
    q = orc.associate(data, pose)
    nn, _ = E.knn_brute(m, q, n_neigh, orc.default_opts()[orc.O_MIN_MATCH_SQ])
    full = np.all(nn >= 0, axis=1)
    assert np.array_equal(nn[rvalid], rnn[rvalid])
    rank = E.neighbour_rank(m, nn[full])
    counts["rank1"] += int((rank == 1).sum())
    counts["rank2"] += int((rank == 2).sum())
    counts["diag"] += int(E.scatter_is_diagonal(m, nn[full]).sum())
    if kind == "s":
        counts["zero_res"] += int(E.plane_residual_zero(m, rnn[rvalid], rcoeffs[rvalid]).sum())
    return counts


@pytest.mark.parametrize("fov", [False, True])
@pytest.mark.parametrize("n_neigh", [5, 10])
@pytest.mark.parametrize("kind", ["s", "c"])
def test_match_degenerate_neighbourhoods(ctx, matcher_maps, kind, n_neigh, fov):
    counts = dict(rank1=0, rank2=0, diag=0, zero_res=0)
    for name, (m, data, pose) in matcher_maps.items():
        rvalid, rcoeffs, rnn = _compare_match(ctx, kind, m, data, pose, n_neigh, fov)
        degeneracy_counts(kind, m, data, pose, n_neigh, rvalid, rcoeffs, rnn, counts)
    need = ["rank1", "rank2", "diag"] + (["zero_res"] if kind == "s" else [])
    assert all(counts[c] >= 100 for c in need), counts


@pytest.mark.parametrize("kind", ["s", "c"])
def test_match_far_from_origin(ctx, far_c1, kind):
    m = far_c1["surf_map"] if kind == "s" else far_c1["corner_map"]
    data = far_c1["surf_scan"] if kind == "s" else far_c1["corner_scan"]
    for n_neigh, fov in ((5, False), (10, True)):
        rvalid, _, _ = _compare_match(ctx, kind, m, data, far_c1["init"], n_neigh, fov)
        assert rvalid.sum() >= 100


# ------------------------------------------------------------------------------------------------ 3. re-association shortcuts
def _context(mloam, p, **env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return mloam.Context(0, p)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k)
            else:
                os.environ[k] = v


def _same_solve(a, b):
    (pa, sa), (pb, sb) = a, b
    assert np.array_equal(pa, pb)
    for key in ("ran", "n_surf", "n_corner", "lm_iterations", "termination", "degenerate"):
        assert sa[key] == sb[key], key
    assert np.array_equal(np.asarray(sa["H"]), np.asarray(sb["H"])) and sa["final_cost"] == sb["final_cost"]


def _scan2map_case(name):
    rng = np.random.default_rng(11)
    surf, corner = E.coplanar_patches(False), E.rods()
    if name == "dup2":  # doubled, not x5: five copies of one point would reject every plane and line fit
        surf = np.ascontiguousarray(np.repeat(surf, 2, axis=0)[rng.permutation(surf.shape[0] * 2)])
        corner = np.ascontiguousarray(np.repeat(corner, 2, axis=0)[rng.permutation(corner.shape[0] * 2)])
    truth = syn.pose7([0.5, -0.25, 0.125], syn.quat_from_rpy(0.0, 0.0, 0.02))
    inv = syn.pose_inv(truth)
    ss = orc.associate(E.near(E.coplanar_patches(False), rng, 1500, 0.05), inv)
    cs = orc.associate(E.near(E.rods(), rng, 600, 0.05), inv)
    init = syn.pose7([0.55, -0.2, 0.1], syn.quat_from_rpy(0.005, -0.004, 0.03))
    return surf, corner, ss, cs, init


@pytest.mark.parametrize("case", ["lattice", "dup2", "far_c1"])
def test_reassociation_shortcuts_bit_identical(mloam, case):
    """scan2map with the keep / ball shortcuts off and on, serial and speculative schedule, and (far C1) the whole-frame
    stream path, graph capture and replay: identical results, and within the pose tolerance of the oracle."""
    if case == "far_c1":
        c = _far_c1()
        surf, corner, ss, cs, init = c["surf_map"], c["corner_map"], c["surf_scan"], c["corner_scan"], c["init"]
    else:
        surf, corner, ss, cs, init = _scan2map_case(case)
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell = 16, 10, 1, 0.5
    results = []
    for seeds in ("1", "0"):
        for fuse in ("0", "1"):
            cx = _context(mloam, p, MLOAM_DISABLE_SEEDS=seeds, MLOAM_FUSE_ITER=fuse)
            cx.map_build(1, surf, 0.5)
            cx.map_build(0, corner, 0.5)
            results.append(cx.scan2map(ss, cs, init))
            if seeds == "0" and fuse == "1":
                cx.profile(True)
                results.append(cx.scan2map(ss, cs, init))
                paths = {k: cx.profile_get(k)[1] for k in ("knn_keep_matched", "knn_keep_rejected", "knn_ball", "knn_blind")}
                cx.profile(False)
                assert paths["knn_ball"] >= 1, paths
                if case == "lattice":  # doubled points leave no slack between the K-th and the (K+1)-th: no keep there
                    assert paths["knn_keep_matched"] + paths["knn_keep_rejected"] >= 1, paths
            cx.close()
    for r in results[1:]:
        _same_solve(results[0], r)
    pose, st = results[0]
    assert st["ran"] == 1 and st["n_surf"] >= 100
    ref, rst = orc.scan2map(surf, corner, ss, cs, init, _opts(10, 1))
    dt, dr = syn.pose_err(pose, ref)
    assert dt <= POSE_TOL and dr <= POSE_TOL, (dt, dr)
    assert st["n_surf"] == int(rst["n_surf"]) and st["n_corner"] == int(rst["n_corner"])
    if case == "far_c1":
        cx = _context(mloam, p, MLOAM_FUSE_ITER="1")
        fr = [cx.frame(c["cloud"], c["ss"], c["se"], surf, corner, init) for _ in range(3)]  # stream, capture, replay
        cx.close()
        for r in fr:
            _same_solve(fr[0], r)
        assert fr[0][1]["n_surf_in"] == ss.shape[0] and fr[0][1]["n_corner_in"] == cs.shape[0]
        dt, dr = syn.pose_err(fr[0][0], ref)
        assert dt <= POSE_TOL and dr <= POSE_TOL, (dt, dr)


def _opts(outer, inner):
    o = orc.default_opts()
    o[orc.O_MAX_OUTER], o[orc.O_MAX_INNER] = outer, inner
    return o


# ------------------------------------------------------------------------------------------------ 4. voxel filters
def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("last", [False, True])
def test_voxel_path_boundary(ctx, last):
    """2047 / 2048 points take the in-CTA filter, 2049 the radix pipeline: the same prefix of one cloud on both."""
    pts = E.heavy_voxel_cloud(np.random.default_rng(3), 2049, 0.4)
    for n in (2047, 2048, 2049):
        out = ctx.voxel_downsample(pts[:n], 0.4, last)
        ref, ok = orc.voxel_grid(pts[:n], 0.4, last)
        assert ok and _same_bits(out, ref) and ref.shape[0] < n // 4


@pytest.mark.parametrize("leaf", [0.2, 0.4, 1.0])
def test_voxel_faces(ctx, leaf):
    pts = E.voxel_face_cloud(np.random.default_rng(int(leaf * 10)), leaf)
    on_face = (pts[:, :3] == np.round(pts[:, :3] / np.float32(leaf)) * np.float32(leaf)).all(1)
    assert on_face.sum() >= 500 and (pts[:, :3] < 0).any()
    for sub in (pts[:2000], pts):  # in-CTA and radix path
        for last in (False, True):
            out = ctx.voxel_downsample(sub, leaf, last)
            ref, ok = orc.voxel_grid(sub, leaf, last)
            assert ok and _same_bits(out, ref)


def test_voxel_one_heavy_voxel(ctx):
    """200k points in one voxel: the float centroid sum must follow the input order."""
    rng = np.random.default_rng(4)
    pts = E.cloud(rng.uniform(0.05, 0.95, (200000, 3)) + [3.0, -2.0, 1.0], rng.integers(0, 64, 200000))
    for last in (False, True):
        out = ctx.voxel_downsample(pts, 1.0, last)
        ref, ok = orc.voxel_grid(pts, 1.0, last)
        assert ok and ref.shape[0] == 1 and _same_bits(out, ref)
    # a different order gives a different float sum: the comparison above does test the order
    perm = pts[rng.permutation(pts.shape[0])]
    assert not _same_bits(orc.voxel_grid(perm, 1.0)[0], orc.voxel_grid(pts, 1.0)[0])


def test_voxel_far_from_origin(ctx, far_c1):
    pts = E.cloud(far_c1["cloud"][:, :3].astype(np.float64) + FAR, far_c1["cloud"][:, 3])
    for leaf, last in ((0.2, True), (0.4, False), (1.0, True)):
        out = ctx.voxel_downsample(pts, leaf, last)
        ref, ok = orc.voxel_grid(pts, leaf, last)
        assert ok and _same_bits(out, ref) and ref.shape[0] > 1000


@pytest.mark.parametrize("n", [1500, 6000])
def test_voxel_int32_index_space(ctx, n):
    """46340 x 46340 x 1 voxels fit PCL's int32 index space, 46341 x 46341 x 1 overflow (the input comes back unchanged),
    on the in-CTA path (n <= 2048) and the radix path, and for the covariance filter."""
    rng = np.random.default_rng(n)
    for span, fits in ((46340, True), (46341, False)):
        pts = E.index_space_cloud(rng, n, span, 1.0)
        assert (E.voxel_index_extent(pts, 1.0) <= 2**31 - 1) == fits
        out = ctx.voxel_downsample(pts, 1.0, True)
        ref, ok = orc.voxel_grid(pts, 1.0, True)
        assert ok == fits and _same_bits(out, ref)
        assert (ref.shape[0] < n) == fits
        cov6 = rng.uniform(0, 0.01, (n, 6)).astype(np.float32)
        tr = (cov6[:, 0] + cov6[:, 3] + cov6[:, 5]).astype(np.float32)
        gp, gc, gt = ctx.voxel_downsample_cov(pts, cov6, tr, 1.0, 1.0)
        rp, rc, rt, rok = orc.voxel_grid_cov(pts, cov6, tr, 1.0, 1.0)
        assert rok == fits and _same_bits(gp, rp) and _same_bits(gc, rc) and _same_bits(gt, rt)


def test_voxel_cov_trace_gate(ctx):
    """A point whose trace equals the threshold exactly is skipped, one just below it is kept."""
    rng = np.random.default_rng(12)
    pts = E.heavy_voxel_cloud(rng, 4000, 0.4)
    cov6 = np.zeros((4000, 6), np.float32)
    cov6[:, 0] = rng.choice(np.float32([0.25, 0.5, 0.75]), 4000)
    tr = cov6[:, 0].copy()
    for thr in (np.float32(0.5), np.nextafter(np.float32(0.5), np.float32(1))):
        gp, gc, gt = ctx.voxel_downsample_cov(pts, cov6, tr, 0.4, float(thr))
        rp, rc, rt, ok = orc.voxel_grid_cov(pts, cov6, tr, 0.4, float(thr))
        assert ok and _same_bits(gp, rp) and _same_bits(gc, rc) and _same_bits(gt, rt)
        assert np.all(gt < thr) if gt.size else True
    assert (tr == np.float32(0.5)).sum() >= 1000


# ------------------------------------------------------------------------------------------------ 5. extraction
LENGTHS = [5, 6, 7, 11, 12, 13, 255, 256, 257, 1023, 1024, 1025, 4095, 4096, 4097]


def _compare_extract(ctx, cloud, ss, se):
    got = ctx.extract_features(cloud, ss, se)
    curv, label = ctx.extract_debug(cloud.shape[0])
    ref = orc.extract_cloud(cloud, ss, se)
    assert np.array_equal(label, ref["label"])
    for k in ("corner_points_sharp", "corner_points_less_sharp", "surf_points_flat", "surf_points_less_flat"):
        assert _same_bits(got[k], ref[k]), k
    return ref


def test_extract_ring_lengths(ctx):
    cloud, ss, se = E.rings_cloud(LENGTHS, np.random.default_rng(1))
    assert list(se - ss) == LENGTHS
    ctx.set_params(n_scans=len(LENGTHS), max_ring_points=0)
    try:
        ref = _compare_extract(ctx, cloud, ss, se)
    finally:
        ctx.set_params(n_scans=64, max_ring_points=0)
    assert ref["corner_points_sharp"].shape[0] >= 20 and ref["surf_points_flat"].shape[0] >= 20


def test_extract_curvature_ties(ctx):
    pattern = np.zeros(16)
    pattern[3], pattern[11], pattern[7] = 40 / 64, -24 / 64, 8 / 64
    lengths = [1000, 999, 640]
    cloud, ss, se = E.rings_cloud(lengths, None, pattern=pattern)
    ctx.set_params(n_scans=len(lengths), max_ring_points=0)
    try:
        ref = _compare_extract(ctx, cloud, ss, se)
    finally:
        ctx.set_params(n_scans=64, max_ring_points=0)
    for s, e in zip(ss, se):
        c = ref["curvature"][s:e]
        assert np.unique(c).size < 0.1 * c.size
    assert ref["corner_points_sharp"].shape[0] >= 6 and ref["surf_points_flat"].shape[0] >= 6


def test_extract_window_and_ring_limits(ctx, mloam):
    """A ring whose on-chip window (scan_end - scan_start + 10) is exactly 12288 points is extracted; one point more is
    an error, not a partial result.  max_ring_points below the longest ring's sort capacity is an error too."""
    rng = np.random.default_rng(2)
    ctx.set_params(n_scans=1, max_ring_points=0)
    try:
        cloud, ss, se = E.rings_cloud([12278], rng)
        _compare_extract(ctx, cloud, ss, se)
        cloud, ss, se = E.rings_cloud([12279], rng)
        with pytest.raises(mloam.MloamError):
            ctx.extract_features(cloud, ss, se)
        cloud, ss, se = E.rings_cloud([300, 1025, 700], rng)
        ctx.set_params(n_scans=3, max_ring_points=1024)
        with pytest.raises(mloam.MloamError):
            ctx.extract_features(cloud, ss, se)
        ctx.set_params(max_ring_points=1025)
        _compare_extract(ctx, cloud, ss, se)
    finally:
        ctx.set_params(n_scans=64, max_ring_points=0)


# ------------------------------------------------------------------------------------------------ 6. normal equations
def _rows_c1(far: bool, huber_straddle: bool = False):
    c = _far_c1() if far else None
    if c is None:
        scene = syn.make_scene()
        traj = syn.trajectory(6)
        surf_map, corner_map = syn.make_submap(scene, 50000)
        cloud, ss, se = syn.make_sweep(scene, traj[4], 16, 1024, seed=4)
        f = orc.extract_cloud(cloud, ss, se)
        cs, _ = orc.voxel_grid(f["corner_points_less_sharp"], 0.2, True)
        sf, _ = orc.voxel_grid(f["surf_points_less_flat"], 0.4, True)
        init = syn.perturb_pose(traj[4], np.random.Generator(np.random.PCG64(11)))
        c = dict(surf_map=surf_map, corner_map=corner_map, surf_scan=sf, corner_scan=cs, init=init)
    vs, cfs, _ = orc.match_from_map("s", c["surf_map"], c["surf_scan"], c["init"])
    vc, cfc, _ = orc.match_from_map("c", c["corner_map"], c["corner_scan"], c["init"])
    pts = np.concatenate([c["surf_scan"][vs][:, :3], c["corner_scan"][vc][:, :3]]).astype(np.float64)
    coeffs = np.concatenate([cfs[vs], cfc[vc]])
    types = np.array([ord("s")] * int(vs.sum()) + [ord("c")] * int(vc.sum()), np.uint8)
    if huber_straddle:  # move every plane so that the residuals spread over 0.02 .. 0.5 around the Huber threshold 0.1
        rng = np.random.default_rng(3)
        s = types == ord("s")
        coeffs[s, 3] += rng.uniform(0.02, 0.5, int(s.sum())) * rng.choice([-1, 1], int(s.sum()))
    # features carry float points and coefficients (PointPlaneFeature): keep the rows exactly representable in float so
    # that the device and the references reduce the same rows
    coeffs = coeffs.astype(np.float32).astype(np.float64)
    return types, pts, coeffs, np.asarray(c["init"], np.float64)


@pytest.mark.parametrize("rows", ["c1", "far_c1", "huber"])
def test_normal_equations_against_fsum(ctx, rows):
    types, pts, coeffs, x = _rows_c1(rows == "far_c1", rows == "huber")
    huber_a = 0.1
    H, g, cost = ctx.normal_equations(types, pts, coeffs, 1.0, huber_a, x)
    rH, rg, rcost, Habs, gabs, cabs = E.normal_eq_fsum(types, pts, coeffs, 1.0, huber_a, x, orc.factor_eval, orc.huber)
    n = types.shape[0]
    assert n >= 500
    assert np.all(np.abs(H - rH) <= E.sum_error_bound(n, Habs))
    assert np.all(np.abs(g - rg) <= E.sum_error_bound(n, gabs))
    assert abs(cost - rcost) <= E.sum_error_bound(n, cabs)
    if rows == "huber":
        r = np.array([orc.factor_eval(0 if t == ord("s") else 1, p, cf, 1.0, x)[0][0] for t, p, cf in zip(types, pts, coeffs)])
        assert (np.abs(r) > huber_a).sum() >= 200 and (np.abs(r) < huber_a).sum() >= 200

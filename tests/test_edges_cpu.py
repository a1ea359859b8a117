"""CPU tests of the edge-case generators (tests/edges.py) and of the references they feed: the cases really contain the
ties, degenerate neighbourhoods and boundaries test_gpu_edges.py claims to hit, and the math.fsum normal equations
hold the oracle to the summation error bound the GPU test uses."""
import numpy as np
import pytest

import edges as E
import oracle_lib as orc
import test_gpu_edges as G


def test_knn_brute_matches_oracle_brute_force():
    rng = np.random.default_rng(1)
    shape = (12, 10, 8)
    m = E.lattice(shape, 0.125)
    q = E.lattice_queries(shape, 0.125, rng=rng, n=300)
    for k in (1, 5, 10):
        idx, sqd = E.knn_brute(m, q, k, 1.0)
        oidx, osqd = orc.knn(m, q, k, brute=True)
        assert np.array_equal(idx, oidx) and np.array_equal(sqd, osqd)
        _, s1 = E.knn_brute(m, q, k, 1.0, extra=1)
        assert E.boundary_ties(s1, k).mean() >= 0.3


def test_knn_brute_radius_and_non_finite():
    m = E.cloud([[1, 0, 0], [np.nan, 0, 0], [0, 2, 0], [0, 0, np.inf]])
    q = E.cloud([[0, 0, 0], [np.nan, 0, 0]])
    idx, sqd = E.knn_brute(m, q, 2, 4.0)
    assert idx.tolist() == [[0, -1], [-1, -1]] and sqd[0, 0] == 1.0 and np.isinf(sqd[0, 1])
    idx, _ = E.knn_brute(m, q, 2, float(np.nextafter(np.float32(4), np.float32(5))))
    assert idx[0].tolist() == [0, 2]


def test_knn_generators_hit_their_edges():
    rng = np.random.default_rng(2)
    assert E.cell_counts(E.dense_cell(rng, 3200, 0.5), 0.5).max() >= 3000
    m = np.concatenate([E.cloud(rng.uniform(1, 20, (50000, 3))), E.cloud([[1e5, 1e5, 1e5]])])
    level, cell = E.grid_level(m, 0.25)
    assert level >= 8 and E.cell_counts(m, cell).max() >= 45000
    line = E.wide_ball_line(0.002)
    ny = int(np.floor(line[:, 1].max() / np.float32(0.002))) + 1
    assert line.shape[0] == 10001 and ny > 2 * 4096 and E.grid_level(line, 0.002)[0] == 0
    base = E.cloud(rng.uniform(-1, 1, (100, 3)))
    dup, reps = E.duplicated(base, rng)
    assert dup.shape[0] == reps.sum() and reps.min() >= 2 and reps.max() <= 40


def test_matcher_maps_are_degenerate():
    """The oracle's neighbour sets on the degenerate maps: rank-1 and rank-2 sets, exactly diagonal scatter matrices and
    exactly zero plane residuals, each at least 100 times (what test_match_degenerate_neighbourhoods requires)."""
    maps = G._matcher_maps(np.random.default_rng(7))
    for kind in ("s", "c"):
        for n_neigh in (5, 10):
            counts = dict(rank1=0, rank2=0, diag=0, zero_res=0)
            for name, (m, data, pose) in maps.items():
                rvalid, rcoeffs, rnn = orc.match_from_map(kind, m, data, pose, n_neigh=n_neigh)
                G.degeneracy_counts(kind, m, data, pose, n_neigh, rvalid, rcoeffs, rnn, counts)
            need = ["rank1", "rank2", "diag"] + (["zero_res"] if kind == "s" else [])
            assert all(counts[c] >= 100 for c in need), (kind, n_neigh, counts)


def test_voxel_generators():
    rng = np.random.default_rng(3)
    assert E.voxel_index_extent(E.index_space_cloud(rng, 100, 46340), 1.0) == 46340 * 46340
    assert E.voxel_index_extent(E.index_space_cloud(rng, 100, 46341), 1.0) == 46341 * 46341 > 2**31 - 1
    for leaf in (0.2, 0.4, 1.0):
        pts = E.voxel_face_cloud(rng, leaf)
        k = pts[:, :3] / np.float32(leaf)
        assert (k == np.round(k)).all(1).sum() >= 500
    pts = E.heavy_voxel_cloud(rng, 2049, 0.4)
    assert orc.voxel_grid(pts, 0.4)[0].shape[0] < 2049 // 4


def test_extraction_generators():
    cloud, ss, se = E.rings_cloud([5, 256, 4097], np.random.default_rng(4))
    assert list(se - ss) == [5, 256, 4097] and se[-1] + 6 == cloud.shape[0]
    pattern = np.zeros(16)
    pattern[3], pattern[11], pattern[7] = 40 / 64, -24 / 64, 8 / 64
    cloud, ss, se = E.rings_cloud([1000, 640], None, pattern=pattern)
    ref = orc.extract_cloud(cloud, ss, se)
    for s, e in zip(ss, se):
        c = ref["curvature"][s:e]
        assert np.unique(c).size < 0.1 * c.size
        assert all(E.curvature_f32(cloud, i) == c[i - s] for i in range(s, s + 40))


@pytest.mark.parametrize("rows", ["c1", "far_c1", "huber"])
def test_oracle_normal_equations_within_fsum_bound(rows):
    """orc.normal_eq against the exactly summed normal equations, within 16 (n + 10) 2^-53 sum |terms| per entry."""
    types, pts, coeffs, x = G._rows_c1(rows == "far_c1", rows == "huber")
    rH, rg, rcost, Habs, gabs, cabs = E.normal_eq_fsum(types, pts, coeffs, 1.0, 0.1, x, orc.factor_eval, orc.huber)
    H, g, cost = orc.normal_eq(types, pts, coeffs, 1.0, 0.1, x)
    n = types.shape[0]
    assert n >= 500
    assert np.all(np.abs(H - rH) <= E.sum_error_bound(n, Habs))
    assert np.all(np.abs(g - rg) <= E.sum_error_bound(n, gabs))
    assert abs(cost - rcost) <= E.sum_error_bound(n, cabs)
    # the bound is not loose enough to pass anything: one row dropped breaks it
    H1, _, _ = orc.normal_eq(types[1:], pts[1:], coeffs[1:], 1.0, 0.1, x)
    assert np.any(np.abs(H1 - rH) > E.sum_error_bound(n, Habs))

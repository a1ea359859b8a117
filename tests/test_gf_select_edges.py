"""Good-feature selection on the device at its edges (-m gpu): k_gf_jaco + k_gf_select through mloam_good_features /
mloam_good_features_odom against the oracle on the scans of tests/gf_select_lib.py (which the CPU suite checks reach their
edges).  Matched flags, the selection and its length are compared exactly, rows to 1e-9 and H to 1e-12."""
import numpy as np
import pytest

import gf_select_lib as G
import oracle_lib as orc

pytestmark = pytest.mark.gpu

_maps = {}


def _map(ctx, slot, mp):
    if _maps.get(slot) is not mp:
        ctx.map_build(slot, mp, 0.5)
        _maps[slot] = mp


def _check(ctx, case, method, ratio, seed):
    slot = 1 if case["kind"] == "s" else 0
    _map(ctx, slot, case["map"])
    cov6 = case.get("cov6")
    out = ctx.good_features(slot, case["kind"], case["scan"], case["pose7"], method, ratio, seed, cov6=cov6)
    ref = orc.good_features(case["kind"], case["map"], case["scan"], case["pose7"], method, ratio, seed, cov6=cov6)
    assert np.array_equal(out["matched"], ref["matched"])
    assert np.allclose(out["jaco"], ref["jaco"], rtol=1e-9, atol=1e-11)
    first = next((i for i in range(min(len(out["sel"]), len(ref["sel"]))) if out["sel"][i] != ref["sel"][i]), None)
    assert len(out["sel"]) == len(ref["sel"]) and np.array_equal(out["sel"], ref["sel"]), (method, ratio, seed, first)
    assert np.allclose(out["H"], ref["H"], rtol=1e-9, atol=1e-12)
    return out, ref


# ------------------------------------------------------------------------------------------------ pool placement
@pytest.mark.parametrize("method,ratio", [(orc.GF_RND, 0.2), (orc.GF_RND, 0.8), (orc.GF_FPS, 0.2), (orc.GF_FPS, 0.8), (orc.GF_GD, 0.2),
                                          (orc.GF_GD, 0.8)])
@pytest.mark.parametrize("n", [22755, 22756, 25599, 25600, 51199, 51200, 70001])
def test_pool_regimes(ctx, n, method, ratio):
    """Shared memory holds the Fenwick tree, visited stamps and matched flags up to n = 22755, drops the flags from 22756, the
    stamps from 25600 and the tree from 51200; 70001 is above the tree's top power 65536."""
    out, _ = _check(ctx, G.pool_scan(n), method, ratio, 7)
    assert len(out["sel"]) == G.num_use_of(n, ratio)


# ------------------------------------------------------------------------------------------------ greedy rounds and batches
@pytest.mark.parametrize("subset,n,ratio", [(1, 4000, 0.8), (2, 4000, 0.5), (31, 31 * 120, 120.5 / (31 * 120)), (32, 32 * 120, 120.5 / (32 * 120)),
                                            (33, 33 * 120, 120.5 / (33 * 120)), (50, 4000, 0.02), (100, 4000, 0.01)])
def test_gd_subset_sizes(ctx, subset, n, ratio):
    assert G.subset_of(n, ratio) == subset
    for seed in (5, 99):
        _check(ctx, G.prefix_scan(n), orc.GF_GD, ratio, seed)


@pytest.mark.parametrize("ratio", [1.0, 0.5 / 4000, 1.5 / 4000])
def test_gd_quota_limits(ctx, ratio):
    """num_use == n (every matched feature, in random order), num_use == 0 and num_use == 1 (a round of n candidates)."""
    out, ref = _check(ctx, G.prefix_scan(4000), orc.GF_GD, ratio, 5)
    if ratio == 1.0:
        assert sorted(out["sel"].tolist()) == np.flatnonzero(ref["matched"]).tolist()
    else:
        assert len(out["sel"]) == 0 and np.array_equal(out["H"], 1e-6 * np.eye(6))


@pytest.mark.parametrize("distinct,copies,ratio", [(8, 40, 0.25), (20, 50, 0.02)])
def test_gd_exact_ties(ctx, distinct, copies, ratio):
    """Duplicated features give equal log dets: the candidate drawn first wins, within a batch (subset 4) and across the two
    batches of a subset-50 round."""
    for seed in (1, 2, 3):
        _check(ctx, G.tie_scan(distinct, copies), orc.GF_GD, ratio, seed)


@pytest.mark.parametrize("ratio", [0.4, 0.1, 0.02])
def test_odometry_corner_ties(ctx, ratio):
    c = G.odom_corner_case()
    _map(ctx, 0, c["map"])
    g = ctx.good_features_odom(0, "c", c["scan"], c["pivot"], c["pose_i"], c["ext"], ratio, 77)
    r = orc.good_features_odom("c", c["map"], c["scan"], c["pivot"], c["pose_i"], c["ext"], ratio, 77)
    assert np.array_equal(g["matched"], r["matched"]) and g["matched"].sum() > 100
    assert np.array_equal(g["jaco"], r["jaco"])
    assert np.array_equal(g["sel"], r["sel"]) and np.allclose(g["H"], r["H"], rtol=1e-9, atol=1e-12)


def test_fps_lattice_ties(ctx):
    """Lattice points equidistant from the last pick on different threads and warps: the smallest index wins."""
    c = G.lattice_scan()
    for seed in (1, 8):
        out, _ = _check(ctx, c, orc.GF_FPS, 0.5, seed)
        assert out["matched"].all()


# ------------------------------------------------------------------------------------------------ exits
def test_exits(ctx):
    _check(ctx, G.mixed_scan(15, 25), orc.GF_GD, 0.05, 2)          # 40-feature pool, subset 20: 20 repeated draws
    _check(ctx, G.mixed_scan(10, 190), orc.GF_GD, 0.6, 2)          # the pool runs out in the middle of a round
    c = G.mixed_scan(100, 1900)                                    # 95 % unmatched: the erase path
    for m in (orc.GF_RND, orc.GF_FPS, orc.GF_GD):
        _check(ctx, c, m, 0.2, 2)
    out, _ = _check(ctx, c, orc.GF_RND, 0.5, 2)                    # fewer matched features than num_use
    assert len(out["sel"]) == 100
    c = G.mixed_scan(200, 200)
    seed = G.seed_with_first_draw(400, lambda k: not c["is_matched"][k])
    _check(ctx, c, orc.GF_FPS, 0.3, seed)                          # fps from an unmatched start point
    out, _ = _check(ctx, G.mixed_scan(100, 200), orc.GF_FPS, 0.5, 2)  # every point visited before the quota
    assert len(out["sel"]) == 100


# ------------------------------------------------------------------------------------------------ non-finite points
def _nan_start_seed(c):
    return G.seed_with_first_draw(c["scan"].shape[0], lambda k: k == int(c["nan_at"][0]))


@pytest.mark.parametrize("case", ["one_nan", "one_nan_all_visited", "nan_start", "nan_tail"])
def test_fps_non_finite(ctx, case):
    """std::min(d, dist[j]) keeps a NaN distance, so a NaN point is never the arg-max; with only NaN points left the pick is
    index 1, visited or not, and a matched index 1 is selected again.  (Picking the NaN point, as fminf would, is invisible in
    the selection of one_nan, where it only delays the walk by an unmatched visit; one_nan_all_visited ends on it.)"""
    c = {"nan_tail": G.nan_tail_scan, "one_nan_all_visited": G.nan_mixed_scan}.get(case, G.nan_scan)()
    seeds = {"one_nan": (3, 12345), "one_nan_all_visited": (2,), "nan_start": (_nan_start_seed(c),), "nan_tail": (3,)}[case]
    for seed in seeds:
        out, _ = _check(ctx, c, orc.GF_FPS, 0.2 if case in ("one_nan", "nan_start") else 0.5, seed)
        if case == "nan_tail":
            assert (out["sel"] == 1).sum() > 100
        if case == "one_nan_all_visited":
            assert out["sel"][-1] == 1 and (out["sel"] == 1).sum() == 2


@pytest.mark.parametrize("method", [orc.GF_RND, orc.GF_GD])
def test_non_finite_rnd_gd(ctx, method):
    for c in (G.nan_scan(), G.nan_tail_scan()):
        out, _ = _check(ctx, c, method, 0.5, 3)
        assert not np.isin(out["sel"], c["nan_at"]).any() and len(set(out["sel"].tolist())) == len(out["sel"])


# ------------------------------------------------------------------------------------------------ k_gf_jaco's sqrt_info clamp
@pytest.mark.parametrize("method", [orc.GF_WO, orc.GF_GD])
def test_sqrt_info_clamp(ctx, method):
    """Per-point traces of 1/9 (the nearest double), one ulp either side, the first trace whose sqrt(1 / trace) is below 3,
    0 and +inf."""
    _check(ctx, G.clamp_scan(), method, 1.0 if method == orc.GF_WO else 0.2, 4)


# ------------------------------------------------------------------------------------------------ mloam_set_params
def test_set_params_refuses_gf_ratio_outside_unit_interval(ctx, mloam):
    c = G.c1()
    ctx.map_build(1, c["surf_map"], 0.5)
    ctx.map_build(0, c["corner_map"], 0.5)
    _maps.clear()
    ctx.set_params(max_outer=3, max_inner=4, gf_method=orc.GF_GD, gf_ratio=0.3, gf_seed=5)
    try:
        pose0, st0 = ctx.scan2map(c["surf_scan"], c["corner_scan"], c["init"])
        for bad in (1.5, float("nan"), -0.1, float("inf")):
            with pytest.raises(mloam.MloamError, match="gf_ratio"):
                ctx.set_params(gf_ratio=bad)
            assert ctx.params.gf_ratio == np.float32(0.3)
        pose1, st1 = ctx.scan2map(c["surf_scan"], c["corner_scan"], c["init"])
    finally:
        ctx.set_params(max_outer=2, max_inner=30, gf_method=0, gf_ratio=1.0, gf_seed=0)
    assert np.array_equal(pose0, pose1)
    for k in ("n_surf", "n_corner", "lm_iterations", "final_cost"):
        assert st0[k] == st1[k], k
    assert 0 < st0["n_surf"] <= int(0.3 * c["surf_scan"].shape[0])  # the selection ran with the ratio that was kept

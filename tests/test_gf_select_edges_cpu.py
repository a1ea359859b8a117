"""Good-feature selection at its edges, without a GPU: the plain-Python statement of goodFeatureMatching's loops
(tests/gf_select_lib.py) against the oracle's restatement, and checks that each generated scan reaches the edge it is for."""
import math

import numpy as np
import pytest

import gf_select_lib as G
import oracle_lib as orc

# generator, ratio the four methods run at
CASES = {
    "prefix": (lambda: G.prefix_scan(4000), 0.2),
    "pool_22756": (lambda: G.pool_scan(22756), 0.2),
    "ties_same_batch": (lambda: G.tie_scan(8, 40), 0.25),
    "ties_across_batches": (lambda: G.tie_scan(20, 50), 0.02),
    "lattice": (G.lattice_scan, 0.5),
    "pool_40_subset_20": (lambda: G.mixed_scan(15, 25), 0.05),
    "empty_mid_round": (lambda: G.mixed_scan(10, 190), 0.6),
    "unmatched_95": (lambda: G.mixed_scan(100, 1900), 0.2),
    "fps_all_visited": (lambda: G.mixed_scan(100, 200), 0.5),
    "one_nan": (G.nan_scan, 0.2),
    "one_nan_all_visited": (G.nan_mixed_scan, 0.5),
    "nan_tail": (G.nan_tail_scan, 0.5),
    "sqrt_info_clamp": (G.clamp_scan, 0.2),
}


def _agree(case, method, ratio, seed):
    """orc.good_features and the Python statement on the oracle's matched flags and rows: same sel in the same order, same H."""
    ref = orc.good_features(case["kind"], case["map"], case["scan"], case["pose7"], method, ratio, seed, cov6=case.get("cov6"))
    sel, H, info = G.select(method, ratio, seed, ref["matched"], ref["jaco"], case["scan"])
    assert np.array_equal(sel, ref["sel"]), (method, ratio, seed, sel[:10], ref["sel"][:10])
    assert np.allclose(H, ref["H"], rtol=1e-12, atol=1e-12)
    return ref, info


@pytest.mark.parametrize("seed", [1, 12345])
@pytest.mark.parametrize("method", [orc.GF_WO, orc.GF_RND, orc.GF_FPS, orc.GF_GD])
@pytest.mark.parametrize("name", list(CASES))
def test_statement_matches_oracle(name, method, seed):
    make, ratio = CASES[name]
    _agree(make(), method, 1.0 if method == orc.GF_WO else ratio, seed)


@pytest.mark.parametrize("ratio", [1.0, 0.4, 0.1, 0.02])
def test_statement_matches_oracle_odometry_corners(ratio):
    """Estimator::goodFeatureMatching's corner rows are all [1 0 0 0 0 0]: every greedy candidate ties with every other."""
    c = G.odom_corner_case()
    ref = orc.good_features_odom(c["kind"], c["map"], c["scan"], c["pivot"], c["pose_i"], c["ext"], ratio, 77)
    m = ref["matched"]
    assert m.sum() > 100 and np.array_equal(ref["jaco"][m], np.tile([1.0, 0, 0, 0, 0, 0], (int(m.sum()), 1)))
    sel, H, info = G.select(orc.GF_WO if ratio == 1.0 else orc.GF_GD, ratio, 77, m, ref["jaco"], c["scan"])
    assert np.array_equal(sel, ref["sel"]) and np.allclose(H, ref["H"], rtol=1e-12, atol=1e-12)
    if 0 < ratio < 1:
        assert all(len(t) == G.subset_of(len(m), ratio) for t in info["ties"]) and len(info["ties"]) == len(sel)


def test_pcg32_and_logdet_are_the_oracles():
    """The two primitives on their own: the draw sequence of the rnd loop over a pool that never shrinks below its size, and
    log det of random SPD matrices against the oracle's logdet_chol and numpy."""
    n = 1000
    sel, _ = orc.gf_select(orc.GF_RND, 0.05, 99, np.ones(n, np.uint8), np.zeros((n, 6)), np.zeros((n, 4), np.float32))
    rng, pool, want = G.Pcg32(99), list(range(n)), []
    for _ in range(len(sel)):
        j = rng.uniform(0, len(pool) - 1)
        want.append(pool.pop(j))
    assert np.array_equal(sel, want)
    r = np.random.default_rng(3)
    for _ in range(20):
        A = r.normal(size=(6, 6))
        M = A @ A.T + 1e-3 * np.eye(6)
        assert G.logdet(M.ravel().tolist()) == orc.lib().orc_logdet(6, orc._p(np.ascontiguousarray(M)))
        assert math.isclose(G.logdet(M.ravel().tolist()), np.linalg.slogdet(M)[1], rel_tol=1e-10)


# ------------------------------------------------------------------------------------------------ each generator reaches its edge
@pytest.mark.parametrize("n", [22755, 22756, 25599, 25600, 51199, 51200, 70001])
def test_pool_scans_have_their_size_and_match(n):
    c = G.pool_scan(n)
    assert c["scan"].shape == (n, 4) and c["scan"].dtype == np.float32
    if n in (22756, 70001):
        m = orc.good_features("s", c["map"], c["scan"], c["pose7"], orc.GF_WO, 1.0, 0)["matched"]
        assert m.mean() > 0.85


def test_pool_regime_boundaries():
    """The kernel's pool placement in 50 * 1024 words of shared memory: Fenwick tree (n + 1), visited stamps (n more),
    matched flags ((n + 3) / 4 words more).  The generated sizes sit on each side of each boundary and above the top power."""
    W = 50 * 1024
    fen = lambda n: n + 1 <= W
    vis = lambda n: 2 * n + 1 <= W
    mat = lambda n: 2 * n + 1 + (n + 3) // 4 <= W
    assert mat(22755) and not mat(22756) and vis(22756)
    assert vis(25599) and not vis(25600) and fen(25600)
    assert fen(51199) and not fen(51200)
    assert 70001 > 65536


@pytest.mark.parametrize("subset,n,ratio", [(1, 4000, 0.8), (2, 4000, 0.5), (31, 31 * 120, 120.5 / (31 * 120)), (32, 32 * 120, 120.5 / (32 * 120)),
                                            (33, 33 * 120, 120.5 / (33 * 120)), (50, 4000, 0.02), (100, 4000, 0.01)])
def test_gd_subset_sizes(subset, n, ratio):
    assert G.subset_of(n, ratio) == subset
    c = G.prefix_scan(n)
    _, info = _agree(c, orc.GF_GD, ratio, 5)
    assert info["max_heap"] == subset and info["exit"] == "quota"


def test_gd_quota_limits():
    n = 4000
    assert G.num_use_of(n, 1.0) == n and G.num_use_of(n, 0.5 / n) == 0 and G.num_use_of(n, 1.5 / n) == 1
    c = G.prefix_scan(n)
    ref, info = _agree(c, orc.GF_GD, 1.0, 5)  # every matched feature, in random order
    assert sorted(ref["sel"].tolist()) == np.flatnonzero(ref["matched"]).tolist() and info["exit"] == "empty"
    ref, info = _agree(c, orc.GF_GD, 0.5 / n, 5)
    assert len(ref["sel"]) == 0
    _, info = _agree(c, orc.GF_GD, 1.5 / n, 5)  # one round of n candidates: the unmatched leave the pool, so it never fills
    assert info["exit"] == "repeat" and info["max_heap"] > 3 * G.BATCH


def test_gd_ties_within_and_across_batches():
    _, info = _agree(G.tie_scan(8, 40), orc.GF_GD, 0.25, 1)
    assert any(len({p // G.BATCH for p in t}) == 1 for t in info["ties"])
    _, info = _agree(G.tie_scan(20, 50), orc.GF_GD, 0.02, 1)
    assert G.subset_of(1000, 0.02) == 50
    assert any(len({p // G.BATCH for p in t}) > 1 for t in info["ties"])


def test_fps_lattice_ties_span_threads_and_warps():
    c = G.lattice_scan()
    ref, info = _agree(c, orc.GF_FPS, 0.5, 1)
    assert ref["matched"].all()
    spread = [t for t in info["fps_ties"] if len({int(j) % 1024 // 32 for j in t}) > 1]
    assert len(spread) > 100 and any(int(t[0]) // 32 == int(t[1]) // 32 and t[0] != t[1] for t in info["fps_ties"])


def test_exits():
    _, info = _agree(G.mixed_scan(15, 25), orc.GF_GD, 0.05, 2)
    assert G.subset_of(40, 0.05) == 20 and info["exit"] == "repeat"
    _, info = _agree(G.mixed_scan(10, 190), orc.GF_GD, 0.6, 2)
    assert info["empty_mid_round"] and info["exit"] == "empty"
    c = G.mixed_scan(100, 1900)
    _, info = _agree(c, orc.GF_GD, 0.2, 2)
    assert info["erased"] > 1000
    ref, info = _agree(c, orc.GF_RND, 0.5, 2)  # fewer matched features than num_use: the pool runs dry
    assert info["exit"] == "empty" and len(ref["sel"]) == 100
    c = G.mixed_scan(200, 200)
    seed = G.seed_with_first_draw(400, lambda k: not c["is_matched"][k])
    ref, info = _agree(c, orc.GF_FPS, 0.3, seed)
    assert not ref["matched"][info["start"]] and info["start"] not in ref["sel"]
    ref, info = _agree(G.mixed_scan(100, 200), orc.GF_FPS, 0.5, 2)
    assert info["exit"] == "visited" and len(ref["sel"]) == 100


def test_non_finite_fps():
    c = G.nan_scan()
    ref, info = _agree(c, orc.GF_FPS, 0.2, 3)  # one NaN point: never the arg-max, so never visited
    assert 137 not in ref["sel"] and info["fallback"] == 0 and not ref["matched"][137]
    n = c["scan"].shape[0]
    seed = G.seed_with_first_draw(n, lambda k: k == 137)
    ref, info = _agree(c, orc.GF_FPS, 0.2, seed)  # a NaN start: every distance is NaN, so the first pick is index 1
    assert info["start"] == 137 and info["fallback"] == 1 and ref["sel"][0] == 1
    ref, info = _agree(G.nan_mixed_scan(), orc.GF_FPS, 0.5, 2)  # every finite point visited: the NaN one is never picked, index 1 is
    assert info["exit"] == "visited" and info["fallback"] == 1 and ref["sel"][-1] == 1 and (ref["sel"] == 1).sum() == 2
    c = G.nan_tail_scan()
    ref, info = _agree(c, orc.GF_FPS, 0.5, 3)  # the NaN tail outlasts the quota: index 1 again and again
    assert info["fallback"] > 100 and (ref["sel"] == 1).sum() == info["fallback"] + 1 and info["exit"] == "quota"
    for m in (orc.GF_RND, orc.GF_GD):
        ref, _ = _agree(c, m, 0.5, 3)
        assert not np.isin(ref["sel"], c["nan_at"]).any() and len(set(ref["sel"].tolist())) == len(ref["sel"])


def test_sqrt_info_clamp_traces():
    c = G.clamp_scan()
    traces = c["traces"]
    cov = c["cov6"].astype(np.float64)
    got = (cov[:, 0] + cov[:, 3]) + cov[:, 5]
    for i, t in enumerate(traces):
        assert got[i] == t
    branch = [t == 0 or math.sqrt(1 / t) >= 3.0 for t in traces]
    assert traces[0] == 1.0 / 9.0 and branch[:3] == [True, True, True] and branch[3] is False
    assert traces[3] > traces[2] and math.isinf(traces[5])
    ref, _ = _agree(c, orc.GF_WO, 1.0, 0)
    m = ref["matched"]
    inf_rows = ref["jaco"][np.arange(len(m)) % len(traces) == 5]
    assert np.all(inf_rows == 0) and m[np.arange(len(m)) % len(traces) == 5].any()

"""The matcher's query schedule and bound-pruned selection (k_match_knn: only blind searches are listed for the next launch,
scan_runs drops candidates beyond the search bound) against MLOAM_KNN_SCHEDULE=0, which lists every ball and blind search
and selects unpruned.  Neighbour lists, anchors (bit patterns, both halves), changed flags, pose, stats and H must be
bit-identical (neighbours compared by original map index), and stage profiling must count the same queries per search path."""
import ctypes as C
import os

import numpy as np
import pytest

import bench
import oracle_lib as orc
import synthetic as syn

pytestmark = pytest.mark.gpu

PATHS = ("knn_keep_matched", "knn_keep_rejected", "knn_ball", "knn_blind")


def _context(mloam, p, schedule):
    os.environ["MLOAM_KNN_SCHEDULE"] = schedule
    try:
        return mloam.Context(0, p)
    finally:
        os.environ.pop("MLOAM_KNN_SCHEDULE")


def _lists(mloam, cx, n_corner, n_surf):
    """(neighbours as original map indices, anchor bits, changed) of the corner and the surf set after the last solve, both
    halves.  Original indices, not positions in the cell-sorted map: those depend on the order of the map build's atomics."""
    out = []
    for s, n in ((0, n_corner), (1, n_surf)):
        nn = np.zeros(2 * n * 10, np.int32)
        anchor = np.zeros(2 * n * 4, np.float32)
        changed = np.zeros(n, np.uint8)
        k = C.c_int(0)
        rc = mloam.lib().mloam_debug_knn_lists(cx._h, s, n, nn.ctypes.data_as(C.c_void_p), anchor.ctypes.data_as(C.c_void_p),
                                               changed.ctypes.data_as(C.c_void_p), C.byref(k))
        assert rc == 0, rc
        out.append((nn[:2 * n * k.value].copy(), anchor.view(np.uint32).copy(), changed))
    return out


def _assert_same(a, b):
    (pa, sa, la), (pb, sb, lb) = a, b
    assert np.array_equal(pa, pb)
    for k in ("ran", "n_surf", "n_corner", "n_surf_in", "n_corner_in", "lm_iterations", "termination", "degenerate"):
        assert sa[k] == sb[k], k
    assert np.array_equal(np.asarray(sa["H"]), np.asarray(sb["H"]))
    assert sa["final_cost"] == sb["final_cost"]
    for s, ((nn_a, an_a, ch_a), (nn_b, an_b, ch_b)) in enumerate(zip(la, lb)):
        assert np.array_equal(nn_a, nn_b), (s, np.nonzero(nn_a != nn_b)[0][:16])
        assert np.array_equal(an_a, an_b), (s, np.nonzero(an_a != an_b)[0][:16])
        assert np.array_equal(ch_a, ch_b), (s, np.nonzero(ch_a != ch_b)[0][:16])


def _scan2map_both(mloam, p, surf_map, corner_map, sf, cs, init, cell):
    res = []
    for schedule in ("0", "1"):
        cx = _context(mloam, p, schedule)
        cx.map_build(1, surf_map, cell)
        cx.map_build(0, corner_map, cell)
        pose, st = cx.scan2map(sf, cs, init)
        res.append((pose, st, _lists(mloam, cx, cs.shape[0], sf.shape[0])))
        cx.close()
    return res


def test_schedule_full_size_frame(mloam):
    """C2 (64 x 2048 sweep, 1M-point keyframe submap, 10 GN iterations): stream path, graph capture and graph replay; then
    the same frame with stage profiling, whose per-path query counts must agree."""
    cfg = bench.CONFIGS["C2"]
    wl = bench.make_workload(syn, cfg, 1, 0, 1)
    fr = wl["frames"][0]
    g = fr["groups"][0]
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = cfg["rings"], cfg["gn_iters"], 1, 0.0, cfg["horizon"]
    res, paths = [], []
    for schedule in ("0", "1"):
        cx = _context(mloam, p, schedule)
        out = []
        for rebuild in (True, False, False, False):
            pose, st = cx.frame(g["cloud"], g["ss"], g["se"], wl["surf_map"], wl["corner_map"], fr["init"], rebuild)
            out.append((pose, st, _lists(mloam, cx, st["n_corner_in"], st["n_surf_in"])))
        cx.profile(True)
        cx.profile_reset()
        out.append(cx.frame(g["cloud"], g["ss"], g["se"], wl["surf_map"], wl["corner_map"], fr["init"], False) + (None,))
        paths.append([cx.profile_get(name)[1] for name in PATHS])
        cx.close()
        res.append(out)
    for a, b in zip(res[0][:-1], res[1][:-1]):
        assert a[1]["ran"] == 1 and a[1]["n_surf"] > 1000
        _assert_same(a, b)
    (pa, sa, _), (pb, sb, _) = res[0][-1], res[1][-1]
    assert np.array_equal(pa, pb) and np.array_equal(np.asarray(sa["H"]), np.asarray(sb["H"]))
    assert paths[0] == paths[1] and paths[0][2] > 0 and paths[0][3] > 0, paths


@pytest.mark.parametrize("cell", [0.5, 2.0])
def test_schedule_coarse_cells(mloam, cell):
    """C1 with a poor initial guess, on the default cell and on a 2 m cell (hundreds of points per cell, so most of a
    staged row lies outside the search ball)."""
    scene = syn.make_scene()
    traj = syn.trajectory(6)
    surf_map, corner_map = syn.make_submap(scene, 50000)
    cloud, ss, se = syn.make_sweep(scene, traj[4], 16, 1024, seed=4)
    f = orc.extract_cloud(cloud, ss, se)
    cs, _ = orc.voxel_grid(f["corner_points_less_sharp"], 0.2, True)
    sf, _ = orc.voxel_grid(f["surf_points_less_flat"], 0.4, True)
    init = np.array(syn.perturb_pose(traj[4], np.random.Generator(np.random.PCG64(11))), dtype=np.float64)
    init[:3] += 0.3
    p = mloam.default_params()
    p.max_outer, p.max_inner, p.map_cell = 10, 1, cell
    a, b = _scan2map_both(mloam, p, surf_map, corner_map, sf, cs, init, cell)
    assert a[1]["n_surf"] > 500
    _assert_same(a, b)


def test_schedule_ties_at_the_bound(mloam):
    """A lattice map and lattice queries (every coordinate a multiple of 1/8, so every squared distance is exact): many
    neighbours at equal distances, at the K-th and (K+1)-th place too.  Some map points sit at exactly 1.05 from a query
    along x, which is the blind search's first selection bound (radius 1 + pad 0.05) as a float, d2 == bound."""
    g = np.arange(-24, 25, dtype=np.float32) / 8.0
    xx, yy = np.meshgrid(g, g, indexing="ij")
    plane = np.stack([xx.ravel(), yy.ravel(), np.zeros(xx.size, np.float32)], 1)
    wall = np.stack([np.full(xx.size, 3.5, np.float32), xx.ravel(), yy.ravel() + 3.0], 1)
    at_bound = np.stack([np.full(9, np.float32(1.05)), (np.arange(9, dtype=np.float32) - 4) / 2, np.zeros(9, np.float32)], 1)
    surf_map = np.concatenate([plane, wall, at_bound]).astype(np.float32)
    surf_map = np.concatenate([surf_map, np.zeros((surf_map.shape[0], 1), np.float32)], 1)
    line = np.stack([np.full(64, 3.5, np.float32), np.full(64, -3.0, np.float32), np.arange(64, dtype=np.float32) / 8.0], 1)
    corner_map = np.concatenate([line, np.zeros((64, 1), np.float32)], 1)
    q = np.arange(-12, 13, dtype=np.float32) / 4.0
    qx, qy = np.meshgrid(q, q, indexing="ij")
    sf = np.stack([qx.ravel(), qy.ravel(), np.zeros(qx.size, np.float32), np.zeros(qx.size, np.float32)], 1)
    cs = np.stack([np.full(16, 3.5, np.float32), np.full(16, -3.0, np.float32), np.arange(16, dtype=np.float32) / 4.0,
                   np.zeros(16, np.float32)], 1)
    init = np.array([0, 0, 0, 0, 0, 0, 1], dtype=np.float64)
    p = mloam.default_params()
    p.max_outer, p.max_inner, p.map_cell = 10, 1, 0.5
    a, b = _scan2map_both(mloam, p, surf_map, corner_map, sf, cs, init, 0.5)
    assert a[1]["ran"] == 1
    _assert_same(a, b)

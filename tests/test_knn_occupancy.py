"""k_match_knn's default instance (at most 72 registers, three CTAs of 256 threads per SM beside one k_eval_candidate block) against
MLOAM_KNN_MB=2 (the same body compiled for two CTAs per SM).  Only register allocation, code layout and residency differ, so neighbour
lists (by original map index), anchors (bit patterns, both halves), changed flags, pose, stats and H must be bit-identical: C2 and C4 on
one GPU at full size on the stream path, the graph capture and the replay, a lattice map with exact ties, and a coarse cell where many
queries search blind.  The occupancy calculator must place three default CTAs on an SM."""
import ctypes as C
import os

import numpy as np
import pytest

import bench
import oracle_lib as orc
import synthetic as syn
from test_knn_schedule import _assert_same, _lists

pytestmark = pytest.mark.gpu


def _context(mloam, p, mb):
    if mb is not None:
        os.environ["MLOAM_KNN_MB"] = mb
    try:
        return mloam.Context(0, p)
    finally:
        os.environ.pop("MLOAM_KNN_MB", None)


def _residency(mloam, cx, k):
    ctas, regs = C.c_int(-1), C.c_int(-1)
    assert mloam.lib().mloam_debug_knn_residency(cx._h, k, C.byref(ctas), C.byref(regs)) == 0
    return ctas.value, regs.value


@pytest.mark.parametrize("name", ["C2", "C4"])
def test_full_size_frames(mloam, name):
    """The bench workload's first frame four times (map rebuilt, then stream path, capture, replay of the same key)."""
    cfg = bench.CONFIGS[name]
    wl = bench.make_workload(syn, cfg, 1, 0, 1)
    fr = wl["frames"][0]
    g = fr["groups"][0]
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = cfg["rings"] * cfg["lidars"], cfg["gn_iters"], 1, 0.0, cfg["horizon"]
    res = []
    for mb in ("2", None):
        cx = _context(mloam, p, mb)
        if cfg["lidars"] > 1:
            cx.set_lidars(cfg["lidars"], g["ext"])
        out = []
        for rebuild in (True, False, False, False):
            pose, st = cx.frame(g["cloud"], g["ss"], g["se"], wl["surf_map"], wl["corner_map"], fr["init"], rebuild)
            out.append((pose, st, _lists(mloam, cx, st["n_corner_in"], st["n_surf_in"])))
        cx.close()
        res.append(out)
    for a, b in zip(*res):
        assert a[1]["ran"] == 1 and a[1]["n_surf"] > 1000
        _assert_same(a, b)


def _scan2map_both(mloam, p, surf_map, corner_map, sf, cs, init, cell):
    res = []
    for mb in ("2", None):
        cx = _context(mloam, p, mb)
        cx.map_build(1, surf_map, cell)
        cx.map_build(0, corner_map, cell)
        pose, st = cx.scan2map(sf, cs, init)
        res.append((pose, st, _lists(mloam, cx, cs.shape[0], sf.shape[0])))
        cx.close()
    return res


def test_ties_on_a_lattice(mloam):
    """Lattice map and queries (coordinates multiples of 1/8: every squared distance is exact), so many neighbours tie, at the K-th
    and (K+1)-th place too, and some map points sit exactly on the blind search's first selection bound."""
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
    p = mloam.default_params()
    p.max_outer, p.max_inner, p.map_cell = 10, 1, 0.5
    a, b = _scan2map_both(mloam, p, surf_map, corner_map, sf, cs, np.array([0, 0, 0, 0, 0, 0, 1], dtype=np.float64), 0.5)
    assert a[1]["ran"] == 1
    _assert_same(a, b)


def test_blind_heavy_coarse_cell(mloam):
    """C1 with a poor initial guess on a 2 m cell: hundreds of points per cell, and the first launch and the queries that moved
    out of their ball search blind."""
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
    p.max_outer, p.max_inner, p.map_cell = 10, 1, 2.0
    a, b = _scan2map_both(mloam, p, surf_map, corner_map, sf, cs, init, 2.0)
    assert a[1]["n_surf"] > 500
    _assert_same(a, b)


def test_residency(mloam):
    """Three default CTAs per SM within the 72-register budget.  MLOAM_KNN_MB=2 selects the instance bounded for two (the launch
    asks for at most two CTAs per SM; the occupancy calculator may place more of it)."""
    p = mloam.default_params()
    for mb in (None, "2"):
        cx = _context(mloam, p, mb)
        try:
            for k in (5, 10):
                ctas, regs = _residency(mloam, cx, k)
                if mb is None:
                    assert ctas == 3 and regs <= 72, (k, ctas, regs)
                else:
                    assert ctas >= 2 and regs <= 128, (k, ctas, regs)
        finally:
            cx.close()

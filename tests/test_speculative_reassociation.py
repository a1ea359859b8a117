"""The speculative scan2map schedule (matcher of GN iteration i + 1 at the candidate pose of iteration i, next to the
evaluation of that candidate) against the serial reference schedule MLOAM_FUSE_ITER=0: results must be bit-identical,
whether the step of an iteration is taken (the speculative lists are used) or not (the previous lists and fit are kept)."""
import os

import numpy as np
import pytest

import bench
import oracle_lib as orc
import synthetic as syn

pytestmark = pytest.mark.gpu


def _context(mloam, p, fuse_iter):
    os.environ["MLOAM_FUSE_ITER"] = fuse_iter
    try:
        return mloam.Context(0, p)
    finally:
        os.environ.pop("MLOAM_FUSE_ITER")


def _assert_same(a, b):
    (pa, sa), (pb, sb) = a, b
    assert np.array_equal(pa, pb)
    for k in ("ran", "n_surf", "n_corner", "lm_iterations", "termination", "degenerate"):
        assert sa[k] == sb[k], k
    assert np.array_equal(np.asarray(sa["H"]), np.asarray(sb["H"]))
    assert sa["final_cost"] == sb["final_cost"]


def test_speculation_full_size_frame(mloam):
    """C2 (64 x 2048 sweep, 1M-point keyframe submap, 10 GN iterations): stream path, graph capture and graph replay."""
    cfg = bench.CONFIGS["C2"]
    wl = bench.make_workload(syn, cfg, 1, 0, 1)
    fr = wl["frames"][0]
    g = fr["groups"][0]
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = cfg["rings"], cfg["gn_iters"], 1, 0.0, cfg["horizon"]
    res = []
    for fuse in ("0", "1"):
        cx = _context(mloam, p, fuse)
        out = [cx.frame(g["cloud"], g["ss"], g["se"], wl["surf_map"], wl["corner_map"], fr["init"], rebuild)
               for rebuild in (True, False, False, False)]
        cx.close()
        res.append(out)
    for a, b in zip(*res):
        assert a[1]["ran"] == 1 and a[1]["n_surf"] > 1000
        _assert_same(a, b)


def test_speculation_with_steps_not_taken(mloam):
    """C1 with a poor initial guess: from GN iteration 7 on the pose no longer moves (the oracle confirms it), so the
    speculative lists of those iterations are discarded and the previous ones are kept."""
    scene = syn.make_scene()
    traj = syn.trajectory(6)
    surf_map, corner_map = syn.make_submap(scene, 50000)
    cloud, ss, se = syn.make_sweep(scene, traj[4], 16, 1024, seed=4)
    f = orc.extract_cloud(cloud, ss, se)
    cs, _ = orc.voxel_grid(f["corner_points_less_sharp"], 0.2, True)
    sf, _ = orc.voxel_grid(f["surf_points_less_flat"], 0.4, True)
    init = np.array(syn.perturb_pose(traj[4], np.random.Generator(np.random.PCG64(11))), dtype=np.float64)
    init[:3] += 0.6
    outer = 10
    poses = []
    for k in (outer - 2, outer - 1):
        o = orc.default_opts()
        o[orc.O_MAX_OUTER], o[orc.O_MAX_INNER] = k, 1
        poses.append(np.asarray(orc.scan2map(surf_map, corner_map, sf, cs, init, o)[0]))
    assert np.array_equal(poses[0], poses[1])  # GN iteration outer - 1 leaves the pose unchanged: a speculation is discarded
    p = mloam.default_params()
    p.max_outer, p.max_inner, p.map_cell = outer, 1, 0.5
    res = []
    for fuse in ("0", "1"):
        cx = _context(mloam, p, fuse)
        cx.map_build(1, surf_map, 0.5)
        cx.map_build(0, corner_map, 0.5)
        res.append(cx.scan2map(sf, cs, init))
        cx.close()
    assert res[0][1]["n_surf"] > 500
    _assert_same(*res)
    # The last GN iteration ended in the acceptance step without taking the step (0: rejected, 1: function tolerance; a zero
    # step would have ended with 2), so its candidate differed from x.  The GN iterations before it that left the pose
    # unchanged are the same computation (same x, same lists), so each of them ended the same way and the evaluation at the
    # next x discarded the speculative lists: the test covers that path, not only the one where the step is taken.
    assert res[1][1]["termination"] in (0, 1), res[1][1]["termination"]

"""GPU tests of mloam_calib_rig, the online-calibration step over the whole rig, and of mloam_calib_frame, its two-LiDAR case: both bit
for bit against the outputs of the former 12-DoF mloam_calib_frame (tests/golden/calib_frame_12dof.npz), mloam_calib_frame's collective
branch on a one-rank communicator, the rig against the oracle's rig restatement (oracle/orc_calib_rig.cpp) on 2, 3, 4 and 16 LiDARs with
and without priors, the edges, every error path, launches that do not depend on the rig size, and a frame path both calls leave alone."""
import ctypes as C
import os

import numpy as np
import pytest

import calib_rig_lib as crl
import oracle_lib as orc
import synthetic as syn

pytestmark = pytest.mark.gpu
POSE_TOL_T = 1e-4  # metres, the parity bound of test_gpu_parity
POSE_TOL_R = 1e-4  # radians
E4 = np.zeros((0, 4), np.float32)
MAX_ERR = [0.0, 0.0]


@pytest.fixture(scope="module")
def rctx(mloam):
    c = mloam.Context(0)
    yield c
    c.close()
    print(f"\ncalib_rig vs oracle: max pose difference {MAX_ERR[0]:.3e} m / {MAX_ERR[1]:.3e} rad")


@pytest.fixture(scope="module")
def case2():
    return syn.make_calib_case(syn.make_scene(), orc.extract_cloud, orc.voxel_grid, 16, 1024, 100_000)


_RIGS = {}


def rig_case(L, idx_ref):
    if (L, idx_ref) not in _RIGS:
        _RIGS[(L, idx_ref)] = crl.make_rig_case(syn.make_scene(), L, 16, 1024, 100_000, idx_ref=idx_ref)
    return _RIGS[(L, idx_ref)]


def _maps(ctx, surf_map, corner_map, own=False):
    ctx.map_build(0, corner_map, 0.25)
    ctx.map_build(1, surf_map, 0.25)
    if own:
        surf_c, _ = orc.voxel_grid(surf_map, 0.2, False)
        corner_c, _ = orc.voxel_grid(corner_map, 0.2, False)
        ctx.map_build(2, corner_c, 0.25)
        ctx.map_build(3, surf_c, 0.25)
        return surf_c, corner_c
    return None, None


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "calib_frame_12dof.npz")


def _equal_golden(g, name, pi, ec, st):
    assert np.array_equal(pi, g[f"{name}.pose_i"]) and np.array_equal(ec, g[f"{name}.ext_cal"])
    for k in crl.CALIB_GOLDEN_STATS:
        assert st[k] == g[f"{name}.{k}"], (k, st[k], g[f"{name}.{k}"])
    assert np.array_equal(np.asarray(st["H"]), g[f"{name}.H"])


@pytest.mark.parametrize("name", list(crl.CALIB_GOLDEN))
def test_calib_frame_and_two_lidar_rig_equal_the_12dof_golden(rctx, name):
    """mloam_calib_frame, and mloam_calib_rig on the same two LiDARs (both idx_ref), give bit for bit what the 12-DoF implementation of
    mloam_calib_frame gave (tests/golden/make_calib_golden.py), with the same launches."""
    g = np.load(GOLDEN)
    kind, outer, inner, groups, own = crl.CALIB_GOLDEN[name]
    cs = crl.calib_golden_inputs(kind)
    assert cs["sha256"] == str(g[f"{name}.inputs_sha256"]), "the seeded inputs changed"
    crl.calib_golden_maps(rctx, cs, own)
    sr, cr, sc, cc = crl.calib_golden_groups(cs, groups)
    l0 = rctx.launch_count()
    pi, ec, st = rctx.calib_frame(sr, cr, sc, cc, cs["pivot"], cs["pose_i_init"], cs["ext_ref"], cs["ext_cal_init"], outer, inner, own_cal_maps=own)
    launches = rctx.launch_count() - l0
    _equal_golden(g, name, pi, ec, st)
    for idx_ref in (0, 1):
        order = [0, 1] if idx_ref == 0 else [1, 0]
        s = [[sr, sc][k] for k in order]
        c = [[cr, cc][k] for k in order]
        e = [[cs["ext_ref"], cs["ext_cal_init"]][k] for k in order]
        l0 = rctx.launch_count()
        rpi, rex, rst, rows = rctx.calib_rig(s, c, cs["pivot"], cs["pose_i_init"], e, idx_ref, max_outer=outer, max_inner=inner, own_cal_maps=own)
        n = rctx.launch_count() - l0
        _equal_golden(g, name, rpi, rex[1 - idx_ref], rst)
        assert np.array_equal(rex[idx_ref], cs["ext_ref"]) and rows.sum() == st["n_surf"] and n == launches


CASES = [  # L, idx_ref, prior (0 off, 1 at the true extrinsics, 2 with ext_ref's target offset too), own maps, outer, inner
    (2, 0, 0, False, 10, 1), (2, 0, 1, False, 2, 4), (3, 0, 0, False, 10, 1), (3, 2, 1, False, 2, 4),
    (4, 0, 0, False, 10, 1), (4, 0, 1, False, 10, 1), (4, 2, 0, True, 2, 4), (4, 2, 1, True, 10, 1),
    (16, 0, 0, False, 2, 4), (16, 2, 1, False, 10, 1), (3, 0, 2, False, 10, 1), (4, 2, 2, False, 2, 4)]


@pytest.mark.parametrize("L,idx_ref,prior,own,outer,inner", CASES)
def test_rig_matches_oracle(rctx, L, idx_ref, prior, own, outer, inner):
    """prior 2: the constant ext_ref's PriorFactor has a non-zero residual, which enters only the cost (and so the function-tolerance
    test): final cost and termination must agree with the oracle, and the cost must carry that residual's 0.5 |r|^2."""
    rc = rig_case(L, idx_ref)
    surf_c, corner_c = _maps(rctx, rc["surf_map"], rc["corner_map"], own)
    kw = {}
    if prior:
        targets = rc["ext"].copy()
        if prior == 2:
            targets[idx_ref] = crl.perturb_ext(rc["ext"][idx_ref], 5, deg=3.0, t=0.2)
        kw = dict(prior7s=targets, prior_pos=2.0, prior_rot=5.0)
    pi, ex, st, rows = rctx.calib_rig(rc["surf"], rc["corner"], rc["pivot"], rc["pose_i_init"], rc["ext_init"], idx_ref, max_outer=outer,
                                      max_inner=inner, own_cal_maps=own, **kw)
    rpi, rex, rst, rrows = crl.calib_rig(rc["surf_map"], rc["corner_map"], rc["surf"], rc["corner"], rc["pivot"], rc["pose_i_init"], rc["ext_init"],
                                         idx_ref, max_outer=outer, max_inner=inner, surf_map_cal=surf_c, corner_map_cal=corner_c, **kw)
    assert st["termination"] == rst["termination"] and st["lm_iterations"] == rst["lm_iterations"]
    assert np.array_equal(rows, rrows) and st["n_surf"] == rst["rows"]
    assert st["final_cost"] == pytest.approx(rst["final_cost"], rel=1e-9, abs=1e-12)
    if prior == 2:
        r_ref, _ = crl.prior_factor_np(rc["ext_init"][idx_ref], kw["prior7s"][idx_ref], 2.0, 5.0)
        assert st["final_cost"] > 0.5 * float(r_ref @ r_ref) > 1e-2
    for got, ref in [(pi, rpi)] + [(ex[n], rex[n]) for n in range(L)]:
        dt, dr = syn.pose_err(got, ref)
        MAX_ERR[0], MAX_ERR[1] = max(MAX_ERR[0], dt), max(MAX_ERR[1], dr)
        assert dt <= POSE_TOL_T and dr <= POSE_TOL_R, (dt, dr)
    assert np.array_equal(ex[idx_ref], rc["ext_init"][idx_ref])


def test_rig_edges(rctx, case2):
    cs = case2
    _maps(rctx, cs["surf_map"], cs["corner_map"])
    ext2 = crl.perturb_ext(cs["ext_cal"], 2)
    ext2[3:] /= np.linalg.norm(ext2[3:])
    e3 = [cs["ext_ref"], cs["ext_cal_init"], ext2]
    pr3 = [cs["ext_ref"], cs["ext_cal"], cs["ext_cal"]]

    def both(surf, corner, ext, **kw):
        g = rctx.calib_rig(surf, corner, cs["pivot"], cs["pose_i_init"], ext, 0, max_outer=3, max_inner=2, **kw)
        r = crl.calib_rig(cs["surf_map"], cs["corner_map"], surf, corner, cs["pivot"], cs["pose_i_init"], ext, 0, max_outer=3, max_inner=2, **kw)
        assert g[2]["termination"] == r[2]["termination"] and g[2]["lm_iterations"] == r[2]["lm_iterations"] and np.array_equal(g[3], r[3])
        for n in range(len(ext)):
            assert max(syn.pose_err(g[1][n], r[1][n])) <= POSE_TOL_T
        assert max(syn.pose_err(g[0], r[0])) <= POSE_TOL_T
        return g

    # a calibrated LiDAR without features: unchanged without a prior, pulled to its prior with one
    g = both([cs["surf_ref"], cs["surf_cal"], E4], [cs["corner_ref"], cs["corner_cal"], E4], e3)
    assert g[3][2] == 0 and np.allclose(g[1][2], ext2, rtol=0, atol=1e-15)
    g = both([cs["surf_ref"], cs["surf_cal"], E4], [cs["corner_ref"], cs["corner_cal"], E4], e3, prior7s=pr3, prior_pos=1.0, prior_rot=1.0)
    assert max(syn.pose_err(g[1][2], cs["ext_cal"])) < max(syn.pose_err(ext2, cs["ext_cal"]))
    # every calibrated LiDAR empty (the frames between two N_CUMU_FEATURE accumulations): pose_i alone
    g = both([cs["surf_ref"], E4, None], [cs["corner_ref"], None, E4], e3)
    assert np.array_equal(g[1][1], e3[1]) or np.allclose(g[1][1], e3[1], rtol=0, atol=1e-15)
    # an empty reference cloud: the extrinsics alone, pose_i unchanged
    g = both([E4, cs["surf_cal"], cs["surf_cal"]], [E4, cs["corner_cal"], cs["corner_cal"]], e3)
    assert g[3][0] == 0 and np.allclose(g[0], cs["pose_i_init"], rtol=0, atol=1e-15)
    # nothing at all
    both([E4, E4], [E4, E4], e3[:2])
    # non-finite points match nothing and change nothing else
    bad = cs["surf_cal"].copy()
    bad[::7, 0] = np.nan
    bad[1::7, 1] = np.inf
    both([cs["surf_ref"], bad], [cs["corner_ref"], cs["corner_cal"]], e3[:2])


def test_rig_error_paths(mloam, rctx, case2):
    cs = case2
    _maps(rctx, cs["surf_map"], cs["corner_map"])
    s, c, e = [cs["surf_ref"], cs["surf_cal"]], [cs["corner_ref"], cs["corner_cal"]], [cs["ext_ref"], cs["ext_cal_init"]]
    bad_pose = cs["pose_i_init"].copy()
    bad_pose[0] = np.nan
    bad_ext = np.array(e)
    bad_ext[1, 4] = np.inf
    for kw in (dict(surf=[s[0]], corner=[c[0]], ext7s=[e[0]]), dict(surf=s * 9, corner=c * 9, ext7s=e * 9), dict(idx_ref=2), dict(idx_ref=-1),
               dict(pose_i7=bad_pose), dict(ext7s=bad_ext), dict(prior7s=[e[0], [np.nan] * 7], prior_pos=1.0), dict(prior_pos=np.inf, prior7s=e),
               dict(prior_rot=1.0), dict(max_outer=0), dict(max_inner=0), dict(huber_a=np.nan)):
        a = dict(surf=s, corner=c, pivot7=cs["pivot"], pose_i7=cs["pose_i_init"], ext7s=e)
        a.update(kw)
        with pytest.raises(mloam.MloamError, match=r"mloam error -1: calib_rig: "):
            rctx.calib_rig(**a)
    # the binding refuses lists whose lengths disagree before the library could read past them
    for kw in (dict(corner=[c[0]]), dict(ext7s=[e[0]]), dict(prior7s=[e[0]], prior_pos=1.0)):
        a = dict(surf=s, corner=c, pivot7=cs["pivot"], pose_i7=cs["pose_i_init"], ext7s=e)
        a.update(kw)
        with pytest.raises(ValueError):
            rctx.calib_rig(**a)
    lib = mloam.lib()
    st = mloam.SolveStats()
    pv, pi, ex = (np.ascontiguousarray(x, np.float64) for x in (cs["pivot"], cs["pose_i_init"], np.array(e)))
    cnt = np.array([-1, 0], np.int32)
    z = np.zeros(2, np.int32)
    p = mloam._p
    assert lib.mloam_calib_rig(rctx._h, 2, 0, None, p(cnt), None, p(z), p(pv), p(pi), p(ex), None, C.c_double(0), C.c_double(0), 1, 1,
                               C.c_double(1.0), 0, C.byref(st), None) == -1
    assert lib.mloam_calib_rig(None, 2, 0, None, p(z), None, p(z), p(pv), p(pi), p(ex), None, C.c_double(0), C.c_double(0), 1, 1,
                               C.c_double(1.0), 0, C.byref(st), None) == -1
    one = np.array([5, 0], np.int32)  # a count without its cloud
    assert lib.mloam_calib_rig(rctx._h, 2, 0, None, p(one), None, p(z), p(pv), p(pi), p(ex), None, C.c_double(0), C.c_double(0), 1, 1,
                               C.c_double(1.0), 0, C.byref(st), None) == -1
    # own_cal_maps without the scan slots, and a context without maps
    fresh = mloam.Context(0)
    try:
        with pytest.raises(mloam.MloamError, match=r"mloam error -4:"):
            fresh.calib_rig(s, c, cs["pivot"], cs["pose_i_init"], e)
        _maps(fresh, cs["surf_map"], cs["corner_map"])
        with pytest.raises(mloam.MloamError, match=r"mloam error -4:"):
            fresh.calib_rig(s, c, cs["pivot"], cs["pose_i_init"], e, own_cal_maps=True)
    finally:
        fresh.close()


def test_rig_with_a_communicator_is_refused(mloam, case2):
    """A communicator is attached with mloam_comm_init (one rank); the rig call is single-GPU and returns MLOAM_E_STATE."""
    import torch  # noqa: F401  (loads the libnccl.so.2 the library resolves)
    cs = case2
    c = mloam.Context(0)
    try:
        lib = mloam.lib()
        uid = C.create_string_buffer(128)
        if lib.mloam_comm_unique_id(uid) != 0 or lib.mloam_comm_init(c._h, 1, 0, uid) != 0:
            pytest.fail("mloam_comm_init with one rank: " + str(lib.mloam_last_error(c._h)))
        _maps(c, cs["surf_map"], cs["corner_map"])
        st = mloam.SolveStats()
        p = mloam._p
        pv, pi, ex = (np.ascontiguousarray(x, np.float64) for x in (cs["pivot"], cs["pose_i_init"], np.array([cs["ext_ref"], cs["ext_cal_init"]])))
        z = np.zeros(2, np.int32)
        assert lib.mloam_calib_rig(c._h, 2, 0, None, p(z), None, p(z), p(pv), p(pi), p(ex), None, C.c_double(0), C.c_double(0), 1, 1,
                                   C.c_double(1.0), 0, C.byref(st), None) == -4
        lib.mloam_comm_destroy(c._h)
    finally:
        c.close()


def test_calib_frame_with_a_one_rank_communicator(mloam, case2):
    """With a communicator attached (one rank), mloam_calib_frame all-reduces each evaluation's sums: the results are those without one, at one
    more launch per evaluation (2 per outer iteration at max_inner 1)."""
    import torch  # noqa: F401  (loads the libnccl.so.2 the library resolves)
    cs = case2
    out = []
    for with_comm in (False, True):
        c = mloam.Context(0)
        try:
            if with_comm:
                lib = mloam.lib()
                uid = C.create_string_buffer(128)
                if lib.mloam_comm_unique_id(uid) != 0 or lib.mloam_comm_init(c._h, 1, 0, uid) != 0:
                    pytest.fail("mloam_comm_init with one rank: " + str(lib.mloam_last_error(c._h)))
            _maps(c, cs["surf_map"], cs["corner_map"])
            l0 = c.launch_count()
            pi, ec, st = c.calib_frame(cs["surf_ref"], cs["corner_ref"], cs["surf_cal"], cs["corner_cal"], cs["pivot"], cs["pose_i_init"],
                                       cs["ext_ref"], cs["ext_cal_init"], 10, 1)
            out.append((pi, ec, st, c.launch_count() - l0))
            if with_comm:
                lib.mloam_comm_destroy(c._h)
        finally:
            c.close()
    (pi, ec, st, n), (pi1, ec1, st1, n1) = out
    assert np.array_equal(pi, pi1) and np.array_equal(ec, ec1) and n1 == n + 2 * 10
    for k in crl.CALIB_GOLDEN_STATS:
        assert st[k] == st1[k], k
    assert np.array_equal(np.asarray(st["H"]), np.asarray(st1["H"]))


def test_rig_launches_do_not_depend_on_the_rig_size(rctx):
    counts = []
    for L in (2, 4):
        rc = rig_case(L, 0)
        _maps(rctx, rc["surf_map"], rc["corner_map"])
        l0 = rctx.launch_count()
        _, _, st, _ = rctx.calib_rig(rc["surf"], rc["corner"], rc["pivot"], rc["pose_i_init"], rc["ext_init"], 0, max_outer=3, max_inner=1)
        counts.append(rctx.launch_count() - l0)
    assert counts[0] == counts[1] == 3 * 7, counts


def test_rig_call_leaves_the_frame_path_alone(mloam, case2):
    """A frame after a calibration call (mloam_calib_rig or mloam_calib_frame) computes and launches what it would without one."""
    cs = case2
    scene = syn.make_scene()
    traj = syn.trajectory(3)
    cloud, ss, se = syn.make_sweep(scene, traj[1], 16, 1024, seed=1)
    surf_map, corner_map = syn.make_submap(scene, 50000)
    init = syn.perturb_pose(traj[1], np.random.Generator(np.random.PCG64(3)))
    p = mloam.default_params()
    p.n_scans = 16
    out = []
    for call in (None, "calib_rig", "calib_frame"):
        c = mloam.Context(0, p)
        try:
            _maps(c, cs["surf_map"], cs["corner_map"])
            c.frame(cloud, ss, se, surf_map, corner_map, init)
            if call:
                _maps(c, cs["surf_map"], cs["corner_map"])
            if call == "calib_rig":
                c.calib_rig([cs["surf_ref"], cs["surf_cal"]], [cs["corner_ref"], cs["corner_cal"]], cs["pivot"], cs["pose_i_init"],
                            [cs["ext_ref"], cs["ext_cal_init"]])
            elif call == "calib_frame":
                c.calib_frame(cs["surf_ref"], cs["corner_ref"], cs["surf_cal"], cs["corner_cal"], cs["pivot"], cs["pose_i_init"], cs["ext_ref"],
                              cs["ext_cal_init"])
            l0 = c.launch_count()
            pose, st = c.frame(cloud, ss, se, surf_map, corner_map, init)
            out.append((pose, st, c.launch_count() - l0))
        finally:
            c.close()
    for o in out[1:]:
        assert np.array_equal(out[0][0], o[0]) and out[0][2] == o[2]
        for k, v in out[0][1].items():
            assert np.array_equal(np.asarray(v), np.asarray(o[1][k])), k

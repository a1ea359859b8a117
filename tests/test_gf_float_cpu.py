"""gd_float on the CPU: the oracle's evalFullHessian against numpy, the ratio policy of lidar_mapper_keyframe.cpp:456-495 over a run of
frames, and the new entry points at the library boundary."""
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import gf_float_lib as gfl
import oracle_lib as orc
import synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def case():
    scene = syn.make_scene()
    traj = syn.trajectory(6)
    surf_map, corner_map = syn.make_submap(scene, 20000)
    cloud, ss, se = syn.make_sweep(scene, traj[4], 16, 512, seed=4)
    f = orc.extract_cloud(cloud, ss, se)
    cs, _ = orc.voxel_grid(f["corner_points_less_sharp"], 0.2, True)
    sf, _ = orc.voxel_grid(f["surf_points_less_flat"], 0.4, True)
    rng = np.random.Generator(np.random.PCG64(11))
    return dict(truth=traj[4], surf_map=surf_map, corner_map=corner_map, corner_scan=cs, surf_scan=sf, init=syn.perturb_pose(traj[4], rng))


def _opts(ratio=0.4):
    o = orc.default_opts()
    o[orc.O_GF_METHOD], o[orc.O_GF_RATIO], o[orc.O_GF_SEED] = orc.GF_GD, ratio, 7
    return o


def _inits(case, n):
    """Pose guesses of n frames: near the truth, except frames 15..24 which start 0.6 m off (fewer matches, a smaller factor)."""
    rng = np.random.Generator(np.random.PCG64(3))
    out = []
    for k in range(1, n + 1):
        x = syn.perturb_pose(case["truth"], rng)
        if 15 <= k <= 24:
            x[0] += 0.6
        out.append(x)
    return out


def test_full_hessian_is_the_serial_sum(case):
    H = None
    n_all = 0
    chain = []
    for kind, mp, sc in (("s", case["surf_map"], case["surf_scan"]), ("c", case["corner_map"], case["corner_scan"])):
        ref = orc.good_features(kind, mp, sc, case["init"], orc.GF_WO, 1.0, 0)
        one, n_one = gfl.full_hessian(kind, mp, sc, case["init"])
        assert n_one == int(ref["matched"].sum()) > 20
        assert one.tobytes() == gfl.serial_hessian(ref["jaco"], ref["matched"]).tobytes()
        assert one.tobytes() == ref["H"].tobytes()  # wo_gf adds the same rows in the same order
        H = gfl.serial_hessian(ref["jaco"], ref["matched"], H)
        n_all += n_one
        chain.append((kind, mp, sc))
    Hc, nc = None, 0
    for kind, mp, sc in chain:  # surf then corner into one mat_H, as :463-467
        Hc, nc = gfl.full_hessian(kind, mp, sc, case["init"], H=Hc, feat_num=nc)
    assert Hc.tobytes() == H.tobytes() and nc == n_all
    ld = orc.lib().orc_logdet
    ld.restype = __import__("ctypes").c_double
    got = ld(6, orc._p(np.ascontiguousarray(Hc)))
    assert abs(got - np.linalg.slogdet(Hc)[1]) <= 1e-12 * abs(got)
    # no features, and features without any map support, leave mat_H and feat_num alone
    H0, n0 = gfl.full_hessian("s", case["surf_map"], np.zeros((0, 4), np.float32), case["init"], H=Hc, feat_num=5)
    far = case["surf_scan"].copy()
    far[:, :3] += 1000.0
    H1, n1 = gfl.full_hessian("s", case["surf_map"], far, case["init"], H=Hc, feat_num=5)
    assert H0.tobytes() == Hc.tobytes() == H1.tobytes() and n0 == n1 == 5


def _run(case, inits, thre, ratio=0.4, gate_fail=()):
    gfl.gf_float_set(True, thre, ratio)
    log = []
    try:
        for k, x in enumerate(inits, 1):
            cm = case["corner_map"][:5] if k in gate_fail else case["corner_map"]
            pose, st = gfl.scan2map(case["surf_map"], cm, case["surf_scan"], case["corner_scan"], x, _opts(ratio))
            g = gfl.gf_float_get()
            log.append(dict(g, pose=pose, n_surf=int(st["n_surf"]), n_corner=int(st["n_corner"]), ran=int(st["ran"])))
    finally:
        gfl.gf_float_set(False)
    return log


def test_policy_over_35_frames(case):
    inits = _inits(case, 35)
    free = _run(case, inits, -1e30)  # every evaluation above the threshold: the ratio stays gf_ratio_ini
    assert [g["frame_cnt"] for g in free] == list(range(1, 36))
    assert [k for k, g in enumerate(free, 1) if g["evaluated"]] == [10, 20, 30]
    f10, f20, f30 = (free[k - 1]["deg_factor"] for k in (10, 20, 30))
    assert f20 < min(f10, f30)  # the frames that start far off see less of the map
    assert all(g["ratio_cur"] == 0.4 for g in free) and free[8]["deg_factor"] == 0.0 and free[10]["deg_factor"] == f10
    assert free[9]["total_feat_num"] > free[19]["total_feat_num"] > 0
    # a threshold between the factors: ini -> 0.8 -> ini, each from its evaluation frame on
    mid = 0.5 * (f20 + min(f10, f30))
    sw = _run(case, inits, mid)
    assert [g["ratio_cur"] for g in sw] == [0.4] * 19 + [0.8] * 10 + [0.4] * 6
    assert [g["deg_factor"] for g in sw] == [g["deg_factor"] for g in free]
    n_in = case["surf_scan"].shape[0]
    assert all(g["n_surf"] <= int(n_in * g["ratio_cur"]) for g in sw)
    assert sw[24]["n_surf"] > int(n_in * 0.4)  # the larger ratio is really used
    # the boundary: `>` against MAP_DEG_THRE as a float — at the float at-or-above the factor 0.8, one float ulp below ini
    at, below = gfl.float_at_or_above(f10)
    assert _run(case, inits[:10], at)[9]["ratio_cur"] == 0.8
    assert _run(case, inits[:10], below)[9]["ratio_cur"] == 0.4
    # the ratio before the first evaluation is min(1, ini), also for ini > 1; after an evaluation above the threshold it is ini itself
    big = _run(case, inits[:10], -1e30, ratio=1.5)
    assert [g["ratio_cur"] for g in big] == [1.0] * 9 + [1.5]


def test_map_gate_failure_counts_but_does_not_evaluate(case):
    inits = _inits(case, 12)
    log = _run(case, inits, -1e30, gate_fail=(10,))
    assert [g["frame_cnt"] for g in log] == list(range(1, 13))
    assert log[9]["ran"] == 0 and not any(g["evaluated"] for g in log)
    assert np.array_equal(log[9]["pose"], inits[9])


def test_mode_off_is_gd_fix(case):
    x = case["init"]
    args = (case["surf_map"], case["corner_map"], case["surf_scan"], case["corner_scan"], x, _opts())
    a, sa = orc.scan2map(*args)  # the oracle's gd_fix
    gfl.gf_float_set(True, -1e30, 0.4)  # on, and the ratio is ini throughout the first nine frames: the same selection
    try:
        b, sb = gfl.scan2map(*args)
        assert gfl.gf_float_get()["frame_cnt"] == 1
    finally:
        gfl.gf_float_set(False)
    c, sc = gfl.scan2map(*args)  # off
    assert gfl.gf_float_get()["frame_cnt"] == 0
    assert a.tobytes() == b.tobytes() == c.tobytes()
    assert int(sa["n_surf"]) == sb["n_surf"] == sc["n_surf"] and sa["H"].tobytes() == sb["H"].tobytes() == sc["H"].tobytes()


def test_entry_points_at_the_boundary(mloam):
    names = ("mloam_full_hessian", "mloam_set_gf_float", "mloam_set_gf_float_threshold", "mloam_gf_float_report")
    hdr = open(os.path.join(ROOT, "include", "mloam_b200.h")).read()
    lib = mloam.lib()
    for n in names:
        assert re.search(r"\bint " + n + r"\(", hdr), n
        assert n in mloam.ABI_SYMBOLS and hasattr(lib, n), n
    # the reference-shaped wrappers: the adapter against the stand-in PCL / Eigen headers, the shim with plain g++
    with tempfile.TemporaryDirectory() as td:
        for src, inc in (("gf_float_adapter_compile_test.cpp", ["-I" + os.path.join(ROOT, "tests", "stubs")]),
                         ("gf_float_shim_compile_test.cpp", ["-I" + os.path.join(ROOT, "m-loam_b200", "host"), "-I" + os.path.join(ROOT, "include")])):
            obj = os.path.join(td, src + ".o")
            out = subprocess.run(["g++", "-std=c++14", "-Wall", "-Werror", *inc, "-c", os.path.join(ROOT, "tests", "stubs", src), "-o", obj],
                                 capture_output=True, text=True)
            assert out.returncode == 0, out.stderr[-3000:]
            syms = subprocess.run(["nm", "-C", obj], capture_output=True, text=True).stdout
            assert "U mloam_full_hessian" in syms, src

"""CPU tests of the rig calibration (mloam_calib_rig): the oracle's rig restatement (oracle/orc_calib_rig.cpp) against orc_calib_frame,
its convergence, its PriorFactor against a numpy statement of prior_factor.hpp, a calibrated LiDAR without rows; the new symbol in the
header, the library and the binding; the adapter's and the shim's wrappers compiled against the stubs, the adapter's host PriorFactor;
the kernels' ptxas budget."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import calib_rig_lib as crl
import oracle_lib as orc
import synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = "/usr/local/cuda/bin/nvcc"


@pytest.fixture(scope="module")
def case2():
    return syn.make_calib_case(syn.make_scene(), orc.extract_cloud, orc.voxel_grid, 16, 1024, 100_000)


@pytest.mark.parametrize("outer,inner", [(10, 1), (2, 4)])
def test_rig_oracle_two_lidars_equals_calib_frame(case2, outer, inner):
    cs = case2
    rpi, rec, rst = orc.calib_frame(cs["surf_map"], cs["corner_map"], cs["surf_ref"], cs["corner_ref"], cs["surf_cal"], cs["corner_cal"], cs["pivot"],
                                    cs["pose_i_init"], cs["ext_ref"], cs["ext_cal_init"], outer, inner)
    pi, ex, st, rows = crl.calib_rig(cs["surf_map"], cs["corner_map"], [cs["surf_ref"], cs["surf_cal"]], [cs["corner_ref"], cs["corner_cal"]],
                                     cs["pivot"], cs["pose_i_init"], [cs["ext_ref"], cs["ext_cal_init"]], 0, max_outer=outer, max_inner=inner)
    assert np.array_equal(pi, rpi) and np.array_equal(ex[1], rec) and np.array_equal(ex[0], cs["ext_ref"])
    assert st == rst and rows.sum() == rst["rows"]
    # the same problem with the reference LiDAR second
    pi1, ex1, st1, rows1 = crl.calib_rig(cs["surf_map"], cs["corner_map"], [cs["surf_cal"], cs["surf_ref"]], [cs["corner_cal"], cs["corner_ref"]],
                                         cs["pivot"], cs["pose_i_init"], [cs["ext_cal_init"], cs["ext_ref"]], 1, max_outer=outer, max_inner=inner)
    assert np.array_equal(pi1, rpi) and np.array_equal(ex1[0], rec) and st1 == rst and np.array_equal(rows1, rows[::-1])


def test_rig_oracle_reduces_every_extrinsic_error():
    rc = crl.make_rig_case(syn.make_scene(), 4, 16, 1024, 100_000)
    pi, ex, st, rows = crl.calib_rig(rc["surf_map"], rc["corner_map"], rc["surf"], rc["corner"], rc["pivot"], rc["pose_i_init"], rc["ext_init"],
                                     0, max_outer=10, max_inner=1)
    assert np.all(rows > 0) and st["rows"] == rows.sum()
    for n in range(1, 4):
        e0, e1 = syn.pose_err(rc["ext_init"][n], rc["ext"][n]), syn.pose_err(ex[n], rc["ext"][n])
        assert e1[0] < 0.5 * e0[0] and e1[1] < 0.5 * e0[1], (n, e0, e1)
    assert np.array_equal(ex[0], rc["ext"][0])
    # with the prior at the true extrinsics the step still converges, and a stiff prior holds every extrinsic at its target
    _, exp, _, _ = crl.calib_rig(rc["surf_map"], rc["corner_map"], rc["surf"], rc["corner"], rc["pivot"], rc["pose_i_init"], rc["ext_init"], 0,
                                 prior7s=rc["ext_init"], prior_pos=1e4, prior_rot=1e4, max_outer=4, max_inner=2)
    for n in range(1, 4):
        assert max(syn.pose_err(exp[n], rc["ext_init"][n])) < 1e-3


def test_prior_factor_matches_the_reference_statement():
    rng = np.random.Generator(np.random.PCG64(5))
    for k in range(20):
        x0 = syn.pose7(rng.normal(0, 1, 3), syn.quat_from_rpy(*rng.normal(0, 0.5, 3)))
        x = crl.perturb_ext(x0, k, deg=float(rng.uniform(0.1, 10)), t=float(rng.uniform(0, 0.3)))
        if k % 3 == 0:
            x[3:] *= 1.0 + 1e-6  # a quaternion off the unit sphere: inverse() divides by the squared norm
        sp, sr = float(rng.uniform(0.1, 10)), float(rng.uniform(0.1, 10))
        r, J = crl.prior_factor(x, x0, sp, sr)
        rn, Jn = crl.prior_factor_np(x, x0, sp, sr)
        assert np.allclose(r, rn, rtol=1e-13, atol=1e-15) and np.allclose(J, Jn, rtol=1e-13, atol=1e-15)
    # the rotation block is LeftQuatMatrix(Q^-1 rot_), not the derivative of the residual: at x != x0 it differs from the numeric one
    x0 = syn.pose7([0, 0, 0], [0, 0, 0, 1])
    x = syn.pose7([0.1, 0, 0], syn.quat_from_rpy(0.3, 0.0, 0.0))
    r, J = crl.prior_factor(x, x0, 1.0, 1.0)
    assert np.allclose(J[3:, 3:], np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1]]) * np.cos(0.15) + np.array([[0, 0, 0], [0, 0, 1], [0, -1, 0]]) * np.sin(0.15))


def test_rig_oracle_leaves_a_calibrated_lidar_without_rows_alone(case2):
    cs = case2
    e4 = np.zeros((0, 4), np.float32)
    ext2 = crl.perturb_ext(cs["ext_cal"], 2)
    ext2[3:] /= np.linalg.norm(ext2[3:])
    pi, ex, st, rows = crl.calib_rig(cs["surf_map"], cs["corner_map"], [cs["surf_ref"], cs["surf_cal"], e4], [cs["corner_ref"], cs["corner_cal"], e4],
                                     cs["pivot"], cs["pose_i_init"], [cs["ext_ref"], cs["ext_cal_init"], ext2], 0, max_outer=3, max_inner=2)
    assert rows[2] == 0 and np.allclose(ex[2], ext2, rtol=0, atol=1e-15)
    # and its prior alone pulls it to the prior's target
    _, exp, _, _ = crl.calib_rig(cs["surf_map"], cs["corner_map"], [cs["surf_ref"], cs["surf_cal"], e4], [cs["corner_ref"], cs["corner_cal"], e4],
                                 cs["pivot"], cs["pose_i_init"], [cs["ext_ref"], cs["ext_cal_init"], ext2], 0,
                                 prior7s=[cs["ext_ref"], cs["ext_cal"], cs["ext_cal"]], prior_pos=1.0, prior_rot=1.0, max_outer=3, max_inner=4)
    assert max(syn.pose_err(exp[2], cs["ext_cal"])) < 0.2 * max(syn.pose_err(ext2, cs["ext_cal"]))


def test_calib_rig_wrappers_compile_against_the_stubs(tmp_path):
    """mloam::calibRig of the adapter (the reference's Pose and PCL clouds, with PriorFactor in the problem assembly) against the stand-in
    PCL / Eigen / Ceres headers, and of the shim with plain g++; both need only exported symbols."""
    stubs, host = os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "m-loam_b200", "host")
    for src, inc in (("calib_rig_adapter_compile_test.cpp", ["-I" + stubs]),
                     ("calib_rig_shim_compile_test.cpp", ["-I" + host, "-I" + os.path.join(ROOT, "include")])):
        obj = str(tmp_path / (src + ".o"))
        out = subprocess.run(["g++", "-std=c++14", "-Wall", "-Werror", *inc, "-c", os.path.join(stubs, src), "-o", obj], capture_output=True, text=True)
        assert out.returncode == 0, out.stderr[-3000:]
        syms = subprocess.run(["nm", "-C", obj], capture_output=True, text=True).stdout
        assert "mloam_calib_rig" in set(re.findall(r"U (mloam_[a-z0-9_]+)", syms)), src


def test_adapter_prior_factor_matches_the_oracle_and_numpy(tmp_path):
    """The adapter's host PriorFactor (what a drop-in estimator.cpp with PRIOR_FACTOR builds its problem from) gives the residual and the
    6 x 7 Jacobian of prior_factor.hpp: the oracle's and the numpy statement's, with a zero 7th column."""
    import ctypes as C
    so = str(tmp_path / "calib_rig_host.so")
    out = subprocess.run(["g++", "-std=c++14", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "tests", "stubs"),
                          os.path.join(ROOT, "tests", "host", "calib_rig_host.cpp"), "-o", so], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-3000:]
    h = C.CDLL(so)
    rng = np.random.Generator(np.random.PCG64(9))
    for k in range(12):
        x0 = syn.pose7(rng.normal(0, 1, 3), syn.quat_from_rpy(*rng.normal(0, 0.5, 3)))
        x = crl.perturb_ext(x0, k, deg=float(rng.uniform(0.1, 10)), t=float(rng.uniform(0, 0.3)))
        sp, sr = float(rng.uniform(0.1, 10)), float(rng.uniform(0.1, 10))
        r, J = np.zeros(6), np.zeros(42)
        h.host_prior_factor(crl._p(x), crl._p(x0), C.c_double(sp), C.c_double(sr), crl._p(r), crl._p(J))
        J = J.reshape(6, 7)
        ro, Jo = crl.prior_factor(x, x0, sp, sr)
        assert np.array_equal(r, ro) and np.array_equal(J[:, :6], Jo) and not J[:, 6].any()
        rn, Jn = crl.prior_factor_np(x, x0, sp, sr)
        assert np.allclose(r, rn, rtol=1e-13, atol=1e-15) and np.allclose(J[:, :6], Jn, rtol=1e-13, atol=1e-15)


def test_calib_rig_symbol_in_header_library_and_binding():
    import importlib.util
    import sys
    hdr = open(os.path.join(ROOT, "include", "mloam_b200.h")).read()
    assert re.search(r"int mloam_calib_rig\(mloam_ctx_t \*ctx, int n_lidars, int idx_ref,", hdr)
    src = open(os.path.join(ROOT, "m-loam_b200", "__init__.py")).read()
    assert '"mloam_calib_rig"' in src and "def calib_rig(" in src
    so = os.path.join(ROOT, "m-loam_b200", "libmloam_b200.so")
    if os.path.exists(so) and shutil.which("nm"):
        syms = subprocess.run(["nm", "-D", "--defined-only", so], capture_output=True, text=True).stdout
        assert re.search(r"\bT mloam_calib_rig\b", syms)


@pytest.mark.skipif(not os.path.exists(NVCC) or shutil.which("c++filt") is None, reason="needs nvcc and c++filt")
def test_calib_rig_kernels_do_not_spill(tmp_path):
    """The LM state machine runs on one warp without a stack frame (every block's step lives in RigState, not in per-thread arrays);
    no kernel of the rig path spills."""
    from test_knn_registers_cpu import _ptxas
    k = _ptxas("calib_rig.cu", tmp_path)
    names = ("k_rig_poses", "k_rig_knn", "k_rig_fit", "k_rig_linearize", "k_rig_lm")
    for n in names:
        regs, frame, st, ld = k[f"mloam::{n}"] if f"mloam::{n}" in k else k[f"void mloam::{n}"]
        assert frame == 0 and st == 0 and ld == 0, (n, regs, frame, st, ld)
        assert regs <= 255
    # the matcher keeps two 256-thread CTAs per SM
    assert 2 * 256 * (k.get("mloam::k_rig_knn") or k["void mloam::k_rig_knn"])[0] <= 65536

"""Test infrastructure of the rig calibration (mloam_calib_rig): the binding of the oracle's restatement (oracle/orc_calib_rig.cpp, built by
oracle/calib_rig.mk), a numpy restatement of PriorFactor (prior_factor.hpp), the synthetic rig case the tests and
tools/bench_calib_rig.py solve, and the cases of tests/golden/calib_frame_12dof.npz."""
from __future__ import annotations

import ctypes as C
import hashlib
import math
import os
import subprocess

import numpy as np

import oracle_lib as orc
import synthetic as syn

_p = orc._p
_lib = None


def lib():
    """oracle/liborc_calib_rig.so (oracle/calib_rig.mk), rebuilt when a source is newer."""
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-C", orc.ORC_DIR, "-f", "calib_rig.mk"], stdout=subprocess.DEVNULL)
        _lib = C.CDLL(os.path.join(orc.ORC_DIR, "liborc_calib_rig.so"))
    return _lib


def _cat(clouds):
    cl = [np.zeros((0, 4), np.float32) if x is None or len(x) == 0 else orc.cloud(x) for x in clouds]
    n = np.array([x.shape[0] for x in cl], np.int32)
    return np.ascontiguousarray(np.concatenate(cl + [np.zeros((1, 4), np.float32)]), np.float32), n


def calib_rig(surf_map, corner_map, surf, corner, pivot, pose_i, ext7s, idx_ref=0, prior7s=None, prior_pos=0.0, prior_rot=0.0, max_outer=2,
              max_inner=4, huber_a=1.0, surf_map_cal=None, corner_map_cal=None, opts=None):
    """orc_calib_rig.  Returns (pose_i, ext7s [L, 7], stats, rows [L])."""
    e4 = np.zeros((0, 4), np.float32)
    maps = [orc.cloud(x) if x is not None and len(x) else e4 for x in (surf_map, corner_map, surf_map_cal, corner_map_cal)]
    L = len(surf)
    hs, ns = _cat(surf)
    hc, nc = _cat(corner)
    opts = orc.default_opts() if opts is None else np.ascontiguousarray(opts, np.float64)
    pv = np.ascontiguousarray(pivot, np.float64)
    pi = np.array(pose_i, np.float64)
    ex = np.array(ext7s, np.float64).reshape(L, 7)
    pr = None if prior7s is None else np.ascontiguousarray(prior7s, np.float64).reshape(L, 7)
    st = np.zeros(4)
    rows = np.zeros(L, np.int32)
    args = []
    for a in maps:
        args += [_p(a), a.shape[0]]
    lib().orc_calib_rig(*args, L, idx_ref, _p(hs), _p(ns), _p(hc), _p(nc), _p(pv), _p(pi), _p(ex), _p(pr), C.c_double(prior_pos),
                        C.c_double(prior_rot), max_outer, max_inner, C.c_double(huber_a), _p(opts), _p(st), _p(rows))
    return pi, ex, {"lm_iterations": int(st[0]), "final_cost": st[1], "rows": int(st[2]), "termination": int(st[3])}, rows


def prior_factor(x7, x07, pos_scale, rot_scale):
    """orc_prior_factor: (r[6], J[6, 6])."""
    r, J = np.zeros(6), np.zeros(36)
    lib().orc_prior_factor(_p(np.ascontiguousarray(x7, np.float64)), _p(np.ascontiguousarray(x07, np.float64)), C.c_double(pos_scale),
                           C.c_double(rot_scale), _p(r), _p(J))
    return r, J.reshape(6, 6)


def _qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz])


def _qinv(q):
    return np.array([-q[0], -q[1], -q[2], q[3]]) / float(np.dot(q, q))


def prior_factor_np(x7, x07, pos_scale, rot_scale):
    """PriorFactor::Evaluate in numpy (prior_factor.hpp:36-71): residual [P - pos_ ; 2 (rot_^-1 Q).vec] scaled by diag(pos I3, rot I3);
    local jacobian diag(I3, LeftQuatMatrix(Q^-1 rot_).topLeftCorner<3,3>()) scaled likewise, as the reference writes it."""
    x, x0 = np.asarray(x7, np.float64), np.asarray(x07, np.float64)
    e = _qmul(_qinv(x0[3:]), x[3:])
    r = np.concatenate([pos_scale * (x[:3] - x0[:3]), rot_scale * (2 * e[:3])])
    m = _qmul(_qinv(x[3:]), x0[3:])
    v, w = m[:3], m[3]
    skew = np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])
    J = np.zeros((6, 6))
    J[:3, :3] = pos_scale * np.eye(3)
    J[3:, 3:] = rot_scale * (w * np.eye(3) + skew)
    return r, J


def perturb_ext(e, k, deg=2.0, t=0.05):
    """An extrinsic off by `deg` degrees and `t` metres, the direction varying with k."""
    s = 1 if k % 2 else -1
    d = math.radians(deg) / math.sqrt(3.0)
    return syn.pose_mul(e, syn.pose7([s * t / math.sqrt(3.0), -t / math.sqrt(3.0), t / math.sqrt(3.0)], syn.quat_from_rpy(d, -s * d, d)))


def make_rig_case(scene, n_lidars, n_rings, horizon, map_points, idx_ref=0, seed=31, submap=None):
    """One rig calibration step: the local map in the pivot frame, frame i's features of LiDAR idx_ref, the other LiDARs' features at the
    pivot (sensor frame, leaf 0.4 / 0.2), truth and initial values (every calibrated extrinsic off by 2 deg / 5 cm)."""
    traj = syn.trajectory(10)
    pivot, pose_i = traj[3], traj[7]
    ext = syn.rig_extrinsics(n_lidars)
    surf_w, corner_w = submap if submap is not None else syn.make_submap(scene, map_points)
    Pinv = syn.pose_inv(pivot)
    surf_map, corner_map = syn.transform_cloud(surf_w, Pinv), syn.transform_cloud(corner_w, Pinv)
    surf, corner = [], []
    for n in range(n_lidars):
        cloud, ss, se = syn.make_sweep(scene, pose_i if n == idx_ref else pivot, n_rings, horizon, seed=seed + n, lidar_id=n, ext=ext[n])
        f = orc.extract_cloud(cloud, ss, se)
        surf.append(orc.voxel_grid(f["surf_points_less_flat"], 0.4, False)[0])
        corner.append(orc.voxel_grid(f["corner_points_less_sharp"], 0.2, False)[0])
    rng = np.random.Generator(np.random.PCG64(seed))
    ext_init = np.array([ext[n] if n == idx_ref else perturb_ext(ext[n], n) for n in range(n_lidars)])
    return dict(surf_map=surf_map, corner_map=corner_map, surf=surf, corner=corner, pivot=pivot, pose_i=pose_i, ext=ext,
                pose_i_init=syn.perturb_pose(pose_i, rng), ext_init=ext_init, idx_ref=idx_ref)


# tests/golden/calib_frame_12dof.npz holds mloam_calib_frame's outputs as its 12-DoF solver computed them, on these cases
# (name: inputs, max_outer, max_inner, feature groups given, the calibrated LiDAR matched against its own maps)
CALIB_GOLDEN = {"case2_10x1": ("case2", 10, 1, "both", False), "case2_2x4": ("case2", 2, 4, "both", False),
                "own_cal_maps": ("case2", 10, 1, "both", True), "ref_only": ("case2", 10, 1, "ref", False),
                "cal_only": ("case2", 10, 1, "cal", False), "c3": ("c3", 10, 1, "both", False)}
CALIB_GOLDEN_STATS = ("termination", "lm_iterations", "n_surf", "final_cost", "n_surf_in", "n_corner_in")
_GOLDEN_INPUTS = {}


def calib_golden_inputs(kind):
    """The seeded inputs of a golden case ("case2": 16 x 1024 sweeps and a 100k-point map; "c3": bench.py C3's 64 x 2048 sweeps and a 2M-point
    map), with the calibration maps of own_cal_maps (leaf 0.2) for case2 and a sha256 over every array."""
    if kind not in _GOLDEN_INPUTS:
        rings, horizon, pts = (16, 1024, 100_000) if kind == "case2" else (64, 2048, 2_000_000)
        cs = syn.make_calib_case(syn.make_scene(), orc.extract_cloud, orc.voxel_grid, rings, horizon, pts)
        if kind == "case2":
            cs["surf_map_cal"] = orc.voxel_grid(cs["surf_map"], 0.2, False)[0]
            cs["corner_map_cal"] = orc.voxel_grid(cs["corner_map"], 0.2, False)[0]
        h = hashlib.sha256()
        for k in sorted(cs):
            a = np.ascontiguousarray(cs[k])
            h.update(f"{k} {a.dtype} {a.shape}".encode())
            h.update(a.tobytes())
        cs["sha256"] = h.hexdigest()
        _GOLDEN_INPUTS[kind] = cs
    return _GOLDEN_INPUTS[kind]


def calib_golden_maps(ctx, cs, own):
    ctx.map_build(0, cs["corner_map"], 0.25)
    ctx.map_build(1, cs["surf_map"], 0.25)
    if own:
        ctx.map_build(2, cs["corner_map_cal"], 0.25)
        ctx.map_build(3, cs["surf_map_cal"], 0.25)


def calib_golden_groups(cs, groups):
    """(surf_ref, corner_ref, surf_cal, corner_cal), None for a group not given."""
    ref = (cs["surf_ref"], cs["corner_ref"]) if groups != "cal" else (None, None)
    cal = (cs["surf_cal"], cs["corner_cal"]) if groups != "ref" else (None, None)
    return ref + cal

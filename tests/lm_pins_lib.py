"""The cases of tests/golden/lm_solve_pins.npz: the device Levenberg-Marquardt solves (mloam_odom_solve, mloam_calib_rig) and the good-feature
selection's log-det greedy, each on seeded inputs, with the outputs to record.  tests/golden/make_lm_golden.py writes the pins and
tests/test_lm_pins.py checks that every pinned value comes out bit for bit."""
import hashlib

import numpy as np

import calib_rig_lib as crl
import oracle_lib as orc
import synthetic as syn

STATS = ("lm_iterations", "termination", "final_cost")

# name: free_mask, max_iterations, start ("near": 2 cm / 0.2 deg off, "far": 0.5 m / 15 deg off), features ("chain": planes and lines
# through a 3-pose chain, "plane": one plane only)
ODOM = {"fm1_converge": (1, 30, "near", "chain"), "fm2_converge": (2, 30, "near", "chain"), "fm3_converge": (3, 30, "near", "chain"),
        "fm1_cap": (1, 2, "near", "chain"), "fm2_cap": (2, 2, "near", "chain"), "fm3_cap": (3, 2, "near", "chain"),
        "fm1_far": (1, 30, "far", "chain"), "fm3_far": (3, 30, "far", "chain"),
        "fm1_plane": (1, 30, "near", "plane"), "fm3_plane": (3, 30, "near", "plane")}

# name: idx_ref, prior (0 off, 1 at the true extrinsics), max_outer, max_inner; three LiDARs
RIG = {"rig3_10x1": (0, 0, 10, 1), "rig3_2x4": (0, 0, 2, 4), "rig3_prior_10x1": (0, 1, 10, 1), "rig3_prior_2x4": (2, 1, 2, 4)}

# name: kind, ratio, seed (stochastic greedy on the log-det of the selection's information matrix)
GD = {"gd_surf": ("s", 0.2, 3), "gd_corner": ("c", 0.3, 12345)}


def _rand_pose(rng):
    return syn.pose7(rng.normal(size=3) * 3, rng.normal(size=4))


def odom_inputs(name):
    """(types, points, coeffs, pivot, pose_i, ext) of an ODOM case: features consistent with the chain pivot^-1 pose_i ext, with 1 cm noise,
    float-valued like the reference's PointPlaneFeature."""
    free_mask, _, start, feats = ODOM[name]
    rng = np.random.default_rng(1000 + list(ODOM).index(name))
    xp, xi, xe = (_rand_pose(rng) for _ in range(3))
    comp = syn.pose_mul(syn.pose_mul(syn.pose_inv(xp), xi), xe)
    R = syn.quat_to_mat(comp[3:])
    n = 1500
    pts = rng.normal(size=(n, 3)) * 6
    types = np.array([ord("c") if feats == "chain" and k % 3 == 0 else ord("s") for k in range(n)], np.uint8)
    coeffs = np.zeros((n, 6))
    plane = rng.normal(size=3)
    plane /= np.linalg.norm(plane)
    for k in range(n):
        lp = R @ pts[k] + comp[:3]
        if types[k] == ord("s"):
            nrm = plane if feats == "plane" else rng.normal(size=3)
            nrm = nrm / np.linalg.norm(nrm)
            coeffs[k, :4] = [*nrm, -nrm @ lp + rng.normal() * 0.01]
        else:
            d = rng.normal(size=3)
            d /= np.linalg.norm(d)
            off = np.cross(d, rng.normal(size=3)) * 0.01
            coeffs[k] = [*(lp + off + 0.1 * d), *(lp + off - 0.1 * d)]
    st, sr = (0.02, 0.004) if start == "near" else (0.5, 0.15)
    d = lambda: syn.pose7(rng.normal(size=3) * st, syn.quat_from_rpy(*(rng.normal(size=3) * sr)))
    xi0 = syn.pose_mul(xi, d()) if free_mask & 1 else xi
    xe0 = syn.pose_mul(xe, d()) if free_mask & 2 else xe
    return types, pts.astype(np.float32).astype(np.float64), coeffs.astype(np.float32).astype(np.float64), xp, xi0, xe0


_RIG = {}


def rig_inputs(idx_ref):
    if idx_ref not in _RIG:
        _RIG[idx_ref] = crl.make_rig_case(syn.make_scene(), 3, 16, 1024, 100_000, idx_ref=idx_ref)
    return _RIG[idx_ref]


_GD = {}


def gd_inputs():
    """bench C1's maps and downsampled scans (16-ring x 1024 sweep, 50k-point submap) and a perturbed pose."""
    if not _GD:
        scene = syn.make_scene()
        traj = syn.trajectory(6)
        surf_map, corner_map = syn.make_submap(scene, 50000)
        cloud, ss, se = syn.make_sweep(scene, traj[4], 16, 1024, seed=4)
        f = orc.extract_cloud(cloud, ss, se)
        _GD.update(surf_map=surf_map, corner_map=corner_map, init=syn.perturb_pose(traj[4], np.random.Generator(np.random.PCG64(11))),
                   c=orc.voxel_grid(f["corner_points_less_sharp"], 0.2, True)[0], s=orc.voxel_grid(f["surf_points_less_flat"], 0.4, True)[0])
    return _GD


def sha256(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        a = np.ascontiguousarray(a)
        h.update(f"{a.dtype} {a.shape}".encode())
        h.update(a.tobytes())
    return h.hexdigest()


def run_all(ctx):
    """Every case on the context: {key: array}, the keys of the pins file."""
    out = {}
    for name, (free_mask, max_it, _, _) in ODOM.items():
        inp = odom_inputs(name)
        xi, xe, st = ctx.odom_solve(*inp, free_mask, max_iterations=max_it)
        out[f"{name}.inputs_sha256"] = np.array(sha256(*inp))
        out[f"{name}.pose_i"], out[f"{name}.ext"] = xi, xe
        for k in STATS:
            out[f"{name}.{k}"] = np.array(st[k])
        out[f"{name}.H"] = np.asarray(st["H"], np.float64)
    for name, (idx_ref, prior, outer, inner) in RIG.items():
        rc = rig_inputs(idx_ref)
        ctx.map_build(0, rc["corner_map"], 0.25)
        ctx.map_build(1, rc["surf_map"], 0.25)
        kw = dict(prior7s=rc["ext"], prior_pos=2.0, prior_rot=5.0) if prior else {}
        pi, ex, st, rows = ctx.calib_rig(rc["surf"], rc["corner"], rc["pivot"], rc["pose_i_init"], rc["ext_init"], idx_ref, max_outer=outer,
                                         max_inner=inner, **kw)
        out[f"{name}.inputs_sha256"] = np.array(sha256(rc["surf_map"], rc["corner_map"], *rc["surf"], *rc["corner"], rc["pivot"],
                                                       rc["pose_i_init"], rc["ext_init"], rc["ext"]))
        out[f"{name}.pose_i"], out[f"{name}.ext"], out[f"{name}.rows"] = pi, ex, rows
        for k in STATS:
            out[f"{name}.{k}"] = np.array(st[k])
        out[f"{name}.H"] = np.asarray(st["H"], np.float64)
    g = gd_inputs()
    ctx.map_build(1, g["surf_map"], 0.5)
    ctx.map_build(0, g["corner_map"], 0.5)
    for name, (kind, ratio, seed) in GD.items():
        r = ctx.good_features(1 if kind == "s" else 0, kind, g[kind], g["init"], orc.GF_GD, ratio, seed)
        out[f"{name}.inputs_sha256"] = np.array(sha256(g[kind], g["surf_map"] if kind == "s" else g["corner_map"], g["init"]))
        out[f"{name}.sel"] = r["sel"]
    return out

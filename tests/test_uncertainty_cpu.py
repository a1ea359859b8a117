"""The oracle's uncertainty-aware frame (with_ua = true): downsampleCurrentScan's per-point uncertainty and trace gate, and
cov_mapping = H^-1 at the returned pose (lidar_mapper_keyframe.cpp:356-421, :600-610), checked against independent restatements."""
import numpy as np
from scipy.spatial.transform import Rotation

import oracle_lib as orc
import uncertainty_lib as ua
import synthetic as syn

COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])


def _multi_case(n_lidars=2, rings=16, horizon=1024, map_pts=60_000, seed=21):
    scene = syn.make_scene()
    traj = syn.trajectory(8)
    surf_map, corner_map = syn.make_submap(scene, map_pts)
    cloud, ss, se, ext = syn.make_multi_sweep(scene, traj[6], n_lidars, rings, horizon, seed=seed)
    init = syn.perturb_pose(traj[6], np.random.Generator(np.random.PCG64(23)))
    return dict(surf_map=surf_map, corner_map=corner_map, cloud=cloud, ss=ss, se=se, ext=ext, init=init, truth=traj[6])


def _expected_cov(pts, ext, ext_cov):
    """orc.point_uncertainty of every point, associated with pose_ext[id]^-1 and evaluated under pose_ext[id], id = int(intensity)."""
    cov = np.zeros((pts.shape[0], 6), np.float32)
    ids = pts[:, 3].astype(np.int32)
    for l in np.unique(ids):
        m = ids == l
        sel = orc.associate(pts[m], ua.pose_inv(ext[l]))
        cov[m] = orc.point_uncertainty(sel, ext[l], ext_cov[l], COV_MEAS)
    return cov


def _trace(c6):
    return c6[:, 0].astype(np.float64) + c6[:, 3].astype(np.float64) + c6[:, 5].astype(np.float64)


def test_frame_uncertainty_and_gate_match_point_uncertainty():
    c = _multi_case()
    ext_cov = ua.ext_covariances(2, seed=5)
    corner_ds, surf_ds = orc.prepare_multi(c["cloud"], c["ss"], c["se"], 2, c["ext"])
    exp_s, exp_c = _expected_cov(surf_ds, c["ext"], ext_cov), _expected_cov(corner_ds, c["ext"], ext_cov)
    tr = np.sort(np.concatenate([_trace(exp_s), _trace(exp_c)]))
    k = int(0.7 * tr.shape[0])
    thr = 0.5 * (tr[k - 1] + tr[k])  # the 70th percentile, between two traces
    o = orc.default_opts()
    o[orc.O_MAX_OUTER], o[orc.O_MAX_INNER] = 3, 1
    pose, st, cov, scans = ua.frame_multi_ua(c["cloud"], c["ss"], c["se"], 2, c["ext"], ext_cov, COV_MEAS, thr, c["surf_map"], c["corner_map"],
                                              c["init"], o)
    for pts, c6, exp, key in ((surf_ds, exp_s, exp_s, "surf"), (corner_ds, exp_c, exp_c, "corner")):
        keep = _trace(exp) <= thr
        assert 0.1 < 1.0 - keep.mean() < 0.5
        assert np.array_equal(scans[key], pts[keep])
        assert np.array_equal(scans[key + "_cov6"], exp[keep])
    assert st["n_surf_in"] == scans["surf"].shape[0] and st["n_corner_in"] == scans["corner"].shape[0]
    assert st["ran"] == 1
    # an infinite threshold keeps every point; zero covariances with a huge threshold reproduce the with_ua = false frame
    pose0, st0 = orc.frame_multi(c["cloud"], c["ss"], c["se"], 2, c["ext"], c["surf_map"], c["corner_map"], c["init"], o)
    pz, stz, covz, sz = ua.frame_multi_ua(c["cloud"], c["ss"], c["se"], 2, c["ext"], np.zeros((2, 6, 6)), COV_MEAS, 1e30, c["surf_map"],
                                           c["corner_map"], c["init"], o)
    assert np.array_equal(pz, pose0) and stz["final_cost"] == st0["final_cost"] and stz["n_surf_in"] == st0["n_surf_in"]
    assert np.allclose(covz @ sz["H"], np.eye(6), atol=1e-9)


def _h_numpy(surf_scan, surf_cov6, corner_scan, corner_cov6, surf_map, corner_map, x_assoc, x, huber_a=0.1):
    """Loss-corrected J^T J of the plane and edge residuals (lidar_map_factor.hpp) of the association at x_assoc, evaluated at x:
    rho'(s) J^T J with Huber rho' = 1 | a / sqrt(s), J w.r.t. [t | rotation vector] applied on the right."""
    vs, cfs, _ = orc.match_from_map("s", surf_map, surf_scan, x_assoc)
    vc, cfc, _ = orc.match_from_map("c", corner_map, corner_scan, x_assoc)
    sis = np.minimum(np.sqrt(1.0 / _trace(surf_cov6[vs])) / 3.0, 1.0)
    sic = np.minimum(np.sqrt(1.0 / _trace(corner_cov6[vc])) / 3.0, 1.0)
    R = Rotation.from_quat(x[3:7]).as_matrix()
    t = x[:3]
    ps, ws, ds = surf_scan[vs][:, :3].astype(np.float64), cfs[vs][:, :3], cfs[vs][:, 3]
    pc, la, lb = corner_scan[vc][:, :3].astype(np.float64), cfc[vc][:, :3], cfc[vc][:, 3:6]

    def skew(v):
        z = np.zeros(v.shape[0])
        return np.stack([np.stack([z, -v[:, 2], v[:, 1]], 1), np.stack([v[:, 2], z, -v[:, 0]], 1), np.stack([-v[:, 1], v[:, 0], z], 1)], 1)

    # plane: r = s (w . (R p + t) + d)
    r_s = sis * (np.einsum("ij,ij->i", ws, ps @ R.T + t) + ds)
    dldth_s = -np.einsum("ij,njk->nik", R, skew(ps))                      # d(R exp(th) p)/dth = -R [p]x
    J_s = sis[:, None] * np.concatenate([ws, np.einsum("ni,nik->nk", ws, dldth_s)], 1)
    # edge: r = s |(l - a) x (l - b)| / |a - b|, l = R p + t
    lp = pc @ R.T + t
    u = np.cross(lp - la, lp - lb)
    nu, nab = np.linalg.norm(u, axis=1), np.linalg.norm(la - lb, axis=1)
    r_c = sic * nu / nab
    drdl = sic[:, None] * np.einsum("ni,nik->nk", u / nu[:, None], skew(lb - la)) / nab[:, None]  # du = [b - a]x dl
    dldth_c = -np.einsum("ij,njk->nik", R, skew(pc))
    J_c = np.concatenate([drdl, np.einsum("ni,nik->nk", drdl, dldth_c)], 1)
    r = np.concatenate([r_s, r_c])
    J = np.concatenate([J_s, J_c])
    s = r * r
    w = np.where(s <= huber_a * huber_a, 1.0, huber_a / np.sqrt(np.maximum(s, 1e-300)))
    return (J * w[:, None]).T @ J


def test_pose_covariance_is_inverse_of_independent_hessian():
    """C1 size (16 x 1024 sweep, 50k-point submap), one association (max_outer 1) so that the last association is the one at
    the initial pose: the oracle's H at the returned pose equals an H assembled here in numpy, and cov_mapping inverts it."""
    scene = syn.make_scene()
    traj = syn.trajectory(6)
    surf_map, corner_map = syn.make_submap(scene, 50000)
    cloud, ss, se = syn.make_sweep(scene, traj[4], 16, 1024, seed=4)
    f = orc.extract_cloud(cloud, ss, se)
    cs, _ = orc.voxel_grid(f["corner_points_less_sharp"], 0.2, True)
    sf, _ = orc.voxel_grid(f["surf_points_less_flat"], 0.4, True)
    init = syn.perturb_pose(traj[4], np.random.Generator(np.random.PCG64(11)))
    ext_cov = ua.ext_covariances(1, seed=3)[0]
    ident = np.array([0, 0, 0, 0, 0, 0, 1.0])
    sc6 = orc.point_uncertainty(sf, ident, ext_cov, COV_MEAS)
    cc6 = orc.point_uncertainty(cs, ident, ext_cov, COV_MEAS)
    assert (np.minimum(np.sqrt(1.0 / _trace(sc6)) / 3.0, 1.0) < 1.0).mean() >= 0.2
    o = orc.default_opts()
    o[orc.O_MAX_OUTER], o[orc.O_MAX_INNER] = 1, 30
    pose, st, cov, H = ua.scan2map_ua_cov(surf_map, corner_map, sf, sc6, cs, cc6, init, o)
    assert st["ran"] == 1 and st["n_surf"] > 500
    Hn = _h_numpy(sf, sc6, cs, cc6, surf_map, corner_map, init, pose)
    assert np.linalg.norm(H - Hn) <= 1e-9 * np.linalg.norm(Hn), np.linalg.norm(H - Hn) / np.linalg.norm(Hn)
    assert np.allclose(cov @ H, np.eye(6), atol=1e-9)
    assert np.linalg.norm(cov - cov.T) <= 1e-9 * np.linalg.norm(cov)
    assert np.all(np.linalg.eigvalsh(0.5 * (cov + cov.T)) > 0)
    # the pose and statistics are those of orc_scan2map_ua, which reports no covariance
    p2, st2 = orc.scan2map_ua(surf_map, corner_map, sf, sc6, cs, cc6, init, o)
    assert np.array_equal(p2, pose) and st2["final_cost"] == st["final_cost"]


def test_pose_covariance_zero_when_map_gated():
    c = _multi_case(n_lidars=1, map_pts=60_000)
    tiny = c["surf_map"][:40]
    _, st, cov, _ = ua.frame_multi_ua(c["cloud"], c["ss"], c["se"], 1, c["ext"], ua.ext_covariances(1), COV_MEAS, 1e30, tiny, c["corner_map"],
                                       c["init"])
    assert st["ran"] == 0 and not cov.any()


def test_ext_covariances_are_seeded_spd():
    a, b = ua.ext_covariances(3, seed=7), ua.ext_covariances(3, seed=7)
    assert a.shape == (3, 6, 6) and np.array_equal(a, b)
    assert np.allclose(a, np.transpose(a, (0, 2, 1)))
    assert np.all(np.linalg.eigvalsh(a) > 0)
    assert np.allclose(ua.ext_covariances(1, seed=7, scale=2.0), 4.0 * ua.ext_covariances(1, seed=7))

"""Test infrastructure of the global map (mloam_global_map): the binding of the oracle's pubGlobalMap / saveGlobalMap restatement
(oracle/orc_mapper.cpp in oracle_lib's library) over a mapper_lib.Mapper, and an independent composition of the same steps from the
oracle's single-step entry points (radius search, position filter, cloudUCTAssociateToMap, VoxelGridCovarianceMLOAM) in numpy."""
from __future__ import annotations

import numpy as np

import mapper_lib as ml
import oracle_lib as orc

SURROUND, SAVE = 0, 1
_p = orc._p


def global_map(mapper: ml.Mapper, mode: int, center7, radius: float, kf_leaf: float, leaf: float):
    """The oracle's global map of a Mapper's keyframes, with their outlier clouds appended in the reference's orders: (chosen ids,
    [map 0 points, map 0 cov6, map 1 points, map 1 cov6]).  center7: the pose whose float position is the centre (SURROUND; the position
    the last save tested when the device call passes NULL)."""
    ct = None if center7 is None else np.ascontiguousarray(center7, np.float64)
    cnt = np.zeros(3, np.int32)
    r = orc.lib().orc_global_map(mapper._h.value, int(mode), _p(ct), float(radius), float(kf_leaf), float(leaf), _p(cnt))
    try:
        ch = np.zeros(max(cnt[0], 1), np.int32)
        out = []
        for which in (0, 1):
            n = int(cnt[1 + which])
            p, c6 = np.zeros((max(n, 1), 4), np.float32), np.zeros((max(n, 1), 6), np.float32)
            orc.lib().orc_global_map_read(r, which, _p(ch), _p(p), _p(c6))
            out += [p[:n], c6[:n]]
        return ch[:cnt[0]].tolist(), out
    finally:
        orc.lib().orc_global_map_free(r)


# ---------------------------------------------------------------------------------------- independent composition
def np_candidates(pos_f32, mode, center_f32=None, radius=None):
    """The keyframes offered to the position filter: radius search order (SURROUND) or id order (SAVE)."""
    if mode == SURROUND:
        return ml.np_radius_search(pos_f32, center_f32, radius)[0]
    return list(range(len(pos_f32)))


def np_chosen(pos_f32, cand, kf_leaf):
    """The position filter over the candidates' positions with intensity = id: the last-listed id of each voxel, in voxel order."""
    if not cand:
        return []
    p = np.asarray(pos_f32, np.float32)[cand]
    return [cand[i] for i in ml.np_position_filter(p, kf_leaf)]


def compose(keyframes, ext7, ext_cov, cov_meas, with_ua, trace_thr, mode, chosen, leaf):
    """keyframes[id] = (pose7, cov 6x6, surf [n,4], corner [m,4]).  Each chosen keyframe's clouds through cloudUCTAssociateToMap with the
    compound of its pose and each extrinsic, concatenated in the mode's order, then VoxelGridCovarianceMLOAM<PointIWithCov>(leaf)."""
    ext7 = np.asarray(ext7, np.float64).reshape(-1, 7)
    L = ext7.shape[0]
    raw = [[], []]
    for i in chosen:
        pose, cov, surf, corner = keyframes[i]
        pc, cc = [], []
        for l in range(L):
            ec = ext_cov[l] if with_ua else np.zeros((6, 6))
            a, b = orc.compound_pose_cov(pose, cov, ext7[l], ec)
            pc.append(a), cc.append(b)
        for t, cl in ((0, surf), (1, corner)):
            if cl.shape[0] == 0:
                continue
            got = orc.cloud_uct_associate(cl, pose, ext7, np.stack(pc), np.stack(cc), cov_meas, with_ua, trace_thr)
            raw[0 if mode == SURROUND else t].append(got)
    out = []
    for parts in raw[:1 if mode == SURROUND else 2]:
        if not parts:
            out += [np.zeros((0, 4), np.float32), np.zeros((0, 6), np.float32)]
            continue
        p, c6, tr, _ = orc.voxel_grid_cov(np.concatenate([x[0] for x in parts]), np.concatenate([x[1] for x in parts]),
                                          np.concatenate([x[2] for x in parts]), leaf, trace_thr)
        out += [p, c6]
    return out

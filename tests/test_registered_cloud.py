"""GPU tests (-m gpu) of the registered clouds (mloam_set_registered / mloam_frame_registered, pubPointCloud): each frame's full-resolution,
surf_last and corner_last clouds through the C ABI against the oracle (oracle/orc_registered.cpp) evaluated at the pose the frame returned, bit
for bit — mloam_frame and mloam_frame_raw, one LiDAR with and without mloam_set_extrinsic and a 3-LiDAR rig, with_ua, DISTORTION and the outlier
cloud, graph replay, the stream path, stage profiling, the look-ahead announcing the other sweep, mloam_frame_device with the caller's sweep
overwritten, a map-gated frame, the closed mapper loop with the keyframe store and a 4 x 64 x 2048 frame —; the frame's other results unchanged
by it and one launch more per frame; its error paths."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import mapper_lib as ml
import registered_lib as rl
import synthetic as syn
import uncertainty_lib as ua

pytestmark = pytest.mark.gpu

E_INVALID, E_STATE = -1, -4
COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])
LEAF = 0.8
RINGS, HORIZON = 16, 512
SINGLE_EXT = syn.pose7([0.4, -0.1, 1.1], syn.quat_from_rpy(0.01, 0.03, 0.25))
UNDIST = [np.stack([syn.pose7([0.09 + 0.01 * l, 0.01 * k, 0.003], syn.quat_from_rpy(0.001 * k, -0.002, 0.02 + 0.003 * l)) for l in range(3)])
          for k in (1, 2)]


def _exts(n):
    out = []
    for l in range(n):
        a = 2 * math.pi * l / n
        out.append([0.3 * math.cos(a), 0.3 * math.sin(a), 0.05 * l, 0.0, 0.0, math.sin(a / 4), math.cos(a / 4)])
    return np.array(out, np.float64)


@pytest.fixture(scope="module")
def scene():
    sc = syn.make_scene()
    surf_map, corner_map = syn.make_submap(sc, 60000)
    return dict(scene=sc, traj=syn.trajectory(6), surf_map=surf_map, corner_map=corner_map)


def _ctx(mloam, n_lidars, env=None):
    env = env or {}
    for k, v in env.items():
        os.environ[k] = v
    try:
        p = mloam.default_params()
        p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = RINGS * n_lidars, 4, 1, 0.5, 1024
        return mloam.Context(0, p)
    finally:
        for k in env:
            os.environ.pop(k)


def _frames(sc, n_lidars, raw, nan_lidar=None):
    """Two sweeps (A, B).  ring-ordered: (cloud, scan_start, scan_end); raw: (raw, counts); nan_lidar: that LiDAR's raw sweep is all non-finite."""
    import front_end_lib as fel
    ext = _exts(n_lidars)
    out = []
    for k in (1, 2):
        pose = sc["traj"][k]
        if raw:
            parts = [fel.raw_sweep(sc["scene"], pose, RINGS, HORIZON, 40 + 31 * k + l, ext=ext[l]) for l in range(n_lidars)]
            if nan_lidar is not None:
                parts[nan_lidar][:, 0] = np.nan
            out.append((np.ascontiguousarray(np.concatenate(parts)), np.array([p.shape[0] for p in parts], np.int32)))
        else:
            cloud, ss, se, _ = syn.make_multi_sweep(sc["scene"], pose, n_lidars, RINGS, HORIZON, seed=40 + k, ext=ext)
            out.append((cloud, ss, se))
    return out


def _ring_ordered(mloam, frames, n_lidars, merge):
    """The oracle's inputs of raw frames: the ring-ordered sweep and its ScanInfo (mloam_front_end, on a context of its own)."""
    cx = _ctx(mloam, n_lidars)
    try:
        if merge:
            cx.set_lidars(n_lidars, _exts(n_lidars))
        cx.set_front_end(RINGS, HORIZON)
        out = []
        for raw, counts in frames:
            cloud, ss, se = cx.front_end(raw, counts)
            out.append((cloud, ss[:n_lidars * RINGS], se[:n_lidars * RINGS]))
        return out
    finally:
        cx.close()


class Cfg:
    def __init__(self, setup="rig", raw=False, with_ua=False, dist=False, outlier=False):
        self.setup, self.raw, self.with_ua, self.dist, self.outlier = setup, raw, with_ua, dist, outlier
        self.L = 3 if setup == "rig" else 1

    def configure(self, cx, reg):
        L = self.L
        if self.setup == "rig":
            cx.set_lidars(L, _exts(L))
        elif self.setup == "single_ext":
            cx.set_extrinsic(SINGLE_EXT)
        cx.set_uncertainty(self.with_ua, ua.ext_covariances(L, seed=3) if self.with_ua else None, COV_MEAS, 1e3)
        if self.outlier:
            cx.set_outlier(LEAF)
        if self.dist:
            cx.set_distortion(True, 0.1)
        if reg:
            cx.set_registered(True)
        if self.raw:
            cx.set_front_end(RINGS, HORIZON)

    def want(self, inp, pose, k):
        cloud, ss, se = inp
        return rl.registered(cloud, ss, se, pose, ext7=_exts(self.L) if self.setup == "rig" else None,
                             single_ext7=SINGLE_EXT if self.setup == "single_ext" else None,
                             poses7=UNDIST[k % 2][:self.L] if self.dist else None, outlier=self.outlier)


def _run(mloam, sc, frames, cfg, reg=True, lookahead=False, graphs=True, prof=False, n_rounds=2):
    """Frames A, B, A, B (the same arrays, so that graphs capture and replay): per frame (pose, stats, frame_scan, outlier, registered clouds,
    the device read of the full-resolution cloud) and the launches of each frame."""
    cx = _ctx(mloam, cfg.L, None if graphs else {"MLOAM_DISABLE_GRAPHS": "1"})
    out, launches = [], []
    try:
        cfg.configure(cx, reg)
        if prof:
            cx.profile(True)
        seq = [frames[k % 2] for k in range(2 * n_rounds)]
        for k, fr in enumerate(seq):
            if lookahead and k + 1 < len(seq):
                (cx.frame_set_next_raw if cfg.raw else cx.frame_set_next)(*seq[k + 1])
            if cfg.dist:
                cx.frame_undistort(UNDIST[k % 2][:cfg.L])
            l0 = cx.launch_count()
            init = sc["traj"][1 + k % 2]
            if cfg.raw:
                pose, st = cx.frame_raw(fr[0], fr[1], sc["surf_map"], sc["corner_map"], init)
            else:
                pose, st = cx.frame(fr[0], fr[1], fr[2], sc["surf_map"], sc["corner_map"], init)
            launches.append(cx.launch_count() - l0)
            regs = [cx.frame_registered(w) for w in range(3)] if reg else None
            dev = cx.frame_registered_device(mloam.REGISTERED_FULL_RES).cpu().numpy() if reg and k == 0 else None
            out.append((pose, dict(st), cx.frame_scan(), cx.frame_outlier() if cfg.outlier else None, regs, dev))
        if prof:
            cx.profile(False)
            out.append(cx.profile_get("registered"))
    finally:
        cx.close()
    return out, launches


def _same(a, b):
    return rl.bits_equal(a, b)


def _inputs(mloam, frames, cfg):
    return _ring_ordered(mloam, frames, cfg.L, cfg.setup == "rig") if cfg.raw else frames


def _check_against_oracle(got, inputs, cfg, tag):
    for k, g in enumerate(got):
        want = cfg.want(inputs[k % 2], g[0], k)
        for t in range(3):
            assert _same(g[4][t], want[t]), (tag, k, t, g[4][t].shape, want[t].shape)
        if g[5] is not None:
            assert _same(g[5], g[4][0]), (tag, k)


def _check_unchanged(got, off, tag):
    for k, (g, o) in enumerate(zip(got, off)):
        assert np.array_equal(g[0], o[0]) and g[1] == o[1], (tag, k)
        assert all(_same(a, b) for a, b in zip(g[2], o[2])), (tag, k)
        if g[3] is not None:
            assert _same(g[3][0], o[3][0]) and _same(g[3][1], o[3][1]), (tag, k)


OPTS = {"plain": {}, "dist": dict(dist=True), "all": dict(with_ua=True, dist=True, outlier=True)}


@pytest.mark.parametrize("opts", list(OPTS))
@pytest.mark.parametrize("path", ["frame", "raw"])
@pytest.mark.parametrize("setup", ["single", "single_ext", "rig"])
def test_matches_oracle(mloam, scene, setup, path, opts):
    """Bit-identical clouds on the stream path and from graph replays, with and without the look-ahead (which announces the other sweep);
    the device read equals the host read; pose, statistics, mloam_frame_scan and the outlier cloud bit-identical to the run with the
    feature off, and one launch more per frame."""
    cfg = Cfg(setup, path == "raw", **OPTS[opts])
    frames = _frames(scene, cfg.L, cfg.raw)
    inputs = _inputs(mloam, frames, cfg)
    for graphs in (True, False):
        for lookahead in (False, True):
            tag = (graphs, lookahead)
            off, off_launches = _run(mloam, scene, frames, cfg, reg=False, lookahead=lookahead, graphs=graphs)
            got, launches = _run(mloam, scene, frames, cfg, lookahead=lookahead, graphs=graphs)
            assert all(g[1]["ran"] == 1 for g in got)
            _check_against_oracle(got, inputs, cfg, tag)
            _check_unchanged(got, off, tag)
            assert launches == [n + 1 for n in off_launches], (tag, launches, off_launches)


def test_stage_profiling(mloam, scene):
    """Stage profiling (event scopes, the look-ahead off): the same clouds, and mloam_profile_get("registered") times one launch a frame."""
    cfg = Cfg("rig", False, with_ua=True, dist=True, outlier=True)
    frames = _frames(scene, 3, False)
    got, _ = _run(mloam, scene, frames, cfg, prof=True, lookahead=True)
    ms, cnt = got.pop()
    assert cnt == len(got) and ms > 0.0
    _check_against_oracle(got, frames, cfg, "prof")


def test_frame_device_caller_overwrites_sweep(mloam, scene):
    """mloam_frame_device with the look-ahead announcing the next device sweep: the caller overwrites each sweep after its call returns; the
    clouds read afterwards are still those of the sweep the frame took."""
    import torch
    cfg = Cfg("rig", False, outlier=True)
    frames = _frames(scene, 3, False)
    dev = [tuple(torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in fr) for fr in frames]
    sm, cm = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (scene["surf_map"], scene["corner_map"]))
    cx = _ctx(mloam, 3)
    try:
        cfg.configure(cx, True)
        seq = [dev[k % 2] for k in range(4)]
        for k, (c, ss, se) in enumerate(seq):
            if k + 1 < len(seq):
                nc, nss, nse = seq[k + 1]
                cx.frame_set_next_device(nc.data_ptr(), nc.shape[0], nss.data_ptr(), nse.data_ptr(), nss.shape[0])
            torch.cuda.synchronize()
            pose, st = cx.frame_device(c.data_ptr(), c.shape[0], ss.data_ptr(), se.data_ptr(), ss.shape[0], sm.data_ptr(), sm.shape[0],
                                       cm.data_ptr(), cm.shape[0], scene["traj"][1 + k % 2])
            keep = c.clone()
            c.fill_(123.0)  # the caller reuses its buffer
            torch.cuda.synchronize()
            got = [cx.frame_registered(w) for w in range(3)]
            d = cx.frame_registered_device(mloam.REGISTERED_SURF).cpu().numpy()
            c.copy_(keep)
            torch.cuda.synchronize()
            want = cfg.want(frames[k % 2], pose, k)
            for t in range(3):
                assert _same(got[t], want[t]), (k, t)
            assert _same(d, got[1]), k
    finally:
        cx.close()


def test_map_gated_frame(mloam, scene):
    """A frame the map gate rejects (too few map points) registers its clouds at the initial pose, as the reference publishes it."""
    cfg = Cfg("rig", False, dist=True, outlier=True)
    frames = _frames(scene, 3, False)
    cx = _ctx(mloam, 3)
    try:
        cfg.configure(cx, True)
        for k in range(3):  # the stream path, the capture, a replay
            cx.frame_undistort(UNDIST[0][:3])
            c, ss, se = frames[0]
            init = scene["traj"][1]
            pose, st = cx.frame(c, ss, se, scene["surf_map"][:40], scene["corner_map"][:8], init)
            assert st["ran"] == 0 and np.array_equal(pose, init)
            want = cfg.want(frames[0], init, 0)
            for t in range(3):
                assert _same(cx.frame_registered(t), want[t]), (k, t)
    finally:
        cx.close()


def test_all_non_finite_raw_lidar(mloam, scene):
    """A raw LiDAR whose every point is non-finite: removeNaN leaves its part empty — no points, no outlier point for it."""
    cfg = Cfg("rig", True, outlier=True, dist=True)
    frames = _frames(scene, 3, True, nan_lidar=1)
    inputs = _inputs(mloam, frames, cfg)
    got, _ = _run(mloam, scene, frames, cfg, lookahead=True)
    _check_against_oracle(got, inputs, cfg, "nan")
    for g in got:
        assert 1.0 not in g[4][0][:, 3].tolist()


def test_c4_frame(mloam, scene):
    """One 4 x 64 x 2048 frame (about 524k points) at full size, with DISTORTION and the outlier cloud, read on the host and on the device."""
    ext = syn.rig_extrinsics(4)
    cloud, ss, se, _ = syn.make_multi_sweep(scene["scene"], scene["traj"][1], 4, 64, 2048, seed=77, ext=ext)
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell = 256, 4, 1, 0.5
    cx = mloam.Context(0, p)
    try:
        cx.set_lidars(4, ext)
        cx.set_outlier(LEAF)
        cx.set_distortion(True, 0.1)
        cx.set_registered(True)
        und = np.concatenate([UNDIST[0], UNDIST[1][:1]])
        cx.frame_undistort(und)
        pose, st = cx.frame(cloud, ss, se, scene["surf_map"], scene["corner_map"], scene["traj"][1])
        assert st["ran"] == 1
        got = [cx.frame_registered(w) for w in range(3)]
        want = rl.registered(cloud, ss, se, pose, ext7=ext, poses7=und, outlier=True)
        assert got[0].shape[0] == cloud.shape[0] + 4
        for t in range(3):
            assert _same(got[t], want[t]), t
            assert _same(cx.frame_registered_device(t).cpu().numpy(), got[t]), t
    finally:
        cx.close()


def test_error_paths(mloam, scene):
    frames = _frames(scene, 3, False)
    lib = mloam.lib()
    cx = _ctx(mloam, 3)
    try:
        cx.set_lidars(3, _exts(3))
        for bad in (-1, 2):
            assert lib.mloam_set_registered(cx._h, bad) == E_INVALID
        cx.set_registered(True)
        n = C.c_int(-1)
        assert lib.mloam_frame_registered(cx._h, 0, None, 0, C.byref(n)) == E_STATE and n.value == 0  # before any frame
        c, ss, se = frames[0]
        cx.set_registered(False)
        cx.frame(c, ss, se, scene["surf_map"], scene["corner_map"], scene["traj"][1])
        assert lib.mloam_frame_registered(cx._h, 0, None, 0, C.byref(n)) == E_STATE  # the frame ran with it off
        cx.set_registered(True)
        pose, _ = cx.frame(c, ss, se, scene["surf_map"], scene["corner_map"], scene["traj"][1])
        for bad in (-1, 3):
            assert lib.mloam_frame_registered(cx._h, bad, None, 0, C.byref(n)) == E_INVALID
            d = C.c_void_p()
            assert lib.mloam_frame_registered_device(cx._h, bad, C.byref(d), C.byref(n)) == E_INVALID
        for w in range(3):
            assert lib.mloam_frame_registered(cx._h, w, None, 0, C.byref(n)) == 0 and n.value > 0
            buf = np.zeros((n.value, 4), np.float32)
            m = C.c_int(-1)  # the capacity rule: too small -> MLOAM_E_INVALID with the size in *n
            assert lib.mloam_frame_registered(cx._h, w, mloam._p(buf), n.value - 1, C.byref(m)) == E_INVALID and m.value == n.value
            assert lib.mloam_frame_registered(cx._h, w, mloam._p(buf), n.value, C.byref(m)) == 0 and m.value == n.value
            assert _same(buf, cx.frame_registered(w))
        assert cx.frame_registered(0).shape[0] == c.shape[0]
        surf, corner = cx.frame_scan()[0], cx.frame_scan()[2]
        cx.scan2map(surf, corner, pose)  # a scan has no sweep
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
            cx.frame_registered(0)
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
            cx.frame_registered_device(1)
    finally:
        cx.close()


def test_communicator_rejected(mloam):
    import torch  # noqa: F401  (torch's NCCL first, as test_keyframe_mapper.py explains)
    cx = _ctx(mloam, 1)
    try:
        try:
            cx.comm_init(1, 0, mloam.Context.comm_unique_id())
        except mloam.MloamError as e:
            pytest.skip(f"no NCCL on this machine: {e}")
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
            cx.set_registered(True)
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
            cx.frame_registered(0)
    finally:
        cx.close()


# ---------------------------------------------------------------------------------------------------- closed mapper loop
N_LOOP = 16


def _loop(mloam, reg):
    """The mapper loop of process() on the device with the keyframe store (3 LiDARs, with_ua, the outlier cloud): per frame (pose, saved,
    frame_scan, registered clouds or None) and, at the end, every keyframe's scan and outlier cloud and both global maps."""
    sc = syn.make_scene()
    traj = syn.trajectory(N_LOOP)
    ext = syn.rig_extrinsics(3)
    sweeps = [syn.make_multi_sweep(sc, traj[k], 3, 16, 1024, seed=60 + k, ext=ext) for k in range(N_LOOP)]
    odom = [syn.pose_mul(traj[k], syn.pose7([0.002 * k, -0.001 * k, 0.0], syn.quat_from_rpy(0.0, 0.0, np.radians(0.02 * k)))) for k in range(N_LOOP)]
    ext_cov = ua.ext_covariances(3, seed=7)
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = 48, 10, 1, 0.5, 1024
    cx = mloam.Context(0, p)
    out = []
    try:
        cx.set_lidars(3, ext)
        cx.set_outlier(LEAF)
        cx.set_registered(reg)
        cx.keyframes_init(0.3, 2.0, 6.0, 1.0, 1e3)
        wmap_wodom = np.array([0, 0, 0, 0, 0, 0, 1.0])
        for k in range(N_LOOP):
            cloud, ss, se, _ = sweeps[k]
            cx.set_uncertainty(True, ext_cov, COV_MEAS, 1e3)
            pred = ml.pose_mul(wmap_wodom, odom[k])
            cx.keyframe_submap(pred)
            pose, st = cx.frame(cloud, ss, se, None, None, pred, False)
            wmap_wodom = ml.pose_mul(pose, ml.pose_inv(odom[k]))
            regs = None
            if reg:
                regs = [cx.frame_registered(w) for w in range(3)]
                want = rl.registered(cloud, ss, se, pose, ext7=ext, outlier=True)
                for t in range(3):
                    assert _same(regs[t], want[t]), (k, t)
            out.append((pose, dict(st), cx.frame_scan(), cx.frame_outlier(), cx.keyframe_save()))
        n_kf = cx.keyframe_query()[0]
        kfs = [(cx.keyframe_scan(i), cx.keyframe_outlier(i)) for i in range(n_kf)]
        gms = [cx.global_map(mode, center=out[-1][0]) for mode in (mloam.GLOBAL_MAP_SURROUND, mloam.GLOBAL_MAP_SAVE)]
    finally:
        cx.close()
    return out, kfs, gms


def test_closed_loop_keyframes_and_global_maps(mloam):
    """The registered clouds of every frame of the closed mapper loop equal the oracle's; poses, statistics, scans, outlier clouds, keyframe
    decisions, the keyframe store's contents and both global maps are bit-identical to the run without them."""
    on, kf_on, gm_on = _loop(mloam, True)
    off, kf_off, gm_off = _loop(mloam, False)
    assert sum(o[4] for o in on) >= 3
    for k, (a, b) in enumerate(zip(on, off)):
        assert np.array_equal(a[0], b[0]) and a[1] == b[1] and a[4] == b[4], k
        assert all(_same(x, y) for x, y in zip(a[2], b[2])) and all(_same(x, y) for x, y in zip(a[3], b[3])), k
    assert len(kf_on) == len(kf_off)
    for (sa, oa), (sb, ob) in zip(kf_on, kf_off):
        assert all(_same(np.asarray(x, np.float32), np.asarray(y, np.float32)) if np.asarray(x).dtype == np.float32 else np.array_equal(x, y)
                   for x, y in zip(sa, sb))
        assert all(_same(x, y) for x, y in zip(oa, ob))
    for ga, gb in zip(gm_on, gm_off):
        assert all(_same(x, y) for x, y in zip(ga, gb))

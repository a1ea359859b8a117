"""GPU tests (-m gpu) of the published clouds as PointCloud2 data (mloam_cloud_msgs / mloam_cloud_msgs_device): every message is byte for
byte the host statement (m-loam_b200/host/mloam_io.hpp packPointCloud2 / packPointCloud2Cov) of what the existing reads return —
mloam_frame_registered for the registered clouds; the submap outputs and mloam_global_map_read, with the cov_trace composed from the
oracle's single steps, for the covariance clouds — over mloam_frame, mloam_frame_raw and mloam_frame_msg, 1 and 3 LiDARs, plain,
DISTORTION and with_ua with the outlier cloud, graph replay and the stream path with and without the look-ahead, a 4 x 64 x 2048 frame,
every frame of the closed mapper loop, both global-map modes and the int32-overflow pass-through; non-finite points keep their bits; odd
and pinned destinations; the device bytes equal the host bytes; one launch per call; frames unchanged by packing; every error path."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import cloud_msgs_lib as cml
import front_end_lib as fel
import global_map_lib as gl
import mapper_lib as ml
import synthetic as syn
import uncertainty_lib as ua
import wire_lib as wl

pytestmark = pytest.mark.gpu

E_INVALID, E_STATE = -1, -4
COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])
RINGS, HORIZON = 16, 512
REG = [0, 1, 2]
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


def _ctx(mloam, n_scans, graphs=True):
    if not graphs:
        os.environ["MLOAM_DISABLE_GRAPHS"] = "1"
    try:
        p = mloam.default_params()
        p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = n_scans, 4, 1, 0.5, 1024
        return mloam.Context(0, p)
    finally:
        os.environ.pop("MLOAM_DISABLE_GRAPHS", None)


def _inputs(sc, L, entry):
    """Sweeps A and B as the entry point takes them: (cloud, ss, se) | (raw, counts) | [message per LiDAR]."""
    ext = _exts(L)
    out = []
    for k in (1, 2):
        pose = sc["traj"][k]
        if entry == "frame":
            cloud, ss, se, _ = syn.make_multi_sweep(sc["scene"], pose, L, RINGS, HORIZON, seed=40 + k, ext=ext)
            out.append((cloud, ss, se))
            continue
        parts = [fel.raw_sweep(sc["scene"], pose, RINGS, HORIZON, 40 + 31 * k + l, ext=ext[l]) for l in range(L)]
        if entry == "raw":
            out.append((np.ascontiguousarray(np.concatenate(parts)), np.array([p.shape[0] for p in parts], np.int32)))
        else:
            out.append([wl.as_arg(wl.pack(p, "xyzi32", rng=np.random.default_rng(k * 7 + l))) for l, p in enumerate(parts)])
    return out


def _configure(mloam, cx, L, entry, variant, inputs):
    cx.set_lidars(L, _exts(L))
    if variant == "ua_outlier":
        cx.set_uncertainty(True, ua.ext_covariances(L, seed=3), COV_MEAS, 1e3)
        cx.set_outlier(0.8)
    if variant == "dist":
        cx.set_distortion(True, 0.1)
    cx.set_registered(True)
    if entry != "frame":
        cx.set_front_end(RINGS, HORIZON)
    if entry == "msg":
        msg = wl.pack(np.zeros((4, 4), np.float32), "xyzi32")
        cx.set_front_end_layout([wl.layout(mloam, msg, None)] * L)


def _frame(cx, entry, fr, sc, init):
    if entry == "frame":
        return cx.frame(fr[0], fr[1], fr[2], sc["surf_map"], sc["corner_map"], init)
    if entry == "raw":
        return cx.frame_raw(fr[0], fr[1], sc["surf_map"], sc["corner_map"], init)
    return cx.frame_msg(fr, sc["surf_map"], sc["corner_map"], init)


def _announce(cx, entry, fr):
    if entry == "frame":
        cx.frame_set_next(*fr)
    elif entry == "raw":
        cx.frame_set_next_raw(*fr)
    else:
        cx.frame_set_next_msg(fr)


def _check_registered(mloam, cx):
    """The three registered messages against packPointCloud2 of mloam_frame_registered, on the host and on the device."""
    reads = [cx.frame_registered(w) for w in REG]
    got = cx.cloud_msgs(REG)
    for w in REG:
        assert got[w] == cml.pack(reads[w]), w
    dev = cx.cloud_msgs_device(REG)
    for w in REG:
        assert dev[w].cpu().numpy().tobytes() == got[w], w
    return reads


def _run(mloam, sc, L, entry, variant, pack, graphs=True, lookahead=True, rounds=2):
    """Frames A, B, A, B (the same arrays, so that graphs capture and replay), packing the registered messages after each when `pack`:
    per frame its pose, stats, launches, frame_scan and registered reads."""
    inputs = _inputs(sc, L, entry)
    cx = _ctx(mloam, RINGS * L, graphs)
    out = []
    try:
        _configure(mloam, cx, L, entry, variant, inputs)
        seq = [inputs[k % 2] for k in range(2 * rounds)]
        for k, fr in enumerate(seq):
            if lookahead and k + 1 < len(seq):
                _announce(cx, entry, seq[k + 1])
            if variant == "dist":
                cx.frame_undistort(UNDIST[k % 2][:L])
            l0 = cx.launch_count()
            pose, st = _frame(cx, entry, fr, sc, sc["traj"][1 + k % 2])
            launches = cx.launch_count() - l0
            reads = _check_registered(mloam, cx) if pack else [cx.frame_registered(w) for w in REG]
            out.append(dict(pose=pose, stats=dict(st), H=st["H"], launches=launches, scan=cx.frame_scan(), reads=reads))
        out.append(dict(captures=cx.profile_get("graph_captures")))
    finally:
        cx.close()
    return out


@pytest.mark.parametrize("variant", ["plain", "dist", "ua_outlier"])
@pytest.mark.parametrize("entry", ["frame", "raw", "msg"])
@pytest.mark.parametrize("n_lidars", [1, 3])
def test_registered_messages(mloam, scene, n_lidars, entry, variant):
    """Graph capture and replay with the look-ahead announced: after every frame the three messages are packPointCloud2 of the reads."""
    out = _run(mloam, scene, n_lidars, entry, variant, True)
    assert all(o["reads"][0].shape[0] > 1000 for o in out[:-1])


@pytest.mark.parametrize("graphs,lookahead", [(True, False), (False, True), (False, False)])
def test_paths_and_no_interference(mloam, scene, graphs, lookahead):
    """The stream path and graph replay, with and without the look-ahead: the messages are right, and poses, stats, launches, scans,
    registered reads and graph captures are bit-identical to the same run that never packs."""
    a = _run(mloam, scene, 3, "raw", "ua_outlier", True, graphs, lookahead)
    b = _run(mloam, scene, 3, "raw", "ua_outlier", False, graphs, lookahead)
    assert a[-1] == b[-1]
    for k, (x, y) in enumerate(zip(a[:-1], b[:-1])):
        assert np.array_equal(x["pose"], y["pose"]) and x["stats"] == y["stats"] and np.array_equal(x["H"], y["H"]), k
        assert x["launches"] == y["launches"], k
        assert all(np.array_equal(p.view(np.uint32), q.view(np.uint32)) for p, q in zip(x["scan"], y["scan"])), k
        assert all(np.array_equal(p.view(np.uint32), q.view(np.uint32)) for p, q in zip(x["reads"], y["reads"])), k


def test_non_finite_full_res_bits(mloam, scene):
    """Non-finite sweep points reach FULL_RES and the message keeps their bit patterns (NaN payloads, infinities)."""
    cloud, ss, se, _ = syn.make_multi_sweep(scene["scene"], scene["traj"][1], 1, RINGS, HORIZON, seed=41, ext=_exts(1))
    cloud = cloud.copy()
    bits = cloud.view(np.uint32)
    bits[0, 0], bits[1, 3] = 0x7FC12345, 0xFFA00001  # a quiet and a signalling NaN with payloads, in x and in the intensity lane
    cloud[2, 1], cloud[3, 2] = np.inf, -np.inf
    cx = _ctx(mloam, RINGS)
    try:
        cx.set_registered(True)
        cx.frame(cloud, ss, se, scene["surf_map"], scene["corner_map"], scene["traj"][1])
        full = cx.frame_registered(0)
        msg = cx.cloud_msgs([mloam.MSG_FULL_RES])[0]
        assert msg == cml.pack(full)
        rec = np.frombuffer(msg, np.uint8).reshape(-1, 32)
        assert (~np.isfinite(full[:4])).any(axis=1).all()  # every altered point reaches FULL_RES non-finite
        assert np.array_equal(rec[:, 16:20].copy().view(np.uint32)[:, 0], full[:, 3].view(np.uint32))
    finally:
        cx.close()


def test_c4_frame_pinned_and_odd_destinations(mloam, scene):
    """One 4 x 64 x 2048 frame with DISTORTION and the outlier cloud: the messages into pageable memory at an odd address and into pinned
    memory equal packPointCloud2 of the reads and the device bytes; each call is one launch."""
    import torch

    ext = syn.rig_extrinsics(4)
    cloud, ss, se, _ = syn.make_multi_sweep(scene["scene"], scene["traj"][1], 4, 64, 2048, seed=77, ext=ext)
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell = 256, 4, 1, 0.5
    cx = mloam.Context(0, p)
    try:
        cx.set_lidars(4, ext)
        cx.set_outlier(0.8)
        cx.set_distortion(True, 0.1)
        cx.set_registered(True)
        cx.frame_undistort(np.concatenate([UNDIST[0], UNDIST[1][:1]]))
        pose, st = cx.frame(cloud, ss, se, scene["surf_map"], scene["corner_map"], scene["traj"][1])
        assert st["ran"] == 1
        want = [cml.pack(cx.frame_registered(w)) for w in REG]
        assert len(want[0]) == 32 * (cloud.shape[0] + 4)
        odd = [np.zeros(len(w) + 1, np.uint8)[1:] for w in want]
        assert all(a.__array_interface__["data"][0] % 2 == 1 for a in odd)
        pinned = [torch.zeros(len(w), dtype=torch.uint8).pin_memory().numpy() for w in want]
        for dst in (odd, pinned):
            l0 = cx.launch_count()
            assert cx.cloud_msgs(REG, out=dst) == want
            assert cx.launch_count() - l0 == 1
            assert [d.tobytes() for d in dst] == want
        assert [t.cpu().numpy().tobytes() for t in cx.cloud_msgs_device(REG)] == want
    finally:
        cx.close()


def _params(mloam, n_scans):
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = n_scans, 10, 1, 0.5, 1024
    return p


def _traj(n, step=0.35, seed=5):
    """A path that saves a keyframe every few frames at DISTANCE_KEYFRAMES 0.9 m."""
    rng = np.random.Generator(np.random.PCG64(seed))
    out = []
    for k in range(n):
        jt = rng.normal(0, 0.01, 3)
        out.append(syn.pose7([-12.0 + step * k + jt[0], 0.3 * np.sin(0.2 * k) + jt[1], 1.8 + jt[2]], syn.quat_from_rpy(0.0, 0.0, 0.02 * np.sin(0.3 * k))))
    return np.stack(out)


class _Store:
    """The keyframes the loop saved and the single-step composition of the clouds the store derives from them, with the cov_trace the
    device filters store (an independent statement: the oracle's store gives points and cov_vec only)."""

    def __init__(self, ext, ext_cov, with_ua, thr):
        self.ext, self.ext_cov, self.with_ua, self.thr = ext, ext_cov, with_ua, thr
        self.kfs, self.merged = [], ([], [])

    def assoc(self, kf_id, t):
        pose, cov, clouds = self.kfs[kf_id]
        return cml.associate(pose, cov, clouds[t], self.ext, self.ext_cov, COV_MEAS, self.with_ua, self.thr)

    def rebuild(self, chosen, leaves):
        """extractSurroundingKeyFrames' `+=` of the chosen keyframes (emptied by a save only) and the two filters."""
        for t in (0, 1):
            self.merged[t].extend(self.assoc(i, t) for i in chosen)
        return [cml.voxel_cov(self.merged[t], leaves[t], self.thr) for t in (0, 1)]

    def save(self, pose, cov, surf, corner):
        self.kfs.append((pose, cov, (surf, corner)))
        self.merged = ([], [])  # clearCloud

    def global_map(self, mode, chosen, leaf):
        """SURROUND: per chosen keyframe surf then corner into map 0; SAVE: surf into map 0, corner into map 1 (no outlier clouds here)."""
        if mode == 0:
            return [cml.voxel_cov([self.assoc(i, t) for i in chosen for t in (0, 1)], leaf, self.thr)]
        return [cml.voxel_cov([self.assoc(i, t) for i in chosen], leaf, self.thr) for t in (0, 1)]


def _gm_check(mloam, cx, om, store, mode, center, radius, kf_leaf, leaf, last_tested=None):
    """One global map: device chosen ids, points and cov_vec equal the oracle's and the composition's; the messages equal
    packPointCloud2Cov of the device reads with the composition's cov_trace.  Returns map 0's (cov6, cov_trace)."""
    g = cx.global_map(mode, center, radius, kf_leaf, leaf)
    chosen = cx.global_map_chosen()
    o_ch, o = gl.global_map(om, mode, center if center is not None else last_tested, radius, kf_leaf, leaf)
    want = store.global_map(mode, chosen, leaf)
    assert chosen == o_ch, mode
    msgs = cx.cloud_msgs([mloam.MSG_GLOBAL_MAP0, mloam.MSG_GLOBAL_MAP1])
    dev = cx.cloud_msgs_device([mloam.MSG_GLOBAL_MAP0, mloam.MSG_GLOBAL_MAP1])
    for m in range(len(want)):
        assert np.array_equal(g[2 * m], o[2 * m]) and np.array_equal(g[2 * m + 1], o[2 * m + 1]), (mode, m)
        assert np.array_equal(g[2 * m], want[m][0]) and np.array_equal(g[2 * m + 1], want[m][1]), (mode, m)
        assert msgs[m] == cml.pack_cov(g[2 * m], g[2 * m + 1], want[m][2]), (mode, m)
    if mode == mloam.GLOBAL_MAP_SURROUND:
        assert msgs[1] == b""
    assert [t.cpu().numpy().tobytes() for t in dev] == msgs
    return want[0][1], want[0][2]


@pytest.mark.parametrize("with_ua", [True, False])
def test_mapper_loop_surround_and_global_maps(mloam, with_ua):
    """The closed mapper loop on a 3-LiDAR rig with the oracle's store in lock-step: SURROUND after every submap is packPointCloud2Cov of
    the submap outputs (surf then corner) with the cov_trace of the single-step composition, and empty after every save; after every save
    both global-map modes and, at the end, a SAVE map whose voxel index overflows int32 (the input passes through with the association's
    cov_trace, which is not the sum of the stored cov_vec).  n = 1 and n = 6 are one launch each."""
    scene = syn.make_scene()
    traj = _traj(30)
    sweeps = [syn.make_multi_sweep(scene, traj[k], 3, 16, 1024, seed=120 + k) for k in range(len(traj))]
    ext = sweeps[0][3]
    thr = 0.08 if with_ua else 10.0
    p = _params(mloam, 48)
    cx = mloam.Context(0, p)
    om = ml.Mapper(0.9, 5.0, 2.6, 1.5, thr)
    lib = mloam.lib()
    ext_cov = ua.ext_covariances(3, seed=1)
    store = _Store(ext, ext_cov, with_ua, thr)
    filt = [cml.voxel_cov([], 1.0, thr)] * 2
    n_saved = n_surround = 0
    try:
        cx.set_lidars(3, ext)
        cx.set_uncertainty(with_ua, ext_cov if with_ua else None, COV_MEAS, 1e3)
        om.set_lidars(ext, ext_cov, COV_MEAS, with_ua)
        cx.set_registered(True)
        cx.keyframes_init(0.9, 5.0, 2.6, 1.5, thr)
        assert cx.cloud_msgs([mloam.MSG_SURROUND, mloam.MSG_GLOBAL_MAP0, mloam.MSG_GLOBAL_MAP1]) == [b"", b"", b""]
        for k, (cloud, ss, se, _) in enumerate(sweeps):
            rb, sp, sc6, cp, cc6 = cx.keyframe_submap(traj[k], want_output=True)
            assert rb == om.submap(traj[k])[0], k
            osp, osc, ocp, occ = om.maps()
            assert np.array_equal(sp, osp) and np.array_equal(sc6, osc) and np.array_equal(cp, ocp) and np.array_equal(cc6, occ), k
            if rb:
                filt = store.rebuild(cx.keyframe_query()[2], (p.surf_leaf, p.corner_leaf))
            assert all(np.array_equal(a, b) for a, b in zip((sp, sc6, cp, cc6), (filt[0][0], filt[0][1], filt[1][0], filt[1][1]))), k
            want = cml.pack_cov(np.concatenate([sp, cp]), np.concatenate([sc6, cc6]), np.concatenate([filt[0][2], filt[1][2]]))
            got = cx.cloud_msgs([mloam.MSG_SURROUND])[0]
            assert got == want, k
            n_surround += len(got) > 0
            cx.frame(cloud, ss, se, None, None, traj[k], False)
            s, _, c, _ = cx.frame_scan()
            saved = cx.keyframe_save(traj[k], np.zeros((6, 6)))
            assert saved == om.save(traj[k], np.zeros((6, 6)), s, c)[0], k
            if saved:
                n_saved += 1
                store.save(traj[k], np.zeros((6, 6)), s, c)
                filt = [cml.voxel_cov([], 1.0, thr)] * 2
                assert cx.cloud_msgs([mloam.MSG_SURROUND]) == [b""], k  # clearCloud
                _gm_check(mloam, cx, om, store, mloam.GLOBAL_MAP_SURROUND, traj[k], 1000.0, 2.5, 0.4)
                _gm_check(mloam, cx, om, store, mloam.GLOBAL_MAP_SAVE, None, 1000.0, 2.5, 0.8)
        assert n_saved >= 5 and n_surround >= 5
        cov6, tr = _gm_check(mloam, cx, om, store, mloam.GLOBAL_MAP_SAVE, None, 1000.0, 1.0, 1e-4)  # ~1e5 voxels per axis: int32 overflow
        summed = (cov6[:, 0] + cov6[:, 3]).astype(np.float32) + cov6[:, 5]
        assert cov6.shape[0] > 1000 and (not with_ua or np.any(summed.view(np.uint32) != tr.view(np.uint32)))  # without with_ua: all zero
        for srcs in ([mloam.MSG_GLOBAL_MAP0], list(range(6))):
            bufs = [np.zeros(len(b), np.uint8) for b in cx.cloud_msgs(srcs)]
            l0 = cx.launch_count()
            cx.cloud_msgs(srcs, out=bufs)
            assert cx.launch_count() - l0 == 1, srcs
            src = (C.c_int * len(srcs))(*srcs)
            ptrs, width = (C.c_void_p * len(srcs))(), (C.c_int * len(srcs))()
            l0 = cx.launch_count()
            assert lib.mloam_cloud_msgs_device(cx._h, len(srcs), src, ptrs, width) == 0 and cx.launch_count() - l0 == 1
            assert all(ptrs[k] % 256 == 0 for k in range(len(srcs)))
    finally:
        cx.close()
        om.close()


def test_error_paths(mloam, scene):
    lib = mloam.lib()
    cx = _ctx(mloam, RINGS)

    def call(srcs, n=None, caps=None, data=None, width=True, null_src=False):
        n = len(srcs) if n is None else n
        src = None if null_src else (C.c_int * max(len(srcs), 1))(*srcs)
        w = (C.c_int * 8)(*([-7] * 8)) if width else None
        d = (C.c_void_p * 8)(*(data or [])) if data is not False else None
        cp = (C.c_size_t * 8)(*(caps or [])) if caps is not False else None
        return lib.mloam_cloud_msgs(cx._h, n, src, d, cp, w), w

    try:
        cloud, ss, se, _ = syn.make_multi_sweep(scene["scene"], scene["traj"][1], 1, RINGS, HORIZON, seed=41, ext=_exts(1))
        assert call([0])[0] == E_STATE  # before any frame
        assert call([3])[0] == E_STATE  # without mloam_keyframes_init
        cx.frame(cloud, ss, se, scene["surf_map"], scene["corner_map"], scene["traj"][1])
        assert call([1])[0] == E_STATE  # the frame ran without the registered clouds
        cx.set_registered(True)
        cx.frame(cloud, ss, se, scene["surf_map"], scene["corner_map"], scene["traj"][1])
        for bad in ([0, 0], [6], [-1], [1, 2, 1]):
            assert call(bad)[0] == E_INVALID, bad
        assert call([], n=0)[0] == E_INVALID and call(list(range(6)) + [0], n=7)[0] == E_INVALID
        assert call([0], null_src=True)[0] == E_INVALID and call([0], width=False)[0] == E_INVALID
        assert call([0], data=False)[0] == E_INVALID and call([0], caps=False)[0] == E_INVALID
        assert call([0, 3])[0] == E_STATE  # a registered source is fine, the map source is not
        rc, w = call([2, 0, 1])  # size query
        assert rc == 0 and w[1] == cloud.shape[0] and w[0] > 0 and w[2] > 0
        full = cx.frame_registered(0)
        n_full, n_corner = w[1], w[0]
        fits, small = np.full(32 * n_full, 0x5A, np.uint8), np.full(32 * n_corner - 1, 0x5A, np.uint8)
        rc, w2 = call([0, 2], data=[fits.ctypes.data, small.ctypes.data], caps=[fits.nbytes, small.nbytes])
        assert rc == E_INVALID and (w2[0], w2[1]) == (n_full, n_corner)  # the widths are set; nothing is copied, not even FULL_RES
        assert (small == 0x5A).all() and (fits == 0x5A).all()
        big = np.zeros(32 * w[1], np.uint8)
        rc, _ = call([0], data=[big.ctypes.data], caps=[big.nbytes])
        assert rc == 0 and big.tobytes() == cml.pack(full)
        ptrs = (C.c_void_p * 1)()
        assert lib.mloam_cloud_msgs_device(cx._h, 1, (C.c_int * 1)(0), None, (C.c_int * 1)()) == E_INVALID
        assert lib.mloam_cloud_msgs_device(cx._h, 1, (C.c_int * 1)(0), ptrs, None) == E_INVALID
        cx.keyframes_init(1.0, 1.0, 30.0, 1.0, 10.0)
        rc, w = call([3, 4, 5])
        assert rc == 0 and list(w)[:3] == [0, 0, 0]  # empty clouds are a success
        cx.set_distortion(True, 0.1)
        with pytest.raises(mloam.MloamError):
            cx.frame(cloud, ss, se, scene["surf_map"], scene["corner_map"], scene["traj"][1])  # no undistortion pose: the frame fails
        assert call([0])[0] == E_STATE and call([4])[0] == 0
    finally:
        cx.close()


def test_communicator_rejected(mloam):
    import torch  # noqa: F401  (torch's NCCL first, as test_keyframe_mapper.py explains)
    cx = _ctx(mloam, RINGS)
    try:
        try:
            cx.comm_init(1, 0, mloam.Context.comm_unique_id())
        except mloam.MloamError as e:
            pytest.skip(f"no NCCL on this machine: {e}")
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
            cx.cloud_msgs([mloam.MSG_SURROUND])
    finally:
        cx.close()

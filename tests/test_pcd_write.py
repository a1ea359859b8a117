"""GPU tests (-m gpu) of the ASCII PCD writer (mloam_cloud_pcd / mloam_cloud_pcd_device / mloam_pcd_encode): every file is byte for byte
host/mloam_io.hpp writePCDASCII (PCL's writer restated with iostreams) of what the existing reads return — mloam_frame_registered, the
submap outputs and mloam_global_map_read in both modes with and without the outlier cloud (cov_trace as mloam_cloud_msgs packs it), and
pose_keyframes_3d from mloam_keyframe_scan / mloam_keyframe_query — after every step of a closed mapper loop; mloam_pcd_encode is the host
writer on 2^24 random bit patterns per layout and on the CPU test's targeted sets, with one-point and odd-sized clouds; the device bytes
equal the host bytes; empty sources give no bytes; one launch per call whatever the sources and sizes; frames around the calls are
bit-identical to frames without them, on graph replay and on the stream path; every error path."""
import ctypes as C
import os

import numpy as np
import pytest

import pcd_write_lib as pw
import synthetic as syn
import uncertainty_lib as ua

pytestmark = pytest.mark.gpu

E_INVALID, E_STATE = -1, -4
COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])
REG = [0, 1, 2]


def _msg_cov(msg: bytes):
    """A PointXYZIWithCov message of mloam_cloud_msgs -> (pts [n,4], cov6 [n,6], trace [n])."""
    rec = np.frombuffer(msg, np.uint8).reshape(-1, 48)
    f = rec.copy().view(np.float32)
    pts = np.concatenate([f[:, :3], f[:, 4:5]], axis=1)
    return np.ascontiguousarray(pts), np.ascontiguousarray(f[:, 5:11]), np.ascontiguousarray(f[:, 11])


def _check(cx, sources, want):
    """cloud_pcd of sources equals want (bytes per source), on the host and on the device, in one launch each."""
    l0 = cx.launch_count()
    got = cx.cloud_pcd(sources, out=[np.zeros(len(w) + 3, np.uint8) for w in want])
    assert cx.launch_count() - l0 == 1
    for s, g, w in zip(sources, got, want):
        assert g == w, s
    l0 = cx.launch_count()
    dev = cx.cloud_pcd_device(sources)
    assert cx.launch_count() - l0 == 1
    assert [t.cpu().numpy().tobytes() for t in dev] == want


def _cov_files(cx, mloam, sources, reads):
    """writePCDASCII of covariance reads (pts, cov6) with the cov_trace mloam_cloud_msgs packs for the same source."""
    msgs = cx.cloud_msgs(sources)
    out = []
    for m, (pts, cov6) in zip(msgs, reads):
        mp, mc, tr = _msg_cov(m)
        assert np.array_equal(mp.view(np.uint32), pts.view(np.uint32)) and np.array_equal(mc.view(np.uint32), cov6.view(np.uint32))
        out.append(pw.write_ascii(pw.XYZI_COV, pts, cov6, tr))
    return out


def _keyframes_file(cx):
    n = cx.keyframe_query()[0]
    pts = np.zeros((n, 4), np.float32)
    for i in range(n):
        pts[i, :3] = cx.keyframe_scan(i)[0][:3].astype(np.float32)
        pts[i, 3] = i
    return pw.write_ascii(pw.XYZI, pts)


def _traj(n, step=0.35, seed=5):
    rng = np.random.Generator(np.random.PCG64(seed))
    out = []
    for k in range(n):
        jt = rng.normal(0, 0.01, 3)
        out.append(syn.pose7([-12.0 + step * k + jt[0], 0.3 * np.sin(0.2 * k) + jt[1], 1.8 + jt[2]],
                             syn.quat_from_rpy(0.0, 0.0, 0.02 * np.sin(0.3 * k))))
    return np.stack(out)


@pytest.mark.parametrize("with_ua,outlier", [(True, True), (False, False)])
def test_mapper_loop_every_source_is_the_host_writer(mloam, with_ua, outlier):
    """A closed mapper loop on a 3-LiDAR rig: after every submap, SURROUND; after every frame, the three registered clouds; after every
    save, pose_keyframes_3d and both global-map modes; every file is writePCDASCII of the reads."""
    scene = syn.make_scene()
    traj = _traj(24)
    sweeps = [syn.make_multi_sweep(scene, traj[k], 3, 16, 1024, seed=120 + k) for k in range(len(traj))]
    ext = sweeps[0][3]
    thr = 0.08 if with_ua else 10.0
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = 48, 10, 1, 0.5, 1024
    cx = mloam.Context(0, p)
    n_saved = n_surround = 0
    try:
        cx.set_lidars(3, ext)
        ext_cov = ua.ext_covariances(3, seed=1)
        cx.set_uncertainty(with_ua, ext_cov if with_ua else None, COV_MEAS, 1e3)
        if outlier:
            cx.set_outlier(0.8)
        cx.set_registered(True)
        cx.keyframes_init(0.9, 5.0, 2.6, 1.5, thr)
        assert cx.cloud_pcd([3, 4, 5, 6]) == [b""] * 4  # empty sources: no bytes
        for k, (cloud, ss, se, _) in enumerate(sweeps):
            _, sp, sc6, cp, cc6 = cx.keyframe_submap(traj[k], want_output=True)
            want = _cov_files(cx, mloam, [mloam.MSG_SURROUND], [(np.concatenate([sp, cp]), np.concatenate([sc6, cc6]))])
            _check(cx, [mloam.MSG_SURROUND], want)
            n_surround += len(want[0]) > 0
            cx.frame(cloud, ss, se, None, None, traj[k], False)
            _check(cx, REG, [pw.write_ascii(pw.XYZI, cx.frame_registered(w)) for w in REG])
            if cx.keyframe_save(traj[k], np.zeros((6, 6))):
                n_saved += 1
                kf = _keyframes_file(cx)
                assert kf.count(b"\n") == 11 + n_saved
                g = cx.global_map(mloam.GLOBAL_MAP_SURROUND, traj[k], 1000.0, 2.5, 0.4)
                _check(cx, [mloam.MSG_GLOBAL_MAP0, mloam.MSG_GLOBAL_MAP1, mloam.PCD_KEYFRAMES],
                       _cov_files(cx, mloam, [mloam.MSG_GLOBAL_MAP0], [g[:2]]) + [b"", kf])
                g = cx.global_map(mloam.GLOBAL_MAP_SAVE, None, 0.0, 10.0, 0.8)
                files = _cov_files(cx, mloam, [mloam.MSG_GLOBAL_MAP0, mloam.MSG_GLOBAL_MAP1], [g[:2], g[2:]])
                _check(cx, [mloam.PCD_KEYFRAMES, mloam.MSG_GLOBAL_MAP0, mloam.MSG_GLOBAL_MAP1], [kf] + files)
        assert n_saved >= 5 and n_surround >= 5
        # all seven sources in one call
        reg = [pw.write_ascii(pw.XYZI, cx.frame_registered(w)) for w in REG]
        _, sp, sc6, cp, cc6 = cx.keyframe_submap(traj[-1], want_output=True)
        sur = _cov_files(cx, mloam, [mloam.MSG_SURROUND], [(np.concatenate([sp, cp]), np.concatenate([sc6, cc6]))])
        src = [6, 5, 4, 3, 2, 1, 0]
        _check(cx, src, [_keyframes_file(cx)] + files[::-1] + sur + reg[::-1])
    finally:
        cx.close()


def _encode_check(cx, clouds):
    """pcd_encode of clouds [(layout, pts[, cov6, trace])] equals the host writer, in one launch."""
    l0 = cx.launch_count()
    got = cx.pcd_encode(clouds)
    assert cx.launch_count() - l0 == 2  # the size query and the copy
    for k, c in enumerate(clouds):
        want = pw.write_ascii(*c)
        if got[k] != want:
            g, w = got[k].split(b"\n"), want.split(b"\n")
            bad = next(i for i in range(min(len(g), len(w))) if g[i] != w[i])
            raise AssertionError((k, bad, g[bad], w[bad]))


def _clouds_of_bits(bits, layout, sizes=None):
    nf = {pw.XYZ: 3, pw.XYZI: 4, pw.XYZI_COV: 11}[layout]
    bits = np.concatenate([bits, np.zeros((-bits.size) % nf, np.uint32)]).reshape(-1, nf)
    out, at = [], 0
    for n in (sizes or [bits.shape[0]]):
        b = bits[at:at + n]
        at += n
        pts = np.zeros((b.shape[0], 4), np.uint32)
        pts[:, :min(nf, 4)] = b[:, :min(nf, 4)]
        pts = pts.view(np.float32)
        if layout == pw.XYZI_COV:
            out.append((layout, pts, np.ascontiguousarray(b[:, 4:10]).view(np.float32), np.ascontiguousarray(b[:, 10]).view(np.float32)))
        else:
            out.append((layout, pts))
    return out


@pytest.mark.parametrize("layout", [pw.XYZ, pw.XYZI, pw.XYZI_COV])
def test_encode_random_bit_patterns(mloam, layout):
    """2^24 random float bit patterns per layout, in clouds of 1, 2, 127, 128, 129 and 1000003 points and the rest."""
    rng = np.random.default_rng(7 + layout)
    bits = rng.integers(0, 1 << 32, size=1 << 24, dtype=np.uint64).astype(np.uint32)
    nf = {pw.XYZ: 3, pw.XYZI: 4, pw.XYZI_COV: 11}[layout]
    n_pts = -(-bits.size // nf)
    sizes = [1, 2, 127, 128, 129, 1000003]
    sizes.append(n_pts - sum(sizes))
    cx = mloam.Context(0)
    try:
        _encode_check(cx, _clouds_of_bits(bits, layout, sizes))
    finally:
        cx.close()


def test_encode_targeted_sets(mloam):
    """The CPU test's targeted sets (every exponent's first and last mantissas, every exact tie, powers of ten, the %f / %e boundaries,
    the special values) through each layout."""
    bits = pw.targeted_bits()
    cx = mloam.Context(0)
    try:
        for layout in (pw.XYZ, pw.XYZI, pw.XYZI_COV):
            _encode_check(cx, _clouds_of_bits(np.roll(bits, layout), layout))
    finally:
        cx.close()


def test_launches_do_not_depend_on_sources_or_sizes(mloam):
    rng = np.random.default_rng(3)
    cx = mloam.Context(0)
    try:
        for clouds in ([(pw.XYZI, rng.standard_normal((1, 4)))],
                       [(pw.XYZ, rng.standard_normal((1000000, 4)))],
                       [(k % 3,) + ((rng.standard_normal((n, 4)),) if k % 3 < 2 else pw.cov_cloud(rng, n))
                        for k, n in enumerate([1, 5, 300, 70000, 2, 9, 1])]):
            sizes = [len(b) for b in cx.pcd_encode(clouds)]
            bufs = [np.zeros(n, np.uint8) for n in sizes]
            l0 = cx.launch_count()
            got = cx.pcd_encode(clouds, out=bufs)
            assert cx.launch_count() - l0 == 1 and [len(g) for g in got] == sizes
    finally:
        cx.close()


def _frames(mloam, sc, write, graphs):
    """Frames A, B, A, B with the look-ahead announced, the registered clouds and the keyframe store on; with `write`, every PCD source
    is written around each frame.  Per frame: pose, stats, launches of the frame call; then the graph captures."""
    if not graphs:
        os.environ["MLOAM_DISABLE_GRAPHS"] = "1"
    try:
        p = mloam.default_params()
        p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = 16, 4, 1, 0.5, 1024
        cx = mloam.Context(0, p)
    finally:
        os.environ.pop("MLOAM_DISABLE_GRAPHS", None)
    ext = syn.rig_extrinsics(1)
    ins = [syn.make_multi_sweep(sc["scene"], sc["traj"][k], 1, 16, 512, seed=40 + k, ext=ext)[:3] for k in (1, 2)]
    out = []
    try:
        cx.set_lidars(1, ext)
        cx.set_registered(True)
        cx.keyframes_init(0.9, 5.0, 2.6, 1.5, 10.0)
        for k in range(4):
            fr = ins[k % 2]
            cx.frame_set_next(*ins[(k + 1) % 2])
            if write and k:
                cx.cloud_pcd(list(range(7)))
                cx.pcd_encode([(pw.XYZI, fr[0][:1000])])
            l0 = cx.launch_count()
            pose, st = cx.frame(fr[0], fr[1], fr[2], sc["surf_map"], sc["corner_map"], sc["traj"][1 + k % 2])
            out.append((pose, dict(st), cx.launch_count() - l0, cx.frame_registered(0)))
            cx.keyframe_save(pose, np.zeros((6, 6)))
            cx.global_map(mloam.GLOBAL_MAP_SAVE, None, 0.0, 10.0, 0.8)
            if write:
                cx.cloud_pcd_device(list(range(7)))
        out.append(cx.profile_get("graph_captures"))
    finally:
        cx.close()
    return out


@pytest.mark.parametrize("graphs", [True, False])
def test_frames_around_the_calls_are_unchanged(mloam, graphs):
    sc = syn.make_scene()
    surf_map, corner_map = syn.make_submap(sc, 60000)
    s = dict(scene=sc, traj=syn.trajectory(4), surf_map=surf_map, corner_map=corner_map)
    a, b = _frames(mloam, s, True, graphs), _frames(mloam, s, False, graphs)
    assert a[-1] == b[-1]
    for k, (x, y) in enumerate(zip(a[:-1], b[:-1])):
        assert np.array_equal(x[0], y[0]) and x[1] == y[1] and x[2] == y[2], k
        assert np.array_equal(x[3].view(np.uint32), y[3].view(np.uint32)), k


def test_error_paths(mloam):
    lib = mloam.lib()
    cx = mloam.Context(0)

    def call(srcs, n=None, caps=None, data=None, nbytes=True, null_src=False):
        n = len(srcs) if n is None else n
        src = None if null_src else (C.c_int * max(len(srcs), 1))(*srcs)
        nb = (C.c_size_t * 8)(*([7] * 8)) if nbytes else None
        d = (C.c_void_p * 8)(*(data or [])) if data is not False else None
        cp = (C.c_size_t * 8)(*(caps or [])) if caps is not False else None
        return lib.mloam_cloud_pcd(cx._h, n, src, d, cp, nb), nb

    def enc(clouds, caps=None, data=None):
        arr = (mloam.PcdCloud * max(len(clouds), 1))()
        for k, (ptr, cov, tr, cnt, lay) in enumerate(clouds):
            arr[k].pts, arr[k].cov6, arr[k].trace, arr[k].count, arr[k].layout = ptr, cov, tr, cnt, lay
        nb = (C.c_size_t * 8)(*([7] * 8))
        return lib.mloam_pcd_encode(cx._h, len(clouds), arr, (C.c_void_p * 8)(*(data or [])), (C.c_size_t * 8)(*(caps or [])), nb), nb

    try:
        sc = syn.make_scene()
        surf_map, corner_map = syn.make_submap(sc, 60000)
        cloud, ss, se, _ = syn.make_multi_sweep(sc, syn.trajectory(2)[1], 1, 16, 512, seed=41)
        init = syn.trajectory(2)[1]
        assert call([0])[0] == E_STATE  # before any frame
        assert call([6])[0] == E_STATE and call([3])[0] == E_STATE  # without mloam_keyframes_init
        cx.frame(cloud, ss, se, surf_map, corner_map, init)
        assert call([1])[0] == E_STATE  # the frame ran without the registered clouds
        cx.set_registered(True)
        cx.frame(cloud, ss, se, surf_map, corner_map, init)
        for bad in ([0, 0], [7], [-1], [1, 2, 1]):
            assert call(bad)[0] == E_INVALID, bad
        assert call([], n=0)[0] == E_INVALID and call(list(range(7)) + [0], n=8)[0] == E_INVALID
        assert call([0], null_src=True)[0] == E_INVALID and call([0], nbytes=False)[0] == E_INVALID
        assert call([0], data=False)[0] == E_INVALID and call([0], caps=False)[0] == E_INVALID
        assert call([0, 6])[0] == E_STATE
        rc, nb = call([2, 0])  # size query
        assert rc == 0 and nb[0] > 0 and nb[1] > nb[0]
        full = pw.write_ascii(pw.XYZI, cx.frame_registered(0))
        assert nb[1] == len(full)
        fits, small = np.full(nb[1], 0x5A, np.uint8), np.full(nb[0] - 1, 0x5A, np.uint8)
        rc, nb2 = call([0, 2], data=[fits.ctypes.data, small.ctypes.data], caps=[fits.nbytes, small.nbytes])
        assert rc == E_INVALID and (nb2[0], nb2[1]) == (nb[1], nb[0])  # the sizes are set; nothing is copied
        assert (small == 0x5A).all() and (fits == 0x5A).all()
        rc, _ = call([0], data=[fits.ctypes.data], caps=[fits.nbytes])
        assert rc == 0 and fits.tobytes() == full
        ptrs = (C.c_void_p * 1)()
        assert lib.mloam_cloud_pcd_device(cx._h, 1, (C.c_int * 1)(0), None, (C.c_size_t * 1)()) == E_INVALID
        assert lib.mloam_cloud_pcd_device(cx._h, 1, (C.c_int * 1)(0), ptrs, None) == E_INVALID
        assert lib.mloam_cloud_pcd_device(cx._h, 1, (C.c_int * 1)(0), ptrs, (C.c_size_t * 1)()) == 0 and ptrs[0] % 256 == 0
        cx.keyframes_init(1.0, 1.0, 30.0, 1.0, 10.0)
        rc, nb = call([3, 4, 5, 6])
        assert rc == 0 and list(nb)[:4] == [0, 0, 0, 0]  # empty clouds are a success
        # mloam_pcd_encode
        pts = np.ones((10, 4), np.float32)
        cov = np.ones((10, 6), np.float32)
        pp, pc = pts.ctypes.data, cov.ctypes.data
        assert enc([(pp, None, None, 10, 3)])[0] == E_INVALID  # a layout that is not one of the three
        assert enc([(pp, None, None, -1, 0)])[0] == E_INVALID
        assert enc([(None, None, None, 10, 0)])[0] == E_INVALID
        assert enc([(pp, None, pc, 10, 2)])[0] == E_INVALID and enc([(pp, pc, None, 10, 2)])[0] == E_INVALID
        assert enc([(pp, None, None, 1 << 26, 2)])[0] == E_INVALID  # could exceed 2^31 - 1 bytes
        assert enc([])[0] == E_INVALID and enc([(pp, None, None, 1, 0)] * 17)[0] == E_INVALID
        rc, nb = enc([(pp, None, None, 10, 1), (None, None, None, 0, 2)])
        assert rc == 0 and nb[1] == 0 and nb[0] == len(pw.write_ascii(pw.XYZI, pts))
        buf = np.zeros(nb[0] - 1, np.uint8)
        rc, nb2 = enc([(pp, None, None, 10, 1)], caps=[buf.nbytes], data=[buf.ctypes.data])
        assert rc == E_INVALID and nb2[0] == nb[0] and not buf.any()
        assert lib.mloam_pcd_encode(cx._h, 1, None, (C.c_void_p * 1)(), (C.c_size_t * 1)(), (C.c_size_t * 1)()) == E_INVALID
    finally:
        cx.close()


def test_communicator_rejected(mloam):
    import torch  # noqa: F401  (torch's NCCL first, as test_keyframe_mapper.py explains)
    cx = mloam.Context(0)
    try:
        try:
            cx.comm_init(1, 0, mloam.Context.comm_unique_id())
        except mloam.MloamError as e:
            pytest.skip(f"no NCCL on this machine: {e}")
        for f in (lambda: cx.cloud_pcd([mloam.PCD_KEYFRAMES]), lambda: cx.pcd_encode([(pw.XYZ, np.ones((3, 4), np.float32))])):
            with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
                f()
    finally:
        cx.close()

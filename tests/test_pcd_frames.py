"""GPU tests (-m gpu) of the PCD decode: mloam_pcd_decode / mloam_pcd_decode_device against host/mloam_io.hpp decodePCDASCII (PCL's
reader restated with istringstream and atof) — bit for bit on millions of printf tokens, on rigs of 1 and 3 files with other layouts,
CRLF, tabs, blank lines and non-finite points, and on a 4 x 64 x 2048 rig; every refused body; mloam_front_end_pcd against
mloam_front_end on the sweep decodePCDASCII gives; and the decode's fixed launch count."""
import math

import numpy as np
import pytest

import front_end_lib as fel
import pcd_lib as pl
import synthetic as syn

pytestmark = pytest.mark.gpu

E_INVALID, E_STATE = -1, -4
RINGS, HORIZON = 16, 1800


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def _same(a, b):
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


def _ctx(mloam, n_scans=16):
    p = mloam.default_params()
    p.n_scans = n_scans
    return mloam.Context(0, p)


def _file(pts, fields, xyz_cols, prec=8, sep=" ", eol="\n", blank_every=0, seed=0):
    """A PCD file of pts (n x 3) with `fields` (pl.XYZ-style); xyz_cols: the token index of x, y, z; the other tokens random."""
    rng = np.random.default_rng(seed)
    n = pts.shape[0]
    cols = [rng.uniform(-5, 5, n).astype(np.float32) for _ in range(sum(f[3] for f in fields))]
    for k in range(3):
        cols[xyz_cols[k]] = pts[:, k]
    body = pl.ascii_body(cols, prec=prec, sep=sep, eol=eol)
    if blank_every:
        lines = body.split(eol.encode())
        body = b"".join(l + eol.encode() + (b"  \t\r\n" if i % blank_every == 0 else b"") for i, l in enumerate(lines[:-1]))
    data = pl.fields_header(fields, n) + body
    h = pl.header(data)
    assert h is not None
    return data, h


def _host_decode(data, h):
    rc, out = pl.decode_ascii(data[h["body"]:], h["points"], h["tokens"], (h["ix"], h["iy"], h["iz"]))
    assert rc == 0
    return out


def _body(data, h):
    return (np.frombuffer(data[h["body"]:], np.uint8), h["points"], h["tokens"], (h["ix"], h["iy"], h["iz"]))


def test_printf_corpora_bit_identical(mloam):
    """%.8g, %.9g and %.17g of 2^21 floats over every exponent (NaN and inf included as PCL writes them) as 3-token lines."""
    rng = np.random.default_rng(7)
    bits = rng.integers(0, 1 << 32, size=3 << 21, dtype=np.uint64).astype(np.uint32)
    f = bits.view(np.float32)
    f[np.isnan(f)] = np.nan  # "nan": the positive quiet NaN, as %g prints it without a sign
    pts = f.reshape(-1, 3)
    cx = _ctx(mloam)
    try:
        for prec in (8, 9, 17):
            data, h = _file(pts, pl.XYZ, (0, 1, 2), prec=prec)
            want = _host_decode(data, h)
            got = cx.pcd_decode([_body(data, h)])
            assert _same(got, want), prec
            if prec >= 9:
                fin = ~np.isnan(pts)
                assert np.array_equal(got[:, :3].view(np.uint32)[fin], pts.view(np.uint32)[fin])
    finally:
        cx.close()


def _rig(n, seed, n_pts=5000):
    rng = np.random.default_rng(seed)
    specs = [
        (pl.XYZ, (0, 1, 2), dict()),
        (pl.XYZI, (0, 1, 2), dict(sep="\t", eol="\r\n", prec=9)),
        ([("_", 1, "U", 4), ("z", 4, "F", 1), ("rgb", 4, "U", 1), ("x", 4, "F", 1), ("y", 4, "F", 1), ("t", 8, "F", 2)], (6, 7, 4),
         dict(blank_every=7, prec=17)),
    ]
    files = []
    for l in range(n):
        fields, cols, kw = specs[l % len(specs)]
        pts = (rng.standard_normal((n_pts + 37 * l, 3)) * 30).astype(np.float32)
        pts[rng.integers(0, pts.shape[0], 25), rng.integers(0, 3, 25)] = np.nan
        pts[rng.integers(0, pts.shape[0], 5), 0] = np.inf
        files.append(_file(pts, fields, cols, seed=seed + l, **kw))
    return files


@pytest.mark.parametrize("n", [1, 3])
def test_rig_decode_host_and_device_bytes(mloam, n):
    import torch

    files = _rig(n, 11)
    want = np.concatenate([_host_decode(d, h) for d, h in files])
    cx = _ctx(mloam)
    try:
        l0 = cx.launch_count()
        got = cx.pcd_decode([_body(d, h) for d, h in files])
        assert cx.launch_count() - l0 == 2  # one count and one parse launch, whatever the file count
        assert _same(got, want)
        dev = [torch.from_numpy(np.frombuffer(d[h["body"]:], np.uint8).copy()).cuda() for d, h in files]
        out = torch.zeros((want.shape[0], 4), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        cx.pcd_decode_device([(t.data_ptr(), t.numel(), h["points"], h["tokens"], (h["ix"], h["iy"], h["iz"])) for t, (_, h) in zip(dev, files)],
                             out.data_ptr())
        assert _same(out.cpu().numpy(), want)
    finally:
        cx.close()


def test_large_rig_4x64x2048(mloam):
    rng = np.random.default_rng(3)
    files = []
    for l in range(4):
        pts = (rng.standard_normal((64 * 2048, 3)) * 40).astype(np.float32)
        files.append(_file(pts, pl.XYZI, (0, 1, 2), seed=l))
    want = np.concatenate([_host_decode(d, h) for d, h in files])
    cx = _ctx(mloam)
    try:
        assert _same(cx.pcd_decode([_body(d, h) for d, h in files]), want)
    finally:
        cx.close()


def test_refused_bodies(mloam):
    good = b"1 2 3\n4 5 6\n"
    cases = [
        (b"1 2 3\n4 5\n", 2),                      # a short line
        (b"1 2 3\n4 x 6\n", 2),                    # a bad token
        (b"1 2 3\n", 2),                           # too few lines
        (b"1 2 3\n4 5 12345678901234567891\n", 2),  # more than 19 significant digits
        (b"1 2 3\n4 5 0x6\n", 2),
        (b"", 1),
    ]
    cx = _ctx(mloam)
    try:
        assert _same(cx.pcd_decode([(good, 2, 3, (0, 1, 2))])[:, :3], np.array([[1, 2, 3], [4, 5, 6]], np.float32))
        for body, points in cases:
            with pytest.raises(mloam.MloamError, match=f"error {E_INVALID}"):
                cx.pcd_decode([(good, 2, 3, (0, 1, 2)), (body, points, 3, (0, 1, 2))])
        for bad in [(good, 0, 3, (0, 1, 2)), (good, 2, 3, (0, 1, 3)), (good, 2, 3, (0, -1, 2)), (good, 2, 0, (0, 0, 0))]:
            with pytest.raises(mloam.MloamError, match=f"error {E_INVALID}"):
                cx.pcd_decode([bad])
        with pytest.raises(mloam.MloamError, match=f"error {E_INVALID}"):
            cx.pcd_decode([(good, 2, 3, (0, 1, 2))] * 17)
        # a refused body leaves the next decode's results as they are
        assert _same(cx.pcd_decode([(good, 2, 3, (0, 1, 2))])[:, :3], np.array([[1, 2, 3], [4, 5, 6]], np.float32))
    finally:
        cx.close()


def _exts(n):
    out = []
    for l in range(n):
        a = 2 * math.pi * l / n
        out.append([0.3 * math.cos(a), 0.3 * math.sin(a), 0.05 * l, 0.0, 0.0, math.sin(a / 4), math.cos(a / 4)])
    return np.array(out, np.float64)


@pytest.mark.parametrize("n", [1, 3])
def test_front_end_pcd_bit_identical(mloam, n):
    sc = syn.make_scene()
    traj = syn.trajectory(3)
    ext = _exts(n)
    files = []
    for l in range(n):
        raw = fel.raw_sweep(sc, traj[1], RINGS, HORIZON, 100 + l, time_field=False, ext=ext[l] if n > 1 else None, n_nan=20)
        files.append(_file(raw[:, :3].copy(), [pl.XYZ, pl.XYZI][l % 2], (0, 1, 2), prec=[8, 9][l % 2], seed=l))
    parts = [_host_decode(d, h) for d, h in files]
    raw = np.ascontiguousarray(np.concatenate(parts))
    counts = np.array([p.shape[0] for p in parts], np.int32)
    cx = _ctx(mloam, n * RINGS)
    try:
        if n > 1:
            cx.set_lidars(n, ext)
        cx.set_front_end(RINGS, HORIZON, 0.5, 0.1, False)
        want, ws, we = cx.front_end(raw, counts)
        got, gs, ge = cx.front_end_pcd([_body(d, h) for d, h in files])
        assert _same(got, want) and np.array_equal(gs, ws) and np.array_equal(ge, we)
        cx.set_front_end(RINGS, HORIZON, 0.5, 0.1, True)  # PointXYZ has no timestamp
        with pytest.raises(mloam.MloamError, match=f"error {E_INVALID}"):
            cx.front_end_pcd([_body(d, h) for d, h in files])
    finally:
        cx.close()
    cx = _ctx(mloam, n * RINGS)
    try:
        with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):  # no front end
            cx.front_end_pcd([_body(d, h) for d, h in files])
    finally:
        cx.close()


# ------------------------------------------------------------------------------------------------ frames
COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])
LAYOUTS = [(pl.XYZ, (0, 1, 2)), (pl.XYZI, (0, 1, 2)),
           ([("_", 1, "U", 4), ("z", 4, "F", 1), ("x", 4, "F", 1), ("y", 4, "F", 1), ("t", 8, "F", 2)], (5, 6, 4))]


@pytest.fixture(scope="module")
def scene():
    sc = syn.make_scene()
    surf_map, corner_map = syn.make_submap(sc, 60000)
    return dict(scene=sc, traj=syn.trajectory(6), surf_map=surf_map, corner_map=corner_map)


def _frame_sweep(sc, pose, n, seed, prec=8, sep=" "):
    """One rig sweep as PCD files (LiDAR l in layout l), and the raw sweep + counts decodePCDASCII gives for them."""
    ext = _exts(n)
    files, parts = [], []
    for l in range(n):
        raw = fel.raw_sweep(sc, pose, RINGS, HORIZON, seed * 31 + l, time_field=False, ext=ext[l] if n > 1 else None, n_nan=20)
        fields, cols = LAYOUTS[l % len(LAYOUTS)]
        d, h = _file(raw[:, :3].copy(), fields, cols, prec=prec, sep=sep, eol="\r\n" if l == 1 else "\n", blank_every=9 if l == 2 else 0,
                     seed=seed + l)
        files.append((d, h))
        parts.append(_host_decode(d, h))
    return dict(files=files, bodies=[_body(d, h) for d, h in files], raw=np.ascontiguousarray(np.concatenate(parts)),
                counts=np.array([p.shape[0] for p in parts], np.int32), ext=ext)


def _frame_sweeps(scene, n, k0=2, count=3, **kw):
    sweeps = [_frame_sweep(scene["scene"], scene["traj"][k], n, 10 + k, **kw) for k in range(k0, k0 + count)]
    inits = [syn.perturb_pose(scene["traj"][k], np.random.Generator(np.random.PCG64(7 + k))) for k in range(k0, k0 + count)]
    return sweeps, inits


def _setup(cx, n, sw, full, undist):
    if n > 1:
        cx.set_lidars(n, sw["ext"])
    cx.set_front_end(RINGS, HORIZON, 0.5, 0.1, False)
    if full:
        cx.set_uncertainty(True, np.stack([np.diag([1e-4, 1e-4, 1e-4, 1e-5, 1e-5, 1e-5])] * n), COV_MEAS, 10.0)
        cx.set_outlier(0.8)
        cx.set_registered(True)
    if undist:
        cx.set_distortion(True, 0.1)


def _undist_poses(n, k):
    a = 0.004 * (k + 1)
    return np.array([[0.4 + 0.05 * k, 0.02, 0.01, 0.0, 0.0, math.sin(a), math.cos(a)]] * n)


def _dev_bodies(sw, keep):
    ts = [__import__("torch").from_numpy(b[0].copy()).cuda() for b in sw["bodies"]]
    keep.append(ts)
    return [(t.data_ptr(), t.numel(), b[1], b[2], b[3]) for t, b in zip(ts, sw["bodies"])]


def _run(mloam, scene, n, sweeps, inits, kind, ahead, graph, full=False, undist=False, second=None):
    """Frames over the sweeps (twice with graphs: the second pass replays, over `second` when given) -> per frame (pose, stats, scan, cov,
    outlier, registered), launches per frame, "undistort_ahead" and "graph_captures".  kind: raw | raw_reuse | pcd | pcd_dev.  raw_reuse
    copies every sweep into one of two host buffers (alternating with the frame, as a dataset replay reuses its buffers) before the call:
    the graph keys of host PCD frames, which never hold the caller's pointer, are those of this run."""
    import torch
    p = mloam.default_params()
    p.n_scans = n * RINGS
    p.max_inner = 1 if graph else 30
    cx = mloam.Context(0, p)
    keep = []
    try:
        _setup(cx, n, sweeps[0], full, undist)
        sm, cm = scene["surf_map"], scene["corner_map"]
        passes = [sweeps] + ([second or sweeps] if graph else [])
        seq = [(s, k) for s in passes for k in range(len(sweeps))]
        dev = kind == "pcd_dev"
        if dev:
            d_bodies = {(id(s), k): _dev_bodies(s[k], keep) for s in passes for k in range(len(sweeps))}
            d_sm, d_cm = torch.from_numpy(sm).cuda(), torch.from_numpy(cm).cuda()
            torch.cuda.synchronize()
        out, launches = [], []
        announced = False
        bufs = [np.empty_like(sweeps[0]["raw"]) for _ in range(2)]
        for i, (s, k) in enumerate(seq):
            if undist and not announced:
                cx.frame_undistort(_undist_poses(n, k))
            nxt = seq[i + 1] if ahead and i + 1 < len(seq) else None
            if nxt is not None:
                ns, nk = nxt
                if kind == "raw":
                    cx.frame_set_next_raw(ns[nk]["raw"], ns[nk]["counts"])
                elif kind == "raw_reuse":
                    np.copyto(bufs[(i + 1) & 1], ns[nk]["raw"])
                    cx.frame_set_next_raw(bufs[(i + 1) & 1], ns[nk]["counts"])
                elif dev:
                    cx.frame_set_next_pcd_device(d_bodies[(id(ns), nk)])
                else:
                    cx.frame_set_next_pcd(ns[nk]["bodies"])
                if undist:
                    cx.frame_set_next_undistort(_undist_poses(n, nk))
            announced = nxt is not None and undist
            l0 = cx.launch_count()
            if kind == "raw":
                res = cx.frame_raw(s[k]["raw"], s[k]["counts"], sm, cm, inits[k])
            elif kind == "raw_reuse":
                if not ahead:
                    np.copyto(bufs[i & 1], s[k]["raw"])
                res = cx.frame_raw(bufs[i & 1], s[k]["counts"], sm, cm, inits[k])
            elif dev:
                res = cx.frame_pcd_device(d_bodies[(id(s), k)], d_sm.data_ptr(), d_sm.shape[0], d_cm.data_ptr(), d_cm.shape[0], inits[k])
            else:
                res = cx.frame_pcd(s[k]["bodies"], sm, cm, inits[k])
            launches.append(cx.launch_count() - l0)
            pose, st = res
            r = [pose, {x: st[x] for x in ("ran", "n_surf", "n_corner", "lm_iterations", "degenerate", "termination", "final_cost", "n_surf_in",
                                           "n_corner_in")}, cx.frame_scan(), cx.pose_covariance()]
            if full:
                r += [cx.frame_outlier(), [cx.frame_registered(w) for w in range(3)]]
            out.append(r)
        return out, launches, cx.profile_get("undistort_ahead")[1], cx.profile_get("graph_captures")[1]
    finally:
        cx.close()


def _assert_same(a, b):
    assert np.array_equal(a[0], b[0]), (a[0], b[0])
    assert a[1] == b[1], (a[1], b[1])
    assert a[1]["ran"] == 1
    for x, y in zip(a[2], b[2]):
        assert _same(x, y)
    assert np.array_equal(a[3], b[3])
    if len(a) > 4:
        for x, y in zip(a[4], b[4]):
            assert _same(x, y)
        for x, y in zip(a[5], b[5]):
            assert x.shape[0] > 0 and _same(x, y)


def _assert_two_more(got_l, ref_l, ahead):
    """The decode's two launches per sweep; with the look-ahead the first frame also decodes the announced sweep and the last frame
    takes its sweep decoded, so the run holds two more launches per frame."""
    d = [a - b for a, b in zip(got_l, ref_l)]
    assert sum(d) == 2 * len(d) and (ahead or d == [2] * len(d)), (d, got_l, ref_l)
    if ahead:
        assert d[1:-1] == [2] * (len(d) - 2), d


@pytest.mark.parametrize("n,full", [(1, False), (3, False), (3, True)])
@pytest.mark.parametrize("graph", [False, True])
def test_frame_pcd_bit_identical_to_frame_raw(mloam, scene, n, full, graph):
    sweeps, inits = _frame_sweeps(scene, n)
    base, base_l, _, base_g = _run(mloam, scene, n, sweeps, inits, "raw", False, graph, full)
    raw_ahead, raw_ahead_l, _, raw_ahead_g = _run(mloam, scene, n, sweeps, inits, "raw", True, graph, full)
    reuse_g = {ahead: _run(mloam, scene, n, sweeps, inits, "raw_reuse", ahead, graph, full)[3] for ahead in (False, True)}
    for kind in ("pcd", "pcd_dev"):
        for ahead in (False, True):
            got, got_l, _, got_g = _run(mloam, scene, n, sweeps, inits, kind, ahead, graph, full)
            for x, y in zip(got, base):
                _assert_same(x, y)
            ref_l, ref_g = (raw_ahead_l, raw_ahead_g) if ahead else (base_l, base_g)
            _assert_two_more(got_l, ref_l, ahead)
            # device bodies are keyed by their pointers as raw sweeps are; host bodies as raw sweeps passed through reused buffers
            want_g = ref_g if kind == "pcd_dev" else reuse_g[ahead]
            assert got_g == want_g, (kind, ahead, got_g, want_g)


@pytest.mark.parametrize("graph", [False, True])
def test_distortion_with_announced_poses(mloam, scene, graph):
    n = 2
    sweeps, inits = _frame_sweeps(scene, n)
    base, _, _, _ = _run(mloam, scene, n, sweeps, inits, "raw", False, graph, undist=True)
    _, raw_l, raw_ua, raw_g = _run(mloam, scene, n, sweeps, inits, "raw", True, graph, undist=True)
    assert raw_ua > 0
    reuse_g = _run(mloam, scene, n, sweeps, inits, "raw_reuse", True, graph, undist=True)[3]
    for kind in ("pcd", "pcd_dev"):
        got, got_l, got_ua, got_g = _run(mloam, scene, n, sweeps, inits, kind, True, graph, undist=True)
        for x, y in zip(got, base):
            _assert_same(x, y)
        want_g = raw_g if kind == "pcd_dev" else reuse_g  # host bodies: keyed as raw sweeps through reused buffers
        assert got_ua == raw_ua and got_g == want_g, (kind, got_ua, raw_ua, got_g, want_g)
        _assert_two_more(got_l, raw_l, True)


@pytest.mark.parametrize("ahead", [False, True])
def test_other_byte_sizes_replay_the_same_graphs(mloam, scene, ahead):
    """The replay pass reads the same sweeps rewritten with two spaces between tokens: larger bodies, the same points (%.9g names its
    float) — no graph is captured beyond the raw run's, and the results stay bit-identical."""
    n = 3
    sweeps, inits = _frame_sweeps(scene, n, prec=9)
    other, _ = _frame_sweeps(scene, n, prec=9, sep="  ")
    assert all(np.array_equal(o["raw"].view(np.uint32), s["raw"].view(np.uint32)) for o, s in zip(other, sweeps))
    assert all(o["bodies"][l][0].size != s["bodies"][l][0].size for o, s in zip(other, sweeps) for l in range(n))
    base, _, _, _ = _run(mloam, scene, n, sweeps, inits, "raw", ahead, True)
    _, _, _, raw_g = _run(mloam, scene, n, sweeps, inits, "raw_reuse", ahead, True)
    got, _, _, got_g = _run(mloam, scene, n, sweeps, inits, "pcd", ahead, True, second=other)  # host bytes: the caller's pointers are not keyed
    for x, y in zip(got, base):
        _assert_same(x, y)
    assert got_g == raw_g, (got_g, raw_g)


@pytest.mark.parametrize("graph", [False, True])
def test_bad_body_in_the_lookahead(mloam, scene, graph):
    """A refused body decoded in the look-ahead fails the call that takes it, which commits nothing; the next good frame is unchanged."""
    n = 3
    sweeps, inits = _frame_sweeps(scene, n, count=3)
    base, _, _, _ = _run(mloam, scene, n, sweeps, inits, "raw", False, graph)
    bad = dict(sweeps[1])
    body = bytearray(bad["bodies"][1][0].tobytes())
    k = body.index(b"\n", len(body) // 2) + 1
    body[k:k + 1] = b"x"  # a bad first token on a line half-way through LiDAR 1's body
    bad["bodies"] = list(bad["bodies"])
    bad["bodies"][1] = (np.frombuffer(bytes(body), np.uint8),) + tuple(bad["bodies"][1][1:])
    p = mloam.default_params()
    p.n_scans = n * RINGS
    p.max_inner = 1 if graph else 30
    cx = mloam.Context(0, p)
    try:
        _setup(cx, n, sweeps[0], False, False)
        sm, cm = scene["surf_map"], scene["corner_map"]
        for _ in range(2 if graph else 1):
            cx.frame_set_next_pcd(bad["bodies"])
            r0 = cx.frame_pcd(sweeps[0]["bodies"], sm, cm, inits[0])
            with pytest.raises(mloam.MloamError, match=f"error {E_INVALID}"):
                cx.frame_pcd(bad["bodies"], sm, cm, inits[1])
            with pytest.raises(mloam.MloamError, match=f"error {E_INVALID}"):  # the same body decoded in the call
                cx.frame_pcd(bad["bodies"], sm, cm, inits[1])
            r2 = cx.frame_pcd(sweeps[2]["bodies"], sm, cm, inits[2])
            for got, want in ((r0, base[0]), (r2, base[2])):
                assert np.array_equal(got[0], want[0]) and got[1]["lm_iterations"] == want[1]["lm_iterations"]
                assert got[1]["final_cost"] == want[1]["final_cost"]
    finally:
        cx.close()


def test_frame_pcd_error_paths(mloam, scene):
    n = 3
    sw = _frame_sweep(scene["scene"], scene["traj"][2], n, 3)
    sm, cm, init = scene["surf_map"], scene["corner_map"], scene["traj"][2]

    def rc(expect, fn, *a):
        with pytest.raises(mloam.MloamError, match=f"error {expect}"):
            fn(*a)

    cx = _ctx(mloam, n * RINGS)
    try:
        cx.set_lidars(n, sw["ext"])
        rc(E_STATE, cx.frame_pcd, sw["bodies"], sm, cm, init)  # no front end
        rc(E_STATE, cx.frame_set_next_pcd, sw["bodies"])
        rc(E_STATE, cx.front_end_pcd, sw["bodies"])
        cx.set_front_end(RINGS, HORIZON, 0.5, 0.1, True)
        rc(E_INVALID, cx.frame_pcd, sw["bodies"], sm, cm, init)  # time_field 1: PointXYZ has no timestamp
        rc(E_INVALID, cx.frame_set_next_pcd_device, [(0, 0) + tuple(b[1:]) for b in sw["bodies"]])
        cx.set_front_end(RINGS, HORIZON, 0.5, 0.1, False)
        b = list(sw["bodies"])
        for broken in [(b[0][0], 0, b[0][2], b[0][3]), (b[0][0], b[0][1], 0, (0, 0, 0)), (b[0][0], b[0][1], b[0][2], (0, 1, 9))]:
            rc(E_INVALID, cx.frame_pcd, [broken] + b[1:], sm, cm, init)
        rc(E_INVALID, cx.frame_pcd, [(b[0][0], b[0][1] + 1, b[0][2], b[0][3])] + b[1:], sm, cm, init)  # too few lines: on the device
        pose, st = cx.frame_pcd(sw["bodies"], sm, cm, init)  # the same calls pass once the bodies are right
        assert st["ran"] == 1
    finally:
        cx.close()


def test_communicator_rejected(mloam, scene):
    import torch  # noqa: F401  (torch's NCCL first, see test_keyframe_mapper.py)
    sw = _frame_sweep(scene["scene"], scene["traj"][2], 1, 3)
    cx = _ctx(mloam, RINGS)
    try:
        try:
            cx.comm_init(1, 0, mloam.Context.comm_unique_id())
        except mloam.MloamError as e:
            pytest.skip(f"no NCCL on this machine: {e}")
        cx.set_front_end(RINGS, HORIZON, 0.5, 0.1, True)  # time_field 1 too: the communicator is reported first
        for fn, a in ((cx.frame_pcd, (sw["bodies"], scene["surf_map"], scene["corner_map"], scene["traj"][2])), (cx.front_end_pcd, (sw["bodies"],)),
                      (cx.frame_set_next_pcd, (sw["bodies"],))):
            with pytest.raises(mloam.MloamError, match=f"error {E_STATE}"):
                fn(*a)
    finally:
        cx.close()

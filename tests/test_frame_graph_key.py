"""The frame graph key (pipeline.cu frame_key): which settings make a frame a new CUDA graph, and which only change what the graph's
staged inputs hold.  One scripted sequence of frames runs on a default context and on an MLOAM_DISABLE_GRAPHS=1 context.  Poses, stats,
the frame's scan, outlier and registered clouds are bit-identical; and after every call of the graph context the capture counter and the
frame's from_graph flag follow the schedule the key implies: a new key runs on the stream, its second sighting captures (and replays),
later sightings replay.

The script changes, one at a time, settings that re-key (a params field, set_extrinsic, set_lidars values and count, each stage switch,
the undistortion pose count, a gd_float evaluation frame, the raw front end, a message sweep, a PCD sweep and its POINTS, rebuild on /
off, the map gate with maps built outside the frame) and values that are staged and must replay the same graph with the new value (the initial pose, the with_ua covariances and
threshold, the outlier leaf, the undistortion poses, the gd_float threshold, the byte sizes of PCD bodies).  A frame's key also holds the half of the feature double
buffer it extracts into, which alternates from frame to frame, so each setting runs six frames: stream, capture and replay per half."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import front_end_lib as fel
import pcd_lib as pl
import synthetic as syn
import wire_lib as wl

pytestmark = pytest.mark.gpu

RINGS, HORIZON = 16, 512
STATS = ("ran", "n_surf", "n_corner", "n_surf_in", "n_corner_in", "lm_iterations", "termination", "degenerate", "final_cost")
COV_MEAS = np.diag([0.0025, 0.0025, 0.0025])


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def _ctx(mloam, graphs):
    if not graphs:
        os.environ["MLOAM_DISABLE_GRAPHS"] = "1"
    try:
        p = mloam.default_params()
        p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = RINGS, 3, 1, 0.5, HORIZON
        return mloam.Context(0, p)
    finally:
        os.environ.pop("MLOAM_DISABLE_GRAPHS", None)


def _graph_state(mloam, cx):
    edges, from_graph = C.c_int(-1), C.c_int(-1)
    assert mloam.lib().mloam_debug_pdl(cx._h, C.byref(edges), C.byref(from_graph)) == 0
    return cx.profile_get("graph_captures")[1], from_graph.value


def _ext(k):
    a = 0.3 * k + 0.1
    return [0.2 * math.cos(a), 0.2 * math.sin(a), 0.05 * k, 0.0, 0.0, math.sin(a / 4), math.cos(a / 4)]


def _ext_cov(n, scale):
    return np.stack([np.diag([1e-4 * scale] * 3 + [2e-5 * scale] * 3)] * n)


def _undist(n, k):
    h = 0.002 * (k + 1)
    return np.array([[0.02 * (k + 1), 0.01, 0.0, 0.0, 0.0, math.sin(h), math.cos(h)]] * n)


@pytest.fixture(scope="module")
def scene():
    sc = syn.make_scene()
    traj = syn.trajectory(4)
    surf_map, corner_map = syn.make_submap(sc, 60000)
    cloud, ss, se = syn.make_sweep(sc, traj[1], RINGS, HORIZON, seed=3)
    rig, rss, rse, _ = syn.make_multi_sweep(sc, traj[1], 2, RINGS, HORIZON, seed=5)
    raw = np.ascontiguousarray(fel.raw_sweep(sc, traj[1], RINGS, HORIZON, seed=7), np.float32)
    msg = wl.pack(raw, "xyzi32", height=2, row_pad=8)

    def pcd(pts, prec):  # one PointXYZ body: %.9g and %.8g lines of the same points differ in byte size only
        return [(pl.ascii_body([pts[:, 0], pts[:, 1], pts[:, 2]], prec=prec), pts.shape[0], 3, (0, 1, 2))]

    return dict(truth=traj[1], surf_map=surf_map, corner_map=corner_map, ring=(np.ascontiguousarray(cloud, np.float32), ss, se),
                rig=(np.ascontiguousarray(rig, np.float32), rss, rse), raw=raw, msg=[wl.as_arg(msg)], msg_layout=msg,
                pcd9=pcd(raw, 9), pcd8=pcd(raw, 8), pcd_short=pcd(raw[:-100], 9))


def _script(mloam, sc):
    """[(label, settings applied before the block's first frame, settings applied before its fourth, frames, sweep, rebuild)].  A new
    label is a new key; a repeated label returns to the key the label had.  sweep: one name, or the names of the first three frames
    and of the rest."""
    tiny_s, tiny_c = sc["surf_map"][:40], sc["corner_map"][:8]
    gf = [("set_params", dict(gf_method=3, gf_ratio=0.5)), ("set_gf_float", True, 1e9)]
    return [
        ("base", [], [], 6, "ring", True),
        ("params", [("set_params", dict(surf_leaf=0.45))], [], 6, "ring", True),
        ("ext a", [("set_extrinsic", _ext(1))], [], 6, "ring", True),
        ("ext b", [("set_extrinsic", _ext(2))], [], 6, "ring", True),
        ("lidars a", [("set_lidars", 1, [_ext(3)])], [], 6, "ring", True),
        ("lidars b", [("set_lidars", 1, [_ext(4)])], [], 6, "ring", True),
        ("with_ua", [("set_uncertainty", True, _ext_cov(1, 1.0), COV_MEAS, 1e30)],
         [("set_uncertainty", True, _ext_cov(1, 40.0), 2 * COV_MEAS, 0.05)], 6, "ring", True),
        ("outlier", [("set_outlier", 0.5)], [("set_outlier", 2.0)], 6, "ring", True),
        ("undistortion", [("set_distortion", True, 0.1)], [], 6, "ring", True),
        ("registered", [("set_registered", True)], [], 6, "ring", True),
        ("raw a", [("set_front_end", RINGS, HORIZON, 0.5)], [], 6, "raw", True),
        ("raw b", [("set_front_end", RINGS, HORIZON, 0.8)], [], 6, "raw", True),
        ("message", [("set_front_end_layout", [wl.layout(mloam, sc["msg_layout"], None)])], [], 6, "msg", True),
        # the bodies' byte sizes are staged: other files of the same POINTS replay the graph captured with the first ones
        ("pcd", [], [], 6, ("pcd9", "pcd8"), True),
        ("pcd points", [], [], 6, "pcd_short", True),
        ("2 lidars a", [("set_lidars", 2, [_ext(5), _ext(6)])], [], 6, "rig", True),
        ("2 lidars b", [("set_lidars", 2, [_ext(5), _ext(7)])], [], 6, "rig", True),
        # maps built outside the frame; the first host build grows the staging the host sweep shares, so it comes before the block
        ("no rebuild", [("map_build", sc["surf_map"], sc["corner_map"])], [], 6, "rig", False),
        ("gate closed", [("map_build", tiny_s, tiny_c)], [], 4, "rig", False),
        ("no rebuild", [("map_build", sc["surf_map"], sc["corner_map"])], [], 4, "rig", False),
        ("gd_float", gf, [("set_gf_float_threshold", -1e9)], 12, "rig", False),
    ]


def _apply(mloam, cx, s):
    if s[0] == "set_params":
        cx.set_params(**s[1])
    elif s[0] == "map_build":
        cx.map_build(mloam.MAP_SURF, s[1], 0.5), cx.map_build(mloam.MAP_CORNER, s[2], 0.5)
    else:
        getattr(cx, s[0])(*s[1:])


def _frame(mloam, cx, on, sc, sweep, rebuild, init, k):
    if on["set_distortion"]:
        cx.frame_undistort(_undist(2 if sweep == "rig" else 1, k))
    sm, cm = (sc["surf_map"], sc["corner_map"]) if rebuild else (None, None)
    if sweep == "raw":
        pose, st = cx.frame_raw(sc["raw"], [sc["raw"].shape[0]], sm, cm, init, rebuild_maps=rebuild)
    elif sweep == "msg":
        pose, st = cx.frame_msg(sc["msg"], sm, cm, init, rebuild_maps=rebuild)
    elif sweep.startswith("pcd"):
        pose, st = cx.frame_pcd(sc[sweep], sm, cm, init, rebuild_maps=rebuild)
    else:
        cloud, ss, se = sc[sweep]
        pose, st = cx.frame(cloud, ss, se, sm, cm, init, rebuild_maps=rebuild)
    out = [pose, [st[f] for f in STATS]]
    out += [_bits(a) for a in cx.frame_scan()]
    if on["set_outlier"]:
        out += [_bits(a) for a in cx.frame_outlier()]
    if on["set_registered"]:
        out += [_bits(cx.frame_registered(w)) for w in (mloam.REGISTERED_FULL_RES, mloam.REGISTERED_SURF, mloam.REGISTERED_CORNER)]
    return out


def test_frame_graph_key_schedule(mloam, scene):
    rng = np.random.Generator(np.random.PCG64(11))
    g, plain = _ctx(mloam, True), _ctx(mloam, False)
    on = dict(set_distortion=False, set_outlier=False, set_registered=False)  # the stages whose outputs the script reads back
    sightings, parity, gf_frames, k = {}, 0, None, 0
    try:
        for label, before, middle, n_frames, sweeps, rebuild in _script(mloam, scene):
            for i in range(n_frames):
                sweep = sweeps if isinstance(sweeps, str) else sweeps[i >= 3]
                for s in before if i == 0 else middle if i == 3 else []:
                    for cx in (g, plain):
                        _apply(mloam, cx, s)
                    on[s[0]] = True
                    if s[0] == "set_gf_float":
                        gf_frames = 0
                if gf_frames is not None:
                    gf_frames += 1
                init = syn.perturb_pose(scene["truth"], rng)  # a new pose guess every frame: staged, never in the key
                c0 = _graph_state(mloam, g)[0]
                got = _frame(mloam, g, on, scene, sweep, rebuild, init, k)
                want = _frame(mloam, plain, on, scene, sweep, rebuild, init, k)
                assert len(got) == len(want)
                for a, b in zip(got, want):
                    assert np.array_equal(np.asarray(a), np.asarray(b)), (label, i)
                key = (label, parity, gf_frames is not None and gf_frames % 10 == 0)
                sightings[key] = sightings.get(key, 0) + 1
                captures, from_graph = _graph_state(mloam, g)
                assert captures - c0 == (1 if sightings[key] == 2 else 0), (label, i, key, sightings[key])
                assert from_graph == (1 if sightings[key] >= 2 else 0), (label, i, key, sightings[key])
                parity ^= 1
                k += 1
        assert g.launch_count() == plain.launch_count()
        assert g.profile_get("graph_capture_failures")[1] == 0
    finally:
        g.close(), plain.close()

"""Programmatic dependent launch along scan2map's GN chain (launch_chain, MLOAM_PDL): it changes when the chain's kernels start, never
what they compute.  Frames with and without it give bit-identical poses, solve statistics, H, eigenvalues, match counts and pose
covariances on the stream path, the graph capture and the replay, with and without the sweep look-ahead, over a keyframe cadence; and
the captured frame graph really has programmatic edges and really ran."""
import ctypes as C
import os

import numpy as np
import pytest

import bench
import synthetic as syn
import uncertainty_lib as ua

pytestmark = pytest.mark.gpu

STATS = ("ran", "n_surf", "n_corner", "n_surf_in", "n_corner_in", "lm_iterations", "termination", "degenerate", "final_cost")
N_FRAMES, STEPS, KEYFRAME_EVERY = 3, 9, 3  # every (frame, rebuild) pair is seen three times: stream path, capture, replay
_WL = {}


def _workload(name):
    if name not in _WL:
        _WL[name] = bench.make_workload(syn, bench.CONFIGS[name], 1, 0, N_FRAMES)
    return _WL[name]


def _context(mloam, name, pdl):
    cfg = bench.CONFIGS[name]
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = cfg["rings"] * cfg["lidars"], cfg["gn_iters"], 1, 0.0, cfg["horizon"]
    os.environ["MLOAM_PDL"] = pdl
    try:
        cx = mloam.Context(0, p)
    finally:
        os.environ.pop("MLOAM_PDL")
    if cfg["lidars"] > 1:
        cx.set_lidars(cfg["lidars"], _workload(name)["frames"][0]["groups"][0]["ext"])
    return cx


def _pdl_state(mloam, cx):
    edges, from_graph = C.c_int(-1), C.c_int(-1)
    assert mloam.lib().mloam_debug_pdl(cx._h, C.byref(edges), C.byref(from_graph)) == 0
    return edges.value, from_graph.value


def _run(mloam, name, pdl, lookahead, with_ua=False):
    """STEPS frames cycling over the workload's frames, the submap rebuilt every KEYFRAME_EVERY-th step."""
    wl = _workload(name)
    cx = _context(mloam, name, pdl)
    out = []
    try:
        if with_ua:
            cx.set_uncertainty(True, ua.ext_covariances(bench.CONFIGS[name]["lidars"], seed=5, scale=1.6), np.diag([0.0025] * 3), 1e30)
        for k in range(STEPS):
            g = wl["frames"][k % N_FRAMES]["groups"][0]
            if lookahead:
                gn = wl["frames"][(k + 1) % N_FRAMES]["groups"][0]
                cx.frame_set_next(gn["cloud"], gn["ss"], gn["se"])
            pose, st = cx.frame(g["cloud"], g["ss"], g["se"], wl["surf_map"], wl["corner_map"], wl["frames"][k % N_FRAMES]["init"],
                                k % KEYFRAME_EVERY == 0)
            out.append((pose, st, cx.pose_covariance(), _pdl_state(mloam, cx)))
    finally:
        cx.close()
    return out


def _assert_same(ref, res):
    for (pa, sa, ca, _), (pb, sb, cb, _) in zip(ref, res):
        assert sa["ran"] == 1 and sa["n_surf"] > 1000
        assert np.array_equal(pa, pb)
        for k in STATS:
            assert sa[k] == sb[k], k
        assert np.array_equal(np.asarray(sa["H"]), np.asarray(sb["H"]))
        assert np.array_equal(np.asarray(sa["eig"]), np.asarray(sb["eig"]))
        assert np.array_equal(ca, cb)


@pytest.mark.parametrize("lookahead", [False, True], ids=["no_lookahead", "lookahead"])
@pytest.mark.parametrize("name", ["C2", "C4"])
def test_pdl_frames_bit_identical(mloam, name, lookahead):
    """C2 and C4 on one GPU at full size: MLOAM_PDL=0 (ordinary launches) against the default."""
    ref = _run(mloam, name, "0", lookahead)
    res = _run(mloam, name, "1", lookahead)
    _assert_same(ref, res)
    gn = bench.CONFIGS[name]["gn_iters"]
    # the first sighting of a frame graph's key runs on the stream path, the later ones from the graph; the key (look-ahead half,
    # parity) is the same for both settings
    assert [r[3][1] for r in res] == [r[3][1] for r in ref]
    assert res[0][3][1] == 0 and res[-2][3][1] == 1 and res[-1][3][1] == 1
    edges = res[-1][3][0]
    print(f"{name} lookahead={lookahead}: {edges} programmatic edges in the last captured frame graph")
    # k_linearize -> k_match_knn and k_match_knn -> k_linearize on the main stream, at every boundary between GN iterations
    assert edges >= 2 * (gn - 1), edges
    assert ref[-1][3][0] == 0


def test_pdl_with_ua_bit_identical(mloam):
    """C2 with the uncertainty-aware mapper: the per-feature weights and k_pose_cov after the last, two-pass k_linearize."""
    ref = _run(mloam, "C2", "0", True, with_ua=True)
    res = _run(mloam, "C2", "1", True, with_ua=True)
    _assert_same(ref, res)
    assert np.abs(res[-1][2]).max() > 0  # the covariance was computed

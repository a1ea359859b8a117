"""The phase stamps of k_linearize's pass 0 (MLOAM_LIN_TRACE=1, read by tools/trace_replay.py --phases): a traced frame computes
what an untraced one does, bit for bit, and every evaluation at x of the solve leaves one slot whose stamps are in phase order."""
import ctypes as C
import os

import numpy as np
import pytest

import bench
import synthetic as syn

pytestmark = pytest.mark.gpu

LIN_TRACE_BLOCK, LIN_TRACE_SLOT, LIN_TRACE_SLOTS = 64, 64 * 64, 16  # solve_kernels.cu


def _context(mloam, p, trace):
    if trace:
        os.environ["MLOAM_LIN_TRACE"] = "1"
    try:
        return mloam.Context(0, p)
    finally:
        os.environ.pop("MLOAM_LIN_TRACE", None)


def _read(mloam, cx):
    buf = np.zeros(LIN_TRACE_SLOTS * LIN_TRACE_SLOT, dtype=np.uint64)
    n = C.c_int(0)
    assert mloam.lib().mloam_debug_lin_trace(cx._h, buf.ctypes.data_as(C.c_void_p), buf.size, C.byref(n)) == 0
    return buf.reshape(LIN_TRACE_SLOTS, 64, LIN_TRACE_BLOCK).astype(np.int64), n.value


def _check_slot(slot):
    blk = slot[slot[:, 0] != 0]
    assert len(blk) > 0
    warps = blk[:, :32].reshape(-1, 4)
    t0 = warps[:, 0].min()
    loop_end = (warps[:, 0] + warps[:, 1]).max()
    assert (warps[:, 2] <= warps[:, 3]).all()  # fit cycles are part of the feature loop's
    assert t0 <= loop_end <= blk[:, 32].max()  # feature loop, then the block partials
    assert (blk[:, 32] <= blk[:, 33]).all()  # each block takes its ticket after writing its partial
    last = blk[blk[:, 34] != 0]
    assert len(last) == 1  # one block ran the tail
    assert blk[:, 33].max() <= last[0, 34] <= last[0, 35]


def test_traced_frames_are_bit_identical_and_ordered(mloam):
    """C2 (64 x 2048 sweep, 1M-point keyframe submap, 10 GN iterations, speculative schedule): stream path, capture, replay."""
    cfg = bench.CONFIGS["C2"]
    wl = bench.make_workload(syn, cfg, 1, 0, 1)
    fr = wl["frames"][0]
    g = fr["groups"][0]
    p = mloam.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell, p.max_ring_points = cfg["rings"], cfg["gn_iters"], 1, 0.0, cfg["horizon"]
    res = []
    for trace in (False, True):
        cx = _context(mloam, p, trace)
        out = []
        for rebuild in (True, False, False, False):
            out.append(cx.frame(g["cloud"], g["ss"], g["se"], wl["surf_map"], wl["corner_map"], fr["init"], rebuild))
            if trace:
                slots, n = _read(mloam, cx)
                assert n == cfg["gn_iters"]  # one evaluation at x per GN iteration
                for s in range(n):
                    _check_slot(slots[s])
        cx.close()
        res.append(out)
    for (pa, sa), (pb, sb) in zip(*res):
        assert sa["ran"] == 1 and sa["n_surf"] > 1000
        assert np.array_equal(pa, pb)
        for k in ("ran", "n_surf", "n_corner", "lm_iterations", "termination", "degenerate", "final_cost"):
            assert sa[k] == sb[k], k
        assert np.array_equal(np.asarray(sa["H"]), np.asarray(sb["H"]))

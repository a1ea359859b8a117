#!/usr/bin/env python
"""Diagnosis tool (not a benchmark): event-timed k_match_knn launches of the C2 surf features against the 900k-point
surf submap, blind search, for a given cell edge / staging threshold (env MLOAM_KNN_TMA_MIN).
usage: knn_micro.py [cell ...]"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import synthetic as syn  # noqa: E402


def main():
    cells = [float(a) for a in sys.argv[1:]] or [0.25]
    m = bench.load_mloam()
    p = m.default_params()
    p.n_scans = 64
    ctx = m.Context(0, p)
    surf_map, corner_map, frames, _ = bench.make_workload(syn, 1, 0, 1)
    f = frames[0]
    feats = ctx.extract_features(f["cloud"], f["ss"], f["se"])
    surf = ctx.voxel_downsample(feats["surf_points_less_flat"], 0.4, True)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    pose = np.asarray(f["init"], np.float64)
    for cell in cells:
        ctx.profile(True)
        ctx.profile_reset()
        for _ in range(5):
            ctx.map_build(1, surf_map, cell)
        ms_b, kb = ctx.profile_get("map_build")
        full = surf
        for n_sub in (32, 256, 1184, 2368, 4736):
            surf = full[:n_sub]
            ctx.profile_reset()
            for _ in range(10):
                ctx.match_from_map(1, "s", surf, pose, want_nn=False)
            ms, k = ctx.profile_get("match")
            print(f"  cell={cell:5.3f} {n_sub:5d} queries: k_match_knn {1e3 * ms / max(k, 1):7.1f} us")
        surf = full
        for warm in (True, False):
            ctx.profile_reset()
            for _ in range(10):
                if not warm:
                    flush.fill_(1)
                    torch.cuda.synchronize()
                valid, _, _ = ctx.match_from_map(1, "s", surf, pose, want_nn=False)
            ms, k = ctx.profile_get("match")
            fms, fk = ctx.profile_get("fit")
            print(f"tma_min={os.environ.get('MLOAM_KNN_TMA_MIN', 'default'):>10s} cell={cell:5.3f} {'warm L2' if warm else 'flushed'}: "
                  f"k_match_knn {1e3 * ms / max(k, 1):7.1f} us  fit {1e3 * fms / max(fk, 1):5.1f} us  build {1e3 * ms_b / max(kb, 1):6.1f} us  "
                  f"features {surf.shape[0]} matched {int(valid.sum())}")
        ctx.profile(False)
        if os.environ.get("MLOAM_KNN_TRACE") == "1":
            import ctypes as C
            valid, _, _ = ctx.match_from_map(1, "s", surf, pose, want_nn=False)
            tr = np.zeros((surf.shape[0], 4), np.uint32)
            rc = m.lib().mloam_debug_knn_trace(ctx._h, tr.ctypes.data_as(C.c_void_p), surf.shape[0])
            cyc = tr[:, 0] & 0x3fffffff
            order = np.argsort(-cyc.astype(np.int64))
            print("trace rc", rc, "cycles: median", int(np.median(cyc)), "p90", int(np.percentile(cyc, 90)), "p99", int(np.percentile(cyc, 99)), "max", int(cyc.max()))
            for q in order[:12]:
                print(f"  q={q:5d} cycles={int(cyc[q]):7d} path={int(tr[q,0]>>30)} ring1_cyc={int(tr[q,1]):6d} ball_cyc={int(tr[q,2]):6d} ring1_pts={int(tr[q,3]>>20)} ball_pts={int((tr[q,3]>>8)&0xfff)} ball_steps={int(tr[q,3]&0xff)} valid={bool(valid[q])}")
            np.save(os.path.join(ROOT, "gpurun_out", "knn_trace.npy"), tr)


def seeded_trace():
    """Trace of the LAST k_match_knn launch of a 10-iteration scan2MapOptimization (a seeded launch: keep / ball / blind mix)."""
    import ctypes as C
    m = bench.load_mloam()
    p = m.default_params()
    p.n_scans, p.max_outer, p.max_inner, p.map_cell = 64, 10, 1, 0.25
    ctx = m.Context(0, p)
    surf_map, corner_map, frames, _ = bench.make_workload(syn, 1, 0, 1)
    f = frames[0]
    feats = ctx.extract_features(f["cloud"], f["ss"], f["se"])
    surf = ctx.voxel_downsample(feats["surf_points_less_flat"], 0.4, True)
    corner = ctx.voxel_downsample(feats["corner_points_less_sharp"], 0.2, True)
    ctx.map_build(1, surf_map, 0.25)
    ctx.map_build(0, corner_map, 0.25)
    ctx.profile(True)
    for _ in range(3):
        ctx.profile_reset()
        pose, st = ctx.scan2map(surf, corner, np.asarray(f["init"], np.float64))
    ms, k = ctx.profile_get("match")
    print(f"scan2map: k_match_knn {1e3 * ms / max(k, 1):7.1f} us avg over {k} launches; features corner {corner.shape[0]} surf {surf.shape[0]}")
    n = corner.shape[0] + surf.shape[0]
    nw = 8 * 4 * torch.cuda.get_device_properties(0).multi_processor_count
    full = np.zeros((n + 1 + nw, 4), np.uint32)
    rc = m.lib().mloam_debug_knn_trace(ctx._h, full.ctypes.data_as(C.c_void_p), n + 1 + nw)
    tr = full[:n]
    tl = full[n + 1:].copy().view(np.uint64).reshape(-1, 2)
    tl = tl[tl[:, 0] > 0]
    t0 = tl[:, 0].min()
    ent, ext = (tl[:, 0] - t0).astype(np.int64), (tl[:, 1] - t0).astype(np.int64)
    print(f"  timeline over {len(tl)} warps [ns]: enter median {int(np.median(ent))} max {int(ent.max())}; exit median {int(np.median(ext))} p90 {int(np.percentile(ext, 90))} max {int(ext.max())}; "
          f"busy median {int(np.median(ext - ent))} max {int((ext - ent).max())}")
    cyc = (tr[:, 0] & 0x3fffffff).astype(np.int64)
    path = tr[:, 0] >> 30
    for pth, name in enumerate(("keep matched", "keep rejected", "ball", "blind")):
        sel = path == pth
        if sel.any():
            print(f"  {name:14s} n={int(sel.sum()):6d} cycles median {int(np.median(cyc[sel])):6d} p90 {int(np.percentile(cyc[sel], 90)):6d} max {int(cyc[sel].max()):6d} sum {int(cyc[sel].sum()):10d}")


if __name__ == "__main__":
    if os.environ.get("KNN_MICRO_SEEDED") == "1":
        seeded_trace()
        sys.exit(0)
    main()

"""Per-frame cost of taking the dataset nodes' ASCII PCD files (%.8g, as pcl::io::savePCDFileASCII writes them) into the frame path:

  host       PCL's read on the host (lines, tokens, istringstream >> float of x / y / z, nothing else checked) + mloam_frame_raw
  pcd        mloam_frame_pcd: the host bodies copied up and decoded on the device (two launches for the rig) inside the frame
  pcd_ahead  mloam_frame_pcd with the next frame's bodies announced (mloam_frame_set_next_pcd): the decode runs in the look-ahead
  decode     mloam_pcd_decode_device alone on bodies already in device memory (CUDA events around the call)

for an Oxford-shaped rig (2 LiDARs x 32 rings x 1800 columns) and a 4 x 64 x 2048 rig, with a 200k-point submap rebuilt every frame and
one LM iteration per GN iteration (the frames replay captured graphs).  Prints the card and its power limit with the numbers.  Run from
the repository root after build():  python tools/bench_pcd.py [--frames N]
"""
import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import front_end_lib as fel  # noqa: E402
import pcd_lib as pl  # noqa: E402
import synthetic as syn  # noqa: E402


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def _exts(n):
    out = []
    for l in range(n):
        a = 2 * math.pi * l / n
        out.append([0.3 * math.cos(a), 0.3 * math.sin(a), 0.05 * l, 0.0, 0.0, math.sin(a / 4), math.cos(a / 4)])
    return np.array(out, np.float64)


def _pcl_read(data, h):
    body = data[h["body"]:]
    out = np.zeros((h["points"], 4), np.float32)
    idx = np.array([h["ix"], h["iy"], h["iz"]], np.int32)
    n = pl.lib().pcd_pcl_read(C.c_char_p(body), C.c_size_t(len(body)), h["points"], C.c_void_p(idx.ctypes.data), C.c_void_p(out.ctypes.data))
    assert n == h["points"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
    args = ap.parse_args()
    import __graft_entry__ as g
    import torch

    m = g._load()
    print(json.dumps({"card": _card()}))
    scene = syn.make_scene()
    traj = syn.trajectory(4)
    sm, cm = syn.make_submap(scene, 200000)
    for name, (nl, rings, cols) in {"oxford_2x32x1800": (2, 32, 1800), "rig_4x64x2048": (4, 64, 2048)}.items():
        ext = _exts(nl)
        frames = []
        for k in range(2):
            files = []
            for l in range(nl):
                raw = fel.raw_sweep(scene, traj[1 + k], rings, cols, 10 * k + l, ext=ext[l])
                data = pl.fields_header(pl.XYZ, raw.shape[0]) + pl.ascii_body([raw[:, 0], raw[:, 1], raw[:, 2]], prec=8)
                files.append((data, pl.header(data)))
            frames.append(dict(files=files, bodies=[(np.frombuffer(d[h["body"]:], np.uint8), h["points"], h["tokens"], (h["ix"], h["iy"], h["iz"]))
                                                    for d, h in files], counts=np.array([h["points"] for _, h in files], np.int32)))
        init = traj[1]
        p = m.default_params()
        p.n_scans = nl * rings
        p.max_inner = 1
        cx = m.Context(0, p)
        try:
            cx.set_lidars(nl, ext)
            cx.set_front_end(rings, cols, 0.5, 0.1, False)
            res = {"rig": name, "body_bytes": int(sum(b[0].nbytes for b in frames[0]["bodies"])), "points": int(frames[0]["counts"].sum())}

            def host(k):
                raw = np.concatenate([_pcl_read(d, h) for d, h in frames[k]["files"]])
                return cx.frame_raw(raw, frames[k]["counts"], sm, cm, init)

            def pcd(k):
                return cx.frame_pcd(frames[k]["bodies"], sm, cm, init)

            def pcd_ahead(k):
                cx.frame_set_next_pcd(frames[k ^ 1]["bodies"])
                return cx.frame_pcd(frames[k]["bodies"], sm, cm, init)

            ref = [host(k)[0] for k in range(2)]
            for key, fn in (("host_pcl_read+frame_raw_ms", host), ("frame_pcd_ms", pcd), ("frame_pcd_lookahead_ms", pcd_ahead)):
                for k in range(4):
                    fn(k & 1)
                t = []
                for i in range(args.frames):
                    t0 = time.perf_counter()
                    pose, _ = fn(i & 1)
                    t.append((time.perf_counter() - t0) * 1e3)
                    assert np.array_equal(pose, ref[i & 1])
                cx.frame_set_next_pcd(None)
                res[key] = round(float(np.median(t)), 3)
            bodies = frames[0]["bodies"]
            dbuf = [torch.from_numpy(b[0].copy()).cuda() for b in bodies]
            out = torch.empty((int(frames[0]["counts"].sum()), 4), dtype=torch.float32, device="cuda")
            darg = [(t.data_ptr(), t.numel(), b[1], b[2], b[3]) for t, b in zip(dbuf, bodies)]
            cx.pcd_decode_device(darg, out.data_ptr())
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t = []
            for _ in range(args.frames):
                torch.cuda.synchronize()
                ev0.record()
                cx.pcd_decode_device(darg, out.data_ptr())
                ev1.record()
                ev1.synchronize()
                t.append(ev0.elapsed_time(ev1))
            res["decode_device_ms"] = round(float(np.median(t)), 3)
            print(json.dumps(res))
        finally:
            cx.close()


if __name__ == "__main__":
    main()

"""2-GPU check of the 12-DoF online-calibration step (launch with torch.distributed.run, 2 ranks):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29541 tests/multi_gpu_calib_check.py

Rank 0 holds the reference LiDAR's features (1x6 rows on pose_i), rank 1 the second LiDAR's (1x6 rows on its extrinsic); both
blocks' packed normal equations and the cost (57 doubles) are summed with one ncclAllReduce per LM evaluation inside mloam_calib_frame.  Both ranks must end
with the same [pose_i | ext_cal], equal (<= 1e-4 m / rad) to the oracle's joint solve."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)


def main():
    import torch
    import torch.distributed as dist

    import oracle_lib as orc
    import synthetic as syn
    from bench import load_mloam

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    assert world == 2
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    m = load_mloam()
    ctx = m.Context(local, m.default_params())
    uid = [m.Context.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    ctx.comm_init(world, rank, uid[0])
    cs = syn.make_calib_case(syn.make_scene(), orc.extract_cloud, orc.voxel_grid, 16, 1024, 100000)
    ctx.map_build(0, cs["corner_map"], 0.25)
    ctx.map_build(1, cs["surf_map"], 0.25)
    ref = (cs["surf_ref"], cs["corner_ref"]) if rank == 0 else (None, None)
    cal = (cs["surf_cal"], cs["corner_cal"]) if rank == 1 else (None, None)
    pi, ec, st = ctx.calib_frame(ref[0], ref[1], cal[0], cal[1], cs["pivot"], cs["pose_i_init"], cs["ext_ref"], cs["ext_cal_init"], 10, 1)
    res = [None] * world
    dist.all_gather_object(res, (pi.tolist(), ec.tolist(), st["n_surf"]))
    ok = True
    if rank == 0:
        if res[0][:2] != res[1][:2]:
            print("FAIL: the ranks ended with different states")
            ok = False
        rpi, rec, rst = orc.calib_frame(cs["surf_map"], cs["corner_map"], cs["surf_ref"], cs["corner_ref"], cs["surf_cal"], cs["corner_cal"], cs["pivot"],
                                        cs["pose_i_init"], cs["ext_ref"], cs["ext_cal_init"], 10, 1)
        (dtp, drp), (dte, dre) = syn.pose_err(pi, rpi), syn.pose_err(ec, rec)
        print(f"calibration x2 GPUs [nccl]: pose_i vs oracle dt={dtp:.3e} dr={drp:.3e}; ext_cal dt={dte:.3e} dr={dre:.3e}; rows {st['n_surf']} vs {rst['rows']}; "
              f"ext rotation error vs truth {syn.pose_err(cs['ext_cal_init'], cs['ext_cal'])[1]:.4f} -> {syn.pose_err(ec, cs['ext_cal'])[1]:.4f} rad")
        if max(dtp, drp, dte, dre) > 1e-4 or st["n_surf"] != rst["rows"]:
            print("FAIL: parity")
            ok = False
    flag = [ok]
    dist.broadcast_object_list(flag, src=0)
    ctx.close()
    dist.destroy_process_group()
    if rank == 0:
        print("MULTI_GPU_CALIB_CHECK", "OK" if flag[0] else "FAILED")
    sys.exit(0 if flag[0] else 1)


if __name__ == "__main__":
    main()

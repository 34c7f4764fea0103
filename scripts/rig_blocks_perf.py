"""Cost of rig calibration on a PREC_BLOCKS context (DESIGN.md "Rig calibration on block-sparse voxel BA").

Workloads: rig_blocks_ref.rig_corridor (bases along a corridor, 4 LiDARs, every plane seen by the slots of the bases
within +-4 of its centre, LiDAR 0 fixed) at 2 000 slots (500 x 4), where the blocks rig runs alternating with the dense
tensor and fp64 rigs on the same scene, and at 20 000 slots (5 000 x 4), where the dense rig does not fit.

Per size and call: ms per LM iteration (host clock around rig_damping_iter, which ends in a device synchronise;
force_hess on and the convergence exit off, so every iteration evaluates), several runs; the split from balm_timings
per iteration (ms_stats + ms_obs: the sweep, ms_syrk: the slot blocks, ms_assemble: factors, priors and the rig
reduction, ms_solve: the rig solve); rig_block_structure's pairs, L blocks, levels and bytes. Then, in a separate
torch.profiler run of rig_evaluate, the two reduction kernels' device time.

    python scripts/rig_blocks_perf.py [--runs 3] [--iters 5] [--sizes 500,5000] [--out FILE]

Prints the card's name and power limit, then one JSON line per record; --out FILE also writes them there.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import balm_b200  # noqa: E402
import rig_blocks_ref as rb  # noqa: E402
from balm_b200 import _lib as L  # noqa: E402

LM = dict(rel_tol=-1.0, force_hess=True, min_planes_per_pose=0, gauge_mode=2)
PRECS = {"blocks": L.PREC_BLOCKS, "tensor": L.PREC_TENSOR, "fp64": L.PREC_FP64}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def context(sc, prec):
    c = balm_b200.Context(sc["n_poses"], 0, PRECS[prec])
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
    if prec == "blocks":
        c.set_block_rig(sc["base_of"], sc["lidar_of"])
    else:
        c.set_rig(sc["base_of"], sc["lidar_of"])
    return c


def timed(c, sc, iters):
    c.reset_counters()
    t0 = time.perf_counter()
    tr = c.rig_damping_iter(sc["base_init"], sc["ext_init"], max_iter=iters, **LM)[2]
    ms = (time.perf_counter() - t0) * 1e3
    tm = c.timings()
    it = len(tr)
    return dict(ms_per_iter=round(ms / it, 3), ms_sweep=round((tm["ms_stats"] + tm["ms_obs"]) / it, 4),
                ms_blocks=round(tm["ms_syrk"] / it, 4), ms_assemble_and_reduce=round(tm["ms_assemble"] / it, 4),
                ms_solve=round(tm["ms_solve"] / it, 4), ms_residual=round(tm["ms_residual"] / it, 4))


def profile(c, sc, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    c.rig_evaluate(sc["base_init"], sc["ext_init"])
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(reps):
            c.rig_evaluate(sc["base_init"], sc["ext_init"])
    out = {}
    for e in p.key_averages():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time_total > 0:
            out[e.key] = out.get(e.key, 0.0) + e.device_time_total / 1000.0
    return {k: round(v / reps, 4) for k, v in sorted(out.items(), key=lambda kv: -kv[1])}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--sizes", default="500,5000", help="base poses per run (4 LiDARs each)")
    ap.add_argument("--profile_reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    gpu = card()
    print("card:", gpu, flush=True)
    with open(a.out if a.out else os.devnull, "w") as f:
        def emit(rec):
            line = json.dumps(dict(card=gpu, **rec))
            print(line, flush=True)
            f.write(line + "\n")

        for B in (int(x) for x in a.sizes.split(",")):
            sc = rb.rig_corridor(B, 4, w=4, seed=3)
            name = f"rig corridor {4 * B} slots ({B} x 4)"
            precs = ["blocks", "tensor", "fp64"] if B <= 500 else ["blocks"]
            ctxs = {p: context(sc, p) for p in precs}
            for p in precs:
                ctxs[p].rig_damping_iter(sc["base_init"], sc["ext_init"], max_iter=2, **LM)  # warm-up of every shape
            for r in range(a.runs):
                for p in precs:
                    emit(dict(workload=name, prec=p, run=r, **timed(ctxs[p], sc, a.iters)))
            blk = ctxs["blocks"]
            emit(dict(workload=name, structure=blk.rig_block_structure(), slot_structure=blk.block_structure()))
            kt = profile(blk, sc, a.profile_reps)
            emit(dict(workload=name, profile="rig_evaluate kernels (ms per call)",
                      reduction_ms={k: v for k, v in kt.items() if "rig_" in k and "blocks_kernel" in k},
                      all_kernels_ms=kt))
            for c in ctxs.values():
                c.close()


if __name__ == "__main__":
    main()

"""Cost of the point-noise covariance on blocks contexts (DESIGN.md "Point-noise covariance on blocks contexts").

Workloads, one call each:
  rig2k    rig_blocks_ref.rig_corridor(500, 4) with every base fixed (LiDAR-to-INS): 2 000 slots, the four
           extrinsics' joint Sigma
           (balm_rig_block_point_covariance), next to the dense fp64 rig's balm_rig_covariance on the same scene
  rig20k   rig_corridor(5000, 4): 20 000 slots, the same call (no dense rig fits)
  marg20k  block_hessian_ref.corridor(20000) over 100 m with fix clusters: every pose's marginal on a 20 000-pose
           blocks context, one call
Per workload: wall ms per call (host clock around the call, which ends in a device synchronise; the variants of a size
alternate, median of --runs), and in a separate torch.profiler run each kernel's device time.

    python scripts/block_point_covariance_perf.py [--runs 3] [--only rig2k,rig20k,marg20k] [--out FILE]

Prints the card's name and power limit, then one JSON line per record; --out FILE also writes them there.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import balm_b200  # noqa: E402
import block_hessian_ref as bref  # noqa: E402
import rig_blocks_ref as rb  # noqa: E402
from balm_b200 import _lib as L  # noqa: E402

PN = 0.01


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def context(sc, prec):
    c = balm_b200.Context(sc["n_poses"], 0, prec)
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc.get("fix10"))
    return c


def workloads(only):
    out = {}
    for name, B in (("rig2k", 500), ("rig20k", 5000)):
        if name not in only:
            continue
        S = rb.rig_corridor(B, 4)
        ctx = context(S, L.PREC_BLOCKS)
        # LiDAR-to-INS (every base fixed): over a drive this long with free bases H_rig fails the 1e-11 pivot rule
        fixed = dict(fixed_bases=range(B), fixed_lidars=())
        ctx.set_block_rig(S["base_of"], S["lidar_of"], **fixed)
        sel = [0, 1, 2, 3]
        # at the LM optimum: away from it H_rig can be indefinite
        b, e, _ = ctx.rig_damping_iter(S["base12"], S["ext12"], max_iter=5, gauge_mode=2, min_planes_per_pose=0)
        calls = {"blocks": lambda ctx=ctx, b=b, e=e, sel=sel: ctx.rig_block_point_covariance(b, e, sel, point_noise=PN,
                                                                                               anchor=-1)}
        if B == 500:
            dense = context(S, L.PREC_FP64)
            dense.set_rig(S["base_of"], S["lidar_of"], **fixed)
            calls["dense_fp64"] = lambda dense=dense, b=b, e=e: dense.rig_covariance(b, e, point_noise=PN, anchor=-1,
                                                                                     want_raw=False)
        out[name] = (ctx, calls)
    if "marg20k" in only:
        bref.min = lambda a, b: 100.0 / 20000  # a 100 m drive: over 1 km H fails the 1e-11 pivot rule
        sc = bref.corridor(20000, w=8, planes_per_pose=30, seed=7, with_fix=True)
        del bref.min
        ctx = context(sc, L.PREC_BLOCKS)
        x, sel = sc["poses_gt"], np.arange(20000)
        out["marg20k"] = (ctx, {"blocks": lambda: ctx.block_point_covariance(x, sel, point_noise=PN, anchor=-1,
                                                                              include_fix=True, joint=False)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--only", default="rig2k,rig20k,marg20k")
    ap.add_argument("--out")
    a = ap.parse_args()
    recs = []

    def emit(r):
        print(json.dumps(r), flush=True)
        recs.append(r)

    print("card:", card(), flush=True)
    wl = workloads(a.only.split(","))
    for name, (ctx, calls) in wl.items():
        st = ctx.block_structure()
        for f in calls.values():  # warm-up: module loads, first allocations
            f()
        times = {k: [] for k in calls}
        for _ in range(a.runs):
            for k, f in calls.items():
                t0 = time.perf_counter()
                f()
                times[k].append(1e3 * (time.perf_counter() - t0))
        for k, ts in times.items():
            emit(dict(workload=name, variant=k, ms_median=float(np.median(ts)), ms=[round(t, 2) for t in ts],
                      slot_pairs=st["pairs"], l_blocks=st["l_blocks"], levels=st["levels"]))
    import torch
    from torch.profiler import ProfilerActivity, profile
    for name, (ctx, calls) in wl.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            calls["blocks"]()
            torch.cuda.synchronize()
        per = {}
        for e in prof.key_averages():
            if e.device_time_total > 0:
                per[e.key[:80]] = (round(e.device_time_total / 1e3, 3), e.count)
        top = sorted(per.items(), key=lambda kv: -kv[1][0])[:14]
        emit(dict(workload=name, profile_ms={k: v[0] for k, v in top}, launches={k: v[1] for k, v in top}))
    if a.out:
        with open(a.out, "w") as f:
            for r in recs:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()

"""Absolute pose priors (balm_set_pose_priors): what a GNSS position prior on every 10th pose adds to an LM iteration,
against no priors on the same handle and factors. Workloads are scripts/robust_factors_perf.py's:

  pyramid  PoseGraph, HBA-shaped window factors
  chain    PoseGraph, laps of a loop with odometry and a closure to the previous lap every 25 poses
  corridor PREC_BLOCKS voxel corridor with odometry and a loop closure every 500 poses

"no priors" and "priors" alternate inside every run on one handle (set_pose_priors / set_pose_priors([])); wall times
are host clocks around synchronised work (force_hess, so every iteration evaluates). A separate profiled run gives
the device time of the prior kernels.

  python scripts/pose_priors_perf.py [--pg-sizes 4541 20000 50000] [--block-sizes 1000 4541 20000] [--runs 3]
                                     [--out FILE]

Prints one JSON line per measurement with the card's name and power limit; --out FILE also writes them there.
"""
import argparse
import json
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]
import balm_b200  # noqa: E402
import block_factors_perf as bfp  # noqa: E402
import robust_factors_perf as rfp  # noqa: E402


def gnss(x, every=10, sigma=0.05, point_noise=0.01):
    """a position prior at every `every`-th pose of x, 1.2 m lever arm, information in the voxel cost's units"""
    idx = np.arange(0, len(x), every)
    lever = np.array([0.0, 0.0, 1.2])
    pos = np.array([x[i, :9].reshape(3, 3).T @ lever + x[i, 9:] for i in idx])
    return balm_b200.position_priors(idx, pos, 2 * point_noise ** 2 / sigma ** 2 * np.eye(3), lever_arm=lever)


def profiled(h, x, iters):
    """device ms per iteration of the prior kernels in a profiled run"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rfp.lm(h, x, iters, rel_tol=-1, force_hess=True)
    out = {}
    for e in prof.events():
        if e.device_type.name != "CUDA" or "prior_" not in e.name:
            continue
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        key = re.search(r"prior_\w+", e.name).group(0)
        out[key] = out.get(key, 0.0) + us / 1e3 / iters
    return out


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--pg-sizes", type=int, nargs="+", default=[4541, 20000, 50000])
    ap.add_argument("--block-sizes", type=int, nargs="+", default=[1000, 4541, 20000])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    gpu = bfp.card()
    print("card:", gpu)
    jobs = [(k, P) for k in ("pyramid", "chain") for P in a.pg_sizes] + [("corridor", P) for P in a.block_sizes]
    with open(a.out if a.out else os.devnull, "w") as f:
        def emit(rec):
            rec["card"] = gpu
            f.write(json.dumps(rec) + "\n")
            f.flush()
            print(json.dumps(rec))

        for kind, P in jobs:
            make, x, _, F = rfp.workload(kind, P)
            priors = gnss(x)
            h = make()
            for r in range(a.runs):
                for with_priors in (False, True):
                    h.set_pose_priors(priors if with_priors else [])
                    emit(dict(rfp.timed(h, x, a.iters), workload=kind, P=P, factors=F,
                              priors=len(priors) if with_priors else 0, run=r))
            h.set_pose_priors(priors)
            emit(dict(workload=kind, P=P, priors=len(priors), profiled_kernel_ms_per_iter=profiled(h, x, a.iters)))
            h.close()


if __name__ == "__main__":
    main()

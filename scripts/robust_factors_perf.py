"""Robust pose factors (balm_set_factor_loss): what a Cauchy loss adds to an LM iteration, against the trivial loss on the
same handle and factors.

  pyramid  PoseGraph, HBA-shaped window factors (scripts/pose_graph_perf.py's set)
  chain    PoseGraph, laps of a loop with odometry and a closure to the previous lap every 25 poses
           (tests/robust_factors_ref.outlier_scene without false closures)
  corridor PREC_BLOCKS voxel corridor with odometry and a loop closure every 500 poses (scripts/block_factors_perf.py)

The two losses alternate inside every run; wall times are host clocks around synchronised work (force_hess, so every
iteration evaluates). A separate profiled run per workload gives the device time of the robust cost and linearisation
kernels. Last, the LM iterations to convergence on the outlier scene with and without the loss.

  python scripts/robust_factors_perf.py [--pg-sizes 4541 20000 50000] [--block-sizes 1000 4541 20000] [--runs 3]
                                        [--out FILE]

Prints one JSON line per measurement with the card's name and power limit; --out FILE also writes them there.
"""
import argparse
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]
import balm_b200  # noqa: E402
import block_factors_perf as bfp  # noqa: E402
import block_hessian_ref as bref  # noqa: E402
import pose_graph_perf as pgp  # noqa: E402
import robust_factors_ref as rr  # noqa: E402
from balm_b200 import _lib as L  # noqa: E402


def workload(kind, P):
    """-> (make a handle with the factors attached, start poses, Cauchy scale)"""
    if kind == "pyramid":
        fs, x = pgp.factor_set(P)
        s, _ = rr.residuals(x, fs, np.zeros(len(fs), np.int32), np.ones(len(fs)))
        c = float(np.sqrt(np.median(s)))
    elif kind == "chain":  # true closures only: random false ones between distant poses would time the fill they cause
        sc = rr.outlier_scene(P, 1, every=25, false_frac=0.0)
        fs, x, c = sc["all"], sc["x0"], rr.cauchy_scale()
    else:
        sc = bref.corridor(P, w=10, planes_per_pose=30, seed=P)
        fs, x, c = bfp.factor_sets(sc, 500, 300)["loops"], sc["poses_init"], rr.cauchy_scale()

        def make():
            h = balm_b200.Context(P, 0, L.PREC_BLOCKS)
            h.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
            h.set_block_factors(fs)
            return h
        return make, x, c, len(fs)

    def make():
        h = balm_b200.PoseGraph(P)
        h.set_pose_factors(fs)
        return h
    return make, x, c, len(fs)


def lm(h, x, iters, **kw):
    if isinstance(h, balm_b200.PoseGraph):
        return h.pose_graph_iter(x, max_iter=iters, gauge_mode=2, **kw)[1]
    return h.damping_iter(x, max_iter=iters, gauge_mode=2, min_planes_per_pose=0, **kw)[1]


def timed(h, x, iters):
    lm(h, x, 1, rel_tol=-1)  # warm-up
    if not isinstance(h, balm_b200.PoseGraph):
        h.reset_counters()
    t0 = time.perf_counter()
    tr = lm(h, x, iters, rel_tol=-1, force_hess=True)
    rec = dict(ms_per_iter=1e3 * (time.perf_counter() - t0) / len(tr))
    if not isinstance(h, balm_b200.PoseGraph):
        tm = h.timings()
        rec["ms_assemble_per_eval"] = tm["ms_assemble"] / max(1, tm["n_eval"])
    return rec


def profiled(h, x, iters):
    """device ms per iteration of the robust kernels (and of every pose-factor kernel) in a profiled run"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        lm(h, x, iters, rel_tol=-1, force_hess=True)
    out = {}
    for e in prof.events():
        if e.device_type.name != "CUDA" or not any(k in e.name for k in ("pg_cost", "pg_linearise", "pg_assemble",
                                                                           "pg_sum")):
            continue
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        key = re.search(r"pg_\w+", e.name).group(0)
        key += "<FactorLoss>" if "FactorLoss" in e.name else "<NoLoss>" if "NoLoss" in e.name else ""
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
            make, x, c, F = workload(kind, P)
            h = make()
            for r in range(a.runs):
                for loss in ("trivial", "cauchy"):
                    h.set_factor_loss(loss, c)
                    emit(dict(timed(h, x, a.iters), workload=kind, P=P, factors=F, loss=loss, run=r))
            for loss in ("trivial", "cauchy"):
                h.set_factor_loss(loss, c)
                emit(dict(workload=kind, P=P, loss=loss, profiled_kernel_ms_per_iter=profiled(h, x, a.iters)))
            h.close()
        for P in (200, 2000):  # iterations to convergence on the outlier scene
            sc = rr.outlier_scene(P, 1)
            for loss in ("trivial", "cauchy"):
                h = balm_b200.PoseGraph(P)
                h.set_pose_factors(sc["all"])
                h.set_factor_loss(loss, rr.cauchy_scale())
                xs, tr = h.pose_graph_iter(sc["x0"], max_iter=100, gauge_mode=2)
                emit(dict(workload="outlier_scene", P=P, loss=loss, iterations=len(tr),
                          max_error_m=rr.max_error(xs, sc["gt"])))
                h.close()


if __name__ == "__main__":
    main()

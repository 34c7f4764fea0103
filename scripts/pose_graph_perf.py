"""Device time of the pose graph (Context.pose_graph_iter) per LM iteration, split into linearisation, assembly, the
dense solve (with the pose update) and the cost passes, at P = 177, 1 000 and 4 541 poses (the length of the
benchmark_realworld sequence, a longer drive, and KITTI 00).

Factor sets have the shape hba() builds: windows of 10 poses every 5, the windows' first poses forming the next layer,
up to one top window of at most 32 (tests/pose_graph_ref.pyramid_factor_poses), each factor noisy relative poses of one
random trajectory with a random window Hessian. Every iteration re-evaluates (force_hess) and runs to max_iter
(rel_tol < 0), so that all iterations do the same work. Per P:
  - wall ms per iteration: host clock around pose_graph_iter, which ends in a device synchronisation;
  - host waits per iteration: one stream synchronisation, plus one per refinement round (Context.timings());
  - the device split: a separate run under torch.profiler (CUDA activities), kernels grouped by name.
Prints one JSON line with the card's name and power limit; --out FILE also writes it there."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]


def factor_set(P, seed=0):
    import pose_graph_ref as pg
    rng = np.random.default_rng(seed)
    truth = np.array([pg.random_pose(rng, 0.5, 3.0) for _ in range(P)])
    factors = [pg.make_factor(rng, truth, s, noise=0.01) for s in pg.pyramid_factor_poses(P, top=32)]
    return factors, pg.perturb(rng, truth, 0.02, 0.1)


def phase(name):
    if "pg_linearise" in name:
        return "linearise"
    if "pg_assemble" in name or "memset" in name.lower():
        return "assembly"
    if "pg_cost" in name or "pg_sum" in name:
        return "cost"
    if "Memcpy" in name:
        return "copies"
    return "solve"  # damping copy, factorisation, substitutions, q1, backward-error check, pose update


def profile(c, x, iters):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprof
    torch.cuda.init()
    with tprof(activities=[ProfilerActivity.CUDA]) as prof:
        c.pose_graph_iter(x, max_iter=iters, rel_tol=-1, gauge_mode=2, force_hess=True)
    split, kernels = {}, {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        split[phase(e.name)] = split.get(phase(e.name), 0.0) + us / 1e3 / iters
        kernels[e.name[:60]] = kernels.get(e.name[:60], 0.0) + us / 1e3 / iters
    return split, dict(sorted(kernels.items(), key=lambda kv: -kv[1])[:12])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="177,1000,4541")
    ap.add_argument("--iters", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import balm_b200
    from hba_perf import gpu_info
    out = dict(gpu=gpu_info(), iters=a.iters, sizes=[])
    for P in [int(s) for s in a.sizes.split(",")]:
        factors, x = factor_set(P)
        c = balm_b200.Context(P)
        t0 = time.perf_counter()
        st = c.set_pose_factors(factors)
        reg_ms = 1e3 * (time.perf_counter() - t0)
        c.pose_graph_iter(x, max_iter=1, rel_tol=-1, gauge_mode=2)  # warm-up
        c.reset_counters()
        t0 = time.perf_counter()
        _, tr = c.pose_graph_iter(x, max_iter=a.iters, rel_tol=-1, gauge_mode=2, force_hess=True)
        wall = 1e3 * (time.perf_counter() - t0) / len(tr)
        tm = c.timings()
        split, kernels = profile(c, x, a.iters)
        out["sizes"].append(dict(P=P, factors=len(factors), not_pd=int(sum(s != 0 for s in st)),
                                 H_and_factor_GB=2 * (6 * P) ** 2 * 8 / 1e9, register_ms=reg_ms, wall_ms_per_iter=wall,
                                 host_waits_per_iter=(len(tr) + tm["refinements"]) / len(tr),
                                 device_ms_per_iter=split, top_kernels_ms_per_iter=kernels,
                                 cost=[tr[0]["r1"], tr[-1]["r2"]]))
        c.close()
        print(json.dumps(out["sizes"][-1]), flush=True)
    s = json.dumps(out)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")
    print(s)


if __name__ == "__main__":
    main()

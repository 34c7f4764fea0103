"""Time of the pose graph per LM iteration on its two solves: the context's dense one (Context.pose_graph_iter) at
P = 177, 400, 700, 1 000 and 4 541 poses (the length of the benchmark_realworld sequence, longer drives, and KITTI 00), and the
block-sparse one (PoseGraph.pose_graph_iter) at those sizes and at 20 000 and 50 000 poses (about 35 and 90 minutes of
10 Hz scans), where the dense system does not fit. At the shared sizes the two paths run alternately in the same call,
and their poses are compared.

Factor sets have the shape hba() builds: windows of 10 poses every 5, the windows' first poses forming the next layer,
up to one top window of at most 32 (tests/pose_graph_ref.pyramid_factor_poses), each factor noisy relative poses of one
random trajectory with a random window Hessian. Every iteration re-evaluates (force_hess) and runs to max_iter
(rel_tol < 0), so that all iterations do the same work. Per P:
  - wall ms per iteration: host clock around pose_graph_iter, which ends in a device synchronisation;
  - host waits per iteration: one stream synchronisation, plus one per refinement round (Context.timings());
  - the device split: a separate run under torch.profiler (CUDA activities), kernels grouped by name; on the sparse
    path also the launch gaps inside its solves (each solve's span, from its damped copy to the end of its check,
    minus the kernel time within it);
  - registration ms; on the sparse path also its excess over the dense registration, which is the host ordering,
    symbolic factorisation and graph capture (the factor upload, check and tables are the same code);
  - sparse: blocks of L, elimination-tree levels and device bytes.
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
    if "pg_linearise" in name or "pg_assemble" in name:
        return "assembly"
    if "memset" in name.lower():
        return "memset"
    if "pg_cost" in name or "pg_sum" in name:
        return "cost"
    if "Memcpy" in name:
        return "copies"
    if "spg_damp" in name or "spg_factor_kernel<true>" in name:
        return "factorisation"  # the level kernels also run the forward substitution of their columns
    if "spg_back" in name or "spg_factor_kernel<false>" in name:
        return "substitutions"
    if "spg_check" in name or "q1_kernel" in name:
        return "check"
    return "solve"  # dense: damping copy, factorisation, substitutions, q1, backward-error check; both: pose update


def profile(c, x, iters):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprof
    torch.cuda.init()
    with tprof(activities=[ProfilerActivity.CUDA]) as prof:
        c.pose_graph_iter(x, max_iter=iters, rel_tol=-1, gauge_mode=2, force_hess=True)
    split, kernels, ev = {}, {}, []
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        split[phase(e.name)] = split.get(phase(e.name), 0.0) + us / 1e3 / iters
        kernels[e.name[:60]] = kernels.get(e.name[:60], 0.0) + us / 1e3 / iters
        ev.append((e.time_range.start, e.time_range.end, us, e.name))
    ev.sort()
    span = busy = 0.0  # sparse solves: from spg_damp_kernel to the end of the next spg_check_kernel
    t0 = None
    for start, end, us, name in ev:
        if "spg_damp" in name:
            t0, inside = start, 0.0
        if t0 is not None:
            inside += us
            if "spg_check" in name:
                span, busy, t0 = span + end - t0, busy + inside, None
    if span > 0:
        split["solve_launch_gaps"] = (span - busy) / 1e3 / iters
        split["solve_span"] = span / 1e3 / iters
    return split, dict(sorted(kernels.items(), key=lambda kv: -kv[1])[:12])


def run(P, factors, x, sparse, iters):
    import balm_b200
    c = balm_b200.PoseGraph(P) if sparse else balm_b200.Context(P)
    t0 = time.perf_counter()
    st = c.set_pose_factors(factors)
    reg_ms = 1e3 * (time.perf_counter() - t0)
    c.pose_graph_iter(x, max_iter=1, rel_tol=-1, gauge_mode=2)  # warm-up
    t0 = time.perf_counter()
    poses, tr = c.pose_graph_iter(x, max_iter=iters, rel_tol=-1, gauge_mode=2, force_hess=True)
    wall = 1e3 * (time.perf_counter() - t0) / len(tr)
    r = dict(path="sparse" if sparse else "dense", register_ms=reg_ms, wall_ms_per_iter=wall,
             not_pd=int(sum(s != 0 for s in st)), cost=[tr[0]["r1"], tr[-1]["r2"]])
    if sparse:
        r.update(c.structure())
    else:
        r["H_and_factor_GB"] = 2 * (6 * P) ** 2 * 8 / 1e9
    c.close()
    return r, poses


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="177,400,700,1000,4541,20000,50000")
    ap.add_argument("--dense_max", type=int, default=4541, help="largest P also run on the dense path")
    ap.add_argument("--reps", type=int, default=3, help="alternating runs of the two paths per shared size")
    ap.add_argument("--iters", type=int, default=4)
    ap.add_argument("--no_profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import balm_b200
    from hba_perf import gpu_info
    out = dict(gpu=gpu_info(), iters=a.iters, sizes=[])
    for P in [int(s) for s in a.sizes.split(",")]:
        factors, x = factor_set(P)
        paths = [False, True] if P <= a.dense_max else [True]
        runs = {p: [] for p in paths}
        poses = {}
        for rep in range(a.reps if len(paths) > 1 else 1):
            for sparse in paths:
                r, poses[sparse] = run(P, factors, x, sparse, a.iters)
                runs[sparse].append(r)
        res = dict(P=P, factors=len(factors))
        for sparse in paths:
            rs = runs[sparse]
            r = dict(rs[-1], wall_ms_per_iter=[q["wall_ms_per_iter"] for q in rs],
                     register_ms=[q["register_ms"] for q in rs])
            if not a.no_profile:
                c = balm_b200.PoseGraph(P) if sparse else balm_b200.Context(P)
                c.set_pose_factors(factors)
                c.pose_graph_iter(x, max_iter=1, rel_tol=-1, gauge_mode=2)
                r["device_ms_per_iter"], r["top_kernels_ms_per_iter"] = profile(c, x, a.iters)
                c.close()
            res[r.pop("path")] = r
        if len(paths) > 1:
            res["max_pose_diff_dense_vs_sparse"] = float(np.abs(poses[True] - poses[False]).max())
            reg = [s - d for s, d in zip(res["sparse"]["register_ms"], res["dense"]["register_ms"])]
            res["sparse"]["register_excess_ms"] = reg
        out["sizes"].append(res)
        print(json.dumps(res), flush=True)
    s = json.dumps(out)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")
    print(s)


if __name__ == "__main__":
    main()

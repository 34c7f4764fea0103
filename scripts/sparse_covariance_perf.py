"""Time of the marginal covariances on the sparse solve (PoseGraph.covariance, Context.block_covariance) beside one LM
iteration of the same handle: PoseGraph pyramids at P = 177, 1 000, 4 541, 20 000 and 50 000 poses (the
pose_graph_perf.py sets) and PREC_BLOCKS corridors at P = 177, 1 000, 4 541 and 20 000 (the block_hessian_perf.py
scenes). The corridors carry fix clusters (anchor = -1) and span at most --blocks_length metres (100): longer ones are too
ill-conditioned in the pose-update coordinates for the covariance's pivot rule. Per P:
  - wall ms of the first covariance call (which also builds the selected-inversion tables) and of repeat calls, host
    clock around the call, which ends in a device synchronisation; the covariance is taken at the LM's output poses;
  - wall ms per LM iteration (force_hess, rel_tol < 0: every iteration evaluates, factors and solves);
  - the device split of one repeat call from torch.profiler (CUDA activities) in a separate run: evaluation, factor
    (undamped copy, anchor, level factorisation), selinv, gather, copies;
  - the selected-inversion terms and the device bytes before and after the first call (the growth is 8 (P + 1) + 4 terms
    + 4 pairs + 288 blocks of L bytes, from which the terms are read back).
Prints one JSON line per (path, P) with the card's name and power limit; --out FILE also writes them there."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]


def phase(name):
    if "spg_selinv" in name:
        return "selinv"
    if "spg_cov_gather" in name:
        return "gather"
    if "spg_damp" in name or "spg_anchor" in name or "spg_factor_kernel" in name:
        return "factor"
    if "Memcpy" in name:
        return "copies"
    if "memset" in name.lower():
        return "memset"
    return "evaluation"


def profile(call):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprof
    torch.cuda.init()
    with tprof(activities=[ProfilerActivity.CUDA]) as prof:
        call()
    split = {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        split[phase(e.name)] = split.get(phase(e.name), 0.0) + us / 1e3
    return split


def timed(call):
    t0 = time.perf_counter()
    out = call()
    return 1e3 * (time.perf_counter() - t0), out


def measure(h, structure, lm, cov, reps, do_profile):
    """h: the handle; structure() -> dict with pairs, l_blocks, device_bytes; lm() -> (poses, iterations);
    cov(poses) -> the covariance call."""
    import balm_b200
    lm()  # warm-up
    t, (x, n) = timed(lm)
    st0 = structure()
    rec = dict(lm_ms_per_iter=t / n, pairs=st0["pairs"], l_blocks=st0["l_blocks"], levels=st0["levels"],
               device_bytes_registered=st0["device_bytes"])
    try:
        first, _ = timed(lambda: cov(x))
    except balm_b200.BalmError as e:
        rec["status"] = e.status
        return rec
    rec["cov_first_ms"] = first
    rec["cov_repeat_ms"] = [timed(lambda: cov(x))[0] for _ in range(reps)]
    st1 = structure()
    grown = st1["device_bytes"] - st0["device_bytes"]
    P = h.N
    rec.update(device_bytes_after=st1["device_bytes"],
               selinv_terms=(grown - 8 * (P + 1) - 4 * max(st0["pairs"], 1) - 288 * st0["l_blocks"]) // 4)
    rec["repeat_over_lm_iter"] = float(np.median(rec["cov_repeat_ms"])) / rec["lm_ms_per_iter"]
    if do_profile:
        rec["device_ms"] = profile(lambda: cov(x))
    return rec


def pose_graph(P, iters, reps, do_profile):
    import balm_b200
    from pose_graph_perf import factor_set
    factors, x0 = factor_set(P)
    s = balm_b200.PoseGraph(P)
    s.set_pose_factors(factors)

    def lm():
        x, tr = s.pose_graph_iter(x0, max_iter=iters, rel_tol=-1, gauge_mode=2, force_hess=True)
        return x, len(tr)
    rec = measure(s, s.structure, lm, lambda x: s.covariance(x, 0), reps, do_profile)
    s.close()
    return dict(path="pose_graph", P=P, factors=len(factors), **rec)


def blocks(P, iters, reps, do_profile, length):
    import balm_b200
    import block_hessian_ref as bref
    from balm_b200 import _lib as L
    # corridor() spreads P poses over min(1 km, P m); H of a long corridor is too ill-conditioned in the pose-update
    # coordinates for the covariance's pivot rule (tests/test_gpu_sparse_covariance.py), so these span `length` metres
    # and carry fix clusters, which fix the gauge (anchor = -1)
    bref.min = lambda a, b: min(1.0, length / P)
    try:
        sc = bref.corridor(P, w=10, planes_per_pose=30, seed=P, with_fix=True)
    finally:
        del bref.min
    c = balm_b200.Context(P, 0, L.PREC_BLOCKS)
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc["fix10"])

    def lm():
        x, tr, _ = c.damping_iter(sc["poses_init"], max_iter=iters, rel_tol=-1, force_hess=True, min_planes_per_pose=0,
                                  gauge_mode=2, hess_includes_fix=True)
        return x, len(tr)
    rec = measure(c, c.block_structure, lm, lambda x: c.block_covariance(x, include_fix=True, anchor=-1), reps,
                  do_profile)
    c.close()
    return dict(path="blocks", P=P, length_m=min(P, length), voxels=len(sc["row_ptr"]) - 1, **rec)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pose_graph_sizes", default="177,1000,4541,20000,50000")
    ap.add_argument("--blocks_sizes", default="177,1000,4541,20000")
    ap.add_argument("--blocks_length", type=float, default=100.0, help="metres the blocks corridors span at most")
    ap.add_argument("--iters", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3, help="repeat covariance calls timed per size")
    ap.add_argument("--no_profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from hba_perf import gpu_info
    gpu = gpu_info()
    print("card:", json.dumps(gpu), flush=True)
    recs = []
    runs = [("pose_graph", a.pose_graph_sizes, pose_graph),
            ("blocks", a.blocks_sizes, lambda *r: blocks(*r, a.blocks_length))]
    for path, sizes, fn in runs:
        for P in [int(v) for v in sizes.split(",") if v]:
            r = dict(fn(P, a.iters, a.reps, not a.no_profile), gpu=gpu)
            recs.append(r)
            print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.writelines(json.dumps(r) + "\n" for r in recs)


if __name__ == "__main__":
    main()

"""Pose factors in a PREC_BLOCKS context (balm_block_set_factors) on corridor scenes (tests/block_hessian_ref.corridor):
ms per LM iteration split by phase (balm_timings; ms_assemble is the factors' linearisation, assembly and cost), the time
to attach the factors, pattern size, blocks of L, elimination-tree levels and device bytes, for three modes:

  blocks    voxels alone
  odometry  plus one odometry factor between consecutive scans (neighbours co-observe: the pattern does not change)
  loops     plus a loop closure every --loop-every poses to the pose --loop-back before it (fill grows)

The modes alternate inside every run; wall times are host clocks around synchronised work.

  python scripts/block_factors_perf.py --sizes 1000 4541 20000 --runs 3 [--out FILE]

Prints one JSON line per (size, run, mode) with the card's name and power limit; --out FILE also writes them there.
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
from balm_b200 import _lib as L  # noqa: E402

MODES = ("blocks", "odometry", "loops")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def factor_sets(sc, loop_every, loop_back):
    """odometry from the truth (0.002 rad, 0.02 m), in the voxel cost's units (points x m^2 at 0.01 m point noise)"""
    info = 2 * 0.01 ** 2 * np.diag(np.r_[np.full(3, 0.002 ** -2), np.full(3, 0.02 ** -2)])
    gt = sc["poses_gt"]
    odo = balm_b200.odometry_factors(gt, info)
    loops = [(a, a - loop_back) for a in range(loop_every, sc["n_poses"], loop_every)]
    return {"blocks": [], "odometry": odo, "loops": odo + balm_b200.odometry_factors(gt, info, edges=loops)}


def one(sc, factors, mode, iters):
    P = sc["n_poses"]
    c = balm_b200.Context(P, 0, L.PREC_BLOCKS)
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
    c.sync()
    t0 = time.perf_counter()
    if factors:
        c.set_block_factors(factors)
    c.sync()
    attach_ms = 1e3 * (time.perf_counter() - t0)
    kw = dict(max_iter=iters, rel_tol=-1, force_hess=True, min_planes_per_pose=0, gauge_mode=2)
    c.damping_iter(sc["poses_init"], max_iter=1, rel_tol=-1, min_planes_per_pose=0, gauge_mode=2)  # warm-up
    c.reset_counters()
    t0 = time.perf_counter()
    _, trace, _ = c.damping_iter(sc["poses_init"], **kw)
    c.sync()
    wall = 1e3 * (time.perf_counter() - t0) / len(trace)
    tm = c.timings()
    n = len(trace)
    rec = dict(P=P, mode=mode, factors=len(factors), ms_per_iter=wall, attach_ms=attach_ms,
               split={k: tm[k] / n for k in ("ms_stats", "ms_obs", "ms_syrk", "ms_assemble", "ms_solve", "ms_residual")},
               refinements=tm["refinements"], not_pd=sum(t["not_pd"] for t in trace),
               r_first=trace[0]["r1"], r_last=trace[-1]["r2"])
    rec.update(c.block_structure())
    c.close()
    return rec


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1000, 4541, 20000])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--w", type=int, default=10, help="co-visibility half-width in poses")
    ap.add_argument("--loop-every", type=int, default=500)
    ap.add_argument("--loop-back", type=int, default=300)
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    gpu = card()
    print("card:", gpu)
    with open(a.out if a.out else os.devnull, "w") as f:
        for P in a.sizes:
            sc = bref.corridor(P, w=a.w, planes_per_pose=30, seed=P)
            sets = factor_sets(sc, a.loop_every, a.loop_back)
            for r in range(a.runs):
                for m in MODES:
                    rec = dict(one(sc, sets[m], m, a.iters), run=r, card=gpu, voxels=len(sc["row_ptr"]) - 1,
                               obs=len(sc["pose_idx"]))
                    f.write(json.dumps(rec) + "\n")
                    f.flush()
                    print(json.dumps(rec))


if __name__ == "__main__":
    main()

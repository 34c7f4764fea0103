"""PREC_BLOCKS against the dense fp64 and tensor contexts on corridor scenes (tests/block_hessian_ref.corridor): ms per
LM iteration split by phase (balm_timings), registration ms, pattern size and device bytes, and the largest pose
difference between the paths. The modes alternate inside every run; wall times are host clocks around synchronised work.

  python scripts/block_hessian_perf.py --sizes 177 500 1000 2000 4541 20000 --runs 3 [--out FILE]

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

MODES = {"fp64": L.PREC_FP64, "tensor": L.PREC_TENSOR, "blocks": L.PREC_BLOCKS}
DENSE_MAX_POSES = 6000  # H + A = 2 (6P)^2 doubles: 20 GB at 6000 poses


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def one(sc, mode, iters):
    P = sc["n_poses"]
    c = balm_b200.Context(P, 0, MODES[mode])
    t0 = time.perf_counter()
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
    c.sync()
    reg_ms = 1e3 * (time.perf_counter() - t0)
    kw = dict(max_iter=iters, rel_tol=-1, force_hess=True, min_planes_per_pose=0, gauge_mode=2)
    c.damping_iter(sc["poses_init"], max_iter=1, rel_tol=-1, min_planes_per_pose=0, gauge_mode=2)  # warm-up
    c.reset_counters()
    t0 = time.perf_counter()
    poses, trace, _ = c.damping_iter(sc["poses_init"], **kw)
    c.sync()
    wall = 1e3 * (time.perf_counter() - t0) / len(trace)
    tm = c.timings()
    n = len(trace)
    rec = dict(P=P, mode=mode, ms_per_iter=wall, reg_ms=reg_ms,
               split={k: tm[k] / n for k in ("ms_stats", "ms_obs", "ms_syrk", "ms_assemble", "ms_solve", "ms_residual")},
               refinements=tm["refinements"])
    if mode == "blocks":
        rec.update(c.block_structure())
    c.close()
    return rec, poses


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[177, 500, 1000, 2000, 4541, 20000])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--w", type=int, default=10, help="co-visibility half-width in poses")
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    gpu = card()
    print("card:", gpu)
    with open(a.out if a.out else os.devnull, "w") as f:
        for P in a.sizes:
            sc = bref.corridor(P, w=a.w, planes_per_pose=30, seed=P)
            modes = ["fp64", "tensor", "blocks"] if P <= DENSE_MAX_POSES else ["blocks"]
            for r in range(a.runs):
                res = {m: one(sc, m, a.iters) for m in modes}
                diff = max((float(np.abs(res[m][1] - res["blocks"][1]).max()) for m in modes if m != "blocks"),
                           default=0.0)
                for m in modes:
                    rec = dict(res[m][0], run=r, card=gpu, max_pose_diff_vs_blocks=diff,
                               voxels=len(sc["row_ptr"]) - 1, obs=len(sc["pose_idx"]))
                    f.write(json.dumps(rec) + "\n")
                    f.flush()
                    print(json.dumps(rec))


if __name__ == "__main__":
    main()

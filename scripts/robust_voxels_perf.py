"""Cost of a robust voxel loss (balm_set_voxel_loss): the trivial loss and Cauchy alternate on one handle, three runs
each, on bench.py's scene shape at C3 (500 poses x 100 000 voxels) and C2 (200 x 20 000) on the tensor path, C3 on the
fp64 path, and block_hessian_perf.py's 4 541-pose corridor on PREC_BLOCKS. Per run: ms per LM iteration (CUDA events
around one damping_iter with force_hess and the convergence exit off), the stats pass per evaluation (ms_stats / n_stats),
and the tensor path's sweep counters (single_sweeps, redone_sweeps: the OBS_INT8 sweep re-armed because column maxima
moved past their scales; reused_sweeps). The loss changes G''s column maxima between evaluations, so redone_sweeps is
the number to watch.

    python scripts/robust_voxels_perf.py [--runs 3] [--iters 5] [--out FILE]

Prints the card's name and power limit, then one JSON line per (workload, loss, run); --out FILE also writes them there.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import balm_b200  # noqa: E402
import block_hessian_ref as bref  # noqa: E402
from balm_b200 import _lib as L  # noqa: E402

LM = dict(rel_tol=-1.0, force_hess=True, min_planes_per_pose=0, gauge_mode=2)
NOISE = 0.01  # bench.py's point noise: Cauchy at 2 sigma


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def workloads():
    def synth(P, M, prec):
        c = balm_b200.Context(P, 0, prec)
        _, init = c.synth_virtual(M, 0, 40, NOISE, 2.0, 10)  # bench.py: PTS, NOISE, RANGE, SEED
        return c, init, 2 * NOISE

    def corridor():
        sc = bref.corridor(4541, w=10, planes_per_pose=30, seed=4541)
        c = balm_b200.Context(sc["n_poses"], 0, L.PREC_BLOCKS)
        c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
        lam, _ = c.voxel_residuals(sc["poses_init"])
        return c, sc["poses_init"], float(np.sqrt(np.median(lam)))  # both sides of c^2 at the start

    yield "C3 tensor", lambda: synth(500, 100000, L.PREC_TENSOR)
    yield "C2 tensor", lambda: synth(200, 20000, L.PREC_TENSOR)
    yield "C3 fp64", lambda: synth(500, 100000, L.PREC_FP64)
    yield "corridor 4541 blocks", corridor


def one(c, init, iters):
    c.reset_counters()
    c.timer_begin()
    _, tr, _ = c.damping_iter(init, max_iter=iters, **LM)
    ms = c.timer_end()
    tm = c.timings()
    return dict(ms_per_iter=round(ms / len(tr), 3), ms_stats=round(tm["ms_stats"] / max(tm["n_stats"], 1), 4),
                accepted="".join("A" if t["accepted"] else "r" for t in tr),
                **{k: tm[k] for k in ("n_eval", "single_sweeps", "redone_sweeps", "reused_sweeps")})


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    gpu = card()
    print("card:", gpu, flush=True)
    with open(a.out if a.out else os.devnull, "w") as f:
        for name, make in workloads():
            c, init, scale = make()
            c.damping_iter(init, max_iter=2, **LM)  # warm-up of both instantiations
            c.set_voxel_loss("cauchy", scale)
            c.damping_iter(init, max_iter=2, **LM)
            for r in range(a.runs):
                for loss in ("trivial", "cauchy"):
                    c.set_voxel_loss(loss, scale)
                    rec = dict(workload=name, loss=loss, scale=scale, run=r, card=gpu, **one(c, init, a.iters))
                    line = json.dumps(rec)
                    print(line, flush=True)
                    f.write(line + "\n")
            c.close()


if __name__ == "__main__":
    main()

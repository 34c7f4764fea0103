"""Voxels, pose factors and priors in one cost on dense contexts (balm_set_joint_cost): what odometry on every pose and
a GNSS position prior on every 10th pose add to an LM iteration. Corridor scenes as scripts/block_hessian_perf.py's
(tests/block_hessian_ref.corridor, every plane seen by the 21 poses within +-10, 30 planes per pose), at 177, 500 and
1 000 poses: the sizes where the dense path is the faster one. Four contexts per size:

  tensor        PREC_TENSOR, voxels only (the baseline the joint cost adds to)
  tensor_joint  PREC_TENSOR, set_joint_cost(True) with the odometry and the priors
  fp64_joint    PREC_FP64, the same
  blocks_joint  PREC_BLOCKS with the same factors and priors (set_block_factors)

All four are created once per size and run alternately, three runs each: wall ms per LM iteration from the host clock
around synchronised work (5 iterations, force_hess, so every one evaluates), and ms_assemble per evaluation from
balm_timings (on the dense contexts the assembly of H and g plus the factors' and priors' kernels; on blocks the
factor and prior kernels alone). One warm-up LM call per context before its first timed run.

  python scripts/joint_cost_perf.py [--sizes 177 500 1000] [--runs 3] [--iters 5] [--out FILE]

Prints one JSON line per measurement with the card's name and power limit; --out FILE also writes them there.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]
import balm_b200  # noqa: E402
import block_hessian_ref as bref  # noqa: E402
from balm_b200 import _lib as L  # noqa: E402
from block_factors_perf import card  # noqa: E402
from pose_priors_perf import gnss  # noqa: E402

MODES = ("tensor", "tensor_joint", "fp64_joint", "blocks_joint")


def odometry(gt):
    """odometry from the truth (0.002 rad, 0.02 m), in the voxel cost's units (points x m^2 at 0.01 m point noise)"""
    info = 2 * 0.01 ** 2 * np.diag(np.r_[np.full(3, 0.002 ** -2), np.full(3, 0.02 ** -2)])
    return balm_b200.odometry_factors(gt, info)


def context(sc, mode, odo, priors):
    prec = {"tensor": L.PREC_TENSOR, "tensor_joint": L.PREC_TENSOR, "fp64_joint": L.PREC_FP64,
            "blocks_joint": L.PREC_BLOCKS}[mode]
    c = balm_b200.Context(sc["n_poses"], 0, prec)
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
    if mode == "blocks_joint":
        c.set_block_factors(odo)
    elif mode != "tensor":
        c.set_pose_factors(odo)
        c.set_joint_cost(True)
    if mode != "tensor":
        c.set_pose_priors(priors)
    return c


def timed(c, x, iters):
    c.reset_counters()
    c.sync()
    t0 = time.perf_counter()
    _, tr, _ = c.damping_iter(x, max_iter=iters, gauge_mode=2, min_planes_per_pose=0, rel_tol=-1, force_hess=True)
    ms = 1e3 * (time.perf_counter() - t0) / len(tr)
    tm = c.timings()
    return dict(ms_per_iter=ms, ms_assemble=tm["ms_assemble"] / max(1, tm["n_eval"]), iters=len(tr),
                launches_per_iter=tm["launches"] / len(tr), r_last=tr[-1]["r2"])


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[177, 500, 1000])
    ap.add_argument("--w", type=int, default=10, help="co-visibility half-width in poses")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    gpu = card()
    print("card:", gpu)
    with open(a.out if a.out else os.devnull, "w") as f:
        def emit(rec):
            rec["card"] = gpu
            f.write(json.dumps(rec) + "\n")
            f.flush()
            print(json.dumps(rec))

        for P in a.sizes:
            sc = bref.corridor(P, w=a.w, planes_per_pose=30, seed=P)
            odo, priors = odometry(sc["poses_gt"]), gnss(sc["poses_gt"])
            x = sc["poses_init"]
            ctx = {m: context(sc, m, odo, priors) for m in MODES}
            for c in ctx.values():  # warm-up
                c.damping_iter(x, max_iter=1, gauge_mode=2, min_planes_per_pose=0, rel_tol=-1)
            for r in range(a.runs):
                for m in MODES:
                    emit(dict(timed(ctx[m], x, a.iters), mode=m, P=P, factors=len(odo), priors=len(priors), run=r))
            for c in ctx.values():
                c.close()


if __name__ == "__main__":
    main()

"""Cost of the rig covariance (DESIGN.md "Rig covariance"): Context.rig_covariance against Context.pose_covariance on
the same context, and the rig call's split into its phases.

Workloads: rig_perf.py's balm_synth_virtual rigs, 500 slots (125 base poses x 4 LiDARs, 100 000 voxels) and 2 000
slots (500 x 4, 20 000 voxels), each on the tensor and the fp64 path; LiDAR 0 fixed, every extrinsic at the identity,
base b at slot 4b's pose, the rig covariance anchored at base 0. The synthetic voxels carry no fix clusters, so the
context's H is singular and pose_covariance refuses after its factorisation (BALM_ERR_NOT_PD): its full call is timed
up to that refusal, and its raw term alone (want_cov=False) as well.

1. Wall time per call: host clocks around calls that end in a device synchronise, the three calls alternating, after
   one warm-up of each.
2. In a separate run, torch.profiler's device kernels of rig_covariance calls, in launch order, split into the raw term
   (up to the first rig_k_kernel), its reduction (that rig_k_kernel and rig_jtk_kernel<false>), the H_rig evaluation
   (up to rig_jtk_kernel<true>), the factorisation (up to the first multi-right-hand-side solve kernel) and the solves.

    python scripts/rig_covariance_perf.py [--reps 5] [--profile_reps 2] [--out FILE]

Prints the card's name and power limit, then one JSON line per record; --out FILE also writes them there.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "scripts")]
import balm_b200  # noqa: E402
from balm_b200 import _lib as L  # noqa: E402
from rig_perf import IDENT, card  # noqa: E402

PN = 0.01
PRECS = {"tensor": L.PREC_TENSOR, "fp64": L.PREC_FP64}


def synth(bases, lidars, M, prec):
    N = bases * lidars
    c = balm_b200.Context(N, 0, prec)
    _, init = c.synth_virtual(M, 0, 40, 0.01, 2.0, 10)  # bench.py: PTS, NOISE, RANGE, SEED
    base_of, lidar_of = np.arange(N) // lidars, np.arange(N) % lidars
    base, ext = init[::lidars].copy(), np.tile(IDENT, (lidars, 1))
    c.set_rig(base_of, lidar_of)
    return c, balm_b200.rig_poses(base, ext, base_of, lidar_of), base, ext


WORKLOADS = [(f"synth {b * 4} slots ({b} x 4), {m // 1000}k voxels, {p}", b, m, p)
             for b, m in ((125, 100000), (500, 20000)) for p in PRECS]


def wall(fn):
    t = time.perf_counter()
    try:
        fn()
        status = "ok"
    except balm_b200.BalmError as e:
        status = f"status {e.status}"
    return (time.perf_counter() - t) * 1e3, status


PHASES = ("raw term", "reduction", "H_rig evaluation", "factor", "solves")


def split(kernels):
    """[(name, ms)] of one call in launch order -> ms per phase"""
    out = dict.fromkeys(PHASES, 0.0)
    phase = 0
    for name, ms in kernels:
        if phase == 0 and "rig_k_kernel" in name:
            phase = 1
        elif phase == 1 and "rig_jtk_kernel" not in name and "rig_k_kernel" not in name:
            phase = 2
        elif phase == 3 and ("mrhs_" in name or "scale_rows" in name):
            phase = 4
        out[PHASES[phase]] += ms
        if phase == 2 and "rig_jtk_kernel<true>" in name:
            phase = 3
    return {k: round(v, 4) for k, v in out.items()}


def profile(c, base, ext, reps):
    from torch.profiler import ProfilerActivity, profile as prof
    c.rig_covariance(base, ext, point_noise=PN, anchor=0)
    rows = []
    for _ in range(reps):
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            c.rig_covariance(base, ext, point_noise=PN, anchor=0)
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "trace.json")
            p.export_chrome_trace(path)
            with open(path) as f:
                ev = json.load(f)["traceEvents"]
        ks = sorted((e for e in ev if e.get("cat") == "kernel"), key=lambda e: e["ts"])
        rows.append(split([(e["name"], e["dur"] / 1000.0) for e in ks]))
    return {k: round(float(np.median([r[k] for r in rows])), 4) for k in PHASES}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile_reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    gpu = card()
    print("card:", gpu, flush=True)
    with open(a.out if a.out else os.devnull, "w") as f:
        def emit(rec):
            line = json.dumps(dict(card=gpu, **rec))
            print(line, flush=True)
            f.write(line + "\n")

        for name, b, m, p in WORKLOADS:
            c, X, base, ext = synth(b, 4, m, PRECS[p])
            calls = (("rig_covariance", lambda: c.rig_covariance(base, ext, point_noise=PN, anchor=0)),
                     ("pose_covariance (to its NOT_PD refusal)", lambda: c.pose_covariance(X, point_noise=PN)),
                     ("pose_covariance raw term only", lambda: c.pose_covariance(X, point_noise=PN, want_cov=False)))
            for _, fn in calls:
                wall(fn)  # warm-up of every shape
            times = {k: [] for k, _ in calls}
            status = {}
            for _ in range(a.reps):
                for k, fn in calls:
                    ms, status[k] = wall(fn)
                    times[k].append(ms)
            for k, _ in calls:
                emit(dict(workload=name, call=k, status=status[k], ms_median=round(float(np.median(times[k])), 2),
                          ms_min=round(min(times[k]), 2), ms_max=round(max(times[k]), 2)))
            emit(dict(workload=name, profile="rig_covariance device ms by phase", **profile(c, base, ext,
                                                                                             a.profile_reps)))
            c.close()


if __name__ == "__main__":
    main()

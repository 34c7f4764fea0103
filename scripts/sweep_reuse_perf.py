"""Tensor path, C3 shape (500 poses x 100 000 voxels, bench.py's scene): the observation sweep skipped on the
re-evaluations that follow rejected LM steps, against BALM_NO_SWEEP_REUSE=1 (sweep again every time).

For each variant, in a process of its own (the hook is read when the context is created), after a 3-iteration warm-up
call: one 10-iteration damping_iter call with bench.py's options (force_hess, convergence exit off) timed with CUDA
events, the accept sequence, the sweep counters and the per-evaluation phases; then the same call under torch.profiler
with the kernel times of the observation sweep, the SYRK and the residual pass. The two variants must return the same
bits (poses and trace).

    python scripts/sweep_reuse_perf.py [--poses 500] [--voxels 100000] [--steps 10] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

LM = dict(u0=0.01, v0=2.0, rel_tol=-1.0, gauge_mode=2, min_planes_per_pose=0, force_hess=True)
KERNELS = ("obs_pass_kernel", "obs_reduce_kernel", "tc_adopt_kernel", "tc_scale_kernel", "syrk_tc_kernel",
           "voxel_sums_kernel", "voxel_eig_kernel")


def child(args):
    sys.path.insert(0, ROOT)
    import torch
    import balm_b200
    c = balm_b200.Context(args.poses, 0, balm_b200.PREC_TENSOR)
    _, init = c.synth_virtual(args.voxels, 0, 40, 0.01, 2.0, 10)  # bench.py: PTS, NOISE, RANGE, SEED
    c.damping_iter(init, max_iter=3, **LM)
    c.reset_counters()
    c.timer_begin()
    poses, tr, _ = c.damping_iter(init, max_iter=args.steps, **LM)
    ms = c.timer_end()
    tm = c.timings()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        c.damping_iter(init, max_iter=args.steps, **LM)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        name = next((k for k in KERNELS if k in e.key), None)
        if name:
            d = kern.setdefault(name, {"calls": 0, "ms": 0.0})
            d["calls"] += e.count
            d["ms"] += e.device_time_total / 1e3
    n_eval = max(tm["n_eval"], 1)
    out = {"reuse": os.environ.get("BALM_NO_SWEEP_REUSE") is None, "gpu": torch.cuda.get_device_name(0),
           "ms_per_iter": ms / args.steps, "accepted": "".join("A" if t["accepted"] else "r" for t in tr),
           "counters": {k: tm[k] for k in ("n_eval", "single_sweeps", "redone_sweeps", "reused_sweeps", "n_stats")},
           "per_eval_ms": {k: round(tm[k] / n_eval, 3) for k in ("ms_stats", "ms_obs", "ms_syrk", "ms_assemble")},
           "per_step_ms": {k: round(tm[k] / args.steps, 3) for k in ("ms_solve", "ms_residual")},
           "profiler_ms_per_call": {k: round(v["ms"], 3) for k, v in kern.items()},
           "profiler_calls": {k: v["calls"] for k, v in kern.items()}}
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        tag = "reuse" if out["reuse"] else "noreuse"
        np.save(os.path.join(args.out, f"poses_{tag}.npy"), poses)
        np.save(os.path.join(args.out, f"trace_{tag}.npy"),
                np.array([[t[k] for k in ("r1", "r2", "q1", "accepted")] for t in tr], dtype=np.float64))
    print(json.dumps(out), flush=True)
    c.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--poses", type=int, default=500)
    ap.add_argument("--voxels", type=int, default=100000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", action="store_true")
    args = ap.parse_args()
    if args.child:
        return child(args)
    res = {}
    for reuse in (False, True):
        env = dict(os.environ)
        env.pop("BALM_NO_SWEEP_REUSE", None)
        if not reuse:
            env["BALM_NO_SWEEP_REUSE"] = "1"
        cmd = [sys.executable, os.path.abspath(__file__), "--child", "--poses", str(args.poses), "--voxels",
               str(args.voxels), "--steps", str(args.steps)] + (["--out", args.out] if args.out else [])
        line = subprocess.run(cmd, env=env, check=True, capture_output=True, text=True).stdout.strip().splitlines()[-1]
        res[reuse] = json.loads(line)
        print(line, flush=True)
    if args.out:
        same = all(np.array_equal(np.load(os.path.join(args.out, f"{k}_reuse.npy")),
                                  np.load(os.path.join(args.out, f"{k}_noreuse.npy"))) for k in ("poses", "trace"))
        print(json.dumps({"bit_identical": same}), flush=True)
    print(json.dumps({"ms_per_iter_saved": round(res[False]["ms_per_iter"] - res[True]["ms_per_iter"], 3)}), flush=True)


if __name__ == "__main__":
    main()

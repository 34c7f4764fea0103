"""Cost of rig calibration (DESIGN.md "Rig calibration"): rig_damping_iter against damping_iter on the same slots, and
the H -> H_rig reduction's kernels on their own.

Workloads: balm_synth_virtual at 500 slots (125 base poses x 4 LiDARs, 100 000 voxels: bench.py's C3 shape) and at
2 000 slots (500 x 4, 20 000 voxels) on the tensor path, and rig_ref's synthetic room rig (12 base poses x 3 LiDARs,
voxels cut at the true poses) on the fp64 path. On the synthetic scenes every LiDAR's extrinsic starts at the
identity and base b at slot 4b's pose; LiDAR 0 is fixed.

Per run, alternating on one context: ms per LM iteration (CUDA events around one call with force_hess and the
convergence exit off) of damping_iter and of rig_damping_iter, with balm_timings' ms_syrk, ms_assemble (the rig call's
includes the reduction) and ms_solve per iteration. Then, in a separate torch.profiler run of rig_evaluate, every
device kernel's time by its full name, and the reduction kernels' effective bandwidth (rig_k_kernel reads H and writes
K = H J, rig_jtk_kernel reads K and writes H_rig): the bytes of H and K they must read and write, over kernel time,
against the H100 SXM's 3.35 TB/s.

    python scripts/rig_perf.py [--runs 3] [--iters 5] [--out FILE]

Prints the card's name and power limit, then one JSON line per record; --out FILE also writes them there.
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
from balm_b200 import _lib as L  # noqa: E402

LM = dict(rel_tol=-1.0, force_hess=True, min_planes_per_pose=0, gauge_mode=2)
HBM = 3.35e12  # H100 SXM data-sheet HBM3 bandwidth, bytes/s
IDENT = np.concatenate([np.eye(3).reshape(9), np.zeros(3)])


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def synth(bases, lidars, M):
    N = bases * lidars
    c = balm_b200.Context(N, 0, L.PREC_TENSOR)
    _, init = c.synth_virtual(M, 0, 40, 0.01, 2.0, 10)  # bench.py: PTS, NOISE, RANGE, SEED
    base_of, lidar_of = np.arange(N) // lidars, np.arange(N) % lidars
    return c, init, base_of, lidar_of, init[::lidars].copy(), np.tile(IDENT, (lidars, 1))


def room():
    import rig_ref as rr
    S = rr.rig_scene()
    sc = rr.cut(S, S["base12"], S["ext12"])
    c = balm_b200.Context(sc["n_poses"], 0, L.PREC_FP64)
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
    X = rr.compose(S["base12"], S["ext12"], S["base_of"], S["lidar_of"])
    return c, X, S["base_of"], S["lidar_of"], S["base12"], S["ext12"]


WORKLOADS = [("synth 500 slots (125 x 4), 100k voxels, tensor", lambda: synth(125, 4, 100000)),
             ("synth 2000 slots (500 x 4), 20k voxels, tensor", lambda: synth(500, 4, 20000)),
             ("room rig 36 slots (12 x 3), fp64", room)]


def reduction_bytes(base_of, lidar_of, B, L_, fixed_lidars=(0,)):
    """bytes the reduction must move: H columns read by rig_k_kernel (each free unknown's slots' six columns), K
    written, the lower block rows of K read by rig_jtk_kernel once per column, and H_rig written"""
    N = len(base_of)
    n = 6 * N
    free = [("b", b) for b in range(B)] + [("l", l) for l in range(L_) if l not in fixed_lidars]
    slots = [int(np.sum(base_of == j)) if k == "b" else int(np.sum(lidar_of == j)) for k, j in free]
    nr = 6 * len(free)
    h_read = sum(6 * s * n for s in slots) * 8
    k_write = nr * n * 8
    suffix = np.cumsum(slots[::-1])[::-1]  # slots of the unknowns at and after each one
    k_read = sum(6 * 6 * int(suffix[u]) for u in range(len(free))) * 8  # column c of unknown v reads 6 rows per slot
    return dict(h_read=h_read, k_write=k_write, k_read=k_read, hrig_write=nr * nr * 8, n_rig=nr)


def timed(c, fn, iters):
    c.reset_counters()
    c.timer_begin()
    tr = fn(iters)
    ms = c.timer_end()
    tm = c.timings()
    it = len(tr)
    return dict(ms_per_iter=round(ms / it, 3), ms_syrk=round(tm["ms_syrk"] / it, 4),
                ms_assemble=round(tm["ms_assemble"] / it, 4), ms_solve=round(tm["ms_solve"] / it, 4))


def profile(c, base, ext, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    c.rig_evaluate(base, ext)
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(reps):
            c.rig_evaluate(base, ext)
    out = {}
    for e in p.key_averages():  # every device kernel of the evaluation, by name
        if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time_total > 0:
            out[e.key] = out.get(e.key, 0.0) + e.device_time_total / 1000.0
    return {k: round(v / reps, 4) for k, v in sorted(out.items(), key=lambda kv: -kv[1])}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--profile_reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    gpu = card()
    print("card:", gpu, flush=True)
    with open(a.out if a.out else os.devnull, "w") as f:
        def emit(rec):
            line = json.dumps(dict(card=gpu, **rec))
            print(line, flush=True)
            f.write(line + "\n")

        for name, make in WORKLOADS:
            c, X, base_of, lidar_of, base, ext = make()
            B, L_ = len(base), len(ext)
            n_rig = c.set_rig(base_of, lidar_of)
            plain = lambda k: c.damping_iter(X, max_iter=k, **LM)[1]
            rig = lambda k: c.rig_damping_iter(base, ext, max_iter=k, **LM)[2]
            plain(2)
            rig(2)  # warm-up of every shape
            for r in range(a.runs):
                for label, fn in (("damping_iter", plain), ("rig_damping_iter", rig)):
                    emit(dict(workload=name, call=label, run=r, n_rig=n_rig, **timed(c, fn, a.iters)))
            by = reduction_bytes(base_of, lidar_of, B, L_)
            kt = profile(c, base, ext, a.profile_reps)  # per rig_evaluate, every kernel by its full name
            rec = dict(workload=name, profile="rig_evaluate kernels", kernel_ms=kt, **by)
            for short, moved in (("rig_k_kernel", by["h_read"] + by["k_write"]),
                                 ("rig_jtk_kernel", by["k_read"] + by["hrig_write"])):
                ms = sum(v for k, v in kt.items() if short in k)
                rec[short + "_ms"] = round(ms, 4)
                rec[short + "_TBps"] = round(moved / (ms * 1e-3) / 1e12, 3)
                rec[short + "_of_peak"] = round(moved / (ms * 1e-3) / HBM, 3)
            emit(rec)
            c.close()


if __name__ == "__main__":
    main()

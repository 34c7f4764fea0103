"""Device time of the persistent sliding window (balm_window_*) on a benchmark_realworld-shaped stream, next to what a
user would otherwise re-run every shift: balm_cut_voxels on the window's points (which loses the fix clusters).

Stream: tests/assoc_ref.synthetic_scans (room 12, 75 000 points per scan, 40 scans), window 20, mg 2, one recut per
scan (the consistency.cpp loop). The fill of the first window is the warm-up; every later shift is timed:
marginalize, then per new scan cut + recut, then push (registration included). Each call ends in a device
synchronisation, so a host clock around it measures the device work. Prints one JSON line; --out FILE also writes
the per-call times there."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the numbers are still valid, but say where they came from
        q = f"nvidia-smi unavailable: {e}"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=40)
    ap.add_argument("--points", type=int, default=75000)
    ap.add_argument("--window", type=int, default=20)
    ap.add_argument("--mg", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the result with every per-call time to this JSON file")
    a = ap.parse_args()
    import assoc_ref
    import scenes
    import balm_b200
    pts, frs, poses = assoc_ref.synthetic_scans(n_poses=a.scans, pts_per_scan=a.points, seed=3, room=12.0)
    P = scenes.pack_poses([r for r, _ in poses], [p for _, p in poses])
    scans = [pts[frs == i].astype(np.float32) for i in range(a.scans)]
    kw = dict(voxel_size=2.0, layer_limit=2, min_ps=15, eigen_value_array=(1 / 16, 1 / 16, 1 / 9))
    N, mg = a.window, a.mg
    c = balm_b200.Context(N, 0, 0)
    ref = balm_b200.Context(N, 0, 0)
    c.window_reset(**kw)
    t = {k: [] for k in ("cut", "recut", "marginalize", "push", "step", "cut_voxels")}

    def timed(key, f):
        c.sync()
        t0 = time.perf_counter()
        r = f()
        c.sync()
        t[key].append(1e3 * (time.perf_counter() - t0))
        return r

    for s in range(N):                                         # warm-up: fill the first window
        c.window_cut(scans[s], P[s], s)
        c.window_recut(s + 1)
    c.window_push(N)
    win_pts = np.concatenate(scans[:N])
    win_frs = np.concatenate([np.full(len(scans[s]), s, np.int32) for s in range(N)])
    ref.cut_voxels(win_pts, win_frs, P[:N], **kw)              # warm-up of the comparison
    first, nxt, sizes = 0, N, []
    while nxt + mg <= a.scans:
        x = P[first:first + N]
        t0 = time.perf_counter()
        timed("marginalize", lambda: c.window_marginalize(mg, x, N))
        first += mg
        for j in range(mg):
            slot = N - mg + j
            timed("cut", lambda: c.window_cut(scans[nxt + j], P[nxt + j], slot))
            timed("recut", lambda: c.window_recut(slot + 1))
        M, K = timed("push", lambda: c.window_push(N))
        t["step"].append(1e3 * (time.perf_counter() - t0))
        nxt += mg
        idx = range(first, first + N)
        win_pts = np.concatenate([scans[s] for s in idx])
        win_frs = np.concatenate([np.full(len(scans[s]), s - first, np.int32) for s in idx])
        Mr, Kr = timed("cut_voxels", lambda: ref.cut_voxels(win_pts, win_frs, P[first:first + N], **kw))
        sizes.append(dict(window_voxels=M, window_obs=K, cut_voxels_voxels=Mr, cut_voxels_obs=Kr, window_points=len(win_pts)))
    res = dict(gpu=gpu_info(), scans=a.scans, points_per_scan=a.points, window=N, mg=mg, shifts=len(t["step"]),
               ms_median={k: float(np.median(v)) for k, v in t.items()},
               ms_min={k: float(np.min(v)) for k, v in t.items()}, per_shift=sizes)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(res, ms_all=t), f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""balm_cut_voxels in root-key slabs, measured on the GPU (DESIGN.md section 7, "Association for drives of any length").

  python scripts/assoc_slabs_perf.py [--street-points 1e8] [--drive-scans 20000] [--drive-points-per-scan 110000]
                                     [--skip-drive] [--out result.json]

1. A synthetic street of about 1e8 points (tests/street_ref.py scans) cut in one pass (BALM_ASSOC_BUDGET_MB raised above
   the one-pass bound: the cut itself needs far less than the bound) and in slabs under the default 16 GB budget: wall
   time of each, the accounted peak scratch, the slab stats, and whether the two registrations are bitwise equal.
2. A drive of more than 2^31 points (about 34 GB of host arrays: one street scan repeated at every pose of a 20 km
   straight drive, which sees the same street from every position) cut under the default budget, then 5 LM iterations
   on PREC_BLOCKS: slab stats, the share of time in the root-count pass, the selection, the per-slab cuts and the
   registration, and the one-pass call's accounted scratch bound (the one-pass call is not run: it cannot fit).
The card's name and power limit are read in the same run. Needs a CUDA device; skips step 2 without 48 GB of free host
memory."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import balm_b200  # noqa: E402
import scenes  # noqa: E402
import street_ref  # noqa: E402
from balm_b200 import _lib as L  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def mem_available_gb():
    for line in open("/proc/meminfo"):
        if line.startswith("MemAvailable:"):
            return int(line.split()[1]) / 2 ** 20
    return 0.0


def poses12(poses):
    return scenes.pack_poses([r for r, _ in poses], [p for _, p in poses])


def timed_cut(c, xyz, frame, p12, budget_mb=None):
    old = os.environ.pop("BALM_ASSOC_BUDGET_MB", None)
    if budget_mb is not None:
        os.environ["BALM_ASSOC_BUDGET_MB"] = str(budget_mb)
    try:
        t = time.perf_counter()
        M, K = c.cut_voxels(xyz, frame, p12)
        ms = 1e3 * (time.perf_counter() - t)
    finally:
        os.environ.pop("BALM_ASSOC_BUDGET_MB", None)
        if old is not None:
            os.environ["BALM_ASSOC_BUDGET_MB"] = old
    return dict(ms=ms, M=M, K=K, **c.cut_stats())


def street(n_points):
    per_scan = 100_000
    n_scans = max(2, int(n_points) // per_scan)
    pts, frs, poses = street_ref.street_scans(n_forward=n_scans - n_scans // 10, n_revisit=n_scans // 10,
                                              pts_per_scan=per_scan, step=2.0)
    xyz = pts.astype(np.float32)
    del pts
    p12 = poses12(poses)
    c = balm_b200.Context(len(poses), 0, L.PREC_FP64)
    n = len(frs)
    timed_cut(c, xyz[:200000], frs[:200000], p12)  # warm-up (module load, cub's first launches)
    stats = c.cut_stats()
    bound = stats["scratch_per_point"] * n + stats["scratch_fixed"]
    one_budget_mb = bound / 2 ** 20 + 1
    runs = {}
    for rep in range(2):  # alternate the two paths
        for name, b in (("one_pass", one_budget_mb), ("slabs", None)):
            r = timed_cut(c, xyz, frs, p12, b)
            runs.setdefault(name, []).append(r)
            if rep == 0:
                runs[name + "_voxels"] = (*c.download_voxels(), *c.download_keys(with_layers=True))
    same = all(np.array_equal(a, b) for a, b in zip(runs.pop("one_pass_voxels"), runs.pop("slabs_voxels")))
    c.close()
    return dict(points=n, scans=len(poses), one_pass_bound_bytes=bound, bitwise_equal=same, **runs)


def long_drive(n_scans, per_scan):
    """one street scan, seen from every pose of a straight drive along x: the facades and the ground are the same at
    every position, so each scan is the template in its own body frame"""
    tpl, _, tpl_poses = street_ref.street_scans(n_forward=1, n_revisit=0, pts_per_scan=per_scan, rng_m=20.0)
    R0, p0 = tpl_poses[0]
    tpl = tpl.astype(np.float32)
    rng = np.random.default_rng(2)
    n = n_scans * per_scan
    t = time.perf_counter()
    xyz = np.empty((n, 3), dtype=np.float32)
    for s in range(n_scans):
        xyz[s * per_scan:(s + 1) * per_scan] = tpl
    frame = np.repeat(np.arange(n_scans, dtype=np.int32), per_scan)
    gen_s = time.perf_counter() - t
    gt = [(R0, p0 + np.array([1.0 * s, 0.0, 0.0])) for s in range(n_scans)]
    init = [(R @ scenes.exp_so3(rng.normal(0, 0.001, 3)), p + rng.normal(0, 0.01, 3)) for R, p in gt]
    init[0] = gt[0]
    p12 = poses12(init)
    c = balm_b200.Context(n_scans, 0, L.PREC_BLOCKS)
    r = timed_cut(c, xyz, frame, p12)
    host_gb = (xyz.nbytes + frame.nbytes) / 1e9
    del xyz, frame
    parts = {k: r[k] for k in ("ms_roots", "ms_select", "ms_cut", "ms_register")}
    total = sum(parts.values())
    r["share"] = {k: v / total for k, v in parts.items()}
    r["restream_factor"] = (r["h2d_bytes"] - 84 * r["K"] - 28 * r["M"]) / (16.0 * n) - 1.0  # root pass = 1 upload
    r["one_pass_bound_bytes"] = r["scratch_per_point"] * n + r["scratch_fixed"]
    t = time.perf_counter()
    poses, trace, _ = c.damping_iter(p12, max_iter=5, min_planes_per_pose=0)
    lm_ms = 1e3 * (time.perf_counter() - t)
    c.close()
    return dict(points=n, scans=n_scans, host_array_gb=host_gb, generate_s=gen_s, cut=r, lm_iterations=len(trace),
                lm_ms=lm_ms, lm_cost=[trace[0]["r1"], trace[-1]["r2"]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--street-points", type=float, default=1e8)
    ap.add_argument("--drive-scans", type=int, default=20000)
    ap.add_argument("--drive-points-per-scan", type=int, default=110000)
    ap.add_argument("--skip-drive", action="store_true")
    ap.add_argument("--out", default=None, help="also write the result to this JSON file")
    a = ap.parse_args()
    out = dict(card=card())
    out["street"] = street(a.street_points)
    print(json.dumps(out, default=float), flush=True)
    need_gb = a.drive_scans * a.drive_points_per_scan * 16 / 2 ** 30 + 12
    if a.skip_drive:
        out["drive"] = "skipped"
    elif mem_available_gb() < need_gb:
        out["drive"] = f"skipped: {mem_available_gb():.0f} GB of host memory available, {need_gb:.0f} GB needed"
    else:
        out["drive"] = long_drive(a.drive_scans, a.drive_points_per_scan)
    out["card_after"] = card()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1, default=float)
    print(json.dumps(out, default=float))


if __name__ == "__main__":
    main()

"""Wall time of hierarchical BA (balm_b200.hba) per layer and for the whole pyramid, with the keyframes merged on the
device (Batch.merge_scans) against the same pyramid with keyframes built on the host by the numpy restatement
(tests/hba_ref.keyframe_ref, which a caller without the device merge would write: download, transform, down-sample).

Workload: 177 synthetic scans of 75 000 points (assoc_ref.synthetic_scans, room 12; the size of benchmark_realworld),
windows of 10 scans every 5, keyframes down-sampled at 0.1 m: 35 windows, then 6, then a top window of 6. Both routes
run in one process, device first (once to warm up every shape, then --repeats times), then the host route; every batch
call ends in a device synchronisation, so the host clock around a call measures its device work. The two routes must
give bitwise-equal poses, statuses and keyframe sizes. Then the device route again with the pose graph
(hba(pose_graph=True)): its total, the pose graph's own wall time, factor count and LM iterations. Prints one JSON line;
--out FILE also writes it there."""
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


def host_merge(self, scans, windows, poses_list, voxel_size):
    import hba_ref
    return [hba_ref.keyframe_ref(scans, w, p, voxel_size) for w, p in zip(windows, poses_list)]


def run(scans, poses, host, pose_graph=False):
    from balm_b200 import Batch, hba
    device_merge = Batch.merge_scans
    if host:
        Batch.merge_scans = host_merge
    try:
        t0 = time.perf_counter()
        res = hba.hba(scans, poses, downsample=0.1, pose_graph=pose_graph)
        total = 1e3 * (time.perf_counter() - t0)
    finally:
        Batch.merge_scans = device_merge
    return res, total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=177)
    ap.add_argument("--points", type=int, default=75000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import assoc_ref
    import scenes
    pts, frs, poses = assoc_ref.synthetic_scans(n_poses=a.scans, pts_per_scan=a.points, room=12.0)
    scans = [pts[frs == i].astype(np.float32) for i in range(a.scans)]
    del pts, frs
    p12 = scenes.pack_poses([r for r, _ in poses], [p for _, p in poses])
    out = dict(gpu=gpu_info(), scans=a.scans, points_per_scan=a.points, window=10, stride=5, downsample=0.1)
    run(scans, p12, host=False)  # warm-up
    dev = [run(scans, p12, host=False) for _ in range(a.repeats)]
    host = run(scans, p12, host=True)

    def layers(res):
        return [dict(windows=len(l["windows"]), cut_ms=l["ms"]["cut"], lm_ms=l["ms"]["lm"], merge_ms=l["ms"]["merge"],
                     iters=int(sum(l["n_iters"])), not_ok=int(sum(s != 0 for s in l["status"])),
                     kf_points=None if l["kf_sizes"] is None else int(sum(l["kf_sizes"])),
                     kf_min_max=None if l["kf_sizes"] is None else [min(l["kf_sizes"]), max(l["kf_sizes"])])
                for l in res["layers"]]
    out["device"] = dict(total_ms=[t for _, t in dev], layers=[layers(r) for r, _ in dev])
    out["host_merge"] = dict(total_ms=host[1], layers=layers(host[0]))
    r0, h0 = dev[0][0], host[0]
    out["bitwise_equal"] = bool(np.array_equal(r0["poses"], h0["poses"]) and all(
        x["status"] == y["status"] and x["kf_sizes"] == y["kf_sizes"] for x, y in zip(r0["layers"], h0["layers"])))
    out["device_runs_bitwise_equal"] = bool(all(np.array_equal(r["poses"], r0["poses"]) for r, _ in dev))
    pgr = [run(scans, p12, host=False, pose_graph=True) for _ in range(a.repeats)]
    out["pose_graph"] = dict(total_ms=[t for _, t in pgr], pose_graph_ms=[r["pose_graph"]["ms"] for r, _ in pgr],
                             factors=pgr[0][0]["pose_graph"]["n_factors"],
                             not_pd=int(sum(s != 0 for s in pgr[0][0]["pose_graph"]["status"])),
                             iters=len(pgr[0][0]["pose_graph"]["trace"]),
                             runs_bitwise_equal=bool(all(np.array_equal(r["poses"], pgr[0][0]["poses"]) for r, _ in pgr)))
    s = json.dumps(out)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")
    print(s)


if __name__ == "__main__":
    main()

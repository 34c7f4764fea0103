"""Hierarchical bundle adjustment on one batch: the layers of HBA's pyramid up to a single top window.

A bottom layer alone (windows of `length` scans every `stride` scans, one BALM window per problem) refines each window's
poses relative to its first scan only; the anchors keep their initial poses, so drift along the trajectory stays. Here
every layer runs on the device as three batch calls: Batch.cut_scans, Batch.damping_iter and Batch.merge_scans, whose
keyframe w (window w's scans in the body frame of its slot 0, down-sampled) becomes item w of the next layer, with the
input pose of the window's slot 0 as its input pose. Layers are built while there are more items than `top_size`; then
one window over all remaining items is the top. The result is carried back down with relative poses only:

    item i of a layer gets  F_w . T_w,0^-1 . T_w,slot(i)

with w the lowest-index window containing i, T that window's refined poses (its input poses when its status is not
BALM_OK) and F_w the final pose of keyframe w. The top's F is the input pose of its slot 0, so the result is in the
input's world frame.

With pose_graph=True the placement above is only the start: every converged window of every layer becomes a factor over
the scans its items stand for (its relative poses, weighted by its BA Hessian; include/balm_b200.h,
balm_set_pose_factors), and one LM solve over all scans fuses them into one trajectory, re-anchored so that scan 0 keeps
its input pose. That solve is dense (Context.pose_graph_iter) for short trajectories and block-sparse (PoseGraph) from
PG_SPARSE_MIN_POSES scans on, so that trajectories of any length fit on the device.

python -m balm_b200.hba --file_path DIR [--out refined.csv] runs it on a benchmark_realworld directory."""
import argparse
import sys
import time

import numpy as np

from . import _lib as L
from . import drivers, io
from .context import Batch, Context, PoseGraph

MAX_POSES = 32  # BALM_BATCH_MAX_POSES
# fuse_windows' crossover from the context's dense pose-graph solve to the sparse one (DESIGN.md "Pose graph",
# scripts/pose_graph_perf.py): measured on an H100, the sparse iteration is faster from here on.
PG_SPARSE_MIN_POSES = 1000
DEFAULT_ASSOC = dict(voxel_size=2.0, layer_limit=2, min_ps=15, eigen_value_array=(1.0 / 16, 1.0 / 16, 1.0 / 9))


def layer_windows(n, length=10, stride=5):
    """Windows of `length` items every `stride` items, the last one cut at n."""
    out, s = [], 0
    while True:
        out.append(list(range(s, min(s + length, n))))
        if s + length >= n:
            return out
        s += stride


def _split(x):
    x = np.asarray(x, dtype=np.float64)
    return x[:9].reshape(3, 3).T, x[9:]  # R row-major, t


def _pack(R, t):
    return np.concatenate([R.T.reshape(9), t])


def relative_chain(F, T0, Tk):
    """F . T0^-1 . Tk of three 12-vectors (R column-major, then t)."""
    RF, tF = _split(F)
    R0, t0 = _split(T0)
    Rk, tk = _split(Tk)
    A = RF @ R0.T
    return _pack(A @ Rk, A @ (tk - t0) + tF)


def propagate(layers):
    """Final poses of the bottom layer's items from the layers hba() records (bottom first, the top last): per layer its
    windows, poses_in (the items' input poses) and poses (per window, the poses its items are carried with)."""
    F = None
    for lay in reversed(layers):
        wins, T = lay["windows"], lay["poses"]
        if F is None:  # the top: slot 0 stays at its input pose
            F = [lay["poses_in"][wins[0][0]]]
        n = len(lay["poses_in"])
        out = [None] * n
        for w, win in enumerate(wins):
            for k, i in enumerate(win):
                if out[i] is None:
                    out[i] = relative_chain(F[w], T[w][0], T[w][k])
        F = out
    return np.array(F)


def fuse_windows(poses_in, poses0, factors, device=0, priors=None):
    """The pose graph's LM (gauge_mode 2) over all scans from poses0, then re-anchored so that scan 0 keeps its input
    pose poses_in[0] -> (poses, dict(status, trace, n_factors, ms)). From PG_SPARSE_MIN_POSES scans on it runs on the
    sparse solve (PoseGraph), below on the context's dense one. priors (set_pose_priors' dicts, by scan index) join the
    pose graph; with any, the result is already in the priors' frame and is not re-anchored (the dict also holds
    prior_status)."""
    t0 = time.perf_counter()
    c = PoseGraph(len(poses0), device) if len(poses0) >= PG_SPARSE_MIN_POSES else Context(len(poses0), device)
    try:
        status = c.set_pose_factors(factors)
        prior_status = c.set_pose_priors(priors) if priors else []
        x, trace = c.pose_graph_iter(poses0, gauge_mode=2)
    finally:
        c.close()
    if not priors:
        x = np.array([relative_chain(poses_in[0], x[0], p) for p in x])
    info = dict(status=status, trace=trace, n_factors=len(factors), ms=1e3 * (time.perf_counter() - t0))
    if priors:
        info["prior_status"] = prior_status
    return x, info


def hba(scans, poses12, length=10, stride=5, downsample=0.1, assoc=None, device=0, top_size=MAX_POSES,
        pose_graph=False, priors=None, voxel_loss=None, **lm_opts):
    """scans: list of (n_s x 3) body-frame points; poses12: P x 12 initial poses. downsample: the keyframes' voxel edge
    (< 0.001: keyframes keep every point); assoc: cut_scans options (DEFAULT_ASSOC when None); lm_opts: damping_iter
    options of every window. Layers are built while more than top_size (<= 32) items remain.
    -> dict(poses = P x 12 final poses, layers = per layer, bottom first and the top last: windows, status, n_iters,
    n_voxels, poses_in (the items' input poses), poses (per window the poses carried down), kf_sizes (None at the top)
    and ms (wall times of cut, lm and merge)). pose_graph: the final poses come from the pose graph over every converged
    window with at least 2 items, started from the propagated ones; the result then also holds pose_graph = dict(status
    per factor, trace, n_factors, ms). priors (pose_graph only): absolute pose priors by scan index, in
    Context.set_pose_priors' format (e.g. position_priors of GNSS fixes); they join that pose graph, and the final poses
    are then in the priors' frame rather than re-anchored to scan 0. voxel_loss: None, or (kind, scale) as
    Batch.set_voxel_loss takes them: a robust voxel cost in every layer's BA, whose weighted H the pose graph's window
    factors then carry."""
    if priors and not pose_graph:
        raise ValueError("hba: priors join the top pose graph: pass pose_graph=True")
    if not (2 <= length <= MAX_POSES and 1 <= stride <= length and 1 <= top_size <= MAX_POSES):
        raise ValueError("hba: needs 2 <= length <= 32, 1 <= stride <= length and 1 <= top_size <= 32")
    poses12 = np.asarray(poses12, dtype=np.float64).reshape(-1, 12)
    if len(scans) != len(poses12) or len(scans) == 0:
        raise ValueError("hba: one pose per scan, at least one scan")
    assoc = dict(DEFAULT_ASSOC if assoc is None else assoc)
    items, x = list(scans), poses12
    scan_of = list(range(len(scans)))  # the bottom scan every item stands for: keyframe w is window w's slot 0
    layers, factors = [], []
    b = Batch(device)
    try:
        if voxel_loss is not None:
            b.set_voxel_loss(*voxel_loss)
        while True:
            top = len(items) <= top_size
            windows = [list(range(len(items)))] if top else layer_windows(len(items), length, stride)
            wposes = [x[w] for w in windows]
            t0 = time.perf_counter()
            mk = b.cut_scans(items, windows, wposes, **assoc)
            t1 = time.perf_counter()
            res = b.damping_iter(wposes, **lm_opts)
            t2 = time.perf_counter()
            T = [p if st == L.OK else wp for (st, p, _, _), wp in zip(res, wposes)]
            lay = dict(windows=windows, status=[r[0] for r in res], n_iters=[len(r[2]) for r in res],
                       n_voxels=[m for m, _ in mk], poses_in=x, poses=T, kf_sizes=None,
                       ms=dict(cut=1e3 * (t1 - t0), lm=1e3 * (t2 - t1), merge=0.0))
            layers.append(lay)
            if pose_graph:
                for win, st, (H, _, _), Tw in zip(windows, lay["status"], b.evaluate(T), T):
                    if st == L.OK and len(win) >= 2:
                        factors.append(dict(poses=[scan_of[i] for i in win], poses_hat=Tw, H=H))
            if top:
                break
            kfs = b.merge_scans(items, windows, T, downsample)
            lay["ms"]["merge"] = 1e3 * (time.perf_counter() - t2)
            lay["kf_sizes"] = [len(k) for k in kfs]
            items, x = kfs, np.array([wp[0] for wp in wposes])
            scan_of = [scan_of[w[0]] for w in windows]
    finally:
        b.close()
    res = dict(poses=propagate(layers), layers=layers)
    if pose_graph:
        if factors:
            res["poses"], res["pose_graph"] = fuse_windows(poses12, res["poses"], factors, device, priors)
        else:
            res["pose_graph"] = dict(status=[], trace=[], n_factors=0, ms=0.0)
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--file_path", required=True, help="directory with alidarPose.csv and full<i>.pcd")
    ap.add_argument("--voxel_size", type=float, default=2.0, help="root voxel edge of the association")
    ap.add_argument("--length", type=int, default=10, help="scans (keyframes) per window")
    ap.add_argument("--stride", type=int, default=5, help="first scans of consecutive windows this far apart")
    ap.add_argument("--downsample", type=float, default=0.1, help="voxel edge of the keyframes")
    ap.add_argument("--top_size", type=int, default=MAX_POSES, help="one top window once at most this many items remain")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--max_scans", type=int, default=None, help="use only the first scans")
    ap.add_argument("--out", default=None, help="write the refined poses in alidarPose.csv format")
    ap.add_argument("--pose_graph", action="store_true", help="fuse every window's relative poses in a pose graph")
    drivers.add_voxel_loss_args(ap)
    a = ap.parse_args(argv)
    R, p, _, scans = io.read_realworld_dir(a.file_path, a.max_scans)
    if len(R) == 0:
        raise ValueError("no poses read")
    R0, p0 = R[0].copy(), p[0].copy()  # re-anchored to pose 0 as benchmark_realworld.cpp:163-168
    p = (p - p0) @ R0
    R = np.einsum("ji,njk->nik", R0, R)
    print("The size of poses: %d" % len(R))
    assoc = dict(DEFAULT_ASSOC, voxel_size=a.voxel_size)
    res = hba(scans, drivers.pack_poses(R, p), a.length, a.stride, a.downsample, assoc, a.device, a.top_size,
              pose_graph=a.pose_graph, voxel_loss=drivers.voxel_loss_arg(ap, a))
    for li, lay in enumerate(res["layers"]):
        guard = sum(st == L.ERR_TOO_FEW_PLANES for st in lay["status"])
        print("layer %d: %d windows, %d iterations, voxels %d, keyframe points %s, cut %.1f ms, LM %.1f ms, merge %.1f ms"
              % (li, len(lay["windows"]), sum(lay["n_iters"]), sum(lay["n_voxels"]),
                 "-" if lay["kf_sizes"] is None else sum(lay["kf_sizes"]), lay["ms"]["cut"], lay["ms"]["lm"],
                 lay["ms"]["merge"]))
        if guard:  # bavoxel.hpp:1079-1085, per window: that window keeps its input poses
            print("%d windows: Initial error too large." % guard)
            print("Please loose plane determination criteria for more planes.")
    if a.pose_graph:
        pg = res["pose_graph"]
        tr = pg["trace"]
        final = "-" if not tr else "%.6g -> %.6g" % (tr[0]["r1"], tr[-1]["r2"] if tr[-1]["accepted"] else tr[-1]["r1"])
        print("pose graph: %d factors (%d not positive definite), %d iterations, cost %s, %.1f ms"
              % (pg["n_factors"], sum(st == L.ERR_NOT_PD for st in pg["status"]), len(tr), final, pg["ms"]))
    if a.out:
        Rf, pf = drivers.unpack_poses(res["poses"])
        io.write_pose_csv(a.out, Rf, pf)
        print("refined poses ->", a.out)
    return 0


if __name__ == "__main__":
    sys.exit(main())

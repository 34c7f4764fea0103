"""Device time of the batched bundle adjustment (balm_b200.Batch) next to what a caller does without it: one Context per
pose count and, for every window, set_voxels + damping_iter, on the fp64 and on the tensor path.

Workloads (HBA's bottom layer splits a trajectory into many short windows): (a) 256 windows x 10 poses x 1 000 planes,
(b) 32 windows x 32 poses x 5 000 planes, and (c) one bottom layer from raw scans: 160 synthetic scans of 20 000
points (assoc_ref.synthetic_scans, room 12), windows of 10 scans every 5 scans (31 windows), associated per window and as
one batch (see run_from_scans), (d) the pose covariance of the windows of (a) and (b) with fix clusters (see
run_covariance), (e) a Monte Carlo sliding window of 64 sequences (see run_sliding_window), (f) the same on the persistent window
maps (see run_persistent_window). For (a) and (b) every window is generated on the GPU by Context.synth_virtual (its own seed) and
read back with download_voxels, so the batch and the loop run on the same host arrays. Two option sets: fixed work
(force_hess, rel_tol < 0, 10 iterations: every LM iteration does the same work) and the defaults. The batch, the fp64 loop
and the tensor loop alternate --repeats times in one process; every call ends in a device synchronisation, so a host clock
around it measures the device work. Registration (set_problems / set_voxels) is timed apart from the LM calls.
A separate torch.profiler run of one fixed-work batch call gives the device time per kernel.
Prints one JSON line; --out FILE also writes it there."""
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


def make_windows(n_windows, n_poses, n_planes, seed0):
    import balm_b200
    c = balm_b200.Context(n_poses, 0, balm_b200.PREC_FP64)
    probs, init = [], []
    for w in range(n_windows):
        _, x0 = c.synth_virtual(n_planes, seed=seed0 + w)
        row_ptr, pose_idx, obs10, coe = c.download_voxels()
        probs.append(dict(n_poses=n_poses, row_ptr=row_ptr, pose_idx=pose_idx, obs10=obs10, coe=coe))
        init.append(x0)
    c.close()
    return probs, init


def run_workload(name, n_windows, n_poses, n_planes, repeats, seed0):
    import balm_b200
    probs, init = make_windows(n_windows, n_poses, n_planes, seed0)
    options = {"fixed": dict(max_iter=10, force_hess=True, rel_tol=-1.0, gauge_mode=2),
               "default": dict()}
    batch = balm_b200.Batch(0)
    ctx = {p: balm_b200.Context(n_poses, 0, p) for p in (balm_b200.PREC_FP64, balm_b200.PREC_TENSOR)}
    out = dict(windows=n_windows, poses=n_poses, planes=n_planes)

    def clock(f):
        t0 = time.perf_counter()
        r = f()
        return r, 1e3 * (time.perf_counter() - t0)

    def loop(c, kw):
        poses, reg, lm, iters = [], 0.0, 0.0, []
        for pr, x0 in zip(probs, init):
            _, t = clock(lambda: c.set_voxels(pr["row_ptr"], pr["pose_idx"], pr["obs10"], pr["coe"]))
            reg += t
            (p, tr, _), t = clock(lambda: c.damping_iter(x0, **kw))
            lm += t
            poses.append(p)
            iters.append(len(tr))
        return poses, reg, lm, iters

    for key, kw in options.items():
        ms = {k: [] for k in ("batch_register", "batch_lm", "fp64_register", "fp64_lm", "tensor_register", "tensor_lm")}
        for rep in range(repeats + 1):  # the first round warms up every shape
            _, t_reg = clock(lambda: batch.set_problems(probs))
            res, t_lm = clock(lambda: batch.damping_iter(init, **kw))
            p64, r64, l64, it64 = loop(ctx[balm_b200.PREC_FP64], kw)
            ptc, rtc, ltc, _ = loop(ctx[balm_b200.PREC_TENSOR], kw)
            if rep == 0:
                continue
            for k, v in (("batch_register", t_reg), ("batch_lm", t_lm), ("fp64_register", r64), ("fp64_lm", l64),
                         ("tensor_register", rtc), ("tensor_lm", ltc)):
                ms[k].append(v)
        dpose = max(float(np.abs(r[1] - p).max()) for r, p in zip(res, p64))
        iters = [len(r[2]) for r in res]
        out[key] = dict(ms=ms, ms_median={k: float(np.median(v)) for k, v in ms.items()},
                        batch_iters_total=int(sum(iters)), loop_iters_total=int(sum(it64)),
                        max_pose_diff_batch_vs_fp64_loop=dpose,
                        same_iteration_counts=bool(iters == it64))
    # one profiled fixed-work call of its own: device time per kernel, summed over the call
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        batch.set_problems(probs)
        batch.damping_iter(init, **options["fixed"])
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            batch.damping_iter(init, **options["fixed"])
            torch.cuda.synchronize()
        per = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = e.cuda_time_total
            if t > 0:
                per[e.key] = dict(ms=t / 1e3, calls=e.count)
        out["profile_fixed_ms_per_kernel"] = per
    except Exception as e:  # the end-to-end numbers above stand on their own
        out["profile_fixed_ms_per_kernel"] = f"profiler failed: {e}"
    batch.close()
    for c in ctx.values():
        c.close()
    return out


def world_cluster(o10, p12):
    """An observation's cluster moved to the world frame by its pose (PointCluster::transform)."""
    R, t = p12[:9].reshape(3, 3).T, p12[9:]
    P = np.array([[o10[0], o10[1], o10[2]], [o10[1], o10[3], o10[4]], [o10[2], o10[4], o10[5]]])
    v, n = o10[6:9], o10[9]
    Rv = R @ v
    Pw = R @ P @ R.T + np.outer(Rv, t) + np.outer(t, Rv) + n * np.outer(t, t)
    vw = Rv + n * t
    return np.array([Pw[0, 0], Pw[0, 1], Pw[0, 2], Pw[1, 1], Pw[1, 2], Pw[2, 2], vw[0], vw[1], vw[2], n])


def run_covariance(name, n_windows, n_poses, n_planes, repeats, seed0):
    """Workload (d): the windows of (a) or (b), each voxel given a fix cluster (its pose-0 observation in the world
    frame at the true poses, what marginalising that scan leaves behind), optimised by one Batch.damping_iter; then
    the pose covariance at the optimum, isotropic point noise 0.01, fix clusters included: (i) a Context (fp64) per
    window, pose_covariance only (set_voxels done beforehand), (ii) the same with set_voxels inside the timed loop,
    (iii) one Batch.pose_covariance. Medians over the repeats, after one warm-up round."""
    import balm_b200
    c = balm_b200.Context(n_poses, 0, balm_b200.PREC_FP64)
    probs, init = [], []
    for w in range(n_windows):
        gt, x0 = c.synth_virtual(n_planes, seed=seed0 + w)
        row_ptr, pose_idx, obs10, coe = c.download_voxels()
        fix10 = np.stack([world_cluster(obs10[row_ptr[v]], gt[pose_idx[row_ptr[v]]]) for v in range(len(coe))])
        probs.append(dict(n_poses=n_poses, row_ptr=row_ptr, pose_idx=pose_idx, obs10=obs10, coe=coe, fix10=fix10))
        init.append(x0)
    c.close()
    batch = balm_b200.Batch(0)
    batch.set_problems(probs)
    res = batch.damping_iter(init, hess_includes_fix=True, gauge_mode=2)
    poses = [r[1] for r in res]
    ctx = balm_b200.Context(n_poses, 0, balm_b200.PREC_FP64)
    kw = dict(point_noise=0.01, include_fix=True)

    def clock(f):
        t0 = time.perf_counter()
        r = f()
        return r, 1e3 * (time.perf_counter() - t0)

    def loop(register_inside):
        out, t = [], 0.0
        for pr, x in zip(probs, poses):
            if register_inside:
                (raw, cov), dt = clock(lambda: (ctx.set_voxels(pr["row_ptr"], pr["pose_idx"], pr["obs10"], pr["coe"],
                                                               pr["fix10"]), ctx.pose_covariance(x, **kw))[1])
            else:
                ctx.set_voxels(pr["row_ptr"], pr["pose_idx"], pr["obs10"], pr["coe"], pr["fix10"])
                (raw, cov), dt = clock(lambda: ctx.pose_covariance(x, **kw))
            t += dt
            out.append((raw, cov))
        return out, t

    ms = {k: [] for k in ("i_context_cov", "ii_context_register_and_cov", "iii_batch_cov")}
    for rep in range(repeats + 1):
        ref, t_i = loop(False)
        _, t_ii = loop(True)
        got, t_iii = clock(lambda: batch.pose_covariance(poses, **kw))
        if rep == 0:
            continue
        for k, v in zip(ms, (t_i, t_ii, t_iii)):
            ms[k].append(v)
    rel = lambda a, b: float(np.abs(a - b).max() / np.abs(b).max())
    out = dict(windows=n_windows, poses=n_poses, planes=n_planes, ms=ms,
               ms_median={k: float(np.median(v)) for k, v in ms.items()},
               statuses=sorted({g[0] for g in got}),
               max_rel_diff_raw_batch_vs_context=max(rel(g[1], r[0]) for g, r in zip(got, ref)),
               max_rel_diff_cov_batch_vs_context=max(rel(g[2], r[1]) for g, r in zip(got, ref)))
    try:  # one profiled batch call of its own: device time per kernel
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            batch.pose_covariance(poses, **kw)
            torch.cuda.synchronize()
        out["profile_ms_per_kernel"] = {e.key: dict(ms=getattr(e, "device_time_total", 0) / 1e3, calls=e.count)
                                        for e in prof.key_averages() if getattr(e, "device_time_total", 0) > 0}
    except Exception as e:
        out["profile_ms_per_kernel"] = f"profiler failed: {e}"
    batch.close()
    ctx.close()
    return out


def layer_windows(n, length=10, stride=5):
    out, s = [], 0
    while True:
        out.append(list(range(s, min(s + length, n))))
        if s + length >= n:
            return out
        s += stride


def run_from_scans(n_scans, pts_per_scan, room, repeats):
    """Workload (c), one HBA bottom layer from raw scans: (i) a Context per window, cut_voxels + damping_iter; (ii) per
    window cut_voxels + download_voxels, then Batch.set_problems + damping_iter; (iii) Batch.cut_scans + damping_iter.
    Association + registration and LM are timed apart."""
    import assoc_ref
    import scenes
    import balm_b200
    pts, frs, poses = assoc_ref.synthetic_scans(n_poses=n_scans, pts_per_scan=pts_per_scan, room=room)
    scans = [pts[frs == i].astype(np.float32) for i in range(n_scans)]
    p12 = scenes.pack_poses([r for r, _ in poses], [p for _, p in poses])
    windows = layer_windows(n_scans)
    wposes = [p12[w] for w in windows]
    wpts = [np.concatenate([scans[s] for s in w]) for w in windows]
    wfr = [np.concatenate([np.full(len(scans[s]), k, dtype=np.int32) for k, s in enumerate(w)]) for w in windows]
    kwc = dict(voxel_size=2.0, eigen_value_array=(1 / 16, 1 / 16, 1 / 9))
    options = {"fixed": dict(max_iter=10, force_hess=True, rel_tol=-1.0, gauge_mode=2, min_planes_per_pose=0),
               "default": dict(min_planes_per_pose=0)}
    ctx = {n: balm_b200.Context(n, 0, balm_b200.PREC_FP64) for n in {len(w) for w in windows}}
    batch = balm_b200.Batch(0)
    out = dict(scans=n_scans, pts_per_scan=pts_per_scan, windows=len(windows), window=10, stride=5,
               points_replicated=int(sum(len(x) for x in wpts)))

    def clock(f):
        t0 = time.perf_counter()
        r = f()
        return r, 1e3 * (time.perf_counter() - t0)

    for key, kw in options.items():
        ms = {k: [] for k in ("i_assoc", "i_lm", "ii_assoc_register", "ii_lm", "iii_cut", "iii_lm")}
        for rep in range(repeats + 1):  # the first round warms up every shape
            ta = tl = 0.0
            p_i = []
            for w, x0 in enumerate(wposes):
                c = ctx[len(windows[w])]
                _, t = clock(lambda: c.cut_voxels(wpts[w], wfr[w], x0, **kwc))
                ta += t
                (p, _, _), t = clock(lambda: c.damping_iter(x0, **kw))
                tl += t
                p_i.append(p)

            def per_window():
                probs = []
                for w, x0 in enumerate(wposes):
                    c = ctx[len(windows[w])]
                    c.cut_voxels(wpts[w], wfr[w], x0, **kwc)
                    rp, pi, ob, co = c.download_voxels()
                    probs.append(dict(n_poses=len(windows[w]), row_ptr=rp, pose_idx=pi, obs10=ob, coe=co))
                batch.set_problems(probs)
            _, t_ii = clock(per_window)
            r_ii, l_ii = clock(lambda: batch.damping_iter(wposes, **kw))
            _, t_iii = clock(lambda: batch.cut_scans(scans, windows, wposes, **kwc))
            r_iii, l_iii = clock(lambda: batch.damping_iter(wposes, **kw))
            if rep == 0:
                continue
            for k, v in (("i_assoc", ta), ("i_lm", tl), ("ii_assoc_register", t_ii), ("ii_lm", l_ii), ("iii_cut", t_iii),
                         ("iii_lm", l_iii)):
                ms[k].append(v)
        out[key] = dict(ms=ms, ms_median={k: float(np.median(v)) for k, v in ms.items()},
                        ii_iii_poses_bitwise_equal=bool(all(np.array_equal(a[1], b[1]) for a, b in zip(r_ii, r_iii))),
                        max_pose_diff_iii_vs_i=max(float(np.abs(a[1] - b).max()) for a, b in zip(r_iii, p_i)),
                        iters_iii=[len(r[2]) for r in r_iii])
    try:  # one profiled cut_scans call of its own: device time per kernel
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            batch.cut_scans(scans, windows, wposes, **kwc)
            torch.cuda.synchronize()
        per = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = e.cuda_time_total
            if t > 0 or "cuda" in e.key.lower():
                per[e.key] = dict(device_ms=t / 1e3, host_ms=e.cpu_time_total / 1e3, calls=e.count)
        out["profile_cut_scans"] = per
    except Exception as e:
        out["profile_cut_scans"] = f"profiler failed: {e}"
    batch.close()
    for c in ctx.values():
        c.close()
    return out


def run_sliding_window(n_seq, window, mg, shifts, pts_per_scan, room):
    """Workload (e), a Monte Carlo sliding window: n_seq independent sequences (assoc_ref.synthetic_scans, one seed
    each), a window of `window` scans cut and optimised once, then `shifts` window shifts, each marginalising the mg
    oldest scans, appending mg new ones, optimising with the fix clusters and propagating the pose covariance:
    (i) a Context (fp64) per sequence, marginalize + mg x append_scan + damping_iter + pose_covariance;
    (ii) one Batch doing the same calls for every sequence. Per shift, the context route marginalises and appends at the
    poses of the batch route, so their registrations must be bitwise equal (checked after every shift, outside the
    timed calls); each route then optimises and propagates on its own. Time per shift for each route."""
    import assoc_ref
    import scenes
    import balm_b200
    n_scans = window + mg * shifts
    scans, windows, init, new_pose = [], [], [], []
    for q in range(n_seq):
        pts, frs, poses = assoc_ref.synthetic_scans(n_poses=n_scans, pts_per_scan=pts_per_scan, seed=100 + q, room=room)
        p12 = scenes.pack_poses([r for r, _ in poses], [p for _, p in poses])
        base = len(scans)
        scans += [pts[frs == i].astype(np.float32) for i in range(n_scans)]
        windows.append(list(range(base, base + window)))
        init.append(p12[:window])
        new_pose.append(p12)
    kwc = dict(voxel_size=2.0, eigen_value_array=(1 / 16, 1 / 16, 1 / 9))
    lm_kw = dict(gauge_mode=2, min_planes_per_pose=0)
    cov_kw = dict(point_noise=0.01, include_fix=True)
    batch = balm_b200.Batch(0)
    batch.cut_scans(scans, windows, init, **kwc)
    x_b = [r[1] for r in batch.damping_iter(init, **lm_kw)]
    ctx = []
    for win, x0 in zip(windows, init):
        c = balm_b200.Context(window, 0, balm_b200.PREC_FP64)
        c.cut_voxels(np.concatenate([scans[s] for s in win]),
                     np.concatenate([np.full(len(scans[s]), k, dtype=np.int32) for k, s in enumerate(win)]), x0, **kwc)
        c.damping_iter(x0, **lm_kw)
        ctx.append(c)

    def clock(f):
        t0 = time.perf_counter()
        r = f()
        return r, 1e3 * (time.perf_counter() - t0)

    parts = ("marginalize", "append", "lm", "cov")
    ms = {"i_context": [], "ii_batch": []}
    ms_part = {r: {k: [] for k in parts} for r in ms}  # per shift, the route's time in each kind of call
    bitwise, dpose, dcov, statuses = True, 0.0, 0.0, set()
    for k in range(shifts):
        new = [[windows[q][0] + window + mg * k + j for q in range(n_seq)] for j in range(mg)]
        shifted = [np.vstack([x[mg:], new_pose[q][window + mg * k:window + mg * (k + 1)]]) for q, x in enumerate(x_b)]
        slots = [window - mg + j for j in range(mg)]
        tb = dict.fromkeys(parts, 0.0)
        _, tb["marginalize"] = clock(lambda: batch.marginalize([mg] * n_seq, x_b))
        for j in range(mg):  # only the scans this call appends: sequence q takes scan q of the list
            _, t = clock(lambda: batch.append_scans([scans[s] for s in new[j]], list(range(n_seq)), [slots[j]] * n_seq,
                                                    shifted))
            tb["append"] += t
        reg = batch.download_voxels(with_keys=True, with_fix=True)  # for the check, not part of the route
        lm, tb["lm"] = clock(lambda: batch.damping_iter(shifted, hess_includes_fix=True, **lm_kw))
        cov, tb["cov"] = clock(lambda: batch.pose_covariance([r[1] for r in lm], **cov_kw))
        tc = dict.fromkeys(parts, 0.0)
        ref = []
        for q, c in enumerate(ctx):
            _, t = clock(lambda: c.marginalize(mg, x_b[q]))
            tc["marginalize"] += t
            for j in range(mg):
                _, t = clock(lambda: c.append_scan(scans[new[j][q]], shifted[q], slots[j]))
                tc["append"] += t
            (p, _, _), t = clock(lambda: c.damping_iter(shifted[q], hess_includes_fix=True, **lm_kw))
            tc["lm"] += t
            (_, cv), t = clock(lambda: c.pose_covariance(p, **cov_kw))
            tc["cov"] += t
            ref.append((p, cv))
        for route, tt in (("ii_batch", tb), ("i_context", tc)):
            ms[route].append(sum(tt.values()))
            for key in parts:
                ms_part[route][key].append(tt[key])
        for c, d in zip(ctx, reg):
            rp, pi, ob, co = c.download_voxels()
            keys, layers = c.download_keys(with_layers=True)
            same = (np.array_equal(rp, d["row_ptr"]) and np.array_equal(pi, d["pose_idx"]) and
                    np.array_equal(ob, d["obs10"]) and np.array_equal(co, d["coe"]) and
                    np.array_equal(c.download_fix(), d["fix10"]) and np.array_equal(keys, d["keys"]) and
                    np.array_equal(layers, d["layers"]))
            bitwise = bitwise and same
        for (st, p, _, _), (cst, _, cv), (pc, cvc) in zip(lm, cov, ref):
            statuses.add(cst)
            dpose = max(dpose, float(np.abs(p - pc).max()))
            dcov = max(dcov, float(np.abs(cv - cvc).max() / np.abs(cvc).max()))
        x_b = [r[1] for r in lm]
    batch.close()
    for c in ctx:
        c.close()
    return dict(sequences=n_seq, window=window, mg=mg, shifts=shifts, pts_per_scan=pts_per_scan, room=room, ms=ms,
                ms_median_per_shift={k: float(np.median(v)) for k, v in ms.items()}, ms_per_call_kind=ms_part,
                ms_per_call_kind_median={r: {k: float(np.median(v)) for k, v in d.items()} for r, d in ms_part.items()},
                registrations_bitwise_equal=bool(bitwise), max_pose_diff_ii_vs_i=dpose,
                max_rel_cov_diff_ii_vs_i=dcov, batch_cov_statuses=sorted(statuses))


def run_persistent_window(n_seq, window, mg, shifts, pts_per_scan):
    """Workload (f), workload (e) on the persistent window maps: n_seq independent sequences of window_ref.growth_scans
    (one seed and step each, scans that keep reaching new space), a window of `window` scans cut, recut, pushed and
    optimised once, then `shifts` window shifts, each marginalising the mg oldest scans at the optimised poses, cutting
    and recutting mg new ones, pushing, optimising with the fix clusters and propagating the pose covariance:
    (i) a Context window (fp64) per sequence; (ii) one Batch window for all of them (balm_batch_window_*). The context
    route marginalises at the batch route's poses, so their pushes must be bitwise equal (checked after every shift,
    outside the timed calls). Also counts, per shift, the voxels the reduced batch path (cut_scans, then marginalize +
    append_scans, workload (e)'s calls) keeps on the same stream."""
    import scenes
    import window_ref
    import balm_b200
    n_scans = window + mg * shifts
    seqs = []
    for q in range(n_seq):
        pts, frs, noisy, _ = window_ref.growth_scans(n_scans=n_scans, pts_per_scan=pts_per_scan, seed=200 + q,
                                                     step=0.3 + 0.01 * (q % 30))
        p12 = scenes.pack_poses([r for r, _ in noisy], [p for _, p in noisy])
        seqs.append(([pts[frs == i].astype(np.float32) for i in range(n_scans)], p12))
    kwc = dict(voxel_size=2.0, layer_limit=2, min_ps=15, eigen_value_array=(1 / 16, 1 / 16, 1 / 9))
    lm_kw = dict(gauge_mode=2, min_planes_per_pose=0)
    cov_kw = dict(point_noise=0.01, include_fix=True)
    B = n_seq

    def clock(f):
        t0 = time.perf_counter()
        r = f()
        return r, 1e3 * (time.perf_counter() - t0)

    def poses_at(q, slot_scans):
        x = np.zeros((window, 12))
        x[:len(slot_scans)] = seqs[q][1][slot_scans]
        return x

    batch = balm_b200.Batch(0)
    batch.window_reset([window] * B, **kwc)
    ctx = [balm_b200.Context(window, 0, balm_b200.PREC_FP64) for _ in range(B)]
    for c in ctx:
        c.window_reset(**kwc)
    init = [poses_at(q, list(range(window))) for q in range(B)]
    for s in range(window):  # fill
        batch.window_cut([seqs[q][0][s] for q in range(B)], list(range(B)), [s] * B, init)
        batch.window_recut([s + 1] * B)
        for q, c in enumerate(ctx):
            c.window_cut(seqs[q][0][s], init[q][s], s)
            c.window_recut(s + 1)
    first_push = batch.window_push([window] * B)
    for c in ctx:
        c.window_push(window)
    x_b = [r[1] for r in batch.damping_iter(init, **lm_kw)]
    for q, c in enumerate(ctx):
        c.damping_iter(init[q], **lm_kw)
    # the reduced path on the same stream, for its voxel counts only
    red = balm_b200.Batch(0)
    cut = red.cut_scans([sc for q in range(B) for sc in seqs[q][0][:window]],
                        [list(range(q * window, (q + 1) * window)) for q in range(B)], init, **kwc)
    x_r = [r[1] for r in red.damping_iter(init, **lm_kw)]
    red_vox = [int(sum(m for m, _ in cut))]

    parts = ("marginalize", "cut", "recut", "push", "lm", "cov")
    ms = {"i_context": [], "ii_batch": []}
    ms_part = {r: {k: [] for k in parts} for r in ms}
    vox = [int(sum(m for m, _ in first_push))]
    bitwise, dpose, statuses, ctx_statuses = True, 0.0, set(), set()
    for k in range(shifts):
        new = [window + mg * k + j for j in range(mg)]
        shifted = [np.vstack([x_b[q][mg:], seqs[q][1][new]]) for q in range(B)]
        tb = dict.fromkeys(parts, 0.0)
        _, tb["marginalize"] = clock(lambda: batch.window_marginalize([mg] * B, x_b, [window] * B))
        for j in range(mg):
            slot = window - mg + j
            _, t = clock(lambda: batch.window_cut([seqs[q][0][new[j]] for q in range(B)], list(range(B)), [slot] * B,
                                                  shifted))
            tb["cut"] += t
            _, t = clock(lambda: batch.window_recut([slot + 1] * B))
            tb["recut"] += t
        pushed, tb["push"] = clock(lambda: batch.window_push([window] * B))
        reg = batch.download_voxels(with_keys=True, with_fix=True)  # for the check, not part of the route
        lm, tb["lm"] = clock(lambda: batch.damping_iter(shifted, hess_includes_fix=True, **lm_kw))
        cov, tb["cov"] = clock(lambda: batch.pose_covariance([r[1] for r in lm], **cov_kw))
        tc = dict.fromkeys(parts, 0.0)
        ref = []
        for q, c in enumerate(ctx):
            _, t = clock(lambda: c.window_marginalize(mg, x_b[q], window))
            tc["marginalize"] += t
            for j in range(mg):
                slot = window - mg + j
                _, t = clock(lambda: c.window_cut(seqs[q][0][new[j]], shifted[q][slot], slot))
                tc["cut"] += t
                _, t = clock(lambda: c.window_recut(slot + 1))
                tc["recut"] += t
            _, t = clock(lambda: c.window_push(window))
            tc["push"] += t
            rp, pi, ob, co = c.download_voxels()
            keys, layers = c.download_keys(with_layers=True)
            d = reg[q]
            bitwise = bitwise and (np.array_equal(rp, d["row_ptr"]) and np.array_equal(pi, d["pose_idx"]) and
                                   np.array_equal(ob, d["obs10"]) and np.array_equal(co, d["coe"]) and
                                   np.array_equal(c.download_fix(), d["fix10"]) and np.array_equal(keys, d["keys"]) and
                                   np.array_equal(layers, d["layers"]))
            (p, _, _), t = clock(lambda: c.damping_iter(shifted[q], hess_includes_fix=True, **lm_kw))
            tc["lm"] += t
            t0 = time.perf_counter()
            try:  # the context reports a singular H (a weakly observed direction) as an error, the batch as a status
                c.pose_covariance(p, **cov_kw)
                ctx_statuses.add(0)  # BALM_OK
            except balm_b200.BalmError as e:
                ctx_statuses.add(e.status)
            tc["cov"] += 1e3 * (time.perf_counter() - t0)
            ref.append(p)
        for route, tt in (("ii_batch", tb), ("i_context", tc)):
            ms[route].append(sum(tt.values()))
            for key in parts:
                ms_part[route][key].append(tt[key])
        for (st, p, _, _), (cst, _, _), pc in zip(lm, cov, ref):
            statuses.add(cst)
            dpose = max(dpose, float(np.abs(p - pc).max()))
        x_b = [r[1] for r in lm]
        vox.append(int(sum(m for m, _ in pushed)))
        # the reduced path: marginalise at its own optimised poses, append the same scans, optimise
        red.marginalize([mg] * B, x_r)
        shifted_r = [np.vstack([x_r[q][mg:], seqs[q][1][new]]) for q in range(B)]
        for j in range(mg):
            app = red.append_scans([seqs[q][0][new[j]] for q in range(B)], list(range(B)), [window - mg + j] * B,
                                   shifted_r)
        red_vox.append(int(sum(m for m, _, _ in app)))
        x_r = [r[1] for r in red.damping_iter(shifted_r, hess_includes_fix=True, **lm_kw)]
    batch.close()
    red.close()
    for c in ctx:
        c.close()
    return dict(sequences=n_seq, window=window, mg=mg, shifts=shifts, pts_per_scan=pts_per_scan, ms=ms,
                ms_median_per_shift={k: float(np.median(v)) for k, v in ms.items()}, ms_per_call_kind=ms_part,
                ms_per_call_kind_median={r: {k: float(np.median(v)) for k, v in d.items()} for r, d in ms_part.items()},
                voxels_per_shift_persistent=vox, voxels_per_shift_reduced=red_vox,
                pushes_bitwise_equal=bool(bitwise), max_pose_diff_ii_vs_i=dpose, batch_cov_statuses=sorted(statuses),
                context_cov_statuses=sorted(ctx_statuses))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--workloads", default="a,b,c")
    ap.add_argument("--out", default=None, help="also write the result to this JSON file")
    a = ap.parse_args()
    shapes = {"a": (256, 10, 1000, 100), "b": (32, 32, 5000, 900)}
    res = dict(gpu=gpu_info(), repeats=a.repeats)
    for w in a.workloads.split(","):
        if w == "c":
            res[w] = run_from_scans(160, 20000, 12.0, a.repeats)
        elif w == "e":
            res[w] = run_sliding_window(64, 10, 2, 5, 20000, 12.0)
        elif w == "f":
            res[w] = run_persistent_window(64, 10, 2, 10, 20000)
        elif w == "d":
            res[w] = {k: run_covariance(k, *shapes[k][:3], a.repeats, shapes[k][3]) for k in ("a", "b")}
        else:
            res[w] = run_workload(w, *shapes[w][:3], a.repeats, shapes[w][3])
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""numpy restatement of the robust voxel cost (DESIGN.md "Robust voxels") on numpy_ref's voxel terms:

  s_v = lambda_min(C_v) of the cluster the pass builds (observations at the poses, + fix cluster where that pass adds it)
  w_v = rho'(s_v),   cost = sum_v coe_v rho(s_v),   H, g = numpy_ref.evaluate of the scene registered with coe_v w_v

(every voxel term of numpy_ref.evaluate is linear in coe_v, so the second line is numpy_ref per voxel scaled by w_v; with
the trivial loss w_v = 1 and everything is numpy_ref's exactly). rho / rho' are robust_factors_ref's (kind 0 trivial,
1 Huber, 2 Cauchy). lm() restates balm_damping_iter's rule on this cost; moving_plane_scene() is the outlier scene the
tests use: a static plane scene plus voxels whose plane moves along its normal from scan to scan."""
import numpy as np

import numpy_ref as nr
import pose_graph_ref as pgr
from robust_factors_ref import CAUCHY, HUBER, NAMES, TRIVIAL, drho, rho  # noqa: F401  (re-exported for the tests)
from scenes import exp_so3, make_scene


def lams(sc, poses, include_fix=False):
    """lambda_min of every voxel, its cluster summed in numpy_ref.evaluate's order"""
    out = np.zeros(len(sc["row_ptr"]) - 1)
    for a in range(len(out)):
        W = [nr._world_cluster(sc["obs10"][s], poses[sc["pose_idx"][s]]) for s in range(sc["row_ptr"][a], sc["row_ptr"][a + 1])]
        P = sum(w[0] for w in W); v = sum(w[1] for w in W); NN = sum(w[2] for w in W)
        if include_fix and sc.get("fix10") is not None:
            f = sc["fix10"][a]
            P = P + np.array([[f[0], f[1], f[2]], [f[1], f[3], f[4]], [f[2], f[4], f[5]]]); v = v + f[6:9]; NN = NN + f[9]
        vb = v / NN
        out[a] = np.linalg.eigh(P / NN - np.outer(vb, vb))[0][0]
    return out


def weights(sc, poses, kind, c, include_fix=False):
    """-> (lam, w) per voxel"""
    lam = lams(sc, poses, include_fix)
    return lam, np.array([drho(kind, c, s) for s in lam])


def cost(sc, poses, kind, c, include_fix=True):
    """sum_v coe_v rho(s_v), summed in voxel order (balm_residual includes the fix clusters)"""
    r = 0.0
    for co, s in zip(sc["coe"], lams(sc, poses, include_fix)):
        r += co * rho(kind, c, s)
    return r


def weighted(sc, w):
    """the scene registered with coe_v w_v: the trivial-loss twin of a robust one"""
    return dict(sc, coe=np.asarray(sc["coe"], dtype=np.float64) * w)


def evaluate(sc, poses, kind, c, include_fix=False):
    """-> (H, g, cost, lam, w) of the robust cost"""
    lam, w = weights(sc, poses, kind, c, include_fix)
    H, g, _ = nr.evaluate(weighted(sc, w), poses, include_fix)
    r = 0.0
    for co, s in zip(sc["coe"], lam):
        r += co * rho(kind, c, s)
    return H, g, r, lam, w


def lm(sc, poses0, kind, c, max_iter=10, u0=0.01, v0=2.0, rel_tol=1e-6, hess_includes_fix=False):
    """balm_damping_iter's rule on the robust cost (bavoxel.hpp:1069-1166): dx = (H + u diag(H))^-1 (-g), the trial
    residual with the fix clusters, accept when it drops, H reused after a rejected step -> (poses, trace, per-iteration
    accepted poses, before any gauge step)"""
    x = np.array(poses0, dtype=np.float64, copy=True)
    u, v = u0, v0
    calc, trace, per = True, [], []
    H = g = None
    r1 = 0.0
    for it in range(max_iter):
        if calc:
            H, g, r1, _, _ = evaluate(sc, x, kind, c, hess_includes_fix)
        D = H.diagonal().copy()
        dx = np.linalg.solve(H + u * np.diag(D), -g)
        q1 = 0.5 * dx @ (u * D * dx - g)
        xt = pgr.pose_update(x, dx)
        r2 = cost(sc, xt, kind, c)
        q = r1 - r2
        t = dict(r1=r1, r2=r2, u=u, v=v, q=q, q1=q1, accepted=False, recomputed_hess=calc)
        if q > 0:
            x = xt
            u *= max(1 - (2 * q / q1 - 1) ** 3, 1.0 / 3.0)
            v, calc = 2.0, True
            t["accepted"] = True
        else:
            u, v, calc = u * v, 2 * v, False
        trace.append(t)
        per.append(x.copy())
        if rel_tol >= 0 and abs(r1 - r2) / r1 < rel_tol:
            break
    return x, trace, per


# ---------------- the moving-plane outlier scene ----------------
NOISE = 0.02   # sigma_p of every point (m)
SPEED = 0.08   # how far a moving plane travels along its normal between consecutive scans (m)
SCALE = 0.03   # the loss scale the tests use: 1.5 sigma_p


def moving_plane_scene(n_poses=8, n_planes=60, n_moving=8, pts_size=40, seed=3, moving_seed=7, drop=0.0,
                       with_fix=False):
    """scenes.make_scene (point noise NOISE) plus n_moving voxels of pts_size points per scan whose plane sits SPEED * j
    further along its normal in scan j. -> (scene with every voxel, the static scene alone); the moving voxels are
    the last n_moving, with empty fix clusters when with_fix gives the static ones theirs."""
    sc = make_scene(n_poses=n_poses, n_planes=n_planes, pts_size=pts_size, point_noise=NOISE, seed=seed, drop=drop,
                    with_fix=with_fix)
    gt = sc["poses_gt"]
    rng = np.random.default_rng(moving_seed)
    row_ptr, pidx, obs, coe = list(sc["row_ptr"]), list(sc["pose_idx"]), list(sc["obs10"]), list(sc["coe"])
    for _ in range(n_moving):
        rot = exp_so3(rng.uniform(-np.pi, np.pi, 3))
        center = rng.uniform(-2, 2, 3)
        nrm = rot[:, 2]
        for j in range(n_poses):
            loc = np.stack([rng.uniform(-.5, .5, pts_size), rng.uniform(-.5, .5, pts_size),
                            rng.normal(0, NOISE, pts_size)], 1)
            w = loc @ rot.T + center + SPEED * j * nrm
            R, p = gt[j, :9].reshape(3, 3).T, gt[j, 9:]
            b = ((w - p) @ R).astype(np.float32).astype(np.float64)
            P, vv = b.T @ b, b.sum(0)
            obs.append([P[0, 0], P[0, 1], P[0, 2], P[1, 1], P[1, 2], P[2, 2], vv[0], vv[1], vv[2], float(pts_size)])
            pidx.append(j)
        row_ptr.append(len(pidx))
        coe.append(float(pts_size * n_poses))
    bad = dict(sc, row_ptr=np.array(row_ptr, dtype=np.int64), pose_idx=np.array(pidx, dtype=np.int32),
               obs10=np.array(obs, dtype=np.float64), coe=np.array(coe, dtype=np.float64),
               fix10=np.concatenate([sc["fix10"], np.zeros((n_moving, 10))]) if with_fix else None)
    return bad, sc


def max_error(poses, gt):
    """largest position error after moving poses by the rigid transform that maps their pose 0 onto gt's"""
    R0, p0 = poses[0, :9].reshape(3, 3).T, poses[0, 9:]
    G0, q0 = gt[0, :9].reshape(3, 3).T, gt[0, 9:]
    A = G0 @ R0.T
    return float(max(np.linalg.norm(A @ (x[9:] - p0) + q0 - y[9:]) for x, y in zip(poses, gt)))

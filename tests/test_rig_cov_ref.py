"""The rig-covariance restatement (tests/rig_cov_ref.py) on the CPU: the identity rig is numpy_cov's pose covariance,
a fixed base pose and an anchor at it give the same covariance, and the extrinsic block does not depend on which base
pose anchors the base poses' gauge; the Monte-Carlo helpers' planar clusters are exactly planar."""
import numpy as np

import numpy_cov as nc
import rig_cov_ref as rc
import rig_ref as rr
import robust_voxels_ref as rv
from scenes import make_scene

PN = 0.01


def _rig_scene():
    """make_scene's scans as 3 bases x two LiDARs (test_gpu_rig.rig_case's "dense" layout, off the origin)"""
    sc = make_scene(n_poses=6, n_planes=30, seed=4)
    X = sc["poses_init"]
    base_of, lidar_of = np.arange(6) // 2, np.arange(6) % 2
    base = X[0::2].copy()
    R0, p0 = X[0, :9].reshape(3, 3).T, X[0, 9:]
    R1, p1 = X[1, :9].reshape(3, 3).T, X[1, 9:]
    ext = np.array([np.concatenate([np.eye(3).reshape(9), np.zeros(3)]),
                    np.concatenate([(R0.T @ R1).T.reshape(9), R0.T @ (p1 - p0)])])
    base[:, 9:] += np.array([30.0, -20.0, 5.0])
    return sc, base_of, lidar_of, base, ext


def _rel(a, b):
    return np.abs(a - b).max() / np.abs(b).max()


def test_identity_rig_is_the_pose_covariance():
    sc = make_scene(n_poses=6, n_planes=30, seed=5, with_fix=True)
    x, N = sc["poses_init"], sc["n_poses"]
    ident = np.concatenate([np.eye(3).reshape(9), np.zeros(3)])[None]
    raw, cov = rc.rig_covariance(sc, x, ident, np.arange(N), np.zeros(N, dtype=int), rr.unknowns(N, 1), pnoise=PN,
                                 include_fix=True)
    R = nc.left_jacobian_point(N, sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], x, sc["fix10"], pnoise=PN)
    H = rv.evaluate(sc, x, rv.TRIVIAL, 1.0, True)[0]
    assert np.array_equal(raw, R)
    assert _rel(cov, nc.pose_covariance(H, R)) < 1e-12


def test_fixed_base_equals_anchor():
    sc, base_of, lidar_of, base, ext = _rig_scene()
    for k in (0, 2):
        fixed = rr.unknowns(3, 2, fixed_bases=(k,))
        raw_f, cov_f = rc.rig_covariance(sc, base, ext, base_of, lidar_of, fixed, pnoise=PN)
        raw_a, cov_a = rc.rig_covariance(sc, base, ext, base_of, lidar_of, rr.unknowns(3, 2), pnoise=PN, anchor=k)
        keep = np.setdiff1d(np.arange(len(raw_a)), np.arange(6 * k, 6 * k + 6))
        assert np.all(cov_a[6 * k:6 * k + 6] == 0) and np.all(cov_a[:, 6 * k:6 * k + 6] == 0)
        assert np.all(raw_a[6 * k:6 * k + 6] == 0) and np.all(raw_a[:, 6 * k:6 * k + 6] == 0)
        assert _rel(raw_a[np.ix_(keep, keep)], raw_f) < 1e-12
        assert _rel(cov_a[np.ix_(keep, keep)], cov_f) < 1e-9


def test_extrinsic_block_is_gauge_free():
    """at a stationary point of the rig cost (no fix clusters, bases free) H_rig has the base poses' common left step
    as a null vector, so every base anchor gives the same extrinsic block"""
    sc, base_of, lidar_of, base, ext = _rig_scene()
    var = rr.unknowns(3, 2)
    base, ext, tr, _ = rr.lm(sc, base, ext, base_of, lidar_of, var, max_iter=40, rel_tol=-1)
    g = rr.evaluate(sc, base, ext, base_of, lidar_of, var)[1]
    covs = [rc.rig_covariance(sc, base, ext, base_of, lidar_of, var, pnoise=PN, anchor=a)[1][18:, 18:] for a in (0, 2)]
    assert _rel(covs[1], covs[0]) < 1e-9, (_rel(covs[1], covs[0]), np.abs(g).max())


def test_planar_moments_are_planar():
    sc, base_of, lidar_of, base, ext = _rig_scene()
    X = rr.compose(base, ext, base_of, lidar_of)
    flat = dict(sc, obs10=rc.planar_moments(sc, X))
    lam_before, lam = rv.lams(sc, X), rv.lams(flat, X)
    assert np.abs(lam).max() < 1e-9 * np.abs(lam_before).max()
    assert np.array_equal(flat["obs10"][:, 9], sc["obs10"][:, 9])

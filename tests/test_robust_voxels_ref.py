"""CPU checks of the robust voxel restatement (tests/robust_voxels_ref.py) that the GPU tests compare against: the
gradient is that of sum coe rho(lambda_min) under the left update, the trivial loss is numpy_ref exactly, the gauge null
space survives the weights, and on the moving-plane scene Cauchy recovers what the trivial loss loses."""
import numpy as np
import pytest

import numpy_ref as nr
import pose_graph_ref as pgr
import robust_voxels_ref as rv


def _fd_gradient(sc, x, kind, c, include_fix, h=1e-5):
    g = np.zeros(6 * len(x))
    for k in range(len(g)):
        d = np.zeros(len(g))
        d[k] = h
        g[k] = (rv.cost(sc, pgr.pose_update(x, d), kind, c, include_fix) -
                rv.cost(sc, pgr.pose_update(x, -d), kind, c, include_fix)) / (2 * h)
    return g


@pytest.mark.parametrize("kind", [rv.HUBER, rv.CAUCHY])
@pytest.mark.parametrize("with_fix", [False, True])
def test_gradient_is_the_robust_cost_gradient(kind, with_fix):
    sc, _ = rv.moving_plane_scene(n_poses=5, n_planes=12, n_moving=3, with_fix=with_fix)
    x = sc["poses_init"]
    c = 0.05  # at the initial poses the static voxels straddle c^2 = 0.0025
    _, g, r, lam, w = rv.evaluate(sc, x, kind, c, include_fix=with_fix)
    if kind == rv.HUBER:  # both branches of Huber are exercised
        assert (lam > c * c).any() and (lam <= c * c).any()
    assert r == pytest.approx(rv.cost(sc, x, kind, c, with_fix), rel=1e-14)
    fd = _fd_gradient(sc, x, kind, c, with_fix)
    assert np.abs(fd - g).max() < 1e-6 * np.abs(g).max()


@pytest.mark.parametrize("with_fix", [False, True])
def test_trivial_is_numpy_ref_exactly(with_fix):
    sc, _ = rv.moving_plane_scene(n_poses=5, n_planes=12, n_moving=3, with_fix=with_fix)
    x = sc["poses_init"]
    H, g, r, _, w = rv.evaluate(sc, x, rv.TRIVIAL, 1.0, include_fix=with_fix)
    Ho, go, ro = nr.evaluate(sc, x, include_fix=with_fix)
    assert (w == 1.0).all()
    assert np.array_equal(H, Ho) and np.array_equal(g, go) and r == ro
    assert rv.cost(sc, x, rv.TRIVIAL, 1.0) == pytest.approx(nr.residual(sc, x), rel=1e-13)  # eigvalsh's last bits


@pytest.mark.parametrize("kind", [rv.HUBER, rv.CAUCHY])
def test_gauge_null_space(kind):
    sc, _ = rv.moving_plane_scene(n_poses=5, n_planes=12, n_moving=3)
    x = sc["poses_init"]
    H, g, _, _, w = rv.evaluate(sc, x, kind, rv.SCALE)
    assert w.min() < 0.5  # the weights are far from uniform
    V = pgr.gauge_vectors(len(x))
    assert np.abs(g @ V).max() < 1e-10 * np.abs(g).max() * np.sqrt(len(g))
    assert np.abs(V.T @ H @ V).max() < 1e-10 * np.abs(H).max() * len(g)


def test_moving_planes_cauchy_recovers():
    bad, clean = rv.moving_plane_scene()
    gt, x0 = clean["poses_gt"], clean["poses_init"]
    e_clean = rv.max_error(rv.lm(clean, x0, rv.TRIVIAL, 1.0, max_iter=15)[0], gt)
    e_triv = rv.max_error(rv.lm(bad, x0, rv.TRIVIAL, 1.0, max_iter=15)[0], gt)
    e_cauchy = rv.max_error(rv.lm(bad, x0, rv.CAUCHY, rv.SCALE, max_iter=15)[0], gt)
    assert e_clean < 0.003
    assert e_cauchy < 2 * e_clean
    assert e_triv > 5 * e_clean
    lam, w = rv.weights(bad, gt, rv.CAUCHY, rv.SCALE)
    assert w[-8:].max() < w[:-8].min()  # every moving voxel ends with a lower weight than any static one

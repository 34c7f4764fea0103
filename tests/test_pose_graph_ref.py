"""The pose-graph oracle (pose_graph_ref.py) against its own definition: zero error at the factor's poses, invariance to a
common left transform, Jacobians and gradient against central finite differences, the gauge null space of H, scale
invariance of the minimiser and exact recovery of a noise-free trajectory."""
import numpy as np
import pytest

import pose_graph_ref as pg


def _scene(seed=0, P=14, noise=0.0):
    rng = np.random.default_rng(seed)
    truth = np.array([pg.random_pose(rng) for _ in range(P)])
    sets = [list(range(0, 6)), list(range(3, 10)), list(range(8, P)), [0, 5, 9, 13], [13, 2]]
    factors = [pg.make_factor(rng, truth, s, noise) for s in sets]
    return rng, truth, factors


def test_error_is_zero_at_the_factor_poses():
    rng, truth, factors = _scene()
    for f in factors:
        e, _, c, _, b = pg.factor_terms(truth, f)
        assert np.abs(e).max() < 1e-12 and abs(c) < 1e-20 and np.abs(b).max() < 1e-9
    # also at the window's own poses, in its own frame
    f = factors[1]
    poses = np.array(truth, copy=True)
    poses[f["poses"]] = f["poses_hat"]
    assert np.abs(pg.factor_terms(poses, f)[0]).max() < 1e-12


def test_cost_is_invariant_to_a_common_left_transform():
    rng, truth, factors = _scene(1, noise=0.02)
    x = pg.perturb(rng, truth, 0.05, 0.2)
    G = pg.random_pose(rng)
    y = np.array([pg.compose(G, p) for p in x])
    c0, c1 = pg.cost(x, factors), pg.cost(y, factors)
    assert c0 > 1e-3 and abs(c0 - c1) <= 1e-12 * c0


def test_jacobians_match_central_differences():
    rng, truth, factors = _scene(2, noise=0.05)
    x = pg.perturb(rng, truth, 0.3, 1.0)
    f = factors[2]
    idx = f["poses"]
    h = 1e-6
    for k in (1, len(idx) - 1):
        _, J = pg.residual(x[idx[0]], x[idx[k]], f["poses_hat"][0], f["poses_hat"][k])
        for who, want in ((k, J), (0, -J)):
            num = np.zeros((6, 6))
            for a in range(6):
                d = np.zeros(6 * len(x))
                d[6 * idx[who] + a] = h
                ep = pg.residual(*(pg.pose_update(x, d)[[idx[0], idx[k]]]), f["poses_hat"][0], f["poses_hat"][k])[0]
                em = pg.residual(*(pg.pose_update(x, -d)[[idx[0], idx[k]]]), f["poses_hat"][0], f["poses_hat"][k])[0]
                num[:, a] = (ep - em) / (2 * h)
            assert np.abs(num - want).max() <= 1e-7 * max(1.0, np.abs(want).max())


def test_gradient_matches_central_differences_of_the_cost():
    rng, truth, factors = _scene(3, noise=0.03)
    x = pg.perturb(rng, truth, 0.2, 0.5)
    P = len(x)
    _, g, _ = pg.evaluate(x, factors, P)
    h = 1e-6
    num = np.zeros(6 * P)
    for j in range(6 * P):
        d = np.zeros(6 * P)
        d[j] = h
        num[j] = (pg.cost(pg.pose_update(x, d), factors) - pg.cost(pg.pose_update(x, -d), factors)) / (2 * h)
    assert np.abs(num - g).max() <= 1e-6 * np.abs(g).max()


def test_hessian_annihilates_the_gauge_directions():
    rng, truth, factors = _scene(4, noise=0.03)
    x = pg.perturb(rng, truth, 0.2, 0.5)
    H, g, _ = pg.evaluate(x, factors, len(x))
    V = pg.gauge_vectors(len(x))
    assert np.abs(H @ V).max() <= 1e-12 * np.abs(H).max()
    assert np.abs(g @ V).max() <= 1e-10 * np.abs(g).max()
    assert np.abs(H - H.T).max() <= 1e-12 * np.abs(H).max()


def _rel_to_first(poses):
    R0, p0 = pg.split(poses[0])
    return np.array([pg.pack(R0.T @ pg.split(p)[0], R0.T @ (pg.split(p)[1] - p0)) for p in poses])


def test_scaling_every_hessian_leaves_the_minimiser():
    rng, truth, factors = _scene(5, noise=0.02)
    x0 = pg.perturb(rng, truth, 0.02, 0.05)
    a, _, _ = pg.lm(x0, factors, len(x0), max_iter=30, rel_tol=1e-14)
    scaled = [dict(f, H=f["H"] * 37.0) for f in factors]
    b, _, _ = pg.lm(x0, scaled, len(x0), max_iter=30, rel_tol=1e-14)
    assert np.abs(_rel_to_first(a) - _rel_to_first(b)).max() < 1e-8


@pytest.mark.parametrize("seed", [6, 7])
def test_noise_free_factors_give_the_trajectory_back(seed):
    rng = np.random.default_rng(seed)
    P = 40
    truth = np.array([pg.random_pose(rng, 0.5, 3.0) for _ in range(P)])
    factors = [pg.make_factor(rng, truth, s) for s in pg.pyramid_factor_poses(P, top=8)]
    x0 = pg.perturb(rng, truth, 0.03, 0.1)
    x, tr, _ = pg.lm(x0, factors, P, max_iter=40, rel_tol=-1)
    assert tr[-1]["r2"] < 1e-20 or min(t["r1"] for t in tr) < 1e-20
    got, want = _rel_to_first(x), _rel_to_first(truth)
    assert np.abs(got - want).max() < 1e-9


def test_log_handles_angles_near_pi_and_zero():
    rng = np.random.default_rng(8)
    for th in (0.0, 1e-9, 1e-3, 0.5, 1.6, 3.0, np.pi - 1e-7):
        a = rng.normal(size=3)
        a /= np.linalg.norm(a)
        phi = pg.log_so3(pg.exp_so3(th * a))
        assert np.abs(pg.exp_so3(phi) - pg.exp_so3(th * a)).max() < 1e-12

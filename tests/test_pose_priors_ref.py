"""CPU checks of the absolute pose prior restatement (tests/pose_priors_ref.py) and of the Python prior builders: the
analytic J and gradient against central finite differences under the left update, for full, position-only and
lever-arm priors under each loss; the units of pose_priors / position_priors; and the LM with priors."""
import numpy as np
import pytest

import balm_b200
import pose_graph_ref as pgr
import pose_priors_ref as ppr
import robust_factors_ref as rfr

LOSSES = [(rfr.TRIVIAL, 1.0), (rfr.HUBER, 0.7), (rfr.CAUCHY, 0.5)]


def _step(x, i, d):
    dx = np.zeros(6 * len(x))
    dx[6 * i:6 * i + 6] = d
    return pgr.pose_update(x, dx)


@pytest.mark.parametrize("kind,c", LOSSES)
@pytest.mark.parametrize("which", ["full", "position", "lever"])
def test_gradient_and_jacobian_against_finite_differences(kind, c, which):
    rng = np.random.default_rng(3)
    x = np.array([pgr.random_pose(rng, 1.0, 30.0) for _ in range(3)])
    pr = ppr.random_priors(rng, x, [1], kinds=(which,))[0]
    pr["pose_hat"] = pgr.compose(x[1], pgr.random_pose(rng, 0.4, 2.0))  # far enough for Huber / Cauchy to bend
    e, J, s, w, _, M, b = ppr.prior_terms(x, pr, kind, c)
    h = 1e-6
    Jn, gn = np.zeros((6, 6)), np.zeros(6)
    for a in range(6):
        d = np.zeros(6)
        d[a] = h
        xp, xm = _step(x, 1, d), _step(x, 1, -d)
        Jn[:, a] = (ppr.prior_terms(xp, pr)[0] - ppr.prior_terms(xm, pr)[0]) / (2 * h)
        gn[a] = (ppr.cost(xp, [], [pr], pk=[kind], ps=[c]) - ppr.cost(xm, [], [pr], pk=[kind], ps=[c])) / (2 * h)
    assert np.abs(Jn - J).max() <= 1e-6 * max(1.0, np.abs(J).max())
    assert np.abs(gn - b).max() <= 1e-6 * max(1.0, np.abs(b).max())
    assert np.linalg.eigvalsh(0.5 * (M + M.T)).min() >= -1e-9 * np.abs(M).max()
    assert w == pytest.approx(rfr.drho(kind, c, s))


def test_position_prior_ignores_the_measured_rotation():
    rng = np.random.default_rng(5)
    x = np.array([pgr.random_pose(rng) for _ in range(2)])
    pr = balm_b200.position_priors([0], [x[0, 9:] + 0.3], np.eye(3), lever_arm=[0.5, -0.2, 1.0])[0]
    other = dict(pr, pose_hat=pgr.compose(pgr.random_pose(rng), pr["pose_hat"]))
    other["pose_hat"][9:] = pr["pose_hat"][9:]
    a, b = ppr.prior_terms(x, pr), ppr.prior_terms(x, other)
    assert a[2] == pytest.approx(b[2], rel=1e-14)
    np.testing.assert_allclose(a[6], b[6], rtol=1e-12, atol=1e-12)
    R, p = pgr.split(x[0])
    np.testing.assert_allclose(a[0][3:], R @ [0.5, -0.2, 1.0] + p - pr["pose_hat"][9:], atol=1e-12)


def test_pose_priors_are_zero_at_the_measurement_and_quadratic():
    rng = np.random.default_rng(7)
    x = np.array([pgr.random_pose(rng) for _ in range(4)])
    om = pgr.random_spd(rng, 6, 100.0)
    prs = balm_b200.pose_priors([0, 2], x[[0, 2]], om)
    assert ppr.cost(x, [], prs) == pytest.approx(0.0, abs=1e-20)
    d = 1e-4 * rng.standard_normal(6)
    xp = _step(x, 2, d)
    J = ppr.prior_terms(x, prs[1])[1]  # info6 is in the residual's coordinates: cost = 1/2 (J d)^T info6 (J d)
    assert ppr.cost(xp, [], prs) == pytest.approx(0.5 * (J @ d) @ om @ (J @ d), rel=1e-3)
    with pytest.raises(ValueError):
        balm_b200.position_priors([0, 1], np.zeros((2, 3)), np.zeros((3, 3, 3)))


def test_lm_with_priors_fixes_the_frame():
    """odometry factors plus GNSS priors on a drifted chain: LM converges to the truth without any re-anchoring, and
    the Hessian of the sum is regular (no gauge null space)"""
    rng = np.random.default_rng(11)
    P = 40
    gt = np.array([pgr.pack(pgr.exp_so3([0, 0, 0.05 * i]), [2.0 * i, 0.1 * i, 0.0]) for i in range(P)])
    factors = [pgr.make_factor(rng, gt, [i, i + 1], cond=10.0) for i in range(P - 1)]
    for f in factors:
        f["H"] *= 100.0
    priors = balm_b200.position_priors(range(0, P, 5), gt[::5, 9:], np.eye(3))
    priors += balm_b200.position_priors(range(2, P, 5), [pgr.split(gt[i])[0] @ [0.3, 0.1, 1.2] + gt[i, 9:]
                                                         for i in range(2, P, 5)], np.eye(3), lever_arm=[0.3, 0.1, 1.2])
    x0 = pgr.perturb(rng, gt, 0.02, 0.5)
    x, trace, _ = ppr.lm(x0, factors, priors, P, max_iter=30, rel_tol=1e-12)
    assert trace[0]["accepted"]
    assert np.abs(x[:, 9:] - gt[:, 9:]).max() < 1e-6
    H, _, _ = ppr.evaluate(x, factors, priors, P)
    ev = np.linalg.eigvalsh(H)
    assert ev.min() > 1e-8 * ev.max()

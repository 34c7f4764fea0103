"""The robust-loss restatement (robust_factors_ref) on the CPU: rho' against differences of rho, the robust gradient
against differences of the robust cost, the reweighted H's gauge and sign, and the outlier scene's claims at 200 poses,
which fix the scene the GPU tests run."""
import numpy as np
import pytest

import pose_graph_ref as pgr
import robust_factors_ref as rr


@pytest.mark.parametrize("kind", [rr.HUBER, rr.CAUCHY])
def test_drho_is_the_derivative_of_rho(kind):
    c = 0.7
    for s in [0.05, 0.3, 0.45, 0.55, 1.0, 7.0, 300.0]:  # c^2 = 0.49: both sides
        h = 1e-6 * s
        fd = (rr.rho(kind, c, s + h) - rr.rho(kind, c, s - h)) / (2 * h)
        assert abs(fd - rr.drho(kind, c, s)) <= 1e-7 * max(1.0, abs(fd)), (kind, s)
    assert rr.rho(rr.TRIVIAL, c, 3.0) == 3.0 and rr.drho(rr.TRIVIAL, c, 3.0) == 1.0
    # below c^2 Huber is the trivial loss exactly; Cauchy is close to it
    assert rr.rho(rr.HUBER, c, 0.2) == 0.2 and rr.drho(rr.HUBER, c, 0.2) == 1.0
    assert abs(rr.rho(rr.CAUCHY, c, 1e-4) - 1e-4) < 1e-7


def _small_set(seed=0, P=8):
    """window and two-pose factors over P poses at perturbed poses, and a scale with factors on both sides of c^2"""
    rng = np.random.default_rng(seed)
    gt = np.array([pgr.random_pose(rng) for _ in range(P)])
    fs = [pgr.make_factor(rng, gt, idx, noise=0.02) for idx in ([0, 1, 2], [2, 3], [3, 4, 5, 6], [6, 7], [7, 0], [1, 5])]
    x = pgr.perturb(rng, gt, 0.02, 0.1)
    s, _ = rr.residuals(x, fs, np.zeros(len(fs), np.int32), np.ones(len(fs)))
    c = np.sqrt(np.median(s))
    return fs, x, P, c, s


def _loss_sets(n, c):
    return {"huber": rr.loss_arrays(n, "huber", c), "cauchy": rr.loss_arrays(n, "cauchy", c),
            "mixed": rr.loss_arrays(n, ["trivial", "huber", "cauchy"] * (n // 3) + ["cauchy"] * (n % 3), c)}


@pytest.mark.parametrize("name", ["huber", "cauchy", "mixed"])
def test_robust_gradient_is_the_derivative_of_the_robust_cost(name):
    fs, x, P, c, s = _small_set()
    assert (s > c * c).any() and (s < c * c).any()
    kinds, scales = _loss_sets(len(fs), c)[name]
    _, g, r = rr.evaluate(x, fs, P, kinds, scales)
    assert r == pytest.approx(rr.cost(x, fs, kinds, scales), rel=1e-15)
    h = 1e-6
    fd = np.zeros(6 * P)
    for q in range(6 * P):
        d = np.zeros(6 * P)
        d[q] = h
        fd[q] = (rr.cost(pgr.pose_update(x, d), fs, kinds, scales) -
                 rr.cost(pgr.pose_update(x, -d), fs, kinds, scales)) / (2 * h)
    err = np.abs(fd - g).max() / np.abs(g).max()
    assert err <= 1e-6, err


@pytest.mark.parametrize("name", ["huber", "cauchy", "mixed"])
def test_reweighted_hessian_is_psd_with_the_gauge_null_space(name):
    fs, x, P, c, _ = _small_set(1)
    kinds, scales = _loss_sets(len(fs), c)[name]
    H, _, _ = rr.evaluate(x, fs, P, kinds, scales)
    assert np.abs(H - H.T).max() <= 1e-12 * np.abs(H).max()
    ev = np.linalg.eigvalsh(H)
    assert ev.min() >= -1e-12 * ev.max()
    assert np.abs(H @ pgr.gauge_vectors(P)).max() <= 1e-10 * np.abs(H).max()
    assert (ev > 1e-9 * ev.max()).sum() == 6 * P - 6
    # every trivial factor contributes its quadratic terms unchanged
    triv = np.zeros(len(fs), np.int32)
    for k, f in zip(kinds, fs):
        if k == rr.TRIVIAL:
            _, _, _, M, b = rr.factor_terms(x, f, k, 1.0)
            _, _, _, M0, b0 = pgr.factor_terms(x, f)
            assert np.array_equal(M, M0) and np.array_equal(b, b0)
    H0 = pgr.evaluate(x, fs, P)[0]
    assert np.abs(rr.evaluate(x, fs, P, triv, scales)[0] - H0).max() <= 1e-13 * np.abs(H0).max()


def test_outlier_scene_claims_at_200_poses():
    """The claims the GPU tests make at 200 and 2000 poses, on the restatement: with false closures the trivial loss is
    off by more than 10x the outlier-free error, Cauchy at c^2 = 2 sigma_p^2 chi2_6(0.999) is within 1.5x of it, and
    every false closure ends with a smaller weight than every true one."""
    P = 200
    sc = rr.outlier_scene(P, 1)
    nt, nf = len(sc["true"]), len(sc["false"])
    assert 0.15 <= nf / (nt + nf) <= 0.25
    c = rr.cauchy_scale()

    def run(fs, kind):
        kinds, scales = rr.loss_arrays(len(fs), kind, c)
        x, tr, _ = rr.lm(sc["x0"], fs, P, kinds, scales, max_iter=60, sparse=True)
        return x, tr, kinds, scales

    x_clean, _, _, _ = run(sc["clean"], "trivial")
    x_triv, _, _, _ = run(sc["all"], "trivial")
    x_rob, tr, kinds, scales = run(sc["all"], "cauchy")
    e_clean, e_triv, e_rob = (rr.max_error(x, sc["gt"]) for x in (x_clean, x_triv, x_rob))
    _, w = rr.residuals(x_rob, sc["all"], kinds, scales)
    no = len(sc["odo"])
    print(f"max error: outlier-free {e_clean:.3f} m, trivial {e_triv:.3f} m, Cauchy {e_rob:.3f} m "
          f"({len(tr)} iterations); w true >= {w[no:no + nt].min():.3f}, w false <= {w[no + nt:].max():.2e}")
    assert e_triv > 10 * e_clean
    assert e_rob < 1.5 * e_clean
    assert w[no + nt:].max() < w[no:no + nt].min()

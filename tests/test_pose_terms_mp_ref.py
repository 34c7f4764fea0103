"""Checks of the extended-precision pose-term reference pose_terms_mp_ref.py itself (CPU): its quaternion Log against
the principal matrix log at every edge angle, its central-difference Jacobians against the closed form of
pose_graph_ref (fp64) and of the same closed form at 50 digits, its costs against the numpy restatements, and its IRLS
gradient against the central-difference gradient of the robust cost."""
import mpmath
import numpy as np
import pytest

import pose_graph_ref as pg
import pose_priors_ref as ppr
import pose_terms_mp_ref as mr
import robust_factors_ref as rfr

# central differences at 50 digits with step 1e-20 keep 30 digits of the residual's size (1 + |p| on translations)
FD_TOL = mpmath.mpf("1e-30")


@pytest.mark.parametrize("axis", range(len(mr.AXES)))
def test_quaternion_log_is_the_matrix_log_at_every_edge_angle(axis):
    a = mr.AXES[axis]
    rng = np.random.default_rng(axis)
    for th in mr.ANGLES + (np.pi,):
        R2 = pg.exp_so3(rng.normal(0, 1, 3))  # D = (X R2) R2^T exactly from fp64 factors: a rotation by th, off by eps
        D = mr.mpa(mr.rot64(th, a) @ R2).dot(mr.mpa(R2.T))
        q, m = mr.log_so3(D), mr.log_so3_logm(D)
        n = mpmath.sqrt(sum(x * x for x in q))
        if th > np.pi - 1e-3:  # the two logs of a rotation by pi differ in sign only; near it they agree
            assert abs(n - mpmath.sqrt(sum(x * x for x in m))) < mpmath.mpf("1e-40")
        if th < np.pi:
            assert max(abs(x - y) for x, y in zip(q, m)) < mpmath.mpf("1e-40"), th


def _mp_closed_form(R0, p0, Rk, pk, Rh0, ph0, Rhk, phk):
    """pose_graph_ref.residual's closed-form J_k at 50 digits (Jl^-1 without its series)"""
    Q = Rh0.dot(R0.T)
    D = Q.dot(Rk).dot(Rhk.T)
    phi = mr.log_so3(D)
    th = mpmath.sqrt(sum(x * x for x in phi))
    h = th / 2
    c2 = (1 - h * mpmath.cot(h)) / (th * th) if th > 0 else mpmath.mpf(1) / 12
    K = mr.hat(phi)
    eye = mr.exp_so3(np.array([mpmath.mpf(0)] * 3, dtype=object))
    w = pk - Rk.dot(Rhk.T).dot(phk)
    J = np.empty((6, 6), dtype=object)
    J[:3, :3] = (eye - K / 2 + c2 * K.dot(K)).dot(Q)
    J[:3, 3:] = mpmath.mpf(0)
    J[3:, :3] = -Q.dot(mr.hat(w))
    J[3:, 3:] = Q
    return J


@pytest.mark.parametrize("theta", [1e-4, 0.05, 0.3, 1.0, 2.5])
def test_central_differences_are_the_closed_form_jacobian(theta):
    rng = np.random.default_rng(int(theta * 1000))
    h0, hk = pg.random_pose(rng), pg.random_pose(rng)
    G = pg.random_pose(rng)
    T0 = pg.compose(G, h0)
    Rhk, phk = pg.split(hk)
    a = rng.standard_normal(3)
    a /= np.linalg.norm(a)
    X = mr.rot64(theta, a)
    Tk = pg.compose(G, pg.pack(X @ Rhk, X @ phk + rng.normal(0, 1, 3)))
    f = dict(poses=np.array([0, 1], dtype=np.int32), poses_hat=np.stack([h0, hk]), H=pg.window_hessian(rng, 2))
    t = mr.factor_terms(np.stack([T0, Tk]), f)
    args = [*mr.pose(T0), *mr.pose(Tk), *mr.pose(h0), *mr.pose(hk)]
    e_mp = mr.factor_residual(*args)
    E = mr._fd(lambda R, p: mr.factor_residual(args[0], args[1], R, p, *args[4:]), args[2], args[3])
    E0 = mr._fd(lambda R, p: mr.factor_residual(R, p, *args[2:]), args[0], args[1])
    e64, J64 = pg.residual(T0, Tk, h0, hk)
    assert np.abs(mr.to_f(e_mp) - e64).max() <= 1e-13 * max(1.0, np.abs(e64).max())
    assert np.abs(mr.to_f(E) - J64).max() <= 1e-13 * np.abs(J64).max()
    assert np.abs(mr.to_f(E0) + J64).max() <= 1e-13 * np.abs(J64).max()
    # the closed form holds exactly for exact rotations: the same poses rotated at 50 digits
    ex = [(mr.exp_so3(mr.log_so3(R)), p) for R, p in (args[0:2], args[2:4], args[4:6], args[6:8])]
    ex = [v for rp in ex for v in rp]
    Emp = mr._fd(lambda R, p: mr.factor_residual(ex[0], ex[1], R, p, *ex[4:]), ex[2], ex[3])
    E0mp = mr._fd(lambda R, p: mr.factor_residual(R, p, *ex[2:]), ex[0], ex[1])
    Jmp = _mp_closed_form(*ex)
    tol = FD_TOL * (1 + max(abs(x) for x in np.concatenate(ex[1::2])))
    assert max(abs(x) for x in (Emp - Jmp).ravel()) < tol
    assert max(abs(x) for x in (E0mp + Jmp).ravel()) < tol  # slot 0: the common left transform
    assert abs(float(t["s"]) - 2 * pg.factor_terms(np.stack([T0, Tk]), f)[2]) <= 1e-12 * float(t["s"])


def test_prior_jacobian_is_the_closed_form_with_the_lever_arm():
    rng = np.random.default_rng(3)
    x = np.array([pg.random_pose(rng, 0.5, 400.0) for _ in range(3)])
    for lever in (None, [2.0, -1.0, 0.5], [500.0, 0.0, -300.0]):
        pr = dict(pose=1, pose_hat=pg.compose(x[1], pg.random_pose(rng, 0.8, 2.0)), H=ppr.random_psd(rng, 6))
        if lever is not None:
            pr["lever_arm"] = np.array(lever)
        R, p = mr.pose(x[1])
        Rh, ph = mr.pose(pr["pose_hat"])
        lv = mr.mpa(np.zeros(3) if lever is None else lever)
        E = mr._fd(lambda R_, p_: mr.prior_residual(R_, p_, Rh, ph, lv), R, p)
        e64, J64, s64, _, _, _, _ = ppr.prior_terms(x, pr)
        assert np.abs(mr.to_f(E) - J64).max() <= 1e-13 * np.abs(J64).max()
        xl = R.dot(lv) + p
        assert max(abs(x_) for x_ in (E[3:, :3] + mr.hat(xl)).ravel()) < FD_TOL * (1 + max(abs(v) for v in xl))
        t = mr.prior_terms(x, pr)
        assert abs(float(t["s"]) - s64) <= 1e-12 * s64


@pytest.mark.parametrize("kind", [rfr.TRIVIAL, rfr.HUBER, rfr.CAUCHY])
def test_costs_match_the_restatements_and_g_is_the_cost_gradient(kind):
    rng = np.random.default_rng(10 + kind)
    P = 5
    truth = np.array([pg.random_pose(rng, 0.5, 3.0) for _ in range(P)])
    factors = [pg.make_factor(rng, truth, s, noise=0.05) for s in ([3, 0, 4], [1, 2], [2, 4, 0, 1])]
    x = pg.perturb(rng, truth, 0.1, 0.3)
    priors = ppr.random_priors(rng, x, [0, 3, 3])
    fk, fs = [kind] * 3, [0.5, 2.0, 1.0]
    pk, ps = [kind] * 3, [0.3, 1.0, 0.1]
    ft = [(f, mr.factor_terms(x, f, k, c)) for f, k, c in zip(factors, fk, fs)]
    pt = [(p, mr.prior_terms(x, p, k, c)) for p, k, c in zip(priors, pk, ps)]
    ref = mr.assemble(ft, pt)
    Hr = np.zeros((6 * P, 6 * P))
    gr = np.zeros(6 * P)
    for (i, j), (B, _) in ref["blocks"].items():
        Hr[6 * i:6 * i + 6, 6 * j:6 * j + 6] = B
        Hr[6 * j:6 * j + 6, 6 * i:6 * i + 6] = B.T
    for i, (v, _) in ref["g"].items():
        gr[6 * i:6 * i + 6] = v
    s_np, w_np = rfr.residuals(x, factors, fk, fs)
    assert np.allclose([float(t["s"]) for _, t in ft], s_np, rtol=1e-12, atol=0)
    assert np.allclose([float(t["w"]) for _, t in ft], w_np, rtol=1e-12, atol=0)
    sq, wq = ppr.residuals(x, priors, pk, ps)
    assert np.allclose([float(t["s"]) for _, t in pt], sq, rtol=1e-12, atol=0)
    assert np.allclose([float(t["w"]) for _, t in pt], wq, rtol=1e-12, atol=0)
    Ho, go, ro = ppr.evaluate(x, factors, priors, P, fk, fs, pk, ps)
    assert abs(ref["cost"] - ro) <= 1e-12 * ro
    assert np.abs(Hr - Ho).max() <= 1e-10 * np.abs(Ho).max()
    Rp = [mr.pose(p) for p in x]
    assert abs(mr.total_cost(Rp, factors, fk, fs, priors, pk, ps) - ref["cost"]) <= 1e-13 * ref["cost"]
    coords = np.arange(6 * P)
    gfd = mr.grad_fd(x, coords, factors, fk, fs, priors, pk, ps)
    gx = np.array([float(v) for v in gfd])
    assert np.abs(gx - gr).max() <= 1e-15 * np.abs(gr).max()  # both rounded from 50 digits

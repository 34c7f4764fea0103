"""CPU checks of the extended-precision covariance reference (tests/cov_mp_ref.py): its vectorised Ls restatement is
numpy_cov.left_jacobian_point's (which test_cov_oracle.py pins to central differences of the C oracle's gradient), its
c_cov convention is the library's isotropic one, and its double-double solve agrees with mpmath at 40 digits."""
import mpmath
import numpy as np
import pytest

import cov_mp_ref as mr
import numpy_cov as nc
import scenes


@pytest.mark.parametrize("drop,with_fix", [(0.0, True), (0.5, True), (0.3, False)])
def test_vectorised_restatement_is_numpy_cov(drop, with_fix):
    sc = scenes.make_scene(n_poses=7, n_planes=10, seed=31, drop=drop, with_fix=with_fix, pts_size=15)
    args = (7, sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc["poses_init"], sc["fix10"])
    cc = mr.random_spd_ccov(sc["obs10"], 0.01, np.random.default_rng(2))
    R, A, E = mr.raw_reference(*args, c_cov=cc)
    ref, Ls = nc.left_jacobian_point(*args, c_cov=cc, return_Ls=True)
    assert np.all(np.abs(R - ref) <= mr.raw_bound(A, E))  # two fp64 restatements: 4e-14 of A apart here
    assert np.all(np.abs(R) <= A) and np.all(E >= 0) and np.all(E <= 1e-12 * A)
    # every observation's Ls, entry for entry, and zero on the rows of poses that do not see the voxel
    for a, slots, rows, L, e_v in mr.voxel_terms(*args):
        for jj, s in enumerate(slots):
            full = Ls[(a, s)]
            assert np.abs(full[rows] - L[jj]).max() <= 1e-13 * np.abs(full).max()
            assert not np.delete(full, rows, axis=0).any()


def test_ccov_convention_is_the_isotropic_one():
    sc = scenes.make_scene(n_poses=5, n_planes=8, seed=32, drop=0.2, with_fix=True, pts_size=12)
    args = (5, sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc["poses_gt"], sc["fix10"])
    iso = mr.raw_reference(*args, pnoise=0.02)[0]
    cc = np.stack([nc.cluster_cov_isotropic(o, 0.02) for o in sc["obs10"]])
    assert np.array_equal(mr.raw_reference(*args, c_cov=cc)[0], iso)
    assert np.array_equal(nc.left_jacobian_point(*args, pnoise=0.02), nc.left_jacobian_point(*args, c_cov=cc))
    # parameters (P00, P01, P02, P11, P12, P22, v0, v1, v2): the isotropic v block is pnoise^2 N I, the (P00, v0) coupling
    # 2 pnoise^2 v0 (Bf = [Bi; I], Bi[0] = (2x, 0, 0))
    assert np.allclose(cc[0][6:, 6:], 0.02 ** 2 * sc["obs10"][0, 9] * np.eye(3), rtol=1e-15, atol=0)
    assert np.isclose(cc[0][0, 6], 0.02 ** 2 * 2 * sc["obs10"][0, 6], rtol=1e-15, atol=0)
    # the layout probe's matrices: (e, f) and (f, e) one, the rest zero; the 45 of them cover every entry once
    cover = sum(mr.pair_ccov(e, f) for e in range(9) for f in range(e, 9))
    assert np.array_equal(cover, np.ones((9, 9)))


def _spd(n, cond, rng):
    Q, _ = np.linalg.qr(rng.normal(size=(n, n)))
    H = (Q * np.logspace(0, np.log10(cond), n)) @ Q.T
    d = np.logspace(0, 3, n)  # badly scaled, as a pose's rotation rows far from the origin are
    return H * d[:, None] * d[None, :]


def test_double_double_solve_agrees_with_mpmath():
    rng = np.random.default_rng(5)
    n = 14
    H = _spd(n, 1e6, rng)
    B = rng.normal(size=(n, 3))
    Xh, Xl = mr.solve_dd(H, B)
    Xm = mr.solve_mp(H, B, dps=40)
    with mpmath.workdps(40):
        err = max(abs((mpmath.mpf(float(Xh[i, j])) + mpmath.mpf(float(Xl[i, j])) - Xm[i][j]) / Xm[i][j])
                  for i in range(n) for j in range(3))
    assert err <= 1e-22  # ~32 digits, times kappa 1e6
    # the fp64 Cholesky solve is within its kappa bound of it, the double-double one far inside
    R = rng.normal(size=(n, n))
    R = R @ R.T
    ref = mr.cov_dd(H, R)
    k = mr.kappa_scaled(H)
    assert k < 1e7
    assert np.all(np.abs(mr.cov_fp64(H, R) - ref) <= mr.cov_bound(ref, k, n, 1.0))
    Xm = mr.solve_mp(H, R, dps=40)
    Ym = mr.solve_mp(H, [[Xm[i][j] for i in range(n)] for j in range(n)], dps=40)  # H^-1 (H^-1 R)^T at 40 digits
    Ymf = np.array([[float(y) for y in r] for r in Ym])
    assert np.all(np.abs(Ymf - ref) <= 4 * mr.EPS * np.abs(Ymf))  # cov_dd is H^-1 R H^-T correctly rounded, nearly


def test_shifted_scene_is_the_same_scene():
    """The moved fix clusters are the moments of the moved points: the cost at the moved poses is the cost."""
    from oracle import oracle_py as orc
    sc = scenes.make_scene(n_poses=4, n_planes=6, seed=33, with_fix=True, pts_size=10)
    x0 = sc["poses_gt"]
    r0 = orc.Oracle(4, sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc["fix10"]).residual(x0)
    x1, f1 = mr.shift_scene(sc, [30.0, -40.0, 12.0], x0)
    r1 = orc.Oracle(4, sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], f1).residual(x1)
    assert abs(r1 - r0) <= 1e-6 * abs(r0)

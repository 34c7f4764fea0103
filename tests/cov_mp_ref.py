"""Extended-precision reference of the pose-covariance propagation (balm_pose_covariance, balm_batch_pose_covariance),
per entry. TEST INFRASTRUCTURE.

Rcov_raw = sum over observations (a, s) of Ls c_s Ls^T, with Ls the dense restatement of tests/numpy_cov.py
(left_jacobian_point, BAs_left.hpp:342-473) evaluated on the rows of the poses that see voxel a only (Ls is zero
elsewhere), vectorised over those poses. Next to it the same sum of |Ls| |c| |Ls|^T, the scale of every rounding error
an fp64 evaluation of the sum can make, and that scale weighted per voxel by e_v below.

Formulation error. Every fp64 evaluation (the device, the C oracle, numpy_cov and this module) forms a voxel's
covariance as C/NN - v_bar v_bar^T from world-frame moments. The moments are of size mean |x|^2 (x the world points), so
that difference carries an absolute error of about eps mean |x|^2, and its eigenvectors -- which Ls and H are built
from -- turn by about eps mean |x|^2 / (lambda_1 - lambda_0); the inverse gaps 1 / (lambda_0 - lambda_k) in Ls move by
the same relative amount. So each voxel's terms are uncertain by
    e_v = eps * mean |x|^2 / (lambda_1 - lambda_0)
relative to |Ls| |c| |Ls|^T, in every implementation alike. Near the origin e_v is tens of eps; 1 km away it is ~1e-9.

Rcov = H^-1 Rcov_raw H^-T: solve_dd solves with H in double-double arithmetic (~32 significant digits: every operation
an error-free transformation of fp64 pairs, Gaussian elimination without pivoting, which is stable for SPD H),
vectorised so n = 198 takes about a second where mpmath's pure-Python arithmetic would take minutes. solve_mp (mpmath at
40 digits) is the check of solve_dd at small n (tests/test_cov_mp_ref.py). cov_fp64 is the LAPACK (Cholesky) form for
large n, whose own error is bounded like the device's (see kappa_scaled).
"""
import mpmath
import numpy as np
import scipy.linalg as sla

import numpy_cov as nc

EPS = np.finfo(np.float64).eps / 2  # unit roundoff 2^-53


# ---------------- Rcov_raw ----------------
def _T(pose12):
    T = np.eye(4)
    T[0:3, 0:3] = pose12[:9].reshape(3, 3).T
    T[0:3, 3] = pose12[9:12]
    return T


def voxel_terms(n_poses, row_ptr, pose_idx, obs10, coe, poses12, fix10=None):
    """Per voxel a: (a, slots, rows, Ls, e_v) with Ls [k, 6k, 9] the k observations' Ls on rows (the 6k coordinates of the
    poses that see the voxel, ascending) and e_v the voxel's formulation error (module docstring). Same formulas and
    names as numpy_cov.left_jacobian_point, the loop over poses p replaced by a batch dimension."""
    T = np.stack([_T(p) for p in np.asarray(poses12, dtype=np.float64)])
    Sp = np.zeros((3, 4)); Sp[0:3, 0:3] = np.eye(3)
    F = np.zeros((4, 4)); F[3, 3] = 1
    l = 0
    for a in range(len(row_ptr) - 1):
        slots = np.arange(row_ptr[a], row_ptr[a + 1])
        seen = np.asarray(pose_idx[slots])
        k = len(seen)
        Ts = T[seen]
        Co = np.stack([nc._C4(obs10[s]) for s in slots])
        TC = Ts @ Co
        C = (np.zeros((4, 4)) if fix10 is None else nc._C4(fix10[a])) + (TC @ Ts.transpose(0, 2, 1)).sum(0)
        NN = C[3, 3]
        C = C / NN
        v_bar = C[0:3, 3]
        lmbd, Uev = np.linalg.eigh(C[0:3, 0:3] - np.outer(v_bar, v_bar))
        u = [Uev[:, 0], Uev[:, 1], Uev[:, 2]]
        e_v = EPS * np.trace(C[0:3, 0:3]) / (lmbd[1] - lmbd[0])
        Ul = np.zeros((6, 4))
        Ul[0:3, 0:3] = nc.hat(-u[l])
        Ul[3:6, 3] = u[l]
        SpTul = Sp.T @ u[l]
        T_FC = Ts.transpose(0, 2, 1) - F @ C              # [k, 4, 4]
        UlTC = Ul @ TC                                      # [k, 6, 4]
        w2 = TC @ T_FC @ SpTul                              # [k, 4]
        g2w = np.zeros((k, 6, 3))
        for i in range(k):
            g2w[i] = nc.g2(w2[i])
        g2_combos = g2w + UlTC @ T_FC @ Sp.T                # [k, 6, 3]
        UlTCF = UlTC @ F
        g1_FC = nc.g1(F @ C @ Sp.T @ u[l])
        Ls = np.zeros((k, 6 * k, 9))
        for jj in range(k):
            Tj = Ts[jj]
            g1_TSu = nc.g1(Tj.T @ SpTul)
            Gkl = T_FC[jj].T @ g1_TSu - Tj @ g1_FC
            G = np.zeros((3, 9))
            for kk in range(3):
                if kk != l:
                    G += 1.0 / (lmbd[l] - lmbd[kk]) / NN * np.outer(u[kk], u[kk]) @ Sp @ Gkl
            Lp = g2_combos @ G - 1.0 / NN * UlTCF @ (Tj @ g1_TSu)   # [k, 6, 9]
            Lp[jj] += Ul @ Tj @ nc.g1(T_FC[jj] @ SpTul)
            Ls[jj] = (2.0 / NN * coe[a]) * Lp.reshape(6 * k, 9)
        rows = (6 * seen[:, None] + np.arange(6)).ravel()
        yield a, slots, rows, Ls, e_v


def accumulate(n_poses, terms, c_cov):
    """sum Ls c Ls^T, sum |Ls| |c| |Ls|^T and sum e_v |Ls| |c| |Ls|^T (each 6N x 6N) over the voxel terms; c_cov[s] the
    9 x 9 covariance of observation s."""
    n = 6 * n_poses
    R, A, E = np.zeros((n, n)), np.zeros((n, n)), np.zeros((n, n))
    for a, slots, rows, Ls, e_v in terms:
        cc = np.asarray(c_cov[slots])
        LC = np.einsum("jre,jef->rjf", Ls, cc).reshape(len(rows), -1)          # [Ls_1 c_1 | Ls_2 c_2 | ...]
        LA = np.einsum("jre,jef->rjf", np.abs(Ls), np.abs(cc)).reshape(len(rows), -1)
        L2 = Ls.transpose(1, 0, 2).reshape(len(rows), -1)                        # [Ls_1 | Ls_2 | ...]
        ix = np.ix_(rows, rows)
        R[ix] += LC @ L2.T
        Av = LA @ np.abs(L2).T
        A[ix] += Av
        E[ix] += e_v * Av
    return R, A, E


def raw_reference(n_poses, row_ptr, pose_idx, obs10, coe, poses12, fix10=None, c_cov=None, pnoise=None):
    """-> (Rcov_raw, sum |Ls| |c| |Ls|^T, sum e_v |Ls| |c| |Ls|^T); c_cov [K, 9, 9] or None for isotropic point noise
    pnoise (numpy_cov.cluster_cov_isotropic, as the library builds it)."""
    if c_cov is None:
        c_cov = np.stack([nc.cluster_cov_isotropic(o, pnoise) for o in obs10])
    terms = voxel_terms(n_poses, row_ptr, pose_idx, obs10, coe, poses12, fix10)
    return accumulate(n_poses, terms, np.asarray(c_cov, dtype=np.float64).reshape(-1, 9, 9))


def raw_bound(A, E, tau_r=32 * EPS, c_f=16.0):
    """Per-entry bound of |Rcov_raw - reference|: tau_r |Ls||c||Ls|^T (the rounding of any fp64 evaluation of the sum:
    each term is a product of a few dozen roundings, and the device reaches it through Q V^T + V Q^T, a different but
    equally short chain) plus c_f sum_v e_v |Ls||c||Ls|^T, the formulation error (module docstring): Ls is a product of
    up to three eigen-quantities (u_0, u_k and 1 / (lambda_0 - lambda_k)), each off by e_v, so Ls moves by up to 3 e_v
    and Ls c Ls^T by up to 6 e_v, rounded up to 8, in the evaluation under test and in the reference independently."""
    return tau_r * A + c_f * E


def random_spd_ccov(obs10, pnoise, rng):
    """Per observation an anisotropic SPD 9 x 9 c_cov with every entry coupled: W W^T / 9 + I / 10 (W standard normal),
    scaled by pnoise^2 N like the isotropic one."""
    K = len(obs10)
    W = rng.normal(size=(K, 9, 9))
    c = W @ W.transpose(0, 2, 1) / 9 + 0.1 * np.eye(9)
    return c * (pnoise * pnoise * np.asarray(obs10)[:, 9])[:, None, None]


def pair_ccov(e, f):
    """The 9 x 9 c_cov with only (e, f) and (f, e) set to one: pins c_cov's parameter order and indexing."""
    c = np.zeros((9, 9))
    c[e, f] = c[f, e] = 1.0
    return c


# ---------------- H^-1 R H^-T ----------------
_SPLITTER = 134217729.0  # 2^27 + 1


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _fast_two_sum(a, b):
    s = a + b
    return s, b - (s - a)


def _split(a):
    t = _SPLITTER * a
    hi = t - (t - a)
    return hi, a - hi


def _two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def dd_add(ah, al, bh, bl):
    s, e = _two_sum(ah, bh)
    t, f = _two_sum(al, bl)
    s, e = _fast_two_sum(s, e + t)
    return _fast_two_sum(s, e + f)


def dd_mul(ah, al, bh, bl):
    p, e = _two_prod(ah, bh)
    return _fast_two_sum(p, e + (ah * bl + al * bh))


def dd_div(ah, al, bh, bl):
    q1 = ah / bh
    ph, pl = dd_mul(q1, 0.0, bh, bl)
    rh, rl = dd_add(ah, al, -ph, -pl)
    q2 = rh / bh
    ph, pl = dd_mul(q2, 0.0, bh, bl)
    rh, rl = dd_add(rh, rl, -ph, -pl)
    q3 = rh / bh
    s, e = _fast_two_sum(q1, q2)
    return dd_add(s, e, q3, 0.0)


def solve_dd(H, Bh, Bl=None):
    """H^-1 B in double-double for SPD H (fp64) and B = Bh + Bl -> (Xh, Xl)."""
    H = np.asarray(H, dtype=np.float64)
    n = len(H)
    Ah, Al = H.copy(), np.zeros_like(H)
    Xh = np.array(Bh, dtype=np.float64, copy=True)
    Xl = np.zeros_like(Xh) if Bl is None else np.array(Bl, dtype=np.float64, copy=True)
    for k in range(n - 1):  # elimination: rows below k -= f A[k]
        fh, fl = dd_div(Ah[k + 1:, k], Al[k + 1:, k], Ah[k, k], Al[k, k])
        fh, fl = fh[:, None], fl[:, None]
        ph, pl = dd_mul(fh, fl, Ah[k, None, k + 1:], Al[k, None, k + 1:])
        Ah[k + 1:, k + 1:], Al[k + 1:, k + 1:] = dd_add(Ah[k + 1:, k + 1:], Al[k + 1:, k + 1:], -ph, -pl)
        ph, pl = dd_mul(fh, fl, Xh[k, None], Xl[k, None])
        Xh[k + 1:], Xl[k + 1:] = dd_add(Xh[k + 1:], Xl[k + 1:], -ph, -pl)
    for k in range(n - 1, -1, -1):  # back substitution, column-oriented
        Xh[k], Xl[k] = dd_div(Xh[k], Xl[k], Ah[k, k], Al[k, k])
        if k:
            ph, pl = dd_mul(Ah[:k, k, None], Al[:k, k, None], Xh[k, None], Xl[k, None])
            Xh[:k], Xl[:k] = dd_add(Xh[:k], Xl[:k], -ph, -pl)
    return Xh, Xl


def cov_dd(H, R):
    """H^-1 R H^-T in double-double, rounded to fp64 (R symmetric: H^-1 (H^-1 R)^T)."""
    Xh, Xl = solve_dd(H, R)
    Yh, Yl = solve_dd(H, Xh.T, Xl.T)
    return Yh + Yl


def cov_fp64(H, R):
    """H^-1 R H^-T through LAPACK's Cholesky in fp64."""
    f = sla.cho_factor(H, lower=True)
    X = sla.cho_solve(f, R)
    return sla.cho_solve(f, X.T)


def solve_mp(H, B, dps=40):
    """H^-1 B in mpmath at dps digits (pure Python Gaussian elimination; small n only); B an array or rows of mpf ->
    rows of mpf."""
    with mpmath.workdps(dps):
        n = len(H)
        A = [[mpmath.mpf(float(x)) for x in r] for r in np.asarray(H)]
        X = [[mpmath.mpf(x) for x in r] for r in B]
        for k in range(n):
            for i in range(k + 1, n):
                f = A[i][k] / A[k][k]
                A[i] = [A[i][j] - f * A[k][j] if j > k else A[i][j] for j in range(n)]
                X[i] = [x - f * y for x, y in zip(X[i], X[k])]
        for k in range(n - 1, -1, -1):
            X[k] = [x / A[k][k] for x in X[k]]
            for i in range(k):
                X[i] = [x - A[i][k] * y for x, y in zip(X[i], X[k])]
        return X


def kappa_scaled(H):
    """2-norm condition number of D^-1/2 H D^-1/2, D = diag(H). A backward-stable LDL^T / Cholesky solve with SPD H is
    accurate to about n eps times this in the scaled coordinates, whatever the diagonal scaling (the rotation block of
    a pose far from the origin is |p|^2 times its translation block); inf when the scaled H is not positive definite."""
    s = 1.0 / np.sqrt(np.diag(H))
    ev = np.linalg.eigvalsh(H * s[:, None] * s[None, :])
    return ev[-1] / ev[0] if ev[0] > 0 else np.inf


def cov_bound(cov_ref, kappa, n, C):
    """Per-entry bound of a solve's error in H^-1 R H^-T at correlation scale: C n kappa eps sqrt(ref_ii ref_jj)."""
    d = np.sqrt(np.abs(np.diag(cov_ref)))
    return C * n * kappa * EPS * np.outer(d, d)


# ---------------- scenes ----------------
def shift_scene(sc, t, poses):
    """The scene moved by world translation t: poses p_i + t, fix clusters' moments of the points x + t
    (P' = P + v t^T + t v^T + N t t^T, v' = v + N t); body-frame observations unchanged. -> (poses, fix10)."""
    t = np.asarray(t, dtype=np.float64)
    x = np.array(poses, dtype=np.float64, copy=True)
    x[:, 9:12] += t
    f = sc["fix10"]
    if f is None:
        return x, None
    f = f.copy()
    iu = ([0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2])
    P = np.stack([nc._C4(o)[0:3, 0:3] for o in f])
    v, N = f[:, 6:9], f[:, 9]
    P = P + v[:, :, None] * t[None, None, :] + t[None, :, None] * v[:, None, :] + N[:, None, None] * np.outer(t, t)
    f[:, 0:6] = P[:, iu[0], iu[1]]
    f[:, 6:9] = v + N[:, None] * t
    return x, f

"""Extended-precision reference of the pose-factor and pose-prior terms of balm_b200/csrc/pose_graph.cu, per entry.
TEST INFRASTRUCTURE.

Independent of the device formulas (and of pose_graph_ref / pose_priors_ref, which restate them): every fp64 input is
taken exactly as an mpmath number and everything below runs at DPS = 50 digits.
  - Residuals from their definitions. Factor slot k >= 1: T = A^-1 T_k with A = T_0 T^_0^-1, D = R R^_k^T and
    e_k = (Log D, p - D p^_k); prior: D = R R^^T, e = (Log D, R l + p - p^). D is formed exactly from the fp64 poses, so
    it is orthogonal only to about eps; Log D is the log of its polar factor D (D^T D)^-1/2, the rotation nearest to D:
    its quaternion is the top eigenvector of Bar-Itzhack's 4 x 4 matrix K(D). For an orthogonal D the spectrum of K is
    {1, -1/3, -1/3, -1/3}, so power iteration on K + I/3 gains a factor of about eps per step from the fp64 eigenvector
    and four steps reach 50 digits. The angle is 2 atan2(|q_v|, q_w), which is accurate at every angle up to pi; the
    polar projection matters near pi, where the matrix log of a D that is not orthogonal moves by (theta / sin theta) eps
    (log_so3_logm, vee(logm(polar(D))), is the check of this closed form, tests/test_pose_terms_mp_ref.py).
  - Jacobians E = de / d(delta) of every slot, slot 0 included, and of the prior pose, by central differences through
    the left update R <- Exp(phi) R, p <- Exp(phi) p + t (Exp by Rodrigues at 50 digits) with step H_STEP = 1e-20:
    truncation about 1e-40, cancellation 20 of the 50 digits. No closed-form J or Jl^-1 is used.
  - Terms: s = e~^T H~ e~, cost 1/2 rho(s), w = rho'(s), M = w E^T H~ E, b = w E^T H~ e~; dense H, g and the total cost.
    grad_fd() is the central-difference gradient of the total robust cost, the check of g without the IRLS formula.

Error scales and the bound. Every fp64 evaluation (the device's included) forms D and A^-1 p out of fp64 products, so
its e carries a formulation error that no arithmetic can remove: about eps on each rotation component and
eps (1 + |p_0| + |p_k| + |p^_0| + |p^_k|) on each translation component (prior: eps (1 + |p| + |l| + |p^|)); write
eps d_e for it (d_e per component, in units of eps). J's rotation-rotation and translation-translation blocks (Jl^-1 Q,
Q) are sums of products of unit-sized numbers and its translation-rotation block holds Q hat(p_k - R_k R^_k^T p^_k),
whose entries carry the translation error; write eps d_E for that (1 on the first two blocks, the translation d_e on the
third). Then per entry, with |.| elementwise and the rounding of the evaluation itself bounded by the same magnitudes:
    s:   scale_s = |e~|^T |H~| (|e~| + 2 d_e)
    M:   scale_M = w (|E| + d_E)^T |H~| (|E| + d_E) + |rho''(s)| scale_s |M / w|
    b:   scale_b = w (|E| + d_E)^T |H~| (|e~| + d_e) + |rho''(s)| scale_s |b / w|
    cost: 1/2 (w scale_s + |rho(s)|)
summed over every term and factor of an entry without credit for cancellation (the slot-0 rows and columns and the
pair sums included, which the device forms by cancelling sums), and
    |device - reference| <= C eps scale,   C = 64,   eps = 2^-53.
C covers the longest chain of roundings one entry passes through on the device -- D (two 3-term products), the log, J
(two more), M (two 6-term sums), the slot-0 sums over up to 31 slots and a pair sum over the factors -- each bounded by
the magnitudes above; errors of sums that long add like a random walk, well inside 64. The same C holds for every case;
ratio() gives the worst ratio of an evaluation's errors to it.
"""
import mpmath
import numpy as np

DPS = 50
EPS = 2.0 ** -53
C = 64.0
H_STEP = mpmath.mpf("1e-20")
TRIVIAL, HUBER, CAUCHY = 0, 1, 2

_MP = mpmath.mp
_MP.dps = DPS

# rotation-residual magnitudes the tests reach: exact zero, the series switch of Jl^-1 at 0.1 and one ulp-scale step
# either side, the series' range, the c > 0 switch of the device's log at pi/2, and the approach to pi
ANGLES = (0.0, 1e-12, 1e-8, 1e-4, 0.1 * (1 - 2.0 ** -40), 0.1, 0.1 * (1 + 2.0 ** -40), 0.25, 1.0,
          np.pi / 2 - 1e-9, np.pi / 2, np.pi / 2 + 1e-9, 2.5, np.pi - 1e-3, np.pi - 1e-6)
# coordinate, diagonal ((1, 1, 0) / sqrt 2 ties two diagonal entries of the device's B near pi) and generic axes
AXES = (np.array([1.0, 0.0, 0.0]), np.array([0.0, 0.0, 1.0]), np.array([1.0, 1.0, 0.0]) / np.sqrt(2.0),
        np.array([1.0, 1.0, 1.0]) / np.sqrt(3.0), np.array([0.48, -0.6, 0.64]))


def rot64(theta, axis):
    """fp64 rotation by theta about the unit axis (Rodrigues, no small-angle cut-off; theta = 0 gives I exactly)"""
    K = np.array([[0.0, -axis[2], axis[1]], [axis[2], 0.0, -axis[0]], [-axis[1], axis[0], 0.0]])
    return np.eye(3) + np.sin(theta) * K + (1.0 - np.cos(theta)) * K @ K


def mpa(x):
    """fp64 array -> object array of exact mpf"""
    x = np.asarray(x, dtype=np.float64)
    return np.array([mpmath.mpf(float(v)) for v in x.ravel()], dtype=object).reshape(x.shape)


def to_f(x):
    return np.array([float(v) for v in np.asarray(x, dtype=object).ravel()]).reshape(np.shape(x))


def pose(p12):
    """pose12 (R column-major, then p) -> (R [3, 3], p [3]) as mpf, exactly"""
    p12 = mpa(p12)
    return p12[:9].reshape(3, 3).T.copy(), p12[9:].copy()


def hat(v):
    z = mpmath.mpf(0)
    return np.array([[z, -v[2], v[1]], [v[2], z, -v[0]], [-v[1], v[0], z]], dtype=object)


def exp_so3(phi):
    """Rodrigues at DPS digits"""
    t = mpmath.sqrt(sum(x * x for x in phi))
    eye = np.array([[mpmath.mpf(int(a == b)) for b in range(3)] for a in range(3)], dtype=object)
    if t == 0:
        return eye
    K = hat(phi)
    return eye + (mpmath.sin(t) / t) * K + ((1 - mpmath.cos(t)) / (t * t)) * K.dot(K)


def _bar_itzhack(D):
    (xx, xy, xz), (yx, yy, yz), (zx, zy, zz) = D
    return np.array([[xx - yy - zz, yx + xy, zx + xz, zy - yz],
                     [yx + xy, yy - xx - zz, zy + yz, xz - zx],
                     [zx + xz, zy + yz, zz - xx - yy, yx - xy],
                     [zy - yz, xz - zx, yx - xy, xx + yy + zz]], dtype=object) / 3


def log_so3(D):
    """vee(Log) of the rotation nearest to D (its polar factor), through the quaternion (module docstring)"""
    K = _bar_itzhack(D)
    lam, V = np.linalg.eigh(to_f(K))
    q = mpa(V[:, np.argmax(lam)])
    Ks = K + np.diag([mpmath.mpf(1) / 3] * 4)
    for _ in range(5):
        q = Ks.dot(q)
        q = q / mpmath.sqrt(sum(x * x for x in q))
    if q[3] < 0:
        q = -q
    nv = mpmath.sqrt(q[0] ** 2 + q[1] ** 2 + q[2] ** 2)
    if nv == 0:
        return np.array([mpmath.mpf(0)] * 3, dtype=object)
    return (2 * mpmath.atan2(nv, q[3]) / nv) * q[:3]


def log_so3_logm(D):
    """vee of the principal matrix log of polar(D) = D (D^T D)^-1/2 (the check of log_so3). The log is taken through
    the eigendecomposition, V diag(log lambda) V^-1: mpmath.logm leaves the principal branch as theta nears pi."""
    Dm = mpmath.matrix(D.tolist())
    P = Dm * mpmath.inverse(mpmath.sqrtm(Dm.T * Dm))
    lam, V = mpmath.eig(P)
    L = V * mpmath.diag([mpmath.log(x) for x in lam]) * mpmath.inverse(V)
    return np.array([mpmath.re(L[2, 1] - L[1, 2]) / 2, mpmath.re(L[0, 2] - L[2, 0]) / 2,
                     mpmath.re(L[1, 0] - L[0, 1]) / 2], dtype=object)


def _update(R, p, d):
    """left update by d (6): R <- Exp(d[:3]) R, p <- Exp(d[:3]) p + d[3:]"""
    X = exp_so3(d[:3])
    return X.dot(R), X.dot(p) + d[3:]


def _fd(fun, R, p):
    """[6, 6] central-difference Jacobian of fun(R, p) (6) under the left update"""
    J = np.empty((6, 6), dtype=object)
    z = mpmath.mpf(0)
    for j in range(6):
        d = np.array([z] * 6, dtype=object)
        d[j] = H_STEP
        J[:, j] = (fun(*_update(R, p, d)) - fun(*_update(R, p, -d))) / (2 * H_STEP)
    return J


def factor_residual(R0, p0, Rk, pk, Rh0, ph0, Rhk, phk):
    """e_k (6) from its definition: T = A^-1 T_k, A = T_0 T^_0^-1"""
    Q = Rh0.dot(R0.T)
    Rs, ps = Q.dot(Rk), Q.dot(pk - p0) + ph0
    D = Rs.dot(Rhk.T)
    return np.concatenate([log_so3(D), ps - D.dot(phk)])


def prior_residual(R, p, Rh, ph, lever):
    return np.concatenate([log_so3(R.dot(Rh.T)), R.dot(lever) + p - ph])


# ---------------- robust losses ----------------
def rho(kind, c, s):
    c2 = c * c
    if kind == HUBER and s > c2:
        return 2 * c * mpmath.sqrt(s) - c2
    if kind == CAUCHY:
        return c2 * mpmath.log1p(s / c2)
    return s


def drho(kind, c, s):
    c2 = c * c
    if kind == HUBER and s > c2:
        return c / mpmath.sqrt(s)
    if kind == CAUCHY:
        return 1 / (1 + s / c2)
    return mpmath.mpf(1)


def d2rho_abs(kind, c, s):
    """|rho''(s)|; on Huber within 1e-6 of its kink the quadratic side's 0 is replaced by the other side's value"""
    c2 = c * c
    if kind == HUBER and s > c2 * (1 - mpmath.mpf("1e-6")):
        return c / (2 * s * mpmath.sqrt(s))
    if kind == CAUCHY:
        return 1 / (c2 * (1 + s / c2) ** 2)
    return mpmath.mpf(0)


# ---------------- terms ----------------
def _base(e, E, Ht, de, dE):
    """The loss-free part of one term: e [m], E [m, n], H~ [m, m] (mpf), d_e [m] and d_E [m, n] (floats, units of eps)
    -> s, M0 = E^T H~ E, b0 = E^T H~ e and their scales without a loss (module docstring)"""
    He = Ht.dot(e)
    aH, ae, aE = np.abs(to_f(Ht)), np.abs(to_f(e)), np.abs(to_f(E)) + dE
    return dict(s=e.dot(He), M0=E.T.dot(Ht.dot(E)), b0=E.T.dot(He), s_scale=ae @ aH @ (ae + 2 * de),
                M0_scale=aE.T @ aH @ aE, b0_scale=aE.T @ aH @ (ae + de))


def with_loss(base, kind=TRIVIAL, c=1.0):
    """_base's term under the loss (kind, c) -> dict(s, w, cost, M, b) (mpf) and their scales"""
    c = mpmath.mpf(float(c))
    s = base["s"]
    w, r = drho(kind, c, s), rho(kind, c, s)
    d2, wf, ss = float(d2rho_abs(kind, c, s)), float(w), base["s_scale"]
    return dict(s=s, w=w, cost=r / 2, M=w * base["M0"], b=w * base["b0"],
                s_scale=ss, w_scale=d2 * ss + wf, cost_scale=0.5 * (wf * ss + abs(float(r))),
                M_scale=wf * base["M0_scale"] + d2 * ss * np.abs(to_f(base["M0"])),
                b_scale=wf * base["b0_scale"] + d2 * ss * np.abs(to_f(base["b0"])))


def factor_base(poses12, f):
    """One factor dict (poses, poses_hat, H) at the global poses -> _base's dict over its 6 N coordinates (slot order)"""
    idx, Th, Hf = f["poses"], f["poses_hat"], f["H"]
    N = len(idx)
    T = [pose(poses12[i]) for i in idx]
    Hh = [pose(h) for h in Th]
    m = 6 * (N - 1)
    e = np.empty(m, dtype=object)
    E = np.array([[mpmath.mpf(0)] * (6 * N) for _ in range(m)], dtype=object)
    de, dE = np.zeros(m), np.zeros((m, 6 * N))
    R0, p0 = T[0]
    Rh0, ph0 = Hh[0]
    for k in range(1, N):
        Rk, pk = T[k]
        Rhk, phk = Hh[k]
        r = slice(6 * (k - 1), 6 * k)
        e[r] = factor_residual(R0, p0, Rk, pk, Rh0, ph0, Rhk, phk)
        E[r, 6 * k:6 * k + 6] = _fd(lambda R, p: factor_residual(R0, p0, R, p, Rh0, ph0, Rhk, phk), Rk, pk)
        E[r, 0:6] = _fd(lambda R, p: factor_residual(R, p, Rk, pk, Rh0, ph0, Rhk, phk), R0, p0)
        dt = 1 + sum(float(mpmath.sqrt(v.dot(v))) for v in (p0, pk, ph0, phk))
        de[r] = [1, 1, 1, dt, dt, dt]
        for col in (0, 6 * k):
            dE[r, col:col + 6] = np.block([[np.ones((3, 3)), np.zeros((3, 3))], [np.full((3, 3), dt), np.ones((3, 3))]])
    return _base(e, E, mpa(np.asarray(Hf)[6:, 6:]), de, dE)


def factor_terms(poses12, f, kind=TRIVIAL, c=1.0):
    return with_loss(factor_base(poses12, f), kind, c)


def prior_base(poses12, pr):
    """One prior dict (pose, pose_hat, H, optional lever_arm) -> _base's dict over its pose's 6 coordinates"""
    R, p = pose(poses12[pr["pose"]])
    Rh, ph = pose(pr["pose_hat"])
    lever = mpa(np.zeros(3) if pr.get("lever_arm") is None else pr["lever_arm"])
    e = prior_residual(R, p, Rh, ph, lever)
    E = _fd(lambda R_, p_: prior_residual(R_, p_, Rh, ph, lever), R, p)
    dt = 1 + sum(float(mpmath.sqrt(v.dot(v))) for v in (p, ph, lever))
    de = np.array([1, 1, 1, dt, dt, dt], dtype=np.float64)
    dE = np.block([[np.ones((3, 3)), np.zeros((3, 3))], [np.full((3, 3), dt), np.ones((3, 3))]])
    return _base(e, E, mpa(pr["H"]), de, dE)


def prior_terms(poses12, pr, kind=TRIVIAL, c=1.0):
    return with_loss(prior_base(poses12, pr), kind, c)


def assemble(factor_list, prior_list=()):
    """Reference H as 6 x 6 blocks, g and the cost from per-term dicts: factor_list of (factor dict, terms), prior_list
    of (prior dict, terms). -> dict(blocks {(i, j), i <= j: (H rows of pose i, columns of pose j [6, 6], its scale)},
    g {pose: (6, scale)}, cost, cost_scale); values rounded from the exact sums"""
    Hx, gx, cost, cost_scale = {}, {}, mpmath.mpf(0), 0.0

    def add(poses, t):
        nonlocal cost, cost_scale
        for a, i in enumerate(poses):
            v, sc = gx.get(i, (np.zeros(6, dtype=object), np.zeros(6)))
            gx[i] = (v + t["b"][6 * a:6 * a + 6], sc + t["b_scale"][6 * a:6 * a + 6])
            for b, j in enumerate(poses):
                if i <= j:
                    v, sc = Hx.get((i, j), (np.zeros((6, 6), dtype=object), np.zeros((6, 6))))
                    Hx[i, j] = (v + t["M"][6 * a:6 * a + 6, 6 * b:6 * b + 6],
                                sc + t["M_scale"][6 * a:6 * a + 6, 6 * b:6 * b + 6])
        cost += t["cost"]
        cost_scale += t["cost_scale"]

    for f, t in factor_list:
        add([int(i) for i in f["poses"]], t)
    for pr, t in prior_list:
        add([int(pr["pose"])], t)
    return dict(blocks={k: (to_f(v), sc) for k, (v, sc) in Hx.items()},
                g={k: (to_f(v), sc) for k, (v, sc) in gx.items()}, cost=float(cost), cost_scale=cost_scale)


def total_cost(Rp, factors, fk, fs, priors=(), pk=(), ps=()):
    """sum of 1/2 rho(s) over factors and priors at the poses Rp (a list of mpf (R, p)) -> mpf"""
    r = mpmath.mpf(0)
    for f, k, c in zip(factors, fk, fs):
        idx, h = f["poses"], [pose(t) for t in f["poses_hat"]]
        e = np.concatenate([factor_residual(*Rp[idx[0]], *Rp[idx[q]], *h[0], *h[q]) for q in range(1, len(idx))])
        r += rho(k, mpmath.mpf(float(c)), e.dot(mpa(np.asarray(f["H"])[6:, 6:]).dot(e))) / 2
    for pr, k, c in zip(priors, pk, ps):
        lever = mpa(np.zeros(3) if pr.get("lever_arm") is None else pr["lever_arm"])
        e = prior_residual(*Rp[pr["pose"]], *pose(pr["pose_hat"]), lever)
        r += rho(k, mpmath.mpf(float(c)), e.dot(mpa(pr["H"]).dot(e))) / 2
    return r


def grad_fd(poses12, coords, factors, fk, fs, priors=(), pk=(), ps=()):
    """central-difference gradient of the total robust cost at the coordinates coords (pose i, direction j: 6 i + j)"""
    base = [pose(p) for p in poses12]
    out = []
    z = mpmath.mpf(0)
    for q in coords:
        i, j = divmod(int(q), 6)
        d = np.array([z] * 6, dtype=object)
        d[j] = H_STEP
        vals = []
        for sgn in (1, -1):
            xs = list(base)
            xs[i] = _update(*base[i], sgn * d)
            vals.append(total_cost(xs, factors, fk, fs, priors, pk, ps))
        out.append((vals[0] - vals[1]) / (2 * H_STEP))
    return out


def ratio(dev, ref, scale):
    """max over entries of |dev - ref| / (C eps scale); entries whose scale is 0 must match exactly (inf otherwise)"""
    dev, ref, scale = np.asarray(dev, dtype=np.float64), np.asarray(ref, dtype=np.float64), np.asarray(scale)
    err = np.abs(dev - ref)
    bound = C * EPS * scale
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))
    return float(r.max()) if r.size else 0.0

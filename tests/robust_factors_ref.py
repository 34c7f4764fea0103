"""numpy restatement of the robust pose factors of balm_b200/csrc/pose_graph.cu (DESIGN.md "Robust pose factors"):

  with s_f = e~^T H~ e~ (twice pose_graph_ref's cost_f), w_f = rho'(s_f) and M_f, b_f pose_graph_ref's terms,
      cost_f = 1/2 rho(s_f),   g_f = w_f b_f,   H_f = w_f M_f   (IRLS: no rho'' term)

  kind 0 (trivial) rho = s; 1 (Huber) s for s <= c^2, else 2 c sqrt(s) - c^2; 2 (Cauchy) c^2 log(1 + s / c^2).

lm() is pose_graph_ref.lm's rule on this cost. outlier_scene() builds the loop-closure scene the tests use: laps of a
closed loop, noisy odometry, true closures between revisits and false (identity) closures between distant poses."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import balm_b200
import pose_graph_ref as pgr

TRIVIAL, HUBER, CAUCHY = 0, 1, 2
NAMES = {"trivial": TRIVIAL, "huber": HUBER, "cauchy": CAUCHY}
POINT_NOISE = 0.01       # sigma_p: the factors' H are 2 sigma_p^2 x information, as a voxel cost's are
CHI2_6_999 = 22.457744484825326  # chi-square quantile, 6 degrees of freedom, p = 0.999


def rho(kind, c, s):
    c2 = c * c
    if kind == HUBER and s > c2:
        return 2.0 * c * np.sqrt(s) - c2
    if kind == CAUCHY:
        return c2 * np.log1p(s / c2)
    return s


def drho(kind, c, s):
    c2 = c * c
    if kind == HUBER and s > c2:
        return c / np.sqrt(s)
    if kind == CAUCHY:
        return 1.0 / (1.0 + s / c2)
    return 1.0


def loss_arrays(n, kind, scale):
    """Python-API style (a name or one per factor; a scalar or one per factor) -> (kinds int array, scales array)"""
    kinds = np.array([NAMES[k] for k in ([kind] * n if isinstance(kind, str) else kind)], dtype=np.int32)
    scales = np.broadcast_to(np.asarray(1.0 if scale is None else scale, dtype=np.float64), (n,)).copy()
    return kinds, scales


def factor_terms(poses, f, kind, c):
    """-> (s, w, cost, w M, w b) of one factor"""
    e, E, q, M, b = pgr.factor_terms(poses, f)
    s = 2.0 * q
    w = drho(kind, c, s)
    return s, w, 0.5 * rho(kind, c, s), w * M, w * b


def _slots(f):
    return np.concatenate([np.arange(6 * i, 6 * i + 6) for i in f["poses"]])


def evaluate(poses, factors, P, kinds, scales, sparse=False):
    """H (dense 6P x 6P, or scipy csc with sparse=True), g, cost of the factors (all taken as active)"""
    rows, cols, vals = [], [], []
    g = np.zeros(6 * P)
    r = 0.0
    for f, k, c in zip(factors, kinds, scales):
        _, _, cf, M, b = factor_terms(poses, f, k, c)
        sl = _slots(f)
        rows.append(np.repeat(sl, len(sl)))
        cols.append(np.tile(sl, len(sl)))
        vals.append(M.ravel())
        g[sl] += b
        r += cf
    H = sp.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(6 * P, 6 * P))
    return (H.tocsc() if sparse else H.toarray()), g, r


def cost(poses, factors, kinds, scales):
    return float(sum(factor_terms(poses, f, k, c)[2] for f, k, c in zip(factors, kinds, scales)))


def residuals(poses, factors, kinds, scales):
    """-> (s, w) per factor"""
    out = np.array([factor_terms(poses, f, k, c)[:2] for f, k, c in zip(factors, kinds, scales)])
    return out[:, 0], out[:, 1]


def lm(poses0, factors, P, kinds, scales, max_iter=10, u0=0.01, v0=2.0, rel_tol=1e-6, sparse=False):
    """pose_graph_ref.lm's rule on the robust cost -> (poses, trace, poses per iteration)"""
    x = np.array(poses0, dtype=np.float64, copy=True)
    u, v = u0, v0
    calc, trace, per = True, [], []
    H = g = None
    r1 = 0.0
    for it in range(max_iter):
        if calc:
            H, g, r1 = evaluate(x, factors, P, kinds, scales, sparse)
        D = H.diagonal().copy()
        if sparse:
            dx = spla.spsolve((H + u * sp.diags(D)).tocsc(), -g)
        else:
            dx = np.linalg.solve(H + u * np.diag(D), -g)
        q1 = 0.5 * dx @ (u * D * dx - g)
        xt = pgr.pose_update(x, dx)
        r2 = cost(xt, factors, kinds, scales)
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


# ---------------- the outlier scene ----------------
def info(rot, tran):
    """information of N(0, rot) / N(0, tran) relative-pose noise, in the voxel cost's units (2 sigma_p^2 x information)"""
    return 2 * POINT_NOISE ** 2 * np.diag(np.r_[np.full(3, rot ** -2), np.full(3, tran ** -2)])


def noisy_relative(rng, gt, edges, om, rot, tran):
    """odometry_factors over edges (a, b) from the truth, each relative pose perturbed on the right by N(0, rot / tran)"""
    out = []
    for a, b in edges:
        Rb, pb = pgr.split(gt[b])
        d = np.concatenate([rng.normal(0, rot, 3), rng.normal(0, tran, 3)])
        hb = pgr.pack(Rb @ pgr.exp_so3(d[:3]), Rb @ d[3:] + pb)
        f = balm_b200.odometry_factors(np.stack([gt[a], hb]), om)[0]
        f["poses"] = np.array([a, b], dtype=np.int32)
        out.append(f)
    return out


def dead_reckoning(odo, x0):
    """poses chained from x0 through the odometry factors' relative poses T^_a^-1 T^_b"""
    out = [np.asarray(x0, dtype=np.float64)]
    for f in odo:
        R0, p0 = pgr.split(f["poses_hat"][0])
        R1, p1 = pgr.split(f["poses_hat"][1])
        Ra, pa = pgr.split(out[-1])
        Rr, pr = R0.T @ R1, R0.T @ (p1 - p0)
        out.append(pgr.pack(Ra @ Rr, Ra @ pr + pa))
    return np.array(out)


ODO_NOISE = (0.001, 0.01)    # rad, m per step
LOOP_NOISE = (0.002, 0.02)   # rad, m per closure


def outlier_scene(P, seed, lap=100, radius=15.0, every=4, false_frac=0.2, min_dist=20.0):
    """P poses on P / lap laps of a circle (each lap 0.3 m higher, with a small wobble), so that pose i >= lap revisits
    pose i - lap. Odometry between consecutive poses, a true closure (i - lap, i) every `every` poses of the later laps,
    and false closures (identity relative pose) between random pose pairs at least min_dist apart, false_frac of all
    closures. -> dict(gt, x0 (dead reckoning), odo, true, false, all (odo + true + false), clean (odo + true))"""
    rng = np.random.default_rng(seed)
    i = np.arange(P)
    th = 2 * np.pi * i / lap
    ps = np.stack([radius * np.cos(th), radius * np.sin(th), 0.3 * (i // lap) + 0.2 * np.sin(3 * th)], 1)
    Rs = [pgr.exp_so3(np.array([0.0, 0.0, t + np.pi / 2])) @ pgr.exp_so3(rng.normal(0, 0.02, 3)) for t in th]
    gt = np.array([pgr.pack(R, p) for R, p in zip(Rs, ps)])
    odo = noisy_relative(rng, gt, [(a, a + 1) for a in range(P - 1)], info(*ODO_NOISE), *ODO_NOISE)
    true = noisy_relative(rng, gt, [(b - lap, b) for b in range(lap, P, every)], info(*LOOP_NOISE), *LOOP_NOISE)
    n_false = int(round(false_frac * len(true) / (1 - false_frac)))
    pairs = set()
    while len(pairs) < n_false:
        a, b = sorted(rng.choice(P, 2, replace=False))
        if np.linalg.norm(ps[a] - ps[b]) >= min_dist:
            pairs.add((int(a), int(b)))
    false = []
    for a, b in sorted(pairs):
        f = balm_b200.odometry_factors(np.stack([gt[a], gt[a]]), info(*LOOP_NOISE))[0]
        f["poses"] = np.array([a, b], dtype=np.int32)
        false.append(f)
    x0 = dead_reckoning(odo, gt[0])
    return dict(gt=gt, x0=x0, odo=odo, true=true, false=false, all=odo + true + false, clean=odo + true)


def cauchy_scale():
    """c of a chi-square gate at p = 0.999 on factors in the voxel cost's units: c^2 = 2 sigma_p^2 chi2_6(0.999)"""
    return np.sqrt(2 * POINT_NOISE ** 2 * CHI2_6_999)


def align_rigid(poses, gt):
    """poses moved by the rigid transform (Kabsch on the positions) that best fits them to gt"""
    p = np.array([pgr.split(x)[1] for x in poses])
    q = np.array([pgr.split(x)[1] for x in gt])
    pm, qm = p.mean(0), q.mean(0)
    U, _, Vt = np.linalg.svd((q - qm).T @ (p - pm))
    A = U @ np.diag([1, 1, np.linalg.det(U @ Vt)]) @ Vt
    t = qm - A @ pm
    return np.array([pgr.pack(A @ pgr.split(x)[0], A @ pgr.split(x)[1] + t) for x in poses])


def max_error(poses, gt):
    """largest position error after rigid alignment"""
    a = align_rigid(poses, gt)
    return float(max(np.linalg.norm(pgr.split(x)[1] - pgr.split(y)[1]) for x, y in zip(a, gt)))

"""numpy restatement of the absolute pose priors of balm_b200/csrc/pose_graph.cu (DESIGN.md "Absolute pose priors"):

  a prior on pose i with measured pose T^ = (R^, p^), body-frame lever arm l and 6 x 6 PSD H, at T = (R, p):
      e = (Log(R R^^T), R l + p - p^),   s = e^T H e,   cost = 1/2 rho(s),
      J = [[Jl^-1(e_rot), 0], [-hat(R l + p), I]]   (left update R <- Exp(dtheta) R, p <- Exp(dtheta) p + dp),
      g = w J^T H e,   M = w J^T H J,   w = rho'(s)   (IRLS: no rho'' term)

evaluate() / cost() / lm() are robust_factors_ref's on the factors plus these priors; lm() takes no gauge step."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import pose_graph_ref as pgr
import robust_factors_ref as rfr


def prior_terms(poses, pr, kind=rfr.TRIVIAL, c=1.0):
    """-> (e, J, s, w, cost, M, b) of one prior dict (pose, pose_hat, H, optional lever_arm)"""
    R, p = pgr.split(poses[pr["pose"]])
    Rh, ph = pgr.split(pr["pose_hat"])
    lever = np.zeros(3) if pr.get("lever_arm") is None else np.asarray(pr["lever_arm"], dtype=np.float64)
    x = R @ lever + p
    phi = pgr.log_so3(R @ Rh.T)
    e = np.concatenate([phi, x - ph])
    J = np.zeros((6, 6))
    J[:3, :3] = pgr.jl_inv(phi)
    J[3:, :3] = -pgr.hat(x)
    J[3:, 3:] = np.eye(3)
    H = np.asarray(pr["H"], dtype=np.float64)
    s = float(e @ H @ e)
    w = rfr.drho(kind, c, s)
    return e, J, s, w, 0.5 * rfr.rho(kind, c, s), w * (J.T @ H @ J), w * (J.T @ H @ e)


def evaluate(poses, factors, priors, P, fk=None, fs=None, pk=None, ps=None, sparse=False):
    """H (dense, or scipy csc with sparse=True), g, cost of the factors (robust_factors_ref.evaluate) plus the priors"""
    fk = np.zeros(len(factors), dtype=np.int32) if fk is None else fk
    fs = np.ones(len(factors)) if fs is None else fs
    pk = np.zeros(len(priors), dtype=np.int32) if pk is None else pk
    ps = np.ones(len(priors)) if ps is None else ps
    if factors:
        H, g, r = rfr.evaluate(poses, factors, P, fk, fs, sparse=True)
    else:
        H, g, r = sp.csc_matrix((6 * P, 6 * P)), np.zeros(6 * P), 0.0
    rows, cols, vals = [], [], []
    for pr, k, c in zip(priors, pk, ps):
        _, _, _, _, cq, M, b = prior_terms(poses, pr, k, c)
        sl = np.arange(6 * pr["pose"], 6 * pr["pose"] + 6)
        rows.append(np.repeat(sl, 6))
        cols.append(np.tile(sl, 6))
        vals.append(M.ravel())
        g[sl] += b
        r += cq
    if priors:
        H = H + sp.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))),
                              shape=(6 * P, 6 * P)).tocsc()
    return (H.tocsc() if sparse else H.toarray()), g, r


def cost(poses, factors, priors, fk=None, fs=None, pk=None, ps=None):
    fk = np.zeros(len(factors), dtype=np.int32) if fk is None else fk
    fs = np.ones(len(factors)) if fs is None else fs
    pk = np.zeros(len(priors), dtype=np.int32) if pk is None else pk
    ps = np.ones(len(priors)) if ps is None else ps
    r = rfr.cost(poses, factors, fk, fs) if factors else 0.0
    return r + float(sum(prior_terms(poses, pr, k, c)[4] for pr, k, c in zip(priors, pk, ps)))


def residuals(poses, priors, pk=None, ps=None):
    """-> (s, w) per prior"""
    pk = np.zeros(len(priors), dtype=np.int32) if pk is None else pk
    ps = np.ones(len(priors)) if ps is None else ps
    out = np.array([prior_terms(poses, pr, k, c)[2:4] for pr, k, c in zip(priors, pk, ps)])
    return out[:, 0], out[:, 1]


def lm(poses0, factors, priors, P, max_iter=10, u0=0.01, v0=2.0, rel_tol=1e-6, sparse=False, **loss):
    """pose_graph_ref.lm's rule on the factors plus the priors -> (poses, trace, poses per iteration)"""
    x = np.array(poses0, dtype=np.float64, copy=True)
    u, v = u0, v0
    calc, trace, per = True, [], []
    H = g = None
    r1 = 0.0
    for it in range(max_iter):
        if calc:
            H, g, r1 = evaluate(x, factors, priors, P, sparse=sparse, **loss)
        D = H.diagonal().copy()
        if sparse:
            dx = spla.spsolve((H + u * sp.diags(D)).tocsc(), -g)
        else:
            dx = np.linalg.solve(H + u * np.diag(D), -g)
        q1 = 0.5 * dx @ (u * D * dx - g)
        xt = pgr.pose_update(x, dx)
        r2 = cost(xt, factors, priors, **loss)
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


# ---------------- scenes ----------------
def random_psd(rng, rank=6, scale=1.0):
    A = rng.standard_normal((6, rank))
    H = scale * (A @ A.T)
    return 0.5 * (H + H.T)


def random_priors(rng, poses, idx, kinds=("full", "position", "lever")):
    """one prior per pose idx[q], cycling through full-pose anchors, position-only priors and lever-arm position priors,
    each measured near the current pose"""
    out = []
    for q, i in enumerate(idx):
        kind = kinds[q % len(kinds)]
        hat = pgr.compose(poses[i], pgr.random_pose(rng, 0.05, 0.3))
        if kind == "full":
            out.append(dict(pose=int(i), pose_hat=hat, H=random_psd(rng, 6)))
        else:
            H = np.zeros((6, 6))
            H[3:, 3:] = random_psd(rng, 3)[:3, :3] + np.eye(3)
            d = dict(pose=int(i), pose_hat=hat, H=H)
            if kind == "lever":
                d["lever_arm"] = rng.uniform(-1.5, 1.5, 3)
            out.append(d)
    return out

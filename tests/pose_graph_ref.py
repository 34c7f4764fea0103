"""numpy restatement of the pose graph of balm_b200/csrc/pose_graph.cu (DESIGN.md, "Pose graph"):

  A window factor f holds N distinct global pose indices idx, the window's refined poses T^_k and its BA Hessian H_f
  ((6N)^2, column-major). With c(T, T^) = (Log(R R^^T), p - R R^^T p^) and A = T_idx[0] T^_0^-1:

      e_k = c(A^-1 T_idx[k], T^_k)   (e_0 = 0),   cost_f = 1/2 sum_{k,l >= 1} e_k^T H_f[k,l] e_l

  in the local coordinates of the pose update (R <- Exp(phi) R, p <- Exp(phi) p + dt). de_k/d(delta_k) = J_k,
  de_k/d(delta_0) = -J_k; M = E^T H~ E and b = E^T H~ e with E that stacked Jacobian, scattered into the dense 6P system.

  lm() is balm_damping_iter's Levenberg-Marquardt rule on this cost (no gauge step)."""
import numpy as np


def split(p12):
    p12 = np.asarray(p12, dtype=np.float64)
    return p12[:9].reshape(3, 3).T, p12[9:]  # R[a, c] = p12[3 c + a]


def pack(R, t):
    return np.concatenate([np.asarray(R).T.reshape(9), t])


def hat(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def exp_so3(phi):
    """exp_so3 of internal.cuh: identity below |phi| = 1e-11."""
    nrm = np.linalg.norm(phi)
    if nrm < 1e-11:
        return np.eye(3)
    K = hat(np.asarray(phi) / nrm)
    return np.eye(3) + np.sin(nrm) * K + (1.0 - np.cos(nrm)) * K @ K


def log_so3(R):
    """Log of a rotation: theta = atan2(|v|, (tr - 1)/2) with v = vee(R - R^T)/2; below 90 degrees phi = theta/|v| v, else
    the axis from the symmetric part (R + R^T)/2 - cos(theta) I = (1 - cos(theta)) a a^T, signed by v."""
    v = 0.5 * np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    c = 0.5 * (R[0, 0] + R[1, 1] + R[2, 2] - 1.0)
    s = np.sqrt(v @ v)
    th = np.arctan2(s, c)
    if c > 0.0:
        return np.zeros(3) if s == 0.0 else (th / s) * v
    B = 0.5 * (R + R.T) - c * np.eye(3)
    i = int(np.argmax(np.diag(B)))
    a = B[:, i] / np.sqrt(B[i, i] * (1.0 - c))
    if a @ v < 0.0:
        a = -a
    return th * a


def jl_inv(phi):
    """Inverse left Jacobian of SO(3): Log(Exp(x) Exp(phi)) = phi + jl_inv(phi) x + O(x^2)."""
    th = np.linalg.norm(phi)
    if th < 0.1:
        t2 = th * th
        c2 = 1.0 / 12 + t2 * (1.0 / 720 + t2 * (1.0 / 30240 + t2 / 1209600))
    else:
        h = 0.5 * th
        c2 = (1.0 - h * np.cos(h) / np.sin(h)) / (th * th)
    K = hat(phi)
    return np.eye(3) - 0.5 * K + c2 * K @ K


def residual(T0, Tk, hat0, hatk):
    """e_k and J_k = de_k/d(delta_k) of one slot k >= 1 (12-vectors)."""
    R0, p0 = split(T0)
    Rk, pk = split(Tk)
    Rh0, ph0 = split(hat0)
    Rhk, phk = split(hatk)
    Q = Rh0 @ R0.T
    Rs, ps = Q @ Rk, Q @ (pk - p0) + ph0            # A^-1 T_k
    D = Rs @ Rhk.T
    phi = log_so3(D)
    e = np.concatenate([phi, ps - D @ phk])
    w = pk - Rk @ Rhk.T @ phk
    J = np.zeros((6, 6))
    J[:3, :3] = jl_inv(phi) @ Q
    J[3:, :3] = -Q @ hat(w)
    J[3:, 3:] = Q
    return e, J


def factor_terms(poses, f):
    """-> (e [N,6], E [6(N-1), 6N], cost, M [6N, 6N], b [6N]) of factor f at the global poses."""
    idx, Th, Hf = f["poses"], f["poses_hat"], f["H"]
    N = len(idx)
    e = np.zeros((N, 6))
    E = np.zeros((6 * (N - 1), 6 * N))
    for k in range(1, N):
        e[k], J = residual(poses[idx[0]], poses[idx[k]], Th[0], Th[k])
        E[6 * (k - 1):6 * k, 6 * k:6 * k + 6] = J
        E[6 * (k - 1):6 * k, :6] = -J
    Ht = Hf[6:, 6:]
    ef = e[1:].ravel()
    cost = 0.5 * ef @ Ht @ ef
    return e, E, cost, E.T @ Ht @ E, E.T @ Ht @ ef


def cost(poses, factors):
    return float(sum(factor_terms(poses, f)[2] for f in factors))


def evaluate(poses, factors, P):
    """Dense H (6P x 6P), g, cost of the factors (all taken as registered with status OK)."""
    H = np.zeros((6 * P, 6 * P))
    g = np.zeros(6 * P)
    r = 0.0
    for f in factors:
        _, _, c, M, b = factor_terms(poses, f)
        sl = np.concatenate([np.arange(6 * i, 6 * i + 6) for i in f["poses"]])
        H[np.ix_(sl, sl)] += M
        g[sl] += b
        r += c
    return H, g, r


def pose_update(poses, dx):
    out = np.array(poses, dtype=np.float64, copy=True)
    for i in range(len(out)):
        R, p = split(out[i])
        dR = exp_so3(dx[6 * i:6 * i + 3])
        out[i] = pack(dR @ R, dR @ p + dx[6 * i + 3:6 * i + 6])
    return out


def gauge_vectors(P):
    """The six directions of a common left transform: the same delta on every pose."""
    return np.tile(np.eye(6), (P, 1))


def pd_ok(Hf):
    """Registration check: H_f restricted to slots >= 1 positive definite, smallest pivot above 1e-11 times the largest."""
    A = np.asarray(Hf)[6:, 6:]
    try:
        L = np.linalg.cholesky(0.5 * (A + A.T))
    except np.linalg.LinAlgError:
        return False
    d = np.diag(L) ** 2
    return bool(d.min() > 1e-11 * d.max())


def lm(poses0, factors, P, max_iter=10, u0=0.01, v0=2.0, rel_tol=1e-6):
    """balm_damping_iter's LM rule on the pose-graph cost -> (poses, trace, poses per iteration)."""
    x = np.array(poses0, dtype=np.float64, copy=True)
    u, v = u0, v0
    calc, trace, per = True, [], []
    H = g = None
    r1 = 0.0
    for it in range(max_iter):
        if calc:
            H, g, r1 = evaluate(x, factors, P)
        D = np.diag(H).copy()
        dx = np.linalg.solve(H + u * np.diag(D), -g)
        q1 = 0.5 * dx @ (u * D * dx - g)
        xt = pose_update(x, dx)
        r2 = cost(xt, factors)
        q = r1 - r2
        t = dict(r1=r1, r2=r2, u=u, v=v, q=q, q1=q1, accepted=False, recomputed_hess=calc)
        if q > 0:
            x = xt
            rho = q / q1
            v = 2.0
            fct = 1 - (2 * rho - 1) ** 3
            u *= max(fct, 1.0 / 3.0)
            calc = True
            t["accepted"] = True
        else:
            u = u * v
            v = 2 * v
            calc = False
        trace.append(t)
        per.append(x.copy())
        if rel_tol >= 0 and abs(r1 - r2) / r1 < rel_tol:
            break
    return x, trace, per


# ---------------- synthetic factor sets ----------------
def random_pose(rng, rot=1.0, tran=5.0):
    return pack(exp_so3(rng.normal(0, rot, 3)), rng.normal(0, tran, 3))


def compose(a, b):
    Ra, pa = split(a)
    Rb, pb = split(b)
    return pack(Ra @ Rb, Ra @ pb + pa)


def random_spd(rng, n, cond=1e3):
    Q, _ = np.linalg.qr(rng.normal(size=(n, n)))
    return (Q * np.geomspace(1.0, cond, n)) @ Q.T


def window_hessian(rng, N, cond=1e3):
    """A BA-like window Hessian: symmetric, 6-dimensional gauge null space of the common left transform, and positive
    definite on slots >= 1."""
    S = random_spd(rng, 6 * (N - 1), cond)
    E = np.zeros((6 * (N - 1), 6 * N))
    for k in range(1, N):
        E[6 * (k - 1):6 * k, :6] = -np.eye(6)
        E[6 * (k - 1):6 * k, 6 * k:6 * k + 6] = np.eye(6)
    H = E.T @ S @ E
    return 0.5 * (H + H.T)


def make_factor(rng, truth, idx, noise=0.0, cond=1e3):
    """Factor over the poses idx of the trajectory `truth`, with its T^ in an arbitrary frame of its own and (noise > 0)
    each T^_k perturbed by N(0, noise) on the left."""
    G = random_pose(rng)
    hatp = np.array([compose(G, truth[i]) for i in idx])
    if noise > 0:
        for k in range(1, len(idx)):
            d = rng.normal(0, noise, 6)
            R, p = split(hatp[k])
            dR = exp_so3(d[:3])
            hatp[k] = pack(dR @ R, dR @ p + d[3:])
    return dict(poses=np.asarray(idx, dtype=np.int32), poses_hat=hatp, H=window_hessian(rng, len(idx), cond))


def perturb(rng, poses, rot, tran):
    out = np.array(poses, copy=True)
    for i in range(len(out)):
        R, p = split(out[i])
        out[i] = pack(exp_so3(rng.normal(0, rot, 3)) @ R, p + rng.normal(0, tran, 3))
    return out


def pyramid_factor_poses(P, length=10, stride=5, top=32):
    """Global pose index sets of HBA-shaped windows: windows of `length` every `stride` over P poses, the slot-0 poses of
    a layer's windows forming the next layer, up to one top window of at most `top` items."""
    items = list(range(P))
    out = []
    while True:
        if len(items) <= top:
            if len(items) >= 2:
                out.append(list(items))
            return out
        wins, s = [], 0
        while True:
            wins.append(items[s:min(s + length, len(items))])
            if s + length >= len(items):
                break
            s += stride
        out += [w for w in wins if len(w) >= 2]
        items = [w[0] for w in wins]

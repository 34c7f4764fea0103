"""scipy.sparse restatement of pose_graph_ref: the same H, g and cost with H a sparse matrix, and the damped LM step
solved by spsolve, so that the oracle reaches trajectories whose dense 6P x 6P system does not fit."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import pose_graph_ref as pg


def evaluate(poses, factors, P):
    """-> (H as a CSC matrix, g, cost) of the factors (all taken as registered with status OK)."""
    rows, cols, vals = [], [], []
    g = np.zeros(6 * P)
    r = 0.0
    for f in factors:
        _, _, c, M, b = pg.factor_terms(poses, f)
        sl = np.concatenate([np.arange(6 * i, 6 * i + 6) for i in f["poses"]])
        rows.append(np.repeat(sl, len(sl)))
        cols.append(np.tile(sl, len(sl)))
        vals.append(M.ravel())
        g[sl] += b
        r += c
    H = sp.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(6 * P, 6 * P))
    return H.tocsc(), g, r


def block_pairs(factors):
    """The (i, j), i <= j, of every nonzero 6x6 block of H, ascending."""
    s = {(min(a, b), max(a, b)) for f in factors for a in f["poses"] for b in f["poses"]}
    return np.array(sorted(s), dtype=np.int64).reshape(-1, 2)


def blocks(H, pairs):
    """-> [n_pairs, 6, 6]: H's rows of pose i and columns of pose j for every pair (i, j)."""
    H = H.tocsr()
    return np.array([H[6 * i:6 * i + 6, 6 * j:6 * j + 6].toarray() for i, j in pairs]).reshape(-1, 6, 6)


def damped_solve(H, g, u):
    """dx = (H + u diag(H))^-1 (-g) and q1 = 1/2 dx.(u D dx - g), as pose_graph_ref.lm computes them."""
    D = H.diagonal()
    dx = spla.spsolve((H + u * sp.diags(D)).tocsc(), -g)
    return dx, 0.5 * dx @ (u * D * dx - g)


def lm_step(poses, factors, P, u=0.01):
    """The first iteration of pose_graph_ref.lm -> (trial poses, r1, r2)."""
    H, g, r1 = evaluate(poses, factors, P)
    dx, _ = damped_solve(H, g, u)
    xt = pg.pose_update(poses, dx)
    return xt, r1, pg.cost(xt, factors)

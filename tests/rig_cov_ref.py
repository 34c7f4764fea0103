"""numpy restatement of the rig covariance (DESIGN.md "Rig covariance", include/balm_b200.h balm_rig_covariance):

  X_s = T_{base_of[s]} E_{lidar_of[s]},   R = numpy_cov.left_jacobian_point at the X_s (coe w with a voxel loss)
  raw = J^T R J,   cov = H~^-1 raw~ H~^-T

with J rig_ref.jacobian, H rig_ref.evaluate's H_rig at the same state, and ~ the anchor's 6 rows and columns deleted
(zeroed, 1 on H's diagonal, 0 on raw's and cov's).

planar_moments() and noisy_moments() serve the Monte-Carlo check: the clusters of a scene moved onto their voxel's
plane at the true poses, and a draw of the clusters those points give with isotropic point noise added."""
import numpy as np

import numpy_cov as nc
import rig_ref as rr
import robust_voxels_ref as rv


def delete(A, anchor, diag):
    """A with the rows and columns of free unknown `anchor` zeroed and diag on its diagonal (anchor -1: A)"""
    A = np.array(A, dtype=np.float64, copy=True)
    if anchor >= 0:
        a = 6 * anchor
        A[a:a + 6, :] = 0.0
        A[:, a:a + 6] = 0.0
        A[a:a + 6, a:a + 6] = diag * np.eye(6)
    return A


def rig_covariance(sc, base12, ext12, base_of, lidar_of, var, pnoise=None, c_cov=None, include_fix=False, anchor=-1,
                   kind=rv.TRIVIAL, c=1.0):
    """-> (raw, cov), n_rig x n_rig in var's order"""
    X = rr.compose(base12, ext12, base_of, lidar_of)
    _, w = rv.weights(sc, X, kind, c, include_fix)
    R = nc.left_jacobian_point(sc["n_poses"], sc["row_ptr"], sc["pose_idx"], sc["obs10"],
                               np.asarray(sc["coe"], dtype=np.float64) * w, X,
                               sc.get("fix10") if include_fix else None, c_cov=c_cov, pnoise=pnoise)
    J = rr.jacobian(base12, base_of, lidar_of, len(base12), var)
    raw = delete(J.T @ R @ J, anchor, 0.0)
    H = delete(rr.evaluate(sc, base12, ext12, base_of, lidar_of, var, include_fix, kind, c)[0], anchor, 1.0)
    Hi = np.linalg.inv(H)
    return raw, delete(Hi @ raw @ Hi.T, anchor, 0.0)


# ---------------- Monte-Carlo helpers ----------------
def _sym(o):
    return np.array([[o[0], o[1], o[2]], [o[1], o[3], o[4]], [o[2], o[4], o[5]]])


def _pack(P, v, n):
    return np.array([P[0, 0], P[0, 1], P[0, 2], P[1, 1], P[1, 2], P[2, 2], v[0], v[1], v[2], n])


def planar_moments(sc, poses):
    """every observation's points moved along their voxel's normal onto the voxel's plane (the least-squares plane of
    all its points at `poses`), as moments in the scan frame -> obs10. At `poses` every voxel is then exactly planar."""
    out = np.array(sc["obs10"], dtype=np.float64, copy=True)
    for a in range(len(sc["row_ptr"]) - 1):
        rng_ = range(sc["row_ptr"][a], sc["row_ptr"][a + 1])
        world = []
        for s in rng_:
            o = sc["obs10"][s]
            R, p = poses[sc["pose_idx"][s]][:9].reshape(3, 3).T, poses[sc["pose_idx"][s]][9:]
            P, v, n = _sym(o), o[6:9], o[9]
            Rv = R @ v
            world.append((R @ P @ R.T + np.outer(Rv, p) + np.outer(p, Rv) + n * np.outer(p, p), Rv + n * p, n, R, p))
        NN = sum(w[2] for w in world)
        cbar = sum(w[1] for w in world) / NN
        u = np.linalg.eigh(sum(w[0] for w in world) / NN - np.outer(cbar, cbar))[1][:, 0]
        Pi, d = np.eye(3) - np.outer(u, u), u * (u @ cbar)  # x -> Pi x + d
        for s, (Pw, vw, n, R, p) in zip(rng_, world):
            P2 = Pi @ Pw @ Pi + np.outer(Pi @ vw, d) + np.outer(d, Pi @ vw) + n * np.outer(d, d)
            v2 = Pi @ vw + n * d
            # back to the scan frame: x_b = R^T (x_w - p)
            Pb = R.T @ (P2 - np.outer(v2, p) - np.outer(p, v2) + n * np.outer(p, p)) @ R
            out[s] = _pack(0.5 * (Pb + Pb.T), R.T @ (v2 - n * p), n)
    return out


def noise_model(obs10):
    """The clusters of n points x_i + e_i, e_i ~ N(0, sigma^2 I), follow from the moments of the x_i alone. With X~ the
    4 x n matrix [x_i; 1] and E the 3 x n noise, the added terms are X~ E^T and E E^T, whose joint law depends on X~
    only through X~ X~^T = [[P, v], [v^T, n]]: any Y with Y Y^T = that matrix (here V diag(sqrt(lambda)), columns in
    descending lambda, so a cluster of n < 4 points has its nonzero columns first) stands in for X~ exactly.
    -> (Y [K, 4, 4], n [K]) of every observation"""
    obs10 = np.asarray(obs10, dtype=np.float64)
    M = np.zeros((len(obs10), 4, 4))
    for s, o in enumerate(obs10):
        M[s, :3, :3], M[s, :3, 3], M[s, 3, :3], M[s, 3, 3] = _sym(o), o[6:9], o[6:9], o[9]
    lam, V = np.linalg.eigh(M)
    Y = (V * np.sqrt(np.maximum(lam, 0.0))[:, None, :])[:, :, ::-1]
    return Y, np.rint(obs10[:, 9]).astype(np.int64)


def noisy_moments(obs10, model, sigma, rng):
    """one draw of the clusters with point noise sigma (model: noise_model(obs10)) -> obs10"""
    Y, n = model
    starts = np.concatenate([[0], np.cumsum(n)[:-1]])
    E = rng.normal(0.0, sigma, (int(n.sum()), 3))
    W = np.add.reduceat(E[:, :, None] * E[:, None, :], starts, axis=0)         # sum e e^T
    idx = starts[:, None] + np.minimum(np.arange(4)[None, :], n[:, None] - 1)  # the first min(n, 4) points
    Z = Y @ E[idx]                                                            # rows: X E^T (3 x 3), then (sum e)^T
    out = np.array(obs10, dtype=np.float64, copy=True)
    XE = Z[:, :3, :]
    P = W + XE + XE.transpose(0, 2, 1)
    out[:, [0, 1, 2, 3, 4, 5]] += P[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
    out[:, 6:9] += Z[:, 3, :]
    return out

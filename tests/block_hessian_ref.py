"""Vectorised numpy / scipy.sparse restatement of numpy_ref.evaluate for the block-sparse Hessian of a PREC_BLOCKS
context, and a corridor scene with local co-visibility.

  H = sum_v coe_v G_v diag(w_v) G_v^T + blockdiag(D_i)

is formed as one sparse product over every observation's three G' columns, and read out as the 6x6 blocks of the pose
pairs (i <= j) that share a voxel plus every diagonal pair, (pairs, 6, 6) with [p, a, c] = H[6 i + a, 6 j + c]."""
import numpy as np
import scipy.sparse as sp

import scenes


def _hat(v):  # (..., 3) -> (..., 3, 3)
    z = np.zeros(v.shape[:-1])
    return np.stack([np.stack([z, -v[..., 2], v[..., 1]], -1), np.stack([v[..., 2], z, -v[..., 0]], -1),
                     np.stack([-v[..., 1], v[..., 0], z], -1)], -2)


def _sym(o):  # (..., 10) -> (..., 3, 3)
    return np.stack([o[..., [0, 1, 2]], o[..., [1, 3, 4]], o[..., [2, 4, 5]]], -2)


def pairs_from_csr(N, row_ptr, pose_idx):
    """The co-visible pose pairs (i <= j) plus every (i, i), ascending: (pairs, 2) int32."""
    M = len(row_ptr) - 1
    vox = np.repeat(np.arange(M), np.diff(row_ptr))
    B = sp.csr_matrix((np.ones(len(pose_idx)), (vox, pose_idx)), shape=(M, N))
    C = sp.triu((B.T @ B) + sp.identity(N), format="coo")
    order = np.lexsort((C.col, C.row))
    return np.stack([C.row[order], C.col[order]], 1).astype(np.int32)


def evaluate(sc, poses12, include_fix=False):
    """-> (pairs (P, 2), blocks (P, 6, 6), g, r) of numpy_ref.evaluate(sc, poses12, include_fix)."""
    N = sc["n_poses"]
    row_ptr, pose_idx, obs, coe = sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"]
    M, K = len(row_ptr) - 1, len(pose_idx)
    vox = np.repeat(np.arange(M), np.diff(row_ptr))
    pz = poses12[pose_idx]
    R = pz[:, :9].reshape(K, 3, 3).transpose(0, 2, 1)
    p = pz[:, 9:12]
    P, v, n = _sym(obs), obs[:, 6:9], obs[:, 9]
    Rv = np.einsum("kab,kb->ka", R, v)
    Pw = R @ P @ R.transpose(0, 2, 1) + Rv[:, :, None] * p[:, None, :] + p[:, :, None] * Rv[:, None, :] + \
        n[:, None, None] * p[:, :, None] * p[:, None, :]
    vw = Rv + n[:, None] * p
    Ps = np.add.reduceat(Pw, row_ptr[:-1], 0)
    vs = np.add.reduceat(vw, row_ptr[:-1], 0)
    NN = np.add.reduceat(n, row_ptr[:-1])
    if include_fix and sc.get("fix10") is not None:
        f = sc["fix10"]
        Ps, vs, NN = Ps + _sym(f), vs + f[:, 6:9], NN + f[:, 9]
    vb = vs / NN[:, None]
    lam, U = np.linalg.eigh(Ps / NN[:, None, None] - vb[:, :, None] * vb[:, None, :])
    r = float(np.sum(coe * lam[:, 0]))
    w = np.stack([-2.0 / NN ** 2, 2.0 / (lam[:, 0] - lam[:, 1]), 2.0 / (lam[:, 0] - lam[:, 2])], 1)
    u = U[vox]  # (K, 3, 3): columns u0, u1, u2
    u0 = u[:, :, 0]
    Mt = Pw - vw[:, :, None] * vb[vox][:, None, :]
    mb = vw - n[:, None] * vb[vox]
    NNk = NN[vox][:, None]
    Mu0 = np.einsum("kab,kb->ka", Mt, u0)

    def gk(uk):
        top = -np.cross(uk, Mu0) - np.cross(u0, np.einsum("kab,kb->ka", Mt, uk))
        bot = uk * np.sum(mb * u0, 1)[:, None] + u0 * np.sum(mb * uk, 1)[:, None]
        return np.concatenate([top, bot], 1) / NNk

    G = np.stack([np.concatenate([-np.cross(u0, vw), n[:, None] * u0], 1), gk(u[:, :, 1]), gk(u[:, :, 2])], 2)
    g = np.zeros(6 * N)
    np.add.at(g, (6 * pose_idx[:, None] + np.arange(6)).ravel(), (coe[vox][:, None] * gk(u0)).ravel())
    # D_i = coe (2/NN V0 TCT V0^T + [[E + E^T, 0], [0, 0]]), E = hat(M u0) hat(u0) / NN
    V0 = np.zeros((K, 6, 4))
    V0[:, :3, :3] = _hat(-u0)
    V0[:, 3:, 3] = u0
    TCT = np.zeros((K, 4, 4))
    TCT[:, :3, :3] = Pw
    TCT[:, :3, 3] = vw
    TCT[:, 3, :3] = vw
    TCT[:, 3, 3] = n
    D = 2.0 / NNk[:, :, None] * V0 @ TCT @ V0.transpose(0, 2, 1)
    E = _hat(Mu0) @ _hat(u0) / NNk[:, :, None]
    D[:, :3, :3] += E + E.transpose(0, 2, 1)
    D *= coe[vox][:, None, None]
    # H = Gs diag(coe w) Gs^T (Gs: 6N x 3M, column 3 v + k holds G[s, :, k] of every observation s of voxel v at the
    # rows of its pose) + blockdiag(sum D)
    rows = (6 * pose_idx[:, None, None] + np.arange(6)[None, :, None]).repeat(3, 2)
    cols = (3 * vox[:, None, None] + np.arange(3)[None, None, :]).repeat(6, 1)
    Gs = sp.csr_matrix((G.ravel(), (rows.ravel(), cols.ravel())), shape=(6 * N, 3 * M))
    H = (Gs @ sp.diags((coe[:, None] * w).ravel()) @ Gs.T).tocsr()
    Dsum = np.zeros((N, 6, 6))
    np.add.at(Dsum, pose_idx, D)
    H = H + sp.block_diag([sp.csr_matrix(d) for d in Dsum], format="csr")
    pairs = pairs_from_csr(N, row_ptr, pose_idx)
    return pairs, blocks_of(H, pairs), g, r


def blocks_of(H, pairs):
    """(P, 6, 6) blocks of a dense or sparse H at the pairs."""
    H = sp.csr_matrix(H)
    ri = (6 * pairs[:, 0, None, None] + np.arange(6)[None, :, None]).repeat(6, 2)
    ci = (6 * pairs[:, 1, None, None] + np.arange(6)[None, None, :]).repeat(6, 1)
    return np.asarray(H[ri.ravel(), ci.ravel()]).reshape(len(pairs), 6, 6)


def to_sparse(N, pairs, blocks):
    """The symmetric 6N x 6N scipy.sparse matrix of the blocks."""
    ri = (6 * pairs[:, 0, None, None] + np.arange(6)[None, :, None]).repeat(6, 2).ravel()
    ci = (6 * pairs[:, 1, None, None] + np.arange(6)[None, None, :]).repeat(6, 1).ravel()
    b = blocks.ravel()
    off = np.repeat(pairs[:, 0] != pairs[:, 1], 36)
    return sp.csr_matrix((np.concatenate([b, b[off]]), (np.concatenate([ri, ci[off]]), np.concatenate([ci, ri[off]]))),
                         shape=(6 * N, 6 * N))


def corridor(N, w=8, planes_per_pose=30, pts=8, point_noise=0.01, seed=0, with_fix=False):
    """N poses along a path (<= 1 km long), planes placed along it; the plane of center index c is seen by the poses
    c - w .. c + w, so every pose sees at least planes_per_pose planes. Same dict as scenes.make_scene."""
    rng = np.random.default_rng(seed)
    step = min(1.0, 1000.0 / N)
    yaw = np.cumsum(rng.normal(0, 0.01, N))
    ps = np.stack([np.cumsum(step * np.cos(yaw)), np.cumsum(step * np.sin(yaw)), 0.1 * np.sin(np.arange(N) * 0.01)], 1)
    Rs = np.stack([scenes.exp_so3(np.array([0.0, 0.0, y]) + rng.normal(0, 0.02, 3)) for y in yaw])
    per_center = -(-planes_per_pose // (w + 1))
    centers = np.repeat(np.arange(N), per_center)
    M = len(centers)
    lo, hi = np.maximum(centers - w, 0), np.minimum(centers + w, N - 1)
    k = hi - lo + 1
    row_ptr = np.concatenate([[0], np.cumsum(k)]).astype(np.int64)
    pose_idx = (np.repeat(lo, k) + np.arange(row_ptr[-1]) - np.repeat(row_ptr[:-1], k)).astype(np.int32)
    normal = rng.normal(0, 1, (M, 3))
    normal /= np.linalg.norm(normal, axis=1)[:, None]
    basis = np.linalg.qr(np.concatenate([normal[:, :, None], rng.normal(0, 1, (M, 3, 2))], 2))[0]
    center = ps[centers] + rng.uniform(-3, 3, (M, 3))
    K = len(pose_idx)
    vox = np.repeat(np.arange(M), k)
    loc = np.stack([rng.normal(0, point_noise, (K, pts)), rng.uniform(-1, 1, (K, pts)), rng.uniform(-1, 1, (K, pts))], 2)
    world = np.einsum("kab,kpb->kpa", basis[vox], loc) + center[vox][:, None, :]
    body = np.einsum("kpa,kab->kpb", world - ps[pose_idx][:, None, :], Rs[pose_idx]).astype(np.float32).astype(np.float64)
    P = np.einsum("kpa,kpb->kab", body, body)
    v = body.sum(1)
    obs = np.concatenate([P[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]], v, np.full((K, 1), float(pts))], 1)
    fix = None
    if with_fix:
        fl = np.stack([rng.normal(0, point_noise, (M, pts)), rng.uniform(-1, 1, (M, pts)), rng.uniform(-1, 1, (M, pts))], 2)
        fw = np.einsum("mab,mpb->mpa", basis, fl) + center[:, None, :]
        FP = np.einsum("mpa,mpb->mab", fw, fw)
        fix = np.concatenate([FP[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]], fw.sum(1), np.full((M, 1), float(pts))], 1)
    poses_gt = scenes.pack_poses(list(Rs), list(ps))
    Rn = [Rs[i] @ scenes.exp_so3(rng.normal(0, 0.5 / 57.3, 3)) for i in range(N)]
    pn = ps + rng.normal(0, 0.05, (N, 3))
    return dict(n_poses=N, row_ptr=row_ptr, pose_idx=pose_idx, obs10=obs, coe=(k * pts).astype(np.float64), fix10=fix,
                poses_gt=poses_gt, poses_init=scenes.pack_poses(Rn, list(pn)))

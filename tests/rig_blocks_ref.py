"""numpy restatement of the block-sparse rig (include/balm_b200.h balm_block_set_rig, DESIGN.md "Rig calibration on
block-sparse voxel BA"), working from a blocks context's slot blocks (block_hessian_ref.evaluate):

  pattern: rig pair (u, v), u <= v over the free unknowns, when some slot of u and some slot of v form a slot pair,
           plus every diagonal pair (u, u)
  pass 1:  K_sv = sum_{t in v} H_st J_t for every slot s and free unknown v with a slot co-observing s
  pass 2:  H_rig(u, v) = sum_{s in u} J_s^T K_sv + the second-order correction of the slots of u (rig_ref.correction's
           blocks), g_rig(u) = sum_{s in u} J_s^T g_s

rig_corridor() is a rig drive along block_hessian_ref.corridor's path: B base poses, L LiDARs, every plane seen by the
slots of the bases within +-w of its centre."""
import numpy as np

import block_hessian_ref as bh
import numpy_ref as nr
import rig_ref as rr
from scenes import exp_so3, pack_poses, unpack_pose


def free_of(base_of, lidar_of, B, var):
    """the free unknowns (indices into var) of every slot, ascending"""
    col = {j: u for u, j in enumerate(var)}
    return [[col[x] for x in (int(base_of[s]), B + int(lidar_of[s])) if x in col] for s in range(len(base_of))]


def pattern(slot_pairs, base_of, lidar_of, B, var):
    """the rig pairs (n, 2) int32, (u, v) with u <= v, ascending"""
    fo = free_of(base_of, lidar_of, B, var)
    S = {(u, u) for u in range(len(var))}
    for i, j in slot_pairs:
        for x in fo[i]:
            for y in fo[j]:
                S.add((min(x, y), max(x, y)))
    return np.array(sorted(S), dtype=np.int32).reshape(-1, 2)


def _jblock(base12, base_of, B, var, s, u):
    """J_s's 6x6 block on free unknown u"""
    if var[u] < B:
        return np.eye(6)
    R, p = unpack_pose(np.asarray(base12[base_of[s]], dtype=np.float64))
    Ad = np.zeros((6, 6))
    Ad[:3, :3] = R
    Ad[3:, :3] = nr.hat(p) @ R
    Ad[3:, 3:] = R
    return Ad


def reduce(slot_pairs, slot_blocks, g, base12, base_of, lidar_of, var):
    """the two passes -> (pairs (n, 2), blocks (n, 6, 6) with [p, a, c] = H_rig[6 u + a, 6 v + c], g_rig)"""
    N, B = len(base_of), len(base12)
    fo = free_of(base_of, lidar_of, B, var)
    H = {}
    nbr = [[] for _ in range(N)]
    for (i, j), b in zip(map(tuple, slot_pairs), slot_blocks):
        H[(i, j)] = b
        nbr[i].append(j)
        if i != j:
            H[(j, i)] = b.T
            nbr[j].append(i)
    K = {}
    for s in range(N):
        for t in sorted(nbr[s]):
            for v in fo[t]:
                K[(s, v)] = K.get((s, v), 0.0) + H[(s, t)] @ _jblock(base12, base_of, B, var, t, v)
    slots = [[] for _ in var]
    for s in range(N):
        for u in fo[s]:
            slots[u].append(s)
    pairs = pattern(slot_pairs, base_of, lidar_of, B, var)
    out = np.zeros((len(pairs), 6, 6))
    for q, (u, v) in enumerate(pairs):
        for s in slots[u]:
            if (s, v) in K:
                out[q] += _jblock(base12, base_of, B, var, s, u).T @ K[(s, v)]
    # the correction: (lidar, same lidar) on phi x phi, (base, lidar) on the base's phi rows
    index = {(int(u), int(v)): q for q, (u, v) in enumerate(pairs)}
    col = {j: u for u, j in enumerate(var)}
    for s in range(N):
        e = col.get(B + int(lidar_of[s]))
        if e is None:
            continue
        R, p = unpack_pose(np.asarray(base12[base_of[s]], dtype=np.float64))
        gp, gt = g[6 * s:6 * s + 3], g[6 * s + 3:6 * s + 6]
        S = 0.5 * (np.outer(gt, p) + np.outer(p, gt)) - (gt @ p) * np.eye(3)
        out[index[(e, e)], :3, :3] += -R.T @ S @ R
        a = col.get(int(base_of[s]))
        if a is not None:
            q = index[(a, e)]
            out[q, :3, :3] += -0.5 * nr.hat(gp) @ R - nr.hat(gt) @ nr.hat(p) @ R
            out[q, :3, 3:] += -nr.hat(gt) @ R
    gr = np.zeros(6 * len(var))
    for u in range(len(var)):
        for s in slots[u]:
            gr[6 * u:6 * u + 6] += _jblock(base12, base_of, B, var, s, u).T @ g[6 * s:6 * s + 6]
    return pairs, out, gr


def rig_corridor(B, L, w=4, planes_per_base=12, pts=8, point_noise=0.01, seed=0):
    """B base poses along block_hessian_ref.corridor's path, L LiDARs (LiDAR 0 at the identity), slot s = b L + l;
    the plane of centre base c is seen by every slot of the bases c - w .. c + w. -> a scenes.make_scene-style dict over
    the B L slots with base_of, lidar_of, base12 / ext12 (truth) and base_init / ext_init (bases 0.5 deg / 5 cm off,
    LiDARs 1.. 1 deg / 5 cm off)"""
    rng = np.random.default_rng(seed)
    N = B * L
    step = min(1.0, 1000.0 / B)
    yaw = np.cumsum(rng.normal(0, 0.05, B))
    ps = np.stack([np.cumsum(step * np.cos(yaw)), np.cumsum(step * np.sin(yaw)), 0.1 * np.sin(np.arange(B) * 0.01)], 1)
    Rs = [exp_so3(np.array([0.0, 0.0, y]) + rng.normal(0, 0.05, 3)) for y in yaw]
    base12 = pack_poses(Rs, list(ps))
    Re = [np.eye(3)] + [exp_so3(np.array([0.05, -0.03, 2 * np.pi * l / L])) for l in range(1, L)]
    pe = [np.zeros(3)] + [np.array([0.3 * np.cos(l), 0.3 * np.sin(l), 0.1]) for l in range(1, L)]
    ext12 = pack_poses(Re, pe)
    base_of = np.repeat(np.arange(B), L).astype(np.int32)
    lidar_of = np.tile(np.arange(L), B).astype(np.int32)
    X = rr.compose(base12, ext12, base_of, lidar_of)
    per_centre = -(-planes_per_base // (w + 1))
    centres = np.repeat(np.arange(B), per_centre)
    M = len(centres)
    lo, hi = np.maximum(centres - w, 0), np.minimum(centres + w, B - 1)
    k = (hi - lo + 1) * L
    row_ptr = np.concatenate([[0], np.cumsum(k)]).astype(np.int64)
    pose_idx = (np.repeat(lo * L, k) + np.arange(row_ptr[-1]) - np.repeat(row_ptr[:-1], k)).astype(np.int32)
    normal = rng.normal(0, 1, (M, 3))
    normal /= np.linalg.norm(normal, axis=1)[:, None]
    basis = np.linalg.qr(np.concatenate([normal[:, :, None], rng.normal(0, 1, (M, 3, 2))], 2))[0]
    centre = ps[centres] + rng.uniform(-3, 3, (M, 3))
    K = len(pose_idx)
    vox = np.repeat(np.arange(M), k)
    loc = np.stack([rng.normal(0, point_noise, (K, pts)), rng.uniform(-1, 1, (K, pts)), rng.uniform(-1, 1, (K, pts))], 2)
    world = np.einsum("kab,kpb->kpa", basis[vox], loc) + centre[vox][:, None, :]
    RX = np.stack([unpack_pose(x)[0] for x in X])
    pX = np.stack([unpack_pose(x)[1] for x in X])
    body = np.einsum("kpa,kab->kpb", world - pX[pose_idx][:, None, :], RX[pose_idx]).astype(np.float32).astype(np.float64)
    P = np.einsum("kpa,kpb->kab", body, body)
    obs = np.concatenate([P[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]], body.sum(1), np.full((K, 1), float(pts))], 1)
    base_init = np.stack([rr.perturb(b, rng, 0.5 / 57.3, 0.05) for b in base12])
    ext_init = ext12.copy()
    for l in range(1, L):
        ext_init[l] = rr.perturb(ext12[l], rng, 1.0 / 57.3, 0.05)
    return dict(n_poses=N, row_ptr=row_ptr, pose_idx=pose_idx, obs10=obs, coe=(k * pts).astype(np.float64), fix10=None,
                base_of=base_of, lidar_of=lidar_of, base12=base12, ext12=ext12, base_init=base_init, ext_init=ext_init)

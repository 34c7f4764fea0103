"""Pose factors built from relative-pose measurements, in the format of Context.set_block_factors /
Context.set_pose_factors / PoseGraph.set_pose_factors (include/balm_b200.h, balm_set_pose_factors), and absolute pose
priors in the format of Context.set_pose_priors / PoseGraph.set_pose_priors (balm_set_pose_priors)."""
import numpy as np


def _hat(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def odometry_factors(poses12, info, edges=None):
    """Two-pose factors, one per edge (a, b) (default: consecutive scans, (i, i + 1)), with poses = [a, b] and
    poses_hat = poses12[[a, b]]: the factor holds the relative pose T^_a^-1 T^_b of poses12.

    info: 6 x 6 information matrix of the relative pose, one per edge (n_edges x 6 x 6) or one shared by all. It is that
    of a right (body-frame) perturbation of scan b, T_b = T_a T^_a^-1 T^_b (Exp psi, rho), in the library's (rotation,
    translation) order, so that to second order cost_f = 1/2 xi^T info xi with xi = (psi, rho). The factor's own
    coordinates are e = c(A^-1 T_b, T^_b) (balm_set_pose_factors); to first order e = Ad xi with
    Ad = [[R^_b, 0], [hat(p^_b) R^_b, R^_b]], so the factor's H is E^T Ad^-T info Ad^-1 E, E = [-I, I], which has the
    gauge null space of a common left transform.

    info must be in the voxel cost's units when the factors join a voxel cost (Context.set_block_factors): coe x lambda,
    i.e. points x m^2, which the Hessians of BA windows already are. How much odometry weighs against the voxels is the
    caller's choice. -> list of factor dicts."""
    poses12 = np.asarray(poses12, dtype=np.float64).reshape(-1, 12)
    if edges is None:
        edges = [(i, i + 1) for i in range(len(poses12) - 1)]
    edges = [(int(a), int(b)) for a, b in edges]
    info = np.asarray(info, dtype=np.float64)
    if info.shape == (6, 6):
        info = np.broadcast_to(info, (len(edges), 6, 6))
    if info.shape != (len(edges), 6, 6):
        raise ValueError(f"odometry_factors: info must be 6 x 6 or {len(edges)} x 6 x 6, got {info.shape}")
    E = np.hstack([-np.eye(6), np.eye(6)])
    out = []
    for (a, b), om in zip(edges, info):
        Rb, pb = poses12[b, :9].reshape(3, 3).T, poses12[b, 9:]
        Ai = np.zeros((6, 6))  # Ad^-1
        Ai[:3, :3] = Ai[3:, 3:] = Rb.T
        Ai[3:, :3] = -Rb.T @ _hat(pb)
        om_e = Ai.T @ om @ Ai
        H = E.T @ om_e @ E
        out.append(dict(poses=np.array([a, b], dtype=np.int32), poses_hat=poses12[[a, b]].copy(), H=0.5 * (H + H.T)))
    return out


def _per_item(x, n, shape, what):
    x = np.asarray(x, dtype=np.float64)
    if x.shape == shape:
        x = np.broadcast_to(x, (n,) + shape)
    if x.shape != (n,) + shape:
        raise ValueError(f"{what} must be {shape} or ({n},) + {shape}, got {x.shape}")
    return x


def pose_priors(idx, poses12, info6):
    """Full-pose anchors: one prior per pose idx[q] at the measured pose poses12[q] (len(idx) x 12), with information
    info6 (6 x 6 in the (rotation, translation) order of the residual e = (Log(R R^^T), p - p^), one per prior or one
    shared by all). Units as odometry_factors': in a voxel cost (Context.set_pose_priors on PREC_BLOCKS) an information
    Omega joins as 2 sigma_p^2 Omega, sigma_p the point noise the voxel cost's coe x lambda stands for. -> list of prior
    dicts."""
    idx = np.asarray(idx, dtype=np.int64).ravel()
    poses12 = np.asarray(poses12, dtype=np.float64).reshape(len(idx), 12)
    info6 = _per_item(info6, len(idx), (6, 6), "pose_priors: info6")
    return [dict(pose=int(i), pose_hat=p.copy(), H=0.5 * (om + om.T)) for i, p, om in zip(idx, poses12, info6)]


def position_priors(idx, positions, info3, lever_arm=None):
    """Position fixes (GNSS, surveyed points): one prior per pose idx[q] on the position positions[q] (len(idx) x 3,
    world frame) of the body point lever_arm (3, e.g. the antenna offset; default the pose origin; one per prior or one
    shared), with information info3 (3 x 3, one per prior or shared): H = blockdiag(0, info3), so the rotation of the
    measured pose is unused. Units as pose_priors'. -> list of prior dicts."""
    idx = np.asarray(idx, dtype=np.int64).ravel()
    positions = np.asarray(positions, dtype=np.float64).reshape(len(idx), 3)
    info3 = _per_item(info3, len(idx), (3, 3), "position_priors: info3")
    lever = None if lever_arm is None else _per_item(lever_arm, len(idx), (3,), "position_priors: lever_arm")
    out = []
    for q, (i, x, om) in enumerate(zip(idx, positions, info3)):
        H = np.zeros((6, 6))
        H[3:, 3:] = 0.5 * (om + om.T)
        hat = np.concatenate([np.eye(3).ravel(), x])
        d = dict(pose=int(i), pose_hat=hat, H=H)
        if lever is not None:
            d["lever_arm"] = lever[q].copy()
        out.append(d)
    return out

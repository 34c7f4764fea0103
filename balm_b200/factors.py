"""Pose factors built from relative-pose measurements, in the format of Context.set_block_factors /
Context.set_pose_factors / PoseGraph.set_pose_factors (include/balm_b200.h, balm_set_pose_factors)."""
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

"""numpy restatement of the point-noise covariance on blocks contexts (DESIGN.md "Point-noise covariance on blocks
contexts", include/balm_b200.h balm_block_point_covariance / balm_rig_block_point_covariance):

  plain:  Sigma_sel = Y^T R Y,  Y = H~^-1 E
  rig:    Sigma_sel = W^T R W,  W = J Y,  Y = H~_rig^-1 E

E the unit columns of the selected unknowns, ~ the anchor's rows and columns deleted (rig_cov_ref.delete: 1 on H's
diagonal), the anchor's rows of Y zeroed before J and R are applied, R numpy_cov.left_jacobian_point's raw term and J
rig_ref.jacobian."""
import numpy as np

import rig_cov_ref as rc


def unit_columns(n, sel):
    E = np.zeros((n, 6 * len(sel)))
    for u, i in enumerate(sel):
        E[6 * i:6 * i + 6, 6 * u:6 * u + 6] = np.eye(6)
    return E


def solve_selected(H, sel, anchor):
    """Y = H~^-1 E with the anchor's rows zeroed"""
    Y = np.linalg.solve(rc.delete(H, anchor, 1.0), unit_columns(len(H), sel))
    if anchor >= 0:
        Y[6 * anchor:6 * anchor + 6] = 0.0
    return Y


def sel_covariance(H, R, sel, anchor=-1):
    Y = solve_selected(H, sel, anchor)
    return Y.T @ R @ Y


def rig_sel_covariance(H_rig, R, J, sel, anchor=-1):
    W = J @ solve_selected(H_rig, sel, anchor)
    return W.T @ R @ W


def raw_blocks(R, pairs):
    """R's 6x6 blocks on the pattern: [p, a, c] = R[6 i + a, 6 j + c]"""
    return np.stack([R[6 * i:6 * i + 6, 6 * j:6 * j + 6] for i, j in pairs])


def covisible(N, row_ptr, pose_idx):
    """[N, N] True where two poses share a voxel (the diagonal of every observing pose included)"""
    m = np.zeros((N, N), bool)
    for v in range(len(row_ptr) - 1):
        p = pose_idx[row_ptr[v]:row_ptr[v + 1]]
        m[np.ix_(p, p)] = True
    return m


def sel_block(A, sel):
    """the (6 s)^2 sub-block of A on the selected unknowns, in sel's order"""
    idx = np.concatenate([np.arange(6 * i, 6 * i + 6) for i in sel])
    return A[np.ix_(idx, idx)]

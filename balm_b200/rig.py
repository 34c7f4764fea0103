"""Rig calibration: the extrinsics of several LiDARs on one vehicle or handheld rig, optimised jointly with the rig's
trajectory in dense voxel BA on the device (DESIGN.md "Rig calibration", include/balm_b200.h balm_set_rig).

Scan slot s of a context is taken by LiDAR lidar_of[s] at time step base_of[s], so it sits at X_s = T_b E_l: one base
pose per time step and one extrinsic per LiDAR, instead of a free pose per scan. MLCC-style calibration fixes a
reference LiDAR (the default); LiDAR-to-INS calibration fixes every base pose at the INS trajectory and frees E.

calibrate_rig alternates the adaptive voxelisation with the LM, as MLCC does: every round cuts the scans into plane
voxels at the poses the previous round composed, then runs Context.rig_damping_iter on them."""
import numpy as np

from . import _lib as L
from .context import Context


def _split(x):
    x = np.asarray(x, dtype=np.float64)
    return x[:9].reshape(3, 3).T, x[9:12]


def rig_poses(base12, ext12, base_of, lidar_of):
    """The scan poses X_s = T_{base_of[s]} E_{lidar_of[s]} (N x 12, R column-major then p) of base poses base12 (B x 12)
    and extrinsics ext12 (L x 12): R = R_T R_E, p = R_T p_E + p_T."""
    base12 = np.asarray(base12, dtype=np.float64).reshape(-1, 12)
    ext12 = np.asarray(ext12, dtype=np.float64).reshape(-1, 12)
    out = np.zeros((len(base_of), 12))
    for s, (b, l) in enumerate(zip(base_of, lidar_of)):
        Rt, pt = _split(base12[b])
        Re, pe = _split(ext12[l])
        out[s, :9] = (Rt @ Re).T.reshape(9)
        out[s, 9:] = Rt @ pe + pt
    return out


def extrinsic_sigmas(cov, n_free_bases):
    """1-sigma rotation (rad) and translation (m) of every free extrinsic from a rig covariance (Context.rig_covariance's
    cov; the free extrinsics follow the n_free_bases free base poses, 6 each as (phi, t)) -> (rot, trans), each
    (free extrinsics x 3), the square roots of the 6 x 6 blocks' diagonals."""
    d = np.sqrt(np.diag(np.asarray(cov, dtype=np.float64))[6 * n_free_bases:]).reshape(-1, 6)
    return d[:, :3], d[:, 3:]


def calibrate_rig(xyz, scan, base_of, lidar_of, base12, ext12, voxel_size=2.0, rounds=3, fixed_bases=(),
                  fixed_lidars=(0,), precision=L.PREC_TENSOR, device=0, layer_limit=2, min_ps=15,
                  eigen_value_array=(1.0 / 16, 1.0 / 16, 1.0 / 9), max_iter=10, gauge_mode=2, min_planes_per_pose=0,
                  **lm):
    """Calibrate a rig from raw scans. xyz: body-frame points (n x 3) of every scan, scan: the slot of every point;
    slot s was taken by LiDAR lidar_of[s] at base pose base_of[s]. base12 (B x 12) / ext12 (L x 12): the initial base
    poses and extrinsics. Each of the `rounds` rounds cuts plane voxels (Context.cut_voxels with voxel_size, layer_limit,
    min_ps, eigen_value_array) at the composed scan poses and runs rig_damping_iter (max_iter, gauge_mode,
    min_planes_per_pose and any other damping_iter keyword in lm). gauge_mode defaults to 2, which keeps the input's
    frame. precision=PREC_BLOCKS runs the block-sparse rig (Context.set_block_rig), for long drives. -> (base12, ext12,
    traces), traces one LM trace per round."""
    base_of = np.asarray(base_of, dtype=np.int32)
    lidar_of = np.asarray(lidar_of, dtype=np.int32)
    base = np.array(base12, dtype=np.float64, copy=True).reshape(-1, 12)
    ext = np.array(ext12, dtype=np.float64, copy=True).reshape(-1, 12)
    ctx = Context(len(base_of), device, precision)
    try:
        set_rig = ctx.set_block_rig if precision == L.PREC_BLOCKS else ctx.set_rig
        set_rig(base_of, lidar_of, fixed_bases=fixed_bases, fixed_lidars=fixed_lidars)
        traces = []
        for _ in range(rounds):
            ctx.cut_voxels(xyz, scan, rig_poses(base, ext, base_of, lidar_of), voxel_size=voxel_size,
                           layer_limit=layer_limit, min_ps=min_ps, eigen_value_array=eigen_value_array)
            base, ext, tr = ctx.rig_damping_iter(base, ext, max_iter=max_iter, gauge_mode=gauge_mode,
                                                 min_planes_per_pose=min_planes_per_pose, **lm)
            traces.append(tr)
        return base, ext, traces
    finally:
        ctx.close()

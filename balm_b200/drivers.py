"""Headless equivalents of the reference's two benchmark programs (SURVEY section 8f, row N4).

  benchmark_realworld   src/benchmark/benchmark_realworld.cpp:144-236 -- read poses + scans, re-anchor to pose 0,
                        adaptive voxelisation (cut_voxel / recut / tras_opt), BALM2::damping_iter, refined poses.
  benchmark_virtual     src/benchmark/benchmark_virtual.cpp:486-640 -- random planes seen from a random trajectory,
                        noisy initial poses, the twin's dampingIter (:375-482: u0 = 0.1, <= 20 iterations), RSME line.

What is left out on purpose: ROS publishers / rviz (`data_show`, `pub_pl_func`) and the interactive "input '1' to
continue" prompts; everything that decides the numbers is kept, including the messages the programs print.
Both run the association and the optimisation on the GPU through libbalm_b200.so; there is no CPU path.
"""
import time

import numpy as np

from . import _lib as L
from . import io
from .context import Context

# benchmark_realworld runs PREC_BLOCKS from this many scans on, whatever `precision` says: a lidar sequence has local
# co-visibility, and the block-sparse Hessian and solve beat the dense ones there (DESIGN.md "Block-sparse voxel BA").
# The mode is chosen by pose count because the context, and with it the mode, exists before the association runs.
BLOCKS_MIN_POSES = 1000


def pack_poses(R, p):
    """[n,3,3], [n,3] -> [n,12] (R column-major, then p): the layout of IMUST::R.data() followed by p."""
    R = np.asarray(R, dtype=np.float64)
    p = np.asarray(p, dtype=np.float64)
    out = np.zeros((len(R), 12))
    out[:, :9] = R.transpose(0, 2, 1).reshape(len(R), 9)
    out[:, 9:] = p
    return out


def unpack_poses(poses12):
    poses12 = np.asarray(poses12, dtype=np.float64)
    return poses12[:, :9].reshape(-1, 3, 3).transpose(0, 2, 1).copy(), poses12[:, 9:].copy()


def log_so3(R):
    """Log of include/tools.hpp:92-97 (theta from the trace, axis from the skew part)."""
    c = min(1.0, max(-1.0, (np.trace(R) - 1.0) * 0.5))
    theta = np.arccos(c) if np.trace(R) <= 3 - 1e-6 else 0.0
    K = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    return 0.5 * K if abs(theta) < 0.001 else 0.5 * theta / np.sin(theta) * K


def rsme(poses_es, poses_gt):
    """rsme of benchmark_virtual.cpp:48-61 -> (rot [rad], tran [m])."""
    Re, pe = unpack_poses(poses_es)
    Rg, pg = unpack_poses(poses_gt)
    rot = sum(float(np.sum(log_so3(Rg[i].T @ Re[i]) ** 2)) for i in range(len(Re)))
    tran = float(np.sum((pe - pg) ** 2))
    return np.sqrt(rot / len(Re)), np.sqrt(tran / len(Re))


def down_sampling_voxel(xyz, voxel_size):
    """down_sampling_voxel of include/tools.hpp:203-242: one point per occupied voxel = the mean of its points (voxel
    index from the float32 quotient with the "-1 for negatives" rule, truncated). The reference keeps a running float32
    mean in hash-map order; here the mean is taken in float64 and the voxels come out sorted -- display data only."""
    xyz = np.asarray(xyz, dtype=np.float32).reshape(-1, 3)
    if voxel_size < 0.001 or len(xyz) == 0:
        return xyz.copy()
    loc = xyz / np.float32(voxel_size)
    loc = np.where(loc < 0, loc - np.float32(1.0), loc)
    key = np.trunc(loc).astype(np.int64)
    _, inv, cnt = np.unique(key, axis=0, return_inverse=True, return_counts=True)
    inv = inv.reshape(-1)
    out = np.zeros((len(cnt), 3))
    np.add.at(out, inv, xyz.astype(np.float64))
    return (out / cnt[:, None]).astype(np.float32)


def data_show(poses12, scans, voxel_size=0.05):
    """The clouds data_show publishes (benchmark_realworld.cpp:108-142), returned instead: every scan down-sampled at
    5 cm, moved to the world frame of pose 0, concatenated (-> /map_show), and the trajectory (-> /map_path, the scan
    index in the curvature field)."""
    R, p = unpack_poses(poses12)
    R0, p0 = R[0].copy(), p[0].copy()
    p = (p - p0) @ R0
    R = np.einsum("ji,njk->nik", R0, R)
    clouds = []
    for i, s in enumerate(scans):
        q = down_sampling_voxel(s, voxel_size).astype(np.float64)
        clouds.append((q @ R[i].T + p[i]).astype(np.float32))
    cloud = np.concatenate(clouds) if clouds else np.zeros((0, 3), np.float32)
    return cloud, p.astype(np.float32)


def add_voxel_loss_args(ap):
    """--voxel_loss {huber,cauchy} --voxel_loss_scale C on an argparse parser (default: no loss)."""
    ap.add_argument("--voxel_loss", choices=["huber", "cauchy"], default=None,
                    help="robust voxel cost (Context.set_voxel_loss); default: none")
    ap.add_argument("--voxel_loss_scale", type=float, default=None,
                    help="its scale in metres, a plane thickness (about 1.5 - 3 point-noise sigmas)")


def voxel_loss_arg(ap, a):
    """The (kind, scale) of add_voxel_loss_args' options, or None."""
    if a.voxel_loss is None:
        return None
    if a.voxel_loss_scale is None:
        ap.error("--voxel_loss needs --voxel_loss_scale")
    return a.voxel_loss, a.voxel_loss_scale


def _print_trace(trace):
    for i, t in enumerate(trace):  # the line of bavoxel.hpp:1132 / benchmark_virtual.cpp:432
        rho = t["q"] / t["q1"] if t["q1"] != 0 else float("nan")
        print("iter%d: (%f %f) u: %f v: %.1f q: %.3f %f %f" % (i, t["r1"], t["r2"], t["u"], t["v"], rho, t["q1"], t["q"]))


def benchmark_realworld(file_path, voxel_size=2.0, device=0, precision=L.PREC_TENSOR, max_scans=None, quiet=False,
                        keep_scans=False, voxel_loss=None):
    """file_path: the directory holding alidarPose.csv and full<i>.pcd (the reference appends
    "/datas/benchmark_realworld/" to its package path, benchmark_realworld.cpp:77). voxel_loss: None, or (kind, scale)
    as Context.set_voxel_loss takes them (a robust voxel cost; the reference has none).
    Returns dict(poses_init, poses, trace, n_voxels, n_obs, seconds) or None when the plane guard fires."""
    say = (lambda *a: None) if quiet else print
    t0 = time.perf_counter()
    R, p, _, scans = io.read_realworld_dir(file_path, max_scans)
    if len(R) == 0:
        raise ValueError("no poses read")
    R0, p0 = R[0].copy(), p[0].copy()  # benchmark_realworld.cpp:163-168
    p = (p - p0) @ R0
    R = np.einsum("ji,njk->nik", R0, R)
    win_size = len(R)
    say("The size of poses: %d" % win_size)
    poses_init = pack_poses(R, p)
    xyz = np.concatenate(scans).astype(np.float32)
    frame = np.concatenate([np.full(len(s), i, dtype=np.int32) for i, s in enumerate(scans)])
    t_read = time.perf_counter()
    ctx = Context(win_size, device, L.PREC_BLOCKS if win_size >= BLOCKS_MIN_POSES else precision)
    if voxel_loss is not None:
        ctx.set_voxel_loss(*voxel_loss)
    try:
        n_vox, n_obs = ctx.cut_voxels(xyz, frame, poses_init, voxel_size=voxel_size, layer_limit=2, min_ps=15,
                                      eigen_value_array=(1.0 / 16, 1.0 / 16, 1.0 / 9))  # :183-185, bavoxel.hpp:8-19
    except L.BalmError as e:
        if e.status != L.ERR_INVALID or "no plane voxels" not in str(e):
            raise
        n_vox, n_obs = 0, 0  # an empty VOX_HESS: the guard below fires, as in the reference
    t_cut = time.perf_counter()
    say("\nThe planes (point association) cut by adaptive voxelization.")
    say("If the planes are too few, the optimization will be degenerated and fail.")
    say("plane voxels: %d, observations: %d (%d points)" % (n_vox, n_obs, len(frame)))
    if n_vox < 3 * win_size:  # :203-209
        say("Initial error too large.")
        say("Please loose plane determination criteria for more planes.")
        say("The optimization is terminated.")
        return None
    try:
        poses, trace, _ = ctx.damping_iter(poses_init)  # BALM2::damping_iter defaults (bavoxel.hpp:1087,1104,1155)
    except L.BalmError as e:
        if e.status != L.ERR_TOO_FEW_PLANES:
            raise
        say("Initial error too large.")  # bavoxel.hpp:1079-1085
        say("Please loose plane determination criteria for more planes.")
        say("The optimization is terminated.")
        return None
    t_ba = time.perf_counter()
    if not quiet:
        _print_trace(trace)
        print("\nread %.2f s, association %.3f s, optimisation %.3f s" % (t_read - t0, t_cut - t_read, t_ba - t_cut))
    res = dict(poses_init=poses_init, poses=poses, trace=trace, n_voxels=n_vox, n_obs=n_obs,
               seconds=dict(read=t_read - t0, association=t_cut - t_read, optimisation=t_ba - t_cut))
    if keep_scans:
        res["scans"] = scans
    return res


def benchmark_virtual(winSize=20, sufSize=150, ptsSize=40, point_noise=0.05, surf_range=2.0, seed=10, device=0,
                      precision=L.PREC_TENSOR, quiet=False):
    """Parameters and defaults of benchmark_virtual.cpp:535-542 (`seed` replaces time(0), :548). The scene is drawn
    by the library's device generator (same distributions as :553-606, different random stream)."""
    say = (lambda *a: None) if quiet else print
    say("winSize: %d" % winSize)
    say("sufSize: %d" % sufSize)
    say("pstSize: %d" % ptsSize)
    ctx = Context(winSize, device, precision)
    gt, init = ctx.synth_virtual(sufSize, pts_size=ptsSize, point_noise=point_noise, surf_range=surf_range, seed=seed)
    t0 = time.perf_counter()
    # the twin's loop: u0 = 0.1, v0 = 2, <= 20 iterations, 1e-6 exit, pose 0 := identity at the end (:380,408,453,472-479)
    poses, trace, _ = ctx.damping_iter(init, max_iter=20, u0=0.1, v0=2.0, rel_tol=1e-6, gauge_mode=1,
                                       min_planes_per_pose=0)
    dt = time.perf_counter() - t0
    rot, tran = rsme(poses, gt)
    rot0, tran0 = rsme(init, gt)
    if not quiet:
        _print_trace(trace)
        print("RSME: %fdeg, %fm" % (rot * 57.3, tran))  # :520
        print("(initial poses: %fdeg, %fm; %d iterations in %.3f s)" % (rot0 * 57.3, tran0, len(trace), dt))
    return dict(poses_gt=gt, poses_init=init, poses=poses, trace=trace, rsme=(rot, tran), rsme_init=(rot0, tran0))

"""numpy restatement of rig calibration (DESIGN.md "Rig calibration", include/balm_b200.h balm_set_rig):

  X_s = T_{base_of[s]} E_{lidar_of[s]},   cost = the voxel cost (robust_voxels_ref, loss included) at the X_s
  unknowns: free base poses ascending, then free extrinsics ascending, 6 each (phi, t), left update of pose_graph_ref
  g_rig = sum_s J_s^T g_s,   H_rig = J^T H J + sum_s d2(g_s . delta_s^(2))

with J_s = [I on base b | Ad(T_b) = [[R, 0], [p^ R, R]] on lidar l] and the second-order part of the composition
(T_b = (R, p), a the base step, e the extrinsic step, c = R e_phi)

  delta_phi^(2) = 1/2 a_phi x c,   delta_t^(2) = a_phi x (R e_t + p x c) - 1/2 c x (c x p).

lm() restates balm_rig_damping_iter (robust_voxels_ref.lm's rule with the rig update); rig_scene() builds the synthetic
rig the tests calibrate: assoc_ref.synthetic_scans' room seen by three LiDARs with limited fields of view on a base
trajectory that turns about all three axes."""
import numpy as np

import assoc_ref
import numpy_ref as nr
import robust_voxels_ref as rv
from scenes import exp_so3, pack_poses, unpack_pose

hat = nr.hat


def compose(base12, ext12, base_of, lidar_of):
    """X_s = T_b E_l of every slot (N x 12)"""
    out = np.zeros((len(base_of), 12))
    for s, (b, l) in enumerate(zip(base_of, lidar_of)):
        Rt, pt = unpack_pose(np.asarray(base12[b], dtype=np.float64))
        Re, pe = unpack_pose(np.asarray(ext12[l], dtype=np.float64))
        out[s] = np.concatenate([(Rt @ Re).T.reshape(9), Rt @ pe + pt])
    return out


def unknowns(B, L, fixed_bases=(), fixed_lidars=(0,)):
    """the free unknowns in order: j < B a base pose, j >= B extrinsic j - B"""
    return [j for j in range(B) if j not in fixed_bases] + [B + l for l in range(L) if l not in fixed_lidars]


def jacobian(base12, base_of, lidar_of, B, var):
    """J (6N x n_rig): d delta_s / d(unknowns), first order"""
    N = len(base_of)
    J = np.zeros((6 * N, 6 * len(var)))
    col = {j: 6 * u for u, j in enumerate(var)}
    for s in range(N):
        b, l = base_of[s], B + lidar_of[s]
        R, p = unpack_pose(base12[b])
        if b in col:
            J[6 * s:6 * s + 6, col[b]:col[b] + 6] = np.eye(6)
        if l in col:
            Ad = np.zeros((6, 6))
            Ad[:3, :3] = R
            Ad[3:, :3] = hat(p) @ R
            Ad[3:, 3:] = R
            J[6 * s:6 * s + 6, col[l]:col[l] + 6] = Ad
    return J


def correction(base12, base_of, lidar_of, B, var, g):
    """sum_s Hessian of q_s = g_s . delta_s^(2) in the unknowns"""
    col = {j: 6 * u for u, j in enumerate(var)}
    Q = np.zeros((6 * len(var), 6 * len(var)))
    for s in range(len(base_of)):
        b, l = base_of[s], B + lidar_of[s]
        if l not in col:
            continue
        R, p = unpack_pose(base12[b])
        gp, gt = g[6 * s:6 * s + 3], g[6 * s + 3:6 * s + 6]
        e = col[l]
        S = 0.5 * (np.outer(gt, p) + np.outer(p, gt)) - (gt @ p) * np.eye(3)
        Q[e:e + 3, e:e + 3] += -R.T @ S @ R
        if b in col:
            a = col[b]
            B1 = -0.5 * hat(gp) @ R - hat(gt) @ hat(p) @ R  # d2 q / d a_phi d e_phi
            B2 = -hat(gt) @ R                               # d2 q / d a_phi d e_t
            Q[a:a + 3, e:e + 3] += B1
            Q[e:e + 3, a:a + 3] += B1.T
            Q[a:a + 3, e + 3:e + 6] += B2
            Q[e + 3:e + 6, a:a + 3] += B2.T
    return Q


def evaluate(sc, base12, ext12, base_of, lidar_of, var, include_fix=False, kind=rv.TRIVIAL, c=1.0):
    """-> (H_rig, g_rig, cost, H_X, g_X) at the composed scan poses"""
    B = len(base12)
    X = compose(base12, ext12, base_of, lidar_of)
    H, g, r, _, _ = rv.evaluate(sc, X, kind, c, include_fix)
    J = jacobian(base12, base_of, lidar_of, B, var)
    return J.T @ H @ J + correction(base12, base_of, lidar_of, B, var, g), J.T @ g, r, H, g


def cost(sc, base12, ext12, base_of, lidar_of, kind=rv.TRIVIAL, c=1.0, include_fix=True):
    return rv.cost(sc, compose(base12, ext12, base_of, lidar_of), kind, c, include_fix)


def update(base12, ext12, var, dx):
    """the left step of dx on every free unknown"""
    B = len(base12)
    allp = np.concatenate([np.asarray(base12, dtype=np.float64), np.asarray(ext12, dtype=np.float64)])
    out = allp.copy()
    for u, j in enumerate(var):
        R, p = unpack_pose(allp[j])
        dR = exp_so3(dx[6 * u:6 * u + 3])
        out[j] = np.concatenate([(dR @ R).T.reshape(9), dR @ p + dx[6 * u + 3:6 * u + 6]])
    return out[:B], out[B:]


def lm(sc, base12, ext12, base_of, lidar_of, var, kind=rv.TRIVIAL, c=1.0, max_iter=10, u0=0.01, v0=2.0, rel_tol=1e-6,
       hess_includes_fix=False):
    """balm_rig_damping_iter's rule -> (base12, ext12, trace, per-iteration accepted (base12, ext12)), no gauge step"""
    base, ext = np.array(base12, dtype=np.float64), np.array(ext12, dtype=np.float64)
    u, v = u0, v0
    calc, trace, per = True, [], []
    H = g = None
    r1 = 0.0
    for it in range(max_iter):
        if calc:
            H, g, r1, _, _ = evaluate(sc, base, ext, base_of, lidar_of, var, hess_includes_fix, kind, c)
        D = H.diagonal().copy()
        dx = np.linalg.solve(H + u * np.diag(D), -g)
        q1 = 0.5 * dx @ (u * D * dx - g)
        bt, et = update(base, ext, var, dx)
        r2 = cost(sc, bt, et, base_of, lidar_of, kind, c)
        q = r1 - r2
        t = dict(r1=r1, r2=r2, u=u, v=v, q=q, q1=q1, accepted=False, recomputed_hess=calc)
        if q > 0:
            base, ext = bt, et
            u *= max(1 - (2 * q / q1 - 1) ** 3, 1.0 / 3.0)
            v, calc = 2.0, True
            t["accepted"] = True
        else:
            u, v, calc = u * v, 2 * v, False
        trace.append(t)
        per.append((base.copy(), ext.copy()))
        if rel_tol >= 0 and abs(r1 - r2) / r1 < rel_tol:
            break
    return base, ext, trace, per


def pose_error(a12, b12):
    """(rotation angle in rad, position distance in m) between two 12-vector poses"""
    Ra, pa = unpack_pose(np.asarray(a12, dtype=np.float64))
    Rb, pb = unpack_pose(np.asarray(b12, dtype=np.float64))
    cosang = np.clip((np.trace(Ra.T @ Rb) - 1) / 2, -1.0, 1.0)
    return float(np.arccos(cosang)), float(np.linalg.norm(pa - pb))


def perturb(p12, rng, rot=2 / 57.3, tra=0.1):
    """p12 moved by a rotation of `rot` rad and a translation of `tra` m in random directions"""
    R, p = unpack_pose(np.asarray(p12, dtype=np.float64))
    a, t = rng.normal(size=3), rng.normal(size=3)
    return np.concatenate([(exp_so3(rot * a / np.linalg.norm(a)) @ R).T.reshape(9), p + tra * t / np.linalg.norm(t)])


# ---------------- the synthetic rig scene ----------------
YAWS = (0.0, np.pi / 3, -np.pi / 3)              # the three LiDARs' yaw on the rig
OFFSETS = ((0.3, 0.0, 0.1), (0.05, 0.3, 0.05), (0.05, -0.3, 0.15))
HALF_FOV = np.deg2rad(50.0)                     # each LiDAR sees +-50 deg of azimuth and +-35 deg of elevation
HALF_VFOV = np.deg2rad(35.0)


def rig_truth(n_base=12):
    """true base poses and extrinsics -> (base12, ext12). The bases turn about a different axis each: roll and pitch
    swing back and forth while the yaw grows, so no one axis is left fixed by every base rotation (an axis a with
    R_b a = a for every b would make the extrinsic's translation along a unobservable with the bases fixed)."""
    Rs = [exp_so3(np.array([0.35 * np.sin(0.7 * i), 0.3 * np.sin(0.45 * i + 1.0) - 0.25, 0.22 * i]))
          for i in range(n_base)]
    ps = [np.array([0.25 * i - 1.5, 0.4 * np.sin(0.5 * i), 0.05 * i]) for i in range(n_base)]
    ext = [(exp_so3(np.array([0.02 * k, -0.015 * k, y])), np.array(o)) for k, (y, o) in enumerate(zip(YAWS, OFFSETS))]
    return pack_poses(Rs, ps), pack_poses([e[0] for e in ext], [e[1] for e in ext])


def perturbed_start(scene, seed=7):
    """the start the calibration tests use: LiDARs 1 and 2 moved 2 deg / 0.1 m, every base pose 0.5 deg / 3 cm
    -> (base12, ext12)"""
    rng = np.random.default_rng(seed)
    ext = scene["ext12"].copy()
    for l in range(1, len(ext)):
        ext[l] = perturb(scene["ext12"][l], rng)
    base = scene["base12"].copy()
    for b in range(len(base)):
        base[b] = perturb(scene["base12"][b], rng, 0.5 / 57.3, 0.03)
    return base, ext


def rig_scene(n_base=12, pts_draw=16000, seed=11):
    """Scans of assoc_ref.synthetic_scans' room: slot s = b * 3 + l is LiDAR l at base pose b, its points the room's
    world points inside the LiDAR's field of view, in its own frame (float32-rounded). -> dict(xyz, scan, base_of,
    lidar_of, base12, ext12) with the true poses."""
    base12, ext12 = rig_truth(n_base)
    L = len(ext12)
    base_of = np.repeat(np.arange(n_base), L).astype(np.int32)
    lidar_of = np.tile(np.arange(L), n_base).astype(np.int32)
    X = compose(base12, ext12, base_of, lidar_of)
    pts, scan = [], []
    for s in range(len(base_of)):
        world, _, _ = assoc_ref.synthetic_scans(n_poses=1, pts_per_scan=pts_draw, seed=seed * 1000 + s)
        R, p = unpack_pose(X[s])
        body = (world - p) @ R
        az = np.arctan2(body[:, 1], body[:, 0])
        el = np.arctan2(body[:, 2], np.linalg.norm(body[:, :2], axis=1))
        keep = (np.abs(az) < HALF_FOV) & (np.abs(el) < HALF_VFOV)
        pts.append(body[keep].astype(np.float32).astype(np.float64))
        scan.append(np.full(keep.sum(), s, dtype=np.int32))
    return dict(xyz=np.concatenate(pts), scan=np.concatenate(scan), base_of=base_of, lidar_of=lidar_of,
                base12=base12, ext12=ext12)


def cut(scene, base12, ext12, voxel_size=2.0):
    """assoc_ref.cut_voxels of the scene's scans at the composed poses -> a numpy_ref scene dict"""
    X = compose(base12, ext12, scene["base_of"], scene["lidar_of"])
    row_ptr, pose_idx, obs10, coe, _ = assoc_ref.cut_voxels(scene["xyz"], scene["scan"],
                                                            [unpack_pose(x) for x in X], voxel_size=voxel_size)
    return dict(n_poses=len(X), row_ptr=row_ptr, pose_idx=pose_idx, obs10=obs10, coe=coe, fix10=None)


def ins_scene(scene, lidar=1):
    """the LiDAR-to-INS case of a rig scene: LiDAR `lidar`'s scans alone, slot b at base pose b, one extrinsic
    -> a scene dict of rig_scene's form (the true poses)"""
    keep = scene["lidar_of"][scene["scan"]] == lidar
    slots = np.nonzero(scene["lidar_of"] == lidar)[0]
    slot_of = np.full(len(scene["lidar_of"]), -1, dtype=np.int32)
    slot_of[slots] = np.arange(len(slots))
    return dict(xyz=scene["xyz"][keep], scan=slot_of[scene["scan"][keep]], base_of=scene["base_of"][slots],
                lidar_of=np.zeros(len(slots), dtype=np.int32), base12=scene["base12"],
                ext12=scene["ext12"][lidar:lidar + 1])

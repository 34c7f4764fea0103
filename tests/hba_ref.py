"""numpy restatements for hierarchical BA (balm_batch_merge_scans, balm_b200.hba):

  keyframe_ref    a window's scans in the body frame of its slot 0, reduced by drivers.down_sampling_voxel, with the
                  transform written elementwise in fp64 in the kernel's order (numpy's `@` sums in another order and may
                  use FMA), so that the device result is reproduced bit for bit
  propagate_ref   the layers' results carried down to the scans, written with 4 x 4 homogeneous matrices
  drift_scene     lidar-like scans of a room from a closed-loop trajectory, with initial poses that drift: a random walk
                  of small errors on every relative motion, so that only the upper layers can correct the anchors
"""
import numpy as np

from balm_b200 import drivers


def _rt(p12):
    p12 = np.asarray(p12, dtype=np.float64)
    return p12[:9].reshape(3, 3).T, p12[9:]  # R[a, c] = p12[3 c + a]


def keyframe_ref(scans, window, poses12, voxel_size):
    """Keyframe of one window: q = R_a^T (R_k b + t_k - t_a) for every point b of every slot k (a = slot 0), each fp64
    operation separately rounded in the order ((r0 b0 + r1 b1) + r2 b2) + t, - t_a, then R_a^T in the same form, rounded
    to float32; then down_sampling_voxel at voxel_size (< 0.001: the points as they are, in (slot, point) order)."""
    Ra, ta = _rt(poses12[0])
    parts = []
    for k, s in enumerate(window):
        R, t = _rt(poses12[k])
        b = np.asarray(scans[s], dtype=np.float32).reshape(-1, 3).astype(np.float64)
        d = [((R[a, 0] * b[:, 0] + R[a, 1] * b[:, 1]) + R[a, 2] * b[:, 2]) + t[a] - ta[a] for a in range(3)]
        q = [(Ra[0, a] * d[0] + Ra[1, a] * d[1]) + Ra[2, a] * d[2] for a in range(3)]
        parts.append(np.stack(q, axis=1).astype(np.float32))
    cloud = np.concatenate(parts) if parts else np.zeros((0, 3), np.float32)
    return drivers.down_sampling_voxel(cloud, voxel_size)


def _h(p12):
    R, t = _rt(p12)
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def _p12(T):
    return np.concatenate([T[:3, :3].T.reshape(9), T[:3, 3]])


def _inv(T):
    """Inverse of a rigid motion, [R^T, -R^T t]: input rotations read from text files are orthonormal only to their
    printed digits, and the general inverse of such a matrix is not the motion's inverse."""
    out = np.eye(4)
    out[:3, :3] = T[:3, :3].T
    out[:3, 3] = -T[:3, :3].T @ T[:3, 3]
    return out


def propagate_ref(layers):
    """layers as balm_b200.hba records them (bottom first, the top last; per layer windows, poses_in and per window the
    poses carried down). Item i of a layer: F_w T_w0^-1 T_wk for the lowest window w holding it in slot k, where F_w
    is the final pose of keyframe w; the top's F is its slot 0's input pose."""
    F = None
    for lay in layers[::-1]:
        wins = lay["windows"]
        if F is None:
            F = [_h(lay["poses_in"][wins[0][0]])]
        owner = {}
        for w, win in enumerate(wins):
            for k, i in enumerate(win):
                owner.setdefault(i, (w, k))
        F = [F[w] @ _inv(_h(lay["poses"][w][0])) @ _h(lay["poses"][w][k])
             for w, k in (owner[i] for i in range(len(lay["poses_in"])))]
    return np.array([_p12(T) for T in F])


def _exp(phi):
    th = np.linalg.norm(phi)
    K = np.array([[0, -phi[2], phi[1]], [phi[2], 0, -phi[0]], [-phi[1], phi[0], 0]])
    if th < 1e-12:
        return np.eye(3) + K
    return np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th ** 2 * K @ K


def drift_scene(n_scans=60, pts_per_scan=6000, room=11.0, seed=21, rot_step=2e-3, tran_step=1.5e-2):
    """-> (scans, poses_gt, poses_init), poses P x 12. The sensor goes round an ellipse inside a box room of half-size
    `room` with a slanted plane and clutter; it sees every face. poses_init[0] = poses_gt[0]; every later relative motion
    is perturbed by N(0, rot_step) rad per axis and N(0, tran_step) m per axis, so the error grows along the path."""
    rng = np.random.default_rng(seed)
    ang = np.linspace(0, 2 * np.pi, n_scans, endpoint=False)
    Rs = [_exp(np.array([0.05 * np.sin(a), 0.04 * np.cos(2 * a), a])) for a in ang]
    ps = [np.array([0.5 * room * np.cos(a), 0.35 * room * np.sin(a), 0.3 * np.sin(3 * a)]) for a in ang]
    scans = []
    for i in range(n_scans):
        n = pts_per_scan
        face = rng.integers(0, 8, n)
        u, v = rng.uniform(-room, room, n), rng.uniform(-room, room, n)
        w = np.zeros((n, 3))
        for f in range(6):
            m = face == f
            ax, sgn = f // 2, (1 if f % 2 else -1)
            w[m, ax] = sgn * room
            w[m, (ax + 1) % 3] = u[m]
            w[m, (ax + 2) % 3] = v[m]
        m = face == 6
        w[m] = np.stack([u[m] * 0.5, v[m] * 0.5, 0.3 * u[m] + 0.2 * v[m] - 0.5 * room], axis=1)
        m = face == 7
        w[m] = rng.normal(0, 0.6, (m.sum(), 3)) + rng.choice([-room / 2, 0.0, room / 2], (m.sum(), 3))
        w += rng.normal(0, 0.01, w.shape)
        scans.append(((w - ps[i]) @ Rs[i]).astype(np.float32))
    gt = [(Rs[i], ps[i]) for i in range(n_scans)]
    init = [gt[0]]
    for i in range(1, n_scans):  # init_i = init_{i-1} . (gt_{i-1}^-1 gt_i) . noise
        Rp, pp = gt[i - 1]
        dR, dp = Rp.T @ Rs[i], Rp.T @ (ps[i] - pp)
        dR = dR @ _exp(rng.normal(0, rot_step, 3))
        dp = dp + rng.normal(0, tran_step, 3)
        Ri, pi = init[-1]
        init.append((Ri @ dR, Ri @ dp + pi))
    pack = lambda P: drivers.pack_poses([r for r, _ in P], [t for _, t in P])
    return scans, pack(gt), pack(init)

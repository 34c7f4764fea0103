"""The restatement of the point-noise covariance on blocks contexts (block_point_cov_ref.py) against the dense
sandwiches it restricts: H~^-1 R H~^-T (numpy_cov) and rig_cov_ref.rig_covariance, on the CPU."""
import numpy as np

import block_hessian_ref as bref
import block_point_cov_ref as bp
import numpy_cov as nc
import rig_cov_ref as rc
import rig_ref as rr
from scenes import make_scene

PN = 0.01


def _rig(sc):
    N = sc["n_poses"]
    base_of, lidar_of = np.arange(N) // 2, np.arange(N) % 2
    base = sc["poses_init"][0::2].copy()
    ext = np.zeros((2, 12))
    ext[0] = ext[1] = np.concatenate([np.eye(3).reshape(9), np.zeros(3)])
    ext[1, 9:] = [0.2, -0.1, 0.05]
    return base_of, lidar_of, base, ext


def _R(sc, X, include_fix):
    return nc.left_jacobian_point(sc["n_poses"], sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], X,
                                  sc.get("fix10") if include_fix else None, pnoise=PN)


def test_raw_term_lives_on_the_covisibility_pattern():
    sc = bref.corridor(24, w=3, planes_per_pose=6, seed=2)
    R = _R(sc, sc["poses_init"], False)
    m = np.kron(bp.covisible(sc["n_poses"], sc["row_ptr"], sc["pose_idx"]), np.ones((6, 6), bool))
    assert not m.all()
    assert np.all(R[~m] == 0.0) and np.abs(R[m]).max() > 0


def test_plain_selection_is_the_sandwich_sub_block():
    sc = make_scene(n_poses=8, n_planes=50, seed=7, with_fix=True)
    x = sc["poses_init"]
    N = sc["n_poses"]
    ident = np.concatenate([np.eye(3).reshape(9), np.zeros(3)])[None]
    var = rr.unknowns(N, 1, fixed_lidars=(0,))
    H = rr.evaluate(sc, x, ident, np.arange(N), np.zeros(N, int), var, True)[0]
    R = _R(sc, x, True)
    for anchor in (-1, 3):
        Hi = np.linalg.inv(rc.delete(H, anchor, 1.0))
        full = rc.delete(Hi @ rc.delete(R, anchor, 0.0) @ Hi.T, anchor, 0.0)
        sel = [5, 0, 3, 7]
        S = bp.sel_covariance(H, R, sel, anchor)
        assert np.abs(S - bp.sel_block(full, sel)).max() < 1e-9 * np.abs(full).max()
        if anchor >= 0:
            a = slice(12, 18)  # anchor 3 is sel[2]
            assert np.all(S[a] == 0) and np.all(S[:, a] == 0)


def test_rig_selection_is_the_rig_sandwich_sub_block():
    sc = make_scene(n_poses=8, n_planes=50, seed=5, with_fix=True)
    base_of, lidar_of, base, ext = _rig(sc)
    var = rr.unknowns(len(base), 2)
    X = rr.compose(base, ext, base_of, lidar_of)
    H_rig = rr.evaluate(sc, base, ext, base_of, lidar_of, var, True)[0]
    J = rr.jacobian(base, base_of, lidar_of, len(base), var)
    R = _R(sc, X, True)
    for anchor in (-1, 1):
        _, full = rc.rig_covariance(sc, base, ext, base_of, lidar_of, var, pnoise=PN, include_fix=True, anchor=anchor)
        for sel in ([len(var) - 1], [4, 0, 2]):
            S = bp.rig_sel_covariance(H_rig, R, J, sel, anchor)
            assert np.abs(S - bp.sel_block(full, sel)).max() < 1e-9 * np.abs(full).max()

"""CPU checks of the rig restatement (rig_ref): its g_rig and H_rig against differences of the cost along the rig's own
update path, the gauge identities, the single-LiDAR identity and the calibration of the synthetic rig scene."""
import numpy as np
import pytest

import rig_ref as rr
import robust_voxels_ref as rv
from scenes import make_scene, unpack_pose

BASE_OF = np.array([0, 0, 1, 1, 2, 2])
LIDAR_OF = np.array([0, 1, 0, 1, 0, 1])


def _inv(p12):
    R, t = unpack_pose(p12)
    return np.concatenate([R.reshape(9), -R.T @ t])  # R^T column-major is R row-major


def two_lidar_rig(with_fix, far=0.0, drop=0.0):
    """make_scene's six scans as three base poses x two LiDARs (E_0 = I, E_1 = the pose of scan 1 in scan 0's frame),
    every base moved by `far` metres"""
    sc = make_scene(n_poses=6, n_planes=30, seed=4, with_fix=with_fix, drop=drop)
    X = sc["poses_init"]
    base = X[0::2].copy()
    ext = np.zeros((2, 12))
    ext[0] = np.concatenate([np.eye(3).reshape(9), np.zeros(3)])
    ext[1] = rr.compose(np.array([_inv(X[0])]), np.array([X[1]]), [0], [0])[0]
    base[:, 9:] += far * np.array([1.0, -0.5, 0.3])
    return sc, base, ext


def _cost_fn(sc, base, ext, var, include_fix):
    return lambda dx: rr.cost(sc, *rr.update(base, ext, var, dx), BASE_OF, LIDAR_OF, include_fix=include_fix)


@pytest.mark.parametrize("with_fix", [False, True])
@pytest.mark.parametrize("far", [0.0, 100.0])
def test_gradient_and_hessian_along_the_update_path(with_fix, far):
    sc, base, ext = two_lidar_rig(with_fix, far)
    var = rr.unknowns(3, 2, fixed_lidars=())  # every unknown free: base and extrinsic steps together
    H, g, _, _, _ = rr.evaluate(sc, base, ext, BASE_OF, LIDAR_OF, var, with_fix)
    f = _cost_fn(sc, base, ext, var, with_fix)
    h = 1e-5
    gfd = np.array([(f(h * e) - f(-h * e)) / (2 * h) for e in np.eye(len(g))])
    assert np.abs(gfd - g).max() < 1e-5 * np.abs(g).max()
    rng = np.random.default_rng(3)
    hh = 1e-5 if far else 1e-4  # 100 m from the origin the third-order terms grow with |p|
    for _ in range(3):
        d = rng.normal(size=len(g))
        sd = (f(hh * d) - 2 * f(0 * d) + f(-hh * d)) / hh ** 2
        assert abs(d @ H @ d - sd) < 1e-4 * abs(sd)


@pytest.mark.parametrize("with_fix", [False, True])
def test_gauge_identities(with_fix):
    sc, base, ext = two_lidar_rig(with_fix, far=20.0)
    var = rr.unknowns(3, 2, fixed_lidars=())
    H, g, _, _, _ = rr.evaluate(sc, base, ext, BASE_OF, LIDAR_OF, var, with_fix)
    scale = np.abs(H).max()
    # a common left step of every base pose: a straight null line -> H d = 0 and g . d = 0 (without fix clusters)
    for k in range(6):
        d = np.zeros(len(g))
        for u in range(3):
            d[6 * u + k] = 1.0
        if not with_fix:
            assert abs(d @ H @ d) < 1e-9 * scale
            assert abs(g @ d) < 1e-9 * np.abs(g).max() * 6
    # T_b -> T_b Q, E_l -> Q^-1 E_l with every extrinsic free leaves every scan pose, so fix clusters too: only
    # g . d = 0 (the path is curved)
    for k in range(6):
        d = np.zeros(len(g))
        for u in range(3):
            R, p = unpack_pose(base[u])
            Ad = np.zeros((6, 6)); Ad[:3, :3] = R; Ad[3:, :3] = rr.hat(p) @ R; Ad[3:, 3:] = R
            d[6 * u:6 * u + 6] = Ad[:, k]
        q = np.zeros(6); q[k] = 1.0
        for l in range(2):  # Q^-1 E_l to first order: -e in E_l's left coordinates
            d[18 + 6 * l:18 + 6 * l + 6] = -q
        assert abs(g @ d) < 1e-10 * np.abs(g).max() * np.abs(d).sum()


@pytest.mark.parametrize("with_fix", [False, True])
def test_single_lidar_identity_is_the_scan_hessian(with_fix):
    sc = make_scene(n_poses=6, n_planes=30, seed=4, with_fix=with_fix)
    ident = np.concatenate([np.eye(3).reshape(9), np.zeros(3)])[None]
    base_of, lidar_of = np.arange(6), np.zeros(6, dtype=int)
    var = rr.unknowns(6, 1, fixed_lidars=(0,))
    H, g, r, HX, gX = rr.evaluate(sc, sc["poses_init"], ident, base_of, lidar_of, var, with_fix)
    assert np.array_equal(H, HX) and np.array_equal(g, gX)


def test_loss_is_the_weighted_scene():
    sc, base, ext = two_lidar_rig(with_fix=False, far=0.0)
    var = rr.unknowns(3, 2)
    X = rr.compose(base, ext, BASE_OF, LIDAR_OF)
    _, w = rv.weights(sc, X, rv.CAUCHY, 0.01)
    H, g, _, _, _ = rr.evaluate(sc, base, ext, BASE_OF, LIDAR_OF, var, False, rv.CAUCHY, 0.01)
    Hw, gw, _, _, _ = rr.evaluate(rv.weighted(sc, w), base, ext, BASE_OF, LIDAR_OF, var, False)
    assert np.allclose(H, Hw, rtol=0, atol=1e-12 * np.abs(H).max()) and np.allclose(g, gw, rtol=0, atol=1e-12 * np.abs(g).max())


def test_rig_scene_calibration():
    """Extrinsics 2 deg / 0.1 m off and base poses 0.5 deg / 3 cm off: two rounds of cut + LM bring both free
    extrinsics at least 10x closer to the truth (seed 7: from 0.035 rad / 0.1 m to at most 0.00116 rad / 0.0058 m)."""
    S = rr.rig_scene()
    base, ext = rr.perturbed_start(S)
    var = rr.unknowns(12, 3)
    for _ in range(2):
        sc = rr.cut(S, base, ext)
        base, ext, tr, _ = rr.lm(sc, base, ext, S["base_of"], S["lidar_of"], var)
        assert tr[0]["accepted"]
    for l in (1, 2):
        dr, dp = rr.pose_error(ext[l], S["ext12"][l])
        assert dr < 0.1 * (2 / 57.3) and dp < 0.1 * 0.1, (l, dr, dp)


def test_lidar_to_ins_calibration():
    """L = 1, every base pose fixed at the truth, LiDAR 1's extrinsic 2 deg / 0.1 m off: three rounds of cut + LM bring
    it at least 10x closer (seed 7: to 0.00120 rad / 0.0029 m). The bases turn about different axes, so no direction
    of the extrinsic's translation is left unobservable."""
    S = rr.ins_scene(rr.rig_scene())
    _, ext0 = rr.perturbed_start(rr.rig_scene())
    base, ext = S["base12"], ext0[1:2]
    var = rr.unknowns(len(base), 1, fixed_bases=range(len(base)), fixed_lidars=())
    for _ in range(3):
        sc = rr.cut(S, base, ext)
        base, ext, tr, _ = rr.lm(sc, base, ext, S["base_of"], S["lidar_of"], var)
        assert tr[0]["accepted"]
    assert np.array_equal(base, S["base12"])
    dr, dp = rr.pose_error(ext[0], S["ext12"][0])
    assert dr < 0.1 * (2 / 57.3) and dp < 0.1 * 0.1, (dr, dp)

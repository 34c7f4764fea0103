"""balm_b200.odometry_factors against the pose-graph restatement pose_graph_ref.py: the factor it builds is zero at the
odometry poses and, to second order, costs 1/2 xi^T info xi for a body-frame perturbation xi of scan b."""
import numpy as np
import pytest

import pose_graph_ref as pgr
from balm_b200 import odometry_factors


def _trajectory(rng, n):
    return np.array([pgr.random_pose(rng, rot=1.0, tran=20.0) for _ in range(n)])


def _info(rng):
    return pgr.random_spd(rng, 6, cond=1e2) * 50.0


def test_zero_at_the_odometry_poses():
    rng = np.random.default_rng(0)
    poses = _trajectory(rng, 6)
    fs = odometry_factors(poses, _info(rng), edges=[(0, 1), (1, 2), (4, 2), (0, 5)])
    for f in fs:
        e = pgr.factor_terms(poses, f)[0]
        assert np.abs(e).max() < 1e-12
    G = pgr.random_pose(rng)  # a common left transform keeps them zero
    moved = np.array([pgr.compose(G, p) for p in poses])
    assert all(np.abs(pgr.factor_terms(moved, f)[0]).max() < 1e-10 for f in fs)


def test_default_edges_and_shapes():
    rng = np.random.default_rng(1)
    poses = _trajectory(rng, 5)
    infos = np.stack([_info(rng) for _ in range(4)])
    fs = odometry_factors(poses, infos)
    assert [list(f["poses"]) for f in fs] == [[0, 1], [1, 2], [2, 3], [3, 4]]
    assert all(f["H"].shape == (12, 12) and np.array_equal(f["poses_hat"], poses[f["poses"]]) for f in fs)
    with pytest.raises(ValueError):
        odometry_factors(poses, infos[:2])


@pytest.mark.parametrize("seed", [2, 3, 4])
def test_cost_is_the_information_form_to_second_order(seed):
    """T_b <- T_b (Exp psi, rho): cost_f / (1/2 xi^T info xi) - 1 shrinks linearly with |xi|."""
    rng = np.random.default_rng(seed)
    poses = _trajectory(rng, 2)
    om = _info(rng)
    f = odometry_factors(poses, om)[0]
    d = rng.normal(size=6)
    d /= np.linalg.norm(d)
    errs = []
    for s in (1e-2, 1e-3, 1e-4):
        xi = s * d
        Rb, pb = pgr.split(poses[1])
        moved = poses.copy()
        moved[1] = pgr.pack(Rb @ pgr.exp_so3(xi[:3]), Rb @ xi[3:] + pb)
        c = pgr.factor_terms(moved, f)[2]
        errs.append(abs(c / (0.5 * xi @ om @ xi) - 1.0))
    print(f"seed {seed}: relative errors {errs}")
    # the first-order term grows with |p^_b| (poses up to ~40 m from the origin here)
    assert errs[2] < 1e-2
    assert errs[1] < 0.2 * errs[0] and errs[2] < 0.2 * errs[1]


def test_pd_and_gauge():
    rng = np.random.default_rng(5)
    poses = _trajectory(rng, 3)
    for f in odometry_factors(poses, _info(rng), edges=[(0, 2), (2, 1)]):
        assert pgr.pd_ok(f["H"])
        assert np.array_equal(f["H"], f["H"].T)
        assert np.abs(f["H"] @ pgr.gauge_vectors(2)).max() <= 1e-10 * np.abs(f["H"]).max()

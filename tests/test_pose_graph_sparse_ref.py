"""The scipy.sparse restatement of the pose graph (pose_graph_sparse_ref.py) against the dense numpy oracle at small P:
blocks, gradient, cost and one damped solve."""
import numpy as np
import pytest

import pose_graph_ref as pg
import pose_graph_sparse_ref as spg


def _factors(P, seed):
    rng = np.random.default_rng(seed)
    truth = np.array([pg.random_pose(rng, 0.5, 3.0) for _ in range(P)])
    sets = pg.pyramid_factor_poses(P, top=8) + [[3, P - 2]]  # plus one long-range factor
    return [pg.make_factor(rng, truth, s, noise=0.01) for s in sets], pg.perturb(rng, truth, 0.05, 0.2)


@pytest.mark.parametrize("P", [12, 60])
def test_sparse_restatement_matches_the_dense_oracle(P):
    factors, x = _factors(P, P)
    Hs, gs, rs = spg.evaluate(x, factors, P)
    Hd, gd, rd = pg.evaluate(x, factors, P)
    assert abs(rs - rd) <= 1e-13 * abs(rd)
    assert np.abs(gs - gd).max() <= 1e-13 * np.abs(gd).max()
    assert np.abs(Hs.toarray() - Hd).max() <= 1e-13 * np.abs(Hd).max()
    pairs = spg.block_pairs(factors)
    nz = {(i, j) for i in range(P) for j in range(i, P) if np.any(Hd[6 * i:6 * i + 6, 6 * j:6 * j + 6] != 0)}
    assert set(map(tuple, pairs.tolist())) == nz
    B = spg.blocks(Hs, pairs)
    for (i, j), b in zip(pairs, B):
        assert np.abs(b - Hd[6 * i:6 * i + 6, 6 * j:6 * j + 6]).max() <= 1e-13 * np.abs(Hd).max()
    u = 0.01
    dx, q1 = spg.damped_solve(Hs, gs, u)
    D = np.diag(Hd)
    dxd = np.linalg.solve(Hd + u * np.diag(D), -gd)
    assert np.abs(dx - dxd).max() <= 1e-9 * np.abs(dxd).max()
    assert abs(q1 - 0.5 * dxd @ (u * D * dxd - gd)) <= 1e-9 * abs(q1)
    xt, r1, r2 = spg.lm_step(x, factors, P, u)
    _, tr, per = pg.lm(x, factors, P, max_iter=1, u0=u)
    assert r1 == tr[0]["r1"] and abs(r2 - tr[0]["r2"]) <= 1e-9 * r1
    assert np.abs(pg.pose_update(x, dxd) - xt).max() <= 1e-9

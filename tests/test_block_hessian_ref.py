"""block_hessian_ref (the restatement the PREC_BLOCKS tests compare against) pinned to numpy_ref.evaluate."""
import numpy as np
import pytest

import block_hessian_ref as bref
import numpy_ref
import scenes


def _scenes():
    yield scenes.make_scene(n_poses=7, n_planes=30, seed=1)
    yield scenes.make_scene(n_poses=9, n_planes=40, seed=2, drop=0.4)
    yield scenes.make_scene(n_poses=8, n_planes=30, seed=3, drop=0.3, with_fix=True)
    yield bref.corridor(30, w=3, planes_per_pose=6, seed=4)
    yield bref.corridor(25, w=2, planes_per_pose=6, seed=5, with_fix=True)


@pytest.mark.parametrize("k", range(5))
@pytest.mark.parametrize("include_fix", [False, True])
def test_matches_numpy_ref(k, include_fix):
    sc = list(_scenes())[k]
    poses = sc["poses_init"]
    H, g, r = numpy_ref.evaluate(sc, poses, include_fix=include_fix)
    pairs, blocks, gb, rb = bref.evaluate(sc, poses, include_fix=include_fix)
    scale = np.abs(H).max()  # the corridor's coordinates make the raw moments cancel: summation order shows at 1e-13
    assert np.abs(blocks - bref.blocks_of(H, pairs)).max() <= 1e-11 * scale
    # nothing of H lies outside the pattern
    assert np.abs(bref.to_sparse(sc["n_poses"], pairs, blocks).toarray() - H).max() <= 1e-11 * scale
    assert np.abs(gb - g).max() <= 1e-11 * np.abs(g).max()
    assert abs(rb - r) <= 1e-10 * abs(r)


def test_pairs_are_the_covisible_pairs():
    sc = bref.corridor(40, w=3, planes_per_pose=6, seed=6)
    N = sc["n_poses"]
    want = {(i, i) for i in range(N)}
    for v in range(len(sc["row_ptr"]) - 1):
        ps = sc["pose_idx"][sc["row_ptr"][v]:sc["row_ptr"][v + 1]]
        want |= {(int(a), int(b)) for a in ps for b in ps if a <= b}
    pairs = bref.pairs_from_csr(N, sc["row_ptr"], sc["pose_idx"])
    assert [tuple(p) for p in pairs] == sorted(want)


def test_corridor_shape():
    sc = bref.corridor(200, w=8, planes_per_pose=30, seed=7)
    counts = np.bincount(sc["pose_idx"], minlength=200)
    assert counts.min() >= 30
    assert np.abs(sc["poses_gt"][:, 9:]).max() < 1100.0
    k = np.diff(sc["row_ptr"])
    assert k.max() == 17 and k.min() >= 2

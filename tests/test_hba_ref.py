"""The numpy restatements of hierarchical BA (tests/hba_ref.py) and the host side of balm_b200.hba, without a GPU:
keyframes at voxel size 0 are the plain transformed concatenation, propagation through unchanged upper layers keeps the
bottom layer's relative poses, and only relative poses matter (gauge freedom)."""
import numpy as np
import pytest

import hba_ref
from balm_b200 import drivers, hba


def _rand_poses(rng, n):
    R = [hba_ref._exp(rng.normal(0, 0.7, 3)) for _ in range(n)]
    return drivers.pack_poses(R, rng.normal(0, 5, (n, 3)))


def _pyramid(rng, n=60, length=10, stride=5, top_size=4):
    """Layer records as hba() keeps them, with random input and refined poses; a keyframe's input pose is that of its
    window's slot 0."""
    layers = []
    x = _rand_poses(rng, n)
    while True:
        top = n <= top_size
        wins = [list(range(n))] if top else hba.layer_windows(n, length, stride)
        if layers:
            x = np.array([layers[-1]["poses_in"][w[0]] for w in layers[-1]["windows"]])
        layers.append(dict(windows=wins, poses_in=x, poses=[_rand_poses(rng, len(w)) for w in wins]))
        if top:
            return layers
        n = len(wins)


def _rel(a, b):
    return np.linalg.inv(hba_ref._h(a)) @ hba_ref._h(b)


def test_layer_windows():
    assert hba.layer_windows(24) == [list(range(0, 10)), list(range(5, 15)), list(range(10, 20)), list(range(15, 24))]
    assert hba.layer_windows(7) == [list(range(7))]
    for n in (11, 33, 177):
        w = hba.layer_windows(n)
        assert sorted(set(i for x in w for i in x)) == list(range(n)) and len(w) < n and w[-1][-1] == n - 1


def test_keyframe_at_voxel_size_zero_is_the_transformed_concatenation():
    rng = np.random.default_rng(1)
    scans = [rng.normal(0, 10, (n, 3)).astype(np.float32) for n in (50, 0, 31, 7)]
    window = [2, 0, 1, 3, 0]
    p12 = _rand_poses(rng, len(window))
    got = hba_ref.keyframe_ref(scans, window, p12, 0.0)
    Ra, ta = hba_ref._rt(p12[0])
    want = np.concatenate([((scans[s].astype(np.float64) @ hba_ref._rt(p12[k])[0].T + hba_ref._rt(p12[k])[1]) - ta) @ Ra
                           for k, s in enumerate(window)])
    assert got.dtype == np.float32 and got.shape == (sum(len(scans[s]) for s in window), 3)
    assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()
    assert np.array_equal(hba_ref.keyframe_ref(scans, window, p12, 0.0009), got)  # below 0.001: no reduction
    assert hba_ref.keyframe_ref(scans, [1], p12[:1], 0.5).shape == (0, 3)


def test_keyframe_reduction_is_the_voxel_mean_in_ascending_order():
    rng = np.random.default_rng(2)
    scans = [rng.uniform(-3, 3, (400, 3)).astype(np.float32) for _ in range(3)]
    p12 = _rand_poses(rng, 3)
    full = hba_ref.keyframe_ref(scans, [0, 1, 2], p12, 0.0)
    kf = hba_ref.keyframe_ref(scans, [0, 1, 2], p12, 1.5)
    loc = full / np.float32(1.5)
    key = np.trunc(np.where(loc < 0, loc - np.float32(1), loc)).astype(np.int64)
    uniq, inv = np.unique(key, axis=0, return_inverse=True)
    assert len(kf) == len(uniq) < len(full)
    for v in (0, len(uniq) // 2, len(uniq) - 1):
        assert np.array_equal(kf[v], (full[inv.reshape(-1) == v].astype(np.float64).sum(0) /
                                      np.sum(inv.reshape(-1) == v)).astype(np.float32))


def test_product_propagation_equals_the_matrix_restatement():
    layers = _pyramid(np.random.default_rng(3))
    assert len(layers) == 3 and len(layers[1]["windows"]) == 2 and len(layers[2]["poses_in"]) == 2
    got, ref = hba.propagate(layers), hba_ref.propagate_ref(layers)
    assert got.shape == (60, 12) and np.abs(got - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())


def test_unchanged_upper_layers_keep_the_bottom_relative_poses():
    layers = _pyramid(np.random.default_rng(4))
    for lay in layers[1:]:  # upper layers leave their inputs as they are
        lay["poses"] = [lay["poses_in"][w] for w in lay["windows"]]
    F = hba_ref.propagate_ref(layers)
    bottom = layers[0]
    seen = set()
    for w, win in enumerate(bottom["windows"]):
        own = [(k, i) for k, i in enumerate(win) if i not in seen]
        seen.update(win)
        for (k0, i0), (k1, i1) in zip(own, own[1:]):
            assert np.abs(_rel(F[i0], F[i1]) - _rel(bottom["poses"][w][k0], bottom["poses"][w][k1])).max() < 1e-12
        # and the window's anchor keeps the input pose of its slot 0 (the keyframe's input pose)
        k, i = own[0]
        want = hba_ref._h(bottom["poses_in"][win[0]]) @ _rel(bottom["poses"][w][0], bottom["poses"][w][k])
        assert np.abs(hba_ref._h(F[i]) - want).max() < 1e-12


@pytest.mark.parametrize("layer", [0, 1, 2])
def test_propagation_is_gauge_free(layer):
    rng = np.random.default_rng(5 + layer)
    layers = _pyramid(rng)
    F = hba_ref.propagate_ref(layers)
    for w in range(len(layers[layer]["windows"])):
        G = hba_ref._h(_rand_poses(rng, 1)[0])
        layers[layer]["poses"][w] = np.array([hba_ref._p12(G @ hba_ref._h(p)) for p in layers[layer]["poses"][w]])
    for f in (hba_ref.propagate_ref, hba.propagate):
        assert np.abs(f(layers) - F).max() <= 1e-12 * max(1.0, np.abs(F).max())


def test_drift_scene_drifts():
    scans, gt, init = hba_ref.drift_scene()
    assert len(scans) == 60 and scans[0].dtype == np.float32 and np.array_equal(gt[0], init[0])
    err = np.linalg.norm(gt[:, 9:] - init[:, 9:], axis=1)
    assert err[-10:].mean() > 2 * err[1:11].mean() and err.max() > 0.1  # the error grows along the path

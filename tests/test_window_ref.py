"""tests/window_ref.py::WindowOctree (the restated persistent octree, oracle of balm_window_*) against the flattened
restatements of tests/assoc_ref.py, which tests/test_reference_pin.py holds to the reference's code, and -- where the
reference is built -- against the reference's own octree (oracle/ref_py.Session) through whole sliding-window runs."""
import numpy as np
import pytest

import assoc_ref
import scenes
import window_ref as wr
from oracle import ref_py as ref


def _window(n, seed, lim, mg=2, **extra):
    kw = dict(voxel_size=2.0, layer_limit=lim, min_ps=15, eigen_value_array=(1 / 16, 1 / 16, 1 / 16))
    kw.update(extra)
    pts, frs, poses = assoc_ref.synthetic_scans(n_poses=n + 1, pts_per_scan=3000, seed=seed)
    poses12 = scenes.pack_poses([r for r, _ in poses], [p for _, p in poses])
    w = wr.WindowOctree(n, **kw)
    for i in range(n):
        w.cut_voxel(pts[frs == i], poses12[i], i)
    w.recut(n)
    return w, kw, pts, frs, poses, poses12


@pytest.mark.parametrize("seed,lim", [(31, 2), (32, 2), (31, 0), (33, 0)])
def test_fresh_map_gives_cut_voxels_then_marginalize_ref_then_append_scan_ref(seed, lim):
    n, mg = 8, 2
    w, kw, pts, frs, poses, poses12 = _window(n, seed, lim)
    win = frs < n
    # 1. a fresh map pushes exactly what assoc_ref.cut_voxels computes
    keys, lay, rp, pi, ob, fx, co = w.export(n)
    rp0, pi0, ob0, co0, keys0, lay0 = assoc_ref.cut_voxels(pts[win], frs[win], poses[:n], with_layers=True, **kw)
    assert len(keys) > 20
    assert np.array_equal(keys, keys0) and np.array_equal(lay, lay0)
    assert np.array_equal(rp, rp0) and np.array_equal(pi, pi0) and np.array_equal(co, co0)
    assert np.all(np.abs(ob - ob0) <= 1e-11 * np.abs(ob0).max(axis=0)) and not fx.any()
    # 2. marginalize right after: exactly assoc_ref.marginalize_ref
    rng = np.random.default_rng(seed)
    opt = poses12[:n].copy()
    opt[:, 9:] += rng.normal(0, 0.005, (n, 3))
    w.marginalize(mg, opt, n)
    keys1, lay1, rp1, pi1, ob1, fx1, co1 = w.export(n - mg)
    r_rp, r_pi, r_ob, r_fx, r_co = assoc_ref.marginalize_ref(n, rp, pi, ob, None, opt, mg, kw["min_ps"])
    assert np.array_equal(rp1, r_rp) and np.array_equal(pi1, r_pi) and np.array_equal(co1, r_co)
    assert np.array_equal(ob1, r_ob)
    assert np.abs(fx1 - r_fx).max() <= 1e-12 * np.abs(r_fx).max()
    # 3./4. one new scan at slot n - mg: the window pushes a superset of append_scan_ref, with identical rows on it
    slot = n - mg
    shifted = np.zeros((n, 12))
    shifted[:slot] = opt[mg:]
    shifted[slot] = poses12[n]
    new = pts[frs == n]
    w.cut_voxel(new, shifted[slot], slot)
    w.recut(slot + 1)
    keys2, lay2, rp2, pi2, ob2, fx2, co2 = w.export(slot + 1)
    k, l, a_rp, a_pi, a_ob, a_fx, a_co, matched = assoc_ref.append_scan_ref(
        keys1, lay1, rp1, pi1, ob1, fx1, co1, new, shifted, slot, **kw)
    assert matched > 0.3 * len(new) and (a_pi == slot).sum() > 5
    where = {(int(a), int(b)): i for i, (a, b) in enumerate(zip(keys2, lay2))}
    for a in range(len(k)):
        i = where[(int(k[a]), int(l[a]))]
        assert np.array_equal(pi2[rp2[i]:rp2[i + 1]], a_pi[a_rp[a]:a_rp[a + 1]]) and co2[i] == a_co[a]
        assert np.all(np.abs(ob2[rp2[i]:rp2[i + 1]] - a_ob[a_rp[a]:a_rp[a + 1]]) <= 1e-11 * np.abs(a_ob).max(axis=0))
        assert np.abs(fx2[i] - a_fx[a]).max() <= 1e-12 * max(1.0, np.abs(a_fx[a]).max())
    assert len(where) >= len(k)


@pytest.mark.parametrize("lim", [0, 2])
def test_growth_scans_exercise_new_roots_resplits_and_dormant_leaves(lim):
    pts, frs, noisy, _ = wr.growth_scans(n_scans=20, pts_per_scan=3000, seed=7)
    P = scenes.pack_poses([r for r, _ in noisy], [p for _, p in noisy])
    scans = [pts[frs == i] for i in range(20)]
    for each in (True, False):
        w = wr.WindowOctree(10, voxel_size=2.0, layer_limit=lim, min_ps=15, eigen_value_array=(1 / 16, 1 / 16, 1 / 9))
        pushes = []
        assert wr.run_schedule(wr.window_schedule(20, 10, 2, each), w, scans, P, P, lambda t, e: pushes.append(e)) == 6
        new_roots, resplit, revived = wr.growth_events(pushes)
        assert new_roots > 0 and revived > 0
        assert resplit > 0 if lim == 2 else resplit == 0


# ---------------- pinned to the reference's own octree ----------------
pinned = pytest.mark.skipif(not ref.available(), reason="oracle/_ref/libbalm_ref.so not built (needs the reference sources at build time, BALM_REFERENCE)")


class _Session:
    """ref_py.Session with WindowOctree's method names."""

    def __init__(self, n, kw):
        self.N = n
        self.s = ref.Session(n, kw["voxel_size"], kw["layer_limit"], kw["min_ps"], kw["eigen_value_array"])

    def cut_voxel(self, x, pose12, slot):
        self.s.cut_voxel(np.asarray(x, dtype=np.float32), pose12, slot)

    def recut(self, w):
        self.s.recut(w)

    def marginalize(self, mg, x, w):
        self.s.marginalize(mg, x, w)

    def export(self, w):
        keys, rp, pi, ob, fx, co, lay = self.s.export(w, with_layers=True)
        return keys.astype(np.int64), lay, rp, pi, ob, fx, co


def assert_same_push(a, b):
    keys, lay, rp, pi, ob, fx, co = a
    k2, l2, rp2, pi2, ob2, fx2, co2 = b
    assert np.array_equal(keys, k2) and np.array_equal(lay, l2)
    assert np.array_equal(rp, rp2) and np.array_equal(pi, pi2) and np.array_equal(co, co2)
    if len(ob):
        assert np.all(np.abs(ob - ob2) <= 1e-11 * np.abs(ob2).max(axis=0))
        assert np.abs(fx - fx2).max() <= 1e-12 * max(1.0, np.abs(fx2).max())


@pinned
@pytest.mark.parametrize("lim", [0, 2])
@pytest.mark.parametrize("recut_each_scan", [True, False])
def test_window_octree_matches_the_reference_octree_over_window_shifts(lim, recut_each_scan):
    n_scans, N, mg = 18, 10, 2
    kw = dict(voxel_size=2.0, layer_limit=lim, min_ps=15, eigen_value_array=(1 / 16, 1 / 16, 1 / 9))
    pts, frs, noisy, _ = wr.growth_scans(n_scans=n_scans, pts_per_scan=3000, seed=11)
    P = scenes.pack_poses([r for r, _ in noisy], [p for _, p in noisy])
    X = P.copy()
    X[:, 9:] += np.random.default_rng(4).normal(0, 0.003, (n_scans, 3))
    scans = [pts[frs == i] for i in range(n_scans)]
    ops = wr.window_schedule(n_scans, N, mg, recut_each_scan)
    mine, theirs = [], []
    wr.run_schedule(ops, wr.WindowOctree(N, **kw), scans, P, X, lambda t, e: mine.append(e))
    assert wr.run_schedule(ops, _Session(N, kw), scans, P, X, lambda t, e: theirs.append(e)) >= 4
    for a, b in zip(mine, theirs):
        assert_same_push(a, b)

"""GPU: the persistent sliding-window octree (balm_window_reset / cut / recut / marginalize / push) against its numpy
restatement tests/window_ref.py::WindowOctree over whole window runs, against the reduced sliding-window calls
(balm_cut_voxels / balm_marginalize / balm_append_scan), and the BA that runs on what it pushes."""
import os

import numpy as np
import pytest

import scenes
import window_ref as wr
from oracle import oracle_py as orc

pytestmark = pytest.mark.gpu

N, MG, N_SCANS = 10, 2, 20


class DeviceWindow:
    """balm_b200.Context's window calls with WindowOctree's method names; export() = push + download."""

    def __init__(self, n, **kw):
        import balm_b200
        self.N = n
        self.c = balm_b200.Context(n, 0, 0)
        self.c.window_reset(**kw)

    def cut_voxel(self, x, pose12, slot):
        self.c.window_cut(x, pose12, slot)

    def recut(self, w):
        self.c.window_recut(w)

    def marginalize(self, mg, x, w):
        self.c.window_marginalize(mg, x, w)

    def export(self, w):
        M, K = self.c.window_push(w)
        if M == 0:
            return (np.zeros(0, np.int64), np.zeros(0, np.int32), np.zeros(1, np.int64), np.zeros(0, np.int32),
                    np.zeros((0, 10)), np.zeros((0, 10)), np.zeros(0))
        keys, lay = self.c.download_keys(with_layers=True)
        rp, pi, ob, co = self.c.download_voxels()
        assert len(pi) == K
        return keys.astype(np.int64), lay, rp, pi, ob, self.c.download_fix(), co


def _same(a, b):
    keys, lay, rp, pi, ob, fx, co = a
    k2, l2, rp2, pi2, ob2, fx2, co2 = b
    assert np.array_equal(keys, k2) and np.array_equal(lay, l2)
    assert np.array_equal(rp, rp2) and np.array_equal(pi, pi2) and np.array_equal(co, co2)
    if len(ob2):
        assert np.all(np.abs(ob - ob2) <= 1e-11 * np.abs(ob2).max(axis=0))
        assert np.abs(fx - fx2).max() <= 1e-12 * max(1.0, np.abs(fx2).max())


def _inputs(seed=7, pts=4000):
    pts_, frs, noisy, _ = wr.growth_scans(n_scans=N_SCANS, pts_per_scan=pts, seed=seed)
    P = scenes.pack_poses([r for r, _ in noisy], [p for _, p in noisy])
    X = P.copy()                                  # the poses a window BA would hand to marginalize
    X[:, 9:] += np.random.default_rng(seed).normal(0, 0.003, (N_SCANS, 3))
    return [pts_[frs == i] for i in range(N_SCANS)], P, X


KW = dict(voxel_size=2.0, min_ps=15, eigen_value_array=(1 / 16, 1 / 16, 1 / 9))


@pytest.mark.parametrize("lim", [0, 2])
@pytest.mark.parametrize("recut_each_scan", [True, False])
def test_device_window_matches_the_restatement_at_every_push(lim, recut_each_scan):
    scans, P, X = _inputs()
    ops = wr.window_schedule(N_SCANS, N, MG, recut_each_scan)
    dev, ref = [], []
    n = wr.run_schedule(ops, DeviceWindow(N, layer_limit=lim, **KW), scans, P, X, lambda t, e: dev.append(e))
    wr.run_schedule(ops, wr.WindowOctree(N, layer_limit=lim, **KW), scans, P, X, lambda t, e: ref.append(e))
    assert n >= 5                                 # the first push and at least 4 shifts
    for a, b in zip(dev, ref):
        _same(a, b)
    new_roots, resplit, revived = wr.growth_events(dev)
    assert new_roots > 0 and revived > 0          # roots grown from new points; a dormant leaf back with its fix cluster
    assert resplit > 0 if lim == 2 else resplit == 0


def test_window_keeps_what_the_reduced_calls_keep_and_more():
    """The same stream through balm_cut_voxels + balm_marginalize + balm_append_scan (the flattened voxel set): at the first
    shift every voxel that path keeps is pushed by the window with identical rows and fix cluster; after the last shift the
    window holds at least as many voxels (it grows new roots and leaves, re-splits and revives). Then the BA of the full
    window (hess_includes_fix) on the pushed set against the CPU oracle on the downloaded set."""
    import balm_b200
    scans, P, X = _inputs(seed=9)
    kw = dict(layer_limit=2, **KW)
    win = DeviceWindow(N, **kw)
    red = balm_b200.Context(N, 0, 0)
    for s in range(N):
        win.cut_voxel(scans[s], P[s], s)
        win.recut(s + 1)
    win.export(N)
    pts = np.concatenate(scans[:N]).astype(np.float32)
    frs = np.concatenate([np.full(len(scans[s]), s, np.int32) for s in range(N)])
    red.cut_voxels(pts, frs, P[:N], **kw)
    first, nxt = 0, N
    while nxt + MG <= N_SCANS:
        x = X[first:first + N]
        win.marginalize(MG, x, N)
        red.marginalize(MG, x, min_ps=kw["min_ps"])
        first += MG
        shifted = np.vstack([X[first:first + N - MG], P[nxt:nxt + MG]])
        for j in range(MG):
            slot = N - MG + j
            win.cut_voxel(scans[nxt + j], P[nxt + j], slot)
            win.recut(slot + 1)
            red.append_scan(scans[nxt + j].astype(np.float32), shifted, slot)
        nxt += MG
        keys, lay, rp, pi, ob, fx, co = win.export(N)
        if first == MG:                           # the first shift: the reduced set is contained in the window's push
            rk, rl = red.download_keys(with_layers=True)
            rrp, rpi, rob, rco = red.download_voxels()
            rfx = red.download_fix()
            where = {(int(a), int(b)): i for i, (a, b) in enumerate(zip(keys, lay))}
            for v in range(len(rk)):
                i = where[(int(rk[v]), int(rl[v]))]
                assert np.array_equal(pi[rp[i]:rp[i + 1]], rpi[rrp[v]:rrp[v + 1]]) and co[i] == rco[v]
                assert np.all(np.abs(ob[rp[i]:rp[i + 1]] - rob[rrp[v]:rrp[v + 1]]) <= 1e-11 * np.abs(rob).max(axis=0))
                assert np.abs(fx[i] - rfx[v]).max() <= 1e-12 * max(1.0, np.abs(rfx[v]).max())
            assert len(rk) > 50
    assert len(keys) >= red.M, (len(keys), red.M)
    # BA on the full window: the pushed set with its fix clusters, against the oracle on the same (downloaded) set
    shifted = np.vstack([X[first:first + N - MG], P[nxt - MG:nxt]])
    p_dev, tr_dev, _ = win.c.damping_iter(shifted, gauge_mode=2, min_planes_per_pose=0, hess_includes_fix=True)
    assert fx[:, 9].max() > 0
    o = orc.Oracle(N, rp, pi, ob, co, fx)
    st, p_ora, tr_ora, _ = o.damping_iter(shifted, gauge_mode=2, min_planes_per_pose=0, hess_includes_fix=True)
    assert [t["accepted"] for t in tr_dev] == [t["accepted"] for t in tr_ora]
    assert np.abs(p_dev - p_ora).max() <= 1e-6


def test_rejected_window_calls_change_nothing():
    import balm_b200
    scans, P, X = _inputs(seed=5, pts=2000)
    c = balm_b200.Context(N, 0, 0)
    with pytest.raises(balm_b200.BalmError) as e:     # no balm_window_reset yet
        c.window_cut(scans[0], P[0], 0)
    assert e.value.status == 1
    with pytest.raises(balm_b200.BalmError) as e:
        c.window_recut(1)
    assert e.value.status == 1
    dev = DeviceWindow.__new__(DeviceWindow)
    dev.N, dev.c = N, c
    c.window_reset(layer_limit=2, **KW)
    ref = wr.WindowOctree(N, layer_limit=2, **KW)
    bad = [lambda: c.window_cut(scans[0], P[0], -1), lambda: c.window_cut(scans[0], P[0], N),
           lambda: c.window_recut(0), lambda: c.window_recut(N + 1), lambda: c.window_marginalize(0, X[:N], 4),
           lambda: c.window_marginalize(4, X[:N], 4), lambda: c.window_marginalize(1, X[:N], N + 1),
           lambda: c.window_push(0), lambda: c.window_push(N + 1)]
    for s in range(4):
        for impl in (dev, ref):
            impl.cut_voxel(scans[s], P[s], s)
            impl.recut(s + 1)
        for f in bad:
            with pytest.raises(balm_b200.BalmError) as e:
                f()
            assert e.value.status == 1
    _same(dev.export(4), ref.export(4))
    for impl in (dev, ref):
        impl.marginalize(2, X[:N], 4)
        impl.cut_voxel(scans[4], P[4], 2)
        impl.recut(3)
    _same(dev.export(3), ref.export(3))


REALWORLD = None
try:
    from oracle import ref_py as _ref
    REALWORLD = os.path.join(_ref.REFERENCE_DIR, "datas", "benchmark_realworld")
except Exception:  # pragma: no cover
    pass


@pytest.mark.skipif(REALWORLD is None or not os.path.exists(os.path.join(REALWORLD, "alidarPose.csv")),
                    reason="the reference's dataset is not in the reference sources directory (BALM_REFERENCE)")
def test_device_window_on_the_reference_dataset():
    """The first 30 scans of datas/benchmark_realworld (every 4th point, re-anchored to pose 0, the constants of
    benchmark_realworld.cpp:163-185), window 10, mg 2, one recut per scan: identical pushes on the device and in the
    restatement."""
    from balm_b200 import io
    n = 30
    R, p, t, raw = io.read_realworld_dir(REALWORLD, max_scans=n)
    R0, p0 = R[0].copy(), p[0].copy()
    P = scenes.pack_poses([R0.T @ R[i] for i in range(n)], [R0.T @ (p[i] - p0) for i in range(n)])
    scans = [sc[::4].astype(np.float32).astype(np.float64) for sc in raw]
    kw = dict(voxel_size=2.0, layer_limit=2, min_ps=15, eigen_value_array=(1 / 16, 1 / 16, 1 / 9))
    ops = wr.window_schedule(n, N, MG, True)
    dev, ref = [], []
    wr.run_schedule(ops, DeviceWindow(N, **kw), scans, P, P, lambda t, e: dev.append(e))
    wr.run_schedule(ops, wr.WindowOctree(N, **kw), scans, P, P, lambda t, e: ref.append(e))
    assert len(dev) == len(ref) >= 10 and len(ref[0][0]) > 100
    for a, b in zip(dev, ref):
        _same(a, b)

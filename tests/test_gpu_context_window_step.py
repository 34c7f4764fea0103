"""GPU: the contracts of a context's reduced sliding-window step (balm_marginalize / balm_append_scan, the one-problem case
of the batch's builds) that the restatement tests do not reach: a rejected call leaves the context as it was, keyless and
fix-less registrations stay so, registrations pushed by the persistent window, and a scan of a million points."""
import numpy as np
import pytest

from balm_b200 import _lib

import assoc_ref
import scenes
import window_ref as wr

pytestmark = pytest.mark.gpu

# the context's association options when no balm_cut_voxels set them (what balm_append_scan judges a pushed set with)
CTX_KW = dict(voxel_size=1.0, layer_limit=2, min_ps=15, eigen_value_array=(1 / 16, 1 / 16, 1 / 16))


def _snapshot(c, poses):
    import balm_b200
    snap = list(c.download_voxels()) + [c.download_fix(), *c.evaluate(poses, include_fix=True)]
    try:
        snap += list(c.download_keys(with_layers=True))
    except balm_b200.BalmError:
        snap.append("no keys")
    return snap


def _assert_same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def _patch_scan(rng, n=300):
    """n body-frame points of one plane patch (z = 0.5) inside the root voxel [0, 1)^3"""
    return np.stack([rng.uniform(0.1, 0.9, n), rng.uniform(0.1, 0.9, n), 0.5 + rng.normal(0, 1e-3, n)], axis=1)


def test_rejected_calls_leave_the_context_as_it_was():
    """One plane voxel seen by three scans at identity poses, the oldest retired into its fix cluster: every rejection
    (marginalising it away, a slot not above the voxel's scans, a re-judgement nothing survives, and both of the last
    two at once, where the slot is reported) returns BALM_ERR_INVALID and leaves registration, fix clusters, keys,
    layers and evaluation bitwise unchanged; the context still takes the next valid call."""
    import balm_b200
    N = 4
    rng = np.random.default_rng(3)
    eye = scenes.pack_poses([np.eye(3)] * N, [np.zeros(3)] * N)
    c = balm_b200.Context(N, 0, 0)
    c.cut_voxels(np.concatenate([_patch_scan(rng) for _ in range(3)]).astype(np.float32),
                 np.repeat(np.arange(3, dtype=np.int32), 300), eye, **CTX_KW)
    assert c.marginalize(1, eye) == (1, 2)
    fix = c.download_fix()
    assert fix[0, 9] == 300 and c.download_keys()[0] & 63 == 63    # a layer-0 leaf with keys and its fix cluster
    # slot 1 turned by 90 degrees about the voxel's x axis: the clusters cross, nothing is planar any more
    R = scenes.exp_so3(np.array([np.pi / 2, 0.0, 0.0]))
    ctr = np.full(3, 0.5)
    crossed = eye.copy()
    crossed[1] = scenes.pack_poses([R], [ctr - R @ ctr])[0]
    new = _patch_scan(rng).astype(np.float32)
    before = _snapshot(c, eye)
    for call, msg in [(lambda: c.marginalize(1, eye, min_ps=10 ** 6), "balm_marginalize: no voxel is left"),
                      (lambda: c.append_scan(new, eye, 1), "`slot` must be above every scan"),
                      (lambda: c.append_scan(new, crossed, 2), "balm_append_scan: no plane voxel survives"),
                      (lambda: c.append_scan(new, crossed, 0), "`slot` must be above every scan")]:
        with pytest.raises(balm_b200.BalmError) as e:
            call()
        assert e.value.status == _lib.ERR_INVALID and msg in str(e.value) and "problem" not in str(e.value)
        _assert_same(_snapshot(c, eye), before)
    assert c.append_scan(new, eye, 2) == (1, 3, 300)
    assert np.array_equal(c.download_fix(), fix)
    c.close()


@pytest.mark.parametrize("with_fix", [False, True])
def test_marginalizing_a_keyless_registration_gives_one_without_keys(with_fix):
    import balm_b200
    N, mg = 9, 2
    sc = scenes.make_scene(n_poses=N, n_planes=120, seed=41, drop=0.4, with_fix=with_fix, pts_size=9)
    c = balm_b200.Context(N, 0, 0)
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc["fix10"])
    M, K = c.marginalize(mg, sc["poses_init"])
    rp, pi, ob, fx, co = assoc_ref.marginalize_ref(N, sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["fix10"],
                                                   sc["poses_init"], mg, 15)
    rp_g, pi_g, ob_g, co_g = c.download_voxels()
    assert (M, K) == (len(co), len(pi))
    assert np.array_equal(rp_g, rp) and np.array_equal(pi_g, pi) and np.array_equal(ob_g, ob) and np.array_equal(co_g, co)
    assert np.abs(c.download_fix() - fx).max() <= 1e-12 * np.abs(fx).max()
    with pytest.raises(balm_b200.BalmError):
        c.download_keys()
    c.close()


def test_a_million_point_scan_on_a_registration_without_fix_clusters():
    """balm_append_scan of a 1.2 M point scan against assoc_ref.append_scan_ref; the cut registration has no fix
    clusters and keeps none (they download as zeros)."""
    import balm_b200
    N = 8
    pts, frs, poses = assoc_ref.synthetic_scans(n_poses=N, pts_per_scan=3000, seed=21)
    P = scenes.pack_poses([r for r, _ in poses], [p for _, p in poses])
    kw = dict(voxel_size=2.0, layer_limit=2, min_ps=15, eigen_value_array=(1 / 16, 1 / 16, 1 / 9))
    win = frs < N - 1
    c = balm_b200.Context(N, 0, 0)
    c.cut_voxels(pts[win].astype(np.float32), frs[win], P, **kw)
    rp, pi, ob, co, keys, lays = assoc_ref.cut_voxels(pts[win], frs[win], poses[:N - 1], with_layers=True, **kw)
    rng = np.random.default_rng(5)
    last = pts[frs == N - 1]
    big = np.concatenate([last + rng.normal(0, 0.003, last.shape) for _ in range(400)]).astype(np.float32)
    M, K, matched = c.append_scan(big, P, N - 1)
    k1, l1, rp1, pi1, ob1, fx1, co1, matched_ref = assoc_ref.append_scan_ref(
        keys, lays, rp, pi, ob, None, co, big.astype(np.float64), P, N - 1, **kw)
    assert len(big) >= 1_000_000 and matched == matched_ref and matched > len(big) // 2
    assert (M, K) == (len(co1), len(pi1))
    kg, lg = c.download_keys(with_layers=True)
    assert np.array_equal(kg.astype(np.int64), k1) and np.array_equal(lg, l1)
    rp_g, pi_g, ob_g, co_g = c.download_voxels()
    assert np.array_equal(rp_g, rp1) and np.array_equal(pi_g, pi1) and np.array_equal(co_g, co1)
    assert np.all(np.abs(ob_g - ob1) <= 1e-11 * np.abs(ob1).max(axis=0))
    assert not c.download_fix().any()
    c.close()


def test_marginalize_and_append_on_a_window_push():
    """A registration pushed by the persistent window (keys, layers and fix clusters) marginalised and appended to by the
    reduced calls, against the restatements."""
    import balm_b200
    N, mg = 10, 2
    pts_, frs, noisy, _ = wr.growth_scans(n_scans=N + 1, pts_per_scan=4000, seed=7)
    P = scenes.pack_poses([r for r, _ in noisy], [p for _, p in noisy])
    scans = [pts_[frs == i] for i in range(N + 1)]
    c = balm_b200.Context(N, 0, 0)
    c.window_reset(**CTX_KW)
    for s in range(N):
        c.window_cut(scans[s], P[s], s)
        c.window_recut(s + 1)
    c.window_push(N)
    keys, lays = c.download_keys(with_layers=True)
    rp, pi, ob, co = c.download_voxels()
    fix = c.download_fix()
    M1, K1 = c.marginalize(mg, P[:N])
    rp1, pi1, ob1, fx1, co1 = assoc_ref.marginalize_ref(N, rp, pi, ob, fix, P[:N], mg, 15)
    keep = np.array([((pi[rp[a]:rp[a + 1]] >= mg).sum() >= 2 and
                      int(ob[rp[a]:rp[a + 1]][pi[rp[a]:rp[a + 1]] >= mg, 9].sum()) >= 15) for a in range(len(co))])
    kg, lg = c.download_keys(with_layers=True)
    assert np.array_equal(kg, keys[keep]) and np.array_equal(lg, lays[keep])
    rp_g, pi_g, ob_g, co_g = c.download_voxels()
    assert (M1, K1) == (len(co1), len(pi1)) and M1 > 0
    assert np.array_equal(rp_g, rp1) and np.array_equal(pi_g, pi1) and np.array_equal(ob_g, ob1)
    assert np.array_equal(co_g, co1)
    assert np.abs(c.download_fix() - fx1).max() <= 1e-12 * np.abs(fx1).max()
    shifted = np.vstack([P[mg:N], P[N:N + 1], P[N:N + 1]])
    slot = N - mg
    M2, K2, matched = c.append_scan(scans[N].astype(np.float32), shifted, slot)
    k2, l2, rp2, pi2, ob2, fx2, co2, matched_ref = assoc_ref.append_scan_ref(
        keys[keep].astype(np.int64), lays[keep], rp1, pi1, ob1, fx1, co1, scans[N].astype(np.float32).astype(np.float64),
        shifted, slot, **CTX_KW)
    assert matched == matched_ref > 0 and (M2, K2) == (len(co2), len(pi2))
    kg, lg = c.download_keys(with_layers=True)
    assert np.array_equal(kg.astype(np.int64), k2) and np.array_equal(lg, l2)
    rp_g, pi_g, ob_g, co_g = c.download_voxels()
    assert np.array_equal(rp_g, rp2) and np.array_equal(pi_g, pi2) and np.array_equal(co_g, co2)
    assert np.all(np.abs(ob_g - ob2) <= 1e-11 * np.abs(ob2).max(axis=0))
    assert np.abs(c.download_fix() - fx2).max() <= 1e-12 * np.abs(fx2).max()
    c.close()

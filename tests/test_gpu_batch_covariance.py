"""Batched pose covariance (balm_batch_pose_covariance, balm_b200.Batch.pose_covariance): every problem of a batch
checked against the numpy restatement of left_jacobian_point / multi_second / H^-1 Rcov H^-T (tests/numpy_cov.py) and
against a fp64 Context holding only that problem. Tolerances are those of tests/test_gpu_covariance.py: Rcov_raw 1e-9,
Rcov 1e-7 relative to the largest entry."""
import numpy as np
import pytest

import numpy_cov as nc
import scenes
from oracle import oracle_py as orc

pytestmark = pytest.mark.gpu

PN = 0.01
IDENT = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0.0])

# N_p = 1, 2, 9, 20 (ragged), 32 (n = 192, the largest problem a batch takes), all with fix clusters; the one-pose
# problem is pose 0 of a two-pose scene (make_scene gives every voxel at least two observations)
SCENES = [
    dict(n_poses=2, n_planes=25, seed=41, keep_pose0=True),
    dict(n_poses=2, n_planes=30, seed=42),
    dict(n_poses=9, n_planes=40, seed=43),
    dict(n_poses=20, n_planes=80, seed=44, drop=0.4),
    dict(n_poses=32, n_planes=60, seed=45),
]


def _scene(kw):
    kw = dict(kw)
    if not kw.pop("keep_pose0", False):
        return scenes.make_scene(pts_size=20, with_fix=True, **kw)
    sc = scenes.make_scene(pts_size=20, with_fix=True, **kw)
    keep = sc["pose_idx"] == 0
    counts = np.add.reduceat(keep.astype(np.int64), sc["row_ptr"][:-1])
    return dict(sc, n_poses=1, row_ptr=np.concatenate([[0], np.cumsum(counts)]).astype(np.int64),
                pose_idx=sc["pose_idx"][keep], obs10=sc["obs10"][keep], poses_gt=sc["poses_gt"][:1],
                poses_init=sc["poses_init"][:1])


def _prob(sc, fix=True):
    return dict(n_poses=sc["n_poses"], row_ptr=sc["row_ptr"], pose_idx=sc["pose_idx"], obs10=sc["obs10"],
                coe=sc["coe"], fix10=sc["fix10"] if fix else None)


def _empty(n_poses):
    return dict(n_poses=n_poses, row_ptr=np.zeros(1, dtype=np.int64), pose_idx=np.zeros(0, dtype=np.int32),
                obs10=np.zeros((0, 10)), coe=np.zeros(0), fix10=None)


def _batch(problems):
    import balm_b200
    b = balm_b200.Batch(0)
    b.set_problems(problems)
    return b


@pytest.fixture(scope="module")
def optimised():
    """The scenes, one batch of them, and every problem's poses after the batched LM (the covariance is taken there)."""
    scs = [_scene(kw) for kw in SCENES]
    b = _batch([_prob(s) for s in scs])
    res = b.damping_iter([s["poses_init"] for s in scs], hess_includes_fix=True, gauge_mode=2)
    assert all(r[0] == 0 for r in res)
    poses = [r[1] for r in res]
    out = b.pose_covariance(poses, point_noise=PN, include_fix=True)
    b.close()
    return scs, poses, out


def _oracle_raw(sc, poses, fix=True):
    return nc.left_jacobian_point(sc["n_poses"], sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], poses,
                                  sc["fix10"] if fix else None, pnoise=PN)


def test_matches_reference_restatement_per_problem(optimised):
    scs, poses, out = optimised
    for sc, x, (st, raw, cov) in zip(scs, poses, out):
        n = 6 * sc["n_poses"]
        assert st == 0 and raw.shape == (n, n) and cov.shape == (n, n)
        ref = _oracle_raw(sc, x)
        assert np.abs(raw - ref).max() <= 1e-9 * np.abs(ref).max(), sc["n_poses"]
        assert np.array_equal(raw, raw.T)
        o = orc.Oracle(sc["n_poses"], sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc["fix10"])
        ref_cov = nc.pose_covariance(o.evaluate(x, include_fix=True)[0], ref)
        assert np.abs(cov - ref_cov).max() <= 1e-7 * np.abs(ref_cov).max(), sc["n_poses"]
        assert np.array_equal(cov, cov.T)
        assert np.linalg.eigvalsh(cov).min() >= -1e-9 * np.abs(cov).max()


def test_agrees_with_context_fp64(optimised):
    import balm_b200
    scs, poses, out = optimised
    for sc, x, (st, raw, cov) in zip(scs, poses, out):
        c = balm_b200.Context(sc["n_poses"], 0, balm_b200.PREC_FP64)
        c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc["fix10"])
        raw_c, cov_c = c.pose_covariance(x, point_noise=PN, include_fix=True)
        c.close()
        assert np.abs(raw - raw_c).max() <= 1e-11 * np.abs(raw_c).max(), sc["n_poses"]
        assert np.abs(cov - cov_c).max() <= 1e-9 * np.abs(cov_c).max(), sc["n_poses"]


def test_explicit_cluster_covariances(optimised):
    scs, poses, out = optimised
    b = _batch([_prob(s) for s in scs])
    cc = [np.stack([nc.cluster_cov_isotropic(o10, PN) for o10 in s["obs10"]]) for s in scs]
    got = b.pose_covariance(poses, c_cov=cc, include_fix=True, want_cov=False)
    b.close()
    for (st, raw2, cov2), (_, raw, _) in zip(got, out):
        assert st == 0 and cov2 is None
        assert np.abs(raw2 - raw).max() <= 1e-12 * np.abs(raw).max()


def test_problem_results_do_not_depend_on_the_batch(optimised):
    scs, poses, _ = optimised
    X, Y, Z = 3, 4, 1  # N_p = 20, 32, 2

    def run(order, at):
        b = _batch([_prob(scs[i]) for i in order])
        r = b.pose_covariance([poses[i] for i in order], point_noise=PN, include_fix=True)
        b.close()
        return r[at]

    alone = run([X], 0)
    for order, at in (([X, Y, Z], 0), ([Y, Z, X], 2), ([Z, X], 1), ([Y, X, Y], 1)):
        st, raw, cov = run(order, at)
        assert st == alone[0] and np.array_equal(raw, alone[1]) and np.array_equal(cov, alone[2])
    b = _batch([_prob(scs[i]) for i in (X, Y, Z)])
    r1 = b.pose_covariance([poses[i] for i in (X, Y, Z)], point_noise=PN, include_fix=True)
    r2 = b.pose_covariance([poses[i] for i in (X, Y, Z)], point_noise=PN, include_fix=True)
    b.close()
    for a, c in zip(r1, r2):
        assert a[0] == c[0] and np.array_equal(a[1], c[1]) and np.array_equal(a[2], c[2])


def test_singular_problems_are_refused_per_problem(optimised):
    import balm_b200
    from balm_b200 import _lib
    scs, poses, out = optimised
    A, F = 2, 3  # anchored N_p = 9; N_p = 20 registered without its fix clusters
    probs = [_prob(scs[A]), _prob(scs[F], fix=False), _empty(3), _prob(scs[4])]
    x = [poses[A], poses[F], np.tile(IDENT, (3, 1)), poses[4]]
    b = _batch(probs)
    got = b.pose_covariance(x, point_noise=PN, include_fix=True)
    assert [g[0] for g in got] == [_lib.OK, _lib.ERR_NOT_PD, _lib.ERR_NOT_PD, _lib.OK]
    for i, j in ((0, A), (3, 4)):  # the anchored problems are bitwise what they are in a batch of anchored ones
        alone = _batch([_prob(scs[j])]).pose_covariance([poses[j]], point_noise=PN, include_fix=True)[0]
        assert np.array_equal(got[i][1], alone[1]) and np.array_equal(got[i][2], alone[2])
    st, raw, cov = got[1]
    assert not cov.any()
    ref = _oracle_raw(scs[F], poses[F], fix=False)  # Rcov_raw is still valid
    assert np.abs(raw - ref).max() <= 1e-9 * np.abs(ref).max()
    st, raw, cov = got[2]
    assert raw.shape == (18, 18) and not raw.any() and not cov.any()
    # without the fix clusters in H every problem is free: all refused, Rcov zero
    free = b.pose_covariance(x, point_noise=PN, include_fix=False)
    assert all(g[0] == _lib.ERR_NOT_PD and not g[2].any() for g in free)
    b.close()
    # the context agrees on every problem that has voxels
    for (st, _, _), p, xp in zip(got, probs, x):
        if len(p["row_ptr"]) == 1:
            continue
        c = balm_b200.Context(p["n_poses"], 0, balm_b200.PREC_FP64)
        c.set_voxels(p["row_ptr"], p["pose_idx"], p["obs10"], p["coe"], p["fix10"])
        try:
            c.pose_covariance(xp, point_noise=PN, include_fix=True)
            st_c = _lib.OK
        except balm_b200.BalmError as e:
            st_c = e.status
        c.close()
        assert st_c == st


def test_rejections_raw_only_and_cut_scans(optimised):
    import assoc_ref
    import balm_b200
    from balm_b200 import _lib
    from balm_b200.context import _p
    scs, poses, out = optimised
    b = balm_b200.Batch(0)  # nothing registered
    x = np.tile(IDENT, (2, 1))
    assert _lib.lib().balm_batch_pose_covariance(b._h, _p(x), None, PN, 1, None, None, None) == _lib.ERR_INVALID
    # want_cov=False: no H is factored, every status is OK, also for a free problem
    b.set_problems([_prob(scs[2]), _prob(scs[3], fix=False)])
    got = b.pose_covariance([poses[2], poses[3]], point_noise=PN, include_fix=True, want_cov=False)
    assert [g[0] for g in got] == [_lib.OK, _lib.OK] and all(g[2] is None for g in got)
    assert np.array_equal(got[0][1], out[2][1])
    with pytest.raises(ValueError):
        b.pose_covariance([poses[2], poses[3]], c_cov=[np.zeros((3, 9, 9)), np.zeros((2, 9, 9))])
    # windows associated on the device (no fix clusters: H is singular, Rcov_raw is valid)
    pts, frs, sp = assoc_ref.synthetic_scans(n_poses=8, pts_per_scan=2500, seed=9)
    scans = [pts[frs == i] for i in range(8)]
    p12 = scenes.pack_poses([r for r, _ in sp], [p for _, p in sp])
    windows = [[0, 1, 2, 3], [2, 3, 4, 5, 6, 7]]
    wposes = [p12[w] for w in windows]
    mk = b.cut_scans(scans, windows, wposes)
    assert all(m > 0 for m, _ in mk)
    got = b.pose_covariance(wposes, point_noise=PN, include_fix=True)
    for d, xw, (st, raw, cov) in zip(b.download_voxels(), wposes, got):
        assert st == _lib.ERR_NOT_PD and not cov.any()
        ref = nc.left_jacobian_point(d["n_poses"], d["row_ptr"], d["pose_idx"], d["obs10"], d["coe"], xw, pnoise=PN)
        assert np.abs(raw - ref).max() <= 1e-9 * np.abs(ref).max()
    b.close()

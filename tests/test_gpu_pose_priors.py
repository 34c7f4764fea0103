"""Absolute pose priors on the device (balm_set_pose_priors, balm_spg_set_pose_priors, balm_prior_residuals): evaluation
and LM parity with tests/pose_priors_ref.py on the dense pose graph, PoseGraph and a PREC_BLOCKS context, bitwise
decompositions, a GNSS corridor with and without outliers, covariances with anchor = -1, refusals, lifetime, the
sparse pattern's growth, the gauge rule, detach, and HBA's pose graph in the priors' frame."""
import numpy as np
import pytest

import balm_b200
import block_hessian_ref as bref
import pose_graph_ref as pgr
import pose_priors_ref as ppr
import robust_factors_ref as rr
from balm_b200 import _lib as L
from test_gpu_block_hessian import _ctx
from test_gpu_sparse_covariance import _dense_sigma

pytestmark = pytest.mark.gpu

LOSSES = [("trivial", None), ("huber", 0.8), ("cauchy", 0.5)]


def _graph(seed=0, P=24):
    """HBA-shaped window factors over P poses at perturbed poses, and priors of every type, two of them on pose 3"""
    rng = np.random.default_rng(seed)
    gt = np.array([pgr.random_pose(rng, 0.3, 20.0) for _ in range(P)])
    factors = [pgr.make_factor(rng, gt, w, noise=0.01, cond=50.0) for w in pgr.pyramid_factor_poses(P, 6, 3, 8)]
    x = pgr.perturb(rng, gt, 0.01, 0.1)
    priors = ppr.random_priors(rng, gt, [3, 3, 7, 11, 12, 20])
    return gt, factors, x, priors


def _loss_args(n, kind, scale):
    k, s = rr.loss_arrays(n, kind, scale)
    return dict(pk=k, ps=s)


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(b).max(), 1e-300)


def _spg_dense(spg, x, N):
    pairs, blocks, g, cost = spg.pose_graph_evaluate(x)
    H = np.zeros((6 * N, 6 * N))
    for (i, j), B in zip(pairs, blocks):
        H[6 * i:6 * i + 6, 6 * j:6 * j + 6] = B
        H[6 * j:6 * j + 6, 6 * i:6 * i + 6] = B.T
    return H, g, cost, pairs, blocks


@pytest.mark.parametrize("kind,scale", LOSSES)
def test_pose_graph_evaluation_against_the_restatement(kind, scale):
    """dense context and PoseGraph against pose_priors_ref (1e-12), spg blocks bitwise the dense entries, residuals"""
    gt, factors, x, priors = _graph(1)
    N = len(gt)
    la = _loss_args(len(priors), kind, scale)
    Hr, gr, cr = ppr.evaluate(x, factors, priors, N, **la)
    c, s = balm_b200.Context(N), balm_b200.PoseGraph(N)
    for h in (c, s):
        assert h.set_pose_factors(factors) == [0] * len(factors)
        assert h.set_pose_priors(priors, kind=kind, scale=scale) == [0] * len(priors)
    H, g, cost = c.pose_graph_evaluate(x)
    assert _rel(H, Hr) <= 1e-12 and _rel(g, gr) <= 1e-12 and abs(cost - cr) <= 1e-12 * abs(cr)
    assert np.array_equal(H, H.T)
    Hs, gs, cs, pairs, blocks = _spg_dense(s, x, N)
    assert np.array_equal(blocks, np.array([H[6 * i:6 * i + 6, 6 * j:6 * j + 6] for i, j in pairs]))
    assert np.array_equal(gs, g) and cs == cost
    sr, wr = ppr.residuals(x, priors, **la)
    for h in (c, s):
        sd, wd = h.prior_residuals(x)
        assert _rel(sd, sr) <= 1e-12 and _rel(wd, wr) <= 1e-12
    c.close()
    s.close()


@pytest.mark.parametrize("spg", [False, True])
def test_pose_graph_lm_parity(spg):
    gt, factors, x, priors = _graph(2)
    N = len(gt)
    h = balm_b200.PoseGraph(N) if spg else balm_b200.Context(N)
    h.set_pose_factors(factors)
    h.set_pose_priors(priors)
    xd, td = h.pose_graph_iter(x, max_iter=8, gauge_mode=2, want_per_iter=True)
    xr, tr, per = ppr.lm(x, factors, priors, N, max_iter=8)
    assert [t["accepted"] for t in td] == [t["accepted"] for t in tr]
    for t, p in zip(td, per):
        assert np.abs(t["poses"] - p).max() <= 1e-9
    assert np.abs(xd - xr).max() <= 1e-9
    h.close()


def _corridor(N=1000, seed=5, every=10, lever=(0.4, -0.3, 1.5), sigma_g=0.05, outliers=()):
    """bref.corridor with odometry factors and GNSS position priors (lever arm) every `every` poses, the start drifted
    by a rigid offset; outliers: prior indices moved by 10 m"""
    sc = bref.corridor(N, w=4, planes_per_pose=30, seed=seed)
    rng = np.random.default_rng(seed)
    gt = sc["poses_gt"]
    odo = rr.noisy_relative(rng, gt, [(a, a + 1) for a in range(N - 1)], rr.info(*rr.ODO_NOISE), *rr.ODO_NOISE)
    idx = np.arange(0, N, every)
    pos = np.array([pgr.split(gt[i])[0] @ np.asarray(lever) + gt[i, 9:] for i in idx])
    pos += rng.normal(0, sigma_g, pos.shape)
    for q in outliers:
        pos[q] += np.array([10.0, -6.0, 0.0]) * 10.0 / np.linalg.norm([10.0, -6.0, 0.0])
    priors = balm_b200.position_priors(idx, pos, 2 * rr.POINT_NOISE ** 2 / sigma_g ** 2 * np.eye(3), lever_arm=lever)
    off = pgr.pack(pgr.exp_so3([0.0, 0.0, 0.02]), [3.0, -2.0, 0.5])
    x0 = np.array([pgr.compose(off, p) for p in sc["poses_init"]])
    return sc, odo, priors, x0


def _blocks_ctx(sc, odo, priors, kind="trivial", scale=None):
    c = _ctx(sc, L.PREC_BLOCKS)
    c.set_block_factors(odo)
    if priors:
        c.set_pose_priors(priors, kind=kind, scale=scale)
    return c


def test_blocks_evaluation_decomposition_and_repeatability():
    """blocks = voxel + factor + prior: the prior part against the restatement, two runs bitwise, sub-ranges voxels only"""
    sc, odo, priors, x0 = _corridor(N=120, every=7)
    priors = priors + ppr.random_priors(np.random.default_rng(1), sc["poses_gt"], [5, 5, 40])
    c0, c1 = _blocks_ctx(sc, odo, []), _blocks_ctx(sc, odo, priors)
    H0, g0, r0 = c0.evaluate(x0)
    H1, g1, r1 = c1.evaluate(x0)
    b1 = c1.download_blocks()
    Hp, gp, cp = ppr.evaluate(x0, [], priors, sc["n_poses"])
    assert np.abs((H1 - H0) - Hp).max() <= 1e-12 * np.abs(H1).max()
    assert np.abs((g1 - g0) - gp).max() <= 1e-12 * np.abs(g1).max()
    assert abs((r1 - r0) - cp) <= 1e-12 * abs(r1)
    assert c1.residual(x0) == r1
    H2, g2, r2 = c1.evaluate(x0)
    assert np.array_equal(H1, H2) and np.array_equal(g1, g2) and r1 == r2
    assert np.array_equal(b1, c1.download_blocks())
    assert c0.block_structure()["pairs"] == c1.block_structure()["pairs"]
    Hs0, _, _ = c0.evaluate(x0, 0, 10)
    Hs1, _, _ = c1.evaluate(x0, 0, 10)
    assert np.array_equal(Hs0, Hs1)
    c0.close()
    c1.close()


def test_blocks_lm_parity_with_the_restatement():
    """a blocks corridor with odometry and priors: its LM against voxels (FP64 context) + pose_priors_ref per iteration"""
    sc, odo, priors, x0 = _corridor(N=60, every=6)
    cb = _blocks_ctx(sc, odo, priors)
    cv = _ctx(sc, L.PREC_FP64)
    N = sc["n_poses"]

    def evaluate(x):
        H, g, r = cv.evaluate(x)
        Hf, gf, rf = ppr.evaluate(x, odo, priors, N)
        return H + Hf, g + gf, r + rf

    xd, td, per = cb.damping_iter(x0, max_iter=6, gauge_mode=2, min_planes_per_pose=0, want_per_iter=True)
    x, u, v, calc = np.array(x0), 0.01, 2.0, True
    for t, p in zip(td, per):
        if calc:
            H, g, r1 = evaluate(x)
        D = np.diag(H).copy()
        dx = np.linalg.solve(H + u * np.diag(D), -g)
        q1 = 0.5 * dx @ (u * D * dx - g)
        xt = pgr.pose_update(x, dx)
        r2 = cv.residual(xt) + ppr.cost(xt, odo, priors)
        q = r1 - r2
        assert (q > 0) == t["accepted"]
        if q > 0:
            x, u, v, calc = xt, u * max(1 - (2 * q / q1 - 1) ** 3, 1.0 / 3.0), 2.0, True
        else:
            u, v, calc = u * v, 2 * v, False
        assert np.abs(p - x).max() <= 1e-9
    cb.close()
    cv.close()


def _gnss_error(x, sc):
    return np.linalg.norm(x[:, 9:] - sc["poses_gt"][:, 9:], axis=1)


def test_gnss_corridor_converges_in_the_priors_frame():
    """a 1 km voxel corridor of 1 000 poses started 3 m off: with odometry and lever-arm GNSS fixes every 10th pose the
    LM (gauge_mode 2, no re-anchoring) lands on the truth's frame"""
    sc, odo, priors, x0 = _corridor(N=1000)
    c = _blocks_ctx(sc, odo, priors)
    x, t, _ = c.damping_iter(x0, max_iter=30, gauge_mode=2, min_planes_per_pose=0)
    err = _gnss_error(x, sc)
    assert _gnss_error(x0, sc).min() > 2.0  # the start is off by metres everywhere
    assert err.max() < 0.3, err.max()
    c.close()


def test_gnss_pose_graph_covariance_with_a_free_anchor():
    """odometry and GNSS on PoseGraph: anchor = -1 is regular, matches the dense inverse, and the converged error is
    within a few sigma of it. (At 1 km from the origin the left-update coordinates couple rotation and position so
    strongly that H's pivots span more than the 1e-11 the pivot test allows, so this runs at 300 m.)"""
    sc, odo, priors, x0 = _corridor(N=300)
    N = sc["n_poses"]
    s = balm_b200.PoseGraph(N)
    s.set_pose_factors(odo)
    s.set_pose_priors(priors)
    x, _ = s.pose_graph_iter(x0, max_iter=30, gauge_mode=2)
    pairs, cov = s.covariance(x, anchor=-1)
    Hs, _, _, _, _ = _spg_dense(s, x, N)
    S, kappa = _dense_sigma(Hs, -1)
    ref = bref.blocks_of(S, pairs)
    assert np.abs(cov - ref).max() <= max(1e-9, 10 * kappa * np.finfo(float).eps) * np.abs(ref).max()
    diag = np.array([cov[p][3:, 3:] for p in range(len(pairs)) if pairs[p, 0] == pairs[p, 1]])
    sigma = np.sqrt(2 * rr.POINT_NOISE ** 2 * np.trace(diag, axis1=1, axis2=2))  # covariance = 2 sigma_p^2 H^-1
    assert (_gnss_error(x, sc) <= 5.0 * sigma).all()
    s.close()


def test_gnss_outliers_cauchy_versus_trivial():
    clean_sc, odo, clean, x0 = _corridor(N=400, seed=6)
    out_idx = (3, 17, 30)
    sc, odo, bad, x0 = _corridor(N=400, seed=6, outliers=out_idx)
    errs = {}
    c = _blocks_ctx(sc, odo, clean)
    errs["clean"] = _gnss_error(c.damping_iter(x0, max_iter=30, gauge_mode=2, min_planes_per_pose=0)[0], sc).max()
    c.close()
    c2 = 2 * rr.POINT_NOISE ** 2 * 16.27  # chi-square, 3 degrees of freedom, p = 0.999, in the cost's units
    for kind in ("trivial", "cauchy"):
        c = _blocks_ctx(sc, odo, bad, kind=kind, scale=np.sqrt(c2))
        x = c.damping_iter(x0, max_iter=40, gauge_mode=2, min_planes_per_pose=0)[0]
        errs[kind] = _gnss_error(x, sc).max()
        if kind == "cauchy":
            _, w = c.prior_residuals(x)
            good = np.setdiff1d(np.arange(len(bad)), out_idx)
            assert w[list(out_idx)].max() < 0.05 < w[good].min()
        c.close()
    assert errs["cauchy"] <= 1.5 * errs["clean"] + 0.01, errs
    assert errs["trivial"] >= 3.0 * errs["clean"], errs


def test_collinear_position_priors_leave_the_roll_free():
    N = 20
    gt = np.array([pgr.pack(np.eye(3), [2.0 * i, 0.0, 0.0]) for i in range(N)])
    rng = np.random.default_rng(3)
    factors = [pgr.make_factor(rng, gt, [i, i + 1], cond=10.0) for i in range(N - 1)]
    s = balm_b200.PoseGraph(N)
    s.set_pose_factors(factors)
    s.set_pose_priors(balm_b200.position_priors([0, 10, 19], gt[[0, 10, 19], 9:], np.eye(3)))
    with pytest.raises(balm_b200.BalmError) as e:
        s.covariance(gt, anchor=-1)
    assert e.value.status == L.ERR_NOT_PD
    s.close()
    bent = gt.copy()
    bent[10:, 10] += 0.5 * np.arange(N - 10)  # the positions of poses 0, 10, 19 span a plane
    s = balm_b200.PoseGraph(N)
    s.set_pose_factors([pgr.make_factor(rng, bent, [i, i + 1], cond=10.0) for i in range(N - 1)])
    s.set_pose_priors(balm_b200.position_priors([0, 10, 19], bent[[0, 10, 19], 9:], np.eye(3)))
    pairs, cov = s.covariance(bent, anchor=-1)
    assert np.isfinite(cov).all()
    s.close()


def test_refusals_and_statuses_keep_the_previous_set():
    gt, factors, x, priors = _graph(3)
    N = len(gt)
    for h in (balm_b200.Context(N), balm_b200.PoseGraph(N)):
        h.set_pose_factors(factors)
        h.set_pose_priors(priors)
        ref = h.prior_residuals(x)
        bad = []
        for field, val in [("pose", N), ("pose", -1), ("pose_hat", np.full(12, np.nan)), ("lever_arm", [np.inf, 0, 0])]:
            bad.append([dict(priors[0], **{field: val})])
        H = np.eye(6)
        H[0, 1] = 1e-3
        bad.append([dict(priors[0], H=H)])
        H = np.eye(6)
        H[2, 2] = np.nan
        bad.append([dict(priors[0], H=H)])
        for b in bad:
            with pytest.raises(balm_b200.BalmError) as e:
                h.set_pose_priors(b)
            assert e.value.status == L.ERR_INVALID
        for kind, scale in [("huber", None), ("cauchy", -1.0), ("cauchy", np.inf)]:
            with pytest.raises(balm_b200.BalmError):
                h.set_pose_priors(priors, kind=kind, scale=scale)
        st = L.lib().balm_set_pose_priors if isinstance(h, balm_b200.Context) else L.lib().balm_spg_set_pose_priors
        k = np.full(len(priors), 7, dtype=np.int32)
        hat = np.ascontiguousarray([p["pose_hat"] for p in priors])
        Hs = np.ascontiguousarray([p["H"].ravel(order="F") for p in priors])
        pose = np.array([p["pose"] for p in priors], dtype=np.int32)
        assert st(h._h, len(priors), pose.ctypes.data, hat.ctypes.data, None, Hs.ctypes.data, k.ctypes.data, None,
                  None) == L.ERR_INVALID
        for a, b in zip(h.prior_residuals(x), ref):
            assert np.array_equal(a, b)
        neg = np.diag([1.0, 1, 1, 1, 1, -1e-6])
        st_ = h.set_pose_priors([priors[0], dict(priors[1], H=neg), dict(priors[2], H=np.zeros((6, 6)))])
        assert st_ == [L.OK, L.ERR_NOT_PD, L.ERR_NOT_PD]
        s_, w_ = h.prior_residuals(x)
        assert s_[1] == s_[2] == w_[1] == w_[2] == 0.0
        h.close()
    c = balm_b200.Context(N)
    c.set_pose_priors(priors)  # priors without factors: the pose graph calls still refuse
    with pytest.raises(balm_b200.BalmError):
        c.pose_graph_evaluate(x)
    c.close()


def test_gauge_modes_refused_with_active_priors():
    gt, factors, x, priors = _graph(4)
    N = len(gt)
    for h in (balm_b200.Context(N), balm_b200.PoseGraph(N)):
        h.set_pose_factors(factors)
        h.set_pose_priors(priors)
        for gm in (0, 1):
            with pytest.raises(balm_b200.BalmError) as e:
                h.pose_graph_iter(x, max_iter=2, gauge_mode=gm)
            assert e.value.status == L.ERR_INVALID and "gauge_mode 2" in str(e.value)
        h.set_pose_priors([dict(priors[0], H=np.zeros((6, 6)))])  # nothing active: the gauge step is allowed again
        h.pose_graph_iter(x, max_iter=2, gauge_mode=0)
        h.close()
    sc, odo, pr, x0 = _corridor(N=40, every=5)
    c = _blocks_ctx(sc, odo, pr)
    with pytest.raises(balm_b200.BalmError):
        c.damping_iter(x0, max_iter=2, gauge_mode=0, min_planes_per_pose=0)
    c.close()


def test_spg_pattern_grows_only_for_a_factor_free_pose_and_detach_is_bitwise():
    gt, factors, x, priors = _graph(5, P=30)
    N = len(gt)
    covered = [f for f in factors if 29 not in f["poses"] and 28 not in f["poses"]]
    s, ref = balm_b200.PoseGraph(N), balm_b200.PoseGraph(N)
    for h in (s, ref):
        h.set_pose_factors(covered)
    base = s.structure()
    s.set_pose_priors(priors)  # poses all covered
    assert s.structure()["pairs"] == base["pairs"]
    s.set_pose_priors(priors + [dict(priors[0], pose=29)])
    assert s.structure()["pairs"] == base["pairs"] + 1
    c = balm_b200.Context(N)
    c.set_pose_factors(covered)
    c.set_pose_priors(priors + [dict(priors[0], pose=29)])
    H, g, cost = c.pose_graph_evaluate(x)
    Hs, gs, cs, pairs, blocks = _spg_dense(s, x, N)
    assert np.array_equal(blocks, np.array([H[6 * i:6 * i + 6, 6 * j:6 * j + 6] for i, j in pairs]))
    assert np.array_equal(gs, g) and cs == cost
    s.set_pose_factors(factors)  # re-registration keeps the priors; pose 29 is covered now
    assert s.prior_residuals(x)[0].shape == (len(priors) + 1,)
    for h in (s, c):
        h.set_pose_priors([])
    ref.set_pose_factors(factors)
    a, b = s.pose_graph_evaluate(x), ref.pose_graph_evaluate(x)
    assert all(np.array_equal(u, v) for u, v in zip(a, b))
    assert s.structure() == ref.structure()
    xa, ta = s.pose_graph_iter(x, max_iter=4)
    xb, tb = ref.pose_graph_iter(x, max_iter=4)
    assert np.array_equal(xa, xb)
    for h in (s, ref, c):
        h.close()


def test_blocks_lifetime_across_registrations_and_detach():
    sc, odo, priors, x0 = _corridor(N=60, every=6)
    c, ref = _blocks_ctx(sc, [], priors), _blocks_ctx(sc, [], [])
    bytes_with = c.block_structure()["device_bytes"]
    assert bytes_with > ref.block_structure()["device_bytes"]
    c.set_block_factors(odo)
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
    H1, g1, r1 = c.evaluate(x0)
    Hp, gp, cp = ppr.evaluate(x0, odo, priors, sc["n_poses"])
    ref.set_block_factors(odo)
    H0, g0, r0 = ref.evaluate(x0)
    assert np.abs((H1 - H0) - (Hp - ppr.evaluate(x0, odo, [], sc["n_poses"])[0])).max() <= 1e-12 * np.abs(H1).max()
    c.set_pose_priors([])
    a, b = c.evaluate(x0), ref.evaluate(x0)
    assert all(np.array_equal(u, v) for u, v in zip(a, b))
    assert c.block_structure() == ref.block_structure()
    kw = dict(max_iter=4, gauge_mode=0, min_planes_per_pose=0)
    assert np.array_equal(c.damping_iter(x0, **kw)[0], ref.damping_iter(x0, **kw)[0])
    c.close()
    ref.close()


def test_hba_pose_graph_in_the_priors_frame():
    """HBA's scene started in a frame 3 m / 0.05 rad away from the truth: with GNSS priors by scan index the fused
    poses come back in the priors' (the truth's) frame; without them they keep scan 0's input frame"""
    import hba_ref
    from balm_b200 import hba
    scans, gt, init = hba_ref.drift_scene()
    off = pgr.pack(pgr.exp_so3([0.0, 0.0, 0.05]), [3.0, -1.0, 0.5])
    start = np.array([pgr.compose(off, p) for p in init])
    idx = np.arange(0, len(gt), 5)
    priors = balm_b200.position_priors(idx, gt[idx, 9:], 10.0 * np.eye(3))
    res = hba.hba(scans, start, pose_graph=True, priors=priors)
    assert res["pose_graph"]["prior_status"] == [0] * len(priors)
    assert np.linalg.norm(res["poses"][:, 9:] - gt[:, 9:], axis=1).max() < 0.05
    free = hba.hba(scans, start, pose_graph=True)
    assert np.abs(free["poses"][0] - start[0]).max() <= 1e-12
    with pytest.raises(ValueError):
        hba.hba(scans, start, priors=priors)

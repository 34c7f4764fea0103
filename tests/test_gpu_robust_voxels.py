"""Robust voxel costs on the device (balm_set_voxel_loss, balm_voxel_residuals and the batch's twins): evaluation against
robust_voxels_ref on every precision and scene shape, the coe w identity, the no-op of a trivial loss, LM parity and
recovery on the moving-plane scene, lifetime across every registration route, refusals, the batch and hba."""
import ctypes as C

import numpy as np
import pytest

import assoc_ref
import balm_b200
import block_hessian_ref as bref
import hba_ref
import robust_voxels_ref as rv
import scenes
from balm_b200 import _lib as L
from balm_b200 import drivers, hba
from test_gpu_block_hessian import _check_eval

pytestmark = pytest.mark.gpu

PRECS = {"fp64": L.PREC_FP64, "tensor": L.PREC_TENSOR, "blocks": L.PREC_BLOCKS}
TOLH = {"fp64": 1e-9, "tensor": 1e-8, "blocks": 1e-9}
SCENES = {
    "dense": lambda: rv.moving_plane_scene()[0],
    "ragged": lambda: rv.moving_plane_scene(n_poses=10, n_planes=80, seed=4, drop=0.4)[0],
    "sparse": lambda: bref.corridor(40, w=4, planes_per_pose=30, seed=1),
    "fix": lambda: rv.moving_plane_scene(n_poses=8, n_planes=40, seed=5, with_fix=True)[0],
}


def _ctx(sc, prec, loss=None, coe=None):
    c = balm_b200.Context(sc["n_poses"], 0, PRECS[prec])
    if loss is not None:
        c.set_voxel_loss(*loss)
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"] if coe is None else coe, sc.get("fix10"))
    return c


def _median_scale(sc, x, include_fix=False):
    """a scale with voxels on both sides of c^2"""
    return float(np.sqrt(np.median(rv.lams(sc, x, include_fix))))


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300)


# ------------------------------------------------------------ 1. evaluation against the restatement --------------------
@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("name", list(SCENES))
@pytest.mark.parametrize("kind", ["huber", "cauchy"])
def test_evaluation_matches_restatement(prec, name, kind):
    sc = SCENES[name]()
    x = sc["poses_init"]
    for include_fix in ((False, True) if sc.get("fix10") is not None else (False,)):
        c = _median_scale(sc, x, include_fix)
        Hr, gr, rr_, lam_r, w_r = rv.evaluate(sc, x, rv.NAMES[kind], c, include_fix)
        assert w_r.min() < 1.0
        ctx = _ctx(sc, prec, (kind, c))
        H, g, r = ctx.evaluate(x, include_fix=include_fix)
        # the residual within 1e-12, or within what the same scene gives without a loss (the corridor's thousand small
        # lambda_min, Jacobi on the device against LAPACK here, differ by a little more)
        r0 = _ctx(sc, prec).evaluate(x, include_fix=include_fix, want_H=False)[2]
        e0 = abs(r0 - rv.cost(sc, x, rv.TRIVIAL, 1.0, include_fix)) / abs(r0)
        assert abs(r - rr_) <= max(1e-12, 2 * e0) * abs(rr_)
        assert _rel(g, gr) <= 1e-10
        assert _rel(H, Hr) <= TOLH[prec]
        lam, w = ctx.voxel_residuals(x, include_fix=include_fix)
        assert _rel(lam, lam_r) <= 1e-9 and _rel(w, w_r) <= 1e-9
        if prec == "blocks":  # the blocks are the fp64 context's dense entries, g and r bitwise
            _check_eval(ctx, _ctx(sc, "fp64", (kind, c)), x, include_fix=include_fix)


@pytest.mark.parametrize("prec", list(PRECS))
def test_batches_and_sub_ranges(prec, monkeypatch):
    """several voxel batches (a 1 MB G' budget) and sub-ranges that sum to the full range"""
    sc = rv.moving_plane_scene(n_poses=8, n_planes=700, n_moving=40, seed=6)[0]
    x = sc["poses_init"]
    c = _median_scale(sc, x)
    Hr, gr, rr_, _, _ = rv.evaluate(sc, x, rv.CAUCHY, c)
    monkeypatch.setenv("BALM_G_BUDGET_MB", "1")
    ctx = _ctx(sc, prec, ("cauchy", c))
    H, g, r = ctx.evaluate(x)
    assert abs(r - rr_) <= 1e-12 * abs(rr_) and _rel(g, gr) <= 1e-10 and _rel(H, Hr) <= TOLH[prec]
    M = len(sc["coe"])
    cuts = [0, 233, 511, M]
    parts = [ctx.evaluate(x, a, b) for a, b in zip(cuts[:-1], cuts[1:])]
    assert _rel(sum(p[0] for p in parts), H) <= (1e-12 if prec != "tensor" else TOLH[prec])  # per-range column scales
    assert _rel(sum(p[1] for p in parts), g) <= 1e-12
    assert abs(sum(p[2] for p in parts) - r) <= 1e-12 * abs(r)
    lam, w = ctx.voxel_residuals(x, 233, 511)
    lam_all, w_all = ctx.voxel_residuals(x)
    assert np.array_equal(lam, lam_all[233:511]) and np.array_equal(w, w_all[233:511])


# ------------------------------------------------------------ 2. the coe w identity ------------------------------------
@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("name", ["dense", "sparse", "fix"])
def test_coe_w_identity(prec, name):
    """H, g, the blocks and the covariances of a robust context are bitwise those of a trivial-loss context registered
    with coe w from voxel_residuals"""
    sc = SCENES[name]()
    x = sc["poses_init"]
    include_fix = sc.get("fix10") is not None
    c = _median_scale(sc, x, include_fix)
    rob = _ctx(sc, prec, ("cauchy", c))
    _, w = rob.voxel_residuals(x, include_fix=include_fix)
    twin = _ctx(sc, prec, coe=sc["coe"] * w)
    H1, g1, _ = rob.evaluate(x, include_fix=include_fix)
    H2, g2, _ = twin.evaluate(x, include_fix=include_fix)
    assert np.array_equal(H1, H2) and np.array_equal(g1, g2)
    x = sc["poses_gt"]  # covariances where H without the anchor is positive definite
    _, w = rob.voxel_residuals(x, include_fix=include_fix)
    twin = _ctx(sc, prec, coe=sc["coe"] * w)
    if prec == "blocks":
        rob.evaluate(x, include_fix=include_fix)
        twin.evaluate(x, include_fix=include_fix)
        assert np.array_equal(rob.download_blocks(), twin.download_blocks())
        anchor = -1 if include_fix else 0
        a, b = rob.block_covariance(x, include_fix, anchor), twin.block_covariance(x, include_fix, anchor)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    elif include_fix:
        a, b = rob.pose_covariance(x, 0.02, include_fix=True), twin.pose_covariance(x, 0.02, include_fix=True)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    else:
        a, b = rob.pose_covariance(x, 0.02, want_cov=False), twin.pose_covariance(x, 0.02, want_cov=False)
        assert np.array_equal(a[0], b[0])


# ------------------------------------------------------------ 3. a trivial loss changes nothing ------------------------
def _everything(ctx, x, prec):
    H, g, r = ctx.evaluate(x)
    p, t, per = ctx.damping_iter(x, max_iter=8, want_per_iter=True, force_hess=True)
    out = [H, g, r, p, t, per]
    if prec == "blocks":
        out.append(ctx.download_blocks())
    tm = ctx.timings()
    out.append({k: v for k, v in tm.items() if not k.startswith("ms_")})
    return out


@pytest.mark.parametrize("prec", list(PRECS))
def test_trivial_loss_is_a_no_op(prec):
    """a context that never had a loss, one with the trivial loss set explicitly and one reset after Cauchy, each after
    the same history (an evaluation, a registration of the same voxels, counters reset): every output bitwise equal"""
    sc = SCENES["dense"]()
    x = sc["poses_init"]
    ctxs = [_ctx(sc, prec), _ctx(sc, prec, ("trivial", None)), _ctx(sc, prec, ("cauchy", 0.03))]
    for i, ctx in enumerate(ctxs):
        ctx.evaluate(x)
        if i:
            ctx.set_voxel_loss("trivial")
        ctx.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
        ctx.reset_counters()
    ref = _everything(ctxs[0], x, prec)
    a = ctxs[1]
    for ctx in ctxs[1:]:
        got = _everything(ctx, x, prec)
        for u, v in zip(got, ref):
            if isinstance(u, (list, dict)):
                assert u == v
            else:
                assert np.array_equal(np.asarray(u), np.asarray(v))
    assert np.array_equal(a.voxel_residuals(x)[1], np.ones(len(sc["coe"])))


# ------------------------------------------------------------ 4. LM on the moving-plane scene --------------------------
@pytest.fixture(scope="module")
def outlier():
    bad, clean = rv.moving_plane_scene()
    x0, gt = clean["poses_init"], clean["poses_gt"]
    ref = rv.lm(bad, x0, rv.CAUCHY, rv.SCALE, max_iter=15)
    e_clean = rv.max_error(rv.lm(clean, x0, rv.TRIVIAL, 1.0, max_iter=15)[0], gt)
    return bad, x0, gt, ref, e_clean


@pytest.mark.parametrize("prec", list(PRECS))
def test_lm_outlier_scene(prec, outlier, monkeypatch):
    bad, x0, gt, (xr, tr, per_r), e_clean = outlier
    runs = []
    for no_reuse in ((False, True) if prec == "tensor" else (False,)):
        if no_reuse:
            monkeypatch.setenv("BALM_NO_SWEEP_REUSE", "1")
        ctx = _ctx(bad, prec, ("cauchy", rv.SCALE))
        p, t, per = ctx.damping_iter(x0, max_iter=15, want_per_iter=True)
        assert [d["accepted"] for d in t] == [d["accepted"] for d in tr]
        for a, b in zip(per, per_r):
            assert np.abs(a - b).max() <= 1e-6
        assert rv.max_error(per[-1], gt) < 2 * e_clean
        tm = ctx.timings()
        print("%s reuse=%s: max error %.4f m (clean %.4f m), single %d redone %d reused %d" % (
            prec, not no_reuse, rv.max_error(per[-1], gt), e_clean, tm["single_sweeps"], tm["redone_sweeps"],
            tm["reused_sweeps"]))
        runs.append(per)
    if len(runs) == 2:
        assert all(np.array_equal(a, b) for a, b in zip(*runs))
    triv = _ctx(bad, prec).damping_iter(x0, max_iter=15, want_per_iter=True)[2]
    assert rv.max_error(triv[-1], gt) > 5 * e_clean


def test_tensor_rejected_steps_with_a_loss(outlier, monkeypatch):
    """force_hess after rejected steps: the sweep reuse (tc_adopt_kernel) and the stats hand-over with weights give the
    bits of sweeping again"""
    bad, x0, _, _, _ = outlier
    runs = []
    for no_reuse in (False, True):
        if no_reuse:
            monkeypatch.setenv("BALM_NO_SWEEP_REUSE", "1")
        ctx = _ctx(bad, "tensor", ("huber", rv.SCALE))
        p, t, per = ctx.damping_iter(x0, max_iter=12, u0=1e-6, rel_tol=-1, want_per_iter=True, force_hess=True)
        runs.append((p, t, per))
        print("reuse=%s accepted %s, timings %s" % (not no_reuse, "".join(str(int(d["accepted"])) for d in t),
                                                     {k: v for k, v in ctx.timings().items() if "sweeps" in k}))
    assert any(not d["accepted"] for d in runs[0][1])
    assert np.array_equal(runs[0][0], runs[1][0]) and runs[0][1] == runs[1][1]


# ------------------------------------------------------------ 5. lifetime and refusals --------------------------------
def _loss_applies(ctx, x, kind, c, include_fix=False):
    lam, w = ctx.voxel_residuals(x, include_fix=include_fix)
    assert np.allclose(w, [rv.drho(kind, c, s) for s in lam], rtol=1e-14, atol=0)
    _, _, r = ctx.evaluate(x, include_fix=include_fix, want_H=False)
    co = ctx.download_voxels()[3]
    assert abs(r - sum(a * rv.rho(kind, c, s) for a, s in zip(co, lam))) <= 1e-11 * abs(r)


@pytest.mark.parametrize("prec", list(PRECS))
def test_loss_survives_every_registration_route(prec):
    N = 10
    pts, frs, poses = assoc_ref.synthetic_scans(n_poses=N, pts_per_scan=4000, seed=21)
    P = scenes.pack_poses([r for r, _ in poses], [p for _, p in poses])
    kw = dict(voxel_size=2.0, layer_limit=2, min_ps=15, eigen_value_array=(1 / 16, 1 / 16, 1 / 9))
    ctx = balm_b200.Context(N, 0, PRECS[prec])
    ctx.set_voxel_loss("cauchy", 0.005)
    win = frs < N - 1
    ctx.cut_voxels(pts[win].astype(np.float32), frs[win], P, **kw)
    _loss_applies(ctx, P, rv.CAUCHY, 0.005)
    ctx.marginalize(2, P)
    _loss_applies(ctx, P, rv.CAUCHY, 0.005, include_fix=True)
    ctx.append_scan(pts[frs == N - 1].astype(np.float32), P, N - 2)
    _loss_applies(ctx, P, rv.CAUCHY, 0.005, include_fix=True)
    ctx.window_reset(**kw)
    for s in range(N):
        ctx.window_cut(pts[frs == s].astype(np.float32), P[s], s)
        ctx.window_recut(s + 1)
    ctx.window_push(N)
    _loss_applies(ctx, P, rv.CAUCHY, 0.005, include_fix=True)
    ctx.set_voxels(np.zeros(1, np.int64), np.zeros(0, np.int32), np.zeros((0, 10)), np.zeros(0))  # the empty set
    assert ctx.voxel_residuals(P)[0].shape == (0,)
    sc = SCENES["dense"]()
    ctx2 = balm_b200.Context(sc["n_poses"], 0, PRECS[prec])
    ctx2.set_voxel_loss("huber", 0.03)
    ctx2.set_voxels(np.zeros(1, np.int64), np.zeros(0, np.int32), np.zeros((0, 10)), np.zeros(0))
    ctx2.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
    _loss_applies(ctx2, sc["poses_init"], rv.HUBER, 0.03)
    if prec != "blocks":  # synth_virtual's dense scene
        gt, init = ctx2.synth_virtual(200, pts_size=20, point_noise=0.02)
        _loss_applies(ctx2, init, rv.HUBER, 0.03)


def test_refusals_keep_the_previous_loss():
    sc = SCENES["dense"]()
    x = sc["poses_init"]
    ctx = _ctx(sc, "fp64", ("cauchy", 0.03))
    w0 = ctx.voxel_residuals(x)[1]
    lib = L.lib()
    for kind, scale in [(3, 0.03), (-1, 0.03), (1, 0.0), (2, -0.1), (2, float("nan")), (1, float("inf"))]:
        assert lib.balm_set_voxel_loss(ctx._h, kind, scale) == L.ERR_INVALID
        assert np.array_equal(ctx.voxel_residuals(x)[1], w0)
    with pytest.raises(ValueError):
        ctx.set_voxel_loss("tukey", 0.03)
    assert lib.balm_set_voxel_loss(None, 0, 1.0) == L.ERR_INVALID
    assert lib.balm_set_voxel_loss(ctx._h, 0, float("nan")) == L.OK  # a trivial loss's scale is ignored
    assert np.array_equal(ctx.voxel_residuals(x)[1], np.ones(len(sc["coe"])))
    with pytest.raises(balm_b200.BalmError):
        ctx.voxel_residuals(x, 5, 2)
    b = balm_b200.Batch()
    assert lib.balm_batch_set_voxel_loss(b._h, 4, 1.0) == L.ERR_INVALID
    assert lib.balm_batch_voxel_residuals(b._h, x.ctypes.data_as(C.c_void_p), 0, None, None) == L.ERR_INVALID


# ------------------------------------------------------------ 6. batch and hba -----------------------------------------
def _problems():
    out = []
    for s in range(5):
        sc = rv.moving_plane_scene(n_poses=4 + s, n_planes=20 + 5 * s, n_moving=2 + s % 3, seed=10 + s,
                                   with_fix=s % 2 == 1)[0]
        out.append(sc)
    return out


def test_batch_matches_restatement_and_context():
    probs = _problems()
    xs = [p["poses_init"] for p in probs]
    c = 0.02
    b = balm_b200.Batch()
    b.set_voxel_loss("cauchy", c)
    b.set_problems([probs[0]])  # the loss belongs to the batch: it survives a change of the problem count
    b.set_problems(probs)
    for include_fix in (False, True):
        res = b.evaluate(xs, include_fix=include_fix)
        lw = b.voxel_residuals(xs, include_fix=include_fix)
        for sc, x, (H, g, r), (lam, w) in zip(probs, xs, res, lw):
            Hr, gr, rr_, lam_r, w_r = rv.evaluate(sc, x, rv.CAUCHY, c, include_fix)
            assert abs(r - rr_) <= 1e-12 * abs(rr_) and _rel(g, gr) <= 1e-10 and _rel(H, Hr) <= 1e-9
            assert _rel(lam, lam_r) <= 1e-9 and _rel(w, w_r) <= 1e-9
    # the coe w identity on the batch's covariance
    lw = b.voxel_residuals(xs, include_fix=True)
    twin = balm_b200.Batch()
    twin.set_problems([dict(sc, coe=sc["coe"] * w) for sc, (_, w) in zip(probs, lw)])
    for u, v in zip(b.pose_covariance(xs, 0.02, include_fix=True), twin.pose_covariance(xs, 0.02, include_fix=True)):
        assert u[0] == v[0] and np.array_equal(u[1], v[1]) and np.array_equal(u[2], v[2])
    # LM per problem: that of a one-problem fp64 context with the same loss
    out = b.damping_iter(xs, max_iter=8, min_planes_per_pose=0, want_per_iter=True)
    for sc, x, (st, p, t, per) in zip(probs, xs, out):
        ctx = _ctx(sc, "fp64", ("cauchy", c))
        p2, t2, per2 = ctx.damping_iter(x, max_iter=8, min_planes_per_pose=0, want_per_iter=True)
        assert st == L.OK and [d["accepted"] for d in t] == [d["accepted"] for d in t2]
        assert np.abs(p - p2).max() <= 1e-9


def _moving_patch(scans, gt, speed=0.03, n=1500, seed=5):
    """scans with a 8 m x 8 m panel at y = 5 m added to every scan, moving `speed` m per scan along its normal"""
    rng = np.random.default_rng(seed)
    out = []
    for i, s in enumerate(scans):
        w = np.stack([rng.uniform(-4, 4, n), np.full(n, 5.0 + speed * i) + rng.normal(0, 0.01, n),
                      rng.uniform(-4, 4, n)], 1)
        R, p = gt[i, :9].reshape(3, 3).T, gt[i, 9:]
        out.append(np.concatenate([s, ((w - p) @ R).astype(np.float32)]))
    return out


def test_hba_with_a_voxel_loss():
    scans, gt, init = hba_ref.drift_scene()
    bad = _moving_patch(scans, gt)
    res_t = hba.hba(bad, init)
    res_c = hba.hba(bad, init, voxel_loss=("cauchy", 0.03))
    rot_t, tran_t = drivers.rsme(res_t["poses"], gt)
    rot_c, tran_c = drivers.rsme(res_c["poses"], gt)
    print("moving patch, hba RMSE rot [deg] / tran [m]: trivial %.4f / %.4f, cauchy %.4f / %.4f"
          % (np.degrees(rot_t), tran_t, np.degrees(rot_c), tran_c))
    assert tran_c < tran_t and rot_c < rot_t
    res_pg = hba.hba(bad, init, pose_graph=True, voxel_loss=("cauchy", 0.03))
    assert res_pg["pose_graph"]["n_factors"] > 0

"""Voxels, pose factors and priors in one cost on FP64 / TENSOR contexts (balm_set_joint_cost): the full-range H, g
and residual against the voxel cost plus the pose graph and the priors' restatement, sub-ranges and a switch without
terms bitwise the voxel cost, LM parity with a blocks context, FP64 and the host oracle, the tensor path's carry-over,
scans without planes, GNSS in the priors' frame, the covariance with priors, the rig, refusals and repeatability."""
import numpy as np
import pytest

import balm_b200
import block_hessian_ref as bref
import pose_graph_ref as pgr
import pose_priors_ref as ppr
import rig_blocks_ref as rb
import rig_ref as rr
import robust_factors_ref as rfr
from balm_b200 import _lib as L
from test_gpu_block_factors import _factors, _noisy_odometry, _odo_info
from test_gpu_block_hessian import _ctx
from test_gpu_pose_priors import _corridor, _gnss_error
from test_gpu_rig_blocks import _states_close
from test_gpu_sparse_covariance import _dense_sigma

pytestmark = pytest.mark.gpu

DENSE = [L.PREC_FP64, L.PREC_TENSOR]
# one kind for voxels, factors and priors; scales near each term's typical sqrt(s), so that some terms are down-weighted
LOSSES = [("trivial", None, None, None), ("huber", 0.012, 0.02, 0.01), ("cauchy", 0.012, 0.02, 0.01)]
# counters that describe what a run did (the ms_* fields are times)
COUNTERS = ("launches", "n_eval", "n_solve", "n_residual", "digit_planes", "single_sweeps", "redone_sweeps",
            "refinements", "n_stats", "reused_sweeps")


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300)


def _status(fn):
    with pytest.raises(balm_b200.BalmError) as e:
        fn()
    return e.value.status


def _pose_err(a, b):
    """largest rotation angle (rad) and position distance (m) between the poses of a and b"""
    a, b = np.reshape(a, (-1, 12)), np.reshape(b, (-1, 12))
    rot = max(np.linalg.norm(pgr.log_so3(pgr.split(x)[0].T @ pgr.split(y)[0])) for x, y in zip(a, b))
    return rot, float(np.linalg.norm(a[:, 9:] - b[:, 9:], axis=1).max())


def _counters(c):
    t = c.timings()
    return {k: t[k] for k in COUNTERS}


def _scene(N=60, seed=31, every=6):
    """bref.corridor with _factors' odometry, loop closures and a window factor, and GNSS priors every `every` poses
    plus two full-pose anchors"""
    sc, _, priors, x0 = _corridor(N=N, seed=seed, every=every)
    fs = _factors(sc, seed, loops=((N // 2 + 5, 3), (N - 5, N // 3)), windows=((10, 11, 12),))
    priors = priors + ppr.random_priors(np.random.default_rng(seed), sc["poses_gt"], [5, N // 2])
    return sc, fs, priors, x0


def _joint(sc, prec, fs, priors, loss=LOSSES[0], on=True):
    kind, cv, cf, cp = loss
    c = balm_b200.Context(sc["n_poses"], 0, prec)
    if kind != "trivial":
        c.set_voxel_loss(kind, cv)
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc.get("fix10"))
    if fs:
        assert c.set_pose_factors(fs) == [L.OK] * len(fs)
        c.set_factor_loss(kind, cf)
    if priors:
        assert c.set_pose_priors(priors, kind=kind, scale=cp) == [L.OK] * len(priors)
    if on:
        c.set_joint_cost(True)
    return c


def _blocks(sc, fs, priors, loss=LOSSES[0]):
    kind, cv, cf, cp = loss
    c = balm_b200.Context(sc["n_poses"], 0, L.PREC_BLOCKS)
    if kind != "trivial":
        c.set_voxel_loss(kind, cv)
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc.get("fix10"))
    c.set_block_factors(fs)
    c.set_factor_loss(kind, cf)
    if priors:
        c.set_pose_priors(priors, kind=kind, scale=cp)
    return c


def _loss_arrays(loss, fs, priors):
    kind, _, cf, cp = loss
    fk, fsc = rfr.loss_arrays(len(fs), kind, cf)
    pk, psc = rfr.loss_arrays(len(priors), kind, cp)
    return dict(fk=fk, fs=fsc, pk=pk, ps=psc)


@pytest.mark.parametrize("prec", DENSE)
@pytest.mark.parametrize("loss", LOSSES, ids=[l[0] for l in LOSSES])
def test_decomposition_and_sub_ranges(prec, loss):
    """factors alone: bitwise the voxel evaluation plus pose_graph_evaluate; with priors: that plus the priors'
    restatement (1e-12); sub-ranges bitwise voxels only; residual the full-range cost"""
    sc, fs, priors, x = _scene()
    N, M = sc["n_poses"], len(sc["row_ptr"]) - 1
    c = _joint(sc, prec, fs, [], loss)
    c0 = _joint(sc, prec, [], [], loss, on=False)
    H0, g0, r0 = c0.evaluate(x)
    Hf, gf, rf = c.pose_graph_evaluate(x)
    H, g, r = c.evaluate(x)
    assert np.array_equal(H, H0 + Hf) and np.array_equal(g, g0 + gf) and r == r0 + rf
    assert np.array_equal(H, H.T)
    assert c.residual(x) == c0.residual(x) + rf == r
    for head, end in [(0, M // 3), (M // 3, M), (M // 2, M // 2 + 1), (5, 5), (0, M - 1)]:
        a, b = c.evaluate(x, head, end), c0.evaluate(x, head, end)
        assert all(np.array_equal(u, v) for u, v in zip(a, b)), (head, end)
    kind, _, _, cp = loss
    c.set_pose_priors(priors, kind=kind, scale=cp)
    Hp, gp, rp = c.evaluate(x)
    la = _loss_arrays(loss, fs, priors)
    Hr, gr, rr_ = ppr.evaluate(x, [], priors, N, pk=la["pk"], ps=la["ps"])
    assert _rel(Hp, H + Hr) <= 1e-12 and _rel(gp, g + gr) <= 1e-12 and abs(rp - (r + rr_)) <= 1e-12 * abs(rp)
    assert np.array_equal(Hp, Hp.T)
    assert c.residual(x) == rp
    a = c.evaluate(x)  # repeatable
    assert all(np.array_equal(u, v) for u, v in zip(a, (Hp, gp, rp)))
    c.close()
    c0.close()


@pytest.mark.parametrize("prec", DENSE)
def test_switch_without_terms_and_switched_off_are_the_voxel_cost(prec):
    """on without terms, and terms with the switch off: evaluations, LM poses, traces and counters bitwise those of a
    context that never had the switch; the switch survives re-registrations and replaced term sets"""
    sc, fs, priors, x = _scene(N=40, seed=33, every=5)
    kw = dict(max_iter=6, gauge_mode=2, min_planes_per_pose=0, want_per_iter=True, force_hess=True)
    ref = _joint(sc, prec, [], [], on=False)
    ref.reset_counters()
    e_ref, lm_ref, ct_ref = ref.evaluate(x), ref.damping_iter(x, **kw), _counters(ref)
    for c in (_joint(sc, prec, [], [], on=True), _joint(sc, prec, fs, priors, on=False)):
        c.reset_counters()
        e, lm = c.evaluate(x), c.damping_iter(x, **kw)
        assert all(np.array_equal(u, v) for u, v in zip(e, e_ref))
        assert np.array_equal(lm[0], lm_ref[0]) and np.array_equal(lm[2], lm_ref[2]) and lm[1] == lm_ref[1]
        assert _counters(c) == ct_ref
        c.close()
    c = _joint(sc, prec, fs, priors)
    e1 = c.evaluate(x)
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
    c.set_pose_factors(fs[:3])
    c.set_pose_factors(fs)
    c.set_pose_priors([])
    c.set_pose_priors(priors)
    assert all(np.array_equal(u, v) for u, v in zip(c.evaluate(x), e1))
    c.set_joint_cost(False)
    assert all(np.array_equal(u, v) for u, v in zip(c.evaluate(x), e_ref))
    c.close()
    ref.close()


@pytest.mark.parametrize("loss", [LOSSES[0], LOSSES[2]], ids=["trivial", "cauchy"])
def test_fp64_lm_against_blocks(loss):
    sc, fs, priors, x0 = _scene(N=60, seed=35, every=6)
    kw = dict(max_iter=8, gauge_mode=2, min_planes_per_pose=0, want_per_iter=True)
    cd, cb = _joint(sc, L.PREC_FP64, fs, priors, loss), _blocks(sc, fs, priors, loss)
    _, td, pd = cd.damping_iter(x0, **kw)
    _, tb, pb = cb.damping_iter(x0, **kw)
    assert [t["accepted"] for t in td] == [t["accepted"] for t in tb]
    gap = np.abs(pd - pb).max()
    print(f"{loss[0]}: FP64 joint against blocks, largest per-iteration pose gap {gap:.2e}")
    assert gap <= 1e-9 and td[-1]["r2"] < td[0]["r1"] and not any(t["not_pd"] for t in td)
    cd.close()
    cb.close()


def _lm_oracle(cv, fs, priors, x0, max_iter, la, u0=0.01, v0=2.0, rel_tol=1e-6):
    """the LM rule on an FP64 voxel context plus pose_priors_ref's factors and priors, on the host"""
    N = cv.N
    x, u, v, calc = np.array(x0, copy=True), u0, v0, True
    acc, per = [], []
    for _ in range(max_iter):
        if calc:
            H, g, r1 = cv.evaluate(x)
            Hp, gp, rp = ppr.evaluate(x, fs, priors, N, **la)
            H, g, r1 = H + Hp, g + gp, r1 + rp
        D = np.diag(H).copy()
        dx = np.linalg.solve(H + u * np.diag(D), -g)
        q1 = 0.5 * dx @ (u * D * dx - g)
        xt = pgr.pose_update(x, dx)
        r2 = cv.residual(xt) + ppr.cost(xt, fs, priors, **la)
        q = r1 - r2
        if q > 0:
            x, u, v, calc = xt, u * max(1 - (2 * q / q1 - 1) ** 3, 1.0 / 3.0), 2.0, True
        else:
            u, v, calc = u * v, 2 * v, False
        acc.append(q > 0)
        per.append(x.copy())
        if rel_tol >= 0 and abs(r1 - r2) / r1 < rel_tol:
            break
    return acc, np.array(per)


@pytest.mark.parametrize("loss", [LOSSES[0], LOSSES[1]], ids=["trivial", "huber"])
def test_lm_against_the_host_oracle_and_tensor_against_fp64(loss):
    """on an all-see-all scene (the project's parity scenes; on a long corridor the tensor path's 1e-8 H error is
    amplified by the conditioning beyond 1e-6 m) with odometry, a window factor, GNSS and full-pose priors"""
    import scenes
    sc = scenes.make_scene(n_poses=30, n_planes=200, seed=26)
    rng = np.random.default_rng(37)
    gt = sc["poses_gt"]
    fs = _noisy_odometry(rng, gt, _odo_info()) + [pgr.make_factor(rng, gt, [3, 14, 27], noise=0.002)]
    priors = balm_b200.position_priors([0, 10, 20, 29], gt[[0, 10, 20, 29], 9:], 1e2 * np.eye(3))
    priors += ppr.random_priors(rng, gt, [4, 4, 22])
    x0 = sc["poses_init"]
    kw = dict(max_iter=8, gauge_mode=2, min_planes_per_pose=0, want_per_iter=True)
    cd, ct = _joint(sc, L.PREC_FP64, fs, priors, loss), _joint(sc, L.PREC_TENSOR, fs, priors, loss)
    cv = _joint(sc, L.PREC_FP64, [], [], loss, on=False)
    _, td, pd = cd.damping_iter(x0, **kw)
    acc, po = _lm_oracle(cv, fs, priors, x0, 8, _loss_arrays(loss, fs, priors))
    assert [t["accepted"] for t in td] == acc
    gap = np.abs(pd - po).max()
    _, tt, pt = ct.damping_iter(x0, **kw)
    assert [t["accepted"] for t in tt] == acc
    rot, pos = np.max([_pose_err(p, q) for p, q in zip(pt, pd)], axis=0)
    print(f"{loss[0]}: FP64 joint against the host oracle {gap:.2e}; TENSOR against FP64 rot {rot:.2e} pos {pos:.2e}")
    assert gap <= 1e-9 and rot <= 1e-6 and pos <= 1e-6
    for c in (cd, ct, cv):
        c.close()


def _tensor_run(sc, fs, priors, monkeypatch, reuse, **kw):
    if reuse:
        monkeypatch.delenv("BALM_NO_SWEEP_REUSE", raising=False)
    else:
        monkeypatch.setenv("BALM_NO_SWEEP_REUSE", "1")
    c = _joint(sc, L.PREC_TENSOR, fs, priors, on=bool(fs or priors))
    c.reset_counters()
    out = c.damping_iter(sc["poses_init"], max_iter=14, force_hess=True, rel_tol=-1.0, want_per_iter=True,
                         min_planes_per_pose=0, gauge_mode=2, **kw)
    ct = _counters(c)
    c.close()
    monkeypatch.delenv("BALM_NO_SWEEP_REUSE", raising=False)
    return out, ct


def test_tensor_carry_over_is_kept(monkeypatch):
    """A forced-Hessian tensor run with rejected steps: the joint cost reuses sweeps after rejections bitwise as a
    fresh sweep would, every evaluation but the first is a speculated single sweep, and the per-voxel stats are handed
    over (one stats pass per run). With terms too weak to move a bit, the run is the voxel-only one and its launch count
    grows by exactly the factor and prior kernels: 10 per evaluation and 6 per trial cost."""
    import scenes
    sc = scenes.make_scene(n_poses=24, n_planes=150, seed=57)
    gt = sc["poses_gt"]
    rng = np.random.default_rng(8)
    fs = _noisy_odometry(rng, gt, _odo_info()) + [pgr.make_factor(rng, gt, [2, 12, 20], noise=0.002)]
    priors = balm_b200.position_priors([0, 11, 23], gt[[0, 11, 23], 9:], 1e3 * np.eye(3))
    (p0, t0, per0), c0 = _tensor_run(sc, fs, priors, monkeypatch, False)
    (p1, t1, per1), c1 = _tensor_run(sc, fs, priors, monkeypatch, True)
    assert np.array_equal(per0, per1) and t0 == t1
    rejected = sum(1 for t in t1[:-1] if not t["accepted"])
    assert rejected >= 1 and c0["reused_sweeps"] == 0 and 1 <= c1["reused_sweeps"] <= rejected, (c1, t1)
    assert c1["single_sweeps"] + c1["redone_sweeps"] == c1["n_eval"] - 1 and c1["n_stats"] == 1, c1
    assert c1["n_residual"] == len(t1) + c1["refinements"]
    weak_fs = [dict(f, H=1e-30 * f["H"]) for f in fs]
    weak_pr = [dict(p, H=1e-30 * p["H"]) for p in priors]
    (pv, tv, perv), cv = _tensor_run(sc, [], [], monkeypatch, True)
    (pw, tw, perw), cw = _tensor_run(sc, weak_fs, weak_pr, monkeypatch, True)
    assert [t["accepted"] for t in tw] == [t["accepted"] for t in tv] and np.abs(perw - perv).max() <= 1e-12
    assert {k: v for k, v in cw.items() if k != "launches"} == {k: v for k, v in cv.items() if k != "launches"}
    assert cw["launches"] - cv["launches"] == 10 * cw["n_eval"] + 6 * cw["n_residual"], (cw, cv)


def _planeless(N=80, gap=np.arange(38, 42)):
    sc = bref.corridor(N, w=4, planes_per_pose=30, seed=34)
    keep = ~np.isin(sc["pose_idx"], gap)
    k = np.add.reduceat(keep.astype(np.int64), sc["row_ptr"][:-1])
    return dict(sc, pose_idx=sc["pose_idx"][keep], obs10=sc["obs10"][keep],
                row_ptr=np.concatenate([[0], np.cumsum(k)]).astype(np.int64))


@pytest.mark.parametrize("prec", DENSE)
def test_scans_without_planes_carried_by_odometry(prec):
    """four scans that see no plane: every step not_pd on the voxel cost; with odometry in the cost the LM converges,
    and to the blocks context's result with the same factors"""
    sc = _planeless()
    odo = _noisy_odometry(np.random.default_rng(4), sc["poses_gt"], _odo_info())
    c = _joint(sc, prec, odo, [], on=False)
    _, t, _ = c.damping_iter(sc["poses_init"], max_iter=3, gauge_mode=2, min_planes_per_pose=0)
    assert all(s["not_pd"] for s in t)
    c.set_joint_cost(True)
    kw = dict(max_iter=30, gauge_mode=2, min_planes_per_pose=0)
    x, t, _ = c.damping_iter(sc["poses_init"], **kw)
    assert not any(s["not_pd"] for s in t) and t[-1]["r2"] < t[0]["r1"]
    cb = _blocks(sc, odo, [])
    xb, tb, _ = cb.damping_iter(sc["poses_init"], **kw)
    rot, pos = _pose_err(x, xb)
    err = rfr.max_error(x, sc["poses_gt"])
    print(f"prec {prec}: {len(t)} iterations, position error after a rigid fit {err:.3f} m; against blocks "
          f"{rot:.1e} rad {pos:.1e} m")
    # the LM stops on rel_tol short of the optimum, where the tensor path's H error still moves the poses by microns
    tol = 1e-6 if prec == L.PREC_FP64 else 1e-5
    assert rot <= tol and pos <= tol and err < 0.1
    c.close()
    cb.close()


@pytest.mark.parametrize("prec", DENSE)
def test_gnss_corridor_in_the_priors_frame(prec):
    sc, odo, priors, x0 = _corridor(N=300)
    c = _joint(sc, prec, odo, priors)
    for gm in (0, 1):
        assert _status(lambda: c.damping_iter(x0, max_iter=2, gauge_mode=gm, min_planes_per_pose=0)) == L.ERR_INVALID
    x, _, _ = c.damping_iter(x0, max_iter=30, gauge_mode=2, min_planes_per_pose=0)
    assert _gnss_error(x0, sc).min() > 2.0 and _gnss_error(x, sc).max() < 0.3, _gnss_error(x, sc).max()
    c.set_joint_cost(False)  # the voxels and odometry alone leave the frame where the start put it
    xv, _, _ = c.damping_iter(x0, max_iter=30, gauge_mode=2, min_planes_per_pose=0)
    assert _gnss_error(xv, sc).min() > 1.0
    c.close()


def test_pose_covariance_with_priors_and_no_fix_clusters():
    """singular without the switch; with it, H_joint^-1 R H_joint^-T from the downloaded matrices, and the blocks
    context's block_point_covariance"""
    sc, fs, priors, x0 = _scene(N=60, seed=39, every=6)
    c = _joint(sc, L.PREC_FP64, fs, priors)
    x, _, _ = c.damping_iter(x0, max_iter=20, gauge_mode=2, min_planes_per_pose=0)
    c.set_joint_cost(False)
    assert _status(lambda: c.pose_covariance(x, point_noise=0.01)) == L.ERR_NOT_PD
    raw_v, _ = c.pose_covariance(x, point_noise=0.01, want_cov=False)
    c.set_joint_cost(True)
    raw, cov = c.pose_covariance(x, point_noise=0.01)
    assert np.array_equal(raw, raw_v)  # the terms shape H only
    H = c.evaluate(x)[0]
    S, kappa = _dense_sigma(H, -1)
    ref = S @ raw @ S.T
    err = _rel(cov, ref)
    print(f"kappa {kappa:.1e}: covariance against the dense inverse {err:.1e}")
    assert err <= max(1e-10, 10 * kappa * np.finfo(float).eps)
    cb = _blocks(sc, fs, priors)
    sel = np.array([0, 7, 30, 59], dtype=np.int32)
    Sb = cb.block_point_covariance(x, sel, point_noise=0.01, anchor=-1)
    idx = np.concatenate([np.arange(6 * s, 6 * s + 6) for s in sel])
    errb = _rel(Sb, cov[np.ix_(idx, idx)])
    print(f"blocks block_point_covariance against the dense joint covariance {errb:.1e}")
    assert errb <= max(1e-9, 100 * kappa * np.finfo(float).eps)
    c.close()
    cb.close()


def test_factors_and_priors_in_the_rig_cost():
    """the dense rig with the joint cost against a block-sparse rig with the same terms; rig_covariance runs with them"""
    sc = rb.rig_corridor(40, 3, w=2, seed=5)
    B, N = 40, 120
    base, ext = sc["base_init"], sc["ext_init"]
    X = rr.compose(sc["base12"], sc["ext12"], sc["base_of"], sc["lidar_of"])
    edges = [(s, s + 3) for s in range(N - 3)] + [(0, N - 3)]
    odo = balm_b200.odometry_factors(X, 1e3 * np.eye(6), edges=edges)
    # two GNSS fixes and a full-pose anchor: the gauge is fixed without a base anchor
    priors = balm_b200.position_priors([0, N - 1], X[[0, N - 1], 9:], 100 * np.eye(3))
    priors += balm_b200.pose_priors([0], X[[0]], 100 * np.eye(6))
    cd, cb = _joint(sc, L.PREC_FP64, odo, priors), _blocks(sc, odo, priors)
    cd.set_rig(sc["base_of"], sc["lidar_of"])
    cb.set_block_rig(sc["base_of"], sc["lidar_of"])
    for gm in (0, 1):
        assert _status(lambda: cd.rig_damping_iter(base, ext, gauge_mode=gm, min_planes_per_pose=0)) == L.ERR_INVALID
    Hd, gd, rd = cd.rig_evaluate(base, ext)
    Hb, gb, rb_ = cb.rig_evaluate(base, ext)
    assert _rel(Hd, Hb) < 1e-10 and _rel(gd, gb) < 1e-10 and abs(rd - rb_) <= 1e-12 * abs(rb_)
    cd.set_joint_cost(False)
    Hv, _, rv = cd.rig_evaluate(base, ext)
    assert rv < rd and not np.array_equal(Hv, Hd)
    cd.set_joint_cost(True)
    kw = dict(max_iter=5, gauge_mode=2, min_planes_per_pose=0, want_per_iter=True)
    bd, ed, td, perd = cd.rig_damping_iter(base, ext, **kw)
    _, _, tb, perb = cb.rig_damping_iter(base, ext, **kw)
    assert [t["accepted"] for t in td] == [t["accepted"] for t in tb] and td[0]["accepted"]
    _states_close(perd, perb, 1e-8)
    bd, ed, _ = cd.rig_damping_iter(bd, ed, max_iter=15, gauge_mode=2, min_planes_per_pose=0)
    raw, cov = cd.rig_covariance(bd, ed, point_noise=0.01, anchor=-1)
    H = cd.rig_evaluate(bd, ed)[0]
    S, kappa = _dense_sigma(H, -1)
    assert np.isfinite(cov).all() and _rel(cov, S @ raw @ S.T) <= max(1e-9, 10 * kappa * np.finfo(float).eps)
    cd.close()
    cb.close()


def test_refusals_and_repeatability():
    sc, fs, priors, x = _scene(N=40, seed=41, every=5)
    cb = _blocks(sc, fs, priors)
    e = cb.evaluate(x)
    assert _status(lambda: cb.set_joint_cost(True)) == L.ERR_INVALID
    assert all(np.array_equal(u, v) for u, v in zip(cb.evaluate(x), e))
    cb.close()
    assert L.lib().balm_set_joint_cost(None, 1) == L.ERR_INVALID
    c = _joint(sc, L.PREC_TENSOR, fs, priors)
    e = c.evaluate(x)
    with pytest.raises(balm_b200.BalmError) as err:
        c.comm_init(0, 2, None)
    assert err.value.status == L.ERR_INVALID and "joint cost" in str(err.value)
    assert all(np.array_equal(u, v) for u, v in zip(c.evaluate(x), e))
    kw = dict(max_iter=6, gauge_mode=2, min_planes_per_pose=0, want_per_iter=True, force_hess=True)
    a, b = c.damping_iter(x, **kw), c.damping_iter(x, **kw)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2]) and a[1] == b[1]
    c.close()

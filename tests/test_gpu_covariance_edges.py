"""GPU: the pose-covariance propagation (balm_pose_covariance / Context.pose_covariance in covariance.cu, and
balm_batch_pose_covariance for explicit c_cov) against the extended-precision reference of tests/cov_mp_ref.py, entry by
entry, at the n-right-hand-side solve's panel and tile edges, at every layout x voxel-batching combination, with
anisotropic and single-entry cluster covariances, far from the origin, and for the context state it leaves behind.

Tolerances (derivations in tests/cov_mp_ref.py):
  Rcov_raw  |raw - ref| <= 32 eps |Ls||c||Ls|^T + 16 sum_v e_v |Ls||c||Ls|^T   (raw_bound; e_v = eps mean|x|^2 / gap)
  Rcov      |cov - ref| <= C n kappa eps sqrt(ref_ii ref_jj), C = 1            (cov_bound)
            with ref = H^-1 raw H^-T from the device's own raw and its own H (Context.evaluate / Batch.evaluate at the
            same poses, pinned to the C oracle's H here), solved in double-double (n <= 198) or by LAPACK's Cholesky
            (n = 780, 1920: its own error obeys the same bound, so the tolerance doubles). kappa is the condition
            number of D^-1/2 H D^-1/2, n eps kappa the forward error of a backward-stable solve in those coordinates,
            and the propagation makes two solves; H^-1 and R meet the scale sqrt(ref_ii ref_jj) of the covariance's
            own correlations. Taking the oracle's H instead would add its difference from the device's (fp64 ~1e-12,
            tensor ~1e-9 relative) times kappa, which is not the propagation's error.
Every bound is checked to be non-vacuous: at most 1e-6 of the quantity it bounds."""
import numpy as np
import pytest

import cov_mp_ref as mr
import scenes
from oracle import oracle_py as orc

pytestmark = pytest.mark.gpu

PN = 0.01
C_COV = 1.0
VACUOUS = 1e-6


def _ctx(sc, prec, fix10="scene"):
    import balm_b200
    c = balm_b200.Context(sc["n_poses"], 0, prec)
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc["fix10"] if isinstance(fix10, str) else fix10)
    return c


def _check_raw(raw, R, A, E, what):
    bound = mr.raw_bound(A, E)
    nz = A > 0
    assert np.all(raw[~nz] == 0), what                      # pose pairs that share no voxel: exactly zero
    assert np.all(bound[nz] <= VACUOUS * A[nz]), what       # non-vacuous
    err = np.abs(raw - R)
    worst = (err[nz] / bound[nz]).max()
    print(f"{what}: Rcov_raw max |err| / bound {worst:.2e}")
    assert worst <= 1.0, what
    assert np.array_equal(raw, raw.T), what


def _check_cov(cov, H, raw, what, lapack=False):
    n = len(H)
    kappa = mr.kappa_scaled(H)
    assert np.isfinite(kappa), what
    ref = mr.cov_fp64(H, raw) if lapack else mr.cov_dd(H, raw)
    bound = mr.cov_bound(ref, kappa, n, C_COV) * (2 if lapack else 1)
    scale = np.sqrt(np.outer(np.diag(ref), np.diag(ref)))
    if bound.max() > VACUOUS * scale.max():
        pytest.fail(f"{what}: kappa(D^-1/2 H D^-1/2) = {kappa:.2e} makes the bound vacuous ({bound.max() / scale.max():.1e})")
    err = np.abs(cov - ref)
    worst = (err / bound).max()
    print(f"{what}: kappa {kappa:.2e}, Rcov max |err| / bound {worst:.2e} (max |err| / scale {(err / scale).max():.1e})")
    assert worst <= 1.0, what
    return kappa


def _check_H(H, sc, poses, fix10, tol):
    o = orc.Oracle(sc["n_poses"], sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], fix10)
    Ho = o.evaluate(poses, include_fix=True)[0]
    assert np.abs(H - Ho).max() <= tol * np.abs(Ho).max()


# ---------------- panel and tile edges of solve_many (64-wide panels, 64-column tiles) ----------------
# n = 60 (one partial panel), 66 (a panel and a 2-row sliver), 192 (three full panels), 198 (three and a sliver),
# 780 (twelve and a 12-row sliver), 1920 (thirty full panels: the backward update loops over up to 29 panels)
EDGES = [(10, 30), (11, 30), (32, 24), (33, 24), (130, 14), (320, 10)]


@pytest.fixture(scope="module")
def edge_runs():
    import balm_b200
    out = {}
    for N, M in EDGES:
        sc = scenes.make_scene(n_poses=N, n_planes=M, seed=100 + N, with_fix=True, pts_size=20)
        x = sc["poses_gt"]
        res = {}
        for prec in (balm_b200.PREC_FP64, balm_b200.PREC_TENSOR):
            c = _ctx(sc, prec)
            raw, cov = c.pose_covariance(x, point_noise=PN, include_fix=True)
            H = c.evaluate(x, include_fix=True)[0]
            c.close()
            res[prec] = (raw, cov, H)
        out[N] = (sc, x, res, mr.raw_reference(N, sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], x, sc["fix10"],
                                                pnoise=PN))
    return out


@pytest.mark.parametrize("N", [e[0] for e in EDGES])
def test_panel_and_tile_edges(edge_runs, N):
    import balm_b200
    sc, x, res, (R, A, E) = edge_runs[N]
    for prec, tolH in ((balm_b200.PREC_FP64, 1e-9), (balm_b200.PREC_TENSOR, 1e-8)):
        raw, cov, H = res[prec]
        what = f"N={N} prec={prec}"
        _check_raw(raw, R, A, E, what)
        _check_H(H, sc, x, sc["fix10"], tolH)
        _check_cov(cov, H, raw, what, lapack=6 * N > 200)
    # Rcov_raw takes the same path in both precisions (the fp64 DMMA SYRK over the same rows, ldg = 6N rounded up to
    # 128 in both); only the SYRK's k-split count could differ, and with 3 M < 512 rows per evaluation both take one
    assert 3 * len(sc["coe"]) < 512
    assert np.array_equal(res[balm_b200.PREC_FP64][0], res[balm_b200.PREC_TENSOR][0])


# ---------------- layouts x voxel batching ----------------
@pytest.mark.parametrize("drop", [0.0, 0.5])
@pytest.mark.parametrize("budget_mb", [None, 1])
def test_layouts_and_voxel_batches(monkeypatch, drop, budget_mb):
    """Dense (every pose sees every voxel, diagonal blocks summed by slot) and sparse (per-pose lists) layouts, in one
    voxel batch and in several: with a 1 MiB row budget a batch holds 2^20 / (8 rows x 128 columns x 8 B) = 128 voxels,
    so M = 300 runs as 128 + 128 + 44 and cov_diag_reduce_kernel adds to the earlier batches' sums."""
    import balm_b200
    sc = scenes.make_scene(n_poses=14, n_planes=300, seed=120, drop=drop, with_fix=True, pts_size=10)
    x = sc["poses_gt"]
    if budget_mb:
        monkeypatch.setenv("BALM_COV_BUDGET_MB", str(budget_mb))
    c = _ctx(sc, balm_b200.PREC_FP64)
    raw, cov = c.pose_covariance(x, point_noise=PN, include_fix=True)
    monkeypatch.delenv("BALM_COV_BUDGET_MB", raising=False)
    H = c.evaluate(x, include_fix=True)[0]
    c.close()
    R, A, E = mr.raw_reference(14, sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], x, sc["fix10"], pnoise=PN)
    what = f"drop={drop} budget={budget_mb}"
    _check_raw(raw, R, A, E, what)
    _check_H(H, sc, x, sc["fix10"], 1e-9)
    _check_cov(cov, H, raw, what)


# ---------------- anisotropic and single-entry cluster covariances ----------------
@pytest.mark.parametrize("drop", [0.0, 0.4])
def test_anisotropic_ccov_context(drop):
    import balm_b200
    sc = scenes.make_scene(n_poses=9, n_planes=40, seed=130, drop=drop, with_fix=True, pts_size=20)
    x = sc["poses_gt"]
    cc = mr.random_spd_ccov(sc["obs10"], PN, np.random.default_rng(131))
    c = _ctx(sc, balm_b200.PREC_FP64)
    raw, cov = c.pose_covariance(x, c_cov=cc, include_fix=True)
    H = c.evaluate(x, include_fix=True)[0]
    c.close()
    R, A, E = mr.raw_reference(9, sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], x, sc["fix10"], c_cov=cc)
    _check_raw(raw, R, A, E, f"context anisotropic drop={drop}")
    _check_cov(cov, H, raw, f"context anisotropic drop={drop}")


def _prob(sc, fix10="scene"):
    return dict(n_poses=sc["n_poses"], row_ptr=sc["row_ptr"], pose_idx=sc["pose_idx"], obs10=sc["obs10"],
                coe=sc["coe"], fix10=sc["fix10"] if isinstance(fix10, str) else fix10)


def _batch(problems):
    import balm_b200
    b = balm_b200.Batch(0)
    b.set_problems(problems)
    return b


def test_anisotropic_ccov_batch():
    """Problems of 1, 2, 17 and 32 poses (batch_cov_solve_kernel at n = 6, 12, 102, 192), each observation its own SPD
    c_cov."""
    rng = np.random.default_rng(140)
    scs = []
    for N, M, drop in ((2, 25, 0.0), (2, 30, 0.0), (17, 50, 0.3), (32, 40, 0.0)):
        scs.append(scenes.make_scene(n_poses=N, n_planes=M, seed=141 + N + M, drop=drop, with_fix=True, pts_size=20))
    s0 = scs[0]  # one pose: pose 0's observations of a two-pose scene
    keep = s0["pose_idx"] == 0
    counts = np.add.reduceat(keep.astype(np.int64), s0["row_ptr"][:-1])
    scs[0] = dict(s0, n_poses=1, row_ptr=np.concatenate([[0], np.cumsum(counts)]).astype(np.int64),
                  pose_idx=s0["pose_idx"][keep], obs10=s0["obs10"][keep], poses_gt=s0["poses_gt"][:1])
    cc = [mr.random_spd_ccov(s["obs10"], PN, rng) for s in scs]
    poses = [s["poses_gt"] for s in scs]
    b = _batch([_prob(s) for s in scs])
    got = b.pose_covariance(poses, c_cov=cc, include_fix=True)
    Hs = [h[0] for h in b.evaluate(poses, include_fix=True)]
    b.close()
    for s, x, c, (st, raw, cov), H in zip(scs, poses, cc, got, Hs):
        N = s["n_poses"]
        assert st == 0
        R, A, E = mr.raw_reference(N, s["row_ptr"], s["pose_idx"], s["obs10"], s["coe"], x, s["fix10"], c_cov=c)
        _check_raw(raw, R, A, E, f"batch anisotropic N={N}")
        _check_H(H, s, x, s["fix10"], 1e-9)
        _check_cov(cov, H, raw, f"batch anisotropic N={N}")


def test_ccov_layout_probe():
    """Every parameter pair (e, f) on its own: c_cov with only (e, f) and (f, e) set, the same for every observation.
    Each of the 45 results is Ls_e Ls_f^T + Ls_f Ls_e^T: any transposed, shifted or dropped index of the user's c_cov
    (context: load_ccov; batch: batch_cov_rows_kernel) or of the terms built from it shows in its own call."""
    import balm_b200
    sc = scenes.make_scene(n_poses=3, n_planes=6, seed=150, drop=0.0, with_fix=True, pts_size=15)
    x = sc["poses_init"]
    K, N = len(sc["obs10"]), 3
    terms = list(mr.voxel_terms(N, sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], x, sc["fix10"]))
    # rounding scale: one column of Ls is computed from the same intermediate products as the other eight, so its
    # error is relative to the whole row of Ls, not to the column -- |Ls| J |Ls|^T with J the all-ones 9 x 9
    _, A, E = mr.accumulate(N, terms, np.ones((K, 9, 9)))
    c = _ctx(sc, balm_b200.PREC_FP64)
    b = _batch([_prob(sc)])
    for e in range(9):
        for f in range(e, 9):
            cc = np.broadcast_to(mr.pair_ccov(e, f), (K, 9, 9)).copy()
            R = mr.accumulate(N, terms, cc)[0]
            raw_c, _ = c.pose_covariance(x, c_cov=cc, include_fix=True, want_cov=False)
            st, raw_b, _ = b.pose_covariance([x], c_cov=[cc], include_fix=True, want_cov=False)[0]
            assert st == 0
            _check_raw(raw_c, R, A, E, f"context c_cov ({e}, {f})")
            _check_raw(raw_b, R, A, E, f"batch c_cov ({e}, {f})")
    c.close()
    b.close()


# ---------------- far from the origin ----------------
SHIFT = np.array([0.6, -0.48, 0.64])  # unit vector


@pytest.mark.parametrize("offset", [0.0, 100.0, 1000.0])
def test_off_origin(offset):
    """The same scene (planes within +-20 m) moved by 0, 100 and 1000 m: poses and fix clusters moved, body-frame
    observations unchanged. With the fix clusters H is accepted by both the context and the batch and matches the
    reference; without them the gauge is free and both refuse it."""
    import balm_b200
    from balm_b200 import _lib
    sc = scenes.make_scene(n_poses=10, n_planes=40, seed=160, with_fix=True, pts_size=20, surf_range=20.0)
    x, fix = mr.shift_scene(sc, offset * SHIFT, sc["poses_gt"])
    c = _ctx(sc, balm_b200.PREC_FP64, fix)
    raw, cov = c.pose_covariance(x, point_noise=PN, include_fix=True)
    H = c.evaluate(x, include_fix=True)[0]
    R, A, E = mr.raw_reference(10, sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], x, fix, pnoise=PN)
    what = f"offset {offset:g} m"
    _check_raw(raw, R, A, E, what)
    kappa = _check_cov(cov, H, raw, what)
    d = np.diag(np.linalg.cholesky(H)) ** 2
    print(f"{what}: LDL^T pivots min/max {d.min() / d.max():.1e}, kappa(H) {np.linalg.cond(H):.1e}, "
          f"kappa(D^-1/2 H D^-1/2) {kappa:.1e}")
    b = _batch([_prob(sc, fix)])
    st, raw_b, cov_b = b.pose_covariance([x], point_noise=PN, include_fix=True)[0]
    assert st == _lib.OK
    _check_raw(raw_b, R, A, E, what + " batch")
    _check_cov(cov_b, b.evaluate([x], include_fix=True)[0][0], raw_b, what + " batch")
    with pytest.raises(balm_b200.BalmError) as e:
        c.pose_covariance(x, point_noise=PN, include_fix=False)
    assert e.value.status == _lib.ERR_NOT_PD
    st, _, cov_b = b.pose_covariance([x], point_noise=PN, include_fix=False)[0]
    assert st == _lib.ERR_NOT_PD and not cov_b.any()
    c.close()
    b.close()


def test_small_scene_one_km_out_is_refused():
    """A 5 m scene 1 km from the origin: in the pose-update coordinates a rotation moves a pose by |p| times the angle,
    so H's rotation rows are ~|p|^2 / (5 m)^2 larger than its translation rows and nearly parallel to them. Scaled,
    kappa(D^-1/2 H D^-1/2) ~ 2e8, while forming H in fp64 from world-frame moments of size |p|^2 costs e_v ~ 1e-9 of
    it: no fp64 H^-1 carries a correct digit (kappa e_v ~ 0.2). The raw-pivot rule (min d <= 1e-11 max d) refuses it,
    which is the right outcome; the same scene at 100 m, and a 40 m scene at 1 km (test_off_origin), are accepted."""
    import balm_b200
    from balm_b200 import _lib
    sc = scenes.make_scene(n_poses=10, n_planes=40, seed=5, with_fix=True, pts_size=20)
    for offset, ok in ((100.0, True), (1000.0, False)):
        x, fix = mr.shift_scene(sc, offset * SHIFT, sc["poses_gt"])
        H = orc.Oracle(10, sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], fix).evaluate(x, include_fix=True)[0]
        kappa = mr.kappa_scaled(H)
        e_v = mr.EPS * offset ** 2 / (1 / 12)
        print(f"5 m scene at {offset:g} m: kappa(D^-1/2 H D^-1/2) {kappa:.1e}, kappa e_v {kappa * e_v:.1e}")
        assert (kappa * e_v < 1e-3) == ok
        c = _ctx(sc, balm_b200.PREC_FP64, fix)
        b = _batch([_prob(sc, fix)])
        st = b.pose_covariance([x], point_noise=PN, include_fix=True)[0][0]
        try:
            c.pose_covariance(x, point_noise=PN, include_fix=True)
            st_c = _lib.OK
        except balm_b200.BalmError as e:
            st_c = e.status
        assert st_c == st == (_lib.OK if ok else _lib.ERR_NOT_PD)
        c.close()
        b.close()


# ---------------- the context after pose_covariance ----------------
@pytest.mark.parametrize("prec", [0, 1])
def test_context_state_after_pose_covariance(monkeypatch, prec):
    """pose_covariance overwrites the stats table, the per-batch CSC lists (several voxel batches here) and the
    evaluated H; an evaluate and a damping_iter afterwards are bitwise those of a context that never ran it (in a
    tensor context that includes the speculative column scales of the LM loop)."""
    sc = scenes.make_scene(n_poses=12, n_planes=300, seed=170, drop=0.4, with_fix=True, pts_size=10)
    x0 = sc["poses_init"]

    def run(cov_first):
        c = _ctx(sc, prec)
        if cov_first:
            monkeypatch.setenv("BALM_COV_BUDGET_MB", "1")
            c.pose_covariance(sc["poses_gt"], point_noise=PN, include_fix=True)
            monkeypatch.delenv("BALM_COV_BUDGET_MB")
        H, g, r = c.evaluate(x0)
        poses, tr, _ = c.damping_iter(x0, max_iter=4, gauge_mode=2, hess_includes_fix=True)
        H2, g2, r2 = c.evaluate(poses, include_fix=True)
        c.close()
        return H, g, r, poses, tr, H2, g2, r2

    a, b = run(True), run(False)
    for u, v in zip(a, b):
        if isinstance(u, list):
            assert u == v
        else:
            assert np.array_equal(u, v)

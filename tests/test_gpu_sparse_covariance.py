"""Marginal pose covariances on the sparse solve (balm_spg_covariance / PoseGraph.covariance, balm_block_covariance /
Context.block_covariance): against dense and sparse inverses of the same H, a Monte-Carlo check of their meaning, and
the call's contracts (gauge, singular cases, repeatability, side effects, memory)."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse.linalg as spla

import balm_b200
import block_hessian_ref as bref
import pose_graph_ref as pg
from balm_b200 import _lib as L
from test_gpu_block_hessian import SCENES, _ctx
from test_gpu_pose_graph_sparse import KINDS, _covered, _factor_set, _pyramid, _sparse

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps


def _dense_sigma(H, anchor):
    """(H without pose anchor's rows and columns)^-1 padded with zeros, and the condition number of what was inverted."""
    keep = np.ones(len(H), bool)
    if anchor >= 0:
        keep[6 * anchor:6 * anchor + 6] = False
    Ht = H[np.ix_(keep, keep)]
    S = np.zeros_like(H)
    S[np.ix_(keep, keep)] = np.linalg.inv(Ht)
    return S, np.linalg.cond(Ht)


def _check_against(cov, pairs, S, kappa, what):
    ref = bref.blocks_of(S, pairs)
    scale = np.abs(ref).max()
    err = np.abs(cov - ref).max() / scale
    # both inverses carry rounding of order kappa eps relative to max |Sigma|; 1e-9 unless kappa says otherwise
    tol = max(1e-9, 10 * kappa * EPS)
    print(f"{what}: kappa {kappa:.1e}, error {err:.1e} of max |Sigma|, tolerance {tol:.0e}")
    assert err <= tol


def _anchor_contract(cov, pairs, anchor):
    touch = (pairs[:, 0] == anchor) | (pairs[:, 1] == anchor)
    assert not cov[touch].any()
    diag = (pairs[:, 0] == pairs[:, 1]) & ~touch
    d = cov[diag]
    assert np.array_equal(d, d.transpose(0, 2, 1))
    assert np.linalg.eigvalsh(d).min() > 0


# ---------------- against a dense inverse ----------------
@pytest.mark.parametrize("kind", KINDS + ["loops"])
def test_pose_graph_against_the_dense_inverse(kind):
    P, factors, x = _factor_set(kind)
    c = balm_b200.Context(P)
    c.set_pose_factors(factors)
    H = c.pose_graph_evaluate(x)[0]
    s = _sparse(P, factors)
    for anchor in (0, P // 2):
        if not _covered(P, factors):  # a pose in no factor: H~ is singular whatever the anchor
            with pytest.raises(balm_b200.BalmError) as e:
                s.covariance(x, anchor)
            assert e.value.status == L.ERR_NOT_PD
            continue
        pairs, cov = s.covariance(x, anchor)
        S, kappa = _dense_sigma(H, anchor)
        _check_against(cov, pairs, S, kappa, f"{kind} anchor {anchor}")
        _anchor_contract(cov, pairs, anchor)
    c.close()
    s.close()


def _converged(sc, prec, include_fix):
    c = _ctx(sc, prec)
    x, _, _ = c.damping_iter(sc["poses_init"], max_iter=10, gauge_mode=2, min_planes_per_pose=0,
                             hess_includes_fix=include_fix)
    return c, x


@pytest.mark.parametrize("name", list(SCENES))
def test_blocks_against_the_dense_inverse(name):
    sc = SCENES[name]()
    with_fix = sc.get("fix10") is not None
    include_fix, anchor = (True, -1) if with_fix else (False, 0)
    cb, x = _converged(sc, L.PREC_BLOCKS, include_fix)
    pairs, cov = cb.block_covariance(x, include_fix=include_fix, anchor=anchor)
    assert np.array_equal(pairs, cb.block_structure(want_pairs=True)["pair_list"])
    H = cb.evaluate(x, include_fix=include_fix)[0]
    S, kappa = _dense_sigma(H, anchor)
    _check_against(cov, pairs, S, kappa, f"{name} blocks")
    _anchor_contract(cov, pairs, anchor)
    # the fp64 context's H agrees with the blocks' to 1e-12 max |H| (test_gpu_block_hessian); Sigma moves by kappa times that
    cd = _ctx(sc, L.PREC_FP64)
    Hd = cd.evaluate(x, include_fix=include_fix)[0]
    Sd, _ = _dense_sigma(Hd, anchor)
    err = np.abs(cov - bref.blocks_of(Sd, pairs)).max() / np.abs(cov).max()
    print(f"{name}: against the fp64 context's H {err:.1e}")
    assert err <= max(1e-9, 10 * kappa * 1e-12)
    cb.close()
    cd.close()


# ---------------- at size, against sparse LU columns ----------------
def _columns(Hs, N, anchor, poses):
    """Sigma[:, 6 q .. 6 q + 6] for each q in poses, from a sparse LU of H without the anchor's rows and columns."""
    keep = np.ones(6 * N, bool)
    if anchor >= 0:
        keep[6 * anchor:6 * anchor + 6] = False
    lu = spla.splu(Hs[keep][:, keep].tocsc())
    out = {}
    for q in poses:
        E = np.zeros((6 * N, 6))
        E[6 * q:6 * q + 6] = np.eye(6)
        X = np.zeros((6 * N, 6))
        X[keep] = lu.solve(E[keep])
        out[q] = X
    return out


def _check_columns(N, pairs, cov, Hs, anchor, what):
    pick = sorted({0, 1, N // 2 - 1, N // 2, N - 1, *np.random.default_rng(0).choice(N, 3, replace=False).tolist()})
    cols = _columns(Hs, N, anchor, [q for q in pick if q != anchor])
    num = den = 0.0
    for p, (i, j) in enumerate(pairs):
        for q, X in cols.items():
            if j == q:
                ref = X[6 * i:6 * i + 6]
            elif i == q:
                ref = X[6 * j:6 * j + 6].T
            else:
                continue
            num = max(num, np.abs(cov[p] - ref).max())
            den = max(den, np.abs(ref).max())
    print(f"{what}: {len(cols)} poses' columns against splu, error {num / den:.1e} of their max |Sigma|")
    assert num <= 1e-9 * den


def test_pose_graph_at_4541_poses():
    N = 4541
    factors, x = _pyramid(N, 13)
    s = _sparse(N, factors)
    pairs, blocks, _, _ = s.pose_graph_evaluate(x)
    pc, cov = s.covariance(x, 0)
    assert np.array_equal(pc, pairs)
    _check_columns(N, pairs, cov, bref.to_sparse(N, pairs, blocks), 0, "pyramid 4541")
    s.close()


def test_blocks_at_5000_poses(monkeypatch):
    # In the pose-update coordinates a rotation moves a pose by its distance from the origin times the angle, and a long
    # chain bends; both condition H worse the longer the corridor. At the truth of 5 000 poses (scipy eigsh): kappa(H)
    # 3e12 over 1 km with fix clusters and 4e12 over 100 m anchored at pose 0 without them, past the 1e-11 pivot rule;
    # 4e8 over 100 m with them. corridor() spreads N poses over min(1 km, N m); this one spans 100 m.
    monkeypatch.setattr(bref, "min", lambda a, b: 100.0 / 5000, raising=False)  # corridor's step = min(1.0, 1000 / N)
    sc = bref.corridor(5000, w=8, planes_per_pose=30, seed=7, with_fix=True)
    monkeypatch.undo()
    c, x = _converged(sc, L.PREC_BLOCKS, True)
    pairs, cov = c.block_covariance(x, include_fix=True, anchor=-1)
    blocks = c.download_blocks()  # H at x: the covariance call's evaluation
    _check_columns(5000, pairs, cov, bref.to_sparse(5000, pairs, blocks), -1, "corridor 5000")
    c.close()


# ---------------- meaning: a Monte-Carlo check ----------------
def test_monte_carlo_consistency():
    """Residuals drawn from the factors' own noise model, placed exactly; the anchored estimate's error in the pose-update
    coordinates has covariance Sigma, so delta_i^T Sigma_ii^-1 delta_i averages 6."""
    P, draws = 40, 400
    rng = np.random.default_rng(21)
    truth = np.array([pg.random_pose(rng, 0.5, 3.0) for _ in range(P)])
    sets = pg.pyramid_factor_poses(P, top=8)
    Hs = [1e6 * pg.window_hessian(rng, len(s), cond=10.0) for s in sets]  # residual std <= 1e-3
    frames = [pg.random_pose(rng) for _ in sets]
    chols = [np.linalg.cholesky(H[6:, 6:]) for H in Hs]
    R0, p0 = pg.split(truth[0])
    chi = np.zeros((draws, P - 1))
    s = balm_b200.PoseGraph(P)
    for d in range(draws):
        factors = []
        for idx, H, G, Lc in zip(sets, Hs, frames, chols):
            eps = np.linalg.solve(Lc.T, rng.normal(size=6 * (len(idx) - 1))).reshape(-1, 6)  # N(0, H[6:, 6:]^-1)
            hat = np.array([pg.compose(G, truth[i]) for i in idx])  # X_k = A^-1 T_k with A = G^-1
            for k in range(1, len(idx)):
                Rx, px = pg.split(hat[k])
                Et = pg.exp_so3(eps[k - 1, :3]).T
                hat[k] = pg.pack(Et @ Rx, Et @ (px - eps[k - 1, 3:]))
            factors.append(dict(poses=np.asarray(idx, np.int32), poses_hat=hat, H=H))
        assert s.set_pose_factors(factors) == [L.OK] * len(factors)
        est, tr = s.pose_graph_iter(truth, max_iter=20, rel_tol=1e-12, gauge_mode=2)
        # aligned at the anchor, est <- T_true0 T_est0^-1 est, and Sigma there: a common left transform changes the
        # pose-update coordinates (by its adjoint), so Sigma and delta must be taken in the same frame
        Re0, pe0 = pg.split(est[0])
        Ra = R0 @ Re0.T
        al = np.array([pg.pack(Ra @ pg.split(e)[0], Ra @ (pg.split(e)[1] - pe0) + p0) for e in est])
        pairs, cov = s.covariance(al, 0)
        diag = {int(i): cov[p] for p, (i, j) in enumerate(pairs) if i == j}
        for i in range(1, P):
            Rn, pn = pg.split(al[i])
            Rt, pt = pg.split(truth[i])
            th = pg.log_so3(Rn @ Rt.T)
            delta = np.concatenate([th, pn - pg.exp_so3(th) @ pt])
            chi[d, i - 1] = delta @ np.linalg.solve(diag[i], delta)
    s.close()
    per_pose = chi.mean(0)
    print(f"pooled mean {chi.mean():.3f}, per pose {per_pose.min():.2f} .. {per_pose.max():.2f}")
    assert 5.6 <= chi.mean() <= 6.4
    assert np.all((per_pose >= 5.0) & (per_pose <= 7.0))


# ---------------- edges and contracts ----------------
def test_singular_and_invalid_calls():
    for kind, anchor in (("split", 0), ("hole", 0), ("pyramid", -1)):
        P, factors, x = _factor_set(kind)
        s = _sparse(P, factors)
        with pytest.raises(balm_b200.BalmError) as e:
            s.covariance(x, anchor)
        assert e.value.status == L.ERR_NOT_PD and "singular" in str(e.value)
        s.close()
    P, factors, x = _factor_set("pyramid")
    s = _sparse(P, factors)
    for anchor in (-2, P):
        with pytest.raises(balm_b200.BalmError) as e:
            s.covariance(x, anchor)
        assert e.value.status == L.ERR_INVALID
    buf = np.zeros(36 * s.structure()["pairs"])
    lib = L.lib()
    assert lib.balm_spg_covariance(s._h, None, 0, buf.ctypes.data) == L.ERR_INVALID
    assert lib.balm_spg_covariance(s._h, x.ctypes.data, 0, None) == L.ERR_INVALID
    s2 = balm_b200.PoseGraph(P)
    assert lib.balm_spg_covariance(s2._h, x.ctypes.data, 0, buf.ctypes.data) == L.ERR_INVALID  # nothing registered
    s.close()
    s2.close()
    sc = SCENES["corridor40"]()
    cb = _ctx(sc, L.PREC_BLOCKS)
    with pytest.raises(balm_b200.BalmError) as e:  # no fix clusters: the gauge is free
        cb.block_covariance(sc["poses_gt"], anchor=-1)
    assert e.value.status == L.ERR_NOT_PD
    for anchor in (-2, sc["n_poses"]):
        with pytest.raises(balm_b200.BalmError) as e:
            cb.block_covariance(sc["poses_gt"], anchor=anchor)
        assert e.value.status == L.ERR_INVALID
    cd = _ctx(sc, L.PREC_FP64)
    out = np.zeros(36 * 1000)
    assert lib.balm_block_covariance(cd._h, sc["poses_gt"].ctypes.data, 0, 0, out.ctypes.data) == L.ERR_INVALID
    assert not out.any()
    empty = balm_b200.Context(sc["n_poses"], 0, L.PREC_BLOCKS)
    assert lib.balm_block_covariance(empty._h, sc["poses_gt"].ctypes.data, 0, 0, out.ctypes.data) == L.ERR_INVALID
    for c in (cb, cd, empty):
        c.close()


def test_repeatable_and_permutation_equivariant():
    P, factors, x = _factor_set("loops", seed=3)
    anchor = 17
    a = _sparse(P, factors)
    pa, ca = a.covariance(x, anchor)
    pa2, ca2 = a.covariance(x, anchor)
    assert np.array_equal(pa, pa2) and np.array_equal(ca, ca2)
    perm = np.random.default_rng(7).permutation(P)  # pose i of the original is pose perm[i] of the permuted set
    fperm = [dict(f, poses=perm[f["poses"]].astype(np.int32)) for f in factors]
    xperm = np.empty_like(x)
    xperm[perm] = x
    b = _sparse(P, fperm)
    pb, cb = b.covariance(xperm, int(perm[anchor]))
    lookup = {(int(i), int(j)): cb[p] for p, (i, j) in enumerate(pb)}
    scale = np.abs(ca).max()
    for p, (i, j) in enumerate(pa):
        u, v = int(perm[i]), int(perm[j])
        blk = lookup[(u, v)] if u <= v else lookup[(v, u)].T
        assert np.abs(blk - ca[p]).max() <= 1e-8 * scale
    a.close()
    b.close()


def test_lm_is_unchanged_by_a_covariance_call():
    P, factors, x = _factor_set("loops", seed=4)
    runs = []
    for with_cov in (False, True):
        s = _sparse(P, factors)
        x1, t1 = s.pose_graph_iter(x, max_iter=3, gauge_mode=2)
        if with_cov:
            y = x1.copy()
            y[:, 9:] += 0.01
            s.covariance(y, 0)  # other poses: blocks, g and the factor change
        x2, t2 = s.pose_graph_iter(x1, max_iter=3, gauge_mode=2)
        runs.append((x2, str(t2)))
        s.close()
    assert np.array_equal(runs[0][0], runs[1][0]) and runs[0][1] == runs[1][1]
    sc = SCENES["corridor300"]()
    runs = []
    for with_cov in (False, True):
        c = _ctx(sc, L.PREC_BLOCKS)
        x1, _, _ = c.damping_iter(sc["poses_init"], max_iter=3, min_planes_per_pose=0)
        if with_cov:
            c.block_covariance(sc["poses_gt"], include_fix=True, anchor=-1)
        x2, t2, _ = c.damping_iter(x1, max_iter=3, min_planes_per_pose=0)
        runs.append((x2, str(t2)))
        c.close()
    assert np.array_equal(runs[0][0], runs[1][0]) and runs[0][1] == runs[1][1]


def test_device_bytes_grow_only_on_the_first_call():
    P, factors, x = _factor_set("loops", seed=5)
    s = _sparse(P, factors)
    reg = s.structure()["device_bytes"]
    s.pose_graph_iter(x, max_iter=2)
    assert s.structure()["device_bytes"] == reg
    s.covariance(x, 0)
    grown = s.structure()["device_bytes"]
    assert grown > reg
    s.covariance(x, 3)
    assert s.structure()["device_bytes"] == grown
    s.set_pose_factors(factors)
    assert s.structure()["device_bytes"] == reg
    s.close()
    sc = SCENES["corridor300"]()
    c = _ctx(sc, L.PREC_BLOCKS)
    reg = c.block_structure()["device_bytes"]
    c.block_covariance(sc["poses_gt"], include_fix=True, anchor=-1)
    assert c.block_structure()["device_bytes"] > reg
    blocks = c.download_blocks()  # H at the covariance call's poses
    H = c.evaluate(sc["poses_gt"], include_fix=True)[0]
    assert np.array_equal(blocks, bref.blocks_of(H, c.block_structure(want_pairs=True)["pair_list"]))
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc["fix10"])
    assert c.block_structure()["device_bytes"] == reg
    c.close()

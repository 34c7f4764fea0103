"""balm_block_point_covariance / balm_rig_block_point_covariance (Context.block_point_covariance,
Context.rig_block_point_covariance): the raw term against an FP64 context's pose_covariance on the pattern, Sigma against
the dense sandwiches and the restatement (tests/block_point_cov_ref.py), the rig against balm_rig_covariance and the plain
call, bitwise properties, scale against scipy.sparse, a Monte-Carlo check of the meaning, and the refusals."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse as sps
import scipy.sparse.linalg as spla
from scipy import stats

import balm_b200
import block_hessian_ref as bref
import block_point_cov_ref as bp
import numpy_cov as nc
import pose_graph_ref as pg
import rig_blocks_ref as rb
import rig_cov_ref as rc
import rig_ref as rr
import robust_voxels_ref as rv
from balm_b200 import _lib as L
from balm_b200.rig import extrinsic_sigmas
from scenes import make_scene, unpack_pose
from test_gpu_rig import rig_case

pytestmark = pytest.mark.gpu

PN = 0.01
TOLRAW = 1e-12   # of max |R|
TOLCOV = 1e-7    # of max |Sigma|


def _ctx(sc, prec, loss=None):
    c = balm_b200.Context(sc["n_poses"], 0, prec)
    if loss is not None:
        c.set_voxel_loss(*loss)
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc.get("fix10"))
    return c


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300)


def _status(fn):
    with pytest.raises(balm_b200.BalmError) as e:
        fn()
    return e.value.status


def _converged(ctx, x):
    """the LM optimum: away from it the voxel cost's H can be indefinite (BALM_ERR_NOT_PD)"""
    return ctx.damping_iter(x, max_iter=20, rel_tol=1e-12, gauge_mode=2, min_planes_per_pose=0)[0]


def _c_cov(sc, seed=3):
    rng = np.random.default_rng(seed)
    return np.stack([nc.cluster_cov_isotropic(o, PN * rng.uniform(0.5, 2.0)) for o in sc["obs10"]])


@pytest.mark.parametrize("name", ["dense", "ragged", "fix"])
@pytest.mark.parametrize("loss", [None, "cauchy"])
def test_raw_blocks_match_the_dense_raw_term(name, loss):
    sc = rig_case(name)[0]
    x = sc["poses_init"]
    include_fix = sc.get("fix10") is not None
    lo = None
    if loss:
        lo = (loss, float(np.sqrt(np.median(rv.lams(sc, x, include_fix)))))
    blk, dense = _ctx(sc, L.PREC_BLOCKS, lo), _ctx(sc, L.PREC_FP64, lo)
    pairs = blk.block_structure(want_pairs=True)["pair_list"]
    for kw in (dict(point_noise=PN), dict(c_cov=_c_cov(sc))):
        Rd, _ = dense.pose_covariance(x, include_fix=include_fix, want_cov=False, **kw)
        _, (p2, raw) = blk.block_point_covariance(x, [0], include_fix=include_fix, anchor=-1 if include_fix else 0,
                                                  want_raw=True, **kw)
        assert np.array_equal(p2, pairs)
        e = np.abs(raw - bp.raw_blocks(Rd, pairs)).max() / np.abs(Rd).max()
        print(f"{name} {loss} {list(kw)[0]}: raw {e:.2e} of max |R|")
        assert e < TOLRAW
        mask = np.zeros((sc["n_poses"],) * 2, bool)
        mask[pairs[:, 0], pairs[:, 1]] = mask[pairs[:, 1], pairs[:, 0]] = True
        assert np.all(Rd[~np.kron(mask, np.ones((6, 6), bool))] == 0)
    blk.close()
    dense.close()


def test_raw_blocks_are_zero_on_factor_only_pairs():
    sc = bref.corridor(40, w=2, planes_per_pose=10, seed=1)
    ctx = _ctx(sc, L.PREC_BLOCKS)
    x = _converged(ctx, sc["poses_init"])
    vox_pairs = {tuple(p) for p in ctx.block_structure(want_pairs=True)["pair_list"]}
    ctx.set_block_factors([dict(poses=[0, 39], poses_hat=x[[0, 39]], H=np.eye(12))])
    pairs = ctx.block_structure(want_pairs=True)["pair_list"]
    _, (_, raw) = ctx.block_point_covariance(x, [5], point_noise=PN, want_raw=True)
    only = [k for k, p in enumerate(pairs) if tuple(p) not in vox_pairs]
    assert only and np.all(raw[only] == 0.0)
    ctx.close()


@pytest.mark.parametrize("name", ["fix", "ragged"])
def test_plain_covariance(name):
    sc = rig_case(name)[0]
    x, N = sc["poses_init"], sc["n_poses"]
    include_fix = sc.get("fix10") is not None
    blk, dense = _ctx(sc, L.PREC_BLOCKS), _ctx(sc, L.PREC_FP64)
    sel = [N - 1, 0, 2]
    if include_fix:  # gauge held by the fix clusters: the dense pose covariance itself
        _, Rc = dense.pose_covariance(x, point_noise=PN, include_fix=True)
        S = blk.block_point_covariance(x, sel, point_noise=PN, include_fix=True, anchor=-1)
        ref = bp.sel_block(Rc, sel)
        print(f"{name}: joint against pose_covariance {_rel(S, ref):.2e}")
        assert _rel(S, ref) < TOLCOV
    for anchor in (0, 2):
        Rd, _ = dense.pose_covariance(x, point_noise=PN, include_fix=include_fix, want_cov=False)
        H, _, _ = dense.evaluate(x, include_fix=include_fix)
        ref = bp.sel_covariance(H, Rd, sel, anchor)
        S = blk.block_point_covariance(x, sel, point_noise=PN, include_fix=include_fix, anchor=anchor)
        Mg = blk.block_point_covariance(x, sel, point_noise=PN, include_fix=include_fix, anchor=anchor, joint=False)
        print(f"{name} anchor {anchor}: joint against the restatement {_rel(S, ref):.2e}")
        assert _rel(S, ref) < TOLCOV
        assert np.array_equal(S, S.T)
        for u in range(len(sel)):
            assert np.array_equal(Mg[u], S[6 * u:6 * u + 6, 6 * u:6 * u + 6])
        a = 6 * sel.index(anchor)
        assert np.all(S[a:a + 6] == 0) and np.all(S[:, a:a + 6] == 0)
    blk.close()
    dense.close()


# (the fix scene's rig LM stops where H_rig without an anchor is still indefinite: the dense call's pivot test takes
# |d|, the blocks calls' positive pivots only)
@pytest.mark.parametrize("name", ["dense", "ragged"])
def test_rig_against_the_dense_rig_covariance(name):
    sc, base_of, lidar_of, base, ext = rig_case(name)
    include_fix = sc.get("fix10") is not None
    anchor = -1 if include_fix else 0
    blk, dense = _ctx(sc, L.PREC_BLOCKS), _ctx(sc, L.PREC_FP64)
    n_rig = blk.set_block_rig(base_of, lidar_of)
    dense.set_rig(base_of, lidar_of)
    F = n_rig // 6
    # at the rig LM's optimum: the blocks calls' pivot test refuses an indefinite H_rig
    base, ext, _ = blk.rig_damping_iter(base, ext, max_iter=20, rel_tol=1e-12, gauge_mode=2, min_planes_per_pose=0,
                                        hess_includes_fix=include_fix)
    for kw in (dict(point_noise=PN), dict(c_cov=_c_cov(sc))):
        _, cov = dense.rig_covariance(base, ext, include_fix=include_fix, anchor=anchor, want_raw=False, **kw)
        for sel in ([F - 1], [F - 1, 1, 0]):
            S = blk.rig_block_point_covariance(base, ext, sel, include_fix=include_fix, anchor=anchor, **kw)
            e = _rel(S, bp.sel_block(cov, sel))
            print(f"{name} {list(kw)[0]} sel {sel}: {e:.2e}")
            assert e < TOLCOV and np.array_equal(S, S.T)
    blk.close()
    dense.close()


def test_identity_rig_is_bitwise_the_plain_call():
    sc = make_scene(n_poses=8, n_planes=50, seed=7, with_fix=True)
    x, N = sc["poses_init"], sc["n_poses"]
    ident = np.concatenate([np.eye(3).reshape(9), np.zeros(3)])[None]
    ctx = _ctx(sc, L.PREC_BLOCKS)
    ctx.set_block_rig(np.arange(N), np.zeros(N))
    sel = [3, 0, 7]
    for anchor in (-1, 2):
        for joint in (True, False):
            a = ctx.block_point_covariance(x, sel, point_noise=PN, include_fix=True, anchor=anchor, joint=joint)
            b = ctx.rig_block_point_covariance(x, ident, sel, point_noise=PN, include_fix=True, anchor=anchor,
                                               joint=joint)
            assert np.array_equal(a, b)
    ctx.close()


def test_bitwise_properties_and_lm_unchanged():
    sc = bref.corridor(300, w=10, planes_per_pose=30, seed=2, with_fix=True)
    a, b = _ctx(sc, L.PREC_BLOCKS), _ctx(sc, L.PREC_BLOCKS)
    x = _converged(a, sc["poses_init"])
    assert np.array_equal(x, _converged(b, sc["poses_init"]))
    sel = [17, 250, 3, 120]
    S = a.block_point_covariance(x, sel, point_noise=PN, anchor=5)
    assert np.array_equal(S, a.block_point_covariance(x, sel, point_noise=PN, anchor=5))
    perm = [2, 0, 3, 1]
    idx = np.concatenate([np.arange(6 * k, 6 * k + 6) for k in perm])
    Sp = a.block_point_covariance(x, [sel[k] for k in perm], point_noise=PN, anchor=5)
    assert np.array_equal(Sp, S[np.ix_(idx, idx)])
    Mg = a.block_point_covariance(x, sel, point_noise=PN, anchor=5, joint=False)
    for u in range(len(sel)):
        assert np.array_equal(Mg[u], S[6 * u:6 * u + 6, 6 * u:6 * u + 6])
    ra = a.damping_iter(x, max_iter=4, rel_tol=-1, gauge_mode=2, min_planes_per_pose=0, want_per_iter=True)
    rb_ = b.damping_iter(x, max_iter=4, rel_tol=-1, gauge_mode=2, min_planes_per_pose=0, want_per_iter=True)
    assert ra[1] == rb_[1] and np.array_equal(ra[0], rb_[0]) and np.array_equal(ra[2], rb_[2])
    a.close()
    b.close()


def test_marginals_in_chunks_equal_one_chunk():
    sc = bref.corridor(300, w=10, planes_per_pose=30, seed=2, with_fix=True)
    ctx = _ctx(sc, L.PREC_BLOCKS)
    x = _converged(ctx, sc["poses_init"])
    sel = np.arange(300)[::-1]
    whole = ctx.block_point_covariance(x, sel, point_noise=PN, anchor=-1, include_fix=True, joint=False)
    os.environ["BALM_COV_BUDGET_MB"] = "8"  # a few unknowns per chunk; the raw term then runs in voxel batches too
    try:
        chunked = ctx.block_point_covariance(x, sel, point_noise=PN, anchor=-1, include_fix=True, joint=False)
    finally:
        del os.environ["BALM_COV_BUDGET_MB"]
    e = _rel(chunked, whole)
    print(f"chunked marginals against one chunk: {e:.2e}")
    assert e < 1e-12
    ctx.close()


def test_5000_poses_against_scipy(monkeypatch):
    N = 5000
    # test_gpu_sparse_covariance's well-conditioned corridor: 100 m long, gauge held by the fix clusters
    monkeypatch.setattr(bref, "min", lambda a, b: 100.0 / N, raising=False)
    sc = bref.corridor(N, w=8, planes_per_pose=30, seed=7, with_fix=True)
    ctx = _ctx(sc, L.PREC_BLOCKS)
    x = sc["poses_gt"]
    sel = [0, 1234, 2500, 4999]
    anchor = -1
    S, (pairs, raw) = ctx.block_point_covariance(x, sel, point_noise=PN, anchor=anchor, include_fix=True,
                                                 want_raw=True)
    blocks = ctx.download_blocks()  # H at x, undamped
    H = bref.to_sparse(N, pairs, blocks).tolil()
    R = bref.to_sparse(N, pairs, raw).tocsr()
    Y = spla.splu(H.tocsc()).solve(bp.unit_columns(6 * N, sel))
    ref = Y.T @ (R @ Y)
    e = _rel(S, ref)
    print(f"N = {N}: Sigma against scipy {e:.2e} of max |Sigma|")
    assert e < TOLCOV
    Mg = ctx.block_point_covariance(x, np.arange(N), point_noise=PN, anchor=anchor, include_fix=True, joint=False)
    for u, i in enumerate(sel):
        assert np.array_equal(Mg[i], S[6 * u:6 * u + 6, 6 * u:6 * u + 6])
    ctx.close()


def test_20000_slots_extrinsic_sigma():
    S = rb.rig_corridor(5000, 4)
    ctx = _ctx(S, L.PREC_BLOCKS)
    # LiDAR-to-INS: every base fixed on the trajectory, the four extrinsics free
    n_rig = ctx.set_block_rig(S["base_of"], S["lidar_of"], fixed_bases=range(5000), fixed_lidars=())
    assert n_rig == 24
    base, ext, _ = ctx.rig_damping_iter(S["base12"], S["ext12"], max_iter=5, gauge_mode=2, min_planes_per_pose=0)
    cov = ctx.rig_block_point_covariance(base, ext, [0, 1, 2, 3], point_noise=0.01, anchor=-1)
    assert np.array_equal(cov, cov.T)
    ev = np.linalg.eigvalsh(cov)
    rot, tra = extrinsic_sigmas(cov, 0)
    print(f"20 000 slots: eigenvalues {ev.min():.2e} .. {ev.max():.2e}; 1-sigma rot {rot} rad, trans {tra} m")
    assert ev.min() > 0
    ctx.close()


# ---------------- meaning: a Monte-Carlo check ----------------
SIGMA = 0.02
DRAWS = 200


def test_monte_carlo_consistency():
    """bases free and anchored at base 0, LiDAR 0 fixed: the extrinsics' error has covariance Sigma, NEES averages 6"""
    S = rr.rig_scene()
    base_t, ext_t = S["base12"], S["ext12"]
    X = rr.compose(base_t, ext_t, S["base_of"], S["lidar_of"])
    sc = rr.cut(S, base_t, ext_t)
    flat = rc.planar_moments(sc, X)
    model = rc.noise_model(flat)
    ctx = balm_b200.Context(len(X), 0, L.PREC_BLOCKS)
    n_rig = ctx.set_block_rig(S["base_of"], S["lidar_of"])
    ctx.set_voxels(sc["row_ptr"], sc["pose_idx"], flat, sc["coe"])
    fb = len(base_t)
    lidars = list(range(1, len(ext_t)))
    sel = [fb + k for k in range(len(lidars))]
    assert n_rig == 6 * (fb + len(lidars))
    cov = ctx.rig_block_point_covariance(base_t, ext_t, sel, point_noise=SIGMA, anchor=0)
    rng = np.random.default_rng(31)
    chi = np.zeros((DRAWS, len(lidars)))
    for d in range(DRAWS):
        ctx.set_voxels(sc["row_ptr"], sc["pose_idx"], rc.noisy_moments(flat, model, SIGMA, rng), sc["coe"])
        _, ext, _ = ctx.rig_damping_iter(base_t, ext_t, max_iter=20, rel_tol=1e-12, gauge_mode=2, min_planes_per_pose=0)
        for k, l in enumerate(lidars):
            Rn, pn = unpack_pose(ext[l])
            Rt, pt = unpack_pose(ext_t[l])
            th = pg.log_so3(Rn @ Rt.T)
            delta = np.concatenate([th, pn - pg.exp_so3(th) @ pt])
            blk = cov[6 * k:6 * k + 6, 6 * k:6 * k + 6]
            chi[d, k] = delta @ np.linalg.solve(blk, delta)
    ctx.close()
    means = chi.mean(0)
    lo, hi = stats.chi2.ppf([0.005, 0.995], 6 * DRAWS) / DRAWS
    print(f"mean NEES {np.round(means, 3)} (99 % band {lo:.3f} .. {hi:.3f})")
    assert np.all((means >= lo) & (means <= hi)), (means, lo, hi)


def test_refusals_write_nothing():
    sc, base_of, lidar_of, base, ext = rig_case("dense")
    x, N = sc["poses_init"], sc["n_poses"]
    lib = L.lib()
    p = lambda arr: None if arr is None else arr.ctypes.data_as(C.c_void_p)
    ctx = _ctx(sc, L.PREC_BLOCKS)
    pairs = ctx.block_structure()["pairs"]
    raw, cov, marg = np.full(36 * pairs, 7.0), np.full(36 * 4, 7.0), np.full(36 * 4, 7.0)
    x12 = np.ascontiguousarray(x)

    def call(h, poses, anchor, sel, cv=cov, include_fix=0):
        s = None if sel is None else np.ascontiguousarray(sel, dtype=np.int32)
        n = 0 if sel is None else len(sel)
        return lib.balm_block_point_covariance(h, p(poses), None, PN, include_fix, anchor, n, p(s), p(raw), p(cv),
                                               p(marg))

    def untouched():
        return np.all(raw == 7.0) and np.all(cov == 7.0) and np.all(marg == 7.0)

    assert call(ctx._h, None, 0, [1, 2]) == L.ERR_INVALID
    for anchor in (-2, N):
        assert call(ctx._h, x12, anchor, [1, 2]) == L.ERR_INVALID
    for sel in ([1, 1], [N], [-1], None):
        assert call(ctx._h, x12, 0, sel) == L.ERR_INVALID
    assert call(ctx._h, x12, -1, [1, 2]) == L.ERR_NOT_PD  # no fix clusters, no anchor: the gauge is free
    assert "singular" in lib.balm_last_error().decode()
    assert untouched()
    os.environ["BALM_COV_BUDGET_MB"] = "0"
    try:
        assert call(ctx._h, x12, 0, [1, 2]) == L.ERR_UNSUPPORTED
    finally:
        del os.environ["BALM_COV_BUDGET_MB"]
    assert untouched()
    dense = _ctx(sc, L.PREC_FP64)
    assert call(dense._h, x12, 0, [1, 2]) == L.ERR_INVALID
    bare = balm_b200.Context(N, 0, L.PREC_BLOCKS)
    assert call(bare._h, x12, 0, [1, 2]) == L.ERR_INVALID
    assert untouched()
    assert call(ctx._h, x12, 0, [1, 2]) == L.OK and not np.any(cov[:144] == 7.0)
    # the rig call
    b12, e12 = np.ascontiguousarray(base), np.ascontiguousarray(ext)
    rcov = np.full(144, 7.0)

    def rcall(h, anchor, sel, b=b12, e=e12):
        s = np.ascontiguousarray(sel, dtype=np.int32)
        return lib.balm_rig_block_point_covariance(h, p(b), p(e), None, PN, 0, anchor, len(s), p(s), p(rcov), None)

    assert rcall(ctx._h, 0, [0]) == L.ERR_INVALID  # no rig
    n_rig = ctx.set_block_rig(base_of, lidar_of)
    F = n_rig // 6
    b12, e12, _ = ctx.rig_damping_iter(b12, e12, max_iter=20, rel_tol=1e-12, gauge_mode=2, min_planes_per_pose=0)
    for anchor in (-2, F - 1, F):  # below -1, the extrinsic, past the end
        assert rcall(ctx._h, anchor, [0]) == L.ERR_INVALID
    for sel in ([0, 0], [F], [-1]):
        assert rcall(ctx._h, 0, sel) == L.ERR_INVALID
    assert rcall(ctx._h, 0, [0], b=None) == L.ERR_INVALID
    assert rcall(ctx._h, -1, [0]) == L.ERR_NOT_PD
    dense.set_rig(base_of, lidar_of)
    assert rcall(dense._h, 0, [0]) == L.ERR_INVALID
    assert np.all(rcov == 7.0)
    assert rcall(ctx._h, 0, [F - 1], b=b12, e=e12) == L.OK and not np.any(rcov[:36] == 7.0)
    for c in (ctx, dense, bare):
        c.close()

"""balm_rig_covariance on the device (Context.rig_covariance, balm_b200.rig.extrinsic_sigmas): against the restatement
(tests/rig_cov_ref.py) on both dense precisions, every rig_case scene, with and without a voxel loss and with both
noise inputs; the identity rig against the context's own pose covariance, bit for bit; repeatability and an unchanged
LM afterwards; the refusals; and a Monte-Carlo check of the covariance's meaning on the room rig."""
import ctypes as C

import numpy as np
import pytest
from scipy import stats

import balm_b200
import numpy_cov as nc
import pose_graph_ref as pg
import rig_cov_ref as rc
import rig_ref as rr
import robust_voxels_ref as rv
from balm_b200 import _lib as L
from balm_b200.rig import extrinsic_sigmas
from scenes import make_scene, unpack_pose
from test_gpu_rig import PRECS, TOLH, _ctx, _rel, _status, rig_case

pytestmark = pytest.mark.gpu

PN = 0.01
TOLRAW = TOLH["fp64"]  # of max |raw|: the raw term runs in fp64 on both precisions
# of max |cov|. The fix scene's H~ (gauge held by the fix clusters alone) has a condition near 1e11, so cov moves by far
# more than TOLH x the condition allows for the tensor path's H; cov is checked against the restatement's sandwich of
# the device's own H_rig (itself at TOLH of the restatement's), and on fp64 also against the whole restatement.
TOLCOV = 1e-6


def _c_cov(sc, seed=3):
    """explicit per-observation cluster covariances: isotropic ones at a different noise level per observation"""
    rng = np.random.default_rng(seed)
    return np.stack([nc.cluster_cov_isotropic(o, PN * rng.uniform(0.5, 2.0)) for o in sc["obs10"]])


@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("name", ["dense", "ragged", "fix"])
@pytest.mark.parametrize("loss", [None, "cauchy"])
def test_rig_covariance_matches_restatement(prec, name, loss):
    sc, base_of, lidar_of, base, ext = rig_case(name)
    X = rr.compose(base, ext, base_of, lidar_of)
    include_fix = sc.get("fix10") is not None
    anchor = -1 if include_fix else 0  # without fix clusters the base poses' gauge is free
    kind, c = rv.TRIVIAL, 1.0
    if loss:
        kind, c = rv.NAMES[loss], float(np.sqrt(np.median(rv.lams(sc, X, include_fix))))
    ctx = _ctx(sc, prec, (loss, c) if loss else None)
    ctx.set_rig(base_of, lidar_of)
    var = rr.unknowns(len(base), 2)
    for noise in ("iso", "c_cov"):
        kw = dict(pnoise=PN) if noise == "iso" else dict(c_cov=_c_cov(sc))
        raw_r, cov_r = rc.rig_covariance(sc, base, ext, base_of, lidar_of, var, include_fix=include_fix, anchor=anchor,
                                         kind=kind, c=c, **kw)
        raw, cov = ctx.rig_covariance(base, ext, point_noise=kw.get("pnoise", 0.0), c_cov=kw.get("c_cov"),
                                      include_fix=include_fix, anchor=anchor)
        H, _, _ = ctx.rig_evaluate(base, ext, include_fix=include_fix)
        Hr = rr.evaluate(sc, base, ext, base_of, lidar_of, var, include_fix, kind, c)[0]
        Hi = np.linalg.inv(rc.delete(H, anchor, 1.0))
        cov_h = rc.delete(Hi @ raw_r @ Hi.T, anchor, 0.0)
        er, eh, ec, ecr = _rel(raw, raw_r), _rel(H, Hr), _rel(cov, cov_h), _rel(cov, cov_r)
        print(f"{prec} {name} {loss} {noise}: raw {er:.2e} H {eh:.2e} cov {ec:.2e} (restatement's H: {ecr:.2e})")
        assert er < TOLRAW and eh < TOLH[prec] and ec < TOLCOV, (er, eh, ec)
        if prec == "fp64":
            assert ecr < TOLCOV
        assert np.array_equal(raw, raw.T)
        if anchor >= 0:
            a = slice(6 * anchor, 6 * anchor + 6)
            for m in (raw, cov):
                assert np.all(m[a] == 0) and np.all(m[:, a] == 0)
    ctx.close()


@pytest.mark.parametrize("prec", list(PRECS))
def test_identity_rig_is_bitwise_the_pose_covariance(prec):
    sc = make_scene(n_poses=8, n_planes=50, seed=7, with_fix=True)
    x, N = sc["poses_init"], sc["n_poses"]
    ident = np.concatenate([np.eye(3).reshape(9), np.zeros(3)])[None]
    ctx = _ctx(sc, prec)
    ctx.set_rig(np.arange(N), np.zeros(N))
    for kw in (dict(point_noise=PN), dict(c_cov=_c_cov(sc))):
        raw_p, cov_p = ctx.pose_covariance(x, include_fix=True, **kw)
        raw, cov = ctx.rig_covariance(x, ident, include_fix=True, anchor=-1, **kw)
        assert np.array_equal(raw, raw_p) and np.array_equal(cov, cov_p)
    ctx.close()


@pytest.mark.parametrize("prec", list(PRECS))
def test_repeatable_and_lm_unchanged(prec):
    sc, base_of, lidar_of, base, ext = rig_case("dense")
    a, b = _ctx(sc, prec), _ctx(sc, prec)
    for c in (a, b):
        c.set_rig(base_of, lidar_of)
    r1, c1 = a.rig_covariance(base, ext, point_noise=PN, anchor=0)
    r2, c2 = a.rig_covariance(base, ext, point_noise=PN, anchor=0)
    assert np.array_equal(r1, r2) and np.array_equal(c1, c2)
    raw_only, none = a.rig_covariance(base, ext, point_noise=PN, anchor=0, want_cov=False)
    assert none is None and np.array_equal(raw_only, r1)
    pa = a.rig_damping_iter(base, ext, gauge_mode=2, want_per_iter=True, rel_tol=-1, max_iter=5)
    pb = b.rig_damping_iter(base, ext, gauge_mode=2, want_per_iter=True, rel_tol=-1, max_iter=5)
    assert pa[2] == pb[2]
    assert np.array_equal(pa[0], pb[0]) and np.array_equal(pa[1], pb[1])
    for (xa, ea), (xb, eb) in zip(pa[3], pb[3]):
        assert np.array_equal(xa, xb) and np.array_equal(ea, eb)
    a.close()
    b.close()


def test_refusals_write_nothing():
    sc, base_of, lidar_of, base, ext = rig_case("dense")
    lib = L.lib()
    p = lambda arr: None if arr is None else arr.ctypes.data_as(C.c_void_p)
    ctx = _ctx(sc, "fp64")
    assert _status(lambda: ctx.rig_covariance(base, ext, point_noise=PN)) == L.ERR_INVALID  # no rig
    n_rig = ctx.set_rig(base_of, lidar_of, fixed_bases=(1,))  # free bases 0, 2 -> free indices 0, 1; extrinsic 1 -> 2
    raw, cov = np.full((n_rig, n_rig), 7.0), np.full((n_rig, n_rig), 7.0)

    def call(b12, e12, anchor, include_fix=0, h=None):
        return lib.balm_rig_covariance(h or ctx._h, p(b12), p(e12), None, PN, include_fix, anchor, p(raw), p(cov))

    b12, e12 = np.ascontiguousarray(base), np.ascontiguousarray(ext)
    assert call(None, e12, 0) == L.ERR_INVALID and call(b12, None, 0) == L.ERR_INVALID
    for anchor in (-2, 2, 3):  # below -1, the extrinsic's free index, past the end
        assert call(b12, e12, anchor) == L.ERR_INVALID
    assert np.all(raw == 7.0) and np.all(cov == 7.0)
    assert call(b12, e12, 0) == L.OK and not np.any(cov == 7.0)
    # no voxels registered
    bare = balm_b200.Context(sc["n_poses"], 0, L.PREC_FP64)
    bare.set_rig(base_of, lidar_of, fixed_bases=(1,))
    raw[:], cov[:] = 7.0, 7.0
    assert call(b12, e12, 0, h=bare._h) == L.ERR_INVALID
    bare.close()
    # every base free, no fix clusters, no anchor: the base poses' gauge leaves H_rig singular
    ctx.set_rig(base_of, lidar_of)
    n_rig = 6 * 4
    raw, cov = np.full((n_rig, n_rig), 7.0), np.full((n_rig, n_rig), 7.0)
    assert call(b12, e12, -1) == L.ERR_NOT_PD
    assert np.all(raw == 7.0) and np.all(cov == 7.0)
    assert "singular" in lib.balm_last_error().decode()
    ctx.close()


# ---------------- meaning: a Monte-Carlo check ----------------
SIGMA = 0.02  # point noise (m)
DRAWS = 200


def _nees_run(S, fixed_bases, fixed_lidars, anchor, seed):
    """voxels cut once at the truth and moved onto their planes; every draw redraws the points with SIGMA, re-aggregates
    the clusters and runs rig_damping_iter from the truth -> (mean NEES per free extrinsic, sigmas)"""
    base_t, ext_t = S["base12"], S["ext12"]
    X = rr.compose(base_t, ext_t, S["base_of"], S["lidar_of"])
    sc = rr.cut(S, base_t, ext_t)
    flat = rc.planar_moments(sc, X)
    model = rc.noise_model(flat)
    ctx = balm_b200.Context(len(X), 0, L.PREC_FP64)
    ctx.set_rig(S["base_of"], S["lidar_of"], fixed_bases=fixed_bases, fixed_lidars=fixed_lidars)
    ctx.set_voxels(sc["row_ptr"], sc["pose_idx"], flat, sc["coe"])
    _, cov = ctx.rig_covariance(base_t, ext_t, point_noise=SIGMA, anchor=anchor, want_raw=False)
    fb = len(base_t) - len(fixed_bases)
    lidars = [l for l in range(len(ext_t)) if l not in fixed_lidars]
    blocks = [cov[6 * (fb + k):6 * (fb + k + 1), 6 * (fb + k):6 * (fb + k + 1)] for k in range(len(lidars))]
    rng = np.random.default_rng(seed)
    chi = np.zeros((DRAWS, len(lidars)))
    for d in range(DRAWS):
        ctx.set_voxels(sc["row_ptr"], sc["pose_idx"], rc.noisy_moments(flat, model, SIGMA, rng), sc["coe"])
        _, ext, _ = ctx.rig_damping_iter(base_t, ext_t, max_iter=20, rel_tol=1e-12, gauge_mode=2,
                                         min_planes_per_pose=0)
        for k, l in enumerate(lidars):
            Rn, pn = unpack_pose(ext[l])
            Rt, pt = unpack_pose(ext_t[l])
            th = pg.log_so3(Rn @ Rt.T)
            delta = np.concatenate([th, pn - pg.exp_so3(th) @ pt])  # the left step from the truth to the estimate
            chi[d, k] = delta @ np.linalg.solve(blocks[k], delta)
    ctx.close()
    return chi.mean(0), extrinsic_sigmas(cov, fb)


@pytest.mark.parametrize("case", ["multi_lidar", "lidar_to_ins"])
def test_monte_carlo_consistency(case):
    """the estimate's error in the extrinsics' update coordinates has covariance cov_rig: its NEES averages 6"""
    S = rr.rig_scene()
    if case == "multi_lidar":  # LiDAR 0 fixed, bases free, anchored at base 0
        means, (rot, tra) = _nees_run(S, (), (0,), 0, seed=31)
    else:                      # every base fixed at the INS trajectory
        S = rr.ins_scene(S)
        means, (rot, tra) = _nees_run(S, tuple(range(len(S["base12"]))), (), -1, seed=32)
    lo, hi = stats.chi2.ppf([0.005, 0.995], 6 * DRAWS) / DRAWS
    print(f"{case}: mean NEES {np.round(means, 3)} (99 % band {lo:.3f} .. {hi:.3f}); 1-sigma rot {rot} rad, "
          f"trans {tra} m")
    assert np.all((means >= lo) & (means <= hi)), (means, lo, hi)

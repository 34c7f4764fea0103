"""Rig calibration on the device (balm_set_rig, balm_rig_evaluate, balm_rig_damping_iter, balm_b200.rig): H_rig and
g_rig against rig_ref on both dense precisions and every scene shape, with and without a voxel loss; the coe w identity;
determinism; LM parity with the restatement; the single-LiDAR identity rig against the context's own calls; calibration
of the synthetic rig and the LiDAR-to-INS case; refusals and lifetime."""
import ctypes as C

import numpy as np
import pytest

import balm_b200
import rig_ref as rr
import robust_voxels_ref as rv
from balm_b200 import _lib as L
from scenes import make_scene, unpack_pose

pytestmark = pytest.mark.gpu

PRECS = {"fp64": L.PREC_FP64, "tensor": L.PREC_TENSOR}
TOLH = {"fp64": 1e-10, "tensor": 1e-8}  # of max |H|; the tensor path's H tolerance (test_gpu_parity.py)
TOLG = {"fp64": 1e-10, "tensor": 1e-10}


def _inv(p12):
    R, t = unpack_pose(p12)
    return np.concatenate([R.reshape(9), -R.T @ t])


def rig_case(name):
    """make_scene's scans as bases x two LiDARs: E_0 = I, E_1 = scan 1 in scan 0's frame (then every slot's pose is
    its composed one, off the truth by the scene's pose noise) -> (scene, base_of, lidar_of, base12, ext12)"""
    kw = dict(dense=dict(n_poses=6, n_planes=30, seed=4), ragged=dict(n_poses=8, n_planes=60, seed=6, drop=0.4),
              fix=dict(n_poses=6, n_planes=30, seed=5, with_fix=True))[name]
    sc = make_scene(**kw)
    N = sc["n_poses"]
    base_of, lidar_of = np.arange(N) // 2, np.arange(N) % 2
    X = sc["poses_init"]
    base = X[0::2].copy()
    ext = np.zeros((2, 12))
    ext[0] = np.concatenate([np.eye(3).reshape(9), np.zeros(3)])
    ext[1] = rr.compose(np.array([_inv(X[0])]), np.array([X[1]]), [0], [0])[0]
    base[:, 9:] += np.array([30.0, -20.0, 5.0])  # away from the origin, so the p-terms of the correction matter
    return sc, base_of, lidar_of, base, ext


def _ctx(sc, prec, loss=None, coe=None):
    c = balm_b200.Context(sc["n_poses"], 0, PRECS[prec])
    if loss is not None:
        c.set_voxel_loss(*loss)
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"] if coe is None else coe, sc.get("fix10"))
    return c


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300)


@pytest.mark.parametrize("prec", list(PRECS))
@pytest.mark.parametrize("name", ["dense", "ragged", "fix"])
@pytest.mark.parametrize("loss", [None, "cauchy"])
def test_rig_evaluate_matches_restatement(prec, name, loss):
    sc, base_of, lidar_of, base, ext = rig_case(name)
    X = rr.compose(base, ext, base_of, lidar_of)
    for include_fix in ((False, True) if sc.get("fix10") is not None else (False,)):
        kind, c = rv.TRIVIAL, 1.0
        if loss:
            kind, c = rv.NAMES[loss], float(np.sqrt(np.median(rv.lams(sc, X, include_fix))))
        ctx = _ctx(sc, prec, (loss, c) if loss else None)
        n_rig = ctx.set_rig(base_of, lidar_of)
        var = rr.unknowns(len(base), 2)
        assert n_rig == 6 * len(var)
        Hr, gr, rr_, _, _ = rr.evaluate(sc, base, ext, base_of, lidar_of, var, include_fix, kind, c)
        H, g, r = ctx.rig_evaluate(base, ext, include_fix=include_fix)
        assert np.abs(H - Hr).max() < TOLH[prec] * np.abs(Hr).max(), (include_fix, _rel(H, Hr))
        # the residual is the context's own; 30 m from the origin lambda_min loses a few digits to cancellation
        assert _rel(g, gr) < TOLG[prec] and abs(r - rr_) < 1e-10 * abs(rr_)
        assert np.array_equal(H, H.T)
        H2, g2, r2 = ctx.rig_evaluate(base, ext, include_fix=include_fix)  # two runs: the same bits
        assert np.array_equal(H, H2) and np.array_equal(g, g2) and r == r2
        if loss:  # coe w identity, bitwise: a trivial-loss context registered with coe w. With identity extrinsics
            # the device's composition is exact, so w read at the host's scan poses is the weight the evaluation used.
            ext_id = np.tile(np.concatenate([np.eye(3).reshape(9), np.zeros(3)]), (2, 1))
            Hl, gl, _ = ctx.rig_evaluate(base, ext_id, include_fix=include_fix)
            _, w = ctx.voxel_residuals(base[base_of], include_fix=include_fix)
            tw = _ctx(sc, prec, coe=np.asarray(sc["coe"]) * w)
            tw.set_rig(base_of, lidar_of)
            Hw, gw, _ = tw.rig_evaluate(base, ext_id, include_fix=include_fix)
            assert np.array_equal(Hl, Hw) and np.array_equal(gl, gw)
            tw.close()
        ctx.close()


# With every extrinsic free the second gauge (T_b Q, Q^-1 E_l) is a null direction of the cost, along which the tensor
# path's H error moves the poses further than 1e-6; both precisions run with the reference LiDAR fixed.
@pytest.mark.parametrize("prec, fixed_lidars", [("fp64", (0,)), ("fp64", ()), ("tensor", (0,))])
def test_lm_parity_with_restatement(prec, fixed_lidars):
    sc, base_of, lidar_of, base, ext = rig_case("dense")
    ctx = _ctx(sc, prec)
    ctx.set_rig(base_of, lidar_of, fixed_lidars=fixed_lidars)
    var = rr.unknowns(len(base), 2, fixed_lidars=fixed_lidars)
    b_ref, e_ref, tr_ref, per_ref = rr.lm(sc, base, ext, base_of, lidar_of, var)
    b, e, tr, per = ctx.rig_damping_iter(base, ext, gauge_mode=2, want_per_iter=True)
    assert [t["accepted"] for t in tr] == [t["accepted"] for t in tr_ref]
    for (pb, pe), (qb, qe) in zip(per, per_ref):
        for x, y in zip(np.concatenate([pb, pe]), np.concatenate([qb, qe])):
            dr, dp = rr.pose_error(x, y)
            assert dr < 1e-6 and dp < 1e-6
    assert np.array_equal(np.concatenate([b, e]), np.concatenate(per[-1]))
    ctx.close()


@pytest.mark.parametrize("with_fix", [False, True])
def test_identity_rig_is_bitwise_the_context(with_fix):
    """B = N, base_of = identity, one LiDAR fixed at the identity: the rig calls are the context's own, bit for bit"""
    sc = make_scene(n_poses=8, n_planes=50, seed=7, with_fix=with_fix)
    x = sc["poses_init"]
    N = sc["n_poses"]
    ident = np.concatenate([np.eye(3).reshape(9), np.zeros(3)])[None]
    a, b = _ctx(sc, "fp64"), _ctx(sc, "fp64")
    assert b.set_rig(np.arange(N), np.zeros(N)) == 6 * N
    for inc in ((False, True) if with_fix else (False,)):
        H, g, r = a.evaluate(x, include_fix=inc)
        Hr, gr, rr_ = b.rig_evaluate(x, ident, include_fix=inc)
        assert np.array_equal(H, Hr) and np.array_equal(g, gr) and r == rr_
    for gauge in (0, 2):
        for force in (False, True):
            p, tr, per = a.damping_iter(x, gauge_mode=gauge, want_per_iter=True, force_hess=force, rel_tol=-1,
                                        hess_includes_fix=with_fix)
            pb, pe, trb, perb = b.rig_damping_iter(x, ident, gauge_mode=gauge, want_per_iter=True, force_hess=force,
                                                   rel_tol=-1, hess_includes_fix=with_fix)
            assert tr == trb
            assert np.array_equal(p, pb) and np.array_equal(pe, ident)
            for q, (qb, _) in zip(per, perb):
                assert np.array_equal(q, qb)
    a.close()
    b.close()


# The restatement's results on the same scenes and start. Multi-LiDAR (test_rig_ref.test_rig_scene_calibration, two
# rounds): worst free extrinsic 0.00116 rad / 0.0058 m; the bounds are twice that, the translation capped at the 10x
# bound 0.01 m. LiDAR-to-INS (test_rig_ref.test_lidar_to_ins_calibration, three rounds): 0.00120 rad / 0.0029 m; the
# bounds are twice that.
CAL_ROT, CAL_POS = 2 * 0.00116, 0.01
INS_ROT, INS_POS = 2 * 0.00120, 2 * 0.0029


@pytest.mark.parametrize("prec", list(PRECS))
def test_calibrate_rig_recovers_extrinsics(prec):
    S = rr.rig_scene()
    base0, ext0 = rr.perturbed_start(S)
    base, ext, traces = balm_b200.calibrate_rig(S["xyz"], S["scan"], S["base_of"], S["lidar_of"], base0, ext0,
                                                precision=PRECS[prec])
    assert len(traces) == 3 and traces[0][0]["accepted"]
    assert np.array_equal(ext[0], ext0[0])  # the reference LiDAR stays fixed
    for l in (1, 2):
        dr, dp = rr.pose_error(ext[l], S["ext12"][l])
        assert dr < CAL_ROT and dp < CAL_POS, (l, dr, dp)


def test_lidar_to_ins():
    """L = 1: LiDAR 1's scans with every base pose fixed at the truth, only the extrinsic free (from 2 deg / 0.1 m off)"""
    S = rr.ins_scene(rr.rig_scene())
    _, ext0 = rr.perturbed_start(rr.rig_scene())
    B = len(S["base12"])
    base, ext, traces = balm_b200.calibrate_rig(S["xyz"], S["scan"], S["base_of"], S["lidar_of"], S["base12"],
                                                ext0[1:2], fixed_bases=range(B), fixed_lidars=(),
                                                precision=L.PREC_FP64)
    assert np.array_equal(base, S["base12"])
    dr, dp = rr.pose_error(ext[0], S["ext12"][0])
    assert dr < INS_ROT and dp < INS_POS, (dr, dp)


def _status(fn):
    with pytest.raises(balm_b200.BalmError) as e:
        fn()
    return e.value.status


def test_refusals_and_lifetime():
    sc, base_of, lidar_of, base, ext = rig_case("dense")
    x = sc["poses_init"]
    blk = balm_b200.Context(sc["n_poses"], 0, L.PREC_BLOCKS)
    assert _status(lambda: blk.set_rig(base_of, lidar_of)) == L.ERR_UNSUPPORTED
    blk.close()
    ctx = _ctx(sc, "fp64")
    assert _status(lambda: ctx.rig_evaluate(base, ext)) == L.ERR_INVALID  # no rig yet
    n_rig = ctx.set_rig(base_of, lidar_of)
    H0, g0, r0 = ctx.rig_evaluate(base, ext)
    N = sc["n_poses"]
    lib, h = L.lib(), ctx._h
    n_out = C.c_int()
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
    bo, lo = i32(base_of), i32(lidar_of)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    # an index out of range, a base and a LiDAR no slot uses, nothing free: refused, the rig kept
    assert lib.balm_set_rig(h, 3, 2, p(i32(np.r_[base_of[:-1], 3])), p(lo), None, None, C.byref(n_out)) == L.ERR_INVALID
    assert lib.balm_set_rig(h, 3, 2, p(bo), p(i32(np.r_[lidar_of[:-1], -1])), None, None, C.byref(n_out)) == L.ERR_INVALID
    assert lib.balm_set_rig(h, 4, 2, p(bo), p(lo), None, None, C.byref(n_out)) == L.ERR_INVALID
    assert lib.balm_set_rig(h, 3, 3, p(bo), p(lo), None, None, C.byref(n_out)) == L.ERR_INVALID
    ones = lambda k: np.ones(k, dtype=np.uint8)
    bf, lf = ones(3), ones(2)
    assert lib.balm_set_rig(h, 3, 2, p(bo), p(lo), p(bf), p(lf), C.byref(n_out)) == L.ERR_INVALID
    H1, g1, r1 = ctx.rig_evaluate(base, ext)
    assert np.array_equal(H0, H1) and np.array_equal(g0, g1) and r0 == r1
    # gauge_mode 0 / 1 with a fixed base pose: refused
    ctx.set_rig(base_of, lidar_of, fixed_bases=(0,))
    for gm in (0, 1):
        assert _status(lambda: ctx.rig_damping_iter(base, ext, gauge_mode=gm)) == L.ERR_INVALID
    ctx.rig_damping_iter(base, ext, gauge_mode=2, max_iter=2)
    # every voxel registration keeps the rig
    ctx.set_rig(base_of, lidar_of)
    ctx.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
    H2, g2, r2 = ctx.rig_evaluate(base, ext)
    assert np.array_equal(H0, H2) and H2.shape == (n_rig, n_rig)
    # the context's own calls ignore the rig; after detach it is bitwise a context that never had one
    fresh = _ctx(sc, "fp64")
    pa, tra, _ = fresh.damping_iter(x, gauge_mode=2, max_iter=4)
    pb, trb, _ = ctx.damping_iter(x, gauge_mode=2, max_iter=4)
    assert tra == trb and np.array_equal(pa, pb)
    assert ctx.set_rig(None, None) == 0
    assert _status(lambda: ctx.rig_evaluate(base, ext)) == L.ERR_INVALID
    assert _status(lambda: ctx.rig_damping_iter(base, ext)) == L.ERR_INVALID
    Ha, ga, ra = fresh.evaluate(x)
    Hb, gb, rb = ctx.evaluate(x)
    assert np.array_equal(Ha, Hb) and np.array_equal(ga, gb) and ra == rb
    pa, tra, _ = fresh.damping_iter(x, gauge_mode=0, max_iter=4)
    pb, trb, _ = ctx.damping_iter(x, gauge_mode=0, max_iter=4)
    assert tra == trb and np.array_equal(pa, pb)
    fresh.close()
    ctx.close()

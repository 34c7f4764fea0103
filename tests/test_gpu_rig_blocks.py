"""Rig calibration on a PREC_BLOCKS context (balm_block_set_rig, balm_rig_block_structure, balm_rig_block_covariance,
and balm_rig_evaluate / balm_rig_damping_iter on such a rig): H_rig and g_rig against rig_ref and the FP64 dense rig;
the identity rig bitwise the blocks context; LM parity; a 2000-slot corridor against the dense rig; calibration; pose
factors and priors in the rig cost; the Laplace covariance; refusals, lifetime and device memory."""
import ctypes as C

import numpy as np
import pytest

import balm_b200
import rig_blocks_ref as rb
import rig_ref as rr
import robust_voxels_ref as rv
from balm_b200 import _lib as L
from scenes import make_scene, unpack_pose
from test_gpu_rig import CAL_POS, CAL_ROT, INS_POS, INS_ROT, rig_case

pytestmark = pytest.mark.gpu


def _ctx(sc, prec=L.PREC_BLOCKS, loss=None):
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


def _states_close(per_a, per_b, tol):
    """every state's rotations (|R_a - R_b|, about sqrt(2) x the angle: rr.pose_error's arccos cannot resolve angles
    below 2e-8) and positions within tol"""
    for (pb, pe), (qb, qe) in zip(per_a, per_b):
        for x, y in zip(np.concatenate([pb, pe]), np.concatenate([qb, qe])):
            (Ra, pa), (Rb, pb_) = unpack_pose(x), unpack_pose(y)
            dr, dp = np.linalg.norm(Ra - Rb), np.linalg.norm(pa - pb_)
            assert dr < tol and dp < tol, (dr, dp)


@pytest.mark.parametrize("name", ["dense", "ragged", "fix"])
@pytest.mark.parametrize("loss", [None, "cauchy"])
def test_rig_evaluate_matches_restatement_and_dense(name, loss):
    sc, base_of, lidar_of, base, ext = rig_case(name)
    X = rr.compose(base, ext, base_of, lidar_of)
    for include_fix in ((False, True) if sc.get("fix10") is not None else (False,)):
        kind, c = rv.TRIVIAL, 1.0
        if loss:
            kind, c = rv.NAMES[loss], float(np.sqrt(np.median(rv.lams(sc, X, include_fix))))
        lo = (loss, c) if loss else None
        blk, dense = _ctx(sc, L.PREC_BLOCKS, lo), _ctx(sc, L.PREC_FP64, lo)
        var = rr.unknowns(len(base), 2)
        assert blk.set_block_rig(base_of, lidar_of) == dense.set_rig(base_of, lidar_of) == 6 * len(var)
        Hr, gr, _, _, _ = rr.evaluate(sc, base, ext, base_of, lidar_of, var, include_fix, kind, c)
        H, g, r = blk.rig_evaluate(base, ext, include_fix=include_fix)
        Hd, gd, rd = dense.rig_evaluate(base, ext, include_fix=include_fix)
        assert np.abs(H - Hr).max() < 1e-10 * np.abs(Hr).max() and _rel(g, gr) < 1e-10
        assert np.abs(H - Hd).max() < 1e-10 * np.abs(Hd).max() and _rel(g, gd) < 1e-10
        _, _, rc = blk.evaluate(X, include_fix=include_fix)  # the context's own residual at the composed poses
        assert abs(r - rc) < 1e-12 * abs(rc) and abs(r - rd) < 1e-10 * abs(rd)
        assert np.array_equal(H, H.T)
        H2, g2, r2 = blk.rig_evaluate(base, ext, include_fix=include_fix)
        assert np.array_equal(H, H2) and np.array_equal(g, g2) and r == r2
        blk.close()
        dense.close()


@pytest.mark.parametrize("with_fix", [False, True])
def test_identity_rig_is_bitwise_the_blocks_context(with_fix):
    sc = make_scene(n_poses=8, n_planes=50, seed=7, with_fix=with_fix)
    x = sc["poses_init"]
    N = sc["n_poses"]
    ident = np.concatenate([np.eye(3).reshape(9), np.zeros(3)])[None]
    a, b = _ctx(sc), _ctx(sc)
    assert b.set_block_rig(np.arange(N), np.zeros(N)) == 6 * N
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


@pytest.mark.parametrize("fixed_lidars", [(0,), ()])
def test_lm_parity(fixed_lidars):
    sc, base_of, lidar_of, base, ext = rig_case("dense")
    blk, dense = _ctx(sc), _ctx(sc, L.PREC_FP64)
    blk.set_block_rig(base_of, lidar_of, fixed_lidars=fixed_lidars)
    dense.set_rig(base_of, lidar_of, fixed_lidars=fixed_lidars)
    var = rr.unknowns(len(base), 2, fixed_lidars=fixed_lidars)
    _, _, tr_ref, per_ref = rr.lm(sc, base, ext, base_of, lidar_of, var)
    b, e, tr, per = blk.rig_damping_iter(base, ext, gauge_mode=2, want_per_iter=True)
    _, _, trd, perd = dense.rig_damping_iter(base, ext, gauge_mode=2, want_per_iter=True)
    acc = [t["accepted"] for t in tr]
    assert acc == [t["accepted"] for t in tr_ref] == [t["accepted"] for t in trd]
    _states_close(per, per_ref, 1e-6)
    # with every extrinsic free the second gauge is a null direction of the cost, along which the two solves' rounding
    # moves the states further (2.4e-9 measured)
    _states_close(per, perd, 1e-9 if fixed_lidars else 1e-8)
    assert np.array_equal(np.concatenate([b, e]), np.concatenate(per[-1]))
    blk.close()
    dense.close()


def test_corridor_2000_slots_against_dense():
    sc = rb.rig_corridor(500, 4, w=4, seed=3)
    base, ext = sc["base_init"], sc["ext_init"]
    blk, dense = _ctx(sc), _ctx(sc, L.PREC_FP64)
    blk.set_block_rig(sc["base_of"], sc["lidar_of"])
    dense.set_rig(sc["base_of"], sc["lidar_of"])
    H, g, _ = blk.rig_evaluate(base, ext)
    Hd, gd, _ = dense.rig_evaluate(base, ext)
    assert np.abs(H - Hd).max() < 1e-10 * np.abs(Hd).max() and _rel(g, gd) < 1e-10
    kw = dict(max_iter=3, gauge_mode=2, min_planes_per_pose=0, want_per_iter=True)
    _, _, tr, per = blk.rig_damping_iter(base, ext, **kw)
    _, _, trd, perd = dense.rig_damping_iter(base, ext, **kw)
    assert [t["accepted"] for t in tr] == [t["accepted"] for t in trd]
    _states_close(per, perd, 1e-8)
    st = blk.rig_block_structure()
    print(f"2000 slots: {st}")
    blk.close()
    dense.close()


def test_calibrate_rig_on_blocks():
    S = rr.rig_scene()
    base0, ext0 = rr.perturbed_start(S)
    base, ext, traces = balm_b200.calibrate_rig(S["xyz"], S["scan"], S["base_of"], S["lidar_of"], base0, ext0,
                                                precision=L.PREC_BLOCKS)
    assert len(traces) == 3 and traces[0][0]["accepted"]
    assert np.array_equal(ext[0], ext0[0])
    for l in (1, 2):
        dr, dp = rr.pose_error(ext[l], S["ext12"][l])
        assert dr < CAL_ROT and dp < CAL_POS, (l, dr, dp)
    S = rr.ins_scene(rr.rig_scene())
    B = len(S["base12"])
    base, ext, _ = balm_b200.calibrate_rig(S["xyz"], S["scan"], S["base_of"], S["lidar_of"], S["base12"], ext0[1:2],
                                           fixed_bases=range(B), fixed_lidars=(), precision=L.PREC_BLOCKS)
    assert np.array_equal(base, S["base12"])
    dr, dp = rr.pose_error(ext[0], S["ext12"][0])
    assert dr < INS_ROT and dp < INS_POS, (dr, dp)


def test_factors_and_priors_in_the_rig_cost():
    sc = rb.rig_corridor(40, 3, w=2, seed=5)
    B, N = 40, 120
    base, ext = sc["base_init"], sc["ext_init"]
    X = rr.compose(sc["base12"], sc["ext12"], sc["base_of"], sc["lidar_of"])
    c = _ctx(sc)
    c.set_block_rig(sc["base_of"], sc["lidar_of"])
    var = rr.unknowns(B, 3)
    n0 = c.rig_block_structure()["pairs"]
    edges = [(s, s + 3) for s in range(N - 3)] + [(0, N - 3)]  # odometry per LiDAR, one loop closure
    assert all(s == 0 for s in c.set_block_factors(balm_b200.odometry_factors(X, 1e3 * np.eye(6), edges=edges)))
    st = c.rig_block_structure(want_pairs=True)
    assert st["pairs"] == n0 + 1 and [0, B - 1] in st["pair_list"].tolist()  # the loop closure's base pair
    c.set_pose_priors(balm_b200.position_priors([0, N - 1], X[[0, N - 1], 9:], 100 * np.eye(3)))
    for gm in (0, 1):
        assert _status(lambda: c.rig_damping_iter(base, ext, gauge_mode=gm, min_planes_per_pose=0)) == L.ERR_INVALID
    Hr, gr, _ = c.rig_evaluate(base, ext)
    Xc = rr.compose(base, ext, sc["base_of"], sc["lidar_of"])
    H, g, _ = c.evaluate(Xc)
    J = rr.jacobian(base, sc["base_of"], sc["lidar_of"], B, var)
    Href = J.T @ H @ J + rr.correction(base, sc["base_of"], sc["lidar_of"], B, var, g)
    assert _rel(Hr, Href) < 1e-12 and _rel(gr, J.T @ g) < 1e-12
    _, _, tr = c.rig_damping_iter(base, ext, gauge_mode=2, max_iter=3, min_planes_per_pose=0)
    assert tr[0]["accepted"]
    c.set_block_factors([])
    assert c.rig_block_structure()["pairs"] == n0
    c.close()


def test_block_covariance():
    # At the LM optimum: H_rig carries the composition's second-order term, which away from it (and on the fix scene,
    # 30 m from the origin, even there) leaves H_rig indefinite, and the Laplace form needs a positive definite one.
    # The gauge is held by a fixed base pose on the ragged scene and by the anchor base 0 on the dense one.
    for name, fixed, anchor in (("ragged", (0,), -1), ("dense", (), 0)):
        sc, base_of, lidar_of, base, ext = rig_case(name)
        c = _ctx(sc)
        n_rig = c.set_block_rig(base_of, lidar_of, fixed_bases=fixed)
        base, ext, _ = c.rig_damping_iter(base, ext, gauge_mode=2)
        H, _, _ = c.rig_evaluate(base, ext)
        keep = np.ones(n_rig, dtype=bool)
        if anchor >= 0:
            keep[6 * anchor:6 * anchor + 6] = False
        S = np.zeros_like(H)
        S[np.ix_(keep, keep)] = np.linalg.inv(H[np.ix_(keep, keep)])
        pairs, cov = c.rig_block_covariance(base, ext, anchor=anchor)
        ref = np.stack([S[6 * u:6 * u + 6, 6 * v:6 * v + 6] for u, v in pairs])
        assert np.abs(cov - ref).max() < 1e-8 * np.abs(ref).max()
        c.close()
    # the base poses' gauge left free: NOT_PD; a call leaves the next rig_damping_iter bitwise as without it
    sc, base_of, lidar_of, base, ext = rig_case("dense")
    a, b = _ctx(sc), _ctx(sc)
    a.set_block_rig(base_of, lidar_of)
    b.set_block_rig(base_of, lidar_of)
    bo, eo, _ = b.rig_damping_iter(base, ext, gauge_mode=2)
    assert _status(lambda: a.rig_block_covariance(bo, eo, anchor=-1)) == L.ERR_NOT_PD
    a.rig_block_covariance(bo, eo, anchor=0)
    ra = a.rig_damping_iter(base, ext, gauge_mode=2, want_per_iter=True)
    rb_ = b.rig_damping_iter(base, ext, gauge_mode=2, want_per_iter=True)
    assert ra[2] == rb_[2] and np.array_equal(ra[0], rb_[0]) and np.array_equal(ra[1], rb_[1])
    a.close()
    b.close()
    # the identity rig's covariance is bitwise the blocks context's
    sc = make_scene(n_poses=8, n_planes=50, seed=7, with_fix=True)
    x = sc["poses_init"]
    ident = np.concatenate([np.eye(3).reshape(9), np.zeros(3)])[None]
    a, b = _ctx(sc), _ctx(sc)
    b.set_block_rig(np.arange(8), np.zeros(8))
    pa, ca = a.block_covariance(x, include_fix=True, anchor=0)
    pb, cb = b.rig_block_covariance(x, ident, include_fix=True, anchor=0)
    assert np.array_equal(pa, pb) and np.array_equal(ca, cb)
    a.close()
    b.close()


def test_refusals_lifetime_and_memory():
    import torch
    sc, base_of, lidar_of, base, ext = rig_case("dense")
    x = sc["poses_init"]
    dense = _ctx(sc, L.PREC_FP64)
    assert _status(lambda: dense.set_block_rig(base_of, lidar_of)) == L.ERR_INVALID
    dense.close()
    blk = _ctx(sc)
    assert _status(lambda: blk.set_rig(base_of, lidar_of)) == L.ERR_UNSUPPORTED
    assert _status(lambda: blk.rig_evaluate(base, ext)) == L.ERR_INVALID  # no rig yet
    blk.set_block_rig(base_of, lidar_of)
    H0, g0, r0 = blk.rig_evaluate(base, ext)
    lib, h = L.lib(), blk._h
    n_out = C.c_int()
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
    bo, lo = i32(base_of), i32(lidar_of)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    f = lib.balm_block_set_rig
    assert f(h, 3, 2, p(i32(np.r_[base_of[:-1], 3])), p(lo), None, None, C.byref(n_out)) == L.ERR_INVALID
    assert f(h, 3, 2, p(bo), p(i32(np.r_[lidar_of[:-1], -1])), None, None, C.byref(n_out)) == L.ERR_INVALID
    assert f(h, 4, 2, p(bo), p(lo), None, None, C.byref(n_out)) == L.ERR_INVALID
    assert f(h, 3, 3, p(bo), p(lo), None, None, C.byref(n_out)) == L.ERR_INVALID
    ones = lambda k: np.ones(k, dtype=np.uint8)
    assert f(h, 3, 2, p(bo), p(lo), p(ones(3)), p(ones(2)), C.byref(n_out)) == L.ERR_INVALID
    H1, g1, r1 = blk.rig_evaluate(base, ext)
    assert np.array_equal(H0, H1) and np.array_equal(g0, g1) and r0 == r1
    assert _status(lambda: blk.rig_covariance(base, ext)) == L.ERR_UNSUPPORTED
    blk.set_block_rig(base_of, lidar_of, fixed_bases=(0,))
    for gm in (0, 1):
        assert _status(lambda: blk.rig_damping_iter(base, ext, gauge_mode=gm)) == L.ERR_INVALID
    blk.rig_damping_iter(base, ext, gauge_mode=2, max_iter=2)
    # after detach the context is bitwise one that never had a rig
    fresh = _ctx(sc)
    assert blk.set_block_rig(None, None) == 0
    assert _status(lambda: blk.rig_evaluate(base, ext)) == L.ERR_INVALID
    Ha, ga, ra = fresh.evaluate(x)
    Hb, gb, rb_ = blk.evaluate(x)
    assert np.array_equal(Ha, Hb) and np.array_equal(ga, gb) and ra == rb_
    pa, tra, _ = fresh.damping_iter(x, gauge_mode=0, max_iter=4)
    pb, trb, _ = blk.damping_iter(x, gauge_mode=0, max_iter=4)
    assert tra == trb and np.array_equal(pa, pb)
    fresh.close()
    blk.close()
    # device bytes: set_block_rig plus the first evaluation, against rig_block_structure (the blocks test's margin);
    # nothing of n_rig x 6N (2000 x 6 x 12000 doubles = 1.1 GB at this size)
    sc = rb.rig_corridor(500, 4, w=4, seed=3)
    c = _ctx(sc)
    c.evaluate(rr.compose(sc["base_init"], sc["ext_init"], sc["base_of"], sc["lidar_of"]))
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    c.set_block_rig(sc["base_of"], sc["lidar_of"])
    c.rig_evaluate(sc["base_init"], sc["ext_init"])
    used = free0 - torch.cuda.mem_get_info(0)[0]
    st = c.rig_block_structure()
    print(f"rig 500 x 4: {st}, mem_get_info delta {used / 2**20:.1f} MiB")
    assert st["device_bytes"] < 64 << 20 and used < 2 * st["device_bytes"] + (64 << 20)
    c.close()

"""Pose factors in the cost of a PREC_BLOCKS context (balm_block_set_factors / Context.set_block_factors): the evaluation
as the bitwise sum of the voxel blocks and the sparse pose graph's factor blocks, the LM against a host oracle built from
an fp64 context and pose_graph_ref, the pure pose graph, plane-poor scans carried by odometry, covariances, registration
routes, refusals and size."""
import numpy as np
import pytest

import assoc_ref
import balm_b200
import block_hessian_ref as bref
import pose_graph_ref as pgr
import scenes
from balm_b200 import _lib as L
from test_gpu_block_hessian import _ctx, _pattern_mask
from test_gpu_sparse_covariance import _dense_sigma

pytestmark = pytest.mark.gpu

POINT_NOISE = 0.01  # bref.corridor's default


def _noisy_odometry(rng, gt, info, rot=0.002, tran=0.02, edges=None):
    """odometry_factors from the truth, each relative pose perturbed on the right by N(0, rot / tran)."""
    edges = [(i, i + 1) for i in range(len(gt) - 1)] if edges is None else edges
    out = []
    for a, b in edges:
        Rb, pb = pgr.split(gt[b])
        d = np.concatenate([rng.normal(0, rot, 3), rng.normal(0, tran, 3)])
        hb = pgr.pack(Rb @ pgr.exp_so3(d[:3]), Rb @ d[3:] + pb)
        f = balm_b200.odometry_factors(np.stack([gt[a], hb]), info)[0]
        f["poses"] = np.array([a, b], dtype=np.int32)
        out.append(f)
    return out


def _odo_info(rot=0.002, tran=0.02):
    """information of the odometry noise above, in the voxel cost's units: the voxel cost is a sum of squared point
    distances, so its Hessian over 2 sigma_p^2 is the information; the factors' H is scaled the same way"""
    return 2 * POINT_NOISE ** 2 * np.diag(np.r_[np.full(3, rot ** -2), np.full(3, tran ** -2)])


def _factors(sc, seed, loops=((35, 3), (55, 20)), windows=((10, 11, 12),)):
    """noisy odometry over every consecutive pair, loop closures (a, b) and HBA-like window factors from the truth"""
    rng = np.random.default_rng(seed)
    gt = sc["poses_gt"]
    fs = _noisy_odometry(rng, gt, _odo_info())
    fs += [pgr.make_factor(rng, gt, list(ab), noise=0.002, cond=1e3) for ab in loops]
    fs += [pgr.make_factor(rng, gt, list(w), noise=0.002, cond=1e3) for w in windows]
    return fs


SCENES = {
    "corridor60": lambda: bref.corridor(60, w=4, planes_per_pose=30, seed=31),
    "corridor80fix": lambda: bref.corridor(80, w=5, planes_per_pose=30, seed=32, with_fix=True),
}


def _pair_index(pairs):
    return {(int(i), int(j)): p for p, (i, j) in enumerate(pairs)}


def _check_decomposition(cb, c0, factors, poses, include_fix=False):
    """cb (voxels + factors) == c0 (the same voxels) + PoseGraph(factors), added on the host in that order, bitwise"""
    Hb, gb, rb = cb.evaluate(poses, include_fix=include_fix)
    pairs = cb.block_structure(want_pairs=True)["pair_list"]
    blocks = cb.download_blocks()
    _, g0, r0 = c0.evaluate(poses, include_fix=include_fix, want_H=False)
    p0, b0 = c0.block_structure(want_pairs=True)["pair_list"], c0.download_blocks()
    spg = balm_b200.PoseGraph(cb.N)
    status = spg.set_pose_factors(factors)
    pp, pb, pg_g, pg_c = spg.pose_graph_evaluate(poses)
    spg.close()
    union = sorted(set(map(tuple, p0.tolist())) | set(map(tuple, pp.tolist())) | {(i, i) for i in range(cb.N)})
    assert pairs.tolist() == [list(t) for t in union]
    idx = _pair_index(pairs)
    exp = np.zeros((len(pairs), 6, 6))
    exp[[idx[tuple(t)] for t in p0.tolist()]] += b0
    exp[[idx[tuple(t)] for t in pp.tolist()]] += pb
    assert np.array_equal(blocks, exp)
    assert np.array_equal(gb, g0 + pg_g) and rb == r0 + pg_c
    mask = _pattern_mask(cb.N, pairs)
    assert not Hb[~mask].any()
    assert np.array_equal(Hb, bref.to_sparse(cb.N, pairs, blocks).toarray())
    return status


def _pair(sc, factors):
    cb, c0 = _ctx(sc, L.PREC_BLOCKS), _ctx(sc, L.PREC_BLOCKS)
    status = cb.set_block_factors(factors)
    return cb, c0, status


@pytest.mark.parametrize("name", list(SCENES))
def test_decomposition_and_sub_ranges(name):
    sc = SCENES[name]()
    fs = _factors(sc, 1)
    cb, c0, status = _pair(sc, fs)
    assert status == [L.OK] * len(fs)
    assert len(cb.block_structure(want_pairs=True)["pair_list"]) > len(c0.block_structure(want_pairs=True)["pair_list"])
    for include_fix in (False, True):
        for x in (sc["poses_init"], sc["poses_gt"]):
            _check_decomposition(cb, c0, fs, x, include_fix)
    M = len(sc["row_ptr"]) - 1
    for head, end in [(0, M // 3), (M // 3, M), (M // 2, M // 2 + 1), (5, 5), (0, M - 1)]:
        H1, g1, r1 = cb.evaluate(sc["poses_init"], head, end)
        H0, g0, r0 = c0.evaluate(sc["poses_init"], head, end)
        assert np.array_equal(H1, H0) and np.array_equal(g1, g0) and r1 == r0
    cb.reset_counters()
    cb.evaluate(sc["poses_init"], want_H=False)
    assert cb.timings()["ms_assemble"] > 0
    # detached: structure, evaluation and LM bitwise those of a context that never had factors
    assert cb.set_block_factors([]) == []
    assert cb.block_structure(want_pairs=True).keys() == c0.block_structure(want_pairs=True).keys()
    s1, s0 = cb.block_structure(want_pairs=True), c0.block_structure(want_pairs=True)
    assert all(np.array_equal(s1[k], s0[k]) for k in s0)
    H1, g1, r1 = cb.evaluate(sc["poses_init"])
    H0, g0, r0 = c0.evaluate(sc["poses_init"])
    assert np.array_equal(H1, H0) and np.array_equal(g1, g0) and r1 == r0
    assert np.array_equal(cb.download_blocks(), c0.download_blocks())
    cb.reset_counters()
    kw = dict(max_iter=5, gauge_mode=2, min_planes_per_pose=0, want_per_iter=True)
    p1, t1, per1 = cb.damping_iter(sc["poses_init"], **kw)
    p0, t0, per0 = c0.damping_iter(sc["poses_init"], **kw)
    assert np.array_equal(per1, per0) and t1 == t0
    assert cb.timings()["ms_assemble"] == 0


def _lm_oracle(cd, factors, x0, max_iter, include_fix, u0=0.01, v0=2.0, rel_tol=1e-6):
    """pose_graph_ref.lm's rule on fp64 voxels + factors: H, g, r from cd.evaluate + pose_graph_ref.evaluate, the trial
    cost from cd.residual + pose_graph_ref.cost"""
    N = cd.N
    x = np.array(x0, copy=True)
    u, v, calc = u0, v0, True
    acc, per = [], []
    for _ in range(max_iter):
        if calc:
            H, g, r1 = cd.evaluate(x, include_fix=include_fix)
            Hf, gf, rf = pgr.evaluate(x, factors, N)
            H, g, r1 = H + Hf, g + gf, r1 + rf
        D = np.diag(H).copy()
        dx = np.linalg.solve(H + u * np.diag(D), -g)
        q1 = 0.5 * dx @ (u * D * dx - g)
        xt = pgr.pose_update(x, dx)
        r2 = cd.residual(xt) + pgr.cost(xt, factors)
        q = r1 - r2
        if q > 0:
            x = xt
            u *= max(1 - (2 * q / q1 - 1) ** 3, 1.0 / 3.0)
            v, calc = 2.0, True
        else:
            u, v, calc = u * v, 2 * v, False
        acc.append(q > 0)
        per.append(x.copy())
        if rel_tol >= 0 and abs(r1 - r2) / r1 < rel_tol:
            break
    return acc, np.array(per)


@pytest.mark.parametrize("name", list(SCENES))
def test_damping_iter_against_the_host_oracle(name):
    sc = SCENES[name]()
    include_fix = sc.get("fix10") is not None
    fs = _factors(sc, 2)
    cb = _ctx(sc, L.PREC_BLOCKS)
    cb.set_block_factors(fs)
    cd = _ctx(sc, L.PREC_FP64)
    _, tb, per_b = cb.damping_iter(sc["poses_init"], max_iter=8, gauge_mode=2, min_planes_per_pose=0,
                                   want_per_iter=True, hess_includes_fix=include_fix)
    acc, per_o = _lm_oracle(cd, fs, sc["poses_init"], 8, include_fix)
    assert [t["accepted"] for t in tb] == acc
    gap = np.abs(per_b - per_o).max()
    print(f"{name}: largest per-iteration pose gap against the host oracle {gap:.2e}")
    assert gap < 1e-9 and tb[-1]["r2"] < tb[0]["r1"] and not any(t["not_pd"] for t in tb)


def test_pure_pose_graph():
    """An empty voxel registration and factors on every pose: PoseGraph's pairs, blocks, g, cost, LM poses and trace"""
    rng = np.random.default_rng(3)
    N = 90
    gt = bref.corridor(N, w=4, seed=33)["poses_gt"]
    fs = _noisy_odometry(rng, gt, _odo_info())
    fs += [pgr.make_factor(rng, gt, idx, noise=0.002) for idx in ([0, 40, 80], [5, 6, 7, 8], [70, 20])]
    x0 = pgr.perturb(rng, gt, 0.01, 0.1)
    c = balm_b200.Context(N, 0, L.PREC_BLOCKS)
    c.set_block_factors(fs)  # before any registration
    c.set_voxels(np.zeros(1, np.int64), np.zeros(0, np.int32), np.zeros((0, 10)), np.zeros(0))
    spg = balm_b200.PoseGraph(N)
    spg.set_pose_factors(fs)
    st, sst = c.block_structure(want_pairs=True), spg.structure()
    assert (st["pairs"], st["l_blocks"], st["levels"]) == (sst["pairs"], sst["l_blocks"], sst["levels"])
    _, g, r = c.evaluate(x0, want_H=False)
    pairs, blocks, pg_g, pg_c = spg.pose_graph_evaluate(x0)
    assert np.array_equal(st["pair_list"], pairs)
    assert np.array_equal(c.download_blocks(), blocks) and np.array_equal(g, pg_g) and r == pg_c
    for gauge_mode in (0, 2):
        p1, t1, _ = c.damping_iter(x0, max_iter=8, gauge_mode=gauge_mode, min_planes_per_pose=0)
        p2, t2 = spg.pose_graph_iter(x0, max_iter=8, gauge_mode=gauge_mode)
        assert np.array_equal(p1, p2) and t1 == t2
        assert t1[-1]["r2"] < t1[0]["r1"]


def test_scans_without_planes_carried_by_odometry():
    sc = bref.corridor(80, w=4, planes_per_pose=30, seed=34)
    gap = np.arange(38, 42)
    keep = ~np.isin(sc["pose_idx"], gap)
    k = np.add.reduceat(keep.astype(np.int64), sc["row_ptr"][:-1])
    sc = dict(sc, pose_idx=sc["pose_idx"][keep], obs10=sc["obs10"][keep],
              row_ptr=np.concatenate([[0], np.cumsum(k)]).astype(np.int64))
    c = _ctx(sc, L.PREC_BLOCKS)
    _, t, _ = c.damping_iter(sc["poses_init"], max_iter=2, min_planes_per_pose=0)
    assert t[0]["not_pd"]
    with pytest.raises(balm_b200.BalmError) as e:
        c.block_covariance(sc["poses_init"])
    assert e.value.status == L.ERR_NOT_PD
    rng = np.random.default_rng(4)
    c.set_block_factors(_noisy_odometry(rng, sc["poses_gt"], _odo_info()))
    x, t, _ = c.damping_iter(sc["poses_init"], max_iter=30, gauge_mode=2, min_planes_per_pose=0)
    assert not any(s["not_pd"] for s in t) and t[-1]["r2"] < t[0]["r1"]
    pairs, cov = c.block_covariance(x)
    sigma = np.sqrt(2 * POINT_NOISE ** 2 * np.array([np.diag(cov[p]) for p in range(len(pairs))
                                                     if pairs[p, 0] == pairs[p, 1]]))
    xa = _align_rigid(x, sc["poses_gt"])
    z = []
    for i in gap:  # the error in the coordinates of the pose update: R = Exp(dth) R_true, p = Exp(dth) p_true + dp
        R, p = pgr.split(xa[i])
        Rt, pt = pgr.split(sc["poses_gt"][i])
        dth = pgr.log_so3(R @ Rt.T)
        z.append(np.concatenate([dth, p - pgr.exp_so3(dth) @ pt]) / sigma[i])
    worst = np.abs(z).max()
    print(f"gap poses after {len(t)} iterations: errors in sigma {np.round(z, 2).tolist()}; "
          f"sigma {sigma[gap].min():.2e} .. {sigma[gap].max():.2e}")
    assert worst < 5


def _align_rigid(poses, gt):
    """poses moved by the rigid transform that best fits them to gt: rotation from every pose's orientation (positions
    along a corridor leave the roll about its axis to noise), then the mean offset of the positions"""
    Rs = [pgr.split(p)[0] for p in poses]
    U, _, Vt = np.linalg.svd(sum(pgr.split(g)[0] @ R.T for g, R in zip(gt, Rs)))
    A = U @ np.diag([1, 1, np.linalg.det(U @ Vt)]) @ Vt
    t = np.mean([pgr.split(g)[1] - A @ pgr.split(p)[1] for g, p in zip(gt, poses)], axis=0)
    return np.array([pgr.pack(A @ R, A @ pgr.split(p)[1] + t) for R, p in zip(Rs, poses)])


def test_covariance_against_the_dense_inverse():
    for name, include_fix, anchor in [("corridor60", False, 0), ("corridor80fix", True, -1)]:
        sc = SCENES[name]()
        fs = _factors(sc, 5)
        cb = _ctx(sc, L.PREC_BLOCKS)
        cb.set_block_factors(fs)
        x, _, _ = cb.damping_iter(sc["poses_init"], max_iter=10, gauge_mode=2, min_planes_per_pose=0,
                                  hess_includes_fix=include_fix)
        pairs, cov = cb.block_covariance(x, include_fix=include_fix, anchor=anchor)
        cd = _ctx(sc, L.PREC_FP64)
        H = cd.evaluate(x, include_fix=include_fix)[0] + pgr.evaluate(x, fs, cb.N)[0]
        S, kappa = _dense_sigma(H, anchor)
        err = np.abs(cov - bref.blocks_of(S, pairs)).max() / np.abs(cov).max()
        print(f"{name} anchor {anchor}: kappa {kappa:.1e}, error {err:.1e} of max |Sigma|")
        assert err <= max(1e-9, 10 * kappa * 1e-12)
        # the next LM call is bitwise what it is without the covariance call
        cc = _ctx(sc, L.PREC_BLOCKS)
        cc.set_block_factors(fs)
        kw = dict(max_iter=3, gauge_mode=2, min_planes_per_pose=0, hess_includes_fix=include_fix)
        assert np.array_equal(cb.damping_iter(x, **kw)[0], cc.damping_iter(x, **kw)[0])


def test_registration_routes():
    N = 10
    pts, frs, poses = assoc_ref.synthetic_scans(n_poses=N, pts_per_scan=4000, seed=21)
    P = scenes.pack_poses([r for r, _ in poses], [p for _, p in poses])
    kw = dict(voxel_size=2.0, layer_limit=2, min_ps=15, eigen_value_array=(1 / 16, 1 / 16, 1 / 9))
    rng = np.random.default_rng(6)
    fs = _noisy_odometry(rng, P, _odo_info()) + [pgr.make_factor(rng, P, [0, 7], noise=0.002)]
    x = pgr.perturb(rng, P, 0.002, 0.02)
    win = frs < N - 1
    cb, c0 = balm_b200.Context(N, 0, L.PREC_BLOCKS), balm_b200.Context(N, 0, L.PREC_BLOCKS)
    cb.set_block_factors(fs)
    for c in (cb, c0):
        c.cut_voxels(pts[win].astype(np.float32), frs[win], P, **kw)
    _check_decomposition(cb, c0, fs, x)
    assert cb.marginalize(2, P) == c0.marginalize(2, P)
    _check_decomposition(cb, c0, fs, x, include_fix=True)
    last = pts[frs == N - 1].astype(np.float32)
    assert cb.append_scan(last, P, N - 2) == c0.append_scan(last, P, N - 2)
    _check_decomposition(cb, c0, fs, x, include_fix=True)
    for c in (cb, c0):
        c.window_reset(**kw)
        for s in range(N):
            c.window_cut(pts[frs == s].astype(np.float32), P[s], s)
            c.window_recut(s + 1)
        c.window_push(N)
    _check_decomposition(cb, c0, fs, x, include_fix=True)


def test_refusals_repeatability_memory():
    sc = SCENES["corridor60"]()
    fs = _factors(sc, 7)
    lib = L.lib()
    for prec in (L.PREC_FP64, L.PREC_TENSOR):  # other contexts: refused, nothing changed
        c = _ctx(sc, prec)
        H0, g0, r0 = c.evaluate(sc["poses_init"])
        assert lib.balm_block_set_factors(c._h, 0, None, None, None, None, None) == L.ERR_INVALID
        with pytest.raises(balm_b200.BalmError) as e:
            c.set_block_factors(fs)
        assert e.value.status == L.ERR_INVALID and "balm_block_set_factors" in str(e.value)
        H1, g1, r1 = c.evaluate(sc["poses_init"])
        assert np.array_equal(H1, H0) and np.array_equal(g1, g0) and r1 == r0
        c.close()
    c0 = _ctx(sc, L.PREC_BLOCKS)
    bytes0 = c0.block_structure()["device_bytes"]
    cb, _, _ = _pair(sc, fs)
    st = cb.block_structure(want_pairs=True)
    H0, g0, r0 = cb.evaluate(sc["poses_init"])
    assert st["device_bytes"] > bytes0
    bad = [dict(f) for f in fs]
    bad[3] = dict(bad[3], poses=np.array([3, 60], dtype=np.int32))  # index out of range
    for factors in (bad, [dict(fs[0], H=np.full((12, 12), np.nan))]):
        with pytest.raises(balm_b200.BalmError) as e:
            cb.set_block_factors(factors)
        assert e.value.status == L.ERR_INVALID and "balm_block_set_factors" in str(e.value)
    st1 = cb.block_structure(want_pairs=True)
    assert all(np.array_equal(st1[k], st[k]) for k in st)
    H1, g1, r1 = cb.evaluate(sc["poses_init"])
    assert np.array_equal(H1, H0) and np.array_equal(g1, g0) and r1 == r0
    # a NOT_PD factor is left out of the pattern and every sum
    singular = pgr.make_factor(np.random.default_rng(8), sc["poses_gt"], [2, 50])
    singular["H"] = np.zeros((12, 12))
    assert cb.set_block_factors(fs + [singular])[-1] == L.ERR_NOT_PD
    st2 = cb.block_structure(want_pairs=True)
    assert np.array_equal(st2["pair_list"], st["pair_list"])
    H2, g2, r2 = cb.evaluate(sc["poses_init"])
    assert np.array_equal(H2, H0) and np.array_equal(g2, g0) and r2 == r0
    # detaching gives the factor set's memory back
    cb.set_block_factors([])
    assert cb.block_structure()["device_bytes"] == bytes0
    # two runs are bitwise equal
    runs = []
    for _ in range(2):
        c = _ctx(sc, L.PREC_BLOCKS)
        c.set_block_factors(fs)
        _, g, r = c.evaluate(sc["poses_init"], want_H=False)
        p, t, _ = c.damping_iter(sc["poses_init"], max_iter=5, gauge_mode=2, min_planes_per_pose=0)
        runs.append((g, r, c.download_blocks(), p, [s["r2"] for s in t]))
        c.close()
    for a, b in zip(*runs):
        assert np.array_equal(np.asarray(a), np.asarray(b))
    assert lib.balm_block_set_factors(None, 0, None, None, None, None, None) == L.ERR_INVALID


def test_20000_poses_with_odometry_and_loop_closures():
    import time
    import torch
    sc = bref.corridor(20000, w=8, planes_per_pose=30, pts=6, seed=8)
    N, gt = sc["n_poses"], sc["poses_gt"]
    rng = np.random.default_rng(9)
    loops = [(a, a - 300) for a in range(500, N, 500)]
    fs = _noisy_odometry(rng, gt, _odo_info()) + \
        balm_b200.odometry_factors(gt, _odo_info(), edges=loops)
    free0 = torch.cuda.mem_get_info(0)[0]
    c = _ctx(sc, L.PREC_BLOCKS)
    base = c.block_structure()
    assert c.set_block_factors(fs) == [L.OK] * len(fs)
    st = c.block_structure()
    used = free0 - torch.cuda.mem_get_info(0)[0]
    print(f"N = 20000: voxels only {base}, with factors {st}, mem_get_info delta {used / 2**30:.2f} GB")
    assert st["device_bytes"] < 4 << 30 and used < 6 << 30
    c.reset_counters()
    t0 = time.perf_counter()
    p, t, _ = c.damping_iter(sc["poses_init"], max_iter=10, gauge_mode=2, min_planes_per_pose=0)
    ms = 1e3 * (time.perf_counter() - t0) / len(t)
    tm = c.timings()
    print(f"N = 20000 with {len(fs)} factors: {ms:.1f} ms per LM iteration, ms_assemble {tm['ms_assemble']:.2f} ms "
          f"over {tm['n_eval']} evaluations, r {t[0]['r1']:.4e} -> {t[-1]['r2']:.4e}")
    assert t[-1]["r2"] < t[0]["r1"] and not any(s["not_pd"] for s in t)

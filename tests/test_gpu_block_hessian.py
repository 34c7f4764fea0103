"""PREC_BLOCKS contexts (block-sparse Hessian, nested-dissection solve) against fp64 contexts on the same scenes, the CPU
oracle and the scipy.sparse restatement block_hessian_ref.py."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import assoc_ref
import block_hessian_ref as bref
import scenes
from balm_b200 import _lib as L

pytestmark = pytest.mark.gpu

SCENES = {
    "corridor40": lambda: bref.corridor(40, w=4, planes_per_pose=30, seed=1),
    "corridor300": lambda: bref.corridor(300, w=10, planes_per_pose=30, seed=2, with_fix=True),
    "dense": lambda: scenes.make_scene(n_poses=12, n_planes=80, seed=3),
    "drop": lambda: scenes.make_scene(n_poses=16, n_planes=120, seed=4, drop=0.4, with_fix=True),
}


def _ctx(sc, prec):
    import balm_b200
    c = balm_b200.Context(sc["n_poses"], 0, prec)
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc.get("fix10"))
    return c


def _pattern_mask(N, pairs):
    m = np.zeros((N, N), bool)
    m[pairs[:, 0], pairs[:, 1]] = m[pairs[:, 1], pairs[:, 0]] = True
    return np.kron(m, np.ones((6, 6), bool))


def _check_eval(cb, cd, poses, head=0, end=None, include_fix=False):
    Hd, gd, rd = cd.evaluate(poses, head, end, include_fix)
    Hb, gb, rb = cb.evaluate(poses, head, end, include_fix)
    assert rb == rd and np.array_equal(gb, gd)  # the same sweep and reductions: bitwise
    st = cb.block_structure(want_pairs=True)
    pairs = st["pair_list"]
    blocks = cb.download_blocks()
    scale = np.abs(Hd).max()
    assert np.abs(blocks - bref.blocks_of(Hd, pairs)).max() <= 1e-12 * scale
    mask = _pattern_mask(cb.N, pairs)
    assert not Hd[~mask].any() and not Hb[~mask].any()  # exact zeros outside the pattern
    assert np.abs(Hb - Hd).max() <= 1e-12 * scale
    return blocks


@pytest.mark.parametrize("name", list(SCENES))
def test_evaluation_matches_fp64(name):
    sc = SCENES[name]()
    cb, cd = _ctx(sc, L.PREC_BLOCKS), _ctx(sc, L.PREC_FP64)
    for include_fix in (False, True):
        _check_eval(cb, cd, sc["poses_init"], include_fix=include_fix)
    M = len(sc["row_ptr"]) - 1
    for head, end in [(0, M // 3), (M // 3, M), (M // 2, M // 2 + 1), (5, 5)]:
        _check_eval(cb, cd, sc["poses_init"], head, end)
    tm = cb.timings()
    assert tm["ms_assemble"] == 0 and tm["ms_syrk"] > 0


@pytest.mark.parametrize("name", list(SCENES))
def test_damping_iter_matches_fp64(name):
    sc = SCENES[name]()
    cb, cd = _ctx(sc, L.PREC_BLOCKS), _ctx(sc, L.PREC_FP64)
    kw = dict(max_iter=8, gauge_mode=2, min_planes_per_pose=0, want_per_iter=True, hess_includes_fix=True)
    pb, tb, per_b = cb.damping_iter(sc["poses_init"], **kw)
    pd, td, per_d = cd.damping_iter(sc["poses_init"], **kw)
    assert [t["accepted"] for t in tb] == [t["accepted"] for t in td]
    gap = np.abs(per_b - per_d).max()
    print(f"{name}: largest per-iteration pose gap blocks vs fp64 {gap:.2e}")
    assert gap < 1e-9 and tb[-1]["r2"] < tb[0]["r1"]


def test_damping_iter_matches_oracle():
    from oracle import oracle_py as orc
    sc = SCENES["drop"]()
    o = orc.Oracle(sc["n_poses"], sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
    cb = _ctx(dict(sc, fix10=None), L.PREC_BLOCKS)
    pb, tb, per_b = cb.damping_iter(sc["poses_init"], gauge_mode=2, want_per_iter=True)
    st, po, to, per_o = o.damping_iter(sc["poses_init"], gauge_mode=2)
    assert [t["accepted"] for t in tb] == [t["accepted"] for t in to]
    assert np.abs(pb - po).max() < 1e-6


def test_repeatable():
    sc = SCENES["corridor300"]()
    runs = []
    for _ in range(2):
        c = _ctx(sc, L.PREC_BLOCKS)
        H, g, r = c.evaluate(sc["poses_init"], want_H=False)
        b = c.download_blocks()
        p, t, _ = c.damping_iter(sc["poses_init"], max_iter=5, min_planes_per_pose=0)
        runs.append((g, r, b, p, [x["r2"] for x in t]))
        c.close()
    for a, b in zip(*runs):
        assert np.array_equal(np.asarray(a), np.asarray(b))


def test_registration_routes():
    """cut_voxels, then marginalize and append_scan; and a window_push stream: after every step the evaluation is the
    fp64 context's."""
    import balm_b200
    N = 10
    pts, frs, poses = assoc_ref.synthetic_scans(n_poses=N, pts_per_scan=4000, seed=21)
    P = scenes.pack_poses([r for r, _ in poses], [p for _, p in poses])
    kw = dict(voxel_size=2.0, layer_limit=2, min_ps=15, eigen_value_array=(1 / 16, 1 / 16, 1 / 9))
    win = frs < N - 1
    cb, cd = balm_b200.Context(N, 0, L.PREC_BLOCKS), balm_b200.Context(N, 0, L.PREC_FP64)
    for c in (cb, cd):
        c.cut_voxels(pts[win].astype(np.float32), frs[win], P, **kw)
    _check_eval(cb, cd, P)
    assert cb.marginalize(2, P) == cd.marginalize(2, P)
    _check_eval(cb, cd, P, include_fix=True)
    last = pts[frs == N - 1].astype(np.float32)
    assert cb.append_scan(last, P, N - 2) == cd.append_scan(last, P, N - 2)
    _check_eval(cb, cd, P, include_fix=True)
    for c in (cb, cd):
        c.window_reset(**kw)
        for s in range(N):
            c.window_cut(pts[frs == s].astype(np.float32), P[s], s)
            c.window_recut(s + 1)
        c.window_push(N)
    _check_eval(cb, cd, P, include_fix=True)


def test_pose_in_no_voxel_is_not_pd():
    sc = bref.corridor(40, w=4, planes_per_pose=30, seed=5)
    keep = sc["pose_idx"] != 17  # pose 17 observes nothing
    k = np.add.reduceat(keep.astype(np.int64), sc["row_ptr"][:-1])
    sc = dict(sc, pose_idx=sc["pose_idx"][keep], obs10=sc["obs10"][keep],
              row_ptr=np.concatenate([[0], np.cumsum(k)]).astype(np.int64))
    for prec in (L.PREC_BLOCKS, L.PREC_FP64):
        c = _ctx(sc, prec)
        c.evaluate(sc["poses_init"], want_H=False)
        assert c.solve(0.01)[2]
        _, t, _ = c.damping_iter(sc["poses_init"], max_iter=2, min_planes_per_pose=0)
        assert t[0]["not_pd"]


def test_empty_registration():
    import balm_b200
    c = balm_b200.Context(7, 0, L.PREC_BLOCKS)
    c.set_voxels(np.zeros(1, np.int64), np.zeros(0, np.int32), np.zeros((0, 10)), np.zeros(0))
    H, g, r = c.evaluate(np.tile(np.eye(4)[:3].T.ravel(), (7, 1)))
    assert not H.any() and not g.any() and r == 0
    st = c.block_structure()
    assert st["pairs"] == 7 and not c.download_blocks().any()


def test_unsupported_calls_change_nothing():
    import balm_b200
    sc = SCENES["corridor40"]()
    c = _ctx(sc, L.PREC_BLOCKS)
    H0, g0, r0 = c.evaluate(sc["poses_init"])
    b0 = c.download_blocks()
    lib, h = L.lib(), c._h
    calls = [lambda: lib.balm_comm_init(h, 0, 2, bytes(128)),
             lambda: lib.balm_pose_covariance(h, sc["poses_init"].ctypes.data, None, 0.0, 0, np.zeros(1).ctypes.data, None),
             lambda: lib.balm_set_pose_factors(h, 1, None, None, None, None, None),
             lambda: lib.balm_pose_graph_evaluate(h, sc["poses_init"].ctypes.data, None, None, None),
             lambda: lib.balm_pose_graph_iter(h, sc["poses_init"].ctypes.data, C.byref(L.LmOpts()), None, None, None),
             lambda: lib.balm_device_views(h, None, None),
             lambda: lib.balm_debug_tc_trace(h, np.zeros(4, np.uint64).ctypes.data, 4),
             lambda: lib.balm_debug_tc_planes(h, None, None, None, None, None),
             lambda: lib.balm_debug_syrk_tc(h, np.zeros(4, np.int8).ctypes.data, 2, 1, np.zeros(4).ctypes.data, 1, 0,
                                            np.zeros(4).ctypes.data)]
    for call in calls:
        assert call() == L.ERR_UNSUPPORTED, lib.balm_last_error()
    assert np.array_equal(c.download_blocks(), b0)
    H1, g1, r1 = c.evaluate(sc["poses_init"])
    assert np.array_equal(H1, H0) and np.array_equal(g1, g0) and r1 == r0
    with pytest.raises(balm_b200.BalmError):
        balm_b200.Context(4, 0, L.PREC_FP64).block_structure()


def test_over_budget_registration_is_refused(monkeypatch):
    import balm_b200
    sc = SCENES["corridor300"]()
    c = _ctx(sc, L.PREC_BLOCKS)
    assert 144 * len(sc["pose_idx"]) > 1 << 20
    monkeypatch.setenv("BALM_G_BUDGET_MB", "1")
    with pytest.raises(balm_b200.BalmError) as e:
        c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
    assert e.value.status == L.ERR_UNSUPPORTED and "G' budget" in str(e.value)
    with pytest.raises(balm_b200.BalmError):
        c.evaluate(sc["poses_init"])  # left unregistered


def test_5000_poses_against_the_restatement():
    sc = bref.corridor(5000, w=8, planes_per_pose=30, seed=7)
    c = _ctx(sc, L.PREC_BLOCKS)
    _, g, r = c.evaluate(sc["poses_init"], want_H=False)
    pairs_r, blocks_r, g_r, r_r = bref.evaluate(sc, sc["poses_init"])
    st = c.block_structure(want_pairs=True)
    assert np.array_equal(st["pair_list"], pairs_r)
    blocks = c.download_blocks()
    pick = np.random.default_rng(0).choice(len(pairs_r), 2000, replace=False)
    # a different formulation of sums whose raw moments cancel at ~1 km: the two agree to 9e-11 of max |H| (measured);
    # against the fp64 context (same arithmetic) the blocks hold to 1e-12 (test_evaluation_matches_fp64)
    assert np.abs(blocks[pick] - blocks_r[pick]).max() <= 1e-9 * np.abs(blocks_r).max()
    assert np.abs(g - g_r).max() <= 1e-8 * np.abs(g_r).max()  # measured 2.4e-10: the same cancellation
    u = 0.01
    dx, q1, bad = c.solve(u)
    A = bref.to_sparse(5000, st["pair_list"], blocks)
    dx_ref = spla.spsolve((A + sp.diags(u * A.diagonal())).tocsc(), -g)
    print(f"N = 5000: dx against spsolve {np.abs(dx - dx_ref).max() / np.abs(dx_ref).max():.1e} of max |dx|")
    assert not bad and np.abs(dx - dx_ref).max() <= 1e-6 * np.abs(dx_ref).max()


def _align(poses, gt):
    """poses moved by the rigid transform that best fits their positions to gt's (BA leaves the global frame free)."""
    pe, pg = poses[:, 9:], gt[:, 9:]
    ce, cg = pe.mean(0), pg.mean(0)
    U, _, Vt = np.linalg.svd((pg - cg).T @ (pe - ce))
    R = U @ np.diag([1, 1, np.linalg.det(U @ Vt)]) @ Vt
    out = poses.copy()
    Re = poses[:, :9].reshape(-1, 3, 3).transpose(0, 2, 1)
    out[:, :9] = (R @ Re).transpose(0, 2, 1).reshape(-1, 9)
    out[:, 9:] = (pe - ce) @ R.T + cg
    return out


def test_20000_poses():
    import torch
    sc = bref.corridor(20000, w=8, planes_per_pose=30, pts=6, seed=8)
    free0 = torch.cuda.mem_get_info(0)[0]
    c = _ctx(sc, L.PREC_BLOCKS)
    st = c.block_structure()
    used = free0 - torch.cuda.mem_get_info(0)[0]
    print(f"N = 20000: {st}, mem_get_info delta {used / 2**30:.2f} GB")
    assert st["device_bytes"] < 4 << 30 and used < 6 << 30
    p, t, _ = c.damping_iter(sc["poses_init"], max_iter=10, gauge_mode=2, min_planes_per_pose=0)
    assert t[-1]["r2"] < t[0]["r1"]
    from balm_b200 import drivers
    rot, tran = drivers.rsme(_align(p, sc["poses_gt"]), sc["poses_gt"])
    rot0, tran0 = drivers.rsme(_align(sc["poses_init"], sc["poses_gt"]), sc["poses_gt"])
    print(f"N = 20000 RMSE {rot * 57.3:.4f} deg {tran:.4f} m (initial {rot0 * 57.3:.3f} deg {tran0:.3f} m)")
    assert rot < 0.3 * rot0 and tran < 0.4 * tran0  # measured: 0.15 and 0.31 of the initial error


def test_driver_route(tmp_path, monkeypatch):
    from balm_b200 import drivers, io
    pts_b, frames, poses = assoc_ref.synthetic_scans(n_poses=10, pts_per_scan=5000, seed=9)
    io.write_pose_csv(tmp_path / "alidarPose.csv", np.stack([r for r, _ in poses]), np.stack([p for _, p in poses]),
                      np.arange(10) * 0.1)
    for i in range(10):
        io.write_pcd(tmp_path / f"full{i}.pcd", pts_b[frames == i])
    ref = drivers.benchmark_realworld(str(tmp_path), voxel_size=2.0, precision=L.PREC_FP64, quiet=True)
    monkeypatch.setattr(drivers, "BLOCKS_MIN_POSES", 0)
    res = drivers.benchmark_realworld(str(tmp_path), voxel_size=2.0, precision=L.PREC_FP64, quiet=True)
    assert [t["accepted"] for t in res["trace"]] == [t["accepted"] for t in ref["trace"]]
    assert np.abs(res["poses"] - ref["poses"]).max() < 1e-9

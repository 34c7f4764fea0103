"""The sparse pose graph (balm_spg_*, balm_b200.PoseGraph) against the context's dense pose graph, the numpy oracle
pose_graph_ref.py and its scipy.sparse restatement pose_graph_sparse_ref.py, and hba(pose_graph=True) on its route."""
import os

import numpy as np
import pytest

import balm_b200
import hba_ref
import pose_graph_ref as pg
import pose_graph_sparse_ref as spg
from balm_b200 import _lib as L, hba

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "realworld_points_small.npz")
KINDS = [2, 10, 11, 21, 22, 32, "pyramid", "all", "many"]


def _factor_set(kind, seed=0):
    """-> (P, factors, poses): test_gpu_pose_graph's factor sets, and the shapes of this file: "loops" (a pyramid with
    long-range two-pose factors across the trajectory), "split" (two pyramids with no factor between them) and "hole"
    (a pyramid over every pose but the last)."""
    rng = np.random.default_rng(seed)
    if isinstance(kind, int):  # one factor of kind poses, scattered indices, plus a small one over its first slots
        P = 40
        sets = [list(rng.permutation(P)[:kind]), [int(i) for i in rng.permutation(P)[:2]]]
    elif kind == "pyramid":  # overlapping windows of 10 every 5, three layers
        P = 90
        sets = pg.pyramid_factor_poses(P, top=8)
    elif kind == "all":  # one factor covering every pose
        P = 32
        sets = [list(rng.permutation(P))]
    elif kind == "many":  # more factors than one block of threads
        P = 700
        sets = [list(range(s, s + 3)) for s in range(0, P - 2, 2)]
    elif kind == "loops":
        P = 300
        sets = pg.pyramid_factor_poses(P, top=32) + [[i, P - 1 - i] for i in range(0, P // 2, 37)]
    elif kind == "split":
        P = 160
        sets = pg.pyramid_factor_poses(80, top=8) + [[80 + i for i in s] for s in pg.pyramid_factor_poses(80, top=8)]
    elif kind == "hole":
        P = 91
        sets = pg.pyramid_factor_poses(90, top=8)
    truth = np.array([pg.random_pose(rng, 0.5, 3.0) for _ in range(P)])
    factors = [pg.make_factor(rng, truth, s, noise=0.01) for s in sets]
    return P, factors, pg.perturb(rng, truth, 0.05, 0.2)


def _covered(P, factors):
    return len({int(i) for f in factors for i in f["poses"]}) == P


def _sparse(P, factors):
    s = balm_b200.PoseGraph(P)
    assert s.set_pose_factors(factors) == [L.OK] * len(factors)
    return s


@pytest.mark.parametrize("kind", KINDS + ["loops", "split"])
def test_evaluation_is_bitwise_the_dense_context(kind):
    P, factors, x = _factor_set(kind)
    c = balm_b200.Context(P)
    c.set_pose_factors(factors)
    H, g, r = c.pose_graph_evaluate(x)
    s = _sparse(P, factors)
    pairs, B, gs, rs = s.pose_graph_evaluate(x)
    assert np.array_equal(pairs, spg.block_pairs(factors))
    assert np.array_equal(B, np.array([H[6 * i:6 * i + 6, 6 * j:6 * j + 6] for i, j in pairs]))
    assert np.array_equal(gs, g) and rs == r
    st = s.structure()
    assert st["pairs"] == len(pairs) and st["l_blocks"] >= len(pairs) and st["levels"] >= 1
    c.close()
    s.close()


def _lm_both(P, factors, x, **kw):
    c = balm_b200.Context(P)
    c.set_pose_factors(factors)
    pd, td = c.pose_graph_iter(x, want_per_iter=True, **kw)
    s = _sparse(P, factors)
    ps, ts = s.pose_graph_iter(x, want_per_iter=True, **kw)
    c.close()
    s.close()
    return (pd, td), (ps, ts)


def _same_lm(td, ts, pd, ps, tol=1e-9):
    assert [t["accepted"] for t in ts] == [t["accepted"] for t in td]
    assert [t["not_pd"] for t in ts] == [t["not_pd"] for t in td]
    r0 = td[0]["r1"]  # the scale of the costs: at the minimum of "all" they fall to the rounding of r0
    for a, b in zip(ts, td):
        assert abs(a["r1"] - b["r1"]) <= 1e-10 * max(b["r1"], r0)
        if not a["not_pd"]:  # the trial poses of a step whose factorisation failed are not comparable
            assert abs(a["r2"] - b["r2"]) <= 1e-10 * max(b["r1"], r0)
        assert np.abs(a["poses"] - b["poses"]).max() <= tol
    assert np.abs(ps - pd).max() <= tol


@pytest.mark.parametrize("kind", KINDS + ["loops", "split", "hole"])
def test_lm_matches_the_dense_path_and_the_oracle(kind):
    P, factors, x = _factor_set(kind, seed=1)
    (pd, td), (ps, ts) = _lm_both(P, factors, x, max_iter=8, gauge_mode=2)
    _same_lm(td, ts, pd, ps)
    if not _covered(P, factors):  # a pose in no factor: H + u diag(H) is singular, every step is rejected
        assert all(t["not_pd"] and not t["accepted"] for t in ts)
        return
    po, tro, per = pg.lm(x, factors, P, max_iter=8)
    assert [t["accepted"] for t in ts] == [t["accepted"] for t in tro]
    r0 = tro[0]["r1"]
    for a, b, p in zip(ts, tro, per):
        assert abs(a["r1"] - b["r1"]) <= 1e-10 * max(b["r1"], r0) and abs(a["r2"] - b["r2"]) <= 1e-10 * max(b["r1"], r0)
        assert np.abs(a["poses"] - p).max() <= 1e-9
    if kind in ("pyramid", "loops", "split"):
        assert ts[-1]["r2"] < 1e-2 * ts[0]["r1"]


def test_gauge_modes_and_forced_hessians_match_the_dense_path():
    P, factors, x = _factor_set("loops", seed=5)
    for kw in (dict(gauge_mode=0), dict(gauge_mode=1, force_hess=True), dict(gauge_mode=2, rel_tol=-1, max_iter=12)):
        (pd, td), (ps, ts) = _lm_both(P, factors, x, **kw)
        _same_lm(td, ts, pd, ps)


def test_two_registrations_are_bitwise_equal():
    P, factors, x = _factor_set("loops", seed=2)
    s = balm_b200.PoseGraph(P)
    out = []
    for _ in range(2):
        st = s.set_pose_factors(factors)
        out.append((st, s.structure(), s.pose_graph_evaluate(x), s.pose_graph_iter(x, max_iter=6, gauge_mode=2)))
    (s1, u1, e1, (p1, t1)), (s2, u2, e2, (p2, t2)) = out
    assert s1 == s2 and u1 == u2 and all(np.array_equal(a, b) for a, b in zip(e1, e2))
    assert np.array_equal(p1, p2) and str(t1) == str(t2)
    s.close()


def test_a_permuted_trajectory_converges_to_the_same_poses():
    P, factors, x = _factor_set("loops", seed=3)
    perm = np.random.default_rng(7).permutation(P)  # pose i of the original is pose perm[i] of the permuted set
    fperm = [dict(f, poses=perm[f["poses"]].astype(np.int32)) for f in factors]
    xperm = np.empty_like(x)
    xperm[perm] = x
    a, b = _sparse(P, factors), _sparse(P, fperm)
    assert a.structure()["pairs"] == b.structure()["pairs"]
    pa, ta = a.pose_graph_iter(x, max_iter=25, rel_tol=-1, gauge_mode=2)
    pb, tb = b.pose_graph_iter(xperm, max_iter=25, rel_tol=-1, gauge_mode=2)
    assert ta[-1]["r2"] < 1e-2 * ta[0]["r1"]
    assert np.abs(pb[perm] - pa).max() <= 1e-8
    a.close()
    b.close()


def test_a_factor_that_is_not_pd_is_reported_and_left_out():
    P, factors, x = _factor_set("pyramid", seed=3)
    bad = [dict(factors[1], H=-factors[1]["H"]), dict(factors[4], H=np.zeros_like(factors[4]["H"]))]
    c = balm_b200.Context(P)
    s = balm_b200.PoseGraph(P)
    fs = factors[:3] + bad + factors[3:]
    assert s.set_pose_factors(fs) == c.set_pose_factors(fs) == [L.OK] * 3 + [L.ERR_NOT_PD] * 2 + [L.OK] * (len(factors) - 3)
    H, g, r = c.pose_graph_evaluate(x)
    pairs, B, gs, rs = s.pose_graph_evaluate(x)
    assert np.array_equal(pairs, spg.block_pairs(factors)) and np.array_equal(gs, g) and rs == r
    Ho, go, ro = pg.evaluate(x, factors, P)
    assert abs(rs - ro) <= 1e-12 * abs(ro)
    c.close()
    s.close()


def test_malformed_registrations_are_rejected_and_the_previous_set_kept():
    P, factors, x = _factor_set(10, seed=4)
    s = balm_b200.PoseGraph(P)
    s.set_pose_factors(factors)
    before = (s.structure(), s.pose_graph_evaluate(x), s.pose_graph_iter(x, max_iter=3))
    f = factors[0]
    bad_sets = [
        [dict(f, poses=np.r_[f["poses"][:-1], P])],                      # index out of range
        [dict(f, poses=np.r_[f["poses"][:-1], -1])],                     # negative index
        [dict(f, poses=np.r_[f["poses"][:-1], f["poses"][0]])],          # repeated index
        [dict(poses=[3], poses_hat=f["poses_hat"][:1], H=np.eye(6))],    # one pose
        [dict(poses=list(range(33)), poses_hat=np.tile(f["poses_hat"][:1], (33, 1)), H=np.eye(198))],  # 33 poses
        [dict(f, H=np.where(np.eye(len(f["H"])) > 0, np.nan, f["H"]))],  # non-finite Hessian
        factors + [dict(f, poses=np.r_[f["poses"][:-1], P + 5])],        # a bad factor after good ones
        [],                                                              # no factor
    ]
    for fs in bad_sets:
        with pytest.raises(balm_b200.BalmError) as e:
            s.set_pose_factors(fs)
        assert e.value.status == L.ERR_INVALID and "balm_spg_set_factors" in str(e.value)
        after = (s.structure(), s.pose_graph_evaluate(x), s.pose_graph_iter(x, max_iter=3))
        assert after[0] == before[0] and all(np.array_equal(u, v) for u, v in zip(before[1], after[1]))
        assert np.array_equal(before[2][0], after[2][0]) and str(before[2][1]) == str(after[2][1])  # q1 may be nan
    with pytest.raises(ValueError):
        s.set_pose_factors([dict(f, H=f["H"][:-6, :-6])])
    s2 = balm_b200.PoseGraph(P)
    for call in (lambda: s2.pose_graph_evaluate(x), lambda: s2.pose_graph_iter(x), s2.structure):
        with pytest.raises(balm_b200.BalmError):
            call()
    s.close()
    s2.close()


# ---------------- sizes the dense context cannot hold ----------------
def _pyramid(P, seed):
    rng = np.random.default_rng(seed)
    truth = np.array([pg.random_pose(rng, 0.5, 3.0) for _ in range(P)])
    factors = [pg.make_factor(rng, truth, s, noise=0.01) for s in pg.pyramid_factor_poses(P, top=32)]
    return factors, pg.perturb(rng, truth, 0.02, 0.1)


def test_20000_poses_against_the_sparse_oracle():
    P = 20000
    factors, x = _pyramid(P, 11)
    s = _sparse(P, factors)
    _, tr = s.pose_graph_iter(x, max_iter=1, rel_tol=-1, gauge_mode=2, want_per_iter=True)
    xt, r1, r2 = spg.lm_step(x, factors, P)
    assert abs(tr[0]["r1"] - r1) <= 1e-10 * r1 and abs(tr[0]["r2"] - r2) <= 1e-10 * r1
    assert np.abs(tr[0]["poses"] - xt).max() <= 1e-9
    _, tr = s.pose_graph_iter(x, gauge_mode=2)
    assert tr[-1]["r2"] < 1e-2 * tr[0]["r1"]
    s.close()


def test_50000_poses_and_the_ordering_as_the_trajectory_grows():
    stats = {}
    for P in (5000, 50000):
        factors, x = _pyramid(P, 12)
        s = _sparse(P, factors)
        stats[P] = s.structure()
        if P == 50000:
            poses, tr = s.pose_graph_iter(x, max_iter=3, gauge_mode=2)
            assert np.all(np.isfinite(poses)) and tr[-1]["r2"] < tr[0]["r1"]
        s.close()
    a, b = stats[5000], stats[50000]
    print("structure at 5000 / 50000 poses:", a, b)
    assert b["l_blocks"] / 50000 <= 1.5 * a["l_blocks"] / 5000
    assert b["levels"] <= 2 * a["levels"]
    assert b["device_bytes"] < 2 * (6 * 50000) ** 2 * 8 / 100  # far below the dense H and factor


# ---------------- hierarchical BA on the sparse route ----------------
def _hba_routes(monkeypatch, *args, **kw):
    dense = hba.hba(*args, pose_graph=True, **kw)
    monkeypatch.setattr(hba, "PG_SPARSE_MIN_POSES", 0)
    sparse = hba.hba(*args, pose_graph=True, **kw)
    again = hba.hba(*args, pose_graph=True, **kw)
    return dense, sparse, again


def test_hba_sparse_route_on_a_drifting_trajectory(monkeypatch):
    scans, gt, init = hba_ref.drift_scene()
    dense, sparse, again = _hba_routes(monkeypatch, scans, init)
    assert np.abs(sparse["poses"] - dense["poses"]).max() <= 1e-9
    assert np.array_equal(sparse["poses"], again["poses"])
    assert sparse["pose_graph"]["status"] == dense["pose_graph"]["status"]


def test_hba_sparse_route_on_the_realworld_slice(monkeypatch):
    d = np.load(GOLD)
    n = len(d["poses"])
    scans = [d["xyz"][d["frame"] == i].astype(np.float32) for i in range(n)]
    x = np.asarray(d["poses"], dtype=np.float64)
    dense, sparse, again = _hba_routes(monkeypatch, scans, x, top_size=8)
    assert np.abs(sparse["poses"] - dense["poses"]).max() <= 1e-9
    assert np.array_equal(sparse["poses"], again["poses"])

"""The pose graph on the device (balm_set_pose_factors, balm_pose_graph_evaluate, balm_pose_graph_iter and
hba(pose_graph=True)) against the numpy oracle pose_graph_ref.py."""
import os

import numpy as np
import pytest

import balm_b200
import hba_ref
import pose_graph_ref as pg
import scenes
from balm_b200 import _lib as L, drivers, hba, io

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "realworld_points_small.npz")


def _factor_set(kind, seed=0):
    """-> (P, factors, poses): noisy factors of `kind` over a random trajectory, and poses away from it."""
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
    truth = np.array([pg.random_pose(rng, 0.5, 3.0) for _ in range(P)])
    factors = [pg.make_factor(rng, truth, s, noise=0.01) for s in sets]
    return P, factors, pg.perturb(rng, truth, 0.05, 0.2)


@pytest.mark.parametrize("kind", [2, 10, 11, 21, 22, 32, "pyramid", "all", "many"])
def test_evaluate_matches_oracle(kind):
    P, factors, x = _factor_set(kind)
    c = balm_b200.Context(P)
    assert c.set_pose_factors(factors) == [L.OK] * len(factors)
    H, g, r = c.pose_graph_evaluate(x)
    Ho, go, ro = pg.evaluate(x, factors, P)
    assert abs(r - ro) <= 1e-12 * abs(ro)
    assert np.abs(g - go).max() <= 1e-10 * np.abs(go).max()
    assert np.abs(H - Ho).max() <= 1e-10 * np.abs(Ho).max()
    assert np.array_equal(H, H.T)
    if kind == "many":
        assert len(factors) > 256
    c.close()


def test_iterations_match_the_oracle_lm():
    P, factors, x = _factor_set("pyramid", seed=1)
    c = balm_b200.Context(P)
    c.set_pose_factors(factors)
    poses, tr = c.pose_graph_iter(x, max_iter=8, gauge_mode=2, want_per_iter=True)
    po, tro, per = pg.lm(x, factors, P, max_iter=8)
    print("pose graph LM:", [(t["accepted"], "%.6g" % t["r2"]) for t in tr])
    assert [t["accepted"] for t in tr] == [t["accepted"] for t in tro]
    for t, to, p in zip(tr, tro, per):
        assert abs(t["r1"] - to["r1"]) <= 1e-10 * to["r1"] and abs(t["r2"] - to["r2"]) <= 1e-10 * to["r1"]
        assert np.abs(t["poses"] - p).max() <= 1e-9
    assert np.abs(poses - po).max() <= 1e-9
    assert tr[-1]["r2"] < 1e-2 * tr[0]["r1"]
    c.close()


def test_two_calls_are_bitwise_equal():
    P, factors, x = _factor_set("pyramid", seed=2)
    c = balm_b200.Context(P)
    s1 = c.set_pose_factors(factors)
    a = c.pose_graph_evaluate(x)
    pa, ta = c.pose_graph_iter(x, max_iter=5, gauge_mode=2)
    s2 = c.set_pose_factors(factors)
    b = c.pose_graph_evaluate(x)
    pb, tb = c.pose_graph_iter(x, max_iter=5, gauge_mode=2)
    assert s1 == s2 and all(np.array_equal(u, v) for u, v in zip(a, b))
    assert np.array_equal(pa, pb) and ta == tb
    c.close()


def test_a_factor_that_is_not_pd_is_reported_and_left_out():
    P, factors, x = _factor_set("pyramid", seed=3)
    bad = [dict(factors[1], H=-factors[1]["H"]), dict(factors[4], H=np.zeros_like(factors[4]["H"]))]
    H = factors[6]["H"].copy()
    H[6:12, :] = 0.0  # slot 1 unconstrained: H~ singular
    H[:, 6:12] = 0.0
    bad.append(dict(factors[6], H=H))
    assert not any(pg.pd_ok(f["H"]) for f in bad)
    c = balm_b200.Context(P)
    st = c.set_pose_factors(factors[:3] + bad + factors[3:])
    assert st == [L.OK] * 3 + [L.ERR_NOT_PD] * 3 + [L.OK] * (len(factors) - 3)
    Hd, gd, rd = c.pose_graph_evaluate(x)
    Ho, go, ro = pg.evaluate(x, factors, P)
    assert abs(rd - ro) <= 1e-12 * abs(ro) and np.abs(gd - go).max() <= 1e-10 * np.abs(go).max()
    assert np.abs(Hd - Ho).max() <= 1e-10 * np.abs(Ho).max()
    c.close()


def test_malformed_registrations_are_rejected_and_the_previous_set_kept():
    P, factors, x = _factor_set(10, seed=4)
    c = balm_b200.Context(P)
    c.set_pose_factors(factors)
    before = c.pose_graph_evaluate(x)
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
            c.set_pose_factors(fs)
        assert e.value.status == L.ERR_INVALID
        after = c.pose_graph_evaluate(x)
        assert all(np.array_equal(u, v) for u, v in zip(before, after))
    with pytest.raises(ValueError):
        c.set_pose_factors([dict(f, H=f["H"][:-6, :-6])])
    assert all(np.array_equal(u, v) for u, v in zip(before, c.pose_graph_evaluate(x)))
    c2 = balm_b200.Context(P)
    with pytest.raises(balm_b200.BalmError):
        c2.pose_graph_evaluate(x)
    with pytest.raises(balm_b200.BalmError):
        c2.pose_graph_iter(x)
    c.close()
    c2.close()


def test_voxel_damping_iter_is_unaffected_by_factors():
    sc = scenes.make_scene(n_poses=12, n_planes=80, seed=3)
    rng = np.random.default_rng(5)
    truth = np.array([pg.random_pose(rng) for _ in range(12)])
    factors = [pg.make_factor(rng, truth, s, 0.01) for s in ([0, 1, 2, 3, 4], [4, 7, 9, 11], [11, 0])]
    out = []
    for with_factors in (False, True):
        c = balm_b200.Context(sc["n_poses"])
        if with_factors:
            c.set_pose_factors(factors)
        c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
        if with_factors:
            c.pose_graph_evaluate(truth)
            c.pose_graph_iter(truth, max_iter=3)
        H, g, r = c.evaluate(sc["poses_init"])
        poses, tr, per = c.damping_iter(sc["poses_init"], gauge_mode=2, want_per_iter=True)
        out.append((H, g, r, poses, tr, per))
        c.close()
    a, b = out
    assert all(np.array_equal(u, v) for u, v in zip(a[:4], b[:4])) and a[4] == b[4] and np.array_equal(a[5], b[5])


# ---------------- hierarchical BA ----------------
@pytest.fixture(scope="module")
def drift():
    return hba_ref.drift_scene()


@pytest.fixture(scope="module")
def drift_runs(drift):
    scans, gt, init = drift
    return hba.hba(scans, init), hba.hba(scans, init, pose_graph=True)


def test_hba_pose_graph_on_a_drifting_trajectory(drift, drift_runs):
    scans, gt, init = drift
    base, res = drift_runs
    for a, b in zip(base["layers"], res["layers"]):  # the pyramid itself is unchanged
        assert a["status"] == b["status"] and all(np.array_equal(x, y) for x, y in zip(a["poses"], b["poses"]))
    p = res["pose_graph"]
    n_ok = sum(st == L.OK and len(w) >= 2 for lay in res["layers"] for st, w in zip(lay["status"], lay["windows"]))
    assert p["n_factors"] == n_ok == len(p["status"]) and len(p["trace"]) >= 1
    assert np.abs(res["poses"][0] - init[0]).max() <= 1e-12
    rot0, tran0 = drivers.rsme(init, gt)
    rot2, tran2 = drivers.rsme(res["poses"], gt)
    assert rot2 < 0.1 * rot0 and tran2 < 0.1 * tran0


# Measured on an H100: initial 0.8632 deg / 0.0975 m, hba pyramid 0.01126 deg / 0.00118 m, hba + pose graph
# 0.01136 deg / 0.00118 m (12 factors, converged: more LM iterations do not move it). The factors' minimum is not the
# ground truth (cost 0.020 there, 0.314 at the ground truth): the top window's Hessian, built on keyframes merged at the
# bottom windows' estimates, overstates how well its relative poses are known. Scaling the top factor by 10 gives
# 0.01160 deg, by 0.1 gives 0.01021 deg. Until the factors carry calibrated weights the pose graph is not better than
# the pyramid in rotation on this scene.
@pytest.mark.xfail(strict=True, reason="the top window's Hessian overweights it: 0.01136 vs 0.01126 deg rotation RMSE")
def test_hba_pose_graph_is_not_worse_than_the_pyramid(drift, drift_runs):
    scans, gt, init = drift
    base, res = drift_runs
    rot1, tran1 = drivers.rsme(base["poses"], gt)
    rot2, tran2 = drivers.rsme(res["poses"], gt)
    p = res["pose_graph"]
    print("drift RMSE rot [deg] / tran [m]: hba pyramid %.5f / %.5f, hba + pose graph %.5f / %.5f;"
          " %d factors, %d LM iterations, %.1f ms"
          % (np.degrees(rot1), tran1, np.degrees(rot2), tran2, p["n_factors"], len(p["trace"]), p["ms"]))
    assert rot2 <= rot1 and tran2 <= tran1


def test_hba_pose_graph_realworld_slice():
    d = np.load(GOLD)
    n = len(d["poses"])
    scans = [d["xyz"][d["frame"] == i].astype(np.float32) for i in range(n)]
    x = np.asarray(d["poses"], dtype=np.float64)
    res = hba.hba(scans, x, top_size=8, pose_graph=True)
    lays = res["layers"]
    assert [len(lay["windows"]) for lay in lays] == [4, 1]
    assert res["poses"].shape == (24, 12) and np.all(np.isfinite(res["poses"]))
    assert res["pose_graph"]["n_factors"] == sum(st == L.OK for lay in lays for st in lay["status"])
    again = hba.hba(scans, x, top_size=8, pose_graph=True)
    assert np.array_equal(res["poses"], again["poses"])


def test_cli_pose_graph_gives_the_function_poses(tmp_path, capsys):
    from test_drivers import _write_dataset
    _write_dataset(tmp_path, n_poses=24, pts=4000)
    out = tmp_path / "refined.csv"
    assert hba.main(["--file_path", str(tmp_path), "--top_size", "8", "--pose_graph", "--out", str(out)]) == 0
    text = capsys.readouterr().out
    assert "The size of poses: 24" in text and "pose graph:" in text
    R, p, _, scans = io.read_realworld_dir(str(tmp_path))
    R0, p0 = R[0].copy(), p[0].copy()
    x = drivers.pack_poses(np.einsum("ji,njk->nik", R0, R), (p - p0) @ R0)
    want = hba.hba(scans, x, top_size=8, pose_graph=True)["poses"]
    Rf, pf, _ = io.read_pose_csv(out)
    assert np.array_equal(drivers.pack_poses(Rf, pf), want)

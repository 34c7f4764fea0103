"""Tensor path inside balm_damping_iter with force_hess: after a rejected step the Hessian is re-evaluated at the
unchanged poses. When the digit planes, column maxima and accumulators of the previous evaluation were written by the
fused sweep with the very scales the re-evaluation adopts, the observation sweep is skipped and they are reused. That
must give the same bits as sweeping again (BALM_NO_SWEEP_REUSE=1): same poses after every iteration, same trace."""
import numpy as np
import pytest

import scenes

pytestmark = pytest.mark.gpu

# long enough to pass the 4-5 descent steps and sit at the converged cost, where about half the steps are rejected
KW = dict(max_iter=14, force_hess=True, rel_tol=-1.0, want_per_iter=True, min_planes_per_pose=0)


def _run(sc, monkeypatch, reuse, env=(), **kw):
    import balm_b200
    for k, v in env:
        monkeypatch.setenv(k, v)
    if reuse:
        monkeypatch.delenv("BALM_NO_SWEEP_REUSE", raising=False)
    else:
        monkeypatch.setenv("BALM_NO_SWEEP_REUSE", "1")
    c = balm_b200.Context(sc["n_poses"], 0, balm_b200.PREC_TENSOR)
    c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc["fix10"])
    c.reset_counters()
    poses, tr, per_iter = c.damping_iter(sc["poses_init"], **{**KW, **kw})
    tm = c.timings()
    c.close()
    for k, _ in env:
        monkeypatch.delenv(k)
    return poses, per_iter, [(t["r1"], t["r2"], t["q1"], t["accepted"]) for t in tr], tm


def _compare(sc, monkeypatch, env=(), **kw):
    p0, pi0, t0, tm0 = _run(sc, monkeypatch, False, env, **kw)
    p1, pi1, t1, tm1 = _run(sc, monkeypatch, True, env, **kw)
    assert np.array_equal(p0, p1) and np.array_equal(pi0, pi1)
    assert t0 == t1
    assert tm0["reused_sweeps"] == 0
    for k in ("n_eval", "single_sweeps", "redone_sweeps", "digit_planes"):
        assert tm0[k] == tm1[k], (k, tm0, tm1)
    # only re-evaluations after a rejected step can reuse, and each of them is a kept single sweep
    rejected = sum(1 for x in t1[:-1] if not x[3])
    assert tm1["reused_sweeps"] <= min(rejected, tm1["single_sweeps"]), (tm1, t1)
    return t1, tm1


@pytest.mark.parametrize("n_poses,n_planes,drop,with_fix,hess_fix", [
    (24, 150, 0.0, False, False),   # dense, one warp tile
    (37, 200, 0.0, True, True),     # partial second tile, fix cluster in the Hessian (stats hand-over on)
    (33, 160, 0.0, True, False),    # fix cluster outside the Hessian (no stats hand-over)
])
def test_reuse_after_rejection_is_bit_identical(n_poses, n_planes, drop, with_fix, hess_fix, monkeypatch):
    sc = scenes.make_scene(n_poses=n_poses, n_planes=n_planes, seed=57, drop=drop, with_fix=with_fix)
    tr, tm = _compare(sc, monkeypatch, hess_includes_fix=hess_fix)
    assert not all(x[3] for x in tr[:-1]), tr      # the converged regime was reached: some step was rejected
    assert tm["reused_sweeps"] >= 1, (tm, tr)


def test_no_reuse_on_sparse_scenes(monkeypatch):
    """Sparse co-visibility (pose-major lists): the planes are cleared before every sweep, so it always runs."""
    sc = scenes.make_scene(n_poses=30, n_planes=220, seed=57, drop=0.4)
    tr, tm = _compare(sc, monkeypatch)
    assert not all(x[3] for x in tr[:-1]), tr
    assert tm["reused_sweeps"] == 0 and tm["single_sweeps"] >= 1, tm


@pytest.mark.parametrize("seed", [3, 4])
def test_no_reuse_when_the_accepted_step_moved_the_scales(seed, monkeypatch):
    """0.5 m of translation noise and u0 = 1e-6: the first step is a large accepted one and moves column maxima across
    powers of two; the evaluation after it keeps its speculated scales (no redone sweep) but finds fresh ones that
    differ, and the next step is rejected. The re-evaluation after that rejection adopts the fresh scales, which differ
    from the ones the kept planes were written with, so it must sweep. Every later re-evaluation at unchanged poses
    finds the scales it swept with and reuses."""
    sc = scenes.make_scene(n_poses=37, n_planes=150, seed=seed, tra_noise=0.5)
    tr, tm = _compare(sc, monkeypatch, u0=1e-6)
    acc = [x[3] for x in tr]
    assert acc[:3] == [1, 0, 0], tr
    assert tm["redone_sweeps"] == 0, tm            # every speculation kept: *spec_ok = 1 before each re-evaluation
    assert tm["reused_sweeps"] == sum(1 for a in acc[:-1] if not a) - 1, (tm, tr)


def test_reuse_with_four_digit_planes(monkeypatch):
    sc = scenes.make_scene(n_poses=24, n_planes=150, seed=58)
    _, tm = _compare(sc, monkeypatch, env=(("BALM_TC_SLICES", "4"),))
    assert tm["digit_planes"] == 4 and tm["reused_sweeps"] >= 1, tm


@pytest.mark.parametrize("skew", [4, -9])
def test_no_reuse_when_every_speculation_fails(skew, monkeypatch):
    """Skewed adopted scales never equal the ones the planes were written with (and every check re-arms the digit
    sweep), so nothing is reused and the result is the hook run's."""
    sc = scenes.make_scene(n_poses=24, n_planes=150, seed=57)
    _, tm = _compare(sc, monkeypatch, env=(("BALM_TC_SPEC_SKEW", str(skew)),))
    assert tm["reused_sweeps"] == 0 and tm["single_sweeps"] == 0, tm


def test_no_reuse_across_voxel_batches(monkeypatch):
    """Several voxel batches: no speculation and no reuse (the planes hold the last batch only)."""
    sc = scenes.make_scene(n_poses=24, n_planes=1200, seed=57)
    _, tm = _compare(sc, monkeypatch, env=(("BALM_G_BUDGET_MB", "1"),))  # 1 MiB of G' -> several voxel batches
    assert tm["reused_sweeps"] == 0 and tm["single_sweeps"] == 0 and tm["redone_sweeps"] == 0, tm


def test_rel_tol_exit(monkeypatch):
    sc = scenes.make_scene(n_poses=24, n_planes=150, seed=57)
    tr, _ = _compare(sc, monkeypatch, rel_tol=1e-9)
    assert len(tr) < KW["max_iter"], tr

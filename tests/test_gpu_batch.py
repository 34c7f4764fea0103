"""Batched bundle adjustment (balm_batch_*, balm_b200.Batch): B independent problems registered together, checked
problem by problem against the CPU oracle and against a Context holding only that problem. Tolerances are those of the
fp64 path (tests/test_gpu_parity.py): residual 1e-12, gradient 1e-10, Hessian 1e-9 relative; per LM iteration
1e-6 rad / 1e-6 m with the same accept / reject sequence."""
import ctypes as C

import numpy as np
import pytest

import scenes
from oracle import oracle_py as orc

pytestmark = pytest.mark.gpu

IDENT = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0.0])


def _prob(sc):
    return dict(n_poses=sc["n_poses"], row_ptr=sc["row_ptr"], pose_idx=sc["pose_idx"], obs10=sc["obs10"],
                coe=sc["coe"], fix10=sc["fix10"])


def _empty(n_poses):
    return dict(n_poses=n_poses, row_ptr=np.zeros(1, dtype=np.int64), pose_idx=np.zeros(0, dtype=np.int32),
                obs10=np.zeros((0, 10)), coe=np.zeros(0), fix10=None)


def _oracle(sc):
    return orc.Oracle(sc["n_poses"], sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc["fix10"])


def _batch(problems):
    import balm_b200
    b = balm_b200.Batch(0)
    b.set_problems(problems)
    return b


def _pose_err(a, b):
    rot = max(np.linalg.norm(orc.log_so3(scenes.unpack_pose(x)[0].T @ scenes.unpack_pose(y)[0])) for x, y in zip(a, b))
    tra = max(np.linalg.norm(x[9:] - y[9:]) for x, y in zip(a, b))
    return rot, tra


def _tr_key(tr):
    return [(t["r1"], t["r2"], t["u"], t["v"], t["q"], t["q1"], t["accepted"], t["recomputed_hess"], t["not_pd"])
            for t in tr]


# N_p 2 .. 32, dense and drop = 0.4, with and without fix clusters
EVAL_SCENES = [
    dict(n_poses=2, n_planes=5, seed=21),
    dict(n_poses=32, n_planes=60, seed=22),
    dict(n_poses=20, n_planes=120, seed=23, drop=0.4),
    dict(n_poses=12, n_planes=50, seed=24, with_fix=True),
    dict(n_poses=9, n_planes=30, seed=25, drop=0.5, with_fix=True),
    dict(n_poses=7, n_planes=40, seed=26),
    dict(n_poses=25, n_planes=80, seed=27, drop=0.4, with_fix=True),
]


def test_evaluate_matches_oracle_per_problem():
    scs = [scenes.make_scene(**kw) for kw in EVAL_SCENES]
    empty_at = 3
    problems = [_prob(s) for s in scs]
    problems.insert(empty_at, _empty(3))  # a problem with no voxels
    b = _batch(problems)
    poses = [s["poses_init"] for s in scs]
    poses.insert(empty_at, np.tile(IDENT, (3, 1)))
    for include_fix in (False, True):
        res = b.evaluate(poses, include_fix=include_fix)
        H, g, r = res[empty_at]
        assert r == 0 and not H.any() and not g.any()
        del res[empty_at]
        for sc, (H, g, r) in zip(scs, res):
            Ho, go, ro = _oracle(sc).evaluate(sc["poses_init"], include_fix=include_fix)
            assert H.shape == (6 * sc["n_poses"],) * 2
            assert abs(r - ro) <= 1e-12 * abs(ro), (sc["n_poses"], r, ro)
            assert np.abs(g - go).max() <= 1e-10 * np.abs(go).max()
            assert np.abs(H - Ho).max() <= 1e-9 * np.abs(Ho).max()
            assert np.array_equal(H, H.T)


# problems of different size, sparsity and start quality, so that they stop at different iterations
LM_SCENES = [
    dict(n_poses=8, n_planes=60, seed=26),
    dict(n_poses=20, n_planes=200, seed=27, drop=0.3),
    dict(n_poses=32, n_planes=80, seed=28),
    dict(n_poses=12, n_planes=60, seed=29, with_fix=True),
    dict(n_poses=6, n_planes=40, seed=30, rot_noise=0.1 / 57.3, tra_noise=0.002),
    dict(n_poses=10, n_planes=50, seed=31, rot_noise=5 / 57.3, tra_noise=0.3),
]


@pytest.fixture(scope="module")
def lm_scenes():
    return [scenes.make_scene(**kw) for kw in LM_SCENES]


def _check_vs_oracle(sc, res, oracle_run):
    st, poses, tr, per = res
    st_o, poses_o, tr_o, per_o = oracle_run
    assert st == 0 and st_o == 0 and len(tr) == len(tr_o)
    assert [t["accepted"] for t in tr] == [t["accepted"] for t in tr_o]
    assert [t["recomputed_hess"] for t in tr] == [t["recomputed_hess"] for t in tr_o]
    for it in range(len(tr)):
        rot, tra = _pose_err(per[it], per_o[it])
        assert rot <= 1e-6 and tra <= 1e-6, (it, rot, tra)
        assert abs(tr[it]["r2"] - tr_o[it]["r2"]) <= 1e-9 * abs(tr_o[it]["r2"])
        assert abs(tr[it]["u"] - tr_o[it]["u"]) <= 1e-5 * tr_o[it]["u"]


def test_damping_iter_matches_oracle_per_problem(lm_scenes):
    b = _batch([_prob(s) for s in lm_scenes])
    init = [s["poses_init"] for s in lm_scenes]
    res = b.damping_iter(init, want_per_iter=True, gauge_mode=2)
    for sc, r in zip(lm_scenes, res):
        _check_vs_oracle(sc, r, _oracle(sc).damping_iter(sc["poses_init"], gauge_mode=2))
    assert len({len(r[2]) for r in res}) > 1, "the problems were meant to stop at different iterations"
    # the final gauge step, per problem (bavoxel.hpp:1159-1164)
    for sc, (st, p0, _, _) in zip(lm_scenes, b.damping_iter(init, gauge_mode=0)):
        _, p0o, _, _ = _oracle(sc).damping_iter(sc["poses_init"], gauge_mode=0)
        assert max(_pose_err(p0, p0o)) <= 1e-6
    # the benchmark_virtual twin: pose 0 exactly the identity, converged to the noise floor
    for sc, (st, p1, tr, _) in zip(lm_scenes, b.damping_iter(init, max_iter=20, u0=0.1, gauge_mode=1,
                                                              hess_includes_fix=True)):
        assert st == 0 and np.array_equal(p1[0], IDENT)
        rot, tra = orc.rmse(p1, sc["poses_gt"])
        assert rot * 57.3 < 0.1 and tra < 0.01, (sc["n_poses"], rot, tra)


def test_damping_iter_agrees_with_context_fp64(lm_scenes):
    import balm_b200
    b = _batch([_prob(s) for s in lm_scenes])
    res = b.damping_iter([s["poses_init"] for s in lm_scenes])
    for sc, (st, poses, tr, _) in zip(lm_scenes, res):
        c = balm_b200.Context(sc["n_poses"], 0, balm_b200.PREC_FP64)
        c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc["fix10"])
        pc, trc, _ = c.damping_iter(sc["poses_init"])
        assert st == 0 and [t["accepted"] for t in tr] == [t["accepted"] for t in trc]
        assert np.abs(poses - pc).max() <= 1e-9, (sc["n_poses"], np.abs(poses - pc).max())
        c.close()


def test_problem_results_do_not_depend_on_the_batch(lm_scenes):
    X, Y, Z, W = lm_scenes[1], lm_scenes[2], lm_scenes[4], lm_scenes[3]
    kw = dict(want_per_iter=True, max_iter=6)

    def run(batch, at):
        out = _batch([_prob(s) for s in batch]).damping_iter([s["poses_init"] for s in batch], **kw)[at]
        return out[1], _tr_key(out[2]), out[3]

    alone = run([X], 0)
    for batch, at in (([X, Y, Z], 0), ([Y, Z, X], 2), ([W, X], 1), ([X], 0)):
        p, t, per = run(batch, at)
        assert np.array_equal(p, alone[0]) and t == alone[1] and np.array_equal(per, alone[2])
    b = _batch([_prob(s) for s in (X, Y, Z)])
    r1 = b.damping_iter([s["poses_init"] for s in (X, Y, Z)], **kw)
    r2 = b.damping_iter([s["poses_init"] for s in (X, Y, Z)], **kw)
    for a, c in zip(r1, r2):
        assert np.array_equal(a[1], c[1]) and _tr_key(a[2]) == _tr_key(c[2]) and np.array_equal(a[3], c[3])
    e1 = b.evaluate([s["poses_init"] for s in (X, Y, Z)])
    e2 = b.evaluate([s["poses_init"] for s in (X, Y, Z)])
    for (Ha, ga, ra), (Hb, gb, rb) in zip(e1, e2):
        assert np.array_equal(Ha, Hb) and np.array_equal(ga, gb) and ra == rb


def test_too_few_planes_is_per_problem(lm_scenes):
    A, Cs = lm_scenes[0], lm_scenes[3]
    T = scenes.make_scene(n_poses=4, n_planes=10, seed=27)  # 10 planes per pose < min_planes_per_pose = 20
    with_t = _batch([_prob(A), _prob(T), _prob(Cs)]).damping_iter([A["poses_init"], T["poses_init"], Cs["poses_init"]])
    without = _batch([_prob(A), _prob(Cs)]).damping_iter([A["poses_init"], Cs["poses_init"]])
    st, pt, tr, _ = with_t[1]
    assert st == 4 and tr == [] and np.array_equal(pt, T["poses_init"])  # reference: printf + exit(0) (bavoxel.hpp:1079)
    for a, c in zip((with_t[0], with_t[2]), without):
        assert a[0] == 0 and np.array_equal(a[1], c[1]) and _tr_key(a[2]) == _tr_key(c[2])


def test_indefinite_damped_system_follows_oracle():
    """Strongly perturbed start with tiny damping: H + uD is indefinite at the start (see
    test_gpu_parity_sizes.test_indefinite_damped_system_vs_pivoted_ldlt). The batched solve factors without pivoting,
    checks the backward error and refines; an unusable step is flagged not_pd and rejected."""
    hard = scenes.make_scene(n_poses=12, n_planes=60, seed=71, rot_noise=12 / 57.3, tra_noise=0.6)
    easy = scenes.make_scene(n_poses=8, n_planes=60, seed=26)
    kw = dict(max_iter=8, u0=1e-4, min_planes_per_pose=0, gauge_mode=2)
    H, g, r = _batch([_prob(hard)]).evaluate([hard["poses_init"]])[0]
    assert np.linalg.eigvalsh(H + 1e-4 * np.diag(np.diag(H)))[0] < 0
    res = _batch([_prob(easy), _prob(hard)]).damping_iter([easy["poses_init"], hard["poses_init"]], want_per_iter=True, **kw)
    st, poses, tr, per = res[1]
    st_o, poses_o, tr_o, per_o = _oracle(hard).damping_iter(hard["poses_init"], **kw)
    assert st == 0 and [t["accepted"] for t in tr] == [t["accepted"] for t in tr_o]
    for it in range(len(tr)):
        assert max(_pose_err(per[it], per_o[it])) <= 1e-6, it
        if tr[it]["not_pd"]:
            assert not tr[it]["accepted"]


def test_bad_input_is_rejected_and_keeps_the_registration(lm_scenes):
    import balm_b200
    from balm_b200 import _lib
    from balm_b200.context import _p
    scs = lm_scenes[:3]
    b = _batch([_prob(s) for s in scs])
    init = [s["poses_init"] for s in scs]
    before = b.damping_iter(init, want_per_iter=True, gauge_mode=2)
    A = _prob(scs[0])

    def rejected(problems):
        with pytest.raises(balm_b200.BalmError) as e:
            b.set_problems(problems)
        assert e.value.status == _lib.ERR_INVALID

    rejected([A, dict(_empty(0))])                                          # 0 poses
    big = scenes.make_scene(n_poses=33, n_planes=30, seed=5)
    rejected([A, _prob(big)])                                               # 33 poses
    bad = dict(A, pose_idx=A["pose_idx"].copy())
    bad["pose_idx"][3] = A["n_poses"]                                      # out of the problem's range
    rejected([bad, A])
    bad = dict(A, pose_idx=A["pose_idx"].copy())
    bad["pose_idx"][1] = bad["pose_idx"][0]                                # not ascending inside a voxel
    rejected([A, bad])
    # the raw call: n_problems < 1, pose_ptr / voxel_ptr / row_ptr not ascending
    L = _lib.lib()
    rp, pi, ob, co = A["row_ptr"], A["pose_idx"], A["obs10"], A["coe"]
    M = len(rp) - 1
    i64 = lambda *v: np.array(v, dtype=np.int64)
    calls = [
        (0, i64(0), i64(0), rp),
        (2, i64(0, 8, 4), i64(0, M // 2, M), rp),          # pose_ptr descending
        (2, i64(0, 4, 8), i64(0, M, M // 2), rp),          # voxel_ptr descending
        (1, i64(0, 8), i64(0, 2), i64(0, 8, 4)),           # row_ptr descending
    ]
    for n, pp, vp, rr in calls:
        assert L.balm_batch_set_voxels(b._h, n, _p(pp), _p(vp), _p(rr), _p(pi), _p(ob), None, _p(co)) == _lib.ERR_INVALID
    with pytest.raises(balm_b200.BalmError) as e:
        b.damping_iter(init, verbose=True)
    assert e.value.status == _lib.ERR_INVALID
    after = b.damping_iter(init, want_per_iter=True, gauge_mode=2)
    for sc, x, y in zip(scs, before, after):
        assert np.array_equal(x[1], y[1]) and _tr_key(x[2]) == _tr_key(y[2]) and np.array_equal(x[3], y[3])
        _check_vs_oracle(sc, y, _oracle(sc).damping_iter(sc["poses_init"], gauge_mode=2))

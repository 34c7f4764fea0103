"""Batched sliding window (balm_batch_marginalize / balm_batch_append_scan, Batch.marginalize / append_scans): every
problem must get bitwise what a fp64 Context holding it alone registers with marginalize / append_scan, whatever else is
in the batch; a problem the context call would leave without voxels is registered empty; untouched problems stay
bitwise as they were; bad input is rejected and keeps the registration. Then the whole window step -- cut, LM,
marginalise, append, LM with fix clusters, pose covariance -- against the per-sequence Context route."""
import ctypes as C

import numpy as np
import pytest

import assoc_ref
import scenes

pytestmark = pytest.mark.gpu

KW = dict(voxel_size=2.0, eigen_value_array=(1 / 16, 1 / 16, 1 / 9))
FIELDS = ("row_ptr", "pose_idx", "obs10", "coe", "fix10")
EMPTY = dict(row_ptr=np.zeros(1, dtype=np.int64), pose_idx=np.zeros(0, dtype=np.int32), obs10=np.zeros((0, 10)),
             coe=np.zeros(0), fix10=np.zeros((0, 10)), keys=np.zeros(0, dtype=np.uint64), layers=np.zeros(0, dtype=np.int32))


def _equal(a, b, fields=FIELDS):
    return all(np.array_equal(np.asarray(a[k]).reshape(np.asarray(b[k]).shape), b[k]) for k in fields)


def _ctx_dict(c, keys=False):
    rp, pi, ob, co = c.download_voxels()
    d = dict(row_ptr=rp, pose_idx=pi, obs10=ob, coe=co, fix10=c.download_fix())
    if keys:
        d["keys"], d["layers"] = c.download_keys(with_layers=True)
    return d


# ---------------------------------------------------------------- marginalise ----------------------------------------
def _marg_problems():
    """(problem dict, poses, mg): N_p 2 .. 32, dense and ragged, with and without fix clusters (some >= 50 points), an
    untouched problem, one whose voxels all vanish and one without voxels."""
    out = []
    for N, drop, fix, mg, seed in [(2, 0.0, False, 1, 1), (7, 0.3, True, 2, 2), (12, 0.0, False, 0, 3),
                                   (12, 0.5, True, 4, 4), (32, 0.4, False, 3, 5), (7, 0.0, True, 1, 6),
                                   (12, 0.2, True, 0, 7)]:
        sc = scenes.make_scene(n_poses=N, n_planes=60, seed=90 + seed, drop=drop, with_fix=fix, pts_size=9)
        if fix:
            sc["fix10"][::3] *= 8.0                    # >= 50 points: these fix clusters absorb nothing (bavoxel.hpp:790)
        p = dict(n_poses=N, row_ptr=sc["row_ptr"], pose_idx=sc["pose_idx"], obs10=sc["obs10"], coe=sc["coe"],
                 fix10=sc["fix10"])
        out.append((p, sc["poses_init"], mg))
    out.append((dict(n_poses=3, **{k: EMPTY[k] for k in FIELDS}), np.tile(scenes.pack_poses([np.eye(3)], [np.zeros(3)]),
                                                                          (3, 1)), 1))
    return out


def _ctx_marginalize(p, poses, mg, min_ps=15):
    """Context.set_voxels + marginalize; mg 0 -> the problem itself; the context's refusal -> empty."""
    import balm_b200
    from balm_b200 import _lib
    if mg == 0:
        return {k: (np.zeros((len(p["coe"]), 10)) if k == "fix10" and p[k] is None else p[k]) for k in FIELDS}
    if len(p["coe"]) == 0:                                    # the context refuses to marginalise no voxels
        return {k: EMPTY[k] for k in FIELDS}
    c = balm_b200.Context(p["n_poses"], 0, balm_b200.PREC_FP64)
    c.set_voxels(p["row_ptr"], p["pose_idx"], p["obs10"], p["coe"], p["fix10"])
    try:
        c.marginalize(mg, poses, min_ps=min_ps)
        d = _ctx_dict(c)
    except balm_b200.BalmError as e:                          # no voxel left with two observing scans
        assert e.status == _lib.ERR_INVALID and "no voxel is left" in str(e)
        d = {k: EMPTY[k] for k in FIELDS}
    c.close()
    return d


def _batch_marginalize(items, min_ps=15):
    import balm_b200
    b = balm_b200.Batch(0)
    b.set_problems([p for p, _, _ in items])
    mk = b.marginalize([m for _, _, m in items], [x for _, x, _ in items], min_ps=min_ps)
    got = b.download_voxels(with_fix=True)
    b.close()
    return mk, got


def test_marginalize_matches_context_per_problem():
    items = _marg_problems()
    mk, got = _batch_marginalize(items)
    for i, ((p, poses, mg), d, (M, K)) in enumerate(zip(items, got, mk)):
        ref = _ctx_marginalize(p, poses, mg)
        assert _equal(d, ref), i
        assert (M, K) == (len(ref["coe"]), len(ref["pose_idx"]))
    assert mk[0] == (0, 0) and mk[-1] == (0, 0)              # every voxel vanishes / no voxels: empty, not an error
    assert all(m > 0 for m, _ in mk[1:-1])
    for i in (2, 6):                                          # mg_size 0: bitwise the registered problem
        assert _equal(got[i], {k: items[i][0][k] for k in FIELDS[:4]}, FIELDS[:4])
    assert not got[2]["fix10"].any()                          # ... given zero fix rows when it had none
    # one problem against the numpy restatement of to_margi + push_voxel
    p, poses, mg = items[3]
    rp, pi, ob, fx, co = assoc_ref.marginalize_ref(p["n_poses"], p["row_ptr"], p["pose_idx"], p["obs10"], p["fix10"],
                                                   poses, mg, 15)
    d = got[3]
    assert np.array_equal(d["row_ptr"], rp) and np.array_equal(d["pose_idx"], pi) and np.array_equal(d["coe"], co)
    assert np.array_equal(d["obs10"], ob)
    assert np.abs(d["fix10"] - fx).max() <= 1e-12 * np.abs(fx).max()


def test_marginalize_independence_and_determinism():
    items = _marg_problems()
    mk, got = _batch_marginalize(items)
    mk2, got2 = _batch_marginalize(items)                     # a second identical call
    assert mk == mk2 and all(_equal(a, b) for a, b in zip(got, got2))
    perm = [3, 0, 7, 5, 1, 6, 2, 4]
    pmk, pgot = _batch_marginalize([items[i] for i in perm])
    for j, i in enumerate(perm):
        assert pmk[j] == mk[i] and _equal(pgot[j], got[i]), i
    for i in (1, 3, 4):                                       # alone
        amk, agot = _batch_marginalize([items[i]])
        assert amk[0] == mk[i] and _equal(agot[0], got[i]), i


def test_fix_round_trip():
    import balm_b200
    items = _marg_problems()[1:-1]
    b = balm_b200.Batch(0)
    b.set_problems([p for p, _, _ in items])
    b.marginalize([max(m, 1) for _, _, m in items], [x for _, x, _ in items])
    poses = [x for _, x, _ in items]
    before = b.evaluate(poses, include_fix=True)
    rt = balm_b200.Batch(0)
    rt.set_problems(b.download_voxels(with_fix=True))
    after = rt.evaluate(poses, include_fix=True)
    for (H0, g0, r0), (H1, g1, r1) in zip(before, after):
        assert np.array_equal(H0, H1) and np.array_equal(g0, g1) and r0 == r1
    b.close()
    rt.close()


# ---------------------------------------------------------------- append ---------------------------------------------
def _append_setup():
    """12 synthetic scans plus an empty one (index 12): windows whose last slot holds the empty scan, so a new scan can
    take it. Windows 0 and 1 share scans and both take scan 10; window 2 takes scan 11; window 3 takes none; window 4 has
    one real scan (no voxels) and takes scan 11."""
    pts, frs, poses = assoc_ref.synthetic_scans(n_poses=12, pts_per_scan=3000, seed=13)
    scans = [pts[frs == i].astype(np.float32) for i in range(12)] + [np.zeros((0, 3), dtype=np.float32)]
    p12 = scenes.pack_poses([r for r, _ in poses], [q for _, q in poses])
    p12 = np.vstack([p12, p12[:1]])
    E = 12
    windows = [list(range(0, 7)) + [E], list(range(3, 10)) + [E], [1, 2, 3, E], [5, 6, 7], [0, E]]
    scan_of = [10, 10, 11, -1, 11]
    slots = [len(w) - 1 for w in windows]
    wposes = []
    for w, s in zip(windows, scan_of):
        x = p12[w].copy()
        if s >= 0:
            x[-1] = p12[s]                                     # the new scan's pose in the slot it takes
        wposes.append(x)
    return scans, windows, wposes, scan_of, slots


def _ctx_cut(scans, win, poses):
    import balm_b200
    from balm_b200 import _lib
    pts = np.concatenate([scans[s] for s in win])
    fr = np.concatenate([np.full(len(scans[s]), k, dtype=np.int32) for k, s in enumerate(win)])
    c = balm_b200.Context(len(win), 0, balm_b200.PREC_FP64)
    try:
        c.cut_voxels(pts, fr, poses, **KW)
    except balm_b200.BalmError as e:
        assert e.status == _lib.ERR_INVALID
        c.close()
        return None
    return c


def _ctx_append(scans, win, poses, scan, slot):
    """Context.cut_voxels + append_scan -> (dict with keys, matched); the context's refusal -> empty."""
    import balm_b200
    from balm_b200 import _lib
    c = _ctx_cut(scans, win, poses)
    if c is None:
        return dict(EMPTY), 0
    if scan < 0:
        d = _ctx_dict(c, keys=True)
        c.close()
        return d, 0
    try:
        _, _, m = c.append_scan(scans[scan], poses, slot)
    except balm_b200.BalmError as e:
        assert e.status == _lib.ERR_INVALID and "survives" in str(e)
        c.close()
        return dict(EMPTY), 0
    d = _ctx_dict(c, keys=True)
    c.close()
    return d, m


def _batch_append(scans, windows, wposes, scan_of, slots):
    import balm_b200
    b = balm_b200.Batch(0)
    b.cut_scans(scans, windows, wposes, **KW)
    res = b.append_scans(scans, scan_of, slots, wposes)
    got = b.download_voxels(with_keys=True, with_fix=True)
    b.close()
    return res, got


ALL = FIELDS + ("keys", "layers")


def test_append_matches_context_per_problem():
    scans, windows, wposes, scan_of, slots = _append_setup()
    res, got = _batch_append(scans, windows, wposes, scan_of, slots)
    for w, (win, x, s, sl, d, (M, K, m)) in enumerate(zip(windows, wposes, scan_of, slots, got, res)):
        ref, mref = _ctx_append(scans, win, x, s, sl)
        assert _equal(d, ref, ALL), w
        assert (M, K, m) == (len(ref["coe"]), len(ref["pose_idx"]), mref), w
    assert all(res[w][2] > 0 and (got[w]["pose_idx"] == slots[w]).any() for w in (0, 1, 2))  # the new scan joined
    assert res[0][2] != res[1][2]                            # one scan, two windows, two different sets of leaves
    assert res[4] == (0, 0, 0)
    # scan_of -1: bitwise the cut registration
    import balm_b200
    b = balm_b200.Batch(0)
    b.cut_scans(scans, windows, wposes, **KW)
    cut = b.download_voxels(with_keys=True, with_fix=True)
    b.close()
    assert _equal(got[3], cut[3], ALL)


def test_append_independence_and_determinism():
    scans, windows, wposes, scan_of, slots = _append_setup()
    res, got = _batch_append(scans, windows, wposes, scan_of, slots)
    res2, got2 = _batch_append(scans, windows, wposes, scan_of, slots)
    assert res == res2 and all(_equal(a, b, ALL) for a, b in zip(got, got2))
    perm = [4, 2, 0, 3, 1]
    pres, pgot = _batch_append(scans, [windows[i] for i in perm], [wposes[i] for i in perm], [scan_of[i] for i in perm],
                               [slots[i] for i in perm])
    for j, i in enumerate(perm):
        assert pres[j] == res[i] and _equal(pgot[j], got[i], ALL), i
    for i in (0, 1, 2):
        ares, agot = _batch_append(scans, [windows[i]], [wposes[i]], [scan_of[i]], [slots[i]])
        assert ares[0] == res[i] and _equal(agot[0], got[i], ALL), i


# ---------------------------------------------------------------- the whole window step ------------------------------
def _rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


def test_sliding_window_matches_context_route():
    """Sequences of different lengths: cut_scans -> damping_iter -> marginalize -> append_scans x 2 ->
    damping_iter(hess_includes_fix) -> pose_covariance(include_fix). Each context step gets the batch's poses, so the
    registrations must be bitwise equal; the LMs agree to 1e-9 with the same accept sequence; the covariance is anchored
    by the fix clusters now (BALM_OK)."""
    import balm_b200
    mg = 2
    Ns = [10, 8, 6]
    scans, windows, init, seqs = [], [], [], []
    for q, N in enumerate(Ns):
        pts, frs, poses = assoc_ref.synthetic_scans(n_poses=N + mg, pts_per_scan=5000, seed=40 + q)
        p12 = scenes.pack_poses([r for r, _ in poses], [p for _, p in poses])
        base = len(scans)
        scans += [pts[frs == i].astype(np.float32) for i in range(N + mg)]
        windows.append(list(range(base, base + N)))
        init.append(p12[:N])
        seqs.append((base, p12))
    b = balm_b200.Batch(0)
    b.cut_scans(scans, windows, init, **KW)
    lm_kw = dict(gauge_mode=2, min_planes_per_pose=0)
    lm = b.damping_iter(init, **lm_kw)
    ctx = []
    for win, x0, (st, p, tr, _) in zip(windows, init, lm):
        c = _ctx_cut(scans, win, x0)
        pc, trc, _ = c.damping_iter(x0, **lm_kw)
        assert st == 0 and [t["accepted"] for t in tr] == [t["accepted"] for t in trc]
        assert np.abs(p - pc).max() <= 1e-9
        ctx.append(c)
    poses = [r[1] for r in lm]
    mk = b.marginalize([mg] * len(Ns), poses)
    got = b.download_voxels(with_keys=True, with_fix=True)
    for c, x, d, (M, K) in zip(ctx, poses, got, mk):
        c.marginalize(mg, x)
        assert _equal(d, _ctx_dict(c, keys=True), ALL) and M > 0
    shifted = [np.vstack([x[mg:], p12[N:N + mg]]) for x, N, (_, p12) in zip(poses, Ns, seqs)]
    for j in range(mg):
        scan_of = [base + N + j for N, (base, _) in zip(Ns, seqs)]
        slots = [N - mg + j for N in Ns]
        res = b.append_scans(scans, scan_of, slots, shifted)
        got = b.download_voxels(with_keys=True, with_fix=True)
        for c, x, s, sl, d, (M, K, m) in zip(ctx, shifted, scan_of, slots, got, res):
            _, _, mc = c.append_scan(scans[s], x, sl)
            assert _equal(d, _ctx_dict(c, keys=True), ALL) and m == mc and m > 0
    lm2 = b.damping_iter(shifted, hess_includes_fix=True, **lm_kw)
    cov = b.pose_covariance([r[1] for r in lm2], point_noise=0.01, include_fix=True)
    for c, x, (st, p, tr, _), (cst, raw, rc) in zip(ctx, shifted, lm2, cov):
        pc, trc, _ = c.damping_iter(x, hess_includes_fix=True, **lm_kw)
        assert st == 0 and [t["accepted"] for t in tr] == [t["accepted"] for t in trc]
        assert np.abs(p - pc).max() <= 1e-9
        assert cst == 0                                        # anchored by the fix clusters
        raw_c, cov_c = c.pose_covariance(p, point_noise=0.01, include_fix=True)
        assert _rel(raw, raw_c) <= 1e-11 and _rel(rc, cov_c) <= 1e-9
        c.close()
    b.close()


# ---------------------------------------------------------------- rejected input -------------------------------------
def test_bad_input_is_rejected_and_keeps_the_registration():
    import balm_b200
    from balm_b200 import _lib
    from balm_b200.context import _p
    scans, windows, wposes, scan_of, slots = _append_setup()
    windows, wposes, scan_of, slots = windows[:3], wposes[:3], scan_of[:3], slots[:3]
    b = balm_b200.Batch(0)
    b.cut_scans(scans, windows, wposes, **KW)
    b.marginalize([0, 1, 0], wposes)
    before = b.download_voxels(with_keys=True, with_fix=True)
    L = _lib.lib()
    P = np.ascontiguousarray(np.concatenate(wposes))
    xyz = np.ascontiguousarray(np.concatenate(scans[:12]), dtype=np.float32)
    sp = np.concatenate([[0], np.cumsum([len(s) for s in scans[:12]])]).astype(np.int64)
    i32 = lambda *v: np.array(v, dtype=np.int32)

    def marg(mg):
        return L.balm_batch_marginalize(b._h, _p(i32(*mg)), _p(P), 15, None, None)

    def app(so, sl, scan_ptr=sp, n_scans=12, pts=xyz):
        return L.balm_batch_append_scan(b._h, _p(i32(*so)), _p(i32(*sl)), n_scans, _p(scan_ptr), _p(pts), _p(P), None,
                                        None, None)

    for mg in ([0, 0, 4], [-1, 0, 0], [8, 0, 0]):              # mg_size outside {0} and [1, N_p)
        assert marg(mg) == _lib.ERR_INVALID, mg
    assert b.n_poses == [8, 8, 4]
    bad = [
        ([10, -1, 12], [7, 0, 3], sp),                         # scan index = n_scans
        ([10, -2, -1], [7, 0, 0], sp),                         # scan index below -1
        ([10, -1, -1], [8, 0, 0], sp),                         # slot = N_p
        ([10, -1, -1], [-1, 0, 0], sp),                        # slot negative
        ([10, 10, -1], [7, 3, 0], sp),                         # slot 3 is not above the scans of problem 1's voxels
        ([10, -1, -1], [7, 0, 0], sp + 1),                     # scan_ptr[0] != 0
        ([10, -1, -1], [7, 0, 0], np.concatenate([sp[:12], [sp[11] - 1]]).astype(np.int64)),  # descending
    ]
    for so, sl, scan_ptr in bad:
        assert app(so, sl, scan_ptr) == _lib.ERR_INVALID, (so, sl)
    sp_empty = np.concatenate([sp, [sp[-1]]]).astype(np.int64)  # scan 12 is empty
    assert app([12, -1, -1], [7, 0, 0], sp_empty, 13) == _lib.ERR_INVALID
    # 2^31 points counted once per problem that takes them: rejected before the points are read
    huge = np.array([0, 1 << 30], dtype=np.int64)
    assert app([0, 0, -1], [7, 7, 0], huge, 1) == _lib.ERR_UNSUPPORTED
    after = b.download_voxels(with_keys=True, with_fix=True)
    assert all(_equal(x, y, ALL) for x, y in zip(before, after))
    # the slot check names the problem
    assert app([10, 10, -1], [7, 3, 0]) == _lib.ERR_INVALID and "problem 1" in L.balm_last_error().decode()
    # the next valid calls work
    assert app(scan_of, slots) == _lib.OK
    assert marg([1, 0, 1]) == _lib.OK
    # a registration without keys cannot take a scan
    rt = balm_b200.Batch(0)
    rt.set_problems(b.download_voxels(with_fix=True))
    with pytest.raises(balm_b200.BalmError) as e:
        rt.append_scans(scans, scan_of, slots, wposes)
    assert e.value.status == _lib.ERR_INVALID
    b.close()
    rt.close()

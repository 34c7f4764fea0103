"""GPU: persistent sliding-window octrees for a batch (balm_batch_window_*, Batch.window_*). Every problem's push must be
bitwise what a fp64 Context window of n_slots[p] slots pushes when driven by the same calls on that problem alone,
whatever else is in the batch and wherever the problem sits in it; a skipped problem (-1 / 0) is a call not made; bad
input is rejected and changes neither the maps nor the registration. Then the whole loop (push, LM with fix clusters,
pose covariance) against the per-sequence Context route, and a longer stream on which the persistent maps keep their
voxels while the reduced batch path (marginalize + append_scans) loses them."""
import numpy as np
import pytest

import scenes
import window_ref as wr

pytestmark = pytest.mark.gpu

KW = dict(voxel_size=2.0, min_ps=15, eigen_value_array=(1 / 16, 1 / 16, 1 / 9))
PTS = 1500


def _gaps(pts, frs, gt, wall_gap, object_gap):
    """Drops from growth_scans' scans the points of its returning wall (y = -4.5, x in [-3.8, 1.8]) in the scans of
    wall_gap and of its object (around (3, 1, -1.4)) in those of object_gap, [lo, hi) each: with windows of 16 or 32
    scans the wall is then out of view for longer than a window and the object appears after the first push."""
    keep = np.ones(len(pts), dtype=bool)
    for i in range(len(gt)):
        R, p = gt[i]
        sel = np.flatnonzero(frs == i)
        w = pts[sel] @ R.T + p
        drop = np.zeros(len(sel), dtype=bool)
        if wall_gap and wall_gap[0] <= i < wall_gap[1]:
            drop |= (np.abs(w[:, 1] + 4.5) < 0.1) & (w[:, 0] > -3.9) & (w[:, 0] < 1.9) & (w[:, 2] > -0.3)
        if object_gap and object_gap[0] <= i < object_gap[1]:
            drop |= (np.hypot(w[:, 0] - 3.0, w[:, 1] - 1.0) < 1.0) & (w[:, 2] < -0.7)
        keep[sel[drop]] = False
    return pts[keep], frs[keep]


def _sequence(seed, step, n_scans, wall_gap=None, object_gap=None, pts=PTS):
    """-> (scans, poses at cut time, poses marginalize re-transforms with)"""
    p, f, noisy, gt = wr.growth_scans(n_scans=n_scans, pts_per_scan=pts, seed=seed, step=step)
    if wall_gap or object_gap:
        p, f = _gaps(p, f, gt, wall_gap, object_gap)
    P = scenes.pack_poses([r for r, _ in noisy], [t for _, t in noisy])
    X = P.copy()
    X[:, 9:] += np.random.default_rng(seed).normal(0, 0.003, (n_scans, 3))
    return [p[f == i].astype(np.float32) for i in range(n_scans)], P, X


# sequence id -> (seed, step, scans, wall gap, object gap); problems (sequence id, n_slots, mg). Problems 0 and 1 share
# one sequence, so every cut they make together reads one scan.
SEQS = {0: (7, 0.5, 20, None, None), 1: (11, 0.4, 26, (16, 22), (12, 18)), 2: (13, 0.3, 44, (16, 36), (12, 36)),
        3: (17, 0.6, 22, None, None)}
PROBLEMS = [(0, 10, 2), (0, 4, 1), (1, 16, 3), (2, 32, 4), (3, 10, 5)]


def _streams():
    return {k: _sequence(*v) for k, v in SEQS.items()}


class CtxWindow:
    """A Context window with window_ref's method names; export() = push + download (keys, layers, row_ptr, pose_idx,
    obs10, fix10, coe)."""

    def __init__(self, n, **kw):
        import balm_b200
        self.N = n
        self.c = balm_b200.Context(n, 0, 0)
        self.c.window_reset(**kw)

    def cut_voxel(self, x, pose12, slot):
        self.c.window_cut(x, pose12, slot)

    def recut(self, w):
        self.c.window_recut(w)

    def marginalize(self, mg, x, w):
        self.c.window_marginalize(mg, x, w)

    def export(self, w):
        M, K = self.c.window_push(w)
        if M == 0:
            return _empty()
        keys, lay = self.c.download_keys(with_layers=True)
        rp, pi, ob, co = self.c.download_voxels()
        return keys.astype(np.int64), lay, rp, pi, ob, self.c.download_fix(), co


def _empty():
    return (np.zeros(0, np.int64), np.zeros(0, np.int32), np.zeros(1, np.int64), np.zeros(0, np.int32), np.zeros((0, 10)),
            np.zeros((0, 10)), np.zeros(0))


def _export(d):
    return (d["keys"].astype(np.int64), d["layers"], d["row_ptr"], d["pose_idx"], d["obs10"], d["fix10"], d["coe"])


def _bitwise(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


class BatchDriver:
    """Drives a Batch window through per-problem schedules (window_ref.window_schedule): every round makes one call of
    the kind the lowest unfinished problem needs next, for every problem whose next op is of that kind; the others are
    skipped (-1 / 0) in that call. on_push(p, export) for each problem that pushes."""

    def __init__(self, problems, streams, lim, recut_each_scan, order=None):
        import balm_b200
        self.problems = problems
        self.streams = streams
        self.order = list(range(len(problems))) if order is None else order
        self.b = balm_b200.Batch(0)
        self.ns = [problems[p][1] for p in self.order]
        self.b.window_reset(self.ns, layer_limit=lim, **KW)
        self.ops = []
        for p in self.order:
            seq, n, mg = problems[p]
            self.ops.append(wr.window_schedule(len(streams[seq][0]), n, mg, recut_each_scan))
        self.pos = [0] * len(problems)

    def done(self):
        return all(i >= len(o) for i, o in zip(self.pos, self.ops))

    def round(self, on_push):
        B = len(self.order)
        live = [q for q in range(B) if self.pos[q] < len(self.ops[q])]
        kind = self.ops[live[0]][self.pos[live[0]]][0]
        take = [q for q in live if self.ops[q][self.pos[q]][0] == kind]
        ops = {q: self.ops[q][self.pos[q]] for q in take}
        for q in take:
            self.pos[q] += 1
        zero = np.zeros((1, 12))
        if kind == "cut":
            names, scans, scan_of, slots, poses = {}, [], [-1] * B, [0] * B, []
            for q in range(B):
                seq = self.problems[self.order[q]][0]
                x = np.tile(zero, (self.ns[q], 1))
                if q in ops:
                    _, s, slot = ops[q]
                    if (seq, s) not in names:
                        names[(seq, s)] = len(scans)
                        scans.append(self.streams[seq][0][s])
                    scan_of[q], slots[q] = names[(seq, s)], slot
                    x[slot] = self.streams[seq][1][s]
                poses.append(x)
            self.b.window_cut(scans, scan_of, slots, poses)
        elif kind == "recut":
            self.b.window_recut([ops[q][1] if q in ops else 0 for q in range(B)])
        elif kind == "marginalize":
            mgs, wcs, poses = [0] * B, [0] * B, []
            for q in range(B):
                x = np.tile(zero, (self.ns[q], 1))
                if q in ops:
                    _, mg, first, w = ops[q]
                    x[:w] = self.streams[self.problems[self.order[q]][0]][2][first:first + w]
                    mgs[q], wcs[q] = mg, w
                poses.append(x)
            self.b.window_marginalize(mgs, poses, wcs)
        else:
            wcs = [ops[q][1] if q in ops else 0 for q in range(B)]
            mk = self.b.window_push(wcs)
            d = self.b.download_voxels(with_keys=True, with_fix=True)
            for q in range(B):
                if q in ops:
                    on_push(self.order[q], _export(d[q]))
                else:
                    assert mk[q] == (0, 0) and len(d[q]["coe"]) == 0
        return kind

    def run(self, on_push):
        while not self.done():
            self.round(on_push)


def _ctx_pushes(problems, streams, lim, recut_each_scan, only=None):
    out = {}
    for p, (seq, n, mg) in enumerate(problems):
        if only is not None and p not in only:
            continue
        sc, P, X = streams[seq]
        out[p] = []
        wr.run_schedule(wr.window_schedule(len(sc), n, mg, recut_each_scan), CtxWindow(n, layer_limit=lim, **KW), sc, P, X,
                        lambda t, e: out[p].append(e))
    return out


@pytest.fixture(scope="module")
def streams():
    return _streams()


@pytest.mark.parametrize("lim", [0, 2])
@pytest.mark.parametrize("recut_each_scan", [True, False])
def test_every_push_matches_a_context_window(streams, lim, recut_each_scan):
    dev = {p: [] for p in range(len(PROBLEMS))}
    BatchDriver(PROBLEMS, streams, lim, recut_each_scan).run(lambda p, e: dev[p].append(e))
    ref = _ctx_pushes(PROBLEMS, streams, lim, recut_each_scan)
    for p in range(len(PROBLEMS)):
        assert len(dev[p]) == len(ref[p]) >= 3, p
        for t, (a, b) in enumerate(zip(dev[p], ref[p])):
            assert _bitwise(a, b), (p, t)
        new_roots, resplit, revived = wr.growth_events(dev[p])
        assert new_roots > 0 and revived > 0, (p, new_roots, revived)
        if lim == 2:
            assert resplit > 0, p
        else:
            assert resplit == 0, p


def test_one_problem_matches_the_restatement(streams):
    """A batch of one problem against window_ref.WindowOctree, with test_gpu_window's tolerances."""
    prob = [(0, 10, 2)]
    dev = {0: []}
    BatchDriver(prob, streams, 2, True).run(lambda p, e: dev[p].append(e))
    sc, P, X = streams[0]
    ref = []
    wr.run_schedule(wr.window_schedule(len(sc), 10, 2, True), wr.WindowOctree(10, layer_limit=2, **KW), sc, P, X,
                    lambda t, e: ref.append(e))
    assert len(dev[0]) == len(ref) >= 5
    for a, b in zip(dev[0], ref):
        keys, lay, rp, pi, ob, fx, co = a
        k2, l2, rp2, pi2, ob2, fx2, co2 = b
        assert np.array_equal(keys, k2) and np.array_equal(lay, l2)
        assert np.array_equal(rp, rp2) and np.array_equal(pi, pi2) and np.array_equal(co, co2)
        if len(ob2):
            assert np.all(np.abs(ob - ob2) <= 1e-11 * np.abs(ob2).max(axis=0))
            assert np.abs(fx - fx2).max() <= 1e-12 * max(1.0, np.abs(fx2).max())


def test_independence_permutation_and_determinism(streams):
    """Problems permuted, a problem run alone, and the same call sequence twice: bitwise equal pushes."""
    probs = PROBLEMS[:3] + PROBLEMS[4:]
    base = {p: [] for p in range(len(probs))}
    BatchDriver(probs, streams, 2, True).run(lambda p, e: base[p].append(e))
    again = {p: [] for p in range(len(probs))}
    BatchDriver(probs, streams, 2, True).run(lambda p, e: again[p].append(e))
    perm = {p: [] for p in range(len(probs))}
    BatchDriver(probs, streams, 2, True, order=[3, 0, 2, 1]).run(lambda p, e: perm[p].append(e))
    alone = {2: []}
    BatchDriver([probs[2]], streams, 2, True).run(lambda p, e: alone[2].append(e))
    for p in range(len(probs)):
        assert len(base[p]) == len(again[p]) == len(perm[p])
        for a, b, c in zip(base[p], again[p], perm[p]):
            assert _bitwise(a, b) and _bitwise(a, c), p
    assert len(alone[2]) == len(base[2]) and all(_bitwise(a, b) for a, b in zip(alone[2], base[2]))


def _download(b):
    return [_export(d) for d in b.download_voxels(with_keys=True, with_fix=True)]


def test_skips_leave_a_map_as_if_the_call_was_not_made(streams):
    """Problem 1 is skipped in a cut, a recut, a marginalise and a push (-1 / 0) that problem 0 takes; its later pushes
    equal those of a context that never saw those calls."""
    import balm_b200
    sc, P, X = streams[0]
    b = balm_b200.Batch(0)
    b.window_reset([10, 10], layer_limit=2, **KW)
    c = [CtxWindow(10, layer_limit=2, **KW) for _ in range(2)]
    z = np.zeros((10, 12))

    def cut(s, slot, who):
        x = [z.copy(), z.copy()]
        for q in who:
            x[q][slot] = P[s]
            c[q].cut_voxel(sc[s], P[s], slot)
        b.window_cut([sc[s]], [0 if q in who else -1 for q in range(2)], [slot, slot], x)

    def recut(w, who):
        for q in who:
            c[q].recut(w)
        b.window_recut([w if q in who else 0 for q in range(2)])

    for s in range(10):
        cut(s, s, (0, 1))
        recut(s + 1, (0, 1))
    cut(10, 9, (0,))              # problem 1 skips a cut into a slot it will fill later
    recut(10, (0,))
    mk = b.window_push([10, 0])
    assert mk[1] == (0, 0)
    assert _bitwise(_download(b)[0], c[0].export(10))
    for q in (0,):
        c[q].marginalize(2, X[:10], 10)
    b.window_marginalize([2, 0], [X[:10], X[:10]], [10, 10])
    for q in (1,):
        c[q].marginalize(3, X[:10], 10)
    b.window_marginalize([0, 3], [X[:10], X[:10]], [0, 10])
    for s, slot in ((11, 8), (12, 9)):
        cut(s, slot, (0,))
        recut(slot + 1, (0,))
    cut(13, 7, (1,))
    recut(8, (1,))
    b.window_push([10, 10])
    d = _download(b)
    assert _bitwise(d[0], c[0].export(10)) and _bitwise(d[1], c[1].export(10))
    assert len(d[0][0]) > 20 and len(d[1][0]) > 20


def test_rejected_calls_change_nothing(streams):
    import ctypes as C
    import balm_b200
    from balm_b200 import _lib as L
    sc, P, X = streams[0]
    b = balm_b200.Batch(0)
    z = [np.zeros((4, 12)), np.zeros((6, 12))]
    with pytest.raises(balm_b200.BalmError) as e:   # no reset yet
        b.window_cut([sc[0]], [0, 0], [0, 0], z)
    assert e.value.status == 1
    with pytest.raises(balm_b200.BalmError) as e:
        b.window_push([1, 1])
    assert e.value.status == 1
    for ns in ([0, 4], [4, 33], []):
        with pytest.raises(balm_b200.BalmError) as e:
            b.window_reset(ns, layer_limit=2, **KW)
        assert e.value.status == 1
    b.window_reset([4, 6], layer_limit=2, **KW)
    c = [CtxWindow(4, layer_limit=2, **KW), CtxWindow(6, layer_limit=2, **KW)]
    for s in range(4):
        x = [z[0].copy(), z[1].copy()]
        x[0][s], x[1][s] = P[s], P[s]
        b.window_cut([sc[s]], [0, 0], [s, s], x)
        b.window_recut([s + 1, s + 1])
        for q in range(2):
            c[q].cut_voxel(sc[s], P[s], s)
            c[q].recut(s + 1)
    b.window_push([4, 4])
    reg = _download(b)
    far = sc[4].copy()
    far[17] = [6e5, 0, 0]                            # outside the +-2^18 root range of a 2 m voxel
    xs = [z[0].copy(), z[1].copy()]
    xs[1][4] = P[4]
    bad = [lambda: b.window_cut([sc[4]], [1, -1], [0, 0], z),                   # scan index
           lambda: b.window_cut([sc[4]], [-2, -1], [0, 0], z),
           lambda: b.window_cut([sc[4]], [-1, 0], [0, 6], z),                   # slot
           lambda: b.window_cut([sc[4]], [0, -1], [-1, 0], z),
           lambda: b.window_cut([sc[4], far], [0, 1], [3, 4], xs),             # point out of range in problem 1 only
           lambda: b.window_recut([5, 0]), lambda: b.window_recut([-1, 0]),     # win_count
           lambda: b.window_marginalize([1, 0], z, [0, 0]),                     # mg_size
           lambda: b.window_marginalize([4, 0], z, [4, 0]), lambda: b.window_marginalize([0, -1], z, [0, 6]),
           lambda: b.window_marginalize([0, 1], z, [0, 7]),
           lambda: b.window_push([0, 7]), lambda: b.window_push([-1, 0])]
    for f in bad:
        with pytest.raises(balm_b200.BalmError) as e:
            f()
        assert e.value.status == 1
    with pytest.raises(balm_b200.BalmError) as e:
        b.window_cut([sc[4], far], [0, 1], [3, 4], xs)
    assert "problem 1" in str(e.value)
    xyz = np.ascontiguousarray(sc[4])
    sp = np.array([5, 3], dtype=np.int64)                                       # scan_ptr not starting at 0
    rc = L.lib().balm_batch_window_cut(b._h, np.array([0, -1], np.int32).ctypes.data_as(C.c_void_p),
                                       np.zeros(2, np.int32).ctypes.data_as(C.c_void_p), 1, sp.ctypes.data_as(C.c_void_p),
                                       xyz.ctypes.data_as(C.c_void_p), np.zeros((10, 12)).ctypes.data_as(C.c_void_p))
    assert rc == 1
    sp = np.array([0, 5, 3], dtype=np.int64)                                    # not ascending
    rc = L.lib().balm_batch_window_cut(b._h, np.array([0, -1], np.int32).ctypes.data_as(C.c_void_p),
                                       np.zeros(2, np.int32).ctypes.data_as(C.c_void_p), 2, sp.ctypes.data_as(C.c_void_p),
                                       xyz.ctypes.data_as(C.c_void_p), np.zeros((10, 12)).ctypes.data_as(C.c_void_p))
    assert rc == 1
    assert all(_bitwise(a, r) for a, r in zip(_download(b), reg))            # the registration is untouched
    # ... and so are the maps: the next valid calls give what the contexts give
    x = [z[0].copy(), z[1].copy()]
    x[1][4] = P[4]
    b.window_cut([sc[4]], [-1, 0], [0, 4], x)
    b.window_recut([0, 5])
    c[1].cut_voxel(sc[4], P[4], 4)
    c[1].recut(5)
    b.window_marginalize([2, 0], [X[:4], X[:6]], [4, 0])
    c[0].marginalize(2, X[:4], 4)
    b.window_push([4, 5])
    d = _download(b)
    assert _bitwise(d[0], c[0].export(4)) and _bitwise(d[1], c[1].export(5))


def _rel(a, b):
    return np.abs(a - b).max() / np.abs(b).max()


def test_whole_loop_matches_the_context_route():
    """Fill, push, LM; then shifts of marginalise at the optimised poses, cut + recut, push, LM with the fix clusters
    (hess_includes_fix) and the pose covariance (include_fix), against a Context window per sequence driven with the
    batch's poses: same pushes; for the LM with fix clusters the same accept sequence and poses within 1e-9, covariances
    as in test_gpu_batch_window. Room scenes (assoc_ref.synthetic_scans, as test_gpu_batch_window uses): their planes
    fix every pose direction, which growth_scans' corridor does not (its translation along the corridor is weakly
    observed, so two correct LMs may part at 1e-8)."""
    import assoc_ref
    import balm_b200
    streams = {}
    for k, n in ((0, 14), (1, 22), (3, 14)):
        pts, frs, poses = assoc_ref.synthetic_scans(n_poses=n, pts_per_scan=5000, seed=40 + k)
        P = scenes.pack_poses([r for r, _ in poses], [t for _, t in poses])
        streams[k] = ([pts[frs == i].astype(np.float32) for i in range(n)], P, P)
    probs = [(0, 10, 2), (1, 16, 3), (3, 10, 2)]
    B = len(probs)
    ns = [n for _, n, _ in probs]
    lm_kw = dict(gauge_mode=2, min_planes_per_pose=0)
    b = balm_b200.Batch(0)
    b.window_reset(ns, layer_limit=2, **KW)
    ctx = [CtxWindow(n, layer_limit=2, **KW) for n in ns]
    P = [streams[s][1] for s, _, _ in probs]
    SC = [streams[s][0] for s, _, _ in probs]
    x = [P[q][:ns[q]].copy() for q in range(B)]
    for s in range(max(ns)):
        who = [q for q in range(B) if s < ns[q]]
        b.window_cut([SC[q][s] if q in who else SC[q][0] for q in range(B)], [q if q in who else -1 for q in range(B)],
                     [s if q in who else 0 for q in range(B)], x)
        b.window_recut([s + 1 if q in who else 0 for q in range(B)])
        for q in who:
            ctx[q].cut_voxel(SC[q][s], P[q][s], s)
            ctx[q].recut(s + 1)
    b.window_push(ns)
    for q in range(B):
        ctx[q].c.window_push(ns[q])
    x = [r[1] for r in b.damping_iter(x, **lm_kw)]  # the poses both routes marginalise with
    nxt = list(ns)
    for k in range(2):
        mgs = [mg for _, _, mg in probs]
        b.window_marginalize(mgs, x, ns)
        shifted = [np.vstack([x[q][mgs[q]:], P[q][nxt[q]:nxt[q] + mgs[q]]]) for q in range(B)]
        for q in range(B):
            ctx[q].marginalize(mgs[q], x[q], ns[q])
        for j in range(max(mgs)):
            who = [q for q in range(B) if j < mgs[q]]
            sl = [ns[q] - mgs[q] + j if q in who else 0 for q in range(B)]
            b.window_cut([SC[q][nxt[q] + j] if q in who else SC[q][0] for q in range(B)],
                         [q if q in who else -1 for q in range(B)], sl, shifted)
            b.window_recut([sl[q] + 1 if q in who else 0 for q in range(B)])
            for q in who:
                ctx[q].cut_voxel(SC[q][nxt[q] + j], shifted[q][sl[q]], sl[q])
                ctx[q].recut(sl[q] + 1)
        nxt = [nxt[q] + mgs[q] for q in range(B)]
        b.window_push(ns)
        d = _download(b)
        for q in range(B):
            assert _bitwise(d[q], ctx[q].export(ns[q])), (k, q)
        lm = b.damping_iter(shifted, hess_includes_fix=True, **lm_kw)
        cov = b.pose_covariance([r[1] for r in lm], point_noise=0.01, include_fix=True)
        for q in range(B):
            st, p, tr, _ = lm[q]
            assert st == 0
            pc, trc, _ = ctx[q].c.damping_iter(shifted[q], hess_includes_fix=True, **lm_kw)
            assert [t["accepted"] for t in tr] == [t["accepted"] for t in trc]
            assert np.abs(p - pc).max() <= 1e-9
            raw_c, cov_c = ctx[q].c.pose_covariance(p, point_noise=0.01, include_fix=True)
            cst, raw, rc = cov[q]
            assert cst == 0
            assert _rel(raw, raw_c) <= 1e-11 and _rel(rc, cov_c) <= 1e-9
        x = [r[1] for r in lm]


def test_longer_stream_keeps_its_voxels():
    """40 scans of 3 000 points, 0.5 m per scan, window 10, mg 2, layer_limit 2, two sequences: the persistent maps'
    last push keeps at least as many voxels as their first, the reduced batch path falls below half of its first."""
    import balm_b200
    N, MG, n_scans = 10, 2, 40
    seqs = [_sequence(seed, 0.5, n_scans, pts=3000) for seed in (3, 5)]
    kw = dict(layer_limit=2, **KW)
    b = balm_b200.Batch(0)
    b.window_reset([N, N], **kw)
    red = balm_b200.Batch(0)
    z = [np.zeros((N, 12)), np.zeros((N, 12))]
    for s in range(N):
        x = [z[0].copy(), z[1].copy()]
        x[0][s], x[1][s] = seqs[0][1][s], seqs[1][1][s]
        b.window_cut([seqs[0][0][s], seqs[1][0][s]], [0, 1], [s, s], x)
        b.window_recut([s + 1, s + 1])
    per = [sum(m for m, _ in b.window_push([N, N]))]
    cut = red.cut_scans([q[0][s] for q in seqs for s in range(N)], [list(range(N)), list(range(N, 2 * N))],
                        [q[1][:N] for q in seqs], **kw)
    rd = [sum(m for m, _ in cut)]
    first, nxt = 0, N
    while nxt + MG <= n_scans:
        xw = [q[2][first:first + N] for q in seqs]
        b.window_marginalize([MG, MG], xw, [N, N])
        red.marginalize([MG, MG], xw)
        first += MG
        shifted = [np.vstack([q[2][first:first + N - MG], q[1][nxt:nxt + MG]]) for q in seqs]
        for j in range(MG):
            slot = N - MG + j
            b.window_cut([q[0][nxt + j] for q in seqs], [0, 1], [slot, slot], shifted)
            b.window_recut([slot + 1, slot + 1])
            app = red.append_scans([q[0][nxt + j] for q in seqs], [0, 1], [slot, slot], shifted)
        nxt += MG
        per.append(sum(m for m, _ in b.window_push([N, N])))
        rd.append(sum(m for m, _, _ in app))
    assert len(per) >= 15
    assert per[-1] >= per[0], per
    assert rd[-1] < rd[0] / 2, rd

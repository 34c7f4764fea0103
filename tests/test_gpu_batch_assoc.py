"""Batched association (balm_batch_cut_voxels, balm_b200.Batch.cut_scans): every window's plane voxels cut from raw scans
on the device and registered in one call. Each window must get bitwise what Context(N_w).cut_voxels registers on its own
points (arrays, keys, layers), whatever else is in the batch; empty windows are registered empty; bad input is rejected
and keeps the previous registration."""
import ctypes as C
import os

import numpy as np
import pytest

import assoc_ref
import scenes

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "realworld_points_small.npz")
EIG = (1 / 16, 1 / 16, 1 / 9)


def layer_windows(n, length=10, stride=5):
    """HBA's bottom layer: windows of `length` scans every `stride` scans, the last one cut at n."""
    out, s = [], 0
    while True:
        out.append(list(range(s, min(s + length, n))))
        if s + length >= n:
            return out
        s += stride


def _context_cut(scans, win, poses12, **kw):
    """Context(N_w).cut_voxels on the window's points with frame = slot -> (row_ptr, pose_idx, obs10, coe, keys, layers);
    a window without a plane voxel -> empty arrays."""
    import balm_b200
    from balm_b200 import _lib
    pts = np.concatenate([scans[s] for s in win]).astype(np.float32)
    fr = np.concatenate([np.full(len(scans[s]), k, dtype=np.int32) for k, s in enumerate(win)])
    c = balm_b200.Context(len(win), 0, balm_b200.PREC_FP64)
    try:
        c.cut_voxels(pts, fr, poses12, **kw)
    except balm_b200.BalmError as e:
        assert e.status == _lib.ERR_INVALID and "no plane voxels" in str(e)
        c.close()
        return (np.zeros(1, dtype=np.int64), np.zeros(0, dtype=np.int32), np.zeros((0, 10)), np.zeros(0),
                np.zeros(0, dtype=np.uint64), np.zeros(0, dtype=np.int32))
    out = c.download_voxels() + c.download_keys(with_layers=True)
    c.close()
    return out


def _same(d, ref):
    rp, pi, ob, co, keys, layers = ref
    return (np.array_equal(d["row_ptr"], rp) and np.array_equal(d["pose_idx"], pi) and np.array_equal(d["obs10"], ob)
            and np.array_equal(d["coe"], co) and np.array_equal(d["keys"], keys) and np.array_equal(d["layers"], layers))


def _cut(scans, windows, poses, **kw):
    import balm_b200
    b = balm_b200.Batch(0)
    mk = b.cut_scans(scans, windows, poses, **kw)
    return b, mk, b.download_voxels(with_keys=True)


def _lm_key(res):
    return [(st, p, [tuple(t.values()) for t in tr]) for st, p, tr, _ in res]


def _lm_equal(a, b):
    return all(x[0] == y[0] and np.array_equal(x[1], y[1]) and x[2] == y[2] for x, y in zip(_lm_key(a), _lm_key(b)))


@pytest.fixture(scope="module")
def realworld():
    d = np.load(GOLD)
    n = len(d["poses"])
    scans = [d["xyz"][d["frame"] == i] for i in range(n)]
    return scans, np.asarray(d["poses"], dtype=np.float64)


def test_realworld_layer_matches_context_and_reference(realworld):
    scans, poses = realworld
    windows = layer_windows(len(scans))
    assert windows == [list(range(0, 10)), list(range(5, 15)), list(range(10, 20)), list(range(15, 24))]
    wposes = [poses[w] for w in windows]
    b, mk, got = _cut(scans, windows, wposes, voxel_size=2.0, eigen_value_array=EIG)
    for win, p12, d, (M, K) in zip(windows, wposes, got, mk):
        ref = _context_cut(scans, win, p12, voxel_size=2.0, eigen_value_array=EIG)
        assert _same(d, ref) and (M, K) == (len(ref[3]), len(ref[1])) and M > 0
        # the numpy restatement, under test_assoc._compare's rules
        pts = np.concatenate([scans[s] for s in win]).astype(np.float64)
        fr = np.concatenate([np.full(len(scans[s]), k, dtype=np.int32) for k, s in enumerate(win)])
        rp0, pi0, obs0, coe0, keys0, lay0 = assoc_ref.cut_voxels(pts, fr, [scenes.unpack_pose(p) for p in p12],
                                                                  with_layers=True, voxel_size=2.0, eigen_value_array=EIG)
        assert np.array_equal(d["row_ptr"], rp0) and np.array_equal(d["pose_idx"], pi0) and np.array_equal(d["coe"], coe0)
        assert np.array_equal(d["keys"].astype(np.int64), keys0) and np.array_equal(d["layers"], lay0)
        assert np.array_equal(d["obs10"][:, 9], obs0[:, 9])
        assert np.all(np.abs(d["obs10"] - obs0) <= 1e-11 * np.abs(obs0).max(axis=0))
    b.close()


def _synthetic():
    """36 overlapping synthetic scans plus three tiny scans of a few scattered points."""
    pts, frs, poses = assoc_ref.synthetic_scans(n_poses=36, pts_per_scan=2500, seed=9)
    scans = [pts[frs == i] for i in range(36)]
    p12 = list(scenes.pack_poses([r for r, _ in poses], [p for _, p in poses]))
    rng = np.random.default_rng(3)
    for _ in range(3):
        scans.append(rng.uniform(-5, 5, (6, 3)).astype(np.float32).astype(np.float64))
        p12.append(p12[0])
    windows = [[0, 1], list(range(0, 32)), list(range(3, 10)), [5], list(range(20, 36)), [36, 37, 38],
               list(range(10, 23)), [30, 31, 32, 33]]
    return scans, np.array(p12), windows


@pytest.mark.parametrize("layer_limit,voxel_size", [(2, 2.0), (1, 2.0), (0, 1.0), (2, 1.0)])
def test_options_shapes_and_empty_windows(layer_limit, voxel_size):
    from balm_b200 import _lib
    scans, p12, windows = _synthetic()
    wposes = [p12[w] for w in windows]
    kw = dict(layer_limit=layer_limit, voxel_size=voxel_size)
    b, mk, got = _cut(scans, windows, wposes, **kw)
    empty = []
    for w, (win, d, (M, K)) in enumerate(zip(windows, got, mk)):
        ref = _context_cut(scans, win, p12[win], **kw)
        assert _same(d, ref), (w, win)
        assert (M, K) == (len(ref[3]), len(ref[1]))
        if M == 0:
            empty.append(w)
    assert 3 in empty and 5 in empty                 # one scan: no voxel has two frames; tiny scans: no plane
    assert mk[1][0] > 0 and mk[2][0] > 0
    res = b.damping_iter(wposes)
    for w in empty:
        st, p, tr, _ = res[w]
        assert st == _lib.ERR_TOO_FEW_PLANES and tr == [] and np.array_equal(p, wposes[w])
    b.close()


def test_independence_and_determinism():
    scans, p12, windows = _synthetic()
    wposes = [p12[w] for w in windows]
    kw = dict(min_planes_per_pose=0, want_per_iter=True, max_iter=6)
    b, _, got = _cut(scans, windows, wposes)
    lm = b.damping_iter(wposes, **kw)
    b2, _, got2 = _cut(scans, windows, wposes)                        # a second identical call
    assert all(_same(x, tuple(y[k] for k in ("row_ptr", "pose_idx", "obs10", "coe", "keys", "layers")))
               for x, y in zip(got, got2))
    assert _lm_equal(lm, b2.damping_iter(wposes, **kw))
    rb, _, rgot = _cut(scans, windows[::-1], wposes[::-1])            # reversed window order
    rlm = rb.damping_iter(wposes[::-1], **kw)[::-1]
    for x, y in zip(got, rgot[::-1]):
        assert _same(x, tuple(y[k] for k in ("row_ptr", "pose_idx", "obs10", "coe", "keys", "layers")))
    assert _lm_equal(lm, rlm)
    for w in (1, 2, 6):                                               # one window alone
        ab, _, agot = _cut(scans, [windows[w]], [wposes[w]])
        assert _same(got[w], tuple(agot[0][k] for k in ("row_ptr", "pose_idx", "obs10", "coe", "keys", "layers")))
        assert _lm_equal([lm[w]], ab.damping_iter([wposes[w]], **kw))
    for x in (b, b2, rb):
        x.close()


def test_lm_after_cut_equals_round_trip_and_context(realworld):
    import balm_b200
    scans, poses = realworld
    windows = layer_windows(len(scans))
    wposes = [poses[w] for w in windows]
    kw = dict(voxel_size=2.0, eigen_value_array=EIG)
    b, _, got = _cut(scans, windows, wposes, **kw)
    lm = b.damping_iter(wposes, want_per_iter=True, min_planes_per_pose=0)
    rt = balm_b200.Batch(0)
    rt.set_problems(b.download_voxels())
    assert _lm_equal(lm, rt.damping_iter(wposes, want_per_iter=True, min_planes_per_pose=0))
    for win, p12, (st, p, tr, _) in zip(windows, wposes, lm):
        pts = np.concatenate([scans[s] for s in win]).astype(np.float32)
        fr = np.concatenate([np.full(len(scans[s]), k, dtype=np.int32) for k, s in enumerate(win)])
        c = balm_b200.Context(len(win), 0, balm_b200.PREC_FP64)
        c.cut_voxels(pts, fr, p12, **kw)
        pc, trc, _ = c.damping_iter(p12, min_planes_per_pose=0)
        assert st == 0 and len(tr) == len(trc) and [t["accepted"] for t in tr] == [t["accepted"] for t in trc]
        assert np.abs(p - pc).max() <= 1e-9, np.abs(p - pc).max()
        c.close()
    b.close()
    rt.close()


def test_bad_input_is_rejected_and_keeps_the_registration(realworld):
    import balm_b200
    from balm_b200 import _lib
    from balm_b200.context import _p
    scans, poses = realworld
    windows = layer_windows(len(scans))[:2]
    wposes = [poses[w] for w in windows]
    b, _, _ = _cut(scans, windows, wposes, voxel_size=2.0, eigen_value_array=EIG)
    before = [r for _, _, r in b.evaluate(wposes)]
    L = _lib.lib()
    i64 = lambda *v: np.array(v, dtype=np.int64)
    i32 = lambda *v: np.array(v, dtype=np.int32)
    xyz = np.ascontiguousarray(np.concatenate(scans[:4]), dtype=np.float32)
    sp = np.concatenate([[0], np.cumsum([len(s) for s in scans[:4]])]).astype(np.int64)
    p12 = np.ascontiguousarray(np.tile(poses[0], (40, 1)))
    far = xyz.copy()
    far[7] = [1e6, 0, 0]                                              # outside the +-2^18 root range at voxel size 2

    def call(n, pp, ps, n_scans, scan_ptr, pts=xyz, layer_limit=2):
        o = _lib.AssocOpts(2.0, layer_limit, 15, (C.c_double * 3)(*EIG))
        return L.balm_batch_cut_voxels(b._h, n, _p(pp), _p(ps), n_scans, _p(scan_ptr), _p(pts), _p(p12), C.byref(o),
                                       None, None)

    ok = (2, i64(0, 2, 4), i32(0, 1, 2, 3), 4, sp)
    assert call(*ok) == _lib.OK
    b.cut_scans(scans, windows, wposes, voxel_size=2.0, eigen_value_array=EIG)
    bad = [
        (0, i64(0), i32(), 4, sp),                                    # no problem
        (2, i64(0, 0, 4), i32(0, 1, 2, 3), 4, sp),                    # a problem without poses
        (1, i64(0, 33), np.zeros(33, dtype=np.int32), 4, sp),         # 33 poses
        (2, i64(0, 3, 2), i32(0, 1, 2), 4, sp),                       # pose_ptr descending
        (2, i64(0, 2, 4), i32(0, 1, 2, 4), 4, sp),                    # pose_scan = n_scans
        (2, i64(0, 2, 4), i32(0, -1, 2, 3), 4, sp),                   # pose_scan negative
        (2, i64(0, 2, 4), i32(0, 1, 2, 3), 4, sp + 1),                # scan_ptr[0] != 0
        (2, i64(0, 2, 4), i32(0, 1, 2, 3), 4, i64(0, sp[2], sp[1], sp[3], sp[4])),  # scan_ptr descending
    ]
    for args in bad:
        assert call(*args) == _lib.ERR_INVALID, args
    for lim in (-1, 3):
        assert call(*ok, layer_limit=lim) == _lib.ERR_INVALID
    assert call(*ok[:4], sp, far) == _lib.ERR_INVALID
    # 2^31 points counted once per pose row that uses them: rejected on the host, before the points are read
    assert call(2, i64(0, 1, 2), i32(0, 0), 1, i64(0, 1 << 30)) == _lib.ERR_UNSUPPORTED
    after = [r for _, _, r in b.evaluate(wposes)]
    assert before == after
    rt = balm_b200.Batch(0)
    rt.set_problems(b.download_voxels())
    with pytest.raises(balm_b200.BalmError) as e:                     # keys exist only after a cut
        rt.download_voxels(with_keys=True)
    assert e.value.status == _lib.ERR_INVALID
    b.close()
    rt.close()

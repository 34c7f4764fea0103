"""Keyframe merge on the device (balm_batch_merge_scans, balm_b200.Batch.merge_scans): every window's scans in the body
frame of its slot 0, down-sampled. Each keyframe must be bitwise tests/hba_ref.keyframe_ref, whatever else is in the
batch; bad input is rejected with the outputs unwritten and the registration untouched."""
import os

import numpy as np
import pytest

import assoc_ref
import hba_ref
import scenes
from balm_b200 import hba

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "realworld_points_small.npz")


def _room(n=24, pts=3000, seed=9, room=12.0):
    pts_, frs, poses = assoc_ref.synthetic_scans(n_poses=n, pts_per_scan=pts, seed=seed, room=room)
    scans = [pts_[frs == i].astype(np.float32) for i in range(n)]
    return scans, scenes.pack_poses([r for r, _ in poses], [p for _, p in poses])


def _check(scans, windows, wposes, voxel_size):
    import balm_b200
    b = balm_b200.Batch(0)
    got = b.merge_scans(scans, windows, wposes, voxel_size)
    b.close()
    assert len(got) == len(windows)
    for w, (win, p12, kf) in enumerate(zip(windows, wposes, got)):
        ref = hba_ref.keyframe_ref(scans, win, p12, voxel_size)
        assert kf.dtype == np.float32 and kf.shape == ref.shape, (w, kf.shape, ref.shape)
        assert np.array_equal(kf, ref), (w, voxel_size)
    return got


@pytest.mark.parametrize("voxel_size", [0.0, 0.05, 0.1, 0.5, 2.0])
def test_overlapping_room_windows_match_the_restatement(voxel_size):
    scans, p12 = _room()
    windows = hba.layer_windows(len(scans)) + [[3, 7, 3], [20]]  # a scan twice in one window, a single scan
    got = _check(scans, windows, [p12[w] for w in windows], voxel_size)
    n_items = sum(len(scans[s]) for w in windows for s in w)
    if voxel_size == 0.0:
        assert sum(len(k) for k in got) == n_items
    else:
        assert 0 < sum(len(k) for k in got) < n_items


@pytest.mark.parametrize("voxel_size", [0.0, 0.1, 1.0])
def test_realworld_slice_matches_the_restatement(voxel_size):
    d = np.load(GOLD)
    n = len(d["poses"])
    scans = [d["xyz"][d["frame"] == i].astype(np.float32) for i in range(n)]
    poses = np.asarray(d["poses"], dtype=np.float64)
    windows = hba.layer_windows(n)
    assert n == 24 and len(windows) == 4
    _check(scans, windows, [poses[w] for w in windows], voxel_size)


def test_empty_scans_and_empty_windows():
    scans, p12 = _room(n=6, pts=1500)
    scans = scans[:3] + [np.zeros((0, 3), np.float32)] + scans[3:] + [np.zeros((0, 3), np.float32)]
    windows = [[0, 3, 1], [3], [3, 7, 3], [2, 4, 5, 6], [7]]
    wposes = [np.tile(p12[0], (len(w), 1)) if w[0] in (3, 7) else p12[[min(s, 5) for s in w]] for w in windows]
    for vs in (0.0, 0.2):
        got = _check(scans, windows, wposes, vs)
        assert [len(got[w]) for w in (1, 2, 4)] == [0, 0, 0] and len(got[0]) > 0
    import balm_b200
    b = balm_b200.Batch(0)
    assert [len(k) for k in b.merge_scans(scans, [[3], [7, 3]], [p12[:1], p12[:2]], 0.2)] == [0, 0]
    b.close()


def test_independence_order_and_determinism():
    import balm_b200
    scans, p12 = _room(n=30, pts=2000, seed=4)
    windows = hba.layer_windows(30) + [[0], list(range(0, 30, 3))]
    wposes = [p12[w] for w in windows]
    b = balm_b200.Batch(0)
    got = b.merge_scans(scans, windows, wposes, 0.1)
    again = b.merge_scans(scans, windows, wposes, 0.1)
    rev = b.merge_scans(scans, windows[::-1], wposes[::-1], 0.1)[::-1]
    for w in range(len(windows)):
        alone = b.merge_scans(scans, [windows[w]], [wposes[w]], 0.1)[0]
        assert np.array_equal(got[w], again[w]) and np.array_equal(got[w], rev[w]) and np.array_equal(got[w], alone)
    b.close()


def test_bad_input_is_rejected_with_outputs_unwritten():
    import balm_b200
    from balm_b200 import _lib
    from balm_b200.context import _p
    scans, p12 = _room(n=8, pts=1500)
    windows = hba.layer_windows(8, 4, 2)
    wposes = [p12[w] for w in windows]
    b = balm_b200.Batch(0)
    b.cut_scans(scans, windows, wposes)
    before = b.download_voxels(with_keys=True)
    L = _lib.lib()
    i64 = lambda *v: np.array(v, dtype=np.int64)
    i32 = lambda *v: np.array(v, dtype=np.int32)
    xyz = np.ascontiguousarray(np.concatenate(scans[:4]), dtype=np.float32)
    sp = np.concatenate([[0], np.cumsum([len(s) for s in scans[:4]])]).astype(np.int64)
    poses = np.ascontiguousarray(np.tile(p12[0], (40, 1)))
    far = poses.copy()
    far[3, 9] = 4e5                                                   # problem 1, slot 1: 1.3e6 voxels of 0.3 away
    kf_ptr = np.full(3, -7, dtype=np.int64)
    kf = np.full((4 * len(xyz), 3), -7, dtype=np.float32)

    def call(n, pp, ps, n_scans, scan_ptr, x=poses, vs=0.3):
        return L.balm_batch_merge_scans(b._h, n, _p(pp), _p(ps), n_scans, _p(scan_ptr), _p(xyz), _p(x), float(vs),
                                        _p(kf_ptr), _p(kf))

    ok = (2, i64(0, 2, 4), i32(0, 1, 2, 3), 4, sp)
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
    for vs in (float("nan"), float("inf"), -float("inf")):
        assert call(*ok, vs=vs) == _lib.ERR_INVALID
    assert call(*ok, x=far) == _lib.ERR_INVALID                       # outside +-2^20, found on the device
    assert "problem 1" in L.balm_last_error().decode()
    far[3, 9] = -4e5
    far[1, 10] = 4e5                                                  # now problem 0 too: the lowest is named
    assert call(*ok, x=far) == _lib.ERR_INVALID and "problem 0" in L.balm_last_error().decode()
    # 2^31 points counted once per pose row that uses them: rejected on the host, before the points are read
    assert call(2, i64(0, 1, 2), i32(0, 0), 1, i64(0, 1 << 30)) == _lib.ERR_UNSUPPORTED
    assert np.all(kf_ptr == -7) and np.all(kf == -7)
    after = b.download_voxels(with_keys=True)
    assert all(all(np.array_equal(x[k], y[k]) for k in x) for x, y in zip(before, after))
    assert call(*ok) == _lib.OK and kf_ptr[0] == 0 and 0 < kf_ptr[2] <= len(xyz) * 2
    b.close()

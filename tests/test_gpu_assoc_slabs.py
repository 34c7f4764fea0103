"""balm_cut_voxels in root-key slabs (BALM_ASSOC_BUDGET_MB below the one-pass bound): bitwise the one-pass cut on the
room scans, a synthetic street drive and the reference's own data, at every layer limit, two voxel sizes, both point
orders and budgets from one pass down to the tightest slab cap; the refusals leave the registration as it was; BA,
marginalisation, scan appending and rig calibration on slabbed voxels are bitwise those on one-pass voxels."""
import contextlib
import os

import numpy as np
import pytest

import assoc_ref
import balm_b200
import rig_ref as rr
import scenes
import street_ref
from balm_b200 import _lib as L

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "realworld_points_small.npz")
EIG = (1 / 16, 1 / 16, 1 / 9)


def _inputs(name):
    """-> (points_body float64 rounded to float32, frames, poses [(R, p)])"""
    if name == "synthetic":
        return assoc_ref.synthetic_scans(n_poses=10, pts_per_scan=5000, seed=9)
    if name == "street":
        return street_ref.street_scans()
    d = np.load(GOLD)
    return d["xyz"].astype(np.float64), d["frame"], [scenes.unpack_pose(p) for p in d["poses"]]


def _poses12(poses):
    return scenes.pack_poses([r for r, _ in poses], [p for _, p in poses])


@contextlib.contextmanager
def _budget(nbytes):
    """BALM_ASSOC_BUDGET_MB = nbytes exactly (a binary fraction of a MiB is exact in the decimal repr)"""
    old = os.environ.get("BALM_ASSOC_BUDGET_MB")
    os.environ["BALM_ASSOC_BUDGET_MB"] = repr(nbytes / 2 ** 20)
    try:
        yield
    finally:
        if old is None:
            del os.environ["BALM_ASSOC_BUDGET_MB"]
        else:
            os.environ["BALM_ASSOC_BUDGET_MB"] = old


def _snap(c):
    return (*c.download_voxels(), *c.download_keys(with_layers=True))


def _same(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


def _error(fn):
    with pytest.raises(balm_b200.BalmError) as e:
        fn()
    return e.value.status, str(e.value)


@pytest.mark.parametrize("layer_limit", [0, 1, 2])
@pytest.mark.parametrize("name", ["synthetic", "street", "realworld"])
def test_slabs_are_bitwise_the_one_pass_cut(name, layer_limit):
    pts, frs, poses = _inputs(name)
    N, n = len(poses), len(frs)
    poses12 = _poses12(poses)
    perm = np.random.default_rng(3).permutation(n)
    c = balm_b200.Context(N, 0, L.PREC_FP64)
    for vs in (2.0, 1.0):
        kw = dict(voxel_size=vs, layer_limit=layer_limit, eigen_value_array=EIG)
        counts = street_ref.root_counts(pts, frs, poses, vs)
        for order in (np.arange(n), perm):
            xyz, fr = pts[order].astype(np.float32), frs[order]
            c.cut_voxels(xyz, fr, poses12, **kw)
            ref = _snap(c)
            st = c.cut_stats()
            assert st["slabs"] == 1 and st["max_slab_points"] == n and st["roots"] == len(counts)
            P, F = st["scratch_per_point"], st["scratch_fixed"]
            assert P == 345 + 120 * (layer_limit + 1) and st["peak_scratch_bytes"] <= P * n + F
            tight = F + P * int(counts.max())
            budgets = [F + P * n, F + P * max(int(counts.max()), n // 4), tight]
            for B in budgets:
                with _budget(B):
                    c.cut_voxels(xyz, fr, poses12, **kw)
                assert _same(_snap(c), ref), (name, layer_limit, vs, B)
                s = c.cut_stats()
                cap = (B - F) // P
                assert s["slabs"] == (1 if B >= F + P * n else street_ref.greedy_slabs(counts, cap)), (s, cap)
                assert s["roots"] == len(counts) and s["peak_scratch_bytes"] <= B and s["max_slab_points"] <= cap
            assert s["slabs"] > 1


def test_refusals_leave_the_registration():
    pts, frs, poses = street_ref.street_scans(n_forward=16, n_revisit=4)
    N, n = len(poses), len(frs)
    poses12 = _poses12(poses)
    xyz = pts.astype(np.float32)
    c = balm_b200.Context(N, 0, L.PREC_FP64)
    c.cut_voxels(xyz, frs, poses12)
    ref, ev = _snap(c), c.evaluate(poses12)
    st = c.cut_stats()
    P, F = st["scratch_per_point"], st["scratch_fixed"]
    counts = street_ref.root_counts(pts, frs, poses, 2.0)
    big = int(counts.max())

    def unchanged():
        assert _same(_snap(c), ref)
        assert all(np.array_equal(a, b) for a, b in zip(c.evaluate(poses12), ev))

    with _budget(F + P * (big - 1)):  # the cap one point below the largest root
        status, msg = _error(lambda: c.cut_voxels(xyz, frs, poses12))
    assert status == L.ERR_UNSUPPORTED and f"holds {big} points" in msg and f"the {big - 1} points" in msg, msg
    unchanged()
    bad_frame = frs.copy()
    bad_frame[n // 2] = N
    far = xyz.copy()
    far[n // 3] = (1e6, 0.0, 0.0)
    noise = np.random.default_rng(1).normal(0, 40.0, (20000, 3)).astype(np.float32)
    cases = [(xyz, bad_frame), (far, frs), (noise, np.repeat(np.arange(N, dtype=np.int32), 20000 // N + 1)[:20000])]
    for p, f in cases:
        one = _error(lambda: c.cut_voxels(p, f, poses12))
        unchanged()
        with _budget(F + P * (len(f) // 5)):
            slab = _error(lambda: c.cut_voxels(p, f, poses12))
        assert slab == one and one[0] == L.ERR_INVALID, (one, slab)
        unchanged()
    assert "frame index" in _error(lambda: c.cut_voxels(xyz, bad_frame, poses12))[1]


@pytest.mark.parametrize("prec", [L.PREC_FP64, L.PREC_BLOCKS])
def test_downstream_is_bitwise(prec):
    pts, frs, poses = street_ref.street_scans()
    N, n = len(poses), len(frs)
    poses12 = _poses12(poses)
    xyz = pts.astype(np.float32)
    a = balm_b200.Context(N, 0, prec)
    a.cut_voxels(xyz, frs, poses12)
    st = a.cut_stats()
    b = balm_b200.Context(N, 0, prec)
    with _budget(st["scratch_fixed"] + st["scratch_per_point"] * (n // 6)):
        for _ in range(2):  # two slabbed calls on one context
            b.cut_voxels(xyz, frs, poses12)
            assert b.cut_stats()["slabs"] > 1 and _same(_snap(b), _snap(a))
    pa, tra, _ = a.damping_iter(poses12, min_planes_per_pose=0)
    pb, trb, _ = b.damping_iter(poses12, min_planes_per_pose=0)
    assert tra == trb and np.array_equal(pa, pb) and len(tra) > 1
    if prec == L.PREC_FP64:
        for c, p in ((a, pa), (b, pb)):
            c.marginalize(2, p)
            p2 = np.concatenate([p[2:], p[-2:]])
            c.append_scan(xyz[frs == N - 1], p2, N - 2)
        assert _same(_snap(a), _snap(b))
        assert np.array_equal(a.download_fix(), b.download_fix())


def test_calibrate_rig_on_blocks_under_a_small_budget():
    S = rr.rig_scene()
    base0, ext0 = rr.perturbed_start(S)
    args = (S["xyz"], S["scan"], S["base_of"], S["lidar_of"], base0, ext0)
    ref = balm_b200.calibrate_rig(*args, precision=L.PREC_BLOCKS)
    probe = balm_b200.Context(len(S["base_of"]), 0, L.PREC_FP64)
    probe.cut_voxels(S["xyz"], S["scan"], rr.compose(base0, ext0, S["base_of"], S["lidar_of"]))
    st = probe.cut_stats()
    n = len(S["scan"])
    with _budget(st["scratch_fixed"] + st["scratch_per_point"] * (n // 3)):
        out = balm_b200.calibrate_rig(*args, precision=L.PREC_BLOCKS)
    assert np.array_equal(out[0], ref[0]) and np.array_equal(out[1], ref[1]) and out[2] == ref[2]

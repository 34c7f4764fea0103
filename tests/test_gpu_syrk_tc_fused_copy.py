"""The tensor SYRK copies the digit planes K-major itself: copier warps of every CTA write the (64-row band, 128-column
block) units a launch's MMAs read, and stamp per-unit readiness flags with a per-launch epoch. Pinned bit for bit to the
exact integer reference of test_gpu_syrk_tc.py: many launches on one context (stale flags of an earlier launch must not
pass for ready), an evaluation after a re-registration of another shape, grids smaller than the SM count (few CTAs copy
everything), trailing empty k-splits and short last bands, in both item shapes; and the copiers' trace counts every
plane tile copied.
"""
import numpy as np
import pytest

import scenes
from test_gpu_syrk_tc import (KS, TILE, _close_contexts, _lib, _ptr, check_product, ldg_of, pad_rows,  # noqa: F401
                              random_case, run_syrk, syrk_reference)

COPY_WORDS = 3


def _ctx(n_poses, monkeypatch, tile=None, trace=False):
    import balm_b200
    if tile is None:
        monkeypatch.delenv("BALM_TC_TILE", raising=False)
    else:
        monkeypatch.setenv("BALM_TC_TILE", tile)
    if trace:
        monkeypatch.setenv("BALM_TC_TRACE", "1")
    else:
        monkeypatch.delenv("BALM_TC_TRACE", raising=False)
    return balm_b200.Context(n_poses, 0, balm_b200.PREC_TENSOR)


def _syrk(c, q, rows, isc, splits):
    L = _lib()
    nb = q.shape[2] // TILE
    part = np.full((splits, nb * (nb + 1) // 2, TILE, TILE), np.nan)
    planes = np.ascontiguousarray(q[:, :rows], dtype=np.int8)
    isc = np.ascontiguousarray(isc, dtype=np.float64)
    st = L.lib().balm_debug_syrk_tc(c._h, _ptr(planes), len(q), rows, _ptr(isc), splits, 0, _ptr(part))
    assert st == 0, L.lib().balm_last_error()
    return part


@pytest.mark.gpu
def test_plane_sets_back_to_back_on_one_context():
    """Launch after launch on one context's stream, with different planes, plane counts and row counts: each must see
    its own copy, never a unit an earlier launch left behind."""
    n_poses = 130
    rng = np.random.default_rng(1200)
    for k, (S, rows, splits) in enumerate([(3, 64 * 9, 3), (3, 64 * 9, 3), (2, 64 * 6 - 5, 2), (4, 64 * 9, 3),
                                           (3, 64 * 2 + 1, 1), (2, 64 * 9, 3)]):
        q, isc = random_case(rng, n_poses, S, rows)
        st, part = run_syrk(n_poses, q, rows, isc, splits)
        assert st == 0, _lib().lib().balm_last_error()
        assert np.array_equal(part, syrk_reference(q, isc, splits)), k


@pytest.mark.gpu
def test_evaluation_after_reregistration_of_another_shape(monkeypatch):
    c = _ctx(60, monkeypatch)
    try:
        for kw in (dict(n_poses=60, n_planes=900, drop=0.5, seed=61), dict(n_poses=60, n_planes=250, seed=62),
                   dict(n_poses=60, n_planes=1400, drop=0.7, seed=63)):
            sc = scenes.make_scene(**kw)
            c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
            H, _, _ = c.evaluate(sc["poses_init"])
            check_product(c, sc, H, c.M)
    finally:
        c.close()


# (n_poses, rows, splits): one tile in two splits; three tiles with trailing empty k-splits; few items with a short
# last band
SMALL = [(12, 64 * 5 - 3, 2), (22, 64 * 2 + 7, 6), (22, 64 * 3, 5), (40, 64 * 4 - 1, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("tile", ["full", "half"])
@pytest.mark.parametrize("S", [2, 3, 4])
def test_small_grids_and_empty_splits(S, tile, monkeypatch):
    c = _ctx(40, monkeypatch, tile=tile)
    try:
        rng = np.random.default_rng(1300 + S)
        for n_poses, rows, splits in SMALL:
            if ldg_of(n_poses) != ldg_of(40):  # the hook uses the context's column count
                continue
            q, isc = random_case(rng, n_poses, S, rows)
            assert np.array_equal(_syrk(c, q, rows, isc, splits), syrk_reference(q, isc, splits))
    finally:
        c.close()
    for n_poses, rows, splits in SMALL:
        if ldg_of(n_poses) == ldg_of(40):
            continue
        c = _ctx(n_poses, monkeypatch, tile=tile)
        try:
            rng = np.random.default_rng(1400 + S + n_poses)
            q, isc = random_case(rng, n_poses, S, rows)
            assert np.array_equal(_syrk(c, q, rows, isc, splits), syrk_reference(q, isc, splits))
        finally:
            c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("S", [2, 3, 4])
def test_copy_trace_counts_every_plane_tile(S, monkeypatch):
    L = _lib()
    n_poses, rows, splits = 200, 64 * 7 * 2 - 9, 2
    rng = np.random.default_rng(1500 + S)
    q, isc = random_case(rng, n_poses, S, rows)
    st, plain = run_syrk(n_poses, q, rows, isc, splits)
    assert st == 0
    c = _ctx(n_poses, monkeypatch, trace=True)
    try:
        traced = _syrk(c, q, rows, isc, splits)
        buf = np.zeros(COPY_WORDS * 1024, dtype=np.uint64)
        L.check(L.lib().balm_debug_tc_copy_trace(c._h, _ptr(buf), len(buf)))
    finally:
        c.close()
    assert np.array_equal(plain, syrk_reference(q, isc, splits))
    assert np.array_equal(traced, plain)
    tr = buf.reshape(-1, COPY_WORDS).astype(np.int64)
    nb = ldg_of(n_poses) // TILE
    assert tr[:, 2].sum() == S * (pad_rows(rows) // KS) * nb
    assert (tr[:, 1] <= tr[:, 0]).all() and tr[:, 0].sum() > 0

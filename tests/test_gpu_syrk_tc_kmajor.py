"""The tensor SYRK's two item shapes: whole 128 x 128 tiles (m64n128 wgmma, taken at S <= 3 when every SM gets an item)
and 128 x 64 column halves, both fed from the K-major copy of the digit planes (tc_kmajor_kernel). BALM_TC_TILE=full|half
forces one at context creation. Both must give the exact integer reference's bits, at the shapes where the whole tiles
are the default (more (tile, k-split) pairs than SMs) and with padding columns, padding rows, several splits and
accumulation; an evaluation's H must not depend on the choice; and the trace counts stages in half-tile units.
"""
import numpy as np
import pytest

import scenes
from test_gpu_syrk_tc import (KS, TILE, _lib, _ptr, item_ranges, ldg_of, pad_rows, random_case,  # noqa: F401
                              syrk_reference)

TRACE_WORDS = 18


def _ctx(n_poses, tile, monkeypatch, trace=False):
    import balm_b200
    monkeypatch.setenv("BALM_TC_TILE", tile)
    if trace:
        monkeypatch.setenv("BALM_TC_TRACE", "1")
    else:
        monkeypatch.delenv("BALM_TC_TRACE", raising=False)
    return balm_b200.Context(n_poses, 0, balm_b200.PREC_TENSOR)


def _syrk(c, q, rows, isc, splits, accumulate=0, part=None):
    L = _lib()
    nb = q.shape[2] // TILE
    if part is None:
        part = np.full((splits, nb * (nb + 1) // 2, TILE, TILE), np.nan)
    planes = np.ascontiguousarray(q[:, :rows], dtype=np.int8)
    isc = np.ascontiguousarray(isc, dtype=np.float64)
    st = L.lib().balm_debug_syrk_tc(c._h, _ptr(planes), len(q), rows, _ptr(isc), splits, accumulate, _ptr(part))
    assert st == 0, L.lib().balm_last_error()
    return part


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# (n_poses, rows, splits): nb (nb + 1) / 2 tiles x splits >= 132 whole-tile items, live columns 6N < ldg, rows not a
# multiple of 64
SHAPES = [(130, 64 * 3 * 5 - 7, 5), (300, 64 * 5 * 2 - 1, 2), (200, 64 * 4 * 3 + 5, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("S", [2, 3])
@pytest.mark.parametrize("n_poses,rows,splits", SHAPES)
def test_whole_tiles_match_halves_and_reference(S, n_poses, rows, splits, monkeypatch):
    nb = ldg_of(n_poses) // TILE
    assert nb * (nb + 1) // 2 * splits >= _sms() and 6 * n_poses < ldg_of(n_poses)
    rng = np.random.default_rng(900 + 10 * S + n_poses)
    q, isc = random_case(rng, n_poses, S, rows)
    ref = syrk_reference(q, isc, splits)
    out = {}
    for tile in ("full", "half"):
        c = _ctx(n_poses, tile, monkeypatch)
        try:
            out[tile] = _syrk(c, q, rows, isc, splits)
        finally:
            c.close()
    assert np.array_equal(out["full"], ref)
    assert np.array_equal(out["half"], ref)


@pytest.mark.gpu
@pytest.mark.parametrize("S", [2, 3])
def test_whole_tiles_accumulate(S, monkeypatch):
    n_poses, splits = 130, 5
    rng = np.random.default_rng(950 + S)
    qa, isc = random_case(rng, n_poses, S, 700)
    qb, _ = random_case(rng, n_poses, S, 300)
    ref_a = syrk_reference(qa, isc, splits)
    for tile in ("full", "half"):
        c = _ctx(n_poses, tile, monkeypatch)
        try:
            pa = _syrk(c, qa, 700, isc, splits, part=np.full_like(ref_a, -7.0))
            assert np.array_equal(pa, ref_a), tile
            pab = _syrk(c, qb, 300, isc, splits, accumulate=1, part=pa.copy())
            assert np.array_equal(pab, syrk_reference(qb, isc, splits, old=ref_a)), tile
        finally:
            c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("slices", [None, 3], ids=["device", "S3"])
def test_evaluation_hessian_is_the_same_under_both_tile_modes(slices, monkeypatch):
    if slices is None:
        monkeypatch.delenv("BALM_TC_SLICES", raising=False)
    else:
        monkeypatch.setenv("BALM_TC_SLICES", str(slices))
    sc = scenes.make_scene(n_poses=200, n_planes=1100, drop=0.8, seed=52)
    res = {}
    for tile in ("full", "half"):
        c = _ctx(sc["n_poses"], tile, monkeypatch)
        try:
            c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
            res[tile] = c.evaluate(sc["poses_init"])
        finally:
            c.close()
    for a, b in zip(res["full"], res["half"]):
        assert np.array_equal(np.asarray(a), np.asarray(b))


@pytest.mark.gpu
def test_traced_whole_tiles_count_half_tile_stages(monkeypatch):
    L = _lib()
    n_poses, rows, splits, S = 130, 64 * 3 * 5 - 7, 5, 3
    rng = np.random.default_rng(990)
    q, isc = random_case(rng, n_poses, S, rows)
    c = _ctx(n_poses, "full", monkeypatch, trace=True)
    try:
        part = _syrk(c, q, rows, isc, splits)
        buf = np.zeros(TRACE_WORDS * 1024, dtype=np.uint64)
        L.check(L.lib().balm_debug_tc_trace(c._h, _ptr(buf), len(buf)))
    finally:
        c.close()
    assert np.array_equal(part, syrk_reference(q, isc, splits))
    tr = buf.reshape(-1, TRACE_WORDS).astype(np.int64)
    nb = ldg_of(n_poses) // TILE
    _, ranges = item_ranges(pad_rows(rows), splits)
    assert tr[:, 0].sum() == nb * (nb + 1) * sum((k1 - k0) // KS for k0, k1 in ranges)
    grid = min(nb * (nb + 1) // 2 * splits, _sms())
    live = tr[:grid]
    assert (live[:, 0] % 2 == 0).all()  # a whole-tile stage counts two half-tile units
    assert (live[:, 7] > 0).all() and (live[:, 12] > 0).all()
    assert not tr[:, 13:16].any()

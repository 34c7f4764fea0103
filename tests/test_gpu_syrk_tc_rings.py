"""The tensor-core SYRK's three shared-memory rings (A, B and the K-major copies BT of B), pinned bit for bit to the exact
integer reference of test_gpu_syrk_tc.py at the row counts where items end at every slot and parity of every ring, with
many items per CTA so that the rings wrap across a CTA's consecutive items, and with the per-role clock trace
(BALM_TC_TRACE) on: the traced instantiation computes the same bits and counts every stage.
"""
import math

import numpy as np
import pytest

# _close_contexts: the autouse fixture that closes run_syrk's cached contexts at the end of this module too
from test_gpu_syrk_tc import (KS, SLICES, TILE, _close_contexts, _lib, _ptr, check_syrk, item_ranges,  # noqa: F401
                              ldg_of, pad_rows, random_case, run_syrk, syrk_reference)

# slots of the A, B and BT rings per digit-plane count (syrk_tc.cu, Rings<S>)
RINGS = {2: (6, 4, 4), 3: (4, 4, 4), 4: (4, 2, 4)}
TRACE_WORDS = 18


def ring_steps(S):
    """Steps per item around every ring's depth, plus the depths' least common multiple and twice that."""
    depths = RINGS[S]
    lcm = math.lcm(*depths)
    return sorted({n for d in depths for n in (d - 1, d, d + 1)} | {lcm, 2 * lcm})


def test_ring_steps_cover_every_depth():
    assert ring_steps(3) == [3, 4, 5, 8]
    assert ring_steps(4) == [1, 2, 3, 4, 5, 8]
    assert ring_steps(2) == [3, 4, 5, 6, 7, 12, 24]


@pytest.mark.gpu
@pytest.mark.parametrize("S", SLICES)
@pytest.mark.parametrize("splits", [1, 2, 3])
def test_rows_at_every_ring_depth(S, splits):
    """Every item gets exactly nsteps 64-row stages (rows = splits x 64 x nsteps), and one short last row."""
    n_poses = 22
    rng = np.random.default_rng(500 + 10 * S + splits)
    for nsteps in ring_steps(S):
        for rows in (splits * KS * nsteps, splits * KS * nsteps - 1):
            q, isc = random_case(rng, n_poses, S, rows)
            check_syrk(n_poses, q, rows, isc, splits)


@pytest.mark.gpu
@pytest.mark.parametrize("S", SLICES)
@pytest.mark.parametrize("nsteps", [1, 2, 3, 5, 7])
def test_rings_wrap_across_items(S, nsteps):
    """120 tiles x 2 halves x 3 splits = 720 items on at most 132 SMs: each CTA runs 5-6 items back to back, whose
    first stages sit at whatever slot and parity the previous item left every ring in."""
    import torch
    n_poses, splits = 300, 3
    nb = ldg_of(n_poses) // TILE
    assert nb * (nb + 1) * splits > torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(600 + 10 * S + nsteps)
    rows = splits * KS * nsteps - 5
    q, isc = random_case(rng, n_poses, S, rows)
    check_syrk(n_poses, q, rows, isc, splits)


def _traced_ctx(n_poses, monkeypatch):
    import balm_b200
    monkeypatch.setenv("BALM_TC_TRACE", "1")
    return balm_b200.Context(n_poses, 0, balm_b200.PREC_TENSOR)


def _trace(c):
    L = _lib()
    buf = np.zeros(TRACE_WORDS * 1024, dtype=np.uint64)
    L.check(L.lib().balm_debug_tc_trace(c._h, _ptr(buf), len(buf)))
    return buf.reshape(-1, TRACE_WORDS).astype(np.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("S", SLICES)
@pytest.mark.parametrize("n_poses,rows,splits", [(22, 64 * 13 - 3, 2), (200, 64 * 7 * 2, 2)])
def test_traced_kernel_is_bit_identical_and_counts_every_stage(S, n_poses, rows, splits, monkeypatch):
    import torch
    L = _lib()
    rng = np.random.default_rng(700 + S + n_poses)
    q, isc = random_case(rng, n_poses, S, rows)
    st, plain = run_syrk(n_poses, q, rows, isc, splits)
    assert st == 0
    assert np.array_equal(plain, syrk_reference(q, isc, splits))
    c = _traced_ctx(n_poses, monkeypatch)
    try:
        traced = np.full_like(plain, np.nan)
        planes = np.ascontiguousarray(q[:, :rows])
        isc_c = np.ascontiguousarray(isc)
        st = L.lib().balm_debug_syrk_tc(c._h, _ptr(planes), S, rows, _ptr(isc_c), splits, 0, _ptr(traced))
        assert st == 0, L.lib().balm_last_error()
        assert np.array_equal(traced, plain)
        tr = _trace(c)
    finally:
        c.close()
    nb = ldg_of(n_poses) // TILE
    items = nb * (nb + 1) * splits
    _, ranges = item_ranges(pad_rows(rows), splits)
    steps = nb * (nb + 1) * sum((k1 - k0) // KS for k0, k1 in ranges)  # both halves of every tile, every split
    assert tr[:, 0].sum() == steps
    grid = min(items, torch.cuda.get_device_properties(0).multi_processor_count)
    live = tr[:grid]
    assert (live[:, 7] > 0).all() and (live[:, 12] > 0).all()  # both consumer warpgroups ran
    assert (live[:, 2] >= live[:, 1]).all()
    for base, n in ((3, 4), (8, 4)):  # the consumers' categories add up to no more than their total
        assert (live[:, base:base + n].sum(axis=1) <= live[:, base + n]).all()
    assert not tr[grid:].any()  # CTAs beyond the grid record nothing


@pytest.mark.gpu
def test_trace_requires_the_variable(monkeypatch):
    import balm_b200
    L = _lib()
    monkeypatch.delenv("BALM_TC_TRACE", raising=False)
    c = balm_b200.Context(4, 0, balm_b200.PREC_TENSOR)
    try:
        buf = np.zeros(TRACE_WORDS, dtype=np.uint64)
        assert L.lib().balm_debug_tc_trace(c._h, _ptr(buf), len(buf)) == L.ERR_INVALID
    finally:
        c.close()

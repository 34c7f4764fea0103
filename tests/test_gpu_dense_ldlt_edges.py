"""The dense damped solve of ldlt.cu (tile-DAG LDL^T, grouped backward substitution, q1, backward-error check and fp64
refinement) at the edges of its grid, groups, tiles and loops, against references it cannot agree with by accident:

  * an exact integer system (L unit lower with entries in {0, +-1}, d_i = +-2^e), on which every intermediate of the
    solve is an integer below 2^53 and every division is by a power of two, so LD, dx, q1 and omega must come back
    bit for bit -- a tile read before its last update, or a skipped update, cannot hide behind refinement;
  * the pivot flag at sub-panel, tile and matrix ends, at the 1e-290 guard and on non-finite input;
  * Hessians of real BA problems against an extended-precision reference, with refinement required NOT to run;
  * refinement under negative damping, where it must run, and is counted once per refined solve.

Caller-supplied systems go through balm_debug_ldlt, which runs balm_solve's own path on scratch buffers."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.linalg as sla

import balm_b200
import nd_symbolic_ref as nd
from balm_b200 import _lib as L

EPS = np.finfo(np.float64).eps
T = 64          # ldlt.cu's tile (BALM_NB) and the chain's step
SUB = 16        # diag_factor's sub-panel
NEAR_ROWS = 4   # dag::NEAR_ROWS: rows k+2 .. k+1+NEAR_ROWS of step k go to the near group
BACK_GROUP = 4  # tile rows per ldl_back_kernel launch
Q1_THREADS = 1024


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def debug_ldlt(c, H, g, u, want_LD=True):
    """balm_debug_ldlt -> (dx, q1, not_pd, LD or None, omega)"""
    H = np.asfortranarray(H, dtype=np.float64)
    g = np.ascontiguousarray(g, dtype=np.float64)
    dx = np.zeros(c.n)
    LD = np.zeros((c.n, c.n), order="F") if want_LD else None
    q1, bad, om = C.c_double(), C.c_int(), C.c_double()
    L.check(L.lib().balm_debug_ldlt(c._h, _p(H), _p(g), float(u), _p(dx), C.byref(q1), C.byref(bad), _p(LD),
                                    C.byref(om)))
    return dx, q1.value, bool(bad.value), LD, om.value


# ---------------------------------------------------------------------------------------------------------------------
# the grid: a host restatement of enqueue_solve_dag's launch and ldl_dag_kernel's dealing

def layout(N, sm_count):
    """What a solve of order n = 6N reaches on a device of sm_count SMs."""
    n = 6 * N
    nt = -(-n // T)
    last = n - (nt - 1) * T
    grid = 1 if nt < 2 else sm_count
    workers = grid - 1
    near = 8 if workers >= 16 else 0
    split = near > 0 and workers - near > 0
    near_tasks = far_tasks = far_rounds = 0
    for k in range(nt - 1):
        r_split = min(k + 2 + NEAR_ROWS, nt) if split else nt
        near_tasks += sum(1 + r - k for r in range(k + 2, r_split))
        step_far = (nt - r_split) + sum(r - k for r in range(r_split, nt))
        far_tasks += step_far
        if step_far:
            far_rounds = max(far_rounds, -(-step_far // (workers - near)))
    return dict(n=n, nt=nt, last=last, last_subpanels=-(-last // SUB), grid=grid, near=near, split=split,
                near_tasks=near_tasks, far_tasks=far_tasks, far_rounds=far_rounds, back_last=nt % BACK_GROUP or BACK_GROUP,
                q1_loops=n > Q1_THREADS)


# N -> (the edge it is there for, the layout that shows it is reached)
SIZES = {
    1: ("one-CTA grid, last tile 6: 1 sub-panel", lambda l: l["grid"] == 1 and l["last_subpanels"] == 1),
    3: ("one-CTA grid, last tile 18: 2 sub-panels", lambda l: l["grid"] == 1 and l["last_subpanels"] == 2),
    8: ("one-CTA grid, last tile 48: 3 sub-panels", lambda l: l["grid"] == 1 and l["last_subpanels"] == 3),
    10: ("one-CTA grid, last tile 60: 4 sub-panels", lambda l: l["grid"] == 1 and l["last"] == 60),
    11: ("chain only, workers idle, last tile 2", lambda l: l["nt"] == 2 and l["grid"] > 1 and l["last"] == 2 and
         l["near_tasks"] == l["far_tasks"] == 0),
    21: ("chain only, workers idle, last tile 62", lambda l: l["nt"] == 2 and l["grid"] > 1 and l["last"] == 62 and
         l["near_tasks"] == l["far_tasks"] == 0),
    32: ("first worker tasks: P(2,0), U(2,1,0), U(2,2,0)", lambda l: l["nt"] == 3 and l["last"] == T and
         l["near_tasks"] == 3 and l["far_tasks"] == 0),
    42: ("npan mod 4 = 0", lambda l: l["nt"] == 4 and l["back_last"] == 4 and l["last"] == 60),
    64: ("largest near-only", lambda l: l["nt"] == 2 + NEAR_ROWS and l["far_tasks"] == 0 and l["last"] == T),
    65: ("first far-group rows: P(6,0), U(6,1..6,0)", lambda l: l["nt"] == 3 + NEAR_ROWS and l["far_tasks"] == 7 and
         l["last"] == 6),
    80: ("far group, npan mod 4 = 0", lambda l: l["nt"] == 8 and l["far_tasks"] > 0 and l["back_last"] == 4 and
         l["last"] == 32),
    171: ("q1 loop (n > 1024), last tile 2", lambda l: l["q1_loops"] and l["nt"] == 17 and l["last"] == 2),
    200: ("C2", lambda l: l["nt"] == 19 and l["last"] == 48 and l["far_rounds"] > 1),
    500: ("the benchmark (C3)", lambda l: l["nt"] == 47 and l["last"] == 56 and l["far_rounds"] > 1),
    512: ("full tiles at benchmark scale", lambda l: l["nt"] == 48 and l["last"] == T),
    1000: ("beyond the benchmark, many rounds of dealing", lambda l: l["nt"] == 94 and l["last"] == 48 and
           l["far_rounds"] >= 20),
}


@pytest.mark.parametrize("sm_count", [17, 78, 114, 132, 148])
def test_sizes_reach_their_edges(sm_count):
    """Every size's edge holds on any device with at least 17 SMs. With fewer, near_ctas = 0 and one group takes every
    row; no H100 has so few SMs, so that dealing is not exercised here."""
    for N in SIZES:
        lay = layout(N, sm_count)
        assert SIZES[N][1](lay), (N, SIZES[N][0], lay)
    assert layout(64, sm_count)["near_tasks"] > layout(42, sm_count)["near_tasks"]
    assert layout(65, sm_count)["split"] and layout(65, sm_count)["near"] == 8
    # the sizes together cover every sub-panel count of the last tile and every size of the last backward group
    assert {layout(N, sm_count)["last_subpanels"] for N in SIZES} == {1, 2, 3, 4}
    assert {layout(N, sm_count)["back_last"] for N in SIZES} == {1, 2, 3, 4}


# ---------------------------------------------------------------------------------------------------------------------
# the exact integer reference

def integer_factor(N, seed, negative=False):
    """L unit lower triangular, entries in {0, +-1}: sparse (1/32) strictly below the diagonal inside each 64 x 64
    diagonal block, dense (1/2) in the blocks below it; d_i = +-2^e, e in [2, 8]."""
    n = 6 * N
    rng = np.random.default_rng(seed)
    R = rng.random((n, n))
    Lm = np.where(R < 1 / 4, 1.0, np.where(R < 1 / 2, -1.0, 0.0))
    for k0 in range(0, n, T):
        Rb = R[k0:k0 + T, k0:k0 + T]
        Lm[k0:k0 + T, k0:k0 + T] = np.where(Rb < 1 / 64, 1.0, np.where(Rb < 1 / 32, -1.0, 0.0))
    Lm = np.tril(Lm, -1)
    Lm[np.diag_indices(n)] = 1.0
    d = 2.0 ** rng.integers(2, 9, size=n)
    if negative:
        d[rng.random(n) < 0.25] *= -1
    x = rng.integers(-8, 9, size=n).astype(np.float64)
    return Lm, d, x


def exact_bounds(Lm, d, A, x):
    """Assert the bounds under which every quantity the device forms is an integer below 2^53, so that the solve is
    exact in fp64 whatever the order of its sums: every Schur complement entry S_ij = sum_{m >= k} L_im d_m L_jm is at
    most sqrt(B_ii B_jj) <= max_i B_ii, B_ii = sum_m L_im^2 |d_m|; the inverses X = L_kk^-1 of the diagonal blocks
    (their 16 x 16 diagonal blocks are diag_factor's inverses) are integers; W = S X^T sums at most n terms of
    |S| |X|; y = D L^T x and w = L^T x, and the residual and q1 sums, are bounded by |A| |x|. -> (max|A|, max|X|)"""
    n = len(d)
    xmax = 0.0
    for k0 in range(0, n, T):
        Lkk = Lm[k0:k0 + T, k0:k0 + T]
        X = sla.solve_triangular(Lkk, np.eye(len(Lkk)), lower=True, unit_diagonal=True)
        assert np.array_equal(X, np.round(X))
        xmax = max(xmax, np.abs(X).max())
    schur = ((Lm * Lm) @ np.abs(d)).max()
    amax = np.abs(A).max()
    limit = 2.0 ** 53
    assert amax <= schur < limit / n
    assert n * schur * xmax < limit                                   # sum |S| |X| over a row: W = S X^T, X assembly
    assert (np.abs(A) @ np.full(n, xmax)).max() < limit
    assert n * 8 * ((np.abs(A) @ np.abs(x)).max() + 3 * 8 * amax) < limit  # g, the residual check and q1 (u <= 3)
    assert np.abs(d).max() * (np.abs(Lm).T @ np.abs(x)).max() * n < limit  # y, w and their partial sums
    return amax, xmax


def integer_system(N, seed, negative=False):
    Lm, d, x = integer_factor(N, seed, negative)
    A = (Lm * d) @ Lm.T
    amax, xmax = exact_bounds(Lm, d, A, x)
    return Lm, d, x, A, -(A @ x), amax, xmax


def damped_input(A, u):
    """H with H + u diag(H) = A: diag(A) is a multiple of 4, so diag(A) / (1 + u) is exact for u = 0, 1, 3."""
    H = A.copy()
    H[np.diag_indices(len(A))] = np.diag(A) / (1 + u)
    assert np.array_equal(np.diag(H) * (1 + u), np.diag(A))
    return H


def exact_q1(H, g, x, u):
    """0.5 x . (u diag(H) x - g) in integers"""
    xi = x.astype(np.int64)
    s = int(np.sum(xi * (np.round(u * np.diag(H)).astype(np.int64) * xi - g.astype(np.int64))))
    assert abs(s) < 2 ** 53
    return 0.5 * s


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _solve_bits(out):
    dx, q1, bad, LD, om = out
    return dx.tobytes(), q1, bad, None if LD is None else LD.tobytes(), om


@pytest.mark.gpu
@pytest.mark.parametrize("N", list(SIZES))
def test_integer_system_bit_for_bit(N):
    """LD, dx, q1 and omega exactly, with no refinement: undamped, with u = 1 and 3 (diag(H) damped on the device),
    indefinite, repeated, on a second context and in the BALM_DAG_TRACE instantiation."""
    lay = layout(N, _sm_count())
    assert SIZES[N][1](lay), (N, SIZES[N][0], lay)
    c, c2 = balm_b200.Context(N, 0, 0), balm_b200.Context(N, 0, 0)
    for negative in (False, True):
        Lm, d, x, A, g, amax, xmax = integer_system(N, seed=N, negative=negative)
        LDref = np.tril(Lm, -1) + np.diag(d)
        print(f"N {N} ({SIZES[N][0]}){' indefinite' if negative else ''}: max|A| {amax:.3g}, max|X| {xmax:g}")
        for u in ((0.0,) if negative else (0.0, 1.0, 3.0)):
            H = damped_input(A, u)
            c.reset_counters()
            out = debug_ldlt(c, H, g, u)
            dx, q1, bad, LD, om = out
            assert not bad and c.timings()["refinements"] == 0, (N, u)
            assert np.array_equal(LD, LDref), (N, u, np.argwhere(LD != LDref)[:4])
            assert np.array_equal(dx, x), (N, u)
            assert q1 == exact_q1(H, g, x, u), (N, u)
            assert om == 0.0, (N, u)
            # repeatable: the same call again, and on another context
            assert _solve_bits(debug_ldlt(c, H, g, u)) == _solve_bits(out)
            assert _solve_bits(debug_ldlt(c2, H, g, u)) == _solve_bits(out)
    # the BALM_DAG_TRACE instantiation: the workspaces read the variable when they are allocated, which for
    # balm_debug_ldlt is every call (test_ba_hessians_against_extended_precision reads back a traced context's clock)
    os.environ["BALM_DAG_TRACE"] = "1"
    try:
        traced = debug_ldlt(c2, H, g, 0.0)
    finally:
        del os.environ["BALM_DAG_TRACE"]
    assert _solve_bits(traced) == _solve_bits(debug_ldlt(c, H, g, 0.0))
    c.close()
    c2.close()


def isolated_pivot(Lm, d, x, j, dj):
    """The integer system with row and column j of L zero off the diagonal and d_j = dj: pivot j is dj whatever the
    order of the sums, and 1 / dj is finite down to 2^-1022, so dx stays x* even when the pivot is flagged."""
    Lm, d = Lm.copy(), d.copy()
    Lm[j, :j] = 0.0
    Lm[j + 1:, j] = 0.0
    d[j] = dj
    A = (Lm * d) @ Lm.T
    exact_bounds(Lm, d, A, x)
    assert A[j, j] == dj and np.count_nonzero(A[j]) == 1
    return Lm, d, A, -(A @ x)


PIVOT_POSITIONS = (0, 15, 16, 47, 63, 64, 64 * 20 + 33, 2944, 2999)  # of n = 3000: sub-panel, tile and matrix ends


@pytest.mark.gpu
def test_zero_pivot_flag_at_every_position():
    """At sub-panel and tile starts and ends, mid-matrix, in the short last tile and in the last column of the
    benchmark's n = 3000: d_j = 0 is flagged and not refined; an isolated pivot d_j = 2^-964, below the |d| > 1e-290
    guard, is flagged with dx = x* and a finite q1, so the pivot flag is the only reason for not_pd; and the next clean
    solve on the context is exact again."""
    N = 500
    c = balm_b200.Context(N, 0, 0)
    Lm, d, x, A, g, _, _ = integer_system(N, seed=7)
    for j in PIVOT_POSITIONS:
        Aj = A - d[j] * np.outer(Lm[:, j], Lm[:, j])   # the same L with d_j = 0 (exact: integers)
        c.reset_counters()
        dx, q1, bad, _, _ = debug_ldlt(c, Aj, -(Aj @ x), 0.0, want_LD=False)
        assert bad and c.timings()["refinements"] == 0, j
        _, _, Ai, gi = isolated_pivot(Lm, d, x, j, 2.0 ** -964)
        dx, q1, bad, _, _ = debug_ldlt(c, Ai, gi, 0.0, want_LD=False)
        assert bad and c.timings()["refinements"] == 0, j
        # row j's term 2^-964 x_j^2 vanishes when q1 is rounded: the fp64 sum of the terms, not the exact one
        assert np.array_equal(dx, x) and np.isfinite(q1) and q1 == 0.5 * np.sum(x * -gi), j
        dx, q1, bad, _, om = debug_ldlt(c, A, g, 0.0, want_LD=False)
        assert not bad and np.array_equal(dx, x) and q1 == exact_q1(A, g, x, 0.0) and om == 0.0, j
    c.close()


@pytest.mark.gpu
def test_pivot_guard_and_non_finite_input():
    """An isolated pivot just below the |d| > 1e-290 guard is flagged; 16 times larger it is solved exactly. A NaN or
    an Inf in one symmetric off-diagonal pair is flagged."""
    N = 500
    j = 64 * 20 + 33
    c = balm_b200.Context(N, 0, 0)
    L0, d0, x = integer_factor(N, seed=8)
    for e, flagged in ((-964, True), (-960, False)):
        assert (2.0 ** e <= 1e-290) == flagged
        Lm, d, A, g = isolated_pivot(L0, d0, x, j, 2.0 ** e)
        c.reset_counters()
        dx, q1, bad, LD, om = debug_ldlt(c, A, g, 0.0)
        assert bad == flagged and c.timings()["refinements"] == 0, e
        if not flagged:
            assert np.array_equal(dx, x) and om == 0.0
            assert np.array_equal(LD, np.tril(Lm, -1) + np.diag(d))
            assert q1 == 0.5 * np.sum(x * -g)
    Lm, d, x, A, g, _, _ = integer_system(65, seed=9)
    c.close()
    c = balm_b200.Context(65, 0, 0)
    for bad_value in (np.nan, np.inf):
        Ab = A.copy()
        Ab[300, 17] = Ab[17, 300] = bad_value
        c.reset_counters()
        assert debug_ldlt(c, Ab, g, 0.0, want_LD=False)[2] and c.timings()["refinements"] == 0, bad_value
    assert np.array_equal(debug_ldlt(c, A, g, 0.0, want_LD=False)[0], x)
    c.close()


@pytest.mark.gpu
def test_debug_ldlt_refuses_bad_arguments():
    c = balm_b200.Context(4, 0, 0)
    with pytest.raises(balm_b200.BalmError) as e:
        L.check(L.lib().balm_debug_ldlt(c._h, None, None, 0.0, None, None, None, None, None))
    assert e.value.status == L.ERR_INVALID
    c.close()
    b = balm_b200.Context(4, 0, L.PREC_BLOCKS)
    with pytest.raises(balm_b200.BalmError) as e:
        debug_ldlt(b, np.eye(24), np.ones(24), 0.0)
    assert e.value.status == L.ERR_INVALID
    b.close()


# ---------------------------------------------------------------------------------------------------------------------
# real BA Hessians against an extended-precision reference

def reference_solve(A, b):
    """LU in fp64, then three rounds of refinement with the residual formed in long double"""
    lu = sla.lu_factor(A)
    x = sla.lu_solve(lu, b)
    Ald, bld = np.asarray(A, np.longdouble), np.asarray(b, np.longdouble)
    for _ in range(3):
        x = x + sla.lu_solve(lu, (bld - Ald @ np.asarray(x, np.longdouble)).astype(np.float64))
    return x


def backward_error(A, b, x):
    """componentwise, the residual in long double"""
    r = np.abs(np.asarray(b, np.longdouble) - np.asarray(A, np.longdouble) @ np.asarray(x, np.longdouble))
    den = np.abs(A) @ np.abs(x) + np.abs(b)
    return float(np.max(np.where(den > 0, r.astype(np.float64) / np.where(den > 0, den, 1.0), 0.0)))


def scaled_eigenvalues(H):
    """eigenvalues of D^-1/2 H D^-1/2, D = diag(H): those of the damped system's scaling are these + u"""
    s = 1.0 / np.sqrt(np.abs(np.diag(H)))
    return np.linalg.eigvalsh(H * s[:, None] * s[None, :])


def check_solve(H, g, u, lam, dx, q1, what):
    """The contract of one unflagged solve -> (omega, forward error over its bound). Unpivoted LDL^T is invariant under
    diagonal scaling, so the forward error is measured in the D^1/2-scaled norm against kappa of the scaled matrix."""
    D = np.diag(H).copy()
    A = H + u * np.diag(D)
    ref = reference_solve(A, -g)
    omega = backward_error(A, -g, dx)
    kappa = np.abs(lam + u).max() / np.abs(lam + u).min()
    s = np.sqrt(np.abs(np.diag(A)))
    fwd = np.linalg.norm(s * (dx - ref)) / np.linalg.norm(s * ref)
    ratio = fwd / (20 * kappa * EPS)
    terms = 0.5 * dx * (u * D * dx - g)
    print(f"{what}: omega {omega:.1e}, forward {fwd:.1e} = {ratio:.2e} of 20 kappa_D eps (kappa_D {kappa:.1e})")
    assert omega <= 2e-12, what
    assert ratio <= 1.0, what
    assert abs(q1 - terms.sum()) <= 1e-12 * np.abs(terms).sum(), what
    return omega, ratio


def chain_trace(c):
    """balm_debug_dag_trace: the chain's [nt][4] timestamps of the context's last factorisation, None without a trace"""
    nt = -(-c.n // T)
    buf = np.zeros(4 * nt, dtype=np.uint64)
    rc = L.lib().balm_debug_dag_trace(c._h, _p(buf), C.c_int(len(buf)))
    if rc == L.ERR_INVALID:
        return None
    L.check(rc)
    return buf.reshape(nt, 4)


def ba_context(N, voxels, seed):
    c = balm_b200.Context(N, 0, 0)
    gt, _ = c.synth_virtual(voxels, seed=seed)
    return c, gt


BA_SIZES = {3: 400, 11: 600, 65: 1000, 130: 1500, 200: 2000, 500: 3000}


@pytest.mark.gpu
@pytest.mark.parametrize("N", list(BA_SIZES))
def test_ba_hessians_against_extended_precision(N):
    """H and g of balm_evaluate at the ground truth (PSD, with the gauge null space), damped by u = 1 .. 1e-6: the
    solve is not refined, its backward error is at rounding level and its forward error within 20 kappa_D eps; repeated
    solves and a context whose first solve ran the BALM_DAG_TRACE instantiation give the same bits."""
    c, gt = ba_context(N, BA_SIZES[N], seed=N)
    H, g, _ = c.evaluate(gt)
    os.environ["BALM_DAG_TRACE"] = "1"
    try:
        ct, gt_t = ba_context(N, BA_SIZES[N], seed=N)
        Ht, gt_g, _ = ct.evaluate(gt_t)
        traced_first = ct.solve(1e-2)
    finally:
        del os.environ["BALM_DAG_TRACE"]
    assert np.array_equal(Ht, H) and np.array_equal(gt_g, g)
    # ct's factorisation took the traced branches (every chain step stamped its start and its publication, in order);
    # c's has no trace buffer at all
    tr = chain_trace(ct)
    assert tr is not None and (tr[:, 0] > 0).all() and (tr[:, 3] >= tr[:, 0]).all() and (tr[1:, 0] >= tr[:-1, 3]).all()
    assert (tr[1:, 1:3] > 0).all() and chain_trace(c) is None
    lam = scaled_eigenvalues(H)
    worst = (0.0, 0.0)
    for u in (1.0, 1e-2, 1e-4, 1e-6):
        c.reset_counters()
        dx, q1, bad = c.solve(u)
        assert not bad and c.timings()["refinements"] == 0, u
        om, ratio = check_solve(H, g, u, lam, dx, q1, f"N {N} u {u:g}")
        worst = (max(worst[0], om), max(worst[1], ratio))
        again = c.solve(u)
        assert np.array_equal(again[0], dx) and again[1:] == (q1, bad)
        traced = ct.solve(u)
        assert np.array_equal(traced[0], dx) and traced[1:] == (q1, bad)
        if u == 1e-2:
            assert np.array_equal(traced_first[0], dx) and traced_first[1:] == (q1, bad)
    print(f"N {N}: worst omega {worst[0]:.1e}, worst forward error / bound {worst[1]:.2e}")
    c.close()
    ct.close()


# ---------------------------------------------------------------------------------------------------------------------
# refinement on the dense path

def leading_minor_crossing(H, poses):
    """A damping u in (-0.95, -0.3) at which the leading principal minor of H + u diag(H) over the first `poses` poses is
    singular: u = -lam for the generalised eigenvalue lam of (H_k, D_k) nearest 0.6."""
    k = 6 * poses
    lam = sla.eigh(H[:k, :k], np.diag(np.diag(H)[:k]), eigvals_only=True)
    lam = lam[(lam > 0.3) & (lam < 0.95)]
    return -lam[np.argmin(np.abs(lam - 0.6))]


def refinement_rounds(n, launches):
    """The rounds of refine_solution a balm_solve ran, from the launches it counted (balm_timings.launches), with
    npan = 64-column panels and G = ceil(npan / 4) backward-substitution groups. The constants restate ldlt.cu's
    launch accounting and change with it: the solve counts 6 + G (enqueue_solve_dag: damp_copy, rhs_init and the
    cooperative factorisation; enqueue_back_substitution: scale_rhs, G ldl_back launches and q1; enqueue_solve_check:
    the residual), every refinement round 5 + npan + G (refine_solution: the copy and npan ldl_fwd_block launches,
    the back substitution without q1, axpy and q1, and the check)."""
    npan = -(-n // T)
    G = -(-npan // BACK_GROUP)
    rounds, rest = divmod(launches - (6 + G), 5 + npan + G)
    assert rest == 0 and 0 <= rounds <= 3, launches
    return rounds


@pytest.mark.gpu
def test_refinement_under_negative_damping():
    """H + u diag(H) with u < 0 is indefinite, and the LDL^T without pivoting may lose digits there; the backward-error
    check must catch it and refine, or flag the step. N = 65 reaches the far group and a multi-CTA forward substitution
    in refinement (m > 256 rows below the first block). A host emulation (the scalar LDL^T in the same order) predicts
    whether omega passes 1e-12: above 1e-11 the device must refine, below 1e-13 it must not. refinements counts refined
    solves, not rounds: at the exact crossing the pivot is rounding-sized, and the solve is flagged after three rounds."""
    N = 65
    c, gt = ba_context(N, 1000, seed=3)
    H, g, _ = c.evaluate(gt)
    n = len(g)
    D = np.diag(H).copy()
    lam = scaled_eigenvalues(H)
    dx0, q10, bad0 = c.solve(1e-3)
    cross = leading_minor_crossing(H, N // 2)
    us = list(np.linspace(-0.95, -0.3, 15)) + [cross * (1 + e) for e in (1e-6, 1e-7, 1e-8)] + [cross]
    c.reset_counters()
    refined_solves, refined_ok, rounds_seen = 0, [], []
    for u in us:
        before = c.timings()
        dx, q1, bad = c.solve(u)
        after = c.timings()
        n_ref = after["refinements"] - before["refinements"]
        rounds = refinement_rounds(n, after["launches"] - before["launches"])
        rounds_seen.append(rounds)
        A = H + u * np.diag(D)
        emulated, _ = nd.ldlt_backward_error(A, -g, range(N))
        print(f"u {u:.12f}: emulated omega {emulated:.1e}, rounds {rounds}, counted {n_ref}, flagged {bad}")
        assert n_ref == (1 if rounds else 0), u
        refined_solves += rounds > 0
        if emulated > 1e-11:
            assert rounds >= 1, u
        if emulated < 1e-13:
            assert rounds == 0, u
        if not bad and rounds:
            check_solve(H, g, u, lam, dx, q1, f"refined u {u:.12f}")
            refined_ok.append((emulated, u, q1))
    assert c.timings()["refinements"] == refined_solves
    assert rounds_seen[-1] == 3 and bad, "the exact crossing: three rounds, then flagged"
    assert refined_ok, "no solve refined and passed"
    # the LM loop takes the same route: the refined q1, bit for bit
    _, u, q1 = max(refined_ok)
    _, tr, _ = c.damping_iter(gt, max_iter=1, u0=u, rel_tol=-1, gauge_mode=2, min_planes_per_pose=0)
    assert not tr[0]["not_pd"] and tr[0]["q1"] == q1
    # balm_debug_ldlt leaves the context's system alone
    H2, g2, _ = c.evaluate(gt)
    assert np.array_equal(H2, H) and np.array_equal(g2, g)
    before = c.solve(1e-3)
    debug_ldlt(c, np.eye(n) * 4.0, np.ones(n), 0.0)
    after = c.solve(1e-3)
    assert np.array_equal(before[0], after[0]) and before[1:] == after[1:]
    assert np.array_equal(before[0], dx0) and before[1:] == (q10, bad0)
    c.close()

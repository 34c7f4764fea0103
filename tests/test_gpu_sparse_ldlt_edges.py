"""The nested-dissection block LDL^T of pose_graph_sparse.cu at the edges of its kernels' loops, against dense fp64
references: the damped solve (backward and forward error, q1, repeatability), its refinement under negative damping,
the selected inversion (block covariances) and one LM iteration, on pose-factor patterns chosen so that every loop of
spg_factor_kernel and spg_selinv_kernel wraps (or just does not), that a row of L is long and that the elimination tree
is deep. Which edge a pattern reaches is read from the host restatement nd_symbolic_ref, and the device's structure is
checked against it.

The solver is reached through a PREC_BLOCKS context with no voxels and the pattern's factors (evaluate gives the dense
H and g, solve(u) dx, q1 and the not-PD flag, timings()["refinements"] the refinements), and through a PoseGraph on the
same factors (its own LM and covariance route)."""
import numpy as np
import pytest
import scipy.linalg as sla

import balm_b200
import nd_symbolic_ref as nd
import pose_graph_ref as pgr
from balm_b200 import _lib as L
from test_gpu_sparse_covariance import _check_against, _dense_sigma

EPS = np.finfo(np.float64).eps
SP_THREADS, SEL_THREADS = 512, 256  # pose_graph_sparse.cu's block sizes


def _clique(n):
    """Factors whose union is the complete graph on n poses: one factor up to 32 poses (a factor's limit), above that
    one over every pair of 16-pose groups."""
    if n <= 32:
        return [list(range(n))]
    g = [list(range(a, min(a + 16, n))) for a in range(0, n, 16)]
    return [g[a] + g[b] for a in range(len(g)) for b in range(a + 1, len(g))]


def _band(P=400, w=32, stride=8):
    """HBA-like windows of w poses every stride poses, and two-pose loop closures (i, P - 1 - i) every 10 poses."""
    wins = [list(range(a, min(a + w, P))) for a in range(0, P - w + stride, stride)]
    return [s for s in wins if len(s) >= 2] + [[i, P - 1 - i] for i in range(0, P // 2, 10)]


def _grid(n=20):
    """Two-pose factors on the 4-neighbour edges of an n x n grid of poses (two-dimensional separators)."""
    return [[r * n + c, r * n + c + 1] for r in range(n) for c in range(n - 1)] + \
           [[r * n + c, (r + 1) * n + c] for r in range(n - 1) for c in range(n)]


PATTERNS = {f"clique{n}": (n, _clique(n)) for n in (16, 17, 33, 34, 43, 44, 86, 87)}
PATTERNS["star"] = (200, [[0, i] for i in range(1, 200)])  # a hub in 199 two-pose factors
PATTERNS.update({f"path{n}": (n, [[i, i + 1] for i in range(n - 1)]) for n in (2, 32, 33, 64, 65)})
PATTERNS["band"] = (400, _band())
PATTERNS["grid"] = (400, _grid())

# the loops the patterns must make wrap, as functions of the restatement (m = blocks below a column's diagonal)
EDGES = {
    "factor_warps": lambda s: s["m_max"] + 1 > SP_THREADS // 32,  # spg_factor_kernel: a column's blocks, a warp each
    "factor_lanes": lambda s: s["terms_max"] > 32,                 # a block's update terms, a lane each
    "factor_rows": lambda s: 6 * s["m_max"] > SP_THREADS,          # off-diagonal rows, a thread each
    "selinv_rows": lambda s: 6 * s["m_max"] > SEL_THREADS,         # spg_selinv_kernel: L^ rows, a thread each
    "selinv_warps": lambda s: s["m_max"] > SEL_THREADS // 32,      # Z blocks, a warp each
    "selinv_lanes": lambda s: s["m_max"] > 32,                     # Z terms and warp 0's diagonal sum, a lane each
    "long_row": lambda s: s["row_max"] > 128,                      # forward substitution over a row's blocks
    "deep_tree": lambda s: s["levels"] > 100,                      # one launch per level, each way
}
# clique pairs (n - 1 below a wrap, n at it)
STRADDLE = [(16, 17, "factor_warps"), (33, 34, "factor_lanes"), (33, 34, "selinv_lanes"), (43, 44, "selinv_rows"),
            (86, 87, "factor_rows")]


def _restatement(name):
    P, sets = PATTERNS[name]
    return nd.symbolic(P, nd.pairs_of(P, sets))


def test_the_patterns_reach_every_edge():
    sym = {name: _restatement(name) for name in PATTERNS}
    for edge, reached in EDGES.items():
        assert [n for n, s in sym.items() if reached(s)], edge
    # the cliques sit on both sides of every wrap: m = n - 1 and n - 1 update terms on the last diagonal block
    for n in (16, 17, 33, 34, 43, 44, 86, 87):
        s = sym[f"clique{n}"]
        assert (s["m_max"], s["terms_max"], s["l_blocks"], s["levels"]) == (n - 1, n - 1, n * (n + 1) // 2, n)
    for lo, hi, edge in STRADDLE:
        assert not EDGES[edge](sym[f"clique{lo}"]) and EDGES[edge](sym[f"clique{hi}"]), edge
    assert sym["star"]["row_max"] == sym["star"]["terms_max"] == 199 and sym["star"]["m_max"] == 1
    for name, s in sym.items():
        print(f"{name}: l_blocks {s['l_blocks']}, levels {s['levels']}, m_max {s['m_max']}, "
              f"terms_max {s['terms_max']}, row_max {s['row_max']}")


def _factors(name, seed):
    P, sets = PATTERNS[name]
    rng = np.random.default_rng(seed)
    truth = np.array([pgr.random_pose(rng, 0.5, 3.0) for _ in range(P)])
    fs = [pgr.make_factor(rng, truth, s, noise=0.01) for s in sets]
    return P, fs, pgr.perturb(rng, truth, 0.05, 0.2)


def _blocks_ctx(P, fs):
    c = balm_b200.Context(P, 0, L.PREC_BLOCKS)
    assert c.set_block_factors(fs) == [L.OK] * len(fs)
    c.set_voxels(np.zeros(1, np.int64), np.zeros(0, np.int32), np.zeros((0, 10)), np.zeros(0))
    return c


def _kappa(A):
    lam = np.abs(np.linalg.eigvalsh(A))
    return lam.max() / lam.min()


def _errors(A, g, dx):
    """-> (componentwise backward error with the residual in long double, dense reference solution, kappa(A))"""
    r = np.abs(np.asarray(-g, np.longdouble) - np.asarray(A, np.longdouble) @ np.asarray(dx, np.longdouble))
    den = np.abs(A) @ np.abs(dx) + np.abs(g)
    omega = float(np.max(np.where(den > 0, r.astype(np.float64) / np.where(den > 0, den, 1.0), 0.0)))
    return omega, np.linalg.solve(A, -g), _kappa(A)


def _check_solve(A, D, g, u, dx, q1, what):
    """The solver's contract on one unflagged solve -> (backward error, forward error over 20 kappa eps |ref|)"""
    omega, ref, kappa = _errors(A, g, dx)
    fwd = np.abs(dx - ref).max()
    bound = 20 * kappa * EPS * np.abs(ref).max()
    terms = 0.5 * dx * (u * D * dx - g)
    print(f"{what}: omega {omega:.1e}, forward {fwd / np.abs(ref).max():.1e} of |ref| (kappa {kappa:.1e})")
    assert omega <= 2e-12, what
    assert fwd <= bound, what
    assert abs(q1 - terms.sum()) <= 1e-9 * np.abs(terms).sum(), what
    return omega, fwd / bound


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PATTERNS))
def test_solve_covariance_and_lm_against_dense_references(name):
    P, fs, x = _factors(name, seed=sorted(PATTERNS).index(name))
    sym = _restatement(name)
    c, c2 = _blocks_ctx(P, fs), _blocks_ctx(P, fs)
    s = balm_b200.PoseGraph(P)
    assert s.set_pose_factors(fs) == [L.OK] * len(fs)
    st, sst = c.block_structure(want_pairs=True), s.structure()
    assert st["pair_list"].tolist() == [list(p) for p in nd.pairs_of(P, PATTERNS[name][1])]
    assert (st["l_blocks"], st["levels"]) == (sst["l_blocks"], sst["levels"]) == (sym["l_blocks"], sym["levels"])

    H, g, _ = c.evaluate(x)
    H2, g2, _ = c2.evaluate(x)
    assert np.array_equal(H2, H) and np.array_equal(g2, g)
    D = np.diag(H).copy()
    for u in (1.0, 0.01, 1e-6):
        dx, q1, bad = c.solve(u)
        assert not bad
        _check_solve(H + u * np.diag(D), D, g, u, dx, q1, f"{name} u {u:g}")
        again, c2_out = c.solve(u), c2.solve(u)
        assert np.array_equal(again[0], dx) and again[1:] == (q1, bad)
        assert np.array_equal(c2_out[0], dx) and c2_out[1:] == (q1, bad)

    bytes0 = sst["device_bytes"]
    for anchor in (sym["order"][0], sym["order"][-1]):
        S, kappa = _dense_sigma(H, anchor)
        pairs, cov = c.block_covariance(x, anchor=anchor)
        _check_against(cov, pairs, S, kappa, f"{name} blocks anchor {anchor}")
        pairs_s, cov_s = s.covariance(x, anchor)
        assert np.array_equal(pairs_s, pairs)
        _check_against(cov_s, pairs_s, S, kappa, f"{name} PoseGraph anchor {anchor}")
        # the selected inversion's tables and Z, built by the first call only
        grown = 8 * (P + 1) + 4 * max(sym["nsel"], 1) + 4 * max(len(pairs), 1) + 288 * sym["l_blocks"]
        assert s.structure()["device_bytes"] == bytes0 + grown

    A = H + 0.01 * np.diag(D)
    ref = np.linalg.solve(A, -g)
    _, tr = s.pose_graph_iter(x, max_iter=1, rel_tol=-1, gauge_mode=2, want_per_iter=True)
    assert tr[0]["accepted"] and not tr[0]["not_pd"]
    expect = pgr.pose_update(x, ref)
    tol = 1e-9 + 20 * _kappa(A) * EPS * np.abs(ref).max() * (1 + np.abs(x[:, 9:]).max())
    assert np.abs(tr[0]["poses"] - expect).max() <= tol
    for h in (c, c2, s):
        h.close()


@pytest.mark.gpu
def test_structure_of_other_patterns():
    """A voxel pattern, the 4541-pose pyramid of test_gpu_sparse_covariance and a 100-pose clique: the device's
    structure is the restatement's."""
    from test_gpu_block_hessian import SCENES, _ctx
    sc = SCENES["corridor300"]()
    c = _ctx(sc, L.PREC_BLOCKS)
    st = c.block_structure(want_pairs=True)
    sym = nd.symbolic(sc["n_poses"], st["pair_list"])
    print(f"corridor300: l_blocks {sym['l_blocks']}, levels {sym['levels']}, m_max {sym['m_max']}, "
          f"terms_max {sym['terms_max']}")
    assert (st["l_blocks"], st["levels"]) == (sym["l_blocks"], sym["levels"])
    c.close()
    rng = np.random.default_rng(0)
    for P, sets in ((4541, pgr.pyramid_factor_poses(4541, top=32)), (100, _clique(100))):
        truth = np.array([pgr.random_pose(rng, 0.5, 3.0) for _ in range(P)])
        s = balm_b200.PoseGraph(P)
        assert s.set_pose_factors([pgr.make_factor(rng, truth, f) for f in sets]) == [L.OK] * len(sets)
        sym = nd.symbolic(P, nd.pairs_of(P, sets))
        assert (s.structure()["l_blocks"], s.structure()["levels"]) == (sym["l_blocks"], sym["levels"])
        s.close()


def _leading_minor_crossing(H, order, poses):
    """A damping u in (-0.95, -0.3) at which the leading principal minor of H + u diag(H) over the first `poses`
    columns of the elimination order is singular: the generalised eigenvalue lam of (H_k, D_k) nearest the middle of
    the range, u = -lam. Damping just past it leaves that pivot of the unpivoted LDL^T tiny and its multipliers large."""
    idx = (6 * np.asarray(order[:poses])[:, None] + np.arange(6)).ravel()
    lam = sla.eigh(H[np.ix_(idx, idx)], np.diag(np.diag(H)[idx]), eigvals_only=True)
    lam = lam[(lam > 0.3) & (lam < 0.95)]
    return -lam[np.argmin(np.abs(lam - 0.6))]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["clique44", "clique87"])
def test_refinement_under_negative_damping(name):
    """H + u diag(H) with u < 0 is indefinite. The LDL^T without pivoting may then lose digits; the solve's residual
    check must catch it and refine, or flag the step. A host emulation (the scalar LDL^T of the same order) predicts
    whether the backward error passes 1e-12: above 1e-11 the device must refine, below 1e-13 it must not."""
    P, fs, x = _factors(name, seed=0)
    order = _restatement(name)["order"]
    c = _blocks_ctx(P, fs)
    H, g, _ = c.evaluate(x)
    D = np.diag(H).copy()
    # the sweep, and damping 1e-6 .. 1e-8 relative past a leading minor's singularity: emulated omega there is
    # 2e-12 .. 4e-12, 1e-11 .. 3e-11 and 2e-10 .. 4e-10 on these seeds, where the sweep passes 1e-11 only by chance
    # (once, at u = -0.3 on clique44)
    cross = _leading_minor_crossing(H, order, P // 2)
    us = list(np.linspace(-0.95, -0.3, 15)) + [cross * (1 + d) for d in (1e-6, 1e-7, 1e-8)]
    refined_ok = []
    for u in us:
        c.reset_counters()
        dx, q1, bad = c.solve(u)
        n_ref = c.timings()["refinements"]
        A = H + u * np.diag(D)
        emulated, _ = nd.ldlt_backward_error(A, -g, order)
        print(f"{name} u {u:.9f}: emulated omega {emulated:.1e}, refined {n_ref}, flagged {bad}")
        if emulated > 1e-11:
            assert n_ref == 1, u
        if emulated < 1e-13:
            assert n_ref == 0, u
        if not bad:
            _check_solve(A, D, g, u, dx, q1, f"{name} u {u:.9f}")
            if n_ref:
                refined_ok.append((emulated, u, q1))
    assert refined_ok, "no solve refined and passed"
    # exact zero pivots: flagged, and a flagged step is not refined
    c.reset_counters()
    assert c.solve(-1.0)[2] and c.timings()["refinements"] == 0
    # the PoseGraph's LM takes the same refinement route (balm_spg_iter): the refined q1, bit for bit
    _, u, q1 = max(refined_ok)
    s = balm_b200.PoseGraph(P)
    s.set_pose_factors(fs)
    _, tr = s.pose_graph_iter(x, max_iter=1, u0=u, rel_tol=-1, gauge_mode=2)
    assert not tr[0]["not_pd"] and tr[0]["q1"] == q1
    s.close()
    c.close()

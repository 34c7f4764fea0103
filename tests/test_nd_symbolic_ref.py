"""The host restatement of the sparse solve's ordering and symbolic factorisation (nd_symbolic_ref.py) against what
those must be whatever the code: a permutation, cliques of the filled pattern, a parent above its children, the closed
forms of a clique and of paths, and the numbers the C++ gives on patterns of the existing tests."""
import numpy as np
import pytest

import nd_symbolic_ref as nd
import pose_graph_ref as pg


def _path(n):
    return [[i, i + 1] for i in range(n - 1)]


def _grid(n):
    return [[r * n + c, r * n + c + 1] for r in range(n) for c in range(n - 1)] + \
           [[r * n + c, (r + 1) * n + c] for r in range(n - 1) for c in range(n)]


CASES = {
    "clique100": (100, [list(range(100))]),
    "path65": (65, _path(65)),
    "grid20": (400, _grid(20)),
    "pyramid90": (90, pg.pyramid_factor_poses(90, top=8)),
    "loops300": (300, pg.pyramid_factor_poses(300, top=32) + [[i, 299 - i] for i in range(0, 150, 37)]),
    "star": (200, [[0, i] for i in range(1, 200)]),
    "scattered": (70, [list(np.random.default_rng(1).permutation(70)[:k]) for k in (5, 9, 2, 30)] + _path(70)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_order_and_structure_invariants(name):
    P, sets = CASES[name]
    pairs = nd.pairs_of(P, sets)
    s = nd.symbolic(P, pairs)
    assert sorted(s["order"]) == list(range(P))
    iperm = np.empty(P, dtype=int)
    iperm[s["order"]] = np.arange(P)
    F = nd.filled_pattern(P, s)
    for i, j in pairs:  # every block of A is a block of L + L^T
        assert F[iperm[i], iperm[j]]
    for j, S in enumerate(s["struct"]):
        assert all(i > j for i in S) and S == sorted(S)
        assert F[np.ix_(S, S)].all()  # struct(j) is a clique of the filled pattern
        if S:
            p = s["parent"][j]
            assert p == S[0] and s["level"][p] > s["level"][j]
            assert set(S[1:]) <= set(s["struct"][p])  # the rest of struct(j) passes up the tree
        else:
            assert s["parent"][j] == -1
    assert s["levels"] == max(s["level"]) + 1
    m = [len(S) for S in s["struct"]]
    assert s["l_blocks"] == P + sum(m) and s["m_max"] == max(m) and s["nsel"] == sum(k * k for k in m)
    # the row counts are the diagonal blocks' update terms
    rows = np.bincount([i for S in s["struct"] for i in S], minlength=P)
    assert s["row_max"] == rows.max() <= s["terms_max"]


@pytest.mark.parametrize("n", [1, 2, 16, 33, 87, 100])
def test_a_clique(n):
    s = nd.symbolic(n, nd.pairs_of(n, [list(range(n))]))
    assert (s["l_blocks"], s["levels"], s["m_max"]) == (n * (n + 1) // 2, n, n - 1)
    assert s["terms_max"] == max(n - 1, 0) and s["nsel"] == sum(k * k for k in range(n))


@pytest.mark.parametrize("n, l_blocks, levels", [(2, 3, 2), (32, 63, 32), (33, 81, 18), (64, 158, 33), (65, 160, 32)])
def test_paths(n, l_blocks, levels):
    """A leaf of 32 keeps index order (a chain of 31 columns); 33 poses are the first cut; longer paths nest."""
    s = nd.symbolic(n, nd.pairs_of(n, _path(n)))
    assert (s["l_blocks"], s["levels"]) == (l_blocks, levels)


def test_the_first_cut_by_hand():
    """33 poses in a path: cut at index 16, the crossing edge (15, 16) covered by its lower pose 15 (a tie of one
    crossing edge each); the left leaf 0..14, the right leaf 16..32, then the separator."""
    s = nd.symbolic(33, nd.pairs_of(33, _path(33)))
    assert s["order"] == list(range(15)) + list(range(16, 33)) + [15]
    # a star: the hub covers every crossing edge on its own
    s = nd.symbolic(200, nd.pairs_of(200, [[0, i] for i in range(1, 200)]))
    assert s["order"][-1] == 0 and s["row_max"] == s["terms_max"] == 199 and s["levels"] == 2


@pytest.mark.parametrize("name, expect", [
    ("clique100", (5050, 100, 99)),
    ("grid20", (10726, 100, 59)),
    ("pyramid4541", (102377, 128, 49)),
])
def test_known_structures(name, expect):
    """l_blocks, levels and m_max that pose_graph_sparse.cu's ordering and symbolic factorisation give on these
    patterns (test_gpu_sparse_ldlt_edges compares the device's structure with the restatement on them)."""
    if name == "pyramid4541":
        P, sets = 4541, pg.pyramid_factor_poses(4541, top=32)
    else:
        P, sets = CASES[name]
    s = nd.symbolic(P, nd.pairs_of(P, sets))
    assert (s["l_blocks"], s["levels"], s["m_max"]) == expect


def test_the_ldlt_emulation():
    """ldlt_backward_error solves a PD system to rounding and reports a small omega; in another order the same."""
    rng = np.random.default_rng(2)
    A = pg.random_spd(rng, 60, cond=1e4)
    b = rng.normal(size=60)
    for order in (list(range(10)), list(rng.permutation(10))):
        om, x = nd.ldlt_backward_error(A, b, order)
        assert om < 1e-14
        assert np.abs(x - np.linalg.solve(A, b)).max() <= 1e-10 * np.abs(x).max()

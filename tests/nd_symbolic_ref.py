"""Python restatement of the host side of the sparse solve in balm_b200/csrc/pose_graph_sparse.cu: the nested-dissection
ordering (nd_order) and the symbolic block factorisation, from the block pairs of H alone.

  nd_order: a vertex set (ascending pose index) of more than ND_LEAF poses is cut at its median index; the separator is a
  greedy vertex cover of the crossing edges, taken from a max-heap of (uncovered crossing edges, -pose) so that the
  lower pose wins a tie, stale entries pushed back with their current count and covered ones skipped. The left half,
  then the right half are ordered recursively, then the separator in ascending index. A leaf keeps index order.

  symbolic: struct(j) = {i > j : A_ij != 0} united with struct(c) \\ {j} of j's children c in the elimination tree,
  parent(j) = min struct(j), level(j) = 1 + the largest level of its children (0 for a leaf).

The quantities returned are the loop bounds of the device kernels: m_j = |struct(j)| blocks below column j's diagonal,
the update terms of every block of L (column k contributes one term to block (i, j) for every i >= j in struct(k),
diagonal blocks included), the off-diagonal blocks of every row, and the elimination tree's levels."""
import heapq

import numpy as np
from scipy.linalg import solve_triangular

ND_LEAF = 32


def adjacency(P, pairs):
    """Sorted neighbour lists of every pose from block pairs (i, j); diagonal pairs and repeats are ignored."""
    nb = [set() for _ in range(P)]
    for i, j in pairs:
        i, j = int(i), int(j)
        if i != j:
            nb[i].add(j)
            nb[j].add(i)
    return [sorted(s) for s in nb]


def pairs_of(P, pose_sets):
    """The block pairs (i <= j) of factors over the given pose index sets, and every diagonal pair."""
    s = {(i, i) for i in range(P)}
    for f in pose_sets:
        s |= {(min(a, b), max(a, b)) for a in f for b in f}
    return sorted(s)


def nd_order(P, adj):
    """-> order, order[k] = the pose of column k."""
    side, cnt, order = [-1] * P, [0] * P, []

    def rec(V):
        if len(V) <= ND_LEAF:
            order.extend(V)
            return
        h = len(V) // 2
        for q, v in enumerate(V):
            side[v] = 1 if q < h else 2
        heap = []
        for v in V:
            n = sum(1 for w in adj[v] if side[w] == 3 - side[v])
            cnt[v] = n
            if n:
                heap.append((-n, v))
        heapq.heapify(heap)
        sep = []
        while heap:
            n, v = heapq.heappop(heap)
            if side[v] == 0 or cnt[v] == 0:
                continue
            if -n != cnt[v]:
                heapq.heappush(heap, (-cnt[v], v))
                continue
            sv = side[v]
            side[v] = 0
            sep.append(v)
            for w in adj[v]:
                if side[w] == 3 - sv:
                    cnt[w] -= 1
        left = [v for v in V if side[v] == 1]
        right = [v for v in V if side[v] == 2]
        for v in V:
            side[v] = -1
        rec(left)
        rec(right)
        order.extend(sorted(sep))

    rec(list(range(P)))
    return order


def symbolic(P, pairs):
    """-> dict of order, struct (list of ascending column lists), parent, level (per column), l_blocks, levels, m_max,
    terms_max (most update terms of one block of L), row_max (most off-diagonal blocks of one row of L) and
    nsel = sum m_j^2 (the selected inversion's terms)."""
    adj = adjacency(P, pairs)
    order = nd_order(P, adj)
    iperm = np.empty(P, dtype=np.int64)
    iperm[order] = np.arange(P)
    struct, children = [None] * P, [[] for _ in range(P)]
    parent, level = [-1] * P, [0] * P
    for j in range(P):
        rows = {int(iperm[w]) for w in adj[order[j]] if iperm[w] > j}
        for c in children[j]:
            level[j] = max(level[j], level[c] + 1)
            rows.update(i for i in struct[c] if i > j)
        struct[j] = sorted(rows)
        if rows:
            parent[j] = struct[j][0]
            children[parent[j]].append(j)
    m = np.array([len(s) for s in struct], dtype=np.int64)
    # update terms per block, keyed i * P + j: column k adds one to every (S[t], S[u]) with t >= u, S = struct(k)
    keys = []
    for k in range(P):
        S = np.asarray(struct[k], dtype=np.int64)
        if len(S):
            t, u = np.tril_indices(len(S))
            keys.append(S[t] * P + S[u])
    terms = np.unique(np.concatenate(keys), return_counts=True)[1] if keys else np.zeros(1, np.int64)
    rows = np.bincount(np.concatenate([np.asarray(s, np.int64) for s in struct] + [np.zeros(0, np.int64)]),
                       minlength=P)
    return dict(order=order, struct=struct, parent=parent, level=level, l_blocks=int(P + m.sum()),
                levels=int(max(level) + 1), m_max=int(m.max()), terms_max=int(terms.max()), row_max=int(rows.max()),
                nsel=int((m * m).sum()))


def filled_pattern(P, sym):
    """Boolean P x P pattern of L + L^T in column order (diagonal included)."""
    F = np.eye(P, dtype=bool)
    for j, s in enumerate(sym["struct"]):
        F[s, j] = F[j, s] = True
    return F


def ldlt_backward_error(A, b, order):
    """Host emulation of the device's decision to refine: the scalar LDL^T without pivoting of A in the pose order
    `order` (6 rows per pose), the solve of A x = b with it, and the componentwise backward error
    omega = max_r |b - A x|_r / (|A| |x| + |b|)_r with the residual formed in long double."""
    idx = (6 * np.asarray(order)[:, None] + np.arange(6)).ravel()
    M = np.array(A[np.ix_(idx, idx)], dtype=np.float64)
    n = len(M)
    d = np.zeros(n)
    for k in range(n):  # right-looking: column k scaled, then the trailing rank-one update
        d[k] = M[k, k]
        c = M[k + 1:, k] / d[k]
        M[k + 1:, k + 1:] -= np.outer(c, M[k + 1:, k])
        M[k + 1:, k] = c
    Lm = np.tril(M, -1)
    y = solve_triangular(Lm, b[idx], lower=True, unit_diagonal=True)
    z = solve_triangular(Lm.T, y / d, lower=False, unit_diagonal=True)
    x = np.empty(n)
    x[idx] = z
    Ald = np.asarray(A, dtype=np.longdouble)
    r = np.abs(np.asarray(b, np.longdouble) - Ald @ np.asarray(x, np.longdouble)).astype(np.float64)
    den = np.abs(A) @ np.abs(x) + np.abs(b)
    return float(np.max(np.where(den > 0, r / np.where(den > 0, den, 1.0), 0.0))), x

"""The tensor-core SYRK (syrk_tc_kernel) pinned bit for bit to an exact integer reference.

The kernel's digit-pair sums T_d = sum_{s+t=d} q_s^T q_t are exact int32 sums, and its epilogue is a fixed sequence of
fp64 operations on them, so its fp64 partial tiles are a deterministic function of the digit planes and the column
factors isc. The reference below recomputes the T_d exactly (float64 matmuls of int8 digits: every partial sum is an
integer below 2^53) and replays the epilogue in the kernel's operation order:

    val = T[S-1];  val = val / 256 + T[d] for d = S-2 .. 0;  w = (val * isc_i) * isc_j;  w += old when accumulating

over the items of the k-split (per = ceil(padded rows / splits) rounded up to 64; item sp covers
[sp * per, min((sp + 1) * per, padded rows)), an empty item still writes its tiles) and the upper-triangle tiles in
row-major order. H's SYRK term is -(0.0 + p_0 + p_1 + ...) over the splits in ascending order. No tolerance anywhere in
the SYRK comparisons: an error confined to the lowest digit plane reaches H only at 256^-(S-1) of its size, far below
the 1e-8 window of the parity tests, but it changes these bits.

The kernel is driven two ways: alone on synthetic digit planes (balm_debug_syrk_tc) at its tile, half-tile, ring, split
and int32-bound edges, and inside balm_evaluate, whose last batch's planes and scales come back through
balm_debug_tc_planes; there the digits are also checked against the observation sweep's fixed point of G'.
"""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

import numpy_ref
import scenes

TILE, KS = 128, 64
MAX_ROWS_PER_ITEM = 32704                 # 4 * 32704 * 2^14 < 2^31
STAGES = {2: 6, 3: 4, 4: 3}               # syrk_tc_kernel's ring depth per digit-plane count (192 KB / stage bytes)
SLICES = [2, 3, 4]


# ---------------------------------------------------------------- the reference ----------------------------------------
def ldg_of(n_poses):
    return (6 * n_poses + TILE - 1) // TILE * TILE


def pad_rows(rows):
    return (rows + KS - 1) // KS * KS


def tile_coords(nb):
    """(bi, bj) of the upper-triangle tiles in the kernel's order (tile_coords_tc: row-major)."""
    return [(bi, bj) for bi in range(nb) for bj in range(bi, nb)]


def item_ranges(rows_padded, splits):
    """per-item rows and the contraction range of every k-split item (decode_item)."""
    per = (-(-rows_padded // splits) + KS - 1) // KS * KS
    return per, [(sp * per, min((sp + 1) * per, rows_padded)) for sp in range(splits)]


def balanced_digits(X, S):
    """The observation sweep's digit split of integers |X| < 2^(8S-2): byte kb of X + 0x80808080 (32-bit) is the digit
    of weight 256^kb plus 128. Plane 0 is the most significant digit."""
    u = (np.asarray(X, dtype=np.int64) + 0x80808080) & 0xFFFFFFFF
    return np.stack([(((u >> (8 * kb)) & 0xFF) - 128).astype(np.int8) for kb in reversed(range(S))])


def digits_value(q):
    """X = sum_s q_s 256^(S-1-s) (int64)."""
    S = len(q)
    return sum(q[s].astype(np.int64) * (256 ** (S - 1 - s)) for s in range(S))


_TORCH_CUDA = None


def _gram(a, b):
    """a^T b of int8-valued float64 matrices, exact (integer partial sums below 2^53 in any summation order)."""
    global _TORCH_CUDA
    if _TORCH_CUDA is None:
        try:
            import torch
            _TORCH_CUDA = torch.cuda.is_available()
        except ImportError:
            _TORCH_CUDA = False
    if _TORCH_CUDA and a.shape[0] * a.shape[1] * b.shape[1] > (1 << 26):
        import torch
        return (torch.from_numpy(a).cuda().T @ torch.from_numpy(b).cuda()).cpu().numpy()
    return a.T @ b


def digit_pair_sums(q, k0, k1, ndig=None):
    """T_d = sum_{s+t=d} q_s[k0:k1]^T q_t[k0:k1] for d < ndig (default S), exact, as float64."""
    S, _, ldg = q.shape
    ndig = S if ndig is None else ndig
    T = np.zeros((ndig, ldg, ldg))
    if k1 <= k0:
        return T
    Q = [q[s, k0:k1].astype(np.float64) for s in range(S)]
    for s in range(S):
        for t in range(s, S):
            if s + t < ndig:
                G = _gram(Q[s], Q[t])
                T[s + t] += G if s == t else G + G.T
    return T


def epilogue(T, isc, old=None):
    """The kernel's epilogue on the digit-pair sums, operation for operation (val * 1/256 is exact, so an FMA
    contraction of val * inv256 + T[d] gives the same bits)."""
    S = len(T)
    val = T[S - 1].copy()
    for d in range(S - 2, -1, -1):
        val = val * (1.0 / 256.0) + T[d]
    w = (val * isc[:, None]) * isc[None, :]
    return w if old is None else w + old


def syrk_reference(q, isc, splits, old=None):
    """Partial tiles [splits][tiles][128][128] of syrk_tc_kernel on the planes q (S x rows_padded x ldg)."""
    S, rows_padded, ldg = q.shape
    coords = tile_coords(ldg // TILE)
    _, ranges = item_ranges(rows_padded, splits)
    part = np.empty((splits, len(coords), TILE, TILE))
    for sp, (k0, k1) in enumerate(ranges):
        w = epilogue(digit_pair_sums(q, k0, k1), isc)
        for t, (bi, bj) in enumerate(coords):
            blk = w[bi * TILE:(bi + 1) * TILE, bj * TILE:(bj + 1) * TILE]
            part[sp, t] = blk if old is None else blk + old[sp, t]
    return part


def assemble(part, n):
    """H's SYRK term as assemble_kernel forms it: -(0.0 + p_0 + p_1 + ...), upper tiles mirrored to the lower half."""
    splits, ntiles = part.shape[:2]
    s = np.zeros(part.shape[1:])
    for sp in range(splits):
        s = s + part[sp]
    nb = int(round((np.sqrt(8 * ntiles + 1) - 1) / 2))
    F = np.zeros((nb * TILE, nb * TILE))
    for t, (bi, bj) in enumerate(tile_coords(nb)):
        F[bi * TILE:(bi + 1) * TILE, bj * TILE:(bj + 1) * TILE] = s[t]
    r = np.arange(nb * TILE)
    F = np.where(r[:, None] <= r[None, :], F, F.T)
    return -F[:n, :n]


def gprime(sc, poses12, include_fix=False):
    """The 3M x 6N matrix G' whose Gram matrix is the SYRK term of H: rows 3a + k = sqrt(coe_a |w_k|) G_a[:, k]^T, a
    restatement of tests/numpy_ref.py's per-voxel G and weights w."""
    N, M = sc["n_poses"], len(sc["row_ptr"]) - 1
    Gp = np.zeros((3 * M, 6 * N))
    for a in range(M):
        sl = range(sc["row_ptr"][a], sc["row_ptr"][a + 1])
        W = [numpy_ref._world_cluster(sc["obs10"][s], poses12[sc["pose_idx"][s]]) for s in sl]
        P = sum(w[0] for w in W); v = sum(w[1] for w in W); NN = sum(w[2] for w in W)
        if include_fix and sc.get("fix10") is not None:
            f = sc["fix10"][a]
            P = P + np.array([[f[0], f[1], f[2]], [f[1], f[3], f[4]], [f[2], f[4], f[5]]]); v = v + f[6:9]; NN = NN + f[9]
        vb = v / NN
        lam, U = np.linalg.eigh(P / NN - np.outer(vb, vb))
        u0 = U[:, 0]
        wk = np.array([-2.0 / NN ** 2, 2.0 / (lam[0] - lam[1]), 2.0 / (lam[0] - lam[2])])
        f = np.sqrt(sc["coe"][a] * np.abs(wk))
        for s, (Pw, vw, nn) in zip(sl, W):
            i = sc["pose_idx"][s]
            Mt = Pw - np.outer(vw, vb)
            mb = vw - nn * vb
            cols = [np.concatenate([-np.cross(u0, vw), nn * u0])]
            for uk in (U[:, 1], U[:, 2]):
                top = -np.cross(uk, Mt @ u0) - np.cross(u0, Mt @ uk)
                bot = uk * (mb @ u0) + u0 * (mb @ uk)
                cols.append(np.concatenate([top, bot]) / NN)
            for k in range(3):
                Gp[3 * a + k, 6 * i:6 * i + 6] = f[k] * cols[k]
    return Gp


# ---------------------------------------------------------------- the reference's own checks (CPU) -------------------
@pytest.mark.parametrize("S", SLICES)
def test_balanced_digit_split_round_trips(S):
    rng = np.random.default_rng(S)
    lim = 2 ** (8 * S - 2)
    X = np.concatenate([rng.integers(-lim + 1, lim, 20000),
                        [0, 1, -1, 127, 128, -128, -129, 255, 256, -256, lim - 1, -(lim - 1), lim // 2, -lim // 2]])
    q = balanced_digits(X, S)
    assert q.shape == (S, len(X)) and q.dtype == np.int8
    assert np.array_equal(digits_value(q), X)
    # the same digits as the textbook balanced base-256 expansion
    for x, col in zip(X[-14:].tolist() + X[:200].tolist(), np.concatenate([q[:, -14:], q[:, :200]], axis=1).T):
        ref, r = [], int(x)
        for _ in range(S):
            d = (r + 128) % 256 - 128
            ref.append(d)
            r = (r - d) // 256
        assert r == 0 and ref[::-1] == col.tolist(), x


@pytest.mark.parametrize("S", SLICES)
def test_reference_with_all_digit_pairs_is_the_integer_product(S):
    rng = np.random.default_rng(10 + S)
    rows, cols = 37, 9
    q = rng.integers(-128, 128, size=(S, rows, cols)).astype(np.int8)
    q[:, :3] = -128
    T = digit_pair_sums(q, 0, rows, ndig=2 * S - 1)
    full = sum(T[d].astype(np.int64).astype(object) * (256 ** (2 * S - 2 - d)) for d in range(2 * S - 1))
    X = digits_value(q).astype(object)
    assert (full == X.T.dot(X)).all()
    # the kernel's sums (d < S) are a prefix of these
    assert np.array_equal(digit_pair_sums(q, 0, rows), T[:S])
    # and split over contraction ranges they add up
    assert np.array_equal(digit_pair_sums(q, 0, 20) + digit_pair_sums(q, 20, rows), T[:S])


def _round(x):
    return float(x)  # Fraction -> nearest double (correctly rounded int / int division)


@pytest.mark.parametrize("S", SLICES)
def test_epilogue_matches_exact_arithmetic(S):
    """Each operation of the replayed epilogue is the correctly rounded result of exact rational arithmetic, and the
    whole stays within a few roundings of the exact value of sum_d 256^-d T_d isc_i isc_j."""
    rng = np.random.default_rng(20 + S)
    n = 6
    T = rng.integers(-(2 ** 31) + 1, 2 ** 31, size=(S, n, n)).astype(np.float64)
    T[:, 0, 0] = [2 ** 31 - 1] * S
    isc = np.concatenate([np.ldexp(1.0, rng.integers(-40, 40, n - 2)), rng.uniform(0.5, 3.0, 2)])
    old = rng.normal(size=(n, n)) * 1e9
    for o in (None, old):
        w = epilogue(T, isc, o)
        for i in range(n):
            for j in range(n):
                val = Fraction(T[S - 1, i, j])
                for d in range(S - 2, -1, -1):
                    val = Fraction(_round(Fraction(_round(val)) / 256 + Fraction(T[d, i, j])))
                x = _round(Fraction(_round(val * Fraction(isc[i]))) * Fraction(isc[j]))
                if o is not None:
                    x = _round(Fraction(x) + Fraction(o[i, j]))
                assert w[i, j] == x, (i, j)
                if o is None:
                    exact = sum(Fraction(T[d, i, j]) / 256 ** d for d in range(S)) * Fraction(isc[i]) * Fraction(isc[j])
                    assert abs(Fraction(w[i, j]) - exact) <= abs(exact) * Fraction(S + 2, 2 ** 52), (i, j)


def test_item_decomposition():
    for rows_padded in (64, 128, 192, 576, 3328, 32704, 65408):
        for splits in range(1, 9):
            per, ranges = item_ranges(rows_padded, splits)
            assert per % KS == 0 and per * splits >= rows_padded and per - KS < -(-rows_padded // splits)
            covered = [k for k0, k1 in ranges for k in range(k0, k1)]
            assert covered == list(range(rows_padded))
    assert item_ranges(192, 4) == (64, [(0, 64), (64, 128), (128, 192), (192, 192)])
    assert item_ranges(pad_rows(65408), 2)[0] == MAX_ROWS_PER_ITEM
    assert item_ranges(pad_rows(65409), 2)[0] > MAX_ROWS_PER_ITEM


# ---------------------------------------------------------------- the kernel alone (balm_debug_syrk_tc) ---------------
def _lib():
    from balm_b200 import _lib as L
    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


_CTX = {}


def _ctx(n_poses):
    """One tensor-precision context per pose count (the hook uses its device, stream and column count only)."""
    if n_poses not in _CTX:
        import balm_b200
        _CTX[n_poses] = balm_b200.Context(n_poses, 0, balm_b200.PREC_TENSOR)
    return _CTX[n_poses]


@pytest.fixture(scope="module", autouse=True)
def _close_contexts():
    yield
    for c in _CTX.values():
        c.close()
    _CTX.clear()


def run_syrk(n_poses, q, rows, isc, splits, accumulate=0, part=None):
    """balm_debug_syrk_tc on the first `rows` rows of q -> (status, part)."""
    L = _lib()
    S, ldg = q.shape[0], q.shape[2]
    assert ldg == ldg_of(n_poses)
    nb = ldg // TILE
    if part is None:
        part = np.full((splits, nb * (nb + 1) // 2, TILE, TILE), np.nan)
    planes = np.ascontiguousarray(q[:, :rows], dtype=np.int8)
    isc = np.ascontiguousarray(isc, dtype=np.float64)
    st = L.lib().balm_debug_syrk_tc(_ctx(n_poses)._h, _ptr(planes), S, rows, _ptr(isc), splits, accumulate,
                                    _ptr(part))
    return st, part


def random_case(rng, n_poses, S, rows, dead=0.1):
    """Digits uniform over the whole int8 range in every plane (zero in the padding rows), power-of-two column factors
    over a wide range, 0 on dead columns and on the column padding [6N, ldg)."""
    ldg = ldg_of(n_poses)
    q = np.zeros((S, pad_rows(rows), ldg), dtype=np.int8)
    q[:, :rows] = rng.integers(-128, 128, size=(S, rows, ldg))
    isc = np.ldexp(1.0, rng.integers(-60, 40, ldg))
    isc[rng.uniform(size=ldg) < dead] = 0.0
    isc[6 * n_poses:] = 0.0
    return q, isc


def check_syrk(n_poses, q, rows, isc, splits, rng=None):
    st, part = run_syrk(n_poses, q, rows, isc, splits)
    assert st == 0, _lib().lib().balm_last_error()
    ref = syrk_reference(q, isc, splits)
    if not np.array_equal(part, ref):
        bad = np.argwhere(part != ref)
        raise AssertionError(f"N={n_poses} S={len(q)} rows={rows} splits={splits}: {len(bad)} entries differ, first "
                             f"(split, tile, row, col) {bad[:4].tolist()}")
    dead = isc == 0
    assert not np.isnan(part).any()
    return part, dead


@pytest.mark.gpu
@pytest.mark.parametrize("S", SLICES)
@pytest.mark.parametrize("n_poses,cases", [
    (1, [(65, 1), (64 * 7, 2)]),        # one block whose column half 1 is all padding
    (10, [(64 * 5 + 3, 1), (300, 3)]),  # n = 60: both halves of the block hold live columns up to the boundary
    (11, [(64 * 5 + 3, 1), (300, 3)]),  # n = 66: two columns past the half boundary
    (21, [(129, 2), (64 * 6, 1)]),      # n = 126: one block
    (22, [(129, 2), (64 * 6, 1)]),      # n = 132: two blocks, three tiles
    (130, [(200, 3), (64 * 4, 1)]),     # 28 tiles; 3 splits -> 168 items on 132 SMs
    (200, [(64 * 6 + 17, 2), (64, 1)]),  # 55 tiles; 2 splits -> 220 items on 132 SMs
])
def test_kernel_columns(S, n_poses, cases):
    rng = np.random.default_rng(1000 * S + n_poses)
    for rows, splits in cases:
        q, isc = random_case(rng, n_poses, S, rows)
        part, dead = check_syrk(n_poses, q, rows, isc, splits)
        nb = ldg_of(n_poses) // TILE
        for t, (bi, bj) in enumerate(tile_coords(nb)):  # dead columns and their rows are exact zeros
            assert not part[:, t][:, dead[bi * TILE:(bi + 1) * TILE], :].any()
            assert not part[:, t][:, :, dead[bj * TILE:(bj + 1) * TILE]].any()


@pytest.mark.gpu
@pytest.mark.parametrize("S", SLICES)
@pytest.mark.parametrize("splits", [1, 2, 3])
def test_kernel_rows_and_ring(S, splits):
    """Row counts around the 64-row stage and around the ring depth (nsteps = stages - 1, stages, stages + 1 and twice
    the stages per item), so that every item ends at a different ring slot and parity."""
    nst = STAGES[S]
    n_poses = 22
    rng = np.random.default_rng(100 * S + splits)
    rows_list = [1, 63, 64, 65] + [64 * k for k in (nst - 1, nst, nst + 1, 2 * nst)]
    if splits > 1:
        rows_list += [splits * 64 * k for k in (nst - 1, nst, nst + 1, 2 * nst)] + [splits * 64 * (nst + 1) - 5]
    for rows in rows_list:
        q, isc = random_case(rng, n_poses, S, rows)
        check_syrk(n_poses, q, rows, isc, splits)


@pytest.mark.gpu
@pytest.mark.parametrize("S", SLICES)
def test_kernel_empty_trailing_items(S):
    """Split counts that leave trailing items without rows: those still write their tiles (zeros)."""
    rng = np.random.default_rng(300 + S)
    for rows, splits in [(192, 4), (130, 4), (256, 5), (256, 7), (1, 3)]:
        q, isc = random_case(rng, 11, S, rows)
        part, _ = check_syrk(11, q, rows, isc, splits)
        per, ranges = item_ranges(pad_rows(rows), splits)
        for sp, (k0, k1) in enumerate(ranges):
            if k1 <= k0:
                assert not part[sp].any()


@pytest.mark.gpu
@pytest.mark.parametrize("S", SLICES)
def test_kernel_int32_bound(S):
    """All digits -128 at exactly 32704 contraction rows per item: T_{S-1} = S * 32704 * 2^14 (2 143 289 344 at S = 4,
    next to 2^31) must come back exact, in one split and in two."""
    n_poses = 1
    ldg = ldg_of(n_poses)
    isc = np.zeros(ldg)
    isc[:6] = np.ldexp(1.0, np.arange(-3, 3))
    for rows, splits in [(MAX_ROWS_PER_ITEM, 1), (2 * MAX_ROWS_PER_ITEM, 2)]:
        q = np.full((S, rows, ldg), -128, dtype=np.int8)
        T = digit_pair_sums(q, 0, MAX_ROWS_PER_ITEM)
        assert T[S - 1, 0, 0] == S * MAX_ROWS_PER_ITEM * 2 ** 14 and T.max() < 2 ** 31
        if S == 4:
            assert T[3, 0, 0] == 2143289344
        check_syrk(n_poses, q, rows, isc, splits)


@pytest.mark.gpu
@pytest.mark.parametrize("S", SLICES)
def test_kernel_accumulates_and_is_deterministic(S):
    """accumulate = 0 overwrites whatever part held; accumulate = 1 adds the next planes' tiles to it (the later voxel
    batches of an evaluation); identical calls give identical bits."""
    rng = np.random.default_rng(400 + S)
    n_poses, splits = 130, 3
    qa, isc = random_case(rng, n_poses, S, 300)
    qb, _ = random_case(rng, n_poses, S, 300)
    qb = qb[:, :pad_rows(250)].copy()
    qb[:, 250:] = 0
    st, pa = run_syrk(n_poses, qa, 300, isc, splits)
    assert st == 0
    ref_a = syrk_reference(qa, isc, splits)
    assert np.array_equal(pa, ref_a)
    st, pa2 = run_syrk(n_poses, qa, 300, isc, splits, part=np.full_like(pa, -7.0))
    assert st == 0 and np.array_equal(pa2, pa)
    st, pab = run_syrk(n_poses, qb, 250, isc, splits, accumulate=1, part=pa.copy())
    assert st == 0
    assert np.array_equal(pab, syrk_reference(qb, isc, splits, old=ref_a))


@pytest.mark.gpu
def test_kernel_rejects_invalid_arguments():
    n_poses = 1
    ldg = ldg_of(n_poses)
    L = _lib()
    isc = np.ones(ldg)
    for S, rows, splits in [(1, 64, 1), (5, 64, 1), (4, 0, 1), (4, 64, 0), (4, 64, -1),
                            (4, MAX_ROWS_PER_ITEM + 1, 1), (2, 2 * MAX_ROWS_PER_ITEM + 1, 2),
                            (3, 3 * MAX_ROWS_PER_ITEM + 64, 3)]:
        q = np.zeros((max(S, 1), max(rows, 1), ldg), dtype=np.int8)
        part = np.full((max(splits, 1), 1, TILE, TILE), 3.0)
        st = L.lib().balm_debug_syrk_tc(_ctx(n_poses)._h, _ptr(q), S, rows, _ptr(isc), splits, 0, _ptr(part))
        assert st == L.ERR_INVALID, (S, rows, splits, st)
        assert (part == 3.0).all()  # nothing launched
    # the largest accepted shapes: 32704 rows per item
    assert run_syrk(n_poses, np.zeros((4, 3 * MAX_ROWS_PER_ITEM, ldg), np.int8), 3 * MAX_ROWS_PER_ITEM - 70, isc,
                    3)[0] == L.OK


# ---------------------------------------------------------------- the product path (balm_debug_tc_planes) -------------
def tc_planes(c):
    """What the last batch's SYRK consumed -> (planes S x rows_padded x ldg, isc, splits)."""
    L = _lib()
    S, rp, sp = C.c_int(), C.c_int64(), C.c_int()
    L.check(L.lib().balm_debug_tc_planes(c._h, None, None, C.byref(S), C.byref(rp), C.byref(sp)))
    q = np.zeros((S.value, rp.value, ldg_of(c.N)), dtype=np.int8)
    isc = np.zeros(ldg_of(c.N))
    L.check(L.lib().balm_debug_tc_planes(c._h, _ptr(q), _ptr(isc), C.byref(S), C.byref(rp), C.byref(sp)))
    return q, isc, sp.value


def check_product(c, sc, H, M, slices=None, check_sweep=False, include_fix=False):
    N, n = sc["n_poses"], 6 * sc["n_poses"]
    q, isc, splits = tc_planes(c)
    S, rows_padded, ldg = q.shape
    assert rows_padded == pad_rows(3 * M) and ldg == ldg_of(N) and 2 <= S <= 4
    if slices is not None:
        assert S == slices
    # (b) column and row padding hold zeros
    assert not q[:, :, n:].any() and not q[:, 3 * M:, :].any()
    # (a) every off-diagonal pose block of H is the assembled reference of these planes, bit for bit
    ref = assemble(syrk_reference(q, isc, splits), n)
    pose = np.arange(n) // 6
    off = pose[:, None] != pose[None, :]
    if not np.array_equal(H[off], ref[off]):
        d = np.abs(H - ref) * off
        raise AssertionError(f"S={S} splits={splits}: {int((d > 0).sum())} entries differ, max {d.max():.3e} "
                             f"of max|H| {np.abs(H).max():.3e}")
    if check_sweep:
        # (c) the digits encode the sweep's fixed point rint(G' sc), sc = 256^(S-1) / isc, to 1 unit per entry
        X = digits_value(q)[:3 * M, :n]
        live = isc[:n] > 0
        assert not X[:, ~live].any()
        assert (np.abs(X).max(axis=0) < 2 ** (8 * S - 2)).all()
        Gp = gprime(sc, sc["poses_init"], include_fix)
        Xr = np.zeros_like(Gp)
        Xr[:, live] = np.rint(Gp[:, live] * (256.0 ** (S - 1) / isc[:n][live]))
        err = np.minimum(np.abs(X - Xr).max(axis=1), np.abs(X + Xr).max(axis=1))  # eigenvector signs are arbitrary
        assert err.max() <= 1, (S, err.max(), int(np.argmax(err)))
        assert np.abs(Xr).max() > 2 ** (8 * S - 4)  # the check is not vacuous
    return S, splits


PRODUCT_SCENES = [
    pytest.param(dict(n_poses=12, n_planes=120), False, id="dense"),
    pytest.param(dict(n_poses=20, n_planes=200, drop=0.4), False, id="drop0.4"),
    pytest.param(dict(n_poses=10, n_planes=80, with_fix=True), True, id="fix"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("slices", [None, 2, 3, 4], ids=["device", "S2", "S3", "S4"])
@pytest.mark.parametrize("kw,include_fix", PRODUCT_SCENES)
def test_product_planes_and_hessian(kw, include_fix, slices, monkeypatch):
    import balm_b200
    if slices is None:
        monkeypatch.delenv("BALM_TC_SLICES", raising=False)
    else:
        monkeypatch.setenv("BALM_TC_SLICES", str(slices))
    sc = scenes.make_scene(seed=51, **kw)
    c = balm_b200.Context(sc["n_poses"], 0, balm_b200.PREC_TENSOR)
    try:
        c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc["fix10"])
        H, _, _ = c.evaluate(sc["poses_init"], include_fix=include_fix)
        check_product(c, sc, H, c.M, slices, check_sweep=True, include_fix=include_fix)
    finally:
        c.close()


@pytest.mark.gpu
def test_product_many_splits_and_items():
    """A registration whose own k-split count exceeds 1 and whose items outnumber the SMs."""
    import balm_b200
    import torch
    sc = scenes.make_scene(n_poses=200, n_planes=1100, drop=0.8, seed=52)
    c = balm_b200.Context(sc["n_poses"], 0, balm_b200.PREC_TENSOR)
    try:
        c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
        H, _, _ = c.evaluate(sc["poses_init"])
        S, splits = check_product(c, sc, H, c.M)
        nb = ldg_of(200) // TILE
        assert splits > 1 and nb * (nb + 1) * splits > torch.cuda.get_device_properties(0).multi_processor_count
    finally:
        c.close()


@pytest.mark.gpu
def test_tc_planes_rejected_without_tensor_evaluation():
    import balm_b200
    L = _lib()
    sc = scenes.make_scene(n_poses=6, n_planes=30, seed=53)
    S = C.c_int()
    for prec in (balm_b200.PREC_FP64, balm_b200.PREC_TENSOR):
        c = balm_b200.Context(6, 0, prec)
        try:
            c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
            assert L.lib().balm_debug_tc_planes(c._h, None, None, C.byref(S), None, None) == L.ERR_INVALID
            c.evaluate(sc["poses_init"])
            st = L.lib().balm_debug_tc_planes(c._h, None, None, C.byref(S), None, None)
            assert st == (L.OK if prec == balm_b200.PREC_TENSOR else L.ERR_INVALID)
            c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])  # same shape: buffers kept, planes stale
            assert L.lib().balm_debug_tc_planes(c._h, None, None, C.byref(S), None, None) == L.ERR_INVALID
        finally:
            c.close()

"""The pose-factor and pose-prior kernels pinned entry by entry to the 50-digit reference pose_terms_mp_ref.py at their
edges: rotation residuals from exactly 0 through the Jl^-1 series switch and the log's pi/2 switch to pi - 1e-6 (in
factors, including false reverse-direction loop closures, and in full-pose priors), positions up to 1e4 m, lever arms
up to 500 m, GNSS position-only priors, factors of 2, 3, 31 and 32 slots in ascending, descending and scattered order,
one pose pair shared by 16 factors, 1 .. 1000 factors and 1 .. 257 priors with NOT_PD ones interleaved, and Huber /
Cauchy losses across and on the kink. Every comparison uses the reference's per-entry scale and its one constant C
(pose_terms_mp_ref's docstring) and prints its worst ratio to the bound. PoseGraph's blocks, g, cost and (s, w) are
bitwise the dense context's."""
import numpy as np
import pytest

import balm_b200
import pose_graph_ref as pg
import pose_priors_ref as ppr
import pose_terms_mp_ref as mr
from balm_b200 import _lib as L

pytestmark = pytest.mark.gpu

NAMES = {mr.TRIVIAL: "trivial", mr.HUBER: "huber", mr.CAUCHY: "cauchy"}
POS_SCALES = (0.0, 1.0, 1e2, 1e4)
S_OVER_C2 = (1e-8, 1 - 1e-6, 1 + 1e-6, 1e8)


def _poses(rng, P, scales=POS_SCALES):
    """P poses with random rotations and positions of size scales[i % len(scales)] (0: exactly at the origin)"""
    out = []
    for i in range(P):
        d = rng.standard_normal(3)
        out.append(pg.pack(pg.exp_so3(rng.normal(0, 1.0, 3)), scales[i % len(scales)] * d / np.linalg.norm(d)))
    return np.array(out)


def _edge_factor(rng, x, a, b, th, axis, t):
    """two-slot factor over poses (a, b) whose residual at x is (th axis, t) up to the rounding of its T^"""
    ha = pg.random_pose(rng)
    Ra, pa = pg.split(x[a])
    Rb, pb = pg.split(x[b])
    Rha, pha = pg.split(ha)
    Q = Rha @ Ra.T
    R, p = Q @ Rb, Q @ (pb - pa) + pha
    X = mr.rot64(th, axis)
    hb = pg.pack(X.T @ R, X.T @ (p - t))
    return dict(poses=np.array([a, b], dtype=np.int32), poses_hat=np.stack([ha, hb]), H=pg.window_hessian(rng, 2))


def _edge_prior(rng, x, i, th, axis, t, lever, kind):
    """prior on pose i whose residual at x is (th axis, t); kind "full" or "gnss" (rotation block of H zero)"""
    R, p = pg.split(x[i])
    X = mr.rot64(th, axis)
    lv = np.zeros(3) if lever is None else np.asarray(lever, dtype=np.float64)
    if kind == "full":
        H = ppr.random_psd(rng, 6)
    else:
        H = np.zeros((6, 6))
        H[3:, 3:] = ppr.random_psd(rng, 3)[:3, :3] + np.eye(3)
    d = dict(pose=int(i), pose_hat=pg.pack(X.T @ R, R @ lv + p - t), H=H)
    if lever is not None:
        d["lever_arm"] = lv
    return d


class Ratios:
    """worst |device - reference| / (C eps scale) per quantity"""

    def __init__(self, label):
        self.label, self.r = label, {}

    def add(self, name, dev, ref, scale):
        self.r[name] = max(self.r.get(name, 0.0), mr.ratio(dev, ref, scale))

    def check(self):
        print(f"{self.label}: worst error / bound " + ", ".join(f"{k} {v:.3g}" for k, v in self.r.items()))
        bad = {k: v for k, v in self.r.items() if not v <= 1.0}
        assert not bad, f"{self.label}: over the bound {bad}"


def _register(h, factors, fk, fs, priors, pk, ps):
    status = h.set_pose_factors(factors)
    if any(k != mr.TRIVIAL for k in fk):
        h.set_factor_loss([NAMES[k] for k in fk], np.asarray(fs, dtype=np.float64))
    pstatus = h.set_pose_priors(priors, [NAMES[k] for k in pk], np.asarray(ps, dtype=np.float64)) if priors else []
    return status, pstatus


def _pin(label, P, x, factors, fbase, fk=None, fs=None, priors=(), pbase=(), pk=None, ps=None, dense=True):
    """Register on a PoseGraph (and with dense a Context), evaluate at x and pin blocks, g, cost and every term's
    (s, w) to the reference built from the per-term bases fbase / pbase (None for a term expected NOT_PD)."""
    fk = [mr.TRIVIAL] * len(factors) if fk is None else list(fk)
    fs = [1.0] * len(factors) if fs is None else list(fs)
    pk = [mr.TRIVIAL] * len(priors) if pk is None else list(pk)
    ps = [1.0] * len(priors) if ps is None else list(ps)
    ft = [(f, mr.with_loss(b, k, c)) for f, b, k, c in zip(factors, fbase, fk, fs) if b is not None]
    pt = [(p, mr.with_loss(b, k, c)) for p, b, k, c in zip(priors, pbase, pk, ps) if b is not None]
    ref = mr.assemble(ft, pt)
    s = balm_b200.PoseGraph(P)
    status, pstatus = _register(s, factors, fk, fs, priors, pk, ps)
    assert status == [L.OK if b is not None else L.ERR_NOT_PD for b in fbase]
    assert pstatus == [L.OK if b is not None else L.ERR_NOT_PD for b in pbase]
    pairs, B, g, cost = s.pose_graph_evaluate(x)
    fs_w = s.factor_residuals(x)
    ps_w = s.prior_residuals(x) if priors else None
    rt = Ratios(label)
    assert sorted(map(tuple, pairs.tolist())) == sorted(ref["blocks"])
    for q, (i, j) in enumerate(pairs.tolist()):
        Br, sc = ref["blocks"].get((i, j), (np.zeros((6, 6)), np.zeros((6, 6))))
        rt.add("H", B[q], Br, sc)
    gr, gsc = np.zeros(6 * P), np.zeros(6 * P)
    for i, (v, sc) in ref["g"].items():
        gr[6 * i:6 * i + 6], gsc[6 * i:6 * i + 6] = v, sc
    rt.add("g", g, gr, gsc)
    rt.add("cost", cost, ref["cost"], ref["cost_scale"])
    for name, sw, terms, base in (("factor", fs_w, [t for _, t in ft], fbase),
                                  ("prior", ps_w, [t for _, t in pt], pbase)):
        if sw is None:
            continue
        sd, wd = sw
        ok = np.array([b is not None for b in base])
        assert not sd[~ok].any() and not wd[~ok].any()
        rt.add(name + " s", sd[ok], [float(t["s"]) for t in terms], [t["s_scale"] for t in terms])
        rt.add(name + " w", wd[ok], [float(t["w"]) for t in terms], [t["w_scale"] for t in terms])
    rt.check()
    if dense:  # the dense context: bitwise the PoseGraph's blocks, g, cost and (s, w)
        c = balm_b200.Context(P)
        _register(c, factors, fk, fs, priors, pk, ps)
        H, gd, rd = c.pose_graph_evaluate(x)
        assert np.array_equal(B, np.array([H[6 * i:6 * i + 6, 6 * j:6 * j + 6] for i, j in pairs]))
        assert np.array_equal(gd, g) and rd == cost
        assert all(np.array_equal(u, v) for u, v in zip(c.factor_residuals(x), fs_w))
        if priors:
            assert all(np.array_equal(u, v) for u, v in zip(c.prior_residuals(x), ps_w))
        c.close()
    s.close()
    return fs_w, ps_w


# ---------------- rotation-residual magnitudes ----------------
@pytest.fixture(scope="module")
def angle_set():
    """one two-slot factor per (edge angle, axis) over scattered pose pairs in both orders -- those near pi are false
    loop closures between passes driven in opposite directions -- plus one at poses equal to their T^; positions up to
    1e4 m"""
    rng = np.random.default_rng(1)
    P = 48
    x = _poses(rng, P)
    factors = []
    for th, axis in ((th, a) for th in mr.ANGLES for a in mr.AXES):
        a, b = (int(v) for v in rng.choice(P, 2, replace=False))
        factors.append(_edge_factor(rng, x, a, b, th, axis, rng.normal(0, 0.1, 3)))
    f0 = dict(poses=np.array([7, 3], dtype=np.int32), poses_hat=x[[7, 3]].copy(), H=pg.window_hessian(rng, 2))
    factors.append(f0)
    return P, x, factors, [mr.factor_base(x, f) for f in factors]


def _loss_for(bases, kinds):
    """(kinds, scales) with each term's s / c^2 cycling through S_OVER_C2"""
    fk, fs = [], []
    for q, (b, k) in enumerate(zip(bases, kinds)):
        sv = float(b["s"]) if b is not None else 1.0
        fk.append(k)
        fs.append(np.sqrt(sv / S_OVER_C2[q % len(S_OVER_C2)]) if sv > 0 else 1.0)
    return fk, fs


@pytest.mark.parametrize("loss", ["trivial", "huber", "cauchy", "mixed"])
def test_factor_rotation_magnitudes(angle_set, loss):
    P, x, factors, bases = angle_set
    if loss == "trivial":
        fk, fs = None, None
    else:
        kinds = {"huber": [mr.HUBER], "cauchy": [mr.CAUCHY], "mixed": [mr.HUBER, mr.CAUCHY, mr.TRIVIAL]}[loss]
        fk, fs = _loss_for(bases, [kinds[q % len(kinds)] for q in range(len(factors))])
    _pin(f"factor angles, {loss}", P, x, factors, bases, fk, fs)


def test_rotation_by_pi_pins_s_and_cost():
    """at theta = pi the sign of e_rot is arbitrary: with H~ = I, s = |e_rot|^2 + |e_trans|^2 = pi^2 and the cost"""
    rng = np.random.default_rng(3)
    P = 6
    x = _poses(rng, P)
    factors = []
    for n, axis in enumerate(mr.AXES):
        f = _edge_factor(rng, x, n, n + 1, np.pi, axis, np.zeros(3))
        f["H"] = np.kron(np.array([[1.0, -1.0], [-1.0, 1.0]]), np.eye(6))
        factors.append(f)
    c = balm_b200.Context(P)
    assert c.set_pose_factors(factors) == [L.OK] * len(factors)
    sd, wd = c.factor_residuals(x)
    _, _, cost = c.pose_graph_evaluate(x)
    bases = [mr.factor_base(x, f) for f in factors]
    rt = Ratios("theta = pi")
    rt.add("s", sd, [float(b["s"]) for b in bases], [b["s_scale"] for b in bases])
    rt.add("s = pi^2", sd, np.full(len(sd), np.pi ** 2), [b["s_scale"] for b in bases])
    rt.add("cost", cost, float(sum(b["s"] for b in bases)) / 2, 0.5 * sum(b["s_scale"] for b in bases))
    rt.check()
    assert np.array_equal(wd, np.ones(len(sd)))
    c.close()


# ---------------- priors ----------------
LEVERS = (None, [2.0, 0.0, 0.0], [0.0, -300.0, 400.0])


@pytest.fixture(scope="module")
def prior_angle_set():
    """full-pose and GNSS priors at every (edge angle, axis), several per pose, registered out of pose order, lever
    arms 0, 2 m and 500 m, positions up to 1e4 m; one two-slot factor so that the pose graph has factors"""
    rng = np.random.default_rng(4)
    P = 12
    x = _poses(rng, P)
    priors = []
    for n, (th, axis) in enumerate((th, a) for th in mr.ANGLES for a in mr.AXES):
        priors.append(_edge_prior(rng, x, int(rng.integers(P)), th, axis, rng.normal(0, 0.2, 3), LEVERS[n % 3],
                                  "gnss" if n % 4 == 3 else "full"))
    factors = [pg.make_factor(rng, x, [5, 2], noise=0.01)]
    return P, x, factors, [mr.factor_base(x, f) for f in factors], priors, [mr.prior_base(x, p) for p in priors]


@pytest.mark.parametrize("loss", ["trivial", "huber", "cauchy", "mixed"])
def test_prior_rotation_magnitudes(prior_angle_set, loss):
    P, x, factors, fb, priors, pb = prior_angle_set
    if loss == "trivial":
        pk, ps = None, None
    else:
        kinds = {"huber": [mr.HUBER], "cauchy": [mr.CAUCHY], "mixed": [mr.CAUCHY, mr.TRIVIAL, mr.HUBER]}[loss]
        pk, ps = _loss_for(pb, [kinds[q % len(kinds)] for q in range(len(priors))])
    _pin(f"prior angles, {loss}", P, x, factors, fb, priors=priors, pbase=pb, pk=pk, ps=ps)


@pytest.fixture(scope="module")
def prior_count_set():
    """257 priors on 300 poses, three of them NOT_PD (H = -I), and one factor"""
    rng = np.random.default_rng(6)
    P = 300
    x = _poses(rng, P)
    priors = []
    for q in range(257):
        pr = _edge_prior(rng, x, int(rng.integers(P)), float(rng.uniform(0, 3.0)), mr.AXES[q % 5],
                         rng.normal(0, 0.5, 3), LEVERS[q % 3], "gnss" if q % 2 else "full")
        if q in (7, 100, 255):
            pr["H"] = -np.eye(6)
        priors.append(pr)
    factors = [pg.make_factor(rng, x, [9, 4], noise=0.01)]
    pb = [None if np.all(p["H"] == -np.eye(6)) else mr.prior_base(x, p) for p in priors]
    return P, x, factors, [mr.factor_base(x, f) for f in factors], priors, pb


@pytest.mark.parametrize("n", [1, 255, 256, 257])
def test_prior_counts_with_not_pd_interleaved(prior_count_set, n):
    P, x, factors, fb, priors, pb = prior_count_set
    _pin(f"{n} priors", P, x, factors, fb, priors=priors[:n], pbase=pb[:n], dense=False)


# ---------------- factor shapes and counts ----------------
@pytest.fixture(scope="module", params=[1.0, 1e4])
def shape_set(request):
    """factors of 32 (scattered), 31 (descending), 3 (ascending) and 2 (descending) slots, and 16 factors sharing the
    pose pair (5, 9) in both orders, some with a third pose between them; positions of size request.param"""
    rng = np.random.default_rng(7)
    P = 64
    truth = _poses(rng, P, (request.param,))
    sets = [list(rng.permutation(P)[:32]), sorted(rng.choice(P, 31, replace=False).tolist(), reverse=True),
            sorted(rng.choice(P, 3, replace=False).tolist()), [40, 12]]
    for q in range(16):
        third = [int(v) for v in rng.choice([i for i in range(P) if i not in (5, 9)], q % 3, replace=False)]
        sets.append(([5] + third + [9]) if q % 2 else ([9] + third + [5]))
    factors = [pg.make_factor(rng, truth, s, noise=0.05) for s in sets]
    x = pg.perturb(rng, truth, 0.2, 0.5)
    return P, x, factors, [mr.factor_base(x, f) for f in factors]


def test_factor_shapes_and_slot_orders(shape_set):
    P, x, factors, bases = shape_set
    _pin(f"factor shapes, |p| ~ {np.abs(x[:, 9:]).max():.0e}", P, x, factors, bases)


def test_factor_shapes_with_mixed_losses(shape_set):
    P, x, factors, bases = shape_set
    kinds = [[mr.HUBER, mr.CAUCHY, mr.TRIVIAL][q % 3] for q in range(len(factors))]
    fk, fs = _loss_for(bases, kinds)
    _pin("factor shapes, mixed losses", P, x, factors, bases, fk, fs)


@pytest.fixture(scope="module")
def count_set():
    """1000 two- and three-slot factors over 2000 poses in scattered order, every 37th NOT_PD (H negated)"""
    rng = np.random.default_rng(8)
    P = 2000
    truth = _poses(rng, P, (1.0, 1e2))
    factors = []
    for q in range(1000):
        idx = [int(v) for v in rng.choice(P, 2 + q % 2, replace=False)]
        f = pg.make_factor(rng, truth, idx, noise=0.05)
        if q % 37 == 5:
            f["H"] = -f["H"]
        factors.append(f)
    x = pg.perturb(rng, truth, 0.05, 0.2)
    return P, x, factors, [mr.factor_base(x, f) if pg.pd_ok(f["H"]) else None for f in factors]


@pytest.mark.parametrize("n", [1, 255, 256, 257, 1000])
def test_factor_counts_with_not_pd_interleaved(count_set, n):
    P, x, factors, bases = count_set
    if n <= 257:  # the first n factors on their own poses, so that the dense context can be compared as well
        used = sorted({int(i) for f in factors[:n] for i in f["poses"]})
        fs = [dict(f, poses=np.searchsorted(used, f["poses"]).astype(np.int32)) for f in factors[:n]]
        _pin(f"{n} factors", len(used), x[used], fs, bases[:n])
    _pin(f"{n} factors over {P} poses", P, x, factors[:n], bases[:n], dense=False)


# ---------------- the Huber kink ----------------
def _kink_scale(s):
    """an fp64 c with fl(c c) == s, or None"""
    c = np.sqrt(s)
    for _ in range(8):
        for cand in (c, np.nextafter(c, np.inf), np.nextafter(c, 0.0)):
            if cand * cand == s:
                return cand
        c = np.nextafter(c, np.inf)
    return None


def test_huber_on_the_kink(angle_set, prior_angle_set):
    """one factor and one prior with s exactly c^2 in fp64: w = 1 exactly (the quadratic branch), and the whole
    evaluation pinned to the reference"""
    P, x, factors, bases = angle_set
    c = balm_b200.Context(P)
    c.set_pose_factors(factors)
    s, _ = c.factor_residuals(x)
    c.close()
    q, ck = next((q, _kink_scale(v)) for q, v in enumerate(s) if v > 1e-6 and _kink_scale(v) is not None)
    fk = [mr.HUBER] * len(factors)
    fs = [np.sqrt(max(float(b["s"]), 1e-30)) * 2.0 for b in bases]
    fs[q] = ck
    sd, wd = _pin("factor Huber kink", P, x, factors, bases, fk, fs)[0]
    assert sd[q] == ck * ck and wd[q] == 1.0
    P, x, factors, fb, priors, pb = prior_angle_set
    c = balm_b200.Context(P)
    c.set_pose_factors(factors)
    c.set_pose_priors(priors)
    s, _ = c.prior_residuals(x)
    c.close()
    q, ck = next((q, _kink_scale(v)) for q, v in enumerate(s) if v > 1e-6 and _kink_scale(v) is not None)
    pk = [mr.HUBER] * len(priors)
    ps = [np.sqrt(max(float(b["s"]), 1e-30)) * 0.5 for b in pb]
    ps[q] = ck
    sd, wd = _pin("prior Huber kink", P, x, factors, fb, priors=priors, pbase=pb, pk=pk, ps=ps)[1]
    assert sd[q] == ck * ck and wd[q] == 1.0


# ---------------- asymmetric factor Hessians ----------------
def _asymmetric(H, rel, seed=0):
    """H plus rel max |H| times an unsymmetric standard normal matrix: symmetric to about rel of its max |entry| only"""
    return H + rel * np.abs(H).max() * np.random.default_rng(seed).standard_normal(H.shape)


def test_asymmetric_factor_hessians_are_refused_by_every_registration():
    """H_f off symmetric by 1e-10 of its max |entry| is refused by balm_set_pose_factors, balm_spg_set_factors and
    balm_block_set_factors, and the previous set stays in force; off by 1e-15 (the rounding of J^T J arithmetic) and
    odometry_factors' H are accepted"""
    rng = np.random.default_rng(9)
    P = 12
    truth = _poses(rng, P, (3.0,))
    factors = [pg.make_factor(rng, truth, s, noise=0.01) for s in ([0, 3, 5], [5, 1], [7, 2, 9, 11])]
    factors += balm_b200.odometry_factors(truth[:4], np.eye(6))
    x = pg.perturb(rng, truth, 0.05, 0.2)
    dense, sparse, blocks = balm_b200.Context(P), balm_b200.PoseGraph(P), balm_b200.Context(P, 0, L.PREC_BLOCKS)
    routes = [(dense, dense.set_pose_factors, "balm_set_pose_factors", lambda: dense.pose_graph_evaluate(x)),
              (sparse, sparse.set_pose_factors, "balm_spg_set_factors", lambda: sparse.pose_graph_evaluate(x)),
              (blocks, blocks.set_block_factors, "balm_block_set_factors",
               lambda: (*blocks.evaluate(x), blocks.download_blocks()))]
    for h, register, who, evaluate in routes:
        assert register(factors) == [L.OK] * len(factors)
        if h is blocks:
            h.set_voxels(np.zeros(1, np.int64), np.zeros(0, np.int32), np.zeros((0, 10)), np.zeros(0))
        before = evaluate()
        bad = [dict(f) for f in factors]
        bad[2] = dict(bad[2], H=_asymmetric(bad[2]["H"], 1e-10))
        with pytest.raises(balm_b200.BalmError) as e:
            register(bad)
        assert e.value.status == L.ERR_INVALID and who in str(e.value) and "not symmetric" in str(e.value)
        assert all(np.array_equal(u, v) for u, v in zip(before, evaluate()))
        near = [dict(f, H=_asymmetric(f["H"], 1e-15, q)) for q, f in enumerate(factors)]
        assert not any(np.array_equal(f["H"], f["H"].T) for f in near)
        assert register(near) == [L.OK] * len(factors)
        h.close()

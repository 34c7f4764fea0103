"""Robust pose factors on the device (balm_set_factor_loss, balm_spg_set_factor_loss, balm_factor_residuals): the no-op
of a trivial loss, evaluation and LM parity with robust_factors_ref on the dense context, PoseGraph and a PREC_BLOCKS
context, the outlier scenes at size, covariances of the reweighted H, refusals, lifetime, repeatability and memory."""
import ctypes as C

import numpy as np
import pytest

import balm_b200
import block_hessian_ref as bref
import pose_graph_ref as pgr
import robust_factors_ref as rr
from balm_b200 import _lib as L
from test_gpu_block_hessian import _ctx
from test_gpu_sparse_covariance import _dense_sigma

pytestmark = pytest.mark.gpu


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _corridor_factors(sc, seed, n_false=1):
    """odometry, true closures (a - 30, a) and n_false identity closures between poses 40 apart on a voxel corridor"""
    rng = np.random.default_rng(seed)
    gt, N = sc["poses_gt"], sc["n_poses"]
    fs = rr.noisy_relative(rng, gt, [(a, a + 1) for a in range(N - 1)], rr.info(*rr.ODO_NOISE), *rr.ODO_NOISE)
    fs += rr.noisy_relative(rng, gt, [(a - 30, a) for a in range(30, N, 10)], rr.info(*rr.LOOP_NOISE), *rr.LOOP_NOISE)
    for a in range(n_false):
        f = balm_b200.odometry_factors(np.stack([gt[a], gt[a]]), rr.info(*rr.LOOP_NOISE))[0]
        f["poses"] = np.array([a, a + 40], dtype=np.int32)
        fs.append(f)
    return fs


def _small_graph(seed=0):
    """a 60-pose outlier scene (two laps of 30) at perturbed poses and a scale with factors on both sides of c^2"""
    sc = rr.outlier_scene(60, seed, lap=30, radius=6.0, every=3, min_dist=6.0)
    x = pgr.perturb(np.random.default_rng(seed), sc["gt"], 0.003, 0.03)
    s, _ = rr.residuals(x, sc["all"], np.zeros(len(sc["all"]), np.int32), np.ones(len(sc["all"])))
    return sc, x, float(np.sqrt(np.median(s))), s


def _losses(n, c):
    return {"huber": ("huber", c), "cauchy": ("cauchy", c),
            "mixed": ((["trivial", "huber", "cauchy"] * n)[:n], c * np.linspace(0.5, 2.0, n))}


def _dense(N, fs):
    c = balm_b200.Context(N, 0, L.PREC_FP64)
    assert c.set_pose_factors(fs) == [L.OK] * len(fs)
    return c


def _spg(N, fs):
    s = balm_b200.PoseGraph(N)
    assert s.set_pose_factors(fs) == [L.OK] * len(fs)
    return s


def _blocks(N, fs):
    c = balm_b200.Context(N, 0, L.PREC_BLOCKS)
    c.set_voxels(np.zeros(1, np.int64), np.zeros(0, np.int32), np.zeros((0, 10)), np.zeros(0))
    assert c.set_block_factors(fs) == [L.OK] * len(fs)
    return c


def _all_outputs(h, x, kind):
    """everything a handle computes from its factors at x: evaluation, LM poses and trace, covariance"""
    lm = dict(max_iter=6, gauge_mode=2, want_per_iter=True)
    if kind == "dense":
        H, g, r = h.pose_graph_evaluate(x)
        p, t = h.pose_graph_iter(x, **lm)
        return [H, g, r, p, [{k: v for k, v in d.items() if k != "poses"} for d in t], [d["poses"] for d in t]]
    if kind == "spg":
        _, b, g, r = h.pose_graph_evaluate(x)
        p, t = h.pose_graph_iter(x, **lm)
        return [b, g, r, p, [{k: v for k, v in d.items() if k != "poses"} for d in t], [d["poses"] for d in t],
                h.covariance(x)[1]]
    H, g, r = h.evaluate(x)
    b = h.download_blocks()
    p, t, per = h.damping_iter(x, min_planes_per_pose=0, **lm)
    return [H, g, r, b, p, t, per, h.block_covariance(x)[1]]


def _same(a, b):
    assert len(a) == len(b)
    for u, v in zip(a, b):
        if isinstance(u, list) and u and isinstance(u[0], dict):
            assert u == v
        else:
            assert np.array_equal(np.asarray(u), np.asarray(v))


# ---------------------------------------------------------------- 1. no-op ------------------------------------------
@pytest.mark.parametrize("kind", ["dense", "spg", "blocks"])
def test_trivial_loss_is_a_no_op(kind):
    sc, x, c, s = _small_graph(1)
    fs, N = sc["all"], 60
    make = {"dense": _dense, "spg": _spg, "blocks": _blocks}[kind]
    ref = _all_outputs(make(N, fs), x, kind)
    h = make(N, fs)
    h.set_factor_loss(["trivial"] * len(fs), np.full(len(fs), np.nan))  # a trivial factor's scale is ignored
    _same(_all_outputs(h, x, kind), ref)
    h.set_factor_loss("cauchy", c)
    h.set_factor_loss("trivial")  # reset
    _same(_all_outputs(h, x, kind), ref)
    # Huber with every s below c^2: the robust kernels with w = 1 exactly give the quadratic terms bitwise
    h.set_factor_loss("huber", 2 * np.sqrt(s.max()))
    assert np.array_equal(h.factor_residuals(x)[1], np.ones(len(fs)))
    _same(_all_outputs(h, x, kind)[:3], ref[:3])


def test_mixed_set_trivial_factors_are_bitwise():
    """robust factors on poses 0..9 only: every block pair and gradient entry away from them is bitwise the quadratic"""
    sc, x, c, _ = _small_graph(2)
    fs, N = sc["all"], 60
    robust = [any(int(i) < 10 for i in f["poses"]) for f in fs]
    s0 = _spg(N, fs)
    pairs, b0, g0, r0 = s0.pose_graph_evaluate(x)
    s1 = _spg(N, fs)
    s1.set_factor_loss(["cauchy" if r else "trivial" for r in robust], 0.1 * c)
    _, b1, g1, r1 = s1.pose_graph_evaluate(x)
    touched = set()
    for f, r in zip(fs, robust):
        if r:
            touched |= {int(i) for i in f["poses"]}
    away = np.array([int(i) not in touched and int(j) not in touched for i, j in pairs])
    assert away.any() and (~away).any()
    assert np.array_equal(b1[away], b0[away]) and not np.array_equal(b1[~away], b0[~away])
    keep = np.repeat([i not in touched for i in range(N)], 6)
    assert np.array_equal(g1[keep], g0[keep]) and r1 != r0


# ---------------------------------------------------------------- 2. evaluation parity -----------------------------
@pytest.mark.parametrize("name", ["huber", "cauchy", "mixed"])
def test_evaluation_against_the_restatement(name):
    sc, x, c, s = _small_graph(3)
    fs, N = sc["all"], 60
    assert (s > c * c).any() and (s < c * c).any()
    kind, scale = _losses(len(fs), c)[name]
    kinds, scales = rr.loss_arrays(len(fs), kind, scale)
    Hr, gr, rr_ = rr.evaluate(x, fs, N, kinds, scales)
    sr, wr = rr.residuals(x, fs, kinds, scales)
    d = _dense(N, fs)
    d.set_factor_loss(kind, scale)
    H, g, r = d.pose_graph_evaluate(x)
    assert np.abs(H - Hr).max() <= 1e-12 * np.abs(Hr).max()
    assert np.abs(g - gr).max() <= 1e-12 * np.abs(gr).max()
    assert abs(r - rr_) <= 1e-12 * abs(rr_)
    for h in (d, _spg(N, fs)):
        h.set_factor_loss(kind, scale)
        sd, wd = h.factor_residuals(x)
        assert np.abs(sd - sr).max() <= 1e-12 * np.abs(sr).max() and np.abs(wd - wr).max() <= 1e-12
    # PoseGraph's blocks are bitwise the dense context's entries; a blocks context bitwise voxels + PoseGraph
    spg = _spg(N, fs)
    spg.set_factor_loss(kind, scale)
    pairs, blocks, g2, r2 = spg.pose_graph_evaluate(x)
    assert np.array_equal(blocks, bref.blocks_of(H, pairs)) and np.array_equal(g2, g) and r2 == r
    vsc = bref.corridor(N, w=4, planes_per_pose=30, seed=41)
    cb, c0 = _ctx(vsc, L.PREC_BLOCKS), _ctx(vsc, L.PREC_BLOCKS)
    cb.set_block_factors(fs)
    cb.set_factor_loss(kind, scale)
    Hb, gb, rb = cb.evaluate(x)
    bb, pb = cb.download_blocks(), cb.block_structure(want_pairs=True)["pair_list"]
    _, g0, r0 = c0.evaluate(x, want_H=False)
    b0, p0 = c0.download_blocks(), c0.block_structure(want_pairs=True)["pair_list"]
    idx = {(int(i), int(j)): q for q, (i, j) in enumerate(pb)}
    exp = np.zeros_like(bb)
    exp[[idx[tuple(t)] for t in p0.tolist()]] += b0
    exp[[idx[tuple(t)] for t in pairs.tolist()]] += blocks
    assert np.array_equal(bb, exp) and np.array_equal(gb, g0 + g2) and rb == r0 + r2


# ---------------------------------------------------------------- 3. LM parity -------------------------------------
def _lm_per_iter(per, trace):
    return [t["accepted"] for t in trace], np.array(per)


def test_pose_graph_lm_against_the_restatement():
    P = 200
    sc = rr.outlier_scene(P, 1)
    fs, c = sc["all"], rr.cauchy_scale()
    kinds, scales = rr.loss_arrays(len(fs), "cauchy", c)
    _, tr, per = rr.lm(sc["x0"], fs, P, kinds, scales, max_iter=10)
    acc = [t["accepted"] for t in tr]
    for h in (_dense(P, fs), _spg(P, fs)):
        h.set_factor_loss("cauchy", c)
        _, t = h.pose_graph_iter(sc["x0"], max_iter=10, gauge_mode=2, want_per_iter=True)
        assert [d["accepted"] for d in t] == acc
        gap = max(np.abs(d["poses"] - p).max() for d, p in zip(t, per))
        print(f"{type(h).__name__}: {len(t)} iterations, largest pose gap {gap:.2e}")
        assert gap < 1e-9


def test_blocks_damping_iter_against_the_restatement():
    sc = bref.corridor(80, w=4, planes_per_pose=30, seed=42)
    fs = _corridor_factors(sc, 3, n_false=2)
    c = rr.cauchy_scale()
    kinds, scales = rr.loss_arrays(len(fs), "cauchy", c)
    cb = _ctx(sc, L.PREC_BLOCKS)
    cb.set_block_factors(fs)
    cb.set_factor_loss("cauchy", c)
    _, tb, per_b = cb.damping_iter(sc["poses_init"], max_iter=8, gauge_mode=2, min_planes_per_pose=0,
                                   want_per_iter=True)
    cd = _ctx(sc, L.PREC_FP64)
    x = np.array(sc["poses_init"], copy=True)
    u, v, calc, acc, per = 0.01, 2.0, True, [], []
    for _ in range(8):  # pose_graph_ref.lm's rule on fp64 voxels + the robust factors
        if calc:
            H, g, r1 = cd.evaluate(x)
            Hf, gf, rf = rr.evaluate(x, fs, cb.N, kinds, scales)
            H, g, r1 = H + Hf, g + gf, r1 + rf
        D = np.diag(H).copy()
        dx = np.linalg.solve(H + u * np.diag(D), -g)
        q1 = 0.5 * dx @ (u * D * dx - g)
        xt = pgr.pose_update(x, dx)
        r2 = cd.residual(xt) + rr.cost(xt, fs, kinds, scales)
        q = r1 - r2
        if q > 0:
            x = xt
            u *= max(1 - (2 * q / q1 - 1) ** 3, 1.0 / 3.0)
            v, calc = 2.0, True
        else:
            u, v, calc = u * v, 2 * v, False
        acc.append(q > 0)
        per.append(x.copy())
        if abs(r1 - r2) / r1 < 1e-6:
            break
    assert [t["accepted"] for t in tb] == acc
    gap = np.abs(per_b - np.array(per)).max()
    print(f"blocks corridor: largest per-iteration pose gap {gap:.2e}")
    assert gap < 1e-9


# ---------------------------------------------------------------- 4. outcome at size -------------------------------
def test_outlier_scene_2000_poses():
    P = 2000
    sc = rr.outlier_scene(P, 1)
    c = rr.cauchy_scale()
    out = {}
    for name, fs, kind in [("clean", sc["clean"], "trivial"), ("trivial", sc["all"], "trivial"),
                           ("cauchy", sc["all"], "cauchy")]:
        s = _spg(P, fs)
        s.set_factor_loss(kind, c)
        x, t = s.pose_graph_iter(sc["x0"], max_iter=60, gauge_mode=2)
        out[name] = (rr.max_error(x, sc["gt"]), len(t), s.factor_residuals(x)[1])
    e0, e1, e2 = (out[k][0] for k in ("clean", "trivial", "cauchy"))
    no, nt = len(sc["odo"]), len(sc["true"])
    w = out["cauchy"][2]
    print(f"2000 poses: max error outlier-free {e0:.3f} m ({out['clean'][1]} it), trivial {e1:.3f} m "
          f"({out['trivial'][1]} it), Cauchy {e2:.3f} m ({out['cauchy'][1]} it); w true >= {w[no:no + nt].min():.3f}, "
          f"w false <= {w[no + nt:].max():.2e}")
    assert e1 > 10 * e0 and e2 < 1.5 * e0
    assert w[no + nt:].max() < w[no:no + nt].min()


def test_blocks_corridor_1000_poses():
    sc = bref.corridor(1000, w=8, planes_per_pose=30, pts=6, seed=43)
    N, gt = sc["n_poses"], sc["poses_gt"]
    rng = np.random.default_rng(44)
    odo = rr.noisy_relative(rng, gt, [(a, a + 1) for a in range(N - 1)], rr.info(*rr.ODO_NOISE), *rr.ODO_NOISE)
    true = rr.noisy_relative(rng, gt, [(a - 300, a) for a in range(300, N, 25)], rr.info(*rr.LOOP_NOISE),
                             *rr.LOOP_NOISE)
    false = []
    for a in rng.choice(N - 400, 7, replace=False):
        f = balm_b200.odometry_factors(np.stack([gt[a], gt[a]]), rr.info(*rr.LOOP_NOISE))[0]
        f["poses"] = np.array([a, a + 400], dtype=np.int32)
        false.append(f)
    c = rr.cauchy_scale()
    err = {}
    for name, fs, kind in [("clean", odo + true, "trivial"), ("trivial", odo + true + false, "trivial"),
                           ("cauchy", odo + true + false, "cauchy")]:
        cb = _ctx(sc, L.PREC_BLOCKS)
        cb.set_block_factors(fs)
        cb.set_factor_loss(kind, c)
        x, t, _ = cb.damping_iter(sc["poses_init"], max_iter=30, gauge_mode=2, min_planes_per_pose=0)
        err[name] = rr.max_error(x, gt)
        print(f"corridor 1000 {name}: max error {err[name]:.3f} m after {len(t)} iterations")
        cb.close()
    assert err["cauchy"] < 1.5 * err["clean"] and err["trivial"] > 1.5 * err["clean"]


# ---------------------------------------------------------------- 5. covariance ------------------------------------
def test_covariance_of_the_reweighted_hessian():
    sc, x, c, _ = _small_graph(4)
    fs, N = sc["all"], 60
    kinds, scales = rr.loss_arrays(len(fs), "cauchy", c)
    s = _spg(N, fs)
    s.set_factor_loss("cauchy", c)
    pairs, cov = s.covariance(x)
    S, kappa = _dense_sigma(rr.evaluate(x, fs, N, kinds, scales)[0], 0)
    err = np.abs(cov - bref.blocks_of(S, pairs)).max() / np.abs(cov).max()
    print(f"PoseGraph: kappa {kappa:.1e}, error {err:.1e}")
    assert err <= max(1e-9, 10 * kappa * 1e-12)
    vsc = bref.corridor(60, w=4, planes_per_pose=30, seed=31)
    fs = _corridor_factors(vsc, 5)
    kinds, scales = rr.loss_arrays(len(fs), "huber", rr.cauchy_scale())
    cb = _ctx(vsc, L.PREC_BLOCKS)
    cb.set_block_factors(fs)
    cb.set_factor_loss("huber", rr.cauchy_scale())
    x, _, _ = cb.damping_iter(vsc["poses_init"], max_iter=10, gauge_mode=2, min_planes_per_pose=0)
    w = cb.factor_residuals(x)[1]
    assert w.min() < 0.5 and w.max() == 1.0  # the false closure is down-weighted, the rest quadratic
    pairs, cov = cb.block_covariance(x)
    cd = _ctx(vsc, L.PREC_FP64)
    S, kappa = _dense_sigma(cd.evaluate(x)[0] + rr.evaluate(x, fs, cb.N, kinds, scales)[0], 0)
    err = np.abs(cov - bref.blocks_of(S, pairs)).max() / np.abs(cov).max()
    print(f"blocks: kappa {kappa:.1e}, error {err:.1e}")
    assert err <= max(1e-9, 10 * kappa * 1e-12)


# ---------------------------------------------------------------- 6. refusals and lifetime -------------------------
def test_refusals_keep_the_previous_loss():
    sc, x, c, _ = _small_graph(5)
    fs, N = sc["all"], 60
    F = len(fs)
    lib = L.lib()
    for h, set_fn, res_fn in [(_dense(N, fs), lib.balm_set_factor_loss, lib.balm_factor_residuals),
                              (_spg(N, fs), lib.balm_spg_set_factor_loss, lib.balm_spg_factor_residuals)]:
        h.set_factor_loss("huber", c)
        before = h.factor_residuals(x)
        k = np.full(F, L.LOSS_CAUCHY, np.int32)
        sc_ = np.full(F, c)
        bad = [(None, F, k, sc_), (h._h, F - 1, k, sc_), (h._h, F + 1, k, sc_)]
        for kv in (3, -1):
            kk = k.copy()
            kk[7] = kv
            bad.append((h._h, F, kk, sc_))
        for sv in (0.0, -1.0, np.nan, np.inf):
            ss = sc_.copy()
            ss[4] = sv
            bad.append((h._h, F, k, ss))
        bad.append((h._h, F, k, None))
        for hh, n, kk, ss in bad:
            assert set_fn(hh, n, _p(kk), _p(ss)) == L.ERR_INVALID
        s_, w_ = h.factor_residuals(x)
        assert np.array_equal(s_, before[0]) and np.array_equal(w_, before[1])
        assert res_fn(h._h, None, None, None) == L.ERR_INVALID and res_fn(None, _p(x), None, None) == L.ERR_INVALID
        # a trivial factor's scale is ignored, and NULL scale is fine when every kind is trivial
        ss = sc_.copy()
        ss[0] = np.nan
        kk = k.copy()
        kk[0] = L.LOSS_TRIVIAL
        assert set_fn(h._h, F, _p(kk), _p(ss)) == L.OK
        assert set_fn(h._h, F, _p(np.zeros(F, np.int32)), None) == L.OK
    # no registered factor set
    assert lib.balm_set_factor_loss(balm_b200.Context(N, 0, L.PREC_FP64)._h, 0, None, None) == L.ERR_INVALID
    assert lib.balm_spg_set_factor_loss(balm_b200.PoseGraph(N)._h, 0, None, None) == L.ERR_INVALID
    cb = balm_b200.Context(N, 0, L.PREC_BLOCKS)
    assert lib.balm_set_factor_loss(cb._h, 0, None, None) == L.ERR_INVALID
    assert lib.balm_factor_residuals(cb._h, _p(x), None, None) == L.ERR_INVALID


def test_lifetime_not_pd_repeatability_memory():
    sc, x, c, _ = _small_graph(6)
    fs, N = sc["all"], 60
    F = len(fs)
    # re-registration resets the loss (all three set calls)
    for make, reg in [(_dense, "set_pose_factors"), (_spg, "set_pose_factors"), (_blocks, "set_block_factors")]:
        h, h0 = make(N, fs), make(N, fs)
        h.set_factor_loss("cauchy", c)
        assert not np.array_equal(h.factor_residuals(x)[1], np.ones(F))
        getattr(h, reg)(fs)
        assert np.array_equal(h.factor_residuals(x)[1], np.ones(F))
        e = h.evaluate(x) if reg == "set_block_factors" else h.pose_graph_evaluate(x)
        e0 = h0.evaluate(x) if reg == "set_block_factors" else h0.pose_graph_evaluate(x)
        _same(list(e), list(e0))
    # blocks: detach resets; voxel re-registration keeps the loss
    vsc = bref.corridor(60, w=4, planes_per_pose=30, seed=31)
    vf = _corridor_factors(vsc, 7, n_false=2)
    cb = _ctx(vsc, L.PREC_BLOCKS)
    cb.set_block_factors(vf)
    cb.set_factor_loss("cauchy", c)
    H1, g1, r1 = cb.evaluate(vsc["poses_init"])
    cb.set_voxels(vsc["row_ptr"], vsc["pose_idx"], vsc["obs10"], vsc["coe"])
    H2, g2, r2 = cb.evaluate(vsc["poses_init"])
    assert np.array_equal(H1, H2) and np.array_equal(g1, g2) and r1 == r2
    cb.set_block_factors([])
    with pytest.raises(balm_b200.BalmError) as e:
        cb.set_factor_loss("cauchy", c)
    assert e.value.status == L.ERR_INVALID
    cb.set_block_factors(vf)
    assert np.array_equal(cb.factor_residuals(vsc["poses_init"])[1], np.ones(len(vf)))
    # NOT_PD factors report s = w = 0, with and without a loss
    singular = dict(fs[0], H=np.zeros((12, 12)))
    s = balm_b200.PoseGraph(N)
    st = s.set_pose_factors(fs + [singular])
    assert st[-1] == L.ERR_NOT_PD
    for kind in ("trivial", "cauchy"):
        s.set_factor_loss(kind, c)
        sv, wv = s.factor_residuals(x)
        assert sv[-1] == 0 and wv[-1] == 0 and (sv[:-1] > 0).all() and (wv[:-1] > 0).all()
    # memory: exactly 28 bytes per factor while a loss is set
    s = _spg(N, fs)
    b0 = s.structure()["device_bytes"]
    s.set_factor_loss("cauchy", c)
    assert s.structure()["device_bytes"] == b0 + 28 * F
    s.set_factor_loss("trivial")
    assert s.structure()["device_bytes"] == b0
    cb = _ctx(vsc, L.PREC_BLOCKS)
    cb.set_block_factors(vf)
    b0 = cb.block_structure()["device_bytes"]
    cb.set_factor_loss("huber", c)
    assert cb.block_structure()["device_bytes"] == b0 + 28 * len(vf)
    # two runs are bitwise equal
    runs = []
    for _ in range(2):
        s = _spg(N, fs)
        s.set_factor_loss(*_losses(F, c)["mixed"])
        runs.append(_all_outputs(s, x, "spg") + list(s.factor_residuals(x)))
    _same(runs[0], runs[1])

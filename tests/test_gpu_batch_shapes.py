"""Batched bundle adjustment and pose covariance (batch.cu, balm_b200.Batch) at the shapes where the batch's index
arithmetic matters, every problem checked against the CPU oracle (oracle/oracle_py.py), the numpy restatement of the
covariance (tests/numpy_cov.py) and a fp64 Context holding only that problem:
- more than one 64-column tile (N_p >= 11) together with more than one 768-row SYRK chunk, in the Hessian's row layout
  (3 rows per voxel) and the covariance's (8 rows per voxel), and the tile, row-chunk and sweep-chunk edges around them;
- more problems than one 128-thread block of the per-problem kernels (batch_lm_kernel, batch_init_kernel, fill_kernel),
  more poses than one block of batch_gauge_kernel, and more voxels than two passes of batch_stats_kernel's grid.
Tolerances are the suite's: tests/test_gpu_parity.py and test_gpu_batch.py for H, g, r and the LM,
tests/test_gpu_batch_covariance.py for Rcov_raw and Rcov."""
import numpy as np
import pytest

import numpy_cov as nc
import scenes
from oracle import oracle_py as orc

IDENT = np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0.0])
PN = 0.01

# batch.cu's work split (test_shape_table_covers_the_boundaries derives the boundaries below from it)
CHUNK = 32           # voxels per warp of the observation sweep
ROWS = 768           # rows per SYRK work item (row chunk)
TILE = 64            # SYRK output tile; G' / covariance rows are padded to a multiple of it
KB = 16              # rows per shared-memory stage of the SYRK
STATS_WARPS = 8      # batch_stats_kernel: one warp per voxel, 8 per block, at most 8 blocks per SM, grid-stride loop
STATS_BLOCKS_PER_SM = 8
BLOCK = 128          # threads per block of batch_lm_kernel, batch_init_kernel, fill_kernel (per problem) and
                     # batch_gauge_kernel (per pose)
H100_SMS = 132       # the most SMs of an H100 (SXM5); on fewer SMs one stats pass covers fewer voxels

# The Hessian's boundary problems, in one batch: N_p at the tile edges, voxel counts at the row-chunk edges
HESS = [
    dict(n_poses=10, n_planes=256, seed=301),                           # 60 of 64 columns; exactly one chunk
    dict(n_poses=11, n_planes=257, seed=302, with_fix=True),            # pose 10 on tiles 0 | 1; a 3-row second chunk
    dict(n_poses=21, n_planes=512, seed=303, drop=0.4, with_fix=True),  # 126 of 128 columns; two full chunks
    dict(n_poses=22, n_planes=700, seed=304, drop=0.3),                 # pose 21 on tiles 1 | 2; 3 chunks, the last partial
    dict(n_poses=32, n_planes=300, seed=305, with_fix=True),            # three full tiles; two chunks
]
HESS_ALONE = (1, 4)  # the problems also run in a batch of their own

# The covariance's boundary problems (8 rows per voxel), all with fix clusters, as tests/test_gpu_batch_covariance.py
COV = [
    dict(n_poses=4, n_planes=96, seed=311),              # exactly one chunk
    dict(n_poses=11, n_planes=97, seed=312),             # 3 upper tiles x (one full chunk + 8 rows)
    dict(n_poses=6, n_planes=192, seed=313, drop=0.3),   # two full chunks
    dict(n_poses=12, n_planes=250, seed=314, drop=0.4),  # 3 upper tiles x 3 chunks, the last partial
]
COV_PTS = 20


def _workload():
    """An HBA bottom layer's shape: 150 windows with fix clusters, mostly 4 .. 12 poses and 100 .. 140 planes, dense and
    ragged, and three of 32 poses x 300+ planes, two of them behind the first 128 problems."""
    out = []
    for i in range(150):
        if i in (31, 129, 149):
            out.append(dict(n_poses=32, n_planes=330 if i == 149 else 300, seed=400 + i, drop=0.3 if i == 129 else 0.0))
        else:
            out.append(dict(n_poses=4 + (5 * i) % 9, n_planes=100 + (37 * i) % 41, seed=400 + i,
                            drop=0.3 if i % 3 == 1 else 0.0))
    return out


WORK = _workload()
WORK_PTS = 8
WORK_ALONE = (0, 127, 128, 129, len(WORK) - 1)  # each also run in a batch of its own
WORK_NUMPY_COV = (0, 128, int(np.argmax([kw["n_poses"] * kw["n_planes"] for kw in WORK])))


def _layout(n_poses, n_voxels, rows_per_voxel):
    """What batch.cu's reg_layout / syrk_items make of one problem."""
    n = 6 * n_poses
    ldp = -(-n // TILE) * TILE
    nt = ldp // TILE
    rows = rows_per_voxel * n_voxels
    chunks = -(-rows // ROWS)
    return dict(n=n, ldp=ldp, pad=ldp - n, upper_tiles=nt * (nt + 1) // 2, chunks=chunks,
                last_rows=rows - (chunks - 1) * ROWS, last_pose_tiles=(6 * (n_poses - 1) // TILE, (n - 1) // TILE),
                last_sweep=n_voxels - (-(-n_voxels // CHUNK) - 1) * CHUNK)


def test_shape_table_covers_the_boundaries():
    """The tables above hold every boundary the GPU tests are meant to cross (checked from (N_p, n_planes) alone;
    make_scene gives one voxel per plane)."""
    h = {(kw["n_poses"], kw["n_planes"]): _layout(kw["n_poses"], kw["n_planes"], 3) for kw in HESS}
    tiles = {np_: l for (np_, _), l in h.items()}
    # tile shapes
    assert tiles[10]["n"] == 60 and tiles[10]["ldp"] == 64 and tiles[10]["pad"] == 4 and tiles[10]["upper_tiles"] == 1
    assert tiles[11]["last_pose_tiles"] == (0, 1)
    assert tiles[21]["n"] == 126 and tiles[21]["ldp"] == 128 and tiles[21]["pad"] == 2
    assert tiles[22]["last_pose_tiles"] == (1, 2)
    assert tiles[32]["pad"] == 0 and tiles[32]["ldp"] == 3 * TILE and tiles[32]["upper_tiles"] == 6
    # the Hessian's row chunks
    nv = {m: l for (_, m), l in h.items()}
    assert nv[256]["chunks"] == 1 and nv[256]["last_rows"] == ROWS
    assert nv[257]["chunks"] == 2 and nv[257]["last_rows"] == 3 and nv[257]["last_rows"] < KB
    assert nv[257]["last_sweep"] == 1
    assert nv[512]["chunks"] == 2 and nv[512]["last_rows"] == ROWS
    assert any(l["chunks"] == 3 and l["last_rows"] < ROWS for l in h.values())
    # the covariance's row chunks
    c = {kw["n_planes"]: _layout(kw["n_poses"], kw["n_planes"], 8) for kw in COV}
    assert c[96]["chunks"] == 1 and c[96]["last_rows"] == ROWS
    assert c[97]["chunks"] == 2 and c[97]["last_rows"] == 8
    assert c[192]["chunks"] == 2 and c[192]["last_rows"] == ROWS
    assert any(m > 192 and m % 96 != 0 for m in c)
    # more than one upper tile and more than one chunk in the same problem, in both row layouts
    assert any(l["upper_tiles"] > 1 and l["chunks"] > 1 for l in h.values())
    assert any(l["upper_tiles"] > 1 and l["chunks"] > 1 for l in c.values())
    # many problems: a second block of every per-problem and per-pose kernel, at least three stats passes
    B = len(WORK)
    P = sum(kw["n_poses"] for kw in WORK)
    M = sum(kw["n_planes"] for kw in WORK)
    assert B > BLOCK and P > BLOCK and M > 2 * STATS_WARPS * STATS_BLOCKS_PER_SM * H100_SMS
    large = [i for i, kw in enumerate(WORK) if kw["n_poses"] == 32 and kw["n_planes"] > ROWS // 3]
    assert any(i >= BLOCK for i in large) and all(0 <= i < B for i in WORK_ALONE + WORK_NUMPY_COV)
    assert {0, BLOCK - 1, BLOCK, BLOCK + 1, B - 1} <= set(WORK_ALONE)
    assert sum(4 <= kw["n_poses"] <= 12 for kw in WORK) > 0.9 * B


# ---------------------------------------------------------------- helpers

def _scene(kw, **extra):
    sc = scenes.make_scene(**kw, **extra)
    assert len(sc["row_ptr"]) - 1 == kw["n_planes"]
    return sc


def _prob(sc):
    return dict(n_poses=sc["n_poses"], row_ptr=sc["row_ptr"], pose_idx=sc["pose_idx"], obs10=sc["obs10"],
                coe=sc["coe"], fix10=sc["fix10"])


def _batch(problems):
    import balm_b200
    b = balm_b200.Batch(0)
    b.set_problems(problems)
    return b


def _oracle(sc):
    return orc.Oracle(sc["n_poses"], sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc["fix10"])


def _pose_err(a, b):
    rot = max(np.linalg.norm(orc.log_so3(scenes.unpack_pose(x)[0].T @ scenes.unpack_pose(y)[0])) for x, y in zip(a, b))
    tra = max(np.linalg.norm(x[9:] - y[9:]) for x, y in zip(a, b))
    return rot, tra


def _tr_key(tr):
    return [(t["r1"], t["r2"], t["u"], t["v"], t["q"], t["q1"], t["accepted"], t["recomputed_hess"], t["not_pd"])
            for t in tr]


def _same_decisions(tr, tr_o, what):
    """The same accept / reject and recomputed-Hessian sequences; on a mismatch the message gives q / r1 of both sides
    at the first differing iteration (a rounding-level q is a tie the test cannot judge)."""
    acc, acc_o = [t["accepted"] for t in tr], [t["accepted"] for t in tr_o]
    if acc != acc_o:
        it = next((i for i, (x, y) in enumerate(zip(acc, acc_o)) if x != y), min(len(acc), len(acc_o)))
        q = [t["q"] / t["r1"] for t in tr[it:it + 1]] + [t["q"] / t["r1"] for t in tr_o[it:it + 1]]
        pytest.fail(f"{what}: accept sequences {acc} / oracle {acc_o} differ at iteration {it}, q / r1 = {q}")
    assert [t["recomputed_hess"] for t in tr] == [t["recomputed_hess"] for t in tr_o], what


class _Contexts:
    """One fp64 Context per pose count, re-registered per problem with set_voxels."""

    def __init__(self):
        self.ctx = {}

    def __call__(self, sc):
        import balm_b200
        n = sc["n_poses"]
        if n not in self.ctx:
            self.ctx[n] = balm_b200.Context(n, 0, balm_b200.PREC_FP64)
        c = self.ctx[n]
        c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc["fix10"])
        return c

    def close(self):
        for c in self.ctx.values():
            c.close()


@pytest.fixture(scope="module")
def contexts():
    c = _Contexts()
    yield c
    c.close()


def _check_eval(sc, got, include_fix):
    H, g, r = got
    Ho, go, ro = _oracle(sc).evaluate(sc["poses_init"], include_fix=include_fix)
    what = (sc["n_poses"], len(sc["coe"]), include_fix)
    assert H.shape == (6 * sc["n_poses"],) * 2
    assert abs(r - ro) <= 1e-12 * abs(ro), (what, r, ro)
    assert np.abs(g - go).max() <= 1e-10 * np.abs(go).max(), what
    assert np.abs(H - Ho).max() <= 1e-9 * np.abs(Ho).max(), what
    assert np.array_equal(H, H.T), what


def _check_cov(sc, x, got, ctx):
    """status OK; Rcov_raw / Rcov exactly symmetric and against the context holding the problem alone."""
    st, raw, cov = got
    n = 6 * sc["n_poses"]
    what = (sc["n_poses"], len(sc["coe"]))
    assert st == 0 and raw.shape == (n, n) and cov.shape == (n, n), what
    assert np.array_equal(raw, raw.T) and np.array_equal(cov, cov.T), what
    raw_c, cov_c = ctx(sc).pose_covariance(x, point_noise=PN, include_fix=True)
    assert np.abs(raw - raw_c).max() <= 1e-11 * np.abs(raw_c).max(), what
    assert np.abs(cov - cov_c).max() <= 1e-9 * np.abs(cov_c).max(), what


def _check_cov_numpy(sc, x, got):
    _, raw, cov = got
    ref = nc.left_jacobian_point(sc["n_poses"], sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], x, sc["fix10"],
                                 pnoise=PN)
    what = (sc["n_poses"], len(sc["coe"]))
    assert np.abs(raw - ref).max() <= 1e-9 * np.abs(ref).max(), what
    ref_cov = nc.pose_covariance(_oracle(sc).evaluate(x, include_fix=True)[0], ref)
    assert np.abs(cov - ref_cov).max() <= 1e-7 * np.abs(ref_cov).max(), what


# ---------------------------------------------------------------- B: the Hessian's boundary problems in one batch

@pytest.fixture(scope="module")
def hess_scenes():
    return [_scene(kw) for kw in HESS]


LM_KW = dict(want_per_iter=True, gauge_mode=2)


@pytest.fixture(scope="module")
def hess_lm(hess_scenes):
    b = _batch([_prob(s) for s in hess_scenes])
    res = b.damping_iter([s["poses_init"] for s in hess_scenes], **LM_KW)
    b.close()
    return res


@pytest.mark.gpu
def test_boundary_evaluate_matches_oracle(hess_scenes):
    b = _batch([_prob(s) for s in hess_scenes])
    for include_fix in (False, True):
        for sc, got in zip(hess_scenes, b.evaluate([s["poses_init"] for s in hess_scenes], include_fix=include_fix)):
            _check_eval(sc, got, include_fix)
    b.close()


@pytest.mark.gpu
def test_boundary_damping_iter_matches_oracle_and_context(hess_scenes, hess_lm, contexts):
    for sc, (st, poses, tr, per) in zip(hess_scenes, hess_lm):
        what = (sc["n_poses"], len(sc["coe"]))
        st_o, poses_o, tr_o, per_o = _oracle(sc).damping_iter(sc["poses_init"], gauge_mode=2)
        assert st == 0 and st_o == 0 and len(tr) == len(tr_o), what
        _same_decisions(tr, tr_o, what)
        for it in range(len(tr)):
            rot, tra = _pose_err(per[it], per_o[it])
            assert rot <= 1e-6 and tra <= 1e-6, (what, it, rot, tra)
            assert abs(tr[it]["r2"] - tr_o[it]["r2"]) <= 1e-9 * abs(tr_o[it]["r2"]), (what, it)
            assert abs(tr[it]["u"] - tr_o[it]["u"]) <= 1e-5 * tr_o[it]["u"], (what, it)
        pc, trc, _ = contexts(sc).damping_iter(sc["poses_init"], gauge_mode=2)
        assert [t["accepted"] for t in tr] == [t["accepted"] for t in trc], what
        assert np.abs(poses - pc).max() <= 1e-9, (what, np.abs(poses - pc).max())


@pytest.mark.gpu
def test_boundary_gauge_modes(hess_scenes):
    b = _batch([_prob(s) for s in hess_scenes])
    init = [s["poses_init"] for s in hess_scenes]
    for mode in (0, 1):
        for sc, (st, p, tr, _) in zip(hess_scenes, b.damping_iter(init, gauge_mode=mode)):
            what = (sc["n_poses"], len(sc["coe"]), mode)
            _, p_o, tr_o, _ = _oracle(sc).damping_iter(sc["poses_init"], gauge_mode=mode)
            assert st == 0, what
            _same_decisions(tr, tr_o, what)
            assert max(_pose_err(p, p_o)) <= 1e-6, what
            if mode == 1:
                assert np.array_equal(p[0], IDENT), what
    b.close()


@pytest.mark.gpu
def test_boundary_problems_do_not_depend_on_the_batch(hess_scenes, hess_lm):
    for i in HESS_ALONE:
        sc = hess_scenes[i]
        b = _batch([_prob(sc)])
        _, p, tr, per = b.damping_iter([sc["poses_init"]], **LM_KW)[0]
        b.close()
        _, pb, trb, perb = hess_lm[i]
        assert np.array_equal(p, pb) and _tr_key(tr) == _tr_key(trb) and np.array_equal(per, perb), i


# ---------------------------------------------------------------- C: the covariance's boundary problems

@pytest.fixture(scope="module")
def cov_run():
    """The scenes, their poses after the batched LM, and the batch's pose covariance there (isotropic point noise, then
    explicit isotropic cluster covariances)."""
    scs = [_scene(kw, pts_size=COV_PTS, with_fix=True) for kw in COV]
    b = _batch([_prob(s) for s in scs])
    res = b.damping_iter([s["poses_init"] for s in scs], hess_includes_fix=True, gauge_mode=2)
    assert all(r[0] == 0 for r in res)
    poses = [r[1] for r in res]
    out = b.pose_covariance(poses, point_noise=PN, include_fix=True)
    cc = [np.stack([nc.cluster_cov_isotropic(o10, PN) for o10 in s["obs10"]]) for s in scs]
    explicit = b.pose_covariance(poses, c_cov=cc, include_fix=True, want_cov=False)
    b.close()
    return scs, poses, out, explicit


@pytest.mark.gpu
def test_boundary_covariance_matches_reference_and_context(cov_run, contexts):
    scs, poses, out, _ = cov_run
    for sc, x, got in zip(scs, poses, out):
        _check_cov(sc, x, got, contexts)
        _check_cov_numpy(sc, x, got)


@pytest.mark.gpu
def test_boundary_covariance_explicit_cluster_covariances(cov_run):
    _, _, out, explicit = cov_run
    for (st, raw2, cov2), (_, raw, _) in zip(explicit, out):
        assert st == 0 and cov2 is None
        assert np.abs(raw2 - raw).max() <= 1e-12 * np.abs(raw).max()


# ---------------------------------------------------------------- D: a workload-shape batch

@pytest.fixture(scope="module")
def work():
    """The workload's scenes, one batch of them, and its LM with the default options."""
    scs = [_scene(kw, pts_size=WORK_PTS, with_fix=True) for kw in WORK]
    b = _batch([_prob(s) for s in scs])
    init = [s["poses_init"] for s in scs]
    lm = b.damping_iter(init, want_per_iter=True)
    yield scs, b, init, lm
    b.close()


@pytest.mark.gpu
def test_workload_evaluate_matches_oracle(work):
    scs, b, init, _ = work
    for include_fix in (False, True):
        for sc, got in zip(scs, b.evaluate(init, include_fix=include_fix)):
            _check_eval(sc, got, include_fix)


@pytest.mark.gpu
def test_workload_damping_iter_matches_oracle(work):
    scs, _, _, lm = work
    for i, (sc, (st, poses, tr, _)) in enumerate(zip(scs, lm)):
        st_o, poses_o, tr_o, _ = _oracle(sc).damping_iter(sc["poses_init"])
        assert st == 0 and st_o == 0, i
        _same_decisions(tr, tr_o, (i, sc["n_poses"]))
        rot, tra = _pose_err(poses, poses_o)
        assert rot <= 1e-6 and tra <= 1e-6, (i, rot, tra)


@pytest.mark.gpu
def test_workload_problems_do_not_depend_on_the_batch(work):
    scs, _, _, lm = work
    for i in WORK_ALONE:
        b = _batch([_prob(scs[i])])
        _, p, tr, per = b.damping_iter([scs[i]["poses_init"]], want_per_iter=True)[0]
        b.close()
        _, pb, trb, perb = lm[i]
        assert np.array_equal(p, pb) and _tr_key(tr) == _tr_key(trb) and np.array_equal(per, perb), i


@pytest.mark.gpu
def test_workload_gauge_mode_1_sets_every_pose_0_to_identity(work):
    scs, b, init, _ = work
    res = b.damping_iter(init, gauge_mode=1)
    assert all(st == 0 and np.array_equal(p[0], IDENT) for st, p, _, _ in res)
    # and the other poses moved with pose 0 as the oracle's gauge step moves them, in the first and the last block
    for i in (0, len(scs) - 1):
        _, p0, _, _ = _oracle(scs[i]).damping_iter(scs[i]["poses_init"], gauge_mode=1)
        assert max(_pose_err(res[i][1], p0)) <= 1e-6, i


@pytest.mark.gpu
def test_workload_covariance(work, contexts):
    scs, b, _, lm = work
    poses = [r[1] for r in lm]
    out = b.pose_covariance(poses, point_noise=PN, include_fix=True)
    for sc, x, got in zip(scs, poses, out):
        _check_cov(sc, x, got, contexts)
    for i in WORK_NUMPY_COV:
        _check_cov_numpy(scs[i], poses[i], out[i])

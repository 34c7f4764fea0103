"""Small end-to-end run for compute-sanitizer (memcheck / racecheck): both precision modes, dense + sparse; the persistent
tile-DAG factorisation with several 64-column steps (n = 240: chain + near/far workers), the sliding-window marginalisation, the pose-covariance propagation, a multi-batch sparse evaluation, the device
association chain balm_cut_voxels -> balm_marginalize -> balm_append_scan (octree keys + layers), and a batch of
independent problems (balm_batch_*: a dense one with fix clusters, a sparse one of 32 poses, an empty one), and a batch
association of overlapping windows with one empty window (balm_batch_cut_voxels), the batch pose covariance of
an anchored, a free and an empty problem (balm_batch_pose_covariance), and the batched marginalise + append of those
windows, the empty one included (balm_batch_marginalize / balm_batch_append_scan), the batch's persistent window maps
(balm_batch_window_*), and the keyframe merge of overlapping windows with an empty scan and an empty window at voxel
sizes 0 and 0.2 (balm_batch_merge_scans), and the sparse pose graph (balm_spg_*) on a small pyramid with a long-range
factor, a factor that is not positive definite and a pose in no factor, and a factor-only PREC_BLOCKS context on an
87-pose clique (the factor, selected-inversion, anchor and refinement kernels past their wrap edges)."""
import os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import balm_b200, scenes
for prec in (0, 1):
    for drop in (0.0, 0.4):
        sc = scenes.make_scene(n_poses=40, n_planes=90, seed=3, drop=drop, pts_size=6, with_fix=True)
        c = balm_b200.Context(40, 0, prec)
        c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"], sc["fix10"])
        H, g, r = c.evaluate(sc["poses_init"])
        poses, tr, _ = c.damping_iter(sc["poses_init"], max_iter=2, min_planes_per_pose=0, hess_includes_fix=True)
        print("prec", prec, "drop", drop, "r", r, "iters", len(tr), flush=True)
        if prec == 0:
            raw, cov = c.pose_covariance(poses, point_noise=0.01, include_fix=True)
            print("  covariance trace", np.trace(cov), flush=True)
            M2, K2 = c.marginalize(3, poses, min_ps=5)
            shifted = np.vstack([poses[3:], np.tile(poses[-1], (3, 1))])
            print("  marginalised ->", M2, K2, "residual", c.residual(shifted), flush=True)
        c.close()
os.environ["BALM_G_BUDGET_MB"] = "1"
sc = scenes.make_scene(n_poses=20, n_planes=120, seed=4, drop=0.5, pts_size=6)
c = balm_b200.Context(20, 0, 1)
c.set_voxels(sc["row_ptr"], sc["pose_idx"], sc["obs10"], sc["coe"])
print("batched sparse r", c.evaluate(sc["poses_init"])[2], flush=True)
c.close()
import assoc_ref
N, mg = 6, 2
pts, frs, poses = assoc_ref.synthetic_scans(n_poses=N + 1, pts_per_scan=1500, seed=13)
p12 = scenes.pack_poses([r for r, _ in poses], [p for _, p in poses])
c = balm_b200.Context(N, 0, 0)
win = frs < N
M0, K0 = c.cut_voxels(pts[win].astype(np.float32), frs[win], p12[:N], voxel_size=2.0, layer_limit=2, min_ps=15,
                      eigen_value_array=(1 / 16, 1 / 16, 1 / 16))
M1, K1 = c.marginalize(mg, p12[:N], min_ps=15)
shifted = np.vstack([p12[mg:N], p12[N:N + 1], p12[N:N + 1]])
M2, K2, matched = c.append_scan(pts[frs == N].astype(np.float32), shifted, N - mg)
keys, layers = c.download_keys(with_layers=True)
print("assoc chain", (M0, K0), (M1, K1), (M2, K2), "matched", matched, "layers", np.bincount(layers, minlength=3), flush=True)
c.close()
scs = [scenes.make_scene(n_poses=6, n_planes=30, seed=5, pts_size=6, with_fix=True),
       scenes.make_scene(n_poses=32, n_planes=40, seed=6, drop=0.4, pts_size=6)]
probs = [dict(n_poses=s["n_poses"], row_ptr=s["row_ptr"], pose_idx=s["pose_idx"], obs10=s["obs10"], coe=s["coe"],
              fix10=s["fix10"]) for s in scs]
probs.append(dict(n_poses=2, row_ptr=np.zeros(1, dtype=np.int64), pose_idx=np.zeros(0, dtype=np.int32),
                  obs10=np.zeros((0, 10)), coe=np.zeros(0)))
b = balm_b200.Batch(0)
b.set_problems(probs)
x = [s["poses_init"] for s in scs] + [np.tile([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0.0], (2, 1))]
print("batch r", [r for _, _, r in b.evaluate(x, include_fix=True)], flush=True)
res = b.damping_iter(x, max_iter=2, min_planes_per_pose=0, hess_includes_fix=True, want_per_iter=True)
print("batch iters", [len(tr) for _, _, tr, _ in res], flush=True)
cov = b.pose_covariance([r[1] for r in res], point_noise=0.01, include_fix=True)
print("batch covariance", [(st, float(np.trace(raw)), float(np.trace(c))) for st, raw, c in cov], flush=True)
b.close()
# batch association: overlapping windows (2 and 4 scans sharing scans) and one empty window (a single scan)
pts, frs, poses = assoc_ref.synthetic_scans(n_poses=6, pts_per_scan=1500, seed=14)
p12 = scenes.pack_poses([r for r, _ in poses], [p for _, p in poses])
scans = [pts[frs == i] for i in range(6)]
windows = [[0, 1, 2, 3], [2, 3, 4, 5], [4]]
b = balm_b200.Batch(0)
mk = b.cut_scans(scans, windows, [p12[w] for w in windows])
res = b.damping_iter([p12[w] for w in windows], max_iter=2, min_planes_per_pose=0)
print("batch cut", mk, "iters", [len(tr) for _, _, tr, _ in res], flush=True)
# batch sliding window on that registration: marginalise the first two windows (the empty one untouched), then append
# the shared scan 5 to both in the slot that frees
x = [r[1] for r in res]
mm = b.marginalize([1, 1, 0], x)
ma = b.append_scans(scans, [5, 5, -1], [3, 3, 0], x)
print("batch marginalise", mm, "append", ma, "fix rows", len(b.download_voxels(with_fix=True)[0]["fix10"]), flush=True)
b.close()
# persistent window maps of a batch: 4 and 3 slots, the shared scan 2 cut into both, one problem skipped in each call,
# a shift of the first problem, a push with one empty range
b = balm_b200.Batch(0)
b.window_reset([4, 3], layer_limit=2)
wx = [p12[:4], p12[2:5]]
for s in range(3):
    b.window_cut(scans, [s, 2 + s], [s, s], wx)
    b.window_recut([s + 1, s + 1])
b.window_cut(scans, [3, -1], [3, 0], wx)
b.window_recut([4, 0])
b.window_marginalize([2, 0], wx, [4, 0])
b.window_cut(scans, [4, -1], [2, 0], [p12[2:6], wx[1]])
b.window_recut([3, 0])
print("batch window push", b.window_push([3, 0]), b.window_push([3, 3]), flush=True)
b.close()
# keyframe merge: overlapping windows, an empty scan inside one of them, an all-empty window, voxel_size 0 and 0.2
b = balm_b200.Batch(0)
mscans = scans + [np.zeros((0, 3), np.float32)]
mwin = [[0, 1, 6, 2], [2, 3, 4], [6]]
mx = [p12[[0, 1, 1, 2]], p12[2:5], p12[:1]]
print("batch merge", [[len(k) for k in b.merge_scans(mscans, mwin, mx, vs)] for vs in (0.0, 0.2)], flush=True)
b.close()
# sparse pose graph: registration, evaluation, LM with refinement checks; then a pose in no factor (not_pd steps)
import pose_graph_ref as pgr
rng = np.random.default_rng(15)
truth = np.array([pgr.random_pose(rng, 0.5, 3.0) for _ in range(81)])
fs = [pgr.make_factor(rng, truth, w, noise=0.01) for w in pgr.pyramid_factor_poses(80, top=8) + [[2, 77]]]
fs.append(dict(fs[0], H=-fs[0]["H"]))
s = balm_b200.PoseGraph(81)
print("sparse pose graph status", s.set_pose_factors(fs).count(0), s.structure(), flush=True)
print("  cost", s.pose_graph_evaluate(pgr.perturb(rng, truth, 0.05, 0.2))[3], flush=True)
print("  not_pd", [t["not_pd"] for t in s.pose_graph_iter(truth, max_iter=2)[1]], flush=True)
s.set_pose_factors(fs[:-1])
print("  iters", len(s.pose_graph_iter(pgr.perturb(rng, truth, 0.05, 0.2), max_iter=3)[1]), flush=True)
s.close()
# a factor-only blocks context on an 87-pose clique: every loop of the factor and selected-inversion kernels wraps
# (86 blocks below the first column's diagonal); a solve just past a singular leading minor of H + u diag(H), which
# refines, one at u = 0.01 and a covariance (anchor kernel, selected inversion, gather)
import nd_symbolic_ref as nd
from test_gpu_sparse_ldlt_edges import PATTERNS, _blocks_ctx, _factors, _leading_minor_crossing
P, fs, x = _factors("clique87", seed=0)
c = _blocks_ctx(P, fs)
H = c.evaluate(x)[0]
u = _leading_minor_crossing(H, nd.symbolic(P, nd.pairs_of(P, PATTERNS["clique87"][1]))["order"], P // 2) * (1 + 1e-8)
print("clique87 blocks solve at u", u, "not_pd", c.solve(u)[2], "refinements", c.timings()["refinements"], flush=True)
print("  u 0.01 not_pd", c.solve(0.01)[2], flush=True)
print("  covariance trace", sum(np.trace(b) for b in c.block_covariance(x, anchor=0)[1]), flush=True)
c.close()
print("SANITIZE_DONE")

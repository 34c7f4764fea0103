"""numpy restatement of the reference's PERSISTENT octree (the sliding window kept across shifts) -- the oracle of the
device window (balm_window_*). A direct transliteration of src/benchmark/bavoxel.hpp:

  cut_voxel                                   :1170-1223   points -> root voxels, pushed into slot `fnum`
  OCTO_TREE_NODE::recut / judge_eigen / cut_func  :737-776, 654-699, 700-735
  OCTO_TREE_NODE::to_margi / OCTO_TREE_ROOT::marginalize  :778-816, 948-963
  OCTO_TREE_NODE::tras_opt -> VOX_HESS::push_voxel        :908-929, 30-51

Every node keeps, per window slot, its body-frame points (vec_orig), their world coordinates (vec_tran) and the clusters
sig_orig / sig_tran, accumulated point by point in push order (np.cumsum adds left to right, as PointCluster::push does).
Nodes are never deleted: a leaf that is not pushed stays in the map with its fix cluster and comes back when later scans
hit it again. This module sits next to tests/assoc_ref.py, whose flattened restatements it reproduces on a fresh map.
"""
import numpy as np

from assoc_ref import DEFAULTS, node_key, root_index


def _moments(x):
    """Per-point PointCluster::push terms (tools.hpp:311-316): [xx xy xz yy yz zz x y z 1]."""
    return np.stack([x[:, 0] * x[:, 0], x[:, 0] * x[:, 1], x[:, 0] * x[:, 2], x[:, 1] * x[:, 1], x[:, 1] * x[:, 2],
                     x[:, 2] * x[:, 2], x[:, 0], x[:, 1], x[:, 2], np.ones(len(x))], axis=1)


def _push(sig, x):
    """sig.push(p) for every row of x, in order."""
    if len(x) == 0:
        return sig
    return np.cumsum(np.vstack([sig[None, :], _moments(x)]), axis=0)[-1]


def transform(o, pose12):
    """PointCluster::transform (tools.hpp:333-339): body-frame cluster -> world frame at pose12 (R column-major, p)."""
    R = pose12[:9].reshape(3, 3).T
    p = pose12[9:12]
    P = np.array([[o[0], o[1], o[2]], [o[1], o[3], o[4]], [o[2], o[4], o[5]]])
    Rv = R @ o[6:9]
    n = o[9]
    Pw = R @ P @ R.T + np.outer(Rv, p) + np.outer(p, Rv) + n * np.outer(p, p)
    return np.array([Pw[0, 0], Pw[0, 1], Pw[0, 2], Pw[1, 1], Pw[1, 2], Pw[2, 2], *(Rv + n * p), n])


def _to_world(x, pose12):
    R = pose12[:9].reshape(3, 3).T
    return x @ R.T + pose12[9:12]


class _Node:
    def __init__(self, n_slots, layer, center, quater, key):
        self.layer, self.center, self.quater, self.key = layer, center, quater, key
        self.split = False
        self.push_state = 0
        self.fix = np.zeros(10)
        self.orig = [np.zeros((0, 3)) for _ in range(n_slots)]
        self.tran = [np.zeros((0, 3)) for _ in range(n_slots)]
        self.sig_orig = np.zeros((n_slots, 10))
        self.sig_tran = np.zeros((n_slots, 10))
        self.leaves = {}

    def walk(self):
        yield self
        for o in sorted(self.leaves):
            yield from self.leaves[o].walk()


class WindowOctree:
    """surf_map of OCTO_TREE_ROOTs with N window slots, driven by the reference's four operations."""

    def __init__(self, n_slots, **kw):
        o = dict(DEFAULTS)
        o.update(kw)
        self.N = int(n_slots)
        self.vs, self.lim, self.min_ps = float(o["voxel_size"]), int(o["layer_limit"]), int(o["min_ps"])
        self.eig = [float(np.float32(e)) for e in o["eigen_value_array"]]   # `float eigen_value_array[]` (:11)
        self.roots = {}

    def nodes(self):
        for k in sorted(self.roots):
            yield from self.roots[k].walk()

    # ---- cut_voxel (:1170-1223) ----
    def cut_voxel(self, points_body, pose12, slot):
        x = np.asarray(points_body, dtype=np.float32).astype(np.float64)
        w = _to_world(x, np.asarray(pose12, dtype=np.float64))
        idx = root_index(w, self.vs)
        uniq, inv = np.unique(idx, axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        for u in range(len(uniq)):
            m = inv == u
            r = tuple(int(v) for v in uniq[u])
            nd = self.roots.get(r)
            if nd is None:
                center = ((0.5 + np.array(r, dtype=np.float64)) * self.vs).astype(np.float32)
                nd = _Node(self.N, 0, center, np.float32(self.vs / 4.0), node_key(r, 7, 7))
                self.roots[r] = nd
            nd.orig[slot] = np.vstack([nd.orig[slot], x[m]])
            nd.tran[slot] = np.vstack([nd.tran[slot], w[m]])
            nd.sig_orig[slot] = _push(nd.sig_orig[slot], x[m])
            nd.sig_tran[slot] = _push(nd.sig_tran[slot], w[m])

    # ---- recut / judge_eigen / cut_func (:654-776) ----
    def _judge(self, nd, win_count):
        W = nd.fix.copy()
        for i in range(win_count):
            W = W + nd.sig_tran[i]
        cen = W[6:9] / W[9]
        cov = np.array([[W[0], W[1], W[2]], [W[1], W[3], W[4]], [W[2], W[4], W[5]]]) / W[9] - np.outer(cen, cen)
        lam = np.linalg.eigvalsh(cov)
        return lam[0] / lam[1] < self.eig[nd.layer]

    def _cut_func(self, nd, i):
        tran, orig = nd.tran[i], nd.orig[i]
        octs = (tran > nd.center.astype(np.float64)[None, :]).astype(np.int64)
        leaf = 4 * octs[:, 0] + 2 * octs[:, 1] + octs[:, 2]
        for lf in range(8):
            m = leaf == lf
            if not m.any():
                continue
            ch = nd.leaves.get(lf)
            if ch is None:
                xyz = np.array([(lf >> 2) & 1, (lf >> 1) & 1, lf & 1])
                cc = (nd.center + (2 * xyz - 1).astype(np.float32) * np.float32(nd.quater)).astype(np.float32)
                k = (nd.key & ~63) | (lf << 3) | 7 if nd.layer == 0 else (nd.key & ~7) | lf
                ch = _Node(self.N, nd.layer + 1, cc, np.float32(nd.quater / np.float32(2)), k)
                nd.leaves[lf] = ch
            ch.orig[i] = np.vstack([ch.orig[i], orig[m]])
            ch.tran[i] = np.vstack([ch.tran[i], tran[m]])
            ch.sig_orig[i] = _push(ch.sig_orig[i], orig[m])
            ch.sig_tran[i] = _push(ch.sig_tran[i], tran[m])
        nd.orig[i] = np.zeros((0, 3))
        nd.tran[i] = np.zeros((0, 3))

    def _recut(self, nd, win_count):
        if not nd.split:
            point_size = nd.fix[9] + nd.sig_orig[:win_count, 9].sum()
            nd.push_state = 0
            if point_size <= self.min_ps:
                return
            if self._judge(nd, win_count):
                if point_size - nd.fix[9] > self.min_ps:
                    nd.push_state = 1
                return
            if nd.layer == self.lim:
                return
            nd.split = True
            for i in range(win_count):
                self._cut_func(nd, i)
        else:
            self._cut_func(nd, win_count - 1)
        for o in sorted(nd.leaves):
            self._recut(nd.leaves[o], win_count)

    def recut(self, win_count):
        for nd in list(self.roots.values()):
            self._recut(nd, win_count)

    # ---- marginalize / to_margi (:778-816, 948-963) ----
    def marginalize(self, mg, poses12, win_count):
        for nd in list(self.nodes()):
            if nd.split:
                continue
            if poses12 is not None:
                for i in range(win_count):
                    nd.sig_tran[i] = transform(nd.sig_orig[i], poses12[i])
                    nd.tran[i] = _to_world(nd.orig[i], poses12[i])
            if nd.fix[9] < 50 and nd.push_state == 1:
                for i in range(mg):
                    nd.fix = nd.fix + nd.sig_tran[i]
            for i in range(mg, win_count):
                nd.sig_orig[i - mg] = nd.sig_orig[i]
                nd.sig_tran[i - mg] = nd.sig_tran[i]
                nd.orig[i - mg] = nd.orig[i]
                nd.tran[i - mg] = nd.tran[i]
            for i in range(win_count - mg, win_count):
                nd.sig_orig[i] = 0.0
                nd.sig_tran[i] = 0.0
                nd.orig[i] = np.zeros((0, 3))
                nd.tran[i] = np.zeros((0, 3))

    # ---- tras_opt -> push_voxel (:908-929, 30-51) ----
    def export(self, win_count):
        """-> keys, layers, row_ptr, pose_idx, obs10, fix10, coe of the pushed nodes in ascending key order."""
        out = []
        for nd in self.nodes():
            if nd.split or nd.push_state != 1:
                continue
            if nd.sig_orig[:win_count, 9].sum() < self.min_ps:
                continue
            slots = [i for i in range(self.N) if nd.sig_orig[i, 9] != 0]
            if len(slots) < 2:
                continue
            out.append((nd.key, nd))
        out.sort(key=lambda e: e[0])
        keys, layers, rp, pi, ob, fx, co = [], [], [0], [], [], [], []
        for k, nd in out:
            slots = [i for i in range(self.N) if nd.sig_orig[i, 9] != 0]
            for i in slots:
                pi.append(i)
                ob.append(nd.sig_orig[i].copy())
            rp.append(len(pi))
            keys.append(k)
            layers.append(nd.layer)
            fx.append(nd.fix.copy())
            co.append(float(sum(nd.sig_orig[i, 9] for i in slots)))
        return (np.array(keys, dtype=np.int64), np.array(layers, dtype=np.int32), np.array(rp, dtype=np.int64),
                np.array(pi, dtype=np.int32), np.array(ob).reshape(-1, 10), np.array(fx).reshape(-1, 10),
                np.array(co))


def growth_scans(n_scans=30, pts_per_scan=4000, seed=7, step=0.5):
    """Seeded lidar-like scans along a trajectory that advances `step` metres along x per scan, built so that a sliding
    window sees all three ways the persistent octree grows:
      - a floor and a side wall that extend with the trajectory: later scans reach voxels no earlier scan saw (new roots);
      - a compact object that appears from scan 12 on (after a window of 10 has been pushed and shifted once), sitting
        on the floor inside a voxel that was a plane leaf (that leaf is split further);
      - a wall seen by scans 0-3 only and again from scan 16 on (dormant for more than a window of 10, then revived with
        the fix cluster it absorbed).
    -> (points_body float32-rounded float64, frames, noisy initial poses as (R, p), ground-truth poses as (R, p))."""
    import scenes
    rng = np.random.default_rng(seed)
    Rs = [scenes.exp_so3(np.array([0.004 * i, -0.003 * i, 0.02 * np.sin(0.3 * i)])) for i in range(n_scans)]
    ps = [np.array([step * i, 0.2 * np.sin(0.4 * i), 0.01 * i]) for i in range(n_scans)]
    pts, frs = [], []
    for i in range(n_scans):
        xi = step * i
        n = pts_per_scan
        parts = []
        nf = int(0.45 * n)   # floor z = -0.5 around the sensor
        parts.append(np.stack([rng.uniform(xi - 6, xi + 6, nf), rng.uniform(-4.5, 4.5, nf), np.full(nf, -0.5)], 1))
        nw = int(0.3 * n)    # side wall y = 4.5
        parts.append(np.stack([rng.uniform(xi - 6, xi + 6, nw), np.full(nw, 4.5), rng.uniform(-0.5, 3.5, nw)], 1))
        if i < 4 or i >= 16:  # the wall that goes out of view and comes back
            nd = int(0.15 * n)
            parts.append(np.stack([rng.uniform(-3.8, 1.8, nd), np.full(nd, -4.5), rng.uniform(-0.5, 3.5, nd)], 1))
        if i >= 12:           # an object below the floor level inside a floor voxel ([2,4] x [0,2] x [-2,0])
            nb = int(0.06 * n)
            parts.append(rng.normal(0, 0.2, (nb, 3)) + np.array([3.0, 1.0, -1.4]))
        nc = int(0.04 * n)    # clutter
        parts.append(rng.normal(0, 0.5, (nc, 3)) + np.array([xi + 2.0, -2.0, 1.5]))
        w = np.vstack(parts)
        w[:, :2] += rng.normal(0, 0.01, (len(w), 2))
        w[:, 2] += rng.normal(0, 0.01, len(w))
        w = w[rng.permutation(len(w))]
        body = (w - ps[i]) @ Rs[i]
        pts.append(body.astype(np.float32).astype(np.float64))
        frs.append(np.full(len(w), i, dtype=np.int32))
    noisy = [(Rs[i] @ scenes.exp_so3(rng.normal(0, 0.002, 3)), ps[i] + rng.normal(0, 0.005, 3)) for i in range(n_scans)]
    noisy[0] = (Rs[0], ps[0])
    return np.concatenate(pts), np.concatenate(frs), noisy, list(zip(Rs, ps))


def window_schedule(n_scans, n_slots, mg, recut_each_scan):
    """The driver loop of a sliding window (benchmark_realworld.cpp / consistency.cpp): fill the window, push, then shift
    by mg scans at a time -> list of ("cut", scan, slot) / ("recut", win_count) / ("push", win_count) /
    ("marginalize", mg, first_scan_of_window, win_count). recut_each_scan: every cut is followed by its own recut;
    otherwise several scans are cut and one recut follows, which leaves points waiting at already-split nodes."""
    ops = []
    for s in range(n_slots):
        ops.append(("cut", s, s))
        if recut_each_scan:
            ops.append(("recut", s + 1))
    if not recut_each_scan:
        ops.append(("recut", n_slots))
    ops.append(("push", n_slots))
    first, nxt = 0, n_slots
    while nxt + mg <= n_scans:
        ops.append(("marginalize", mg, first, n_slots))
        first += mg
        for j in range(mg):
            slot = n_slots - mg + j
            ops.append(("cut", nxt + j, slot))
            if recut_each_scan:
                ops.append(("recut", slot + 1))
        if not recut_each_scan:
            ops.append(("recut", n_slots))
        ops.append(("push", n_slots))
        nxt += mg
    return ops


def run_schedule(ops, impl, scans, poses12, window_poses12, on_push):
    """Applies `ops` to `impl` (cut_voxel / recut / marginalize / export, as WindowOctree has them). scans[i]: body points
    of scan i; poses12[i]: its pose at cut time; window_poses12[i]: the pose marginalize re-transforms it with (what a BA
    of the window would have produced). on_push(step, export_result) is called at every push."""
    n_push = 0
    for op in ops:
        if op[0] == "cut":
            impl.cut_voxel(scans[op[1]], poses12[op[1]], op[2])
        elif op[0] == "recut":
            impl.recut(op[1])
        elif op[0] == "marginalize":
            mg, first, w = op[1:]
            x = np.zeros((impl.N, 12))
            x[:w] = window_poses12[first:first + w]
            impl.marginalize(mg, x, w)
        else:
            on_push(n_push, impl.export(op[1]))
            n_push += 1
    return n_push


def growth_events(pushes):
    """From the successive pushes (keys, layers, ..., fix10 at index 5) -> counts of (new root pushed, child pushed
    after its parent had been pushed as a leaf, leaf pushed again after an absence with a non-empty fix cluster)."""
    seen_roots, seen, prev = set(), set(), set()
    new_roots = resplit = revived = 0
    for t, p in enumerate(pushes):
        keys, layers, fix = p[0], p[1], p[5]
        cur = set()
        for k, l, f in zip(keys, layers, fix):
            k, l = int(k), int(l)
            cur.add((k, l))
            root = k | 63
            if t > 0 and root not in seen_roots:
                new_roots += 1
            if l >= 1:
                parent = (k | 63, 0) if l == 1 else (k | 7, 1)
                if parent in seen:
                    resplit += 1
            if (k, l) in seen and (k, l) not in prev and f[9] > 0:
                revived += 1
        for k, l in cur:
            seen_roots.add(k | 63)
        seen |= cur
        prev = cur
    return new_roots, resplit, revived

"""Thin object wrapper over the C ABI context (include/balm_b200.h)."""
import ctypes as C

import numpy as np

from . import _lib as L


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _trace_dicts(trace):
    """balm_trace records -> one dict per LM iteration."""
    return [dict(r1=t.r1, r2=t.r2, u=t.u, v=t.v, q=t.q, q1=t.q1, accepted=bool(t.accepted),
                 recomputed_hess=bool(t.recomputed_hess), not_pd=bool(t.not_pd)) for t in trace]


def _set_pose_factors(fn, handle, factors):
    """Marshal window factors for balm_set_pose_factors / balm_spg_set_factors -> per factor status."""
    idx = [np.asarray(f["poses"], dtype=np.int64).ravel() for f in factors]
    hat, Hs = [], []
    for f, i in zip(factors, idx):
        n = 6 * len(i)
        hat.append(np.asarray(f["poses_hat"], dtype=np.float64).reshape(len(i), 12))
        H = np.asarray(f["H"], dtype=np.float64)
        if H.shape != (n, n):
            raise ValueError(f"set_pose_factors: H of a {len(i)}-pose factor must be {n} x {n}, got {H.shape}")
        Hs.append(H.ravel(order="F"))
    ptr = np.concatenate([[0], np.cumsum([len(i) for i in idx])]).astype(np.int64)
    pose = np.ascontiguousarray(np.concatenate(idx) if idx else np.zeros(0), dtype=np.int32)
    hat = np.ascontiguousarray(np.concatenate(hat) if hat else np.zeros((0, 12)), dtype=np.float64)
    Hc = np.ascontiguousarray(np.concatenate(Hs) if Hs else np.zeros(0), dtype=np.float64)
    status = np.zeros(len(factors), dtype=np.int32)
    L.check(fn(handle, len(factors), _p(ptr), _p(pose), _p(hat), _p(Hc), _p(status)))
    return [int(s) for s in status]


_LOSS = {"trivial": L.LOSS_TRIVIAL, "huber": L.LOSS_HUBER, "cauchy": L.LOSS_CAUCHY}


def _loss_arrays(who, kinds, scale):
    """Loss names, one per term, and scale a scalar or one per term (unused for trivial terms) -> the int32 kind and
    float64 scale arrays of balm_set_factor_loss / balm_set_pose_priors (scale None: None); `who` prefixes errors."""
    if any(k not in _LOSS for k in kinds):
        raise ValueError(f"{who}: kinds must be in {sorted(_LOSS)}, got {sorted(set(kinds) - set(_LOSS))}")
    k = np.array([_LOSS[x] for x in kinds], dtype=np.int32)
    sc = None if scale is None else np.ascontiguousarray(np.broadcast_to(np.asarray(scale, dtype=np.float64), k.shape))
    return k, sc


def _set_factor_loss(fn, handle, n_factors, kind, scale):
    """balm_set_factor_loss / balm_spg_set_factor_loss: kind a loss name or one per factor, scale a scalar or one per
    factor (ignored for trivial factors); kind="trivial" resets every factor."""
    if isinstance(kind, str) and kind == "trivial":
        L.check(fn(handle, n_factors, None, None))
        return
    k, sc = _loss_arrays("set_factor_loss", [kind] * n_factors if isinstance(kind, str) else kind, scale)
    L.check(fn(handle, len(k), _p(k), _p(sc)))


def _set_voxel_loss(fn, handle, kind, scale):
    """balm_set_voxel_loss / balm_batch_set_voxel_loss: kind a loss name as set_factor_loss', scale c in metres (a
    plane thickness; unused for "trivial")."""
    if kind not in _LOSS:
        raise ValueError(f"set_voxel_loss: kind must be in {sorted(_LOSS)}, got {kind!r}")
    L.check(fn(handle, _LOSS[kind], 0.0 if scale is None else float(scale)))


def _factor_residuals(fn, handle, n_factors, poses12):
    """balm_factor_residuals / balm_spg_factor_residuals -> (s, w), one entry per factor of the registered set."""
    poses12 = np.ascontiguousarray(poses12, dtype=np.float64)
    s, w = np.zeros(n_factors), np.zeros(n_factors)
    L.check(fn(handle, _p(poses12), _p(s), _p(w)))
    return s, w


def _set_pose_priors(fn, handle, N, priors, kind, scale):
    """Marshal absolute pose priors for balm_set_pose_priors / balm_spg_set_pose_priors -> per prior status. Each prior
    is a dict pose, pose_hat (12), H (6 x 6), optional lever_arm (3); kind a loss name or one per prior, scale a scalar
    or one per prior. [] detaches the set."""
    n = len(priors)
    if n == 0:
        L.check(fn(handle, 0, None, None, None, None, None, None, None))
        return []
    pose = np.array([int(p["pose"]) for p in priors], dtype=np.int32)
    hat = np.ascontiguousarray([np.asarray(p["pose_hat"], dtype=np.float64).reshape(12) for p in priors])
    Hs = []
    for p in priors:
        H = np.asarray(p["H"], dtype=np.float64)
        if H.shape != (6, 6):
            raise ValueError(f"set_pose_priors: H must be 6 x 6, got {H.shape}")
        Hs.append(H.ravel(order="F"))
    H = np.ascontiguousarray(Hs)
    lever = None
    if any(p.get("lever_arm") is not None for p in priors):
        lever = np.ascontiguousarray([np.zeros(3) if p.get("lever_arm") is None else
                                      np.asarray(p["lever_arm"], dtype=np.float64).reshape(3) for p in priors])
    kinds = [kind] * n if isinstance(kind, str) else list(kind)
    k, sc = (None, None) if all(x == "trivial" for x in kinds) else _loss_arrays("set_pose_priors", kinds, scale)
    status = np.zeros(n, dtype=np.int32)
    L.check(fn(handle, n, _p(pose), _p(hat), _p(lever), _p(H), _p(k), _p(sc), _p(status)))
    return [int(s) for s in status]


def _lm_args(rows, want_per_iter, max_iter, u0, v0, rel_tol, *flags, problems=1):
    """An LM call's LmOpts (flags: hess_includes_fix, gauge_mode, min_planes_per_pose, verbose, force_hess), room for
    max(1, max_iter) trace records and an iteration count per problem, and with want_per_iter the state after every
    iteration (max_iter x rows x 12)."""
    return (L.LmOpts(max_iter, u0, v0, rel_tol, *map(int, flags)), (L.Trace * (problems * max(1, max_iter)))(),
            (C.c_int * problems)(), np.zeros((max_iter, rows, 12)) if want_per_iter else None)


def _pose_graph_iter(fn, handle, N, poses12, max_iter, u0, v0, rel_tol, gauge_mode, verbose, want_per_iter, force_hess):
    """balm_pose_graph_iter / balm_spg_iter -> (poses, trace dicts)."""
    poses = np.array(poses12, dtype=np.float64, order="C", copy=True)
    opts, trace, n_it, per_iter = _lm_args(N, want_per_iter, max_iter, u0, v0, rel_tol, 0, gauge_mode, 0, verbose,
                                           force_hess)
    L.check(fn(handle, _p(poses), C.byref(opts), trace, n_it, _p(per_iter)))
    tr = _trace_dicts(trace[:n_it[0]])
    if want_per_iter:
        for t, p in zip(tr, per_iter):
            t["poses"] = p
    return poses, tr


def _block_structure(fn, handle, want_pairs):
    """balm_block_structure / balm_rig_block_structure / balm_spg_structure -> dict(pairs, l_blocks, levels,
    device_bytes), with want_pairs also "pair_list", the (pairs, 2) int32 array of (i, j), i <= j, ascending."""
    st = np.zeros(4, dtype=np.int64)
    L.check(fn(handle, _p(st), None))
    out = dict(pairs=int(st[0]), l_blocks=int(st[1]), levels=int(st[2]), device_bytes=int(st[3]))
    if want_pairs:
        pr = np.zeros((out["pairs"], 2), dtype=np.int32)
        L.check(fn(handle, _p(st), _p(pr)))
        out["pair_list"] = pr
    return out


def _covariance(fn, handle, state, n_pairs, *args):
    """balm_spg_covariance / balm_block_covariance / balm_rig_block_covariance at state (poses12, or base12 and ext12)
    -> [n_pairs, 6, 6] blocks (rows of unknown i, columns of unknown j)."""
    state = [np.ascontiguousarray(x, dtype=np.float64) for x in state]
    cov = np.zeros((n_pairs, 36))
    L.check(fn(handle, *map(_p, state), *args, _p(cov)))
    return cov.reshape(-1, 6, 6).transpose(0, 2, 1)


def _block_point_covariance(fn, handle, state, sel, point_noise, c_cov, include_fix, anchor, joint, *raw):
    """balm_block_point_covariance / balm_rig_block_point_covariance at state (poses12, or base12 and ext12); raw: the
    plain call's raw_blocks pointer -> the joint (6 s x 6 s) Sigma in sel's order, or the (s, 6, 6) marginals."""
    state = [np.ascontiguousarray(x, dtype=np.float64) for x in state]
    sel = np.ascontiguousarray(sel, dtype=np.int32).reshape(-1)
    cc = None if c_cov is None else np.ascontiguousarray(c_cov, dtype=np.float64).reshape(-1, 81)
    s = len(sel)
    cov = np.zeros((6 * s, 6 * s), order="F") if joint else None
    marg = None if joint else np.zeros((s, 36))
    L.check(fn(handle, *map(_p, state), _p(cc), float(point_noise), int(include_fix), int(anchor), s, _p(sel), *raw,
               _p(cov), _p(marg)))
    return cov if joint else marg.reshape(s, 6, 6).transpose(0, 2, 1).copy()


class Context:
    """One GPU, one registered set of plane voxels, N poses."""

    def __init__(self, n_poses, device=0, precision=L.PREC_FP64):
        self._h = C.c_void_p()
        self.N = int(n_poses)
        self.n = 6 * self.N
        self._n_factors = 0  # the registered pose factor set's size
        self._n_priors = 0   # the registered pose prior set's size
        self._rig = None     # (n_base, n_lidar, n_rig) of the rig set by set_rig
        L.check(L.lib().balm_create(C.byref(self._h), self.N, int(device), int(precision)))

    def close(self):
        if self._h:
            L.lib().balm_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- problem ----
    def set_voxels(self, row_ptr, pose_idx, obs10, coe, fix10=None):
        row_ptr = np.ascontiguousarray(row_ptr, dtype=np.int64)
        pose_idx = np.ascontiguousarray(pose_idx, dtype=np.int32)
        obs10 = np.ascontiguousarray(obs10, dtype=np.float64)
        coe = np.ascontiguousarray(coe, dtype=np.float64)
        fix10 = None if fix10 is None else np.ascontiguousarray(fix10, dtype=np.float64)
        self.M = len(row_ptr) - 1
        L.check(L.lib().balm_set_voxels(self._h, self.M, _p(row_ptr), _p(pose_idx), _p(obs10), _p(fix10), _p(coe)))

    def synth_virtual(self, n_voxels, first_voxel=0, pts_size=40, point_noise=0.01, surf_range=2.0, seed=10):
        gt = np.zeros((self.N, 12))
        init = np.zeros((self.N, 12))
        L.check(L.lib().balm_synth_virtual(self._h, int(n_voxels), int(first_voxel), int(pts_size),
                                           float(point_noise), float(surf_range), int(seed), _p(gt), _p(init)))
        self.M = int(n_voxels)
        return gt, init

    def cut_voxels(self, xyz, frame, poses12, voxel_size=2.0, layer_limit=2, min_ps=15,
                   eigen_value_array=(1.0 / 16, 1.0 / 16, 1.0 / 9)):
        """GPU association (cut_voxel + recut + tras_opt): raw body-frame points + poses -> registered plane voxels."""
        xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
        frame = np.ascontiguousarray(frame, dtype=np.int32)
        poses12 = np.ascontiguousarray(poses12, dtype=np.float64)
        o = L.AssocOpts(float(voxel_size), int(layer_limit), int(min_ps), (C.c_double * 3)(*eigen_value_array))
        M, K = C.c_int64(), C.c_int64()
        L.check(L.lib().balm_cut_voxels(self._h, len(frame), _p(xyz), _p(frame), _p(poses12), C.byref(o), C.byref(M),
                                        C.byref(K)))
        self.M = M.value
        return M.value, K.value

    def cut_stats(self):
        """The last successful cut_voxels: slabs (1 in one pass), the points of the largest slab, root voxels, peak
        device scratch bytes, host-to-device bytes, the scratch bound's bytes per point and fixed bytes, and the wall
        times (ms) of the root-count pass, the slab selection, the cuts and the registration."""
        st = np.zeros(11, dtype=np.int64)
        L.check(L.lib().balm_cut_voxels_stats(self._h, _p(st)))
        keys = ("slabs", "max_slab_points", "roots", "peak_scratch_bytes", "h2d_bytes", "scratch_per_point",
                "scratch_fixed")
        out = {k: int(v) for k, v in zip(keys, st)}
        out.update({k: st[7 + i] / 1e3 for i, k in enumerate(("ms_roots", "ms_select", "ms_cut", "ms_register"))})
        return out

    def download_voxels(self):
        K = L.lib().balm_num_obs(self._h)
        row_ptr = np.zeros(self.M + 1, dtype=np.int64)
        pose_idx = np.zeros(K, dtype=np.int32)
        obs10 = np.zeros((K, 10))
        coe = np.zeros(self.M)
        L.check(L.lib().balm_download_voxels(self._h, _p(row_ptr), _p(pose_idx), _p(obs10), _p(coe)))
        return row_ptr, pose_idx, obs10, coe

    def download_voxel_range(self, head, end):
        """CSR arrays of voxels [head, end) only (row_ptr re-based to 0)."""
        K = C.c_int64()
        L.check(L.lib().balm_download_voxel_range(self._h, int(head), int(end), None, None, None, None, C.byref(K)))
        row_ptr = np.zeros(end - head + 1, dtype=np.int64)
        pose_idx = np.zeros(K.value, dtype=np.int32)
        obs10 = np.zeros((K.value, 10))
        coe = np.zeros(end - head)
        L.check(L.lib().balm_download_voxel_range(self._h, int(head), int(end), _p(row_ptr), _p(pose_idx), _p(obs10),
                                                  _p(coe), C.byref(K)))
        return row_ptr, pose_idx, obs10, coe

    # ---- evaluation ----
    def evaluate(self, poses12, head=0, end=None, include_fix=False, want_H=True):
        poses12 = np.ascontiguousarray(poses12, dtype=np.float64)
        H = np.zeros((self.n, self.n), order="F") if want_H else None
        g = np.zeros(self.n)
        r = C.c_double()
        end = self.M if end is None else end
        L.check(L.lib().balm_evaluate(self._h, _p(poses12), head, end, int(include_fix), _p(H), _p(g), C.byref(r)))
        return H, g, r.value

    def residual(self, poses12):
        poses12 = np.ascontiguousarray(poses12, dtype=np.float64)
        r = C.c_double()
        L.check(L.lib().balm_residual(self._h, _p(poses12), C.byref(r)))
        return r.value

    def set_voxel_loss(self, kind, scale=None):
        """Robust loss of every voxel (include/balm_b200.h, balm_set_voxel_loss): kind "trivial", "huber" or "cauchy" of
        s_v = lambda_min (m^2) at scale c in metres. Voxel v then costs coe_v rho(s_v) and its H and g are weighted by
        w_v = rho'(s_v) in every evaluation, LM and covariance. Useful c: 1.5 - 3 point-noise sigmas. "trivial" resets;
        the loss survives every voxel registration."""
        _set_voxel_loss(L.lib().balm_set_voxel_loss, self._h, kind, scale)

    def voxel_residuals(self, poses12, head=0, end=None, include_fix=False):
        """-> (lam, w): lambda_min and its weight rho'(lambda_min) of voxels [head, end) at poses12 (w = 1 without a
        loss); w is bitwise the weight an evaluation at these poses applies."""
        poses12 = np.ascontiguousarray(poses12, dtype=np.float64)
        end = self.M if end is None else end
        lam, w = np.zeros(max(0, end - head)), np.zeros(max(0, end - head))
        L.check(L.lib().balm_voxel_residuals(self._h, _p(poses12), int(head), int(end), int(include_fix), _p(lam), _p(w)))
        return lam, w

    def block_structure(self, want_pairs=False):
        """PREC_BLOCKS contexts: -> dict(pairs, l_blocks, levels, device_bytes): block pairs (i <= j) of H, blocks of the
        factor L, levels of its elimination tree and the device memory the context holds; with want_pairs also
        "pair_list", the (pairs, 2) int32 array of (i, j), ascending."""
        return _block_structure(L.lib().balm_block_structure, self._h, want_pairs)

    def download_blocks(self):
        """PREC_BLOCKS contexts: the last evaluation's blocks, (pairs, 6, 6) with [p, a, c] = H[6 i + a, 6 j + c] of
        pair p = (i, j) in block_structure's order."""
        npairs = self.block_structure()["pairs"]
        b = np.zeros((npairs, 36))
        L.check(L.lib().balm_download_blocks(self._h, _p(b)))
        return b.reshape(npairs, 6, 6).transpose(0, 2, 1).copy()

    def block_covariance(self, poses12, include_fix=False, anchor=0):
        """PREC_BLOCKS contexts: Sigma = (H without pose anchor's rows and columns)^-1 on H's block pattern, H as
        evaluate(poses12, include_fix=include_fix) returns it (anchor=-1: nothing deleted; fix clusters must then fix the
        gauge). -> (pairs [n_pairs, 2] (i <= j), cov [n_pairs, 6, 6]) with cov[p, a, c] = Sigma[6 i + a, 6 j + c]."""
        pairs = self.block_structure(want_pairs=True)["pair_list"]
        return pairs, _covariance(L.lib().balm_block_covariance, self._h, (poses12,), len(pairs), int(include_fix),
                                  int(anchor))

    def block_point_covariance(self, poses12, sel, point_noise=0.0, c_cov=None, include_fix=False, anchor=0, joint=True,
                               want_raw=False):
        """PREC_BLOCKS contexts: pose_covariance's Rcov restricted to the poses sel, without a 6N x 6N matrix
        (include/balm_b200.h, balm_block_point_covariance): Sigma = Y^T R Y, Y = H~^-1 E, H~ as block_covariance's (anchor
        -1 or a pose, deleted; its entries 0), R the raw term. -> the joint (6 s x 6 s) Sigma in sel's order, or with
        joint=False the (s, 6, 6) marginals (all poses of a long drive fit one call); with want_raw also (pairs [n_pairs, 2],
        raw [n_pairs, 6, 6]) with raw[p, a, c] = R[6 i + a, 6 j + c]. c_cov: K x 9 x 9 or None (isotropic point_noise)."""
        pairs = self.block_structure(want_pairs=True)["pair_list"] if want_raw else None
        raw = np.zeros((len(pairs), 36)) if want_raw else None
        out = _block_point_covariance(L.lib().balm_block_point_covariance, self._h, (poses12,), sel, point_noise, c_cov,
                                      include_fix, anchor, joint, _p(raw))
        if want_raw:
            return out, (pairs, raw.reshape(-1, 6, 6).transpose(0, 2, 1).copy())
        return out

    def set_block_factors(self, factors):
        """PREC_BLOCKS contexts: pose factors (set_pose_factors' dicts, e.g. from odometry_factors) in the cost, added to
        the voxel cost in every evaluation over all voxels, damping_iter, block_covariance (include/balm_b200.h,
        balm_block_set_factors). Their H must be in the voxel cost's units (points x m^2). min_planes_per_pose still
        counts voxels only: pass 0 when factors carry scans that see no plane. [] detaches the set; a rejected call
        keeps the previous one. -> per factor OK or ERR_NOT_PD (left out of the cost)."""
        if not factors:
            L.check(L.lib().balm_block_set_factors(self._h, 0, None, None, None, None, None))
            self._n_factors = 0
            return []
        status = _set_pose_factors(L.lib().balm_block_set_factors, self._h, factors)
        self._n_factors = len(status)
        return status

    def set_factor_loss(self, kind, scale=None):
        """Robust loss of the registered pose factors (set_pose_factors', or set_block_factors' on PREC_BLOCKS contexts;
        include/balm_b200.h, balm_set_factor_loss): kind "trivial", "huber" or "cauchy", or one of those per factor;
        scale c (units of sqrt(s), s = e~^T H~ e~) a scalar or one per factor. Every evaluation, LM and covariance of the
        factors then uses cost 1/2 rho(s), gradient rho'(s) b and the reweighted H rho'(s) M. kind="trivial" resets; a
        new factor set starts trivial."""
        _set_factor_loss(L.lib().balm_set_factor_loss, self._h, self._n_factors, kind, scale)

    def factor_residuals(self, poses12):
        """-> (s, w): s_f = e~^T H~ e~ and w_f = rho'(s_f) of every registered factor at poses12 (0, 0 for a factor left
        out as ERR_NOT_PD; w = 1 without a loss)."""
        return _factor_residuals(L.lib().balm_factor_residuals, self._h, self._n_factors, poses12)

    def set_pose_priors(self, priors, kind="trivial", scale=None):
        """Absolute pose priors (include/balm_b200.h, balm_set_pose_priors): list of dict(pose, pose_hat (12), H (6 x 6,
        (rotation, translation) order, positive semi-definite), optional lever_arm (3, body frame)), e.g. from
        pose_priors / position_priors. Prior cost 1/2 rho(e^T H e) with e = (Log(R R^^T), R l + p - p^). They join the
        pose-graph cost (pose_graph_evaluate / pose_graph_iter), and on PREC_BLOCKS contexts, or FP64 / TENSOR ones with
        set_joint_cost on, every evaluation over all voxels, damping_iter, the rig calls and the covariances. With an
        active prior pass gauge_mode=2 and use anchor=-1. kind / scale as set_factor_loss'. [] detaches; the set survives
        factor and voxel registrations. -> per prior OK or ERR_NOT_PD (left out of the cost)."""
        status = _set_pose_priors(L.lib().balm_set_pose_priors, self._h, self.N, priors, kind, scale)
        self._n_priors = len(status)
        return status

    def prior_residuals(self, poses12):
        """-> (s, w): s_q = e^T H_q e and w_q = rho'(s_q) of every registered prior at poses12 (0, 0 for NOT_PD ones)."""
        return _factor_residuals(L.lib().balm_prior_residuals, self._h, self._n_priors, poses12)

    def set_joint_cost(self, on=True):
        """FP64 / TENSOR contexts: with on, the registered pose factors (set_pose_factors, with set_factor_loss) and
        priors (set_pose_priors) join every evaluation over all voxels, as on PREC_BLOCKS contexts (include/balm_b200.h,
        balm_set_joint_cost): evaluate (head 0, end M), residual, damping_iter, the rig calls and pose_covariance (H only;
        the raw term stays voxels only), summed as voxels, then factors, then priors. A sub-range evaluation stays voxels
        only. Odometry then carries scans that see no plane (pass min_planes_per_pose=0), and GNSS priors fix the frame
        (pass gauge_mode=2). The switch survives every registration of voxels, factors and priors; on=False restores the
        voxel cost bitwise. Refused on PREC_BLOCKS contexts and with a communicator attached."""
        L.check(L.lib().balm_set_joint_cost(self._h, int(bool(on))))

    def solve(self, u):
        dx = np.zeros(self.n)
        q1 = C.c_double()
        bad = C.c_int()
        L.check(L.lib().balm_solve(self._h, float(u), _p(dx), C.byref(q1), C.byref(bad)))
        return dx, q1.value, bool(bad.value)

    def damping_iter(self, poses12, max_iter=10, u0=0.01, v0=2.0, rel_tol=1e-6, hess_includes_fix=False,
                     gauge_mode=0, min_planes_per_pose=20, verbose=False, want_per_iter=False, force_hess=False):
        """LM from poses12 -> (poses, trace, per-iteration poses or None). On PREC_BLOCKS contexts, and on FP64 / TENSOR
        ones with set_joint_cost on, the cost holds the pose factors and priors; with an active prior gauge_mode 0 and 1
        are refused (pass 2). min_planes_per_pose counts voxels only: pass 0 when factors carry plane-poor scans."""
        poses = np.array(poses12, dtype=np.float64, order="C", copy=True)
        opts, trace, n_it, per_iter = _lm_args(self.N, want_per_iter, max_iter, u0, v0, rel_tol, hess_includes_fix,
                                               gauge_mode, min_planes_per_pose, verbose, force_hess)
        L.check(L.lib().balm_damping_iter(self._h, _p(poses), C.byref(opts), trace, n_it, _p(per_iter)))
        return poses, _trace_dicts(trace[:n_it[0]]), (per_iter[:n_it[0]] if want_per_iter else None)

    # ---- rig calibration ----
    def set_rig(self, base_of, lidar_of, fixed_bases=(), fixed_lidars=(0,)):
        """Drive the N scan slots by base poses and LiDAR extrinsics (include/balm_b200.h, balm_set_rig): slot s is
        scanned at T_{base_of[s]} E_{lidar_of[s]}. fixed_bases / fixed_lidars list the unknowns held fixed; the default
        fixes LiDAR 0 as the reference (the extrinsics' gauge). base_of=None detaches the rig. -> n_rig, 6 x the free
        unknowns."""
        return self._set_rig(L.lib().balm_set_rig, "set_rig", base_of, lidar_of, fixed_bases, fixed_lidars)

    def set_block_rig(self, base_of, lidar_of, fixed_bases=(), fixed_lidars=(0,)):
        """set_rig on a PREC_BLOCKS context (include/balm_b200.h, balm_block_set_rig): H_rig held as 6x6 blocks and
        solved sparse, the context's pose factors and priors part of the rig cost. rig_evaluate, rig_damping_iter,
        rig_block_structure and rig_block_covariance then take the rig."""
        return self._set_rig(L.lib().balm_block_set_rig, "set_block_rig", base_of, lidar_of, fixed_bases, fixed_lidars)

    def _set_rig(self, fn, who, base_of, lidar_of, fixed_bases, fixed_lidars):
        n_rig = C.c_int()
        if base_of is None:
            L.check(fn(self._h, 0, 0, None, None, None, None, C.byref(n_rig)))
            self._rig = None
            return 0
        base_of = np.ascontiguousarray(base_of, dtype=np.int32)
        lidar_of = np.ascontiguousarray(lidar_of, dtype=np.int32)
        if base_of.shape != (self.N,) or lidar_of.shape != (self.N,):
            raise ValueError(f"{who}: base_of and lidar_of need one entry per slot ({self.N})")
        B = int(base_of.max()) + 1 if self.N else 0
        nl = int(lidar_of.max()) + 1 if self.N else 0
        bf = np.zeros(B, dtype=np.uint8)
        lf = np.zeros(nl, dtype=np.uint8)
        for name, idx, arr in (("fixed_bases", fixed_bases, bf), ("fixed_lidars", fixed_lidars, lf)):
            for i in idx:
                if not 0 <= int(i) < len(arr):
                    raise ValueError(f"{who}: {name} entry {i} outside [0, {len(arr)})")
                arr[int(i)] = 1
        L.check(fn(self._h, B, nl, _p(base_of), _p(lidar_of), _p(bf), _p(lf), C.byref(n_rig)))
        self._rig = (B, nl, n_rig.value)
        return n_rig.value

    def rig_block_structure(self, want_pairs=False):
        """set_block_rig's rig: -> dict(pairs, l_blocks, levels, device_bytes) as block_structure, over the rig's free
        unknowns (set_rig's order); with want_pairs also "pair_list", the (pairs, 2) int32 array of (u, v), u <= v."""
        return _block_structure(L.lib().balm_rig_block_structure, self._h, want_pairs)

    def rig_block_covariance(self, base12, ext12, include_fix=False, anchor=-1):
        """set_block_rig's rig: Sigma = (H_rig without free base anchor's rows and columns)^-1 on the rig's block
        pattern, H_rig as rig_evaluate returns it (anchor=-1: nothing deleted). -> (pairs [n_pairs, 2] (u <= v),
        cov [n_pairs, 6, 6]) with cov[p, a, c] = Sigma[6 u + a, 6 v + c]."""
        base12, ext12, _ = self._rig_shapes(base12, ext12)
        pairs = self.rig_block_structure(want_pairs=True)["pair_list"]
        return pairs, _covariance(L.lib().balm_rig_block_covariance, self._h, (base12, ext12), len(pairs),
                                  int(include_fix), int(anchor))

    def rig_block_point_covariance(self, base12, ext12, sel, point_noise=0.0, c_cov=None, include_fix=False, anchor=-1,
                                   joint=True):
        """set_block_rig's rig: rig_covariance's cov restricted to the free unknowns sel (set_rig's order), without an
        n_rig x n_rig or 6N x 6N matrix (include/balm_b200.h, balm_rig_block_point_covariance). anchor as
        rig_block_covariance. -> the joint (6 s x 6 s) Sigma in sel's order, or with joint=False the (s, 6, 6) marginals.
        balm_b200.rig.extrinsic_sigmas(cov, 0) reads it when sel lists the free extrinsics."""
        base12, ext12, _ = self._rig_shapes(base12, ext12)
        return _block_point_covariance(L.lib().balm_rig_block_point_covariance, self._h, (base12, ext12), sel,
                                       point_noise, c_cov, include_fix, anchor, joint)

    def _rig_shapes(self, base12, ext12):
        if getattr(self, "_rig", None) is None:
            raise L.BalmError(L.ERR_INVALID, "no rig set (set_rig)")
        B, nl, n_rig = self._rig
        base12 = np.array(base12, dtype=np.float64, order="C", copy=True).reshape(B, 12)
        ext12 = np.array(ext12, dtype=np.float64, order="C", copy=True).reshape(nl, 12)
        return base12, ext12, n_rig

    def rig_evaluate(self, base12, ext12, include_fix=False):
        """-> (H_rig, g_rig, residual) at base poses base12 (B x 12) and extrinsics ext12 (L x 12), the unknowns in
        set_rig's order: free base poses ascending, then free extrinsics ascending, 6 each."""
        base12, ext12, n_rig = self._rig_shapes(base12, ext12)
        H = np.zeros((n_rig, n_rig), order="F")
        g = np.zeros(n_rig)
        r = C.c_double()
        L.check(L.lib().balm_rig_evaluate(self._h, _p(base12), _p(ext12), int(include_fix), _p(H), _p(g), C.byref(r)))
        return H, g, r.value

    def rig_damping_iter(self, base12, ext12, max_iter=10, u0=0.01, v0=2.0, rel_tol=1e-6, hess_includes_fix=False,
                         gauge_mode=0, min_planes_per_pose=20, verbose=False, want_per_iter=False, force_hess=False):
        """damping_iter's LM on the rig's unknowns -> (base12, ext12, trace) and, with want_per_iter, the accepted
        (base12, ext12) after every iteration as a fourth item. gauge_mode 0 / 1 re-anchor the base poses to base 0
        (refused while a base pose is fixed: pass 2). With set_joint_cost on (or a set_block_rig rig) the pose factors
        and priors act at the composed scan poses, and an active prior also refuses gauge_mode 0 and 1."""
        base12, ext12, _ = self._rig_shapes(base12, ext12)
        B, nl = len(base12), len(ext12)
        opts, trace, n_it, per_iter = _lm_args(B + nl, want_per_iter, max_iter, u0, v0, rel_tol, hess_includes_fix,
                                               gauge_mode, min_planes_per_pose, verbose, force_hess)
        L.check(L.lib().balm_rig_damping_iter(self._h, _p(base12), _p(ext12), C.byref(opts), trace, n_it,
                                              _p(per_iter)))
        tr = _trace_dicts(trace[:n_it[0]])
        if not want_per_iter:
            return base12, ext12, tr
        per = [(p[:B].copy(), p[B:].copy()) for p in per_iter[:n_it[0]]]
        return base12, ext12, tr, per

    def rig_covariance(self, base12, ext12, point_noise=0.0, c_cov=None, include_fix=False, anchor=-1, want_raw=True,
                       want_cov=True):
        """pose_covariance on the rig's unknowns (include/balm_b200.h, balm_rig_covariance) -> (raw, cov), n_rig x n_rig
        in set_rig's order: raw = J^T Rcov_raw J at the composed scan poses, cov = H_rig^-1 raw H_rig^-T. anchor: -1 or
        the free index of a free base pose, deleted from both (its rows and columns 0); pass a base anchor when the base
        poses' gauge is free (no fixed base and no fix clusters in H), -1 when every base pose is fixed."""
        base12, ext12, n_rig = self._rig_shapes(base12, ext12)
        cc = None if c_cov is None else np.ascontiguousarray(c_cov, dtype=np.float64).reshape(-1, 81)
        raw = np.zeros((n_rig, n_rig), order="F") if want_raw else None
        cov = np.zeros((n_rig, n_rig), order="F") if want_cov else None
        L.check(L.lib().balm_rig_covariance(self._h, _p(base12), _p(ext12), _p(cc), float(point_noise), int(include_fix),
                                            int(anchor), _p(raw), _p(cov)))
        return raw, cov

    def marginalize(self, mg_size, poses12, min_ps=15):
        """OCTO_TREE_ROOT::marginalize on the registered voxel set (bavoxel.hpp:948-963, 778-816) -> (n_voxels, n_obs)."""
        poses12 = np.ascontiguousarray(poses12, dtype=np.float64)
        M, K = C.c_int64(), C.c_int64()
        L.check(L.lib().balm_marginalize(self._h, int(mg_size), _p(poses12), int(min_ps), C.byref(M), C.byref(K)))
        self.M = M.value
        return M.value, K.value

    def append_scan(self, xyz, poses12, slot):
        """Associates a new scan (body-frame points) with the voxel set in HBM: observation in pose slot `slot`, every voxel
        re-judged as recut / judge_eigen do. -> (n_voxels, n_obs, n_points_matched)."""
        xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
        poses12 = np.ascontiguousarray(poses12, dtype=np.float64)
        M, K, m = C.c_int64(), C.c_int64(), C.c_int64()
        L.check(L.lib().balm_append_scan(self._h, len(xyz), _p(xyz), _p(poses12), int(slot), C.byref(M), C.byref(K), C.byref(m)))
        self.M = M.value
        return M.value, K.value, m.value

    def download_keys(self, with_layers=False):
        keys = np.zeros(self.M, dtype=np.uint64)
        layers = np.zeros(self.M, dtype=np.int32)
        L.check(L.lib().balm_download_keys(self._h, _p(keys), _p(layers)))
        return (keys, layers) if with_layers else keys

    def download_fix(self):
        fix = np.zeros((self.M, 10))
        L.check(L.lib().balm_download_fix(self._h, _p(fix)))
        return fix

    # ---- persistent sliding-window octree ----
    def window_reset(self, voxel_size=2.0, layer_limit=2, min_ps=15, eigen_value_array=(1.0 / 16, 1.0 / 16, 1.0 / 9)):
        """Empty window map (the reference's surf_map) with these association parameters."""
        o = L.AssocOpts(float(voxel_size), int(layer_limit), int(min_ps), (C.c_double * 3)(*eigen_value_array))
        L.check(L.lib().balm_window_reset(self._h, C.byref(o)))

    def window_cut(self, xyz, pose12, slot):
        """cut_voxel: a scan's body-frame points, at pose12, into window slot `slot`."""
        xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
        pose12 = np.ascontiguousarray(pose12, dtype=np.float64).reshape(12)
        L.check(L.lib().balm_window_cut(self._h, len(xyz), _p(xyz), _p(pose12), int(slot)))

    def window_recut(self, win_count):
        """recut(win_count) on every root."""
        L.check(L.lib().balm_window_recut(self._h, int(win_count)))

    def window_marginalize(self, mg_size, poses12, win_count):
        """marginalize(mg_size, x_poses, win_count) on every root; poses12: N x 12 (the window's optimised poses) or None."""
        p = None if poses12 is None else np.ascontiguousarray(poses12, dtype=np.float64).reshape(self.N, 12)
        L.check(L.lib().balm_window_marginalize(self._h, int(mg_size), _p(p), int(win_count)))

    def window_push(self, win_count):
        """tras_opt(win_count): registers the pushed nodes as the voxel set -> (n_voxels, n_obs)."""
        M, K = C.c_int64(), C.c_int64()
        L.check(L.lib().balm_window_push(self._h, int(win_count), C.byref(M), C.byref(K)))
        self.M = M.value
        return M.value, K.value

    def pose_covariance(self, poses12, point_noise=0.0, c_cov=None, include_fix=False, want_raw=True, want_cov=True):
        """left_jacobian_point / multi_second / H^-1 Rcov H^-T (BAs_left.hpp:342-473, 995-1023, 1089-1096).
        -> (Rcov_raw, Rcov); c_cov: K x 9 x 9 per-observation cluster covariances, or None for isotropic point noise.
        With set_joint_cost on, H is the joint H of voxels, pose factors and priors (priors can fix the gauge without fix
        clusters); Rcov_raw stays the voxels' term."""
        poses12 = np.ascontiguousarray(poses12, dtype=np.float64)
        cc = None if c_cov is None else np.ascontiguousarray(c_cov, dtype=np.float64).reshape(-1, 81)
        raw = np.zeros((self.n, self.n), order="F") if want_raw else None
        cov = np.zeros((self.n, self.n), order="F") if want_cov else None
        L.check(L.lib().balm_pose_covariance(self._h, _p(poses12), _p(cc), float(point_noise), int(include_fix), _p(raw),
                                             _p(cov)))
        return raw, cov

    # ---- pose graph ----
    def set_pose_factors(self, factors):
        """Window factors (include/balm_b200.h, balm_set_pose_factors): list of dict(poses = N_f distinct global pose
        indices, poses_hat = N_f x 12 refined window poses, H = (6 N_f)^2 window BA Hessian, symmetric to 1e-12 of its
        max |entry|). Replaces the previous factor set; a rejected call keeps it. They make the pose-graph cost, and with set_joint_cost on they also join the voxel
        cost (H in its units: points x m^2, as odometry_factors gives). -> per factor OK or ERR_NOT_PD (left out of the
        cost)."""
        status = _set_pose_factors(L.lib().balm_set_pose_factors, self._h, factors)
        self._n_factors = len(status)
        return status

    def pose_graph_evaluate(self, poses12, want_H=True):
        """-> (H, g, cost) of the registered factors at poses12 (H dense n x n, None with want_H=False)."""
        poses12 = np.ascontiguousarray(poses12, dtype=np.float64)
        H = np.zeros((self.n, self.n), order="F") if want_H else None
        g = np.zeros(self.n)
        r = C.c_double()
        L.check(L.lib().balm_pose_graph_evaluate(self._h, _p(poses12), _p(H), _p(g), C.byref(r)))
        return H, g, r.value

    def pose_graph_iter(self, poses12, max_iter=10, u0=0.01, v0=2.0, rel_tol=1e-6, gauge_mode=0, verbose=False,
                        want_per_iter=False, force_hess=False):
        """damping_iter's LM on the pose-graph cost -> (poses, trace); with want_per_iter every trace record also holds
        the accepted poses after its iteration under "poses"."""
        return _pose_graph_iter(L.lib().balm_pose_graph_iter, self._h, self.N, poses12, max_iter, u0, v0, rel_tol,
                                gauge_mode, verbose, want_per_iter, force_hess)

    # ---- multi-GPU ----
    @staticmethod
    def comm_unique_id():
        buf = (C.c_char * 128)()
        L.check(L.lib().balm_comm_unique_id(buf))
        return bytes(buf)

    def comm_init(self, rank, world, unique_id):
        buf = (C.c_char * 128).from_buffer_copy(unique_id) if unique_id is not None else None
        L.check(L.lib().balm_comm_init(self._h, int(rank), int(world), buf))

    # ---- instrumentation ----
    def timings(self):
        t = L.Timings()
        L.check(L.lib().balm_get_timings(self._h, C.byref(t)))
        reused = C.c_int()
        L.check(L.lib().balm_get_reused_sweeps(self._h, C.byref(reused)))
        return {**{k: getattr(t, k) for k, _ in L.Timings._fields_}, "reused_sweeps": reused.value}

    def reset_counters(self):
        L.check(L.lib().balm_reset_counters(self._h))

    def timer_begin(self):
        L.check(L.lib().balm_timer_begin(self._h))

    def timer_end(self):
        ms = C.c_float()
        L.check(L.lib().balm_timer_end(self._h, C.byref(ms)))
        return ms.value

    def sync(self):
        L.check(L.lib().balm_sync(self._h))


class Batch:
    """One GPU, B independent small problems (at most 32 poses each) registered together; evaluation and LM run for all
    of them at once, each problem with its own damping, accept / reject and stopping (include/balm_b200.h, balm_batch_*)."""

    def __init__(self, device=0):
        self._h = C.c_void_p()
        self.n_poses = []
        self._win_slots = None
        L.check(L.lib().balm_batch_create(C.byref(self._h), int(device)))

    def close(self):
        if self._h:
            L.lib().balm_batch_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_problems(self, problems):
        """problems: list of dicts with n_poses and the arrays Context.set_voxels takes (row_ptr, pose_idx, obs10, coe,
        optional fix10). Problems without fix clusters get zero fix rows when others have them."""
        n_poses = [int(p["n_poses"]) for p in problems]
        row_ptrs = [np.asarray(p["row_ptr"], dtype=np.int64) for p in problems]
        n_vox = [len(rp) - 1 for rp in row_ptrs]
        pose_ptr = np.concatenate([[0], np.cumsum(n_poses)]).astype(np.int64)
        voxel_ptr = np.concatenate([[0], np.cumsum(n_vox)]).astype(np.int64)
        row_ptr, base = [np.zeros(1, dtype=np.int64)], 0
        for rp in row_ptrs:
            row_ptr.append(rp[1:] + base)
            base += int(rp[-1])
        row_ptr = np.ascontiguousarray(np.concatenate(row_ptr), dtype=np.int64)
        pose_idx = np.ascontiguousarray(np.concatenate([np.asarray(p["pose_idx"], dtype=np.int32).ravel()
                                                        for p in problems]), dtype=np.int32)
        obs10 = np.ascontiguousarray(np.concatenate([np.asarray(p["obs10"], dtype=np.float64).reshape(-1, 10)
                                                     for p in problems]), dtype=np.float64)
        coe = np.ascontiguousarray(np.concatenate([np.asarray(p["coe"], dtype=np.float64).ravel() for p in problems]),
                                   dtype=np.float64)
        fix10 = None
        if any(p.get("fix10") is not None for p in problems):
            fix10 = np.ascontiguousarray(np.concatenate([
                np.zeros((m, 10)) if p.get("fix10") is None else np.asarray(p["fix10"], dtype=np.float64).reshape(-1, 10)
                for p, m in zip(problems, n_vox)]), dtype=np.float64)
        L.check(L.lib().balm_batch_set_voxels(self._h, len(problems), _p(pose_ptr), _p(voxel_ptr), _p(row_ptr),
                                              _p(pose_idx), _p(obs10), _p(fix10), _p(coe)))
        self.n_poses = n_poses
        self._pose_ptr = pose_ptr

    def cut_scans(self, scans, windows, poses_list, voxel_size=2.0, layer_limit=2, min_ps=15,
                  eigen_value_array=(1.0 / 16, 1.0 / 16, 1.0 / 9)):
        """Association for every window on the device (include/balm_b200.h, balm_batch_cut_voxels). scans: list of
        (n_s x 3) body-frame points, each uploaded once; windows: per problem the scan indices of its slots (1 .. 32);
        poses_list: per window its N_w x 12 initial poses. Window w gets what Context(N_w).cut_voxels registers on its
        scans' points with frame = slot. A window without a plane voxel is registered empty. -> per window (M, K)."""
        scans = [np.asarray(s, dtype=np.float32).reshape(-1, 3) for s in scans]
        n_poses = [len(w) for w in windows]
        scan_ptr = np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.int64)
        pose_ptr = np.concatenate([[0], np.cumsum(n_poses)]).astype(np.int64)
        pose_scan = np.ascontiguousarray(np.concatenate([np.asarray(w, dtype=np.int64).ravel() for w in windows]),
                                         dtype=np.int32)
        xyz = np.ascontiguousarray(np.concatenate(scans) if scans else np.zeros((0, 3)), dtype=np.float32)
        poses = np.ascontiguousarray(np.concatenate([np.asarray(p, dtype=np.float64).reshape(n, 12)
                                                     for p, n in zip(poses_list, n_poses)]), dtype=np.float64)
        o = L.AssocOpts(float(voxel_size), int(layer_limit), int(min_ps), (C.c_double * 3)(*eigen_value_array))
        M = np.zeros(len(windows), dtype=np.int64)
        K = np.zeros(len(windows), dtype=np.int64)
        L.check(L.lib().balm_batch_cut_voxels(self._h, len(windows), _p(pose_ptr), _p(pose_scan), len(scans),
                                              _p(scan_ptr), _p(xyz), _p(poses), C.byref(o), _p(M), _p(K)))
        self.n_poses = n_poses
        self._pose_ptr = pose_ptr
        return [(int(m), int(k)) for m, k in zip(M, K)]

    def merge_scans(self, scans, windows, poses_list, voxel_size):
        """Keyframes on the device (include/balm_b200.h, balm_batch_merge_scans): per window, its scans' points in the
        body frame of its slot 0 at poses_list[w], down-sampled at voxel_size (< 0.001: not reduced). scans / windows as
        cut_scans. Leaves the registration alone. -> per window an (n_w x 3) float32 cloud, voxels in ascending order."""
        scans = [np.asarray(s, dtype=np.float32).reshape(-1, 3) for s in scans]
        n_poses = [len(w) for w in windows]
        scan_ptr = np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.int64)
        pose_ptr = np.concatenate([[0], np.cumsum(n_poses)]).astype(np.int64)
        pose_scan = np.ascontiguousarray(np.concatenate([np.asarray(w, dtype=np.int64).ravel() for w in windows]),
                                         dtype=np.int32)
        xyz = np.ascontiguousarray(np.concatenate(scans) if scans else np.zeros((0, 3)), dtype=np.float32)
        poses = np.ascontiguousarray(np.concatenate([np.asarray(p, dtype=np.float64).reshape(n, 12)
                                                     for p, n in zip(poses_list, n_poses)]), dtype=np.float64)
        n_items = int(sum(scan_ptr[s + 1] - scan_ptr[s] for s in pose_scan))
        kf_ptr = np.zeros(len(windows) + 1, dtype=np.int64)
        kf = np.zeros((n_items, 3), dtype=np.float32)
        L.check(L.lib().balm_batch_merge_scans(self._h, len(windows), _p(pose_ptr), _p(pose_scan), len(scans),
                                               _p(scan_ptr), _p(xyz), _p(poses), float(voxel_size), _p(kf_ptr), _p(kf)))
        return [kf[kf_ptr[w]:kf_ptr[w + 1]].copy() for w in range(len(windows))]

    def marginalize(self, mg_sizes, poses_list, min_ps=15):
        """Context.marginalize per problem, all in one call (include/balm_b200.h, balm_batch_marginalize): the oldest
        mg_sizes[p] scans of problem p folded into its fix clusters at its poses; 0 leaves a problem unchanged. A problem
        left without a voxel is registered empty. -> per problem (M, K)."""
        mg = np.ascontiguousarray(mg_sizes, dtype=np.int32)
        poses = self._concat(poses_list)
        M = np.zeros(len(self.n_poses), dtype=np.int64)
        K = np.zeros(len(self.n_poses), dtype=np.int64)
        L.check(L.lib().balm_batch_marginalize(self._h, _p(mg), _p(poses), int(min_ps), _p(M), _p(K)))
        return [(int(m), int(k)) for m, k in zip(M, K)]

    def append_scans(self, scans, scan_of, slots, poses_list):
        """Context.append_scan per problem, all in one call (include/balm_b200.h, balm_batch_append_scan). scans: list
        of (n_s x 3) body-frame points, each uploaded once; scan_of[p]: the scan problem p takes in slot slots[p], or -1
        (problem unchanged). Needs a registration from cut_scans. A problem left without voxels is registered empty,
        with 0 points matched. -> per problem (M, K, points matched)."""
        scans = [np.asarray(s, dtype=np.float32).reshape(-1, 3) for s in scans]
        scan_ptr = np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.int64)
        xyz = np.ascontiguousarray(np.concatenate(scans) if scans else np.zeros((0, 3)), dtype=np.float32)
        scan_of = np.ascontiguousarray(scan_of, dtype=np.int32)
        slots = np.ascontiguousarray(slots, dtype=np.int32)
        poses = self._concat(poses_list)
        B = len(self.n_poses)
        M, K, m = (np.zeros(B, dtype=np.int64) for _ in range(3))
        L.check(L.lib().balm_batch_append_scan(self._h, _p(scan_of), _p(slots), len(scans), _p(scan_ptr), _p(xyz),
                                               _p(poses), _p(M), _p(K), _p(m)))
        return [(int(a), int(b), int(c)) for a, b, c in zip(M, K, m)]

    # ---- persistent sliding-window octrees, one per problem ----
    def window_reset(self, n_slots, voxel_size=2.0, layer_limit=2, min_ps=15,
                     eigen_value_array=(1.0 / 16, 1.0 / 16, 1.0 / 9)):
        """Empty window maps (include/balm_b200.h, balm_batch_window_*): problem p gets n_slots[p] (1 .. 32) slots, every
        problem these association parameters. Problem p is a Context(n_slots[p]) window driven by the same calls."""
        ns = np.ascontiguousarray([int(n) for n in n_slots], dtype=np.int32)
        o = L.AssocOpts(float(voxel_size), int(layer_limit), int(min_ps), (C.c_double * 3)(*eigen_value_array))
        L.check(L.lib().balm_batch_window_reset(self._h, len(ns), _p(ns), C.byref(o)))
        self._win_slots = [int(n) for n in ns]

    def _win_poses(self, poses_list):
        if self._win_slots is None:  # no window_reset yet: the library refuses the call
            return np.zeros((1, 12))
        assert len(poses_list) == len(self._win_slots)
        return np.ascontiguousarray(np.concatenate([np.asarray(p, dtype=np.float64).reshape(n, 12)
                                                    for p, n in zip(poses_list, self._win_slots)]), dtype=np.float64)

    def window_cut(self, scans, scan_of, slots, poses_list):
        """Context.window_cut per problem, all in one call. scans: list of (n_s x 3) body-frame points, each uploaded once;
        scan_of[p]: the scan problem p takes into slot slots[p] at its pose poses_list[p][slots[p]], or -1 (map left
        alone); poses_list: per problem its n_slots[p] x 12 poses."""
        scans = [np.asarray(s, dtype=np.float32).reshape(-1, 3) for s in scans]
        scan_ptr = np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.int64)
        xyz = np.ascontiguousarray(np.concatenate(scans) if scans else np.zeros((0, 3)), dtype=np.float32)
        scan_of = np.ascontiguousarray(scan_of, dtype=np.int32)
        slots = np.ascontiguousarray(slots, dtype=np.int32)
        poses = self._win_poses(poses_list)
        L.check(L.lib().balm_batch_window_cut(self._h, _p(scan_of), _p(slots), len(scans), _p(scan_ptr), _p(xyz),
                                              _p(poses)))

    def window_recut(self, win_counts):
        """Context.window_recut(win_counts[p]) per problem; 0 leaves a map alone."""
        w = np.ascontiguousarray(win_counts, dtype=np.int32)
        L.check(L.lib().balm_batch_window_recut(self._h, _p(w)))

    def window_marginalize(self, mg_sizes, poses_list, win_counts):
        """Context.window_marginalize(mg_sizes[p], poses_list[p], win_counts[p]) per problem; mg 0 leaves a map alone.
        poses_list: per problem n_slots[p] x 12 poses, or None (no re-transform)."""
        mg = np.ascontiguousarray(mg_sizes, dtype=np.int32)
        w = np.ascontiguousarray(win_counts, dtype=np.int32)
        poses = None if poses_list is None else self._win_poses(poses_list)
        L.check(L.lib().balm_batch_window_marginalize(self._h, _p(mg), _p(poses), _p(w)))

    def window_push(self, win_counts):
        """Context.window_push(win_counts[p]) per problem, registered as the batch's problems (n_poses = n_slots, fix
        clusters, keys); win_counts[p] == 0 gives problem p an empty voxel range. -> per problem (M, K)."""
        w = np.ascontiguousarray(win_counts, dtype=np.int32)
        B = len(self._win_slots or [])
        M = np.zeros(B, dtype=np.int64)
        K = np.zeros(B, dtype=np.int64)
        L.check(L.lib().balm_batch_window_push(self._h, _p(w), _p(M), _p(K)))
        self.n_poses = list(self._win_slots)
        self._pose_ptr = np.concatenate([[0], np.cumsum(self.n_poses)]).astype(np.int64)
        return [(int(m), int(k)) for m, k in zip(M, K)]

    def download_voxels(self, with_keys=False, with_fix=False):
        """The current registration, per problem a dict set_problems accepts (row_ptr re-based to 0); with_keys adds
        keys and layers (only after cut_scans), with_fix the fix clusters fix10 (zero rows where a voxel has none)."""
        B, P, M, K = C.c_int(), C.c_int64(), C.c_int64(), C.c_int64()
        L.check(L.lib().balm_batch_sizes(self._h, C.byref(B), C.byref(P), C.byref(M), C.byref(K)))
        voxel_ptr = np.zeros(B.value + 1, dtype=np.int64)
        row_ptr = np.zeros(M.value + 1, dtype=np.int64)
        pose_idx = np.zeros(K.value, dtype=np.int32)
        obs10 = np.zeros((K.value, 10))
        coe = np.zeros(M.value)
        keys = np.zeros(M.value, dtype=np.uint64) if with_keys else None
        layers = np.zeros(M.value, dtype=np.int32) if with_keys else None
        L.check(L.lib().balm_batch_download_voxels(self._h, _p(voxel_ptr), _p(row_ptr), _p(pose_idx), _p(obs10), _p(coe),
                                                   _p(keys), _p(layers)))
        fix10 = None
        if with_fix:
            fix10 = np.zeros((M.value, 10))
            L.check(L.lib().balm_batch_download_fix(self._h, _p(fix10)))
        out = []
        for b in range(B.value):
            v0, v1 = int(voxel_ptr[b]), int(voxel_ptr[b + 1])
            s0, s1 = int(row_ptr[v0]), int(row_ptr[v1])
            d = dict(n_poses=int(self._pose_ptr[b + 1] - self._pose_ptr[b]), row_ptr=row_ptr[v0:v1 + 1] - s0,
                     pose_idx=pose_idx[s0:s1].copy(), obs10=obs10[s0:s1].copy(), coe=coe[v0:v1].copy())
            if with_keys:
                d.update(keys=keys[v0:v1].copy(), layers=layers[v0:v1].copy())
            if with_fix:
                d.update(fix10=fix10[v0:v1].copy())
            out.append(d)
        return out

    def _concat(self, poses_list):
        assert len(poses_list) == len(self.n_poses)
        return np.ascontiguousarray(np.concatenate([np.asarray(p, dtype=np.float64).reshape(n, 12)
                                                    for p, n in zip(poses_list, self.n_poses)]), dtype=np.float64)

    def evaluate(self, poses_list, include_fix=False):
        """left_evaluate_acc2 per problem -> list of (H, g, r)."""
        poses = self._concat(poses_list)
        ns = [6 * n for n in self.n_poses]
        H = np.zeros(sum(n * n for n in ns))
        g = np.zeros(6 * len(poses))
        r = np.zeros(len(ns))
        L.check(L.lib().balm_batch_evaluate(self._h, _p(poses), int(include_fix), _p(H), _p(g), _p(r)))
        out, ho = [], 0
        for b, n in enumerate(ns):
            g0 = 6 * int(self._pose_ptr[b])
            out.append((H[ho:ho + n * n].reshape(n, n, order="F"), g[g0:g0 + n].copy(), float(r[b])))
            ho += n * n
        return out

    def set_voxel_loss(self, kind, scale=None):
        """Context.set_voxel_loss for every voxel of every problem (evaluate, damping_iter, pose_covariance); the loss
        belongs to the batch and survives every registration."""
        _set_voxel_loss(L.lib().balm_batch_set_voxel_loss, self._h, kind, scale)

    def voxel_residuals(self, poses_list, include_fix=False):
        """Context.voxel_residuals per problem -> list of (lam, w), each over the problem's voxels in registration order."""
        poses = self._concat(poses_list)
        B, M = C.c_int(), C.c_int64()
        L.check(L.lib().balm_batch_sizes(self._h, C.byref(B), None, C.byref(M), None))
        lam, w = np.zeros(M.value), np.zeros(M.value)
        L.check(L.lib().balm_batch_voxel_residuals(self._h, _p(poses), int(include_fix), _p(lam), _p(w)))
        voxel_ptr = np.zeros(B.value + 1, dtype=np.int64)
        L.check(L.lib().balm_batch_download_voxels(self._h, _p(voxel_ptr), None, None, None, None, None, None))
        return [(lam[voxel_ptr[b]:voxel_ptr[b + 1]].copy(), w[voxel_ptr[b]:voxel_ptr[b + 1]].copy())
                for b in range(B.value)]

    def damping_iter(self, poses_list, max_iter=10, u0=0.01, v0=2.0, rel_tol=1e-6, hess_includes_fix=False,
                     gauge_mode=0, min_planes_per_pose=20, verbose=False, want_per_iter=False, force_hess=False):
        """damping_iter per problem, all advanced together -> list of (status, poses, trace, per_iter)."""
        poses = self._concat(poses_list)
        B, P = len(self.n_poses), len(poses)
        opts, trace, n_it, per_iter = _lm_args(P, want_per_iter, max_iter, u0, v0, rel_tol, hess_includes_fix,
                                               gauge_mode, min_planes_per_pose, verbose, force_hess, problems=B)
        status = np.zeros(B, dtype=np.int32)
        L.check(L.lib().balm_batch_damping_iter(self._h, _p(poses), C.byref(opts), _p(status), n_it, trace,
                                                _p(per_iter)))
        out = []
        for b in range(B):
            p0, p1 = int(self._pose_ptr[b]), int(self._pose_ptr[b + 1])
            tr = _trace_dicts(trace[b * max_iter:b * max_iter + n_it[b]])
            out.append((int(status[b]), poses[p0:p1].copy(), tr,
                        per_iter[:n_it[b], p0:p1].copy() if want_per_iter else None))
        return out

    def pose_covariance(self, poses_list, point_noise=0.0, c_cov=None, include_fix=False, want_raw=True, want_cov=True):
        """Context.pose_covariance per problem, all in one call (include/balm_b200.h, balm_batch_pose_covariance) -> per
        problem (status, Rcov_raw, Rcov). c_cov: per problem a K_p x 9 x 9 array of its observations' cluster
        covariances (concatenated as set_problems concatenates obs10), or None for isotropic point noise. status is
        ERR_NOT_PD (Rcov zero) where H is singular, e.g. without fix clusters; always OK with want_cov=False."""
        poses = self._concat(poses_list)
        ns = [6 * n for n in self.n_poses]
        cc = None
        if c_cov is not None:
            cc = np.ascontiguousarray(np.concatenate([np.asarray(c, dtype=np.float64).reshape(-1, 81) for c in c_cov]),
                                      dtype=np.float64)
            K = C.c_int64()
            L.check(L.lib().balm_batch_sizes(self._h, None, None, None, C.byref(K)))
            if len(cc) != K.value:
                raise ValueError(f"c_cov has {len(cc)} observations, the registration {K.value}")
        size = sum(n * n for n in ns)
        raw = np.zeros(size) if want_raw else None
        cov = np.zeros(size) if want_cov else None
        status = np.zeros(len(ns), dtype=np.int32)
        L.check(L.lib().balm_batch_pose_covariance(self._h, _p(poses), _p(cc), float(point_noise), int(include_fix),
                                                   _p(status), _p(raw), _p(cov)))
        out, o = [], 0
        for b, n in enumerate(ns):
            out.append((int(status[b]), raw[o:o + n * n].reshape(n, n, order="F") if want_raw else None,
                        cov[o:o + n * n].reshape(n, n, order="F") if want_cov else None))
            o += n * n
        return out


class PoseGraph:
    """The pose graph of Context.set_pose_factors for trajectories of any length (include/balm_b200.h, balm_spg_*): H is
    kept as its nonzero 6x6 blocks and the damped system is solved by a block-sparse LDL^T, so memory grows with the
    number of blocks rather than with (6 n_poses)^2."""

    def __init__(self, n_poses, device=0):
        self._h = C.c_void_p()
        self.N = int(n_poses)
        self.n = 6 * self.N
        self._n_factors = 0
        self._n_priors = 0
        L.check(L.lib().balm_spg_create(C.byref(self._h), self.N, int(device)))

    def close(self):
        if self._h:
            L.lib().balm_spg_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_pose_factors(self, factors):
        """Context.set_pose_factors' factors (H_f symmetric to 1e-12 of its max |entry|), checks and result; also orders
        the poses and factors the pattern."""
        status = _set_pose_factors(L.lib().balm_spg_set_factors, self._h, factors)
        self._n_factors = len(status)
        return status

    def set_factor_loss(self, kind, scale=None):
        """Context.set_factor_loss on this handle's factors (evaluate, iterate and covariance use the robust cost)."""
        _set_factor_loss(L.lib().balm_spg_set_factor_loss, self._h, self._n_factors, kind, scale)

    def factor_residuals(self, poses12):
        """Context.factor_residuals on this handle's factors -> (s, w)."""
        return _factor_residuals(L.lib().balm_spg_factor_residuals, self._h, self._n_factors, poses12)

    def set_pose_priors(self, priors, kind="trivial", scale=None):
        """Context.set_pose_priors on this handle (evaluate, iterate and covariance include them). A prior on a pose
        that no factor covers adds that pose's diagonal block to the pattern."""
        status = _set_pose_priors(L.lib().balm_spg_set_pose_priors, self._h, self.N, priors, kind, scale)
        self._n_priors = len(status)
        return status

    def prior_residuals(self, poses12):
        """Context.prior_residuals on this handle's priors -> (s, w)."""
        return _factor_residuals(L.lib().balm_spg_prior_residuals, self._h, self._n_priors, poses12)

    def structure(self):
        """-> dict(pairs, l_blocks, levels, device_bytes): nonzero block pairs of H, blocks of the factor L, levels of
        its elimination tree and the device memory the handle holds."""
        return _block_structure(L.lib().balm_spg_structure, self._h, False)

    def pose_graph_evaluate(self, poses12):
        """-> (pairs [n_pairs, 2] (i <= j), blocks [n_pairs, 6, 6] (H rows of pose i, columns of pose j), g, cost)."""
        poses12 = np.ascontiguousarray(poses12, dtype=np.float64)
        pairs = _block_structure(L.lib().balm_spg_structure, self._h, True)["pair_list"]
        blocks = np.zeros((len(pairs), 36))
        g = np.zeros(self.n)
        r = C.c_double()
        L.check(L.lib().balm_spg_evaluate(self._h, _p(poses12), _p(blocks), _p(g), C.byref(r)))
        return pairs, blocks.reshape(-1, 6, 6).transpose(0, 2, 1), g, r.value

    def covariance(self, poses12, anchor=0):
        """Marginal covariances: Sigma = (H without pose anchor's rows and columns)^-1 on H's block pattern, H the
        Gauss-Newton Hessian at poses12 (anchor=-1: nothing deleted, which leaves the gauge free: ERR_NOT_PD).
        -> (pairs [n_pairs, 2] (i <= j), cov [n_pairs, 6, 6]) with cov[p, a, c] = Sigma[6 i + a, 6 j + c]."""
        pairs = _block_structure(L.lib().balm_spg_structure, self._h, True)["pair_list"]
        return pairs, _covariance(L.lib().balm_spg_covariance, self._h, (poses12,), len(pairs), int(anchor))

    def pose_graph_iter(self, poses12, max_iter=10, u0=0.01, v0=2.0, rel_tol=1e-6, gauge_mode=0, verbose=False,
                        want_per_iter=False, force_hess=False):
        """Context.pose_graph_iter on the sparse solve: same arguments, poses and trace dicts."""
        return _pose_graph_iter(L.lib().balm_spg_iter, self._h, self.N, poses12, max_iter, u0, v0, rel_tol, gauge_mode,
                                verbose, want_per_iter, force_hess)

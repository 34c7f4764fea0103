"""ctypes binding of libbalm_b200.so (include/balm_b200.h). Fails loudly when the CUDA library is missing:
there is no CPU fallback in the product path."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libbalm_b200.so")

OK, ERR_INVALID, ERR_CUDA, ERR_NOT_PD, ERR_TOO_FEW_PLANES, ERR_NCCL, ERR_UNSUPPORTED = range(7)
PREC_FP64, PREC_TENSOR, PREC_BLOCKS = 0, 1, 2
LOSS_TRIVIAL, LOSS_HUBER, LOSS_CAUCHY = 0, 1, 2


class LmOpts(C.Structure):
    _fields_ = [("max_iter", C.c_int), ("u0", C.c_double), ("v0", C.c_double), ("rel_tol", C.c_double),
                ("hess_includes_fix", C.c_int), ("gauge_mode", C.c_int), ("min_planes_per_pose", C.c_int),
                ("verbose", C.c_int), ("force_hess", C.c_int)]


class Trace(C.Structure):
    _fields_ = [("r1", C.c_double), ("r2", C.c_double), ("u", C.c_double), ("v", C.c_double), ("q", C.c_double),
                ("q1", C.c_double), ("accepted", C.c_int), ("recomputed_hess", C.c_int), ("not_pd", C.c_int)]


class Timings(C.Structure):
    _fields_ = [(k, C.c_float) for k in ("ms_stats", "ms_obs", "ms_slice", "ms_syrk", "ms_assemble",
                                         "ms_allreduce", "ms_solve", "ms_residual", "ms_update")] + \
               [("launches", C.c_int), ("n_eval", C.c_int), ("n_solve", C.c_int), ("n_residual", C.c_int),
                ("digit_planes", C.c_int), ("single_sweeps", C.c_int), ("redone_sweeps", C.c_int),
                ("refinements", C.c_int), ("n_stats", C.c_int)]


class AssocOpts(C.Structure):
    _fields_ = [("voxel_size", C.c_double), ("layer_limit", C.c_int), ("min_ps", C.c_int),
                ("eigen_value_array", C.c_double * 3)]


class BalmError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__(f"balm_b200 status {status}: {msg}")
        self.status = status


_lib = None

# every symbol include/balm_b200.h declares (tests check that the library exports all of them)
SYMBOLS = ["balm_last_error", "balm_version", "balm_create", "balm_destroy", "balm_set_voxels",
           "balm_set_voxels_dev", "balm_evaluate", "balm_residual", "balm_solve", "balm_damping_iter",
           "balm_default_lm_opts", "balm_comm_unique_id", "balm_comm_init", "balm_get_timings", "balm_get_reused_sweeps",
           "balm_reset_counters", "balm_sync", "balm_timer_begin", "balm_timer_end", "balm_device_views", "balm_debug_dag_trace",
           "balm_debug_ldlt", "balm_debug_syrk_tc", "balm_debug_tc_planes", "balm_debug_tc_trace", "balm_debug_tc_copy_trace", "balm_synth_virtual",
           "balm_download_voxels", "balm_download_voxel_range", "balm_num_obs", "balm_default_assoc_opts", "balm_cut_voxels", "balm_cut_voxels_stats", "balm_pose_covariance", "balm_marginalize", "balm_download_fix", "balm_append_scan",
           "balm_download_keys", "balm_window_reset", "balm_window_cut", "balm_window_recut", "balm_window_marginalize",
           "balm_window_push", "balm_batch_create", "balm_batch_destroy", "balm_batch_set_voxels", "balm_batch_evaluate",
           "balm_batch_damping_iter", "balm_batch_cut_voxels", "balm_batch_sizes", "balm_batch_download_voxels",
           "balm_batch_pose_covariance", "balm_batch_marginalize", "balm_batch_append_scan", "balm_batch_download_fix",
           "balm_batch_window_reset", "balm_batch_window_cut", "balm_batch_window_recut", "balm_batch_window_marginalize",
           "balm_batch_window_push", "balm_batch_merge_scans", "balm_set_pose_factors", "balm_pose_graph_evaluate",
           "balm_pose_graph_iter", "balm_spg_create", "balm_spg_destroy", "balm_spg_set_factors", "balm_spg_structure",
           "balm_spg_evaluate", "balm_spg_iter", "balm_spg_covariance", "balm_block_structure", "balm_download_blocks",
           "balm_block_covariance", "balm_block_set_factors", "balm_set_factor_loss", "balm_factor_residuals",
           "balm_spg_set_factor_loss", "balm_spg_factor_residuals", "balm_set_pose_priors", "balm_prior_residuals",
           "balm_set_joint_cost",
           "balm_spg_set_pose_priors", "balm_spg_prior_residuals", "balm_set_voxel_loss", "balm_voxel_residuals",
           "balm_batch_set_voxel_loss", "balm_batch_voxel_residuals",
           "balm_set_rig", "balm_rig_evaluate", "balm_rig_damping_iter", "balm_rig_covariance",
           "balm_block_set_rig", "balm_rig_block_structure", "balm_rig_block_covariance",
           "balm_block_point_covariance", "balm_rig_block_point_covariance"]


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; "
                              f"g.build()'` (nvcc, sm_90a). balm_b200 has no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        L.balm_last_error.restype = C.c_char_p
        L.balm_num_obs.restype = C.c_int64
        L.balm_num_obs.argtypes = [C.c_void_p]
        L.balm_create.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int]
        L.balm_destroy.argtypes = [C.c_void_p]
        L.balm_set_voxels.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 5
        L.balm_set_voxels_dev.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 5 + [C.c_int64]
        L.balm_evaluate.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
                                    C.POINTER(C.c_double)]
        L.balm_residual.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_double)]
        L.balm_solve.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int)]
        L.balm_damping_iter.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(LmOpts), C.c_void_p, C.POINTER(C.c_int),
                                        C.c_void_p]
        L.balm_default_lm_opts.argtypes = [C.POINTER(LmOpts)]
        L.balm_comm_unique_id.argtypes = [C.c_void_p]
        L.balm_comm_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.balm_get_timings.argtypes = [C.c_void_p, C.POINTER(Timings)]
        L.balm_get_reused_sweeps.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
        L.balm_reset_counters.argtypes = [C.c_void_p]
        L.balm_sync.argtypes = [C.c_void_p]
        L.balm_timer_begin.argtypes = [C.c_void_p]
        L.balm_timer_end.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
        L.balm_device_views.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
        L.balm_debug_ldlt.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p,
                                      C.POINTER(C.c_double), C.POINTER(C.c_int), C.c_void_p, C.POINTER(C.c_double)]
        L.balm_debug_syrk_tc.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_int,
                                         C.c_void_p]
        L.balm_debug_tc_planes.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int),
                                           C.POINTER(C.c_int64), C.POINTER(C.c_int)]
        L.balm_debug_tc_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.balm_debug_tc_copy_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.balm_synth_virtual.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_double, C.c_double,
                                         C.c_uint64, C.c_void_p, C.c_void_p]
        L.balm_download_voxels.argtypes = [C.c_void_p] + [C.c_void_p] * 4
        L.balm_download_voxel_range.argtypes = [C.c_void_p, C.c_int64, C.c_int64] + [C.c_void_p] * 4 + [C.POINTER(C.c_int64)]
        L.balm_default_assoc_opts.argtypes = [C.POINTER(AssocOpts)]
        L.balm_cut_voxels.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(AssocOpts),
                                      C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.balm_cut_voxels_stats.argtypes = [C.c_void_p, C.c_void_p]
        L.balm_pose_covariance.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_void_p, C.c_void_p]
        L.balm_marginalize.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.balm_download_fix.argtypes = [C.c_void_p, C.c_void_p]
        L.balm_append_scan.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int64),
                                       C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.balm_download_keys.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.balm_window_reset.argtypes = [C.c_void_p, C.POINTER(AssocOpts)]
        L.balm_window_cut.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int]
        L.balm_window_recut.argtypes = [C.c_void_p, C.c_int]
        L.balm_window_marginalize.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        L.balm_window_push.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.balm_batch_create.argtypes = [C.POINTER(C.c_void_p), C.c_int]
        L.balm_batch_destroy.argtypes = [C.c_void_p]
        L.balm_batch_set_voxels.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 7
        L.balm_batch_evaluate.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.balm_batch_damping_iter.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(LmOpts), C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p]
        L.balm_batch_cut_voxels.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 3 + \
                                           [C.POINTER(AssocOpts), C.c_void_p, C.c_void_p]
        L.balm_batch_merge_scans.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 3 + \
                                            [C.c_double, C.c_void_p, C.c_void_p]
        L.balm_batch_sizes.argtypes = [C.c_void_p, C.POINTER(C.c_int)] + [C.POINTER(C.c_int64)] * 3
        L.balm_batch_download_voxels.argtypes = [C.c_void_p] + [C.c_void_p] * 7
        L.balm_batch_pose_covariance.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_int] + \
                                                [C.c_void_p] * 3
        L.balm_batch_marginalize.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.balm_batch_append_scan.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 6
        L.balm_batch_download_fix.argtypes = [C.c_void_p, C.c_void_p]
        L.balm_batch_window_reset.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.POINTER(AssocOpts)]
        L.balm_batch_window_cut.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 3
        L.balm_batch_window_recut.argtypes = [C.c_void_p, C.c_void_p]
        L.balm_batch_window_marginalize.argtypes = [C.c_void_p] + [C.c_void_p] * 3
        L.balm_batch_window_push.argtypes = [C.c_void_p] + [C.c_void_p] * 3
        L.balm_set_pose_factors.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 5
        L.balm_pose_graph_evaluate.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_double)]
        L.balm_pose_graph_iter.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(LmOpts), C.c_void_p, C.POINTER(C.c_int),
                                           C.c_void_p]
        L.balm_spg_create.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_int]
        L.balm_spg_destroy.argtypes = [C.c_void_p]
        L.balm_spg_destroy.restype = None
        L.balm_spg_set_factors.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 5
        L.balm_spg_structure.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.balm_spg_evaluate.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_double)]
        L.balm_spg_iter.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(LmOpts), C.c_void_p, C.POINTER(C.c_int), C.c_void_p]
        L.balm_spg_covariance.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.balm_block_structure.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.balm_download_blocks.argtypes = [C.c_void_p, C.c_void_p]
        L.balm_block_covariance.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.balm_block_set_factors.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 5
        L.balm_set_factor_loss.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.balm_factor_residuals.argtypes = [C.c_void_p] + [C.c_void_p] * 3
        L.balm_spg_set_factor_loss.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.balm_spg_factor_residuals.argtypes = [C.c_void_p] + [C.c_void_p] * 3
        L.balm_set_pose_priors.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 7
        L.balm_prior_residuals.argtypes = [C.c_void_p] + [C.c_void_p] * 3
        L.balm_set_joint_cost.argtypes = [C.c_void_p, C.c_int]
        L.balm_spg_set_pose_priors.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 7
        L.balm_spg_prior_residuals.argtypes = [C.c_void_p] + [C.c_void_p] * 3
        L.balm_set_voxel_loss.argtypes = [C.c_void_p, C.c_int, C.c_double]
        L.balm_voxel_residuals.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]
        L.balm_batch_set_voxel_loss.argtypes = [C.c_void_p, C.c_int, C.c_double]
        L.balm_batch_voxel_residuals.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.balm_set_rig.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 4 + [C.POINTER(C.c_int)]
        L.balm_rig_evaluate.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                        C.POINTER(C.c_double)]
        L.balm_rig_damping_iter.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(LmOpts), C.c_void_p,
                                            C.POINTER(C.c_int), C.c_void_p]
        L.balm_rig_covariance.argtypes = [C.c_void_p] + [C.c_void_p] * 3 + [C.c_double, C.c_int, C.c_int, C.c_void_p,
                                                                              C.c_void_p]
        L.balm_block_set_rig.argtypes = L.balm_set_rig.argtypes
        L.balm_rig_block_structure.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.balm_rig_block_covariance.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.balm_block_point_covariance.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_int,
                                                  C.c_int] + [C.c_void_p] * 4
        L.balm_rig_block_point_covariance.argtypes = [C.c_void_p] + [C.c_void_p] * 3 + [C.c_double, C.c_int, C.c_int,
                                                                                          C.c_int] + [C.c_void_p] * 3
        _lib = L
    return _lib


def check(status):
    if status != OK:
        raise BalmError(status, lib().balm_last_error().decode(errors="replace"))

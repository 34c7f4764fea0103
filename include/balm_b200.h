/*
 * balm_b200.h -- C ABI of libbalm_b200.so: the H100-native (sm_90a) replacement for the inner optimisation loop of
 * BALM 2.0 (VOX_HESS factor evaluation + BALM2::damping_iter()).
 *
 * The reference has no FFI/plugin interface: its seam is the header-level C++ API of
 * src/benchmark/bavoxel.hpp.  Every entry point below names the reference interface it
 * replaces (file:line relative to the reference BALM sources).  include/bavoxel_b200.hpp is the C++ shim that keeps the
 * reference's class/method names on top of this ABI; balm_b200/ (Python) mirrors the same names via ctypes.
 * INTEGRATION.md shows the binding a BALM maintainer adds.
 *
 * Conventions (same as the reference, SURVEY.md section 8b):
 *   poses12 : N x 12 doubles; per pose R column-major (Eigen default) then p    -- IMUST::R, IMUST::p
 *                                                                    (include/tools.hpp:141-201)
 *   obs10   : K x 10 doubles; per (voxel,pose) observation P00,P01,P02,P11,P12,P22,v0,v1,v2,N
 *                                                      -- PointCluster{P,v,N} (include/tools.hpp:290-349)
 *   row_ptr : M+1 int64 CSR offsets voxel -> observations; pose_idx : K int32, ascending inside a voxel.
 *             A slot is present iff PointCluster::N != 0 (bavoxel.hpp:34,332).
 *   coe     : M doubles, push_voxel weight (bavoxel.hpp:42-48)
 *   fix10   : M x 10 doubles or NULL, the fixed / marginalised cluster sig_vecs[a] (bavoxel.hpp:47,441)
 *   H       : n x n doubles, column-major, full symmetric, n = 6N; block (i,j) at rows 6i.., cols 6j..
 *             (bavoxel.hpp:394,416); g : n; unknown order per pose [phi(3), dt(3)] (DVEL = 6, tools.hpp:20)
 * All pointers are HOST pointers unless the name ends in _dev.  No torch/Eigen types cross this boundary.
 * A context owns one CUDA stream and is not re-entrant; distinct contexts are independent.
 */
#ifndef BALM_B200_H
#define BALM_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct balm_ctx balm_ctx;

typedef enum {
  BALM_OK = 0,
  BALM_ERR_INVALID = 1,        /* bad argument / call order */
  BALM_ERR_CUDA = 2,           /* CUDA runtime error, see balm_last_error() */
  BALM_ERR_NOT_PD = 3,         /* (H + u D) had a zero/tiny pivot; LM treats it as a rejected step */
  BALM_ERR_TOO_FEW_PLANES = 4, /* reference prints + exit(0) (bavoxel.hpp:1079-1085) */
  BALM_ERR_NCCL = 5,
  BALM_ERR_UNSUPPORTED = 6
} balm_status;

/* Arithmetic of the rank-3M Hessian accumulation  H -= G' G'^T  (bavoxel.hpp:385,392,410-416). */
typedef enum {
  BALM_PREC_FP64 = 0,   /* fp64 DMMA accumulation (BASELINE config C2, "fp64 accumulation") */
  BALM_PREC_TENSOR = 1, /* int8 tensor-core split-integer (Ozaki) accumulation, exact int32 sums, fp64 result */
  BALM_PREC_BLOCKS = 2  /* fp64, H held as the 6x6 blocks of the pose pairs sharing a voxel (plus every diagonal pair)
                           and the damped system solved by the sparse pose graph's nested-dissection block LDL^T (DESIGN.md
                           "Block-sparse voxel BA"). Nothing of size (6N)^2 is allocated, so windows of thousands of
                           scans with local co-visibility fit. g, the residual and the diagonal blocks' sweep terms are
                           bitwise those of BALM_PREC_FP64. Single batch: 144 B per observation must fit the G' budget
                           (16 GB, BALM_G_BUDGET_MB), else the registration is BALM_ERR_UNSUPPORTED and leaves the
                           context without voxels, as do 2^31 observation pairs or 2^30 block pairs. balm_comm_init,
                           balm_pose_covariance, balm_set_pose_factors, balm_pose_graph_*, balm_device_views and the
                           tensor debug aids return BALM_ERR_UNSUPPORTED on such a context and change nothing;
                           balm_evaluate's H (when not NULL) is the dense matrix expanded from the blocks. Pose factors
                           join the voxel cost through balm_block_set_factors (on FP64 / TENSOR contexts through
                           balm_set_joint_cost). */
} balm_precision;

/* Robust losses of pose factors (balm_set_factor_loss), rho of s = e~^T H~ e~ at scale c > 0 (units of sqrt(s)), and of
 * voxels (balm_set_voxel_loss), rho of s = lambda_min at a scale c in metres. */
typedef enum {
  BALM_LOSS_TRIVIAL = 0, /* rho = s */
  BALM_LOSS_HUBER = 1,   /* rho = s for s <= c^2, else 2 c sqrt(s) - c^2 */
  BALM_LOSS_CAUCHY = 2   /* rho = c^2 log(1 + s / c^2) */
} balm_loss;

typedef struct {
  int max_iter;             /* 10  (bavoxel.hpp:1104); benchmark_virtual twin: 20 (benchmark_virtual.cpp:408) */
  double u0;                /* 0.01 (bavoxel.hpp:1087); twin: 0.1 (benchmark_virtual.cpp:380) */
  double v0;                /* 2 */
  double rel_tol;           /* 1e-6 (bavoxel.hpp:1155); < 0 disables the convergence exit (timing runs) */
  int hess_includes_fix;    /* 0: bavoxel.hpp:325 (fix ignored in H,g); 1: benchmark_virtual.cpp:241-243 */
  int gauge_mode;           /* 0: bavoxel.hpp:1159-1164; 1: benchmark_virtual.cpp:472-479; 2: none */
  int min_planes_per_pose;  /* 20 (bavoxel.hpp:1079); 0 disables the precheck */
  int verbose;              /* 1: print the reference's per-iteration line (bavoxel.hpp:1132) */
  int force_hess;           /* 1: re-evaluate H,g every iteration even after a rejected step (benchmarks: makes
                               every LM iteration the same amount of work; the reference reuses H, :1148) */
} balm_lm_opts;

typedef struct {
  double r1, r2, u, v, q, q1; /* exactly the values printed at bavoxel.hpp:1132 */
  int accepted;
  int recomputed_hess;
  int not_pd;
} balm_trace;

/* Per-phase device time (CUDA events on the ctx stream), SUMMED since balm_reset_counters(), with the
 * number of evaluations / solves / residual passes that contributed and the kernels launched. */
typedef struct {
  float ms_stats, ms_obs, ms_slice, ms_syrk, ms_assemble, ms_allreduce, ms_solve, ms_residual, ms_update;
  int launches;   /* kernels launched by the library since balm_reset_counters() */
  int n_eval, n_solve, n_residual;
  int digit_planes; /* tensor path: int8 digit planes used by the last evaluation (3 or 4, chosen on the device) */
  int single_sweeps; /* tensor path: evaluations whose one fused observation sweep (column scales speculated from the
                        previous evaluation) was accepted ... */
  int redone_sweeps; /* ... and those whose scales failed the check, so the digit-plane sweep ran again */
  int refinements;   /* solves whose backward-error check asked for fp64 iterative refinement (indefinite H + uD) */
  int n_stats;       /* evaluations that ran the per-voxel eigen pass themselves (ms_stats sums only these): inside
                        balm_damping_iter the residual pass of the previous step usually hands its results over */
} balm_timings;

const char *balm_last_error(void);
int balm_version(void);

/* ctx lifetime. `device` is the CUDA ordinal. Replaces constructing VOX_HESS + BALM2 (bavoxel.hpp:21,984). */
int balm_create(balm_ctx **out, int n_poses, int device, int precision);
int balm_destroy(balm_ctx *ctx);

/* Registers all plane voxels at once = the sequence of VOX_HESS::push_voxel calls (bavoxel.hpp:30-51) made by
 * OCTO_TREE_NODE::tras_opt (bavoxel.hpp:908-929). Host arrays are copied (H2D) and may be freed on return. */
int balm_set_voxels(balm_ctx *ctx, int64_t n_voxels, const int64_t *row_ptr, const int32_t *pose_idx,
                    const double *obs10, const double *fix10, const double *coe);
/* n_voxels == 0 registers an EMPTY shard (row_ptr = {0}): evaluations contribute zeros and the rank still takes part
 * in every collective of a multi-GPU job. */
/* Same, but the arrays already live in device memory of ctx's GPU (used for HBM-resident timing). */
int balm_set_voxels_dev(balm_ctx *ctx, int64_t n_voxels, const int64_t *row_ptr_dev, const int32_t *pose_idx_dev,
                        const double *obs10_dev, const double *fix10_dev, const double *coe_dev, int64_t n_obs);

/* VOX_HESS::left_evaluate_acc2(xs, head, end, Hess, JacT, residual) (bavoxel.hpp:304-426).
 * H (n*n) and g (n) may be NULL to keep the result on the device only. With a communicator attached
 * (balm_comm_init) the result is the all-reduced sum over ranks = divide_thread_left's reduction
 * (bavoxel.hpp:1049-1056). head/end select a voxel range of THIS rank's voxels ([0,M) = all). */
int balm_evaluate(balm_ctx *ctx, const double *poses12, int64_t head, int64_t end, int include_fix, double *H,
                  double *g, double *residual);
/* VOX_HESS::evaluate_only_residual(xs, residual) (bavoxel.hpp:428-470) */
int balm_residual(balm_ctx *ctx, const double *poses12, double *residual);
/* D = diag(H); dx = (H + u D)^-1 (-g); q1 = 0.5 dx.(u D dx - g) on the H,g of the last balm_evaluate
 * (bavoxel.hpp:1113-1114,1127). not_pd set when the LDL^T met a zero/tiny pivot. dx (n) may be NULL. */
int balm_solve(balm_ctx *ctx, double u, double *dx, double *q1, int *not_pd);
/* BALM2::damping_iter(x_stats, voxhess) (bavoxel.hpp:1069-1166). poses12 updated in place.
 * trace: room for opts->max_iter entries (may be NULL). poses_per_iter: max_iter*N*12 doubles or NULL,
 * receives the accepted pose set after every iteration (before the gauge step) for parity checks.
 * On a BALM_PREC_BLOCKS context, or a dense one with the joint cost on (balm_set_joint_cost), with an active pose prior
 * (balm_set_pose_priors) gauge_mode 0 and 1 are BALM_ERR_INVALID: the priors fix the frame, and re-anchoring to pose 0
 * would move the result off them; pass 2. */
int balm_damping_iter(balm_ctx *ctx, double *poses12, const balm_lm_opts *opts, balm_trace *trace, int *n_iters,
                      double *poses_per_iter);
void balm_default_lm_opts(balm_lm_opts *opts);

/* Robust voxel cost (DESIGN.md "Robust voxels"): one loss kind (balm_loss) and scale c > 0 in metres -- a plane
 * thickness -- for every voxel of the context. With s_v = lambda_min(C_v) (m^2) of the cluster the pass builds (its
 * observations at the given poses, plus the fix cluster exactly where that pass adds it) and w_v = rho'(s_v), voxel v
 * contributes cost coe_v rho(s_v) (no 1/2: a trivial loss is the plain cost), gradient w_v coe_v grad(lambda_min) and
 * Hessian w_v times the voxel's Hessian without a loss (iteratively reweighted; the rho'' term is left out). Every H, g
 * and covariance therefore equals that of a trivial-loss context registered with coe_v w_v, the weights frozen at the
 * given poses. The loss applies to every call that evaluates voxels: balm_evaluate (any range), balm_residual,
 * balm_damping_iter, balm_solve, balm_download_blocks, balm_pose_covariance and balm_block_covariance. Useful scales:
 * inliers with point noise sigma_p have sqrt(lambda_min) slightly below sigma_p, so c = 1.5 - 3 sigma_p.
 * BALM_LOSS_TRIVIAL resets (scale ignored); a trivial loss's outputs are bitwise those without one. BALM_ERR_INVALID, the
 * previous loss kept, for a kind outside BALM_LOSS_* or a non-trivial kind without a finite scale > 0. Works on every
 * precision; the loss belongs to the context and survives every voxel registration (balm_set_voxels, _dev,
 * balm_cut_voxels, balm_marginalize, balm_append_scan, balm_window_push, balm_synth_virtual, the empty set). With a
 * communicator attached every rank must set the same loss (it is not checked). */
int balm_set_voxel_loss(balm_ctx *ctx, int kind, double scale);
/* s_v = lambda_min and w_v = rho'(s_v) of the voxels [head, end) of this rank at poses12, into lam and w (end - head
 * each; either may be NULL), with the fix clusters when include_fix. w is bitwise the weight an evaluation at these
 * poses applies (1 without a loss). Waits once. BALM_ERR_INVALID for a null ctx or poses12, no registered voxels or a
 * bad range. */
int balm_voxel_residuals(balm_ctx *ctx, const double *poses12, int64_t head, int64_t end, int include_fix, double *lam,
                         double *w);

/* Association on the GPU (SURVEY.md section 8f, row N1): raw scans + initial poses -> plane voxels, registered in the
 * ctx exactly as balm_set_voxels would. Replaces the loop  cut_voxel(surf_map, *pl_fulls[i], x_buf[i], i)  over all scans
 * followed by  recut(win_size); tras_opt(voxhess, win_size)  over all root voxels
 * (benchmark_realworld.cpp:187-200 -> bavoxel.hpp:1170-1223, 737-776, 908-929, 30-51).
 * xyz: n_points x 3 float32 in the BODY frame (the PCD floats), frame: n_points pose indices, poses12: N x 12.
 * opts may be NULL (reference constants: voxel_size 1, layer_limit 2, min_ps 15, eigen ratios 1/16). */
typedef struct {
  double voxel_size;          /* bavoxel.hpp:15; benchmark_realworld.launch sets 2 */
  int layer_limit;            /* bavoxel.hpp:8  (0..2) */
  int min_ps;                 /* bavoxel.hpp:12 */
  double eigen_value_array[3];/* bavoxel.hpp:11; benchmark_realworld.cpp:183-185 sets {1/16, 1/16, 1/9} */
} balm_assoc_opts;
void balm_default_assoc_opts(balm_assoc_opts *opts);
/* Device memory: BALM_ASSOC_BUDGET_MB (read at every call, default 16384; fractions allowed) bounds the association's
 * device scratch. The bound of the call is n_points x P + F bytes, P = 345 + 120 (layer_limit + 1) per point (one
 * segment per point per layer, the worst case) and F = 200 N + 1 MiB; balm_cut_voxels_stats reports both. When it fits
 * the budget (and n_points < 2^31) the points are cut in one pass. Otherwise they are cut in root-key slabs: a pass over
 * the points counts every root voxel's points, the roots are grouped in ascending key order into slabs of at most
 * cap = (budget - F) / P points (and < 2^31), and each slab's points are selected in their input order and cut on their
 * own, then every slab's voxels are registered at once. The result is bitwise that of the one-pass cut (every decision
 * about a voxel depends only on the points of its root voxel; DESIGN.md section 7), so n_points may be 2^31 or more.
 * The device peak is the larger of the budget and the registration; the slabs' voxels are staged in host memory (84 B
 * per observation, 28 B per voxel) on top of the caller's points (16 B per point: xyz and frame), and the slab path
 * streams the points through two pinned buffers of at most 2^23 points. Errors, each leaving the registered voxel set
 * as it was: BALM_ERR_INVALID for a frame outside [0, N), a point outside the +-2^18 root-voxel range, or no plane
 * voxel; BALM_ERR_UNSUPPORTED (slab path) for a root voxel holding more than cap points (the message gives both), a
 * table of the roots that does not fit the budget, or 2^31 or more observations. */
int balm_cut_voxels(balm_ctx *ctx, int64_t n_points, const float *xyz, const int32_t *frame, const double *poses12,
                    const balm_assoc_opts *opts, int64_t *n_voxels_out, int64_t *n_obs_out);
/* The last successful balm_cut_voxels, into stats[BALM_CUT_STATS]: [0] slabs (1 in one pass), [1] points in the largest
 * slab, [2] root voxels, [3] peak device scratch bytes (as allocated by the call, counted by request), [4] host-to-device
 * bytes (points, poses, and in the slab path every re-streamed chunk and the registration's upload), [5] P and [6] F of
 * the scratch bound above, then wall times in microseconds: [7] root-count pass, [8] slab selection, [9] cuts (the whole
 * cut in one pass), [10] registration. All zero before the first cut. */
#define BALM_CUT_STATS 11
int balm_cut_voxels_stats(balm_ctx *ctx, int64_t *stats);

/* Sliding-window marginalisation of the registered voxel set (SURVEY.md section 8f, row N2) =
 * OCTO_TREE_ROOT::marginalize -> OCTO_TREE_NODE::to_margi on every plane leaf (bavoxel.hpp:948-963, 778-816) followed by
 * the re-registration tras_opt -> push_voxel would make (bavoxel.hpp:908-929, 30-51): the clusters of the oldest mg_size
 * scans, transformed by poses12 (the optimised poses, N x 12), are added to the voxel's fix cluster when that holds fewer
 * than 50 points (:790), the remaining scans shift down by mg_size (pose slot i := old slot i + mg_size; the caller shifts
 * its pose array the same way, consistency.cpp:137-140), voxels left with fewer than min_ps points or fewer than two
 * observing scans are not pushed, coe = points left. Everything stays in HBM; the context is re-registered as if
 * balm_set_voxels had been called with the new set (n_poses unchanged: the last mg_size slots are empty until new scans
 * are associated). balm_download_fix copies the fix clusters (M x 10) back. */
int balm_marginalize(balm_ctx *ctx, int mg_size, const double *poses12, int min_ps, int64_t *n_voxels_out,
                     int64_t *n_obs_out);
int balm_download_fix(balm_ctx *ctx, double *fix10);
/* The other half of the sliding window: a NEW scan is associated with the voxel set already in HBM (which must come from
 * balm_cut_voxels: it carries the 63-bit octree key of every voxel). Every point (xyz: n_points x 3 float32, body frame)
 * is transformed by poses12[slot], finds the plane leaf that contains it with the arithmetic of cut_voxel / cut_func
 * (bavoxel.hpp:1170-1223, 700-735), and the body-frame moments of a leaf's new points become its observation in pose
 * slot `slot` (which must lie above every scan already in the window); then EVERY voxel is re-judged as recut does
 * (bavoxel.hpp:737-776 -> judge_eigen :654-699) from its fix cluster and all its clusters transformed by poses12 (N x 12):
 * still planar (eigen ratio below the threshold of its layer), more than min_ps window points, at least two scans ->
 * kept with coe = window points; otherwise dropped. Not done here (it happens at the next full balm_cut_voxels): new
 * roots / leaves from points outside the registered planes, re-splitting a leaf that stopped being planar.
 * n_matched_out: points that fell into a registered voxel. balm_download_keys copies the M voxel keys
 * ([root x|y|z biased by 2^18, 19 bits each | octant at layer 1 | octant at layer 2], 7 = not split) and their octree
 * layers (0..2; a digit 7 is also octant 7, the layer tells the two apart); either pointer may be NULL. */
int balm_append_scan(balm_ctx *ctx, int64_t n_points, const float *xyz, const double *poses12, int slot,
                     int64_t *n_voxels_out, int64_t *n_obs_out, int64_t *n_matched_out);
int balm_download_keys(balm_ctx *ctx, uint64_t *keys, int32_t *layers);

/* Persistent sliding-window octree in HBM = the reference's surf_map of OCTO_TREE_ROOTs kept across window shifts
 * (consistency.cpp / benchmark_realworld.cpp driver loops). Window slots are the ctx's N pose slots. Unlike
 * balm_append_scan / balm_marginalize, which work on the flattened voxel set, the window keeps every node the reference
 * keeps: points outside the known planes grow new roots and leaves, a leaf that stops being planar is split further, and
 * a leaf that is not pushed stays in the map, dormant, with its fix cluster until later scans hit it again. Nodes are
 * never deleted (the reference never deletes them either): the map grows with the trajectory, by 120 + 160 * N bytes
 * per node (key, problem, flags, fix cluster, lookup entry, and sig_orig + sig_tran for every slot), plus 56 bytes per
 * point held. This is the one-problem case of balm_batch_window_* below.
 * The window is independent of the registered voxel set: balm_set_voxels, balm_cut_voxels, balm_append_scan,
 * balm_marginalize and balm_synth_virtual do not touch it; balm_destroy frees it. A rejected call (BALM_ERR_INVALID:
 * slot outside [0, N), win_count outside [1, N], mg_size outside [1, win_count), no balm_window_reset before) leaves the
 * window unchanged. */
int balm_window_reset(balm_ctx *ctx, const balm_assoc_opts *opts);
/* empty map with these association parameters (opts NULL = balm_default_assoc_opts; eigen ratios rounded to float) */
int balm_window_cut(balm_ctx *ctx, int64_t n_points, const float *xyz, const double *pose12, int slot);
/* cut_voxel(surf_map, scan, x, slot) (bavoxel.hpp:1170-1223): xyz n_points x 3 float32 in the body frame, pose12 the
 * scan's pose; every point's world coordinate R p + t (fp64) picks its root voxel (created on first use), and the point
 * is pushed into that root's slot `slot` -- also when the root is already split: such points wait for the next recut. */
int balm_window_recut(balm_ctx *ctx, int win_count);
/* OCTO_TREE_NODE::recut(win_count) on every root (bavoxel.hpp:737-776, judge_eigen :654-699, cut_func :700-735): a node
 * that is not split is judged from fix_point + sig_tran of the slots < win_count (push_state = 1 when planar with more
 * than min_ps window points); a node that is not planar below layer_limit is split for good and the points of its slots
 * < win_count move to the octant children; a node split earlier moves the points of slot win_count - 1 only. */
int balm_window_marginalize(balm_ctx *ctx, int mg_size, const double *poses12 /* N x 12 or NULL */, int win_count);
/* OCTO_TREE_ROOT::marginalize(mg_size, x_poses, win_count) (bavoxel.hpp:948-963, to_margi :778-816) on every node that
 * is not split: with poses12, sig_tran and vec_tran of the slots < win_count are re-transformed by them; a node with
 * push_state 1 and fewer than 50 fix points adds sig_tran of the slots < mg_size to its fix cluster; slots mg_size ..
 * win_count - 1 shift down by mg_size and the top mg_size slots are cleared (their points are gone). */
int balm_window_push(balm_ctx *ctx, int win_count, int64_t *n_voxels_out, int64_t *n_obs_out);
/* tras_opt(voxhess, win_count) on every root (bavoxel.hpp:908-929, push_voxel :30-51): every node that is not split,
 * has push_state 1, at least min_ps points in the slots < win_count and at least two non-empty slots is registered in
 * the ctx as balm_set_voxels would (rows = its non-empty sig_orig slots, fix cluster = its fix_point, coe = its points),
 * in ascending node key; balm_download_keys / balm_download_fix read them back. No such node -> an empty voxel set. */

/* Batched bundle adjustment: B independent small problems (an HBA bottom layer of short windows, one BALM2 per window)
 * registered once and optimised together on one GPU. A batch has its own handle and stream: it does not allocate the
 * dense n x n buffers of a balm_ctx, so a batch of 400 problems of 10 poses pays for 400 blocks of 60 x 60, not for one
 * matrix of 24 000^2. fp64 arithmetic throughout (the BALM_PREC_FP64 contract); no tensor path, no communicator.
 * Problem p owns the poses [pose_ptr[p], pose_ptr[p+1]) of the concatenated pose array (1 <= count <=
 * BALM_BATCH_MAX_POSES) and the voxels [voxel_ptr[p], voxel_ptr[p+1]) (may be empty). row_ptr / obs10 / coe / fix10 as
 * balm_set_voxels, over all voxels (fix10: every voxel or NULL; all-zero rows for problems without fix clusters).
 * pose_idx is problem-local (0 .. N_p - 1), ascending inside a voxel. Host arrays, copied. A malformed registration
 * (n_problems < 1; a problem with 0 or more than BALM_BATCH_MAX_POSES poses; pose_ptr / voxel_ptr / row_ptr not starting
 * at 0 or not ascending; pose_idx out of its problem's range or not ascending inside a voxel -- checked on the device)
 * returns BALM_ERR_INVALID and leaves the previous registration in place. */
#define BALM_BATCH_MAX_POSES 32   /* per problem: 6N <= 192 unknowns */
typedef struct balm_batch balm_batch;
int balm_batch_create(balm_batch **out, int device);
int balm_batch_destroy(balm_batch *b);
int balm_batch_set_voxels(balm_batch *b, int n_problems, const int64_t *pose_ptr, const int64_t *voxel_ptr,
                          const int64_t *row_ptr, const int32_t *pose_idx, const double *obs10,
                          const double *fix10, const double *coe);
/* left_evaluate_acc2 per problem, at poses12 (P x 12, P = pose_ptr[B]). H: the problems' full column-major (6N_p)^2
 * blocks one after the other, g: 6P, residual: B. H, g may be NULL. */
int balm_batch_evaluate(balm_batch *b, const double *poses12, int include_fix, double *H, double *g, double *residual);
/* balm_set_voxel_loss for a batch: one loss for every voxel of every problem, used by balm_batch_evaluate,
 * balm_batch_damping_iter and balm_batch_pose_covariance. Same refusals; it belongs to the batch and survives every
 * registration (set_voxels, cut_voxels, marginalize, append_scan, window_push), whatever the problem count. */
int balm_batch_set_voxel_loss(balm_batch *b, int kind, double scale);
/* balm_voxel_residuals over all voxels of the registration, in registration order (voxel_ptr[B] each). */
int balm_batch_voxel_residuals(balm_batch *b, const double *poses12, int include_fix, double *lam, double *w);
/* balm_damping_iter per problem, all problems advanced together: each problem's iterations are exactly those of
 * balm_damping_iter on a BALM_PREC_FP64 context holding only that problem (precheck, u0 / v0, accept rule, reused H after a
 * rejected step unless force_hess, rel_tol exit, hess_includes_fix, gauge_mode on the problem's own pose 0). A converged
 * problem stops; the others go on. poses12: P x 12, updated in place for problems with status BALM_OK.
 * status[B]: BALM_OK or BALM_ERR_TOO_FEW_PLANES (that problem is left untouched, n_iters 0). n_iters[B].
 * trace: [B][max_iter] or NULL (entries past a problem's n_iters are zero); poses_per_iter: [max_iter][P][12] or NULL
 * (a problem's rows past its n_iters repeat its last poses; rows past the batch's last iteration are not written). opts->verbose != 0 is rejected (BALM_ERR_INVALID): the traces are
 * returned instead of printed. The host waits once per iteration. */
int balm_batch_damping_iter(balm_batch *b, double *poses12, const balm_lm_opts *opts, int *status, int *n_iters,
                            balm_trace *trace, double *poses_per_iter);
/* Association for a batch: the plane voxels of every problem cut from raw scans on the device and registered as
 * balm_batch_set_voxels would register them. Scans are given once: scan s is xyz[scan_ptr[s] .. scan_ptr[s+1]) (float32,
 * body frame). Problem p owns the pose rows [pose_ptr[p], pose_ptr[p+1]) of poses12 (P x 12, the initial poses, the
 * same array later passed to balm_batch_damping_iter); pose row j is scan pose_scan[j] in slot j - pose_ptr[p].
 * Windows may share scans (HBA windows overlap by half); each problem sees only its own slots.
 * Problem p's voxels are bitwise those balm_cut_voxels registers on a context of N_p poses given the points of its scans
 * concatenated in slot order, frame = slot, and its pose rows (ascending node key; row_ptr, pose_idx = slot, obs10, coe,
 * keys, layers). opts as balm_cut_voxels (NULL: the defaults; eigen ratios rounded to float). A problem without a plane
 * voxel gets an empty voxel range; balm_batch_damping_iter then reports BALM_ERR_TOO_FEW_PLANES for it unless
 * min_planes_per_pose is 0. No fix clusters (balm_batch_marginalize adds them). A problem's result depends on nothing else in the batch; two calls are
 * bitwise equal. Points are uploaded once; host synchronisations and allocations are a fixed number per octree layer,
 * whatever the number of problems. BALM_ERR_INVALID (the previous registration stays in place): the problem-table checks
 * of balm_batch_set_voxels, scan_ptr not starting at 0 or not ascending, a pose_scan entry outside [0, n_scans),
 * layer_limit outside 0..2, a point outside the +-2^18 root-voxel range. BALM_ERR_UNSUPPORTED, before anything is
 * allocated: 2^31 or more points, counted once per pose row that uses them (or in xyz). n_voxels_out / n_obs_out: [B]
 * or NULL. */
int balm_batch_cut_voxels(balm_batch *b, int n_problems, const int64_t *pose_ptr, const int32_t *pose_scan,
                          int n_scans, const int64_t *scan_ptr, const float *xyz, const double *poses12,
                          const balm_assoc_opts *opts, int64_t *n_voxels_out, int64_t *n_obs_out);
/* Keyframes of a batch, the step between two layers of hierarchical BA: every window's scans merged into one down-sampled
 * cloud in the body frame of its slot 0, on the device. The problem table and scan pool have the meaning they have in
 * balm_batch_cut_voxels (scans given once, windows may share scans, pose row j is scan pose_scan[j] in slot
 * j - pose_ptr[p]); poses12 holds the rows as balm_batch_damping_iter returns them (P x 12, read only).
 * Keyframe p: every point b of every slot k, expressed in the body frame of the problem's anchor a = slot 0,
 *   q = R_a^T (R_k b + t_k - t_a),
 * reduced by down_sampling_voxel (tools.hpp:203-242) at voxel_size: one point per occupied voxel, the mean of its points.
 * It is kf_xyz[kf_ptr[p] .. kf_ptr[p+1]) (float32 x 3), voxels in ascending (ix, iy, iz). kf_ptr: [B + 1]; the caller
 * sizes kf_xyz for n_items = sum_j |scan pose_scan[j]| points (it may be NULL when that is 0). voxel_size < 0.001: no
 * reduction, as in the reference: keyframe p is its transformed points in (slot, point) order.
 * The arithmetic is fixed so that a numpy restatement reproduces it bit for bit: the transform in fp64, each operation
 * correctly rounded in the order written, without contraction: ((r0 b0 + r1 b1) + r2 b2) + t, then - t_a, then R_a^T in
 * the same form, rounded to float32; voxel index = the float32 quotient q / (float)voxel_size, minus 1 if negative,
 * truncated; mean = the fp64 sum of a voxel's float32 points in item order (slot, then point) over their count, rounded
 * to float32. The reference keeps a float32 running mean in hash-map order instead; this deterministic mean is the one
 * balm_b200.drivers.down_sampling_voxel takes. A problem's keyframe does not depend on the rest of the batch or on its
 * position in it; two calls are bitwise equal. The registration and the window maps are not touched.
 * Host waits: 3 stream synchronisations (entry, the B + 1 offsets, the keyframes; 2 without reduction); about 20 device
 * allocations, freed by the call, whatever B. BALM_ERR_INVALID leaves kf_ptr and kf_xyz unwritten: the problem-table
 * checks of balm_batch_set_voxels, scan_ptr not starting at 0 or not ascending, a pose_scan entry outside [0, n_scans),
 * a non-finite voxel_size, a voxel index outside +-2^20 (checked on the device; the message names the lowest such
 * problem). BALM_ERR_UNSUPPORTED, before anything is allocated: 2^31 or more points, counted once per pose row that uses
 * them (or in xyz). */
int balm_batch_merge_scans(balm_batch *b, int n_problems, const int64_t *pose_ptr, const int32_t *pose_scan,
                           int n_scans, const int64_t *scan_ptr, const float *xyz, const double *poses12,
                           double voxel_size, int64_t *kf_ptr, float *kf_xyz);
/* Sizes of the current registration, then a copy of it (any pointer may be NULL): voxel_ptr [B + 1], row_ptr [M + 1]
 * (over all voxels), pose_idx [K] (problem-local), obs10 [K x 10], coe [M]; keys / layers [M] as balm_download_keys, per
 * problem in ascending key, only after balm_batch_cut_voxels (non-NULL otherwise -> BALM_ERR_INVALID). Fix clusters
 * are not copied (balm_batch_download_fix below). No registration -> BALM_ERR_INVALID. */
int balm_batch_sizes(balm_batch *b, int *n_problems, int64_t *n_poses, int64_t *n_voxels, int64_t *n_obs);
int balm_batch_download_voxels(balm_batch *b, int64_t *voxel_ptr, int64_t *row_ptr, int32_t *pose_idx, double *obs10,
                               double *coe, uint64_t *keys, int32_t *layers);
/* The sliding-window step for a batch (balm_marginalize + balm_append_scan per problem, all problems in one call each).
 * poses12: P x 12, the problems' pose rows as balm_batch_damping_iter returns them (read only); N_p does not change.
 * balm_batch_marginalize: problem p with mg_size[p] in [1, N_p) gets exactly what balm_marginalize(ctx_p, mg_size[p],
 * its pose rows, min_ps) registers on a BALM_PREC_FP64 context holding only problem p: row_ptr, pose_idx shifted down by
 * mg_size[p], obs10 moved (not recomputed), fix clusters (a fix cluster of 50 or more points absorbs nothing, :790), coe,
 * and keys and layers compacted when the registration carries them. mg_size[p] == 0 leaves problem p bitwise untouched.
 * Where the context call would fail (no voxel is left with two observing scans) or the problem has no voxels, the problem
 * gets an empty voxel range (n_voxels_out[p] = 0). Afterwards the registration holds fix clusters for every voxel (zero
 * rows for untouched problems that had none). n_voxels_out / n_obs_out: [B] or NULL.
 * balm_batch_append_scan: scans are given once, as in balm_batch_cut_voxels (scan s = xyz[scan_ptr[s] .. scan_ptr[s+1]),
 * float32, body frame); one scan may serve several problems. Problem p with scan_of[p] >= 0 gets exactly what
 * balm_append_scan(ctx_p, that scan, its pose rows, slot[p]) registers: keys, layers, row_ptr, pose_idx, obs10, fix
 * clusters (kept only if the registration has them), coe and n_matched_out[p]. scan_of[p] == -1 leaves problem p bitwise
 * untouched. The registration must carry keys (balm_batch_cut_voxels, possibly followed by these two calls): the leaves
 * are found and re-judged with the association options of that cut. Where the context call would fail (no plane voxel
 * survives) the problem gets an empty voxel range and n_matched_out[p] = 0. n_voxels_out / n_obs_out / n_matched_out:
 * [B] or NULL.
 * Both: BALM_ERR_INVALID leaves the previous registration in place: no registration; mg_size outside {0} and [1, N_p);
 * scan_of outside -1 and [0, n_scans); slot outside [0, N_p); an empty scan; scan_ptr not starting at 0 or not
 * ascending; a registration without keys (append); a slot not above every scan already observing one of the problem's
 * voxels (checked on the device; the message names the lowest such problem). BALM_ERR_UNSUPPORTED, before anything is
 * allocated: 2^31 or more points, counted once per problem that takes them (or in xyz). A problem's result depends on
 * nothing else in the batch; two calls are bitwise equal. Host waits and allocations are a fixed number per call,
 * whatever B: 5 stream synchronisations in each call (entry, per-problem offsets, emission, and the registration's check
 * and workspaces as in balm_batch_set_voxels), and about 40 (marginalise) or 50 (append) device allocations, most of
 * them the new registration's arrays and workspaces.
 * balm_batch_download_fix: the registration's fix clusters, M x 10 (zero rows where a voxel has none, all zero when the
 * registration has no fix clusters). */
int balm_batch_marginalize(balm_batch *b, const int *mg_size, const double *poses12, int min_ps, int64_t *n_voxels_out,
                           int64_t *n_obs_out);
int balm_batch_append_scan(balm_batch *b, const int32_t *scan_of, const int *slot, int n_scans, const int64_t *scan_ptr,
                           const float *xyz, const double *poses12, int64_t *n_voxels_out, int64_t *n_obs_out,
                           int64_t *n_matched_out);
int balm_batch_download_fix(balm_batch *b, double *fix10);
/* Persistent sliding-window octrees for a batch: B independent window maps (balm_window_* above), one per problem, kept
 * in HBM across shifts and driven together; balm_batch_window_push turns them into the batch's registration, so
 * balm_batch_damping_iter, balm_batch_pose_covariance, balm_batch_marginalize and balm_batch_append_scan run on it.
 * balm_batch_window_reset: problem p gets n_slots[p] (1 .. BALM_BATCH_MAX_POSES) window slots and owns the pose rows
 * [sum_{q<p} n_slots[q], ...) of every poses12 (P x 12, P = sum n_slots), laid out as in the other batch calls; opts as
 * balm_window_reset (NULL = defaults), the same for every problem. Replaces any earlier window maps.
 * balm_batch_window_cut: scans are given once (scan s = xyz[scan_ptr[s] .. scan_ptr[s+1]), float32, body frame); one scan
 * may serve several problems, at different poses and slots. Problem p with scan_of[p] >= 0 takes that scan into slot
 * slot[p] at pose row pose_base[p] + slot[p]; scan_of[p] == -1 leaves its map alone.
 * balm_batch_window_recut / marginalize / push: win_count[p] (and mg_size[p]) as the balm_window_* call of that name;
 * win_count[p] == 0 (marginalize: mg_size[p] == 0) leaves problem p's map alone, and push gives it an empty voxel range.
 * After any sequence of these calls, problem p's push is bitwise what balm_window_push registers on a context of
 * n_slots[p] poses reset with the same opts and driven by the same calls on its scans, pose rows, slots and counts (a
 * skipped problem = a call not made): keys, layers, row_ptr, pose_idx, obs10, fix clusters, coe, M and K. A problem's
 * result does not depend on the rest of the batch or on its position in it; two identical call sequences are bitwise
 * equal. Push replaces the registration (N_p = n_slots[p], fix clusters always present, keys, layers and the association
 * options carried); n_voxels_out / n_obs_out: [B] or NULL. The window maps are independent of the registration:
 * balm_batch_set_voxels, cut_voxels, marginalize and append_scan do not touch them; balm_batch_destroy frees them.
 * Memory: 120 + 160 * max n_slots bytes per node and 56 bytes per point held, summed over the problems. Host waits per
 * call are a fixed number whatever B (recut: a fixed number per octree layer).
 * BALM_ERR_INVALID leaves both the window maps and the registration unchanged: no balm_batch_window_reset before;
 * n_problems < 1 or n_slots outside 1 .. BALM_BATCH_MAX_POSES; scan_of outside -1 and [0, n_scans); slot outside
 * [0, n_slots[p]); scan_ptr not starting at 0 or not ascending; win_count outside 0 and [1, n_slots[p]]; mg_size outside
 * 0 and [1, win_count[p]); a point outside the +-2^18 root-voxel range (checked on the device before any map changes).
 * BALM_ERR_UNSUPPORTED, before anything is allocated: 2^31 or more points, counted once per problem that takes them (or
 * in xyz, or in the maps). Messages name the lowest offending problem. */
int balm_batch_window_reset(balm_batch *b, int n_problems, const int *n_slots, const balm_assoc_opts *opts);
int balm_batch_window_cut(balm_batch *b, const int32_t *scan_of, const int *slot, int n_scans, const int64_t *scan_ptr,
                          const float *xyz, const double *poses12);
int balm_batch_window_recut(balm_batch *b, const int *win_count);
int balm_batch_window_marginalize(balm_batch *b, const int *mg_size, const double *poses12 /* P x 12 or NULL */,
                                  const int *win_count);
int balm_batch_window_push(balm_batch *b, const int *win_count, int64_t *n_voxels_out, int64_t *n_obs_out);
/* balm_pose_covariance per problem, all problems in one call: problem p's results are those of balm_pose_covariance on
 * a BALM_PREC_FP64 context holding only problem p, at its rows of poses12 (P x 12, read only). c_cov81: K x 81 in
 * registration order (the order of obs10), or NULL for isotropic point noise of standard deviation point_noise.
 * include_fix as balm_pose_covariance. Outputs, each may be NULL: Rcov_raw and Rcov hold the problems' (6N_p)^2
 * column-major blocks one after the other (the layout of balm_batch_evaluate's H); status[B].
 * Rcov_p = H_p^-1 Rcov_raw_p H_p^-1 with H_p evaluated at the poses (fix clusters as include_fix) and factored without
 * damping or pivoting; it is made exactly symmetric by copying its upper triangle to the lower one. status[p] is BALM_OK,
 * or BALM_ERR_NOT_PD when H_p is singular under balm_pose_covariance's criterion (a zero / tiny / non-finite LDL^T pivot,
 * or min |d| <= 1e-11 max |d|): that problem's Rcov block is zero, its Rcov_raw block is still valid. A problem without
 * voxels has a zero Rcov_raw and BALM_ERR_NOT_PD. Registrations from balm_batch_cut_voxels have no fix clusters, so every
 * problem's H is singular (free gauge) and reports BALM_ERR_NOT_PD; their Rcov_raw is valid. balm_batch_marginalize
 * gives them fix clusters that anchor the gauge (include_fix = 1). With Rcov == NULL, H is
 * neither evaluated nor factored and every status is BALM_OK. The call returns BALM_OK when it ran, whatever the
 * statuses; BALM_ERR_INVALID without a registration. A problem's results do not depend on the rest of the batch; two
 * calls are bitwise equal. The host waits once. Device scratch allocated and freed by one call, in doubles:
 *   sum_p 8 M_p ldp_p (rows; ldp_p = 6 N_p rounded up to 64) + 21 K (per-observation diagonal blocks)
 *   + 672 sum_p ceil(M_p / 32) (per-chunk diagonal partials) + 4096 sum_p T_p (T_p + 1) / 2 ceil(8 M_p / 768)
 *   (SYRK partials, T_p = ldp_p / 64) + sum_p (6 N_p)^2 (Rcov_raw), + sum_p (6 N_p)^2 more with Rcov, + 81 K with c_cov81;
 *   plus 16 bytes per SYRK item, 8 bytes per problem and, with Rcov, 4 bytes per problem. */
int balm_batch_pose_covariance(balm_batch *b, const double *poses12, const double *c_cov81, double point_noise,
                               int include_fix, int *status, double *Rcov_raw, double *Rcov);

/* Pose-covariance propagation of the consistency experiment (SURVEY.md section 8f, row N3):
 *   Rcov_raw = sum over observations of  Ls c_cov Ls^T      -- VOX_HESS::left_jacobian_point + BALM2::multi_second
 *                                                              (src/simulation/BAs_left.hpp:342-473, 995-1023)
 *   Rcov     = H^-1 Rcov_raw H^-T                            -- the tail of BALM2::damping_iter (BAs_left.hpp:1089-1096)
 * at the poses given (normally the output of balm_damping_iter). c_cov81: K x 81 doubles, the 9 x 9 covariance of every
 * cluster's parameters (P00,P01,P02,P11,P12,P22,v0,v1,v2) in the order of obs10, i.e. PointCluster::c_cov
 * (src/simulation/toolss.hpp:288,341); NULL derives it from the cluster moments for isotropic point noise of standard
 * deviation point_noise, which is exactly what PointCluster::push accumulates (toolss.hpp:311-343). include_fix: the fix
 * clusters take part in the voxel statistics and in H (BAs_left.hpp:183-185); without them H is singular (gauge) and the
 * call fails with BALM_ERR_NOT_PD when Rcov is requested. Either output (n x n, column-major, symmetric) may be NULL.
 * With the joint cost on (balm_set_joint_cost) H is the joint H of voxels, pose factors and priors, so priors can fix
 * the gauge without fix clusters; Rcov_raw stays the voxels' term (the terms' information matrices are cost weights,
 * not a point-noise model). */
int balm_pose_covariance(balm_ctx *ctx, const double *poses12, const double *c_cov81, double point_noise, int include_fix,
                         double *Rcov_raw, double *Rcov);

/* Pose graph (hierarchical BA's top-down step, DESIGN.md "Pose graph"): window factors over the ctx's N poses, each from
 * one converged BA window. Factor f has the N_f = factor_ptr[f+1] - factor_ptr[f] (2 .. BALM_BATCH_MAX_POSES) distinct
 * global pose indices factor_pose[factor_ptr[f] ..], the window's refined poses T^_k (poses_hat12, 12 doubles per slot in
 * the same order) and its BA Hessian H_f ((6 N_f)^2 doubles, column-major, symmetric, as balm_batch_evaluate returns it;
 * the factors' Hessians concatenated). With c(T, T^) = (Log(R R^^T), p - R R^^T p^) and A = T_idx[0] T^_0^-1:
 *   e_k = c(A^-1 T_idx[k], T^_k),   cost_f = 1/2 sum_{k,l >= 1} e_k^T H_f[k,l] e_l,
 * the second-order model of the window's BA cost with slot 0 pinned; the total is the sum over factors.
 * status_out (n_factors, may be NULL): BALM_OK, or BALM_ERR_NOT_PD when H_f restricted to slots >= 1 is not positive
 * definite (pivot test of balm_batch_pose_covariance, or a non-positive pivot); such a factor is left out of every sum.
 * BALM_ERR_INVALID (nothing registered, the previous factor set kept) for n_factors < 1, factor_ptr[0] != 0, a factor
 * with fewer than 2 or more than BALM_BATCH_MAX_POSES poses, an index outside [0, N) or repeated within a factor, a
 * non-finite T^ / H entry, or an H_f not symmetric to 1e-12 of its max |entry| (the cost reads its symmetric part,
 * the gradient its rows). The factor set is independent of the voxel registration; it is replaced by the next call.
 * With balm_set_joint_cost on, the set (with its balm_set_factor_loss) also joins the context's voxel cost. */
int balm_set_pose_factors(balm_ctx *ctx, int n_factors, const int64_t *factor_ptr, const int32_t *factor_pose,
                          const double *poses_hat12, const double *H, int32_t *status_out);
/* balm_evaluate's analogue for the registered factors: dense H (n x n, column-major, exactly symmetric, 6-dimensional
 * gauge null space), g (n) and the cost at poses12. H and g may be NULL. */
int balm_pose_graph_evaluate(balm_ctx *ctx, const double *poses12, double *H, double *g, double *cost);
/* balm_damping_iter on the pose-graph cost: the same LM rule (u0, v0, q / q1, rel_tol, max_iter, force_hess, verbose),
 * solve, refinement, pose update and gauge_mode, with the factor evaluation in place of the voxel evaluation.
 * min_planes_per_pose and hess_includes_fix have no meaning here and are ignored. BALM_ERR_INVALID with a communicator
 * attached (single GPU only) or without registered factors, and for gauge_mode 0 or 1 while a pose prior is active
 * (balm_set_pose_priors: the priors fix the frame; pass 2). */
int balm_pose_graph_iter(balm_ctx *ctx, double *poses12, const balm_lm_opts *opts, balm_trace *trace, int *n_iters,
                         double *poses_per_iter);

/* Rig calibration (DESIGN.md "Rig calibration"): the ctx's N scan slots driven by n_base base poses T_b and n_lidar
 * extrinsics E_l (body-frame poses of the LiDARs): slot s is scanned at X_s = T_b E_l with b = base_of[s] and
 * l = lidar_of[s] (R = R_T R_E, p = R_T p_E + p_T). The cost is the ctx's voxel cost, voxel loss included, at those X_s.
 * Unknowns are the base poses and extrinsics not fixed by base_fixed / lidar_fixed (nonzero = fixed; NULL: none), free
 * base poses ascending then free extrinsics ascending, 6 each (phi, t), updated by the left rule of balm_damping_iter;
 * *n_rig_out = 6 x the free count. With every extrinsic free the cost has a second gauge (T_b Q, Q^-1 E_l): fix one
 * reference LiDAR, as MLCC does. The rig belongs to the ctx: every voxel registration keeps it, and balm_evaluate,
 * balm_damping_iter, the pose-graph and covariance calls ignore it. n_base == 0 detaches it. Refused, with the previous
 * rig kept: BALM_ERR_UNSUPPORTED on a BALM_PREC_BLOCKS ctx (it takes balm_block_set_rig); BALM_ERR_INVALID with a communicator attached, for a base or
 * LiDAR index out of range, a base or LiDAR no slot uses, or when every unknown is fixed. Device memory: the rig holds
 * K = H J (n_rig x 6N doubles), H_rig and its factor (2 n_rig^2) on top of the ctx's H and factor (2 (6N)^2); a rig with
 * about one free unknown per slot (n_rig ~ 6N) therefore needs about twice the ctx's dense memory, and balm_set_rig
 * returns BALM_ERR_CUDA (out of memory), the previous rig kept, when that does not fit. balm_rig_evaluate and
 * balm_rig_damping_iter are refused (BALM_ERR_INVALID) once a communicator is attached. */
int balm_set_rig(balm_ctx *ctx, int n_base, int n_lidar, const int32_t *base_of, const int32_t *lidar_of,
                 const uint8_t *base_fixed, const uint8_t *lidar_fixed, int *n_rig_out);
/* H_rig (n_rig x n_rig, column-major, exactly symmetric), g_rig (n_rig) and the residual at base12 (n_base x 12) and
 * ext12 (n_lidar x 12); the voxels' H and g without (include_fix 0) or with the fix clusters, as balm_evaluate over all
 * voxels. With H_st, g_s the ctx's H and g at the scan poses and J_s = [I on base b | Ad(T_b) on lidar l]:
 * H_rig = sum J_s^T H_st J_t + the second-order part of the composition contracted with g_s, the exact Hessian in these
 * coordinates; g_rig = sum J_s^T g_s. Fixed order, no atomics: two calls give the same bits. H and g may be NULL.
 * BALM_ERR_INVALID without a rig or registered voxels. */
int balm_rig_evaluate(balm_ctx *ctx, const double *base12, const double *ext12, int include_fix, double *H, double *g,
                      double *residual);
/* Point noise propagated to the rig's unknowns (DESIGN.md "Rig covariance"), at base12 / ext12 (normally the output of
 * balm_rig_damping_iter). With X_s the composed scan poses, R balm_pose_covariance's Rcov_raw at them (c_cov81,
 * point_noise and include_fix as there) and J the rig's first-order Jacobian of balm_rig_evaluate:
 *   raw = J^T R J,   cov = H~^-1 raw~ H~^-T,
 * H balm_rig_evaluate's H_rig at the same state and include_fix, factored without damping. anchor: -1, or the free
 * index of a free base pose (in [0, free bases)), whose 6 rows and columns are deleted from H_rig and raw (as the
 * anchor of balm_block_covariance); its entries are exactly 0 in both outputs. With free base poses and no fix clusters
 * the cost keeps the base poses' left gauge: pass a base anchor; the extrinsic block of cov does not depend on which.
 * LiDAR-to-INS (every base pose fixed) uses -1. Both outputs are n_rig x n_rig, column-major, in balm_set_rig's order;
 * either may be NULL (not both), and without cov no H_rig is evaluated. BALM_ERR_INVALID, nothing written, without a
 * rig, with a communicator attached, without registered voxels, for a NULL state, or for an anchor that is neither -1
 * nor a free base index (an extrinsic cannot be the anchor). BALM_ERR_NOT_PD, nothing written, when H~ is singular
 * (balm_pose_covariance's pivot test over the pivots outside the anchor). The rig's state, the poses and the next
 * balm_rig_damping_iter are unaffected. Device memory on top of the rig's: R ((6N)^2 doubles) and the scratch of
 * balm_pose_covariance's raw term, and raw (n_rig^2); the rig's K, H_rig and factor are reused. */
int balm_rig_covariance(balm_ctx *ctx, const double *base12, const double *ext12, const double *c_cov81,
                        double point_noise, int include_fix, int anchor, double *raw, double *cov);
/* balm_damping_iter's LM on the rig cost: the same opts (u0, v0, rel_tol, max_iter, hess_includes_fix, force_hess,
 * verbose; min_planes_per_pose counts voxels per scan slot), accept rule and refinement, with the solve on H_rig.
 * base12 / ext12 are updated in place. rig_per_iter: max_iter x (n_base + n_lidar) x 12 (base poses, then extrinsics,
 * after every iteration, before the gauge step) or NULL. gauge_mode 0 / 1 re-anchors the base poses to base 0
 * (extrinsics are body-frame and stay); BALM_ERR_INVALID for gauge_mode 0 or 1 while a base pose is fixed (the fixed
 * poses set the frame; pass 2), and without a rig or registered voxels. */
int balm_rig_damping_iter(balm_ctx *ctx, double *base12, double *ext12, const balm_lm_opts *opts, balm_trace *trace,
                          int *n_iters, double *rig_per_iter);

/* Rig calibration on a BALM_PREC_BLOCKS ctx (DESIGN.md "Rig calibration on block-sparse voxel BA"): balm_set_rig's
 * arguments, checks, error codes and lifetime (n_base == 0 detaches; a refused call keeps the previous rig);
 * BALM_ERR_INVALID on any other precision. Nothing of size n_rig x 6N or n_rig^2 is held: H_rig is kept as the 6x6
 * blocks of the rig pairs (u, v), u <= v over the free unknowns, for which some slot of u and some slot of v form a
 * block pair of the ctx (balm_block_structure's pattern, pose factors and priors included), plus every diagonal pair,
 * and solved by the nested-dissection block LDL^T of the ctx. The rig's pattern follows the ctx's: every rig call after
 * a voxel registration, balm_block_set_factors or balm_set_pose_priors rebuilds it (BALM_ERR_UNSUPPORTED from that call
 * when it is too large to index). balm_rig_evaluate (H expanded on the host from the blocks) and balm_rig_damping_iter
 * take such a rig with their usual arguments and meaning; the cost is the ctx's full cost: voxels, then pose factors,
 * then priors, all at the composed scan poses (with an active prior gauge_mode 0 and 1 are BALM_ERR_INVALID, as for
 * balm_damping_iter). balm_rig_covariance is BALM_ERR_UNSUPPORTED for it. */
int balm_block_set_rig(balm_ctx *ctx, int n_base, int n_lidar, const int32_t *base_of, const int32_t *lidar_of,
                       const uint8_t *base_fixed, const uint8_t *lidar_fixed, int *n_rig_out);
/* The block-sparse rig's pattern, as balm_block_structure: stats[0] rig block pairs, stats[1] blocks of its L,
 * stats[2] elimination-tree levels, stats[3] device bytes the rig holds (tables, states, K blocks, blocks, solver);
 * pairs (may be NULL): 2 x stats[0] int32, the (u, v), u <= v, in balm_set_rig's unknown order, ascending.
 * BALM_ERR_INVALID without a balm_block_set_rig rig or registered voxels. */
int balm_rig_block_structure(balm_ctx *ctx, int64_t stats[4], int32_t *pairs);
/* Sigma = H~_rig^-1 on the rig's block pattern (balm_rig_block_structure's order, [pairs][36] column-major, rows of u),
 * H~_rig balm_rig_evaluate's H_rig at base12 / ext12 and include_fix without the anchor's rows and columns: the
 * Laplace form balm_block_covariance gives for scan poses. anchor: -1 or the free index of a free base pose (as
 * balm_rig_covariance); its blocks are 0. H_rig holds the composition's second-order term, so away from the optimum it
 * can be indefinite: pass balm_rig_damping_iter's result. BALM_ERR_NOT_PD when H~_rig is singular or indefinite
 * (balm_block_covariance's test),
 * BALM_ERR_INVALID without a balm_block_set_rig rig or registered voxels, for a NULL argument or a bad anchor. The next
 * balm_rig_damping_iter is unaffected. */
int balm_rig_block_covariance(balm_ctx *ctx, const double *base12, const double *ext12, int include_fix, int anchor,
                              double *cov);
/* balm_rig_covariance's point-noise covariance on a balm_block_set_rig rig (DESIGN.md "Point-noise covariance on blocks
 * contexts"), restricted to the n_sel distinct free unknowns sel (free indices in balm_set_rig's order, in [0, n_rig / 6)):
 *   Sigma_sel = W^T R W,   W = J Y,   Y = H~_rig^-1 E,
 * E the unit columns of the selection, H~_rig balm_rig_block_covariance's undamped H_rig without the anchor's rows and
 * columns, J the rig's first-order Jacobian and R balm_block_point_covariance's raw term at the composed scan poses
 * (c_cov81, point_noise and include_fix as in balm_pose_covariance). This is balm_rig_covariance's cov restricted to the
 * selection; nothing of size n_rig^2 or (6N)^2 is formed. cov: (6 n_sel)^2 doubles, column-major, exactly symmetric, in
 * sel's order, or NULL; marg: n_sel x 36 doubles (unknown u's 6x6 block, column-major), bitwise the diagonal blocks of
 * cov, or NULL (not both). anchor: as balm_rig_block_covariance; its entries are exactly 0. BALM_ERR_INVALID, nothing
 * written, on any other kind of ctx, without a balm_block_set_rig rig or registered voxels, with a communicator attached,
 * for a NULL state, a bad anchor, n_sel < 1 or a sel entry repeated or out of range. BALM_ERR_NOT_PD, nothing written,
 * under balm_block_covariance's pivot test. BALM_ERR_UNSUPPORTED, nothing written, when cov's buffers exceed the budget
 * below. The rig, the ctx and the next balm_rig_damping_iter are as without the call. Device memory, freed by the call,
 * in doubles: balm_block_point_covariance's raw-term scratch, and with F free unknowns, C right-hand sides per chunk
 * (6 n_sel for cov; marg alone: as many whole unknowns as fit) and S = ceil(6N / 384):
 *   C (6F + 12N) (Y, W, Z) + 36 S pairs (partial sums; pairs = n_sel (n_sel + 1) / 2 with cov, else C / 6)
 *   + 36 n_sel^2 with cov, else 36 n_sel (outputs), plus 4 (F + n_sel) bytes.
 * BALM_COV_BUDGET_MB (default 4096) bounds the first two terms and the outputs. */
int balm_rig_block_point_covariance(balm_ctx *ctx, const double *base12, const double *ext12, const double *c_cov81,
                                    double point_noise, int include_fix, int anchor, int n_sel, const int32_t *sel,
                                    double *cov, double *marg);

/* Sparse pose graph (DESIGN.md "Pose graph", "Sparse solve"): the same factors, cost and LM as balm_set_pose_factors /
 * balm_pose_graph_iter, with H held as its nonzero 6x6 blocks and the damped system solved by a block LDL^T in a
 * nested-dissection order. Device memory grows with the number of blocks, not with (6P)^2, so trajectories of any
 * length fit; the context's dense pose graph is the faster choice for short ones. A balm_spg is a handle of its own
 * (it takes no balm_ctx call) that owns a BALM_PREC_BLOCKS context without voxels, whose block pattern holds the factor
 * pairs and the diagonal pairs of the prior poses only; each balm_spg_* call runs that context's code after its own
 * checks (balm_block_set_factors, balm_block_structure, balm_evaluate, balm_damping_iter, balm_block_covariance, ...).
 * balm_spg_create: n_poses >= 1 poses on `device`; allocates O(n_poses) device memory only. */
typedef struct balm_spg balm_spg;
int balm_spg_create(balm_spg **out, int n_poses, int device);
void balm_spg_destroy(balm_spg *spg);
/* balm_set_pose_factors' arguments, checks, messages, NOT_PD status and rejection rule (a rejected call keeps the
 * previous set). A registration also orders the poses, builds the symbolic factorisation and captures the per-solve
 * launches in a CUDA graph; BALM_ERR_UNSUPPORTED (previous set kept) when the pattern is too large to index. */
int balm_spg_set_factors(balm_spg *spg, int n_factors, const int64_t *factor_ptr, const int32_t *factor_pose,
                         const double *poses_hat12, const double *H, int32_t *status_out);
/* stats: [0] nonzero block pairs (i <= j) of H, [1] blocks of L, [2] elimination-tree levels, [3] device bytes the
 * handle holds (factors and their staging, tables, L, vectors), as balm_block_structure counts them.
 * pairs (may be NULL, so that a first call can size it): 2 int32 (i, j) per block pair, ascending in (i, j). */
int balm_spg_structure(balm_spg *spg, int64_t stats[4], int32_t *pairs);
/* balm_pose_graph_evaluate with H as blocks: 36 doubles per block pair (rows of pose i, columns of pose j,
 * column-major) in balm_spg_structure's order, bitwise the context's dense entries. blocks and g may be NULL. */
int balm_spg_evaluate(balm_spg *spg, const double *poses12, double *blocks, double *g, double *cost);
/* balm_pose_graph_iter's contract (LM rule, force_hess, rel_tol, gauge_mode, trace records, refinement and not_pd
 * rules, gauge_mode 0 / 1 refused while a pose prior is active) on the sparse solve. */
int balm_spg_iter(balm_spg *spg, double *poses12, const balm_lm_opts *opts, balm_trace *trace, int *n_iters,
                  double *poses_per_iter);
/* Marginal pose covariances (DESIGN.md "Marginal covariances"): H evaluated undamped at poses12, the 6 rows and columns
 * of pose `anchor` deleted when anchor >= 0 (H~), and Sigma = H~^-1 restricted to H's block pattern: 36 doubles per
 * block pair (rows of pose i, columns of pose j, column-major) in balm_spg_structure's order, written to cov. Blocks
 * touching the anchor are 0; diagonal blocks are exactly symmetric. Coordinates are those of the LM pose update,
 * delta = (dtheta, dp) with T <- (Exp(dtheta) R, Exp(dtheta) p + dp); the factors' H are information matrices, so Sigma
 * is the Laplace covariance of the estimate. H has the 6-dimensional gauge null space of a common left transform:
 * anchor = 0 is the normal call. anchor in [-1, N).
 * BALM_ERR_NOT_PD (cov not written) when H~ is singular: a bad pivot, or over every column but the anchor's the smallest
 * LDL^T pivot is not > 1e-11 x the largest (e.g. two unconnected components, a pose in no factor, anchor = -1).
 * BALM_ERR_INVALID for a null argument, no registered factors or an anchor out of range; BALM_ERR_UNSUPPORTED, with
 * nothing changed, when the selected-inversion tables are too large to index.
 * The first call after a registration builds those tables (device bytes grow by 288 per block of L, 4 per term with
 * Sigma_j |struct(j)|^2 terms, 4 per pair and 8 per pose; balm_spg_structure's stats[3] counts them); later calls reuse
 * them until the next
 * registration. Afterwards the handle's blocks, g and factor storage hold this call's evaluation (H at poses12, undamped);
 * the next balm_spg_iter re-evaluates and refactors, so its results are bitwise those without the covariance call.
 * The call waits for the device twice (the pivot test and the copy-out), the first one also while it builds the
 * tables. */
int balm_spg_covariance(balm_spg *spg, const double *poses12, int anchor, double *cov);
/* balm_set_factor_loss and balm_factor_residuals on the handle's factor set: same losses, meaning (balm_spg_evaluate,
 * balm_spg_iter and balm_spg_covariance use the robust cost, gradient and reweighted H), checks and lifetime
 * (balm_spg_set_factors resets the loss); balm_spg_structure's stats[3] counts the 28 bytes per factor. */
int balm_spg_set_factor_loss(balm_spg *spg, int n_factors, const int32_t *kind, const double *scale);
int balm_spg_factor_residuals(balm_spg *spg, const double *poses12, double *s, double *w);

/* Block-sparse Hessian of a BALM_PREC_BLOCKS context (BALM_ERR_INVALID on any other, or before a registration).
 * stats: [0] block pairs (i <= j) of H, [1] blocks of the factor L, [2] elimination-tree levels, [3] device bytes the
 * context holds. pairs (may be NULL, so that a first call can size it): 2 int32 (i, j) per block pair, ascending. */
int balm_block_structure(balm_ctx *ctx, int64_t stats[4], int32_t *pairs);
/* The last evaluation's blocks, bitwise what the solve consumed: 36 doubles per pair (rows of pose i, columns of pose
 * j, column-major) in balm_block_structure's order. */
int balm_download_blocks(balm_ctx *ctx, double *blocks);
/* balm_spg_covariance's Sigma on a BALM_PREC_BLOCKS context: H~^-1 on H's block pattern, in balm_block_structure's order,
 * with H as balm_evaluate returns it at poses12 over every voxel (include_fix as in balm_pose_covariance). This is the
 * inverse of the library's Hessian, not balm_pose_covariance's propagated point noise: scaling it by a point-noise model
 * is the caller's job. A registration whose fix clusters anchor the gauge can use anchor = -1 with include_fix = 1;
 * without them anchor = -1 is BALM_ERR_NOT_PD. BALM_ERR_INVALID also on any other kind of context or before a
 * registration. Tables, errors and side effects as balm_spg_covariance's: afterwards balm_download_blocks returns H at
 * poses12, and the next balm_damping_iter is bitwise what it would have been without this call. */
int balm_block_covariance(balm_ctx *ctx, const double *poses12, int include_fix, int anchor, double *cov);
/* Point noise propagated to selected poses of a BALM_PREC_BLOCKS context (DESIGN.md "Point-noise covariance on blocks
 * contexts"): balm_pose_covariance's Rcov restricted to the n_sel distinct poses sel (in [0, N)), without any 6N x 6N
 * matrix:
 *   Sigma_sel = Y^T R Y,   Y = H~^-1 E,
 * E the unit columns of the selection, H~ balm_block_covariance's undamped H at poses12 (include_fix as there) with the
 * anchor's rows and columns replaced by I, and R balm_pose_covariance's Rcov_raw (c_cov81, point_noise, include_fix as
 * there). R couples exactly the poses that share a voxel, so it lives on the block pattern: raw_blocks (NULL or
 * 36 doubles per pair in balm_block_structure's order, rows of pose i, column-major) receives it; pairs that only a pose
 * factor or a prior gives are 0. Pose factors and priors shape H only: their information matrices are cost weights, not a
 * noise model, so they add nothing to R. cov: (6 n_sel)^2 doubles, column-major, exactly symmetric, in sel's order;
 * marg: n_sel x 36 doubles (pose sel[u]'s block, column-major), bitwise the diagonal blocks of cov. anchor: -1 or a
 * pose, as balm_block_covariance; its entries are exactly 0. Any of the three outputs may be NULL, not all; with cov and
 * marg NULL nothing is factored and sel is not read. With cov NULL the marginals go in chunks that fit the budget, so
 * every pose of a long drive can be asked for in one call. Errors, each writing nothing: BALM_ERR_INVALID on any other
 * kind of ctx, before a registration or without voxels, with a communicator attached, for a NULL poses12, a bad anchor,
 * n_sel < 1 or a sel entry repeated or out of range (when cov or marg is asked for); BALM_ERR_NOT_PD under
 * balm_block_covariance's pivot test; BALM_ERR_UNSUPPORTED when cov's buffers exceed the budget. The ctx and the next
 * balm_damping_iter are as without the call (balm_download_blocks then returns H at poses12, as after
 * balm_block_covariance). Device memory, freed by the call, in doubles: the raw term's 36 pairs + 21 K + 21 N + 10 M
 * + 48 x (observations of its largest voxel batch; batches are cut to fit the budget) + 81 K with c_cov81, and for Sigma
 * balm_rig_block_point_covariance's terms with F = N. BALM_COV_BUDGET_MB (default 4096) bounds the batches and Sigma's
 * buffers. */
int balm_block_point_covariance(balm_ctx *ctx, const double *poses12, const double *c_cov81, double point_noise,
                                int include_fix, int anchor, int n_sel, const int32_t *sel, double *raw_blocks,
                                double *cov, double *marg);
/* Pose factors in the cost of a BALM_PREC_BLOCKS context (DESIGN.md "Voxels and pose factors in one cost"): odometry
 * between consecutive scans, loop closures, HBA window factors. Arguments, checks, error messages, per-factor status
 * (BALM_ERR_NOT_PD factors are left out of the pattern and every sum) and factor cost are balm_set_pose_factors'; H_f must
 * be in the voxel cost's units (coe x lambda: points x m^2, as balm_batch_evaluate's H is). n_factors == 0 (the arrays may
 * be NULL) detaches the factor set. Once attached, the context's cost is the voxel cost plus the sum of the active
 * factors' costs in every evaluation over the whole voxel range (head == 0, end == M, also M == 0): balm_evaluate's H, g
 * and residual, balm_residual, balm_damping_iter, balm_solve, balm_download_blocks and balm_block_covariance. A
 * sub-range evaluation stays voxels only, bitwise what it is without factors. min_planes_per_pose still counts voxels:
 * pass 0 when factors carry scans that see no plane. balm_block_structure reports the union pattern (voxel pairs, the
 * active factors' pairs, every diagonal pair) and counts the factor set's bytes; balm_timings.ms_assemble is the factor
 * linearisation, assembly and cost time (0 without factors).
 * The set is independent of the voxel registration: it may be set before one and survives every registration route.
 * Factor indices are pose slots, so after a window shift re-setting them is the caller's job.
 * BALM_ERR_INVALID on any other kind of context, with nothing changed; a rejected call (invalid arguments, or
 * BALM_ERR_UNSUPPORTED when the union pattern is too large to index) keeps the previous set and pattern. */
int balm_block_set_factors(balm_ctx *ctx, int n_factors, const int64_t *factor_ptr, const int32_t *factor_pose,
                           const double *poses_hat12, const double *H, int32_t *status_out);
/* Robust pose factors (DESIGN.md "Robust pose factors"): a loss kind[f] (balm_loss) and scale[f] for every factor of
 * the context's registered set (balm_set_pose_factors' on FP64 / TENSOR contexts, balm_block_set_factors' on a
 * BALM_PREC_BLOCKS context). With s_f = e~^T H~ e~ (twice the quadratic cost_f) and w_f = rho'(s_f), factor f then
 * contributes cost 1/2 rho(s_f), gradient w_f b_f (the exact gradient of that cost) and Hessian w_f M_f, the iteratively
 * reweighted Gauss-Newton term without the second-order rho'' part, in every call that evaluates the factors:
 * balm_pose_graph_evaluate / _iter, and on a blocks context balm_evaluate, balm_residual, balm_damping_iter,
 * balm_solve, balm_download_blocks and balm_block_covariance (whose Sigma is then the inverse of the reweighted H at
 * poses12). A trivial factor's terms are bitwise those without a loss, also next to robust ones. scale is in units of
 * sqrt(s): for factors in the voxel cost's units (2 sigma_p^2 x information, see odometry_factors) and a chi-square
 * gate at probability p, c^2 = 2 sigma_p^2 chi2_6(p). kind == NULL resets every factor to trivial (scale unused).
 * BALM_ERR_INVALID, the previous loss kept, for a null ctx, no registered factor set (a blocks context with none
 * attached), n_factors not the registered count, a kind outside BALM_LOSS_*, or a non-trivial kind whose scale is not
 * finite and > 0 (a trivial factor's scale is ignored; scale may be NULL when every kind is trivial). The loss belongs to
 * the factor set: registering or detaching a set resets it to trivial; voxel registrations keep it. It changes no
 * pattern, so nothing is refactored symbolically or re-captured. While a kind is non-trivial the set holds 28 more
 * device bytes per factor (kind, scale, s_f, w_f), counted in balm_block_structure's stats[3]. */
int balm_set_factor_loss(balm_ctx *ctx, int n_factors, const int32_t *kind, const double *scale);
/* s_f and w_f = rho'(s_f) of every factor of the registered set at poses12, into s and w (n_factors each; either may
 * be NULL). Factors left out as BALM_ERR_NOT_PD report s = w = 0; without a loss w = 1 for the others, which serves
 * chi-square gating of candidate closures. Enqueues the cost pass only and waits once. BALM_ERR_INVALID for a null ctx
 * or poses12, or no registered factor set. */
int balm_factor_residuals(balm_ctx *ctx, const double *poses12, double *s, double *w);

/* Absolute pose priors (DESIGN.md "Absolute pose priors"): GNSS positions, surveyed control points, full-pose anchors.
 * Prior q names a pose slot pose[q] and holds a measured pose T^ = (R^, p^) (poses_hat12, 12 doubles each), a body-frame
 * lever arm l (lever3, 3 doubles each; NULL: all 0), a 6 x 6 symmetric positive semi-definite H_q (H36, 36 doubles each,
 * column-major, (rotation, translation) order, in the units of the cost it joins) and a loss kind[q] / scale[q] as
 * balm_set_factor_loss's (kind NULL: all trivial). With T = (R, p) of the pose:
 *   e = (Log(R R^^T), R l + p - p^),   s_q = e^T H_q e,   cost_q = 1/2 rho(s_q),
 * gradient w J^T H_q e and Hessian w J^T H_q J with w = rho'(s_q), J = [[Jl^-1(e_rot), 0], [-hat(R l + p), I]] under the
 * library's left update. A position-only (GNSS) prior is H_q = blockdiag(0, Omega_p), its R^ unused; a full-pose
 * anchor is any positive definite H_q with l = 0. The priors join the pose-graph cost (balm_pose_graph_evaluate /
 * _iter) on FP64 / TENSOR contexts, and the voxel cost there while balm_set_joint_cost is on; on a BALM_PREC_BLOCKS
 * context they join every evaluation over the whole voxel range, as
 * balm_block_set_factors' factors do (balm_evaluate, balm_residual, balm_damping_iter, balm_solve, balm_download_blocks,
 * balm_block_covariance); every sum adds voxels, then factors, then priors. A prior touches only its pose's diagonal
 * block, so a blocks context's pattern does not change.
 * n_priors == 0 (the arrays may be NULL) detaches the set; several priors may name the same pose. The set belongs to the
 * context, independent of the factor set, its loss and the voxel registration; it survives all of them. The pose
 * graph calls still need a registered factor set.
 * status_out (n_priors, may be NULL): BALM_OK, or BALM_ERR_NOT_PD when H_q has an eigenvalue below -1e-12 lambda_max or
 * is zero; such a prior is left out of every sum. BALM_ERR_INVALID, the previous set kept, for a pose outside [0, N), a
 * non-finite T^, l, H or scale, an H not symmetric to 1e-12 of its max |entry|, a kind outside BALM_LOSS_*, or a
 * non-trivial kind without a finite scale > 0.
 * Gauge: with an active prior the cost has no gauge null space, so balm_damping_iter (blocks, or joint cost),
 * balm_rig_damping_iter (joint cost or blocks), balm_pose_graph_iter and balm_spg_iter refuse gauge_mode 0 and 1
 * (BALM_ERR_INVALID: pass 2), and anchor = -1 is the natural covariance call.
 * balm_block_structure's / balm_spg_structure's stats[3] count the set's device bytes. */
int balm_set_pose_priors(balm_ctx *ctx, int n_priors, const int32_t *pose, const double *poses_hat12,
                         const double *lever3, const double *H36, const int32_t *kind, const double *scale,
                         int32_t *status_out);
/* s_q and w_q = rho'(s_q) of every prior at poses12 into s and w (n_priors each; either may be NULL); NOT_PD priors
 * report 0, 0. Waits once. BALM_ERR_INVALID without a registered prior set. */
int balm_prior_residuals(balm_ctx *ctx, const double *poses12, double *s, double *w);
/* Voxels, pose factors and priors in one cost on an FP64 / TENSOR context (DESIGN.md "Voxels, factors and priors in one
 * cost on dense contexts"). on != 0: the registered factor set (balm_set_pose_factors, with its balm_set_factor_loss) and
 * prior set (balm_set_pose_priors) join every evaluation over the whole voxel range (head == 0, end == M), summed as
 * voxels, then factors, then priors, as on a BALM_PREC_BLOCKS context: balm_evaluate, balm_residual,
 * balm_damping_iter, balm_solve (on the last evaluation), balm_rig_evaluate, balm_rig_damping_iter and
 * balm_rig_covariance (the terms act at the composed scan poses, before the rig reduction) and balm_pose_covariance
 * (the terms shape H only; Rcov_raw stays voxels only). A sub-range evaluation stays voxels only, bitwise;
 * balm_voxel_residuals and the pose-graph calls are unchanged. With an active prior balm_damping_iter and
 * balm_rig_damping_iter refuse gauge_mode 0 and 1. min_planes_per_pose still counts voxels: pass 0 when factors carry
 * scans that see no plane. The tensor path keeps its once-per-step observation read (the trial pass's digit planes,
 * sweep reuse after a rejected step, the stats hand-over): the terms read no observation. on == 0 (the default)
 * restores the voxel cost, bitwise. The switch belongs to the context: it survives every voxel registration and every
 * replacement or detachment of the factor and prior sets. The first call with on != 0 allocates 6N + 1 doubles.
 * BALM_ERR_INVALID, nothing changed, for a null ctx, a BALM_PREC_BLOCKS context (whose voxel cost always holds its
 * terms) or a communicator attached; balm_comm_init with world > 1 is refused while the switch is on. */
int balm_set_joint_cost(balm_ctx *ctx, int on);
/* balm_set_pose_priors and balm_prior_residuals on a sparse pose graph: same arguments, checks, meaning (balm_spg_evaluate,
 * _iter and _covariance) and lifetime (the set survives balm_spg_set_factors). A prior on a pose that no active factor
 * covers adds that pose's diagonal pair to the pattern, which is then re-ordered and re-captured; only a change of the
 * pattern's pairs does that. */
int balm_spg_set_pose_priors(balm_spg *spg, int n_priors, const int32_t *pose, const double *poses_hat12,
                             const double *lever3, const double *H36, const int32_t *kind, const double *scale,
                             int32_t *status_out);
int balm_spg_prior_residuals(balm_spg *spg, const double *poses12, double *s, double *w);

/* Multi-GPU: voxels are sharded across ranks by the caller (each rank registers its own shard); the library
 * all-reduces [H | g | r] with NCCL after every evaluation and the scalar after every residual pass.
 * unique_id: 128 bytes from balm_comm_unique_id() on rank 0, broadcast by the caller (torch.distributed, MPI). */
int balm_comm_unique_id(void *out128);
int balm_comm_init(balm_ctx *ctx, int rank, int world, const void *unique_id128);

/* Instrumentation */
int balm_get_timings(balm_ctx *ctx, balm_timings *out);
/* Tensor path, since balm_reset_counters(): re-evaluations after a rejected step (force_hess) that ran no observation
 * sweep, because the digit planes and accumulators of the same poses and column scales were still in place. They are
 * also counted in balm_timings.single_sweeps. */
int balm_get_reused_sweeps(balm_ctx *ctx, int *out);
int balm_reset_counters(balm_ctx *ctx);
int balm_sync(balm_ctx *ctx);
/* CUDA-event bracket on the ctx stream: begin records, end records + synchronises and returns elapsed ms. */
int balm_timer_begin(balm_ctx *ctx);
int balm_timer_end(balm_ctx *ctx, float *ms);
/* Debug aid: with BALM_DAG_TRACE=1 in the environment, device timestamps (ns) of the last factorisation: 4 per 64-column
 * step of the chain, then 3 per CTA (start, end, tasks executed). */
int balm_debug_dag_trace(balm_ctx *ctx, unsigned long long *out, int max_entries);
/* Debug aid: the dense damped solve of balm_solve(u) -- tile-DAG LDL^T, backward substitution, q1, the backward-error
 * check, fp64 refinement, the not_pd rule and the timings counters -- on a caller-supplied system, so that it can be
 * compared bit for bit with an exact reference. H is n x n column-major and symmetric and g has length n, n = 6N of
 * ctx; both are copied to scratch buffers, which (with the factor workspaces) the call allocates and frees. It neither
 * needs nor touches a registration, an evaluation or the context's H, g and factors. dx, q1 and not_pd mean what they
 * mean in balm_solve. LD (may be NULL) receives the n x n column-major factor: L strictly below the diagonal, d on it,
 * zeros above. omega (may be NULL) receives the componentwise backward error of the final check. BALM_ERR_INVALID on a
 * BALM_PREC_BLOCKS context or for a NULL H or g. */
int balm_debug_ldlt(balm_ctx *ctx, const double *H, const double *g, double u, double *dx, double *q1, int *not_pd,
                    double *LD, double *omega);
/* Debug aid: with BALM_TC_TRACE=1 in the environment when a tensor-precision ctx is created, the last tensor SYRK launch
 * (of an evaluation or of balm_debug_syrk_tc) records clock64 sums per role, 18 words per CTA, CTA b at 18 b (CTAs
 * beyond the launch's grid hold zeros):
 *   0 stages (64-row contraction steps) the CTA consumed, in 128 x 64 half-tile units (a stage of a whole 128 x 128
 *   tile counts 2); 1, 2 %globaltimer (ns) at the start and the end of consumer warp 0, whose total below spans the same
 *   interval;
 *   3..7 consumer warp 0 and 8..12 consumer warp 4 (one per warpgroup): waiting on the stage full, in the warpgroup's
 *   vote that it arrived, in wgmma.wait_group, epilogue, total;
 *   13..15 zero (there is no transposer warp any more);
 *   16 producer: waiting on a free slot; 17 producer: waiting on the readiness flags of the stage's copy units.
 * Copies min(max_entries, 18 x SM count) words; BALM_ERR_INVALID when the ctx records no trace. Without the variable
 * the SYRK runs an instantiation that reads no clock. BALM_TC_TILE=half|full at ctx creation forces the SYRK's item
 * shape (default: whole tiles at S <= 3 when tiles x k-splits >= the SM count). */
int balm_debug_tc_trace(balm_ctx *ctx, unsigned long long *out, int max_entries);
/* Debug aid: the same launch's copier warps (which copy the digit planes K-major, one 64-row x 128-column tile of one
 * plane at a time), 3 words per CTA, CTA b at 3 b: 0 clock64 sum over its copier warps of the time spent on their copy
 * units; 1 of that, the time waiting on their loads; 2 plane tiles copied (summed over CTAs: digit planes x
 * ceil(rows / 64) x ldg / 128). Copies min(max_entries, 3 x SM count) words; BALM_ERR_INVALID as balm_debug_tc_trace. */
int balm_debug_tc_copy_trace(balm_ctx *ctx, unsigned long long *out, int max_entries);
/* Debug aid: the tensor path's SYRK kernel alone, on caller-supplied digit planes, so that its fp64 partial tiles can be
 * compared bit for bit with an exact integer reference. Uses ctx's device, stream and column count ldg = 6N rounded up
 * to 128 (tiles = T (T + 1) / 2 upper-triangle tiles of 128 x 128, T = ldg / 128); neither needs nor touches a
 * registration or an evaluation. planes: S (2..4) int8 planes of rows x ldg, plane 0 the most significant digit, column
 * index fastest; rows are padded to a multiple of 64 with zeros. isc: ldg column factors. part (in/out):
 * splits x tiles x 128 x 128 doubles, tile t of split sp at (sp * tiles + t) * 16384, row-major; accumulate = 0
 * overwrites it, 1 adds to it. The rows go to `splits` k-split items of per = ceil(padded rows / splits) rounded up to
 * 64 rows each; BALM_ERR_INVALID before any launch for S outside 2..4, rows outside 1..2^30, splits < 1 or per > 32704
 * (the int32 exactness bound: 4 * 32704 * 2^14 < 2^31). A pipeline timeout is BALM_ERR_CUDA. Device scratch is
 * allocated and freed by the call. */
int balm_debug_syrk_tc(balm_ctx *ctx, const int8_t *planes, int S, int64_t rows, const double *isc, int splits,
                       int accumulate, double *part);
/* Debug aid: after a tensor-path evaluation, what the SYRK consumed in its last voxel batch: the S digit planes (their
 * first rows_padded rows, S x rows_padded x ldg int8, layout as above), the ldg column factors isc, S and the context's
 * k-split count. NULL arrays are not written, so a first call sizes the buffers. BALM_ERR_INVALID on an fp64 context or
 * before any evaluation of the registered voxels. */
int balm_debug_tc_planes(balm_ctx *ctx, int8_t *planes, double *isc, int *S, int64_t *rows_padded, int *splits);
/* Device pointers of the last evaluation's H (n*n col-major), g (n) -- for zero-copy consumers. */
int balm_device_views(balm_ctx *ctx, double **H_dev, double **g_dev);

/* Synthetic scene of the benchmark_virtual shape generated directly in HBM
 * (benchmark_virtual.cpp:547-606 scene, :491-503 pose noise, :391 coe): every pose sees every plane,
 * pts_size points per observation. Outputs are device buffers owned by the ctx and registered as its voxels;
 * poses_gt / poses_init (N*12 host doubles) receive ground truth and perturbed start. first_voxel offsets the
 * plane ids so ranks generate disjoint shards of one global scene. */
int balm_synth_virtual(balm_ctx *ctx, int64_t n_voxels, int64_t first_voxel, int pts_size, double point_noise,
                       double surf_range, uint64_t seed, double *poses_gt, double *poses_init);
/* Copies the registered voxels back to host arrays (K*10, K, M+1, M) -- lets tests/bench feed the oracle and
 * the host-buffer (e2e) path with the very scene generated above. Any pointer may be NULL. */
int balm_download_voxels(balm_ctx *ctx, int64_t *row_ptr, int32_t *pose_idx, double *obs10, double *coe);
/* Same for the voxels [head, end) only (row_ptr re-based to 0: end-head+1 entries); n_obs_out receives the number of
 * observations in the range, so a first call with NULL arrays sizes the buffers. Lets a parity test compare
 * balm_evaluate(head, end) of a full-size problem (BASELINE C3: 4 GB of observations) with the CPU oracle on exactly
 * the same voxels. */
int balm_download_voxel_range(balm_ctx *ctx, int64_t head, int64_t end, int64_t *row_ptr, int32_t *pose_idx,
                              double *obs10, double *coe, int64_t *n_obs_out);
int64_t balm_num_obs(balm_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif

// internal.cuh -- shared declarations of libbalm_b200 (not part of the ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <algorithm>
#include <cmath>
#include <functional>
#include <string>
#include <vector>
#include "../../include/balm_b200.h"

#define BALM_SCAL_RCUR 16
#define BALM_SCAL_RTRIAL 17
#define BALM_STATS_STRIDE 40  // doubles per voxel in the stats table: [0..19] eigen data (vb, u0..u2, 1/NN, the three
                              // sqrt(coe|w_k|), coe, lambda), [20..39] the observation sweep's record (see obs_pass_kernel)
#define BALM_SWEEP_OFF 20
#define BALM_SWEEP_WORDS 20
#define BALM_ACC 33           // per-pose accumulators of the observation pass: g(6) + sym 6x6 diag block (21)
                              // + exact fp64 sums of squares of the 6 G' columns (diagonal of G'^T G')
#define BALM_NB 64            // LDL^T panel width
constexpr double SOLVE_OMEGA_TOL = 1e-12;  // componentwise backward error of a damped solve accepted without refinement
#define BALM_SYRK_TILE 128
// int32 exactness bound of the tensor SYRK: contraction rows of one (tile, k-split) item, a multiple of 64.
// A digit-pair sum T_d adds at most 4 * rows products of magnitude <= 2^14: 4 * 32704 * 2^14 < 2^31.
#define BALM_TC_MAX_ROWS_PER_ITEM 32704
// BALM_TC_TRACE: words per CTA of the tensor SYRK's per-role clock trace (layout: balm_debug_tc_trace)
#define BALM_TC_TRACE_WORDS 18
// ... and words per CTA of its copier warps' trace, stored after every CTA's role words (balm_debug_tc_copy_trace)
#define BALM_TC_COPY_TRACE_WORDS 3

void balm_set_error(const std::string &s);
struct WindowState;  // the persistent sliding-window octree (assoc.cu)
void window_free(WindowState *w);
struct PoseGraph;    // the registered window factors (pose_graph.cu)
void pose_graph_free(PoseGraph *p);
struct BlockHessian;  // the block pattern of a BALM_PREC_BLOCKS context (blocks.cu)
void block_hessian_free(BlockHessian *b);
struct PriorSet;      // the registered absolute pose priors (pose_graph.cu)
void prior_set_free(PriorSet *p);
struct Rig;           // balm_set_rig's slot assignment, unknowns and reduced system (rig.cu)
void rig_free(Rig *r);
struct SparseSolver;  // nested-dissection ordering, symbolic factorisation and the per-solve CUDA graph

#define CUDA_TRY(expr)                                                                        \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      char _b[512];                                                                           \
      snprintf(_b, sizeof(_b), "%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      balm_set_error(_b);                                                                     \
      return BALM_ERR_CUDA;                                                                   \
    }                                                                                         \
  } while (0)

// ---------------- host helpers ----------------
// returns the status of x from the calling function unless it is BALM_OK
#define TRY(x)                      \
  do {                              \
    const int _s = (x);             \
    if (_s != BALM_OK) return _s;   \
  } while (0)

template <typename T>
int dev_alloc(T **p, size_t count) {  // count elements of T (at least one, so that the pointer is never null)
  CUDA_TRY(cudaMalloc((void **)p, sizeof(T) * (count ? count : 1)));
  return BALM_OK;
}

// Device scratch of one call: every buffer taken from the pool is freed on ANY exit path (the early returns of TRY /
// CUDA_TRY, a rejected registration, a bad frame index ...), so a failed call leaks nothing. drop frees one early.
// bytes / peak count the bytes requested from the pool and from every pool nested in it (constructed with it as up), so
// the outermost pool of a call sees the call's whole scratch.
struct ScratchPool {
  std::vector<std::pair<void *, size_t>> ptrs;
  ScratchPool *up = nullptr;
  size_t bytes = 0, peak = 0;
  ScratchPool() = default;
  explicit ScratchPool(ScratchPool *outer) : up(outer) {}
  ScratchPool(const ScratchPool &) = delete;
  ScratchPool &operator=(const ScratchPool &) = delete;
  ~ScratchPool() {
    for (auto &q : ptrs) { cudaFree(q.first); count(-(long long)q.second); }
  }
  template <typename T>
  int get(T **p, size_t n) {
    TRY(dev_alloc(p, n));
    const size_t b = sizeof(T) * (n ? n : 1);
    ptrs.push_back({(void *)*p, b});
    count((long long)b);
    return BALM_OK;
  }
  void drop(void *q) {
    release(q);
    cudaFree(q);
  }
  void release(void *q) {  // the caller keeps q: it is no longer freed on exit
    if (!q) return;
    for (size_t i = 0; i < ptrs.size(); i++)
      if (ptrs[i].first == q) {
        count(-(long long)ptrs[i].second);
        ptrs[i] = ptrs.back();
        ptrs.pop_back();
        break;
      }
  }
  void count(long long d) {
    for (ScratchPool *s = this; s; s = s->up) {
      s->bytes = (size_t)((long long)s->bytes + d);
      s->peak = std::max(s->peak, s->bytes);
    }
  }
};

// The workspaces of the dense LDL^T solve of one system of order n (ldlt.cu allocates them on the system's first solve).
struct LdltWork {
  double *Xinv = nullptr;                   // [panels][64*64] inverses of the unit-lower diagonal blocks
  double *dinv = nullptr;                   // [n] 1/d
  double *dval = nullptr;                   // [n] d (the tile-DAG factorisation scales its operands with it)
  double *sol = nullptr;                    // [n] right-hand side / forward-substitution vector
  double *ysol = nullptr;                   // [n] forward-substitution result y (kept apart from the running rhs `sol`)
  double *rres = nullptr;                   // [n] residual b - A x of the last solve (backward-error check)
  double *rdelta = nullptr;                 // [n] refinement correction
  int *dag_flags = nullptr;                 // tile-DAG dependency counters: upd | pdone [nt*nt], xdone | rhs_cnt [nt]
  unsigned long long *dag_trace = nullptr;  // BALM_DAG_TRACE: device timestamps of the last factorisation
};
void ldlt_work_free(LdltWork *w);

// One damped system (H + u diag(H)) dx = -g of order n (H column-major n x n): the context's own, or a rig's reduced
// one. The solve factors into A [n*n] and w, writes dvec = diag(H) and dx, and uses the context's scal / flags.
struct DenseSystem {
  int n;
  const double *H, *g;
  double *dx, *dvec, *A;
  LdltWork *w;
};

struct balm_ctx {
  int N = 0, n = 0, ldg = 0, Np = 0, device = 0, prec = 0;
  cudaStream_t stream = nullptr;
  bool lm_active = false;     // inside balm_damping_iter (scale speculation and stats hand-over are loop-local)
  bool reuse_ws = false;      // the registration in progress has the shape of the previous one: buffers are kept
  bool defer = false;         // inside balm_damping_iter: phases are enqueued back to back, one host sync per iteration
  bool pending_eval = false;  // an evaluation's events / flags still have to be read (defer mode)
  bool pending_stats_cached = false;
  bool eval_same_poses = false;  // the evaluation in progress follows a rejected LM step: the previous one had its poses
  int sm_count = 132;

  // ---- registered problem (device) ----
  int64_t M = 0, K = 0, Kp = 0;
  bool dense = false;   // every voxel observed by every pose, slot j == pose j
  int max_k = 0;
  double *obs = nullptr;          // SoA [10][Kp], voxel-major (CSR order)
  int *pose_idx = nullptr;        // [K]
  long long *row_ptr = nullptr;   // [M+1]
  double *coe = nullptr;          // [M]
  double *fix = nullptr;          // SoA [10][M] or null
  int *csc_ptr = nullptr, *csc_obs = nullptr, *csc_vox = nullptr;  // pose-major lists (sparse problems)
  int csc_max_len = 0;
  int *csc_lo = nullptr, *csc_hi = nullptr;  // [N] segment of every pose's list inside the current voxel batch (null: whole list)
  int min_planes = 0;             // min over poses of #voxels observing it (precheck, bavoxel.hpp:1071-1085)
  int *planes = nullptr;          // [2][N] device: this rank's per-pose voxel counts | their all-reduced sum
  bool registered = false;        // a voxel set (possibly empty: a rank whose shard has no voxels) is registered
  unsigned long long *vox_key = nullptr;  // [M] 63-bit octree key of every voxel (ascending) when the set came from
                                          // balm_cut_voxels: lets balm_append_scan find the leaf a new point falls into
  int *vox_layer = nullptr;       // [M] octree layer of every voxel (a key digit 7 is BOTH octant 7 and "not split":
                                  // the layer says which)
  bool has_keys = false;
  int64_t cut_stats[BALM_CUT_STATS] = {};  // balm_cut_voxels_stats: the last successful balm_cut_voxels
  balm_assoc_opts assoc{1.0, 2, 15, {1.0 / 16, 1.0 / 16, 1.0 / 16}};  // association options of that call
  WindowState *win = nullptr;     // balm_window_* state (independent of the registered voxel set)
  PoseGraph *pg = nullptr;        // balm_set_pose_factors' window factors (independent of the registered voxel set);
                                  // BALM_PREC_BLOCKS: balm_block_set_factors' factors, part of the cost
  BlockHessian *bh = nullptr;     // BALM_PREC_BLOCKS: the registered set's block pattern, terms, blocks and solver
  bool every_diagonal = true;     // BALM_PREC_BLOCKS: the pattern holds every diagonal pair; false for a balm_spg's
                                  // context, whose pattern holds only those of its factors and priors
  PriorSet *pr = nullptr;         // balm_set_pose_priors' priors (independent of the factor and the voxel set): part of
                                  // the pose-graph cost, and on BALM_PREC_BLOCKS of every full-range evaluation
  bool joint_cost = false;        // balm_set_joint_cost (FP64 / TENSOR): pg and pr join every full-range evaluation
  double *joint_fg = nullptr;     // [n + 1] the joint cost's factor g | cost, before they are added onto c->g | r
  int vloss_kind = BALM_LOSS_TRIVIAL;  // balm_set_voxel_loss: the loss of every voxel (independent of the voxel set)
  double vloss_scale = 1.0;
  Rig *rig = nullptr;             // balm_set_rig's rig (independent of the voxel set: N is fixed at creation)

  // ---- optimiser state (device) ----
  double *poses = nullptr, *poses_trial = nullptr;  // [12N]
  double *H = nullptr, *g = nullptr;                // [n*n + n + 8] contiguous: H | g | r  (one all-reduce);
                                                    // BALM_PREC_BLOCKS: no H, g [n + 8] (g | r)
  double *A = nullptr;                              // [n*n] factor workspace (none in BALM_PREC_BLOCKS)
  double *dx = nullptr;                             // [n]
  double *dvec = nullptr;                           // [n] diag(H)
  LdltWork lw;                                      // the factor workspaces of the solve of H
  unsigned long long *tc_trace = nullptr;           // BALM_TC_TRACE: per-CTA clocks of the last tensor SYRK launch
  double *scal = nullptr;                           // device scalars [32]: 0 r(eval) 1 q1 2 r(residual) 3 u 4..15 gauge
                                                    // snapshot, 16/17 this rank's residual at the current / trial poses
  double *h_scal = nullptr;                         // pinned host mirror [16]
  int *flags = nullptr;                             // device flags [4] (0: ldlt bad pivot)
  int *h_flags = nullptr;

  // ---- evaluation workspaces ----
  int64_t VB = 0;                 // voxels per batch
  double *stats = nullptr;        // [VB][20]
  double *vsums = nullptr;        // [VB][10] per-voxel cluster sums (stats pass: streaming kernel -> eigen kernel)
  double *stats_trial = nullptr;  // [M][20] stats of the LM trial poses (single-batch problems): an accepted step
                                  // hands them to the next evaluation instead of recomputing them
  double *G = nullptr;            // [3*VB][ldg] fp64 scaled factor matrix G' (MN-major: pose index contiguous);
                                  // BALM_PREC_BLOCKS: [K][18] the three scaled G' rows of every observation (CSR order)
  int obs_chunks = 0;
  double *obs_part = nullptr;     // [obs_chunks][27][Np]
  double *accum = nullptr;        // [BALM_ACC][Np] reduced g / diag-block / sum-of-squares accumulators
  double *accum_batch = nullptr;  // same, current batch only
  int res_blocks = 0;
  double *res_part = nullptr;     // [res_blocks]
  int syrk_splits = 0, syrk_tiles = 0, syrk_nb = 0;
  double *syrk_part = nullptr;    // [splits][tiles][128*128]

  // ---- tensor path (int8 split-integer) ----
  int8_t *Gq = nullptr;           // [4][rows_alloc][ldg] int8 digit planes of rint(G' * sc) (3 or 4 used per batch)
  unsigned long long *colmax = nullptr;  // [ldg] bit patterns of max |G'[:,j]| of the current batch
  void *tmap = nullptr;           // CUtensorMap storage
  int tc_tile = 0;                // BALM_TC_TILE: 0 = whole tiles when every SM gets one, 1 = column halves, 2 = whole

  // ---- multi-GPU ----
  void *comm = nullptr;
  double *Hpack = nullptr;        // [n(n+1)/2 + n + 1] lower triangle of H | g | r: what the all-reduce carries
  int rank = 0, world = 1;

  // ---- instrumentation ----
  balm_timings tm{};
  int reused_sweeps = 0;  // balm_get_reused_sweeps (kept out of balm_timings, whose layout is fixed)
  cudaEvent_t ev[16] = {};
  long long launches = 0;
};

// BALM_ERR_UNSUPPORTED for a call that needs the dense H on a BALM_PREC_BLOCKS context (which has none), else BALM_OK
inline int refuse_blocks(const balm_ctx *c, const char *who) {
  if (c->prec != BALM_PREC_BLOCKS) return BALM_OK;
  balm_set_error(std::string(who) + ": not available on a BALM_PREC_BLOCKS context (it holds no dense H)");
  return BALM_ERR_UNSUPPORTED;
}

// balm_set_voxel_loss / balm_batch_set_voxel_loss arguments: a kind of balm_loss, a finite scale > 0 unless trivial
inline int check_voxel_loss(const char *who, int kind, double scale) {
  if (kind != BALM_LOSS_TRIVIAL && kind != BALM_LOSS_HUBER && kind != BALM_LOSS_CAUCHY) {
    balm_set_error(std::string(who) + ": loss kind " + std::to_string(kind) + " (0, 1, 2 allowed)");
    return BALM_ERR_INVALID;
  }
  if (kind != BALM_LOSS_TRIVIAL && !(std::isfinite(scale) && scale > 0.0)) {
    balm_set_error(std::string(who) + ": a robust loss needs a finite scale > 0");
    return BALM_ERR_INVALID;
  }
  return BALM_OK;
}

// The pure quadratic as a loss argument: the NoLoss instantiation of a kernel templated on its loss is that kernel as
// without robust losses (the voxel stats kernels, the pose factors' and priors' cost and linearisation kernels)
struct NoLoss {};

// The voxel loss as the stats kernels take it (voxel_eig_kernel, batch_stats_kernel): kind / scale of
// balm_set_voxel_loss, and with lam non-null the per-voxel readout lam[i] = lambda_min, w[i] = rho'(lambda_min)
// (i: the voxel's index from the start of the launch's range).
struct VoxelLoss {
  int kind;
  double scale;
  double *lam, *w;
};

// ---------------- device math ----------------
#ifdef __CUDACC__

// rho(s) and rho'(s) of BALM_LOSS_HUBER / BALM_LOSS_CAUCHY at scale c; BALM_LOSS_TRIVIAL: s and 1. Shared by the pose
// factors and priors (pose_graph.cu) and the voxels (factor_kernels.cu, batch.cu).
__device__ __forceinline__ void loss_rho(int kind, double c, double s, double *rho, double *drho) {
  const double c2 = c * c;
  if (kind == BALM_LOSS_HUBER && s > c2) {
    const double r = sqrt(s);
    *rho = 2.0 * c * r - c2;
    *drho = c / r;
  } else if (kind == BALM_LOSS_CAUCHY) {
    *rho = c2 * log1p(s / c2);
    *drho = 1.0 / (1.0 + s / c2);
  } else {
    *rho = s;
    *drho = 1.0;
  }
}

// The accept rule of BALM2::damping_iter (bavoxel.hpp:1127-1155), on the host (damping_iter, balm_api.cu) and per
// problem on the device (batch_lm_kernel): q = r1 - r2 (-1 for an unusable step, not_pd or a non-finite r2, which is then
// rejected); on acceptance (q > 0) u *= max(1/3, 1 - (2 rho - 1)^3) with rho = q / q1 and v = 2, else u *= v and
// v *= 2. *t receives the iteration's trace record and *stop the rel_tol exit; returns whether the step is accepted.
// pow is the C library's on the host and CUDA's on the device, as in the reference and the batch respectively.
__host__ __device__ inline bool lm_rule(double r1, double r2, double q1, int not_pd, int calc_hess, double rel_tol,
                                        double *u, double *v, balm_trace *t, bool *stop) {
  double q = r1 - r2;
  if (not_pd || !isfinite(r2)) q = -1.0;
  *t = balm_trace{r1, r2, *u, *v, q, q1, 0, calc_hess, not_pd};
  *stop = rel_tol >= 0 && fabs(r1 - r2) / r1 < rel_tol;  // bavoxel.hpp:1155
  if (q > 0) {  // bavoxel.hpp:1134-1143
    const double rho = q / q1;
    *v = 2;
    const double f = 1 - pow(2 * rho - 1, 3.0);
    *u *= (f < (1.0 / 3.0) ? (1.0 / 3.0) : f);
    t->accepted = 1;
    return true;
  }
  *u = *u * *v;  // bavoxel.hpp:1144-1149
  *v = 2 * *v;
  return false;
}

struct WC {  // world-frame cluster
  double p00, p01, p02, p11, p12, p22, v0, v1, v2, n;
};

// PointCluster::transform (tools.hpp:333-339) on packed symmetric storage. R row-major r[9].
__device__ __forceinline__ WC world_cluster(const double *o, const double *r, const double *p) {
  // Rv
  const double rv0 = r[0] * o[6] + r[1] * o[7] + r[2] * o[8];
  const double rv1 = r[3] * o[6] + r[4] * o[7] + r[5] * o[8];
  const double rv2 = r[6] * o[6] + r[7] * o[7] + r[8] * o[8];
  // X = R * P  (P symmetric: o0 o1 o2 / o1 o3 o4 / o2 o4 o5)
  const double x00 = r[0] * o[0] + r[1] * o[1] + r[2] * o[2];
  const double x01 = r[0] * o[1] + r[1] * o[3] + r[2] * o[4];
  const double x02 = r[0] * o[2] + r[1] * o[4] + r[2] * o[5];
  const double x10 = r[3] * o[0] + r[4] * o[1] + r[5] * o[2];
  const double x11 = r[3] * o[1] + r[4] * o[3] + r[5] * o[4];
  const double x12 = r[3] * o[2] + r[4] * o[4] + r[5] * o[5];
  const double x20 = r[6] * o[0] + r[7] * o[1] + r[8] * o[2];
  const double x21 = r[6] * o[1] + r[7] * o[3] + r[8] * o[4];
  const double x22 = r[6] * o[2] + r[7] * o[4] + r[8] * o[5];
  const double N = o[9];
  WC w;
  // R P R^T + (Rv) p^T + p (Rv)^T + N p p^T
  w.p00 = x00 * r[0] + x01 * r[1] + x02 * r[2] + 2.0 * rv0 * p[0] + N * p[0] * p[0];
  w.p01 = x00 * r[3] + x01 * r[4] + x02 * r[5] + rv0 * p[1] + rv1 * p[0] + N * p[0] * p[1];
  w.p02 = x00 * r[6] + x01 * r[7] + x02 * r[8] + rv0 * p[2] + rv2 * p[0] + N * p[0] * p[2];
  w.p11 = x10 * r[3] + x11 * r[4] + x12 * r[5] + 2.0 * rv1 * p[1] + N * p[1] * p[1];
  w.p12 = x10 * r[6] + x11 * r[7] + x12 * r[8] + rv1 * p[2] + rv2 * p[1] + N * p[1] * p[2];
  w.p22 = x20 * r[6] + x21 * r[7] + x22 * r[8] + 2.0 * rv2 * p[2] + N * p[2] * p[2];
  w.v0 = rv0 + N * p[0];
  w.v1 = rv1 + N * p[1];
  w.v2 = rv2 + N * p[2];
  w.n = N;
  return w;
}

// pose12 (R column-major, p) -> row-major r[9], p[3]
__device__ __forceinline__ void load_pose(const double *__restrict__ pose12, double *r, double *p) {
#pragma unroll
  for (int c = 0; c < 3; c++)
#pragma unroll
    for (int rr = 0; rr < 3; rr++) r[rr * 3 + c] = __ldg(pose12 + c * 3 + rr);
  p[0] = __ldg(pose12 + 9);
  p[1] = __ldg(pose12 + 10);
  p[2] = __ldg(pose12 + 11);
}

// streaming load: read-only path, do not allocate in L1 (the observations are read exactly once per kernel)
__device__ __forceinline__ double ld_stream(const double *p) {
  double v;
  asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];\n" : "=d"(v) : "l"(p));
  return v;
}

template <bool PLAIN>
__device__ __forceinline__ void load_pose_any(const double *pose12, double *r, double *p) {
  if (PLAIN) {  // shared-memory table
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
      for (int rr = 0; rr < 3; rr++) r[rr * 3 + c] = pose12[c * 3 + rr];
    p[0] = pose12[9]; p[1] = pose12[10]; p[2] = pose12[11];
  } else {
    load_pose(pose12, r, p);
  }
}

#define BALM_JROT(app, aqq, apq, arp, arq, vp0, vp1, vp2, vq0, vq1, vq2)        \
  if (apq != 0.0) {                                                             \
    const double th = (aqq - app) / (2.0 * apq);                                \
    const double t = copysign(1.0, th) / (fabs(th) + sqrt(th * th + 1.0));      \
    const double c = rsqrt(t * t + 1.0);                                        \
    const double s = t * c;                                                     \
    app -= t * apq;                                                             \
    aqq += t * apq;                                                             \
    apq = 0.0;                                                                  \
    const double trp = arp, trq = arq;                                          \
    arp = c * trp - s * trq;                                                    \
    arq = s * trp + c * trq;                                                    \
    double a_, b_;                                                              \
    a_ = vp0; b_ = vq0; vp0 = c * a_ - s * b_; vq0 = s * a_ + c * b_;           \
    a_ = vp1; b_ = vq1; vp1 = c * a_ - s * b_; vq1 = s * a_ + c * b_;           \
    a_ = vp2; b_ = vq2; vp2 = c * a_ - s * b_; vq2 = s * a_ + c * b_;           \
  }

// Symmetric 3x3 eigen-decomposition by cyclic Jacobi; eigenvalues ascending, eigenvectors u0,u1,u2.
// Stands in for Eigen::SelfAdjointEigenSolver<Matrix3d> (bavoxel.hpp:345,452).
__device__ __forceinline__ void eig3_jacobi(double a00, double a01, double a02, double a11, double a12, double a22,
                                            double *lam, double *u0, double *u1, double *u2) {
  double v00 = 1, v01 = 0, v02 = 0, v10 = 0, v11 = 1, v12 = 0, v20 = 0, v21 = 0, v22 = 1;  // v[r][c]
  const double scale = fabs(a00) + fabs(a11) + fabs(a22);
#pragma unroll 1
  for (int sweep = 0; sweep < 16; sweep++) {
    const double off = fabs(a01) + fabs(a02) + fabs(a12);
    if (off <= 1e-40 * scale) break;
    BALM_JROT(a00, a11, a01, a02, a12, v00, v10, v20, v01, v11, v21)  // (p,q)=(0,1), r=2
    BALM_JROT(a00, a22, a02, a01, a12, v00, v10, v20, v02, v12, v22)  // (0,2), r=1
    BALM_JROT(a11, a22, a12, a01, a02, v01, v11, v21, v02, v12, v22)  // (1,2), r=0
  }
  double d0 = a00, d1 = a11, d2 = a22;
  double e0[3] = {v00, v10, v20}, e1[3] = {v01, v11, v21}, e2[3] = {v02, v12, v22};
#define BALM_CSWAP(da, db, ea, eb)                                        \
  if (da > db) {                                                          \
    double t_ = da; da = db; db = t_;                                     \
    _Pragma("unroll") for (int q_ = 0; q_ < 3; q_++) { t_ = ea[q_]; ea[q_] = eb[q_]; eb[q_] = t_; } \
  }
  BALM_CSWAP(d0, d1, e0, e1)
  BALM_CSWAP(d1, d2, e1, e2)
  BALM_CSWAP(d0, d1, e0, e1)
#undef BALM_CSWAP
  lam[0] = d0; lam[1] = d1; lam[2] = d2;
#pragma unroll
  for (int q = 0; q < 3; q++) { u0[q] = e0[q]; u1[q] = e1[q]; u2[q] = e2[q]; }
}

// The stats row of one voxel: [0..19] eigen data, [20..39] the observation sweep's record with every per-voxel factor
// folded into the vectors it multiplies (so the sweep spends no instruction on them):
//   vb, u0, a_k = sqrt(coe |w_k|)/NN u_k (k = 1,2; w_k = 2/(l0 - l_k), bavoxel.hpp:392), ug = 2 coe/NN u0,
//   uh = sqrt(coe |w_0|) u0 (w_0 = -2/NN^2, bavoxel.hpp:385), f = 2 coe/NN, s0 = vb . u0
__device__ __forceinline__ void store_stats_row(double *row, double vb0, double vb1, double vb2, const double *u0,
                                                const double *u1, const double *u2, double inv, double coe,
                                                const double *lam) {
  const double c0 = sqrt(2.0 * coe) * inv, c1 = sqrt(2.0 * coe / (lam[1] - lam[0])), c2 = sqrt(2.0 * coe / (lam[2] - lam[0]));
  double2 *st = reinterpret_cast<double2 *>(row);
  st[0] = make_double2(vb0, vb1);
  st[1] = make_double2(vb2, u0[0]);
  st[2] = make_double2(u0[1], u0[2]);
  st[3] = make_double2(u1[0], u1[1]);
  st[4] = make_double2(u1[2], u2[0]);
  st[5] = make_double2(u2[1], u2[2]);
  st[6] = make_double2(inv, c0);
  st[7] = make_double2(c1, c2);
  st[8] = make_double2(coe, lam[0]);
  st[9] = make_double2(lam[1], lam[2]);
  const double f = 2.0 * coe * inv, k1 = c1 * inv, k2 = c2 * inv;
  st[10] = make_double2(vb0, vb1);
  st[11] = make_double2(vb2, u0[0]);
  st[12] = make_double2(u0[1], u0[2]);
  st[13] = make_double2(k1 * u1[0], k1 * u1[1]);
  st[14] = make_double2(k1 * u1[2], k2 * u2[0]);
  st[15] = make_double2(k2 * u2[1], k2 * u2[2]);
  st[16] = make_double2(f * u0[0], f * u0[1]);
  st[17] = make_double2(f * u0[2], c0 * u0[0]);
  st[18] = make_double2(c0 * u0[1], c0 * u0[2]);
  st[19] = make_double2(f, vb0 * u0[0] + vb1 * u0[1] + vb2 * u0[2]);
}

// One observation of the Hessian sweep (left_evaluate_acc2 per-observation loop, bavoxel.hpp:365-402): the three
// scaled G' rows of the observing pose (6 values each), handed to emit(gv) as soon as they are computed, and, with GRAD,
// its gradient and upper diagonal-block terms added to acc[0..26] after that. o: the observation, r/p: its pose
// (row-major R), st: the voxel's sweep record (words 20..39 of its stats row, store_stats_row). Shared by
// obs_pass_kernel and the batched sweep (batch.cu).
template <bool GRAD, typename Emit>
__device__ __forceinline__ void obs_terms(const double *o, const double *r, const double *p, const double *st,
                                          double *acc, Emit emit) {
  // ---- per-voxel sweep record (written by the eigen half of the stats pass, words 20..39 of the stats row) ----
  //   vb = mean, u0 = plane normal, a_k = sqrt(coe |w_k|)/NN u_k (k = 1, 2: the G' rows come out scaled),
  //   ug = 2 coe/NN u0, uh = sqrt(2 coe)/NN u0, f = 2 coe/NN, s0 = vb . u0
  const double *vb = st, *u0 = st + 3, *a1 = st + 6, *a2 = st + 9, *ug = st + 12, *uh = st + 15;
  const double f = st[18], s0 = st[19];
  // ---- world-frame cluster (PointCluster::transform, tools.hpp:333-339): P' = R P R^T + v' p^T + p (R v)^T ----
  const double rv0 = r[0] * o[6] + r[1] * o[7] + r[2] * o[8];
  const double rv1 = r[3] * o[6] + r[4] * o[7] + r[5] * o[8];
  const double rv2 = r[6] * o[6] + r[7] * o[7] + r[8] * o[8];
  const double n = o[9];
  const double vw[3] = {rv0 + n * p[0], rv1 + n * p[1], rv2 + n * p[2]};
  double p00, p01, p02, p11, p12, p22;
  {
    const double x00 = r[0] * o[0] + r[1] * o[1] + r[2] * o[2];
    const double x01 = r[0] * o[1] + r[1] * o[3] + r[2] * o[4];
    const double x02 = r[0] * o[2] + r[1] * o[4] + r[2] * o[5];
    const double x10 = r[3] * o[0] + r[4] * o[1] + r[5] * o[2];
    const double x11 = r[3] * o[1] + r[4] * o[3] + r[5] * o[4];
    const double x12 = r[3] * o[2] + r[4] * o[4] + r[5] * o[5];
    const double x20 = r[6] * o[0] + r[7] * o[1] + r[8] * o[2];
    const double x21 = r[6] * o[1] + r[7] * o[3] + r[8] * o[4];
    const double x22 = r[6] * o[2] + r[7] * o[4] + r[8] * o[5];
    p00 = x00 * r[0] + x01 * r[1] + x02 * r[2] + vw[0] * p[0] + p[0] * rv0;
    p01 = x00 * r[3] + x01 * r[4] + x02 * r[5] + vw[0] * p[1] + p[0] * rv1;
    p02 = x00 * r[6] + x01 * r[7] + x02 * r[8] + vw[0] * p[2] + p[0] * rv2;
    p11 = x10 * r[3] + x11 * r[4] + x12 * r[5] + vw[1] * p[1] + p[1] * rv1;
    p12 = x10 * r[6] + x11 * r[7] + x12 * r[8] + vw[1] * p[2] + p[1] * rv2;
    p22 = x20 * r[6] + x21 * r[7] + x22 * r[8] + vw[2] * p[2] + p[2] * rv2;
  }
  // M = [P' - v' vb^T ; (v' - n vb)^T]  (= TC_i * [R_i | p_i - vb]^T, bavoxel.hpp:368-370)
  const double m00 = p00 - vw[0] * vb[0], m01 = p01 - vw[0] * vb[1], m02 = p02 - vw[0] * vb[2];
  const double m10 = p01 - vw[1] * vb[0], m11 = p11 - vw[1] * vb[1], m12 = p12 - vw[1] * vb[2];
  const double m20 = p02 - vw[2] * vb[0], m21 = p12 - vw[2] * vb[1], m22 = p22 - vw[2] * vb[2];
  const double mb[3] = {vw[0] - n * vb[0], vw[1] - n * vb[1], vw[2] - n * vb[2]};
  const double t0[3] = {m00 * u0[0] + m01 * u0[1] + m02 * u0[2], m10 * u0[0] + m11 * u0[1] + m12 * u0[2],
                        m20 * u0[0] + m21 * u0[1] + m22 * u0[2]};
  const double s0p = mb[0] * u0[0] + mb[1] * u0[1] + mb[2] * u0[2];

  // ---- G' rows (3 per voxel), 6 contiguous values per pose:  row 0 = sqrt(coe|w0|) a_i, a_i = [-u0 x v' ; n u0]
  // (bavoxel.hpp:380,385); rows k = 1,2 = sqrt(coe|w_k|) g_k^i, g_k^i = (U_k M u_0 + U_0 M u_k)/NN with
  // U_k = [hat(-u_k) 0; 0 u_k] (bavoxel.hpp:371-378,392) -- the scale factors ride on the record's vectors ----
  double gv[3][6];
  gv[0][0] = vw[1] * uh[2] - vw[2] * uh[1];
  gv[0][1] = vw[2] * uh[0] - vw[0] * uh[2];
  gv[0][2] = vw[0] * uh[1] - vw[1] * uh[0];
  gv[0][3] = n * uh[0]; gv[0][4] = n * uh[1]; gv[0][5] = n * uh[2];
#pragma unroll
  for (int k = 1; k < 3; k++) {
    const double *ak = k == 1 ? a1 : a2;
    const double ma[3] = {m00 * ak[0] + m01 * ak[1] + m02 * ak[2], m10 * ak[0] + m11 * ak[1] + m12 * ak[2],
                          m20 * ak[0] + m21 * ak[1] + m22 * ak[2]};
    const double sa = mb[0] * ak[0] + mb[1] * ak[1] + mb[2] * ak[2];
    // -(a_k x t0 + u0 x (M a_k)) = t0 x a_k + (M a_k) x u0
    gv[k][0] = t0[1] * ak[2] - t0[2] * ak[1] + ma[1] * u0[2] - ma[2] * u0[1];
    gv[k][1] = t0[2] * ak[0] - t0[0] * ak[2] + ma[2] * u0[0] - ma[0] * u0[2];
    gv[k][2] = t0[0] * ak[1] - t0[1] * ak[0] + ma[0] * u0[1] - ma[1] * u0[0];
    gv[k][3] = ak[0] * s0p + u0[0] * sa;
    gv[k][4] = ak[1] * s0p + u0[1] * sa;
    gv[k][5] = ak[2] * s0p + u0[2] * sa;
  }
  emit(gv);
  if (!GRAD) return;
  // ---- gradient: coe g_0^i = [t0 x ug ; ug (mb . u0)]  (bavoxel.hpp:381) ----
  acc[0] += t0[1] * ug[2] - t0[2] * ug[1];
  acc[1] += t0[2] * ug[0] - t0[0] * ug[2];
  acc[2] += t0[0] * ug[1] - t0[1] * ug[0];
  acc[3] += ug[0] * s0p; acc[4] += ug[1] * s0p; acc[5] += ug[2] * s0p;
  // ---- diagonal block coe*( 2/NN * U0 TCT U0^T + [[Ell+Ell^T,0],[0,0]] )  (bavoxel.hpp:387-388,397-402), upper
  // triangle in row-major order acc[6..26]. Columns 3..5: f a_i u0^T. Top-left 3x3: with |u0| = 1,
  //   hat(u0) P' hat(u0)^T = -P' + u0 q^T + q u0^T - tr(P') u0 u0^T + (tr(P') - u0.q) I,  q = P' u0 = t0 + s0 v',
  // and Ell + Ell^T = (u0 t0^T + t0 u0^T - 2 (t0.u0) I)/NN, so the block is
  //   -f P' + ug z^T + z ug^T + f kappa I,  z = 1.5 t0 + s0 v' - tr(P')/2 u0,  kappa = tr(P') - 2 u0.t0 - s0 u0.v' ----
  {
    const double ag[6] = {vw[1] * ug[2] - vw[2] * ug[1], vw[2] * ug[0] - vw[0] * ug[2], vw[0] * ug[1] - vw[1] * ug[0],
                          n * ug[0], n * ug[1], n * ug[2]};
    const double trp = p00 + p11 + p22, hh = 0.5 * trp;
    const double z[3] = {1.5 * t0[0] + s0 * vw[0] - hh * u0[0], 1.5 * t0[1] + s0 * vw[1] - hh * u0[1],
                         1.5 * t0[2] + s0 * vw[2] - hh * u0[2]};
    const double ut = u0[0] * t0[0] + u0[1] * t0[1] + u0[2] * t0[2];
    const double uv = u0[0] * vw[0] + u0[1] * vw[1] + u0[2] * vw[2];
    const double fk = f * (trp - 2.0 * ut - s0 * uv);
    // rows 0..2: [ TL(rr, rr..2) | ag[rr] u0^T ]; rows 3..5: ag[rr] u0[rr-3 ..]
    acc[6]  += fk - f * p00 + 2.0 * (ug[0] * z[0]);
    acc[7]  += ug[0] * z[1] + z[0] * ug[1] - f * p01;
    acc[8]  += ug[0] * z[2] + z[0] * ug[2] - f * p02;
    acc[9]  += ag[0] * u0[0]; acc[10] += ag[0] * u0[1]; acc[11] += ag[0] * u0[2];
    acc[12] += fk - f * p11 + 2.0 * (ug[1] * z[1]);
    acc[13] += ug[1] * z[2] + z[1] * ug[2] - f * p12;
    acc[14] += ag[1] * u0[0]; acc[15] += ag[1] * u0[1]; acc[16] += ag[1] * u0[2];
    acc[17] += fk - f * p22 + 2.0 * (ug[2] * z[2]);
    acc[18] += ag[2] * u0[0]; acc[19] += ag[2] * u0[1]; acc[20] += ag[2] * u0[2];
    acc[21] += ag[3] * u0[0]; acc[22] += ag[3] * u0[1]; acc[23] += ag[3] * u0[2];
    acc[24] += ag[4] * u0[1]; acc[25] += ag[4] * u0[2];
    acc[26] += ag[5] * u0[2];
  }
}

__device__ __forceinline__ void cross3(const double *a, const double *b, double *c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// ---- pose-covariance propagation (covariance.cu, batch.cu): the per-observation terms of left_jacobian_point ----
__device__ __forceinline__ void hat3(const double *v, double *M /*3x3 row-major*/) {
  M[0] = 0; M[1] = -v[2]; M[2] = v[1];
  M[3] = v[2]; M[4] = 0; M[5] = -v[0];
  M[6] = -v[1]; M[7] = v[0]; M[8] = 0;
}
// g1(w): 4 x 9 (BAs_left.hpp:321-331), row-major
__device__ __forceinline__ void g1_mat(const double *w, double *X /*[4][9]*/) {
#pragma unroll
  for (int e = 0; e < 36; e++) X[e] = 0.0;
  X[0] = w[0]; X[1] = w[1]; X[2] = w[2]; X[6] = w[3];
  X[9 + 1] = w[0]; X[9 + 3] = w[1]; X[9 + 4] = w[2]; X[9 + 7] = w[3];
  X[18 + 2] = w[0]; X[18 + 4] = w[1]; X[18 + 5] = w[2]; X[18 + 8] = w[3];
  X[27 + 6] = w[0]; X[27 + 7] = w[1]; X[27 + 8] = w[2];
}

// c_cov (9x9, row-major) of a cluster under isotropic point noise, from its moments (toolss.hpp:311-343):
// Bi = x Ex + y Ey + z Ez  ->  sum Bf Bf^T = [[sum_kl P_kl E_k E_l^T, sum_k v_k E_k], [sym, N I]]
__device__ __forceinline__ void cluster_cov_iso(const double *o, double pn2, double *C /*[81]*/) {
  const double P[3][3] = {{o[0], o[1], o[2]}, {o[1], o[3], o[4]}, {o[2], o[4], o[5]}};
  // E_k as (row, col, value) triplets: Ex: (0,0,2) (1,1,1) (2,2,1); Ey: (1,0,1) (3,1,2) (4,2,1); Ez: (2,0,1) (4,1,1) (5,2,2)
  const int Er[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
  const double Ev[3][3] = {{2, 1, 1}, {1, 2, 1}, {1, 1, 2}};
#pragma unroll
  for (int e = 0; e < 81; e++) C[e] = 0.0;
  for (int k = 0; k < 3; k++)
    for (int l = 0; l < 3; l++)
      for (int cc = 0; cc < 3; cc++)  // (E_k E_l^T)[r1][r2] = sum_c E_k[r1][c] E_l[r2][c]; column c holds one entry per E
        C[Er[k][cc] * 9 + Er[l][cc]] += P[k][l] * Ev[k][cc] * Ev[l][cc];
  for (int k = 0; k < 3; k++)
    for (int cc = 0; cc < 3; cc++) {
      C[Er[k][cc] * 9 + 6 + cc] += o[6 + k] * Ev[k][cc];
      C[(6 + cc) * 9 + Er[k][cc]] += o[6 + k] * Ev[k][cc];
    }
  for (int d = 0; d < 3; d++) C[(6 + d) * 9 + 6 + d] = o[9];
#pragma unroll
  for (int e = 0; e < 81; e++) C[e] *= pn2;
}

// Everything one observation contributes to the covariance sum (covariance.cu explains the factorisation).
struct CovTerms {
  double Z[4][9];   // [G_j ; -h_j^T / NN]
  double E[6][9];
  double Q[6][4];   // [A_p | a_p]
};

// o: the observation, pose12: its pose, st: the voxel's stats row (store_stats_row: vb, u0..u2, 1/NN, coe, lambda)
__device__ __forceinline__ void cov_terms(const double *o, const double *pose12, const double *st, CovTerms &t) {
  double r[9], p[3];
  load_pose(pose12, r, p);  // row-major R
  const double *vb = st, *u0 = st + 3, *u1 = st + 6, *u2 = st + 9;
  const double inv = st[12];
  const double lam0 = st[17], lam1 = st[18], lam2 = st[19];
  const WC w = world_cluster(o, r, p);
  // m = P' - v' vb^T, mb = v' - n vb  (= TC [R | p - vb]^T, as in the observation sweep)
  const double m[3][3] = {{w.p00 - w.v0 * vb[0], w.p01 - w.v0 * vb[1], w.p02 - w.v0 * vb[2]},
                          {w.p01 - w.v1 * vb[0], w.p11 - w.v1 * vb[1], w.p12 - w.v1 * vb[2]},
                          {w.p02 - w.v2 * vb[0], w.p12 - w.v2 * vb[1], w.p22 - w.v2 * vb[2]}};
  const double mb[3] = {w.v0 - w.n * vb[0], w.v1 - w.n * vb[1], w.v2 - w.n * vb[2]};
  double t0[3], s0 = 0.0;
  for (int a = 0; a < 3; a++) { t0[a] = m[a][0] * u0[0] + m[a][1] * u0[1] + m[a][2] * u0[2]; s0 += mb[a] * u0[a]; }
  // A_p = [hat(t0) - hat(u0) m ; s0 I + u0 mb^T]
  double Ht[9], Hu[9];
  hat3(t0, Ht);
  hat3(u0, Hu);
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) {
      t.Q[a][b] = Ht[a * 3 + b] - (Hu[a * 3] * m[0][b] + Hu[a * 3 + 1] * m[1][b] + Hu[a * 3 + 2] * m[2][b]);
      t.Q[3 + a][b] = (a == b ? s0 : 0.0) + u0[a] * mb[b];
    }
  // a_p = [-u0 x v' ; n u0]
  const double vw[3] = {w.v0, w.v1, w.v2};
  double cuv[3];
  cross3(u0, vw, cuv);
  for (int a = 0; a < 3; a++) { t.Q[a][3] = -cuv[a]; t.Q[3 + a][3] = w.n * u0[a]; }
  // ub = R^T u0, w4 = [ub ; p.u0], w5 = [ub ; (p - vb).u0]
  double ub[3];
  for (int a = 0; a < 3; a++) ub[a] = r[a] * u0[0] + r[3 + a] * u0[1] + r[6 + a] * u0[2];
  const double pu = p[0] * u0[0] + p[1] * u0[1] + p[2] * u0[2];
  const double vu = vb[0] * u0[0] + vb[1] * u0[1] + vb[2] * u0[2];
  const double w4[4] = {ub[0], ub[1], ub[2], pu}, w5[4] = {ub[0], ub[1], ub[2], pu - vu};
  double X[36];
  // B_j = [R | p - vb] g1(w4) - (vb.u0) [0 | R]   (3 x 9)
  g1_mat(w4, X);
  double B[3][9];
  for (int a = 0; a < 3; a++)
    for (int e = 0; e < 9; e++)
      B[a][e] = r[a * 3] * X[e] + r[a * 3 + 1] * X[9 + e] + r[a * 3 + 2] * X[18 + e] + (p[a] - vb[a]) * X[27 + e];
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) B[a][6 + b] -= vu * r[a * 3 + b];
  // G_j = Mk B_j / NN,  Mk = sum_{k=1,2} u_k u_k^T / (lam0 - lam_k)
  const double f1 = 1.0 / (lam0 - lam1), f2 = 1.0 / (lam0 - lam2);
  for (int e = 0; e < 9; e++) {
    const double d1 = u1[0] * B[0][e] + u1[1] * B[1][e] + u1[2] * B[2][e];
    const double d2 = u2[0] * B[0][e] + u2[1] * B[1][e] + u2[2] * B[2][e];
    for (int a = 0; a < 3; a++) t.Z[a][e] = (f1 * u1[a] * d1 + f2 * u2[a] * d2) * inv;
    t.Z[3][e] = 0.0;
  }
  for (int b = 0; b < 3; b++) t.Z[3][6 + b] = -ub[b] * inv;  // -h_j^T / NN, h_j = [0_6, R^T u0]
  // E_p = U_l T g1(w5): top = -hat(u0) (R X03 + p X3), bottom = u0 X3
  g1_mat(w5, X);
  for (int e = 0; e < 9; e++) {
    double y[3];
    for (int a = 0; a < 3; a++) y[a] = r[a * 3] * X[e] + r[a * 3 + 1] * X[9 + e] + r[a * 3 + 2] * X[18 + e] + p[a] * X[27 + e];
    double cy[3];
    cross3(u0, y, cy);
    for (int a = 0; a < 3; a++) { t.E[a][e] = -cy[a]; t.E[3 + a][e] = u0[a] * X[27 + e]; }
  }
}

// acc[0..9] += upper triangle of Z c Z^T (4x4), row-major: one observation's part of the voxel's Wz
__device__ __forceinline__ void cov_wz_add(const CovTerms &t, const double *C, double *acc) {
  double ZC[4][9];
  for (int i = 0; i < 4; i++)
    for (int e = 0; e < 9; e++) {
      double x = 0.0;
      for (int f = 0; f < 9; f++) x += t.Z[i][f] * C[f * 9 + e];
      ZC[i][e] = x;
    }
  int q = 0;
  for (int i = 0; i < 4; i++)
    for (int j = i; j < 4; j++) {
      double x = 0.0;
      for (int e = 0; e < 9; e++) x += ZC[i][e] * t.Z[j][e];
      acc[q++] += x;
    }
}

// One observation's six columns of its voxel's eight rows (c2 Q^T | c2 V^T): g[m * ld + i], m = 0..7, i = 0..5 (g points
// at column 6 p of the voxel's first row), and its diagonal block c2^2 D = c2^2 E c E^T, upper triangle row-major -> d[21]
__device__ __forceinline__ void cov_obs_rows(const CovTerms &t, const double *C, const double (&Wz)[4][4], double c2,
                                             double *g, int ld, double *d) {
  // EC = E c (6x9);  Y^T = E c Z^T (6x4);  D = E c E^T (6x6)
  double EC[6][9];
  for (int i = 0; i < 6; i++)
    for (int e = 0; e < 9; e++) {
      double x = 0.0;
      for (int f = 0; f < 9; f++) x += t.E[i][f] * C[f * 9 + e];
      EC[i][e] = x;
    }
  for (int i = 0; i < 6; i++) {
    for (int mcol = 0; mcol < 4; mcol++) {
      double yt = 0.0;
      for (int e = 0; e < 9; e++) yt += EC[i][e] * t.Z[mcol][e];
      double qw = 0.0;
      for (int f = 0; f < 4; f++) qw += t.Q[i][f] * Wz[f][mcol];
      g[(size_t)mcol * ld + i] = c2 * t.Q[i][mcol];
      g[(size_t)(4 + mcol) * ld + i] = c2 * (0.5 * qw + yt);
    }
  }
  int q = 0;
  for (int i = 0; i < 6; i++)
    for (int j = i; j < 6; j++) {
      double x = 0.0;
      for (int e = 0; e < 9; e++) x += EC[i][e] * t.E[j][e];
      d[q++] = c2 * c2 * x;
    }
}

// Exp (tools.hpp:56-71), row-major output
__device__ __forceinline__ void exp_so3(const double *phi, double *R) {
  const double nrm = sqrt(phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2]);
  R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1;
  if (nrm >= 1e-11) {
    const double x = phi[0] / nrm, y = phi[1] / nrm, z = phi[2] / nrm;
    const double s = sin(nrm), c1 = 1.0 - cos(nrm);
    const double K[9] = {0, -z, y, z, 0, -x, -y, x, 0};
    const double KK[9] = {-(y * y + z * z), x * y, x * z, x * y, -(x * x + z * z), y * z, x * z, y * z, -(x * x + y * y)};
#pragma unroll
    for (int i = 0; i < 9; i++) R[i] += s * K[i] + c1 * KK[i];
  }
}

// R <- Exp(phi) R, p <- Exp(phi) p + dt  (bavoxel.hpp:1123-1125) for one pose; dx6 = [phi | dt]
__device__ __forceinline__ void pose_update_one(const double *pin, const double *dx6, double *pout) {
  double dR[9], r[9], p[3];
  exp_so3(dx6, dR);
  load_pose(pin, r, p);
  double rn[9], pn[3];
#pragma unroll
  for (int a = 0; a < 3; a++) {
#pragma unroll
    for (int b = 0; b < 3; b++) rn[a * 3 + b] = dR[a * 3] * r[b] + dR[a * 3 + 1] * r[3 + b] + dR[a * 3 + 2] * r[6 + b];
    pn[a] = dR[a * 3] * p[0] + dR[a * 3 + 1] * p[1] + dR[a * 3 + 2] * p[2] + dx6[3 + a];
  }
#pragma unroll
  for (int c = 0; c < 3; c++)
#pragma unroll
    for (int a = 0; a < 3; a++) pout[c * 3 + a] = rn[a * 3 + c];
  pout[9] = pn[0]; pout[10] = pn[1]; pout[11] = pn[2];
}

// x <- T_0^-1 x (bavoxel.hpp:1159-1164) for one pose, T_0 read from pose0 (a snapshot when x is pose 0 itself);
// to_identity writes the exact identity instead (pose 0 under benchmark_virtual.cpp:472-479)
__device__ __forceinline__ void gauge_one(double *pose, const double *pose0, bool to_identity) {
  double r0[9], p0[3], r[9], p[3];
  load_pose(pose0, r0, p0);
  load_pose(pose, r, p);
  double rn[9], pn[3];
  const double d[3] = {p[0] - p0[0], p[1] - p0[1], p[2] - p0[2]};
#pragma unroll
  for (int a = 0; a < 3; a++) {
    pn[a] = r0[a] * d[0] + r0[3 + a] * d[1] + r0[6 + a] * d[2];
#pragma unroll
    for (int b = 0; b < 3; b++) rn[a * 3 + b] = r0[a] * r[b] + r0[3 + a] * r[3 + b] + r0[6 + a] * r[6 + b];
  }
  if (to_identity) {
    rn[0] = 1; rn[1] = 0; rn[2] = 0; rn[3] = 0; rn[4] = 1; rn[5] = 0; rn[6] = 0; rn[7] = 0; rn[8] = 1;
    pn[0] = pn[1] = pn[2] = 0;
  }
#pragma unroll
  for (int c = 0; c < 3; c++)
#pragma unroll
    for (int a = 0; a < 3; a++) pose[c * 3 + a] = rn[a * 3 + c];
  pose[9] = pn[0]; pose[10] = pn[1]; pose[11] = pn[2];
}

// ---- packed lower-triangle LDL^T of a small system in shared memory (batch.cu's solves, pose_graph.cu's check) ----
__device__ __forceinline__ int tri_idx(int i, int j, int n) { return j * n - j * (j - 1) / 2 + (i - j); }  // i >= j

// Unpivoted right-looking LDL^T of the packed lower triangle in A, in place (unit-lower L below the diagonal, D on it);
// col: n doubles of scratch. Stops at a zero / tiny / non-finite pivot (ldlt.cu's criterion) and returns true then.
// Block-wide over THREADS threads; the result is the same in every thread.
template <int THREADS>
__device__ __forceinline__ bool ldl_factor(double *A, int n, double *col) {
  const int tid = threadIdx.x;
  for (int k = 0; k < n; k++) {
    const int kk = tri_idx(k, k, n);
    const double dk = A[kk];
    if (!(fabs(dk) > 1e-290 && fabs(dk) < 1e300)) return true;
    for (int i = k + 1 + tid; i < n; i += THREADS) {
      const double t = A[kk + i - k];
      col[i] = t;
      A[kk + i - k] = t / dk;
    }
    __syncthreads();
    const int lane = tid & 31, warp = tid >> 5;
    for (int j = k + 1 + warp; j < n; j += THREADS / 32) {
      const double cj = col[j];
      double *Aj = A + tri_idx(j, j, n);
      for (int i = j + lane; i < n; i += 32) Aj[i - j] -= A[kk + i - k] * cj;
    }
    __syncthreads();
  }
  return false;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// 16-byte global -> shared copy through L2 (cp.async.cg)
__device__ __forceinline__ void cp_async16(void *smem, const void *gmem) {
  unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(sa), "l"(gmem));
}

// fp64 tensor-core MMA (DMMA): 8x8 C fragment (c0, c1) += 8x4 A fragment (a) * 4x8 B fragment (b)
__device__ __forceinline__ void dmma_8x8x4(double &c0, double &c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

#endif  // __CUDACC__

// ---------------- kernel launchers (defined in the .cu files) ----------------
// The stats pass of voxels [v0, v1) under the context's voxel loss; lam_out / w_out (both or neither; need stats_out):
// the per-voxel readout of balm_voxel_residuals, index v - v0.
int launch_voxel_stats(balm_ctx *c, const double *poses, int64_t v0, int64_t v1, double *stats_out, bool use_fix,
                       double *residual_out_dev, double *lam_out = nullptr, double *w_out = nullptr);
int launch_obs_pass(balm_ctx *c, const double *poses, int64_t v0, int64_t v1, bool first_batch);
int launch_obs_colmax(balm_ctx *c, const double *poses, int64_t v0, int64_t v1, bool first_batch);
int launch_obs_int8(balm_ctx *c, const double *poses, int64_t v0, int64_t v1, bool first_batch, const double *sc,
                    int8_t *Gq, int64_t plane_stride, const int *S_dev, int S_alloc, int64_t rows_padded, bool fused,
                    const int *skip);
int tensor_obs_and_syrk(balm_ctx *c, const double *poses, int64_t v0, int64_t v1, bool first_batch);
int launch_syrk_f64(balm_ctx *c, int64_t rows, bool first_batch);
// Dacc null: the Hessian, H = -S + blockdiag(accum rows 6..26) and g, into c->H / c->g (or the all-reduce pack).
// Else R = +S + blockdiag(Dacc), Dacc [21][N]: Rcov_raw of covariance.cu, whose rows always go through the fp64 SYRK.
// S: the SYRK partials in c->syrk_part, summed over the splits in ascending order.
int launch_assemble(balm_ctx *c, const double *Dacc = nullptr, double *R = nullptr);
int build_pose_major_lists(balm_ctx *c, const int *planes_host);
int launch_csc_batch(balm_ctx *c, int64_t v0, int64_t v1);
// the context's own system: c->n, c->H, c->g, c->dx, c->dvec, c->A, c->lw
inline DenseSystem ctx_system(balm_ctx *c) { return DenseSystem{c->n, c->H, c->g, c->dx, c->dvec, c->A, &c->lw}; }
// (H + u diag(H)) dx = -g of s with u into scal[3], q1 into scal[1], flags[0] bad pivot, flags[4] backward-error check
// failed (enqueued; allocates s.w on its first call)
int launch_ldlt_solve(balm_ctx *c, const DenseSystem &s, double u);
// fp64 iterative refinement of s.dx with the factors of the last launch_ldlt_solve of s (waits)
int refine_solution(balm_ctx *c, const DenseSystem &s, int *still_bad);
// ---- pose-covariance pieces (covariance.cu) ----
// Rcov_raw at the device poses into a new n x n buffer of pool, *R_out (enqueued; the voxel statistics, G rows, SYRK
// partials and the assembly of balm_pose_covariance)
int cov_raw_dev(balm_ctx *c, ScratchPool &pool, const double *poses_dev, const double *ccov_host, double point_noise,
                bool include_fix, double **R_out);
// A BALM_PREC_BLOCKS context's raw term at the device poses into raw [pairs][36] on its slot pattern (enqueued; voxel
// batches under BALM_COV_BUDGET_MB with cov_raw_dev's stats and rows, each observation's rows stored on their own)
int cov_raw_blocks_dev(balm_ctx *c, ScratchPool &pool, const double *poses_dev, const double *ccov_host,
                       double point_noise, bool include_fix, double *raw);
// The joint (n_sel x 6)^2 covariance of the selection, or its marginals alone, fit BALM_COV_BUDGET_MB (P: the solver's
// unknowns, N: slots)
bool block_point_cov_fits(int P, int N, int n_sel, bool joint);
// Sigma_sel = W^T R W, W = J Y, Y = A^-1 E after sparse_factor_undamped(sp, anchor): rig null for the context's own
// unknowns (J = I), else the rig at state; sel [n_sel] distinct unknowns; raw the device raw term on the slot pattern.
// cov_host (6 n_sel)^2 column-major or null (then the marginals in chunks), marg_host [n_sel][36] or null. Waits.
int block_point_cov_dev(balm_ctx *c, SparseSolver *sp, const Rig *rig, const double *state, int anchor, int n_sel,
                        const int32_t *sel, const double *raw, double *cov_host, double *marg_host);
// undamped LDL^T of s (launch_ldlt_solve with u = 0), then one wait: BALM_ERR_NOT_PD with singular_msg for a bad pivot
// or min |d| not above 1e-11 max |d|, pivots [skip, skip + 6) left out of both (skip -1: none)
int cov_factor(balm_ctx *c, const DenseSystem &s, int skip, const char *singular_msg);
// B <- H^-1 B H^-T with the factors of the last cov_factor of s (enqueued)
int cov_sandwich(balm_ctx *c, const DenseSystem &s, double *B);
// rows and columns [a0, a0 + 6) of the n x n matrix A set to 0, its diagonal there to diag (enqueued)
int cov_delete_block(balm_ctx *c, double *A, int n, int a0, double diag);
int launch_pose_update(balm_ctx *c, const double *poses_in, const double *dx, double *poses_out);
// snap: 12 doubles of device scratch for pose 0
int launch_gauge(cudaStream_t st, int N, double *poses, double *snap, int mode);
// q1 = 1/2 x.(u D x - g) -> scal[1], u = *u_dev
int launch_q1(cudaStream_t st, const double *x, const double *g, const double *dvec, int n, const double *u_dev,
              double *scal);
int launch_synth(balm_ctx *c, int64_t n_voxels, int64_t first_voxel, int pts, double noise, double range,
                 uint64_t seed, const double *poses_gt_dev);
int factor_kernels_setup();
int syrk_f64_setup();
int ldlt_setup();
int covariance_setup();
int pose_graph_setup();
int tensor_syrk_init(balm_ctx *c);
void tensor_syrk_free(balm_ctx *c);
int tensor_syrk_check(balm_ctx *c);
int tensor_syrk_check_enqueue(balm_ctx *c);
int tensor_syrk_check_finish(balm_ctx *c);
void tensor_syrk_new_problem(balm_ctx *c);

// ---------------- pose graph (pose_graph.cu) ----------------
// After those checks: uploads the factors on st, runs the PD check (per factor status) and builds the assembly tables
// -> a new set in *out (the caller replaces its own with it).
int pose_graph_build(cudaStream_t st, int P, int n_factors, const int64_t *factor_ptr, const int32_t *factor_pose,
                     const double *poses_hat12, const double *H, std::vector<int> *status, PoseGraph **out,
                     long long *launches);
// H | g | scal[0] of the registered factors at the device poses (enqueued, no wait)
int pose_graph_eval(balm_ctx *c, const double *poses);
// the same sums with one 6x6 block per pair (column-major, in pose_graph_pairs order) instead of dense H (enqueued)
int pose_graph_eval_blocks(const PoseGraph *p, cudaStream_t st, const double *poses, double *blocks, double *g,
                           double *cost, long long *launches);
// The factor term on a larger block pattern (enqueued): pair p's sum added onto blocks[map[p]], the factor g into
// g [6P] and the cost into *cost
int pose_graph_add_blocks(const PoseGraph *p, cudaStream_t st, const double *poses, double *blocks, const int *map,
                          double *g, double *cost, long long *launches);
// The factor term on an evaluated dense H (6P x 6P, enqueued): pair (i, j)'s sum added onto H at (i, j) and at its
// transpose, the factor g into g [6P] and the cost into *cost
int pose_graph_add_dense(const PoseGraph *p, cudaStream_t st, const double *poses, double *H, double *g, double *cost,
                         long long *launches);
// the cost at the device poses into the device scalar *out (enqueued, no wait)
int pose_graph_cost(const PoseGraph *p, cudaStream_t st, const double *poses, double *out, long long *launches);
// the (i, j), i <= j, of every nonzero 6x6 block pair of H, ascending in (i, j)
const std::vector<int2> &pose_graph_pairs(const PoseGraph *p);
// device bytes the registered set holds (factors, staging, tables, and the loss arrays while a loss is set)
long long pose_graph_bytes(const PoseGraph *p);
int pose_graph_n_factors(const PoseGraph *p);
// balm_set_factor_loss after its argument checks: kind [F] (null: all trivial) and scale [F]; waits for the upload
int pose_graph_set_loss(PoseGraph *p, cudaStream_t st, const int32_t *kind, const double *scale);
// balm_factor_residuals: s_f and rho'(s_f) of every factor at the device poses (0 for inactive factors) into the host
// arrays s and w [F] (either may be null); enqueues the cost pass and waits once
int term_residuals(const PoseGraph *p, cudaStream_t st, const double *poses, double *s, double *w, long long *launches);

// ---------------- absolute pose priors (pose_graph.cu) ----------------
// After the argument checks: uploads n priors (pose [n], hat12 [12n], lever3 [3n] or null, H36 [36n] column-major,
// kind [n] or null, scale [n]), decides each prior's status (BALM_OK, or BALM_ERR_NOT_PD when H has an eigenvalue below
// -1e-12 lambda_max or is zero; such a prior is in no sum) and builds the assembly tables -> a new set in *out (waits)
int prior_set_build(cudaStream_t st, int n, const int32_t *pose, const double *hat12, const double *lever3,
                    const double *H36, const int32_t *kind, const double *scale, std::vector<int> *status,
                    PriorSet **out);
// the index in `pairs` (ascending (i, j)) of the diagonal block of every pose with an active prior (waits)
int prior_set_map(PriorSet *p, cudaStream_t st, const std::vector<int2> &pairs);
// an active prior exists (p may be null)
bool prior_set_active(const PriorSet *p);
// the poses with active priors, ascending
const std::vector<int> &prior_set_poses(const PriorSet *p);
long long prior_set_bytes(const PriorSet *p);
// the priors' H and g at the device poses added onto the dense H (n x n) / onto the diagonal blocks of the mapped
// pattern, and onto g; their cost added onto *cost (enqueued)
int prior_add_dense(const PriorSet *p, cudaStream_t st, const double *poses, double *H, size_t n, double *g,
                    double *cost, long long *launches);
int prior_add_blocks(const PriorSet *p, cudaStream_t st, const double *poses, double *blocks, double *g, double *cost,
                     long long *launches);
// the priors' cost at the device poses added onto the device scalar *cost (enqueued)
int prior_add_cost(const PriorSet *p, cudaStream_t st, const double *poses, double *cost, long long *launches);
// balm_prior_residuals: s and rho'(s) of every prior (0 for NOT_PD ones) into the host arrays s, w [n] (either may be
// null); waits once
int term_residuals(const PriorSet *p, cudaStream_t st, const double *poses, double *s, double *w, long long *launches);

// ---------------- rig (rig.cu) ----------------
// After the argument checks: the rig of N slots (base_of / lidar_of [N] host, base_fixed [B] / lidar_fixed [L] host or
// null: none fixed), its slot tables and the buffers of its reduced system -> a new rig in *out (waits). sparse: the
// block-sparse rig of a BALM_PREC_BLOCKS context (no dense H_rig, K or factor; its pattern comes with rig_blocks_sync)
int rig_build(cudaStream_t st, int N, int B, int L, const int32_t *base_of, const int32_t *lidar_of,
              const uint8_t *base_fixed, const uint8_t *lidar_fixed, bool sparse, Rig **out);
int rig_n(const Rig *r);  // n_rig = 6 x free unknowns
int rig_bases(const Rig *r);
int rig_lidars(const Rig *r);
bool rig_any_base_fixed(const Rig *r);
int rig_free_bases(const Rig *r);  // free base poses: free indices [0, rig_free_bases) are base poses
// the reduced system H_rig | g_rig, dx, and the rig's own factor workspaces
DenseSystem rig_system(Rig *r);
// device [12 (B + L)] base poses then extrinsics: the current state, or the trial one; rig_swap_states exchanges them
double *rig_state(Rig *r, bool trial);
void rig_swap_states(Rig *r);
// the scan poses X_s = T_base_of[s] E_lidar_of[s] of every slot into poses [12N] (enqueued)
int rig_compose(const Rig *r, cudaStream_t st, const double *state, double *poses, long long *launches);
// H_rig and g_rig at state from the context's H [6N x 6N] and g [6N] (enqueued): K = H J, then J^T K on the lower
// blocks plus the second-order correction, each sum in ascending slot order, mirrored; no atomics
int rig_reduce(const Rig *r, cudaStream_t st, const double *state, const double *H, const double *g,
               long long *launches);
// raw_rig = J^T R J at state for any symmetric R [6N x 6N] (enqueued): rig_reduce's sums without the correction and
// without g, through the rig's K, into out [n_rig x n_rig] (column-major, mirrored)
int rig_reduce_raw(const Rig *r, cudaStream_t st, const double *state, const double *R, double *out,
                   long long *launches);
// ---- block-sparse rig (rig_sparse) ----
bool rig_sparse(const Rig *r);
// The rig's block pattern, K tables, blocks and SparseSolver (on scal / flags) from the slot pattern slot_pairs of
// generation gen, unless it was derived from that generation already (waits when it builds). BALM_ERR_UNSUPPORTED
// (message prefixed with who) when too large to index; the rig then keeps its previous pattern.
int rig_blocks_sync(Rig *r, cudaStream_t st, const std::vector<int2> &slot_pairs, long long gen, double *scal,
                    int *flags, const char *who);
// H_rig's blocks and g_rig at state from the slot blocks Hb and g [6N] (enqueued): K_sv = sum_t H_st J_t, then
// J^T K plus the correction per rig pair, every sum in ascending slot order; no atomics
int rig_reduce_blocks(const Rig *r, cudaStream_t st, const double *state, const double *Hb, const double *g,
                      long long *launches);
const std::vector<int2> &rig_pairs(const Rig *r);  // (u, v), u <= v, ascending over the free unknowns
const double *rig_blocks(const Rig *r);            // device [pairs][36], column-major, rows of u
SparseSolver *rig_solver(const Rig *r);
// device bytes the rig holds (tables, states, vectors, pattern, blocks and solver); l_blocks / levels of its L
long long rig_blocks_bytes(const Rig *r, int64_t *l_blocks, int64_t *levels);
// W = J Y at state (enqueued): Y [6 x free unknowns][ld] row-major with unknown u's rows at 6 col[u] (device col),
// W [6N][ld], the first ncols columns
int rig_apply_j(const Rig *r, cudaStream_t st, const double *state, const int *col, const double *Y, int ld, int ncols,
                double *W, long long *launches);
// state_out = the left step of the rig's dx on every free unknown of state, fixed ones copied (enqueued)
int rig_update(const Rig *r, cudaStream_t st, const double *state, double *state_out, long long *launches);

// ---------------- sparse pose graph (pose_graph_sparse.cu) ----------------
void sparse_solver_free(SparseSolver *s);
// Symbolic factorisation of the pairs' block pattern over P poses (host), device tables and the captured solve on st.
// dvec, dx, scal and flags are the handle's buffers the solve reads and writes (as the context's launch_ldlt_solve).
// who: prefix of the BALM_ERR_UNSUPPORTED message when the pattern is too large to index.
int sparse_solver_build(cudaStream_t st, int P, const std::vector<int2> &pairs, const double *blocks, const double *g,
                        double *dvec, double *dx, double *scal, int *flags, const char *who, SparseSolver **out);
// blocks of L, elimination-tree levels and device bytes held
void sparse_solver_stats(const SparseSolver *s, int64_t *l_blocks, int64_t *levels, int64_t *bytes);
// (H + u diag(H)) dx = -g with u in scal[3]: damped copy, factorisation, substitutions, q1 -> scal[1], the backward-error
// check (flags[0] bad pivot, flags[4] check failed, scal[20] omega); one graph launch, enqueued
int sparse_solve(SparseSolver *s, cudaStream_t st);
// refine_solution's rounds with the same factors; *still_bad when omega stayed above the tolerance (waits)
int sparse_refine(SparseSolver *s, cudaStream_t st, int *h_flags, double *h_scal, int *still_bad);
// Marginal covariances: cov (host, [pairs][36] in the registration's pair order, rows of pose i, columns of pose j,
// column-major) = (H without the anchor's rows and columns)^-1 on H's block pattern, 0 on the anchor's blocks (anchor in
// [-1, P), checked by the caller). The first call builds the selected-inversion tables (BALM_ERR_UNSUPPORTED, before
// eval and with nothing changed, when too large). eval leaves H in the solver's blocks (enqueued); then the undamped
// factorisation overwrites L, D, dvec and scal[3], BALM_ERR_NOT_PD (message prefixed with who) when it is singular.
// Waits twice (pivot test, copy-out), and once more on the first call while it builds the tables.
int sparse_covariance(SparseSolver *s, cudaStream_t st, int anchor, const std::function<int()> &eval, const char *who,
                      double *cov, long long *launches);
// The undamped factorisation of the solver's blocks with pose anchor's rows and columns replaced by I (anchor -1: none)
// and the singularity test of sparse_covariance, which runs it after eval: BALM_ERR_NOT_PD (message prefixed with who)
// when singular. Overwrites L, D, dvec and scal[3]; waits once.
int sparse_factor_undamped(SparseSolver *s, cudaStream_t st, int anchor, const char *who, long long *launches);
// Y <- A^-1 Y for the last sparse_factor_undamped's A: Y [6P][ld] row-major, rows in column (elimination) order, the
// first ncols columns (enqueued). A column's result does not depend on the other columns.
int sparse_solve_many(SparseSolver *s, cudaStream_t st, double *Y, int ld, int ncols, long long *launches);
// the column of every pose (host; filled by sparse_factor_undamped), the number of poses, and every pose's pairs (device
// pp_ptr [P + 1], pp: (2 pair + transposed, other pose), ascending in the other pose)
const std::vector<int> &sparse_solver_columns(SparseSolver *s);
int sparse_solver_size(const SparseSolver *s);
void sparse_solver_pose_pairs(const SparseSolver *s, const int **pp_ptr, const int2 **pp);

// ---------------- block-sparse Hessian of a BALM_PREC_BLOCKS context (blocks.cu) ----------------
// The registered voxels' pair pattern and update terms, then the union pattern with c->pg's factor pairs and c->pr's
// diagonal pairs and its symbolic factorisation -> c->bh (replacing the previous one). BALM_ERR_UNSUPPORTED (message
// prefixed with who) when the terms or pairs are too many to index; c->bh is then kept.
int block_hessian_build(balm_ctx *c, const char *who);
// The union pattern of c->bh's voxel pairs, pg's pairs (pg may be null) and c->pr's diagonal pairs replaces c->bh's, the
// voxel terms kept; on an error c->bh is unchanged.
int blocks_repattern(balm_ctx *c, const PoseGraph *pg, const char *who);
// The prior set pr (may be null) in place of c->pr: c->bh's pattern is rebuilt only when its union with pr's diagonal
// pairs differs from the current one (never when it holds every diagonal pair), and pr's diagonal table points into
// it; on an error c->bh is unchanged.
int blocks_set_priors(balm_ctx *c, PriorSet *pr, const char *who);
// c->pg's factor blocks, g and cost at poses added onto the evaluated blocks, c->g and the residual c->g[n] (enqueued);
// stored there when the pattern is the factor pairs alone and there is no voxel term
int blocks_add_factors(balm_ctx *c, const double *poses);
// c->pg's cost at poses added onto the device scalar *r (enqueued; stored when there is no voxel term, as above)
int blocks_add_factor_cost(balm_ctx *c, const double *poses, double *r);
// c->pr's blocks, g and cost at poses added onto the evaluated blocks (after the factors'), c->g and the residual
// c->g[n] (enqueued)
int blocks_add_priors(balm_ctx *c, const double *poses);
// An FP64 / TENSOR context's joint cost (balm_set_joint_cost): c->pg's H added onto the evaluated dense c->H, its g and
// cost through c->joint_fg onto c->g and the residual c->g[n] (enqueued)
int joint_add_factors(balm_ctx *c, const double *poses);
// c->pg's cost at poses through c->joint_fg onto the device scalar *r (enqueued)
int joint_add_factor_cost(balm_ctx *c, const double *poses, double *r);
// the blocks of voxels [head, end) from c->G (the per-observation store) and the accumulators, g from the accumulators
int launch_blocks(balm_ctx *c, int64_t head, int64_t end);
// the blocks and c->g | r zeroed before an evaluation without voxel term (nothing when the pattern is the factor pairs
// alone: blocks_add_factors then stores every block, g and r)
int blocks_zero(balm_ctx *c);
const std::vector<int2> &blocks_pairs(const BlockHessian *b);
const double *blocks_device(const BlockHessian *b);
SparseSolver *blocks_solver(const BlockHessian *b);
// the slot pattern's generation: it changes whenever blocks.cu builds a new pattern
long long blocks_generation(const BlockHessian *b);
// device bytes of the pattern, terms, blocks and solver; l_blocks / levels of the factorisation
long long blocks_bytes(const BlockHessian *b, int64_t *l_blocks, int64_t *levels);
// The point-noise raw term R on the pattern (covariance.cu has its terms), one voxel batch [v0, v1): raw [pairs][36]
// = (add ? raw : 0) + sum over the batch's update terms of the partner-row products of rows [obs - row_ptr[v0]][8][6]
// (c2 Q^T | c2 V^T of covariance.cu), plus Dacc [21][N] on the diagonal pairs when Dacc is not null (enqueued).
// BALM_ERR_INVALID without voxel pairs.
int launch_raw_blocks(balm_ctx *c, const double *rows, int64_t v0, int64_t v1, const double *Dacc, bool add, double *raw);

// ---------------- association (assoc.cu) ----------------
// The plane voxels of one or more problems cut from raw scans. Host arrays; xyz (n_points x 3 float32, body frame) and
// poses12 are uploaded once. Either frame != NULL: one problem whose pose rows are its frames (balm_cut_voxels; the
// points of frame f are in slot f), or a problem table: problem p owns the rows [pose_ptr[p], pose_ptr[p+1]) and row j
// is the scan pose_scan[j] = points [scan_ptr[s], scan_ptr[s+1]) in slot j - pose_ptr[p]; n_items = the sum of the
// rows' point counts (< 2^31, checked by the caller). With on_device (one problem only) xyz and frame are device arrays
// that stay with the caller. outer: the pool the call's scratch is counted in (may be null); stats: the call's
// host-to-device bytes and its root voxels are added to it (may be null).
struct AssocStats {
  int64_t h2d_bytes = 0, roots = 0;
};
struct AssocInput {
  const char *who;  // prefix of error messages
  int64_t n_points;
  const float *xyz;
  int n_rows;  // pose rows when frame != NULL
  const double *poses12;
  const int32_t *frame;
  int n_problems;
  const int64_t *pose_ptr;
  const int32_t *pose_scan;
  const int64_t *scan_ptr;
  int64_t n_items;
  bool on_device = false;
  ScratchPool *outer = nullptr;
  AssocStats *stats = nullptr;
};
// Scratch bound of assoc_cut's one-problem mode, in bytes: n points x assoc_bytes_per_point(layer_limit) +
// assoc_bytes_fixed(n_rows) covers every buffer the call (and balm_cut_voxels' slab path around it) takes at once.
int64_t assoc_bytes_per_point(int layer_limit);
int64_t assoc_bytes_fixed(int n_rows);
// balm_cut_voxels' slab path (assoc.cu): the points of in (host arrays, one problem, any n_points) cut in root-key slabs
// of at most `cap` points each, every slab's voxels staged on the host (the caller registers them).
struct CutSlabStats {
  int64_t slabs = 0, max_slab = 0, roots = 0, h2d_bytes = 0;
  double ms_roots = 0, ms_select = 0, ms_cut = 0;
};
struct SlabVoxels {  // the staged registration: M voxels, K observations, host arrays
  int64_t M = 0, K = 0;
  std::vector<long long> row_ptr;
  std::vector<int> pose_idx, layer;
  std::vector<double> obs[10], coe;
  std::vector<unsigned long long> key;
};
// Where the voxels are emitted (device arrays): observation o, column c at obs[c * obs_cstride + o * obs_ostride]
// (SoA of a context or AoS of a batch), pose_idx = slot, row_ptr [M + 1], coe, key and layer [M].
struct AssocEmit {
  double *obs;
  int64_t obs_cstride, obs_ostride;
  int *pose_idx;
  long long *row_ptr;
  double *coe;
  unsigned long long *key;
  int *layer;
};
// Called once the sizes are known: M voxels, K observations, per problem voxel_ptr / obs_ptr [B + 1]. Allocates the
// destination and fills *out, or returns an error that ends the call.
using AssocRegister = std::function<int(int64_t M, int64_t K, const int64_t *voxel_ptr, const int64_t *obs_ptr,
                                        AssocEmit *out)>;
balm_assoc_opts resolve_assoc_opts(const balm_assoc_opts *opts);  // opts or the defaults, eigen ratios rounded to float
// opts: from resolve_assoc_opts, layer_limit in 0..2 (checked by the caller)
int assoc_cut(cudaStream_t st, const AssocInput &in, const balm_assoc_opts &opts, const AssocRegister &reg,
              long long *launches);
// budget: device scratch bytes; cap: points per slab (< 2^31). Fills out on success; on any error nothing is staged.
int assoc_cut_slabs(cudaStream_t st, const AssocInput &in, const balm_assoc_opts &opts, size_t budget, int64_t cap,
                    ScratchPool &outer, SlabVoxels *out, CutSlabStats *stats, long long *launches);
// Keyframes of a batch (balm_batch_merge_scans): the problem table and scan pool of AssocInput's batch form, checked by
// the caller; n_items (< 2^31) = the rows' point counts summed. Writes kf_ptr [B + 1] and kf_xyz (host) only on success;
// BALM_ERR_INVALID names the lowest problem with a voxel index outside +-2^20.
struct MergeInput {
  const char *who;
  int n_problems;
  const int64_t *pose_ptr;
  const int32_t *pose_scan;
  const int64_t *scan_ptr;
  int64_t n_points;
  const float *xyz;
  const double *poses12;
  double voxel_size;
  int64_t n_items;
};
int merge_scans_build(cudaStream_t st, const MergeInput &in, int64_t *kf_ptr, float *kf_xyz, long long *launches);

// The sliding-window steps of a batch (balm_batch_marginalize / balm_batch_append_scan) and of a context, its one-problem
// case (balm_marginalize / balm_append_scan). The registration they read: problem p owns the pose rows [pose_ptr[p],
// pose_ptr[p+1]) and the voxels [voxel_ptr[p], voxel_ptr[p+1]) (host tables [B + 1]); device arrays vox_prob [M] (null:
// every voxel is problem 0, B = 1), row_ptr [M + 1], pose_idx [K] (problem-local), obs: column c of observation o at
// obs[c * obs_cstride + o * obs_ostride] (AoS [K][10] of a batch, SoA [10][Kp] of a context), fix likewise per voxel or
// null, coe [M], key / layer [M] (null: not carried; appending needs them). poses12: the host's P x 12 poses.
struct BatchVoxels {
  int B;
  int64_t M;
  const int64_t *pose_ptr, *voxel_ptr;
  const int *vox_prob;
  const long long *row_ptr;
  const int *pose_idx;
  const double *obs;
  int64_t obs_cstride, obs_ostride;
  const double *fix;
  int64_t fix_cstride, fix_vstride;
  const double *coe;
  const unsigned long long *key;
  const int *layer;
  const double *poses12;
};
// Where the new registration is emitted (device arrays, AoS): row_ptr [M + 1], pose_idx / obs [K], fix / coe / key /
// layer [M]; fix is always written by marginalisation, by appending only when the input has one; key / layer when the
// input has them.
struct WindowEmit {
  long long *row_ptr;
  int *pose_idx;
  double *obs, *fix, *coe;
  unsigned long long *key;
  int *layer;
};
// Called once the sizes are known: per problem voxel_ptr / obs_ptr [B + 1] of the new registration. Allocates the
// destination and fills *out, or returns an error that ends the call.
using WindowRegister = std::function<int(const int64_t *voxel_ptr, const int64_t *obs_ptr, WindowEmit *out)>;
// mg_size [B]: 0 (problem copied unchanged) or in [1, N_p) (checked by the caller)
int batch_marginalize_build(cudaStream_t st, const BatchVoxels &in, const int *mg_size, int min_ps,
                            const WindowRegister &reg, long long *launches);
// scan_of [B] (-1: problem copied unchanged) and slot [B] checked by the caller; scan s = xyz[scan_ptr[s] ..
// scan_ptr[s+1]) of n_points; n_matched [B]. BALM_ERR_INVALID, before reg is called, when a slot is not above every scan
// already observing one of its problem's voxels: batch, the message of balm_batch_append_scan naming the lowest such
// problem, else that of balm_append_scan.
int batch_append_build(cudaStream_t st, const BatchVoxels &in, const balm_assoc_opts &o, const int32_t *scan_of,
                       const int *slot, const int64_t *scan_ptr, const float *xyz, int64_t n_points,
                       const WindowRegister &reg, int64_t *n_matched, bool batch, long long *launches);

// The persistent sliding-window octree of B problems (balm_window_* with B = 1, balm_batch_window_*). Problem p has
// n_slots[p] slots and owns the pose rows [sum_{q<p} n_slots[q], ...) of every poses12 (host, P x 12). Arguments are
// checked by the callers (who: prefix of error messages); per-problem arrays have B entries, 0 / -1 = problem left
// alone. A rejected call (BALM_ERR_INVALID / UNSUPPORTED before anything changed) leaves the window as it was.
// reset: o from resolve_assoc_opts, replaces *ws; batch: errors name the problem, 2^31 points are UNSUPPORTED.
int window_reset_build(WindowState **ws, const char *who, int B, const int *n_slots, const balm_assoc_opts &o, bool batch);
const std::vector<int> &window_slots(const WindowState *w);
const balm_assoc_opts &window_opts(const WindowState *w);
// cut: problem p takes scan scan_of[p] (xyz[scan_ptr[s] .. scan_ptr[s+1]) of the n_scans) into slot slot[p], at pose
// row pose_base[p] + slot[p]
int window_cut_build(cudaStream_t st, WindowState &w, const char *who, const int32_t *scan_of, const int *slot,
                     int n_scans, const int64_t *scan_ptr, const float *xyz, const double *poses12, long long *launches);
int window_recut_build(cudaStream_t st, WindowState &w, const int *win_count, long long *launches);
// poses12 may be null (no re-transform)
int window_marginalize_build(cudaStream_t st, WindowState &w, const int *mg, const double *poses12, const int *win_count,
                             long long *launches);
// the pushed nodes of every problem in ascending (problem, key), emitted where reg says (fix, key and layer always)
int window_push_build(cudaStream_t st, WindowState &w, const int *win_count, const WindowRegister &reg,
                      long long *launches);

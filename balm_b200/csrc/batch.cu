// batch.cu -- batched bundle adjustment: B independent small problems (at most BALM_BATCH_MAX_POSES poses each),
// registered once and optimised together, each with its own LM state (include/balm_b200.h, balm_batch_*).
//
// Per LM iteration, enqueued back to back on the batch's stream, every kernel masked per problem:
//   batch_stats_kernel<true>   per voxel: cluster sums, eigen-decomposition, stats row, residual term (= the stats pass)
//   batch_residual_kernel      per problem: fixed-order sum of its voxels' residual terms -> r1
//   batch_obs_kernel           per 32-voxel chunk of one problem (chunk_walk): G' rows (fp64, dense per problem) and the
//                              per-pose gradient / diagonal-block partials (obs_terms, shared with obs_pass_kernel)
//   batch_syrk_kernel<3, 0>    per (problem, 64x64 upper tile, 768-row chunk): DMMA partial of G'^T G'
//   batch_assemble_kernel<27, 6, true, true>  per (problem, 64-column block): H = -sum of partials + blockdiag, g
//   batch_solve_kernel         per problem, one CTA: unpivoted LDL^T of H + uD in shared memory, backward error, up to
//                              3 rounds of refinement, q1, trial poses
//   batch_stats_kernel<false> + batch_residual_kernel at the trial poses -> r2
//   batch_lm_kernel            one thread per problem: accept / reject, u, v, trace, stop
// The host waits once per iteration, for the number of problems still active. Every split of work depends on the
// problem alone and every sum runs in a fixed order (no floating-point atomics), so a problem's results do not depend on
// the other problems of the batch or on its position in it.
//
// The pose covariance (balm_batch_pose_covariance) follows the same rules, with the per-observation terms of covariance.cu:
//   batch_stats_kernel<true>    (inside enqueue_eval when Rcov is wanted, which also gives H) at the given poses
//   batch_cov_rows_kernel       per voxel: Wz, the eight rows c2 Q^T | c2 V^T (8 M_p x ldp per problem), c2^2 D per obs
//   batch_cov_diag_kernel       per 32-voxel chunk (chunk_walk): per-pose partial sums of the c2^2 D blocks
//   batch_syrk_kernel<8, 4>     per (problem, tile, 768-row chunk): partial of Q V^T + V Q^T (A = partner row ^ 4)
//   batch_assemble_kernel<21, 0, false, false>  per (problem, 64-column block): Rcov_raw = + sum of partials + blockdiag
//   batch_cov_solve_kernel      per problem, one CTA: LDL^T of H, singularity test, H^-1 Rcov_raw H^-1, symmetrised
//
// The batch's persistent window maps (balm_batch_window_*) live in assoc.cu's WindowState, one state for every problem;
// balm_batch_window_push emits the pushed nodes straight into a new registration (reg_layout / reg_finish / install).
#include <math.h>
#include <string.h>
#include <algorithm>
#include <type_traits>
#include <vector>
#include "internal.cuh"

namespace {

constexpr int CHUNK = 32;                      // voxels per warp of the observation sweep
constexpr int ROWS = 768;                      // G' rows (256 voxels) per SYRK work item
constexpr int TILE = 64;                       // SYRK output tile
constexpr int KB = 16;                         // G' rows per shared-memory stage of the SYRK
constexpr int LDS = TILE + 4;
constexpr int MAXN = 6 * BALM_BATCH_MAX_POSES;  // 192 unknowns
constexpr int SOLVE_THREADS = 256;
constexpr double OMEGA_TOL = 1e-12;            // componentwise backward error accepted without refinement (ldlt.cu)
constexpr int SOLVE_SMEM = (MAXN * (MAXN + 1) / 2 + 5 * MAXN) * (int)sizeof(double);

struct Prob {                  // layout of one problem, built on the host at registration
  int pose_base, np, n, ldp;   // first pose in the concatenated array, poses, 6 np, G' row stride (n rounded up to 64)
  int ochunk_base, n_ochunks;  // its observation-sweep chunks
  long long vox_base, nvox;    // its voxels
  long long goff, hoff;        // offsets of its G' and H
};

struct Dev {  // what the kernels read
  const Prob *prob;
  const int *vox_prob;
  const long long *row_ptr;
  const int *pose_idx;
  const double *obs;  // AoS [K][10]
  const double *fix;  // AoS [M][10] or null
  const double *coe;
  int64_t M, K;
};

// ---- per voxel: the world-frame cluster sum over its observations (+ fix), eig, residual term, stats row; with
// VoxelLoss the residual term coe rho(lambda_0) and coe w in the stats row (voxel_eig_kernel's rule) ----
template <bool STORE, typename Loss>
__global__ void __launch_bounds__(256) batch_stats_kernel(Dev d, const double *poses, const int *mask, int use_fix,
                                                          double *stats, double *res_v, Loss loss) {
  constexpr bool robust = std::is_same<Loss, VoxelLoss>::value;
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * 8;
  for (int64_t v = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); v < d.M; v += nw) {
    const int b = d.vox_prob[v];
    if (!mask[b]) continue;
    const double *pz = poses + 12 * (size_t)d.prob[b].pose_base;
    const long long s0 = d.row_ptr[v];
    const int k = (int)(d.row_ptr[v + 1] - s0);  // <= BALM_BATCH_MAX_POSES (checked at registration)
    double acc[10];
#pragma unroll
    for (int c = 0; c < 10; c++) acc[c] = 0.0;
    if (lane < k) {
      const double *o = d.obs + (size_t)(s0 + lane) * 10;
      double r[9], p[3];
      load_pose(pz + 12 * d.pose_idx[s0 + lane], r, p);
      const WC w = world_cluster(o, r, p);
      acc[0] = w.p00; acc[1] = w.p01; acc[2] = w.p02; acc[3] = w.p11; acc[4] = w.p12;
      acc[5] = w.p22; acc[6] = w.v0;  acc[7] = w.v1;  acc[8] = w.v2;  acc[9] = w.n;
    }
#pragma unroll
    for (int c = 0; c < 10; c++) {
      acc[c] = warp_sum(acc[c]);
      if (use_fix && d.fix) acc[c] += d.fix[(size_t)v * 10 + c];
    }
    if (lane == 0) {
      const double inv = 1.0 / acc[9];
      const double vb0 = acc[6] * inv, vb1 = acc[7] * inv, vb2 = acc[8] * inv;
      double lam[3], u0[3], u1[3], u2[3];
      eig3_jacobi(acc[0] * inv - vb0 * vb0, acc[1] * inv - vb0 * vb1, acc[2] * inv - vb0 * vb2,
                  acc[3] * inv - vb1 * vb1, acc[4] * inv - vb1 * vb2, acc[5] * inv - vb2 * vb2, lam, u0, u1, u2);
      const double coe = d.coe[v];
      if constexpr (robust) {
        double rho, w;
        loss_rho(loss.kind, loss.scale, lam[0], &rho, &w);
        res_v[v] = coe * rho;
        if (loss.lam) { loss.lam[v] = lam[0]; loss.w[v] = w; }
        if (STORE) store_stats_row(stats + (size_t)v * BALM_STATS_STRIDE, vb0, vb1, vb2, u0, u1, u2, inv, coe * w, lam);
      } else {
        res_v[v] = coe * lam[0];
        if (STORE) store_stats_row(stats + (size_t)v * BALM_STATS_STRIDE, vb0, vb1, vb2, u0, u1, u2, inv, coe, lam);
      }
    }
  }
}

// ---- per problem: fixed-order sum of its voxels' residual terms ----
__global__ void __launch_bounds__(128) batch_residual_kernel(const Prob *prob, const int *mask, const double *res_v,
                                                             double *out) {
  __shared__ double red[4];
  const int b = blockIdx.x;
  if (!mask[b]) return;
  const Prob pr = prob[b];
  double s = 0.0;
  for (long long v = threadIdx.x; v < pr.nvox; v += 128) s += res_v[pr.vox_base + v];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) out[b] = (red[0] + red[1]) + (red[2] + red[3]);
}

// ---- the voxels of chunk c (of CHUNK voxels) of problem pr in ascending order, one warp, lane = problem-local pose:
// f(v, s) for every voxel v that the lane's pose observes, s its observation. slot_of: 32 ints of the warp's own ----
template <typename F>
__device__ __forceinline__ void chunk_walk(const Dev &d, const Prob &pr, int c, int *slot_of, F f) {
  const int lane = threadIdx.x & 31;
  const long long v0 = pr.vox_base + (long long)(c - pr.ochunk_base) * CHUNK;
  const long long v1 = v0 + CHUNK < pr.vox_base + pr.nvox ? v0 + CHUNK : pr.vox_base + pr.nvox;
  for (long long v = v0; v < v1; v++) {
    const long long s0 = d.row_ptr[v];
    const int k = (int)(d.row_ptr[v + 1] - s0);
    slot_of[lane] = -1;
    __syncwarp();
    if (lane < k) slot_of[d.pose_idx[s0 + lane]] = lane;  // pose_idx < np <= 32 (checked at registration)
    __syncwarp();
    const int slot = slot_of[lane];
    __syncwarp();
    if (slot >= 0) f(v, s0 + slot);
  }
}

// ---- per chunk of CHUNK voxels of one problem, one warp, lane = problem-local pose ----
__global__ void __launch_bounds__(128) batch_obs_kernel(Dev d, const double *poses, const int *mask,
                                                        const int *ochunk_prob, int n_ochunks, const double *stats,
                                                        double *G, double *opart) {
  __shared__ int slot_of[4][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = blockIdx.x * 4 + warp;
  if (c >= n_ochunks) return;
  const int b = ochunk_prob[c];
  if (!mask[b]) return;
  const Prob pr = d.prob[b];
  const bool active = lane < pr.np;
  double r[9], p[3];
  if (active) load_pose(poses + 12 * (size_t)(pr.pose_base + lane), r, p);
  double acc[27];
#pragma unroll
  for (int q = 0; q < 27; q++) acc[q] = 0.0;
  chunk_walk(d, pr, c, slot_of[warp], [&](long long v, long long s) {
    double o[10], st[BALM_SWEEP_WORDS];
    const double2 *o2 = reinterpret_cast<const double2 *>(d.obs + (size_t)s * 10);
    const double2 *st2 = reinterpret_cast<const double2 *>(stats + (size_t)v * BALM_STATS_STRIDE + BALM_SWEEP_OFF);
#pragma unroll
    for (int q = 0; q < 5; q++) {
      const double2 x = __ldg(o2 + q);
      o[2 * q] = x.x;
      o[2 * q + 1] = x.y;
    }
#pragma unroll
    for (int q = 0; q < BALM_SWEEP_WORDS / 2; q++) {
      const double2 x = __ldg(st2 + q);
      st[2 * q] = x.x;
      st[2 * q + 1] = x.y;
    }
    double *g0 = G + pr.goff + (size_t)(3 * (v - pr.vox_base)) * pr.ldp + 6 * lane;
    obs_terms<true>(o, r, p, st, acc, [&](const double (&gv)[3][6]) {
#pragma unroll
      for (int rr = 0; rr < 3; rr++) {
        double2 *qd = reinterpret_cast<double2 *>(g0 + (size_t)rr * pr.ldp);
#pragma unroll
        for (int h = 0; h < 3; h++) qd[h] = make_double2(gv[rr][2 * h], gv[rr][2 * h + 1]);
      }
    });
  });
  if (active) {
    double *pp = opart + (size_t)c * 27 * 32 + lane;
#pragma unroll
    for (int q = 0; q < 27; q++) pp[q * 32] = acc[q];
  }
}

// ---- per (problem, upper 64x64 tile, 768-row chunk): partial of A^T G with DMMA, 2 x 2 warps of 32 x 32 ----
// RPV rows per voxel, problem p's rows at G + goff_p / 3 * RPV (the layout of G', 3 rows per voxel, with RPV rows).
// A is G (XOR = 0: the Hessian's G'^T G') or G with every row replaced by its partner row ^ XOR (XOR = 4: the eight
// covariance rows c2 Q^T | c2 V^T of a voxel give Q V^T + V Q^T). ROWS is a multiple of 8, so a partner never
// straddles a chunk.
template <int RPV, int XOR>
__global__ void __launch_bounds__(128) batch_syrk_kernel(const Prob *prob, const int *mask, const int4 *items,
                                                         const double *G, double *spart) {
  __shared__ __align__(16) double sA[KB][LDS], sB[KB][LDS];
  const int4 it = items[blockIdx.x];  // (problem, tile row, tile column, row chunk)
  if (!mask[it.x]) return;
  const Prob pr = prob[it.x];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 1, wn = warp & 1, fr = lane >> 2, fk = lane & 3;
  const long long rows = RPV * pr.nvox, k_begin = (long long)it.w * ROWS;
  const long long k_end = k_begin + ROWS < rows ? k_begin + ROWS : rows;
  const double *G0 = G + (RPV == 3 ? pr.goff : pr.goff / 3 * RPV);
  const double *gA = G0 + it.y * TILE, *gB = G0 + it.z * TILE;
  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j][0] = acc[i][j][1] = 0.0;
  for (long long k0 = k_begin; k0 < k_end; k0 += KB) {
    for (int e = tid; e < KB * TILE / 2; e += 128) {
      const int rr = e / (TILE / 2), cc = (e % (TILE / 2)) * 2;
      const long long kr = k0 + rr;
      double2 va = make_double2(0.0, 0.0), vb = va;
      if (kr < k_end) {
        va = *reinterpret_cast<const double2 *>(gA + (size_t)(kr ^ XOR) * pr.ldp + cc);
        vb = *reinterpret_cast<const double2 *>(gB + (size_t)kr * pr.ldp + cc);
      }
      *reinterpret_cast<double2 *>(&sA[rr][cc]) = va;
      *reinterpret_cast<double2 *>(&sB[rr][cc]) = vb;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < KB; kk += 4) {
      double af[4], bf[4];
#pragma unroll
      for (int i = 0; i < 4; i++) af[i] = sA[kk + fk][wm * 32 + i * 8 + fr];
#pragma unroll
      for (int j = 0; j < 4; j++) bf[j] = sB[kk + fk][wn * 32 + j * 8 + fr];
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) dmma_8x8x4(acc[i][j][0], acc[i][j][1], af[i], bf[j]);
    }
    __syncthreads();
  }
  double *out = spart + (size_t)blockIdx.x * TILE * TILE;
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int row = wm * 32 + i * 8 + fr, col = wn * 32 + j * 8 + 2 * fk;
      *reinterpret_cast<double2 *>(out + row * TILE + col) = make_double2(acc[i][j][0], acc[i][j][1]);
    }
}

// ---- per (problem, 64-column block): H = -sum (NEG) or +sum over row chunks of the SYRK partials, then + blockdiag;
// the diagonal blocks are the chunk-ordered sums of the problem's per-chunk partials (W words per pose, the block's
// upper triangle row-major from word OFF), and with GRAD words 0..5 are the gradient, written to g.
// range[p] = (first SYRK item, row chunks) of problem p. Element (i, j) and (j, i) are computed from the same upper
// partial, so H is exactly symmetric. The Hessian is <27, 6, true, true>, Rcov_raw <21, 0, false, false>. ----
template <int W, int OFF, bool NEG, bool GRAD>
__global__ void __launch_bounds__(256) batch_assemble_kernel(const Prob *prob, const int *mask, const int2 *range,
                                                             const double *part, const double *spart, double *H,
                                                             double *g) {
  __shared__ double accs[W][32];
  const int b = blockIdx.x;
  if (!mask[b]) return;
  const Prob pr = prob[b];
  const int n = pr.n, nt = pr.ldp / TILE;
  if (blockIdx.y * TILE >= n) return;
  const int2 ir = range[b];
  for (int e = threadIdx.x; e < W * pr.np; e += 256) {
    const int q = e / pr.np, i = e % pr.np;
    double s = 0.0;
    for (int c = 0; c < pr.n_ochunks; c++) s += part[((size_t)(pr.ochunk_base + c) * W + q) * 32 + i];
    accs[q][i] = s;
  }
  __syncthreads();
  double *Hb = H + pr.hoff;
  const int j_end = (blockIdx.y + 1) * TILE < n ? (blockIdx.y + 1) * TILE : n;
  for (int j = blockIdx.y * TILE; j < j_end; j++) {
    for (int i = threadIdx.x; i < n; i += 256) {
      const int rr = i < j ? i : j, cc = i < j ? j : i;
      const int bi = rr / TILE, bj = cc / TILE;
      const int t = bi * nt - bi * (bi - 1) / 2 + (bj - bi);
      const double *src = spart + (size_t)(ir.x + t * ir.y) * TILE * TILE + (rr % TILE) * TILE + cc % TILE;
      double s = 0.0;
      for (int c = 0; c < ir.y; c++) s += src[(size_t)c * TILE * TILE];
      double h = NEG ? -s : s;
      const int pi = rr / 6;
      if (pi == cc / 6) {
        const int r6 = rr % 6, c6 = cc % 6;
        h += accs[OFF + r6 * 6 - r6 * (r6 - 1) / 2 + (c6 - r6)][pi];
      }
      Hb[(size_t)j * n + i] = h;
    }
  }
  if (GRAD && blockIdx.y == 0)
    for (int i = threadIdx.x; i < n; i += 256) g[6 * (size_t)pr.pose_base + i] = accs[i % 6][i / 6];
}

// ---- damped solve, one CTA per problem, the packed lower triangle of H + uD in shared memory (tri_idx, ldl_factor:
// internal.cuh) ----
// w <-(L D L^T)^-1 w with the factors in A (unit-lower L below the diagonal, D on it)
__device__ void ldl_apply(const double *A, int n, double *w) {
  for (int k = 0; k < n; k++) {  // L y = w
    const double wk = w[k];
    for (int i = k + 1 + threadIdx.x; i < n; i += SOLVE_THREADS) w[i] -= A[tri_idx(i, k, n)] * wk;
    __syncthreads();
  }
  for (int i = threadIdx.x; i < n; i += SOLVE_THREADS) w[i] /= A[tri_idx(i, i, n)];
  __syncthreads();
  for (int k = n - 1; k >= 0; k--) {  // L^T x = y
    const double xk = w[k];
    for (int i = threadIdx.x; i < k; i += SOLVE_THREADS) w[i] -= A[tri_idx(k, i, n)] * xk;
    __syncthreads();
  }
}

// componentwise backward error of x for (H + uD) x = -g, computed from H (Oettli-Prager, as solve_residual_kernel):
// rres = b - A x; returns whether it exceeds OMEGA_TOL anywhere
__device__ bool backward_error(const double *Hb, const double *gb, int n, double u, const double *x, double *rres) {
  bool bad = false;
  const int i = threadIdx.x;
  if (i < n) {
    double s = 0.0, sa = 0.0;
    for (int j = 0; j < n; j++) {  // H exactly symmetric: row i = column i
      double h = Hb[(size_t)j * n + i];
      if (j == i) h += u * h;
      const double t = h * x[j];
      s += t;
      sa += fabs(t);
    }
    const double b = -gb[i], r = b - s, den = sa + fabs(b);
    rres[i] = r;
    const double om = den > 0.0 ? fabs(r) / den : 0.0;
    bad = !(om <= OMEGA_TOL);
  }
  return __syncthreads_or(bad) != 0;
}

// q1 = 0.5 dx.(u D dx - g)  (bavoxel.hpp:1127), block-wide, fixed order
__device__ double damped_q1(const double *x, const double *D, const double *gb, int n, double u, double *red) {
  const int tid = threadIdx.x;
  double part = tid < n ? x[tid] * (u * D[tid] * x[tid] - gb[tid]) : 0.0;
  part = warp_sum(part);
  if ((tid & 31) == 0) red[tid >> 5] = part;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int q = 0; q < SOLVE_THREADS / 32; q++) s += red[q];
  __syncthreads();
  return 0.5 * s;
}

__global__ void __launch_bounds__(SOLVE_THREADS) batch_solve_kernel(const Prob *prob, const int *active, const double *H,
                                                                    const double *g, const double *uvec,
                                                                    const double *poses, double *trial, double *q1_out,
                                                                    int *notpd_out) {
  extern __shared__ double sm[];
  __shared__ double red[SOLVE_THREADS / 32];
  const int b = blockIdx.x;
  if (!active[b]) return;
  const Prob pr = prob[b];
  const int n = pr.n, tid = threadIdx.x;
  double *A = sm, *D = A + n * (n + 1) / 2, *x = D + MAXN, *w = x + MAXN, *rres = w + MAXN, *col = rres + MAXN;
  const double *Hb = H + pr.hoff, *gb = g + 6 * (size_t)pr.pose_base;
  const double u = uvec[b];
  for (int e = tid; e < n * n; e += SOLVE_THREADS) {  // A = H + u diag(H), as damp_copy_kernel
    const int j = e / n, i = e % n;
    if (i < j) continue;
    double h = Hb[e];
    if (i == j) {
      D[i] = h;
      h += u * h;
    }
    A[tri_idx(i, j, n)] = h;
  }
  for (int i = tid; i < n; i += SOLVE_THREADS) x[i] = -gb[i];
  __syncthreads();
  // a zero / tiny / non-finite pivot makes the step not_pd
  const bool pivot_bad = ldl_factor<SOLVE_THREADS>(A, n, col);
  int not_pd = pivot_bad ? 1 : 0;
  double q1 = 0.0;
  if (!pivot_bad) {
    ldl_apply(A, n, x);
    bool omega_bad = backward_error(Hb, gb, n, u, x, rres);
    q1 = damped_q1(x, D, gb, n, u, red);
    not_pd = isfinite(q1) ? 0 : 1;
    if (!not_pd && omega_bad) {  // fp64 iterative refinement with the same factors (refine_solution)
      for (int round = 0; round < 3 && omega_bad; round++) {
        for (int i = tid; i < n; i += SOLVE_THREADS) w[i] = rres[i];
        __syncthreads();
        ldl_apply(A, n, w);
        for (int i = tid; i < n; i += SOLVE_THREADS) x[i] += w[i];
        __syncthreads();
        omega_bad = backward_error(Hb, gb, n, u, x, rres);
      }
      q1 = damped_q1(x, D, gb, n, u, red);
      if (omega_bad || !isfinite(q1)) not_pd = 1;
    }
  } else {
    for (int i = tid; i < n; i += SOLVE_THREADS) x[i] = 0.0;
    __syncthreads();
  }
  if (tid < pr.np) {
    const size_t o = 12 * (size_t)(pr.pose_base + tid);
    pose_update_one(poses + o, x + 6 * tid, trial + o);
  }
  if (tid == 0) {
    q1_out[b] = q1;
    notpd_out[b] = not_pd;
  }
}

struct LmArgs {
  const Prob *prob;
  int B, it, max_iter, force_hess;
  double rel_tol;
  const double *r_eval, *r2, *q1;
  const int *notpd;
  double *r1, *u, *v;
  int *active, *calc, *evalm, *n_iters, *n_active;
  double *poses;
  const double *trial;
  balm_trace *trace;  // [B][max_iter]
};

// ---- LM control, one thread per problem: the host loop of balm_damping_iter (bavoxel.hpp:1129-1155) ----
__global__ void batch_lm_kernel(LmArgs a) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.B || !a.active[b]) return;
  const int calc = a.calc[b];
  const double r1 = calc ? a.r_eval[b] : a.r1[b];
  double u = a.u[b], v = a.v[b];
  balm_trace t;
  bool stop;
  const bool accepted = lm_rule(r1, a.r2[b], a.q1[b], a.notpd[b], calc, a.rel_tol, &u, &v, &t, &stop);
  if (accepted) {
    const Prob pr = a.prob[b];
    for (int e = 0; e < 12 * pr.np; e++) a.poses[12 * (size_t)pr.pose_base + e] = a.trial[12 * (size_t)pr.pose_base + e];
  }
  const int next_calc = accepted ? 1 : a.force_hess;
  a.trace[(size_t)b * a.max_iter + a.it] = t;
  a.n_iters[b] = a.it + 1;
  a.r1[b] = r1;
  a.u[b] = u;
  a.v[b] = v;
  a.calc[b] = next_calc;
  stop = stop || a.it + 1 >= a.max_iter;
  a.evalm[b] = stop ? 0 : next_calc;
  if (stop) a.active[b] = 0;
  else atomicAdd(a.n_active, 1);
}

// ---- gauge step per pose, pose 0 of each problem read from a snapshot ----
__global__ void batch_gauge_kernel(const Prob *prob, const int *pose_prob, const int *status, int P, double *poses,
                                   const double *snapshot, int mode) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P) return;
  const int b = pose_prob[j];
  if (status[b] != BALM_OK) return;
  const int base = prob[b].pose_base;
  gauge_one(poses + 12 * (size_t)j, snapshot + 12 * (size_t)base, mode == 1 && j == base);
}

// ---- registration: per voxel, the CSR invariants and the per-pose voxel counts ----
__global__ void batch_check_kernel(Dev d, int *bad, int *planes) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= d.M) return;
  const Prob pr = d.prob[d.vox_prob[v]];
  const long long s0 = d.row_ptr[v], s1 = d.row_ptr[v + 1];
  if (s0 < 0 || s1 < s0 || s1 > d.K || s1 - s0 > pr.np) { atomicOr(bad, 1); return; }
  int prev = -1;
  for (long long s = s0; s < s1; s++) {
    const int p = d.pose_idx[s];
    if (p <= prev || p >= pr.np) { atomicOr(bad, 1); return; }
    prev = p;
  }
  for (long long s = s0; s < s1; s++) atomicAdd(&planes[pr.pose_base + d.pose_idx[s]], 1);
}

__global__ void batch_init_kernel(int B, const int *status, int max_iter, double u0, double v0, double *u, double *v,
                                  int *active, int *calc, int *evalm, int *n_iters) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int on = status[b] == BALM_OK && max_iter > 0;
  u[b] = u0; v[b] = v0; active[b] = on; calc[b] = 1; evalm[b] = on; n_iters[b] = 0;
}

__global__ void fill_kernel(int *p, int n, int val) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = val;
}

// ---------------- pose covariance (balm_batch_pose_covariance; the mathematics is covariance.cu's) ----------------
// Per lane of the rows kernel, in shared memory: its CovTerms (padded by one double: a stride of 115 doubles leaves at
// most two lanes on a bank) and its 9 x 9 c_cov. In registers they would not fit next to E c.
constexpr int COV_TSTRIDE = (int)(sizeof(CovTerms) / sizeof(double)) + 1;
constexpr int COV_SMEM = 32 * (COV_TSTRIDE + 81) * (int)sizeof(double);

// ---- per voxel, a CTA of one warp, lane = observation (k <= 32): Wz = sum_j Z_j c_j Z_j^T (fixed-order shuffle reduction),
// then the voxel's eight rows c2 Q^T | c2 V^T into the problem's row buffer and every observation's c2^2 D block ----
__global__ void __launch_bounds__(32) batch_cov_rows_kernel(Dev d, const double *poses, const double *stats,
                                                            const double *ccov, double pn2, double *rows, double *Dobs) {
  extern __shared__ double cov_sm[];
  __shared__ double Wz[4][4];  // the voxel's, the same in every lane
  const int lane = threadIdx.x;
  CovTerms &t = *reinterpret_cast<CovTerms *>(cov_sm + lane * COV_TSTRIDE);
  double *C = cov_sm + 32 * COV_TSTRIDE + lane * 81;
  const int64_t v = blockIdx.x;
  const Prob pr = d.prob[d.vox_prob[v]];
  const long long s0 = d.row_ptr[v];
  const int k = (int)(d.row_ptr[v + 1] - s0);
  const long long s = s0 + lane;
  const double *st = stats + (size_t)v * BALM_STATS_STRIDE;
  double acc[10];
#pragma unroll
  for (int e = 0; e < 10; e++) acc[e] = 0.0;
  const int p = lane < k ? d.pose_idx[s] : 0;
  if (lane < k) {
    double o[10];
#pragma unroll
    for (int c = 0; c < 10; c++) o[c] = d.obs[(size_t)s * 10 + c];
    if (ccov) {
      for (int e = 0; e < 81; e++) C[e] = ccov[(size_t)s * 81 + e];
    } else {
      cluster_cov_iso(o, pn2, C);
    }
    cov_terms(o, poses + 12 * (size_t)(pr.pose_base + p), st, t);
    cov_wz_add(t, C, acc);
  }
#pragma unroll
  for (int e = 0; e < 10; e++) acc[e] = warp_sum(acc[e]);
  if (lane == 0) {
    int q = 0;
    for (int i = 0; i < 4; i++)
      for (int j = i; j < 4; j++) { Wz[i][j] = acc[q]; Wz[j][i] = acc[q]; q++; }
  }
  __syncwarp();
  if (lane < k) {
    const double c2 = st[16] * 2.0 * st[12];  // coe * 2 / NN
    double *g = rows + pr.goff / 3 * 8 + (size_t)(8 * (v - pr.vox_base)) * pr.ldp + 6 * p;
    cov_obs_rows(t, C, Wz, c2, g, pr.ldp, Dobs + (size_t)s * 21);
  }
}

// ---- per chunk of CHUNK voxels of one problem, one warp, lane = problem-local pose: the sum of the pose's c2^2 D
// blocks over the chunk's voxels in ascending order ----
__global__ void __launch_bounds__(128) batch_cov_diag_kernel(Dev d, const int *ochunk_prob, int n_ochunks,
                                                             const double *Dobs, double *dpart) {
  __shared__ int slot_of[4][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = blockIdx.x * 4 + warp;
  if (c >= n_ochunks) return;
  const Prob pr = d.prob[ochunk_prob[c]];
  double acc[21];
#pragma unroll
  for (int q = 0; q < 21; q++) acc[q] = 0.0;
  chunk_walk(d, pr, c, slot_of[warp], [&](long long, long long s) {
    const double *dd = Dobs + (size_t)s * 21;
#pragma unroll
    for (int q = 0; q < 21; q++) acc[q] += dd[q];
  });
  if (lane < pr.np) {
    double *pp = dpart + (size_t)c * 21 * 32 + lane;
#pragma unroll
    for (int q = 0; q < 21; q++) pp[q * 32] = acc[q];
  }
}

// ---- per problem, one CTA: undamped LDL^T of H in shared memory, the singularity test of cov_factor, then
// Rcov = H^-1 R H^-1 as two sweeps over n right-hand sides, thread t owning right-hand side t (R and the result in
// global memory, n^2 doubles being too many for shared memory; every access below is coalesced across threads).
// The result is made exactly symmetric by copying its upper triangle to the lower one. ----
// x <- (L D L^T)^-1 x for the vector x[i * n] (i = 0 .. n-1), the factors in A; one thread
__device__ __forceinline__ void ldl_apply_strided(const double *A, int n, double *x) {
  for (int i = 0; i < n; i++) {  // L y = x
    double s = x[(size_t)i * n];
    for (int k = 0; k < i; k++) s -= A[tri_idx(i, k, n)] * x[(size_t)k * n];
    x[(size_t)i * n] = s;
  }
  for (int i = n - 1; i >= 0; i--) {  // L^T x = D^-1 y
    double s = x[(size_t)i * n] / A[tri_idx(i, i, n)];
    for (int k = n - 1; k > i; k--) s -= A[tri_idx(k, i, n)] * x[(size_t)k * n];
    x[(size_t)i * n] = s;
  }
}

__global__ void __launch_bounds__(SOLVE_THREADS) batch_cov_solve_kernel(const Prob *prob, const double *H,
                                                                        const double *Rraw, double *Rcov, int *status) {
  extern __shared__ double sm[];
  __shared__ int singular;
  const int b = blockIdx.x;
  const Prob pr = prob[b];
  const int n = pr.n, tid = threadIdx.x;
  double *A = sm, *col = A + n * (n + 1) / 2;
  const double *Hb = H + pr.hoff, *Rb = Rraw + pr.hoff;
  double *X = Rcov + pr.hoff;
  for (int e = tid; e < n * n; e += SOLVE_THREADS) {
    const int j = e / n, i = e % n;
    if (i >= j) A[tri_idx(i, j, n)] = Hb[e];
  }
  __syncthreads();
  const bool pivot_bad = ldl_factor<SOLVE_THREADS>(A, n, col);
  if (tid == 0) {
    // a singular H (free gauge) pivots at rounding level relative to the others rather than at zero
    double dmin = 1e300, dmax = 0.0;
    for (int i = 0; i < n && !pivot_bad; i++) {
      const double dd = fabs(A[tri_idx(i, i, n)]);
      dmin = fmin(dmin, dd);
      dmax = fmax(dmax, dd);
    }
    singular = pivot_bad || !(dmin > 1e-11 * dmax);
    status[b] = singular ? BALM_ERR_NOT_PD : BALM_OK;
  }
  __syncthreads();
  if (singular) {
    for (int e = tid; e < n * n; e += SOLVE_THREADS) X[e] = 0.0;
    return;
  }
  // X[t + i n] = (H^-1 R)(i, t): right-hand side t is column t of R, read as row t (R is exactly symmetric)
  if (tid < n) {
    for (int i = 0; i < n; i++) X[tid + (size_t)i * n] = Rb[tid + (size_t)i * n];
    ldl_apply_strided(A, n, X + tid);
  }
  __syncthreads();
  // transpose in place: X[t + i n] = (H^-1 R)(t, i), so right-hand side t of the second sweep is row t of H^-1 R
  for (int e = tid; e < n * n; e += SOLVE_THREADS) {
    const int i = e % n, j = e / n;
    if (i < j) {
      const double a = X[e], c = X[j + (size_t)i * n];
      X[e] = c;
      X[j + (size_t)i * n] = a;
    }
  }
  __syncthreads();
  // X[t + i n] = (H^-1 (H^-1 R)^T)(i, t) = (H^-1 R H^-1)(i, t): column-major, X holds the transpose of the result,
  // which is the result up to rounding; its upper triangle is kept
  if (tid < n) ldl_apply_strided(A, n, X + tid);
  __syncthreads();
  for (int e = tid; e < n * n; e += SOLVE_THREADS) {
    const int i = e % n, j = e / n;
    if (i > j) X[e] = X[j + (size_t)i * n];
  }
}

}  // namespace

// One registration: the problems, their voxels and every workspace sized for them. A new registration is built and
// checked completely before it replaces the previous one.
struct BatchReg {
  int B = 0, P = 0, n_ochunks = 0, n_items = 0;
  int64_t M = 0, K = 0;
  std::vector<Prob> hprob;
  std::vector<int> min_planes;  // per problem: the fewest voxels observing one of its poses
  size_t H_size = 0, G_size = 0;
  Prob *prob = nullptr;
  int *vox_prob = nullptr, *pose_prob = nullptr, *ochunk_prob = nullptr;
  int4 *items = nullptr;       // the Hessian SYRK's (syrk_items)
  int2 *item_range = nullptr;
  long long *row_ptr = nullptr;
  int *pose_idx = nullptr;
  double *obs = nullptr, *fix = nullptr, *coe = nullptr;
  unsigned long long *key = nullptr;  // [M] octree keys and layers when the voxels were cut from scans, else null
  int *layer = nullptr;
  balm_assoc_opts assoc{};            // with keys: the options of that cut (balm_batch_append_scan judges with them)
  double *G = nullptr, *stats = nullptr, *res_v = nullptr, *opart = nullptr, *spart = nullptr, *H = nullptr, *g = nullptr;
  double *poses = nullptr, *trial = nullptr;
  double *r_eval = nullptr, *r2 = nullptr, *r1 = nullptr, *q1 = nullptr, *u = nullptr, *v = nullptr;
  int *ints = nullptr;  // [7][B]: notpd, active, calc, evalm, n_iters, status, ones; then n_active
  int *notpd() { return ints; }
  int *active() { return ints + B; }
  int *calc() { return ints + 2 * B; }
  int *evalm() { return ints + 3 * B; }
  int *n_iters() { return ints + 4 * B; }
  int *status() { return ints + 5 * B; }
  int *ones() { return ints + 6 * B; }
  int *n_active() { return ints + 7 * B; }
  Dev dev() const { return Dev{prob, vox_prob, row_ptr, pose_idx, obs, fix, coe, M, K}; }
  ~BatchReg() {
    void *ptrs[] = {prob, vox_prob, pose_prob, ochunk_prob, items, item_range, row_ptr, pose_idx, obs, fix, coe, key, layer, G,
                    stats, res_v, opart, spart, H, g, poses, trial, r_eval, r2, r1, q1, u, v, ints};
    for (void *p : ptrs) cudaFree(p);
  }
};

struct balm_batch {
  int device = 0, sm_count = 132;
  cudaStream_t stream = nullptr;
  BatchReg *reg = nullptr;
  WindowState *win = nullptr;  // balm_batch_window_* maps (independent of the registration)
  int *h_count = nullptr;  // pinned: problems still active after an iteration
  int vloss_kind = BALM_LOSS_TRIVIAL;  // balm_batch_set_voxel_loss: every voxel's loss (independent of the registration)
  double vloss_scale = 1.0;
};

namespace {

template <typename T>
int upload(T **p, const T *src, size_t count, cudaStream_t st) {
  TRY(dev_alloc(p, count));
  if (count) CUDA_TRY(cudaMemcpyAsync(*p, src, sizeof(T) * count, cudaMemcpyHostToDevice, st));
  return BALM_OK;
}
int invalid(const std::string &msg) {
  balm_set_error(msg);
  return BALM_ERR_INVALID;
}

// The problem table of a registration: n_problems >= 1, pose_ptr[0] = 0 and 1 .. BALM_BATCH_MAX_POSES poses each.
int check_pose_ptr(const char *who, int n_problems, const int64_t *pose_ptr) {
  const std::string w = who;
  if (n_problems < 1) return invalid(w + ": n_problems must be >= 1");
  if (pose_ptr[0] != 0) return invalid(w + ": pose_ptr[0] must be 0");
  for (int b = 0; b < n_problems; b++) {
    const int64_t np = pose_ptr[b + 1] - pose_ptr[b];
    if (np < 1 || np > BALM_BATCH_MAX_POSES)
      return invalid(w + ": every problem needs 1 .. BALM_BATCH_MAX_POSES poses (pose_ptr ascending)");
  }
  return BALM_OK;
}

// The SYRK items of every problem for rpv rows per voxel (3: G', 8: the covariance rows): per problem its upper tiles x
// chunks of ROWS rows, item (problem, tile row, tile column, row chunk); range[p] = (first item, row chunks) of problem p.
void syrk_items(const std::vector<Prob> &hprob, int rpv, std::vector<int4> &items, std::vector<int2> &range) {
  items.clear();
  range.resize(hprob.size());
  for (size_t b = 0; b < hprob.size(); b++) {
    const Prob &p = hprob[b];
    const int nt = p.ldp / TILE, nrc = (int)((rpv * p.nvox + ROWS - 1) / ROWS);
    range[b] = make_int2((int)items.size(), nrc);
    for (int ti = 0; ti < nt; ti++)
      for (int tj = ti; tj < nt; tj++)
        for (int c = 0; c < nrc; c++) items.push_back(make_int4((int)b, ti, tj, c));
  }
}

// batch_stats_kernel at poses for every problem with mask[b] != 0 under the batch's voxel loss: the residual terms, and
// with stats non-null the stats rows; lam / w (both or neither; need stats): the per-voxel readout of
// balm_batch_voxel_residuals.
void enqueue_stats(balm_batch *bt, BatchReg *r, const double *poses, const int *mask, bool use_fix, double *stats,
                   double *lam = nullptr, double *w = nullptr) {
  if (r->M == 0) return;
  const int blocks = (int)std::min<int64_t>((r->M + 7) / 8, (int64_t)bt->sm_count * 8);
  const int fx = use_fix ? 1 : 0;
  // without a loss (and outside the readout) the NoLoss kernels, the only ones that run
  if (bt->vloss_kind != BALM_LOSS_TRIVIAL || lam) {
    const VoxelLoss loss{bt->vloss_kind, bt->vloss_scale, lam, w};
    if (stats) batch_stats_kernel<true><<<blocks, 256, 0, bt->stream>>>(r->dev(), poses, mask, fx, stats, r->res_v, loss);
    else batch_stats_kernel<false><<<blocks, 256, 0, bt->stream>>>(r->dev(), poses, mask, fx, nullptr, r->res_v, loss);
  } else if (stats) {
    batch_stats_kernel<true><<<blocks, 256, 0, bt->stream>>>(r->dev(), poses, mask, fx, stats, r->res_v, NoLoss{});
  } else {
    batch_stats_kernel<false><<<blocks, 256, 0, bt->stream>>>(r->dev(), poses, mask, fx, nullptr, r->res_v, NoLoss{});
  }
}

// The evaluation of every problem with mask[b] != 0 at r->poses: r_eval, H, g.
int enqueue_eval(balm_batch *bt, BatchReg *r, const int *mask, bool use_fix) {
  cudaStream_t st = bt->stream;
  enqueue_stats(bt, r, r->poses, mask, use_fix, r->stats);
  batch_residual_kernel<<<r->B, 128, 0, st>>>(r->prob, mask, r->res_v, r->r_eval);
  if (r->n_ochunks > 0)
    batch_obs_kernel<<<(r->n_ochunks + 3) / 4, 128, 0, st>>>(r->dev(), r->poses, mask, r->ochunk_prob, r->n_ochunks,
                                                             r->stats, r->G, r->opart);
  if (r->n_items > 0) batch_syrk_kernel<3, 0><<<r->n_items, 128, 0, st>>>(r->prob, mask, r->items, r->G, r->spart);
  batch_assemble_kernel<27, 6, true, true><<<dim3(r->B, MAXN / TILE), 256, 0, st>>>(r->prob, mask, r->item_range, r->opart,
                                                                                    r->spart, r->H, r->g);
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

// The residual (fix clusters included, as evaluate_only_residual) at the trial poses of every active problem: r2.
int enqueue_trial_residual(balm_batch *bt, BatchReg *r) {
  enqueue_stats(bt, r, r->trial, r->active(), true, nullptr);
  batch_residual_kernel<<<r->B, 128, 0, bt->stream>>>(r->prob, r->active(), r->res_v, r->r2);
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

}  // namespace

extern "C" int balm_batch_create(balm_batch **out, int device) {
  if (!out) return invalid("balm_batch_create: bad arguments");
  int ndev = 0;
  CUDA_TRY(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) { balm_set_error("balm_batch_create: no such CUDA device"); return BALM_ERR_CUDA; }
  CUDA_TRY(cudaSetDevice(device));
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  CUDA_TRY(cudaFuncSetAttribute(batch_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SOLVE_SMEM));
  CUDA_TRY(cudaFuncSetAttribute(batch_cov_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SOLVE_SMEM));
  CUDA_TRY(cudaFuncSetAttribute(batch_cov_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, COV_SMEM));
  balm_batch *b = new balm_batch();
  b->device = device;
  b->sm_count = prop.multiProcessorCount;
  if (cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaMallocHost((void **)&b->h_count, sizeof(int)) != cudaSuccess) {
    balm_set_error("balm_batch_create: stream / pinned buffer allocation failed");
    if (b->stream) cudaStreamDestroy(b->stream);
    delete b;
    return BALM_ERR_CUDA;
  }
  *out = b;
  return BALM_OK;
}

extern "C" int balm_batch_destroy(balm_batch *b) {
  if (!b) return BALM_OK;
  cudaSetDevice(b->device);
  cudaStreamSynchronize(b->stream);
  delete b->reg;
  window_free(b->win);
  cudaFreeHost(b->h_count);
  cudaStreamDestroy(b->stream);
  delete b;
  return BALM_OK;
}

// Host-side layout of a registration of M = voxel_ptr[B] voxels and K observations: problems, observation-sweep chunks,
// SYRK items, voxel -> problem, pose -> problem.
static int reg_layout(balm_batch *bt, BatchReg *r, int B, const int64_t *pose_ptr, const int64_t *voxel_ptr, int64_t K) {
  cudaStream_t st = bt->stream;
  r->B = B;
  r->P = (int)pose_ptr[B];
  r->M = voxel_ptr[B];
  r->K = K;
  std::vector<int> vox_prob((size_t)r->M), pose_prob((size_t)r->P), ochunk_prob;
  r->hprob.resize(B);
  long long goff = 0, hoff = 0;
  for (int b = 0; b < B; b++) {
    Prob &p = r->hprob[b];
    p.pose_base = (int)pose_ptr[b];
    p.np = (int)(pose_ptr[b + 1] - pose_ptr[b]);
    p.n = 6 * p.np;
    p.ldp = (p.n + TILE - 1) / TILE * TILE;
    p.vox_base = voxel_ptr[b];
    p.nvox = voxel_ptr[b + 1] - voxel_ptr[b];
    p.ochunk_base = (int)ochunk_prob.size();
    p.n_ochunks = (int)((p.nvox + CHUNK - 1) / CHUNK);
    ochunk_prob.insert(ochunk_prob.end(), (size_t)p.n_ochunks, b);
    p.goff = goff;
    p.hoff = hoff;
    goff += 3 * p.nvox * p.ldp;
    hoff += (long long)p.n * p.n;
    std::fill(vox_prob.begin() + p.vox_base, vox_prob.begin() + p.vox_base + p.nvox, b);
    std::fill(pose_prob.begin() + p.pose_base, pose_prob.begin() + p.pose_base + p.np, b);
  }
  std::vector<int4> items;
  std::vector<int2> range;
  syrk_items(r->hprob, 3, items, range);
  r->n_ochunks = (int)ochunk_prob.size();
  r->n_items = (int)items.size();
  r->G_size = (size_t)goff;
  r->H_size = (size_t)hoff;
  TRY(upload(&r->prob, r->hprob.data(), (size_t)B, st));
  TRY(upload(&r->vox_prob, vox_prob.data(), vox_prob.size(), st));
  TRY(upload(&r->pose_prob, pose_prob.data(), pose_prob.size(), st));
  TRY(upload(&r->ochunk_prob, ochunk_prob.data(), ochunk_prob.size(), st));
  TRY(upload(&r->items, items.data(), items.size(), st));
  TRY(upload(&r->item_range, range.data(), range.size(), st));
  return BALM_OK;
}

// With row_ptr / pose_idx / obs / coe (/ fix) in place: the per-voxel checks on the device, the per-pose plane counts
// of the precheck, and the workspaces.
static int reg_finish(balm_batch *bt, BatchReg *r) {
  cudaStream_t st = bt->stream;
  const int B = r->B;
  TRY(dev_alloc(&r->ints, 7 * (size_t)B + 1));
  int *d_planes = nullptr;
  TRY(dev_alloc(&d_planes, (size_t)r->P));
  CUDA_TRY(cudaMemsetAsync(d_planes, 0, sizeof(int) * r->P, st));
  CUDA_TRY(cudaMemsetAsync(r->n_active(), 0, sizeof(int), st));  // serves as the check's error flag here
  if (r->M > 0) batch_check_kernel<<<(unsigned)((r->M + 127) / 128), 128, 0, st>>>(r->dev(), r->n_active(), d_planes);
  std::vector<int> planes((size_t)r->P);
  int bad = 0;
  CUDA_TRY(cudaMemcpyAsync(&bad, r->n_active(), sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(planes.data(), d_planes, sizeof(int) * r->P, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  cudaFree(d_planes);
  if (bad) return invalid("balm_batch_set_voxels: inside a voxel, pose_idx must be ascending and in [0, N_p) of its problem");
  r->min_planes.resize(B);
  for (int b = 0; b < B; b++) {
    const Prob &p = r->hprob[b];
    r->min_planes[b] = *std::min_element(planes.begin() + p.pose_base, planes.begin() + p.pose_base + p.np);
  }
  // workspaces
  TRY(dev_alloc(&r->G, r->G_size));
  CUDA_TRY(cudaMemsetAsync(r->G, 0, sizeof(double) * r->G_size, st));  // columns of non-observing poses stay zero
  TRY(dev_alloc(&r->stats, (size_t)r->M * BALM_STATS_STRIDE));
  TRY(dev_alloc(&r->res_v, (size_t)r->M));
  TRY(dev_alloc(&r->opart, (size_t)r->n_ochunks * 27 * 32));
  TRY(dev_alloc(&r->spart, (size_t)r->n_items * TILE * TILE));
  TRY(dev_alloc(&r->H, r->H_size));
  TRY(dev_alloc(&r->g, 6 * (size_t)r->P));
  TRY(dev_alloc(&r->poses, 12 * (size_t)r->P));
  TRY(dev_alloc(&r->trial, 12 * (size_t)r->P));
  double **scal[] = {&r->r_eval, &r->r2, &r->r1, &r->q1, &r->u, &r->v};
  for (double **p : scal) TRY(dev_alloc(p, (size_t)B));
  fill_kernel<<<(B + 127) / 128, 128, 0, st>>>(r->ones(), B, 1);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaStreamSynchronize(st));
  return BALM_OK;
}

static int build_registration(balm_batch *bt, BatchReg *r, int B, const int64_t *pose_ptr, const int64_t *voxel_ptr,
                              const int64_t *row_ptr, const int32_t *pose_idx, const double *obs10,
                              const double *fix10, const double *coe) {
  cudaStream_t st = bt->stream;
  TRY(reg_layout(bt, r, B, pose_ptr, voxel_ptr, row_ptr[voxel_ptr[B]]));
  TRY(upload(&r->row_ptr, reinterpret_cast<const long long *>(row_ptr), (size_t)r->M + 1, st));
  TRY(upload(&r->pose_idx, pose_idx, (size_t)r->K, st));
  TRY(upload(&r->obs, obs10, (size_t)r->K * 10, st));
  if (fix10) TRY(upload(&r->fix, fix10, (size_t)r->M * 10, st));
  TRY(upload(&r->coe, coe, (size_t)r->M, st));
  return reg_finish(bt, r);
}

// Replaces the registration with r once r is complete; otherwise deletes r and keeps the previous one.
static int install(balm_batch *bt, BatchReg *r, int rc) {
  if (rc != BALM_OK) {
    cudaStreamSynchronize(bt->stream);
    delete r;
    return rc;
  }
  delete bt->reg;
  bt->reg = r;
  return BALM_OK;
}

extern "C" int balm_batch_set_voxels(balm_batch *bt, int n_problems, const int64_t *pose_ptr, const int64_t *voxel_ptr,
                                     const int64_t *row_ptr, const int32_t *pose_idx, const double *obs10,
                                     const double *fix10, const double *coe) {
  if (!bt || !pose_ptr || !voxel_ptr || !row_ptr) return invalid("balm_batch_set_voxels: bad arguments");
  TRY(check_pose_ptr("balm_batch_set_voxels", n_problems, pose_ptr));
  if (voxel_ptr[0] != 0) return invalid("balm_batch_set_voxels: voxel_ptr[0] must be 0");
  for (int b = 0; b < n_problems; b++)
    if (voxel_ptr[b + 1] < voxel_ptr[b]) return invalid("balm_batch_set_voxels: voxel_ptr must be ascending");
  const int64_t M = voxel_ptr[n_problems];
  if (row_ptr[0] != 0) return invalid("balm_batch_set_voxels: row_ptr[0] must be 0");
  const int64_t K = row_ptr[M];
  if (K < 0 || (K > 0 && (!pose_idx || !obs10)) || (M > 0 && !coe)) return invalid("balm_batch_set_voxels: bad arguments");
  if (K >= ((int64_t)1 << 31) || pose_ptr[n_problems] >= ((int64_t)1 << 31)) {
    balm_set_error("balm_batch_set_voxels: more than 2^31 observations or poses");
    return BALM_ERR_UNSUPPORTED;
  }
  CUDA_TRY(cudaSetDevice(bt->device));
  CUDA_TRY(cudaStreamSynchronize(bt->stream));
  BatchReg *r = new BatchReg();
  return install(bt, r, build_registration(bt, r, n_problems, pose_ptr, voxel_ptr, row_ptr, pose_idx, obs10, fix10, coe));
}

extern "C" int balm_batch_cut_voxels(balm_batch *bt, int n_problems, const int64_t *pose_ptr, const int32_t *pose_scan,
                                     int n_scans, const int64_t *scan_ptr, const float *xyz, const double *poses12,
                                     const balm_assoc_opts *opts, int64_t *n_voxels_out, int64_t *n_obs_out) {
  if (!bt || !pose_ptr || !pose_scan || !scan_ptr || !poses12 || n_scans < 1)
    return invalid("balm_batch_cut_voxels: bad arguments");
  TRY(check_pose_ptr("balm_batch_cut_voxels", n_problems, pose_ptr));
  if (scan_ptr[0] != 0) return invalid("balm_batch_cut_voxels: scan_ptr[0] must be 0");
  for (int s = 0; s < n_scans; s++)
    if (scan_ptr[s + 1] < scan_ptr[s]) return invalid("balm_batch_cut_voxels: scan_ptr must be ascending");
  const balm_assoc_opts o = resolve_assoc_opts(opts);
  if (o.layer_limit < 0 || o.layer_limit > 2) return invalid("balm_batch_cut_voxels: layer_limit must be in 0..2");
  const int64_t P = pose_ptr[n_problems], n_points = scan_ptr[n_scans];
  int64_t n_items = 0;  // points replicated over the windows that use them
  for (int64_t j = 0; j < P; j++) {
    const int s = pose_scan[j];
    if (s < 0 || s >= n_scans) return invalid("balm_batch_cut_voxels: pose_scan entry outside [0, n_scans)");
    n_items += scan_ptr[s + 1] - scan_ptr[s];
  }
  if (n_points > 0 && !xyz) return invalid("balm_batch_cut_voxels: bad arguments");
  if (n_items >= ((int64_t)1 << 31) || n_points >= ((int64_t)1 << 31)) {
    balm_set_error("balm_batch_cut_voxels: 2^31 or more points, counted once per pose row that uses them");
    return BALM_ERR_UNSUPPORTED;
  }
  CUDA_TRY(cudaSetDevice(bt->device));
  CUDA_TRY(cudaStreamSynchronize(bt->stream));
  BatchReg *r = new BatchReg();
  std::vector<int64_t> obs_ptr;
  const AssocInput in{"balm_batch_cut_voxels", n_points, xyz, (int)P, poses12, nullptr, n_problems, pose_ptr, pose_scan,
                      scan_ptr, n_items};
  const AssocRegister reg = [&](int64_t M, int64_t K, const int64_t *voxel_ptr, const int64_t *optr, AssocEmit *out) {
    TRY(reg_layout(bt, r, n_problems, pose_ptr, voxel_ptr, K));
    TRY(dev_alloc(&r->row_ptr, (size_t)M + 1));
    TRY(dev_alloc(&r->pose_idx, (size_t)K));
    TRY(dev_alloc(&r->obs, (size_t)K * 10));
    TRY(dev_alloc(&r->coe, (size_t)M));
    TRY(dev_alloc(&r->key, (size_t)M));
    TRY(dev_alloc(&r->layer, (size_t)M));
    *out = AssocEmit{r->obs, 1, 10, r->pose_idx, r->row_ptr, r->coe, r->key, r->layer};
    r->assoc = o;
    obs_ptr.assign(optr, optr + n_problems + 1);
    return (int)BALM_OK;
  };
  long long launches = 0;
  int rc = assoc_cut(bt->stream, in, o, reg, &launches);
  if (rc == BALM_OK) rc = reg_finish(bt, r);
  if (rc == BALM_OK)
    for (int b = 0; b < n_problems; b++) {
      if (n_voxels_out) n_voxels_out[b] = r->hprob[b].nvox;
      if (n_obs_out) n_obs_out[b] = obs_ptr[b + 1] - obs_ptr[b];
    }
  return install(bt, r, rc);
}

extern "C" int balm_batch_merge_scans(balm_batch *bt, int n_problems, const int64_t *pose_ptr, const int32_t *pose_scan,
                                      int n_scans, const int64_t *scan_ptr, const float *xyz, const double *poses12,
                                      double voxel_size, int64_t *kf_ptr, float *kf_xyz) {
  if (!bt || !pose_ptr || !pose_scan || !scan_ptr || !poses12 || !kf_ptr || n_scans < 1)
    return invalid("balm_batch_merge_scans: bad arguments");
  TRY(check_pose_ptr("balm_batch_merge_scans", n_problems, pose_ptr));
  if (scan_ptr[0] != 0) return invalid("balm_batch_merge_scans: scan_ptr[0] must be 0");
  for (int s = 0; s < n_scans; s++)
    if (scan_ptr[s + 1] < scan_ptr[s]) return invalid("balm_batch_merge_scans: scan_ptr must be ascending");
  if (!std::isfinite(voxel_size)) return invalid("balm_batch_merge_scans: voxel_size must be finite");
  const int64_t P = pose_ptr[n_problems], n_points = scan_ptr[n_scans];
  int64_t n_items = 0;
  for (int64_t j = 0; j < P; j++) {
    const int s = pose_scan[j];
    if (s < 0 || s >= n_scans) return invalid("balm_batch_merge_scans: pose_scan entry outside [0, n_scans)");
    n_items += scan_ptr[s + 1] - scan_ptr[s];
  }
  if ((n_points > 0 && !xyz) || (n_items > 0 && !kf_xyz)) return invalid("balm_batch_merge_scans: bad arguments");
  if (n_items >= ((int64_t)1 << 31) || n_points >= ((int64_t)1 << 31)) {
    balm_set_error("balm_batch_merge_scans: 2^31 or more points, counted once per pose row that uses them");
    return BALM_ERR_UNSUPPORTED;
  }
  CUDA_TRY(cudaSetDevice(bt->device));
  CUDA_TRY(cudaStreamSynchronize(bt->stream));
  const MergeInput in{"balm_batch_merge_scans", n_problems, pose_ptr, pose_scan, scan_ptr, n_points, xyz, poses12,
                      voxel_size, n_items};
  long long launches = 0;
  const int rc = merge_scans_build(bt->stream, in, kf_ptr, kf_xyz, &launches);
  if (rc != BALM_OK) cudaStreamSynchronize(bt->stream);
  return rc;
}

// ---- sliding window (assoc.cu: batch_marginalize_build / batch_append_build) ----
// The registration as those steps read it; pose_ptr / voxel_ptr receive the host tables it points into.
static BatchVoxels window_input(const BatchReg *r, const double *poses12, std::vector<int64_t> &pose_ptr,
                                std::vector<int64_t> &voxel_ptr) {
  pose_ptr.resize((size_t)r->B + 1);
  voxel_ptr.resize((size_t)r->B + 1);
  for (int b = 0; b < r->B; b++) {
    pose_ptr[b] = r->hprob[b].pose_base;
    voxel_ptr[b] = r->hprob[b].vox_base;
  }
  pose_ptr[r->B] = r->P;
  voxel_ptr[r->B] = r->M;
  return BatchVoxels{r->B, r->M, pose_ptr.data(), voxel_ptr.data(), r->vox_prob, r->row_ptr, r->pose_idx, r->obs, 1, 10,
                     r->fix, 1, 10, r->coe, r->key, r->layer, poses12};
}

// The new registration r of old's problems with the sizes the step found: layout, then the arrays it emits into (fix
// clusters when `fix`, keys and layers when old has them, and old's association options).
static int window_register(balm_batch *bt, const BatchReg *old, BatchReg *r, const int64_t *pose_ptr,
                           const int64_t *voxel_ptr, const int64_t *obs_ptr, bool fix, WindowEmit *out) {
  const int64_t M = voxel_ptr[old->B], K = obs_ptr[old->B];
  TRY(reg_layout(bt, r, old->B, pose_ptr, voxel_ptr, K));
  TRY(dev_alloc(&r->row_ptr, (size_t)M + 1));
  TRY(dev_alloc(&r->pose_idx, (size_t)K));
  TRY(dev_alloc(&r->obs, (size_t)K * 10));
  TRY(dev_alloc(&r->coe, (size_t)M));
  if (fix) TRY(dev_alloc(&r->fix, (size_t)M * 10));
  if (old->key) {
    TRY(dev_alloc(&r->key, (size_t)M));
    TRY(dev_alloc(&r->layer, (size_t)M));
  }
  r->assoc = old->assoc;
  *out = WindowEmit{r->row_ptr, r->pose_idx, r->obs, r->fix, r->coe, r->key, r->layer};
  return BALM_OK;
}

extern "C" int balm_batch_marginalize(balm_batch *bt, const int *mg_size, const double *poses12, int min_ps,
                                      int64_t *n_voxels_out, int64_t *n_obs_out) {
  if (!bt || !mg_size || !poses12) return invalid("balm_batch_marginalize: bad arguments");
  const BatchReg *old = bt->reg;
  if (!old) return invalid("balm_batch_marginalize: no problems registered");
  for (int b = 0; b < old->B; b++)
    if (mg_size[b] < 0 || mg_size[b] >= old->hprob[b].np)
      return invalid("balm_batch_marginalize: problem " + std::to_string(b) + ": mg_size must be 0 or in [1, N_p)");
  CUDA_TRY(cudaSetDevice(bt->device));
  CUDA_TRY(cudaStreamSynchronize(bt->stream));
  std::vector<int64_t> pose_ptr, voxel_ptr, obs_ptr;
  const BatchVoxels in = window_input(old, poses12, pose_ptr, voxel_ptr);
  BatchReg *r = new BatchReg();
  const WindowRegister reg = [&](const int64_t *vp, const int64_t *op, WindowEmit *out) {
    obs_ptr.assign(op, op + old->B + 1);
    return window_register(bt, old, r, pose_ptr.data(), vp, op, true, out);
  };
  long long launches = 0;
  int rc = batch_marginalize_build(bt->stream, in, mg_size, min_ps, reg, &launches);
  if (rc == BALM_OK) rc = reg_finish(bt, r);
  if (rc == BALM_OK)
    for (int b = 0; b < old->B; b++) {
      if (n_voxels_out) n_voxels_out[b] = r->hprob[b].nvox;
      if (n_obs_out) n_obs_out[b] = obs_ptr[b + 1] - obs_ptr[b];
    }
  return install(bt, r, rc);
}

extern "C" int balm_batch_append_scan(balm_batch *bt, const int32_t *scan_of, const int *slot, int n_scans,
                                      const int64_t *scan_ptr, const float *xyz, const double *poses12,
                                      int64_t *n_voxels_out, int64_t *n_obs_out, int64_t *n_matched_out) {
  if (!bt || !scan_of || !slot || !scan_ptr || !poses12 || n_scans < 1)
    return invalid("balm_batch_append_scan: bad arguments");
  const BatchReg *old = bt->reg;
  if (!old) return invalid("balm_batch_append_scan: no problems registered");
  if (!old->key) return invalid("balm_batch_append_scan: needs a registration from balm_batch_cut_voxels (octree keys)");
  if (scan_ptr[0] != 0) return invalid("balm_batch_append_scan: scan_ptr[0] must be 0");
  for (int s = 0; s < n_scans; s++)
    if (scan_ptr[s + 1] < scan_ptr[s]) return invalid("balm_batch_append_scan: scan_ptr must be ascending");
  int64_t n_items = 0;  // points replicated over the problems that take them
  for (int b = 0; b < old->B; b++) {
    const std::string w = "balm_batch_append_scan: problem " + std::to_string(b);
    const int s = scan_of[b];
    if (s == -1) continue;
    if (s < 0 || s >= n_scans) return invalid(w + ": scan index outside [0, n_scans)");
    if (slot[b] < 0 || slot[b] >= old->hprob[b].np) return invalid(w + ": slot outside [0, N_p)");
    if (scan_ptr[s + 1] - scan_ptr[s] < 1) return invalid(w + ": empty scan");
    n_items += scan_ptr[s + 1] - scan_ptr[s];
  }
  const int64_t n_points = scan_ptr[n_scans];
  if (n_points > 0 && !xyz) return invalid("balm_batch_append_scan: bad arguments");
  if (n_items >= ((int64_t)1 << 31) || n_points >= ((int64_t)1 << 31)) {
    balm_set_error("balm_batch_append_scan: 2^31 or more points, counted once per problem that takes them (or in xyz)");
    return BALM_ERR_UNSUPPORTED;
  }
  CUDA_TRY(cudaSetDevice(bt->device));
  CUDA_TRY(cudaStreamSynchronize(bt->stream));
  std::vector<int64_t> pose_ptr, voxel_ptr, obs_ptr, matched((size_t)old->B);
  const BatchVoxels in = window_input(old, poses12, pose_ptr, voxel_ptr);
  BatchReg *r = new BatchReg();
  const WindowRegister reg = [&](const int64_t *vp, const int64_t *op, WindowEmit *out) {
    obs_ptr.assign(op, op + old->B + 1);
    return window_register(bt, old, r, pose_ptr.data(), vp, op, old->fix != nullptr, out);
  };
  long long launches = 0;
  int rc = batch_append_build(bt->stream, in, old->assoc, scan_of, slot, scan_ptr, xyz, n_points, reg, matched.data(),
                              true, &launches);
  if (rc == BALM_OK) rc = reg_finish(bt, r);
  if (rc == BALM_OK)
    for (int b = 0; b < old->B; b++) {
      if (n_voxels_out) n_voxels_out[b] = r->hprob[b].nvox;
      if (n_obs_out) n_obs_out[b] = obs_ptr[b + 1] - obs_ptr[b];
      if (n_matched_out) n_matched_out[b] = matched[b];
    }
  return install(bt, r, rc);
}

// ---- persistent sliding-window octree (assoc.cu: window_*_build, the maps of every problem in one state) ----
// The window's problems and per-problem counts (win_count / mg_size: 0 or in [lo, hi_p]) checked before anything runs.
static int window_ready(balm_batch *bt, const char *who) {
  if (!bt) return invalid(std::string(who) + ": bad arguments");
  if (!bt->win) return invalid(std::string(who) + ": call balm_batch_window_reset first");
  return BALM_OK;
}
static int check_win_count(const char *who, const std::vector<int> &ns, const int *win_count) {
  if (!win_count) return invalid(std::string(who) + ": bad arguments");
  for (size_t b = 0; b < ns.size(); b++)
    if (win_count[b] < 0 || win_count[b] > ns[b])
      return invalid(std::string(who) + ": problem " + std::to_string(b) + ": win_count must be 0 or in [1, n_slots]");
  return BALM_OK;
}

extern "C" int balm_batch_window_reset(balm_batch *bt, int n_problems, const int *n_slots, const balm_assoc_opts *opts) {
  if (!bt || !n_slots || n_problems < 1) return invalid("balm_batch_window_reset: bad arguments");
  for (int b = 0; b < n_problems; b++)
    if (n_slots[b] < 1 || n_slots[b] > BALM_BATCH_MAX_POSES)
      return invalid("balm_batch_window_reset: problem " + std::to_string(b) + ": n_slots must be in 1 .. BALM_BATCH_MAX_POSES");
  CUDA_TRY(cudaSetDevice(bt->device));
  CUDA_TRY(cudaStreamSynchronize(bt->stream));
  return window_reset_build(&bt->win, "balm_batch_window_reset", n_problems, n_slots, resolve_assoc_opts(opts), true);
}

extern "C" int balm_batch_window_cut(balm_batch *bt, const int32_t *scan_of, const int *slot, int n_scans,
                                     const int64_t *scan_ptr, const float *xyz, const double *poses12) {
  const char *who = "balm_batch_window_cut";
  TRY(window_ready(bt, who));
  if (!scan_of || !slot || !scan_ptr || !poses12 || n_scans < 1) return invalid("balm_batch_window_cut: bad arguments");
  if (scan_ptr[0] != 0) return invalid("balm_batch_window_cut: scan_ptr[0] must be 0");
  for (int s = 0; s < n_scans; s++)
    if (scan_ptr[s + 1] < scan_ptr[s]) return invalid("balm_batch_window_cut: scan_ptr must be ascending");
  const std::vector<int> &ns = window_slots(bt->win);
  int64_t n_items = 0;  // points replicated over the problems that take them
  for (size_t b = 0; b < ns.size(); b++) {
    const std::string w = "balm_batch_window_cut: problem " + std::to_string(b);
    const int s = scan_of[b];
    if (s == -1) continue;
    if (s < 0 || s >= n_scans) return invalid(w + ": scan index outside [0, n_scans)");
    if (slot[b] < 0 || slot[b] >= ns[b]) return invalid(w + ": slot outside [0, n_slots)");
    n_items += scan_ptr[s + 1] - scan_ptr[s];
  }
  const int64_t n_points = scan_ptr[n_scans];
  if (n_points > 0 && !xyz) return invalid("balm_batch_window_cut: bad arguments");
  if (n_items >= ((int64_t)1 << 31) || n_points >= ((int64_t)1 << 31)) {
    balm_set_error("balm_batch_window_cut: 2^31 or more points, counted once per problem that takes them (or in xyz)");
    return BALM_ERR_UNSUPPORTED;
  }
  CUDA_TRY(cudaSetDevice(bt->device));
  CUDA_TRY(cudaStreamSynchronize(bt->stream));
  long long launches = 0;
  return window_cut_build(bt->stream, *bt->win, who, scan_of, slot, n_scans, scan_ptr, xyz, poses12, &launches);
}

extern "C" int balm_batch_window_recut(balm_batch *bt, const int *win_count) {
  TRY(window_ready(bt, "balm_batch_window_recut"));
  TRY(check_win_count("balm_batch_window_recut", window_slots(bt->win), win_count));
  CUDA_TRY(cudaSetDevice(bt->device));
  CUDA_TRY(cudaStreamSynchronize(bt->stream));
  long long launches = 0;
  return window_recut_build(bt->stream, *bt->win, win_count, &launches);
}

extern "C" int balm_batch_window_marginalize(balm_batch *bt, const int *mg_size, const double *poses12,
                                             const int *win_count) {
  TRY(window_ready(bt, "balm_batch_window_marginalize"));
  const std::vector<int> &ns = window_slots(bt->win);
  TRY(check_win_count("balm_batch_window_marginalize", ns, win_count));
  if (!mg_size) return invalid("balm_batch_window_marginalize: bad arguments");
  for (size_t b = 0; b < ns.size(); b++)
    if (mg_size[b] != 0 && (mg_size[b] < 1 || mg_size[b] >= win_count[b]))
      return invalid("balm_batch_window_marginalize: problem " + std::to_string(b) +
                     ": mg_size must be 0 or in [1, win_count)");
  CUDA_TRY(cudaSetDevice(bt->device));
  CUDA_TRY(cudaStreamSynchronize(bt->stream));
  long long launches = 0;
  return window_marginalize_build(bt->stream, *bt->win, mg_size, poses12, win_count, &launches);
}

extern "C" int balm_batch_window_push(balm_batch *bt, const int *win_count, int64_t *n_voxels_out, int64_t *n_obs_out) {
  TRY(window_ready(bt, "balm_batch_window_push"));
  const std::vector<int> &ns = window_slots(bt->win);
  TRY(check_win_count("balm_batch_window_push", ns, win_count));
  CUDA_TRY(cudaSetDevice(bt->device));
  CUDA_TRY(cudaStreamSynchronize(bt->stream));
  const int B = (int)ns.size();
  std::vector<int64_t> pose_ptr((size_t)B + 1, 0), obs_ptr;
  for (int b = 0; b < B; b++) pose_ptr[b + 1] = pose_ptr[b] + ns[b];
  BatchReg *r = new BatchReg();
  const WindowRegister reg = [&](const int64_t *vp, const int64_t *op, WindowEmit *out) {
    const int64_t M = vp[B], K = op[B];
    obs_ptr.assign(op, op + B + 1);
    TRY(reg_layout(bt, r, B, pose_ptr.data(), vp, K));
    TRY(dev_alloc(&r->row_ptr, (size_t)M + 1));
    TRY(dev_alloc(&r->pose_idx, (size_t)K));
    TRY(dev_alloc(&r->obs, (size_t)K * 10));
    TRY(dev_alloc(&r->coe, (size_t)M));
    TRY(dev_alloc(&r->fix, (size_t)M * 10));
    TRY(dev_alloc(&r->key, (size_t)M));
    TRY(dev_alloc(&r->layer, (size_t)M));
    r->assoc = window_opts(bt->win);
    *out = WindowEmit{r->row_ptr, r->pose_idx, r->obs, r->fix, r->coe, r->key, r->layer};
    return (int)BALM_OK;
  };
  long long launches = 0;
  int rc = window_push_build(bt->stream, *bt->win, win_count, reg, &launches);
  if (rc == BALM_OK) rc = reg_finish(bt, r);
  if (rc == BALM_OK)
    for (int b = 0; b < B; b++) {
      if (n_voxels_out) n_voxels_out[b] = r->hprob[b].nvox;
      if (n_obs_out) n_obs_out[b] = obs_ptr[b + 1] - obs_ptr[b];
    }
  return install(bt, r, rc);
}

extern "C" int balm_batch_download_fix(balm_batch *bt, double *fix10) {
  if (!bt || !fix10) return invalid("balm_batch_download_fix: bad arguments");
  const BatchReg *r = bt->reg;
  if (!r) return invalid("balm_batch_download_fix: no problems registered");
  CUDA_TRY(cudaSetDevice(bt->device));
  if (!r->fix) {
    memset(fix10, 0, sizeof(double) * 10 * (size_t)r->M);
    return BALM_OK;
  }
  if (r->M) CUDA_TRY(cudaMemcpyAsync(fix10, r->fix, sizeof(double) * 10 * r->M, cudaMemcpyDeviceToHost, bt->stream));
  CUDA_TRY(cudaStreamSynchronize(bt->stream));
  return BALM_OK;
}

extern "C" int balm_batch_sizes(balm_batch *bt, int *n_problems, int64_t *n_poses, int64_t *n_voxels, int64_t *n_obs) {
  if (!bt) return invalid("balm_batch_sizes: bad arguments");
  const BatchReg *r = bt->reg;
  if (!r) return invalid("balm_batch_sizes: no problems registered");
  if (n_problems) *n_problems = r->B;
  if (n_poses) *n_poses = r->P;
  if (n_voxels) *n_voxels = r->M;
  if (n_obs) *n_obs = r->K;
  return BALM_OK;
}

extern "C" int balm_batch_download_voxels(balm_batch *bt, int64_t *voxel_ptr, int64_t *row_ptr, int32_t *pose_idx,
                                          double *obs10, double *coe, uint64_t *keys, int32_t *layers) {
  if (!bt) return invalid("balm_batch_download_voxels: bad arguments");
  const BatchReg *r = bt->reg;
  if (!r) return invalid("balm_batch_download_voxels: no problems registered");
  if ((keys || layers) && !r->key)
    return invalid("balm_batch_download_voxels: keys and layers exist only after balm_batch_cut_voxels");
  CUDA_TRY(cudaSetDevice(bt->device));
  cudaStream_t st = bt->stream;
  if (voxel_ptr) {
    for (int b = 0; b < r->B; b++) voxel_ptr[b] = r->hprob[b].vox_base;
    voxel_ptr[r->B] = r->M;
  }
  if (row_ptr) CUDA_TRY(cudaMemcpyAsync(row_ptr, r->row_ptr, sizeof(int64_t) * (r->M + 1), cudaMemcpyDeviceToHost, st));
  if (pose_idx && r->K) CUDA_TRY(cudaMemcpyAsync(pose_idx, r->pose_idx, sizeof(int32_t) * r->K, cudaMemcpyDeviceToHost, st));
  if (obs10 && r->K) CUDA_TRY(cudaMemcpyAsync(obs10, r->obs, sizeof(double) * 10 * r->K, cudaMemcpyDeviceToHost, st));
  if (coe && r->M) CUDA_TRY(cudaMemcpyAsync(coe, r->coe, sizeof(double) * r->M, cudaMemcpyDeviceToHost, st));
  if (keys && r->M) CUDA_TRY(cudaMemcpyAsync(keys, r->key, sizeof(uint64_t) * r->M, cudaMemcpyDeviceToHost, st));
  if (layers && r->M) CUDA_TRY(cudaMemcpyAsync(layers, r->layer, sizeof(int32_t) * r->M, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return BALM_OK;
}

extern "C" int balm_batch_evaluate(balm_batch *bt, const double *poses12, int include_fix, double *H, double *g,
                                   double *residual) {
  if (!bt || !poses12 || !residual) return invalid("balm_batch_evaluate: bad arguments");
  BatchReg *r = bt->reg;
  if (!r) return invalid("balm_batch_evaluate: no problems registered");
  CUDA_TRY(cudaSetDevice(bt->device));
  cudaStream_t st = bt->stream;
  CUDA_TRY(cudaMemcpyAsync(r->poses, poses12, sizeof(double) * 12 * r->P, cudaMemcpyHostToDevice, st));
  TRY(enqueue_eval(bt, r, r->ones(), include_fix != 0));
  if (H) CUDA_TRY(cudaMemcpyAsync(H, r->H, sizeof(double) * r->H_size, cudaMemcpyDeviceToHost, st));
  if (g) CUDA_TRY(cudaMemcpyAsync(g, r->g, sizeof(double) * 6 * r->P, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(residual, r->r_eval, sizeof(double) * r->B, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return BALM_OK;
}

extern "C" int balm_batch_damping_iter(balm_batch *bt, double *poses12, const balm_lm_opts *o, int *status,
                                       int *n_iters, balm_trace *trace, double *poses_per_iter) {
  if (!bt || !poses12 || !o || !status || !n_iters) return invalid("balm_batch_damping_iter: bad arguments");
  if (o->verbose != 0) return invalid("balm_batch_damping_iter: verbose is not supported (the traces are returned)");
  BatchReg *r = bt->reg;
  if (!r) return invalid("balm_batch_damping_iter: no problems registered");
  CUDA_TRY(cudaSetDevice(bt->device));
  cudaStream_t st = bt->stream;
  const int B = r->B, max_iter = o->max_iter > 0 ? o->max_iter : 0;
  for (int b = 0; b < B; b++) {  // bavoxel.hpp:1071-1085, per problem
    status[b] = (o->min_planes_per_pose > 0 && r->min_planes[b] < o->min_planes_per_pose) ? BALM_ERR_TOO_FEW_PLANES : BALM_OK;
    n_iters[b] = 0;
  }
  ScratchPool pool;
  balm_trace *d_trace = nullptr;
  TRY(pool.get(&d_trace, (size_t)B * std::max(1, max_iter)));
  const size_t pbytes = sizeof(double) * 12 * r->P;
  CUDA_TRY(cudaMemcpyAsync(r->poses, poses12, pbytes, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(r->status(), status, sizeof(int) * B, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemsetAsync(d_trace, 0, sizeof(balm_trace) * B * std::max(1, max_iter), st));
  batch_init_kernel<<<(B + 127) / 128, 128, 0, st>>>(B, r->status(), max_iter, o->u0, o->v0, r->u, r->v, r->active(),
                                                     r->calc(), r->evalm(), r->n_iters());
  CUDA_TRY(cudaGetLastError());
  bool any = false;
  for (int b = 0; b < B; b++) any = any || status[b] == BALM_OK;
  LmArgs a{r->prob, B, 0, max_iter, o->force_hess != 0 ? 1 : 0, o->rel_tol, r->r_eval, r->r2, r->q1, r->notpd(),
           r->r1, r->u, r->v, r->active(), r->calc(), r->evalm(), r->n_iters(), r->n_active(), r->poses, r->trial,
           d_trace};
  for (int it = 0; any && it < max_iter; it++) {
    TRY(enqueue_eval(bt, r, r->evalm(), o->hess_includes_fix != 0));
    batch_solve_kernel<<<B, SOLVE_THREADS, SOLVE_SMEM, st>>>(r->prob, r->active(), r->H, r->g, r->u, r->poses,
                                                             r->trial, r->q1, r->notpd());
    CUDA_TRY(cudaGetLastError());
    TRY(enqueue_trial_residual(bt, r));
    CUDA_TRY(cudaMemsetAsync(r->n_active(), 0, sizeof(int), st));
    a.it = it;
    batch_lm_kernel<<<(B + 127) / 128, 128, 0, st>>>(a);
    CUDA_TRY(cudaGetLastError());
    if (poses_per_iter)
      CUDA_TRY(cudaMemcpyAsync(poses_per_iter + (size_t)it * 12 * r->P, r->poses, pbytes, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(bt->h_count, r->n_active(), sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    any = *bt->h_count > 0;
  }
  if (o->gauge_mode == 0 || o->gauge_mode == 1) {
    CUDA_TRY(cudaMemcpyAsync(r->trial, r->poses, pbytes, cudaMemcpyDeviceToDevice, st));  // pose-0 snapshots
    batch_gauge_kernel<<<(r->P + 127) / 128, 128, 0, st>>>(r->prob, r->pose_prob, r->status(), r->P, r->poses, r->trial,
                                                           o->gauge_mode);
    CUDA_TRY(cudaGetLastError());
  }
  CUDA_TRY(cudaMemcpyAsync(poses12, r->poses, pbytes, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(n_iters, r->n_iters(), sizeof(int) * B, cudaMemcpyDeviceToHost, st));
  if (trace && max_iter > 0)
    CUDA_TRY(cudaMemcpyAsync(trace, d_trace, sizeof(balm_trace) * B * max_iter, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return BALM_OK;
}

extern "C" int balm_batch_pose_covariance(balm_batch *bt, const double *poses12, const double *c_cov81, double point_noise,
                                          int include_fix, int *status, double *Rcov_raw, double *Rcov) {
  if (!bt || !poses12) return invalid("balm_batch_pose_covariance: bad arguments");
  BatchReg *r = bt->reg;
  if (!r) return invalid("balm_batch_pose_covariance: no problems registered");
  if (r->M >= ((int64_t)1 << 31)) {
    balm_set_error("balm_batch_pose_covariance: 2^31 or more voxels");
    return BALM_ERR_UNSUPPORTED;
  }
  CUDA_TRY(cudaSetDevice(bt->device));
  cudaStream_t st = bt->stream;
  const int B = r->B;
  std::vector<int4> items;  // the covariance SYRK's: 8 rows per voxel
  std::vector<int2> range;
  syrk_items(r->hprob, 8, items, range);
  ScratchPool pool;
  double *rows = nullptr, *Dobs = nullptr, *dpart = nullptr, *spart = nullptr, *raw = nullptr, *cov = nullptr,
         *ccov = nullptr;
  int4 *d_items = nullptr;
  int2 *d_range = nullptr;
  int *d_status = nullptr;
  const size_t n_rows = r->G_size / 3 * 8;
  TRY(pool.get(&rows, n_rows));
  TRY(pool.get(&Dobs, (size_t)r->K * 21));
  TRY(pool.get(&dpart, (size_t)r->n_ochunks * 21 * 32));
  TRY(pool.get(&spart, items.size() * TILE * TILE));
  TRY(pool.get(&raw, r->H_size));
  TRY(pool.get(&d_items, items.size()));
  TRY(pool.get(&d_range, (size_t)B));
  if (Rcov) {
    TRY(pool.get(&cov, r->H_size));
    TRY(pool.get(&d_status, (size_t)B));
  }
  if (c_cov81) {
    TRY(pool.get(&ccov, (size_t)r->K * 81));
    if (r->K) CUDA_TRY(cudaMemcpyAsync(ccov, c_cov81, sizeof(double) * 81 * r->K, cudaMemcpyHostToDevice, st));
  }
  if (!items.empty())
    CUDA_TRY(cudaMemcpyAsync(d_items, items.data(), sizeof(int4) * items.size(), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(d_range, range.data(), sizeof(int2) * B, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(r->poses, poses12, sizeof(double) * 12 * r->P, cudaMemcpyHostToDevice, st));
  const Dev d = r->dev();
  // the voxel statistics at these poses (fix clusters as include_fix): with Rcov, the evaluation of H computes them
  if (Rcov) TRY(enqueue_eval(bt, r, r->ones(), include_fix != 0));
  else enqueue_stats(bt, r, r->poses, r->ones(), include_fix != 0, r->stats);
  CUDA_TRY(cudaMemsetAsync(rows, 0, sizeof(double) * n_rows, st));  // columns of non-observing poses stay zero
  if (r->M > 0) {  // one CTA per voxel: a grid-stride loop would cost the kernel a spill
    batch_cov_rows_kernel<<<(unsigned)r->M, 32, COV_SMEM, st>>>(d, r->poses, r->stats, ccov, point_noise * point_noise, rows,
                                                        Dobs);
  }
  if (r->n_ochunks > 0)
    batch_cov_diag_kernel<<<(r->n_ochunks + 3) / 4, 128, 0, st>>>(d, r->ochunk_prob, r->n_ochunks, Dobs, dpart);
  if (!items.empty())
    batch_syrk_kernel<8, 4><<<(unsigned)items.size(), 128, 0, st>>>(r->prob, r->ones(), d_items, rows, spart);
  batch_assemble_kernel<21, 0, false, false><<<dim3(B, MAXN / TILE), 256, 0, st>>>(r->prob, r->ones(), d_range, dpart,
                                                                                    spart, raw, nullptr);
  if (Rcov) batch_cov_solve_kernel<<<B, SOLVE_THREADS, SOLVE_SMEM, st>>>(r->prob, r->H, raw, cov, d_status);
  CUDA_TRY(cudaGetLastError());
  if (Rcov_raw) CUDA_TRY(cudaMemcpyAsync(Rcov_raw, raw, sizeof(double) * r->H_size, cudaMemcpyDeviceToHost, st));
  if (Rcov) CUDA_TRY(cudaMemcpyAsync(Rcov, cov, sizeof(double) * r->H_size, cudaMemcpyDeviceToHost, st));
  if (Rcov && status) CUDA_TRY(cudaMemcpyAsync(status, d_status, sizeof(int) * B, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  if (!Rcov && status)
    for (int b = 0; b < B; b++) status[b] = BALM_OK;
  return BALM_OK;
}

extern "C" int balm_batch_set_voxel_loss(balm_batch *bt, int kind, double scale) {
  if (!bt) return invalid("balm_batch_set_voxel_loss: bad arguments");
  TRY(check_voxel_loss("balm_batch_set_voxel_loss", kind, scale));
  bt->vloss_kind = kind;
  bt->vloss_scale = kind == BALM_LOSS_TRIVIAL ? 1.0 : scale;  // a trivial loss's scale is unused
  return BALM_OK;
}

extern "C" int balm_batch_voxel_residuals(balm_batch *bt, const double *poses12, int include_fix, double *lam, double *w) {
  if (!bt || !poses12) return invalid("balm_batch_voxel_residuals: bad arguments");
  BatchReg *r = bt->reg;
  if (!r) return invalid("balm_batch_voxel_residuals: no problems registered");
  CUDA_TRY(cudaSetDevice(bt->device));
  cudaStream_t st = bt->stream;
  ScratchPool pool;
  double *d_out = nullptr;
  TRY(pool.get(&d_out, 2 * (size_t)r->M));
  CUDA_TRY(cudaMemcpyAsync(r->poses, poses12, sizeof(double) * 12 * r->P, cudaMemcpyHostToDevice, st));
  // the evaluation's own stats instantiation, so that w is bitwise the weight an evaluation at these poses applies
  enqueue_stats(bt, r, r->poses, r->ones(), include_fix != 0, r->stats, d_out, d_out + r->M);
  CUDA_TRY(cudaGetLastError());
  if (lam && r->M) CUDA_TRY(cudaMemcpyAsync(lam, d_out, sizeof(double) * r->M, cudaMemcpyDeviceToHost, st));
  if (w && r->M) CUDA_TRY(cudaMemcpyAsync(w, d_out + r->M, sizeof(double) * r->M, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return BALM_OK;
}

// covariance.cu -- pose-covariance propagation of the consistency experiment (SURVEY.md 8f row N3):
//
//   Rcov_raw = sum over observations (a, j) of  Ls c_cov_j Ls^T ,  Ls = d(gradient)/d(9 parameters of cluster (a, j))
//   Rcov     = H^-1 Rcov_raw H^-T
// = VOX_HESS::left_jacobian_point + BALM2::multi_second + the last lines of BALM2::damping_iter
//   (src/simulation/BAs_left.hpp:342-473, 995-1023, 1089-1096), with c_cov as PointCluster::push
//   accumulates it under isotropic point noise (src/simulation/toolss.hpp:311-343) or given per observation.
//
// The reference forms a dense 6N x 9 matrix Ls per observation and adds the 6N x 6N product Ls c Ls^T. Written out, the
// block of Ls for pose p is (c2 = coe 2/NN)
//     Ls_j[p] = c2 ( Q_p Z_j + [j == p] E_p ),   Q_p = [A_p | a_p] (6x4),  Z_j = [G_j ; -h_j^T/NN] (4x9),  E_p (6x9)
// (A_p = g2_combos[p], a_p = (U_l TC_p)[:,3] -- the same vector as in the Hessian, G_j as in the reference), hence per voxel
//     sum_j Ls_j c_j Ls_j^T [p,q] = c2^2 ( Q_p Wz Q_q^T + Q_p Y_q + Y_p^T Q_q^T + [p == q] D_p ),
//     Wz = sum_j Z_j c_j Z_j^T (4x4),  Y_q = Z_q c_q E_q^T (4x6),  D_p = E_p c_p E_p^T (6x6)
//   = c2^2 ( Q V^T + V Q^T )[p,q] + [p == q] c2^2 D_p ,   V_p = Q_p Wz/2 + Y_p^T .
// So the whole sum is a symmetric rank-8M product of the same shape as the Hessian accumulation: eight rows per voxel
// (four of c2 Q^T, four of c2 V^T, 6N columns each), accumulated by the fp64 DMMA SYRK kernel with the A operand taken
// from the partner row (row ^ 4), plus 6x6 diagonal blocks -- O(M N^2) tensor-core work instead of the reference's
// O(K N^2) dense rank-9 updates. H^-1 (.) H^-T reuses the LDL^T factors of the solve with n right-hand sides.
#include <math.h>
#include <stdlib.h>
#include <algorithm>
#include <vector>
#include "internal.cuh"

int launch_syrk_f64_on(balm_ctx *c, const double *G, int64_t rows, bool first_batch, int row_xor);

namespace {

struct CovArgs {
  const double *obs;
  int64_t Kp;
  const int *pose_idx;
  const long long *row_ptr;
  const double *poses;
  const double *stats;   // [nv][20] of the batch (v0-based)
  const double *ccov;    // [K][81] row-major or null
  double pn2;
  int64_t v0, v1;
  int N, ldg;
  double *Wz;            // [nv][10]
  double *G;             // [8*nv][ldg]
  double *Dobs;          // [K][21] (global observation index)
  long long obs0;        // PER_OBS rows: the observation of G's first 48 entries
};

__device__ __forceinline__ void load_obs(const CovArgs &a, long long s, double *o) {
#pragma unroll
  for (int c = 0; c < 10; c++) o[c] = a.obs[c * a.Kp + s];
}
__device__ __forceinline__ void load_ccov(const CovArgs &a, long long s, const double *o, double *C) {
  if (a.ccov) {
    for (int e = 0; e < 81; e++) C[e] = a.ccov[(size_t)s * 81 + e];
  } else {
    cluster_cov_iso(o, a.pn2, C);
  }
}

// pass 1: Wz[v] = sum_j Z_j c_j Z_j^T   (one warp per voxel, fixed-order shuffle reduction)
__global__ void __launch_bounds__(128) cov_wz_kernel(CovArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t v = a.v0 + (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
  if (v >= a.v1) return;
  const long long s0 = a.row_ptr[v], s1 = a.row_ptr[v + 1];
  const double *st = a.stats + (v - a.v0) * BALM_STATS_STRIDE;
  double acc[10];
  for (int e = 0; e < 10; e++) acc[e] = 0.0;
  for (long long s = s0 + lane; s < s1; s += 32) {
    double o[10], C[81];
    load_obs(a, s, o);
    load_ccov(a, s, o, C);
    CovTerms t;
    cov_terms(o, a.poses + 12 * a.pose_idx[s], st, t);
    cov_wz_add(t, C, acc);
  }
  for (int e = 0; e < 10; e++) acc[e] = warp_sum(acc[e]);
  if (lane == 0)
    for (int e = 0; e < 10; e++) a.Wz[(v - a.v0) * 10 + e] = acc[e];
}

// pass 2: the eight rows of a voxel (c2 Q^T | c2 V^T) and the diagonal block c2^2 D_p of every observation; PER_OBS:
// every observation's six columns of them at G + 48 (s - obs0), [8][6] row-major (a blocks context's raw term)
template <bool PER_OBS>
__global__ void __launch_bounds__(128) cov_rows_kernel(CovArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t v = a.v0 + (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
  if (v >= a.v1) return;
  const long long s0 = a.row_ptr[v], s1 = a.row_ptr[v + 1];
  const double *st = a.stats + (v - a.v0) * BALM_STATS_STRIDE;
  const double c2 = st[16] * 2.0 * st[12];  // coe * 2 / NN
  double Wz[4][4];
  {
    const double *wz = a.Wz + (v - a.v0) * 10;
    int q = 0;
    for (int i = 0; i < 4; i++)
      for (int j = i; j < 4; j++) { Wz[i][j] = wz[q]; Wz[j][i] = wz[q]; q++; }
  }
  for (long long s = s0 + lane; s < s1; s += 32) {
    double o[10], C[81];
    load_obs(a, s, o);
    load_ccov(a, s, o, C);
    CovTerms t;
    const int p = a.pose_idx[s];
    cov_terms(o, a.poses + 12 * p, st, t);
    if (PER_OBS) cov_obs_rows(t, C, Wz, c2, a.G + 48 * (size_t)(s - a.obs0), 6, a.Dobs + (size_t)s * 21);
    else cov_obs_rows(t, C, Wz, c2, a.G + (size_t)(8 * (v - a.v0)) * a.ldg + 6 * p, a.ldg, a.Dobs + (size_t)s * 21);
  }
}

// per pose: sum of its observations' diagonal blocks in ascending voxel order (dense: s = v N + p; sparse: the lists)
__global__ void cov_diag_reduce_kernel(const double *Dobs, int N, int64_t M, int dense, const int *csc_ptr,
                                       const int *csc_obs, double *Dacc /*[21][N]*/, int add, int64_t v0, int64_t v1,
                                       const int *csc_lo, const int *csc_hi) {
  const int p = blockIdx.x, q = threadIdx.x;
  if (q >= 21) return;
  double s = 0.0;
  if (dense) {
    for (int64_t v = v0; v < v1; v++) s += Dobs[((size_t)v * N + p) * 21 + q];
  } else {
    for (int t = csc_lo[p]; t < csc_hi[p]; t++) s += Dobs[(size_t)csc_obs[t] * 21 + q];
  }
  Dacc[(size_t)q * N + p] = add ? Dacc[(size_t)q * N + p] + s : s;
}

// ---- n right-hand sides through the LDL^T factors of the solve (A: L below the diagonal, Xinv: L_jj^-1, dinv) ----
constexpr int NB = BALM_NB;
constexpr int MRHS_SMEM = 2 * NB * (NB + 1) * (int)sizeof(double);
// B[j0 .. j0+nbw) rows, column tile blockIdx.x*64:  B <- X B  (TRANS = 0) or  B <- X^T B  (TRANS = 1)
template <int TRANS>
__global__ void __launch_bounds__(256) mrhs_diag_kernel(const double *Xcm, double *B, int n, int j0, int nbw, const double *rowscale) {
  extern __shared__ double cov_smem[];
  double (*sX)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(cov_smem);
  double (*sB)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(cov_smem + NB * (NB + 1));
  const int tid = threadIdx.x, c0 = blockIdx.x * NB;
  for (int e = tid; e < NB * NB; e += 256) {
    const int rI = e & (NB - 1), cI = e >> 6;
    sX[rI][cI] = Xcm[cI * NB + rI];  // X[r][c]
    const int col = c0 + cI;
    double b = (rI < nbw && col < n) ? B[(size_t)col * n + j0 + rI] : 0.0;
    if (rowscale && rI < nbw) b *= rowscale[j0 + rI];
    sB[rI][cI] = b;
  }
  __syncthreads();
  for (int e = tid; e < NB * NB; e += 256) {
    const int rI = e & (NB - 1), cI = e >> 6;
    double s = 0.0;
    if (TRANS) { for (int k = rI; k < NB; k++) s += sX[k][rI] * sB[k][cI]; }   // X^T is upper triangular
    else { for (int k = 0; k <= rI; k++) s += sX[rI][k] * sB[k][cI]; }
    const int col = c0 + cI;
    if (rI < nbw && col < n) B[(size_t)col * n + j0 + rI] = s;
  }
}
// forward: B[i0.., c0..] -= L[i0.., j0..j0+nbw) B[j0.., c0..]   (grid: row tiles below x column tiles)
__global__ void __launch_bounds__(256) mrhs_fwd_update_kernel(const double *A, double *B, int n, int j0, int nbw) {
  extern __shared__ double cov_smem[];
  double (*sL)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(cov_smem);
  double (*sB)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(cov_smem + NB * (NB + 1));
  const int tid = threadIdx.x, i0 = j0 + nbw + blockIdx.x * NB, c0 = blockIdx.y * NB;
  for (int e = tid; e < NB * NB; e += 256) {
    const int rI = e & (NB - 1), kI = e >> 6;
    sL[rI][kI] = (i0 + rI < n && kI < nbw) ? A[(size_t)(j0 + kI) * n + i0 + rI] : 0.0;
    sB[rI][kI] = (rI < nbw && c0 + kI < n) ? B[(size_t)(c0 + kI) * n + j0 + rI] : 0.0;  // sB[k][col]
  }
  __syncthreads();
  for (int e = tid; e < NB * NB; e += 256) {
    const int rI = e & (NB - 1), cI = e >> 6;
    if (i0 + rI >= n || c0 + cI >= n) continue;
    double s = 0.0;
    for (int k = 0; k < NB; k++) s += sL[rI][k] * sB[k][cI];
    B[(size_t)(c0 + cI) * n + i0 + rI] -= s;
  }
}
// backward: B[j0.., c0..] -= sum over row blocks r > j of L[r.., j0..]^T B[r.., c0..]   (one CTA per column tile)
__global__ void __launch_bounds__(256) mrhs_bwd_update_kernel(const double *A, double *B, int n, int j0, int nbw) {
  extern __shared__ double cov_smem[];
  double (*sL)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(cov_smem);
  double (*sB)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(cov_smem + NB * (NB + 1));
  const int tid = threadIdx.x, c0 = blockIdx.x * NB;
  double acc[16];
  for (int q = 0; q < 16; q++) acc[q] = 0.0;
  for (int i0 = j0 + nbw; i0 < n; i0 += NB) {
    __syncthreads();
    for (int e = tid; e < NB * NB; e += 256) {
      const int rI = e & (NB - 1), kI = e >> 6;
      sL[rI][kI] = (i0 + rI < n && kI < nbw) ? A[(size_t)(j0 + kI) * n + i0 + rI] : 0.0;   // L[i0+r][j0+k]
      sB[rI][kI] = (i0 + rI < n && c0 + kI < n) ? B[(size_t)(c0 + kI) * n + i0 + rI] : 0.0;  // B[i0+r][c0+col]
    }
    __syncthreads();
    for (int q = 0; q < 16; q++) {
      const int e = tid + q * 256, kI = e & (NB - 1), cI = e >> 6;  // output (row j0+kI, col c0+cI)
      double s = 0.0;
      for (int rI = 0; rI < NB; rI++) s += sL[rI][kI] * sB[rI][cI];
      acc[q] += s;
    }
  }
  for (int q = 0; q < 16; q++) {
    const int e = tid + q * 256, kI = e & (NB - 1), cI = e >> 6;
    if (kI < nbw && c0 + cI < n) B[(size_t)(c0 + cI) * n + j0 + kI] -= acc[q];
  }
}
__global__ void transpose_inplace_kernel(double *B, int n) {
  const int i = blockIdx.x * 32 + threadIdx.x, j = blockIdx.y * 32 + threadIdx.y;
  if (i < n && j < i) {
    const double a = B[(size_t)j * n + i], b = B[(size_t)i * n + j];
    B[(size_t)j * n + i] = b;
    B[(size_t)i * n + j] = a;
  }
}

__global__ void scale_rows_kernel(double *B, const double *dinv, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
  if (i < n) B[(size_t)j * n + i] *= dinv[i];
}

// B <- (L D L^T)^-1 B for all n columns of s's last factor: forward sweep (B_j <- X_j B_j, rows below -= L21 B_j),
// rows scaled by 1/d, backward sweep (B_j <- X_j^T (B_j - sum_{r>j} L_rj^T B_r))
int solve_many(balm_ctx *c, const DenseSystem &s, double *B) {
  const int n = s.n, ct = (n + NB - 1) / NB;
  cudaStream_t st = c->stream;
  int launches = 0;
  for (int j0 = 0, pi = 0; j0 < n; j0 += NB, pi++) {
    const int nbw = std::min(NB, n - j0), m = n - j0 - nbw;
    mrhs_diag_kernel<0><<<ct, 256, MRHS_SMEM, st>>>(s.w->Xinv + (size_t)pi * NB * NB, B, n, j0, nbw, nullptr);
    if (m > 0) mrhs_fwd_update_kernel<<<dim3((m + NB - 1) / NB, ct), 256, MRHS_SMEM, st>>>(s.A, B, n, j0, nbw);
    launches += 2;
  }
  scale_rows_kernel<<<dim3((n + 255) / 256, n), 256, 0, st>>>(B, s.w->dinv, n);
  launches++;
  const int npan = (n + NB - 1) / NB;
  for (int pi = npan - 1; pi >= 0; pi--) {
    const int j0 = pi * NB, nbw = std::min(NB, n - j0);
    if (j0 + nbw < n) mrhs_bwd_update_kernel<<<ct, 256, MRHS_SMEM, st>>>(s.A, B, n, j0, nbw);
    mrhs_diag_kernel<1><<<ct, 256, MRHS_SMEM, st>>>(s.w->Xinv + (size_t)pi * NB * NB, B, n, j0, nbw, nullptr);
    launches += 2;
  }
  c->launches += launches;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

// rows and columns [a0, a0 + 6) of the n x n matrix A set to 0, diagonal to diag
__global__ void delete_block_kernel(double *A, int n, int a0, double diag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, k = blockIdx.y;
  if (i >= n) return;
  const double v = i == a0 + k ? diag : 0.0;
  A[(size_t)(a0 + k) * n + i] = v;  // column a0 + k
  A[(size_t)i * n + a0 + k] = v;    // row a0 + k
}

}  // namespace

int covariance_setup() {
  CUDA_TRY(cudaFuncSetAttribute(mrhs_diag_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, MRHS_SMEM));
  CUDA_TRY(cudaFuncSetAttribute(mrhs_diag_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, MRHS_SMEM));
  CUDA_TRY(cudaFuncSetAttribute(mrhs_fwd_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MRHS_SMEM));
  CUDA_TRY(cudaFuncSetAttribute(mrhs_bwd_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MRHS_SMEM));
  return BALM_OK;
}

// bytes of device scratch a covariance call's batched buffers may take
static size_t cov_budget() {
  size_t budget = (size_t)4 << 30;
  if (const char *e = getenv("BALM_COV_BUDGET_MB")) budget = (size_t)atoll(e) << 20;
  return budget;
}

int cov_raw_dev(balm_ctx *c, ScratchPool &pool, const double *poses_dev, const double *ccov_host, double point_noise,
                bool include_fix, double **R_out) {
  const int n = c->n, N = c->N;
  const int64_t M = c->M, K = c->K;
  cudaStream_t st = c->stream;
  // voxels per batch: the stats table holds VB voxels; the row buffer gets its own budget
  const size_t budget = cov_budget();
  int64_t vb = std::min<int64_t>(c->VB, (int64_t)(budget / ((size_t)8 * c->ldg * sizeof(double))));
  vb = std::max<int64_t>(1, std::min<int64_t>(vb, M));
  double *G = nullptr, *Wz = nullptr, *Dobs = nullptr, *Dacc = nullptr, *R = nullptr, *ccov = nullptr;
  TRY(pool.get(&G, (size_t)8 * vb * c->ldg));
  TRY(pool.get(&Wz, (size_t)vb * 10));
  TRY(pool.get(&Dobs, (size_t)K * 21));
  TRY(pool.get(&Dacc, (size_t)21 * N));
  TRY(pool.get(&R, (size_t)n * n));
  if (ccov_host) {
    TRY(pool.get(&ccov, (size_t)K * 81));
    CUDA_TRY(cudaMemcpyAsync(ccov, ccov_host, sizeof(double) * (size_t)K * 81, cudaMemcpyHostToDevice, st));
  }
  bool first = true;
  for (int64_t v0 = 0; v0 < M; v0 += vb) {
    const int64_t v1 = std::min(M, v0 + vb), nv = v1 - v0;
    TRY(launch_csc_batch(c, v0, v1));
    double *rdummy = c->scal + 21;
    CUDA_TRY(cudaMemsetAsync(rdummy, 0, sizeof(double), st));
    TRY(launch_voxel_stats(c, poses_dev, v0, v1, c->stats, include_fix, rdummy));
    CUDA_TRY(cudaMemsetAsync(G, 0, sizeof(double) * (size_t)8 * nv * c->ldg, st));
    CovArgs a{c->obs, c->Kp, c->pose_idx, c->row_ptr, poses_dev, c->stats, ccov, point_noise * point_noise, v0, v1, N,
              c->ldg, Wz, G, Dobs, 0};
    const unsigned grid = (unsigned)((nv + 3) / 4);
    cov_wz_kernel<<<grid, 128, 0, st>>>(a);
    cov_rows_kernel<false><<<grid, 128, 0, st>>>(a);
    cov_diag_reduce_kernel<<<N, 32, 0, st>>>(Dobs, N, M, c->dense ? 1 : 0, c->csc_ptr, c->csc_obs, Dacc, first ? 0 : 1, v0,
                                             v1, c->csc_lo, c->csc_hi);
    c->launches += 3;
    TRY(launch_syrk_f64_on(c, G, 8 * nv, first, /*row_xor=*/4));
    first = false;
  }
  TRY(launch_csc_batch(c, 0, M));
  TRY(launch_assemble(c, Dacc, R));
  *R_out = R;
  return BALM_OK;
}

int cov_factor(balm_ctx *c, const DenseSystem &s, int skip, const char *singular_msg) {
  const int n = s.n;
  cudaStream_t st = c->stream;
  TRY(launch_ldlt_solve(c, s, 0.0));
  CUDA_TRY(cudaMemcpyAsync(c->h_flags, c->flags, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  // a singular H (free gauge: no fix clusters in it) does not produce an exact zero pivot in floating point but
  // pivots at rounding level relative to the others: refuse instead of returning 1e16-sized garbage
  std::vector<double> dinv_h((size_t)n);
  CUDA_TRY(cudaMemcpy(dinv_h.data(), s.w->dinv, sizeof(double) * n, cudaMemcpyDeviceToHost));
  double dmin = 1e300, dmax = 0.0;
  for (int i = 0; i < n; i++) {
    if (skip >= 0 && i >= skip && i < skip + 6) continue;
    const double d = fabs(1.0 / dinv_h[i]);
    dmin = std::min(dmin, d);
    dmax = std::max(dmax, d);
  }
  if (c->h_flags[0] || !(dmin > 1e-11 * dmax)) {
    balm_set_error(singular_msg);
    return BALM_ERR_NOT_PD;
  }
  return BALM_OK;
}

int cov_sandwich(balm_ctx *c, const DenseSystem &s, double *B) {
  const int n = s.n;
  TRY(solve_many(c, s, B));                                   // H^-1 B
  transpose_inplace_kernel<<<dim3((n + 31) / 32, (n + 31) / 32), dim3(32, 32), 0, c->stream>>>(B, n);
  TRY(solve_many(c, s, B));                                   // H^-1 (H^-1 B)^T = H^-1 B H^-T
  c->launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int cov_delete_block(balm_ctx *c, double *A, int n, int a0, double diag) {
  delete_block_kernel<<<dim3((n + 127) / 128, 6), 128, 0, c->stream>>>(A, n, a0, diag);
  c->launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

// ---------------- point-noise covariance on a BALM_PREC_BLOCKS context (DESIGN.md "Point-noise covariance on blocks
// contexts") ----------------
// Sigma_sel = W^T R W with W = J Y, Y = A^-1 E: E the unit columns of the selected unknowns, A the undamped factor of
// H (or H_rig) with the anchor's rows and columns replaced by I, J the identity (plain) or the rig's Jacobian, R the raw
// term on the slot pattern. Y, W and Z = R W are 6 x (rows) x (columns) dense, row-major; nothing 6N x 6N exists.
namespace {

constexpr int PC_TILE = 32;  // right-hand sides per CTA of the row kernels
constexpr int PC_SEG = 384;  // rows of one partial sum of W^T Z (fixed: the sums do not depend on the columns' chunk)

// Y[6 col[sel[u0 + u]] + k][6 u + k] = 1 (Y zeroed before)
__global__ void pc_unit_kernel(const int *selcol, int u0, int nu, int ld, double *Y) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 6 * nu) return;
  const int u = t / 6, k = t % 6;
  Y[(6 * (size_t)selcol[u0 + u] + k) * ld + 6 * u + k] = 1.0;
}

// W[6 p + r][c] = Y[6 col[p] + r][c]: the plain context's J = I, rows back in pose order
__global__ void __launch_bounds__(6 * PC_TILE) pc_gather_kernel(const double *Y, const int *col, int ld, int ncols,
                                                                double *W) {
  const int p = blockIdx.y, r = threadIdx.x / PC_TILE, c = blockIdx.x * PC_TILE + threadIdx.x % PC_TILE;
  if (c < ncols) W[(6 * (size_t)p + r) * ld + c] = Y[(6 * (size_t)col[p] + r) * ld + c];
}

// Z = R W, row block i: sum over pose i's pairs in ascending other pose (2 pair + transposed, other pose), each block's
// six columns in ascending order
__global__ void __launch_bounds__(6 * PC_TILE) pc_rw_kernel(const double *raw, const int *pp_ptr, const int2 *pp,
                                                            const double *W, int ld, int ncols, double *Z) {
  const int i = blockIdx.y, a = threadIdx.x / PC_TILE, c = blockIdx.x * PC_TILE + threadIdx.x % PC_TILE;
  if (c >= ncols) return;
  double s = 0.0;
  for (int q = pp_ptr[i]; q < pp_ptr[i + 1]; q++) {
    const int2 e = pp[q];
    const double *B = raw + 36 * (size_t)(e.x >> 1), *w = W + 6 * (size_t)e.y * ld + c;
    for (int cc = 0; cc < 6; cc++) s = fma(B[(e.x & 1) ? 6 * a + cc : 6 * cc + a], w[(size_t)cc * ld], s);
  }
  Z[(6 * (size_t)i + a) * ld + c] = s;
}

// the 6x6 block pair t of the chunk: joint (I, J) = the t-th of I >= J, row-major over I, then ordered so that
// sel[I] >= sel[J] (a block is W_I^T Z_J for the same two unknowns whatever their places in sel); marginals (t, t)
__device__ __forceinline__ void pc_pair(int t, int joint, const int *sel, int &I, int &J) {
  if (!joint) { I = J = t; return; }
  int i = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while ((long long)(i + 1) * (i + 2) / 2 <= t) i++;
  while ((long long)i * (i + 1) / 2 > t) i--;
  I = i;
  J = t - i * (i + 1) / 2;
  if (sel[I] < sel[J]) { const int k = I; I = J; J = k; }
}

// part[seg][t][6 b + a] = sum over rows of segment seg, ascending, of W[row][6 I + a] Z[row][6 J + b]
__global__ void __launch_bounds__(128) pc_dot_kernel(const double *W, const double *Z, int ld, int rows, int npairs,
                                                     int joint, const int *sel, double *part) {
  const int t = blockIdx.x * 128 + threadIdx.x, seg = blockIdx.y;
  if (t >= npairs) return;
  int I, J;
  pc_pair(t, joint, sel, I, J);
  double acc[36];
#pragma unroll
  for (int e = 0; e < 36; e++) acc[e] = 0.0;
  const int r1 = min(rows, (seg + 1) * PC_SEG);
  for (int r = seg * PC_SEG; r < r1; r++) {
    double w[6], z[6];
#pragma unroll
    for (int a = 0; a < 6; a++) {
      w[a] = W[(size_t)r * ld + 6 * I + a];
      z[a] = Z[(size_t)r * ld + 6 * J + a];
    }
#pragma unroll
    for (int b = 0; b < 6; b++)
#pragma unroll
      for (int a = 0; a < 6; a++) acc[6 * b + a] = fma(w[a], z[b], acc[6 * b + a]);
  }
  double *o = part + ((size_t)seg * npairs + t) * 36;
#pragma unroll
  for (int e = 0; e < 36; e++) o[e] = acc[e];
}

// the segments summed in ascending order; entry (6 I + a, 6 J + b) with (I > J or a >= b) written to both of its
// places: joint into cov (n6 x n6, column-major), marginals into marg [u0 + t][36] (column-major)
__global__ void pc_reduce_kernel(const double *part, int nseg, int npairs, int joint, const int *sel, int u0, int n6,
                                 double *cov, double *marg) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= 36LL * npairs) return;
  const int t = (int)(g / 36), e = (int)(g % 36), a = e % 6, b = e / 6;
  int I, J;
  pc_pair(t, joint, sel, I, J);
  if (I == J && a < b) return;
  double v = 0.0;
  for (int s = 0; s < nseg; s++) v += part[((size_t)s * npairs + t) * 36 + e];
  if (joint) {
    const size_t r = 6 * (size_t)I + a, c = 6 * (size_t)J + b;
    cov[c * n6 + r] = v;
    cov[r * n6 + c] = v;
  } else {
    double *m = marg + 36 * ((size_t)u0 + t);
    m[6 * b + a] = v;
    m[6 * a + b] = v;
  }
}

}  // namespace

int cov_raw_blocks_dev(balm_ctx *c, ScratchPool &pool, const double *poses_dev, const double *ccov_host,
                       double point_noise, bool include_fix, double *raw) {
  const int N = c->N;
  const int64_t M = c->M, K = c->K;
  cudaStream_t st = c->stream;
  // voxel batches: every observation's 48 row entries of a batch within the budget, and at most the stats table's VB
  std::vector<long long> rp((size_t)M + 1);
  CUDA_TRY(cudaMemcpyAsync(rp.data(), c->row_ptr, sizeof(long long) * (M + 1), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  const long long max_obs = std::max<long long>(1, (long long)(cov_budget() / (48 * sizeof(double))));
  std::vector<int64_t> cut{0};
  long long rows_max = 0;
  while (cut.back() < M) {
    const int64_t v0 = cut.back();
    int64_t v1 = v0 + 1;
    while (v1 < M && v1 - v0 < c->VB && rp[v1 + 1] - rp[v0] <= max_obs) v1++;
    rows_max = std::max(rows_max, rp[v1] - rp[v0]);
    cut.push_back(v1);
  }
  int64_t vb = 0;
  for (size_t b = 1; b < cut.size(); b++) vb = std::max(vb, cut[b] - cut[b - 1]);
  double *rows = nullptr, *Wz = nullptr, *Dobs = nullptr, *Dacc = nullptr, *ccov = nullptr;
  TRY(pool.get(&rows, 48 * (size_t)rows_max));
  TRY(pool.get(&Wz, (size_t)vb * 10));
  TRY(pool.get(&Dobs, (size_t)K * 21));
  TRY(pool.get(&Dacc, (size_t)21 * N));
  if (ccov_host) {
    TRY(pool.get(&ccov, (size_t)K * 81));
    CUDA_TRY(cudaMemcpyAsync(ccov, ccov_host, sizeof(double) * (size_t)K * 81, cudaMemcpyHostToDevice, st));
  }
  for (size_t b = 1; b < cut.size(); b++) {
    const int64_t v0 = cut[b - 1], v1 = cut[b], nv = v1 - v0;
    const bool first = b == 1, last = b + 1 == cut.size();
    TRY(launch_csc_batch(c, v0, v1));
    double *rdummy = c->scal + 21;
    CUDA_TRY(cudaMemsetAsync(rdummy, 0, sizeof(double), st));
    TRY(launch_voxel_stats(c, poses_dev, v0, v1, c->stats, include_fix, rdummy));
    CovArgs a{c->obs, c->Kp, c->pose_idx, c->row_ptr, poses_dev, c->stats, ccov, point_noise * point_noise, v0, v1, N,
              6, Wz, rows, Dobs, rp[v0]};
    const unsigned grid = (unsigned)((nv + 3) / 4);
    cov_wz_kernel<<<grid, 128, 0, st>>>(a);
    cov_rows_kernel<true><<<grid, 128, 0, st>>>(a);
    cov_diag_reduce_kernel<<<N, 32, 0, st>>>(Dobs, N, M, c->dense ? 1 : 0, c->csc_ptr, c->csc_obs, Dacc, first ? 0 : 1, v0,
                                             v1, c->csc_lo, c->csc_hi);
    c->launches += 3;
    TRY(launch_raw_blocks(c, rows, v0, v1, last ? Dacc : nullptr, !first, raw));
  }
  TRY(launch_csc_batch(c, 0, M));
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

// columns per chunk (a multiple of 6) that fit the budget, 0 when not even one unknown's do
static int pc_chunk_cols(int P, int N, int n_sel, bool joint) {
  const size_t nseg = ((size_t)6 * N + PC_SEG - 1) / PC_SEG;
  const size_t per_col = sizeof(double) * ((size_t)6 * P + 12 * (size_t)N);
  const size_t budget = cov_budget();
  if (joint) {
    const size_t pairs = (size_t)n_sel * (n_sel + 1) / 2;
    const size_t need = per_col * 6 * n_sel + sizeof(double) * 36 * (pairs * nseg + (size_t)n_sel * n_sel);
    return need <= budget ? 6 * n_sel : 0;
  }
  const size_t per_unknown = 6 * per_col + sizeof(double) * 36 * nseg;
  const size_t avail = budget > sizeof(double) * 36 * (size_t)n_sel ? budget - sizeof(double) * 36 * (size_t)n_sel : 0;
  return 6 * (int)std::min<size_t>((size_t)n_sel, avail / per_unknown);
}

bool block_point_cov_fits(int P, int N, int n_sel, bool joint) { return pc_chunk_cols(P, N, n_sel, joint) > 0; }

int block_point_cov_dev(balm_ctx *c, SparseSolver *sp, const Rig *rig, const double *state, int anchor, int n_sel,
                        const int32_t *sel, const double *raw, double *cov_host, double *marg_host) {
  const int N = c->N, P = sparse_solver_size(sp);
  cudaStream_t st = c->stream;
  const bool joint = cov_host != nullptr;
  const std::vector<int> &col = sparse_solver_columns(sp);
  const int *pp_ptr = nullptr;
  const int2 *pp = nullptr;
  sparse_solver_pose_pairs(blocks_solver(c->bh), &pp_ptr, &pp);
  // the marginals alone go in chunks that fit the budget; the joint in one (checked by the caller)
  const int C = pc_chunk_cols(P, N, n_sel, joint);
  if (C == 0) {
    balm_set_error("point covariance: one unknown's right-hand sides exceed BALM_COV_BUDGET_MB");
    return BALM_ERR_UNSUPPORTED;
  }
  const int chunk = C / 6, nseg = (6 * N + PC_SEG - 1) / PC_SEG;
  const int max_pairs = joint ? n_sel * (n_sel + 1) / 2 : chunk;
  std::vector<int> selcol(n_sel);
  for (int u = 0; u < n_sel; u++) selcol[u] = col[sel[u]];
  ScratchPool pool;
  int *d_col = nullptr, *d_selcol = nullptr, *d_sel = nullptr;
  double *Y = nullptr, *W = nullptr, *Z = nullptr, *part = nullptr, *out = nullptr;
  TRY(pool.get(&d_col, (size_t)P));
  TRY(pool.get(&d_selcol, (size_t)n_sel));
  TRY(pool.get(&d_sel, (size_t)n_sel));
  TRY(pool.get(&Y, (size_t)6 * P * C));
  TRY(pool.get(&W, (size_t)6 * N * C));
  TRY(pool.get(&Z, (size_t)6 * N * C));
  TRY(pool.get(&part, (size_t)nseg * max_pairs * 36));
  TRY(pool.get(&out, joint ? (size_t)36 * n_sel * n_sel : (size_t)36 * n_sel));
  CUDA_TRY(cudaMemcpyAsync(d_col, col.data(), sizeof(int) * P, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(d_selcol, selcol.data(), sizeof(int) * n_sel, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(d_sel, sel, sizeof(int) * n_sel, cudaMemcpyHostToDevice, st));
  for (int u0 = 0; u0 < n_sel; u0 += chunk) {
    const int nu = std::min(chunk, n_sel - u0), nc = 6 * nu;
    const unsigned tiles = (unsigned)((nc + PC_TILE - 1) / PC_TILE);
    CUDA_TRY(cudaMemsetAsync(Y, 0, sizeof(double) * (size_t)6 * P * C, st));
    pc_unit_kernel<<<(6 * nu + 127) / 128, 128, 0, st>>>(d_selcol, u0, nu, C, Y);
    TRY(sparse_solve_many(sp, st, Y, C, nc, &c->launches));
    // the anchor's unit rows deleted: its entries are exactly 0
    if (anchor >= 0) CUDA_TRY(cudaMemsetAsync(Y + (size_t)6 * col[anchor] * C, 0, sizeof(double) * 6 * C, st));
    if (rig) TRY(rig_apply_j(rig, st, state, d_col, Y, C, nc, W, &c->launches));
    else pc_gather_kernel<<<dim3(tiles, N), 6 * PC_TILE, 0, st>>>(Y, d_col, C, nc, W);
    pc_rw_kernel<<<dim3(tiles, N), 6 * PC_TILE, 0, st>>>(raw, pp_ptr, pp, W, C, nc, Z);
    const int npairs = joint ? max_pairs : nu;
    pc_dot_kernel<<<dim3((npairs + 127) / 128, nseg), 128, 0, st>>>(W, Z, C, 6 * N, npairs, joint ? 1 : 0, d_sel,
                                                                    part);
    pc_reduce_kernel<<<(unsigned)((36LL * npairs + 255) / 256), 256, 0, st>>>(part, nseg, npairs, joint ? 1 : 0, d_sel,
                                                                             u0, 6 * n_sel, out, out);
    c->launches += 5 + (rig ? 0 : 1);
    CUDA_TRY(cudaGetLastError());
  }
  if (joint) {
    CUDA_TRY(cudaMemcpyAsync(cov_host, out, sizeof(double) * 36 * (size_t)n_sel * n_sel, cudaMemcpyDeviceToHost, st));
    if (marg_host)  // the joint's diagonal blocks
      for (int u = 0; u < n_sel; u++)
        for (int b = 0; b < 6; b++)
          CUDA_TRY(cudaMemcpyAsync(marg_host + 36 * (size_t)u + 6 * b, out + (6 * (size_t)u + b) * 6 * n_sel + 6 * u,
                                   sizeof(double) * 6, cudaMemcpyDeviceToHost, st));
  } else {
    CUDA_TRY(cudaMemcpyAsync(marg_host, out, sizeof(double) * 36 * (size_t)n_sel, cudaMemcpyDeviceToHost, st));
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  return BALM_OK;
}

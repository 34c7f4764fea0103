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

// pass 2: the eight rows of a voxel (c2 Q^T | c2 V^T) and the diagonal block c2^2 D_p of every observation
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
    cov_obs_rows(t, C, Wz, c2, a.G + (size_t)(8 * (v - a.v0)) * a.ldg + 6 * p, a.ldg, a.Dobs + (size_t)s * 21);
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

// Defined in balm_api.cu
int balm_cov_evaluate_hessian(balm_ctx *c, const double *poses_dev, bool include_fix);

int cov_raw_dev(balm_ctx *c, ScratchPool &pool, const double *poses_dev, const double *ccov_host, double point_noise,
                bool include_fix, double **R_out) {
  const int n = c->n, N = c->N;
  const int64_t M = c->M, K = c->K;
  cudaStream_t st = c->stream;
  // voxels per batch: the stats table holds VB voxels; the row buffer gets its own budget
  size_t budget = (size_t)4 << 30;
  if (const char *e = getenv("BALM_COV_BUDGET_MB")) budget = (size_t)atoll(e) << 20;
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
              c->ldg, Wz, G, Dobs};
    const unsigned grid = (unsigned)((nv + 3) / 4);
    cov_wz_kernel<<<grid, 128, 0, st>>>(a);
    cov_rows_kernel<<<grid, 128, 0, st>>>(a);
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

// Defined in balm_api.cu
int balm_cov_evaluate_hessian(balm_ctx *c, const double *poses_dev, bool include_fix);

int pose_covariance_dev(balm_ctx *c, const double *poses_dev, const double *ccov_host, double point_noise, bool include_fix,
                        double *Rraw_host, double *Rcov_host) {
  const int n = c->n;
  cudaStream_t st = c->stream;
  if (c->M < 1) { balm_set_error("balm_pose_covariance: no voxels registered"); return BALM_ERR_INVALID; }
  ScratchPool pool;
  double *R = nullptr;
  TRY(cov_raw_dev(c, pool, poses_dev, ccov_host, point_noise, include_fix, &R));
  if (Rraw_host) CUDA_TRY(cudaMemcpyAsync(Rraw_host, R, sizeof(double) * (size_t)n * n, cudaMemcpyDeviceToHost, st));
  if (Rcov_host) {
    // H at these poses (divide_thread, BAs_left.hpp:1091), factored without damping, then H^-1 R H^-T
    TRY(balm_cov_evaluate_hessian(c, poses_dev, include_fix));
    const DenseSystem sys = ctx_system(c);
    TRY(cov_factor(c, sys, -1,
                   "balm_pose_covariance: H is singular (gauge freedom not fixed: no fix clusters in the Hessian)"));
    TRY(cov_sandwich(c, sys, R));
    CUDA_TRY(cudaMemcpyAsync(Rcov_host, R, sizeof(double) * (size_t)n * n, cudaMemcpyDeviceToHost, st));
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  return BALM_OK;
}

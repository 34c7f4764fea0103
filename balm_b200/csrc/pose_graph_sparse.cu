// pose_graph_sparse.cu -- the block-sparse damped solve of the sparse pose graph (include/balm_b200.h, balm_spg_*;
// DESIGN.md "Pose graph", "Sparse solve"). A = H + u diag(H) over P poses, H the pose graph's 6x6 block pattern, is
// factored as P L D P^T (unit-lower L of 6x6 blocks, diagonal D, no pivoting) in a nested-dissection order, and
// (H + u diag(H)) dx = -g solved with it. Nothing of size (6P)^2 exists.
// Registration (host, once per factor set): the ordering, the elimination tree and its levels, every column's block
// rows, every block's update terms and every row's blocks; then the per-solve launch sequence is captured in a CUDA
// graph. fp64 throughout; every sum runs in a fixed order and there are no floating-point atomics, so solves repeat bit
// for bit.
//   spg_damp_kernel      per (block of L, entry): the pair's block of H (transposed when the order swaps it) or a
//                        zero fill block; diagonal blocks add u diag(H) and write diag(H)
//   spg_factor_kernel    per column of one elimination-tree level, one CTA: the column's blocks minus their update
//                        terms (a warp per block), the diagonal block's 6x6 LDL^T, the off-diagonal blocks scaled, then
//                        the column's forward substitution (FACTOR = false: the substitution only, for refinement)
//   spg_back_kernel      per column of one level, top level first, one warp: D^-1 and the backward substitution
//   spg_check_kernel     per row: r = -g - A dx over the pose's pairs in ascending order, the componentwise backward
//                        error omega (the dense solve's check, same tolerance)
// Marginal covariances (sparse_covariance; DESIGN.md "Marginal covariances"): H factored undamped with one pose held
// fixed, then the entries of H^-1 on L's pattern by selected inversion, gathered onto H's pattern.
//   spg_anchor_kernel    one CTA: the anchor's row and column of L's blocks zeroed, its diagonal block I
//   spg_selinv_kernel    per column of one level, top level first, one CTA: L^ = L L_jj^-1 in place, the column's Z
//                        blocks from its ancestors' (a warp per block), then its diagonal block
//   spg_cov_gather_kernel  per (pair, entry): Z's block of every pair of H
// Point-noise covariance on blocks contexts (sparse_solve_many; DESIGN.md "Point-noise covariance on blocks contexts"):
// the same undamped, anchored factorisation (sparse_factor_undamped), then many right-hand sides at once.
//   spg_fwd_many_kernel / spg_back_many_kernel  per (column of one level, tile of right-hand sides), one CTA: the
//                        forward / backward substitution of spg_factor_kernel<false> / spg_back_kernel, in place
#include <math.h>
#include <algorithm>
#include <memory>
#include <queue>
#include <vector>
#include "internal.cuh"

namespace {

constexpr int SP_THREADS = 512;
constexpr int SEL_THREADS = 256;  // spg_selinv_kernel: its 36-entry accumulators need more than 128 registers
constexpr int ND_LEAF = 32;  // nested dissection stops at this many poses; a leaf keeps index order

struct SpView {      // L and D as the level kernels read them
  const int *colptr;  // [P+1] blocks of column j: colptr[j] (the diagonal) .. colptr[j+1], rows ascending
  const int *rowidx;  // [nb] block row
  const int *lcol;    // [nb] block column
  const long long *tptr;  // [nb+1] update terms of every block
  const int2 *term;   // (position of L_ik, position of L_jk), ascending k
  const int *rptr, *rpos;  // [P+1] / [nb - P] off-diagonal blocks of every row, ascending column
  const int *perm;    // [P] pose of column j
  double *Lx;         // [nb][36] column-major blocks
  double *D;          // [6P]
  int *flags;
};

__device__ __forceinline__ bool bad_pivot(double d) { return !(fabs(d) > 1e-290 && fabs(d) < 1e300); }  // as ldlt.cu

__global__ void __launch_bounds__(256) spg_damp_kernel(const double *Hb, const int *lsrc, SpView v, long long nb,
                                                       const double *u_dev, double *dvec) {
  const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
  if (t >= 36 * nb) return;
  const long long b = t / 36;
  const int e = (int)(t % 36), a = e % 6, c = e / 6;
  const int s = lsrc[b];  // 2 pair + transposed, or -1
  double h = 0.0;
  if (s >= 0) h = Hb[36 * (size_t)(s >> 1) + ((s & 1) ? 6 * a + c : 6 * c + a)];
  const int j = v.lcol[b];
  if (b == v.colptr[j] && a == c) {
    dvec[6 * (size_t)v.perm[j] + a] = h;
    h += *u_dev * h;
  }
  v.Lx[t] = h;
}

// One CTA per column j of a level: every column L_jk it depends on belongs to a lower level (k is a descendant of j).
template <bool FACTOR>
__global__ void __launch_bounds__(SP_THREADS) spg_factor_kernel(SpView v, const int *cols, const double *rhs, double sgn,
                                                                double *y) {
  __shared__ double W[36], d[6], yj[6];
  const int j = cols[blockIdx.x], tid = threadIdx.x;
  const int b0 = v.colptr[j], b1 = v.colptr[j + 1];
  double *Ljj = v.Lx + 36 * (size_t)b0;
  if (FACTOR) {
    // W_ij = A_ij - sum_k L_ik D_k L_jk^T: one warp per block, lane l summing the terms l, l + 32, ... in ascending k,
    // then the lanes' sums in a fixed butterfly
    const int lane = tid & 31;
    for (int b = b0 + (tid >> 5); b < b1; b += SP_THREADS / 32) {
      double acc[36];
#pragma unroll
      for (int e = 0; e < 36; e++) acc[e] = 0.0;
      for (long long t = v.tptr[b] + lane; t < v.tptr[b + 1]; t += 32) {
        const int2 tk = v.term[t];
        const double *Li = v.Lx + 36 * (size_t)tk.x, *Lj = v.Lx + 36 * (size_t)tk.y, *Dk = v.D + 6 * (size_t)v.lcol[tk.x];
#pragma unroll
        for (int m = 0; m < 6; m++) {
          double li[6], lj[6];
          const double dk = Dk[m];
#pragma unroll
          for (int a = 0; a < 6; a++) {
            li[a] = Li[6 * m + a] * dk;
            lj[a] = Lj[6 * m + a];
          }
#pragma unroll
          for (int c = 0; c < 6; c++)
#pragma unroll
            for (int a = 0; a < 6; a++) acc[6 * c + a] = fma(li[a], lj[c], acc[6 * c + a]);
        }
      }
      double *Lb = v.Lx + 36 * (size_t)b;
#pragma unroll
      for (int e = 0; e < 36; e++) {
        const double s = Lb[e] - warp_sum(acc[e]);
        if (lane == (e & 31)) {
          if (b == b0) W[e] = s;
          else Lb[e] = s;
        }
      }
    }
    __syncthreads();
    if (tid == 0) {  // W_jj = L_jj D_j L_jj^T from its lower triangle, column by column
      bool bad = false;
      for (int m = 0; m < 6; m++) {
        double dm = W[7 * m];
        for (int p = 0; p < m; p++) dm -= W[6 * p + m] * W[6 * p + m] * d[p];
        bad = bad || bad_pivot(dm);
        d[m] = dm;
        for (int r = m + 1; r < 6; r++) {
          double s = W[6 * m + r];
          for (int p = 0; p < m; p++) s -= W[6 * p + r] * W[6 * p + m] * d[p];
          W[6 * m + r] = s / dm;
        }
      }
      for (int m = 0; m < 6; m++) {
        v.D[6 * (size_t)j + m] = d[m];
        for (int r = 0; r < 6; r++) Ljj[6 * m + r] = r == m ? 1.0 : r > m ? W[6 * m + r] : 0.0;
      }
      if (bad) atomicOr(&v.flags[0], 1);
    }
    __syncthreads();
    // L_ij D_j L_jj^T = W_ij, one thread per row of an off-diagonal block
    for (int q = tid; q < 6 * (b1 - b0 - 1); q += SP_THREADS) {
      double *B = v.Lx + 36 * (size_t)(b0 + 1 + q / 6);
      const int a = q % 6;
      double yr[6];
      for (int m = 0; m < 6; m++) {
        double s = B[6 * m + a];
        for (int p = 0; p < m; p++) s -= yr[p] * W[6 * p + m];
        yr[m] = s;
      }
      for (int m = 0; m < 6; m++) B[6 * m + a] = yr[m] / d[m];
    }
  }
  // y_j = L_jj^-1 (b_j - sum_k L_jk y_k), b = sgn rhs in pose order
  if (tid < 6) {
    double s = sgn * rhs[6 * (size_t)v.perm[j] + tid];
    for (int q = v.rptr[j]; q < v.rptr[j + 1]; q++) {
      const int p = v.rpos[q];
      const double *B = v.Lx + 36 * (size_t)p, *yk = y + 6 * (size_t)v.lcol[p];
      for (int m = 0; m < 6; m++) s -= B[6 * m + tid] * yk[m];
    }
    yj[tid] = s;
  }
  __syncthreads();
  if (tid == 0) {
    for (int m = 0; m < 6; m++) {
      double s = yj[m];
      for (int p = 0; p < m; p++) s -= Ljj[6 * p + m] * yj[p];
      yj[m] = s;
      y[6 * (size_t)j + m] = s;
    }
  }
}

// x_j = L_jj^-T (D_j^-1 y_j - sum_i L_ij^T x_i) over the column's off-diagonal blocks in ascending row order; x in
// column order, and into out in pose order (ACCUM: out += x, the refinement's correction)
template <bool ACCUM>
__global__ void __launch_bounds__(32) spg_back_kernel(SpView v, const int *cols, const double *y, double *x,
                                                      double *out) {
  __shared__ double z[6];
  const int j = cols[blockIdx.x], tid = threadIdx.x;
  const int b0 = v.colptr[j], b1 = v.colptr[j + 1];
  if (tid < 6) {
    double s = y[6 * (size_t)j + tid] / v.D[6 * (size_t)j + tid];
    for (int b = b0 + 1; b < b1; b++) {
      const double *B = v.Lx + 36 * (size_t)b, *xi = x + 6 * (size_t)v.rowidx[b];
      for (int c = 0; c < 6; c++) s -= B[6 * tid + c] * xi[c];
    }
    z[tid] = s;
  }
  __syncwarp();
  if (tid == 0) {
    const double *Ljj = v.Lx + 36 * (size_t)b0;
    const size_t o = 6 * (size_t)v.perm[j];
    for (int m = 5; m >= 0; m--) {
      double s = z[m];
      for (int p = m + 1; p < 6; p++) s -= Ljj[6 * m + p] * z[p];
      z[m] = s;
      x[6 * (size_t)j + m] = s;
      if (ACCUM) out[o + m] += s;
      else out[o + m] = s;
    }
  }
}

// the backward error of dx: row 6i + a of A dx over pose i's pairs (2 pair + transposed, other pose) in ascending order
__global__ void __launch_bounds__(256) spg_check_kernel(const double *Hb, const int *pp_ptr, const int2 *pp,
                                                        const double *g, const double *x, int P, const double *u_dev,
                                                        double tol, double *rres, int *flags, double *omega_out) {
  const int r = blockIdx.x * 256 + threadIdx.x;
  if (r >= 6 * P) return;
  const int i = r / 6, a = r % 6;
  const double u = *u_dev;
  double s = 0.0, sa = 0.0;
  for (int q = pp_ptr[i]; q < pp_ptr[i + 1]; q++) {
    const int2 e = pp[q];
    const double *B = Hb + 36 * (size_t)(e.x >> 1);
    for (int c = 0; c < 6; c++) {
      double h = B[(e.x & 1) ? 6 * a + c : 6 * c + a];
      if (e.y == i && c == a) h += u * h;
      const double t = h * x[6 * (size_t)e.y + c];
      s += t;
      sa += fabs(t);
    }
  }
  const double b = -g[r], res = b - s, den = sa + fabs(b);
  rres[r] = res;
  const double om = den > 0.0 ? fabs(res) / den : 0.0;
  if (!(om <= tol)) atomicOr(&flags[4], 1);
  atomicMax(reinterpret_cast<unsigned long long *>(omega_out), (unsigned long long)__double_as_longlong(om));
}

// The covariance's anchored copy: after spg_damp_kernel with u = 0, every block of column ac and of row ac becomes 0 and
// the diagonal block I, so that the factorisation is that of H without the anchor's rows and columns (one CTA).
__global__ void __launch_bounds__(256) spg_anchor_kernel(SpView v, int ac) {
  const int c0 = v.colptr[ac], nc = v.colptr[ac + 1] - c0, r0 = v.rptr[ac], nr = v.rptr[ac + 1] - r0;
  for (int t = threadIdx.x; t < 36 * (nc + nr); t += 256) {
    const int q = t / 36, e = t % 36;
    const int b = q < nc ? c0 + q : v.rpos[r0 + q - nc];
    v.Lx[36 * (size_t)b + e] = (b == c0 && e % 7 == 0) ? 1.0 : 0.0;
  }
}

// Selected inversion (Takahashi), one CTA per column j of a level, top level first: with L^_kj = L_kj L_jj^-1 and
// S = struct(j),
//   Z_ij = -sum_{k in S} Z_ik L^_kj   (i in S),      Z_jj = L_jj^-T D_j^-1 L_jj^-1 - sum_{k in S} L^_kj^T Z_kj,
// where every Z_ik belongs to an ancestor column (S is a clique of L's pattern). Block t of the column's off-diagonal
// blocks sums the terms sterm[sptr[j] + t m + u], u = 0 .. m - 1 (ascending k = S[u]): 2 position of Z_ik's block
// (max, min) + transposed; L^_kj is the column's block 1 + u. L_Sj is overwritten with L^_Sj (nothing else reads it
// before the next factorisation).
__global__ void __launch_bounds__(SEL_THREADS) spg_selinv_kernel(SpView v, const int *cols, const long long *sptr,
                                                                const int *sterm, double *Z) {
  __shared__ double Minv[36], S[36];
  const int j = cols[blockIdx.x], tid = threadIdx.x, lane = tid & 31;
  const int b0 = v.colptr[j], m = v.colptr[j + 1] - b0 - 1;
  const double *Ljj = v.Lx + 36 * (size_t)b0;
  // L^_kj: x L_jj = b for every row b of an off-diagonal block, one thread per row
  for (int q = tid; q < 6 * m; q += SEL_THREADS) {
    double *B = v.Lx + 36 * (size_t)(b0 + 1 + q / 6);
    const int a = q % 6;
    double x[6];
#pragma unroll
    for (int c = 5; c >= 0; c--) {
      double s = B[6 * c + a];
#pragma unroll
      for (int r = c + 1; r < 6; r++) s -= x[r] * Ljj[6 * c + r];
      x[c] = s;
    }
#pragma unroll
    for (int c = 0; c < 6; c++) B[6 * c + a] = x[c];
  }
  if (tid == SEL_THREADS - 1) {  // L_jj^-1, unit lower, column-major
    for (int c = 0; c < 6; c++)
      for (int r = 0; r < 6; r++) {
        double s = r == c ? 1.0 : 0.0;
        for (int p = c; p < r; p++) s -= Ljj[6 * p + r] * Minv[6 * c + p];
        Minv[6 * c + r] = r < c ? 0.0 : s;
      }
  }
  __syncthreads();
  // Z_ij: one warp per block, lane l summing the terms l, l + 32, ..., then the lanes' sums in a fixed butterfly
  for (int t = tid >> 5; t < m; t += SEL_THREADS / 32) {
    double acc[36];
#pragma unroll
    for (int e = 0; e < 36; e++) acc[e] = 0.0;
    const int *w = sterm + sptr[j] + (long long)t * m;
    for (int u = lane; u < m; u += 32) {
      const int x = w[u];
      const double *Zk = Z + 36 * (size_t)(x >> 1), *Lk = v.Lx + 36 * (size_t)(b0 + 1 + u);
      const int sa = (x & 1) ? 6 : 1, sp = (x & 1) ? 1 : 6;  // Z_ik[a][p] = Zk[sa a + sp p]
#pragma unroll
      for (int p = 0; p < 6; p++) {
        double zi[6], lk[6];
#pragma unroll
        for (int a = 0; a < 6; a++) {
          zi[a] = Zk[sa * a + sp * p];
          lk[a] = Lk[6 * a + p];
        }
#pragma unroll
        for (int c = 0; c < 6; c++)
#pragma unroll
          for (int a = 0; a < 6; a++) acc[6 * c + a] = fma(zi[a], lk[c], acc[6 * c + a]);
      }
    }
    double *Zb = Z + 36 * (size_t)(b0 + 1 + t);
#pragma unroll
    for (int e = 0; e < 36; e++) {
      const double s = -warp_sum(acc[e]);
      if (lane == (e & 31)) Zb[e] = s;
    }
  }
  __syncthreads();
  // sum_k L^_kj^T Z_kj over the column's blocks by warp 0, the same lane split and butterfly
  if (tid < 32) {
    double acc[36];
#pragma unroll
    for (int e = 0; e < 36; e++) acc[e] = 0.0;
    for (int u = lane; u < m; u += 32) {
      const double *Lk = v.Lx + 36 * (size_t)(b0 + 1 + u), *Zk = Z + 36 * (size_t)(b0 + 1 + u);
#pragma unroll
      for (int p = 0; p < 6; p++) {
        double lk[6], zk[6];
#pragma unroll
        for (int a = 0; a < 6; a++) {
          lk[a] = Lk[6 * a + p];
          zk[a] = Zk[6 * a + p];
        }
#pragma unroll
        for (int c = 0; c < 6; c++)
#pragma unroll
          for (int a = 0; a < 6; a++) acc[6 * c + a] = fma(lk[a], zk[c], acc[6 * c + a]);
      }
    }
#pragma unroll
    for (int e = 0; e < 36; e++) {
      const double s = warp_sum(acc[e]);
      if (lane == (e & 31)) S[e] = s;
    }
  }
  __syncthreads();
  if (tid < 36) {  // entry (hi, lo) of the lower triangle into both of its places: exactly symmetric
    const int a = tid % 6, c = tid / 6, hi = a > c ? a : c, lo = a > c ? c : a;
    double e = 0.0;
    for (int r = hi; r < 6; r++) e += Minv[6 * hi + r] * Minv[6 * lo + r] / v.D[6 * (size_t)j + r];
    Z[36 * (size_t)b0 + tid] = e - S[6 * lo + hi];
  }
}

// Many right-hand sides (sparse_solve_many): Y [6P rows in column order][ld], row-major, one CTA per (column j of a
// level, tile of MANY_TILE right-hand sides), thread (row a of the column, right-hand side c). Every right-hand side is
// summed in the single-RHS kernels' order, independently of the tile it lands in.
constexpr int MANY_TILE = 32;
//   forward: y_j = L_jj^-1 (y_j - sum_k L_jk y_k) over row j's off-diagonal blocks in ascending column
__global__ void __launch_bounds__(6 * MANY_TILE) spg_fwd_many_kernel(SpView v, const int *cols, double *Y, int ld,
                                                                     int ncols) {
  __shared__ double sy[6][MANY_TILE];
  const int j = cols[blockIdx.x], a = threadIdx.x / MANY_TILE, ci = threadIdx.x % MANY_TILE;
  const int c = blockIdx.y * MANY_TILE + ci;
  if (c < ncols) {
    double s = Y[(6 * (size_t)j + a) * ld + c];
    for (int q = v.rptr[j]; q < v.rptr[j + 1]; q++) {
      const int p = v.rpos[q];
      const double *B = v.Lx + 36 * (size_t)p, *yk = Y + 6 * (size_t)v.lcol[p] * ld + c;
      for (int m = 0; m < 6; m++) s -= B[6 * m + a] * yk[(size_t)m * ld];
    }
    sy[a][ci] = s;
  }
  __syncthreads();
  if (a == 0 && c < ncols) {
    const double *Ljj = v.Lx + 36 * (size_t)v.colptr[j];
    double y[6];
    for (int m = 0; m < 6; m++) {
      double s = sy[m][ci];
      for (int p = 0; p < m; p++) s -= Ljj[6 * p + m] * y[p];
      y[m] = s;
      Y[(6 * (size_t)j + m) * ld + c] = s;
    }
  }
}
//   backward: x_j = L_jj^-T (D_j^-1 y_j - sum_i L_ij^T x_i) over the column's off-diagonal blocks in ascending row
__global__ void __launch_bounds__(6 * MANY_TILE) spg_back_many_kernel(SpView v, const int *cols, double *Y, int ld,
                                                                      int ncols) {
  __shared__ double sz[6][MANY_TILE];
  const int j = cols[blockIdx.x], a = threadIdx.x / MANY_TILE, ci = threadIdx.x % MANY_TILE;
  const int c = blockIdx.y * MANY_TILE + ci;
  const int b0 = v.colptr[j], b1 = v.colptr[j + 1];
  if (c < ncols) {
    double s = Y[(6 * (size_t)j + a) * ld + c] / v.D[6 * (size_t)j + a];
    for (int b = b0 + 1; b < b1; b++) {
      const double *B = v.Lx + 36 * (size_t)b, *xi = Y + 6 * (size_t)v.rowidx[b] * ld + c;
      for (int cc = 0; cc < 6; cc++) s -= B[6 * a + cc] * xi[(size_t)cc * ld];
    }
    sz[a][ci] = s;
  }
  __syncthreads();
  if (a == 0 && c < ncols) {
    const double *Ljj = v.Lx + 36 * (size_t)b0;
    double z[6];
    for (int m = 5; m >= 0; m--) {
      double s = sz[m][ci];
      for (int p = m + 1; p < 6; p++) s -= Ljj[6 * m + p] * z[p];
      z[m] = s;
      Y[(6 * (size_t)j + m) * ld + c] = s;
    }
  }
}

// cov, per (pair, entry): the pair's block of Z (zsrc: 2 position + transposed, the inverse of lsrc); 0 on the anchor
// column ac's row and column
__global__ void __launch_bounds__(256) spg_cov_gather_kernel(const double *Z, const int *zsrc, SpView v, long long npairs,
                                                             int ac, double *cov) {
  const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
  if (t >= 36 * npairs) return;
  const int s = zsrc[t / 36], e = (int)(t % 36), r = e % 6, c = e / 6, pos = s >> 1;
  const double z = Z[36 * (size_t)pos + ((s & 1) ? 6 * r + c : 6 * c + r)];
  cov[t] = (v.rowidx[pos] == ac || v.lcol[pos] == ac) ? 0.0 : z;
}

// ---- ordering: nested dissection of the pose graph (xadj / adj: CSR of every pose's neighbours) ----
// A vertex set (ascending pose index) of more than ND_LEAF poses is cut at its median index; the separator is a greedy
// vertex cover of the crossing edges (most uncovered crossing edges first, the lower index on a tie). The two halves
// without it are ordered recursively, then the separator in ascending index.
void nd_order(const std::vector<int> &V, const std::vector<long long> &xadj, const std::vector<int> &adj,
              std::vector<int> &side, std::vector<int> &cnt, std::vector<int> &order) {
  if ((int)V.size() <= ND_LEAF) {
    order.insert(order.end(), V.begin(), V.end());
    return;
  }
  const size_t h = V.size() / 2;
  for (size_t q = 0; q < V.size(); q++) side[V[q]] = q < h ? 1 : 2;
  std::priority_queue<std::pair<int, int>> heap;  // (crossing edges, -pose)
  for (int v : V) {
    int n = 0;
    for (long long q = xadj[v]; q < xadj[v + 1]; q++) n += side[adj[q]] == 3 - side[v];
    cnt[v] = n;
    if (n) heap.push({n, -v});
  }
  std::vector<int> sep;
  while (!heap.empty()) {
    const int n = heap.top().first, v = -heap.top().second;
    heap.pop();
    if (side[v] == 0 || cnt[v] == 0) continue;
    if (n != cnt[v]) { heap.push({cnt[v], -v}); continue; }
    const int sv = side[v];
    side[v] = 0;  // separator
    sep.push_back(v);
    for (long long q = xadj[v]; q < xadj[v + 1]; q++)
      if (side[adj[q]] == 3 - sv) cnt[adj[q]]--;
  }
  std::vector<int> left, right;
  for (int v : V) {
    if (side[v] == 1) left.push_back(v);
    else if (side[v] == 2) right.push_back(v);
    side[v] = -1;
  }
  std::sort(sep.begin(), sep.end());
  nd_order(left, xadj, adj, side, cnt, order);
  nd_order(right, xadj, adj, side, cnt, order);
  order.insert(order.end(), sep.begin(), sep.end());
}

}  // namespace

struct SparseSolver {
  int P = 0;
  long long nb = 0, nterm = 0, bytes = 0;
  std::vector<int> lev_ptr;  // host: level l's columns are levcols[lev_ptr[l] .. lev_ptr[l+1])
  int *perm = nullptr, *colptr = nullptr, *rowidx = nullptr, *lcol = nullptr, *lsrc = nullptr, *rptr = nullptr,
      *rpos = nullptr, *levcols = nullptr, *pp_ptr = nullptr;
  long long *tptr = nullptr;
  int2 *term = nullptr, *pp = nullptr;
  double *Lx = nullptr, *D = nullptr, *y = nullptr, *xs = nullptr, *rres = nullptr;
  const double *Hb = nullptr, *g = nullptr;
  double *dvec = nullptr, *dx = nullptr, *scal = nullptr;
  int *flags = nullptr;
  cudaGraphExec_t exec = nullptr;
  // selected inversion (sparse_covariance), built by its first call: terms of every column (sptr [P+1], sterm), the
  // inverse of lsrc (zsrc [pairs]), Z [nb][36], and on the host the column of every pose
  long long npairs = 0, nsel = 0;
  long long *sptr = nullptr;
  int *sterm = nullptr, *zsrc = nullptr;
  double *Z = nullptr;
  std::vector<int> col_of;
  ~SparseSolver() {
    if (exec) cudaGraphExecDestroy(exec);
    cudaFree(perm); cudaFree(colptr); cudaFree(rowidx); cudaFree(lcol); cudaFree(lsrc); cudaFree(rptr); cudaFree(rpos);
    cudaFree(levcols); cudaFree(pp_ptr); cudaFree(tptr); cudaFree(term); cudaFree(pp); cudaFree(Lx); cudaFree(D);
    cudaFree(y); cudaFree(xs); cudaFree(rres); cudaFree(sptr); cudaFree(sterm); cudaFree(zsrc); cudaFree(Z);
  }
  SpView view() const { return SpView{colptr, rowidx, lcol, tptr, term, rptr, rpos, perm, Lx, D, flags}; }
  template <typename T>
  int alloc(T **p, size_t count) {
    TRY(dev_alloc(p, count));
    bytes += (long long)(sizeof(T) * (count ? count : 1));
    return BALM_OK;
  }
  template <typename T>
  int put(T **p, const std::vector<T> &h, cudaStream_t st) {
    TRY(alloc(p, h.size()));
    if (!h.empty()) CUDA_TRY(cudaMemcpyAsync(*p, h.data(), sizeof(T) * h.size(), cudaMemcpyHostToDevice, st));
    return BALM_OK;
  }
};

void sparse_solver_free(SparseSolver *s) { delete s; }

void sparse_solver_stats(const SparseSolver *s, int64_t *l_blocks, int64_t *levels, int64_t *bytes) {
  *l_blocks = s->nb;
  *levels = (int64_t)s->lev_ptr.size() - 1;
  *bytes = s->bytes;
}

static int too_large(const char *who, const char *what) {
  balm_set_error(std::string(who) + ": " + what);
  return BALM_ERR_UNSUPPORTED;
}

// The forward sweep over the levels upwards, then the backward sweep downwards (enqueued).
template <bool REFINE>
static int enqueue_substitutions(SparseSolver &s, cudaStream_t st, const double *rhs, double sgn, double *out) {
  const SpView v = s.view();
  const int nlev = (int)s.lev_ptr.size() - 1;
  for (int l = 0; l < nlev; l++)
    spg_factor_kernel<!REFINE><<<s.lev_ptr[l + 1] - s.lev_ptr[l], SP_THREADS, 0, st>>>(v, s.levcols + s.lev_ptr[l], rhs,
                                                                                       sgn, s.y);
  for (int l = nlev - 1; l >= 0; l--)
    spg_back_kernel<REFINE><<<s.lev_ptr[l + 1] - s.lev_ptr[l], 32, 0, st>>>(v, s.levcols + s.lev_ptr[l], s.y, s.xs, out);
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

static int enqueue_check(SparseSolver &s, cudaStream_t st) {
  CUDA_TRY(cudaMemsetAsync(s.scal + 20, 0, sizeof(double), st));
  spg_check_kernel<<<(6 * s.P + 255) / 256, 256, 0, st>>>(s.Hb, s.pp_ptr, s.pp, s.g, s.dx, s.P, s.scal + 3,
                                                          SOLVE_OMEGA_TOL, s.rres, s.flags, s.scal + 20);
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int sparse_solver_build(cudaStream_t st, int P, const std::vector<int2> &pairs, const double *blocks, const double *g,
                        double *dvec, double *dx, double *scal, int *flags, const char *who, SparseSolver **out) {
  std::unique_ptr<SparseSolver> s(new SparseSolver());
  s->P = P;
  const long long npairs = (long long)pairs.size();
  s->npairs = npairs;
  if (npairs >= (1LL << 30)) return too_large(who, "too many block pairs");
  // the pose graph's adjacency
  std::vector<long long> xadj(P + 1, 0);
  for (const int2 &p : pairs)
    if (p.x != p.y) { xadj[p.x + 1]++; xadj[p.y + 1]++; }
  for (int i = 0; i < P; i++) xadj[i + 1] += xadj[i];
  std::vector<int> adj(xadj[P]);
  {
    std::vector<long long> fill(xadj.begin(), xadj.end() - 1);
    for (const int2 &p : pairs)
      if (p.x != p.y) { adj[fill[p.x]++] = p.y; adj[fill[p.y]++] = p.x; }
  }
  // ordering: order[k] = the pose of column k
  std::vector<int> order, iperm(P), V(P), side(P, -1), cnt(P, 0);
  order.reserve(P);
  for (int i = 0; i < P; i++) V[i] = i;
  nd_order(V, xadj, adj, side, cnt, order);
  for (int k = 0; k < P; k++) iperm[order[k]] = k;
  // symbolic factorisation: struct(j) = {i > j : A_ij != 0} united with struct(c) \ {j} of j's children c
  std::vector<std::vector<int>> cstruct(P), children(P);
  std::vector<int> mark(P, -1), level(P, 0);
  for (int j = 0; j < P; j++) {
    std::vector<int> &rows = cstruct[j];
    const int pj = order[j];
    for (long long q = xadj[pj]; q < xadj[pj + 1]; q++) {
      const int i = iperm[adj[q]];
      if (i > j && mark[i] != j) { mark[i] = j; rows.push_back(i); }
    }
    for (int c : children[j]) {
      level[j] = std::max(level[j], level[c] + 1);
      for (int i : cstruct[c])
        if (i > j && mark[i] != j) { mark[i] = j; rows.push_back(i); }
    }
    std::sort(rows.begin(), rows.end());
    if (!rows.empty()) children[rows[0]].push_back(j);  // the elimination tree's parent
  }
  // L's blocks: column j holds its diagonal block, then struct(j) ascending
  std::vector<int> colptr(P + 1, 0);
  for (int j = 0; j < P; j++) {
    const long long n = (long long)colptr[j] + 1 + (long long)cstruct[j].size();
    if (n >= (1LL << 31) / 36) return too_large(who, "too many blocks of L");
    colptr[j + 1] = (int)n;
  }
  const long long nb = colptr[P];
  s->nb = nb;
  std::vector<int> rowidx(nb), lcol(nb), lsrc(nb, -1), rcnt(P + 1, 0);
  for (int j = 0; j < P; j++) {
    rowidx[colptr[j]] = j;
    lcol[colptr[j]] = j;
    for (size_t q = 0; q < cstruct[j].size(); q++) {
      rowidx[colptr[j] + 1 + q] = cstruct[j][q];
      lcol[colptr[j] + 1 + q] = j;
      rcnt[cstruct[j][q] + 1]++;
    }
  }
  // where every pair of H lands in L: block (max, min) of its two columns, transposed when the pair's first pose comes
  // later in the order
  for (long long p = 0; p < npairs; p++) {
    const int a = iperm[pairs[p].x], b = iperm[pairs[p].y];
    const int col = std::min(a, b), row = std::max(a, b);
    const int *r0 = rowidx.data() + colptr[col], *r1 = rowidx.data() + colptr[col + 1];
    const int pos = (int)(std::lower_bound(r0, r1, row) - rowidx.data());
    lsrc[pos] = (int)(2 * p + (a < b ? 1 : 0));
  }
  // every row's off-diagonal blocks, ascending column
  std::vector<int> rptr(P + 1, 0), rpos(nb - P);
  for (int i = 0; i < P; i++) rptr[i + 1] = rptr[i] + rcnt[i + 1];
  {
    std::vector<int> fill(rptr.begin(), rptr.end() - 1);
    for (int k = 0; k < P; k++)
      for (int b = colptr[k] + 1; b < colptr[k + 1]; b++) rpos[fill[rowidx[b]]++] = b;
  }
  // update terms: column k contributes L_ik D_k L_jk^T to block (i, j) for every i >= j in struct(k); struct(k) above j
  // lies in column j's rows (the elimination tree), so one merge walk finds every block. Two passes: count, fill, both
  // over k ascending, so that every block's terms are in ascending k.
  std::vector<long long> tptr(nb + 1, 0);
  for (int pass = 0; pass < 2; pass++) {
    std::vector<long long> fill;
    std::vector<int2> term;
    if (pass == 1) {
      for (long long b = 0; b < nb; b++) tptr[b + 1] += tptr[b];
      s->nterm = tptr[nb];
      fill.assign(tptr.begin(), tptr.end() - 1);
      term.resize(s->nterm);
    }
    for (int k = 0; k < P; k++) {
      const int k0 = colptr[k] + 1, m = colptr[k + 1] - k0;
      for (int u = 0; u < m; u++) {
        const int j = rowidx[k0 + u];
        int q = colptr[j];
        for (int t = u; t < m; t++) {
          const int i = rowidx[k0 + t];
          while (rowidx[q] != i) q++;
          if (pass == 0) tptr[q + 1]++;
          else term[fill[q]++] = make_int2(k0 + t, k0 + u);
        }
      }
    }
    if (pass == 1) TRY(s->put(&s->term, term, st));
  }
  // the levels, columns ascending inside a level
  const int nlev = P ? 1 + *std::max_element(level.begin(), level.end()) : 0;
  std::vector<int> lev_ptr(nlev + 1, 0), levcols(P);
  for (int j = 0; j < P; j++) lev_ptr[level[j] + 1]++;
  for (int l = 0; l < nlev; l++) lev_ptr[l + 1] += lev_ptr[l];
  {
    std::vector<int> fill(lev_ptr.begin(), lev_ptr.end() - 1);
    for (int j = 0; j < P; j++) levcols[fill[level[j]]++] = j;
  }
  s->lev_ptr = lev_ptr;
  // every pose's pairs for the residual check, ascending in the other pose
  std::vector<int> pp_ptr(P + 1, 0);
  for (const int2 &p : pairs) {
    pp_ptr[p.x + 1]++;
    if (p.x != p.y) pp_ptr[p.y + 1]++;
  }
  for (int i = 0; i < P; i++) pp_ptr[i + 1] += pp_ptr[i];
  std::vector<int2> pp(pp_ptr[P]);
  {
    std::vector<int> fill(pp_ptr.begin(), pp_ptr.end() - 1);
    for (long long p = 0; p < npairs; p++) {
      pp[fill[pairs[p].x]++] = make_int2((int)(2 * p), pairs[p].y);
      if (pairs[p].x != pairs[p].y) pp[fill[pairs[p].y]++] = make_int2((int)(2 * p + 1), pairs[p].x);
    }
    for (int i = 0; i < P; i++)
      std::sort(pp.begin() + pp_ptr[i], pp.begin() + pp_ptr[i + 1], [](const int2 &a, const int2 &b) { return a.y < b.y; });
  }
  TRY(s->put(&s->perm, order, st));
  TRY(s->put(&s->colptr, colptr, st));
  TRY(s->put(&s->rowidx, rowidx, st));
  TRY(s->put(&s->lcol, lcol, st));
  TRY(s->put(&s->lsrc, lsrc, st));
  TRY(s->put(&s->tptr, tptr, st));
  TRY(s->put(&s->rptr, rptr, st));
  TRY(s->put(&s->rpos, rpos, st));
  TRY(s->put(&s->levcols, levcols, st));
  TRY(s->put(&s->pp_ptr, pp_ptr, st));
  TRY(s->put(&s->pp, pp, st));
  TRY(s->alloc(&s->Lx, 36 * (size_t)nb));
  TRY(s->alloc(&s->D, 6 * (size_t)P));
  TRY(s->alloc(&s->y, 6 * (size_t)P));
  TRY(s->alloc(&s->xs, 6 * (size_t)P));
  TRY(s->alloc(&s->rres, 6 * (size_t)P));
  CUDA_TRY(cudaStreamSynchronize(st));  // the host tables above are freed on return
  s->Hb = blocks;
  s->g = g;
  s->dvec = dvec;
  s->dx = dx;
  s->scal = scal;
  s->flags = flags;
  // the per-solve launch sequence as one graph: 2 levels + 4 launches and 3 memsets per solve
  cudaGraph_t graph = nullptr;
  CUDA_TRY(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  int rc = BALM_OK;
  if (cudaMemsetAsync(flags, 0, sizeof(int) * 8, st) != cudaSuccess) rc = BALM_ERR_CUDA;
  if (rc == BALM_OK && nb)
    spg_damp_kernel<<<(unsigned)((36 * nb + 255) / 256), 256, 0, st>>>(blocks, s->lsrc, s->view(), nb, scal + 3, dvec);
  if (rc == BALM_OK) rc = enqueue_substitutions<false>(*s, st, g, -1.0, dx);
  if (rc == BALM_OK) rc = launch_q1(st, dx, g, dvec, 6 * P, scal + 3, scal);
  if (rc == BALM_OK) rc = enqueue_check(*s, st);
  const cudaError_t ce = cudaStreamEndCapture(st, &graph);
  if (rc != BALM_OK) { if (graph) cudaGraphDestroy(graph); return rc; }
  CUDA_TRY(ce);
  const cudaError_t ie = cudaGraphInstantiate(&s->exec, graph, 0);
  cudaGraphDestroy(graph);
  CUDA_TRY(ie);
  *out = s.release();
  return BALM_OK;
}

int sparse_solve(SparseSolver *s, cudaStream_t st) {
  CUDA_TRY(cudaGraphLaunch(s->exec, st));
  return BALM_OK;
}

int sparse_refine(SparseSolver *s, cudaStream_t st, int *h_flags, double *h_scal, int *still_bad) {
  *still_bad = 1;
  for (int round = 0; round < 3; round++) {
    // A delta = r with the same factors, dx += delta
    TRY(enqueue_substitutions<true>(*s, st, s->rres, 1.0, s->dx));
    TRY(launch_q1(st, s->dx, s->g, s->dvec, 6 * s->P, s->scal + 3, s->scal));
    CUDA_TRY(cudaMemsetAsync(s->flags + 4, 0, sizeof(int), st));
    TRY(enqueue_check(*s, st));
    CUDA_TRY(cudaMemcpyAsync(h_flags + 4, s->flags + 4, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(h_scal + 1, s->scal + 1, sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (h_flags[4] == 0) { *still_bad = 0; break; }
  }
  return BALM_OK;
}

// The selected inversion's tables from the registered structure (host, once): column k with S = struct(k), m = |S|,
// gives its block t the terms u = 0 .. m - 1 at sptr[k] + t m + u: the position of block (S[max(t,u)], S[min(t,u)])
// (found by the factor table's merge walk down column S[min]) times 2, + 1 when t < u (Z_ik read transposed).
static int selinv_build(SparseSolver &s, cudaStream_t st, const char *who) {
  const int P = s.P;
  const long long nb = s.nb;
  std::vector<int> colptr(P + 1), rowidx(nb), lsrc(nb), perm(P);
  CUDA_TRY(cudaMemcpyAsync(colptr.data(), s.colptr, sizeof(int) * (P + 1), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(rowidx.data(), s.rowidx, sizeof(int) * nb, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(lsrc.data(), s.lsrc, sizeof(int) * nb, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(perm.data(), s.perm, sizeof(int) * P, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  std::vector<long long> sptr(P + 1, 0);
  for (int k = 0; k < P; k++) {
    const long long m = colptr[k + 1] - colptr[k] - 1;
    sptr[k + 1] = sptr[k] + m * m;
  }
  const long long nsel = sptr[P];
  // int positions of Z (< 2^31 / 36, packed with the flag) are always in range; the count is what can outgrow a card
  if (nsel >= (1LL << 33)) return too_large(who, "2^33 or more selected-inversion terms");
  std::vector<int> sterm(nsel), zsrc(s.npairs);
  for (int k = 0; k < P; k++) {
    const int k0 = colptr[k] + 1, m = colptr[k + 1] - k0;
    int *w = sterm.data() + sptr[k];
    for (int u = 0; u < m; u++) {
      int q = colptr[rowidx[k0 + u]];
      for (int t = u; t < m; t++) {
        while (rowidx[q] != rowidx[k0 + t]) q++;
        w[(size_t)t * m + u] = 2 * q;
        if (t != u) w[(size_t)u * m + t] = 2 * q + 1;
      }
    }
  }
  for (long long b = 0; b < nb; b++)
    if (lsrc[b] >= 0) zsrc[lsrc[b] >> 1] = (int)(2 * b + (lsrc[b] & 1));
  s.col_of.assign(P, 0);
  for (int j = 0; j < P; j++) s.col_of[perm[j]] = j;
  ScratchPool pool;  // nothing is kept unless every allocation succeeds
  long long *d_sptr = nullptr;
  int *d_sterm = nullptr, *d_zsrc = nullptr;
  double *d_Z = nullptr;
  long long bytes = 0;
  auto get = [&](auto **p, size_t n) {
    bytes += (long long)(sizeof(**p) * (n ? n : 1));
    return pool.get(p, n);
  };
  TRY(get(&d_sptr, sptr.size()));
  TRY(get(&d_sterm, sterm.size()));
  TRY(get(&d_zsrc, zsrc.size()));
  TRY(get(&d_Z, 36 * (size_t)nb));
  CUDA_TRY(cudaMemcpyAsync(d_sptr, sptr.data(), sizeof(long long) * sptr.size(), cudaMemcpyHostToDevice, st));
  if (nsel) CUDA_TRY(cudaMemcpyAsync(d_sterm, sterm.data(), sizeof(int) * nsel, cudaMemcpyHostToDevice, st));
  if (s.npairs) CUDA_TRY(cudaMemcpyAsync(d_zsrc, zsrc.data(), sizeof(int) * zsrc.size(), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaStreamSynchronize(st));  // the host tables are freed on return
  for (void *q : {(void *)d_sptr, (void *)d_sterm, (void *)d_zsrc, (void *)d_Z}) pool.release(q);
  s.sptr = d_sptr;
  s.sterm = d_sterm;
  s.zsrc = d_zsrc;
  s.Z = d_Z;
  s.nsel = nsel;
  s.bytes += bytes;
  return BALM_OK;
}

// The column of every pose, on the host (once)
static int col_of_build(SparseSolver &s, cudaStream_t st) {
  if ((int)s.col_of.size() == s.P) return BALM_OK;
  std::vector<int> perm(s.P);
  CUDA_TRY(cudaMemcpyAsync(perm.data(), s.perm, sizeof(int) * s.P, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  s.col_of.assign(s.P, 0);
  for (int j = 0; j < s.P; j++) s.col_of[perm[j]] = j;
  return BALM_OK;
}

int sparse_factor_undamped(SparseSolver *s, cudaStream_t st, int anchor, const char *who, long long *launches) {
  TRY(col_of_build(*s, st));
  const SpView v = s->view();
  const int P = s->P, nlev = (int)s->lev_ptr.size() - 1, ac = anchor >= 0 ? s->col_of[anchor] : -1;
  // the undamped copy (u = 0 in scal[3]; the next solve writes its own), the anchor's blocks, the factorisation (its
  // forward substitution on g runs into the scratch y)
  CUDA_TRY(cudaMemsetAsync(s->flags, 0, sizeof(int) * 8, st));
  CUDA_TRY(cudaMemsetAsync(s->scal + 3, 0, sizeof(double), st));
  if (s->nb) spg_damp_kernel<<<(unsigned)((36 * s->nb + 255) / 256), 256, 0, st>>>(s->Hb, s->lsrc, v, s->nb, s->scal + 3,
                                                                                   s->dvec);
  if (ac >= 0) spg_anchor_kernel<<<1, 256, 0, st>>>(v, ac);
  for (int l = 0; l < nlev; l++)
    spg_factor_kernel<true><<<s->lev_ptr[l + 1] - s->lev_ptr[l], SP_THREADS, 0, st>>>(v, s->levcols + s->lev_ptr[l], s->g,
                                                                                      -1.0, s->y);
  CUDA_TRY(cudaGetLastError());
  *launches += 2 + nlev;
  // singular: a bad pivot, or over every column but the anchor's min d <= 1e-11 max d (balm_pose_covariance's rule
  // with positive pivots; the anchor's unit pivots would hide the scale of H)
  std::vector<double> d(6 * (size_t)P);
  int bad = 0;
  CUDA_TRY(cudaMemcpyAsync(d.data(), s->D, sizeof(double) * d.size(), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(&bad, s->flags, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  double dmin = INFINITY, dmax = 0.0;
  for (int j = 0; j < P; j++)
    if (j != ac)
      for (int m = 0; m < 6; m++) {
        dmin = std::min(dmin, d[6 * (size_t)j + m]);
        dmax = std::max(dmax, d[6 * (size_t)j + m]);
      }
  if (bad || !(dmin > 0.0 && dmin > 1e-11 * dmax && dmax < INFINITY)) {
    balm_set_error(std::string(who) + ": H with the anchor's rows and columns deleted is singular");
    return BALM_ERR_NOT_PD;
  }
  return BALM_OK;
}

int sparse_covariance(SparseSolver *s, cudaStream_t st, int anchor, const std::function<int()> &eval, const char *who,
                      double *cov, long long *launches) {
  if (!s->Z) TRY(selinv_build(*s, st, who));
  TRY(eval());
  TRY(sparse_factor_undamped(s, st, anchor, who, launches));
  const SpView v = s->view();
  const int nlev = (int)s->lev_ptr.size() - 1, ac = anchor >= 0 ? s->col_of[anchor] : -1;
  // Z top level first, then cov gathered into L's storage (no longer needed) and copied out
  for (int l = nlev - 1; l >= 0; l--)
    spg_selinv_kernel<<<s->lev_ptr[l + 1] - s->lev_ptr[l], SEL_THREADS, 0, st>>>(v, s->levcols + s->lev_ptr[l], s->sptr,
                                                                                s->sterm, s->Z);
  if (s->npairs)
    spg_cov_gather_kernel<<<(unsigned)((36 * s->npairs + 255) / 256), 256, 0, st>>>(s->Z, s->zsrc, v, s->npairs, ac, s->Lx);
  CUDA_TRY(cudaGetLastError());
  *launches += nlev + 1;
  CUDA_TRY(cudaMemcpyAsync(cov, s->Lx, sizeof(double) * 36 * s->npairs, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return BALM_OK;
}

int sparse_solve_many(SparseSolver *s, cudaStream_t st, double *Y, int ld, int ncols, long long *launches) {
  const SpView v = s->view();
  const int nlev = (int)s->lev_ptr.size() - 1;
  const unsigned tiles = (unsigned)((ncols + MANY_TILE - 1) / MANY_TILE);
  if (ncols < 1) return BALM_OK;
  for (int l = 0; l < nlev; l++)
    spg_fwd_many_kernel<<<dim3(s->lev_ptr[l + 1] - s->lev_ptr[l], tiles), 6 * MANY_TILE, 0, st>>>(
        v, s->levcols + s->lev_ptr[l], Y, ld, ncols);
  for (int l = nlev - 1; l >= 0; l--)
    spg_back_many_kernel<<<dim3(s->lev_ptr[l + 1] - s->lev_ptr[l], tiles), 6 * MANY_TILE, 0, st>>>(
        v, s->levcols + s->lev_ptr[l], Y, ld, ncols);
  CUDA_TRY(cudaGetLastError());
  *launches += 2 * nlev;
  return BALM_OK;
}

const std::vector<int> &sparse_solver_columns(SparseSolver *s) { return s->col_of; }
int sparse_solver_size(const SparseSolver *s) { return s->P; }
void sparse_solver_pose_pairs(const SparseSolver *s, const int **pp_ptr, const int2 **pp) {
  *pp_ptr = s->pp_ptr;
  *pp = s->pp;
}

// pose_graph.cu -- the pose graph of hierarchical BA's top-down step (include/balm_b200.h, balm_set_pose_factors,
// balm_pose_graph_evaluate, balm_pose_graph_iter; DESIGN.md "Pose graph"). A window factor f holds N_f (2..32) global
// pose indices idx, the window's refined poses T^_k and its BA Hessian H_f; with A = T_idx[0] T^_0^-1
//     e_k = c(A^-1 T_idx[k], T^_k)  (e_0 = 0),   c(T, T^) = (Log(R R^^T), p - R R^^T p^),
//     cost_f = 1/2 sum_{k,l >= 1} e_k^T H_f[k,l] e_l.
// fp64 throughout; every sum runs in a fixed order and there are no floating-point atomics, so results repeat bit for bit.
//   pg_check_kernel      per factor, one CTA: LDL^T of H_f restricted to slots >= 1 in shared memory -> status
//   pg_linearise_kernel  per active factor, one CTA: e_k, J_k (shared), M = E^T H~ E and b = E^T H~ e -> staging
//   pg_assemble_kernel   per (global 6x6 block pair i <= j, entry): the pair's (factor, slot, slot) terms in factor order
//                        -> H (i, j) and (j, i) from one sum; per gradient entry: the pose's slots in factor order -> g
//                        (outputs: dense H, stored or added onto the voxel H of a joint cost, or a blocks context's
//                        blocks: stored, or added onto its voxel blocks)
//   pg_cost_kernel       per active factor, one CTA: cost_f
//   pg_sum_kernel        one CTA: the factors' costs in factor order -> a device scalar
// Absolute pose priors (DESIGN.md "Absolute pose priors"; PriorSet, balm_set_pose_priors): prior_cost_kernel and
// prior_linearise_kernel per active prior, prior_assemble_kernel per (pose with priors, entry) adding the pose's sums onto
// the diagonal block and g after the factors; run only while a prior is active.
// Robust losses (DESIGN.md "Robust pose factors"): with s = e~^T H~ e~ a term's cost becomes 1/2 rho(s), its b rho'(s) b
// and its M rho'(s) M (IRLS). Factors and priors each own one TermLoss, the loss core: the per-term arrays, the robust
// flag, their bytes, the readout and the evaluation order. The <FactorLoss> instantiations of the cost kernels (write s
// and w = rho'(s)) and the linearisations (scale M and b by w) run only when an active term has a non-trivial loss; the
// <NoLoss> ones are the kernels without a loss.
#include <math.h>
#include <type_traits>
#include <algorithm>
#include <memory>
#include <vector>
#include "internal.cuh"

namespace {

constexpr int PG_THREADS = 256;
constexpr int PG_MAXN = BALM_BATCH_MAX_POSES;  // poses per factor
constexpr int PG_MAXM = 6 * (PG_MAXN - 1);     // unknowns of H~ (slots >= 1)
constexpr int CHECK_SMEM = (PG_MAXM * (PG_MAXM + 1) / 2 + PG_MAXM) * (int)sizeof(double);

// Log of a rotation (row-major): theta = atan2(|v|, (tr - 1)/2), v = vee(R - R^T)/2; below 90 degrees phi = theta/|v| v,
// else the axis from the symmetric part (R + R^T)/2 - cos(theta) I = (1 - cos(theta)) a a^T, signed by v
__device__ __forceinline__ void log_so3(const double *R, double *phi) {
  const double v[3] = {0.5 * (R[7] - R[5]), 0.5 * (R[2] - R[6]), 0.5 * (R[3] - R[1])};
  const double c = 0.5 * (R[0] + R[4] + R[8] - 1.0);
  const double s = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  const double th = atan2(s, c);
  if (c > 0.0) {
    const double f = s == 0.0 ? 0.0 : th / s;
    for (int a = 0; a < 3; a++) phi[a] = f * v[a];
    return;
  }
  double B[9];
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) B[a * 3 + b] = 0.5 * (R[a * 3 + b] + R[b * 3 + a]) - (a == b ? c : 0.0);
  int i = 0;
  if (B[4] > B[0]) i = 1;
  if (B[8] > B[i * 4]) i = 2;
  const double den = sqrt(B[i * 4] * (1.0 - c));
  double ax[3] = {B[i] / den, B[3 + i] / den, B[6 + i] / den};
  const double sg = ax[0] * v[0] + ax[1] * v[1] + ax[2] * v[2] < 0.0 ? -th : th;
  for (int a = 0; a < 3; a++) phi[a] = sg * ax[a];
}

// e (6) and, when J is not null, J = de/d(delta_k) (row-major 6 x 6) of slot k >= 1: T0 / Tk the current poses of the
// factor's slots 0 and k, h0 / hk its T^_0 and T^_k (pose12 layout). With Q = R^_0 R_0^T and phi = e[0..2]:
//   J = [[Jl^-1(phi) Q, 0], [-Q hat(p_k - R_k R^_k^T p^_k), Q]].
// Not inlined, so that the linearisation and the cost pass compute bitwise the same e.
__device__ __noinline__ void pg_residual(const double *T0, const double *Tk, const double *h0, const double *hk,
                                         double *e, double *J) {
  double r0[9], p0[3], rk[9], pk[3], rh0[9], ph0[3], rhk[9], phk[3];
  load_pose(T0, r0, p0);
  load_pose(Tk, rk, pk);
  load_pose(h0, rh0, ph0);
  load_pose(hk, rhk, phk);
  double Q[9], Rs[9], D[9], ps[3];
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) Q[a * 3 + b] = rh0[a * 3] * r0[b * 3] + rh0[a * 3 + 1] * r0[b * 3 + 1] + rh0[a * 3 + 2] * r0[b * 3 + 2];
  const double dp[3] = {pk[0] - p0[0], pk[1] - p0[1], pk[2] - p0[2]};
  for (int a = 0; a < 3; a++) {
    for (int b = 0; b < 3; b++) Rs[a * 3 + b] = Q[a * 3] * rk[b] + Q[a * 3 + 1] * rk[3 + b] + Q[a * 3 + 2] * rk[6 + b];
    ps[a] = Q[a * 3] * dp[0] + Q[a * 3 + 1] * dp[1] + Q[a * 3 + 2] * dp[2] + ph0[a];
  }
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) D[a * 3 + b] = Rs[a * 3] * rhk[b * 3] + Rs[a * 3 + 1] * rhk[b * 3 + 1] + Rs[a * 3 + 2] * rhk[b * 3 + 2];
  log_so3(D, e);
  for (int a = 0; a < 3; a++) e[3 + a] = ps[a] - (D[a * 3] * phk[0] + D[a * 3 + 1] * phk[1] + D[a * 3 + 2] * phk[2]);
  if (!J) return;
  double w[3];  // p_k - R_k R^_k^T p^_k
  for (int a = 0; a < 3; a++) {
    double m[3];
    for (int b = 0; b < 3; b++) m[b] = rk[a * 3] * rhk[b * 3] + rk[a * 3 + 1] * rhk[b * 3 + 1] + rk[a * 3 + 2] * rhk[b * 3 + 2];
    w[a] = pk[a] - (m[0] * phk[0] + m[1] * phk[1] + m[2] * phk[2]);
  }
  // Jl^-1(phi) = I - 1/2 hat(phi) + c2 hat(phi)^2, c2 = (1 - (th/2) cot(th/2)) / th^2 (series below th = 0.1)
  const double t2 = e[0] * e[0] + e[1] * e[1] + e[2] * e[2], th = sqrt(t2);
  double c2;
  if (th < 0.1) {
    c2 = 1.0 / 12 + t2 * (1.0 / 720 + t2 * (1.0 / 30240 + t2 / 1209600));
  } else {
    const double h = 0.5 * th;
    c2 = (1.0 - h * cos(h) / sin(h)) / t2;
  }
  const double K[9] = {0, -e[2], e[1], e[2], 0, -e[0], -e[1], e[0], 0};
  const double W[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
  double Ji[9];
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++)
      Ji[a * 3 + b] = (a == b ? 1.0 : 0.0) - 0.5 * K[a * 3 + b] + c2 * (e[a] * e[b] - (a == b ? t2 : 0.0));
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) {
      J[a * 6 + b] = Ji[a * 3] * Q[b] + Ji[a * 3 + 1] * Q[3 + b] + Ji[a * 3 + 2] * Q[6 + b];
      J[a * 6 + 3 + b] = 0.0;
      J[(3 + a) * 6 + b] = -(Q[a * 3] * W[b] + Q[a * 3 + 1] * W[3 + b] + Q[a * 3 + 2] * W[6 + b]);
      J[(3 + a) * 6 + 3 + b] = Q[a * 3 + b];
    }
}

// ---- registration: H~ = H_f restricted to slots >= 1 must be positive definite. The pivot test of
// batch_cov_solve_kernel (zero / tiny / non-finite pivot, or min |d| <= 1e-11 max |d|), and every pivot positive ----
__global__ void __launch_bounds__(PG_THREADS) pg_check_kernel(const long long *fptr, const long long *hoff,
                                                              const double *H, int *status) {
  extern __shared__ double sm[];
  const int f = blockIdx.x, tid = threadIdx.x;
  const int n6 = 6 * (int)(fptr[f + 1] - fptr[f]), n = n6 - 6;
  double *A = sm, *col = A + n * (n + 1) / 2;
  const double *Hf = H + hoff[f];
  for (int e = tid; e < n * n; e += PG_THREADS) {
    const int j = e / n, i = e % n;
    if (i >= j) A[tri_idx(i, j, n)] = Hf[(size_t)(j + 6) * n6 + i + 6];
  }
  __syncthreads();
  const bool pivot_bad = ldl_factor<PG_THREADS>(A, n, col);
  if (tid == 0) {
    double dmin = 1e300, dmax = 0.0;
    bool neg = false;
    for (int i = 0; i < n && !pivot_bad; i++) {
      const double d = A[tri_idx(i, i, n)];
      neg = neg || !(d > 0.0);
      dmin = fmin(dmin, fabs(d));
      dmax = fmax(dmax, fabs(d));
    }
    status[f] = pivot_bad || neg || !(dmin > 1e-11 * dmax) ? BALM_ERR_NOT_PD : BALM_OK;
  }
}

struct FactorView {  // one factor as the per-factor kernels read it
  const long long *fptr, *hoff;
  const int *pose;    // [S] global pose index of every slot
  const double *hat;  // [S][12] T^
  const double *H;    // per factor (6N)^2, column-major
};

// e_k (and J_k) of slots 1..N-1 of factor f into shared memory, threads 1..N-1
__device__ __forceinline__ void factor_residuals(const FactorView &fv, int f, const double *poses, double (*se)[6],
                                                 double (*sJ)[36]) {
  const long long s0 = fv.fptr[f];
  const int N = (int)(fv.fptr[f + 1] - s0), k = threadIdx.x;
  if (k > 0 && k < N)
    pg_residual(poses + 12 * (size_t)fv.pose[s0], poses + 12 * (size_t)fv.pose[s0 + k], fv.hat + 12 * s0,
                fv.hat + 12 * (s0 + k), se[k], sJ ? sJ[k] : nullptr);
  __syncthreads();
}

struct FactorLoss {   // per term (factor or prior): kind (BALM_LOSS_*), scale c, outputs s and w = rho'(s)
  int *kind;          // null: every term trivial
  double *scale, *s, *w;
};

// A term's cost from its s, index q of the loss arrays: with FactorLoss 1/2 rho(s), and s, w = rho'(s) to the loss's
// outputs; with NoLoss 1/2 s
template <typename Loss>
__device__ __forceinline__ double term_cost(const Loss &loss, int q, double s) {
  if constexpr (std::is_same<Loss, FactorLoss>::value) {
    double rho, drho;
    loss_rho(loss.kind ? loss.kind[q] : BALM_LOSS_TRIVIAL, loss.kind ? loss.scale[q] : 1.0, s, &rho, &drho);
    loss.s[q] = s;
    loss.w[q] = drho;
    s = rho;
  }
  return 0.5 * s;
}

// ---- per active factor: M (6N x 6N, column-major, at the factor's H offset) and b (6 per slot); with FactorLoss both
// scaled by w_f, which the cost pass before has written ----
template <typename Loss>
__global__ void __launch_bounds__(PG_THREADS) pg_linearise_kernel(FactorView fv, const int *act, const double *poses,
                                                                  double *M, double *b, Loss loss) {
  constexpr bool robust = std::is_same<Loss, FactorLoss>::value;
  __shared__ double se[PG_MAXN][6], sJ[PG_MAXN][36];
  const int f = act[blockIdx.x], tid = threadIdx.x;
  const long long s0 = fv.fptr[f];
  const int N = (int)(fv.fptr[f + 1] - s0), n6 = 6 * N, nb = N - 1;
  const double *Hf = fv.H + fv.hoff[f];
  double *Mf = M + fv.hoff[f], *bf = b + 6 * s0;
  double wf = 1.0;
  if constexpr (robust) wf = loss.w[f];
  factor_residuals(fv, f, poses, se, sJ);
  // k, l >= 1: M[k,l] = J_k^T H_f[k,l] J_l, b_k = J_k^T sum_l H_f[k,l] e_l
  const int nm = nb * nb * 36;
  for (int q = tid; q < nm + nb * 6; q += PG_THREADS) {
    if (q < nm) {
      const int a = q % 6, c6 = (q / 6) % 6, blk = q / 36, k = 1 + blk % nb, l = 1 + blk / nb;
      const double *Hkl = Hf + (size_t)(6 * l) * n6 + 6 * k;  // H_f[6k + c, 6l + d] = Hkl[d n6 + c]
      double s = 0.0;
      for (int d = 0; d < 6; d++) {
        double t = 0.0;
        for (int c = 0; c < 6; c++) t += sJ[k][c * 6 + a] * Hkl[(size_t)d * n6 + c];
        s += t * sJ[l][d * 6 + c6];
      }
      if constexpr (robust) s *= wf;
      Mf[(size_t)(6 * l + c6) * n6 + 6 * k + a] = s;
    } else {
      const int r = q - nm, a = r % 6, k = 1 + r / 6;
      double s = 0.0;
      for (int c = 0; c < 6; c++) {
        double t = 0.0;
        for (int l = 1; l < N; l++)
          for (int d = 0; d < 6; d++) t += Hf[(size_t)(6 * l + d) * n6 + 6 * k + c] * se[l][d];
        s += sJ[k][c * 6 + a] * t;
      }
      if constexpr (robust) s *= wf;
      bf[6 * k + a] = s;
    }
  }
  __syncthreads();  // the block's global writes above are visible to it from here on
  // slot 0 by the invariance to a common left transform (k, l >= 1, ascending): M[0,m] = -sum_k M[k,m],
  // M[m,0] = -sum_l M[m,l], M[0,0] = sum_l sum_k M[k,l], b_0 = -sum_k b_k
  for (int q = tid; q < 2 * nb * 36 + 36 + 6; q += PG_THREADS) {
    if (q < 2 * nb * 36) {
      const int a = q % 6, c6 = (q / 6) % 6, m = 1 + (q / 36) % nb;
      double s = 0.0;
      if (q < nb * 36) {
        for (int k = 1; k < N; k++) s += Mf[(size_t)(6 * m + c6) * n6 + 6 * k + a];
        Mf[(size_t)(6 * m + c6) * n6 + a] = -s;
      } else {
        for (int l = 1; l < N; l++) s += Mf[(size_t)(6 * l + c6) * n6 + 6 * m + a];
        Mf[(size_t)c6 * n6 + 6 * m + a] = -s;
      }
    } else if (q < 2 * nb * 36 + 36) {
      const int r = q - 2 * nb * 36, a = r % 6, c6 = r / 6;
      double s = 0.0;
      for (int l = 1; l < N; l++)
        for (int k = 1; k < N; k++) s += Mf[(size_t)(6 * l + c6) * n6 + 6 * k + a];
      Mf[(size_t)c6 * n6 + a] = s;
    } else {
      const int a = q - 2 * nb * 36 - 36;
      double s = 0.0;
      for (int k = 1; k < N; k++) s += bf[6 * k + a];
      bf[a] = -s;
    }
  }
}

// ---- H and g: one thread per (block pair, entry), then one per gradient entry. The pair sums go to `out`: dense H
// (zeroed beforehand) for the context; on a BALM_PREC_BLOCKS context one 6x6 block per pair when the factor pairs are
// its whole pattern (the sparse pose graph's usual case), else added onto its union pattern's blocks (DESIGN.md "Voxels
// and pose factors in one cost"); with an FP64 / TENSOR context's joint cost, added onto its voxel H (DESIGN.md "Voxels,
// factors and priors in one cost on dense contexts"). ----
struct DenseH {  // H (6P)^2 column-major: entry (a, c6) of pair (i, j) at (6i + a, 6j + c6) and its transpose
  double *H;
  __device__ __forceinline__ void operator()(size_t n, long long p, int2 ij, int a, int c6, double s) const {
    H[(6 * (size_t)ij.y + c6) * n + 6 * (size_t)ij.x + a] = s;
    if (ij.x != ij.y) H[(6 * (size_t)ij.x + a) * n + 6 * (size_t)ij.y + c6] = s;
  }
};
struct PairBlocks {  // block p (36, column-major) = H rows 6i.., columns 6j..
  double *B;
  __device__ __forceinline__ void operator()(size_t, long long p, int2, int a, int c6, double s) const {
    B[36 * p + 6 * c6 + a] = s;
  }
};
struct AddBlocks {  // a BALM_PREC_BLOCKS context's union pattern: block map[p] (36, column-major) += pair p's sum
  double *B;
  const int *map;
  __device__ __forceinline__ void operator()(size_t, long long p, int2, int a, int c6, double s) const {
    B[36 * (size_t)map[p] + 6 * c6 + a] += s;
  }
};
struct AddDenseH {  // an FP64 / TENSOR context's joint cost: DenseH's entries added onto the voxel H, one add per entry
  double *H;
  __device__ __forceinline__ void operator()(size_t n, long long, int2 ij, int a, int c6, double s) const {
    H[(6 * (size_t)ij.y + c6) * n + 6 * (size_t)ij.x + a] += s;
    if (ij.x != ij.y) H[(6 * (size_t)ij.x + a) * n + 6 * (size_t)ij.y + c6] += s;
  }
};

template <typename Out>
__global__ void __launch_bounds__(PG_THREADS) pg_assemble_kernel(const long long *fptr, const long long *hoff,
                                                                 const int2 *pair, const int *pair_ptr, const int3 *term,
                                                                 long long n_pairs, const double *M, const int *gp_ptr,
                                                                 const long long *gp_slot, const double *b, int P,
                                                                 Out out, double *g) {
  const long long t = (long long)blockIdx.x * PG_THREADS + threadIdx.x;
  const size_t n = 6 * (size_t)P;
  if (t < 36 * n_pairs) {
    const long long p = t / 36;
    const int e = (int)(t % 36), a = e % 6, c6 = e / 6;
    const int2 ij = pair[p];
    // a diagonal pair sums its lower entries for both (a, c6) and (c6, a): the block comes out exactly symmetric
    const int ra = ij.x == ij.y ? max(a, c6) : a, rc = ij.x == ij.y ? min(a, c6) : c6;
    double s = 0.0;
    for (int q = pair_ptr[p]; q < pair_ptr[p + 1]; q++) {
      const int3 fkl = term[q];
      const int n6 = 6 * (int)(fptr[fkl.x + 1] - fptr[fkl.x]);
      s += M[hoff[fkl.x] + (size_t)(6 * fkl.z + rc) * n6 + 6 * fkl.y + ra];
    }
    out(n, p, ij, a, c6, s);
  } else if (t < 36 * n_pairs + 6 * (long long)P) {
    const long long r = t - 36 * n_pairs;
    const int i = (int)(r / 6), a = (int)(r % 6);
    double s = 0.0;
    for (int q = gp_ptr[i]; q < gp_ptr[i + 1]; q++) s += b[6 * gp_slot[q] + a];
    g[6 * (size_t)i + a] = s;
  }
}

// ---- per active factor: cost_f = 1/2 e~^T H~ e~, thread r owning row 6 + r of H~; with FactorLoss s_f = e~^T H~ e~,
// cost_f = 1/2 rho(s_f) and s_f, w_f = rho'(s_f) to the loss's outputs ----
template <typename Loss>
__global__ void __launch_bounds__(PG_THREADS) pg_cost_kernel(FactorView fv, const int *act, const double *poses,
                                                             double *cost_part, Loss loss) {
  __shared__ double se[PG_MAXN][6];
  __shared__ double red[PG_THREADS / 32];
  const int f = act[blockIdx.x], tid = threadIdx.x;
  const int N = (int)(fv.fptr[f + 1] - fv.fptr[f]), n6 = 6 * N;
  const double *Hf = fv.H + fv.hoff[f];
  factor_residuals(fv, f, poses, se, nullptr);
  const double *ef = &se[0][0];
  double part = 0.0;
  if (tid < n6 - 6) {
    const int r = 6 + tid;
    double t = 0.0;
    for (int c = 6; c < n6; c++) t += Hf[(size_t)c * n6 + r] * ef[c];
    part = ef[r] * t;
  }
  part = warp_sum(part);
  if ((tid & 31) == 0) red[tid >> 5] = part;
  __syncthreads();
  if (tid == 0) {
    double s = 0.0;
    for (int q = 0; q < PG_THREADS / 32; q++) s += red[q];
    cost_part[blockIdx.x] = term_cost(loss, f, s);
  }
}

__global__ void __launch_bounds__(PG_THREADS) pg_sum_kernel(const double *part, int n, double *out) {
  __shared__ double red[PG_THREADS / 32];
  const int tid = threadIdx.x;
  double s = 0.0;
  for (int i = tid; i < n; i += PG_THREADS) s += part[i];
  s = warp_sum(s);
  if ((tid & 31) == 0) red[tid >> 5] = s;
  __syncthreads();
  if (tid == 0) {
    double r = 0.0;
    for (int q = 0; q < PG_THREADS / 32; q++) r += red[q];
    *out = r;
  }
}

// ---- absolute pose priors (DESIGN.md "Absolute pose priors"): prior q on pose i with measured pose T^ = (R^, p^),
// body-frame lever arm l and 6x6 H_q (column-major, (rotation, translation) order):
//   e = (Log(R R^^T), R l + p - p^),   s_q = e^T H_q e,   cost_q = 1/2 rho(s_q),
//   J = de/d(delta) = [[Jl^-1(e_rot), 0], [-hat(R l + p), I]] under the left update,   M_q = w J^T H_q J, b_q = w J^T H_q e
// with w = rho'(s_q) (1 without a loss). One thread per active prior; the active priors are held sorted by pose, prior
// order within a pose, so that prior_assemble_kernel sums a contiguous range. ----

// e (6) and, when J is not null, J (row-major 6 x 6). Not inlined, so that the cost and the linearisation compute
// bitwise the same e.
__device__ __noinline__ void prior_residual(const double *T, const double *hat, const double *lever, double *e,
                                            double *J) {
  double r[9], p[3], rh[9], ph[3], D[9], x[3];
  load_pose(T, r, p);
  load_pose(hat, rh, ph);
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) D[a * 3 + b] = r[a * 3] * rh[b * 3] + r[a * 3 + 1] * rh[b * 3 + 1] + r[a * 3 + 2] * rh[b * 3 + 2];
  log_so3(D, e);
  for (int a = 0; a < 3; a++) {
    x[a] = r[a * 3] * lever[0] + r[a * 3 + 1] * lever[1] + r[a * 3 + 2] * lever[2] + p[a];  // R l + p
    e[3 + a] = x[a] - ph[a];
  }
  if (!J) return;
  // Jl^-1(phi) = I - 1/2 hat(phi) + c2 hat(phi)^2, c2 = (1 - (th/2) cot(th/2)) / th^2 (series below th = 0.1)
  const double t2 = e[0] * e[0] + e[1] * e[1] + e[2] * e[2], th = sqrt(t2);
  double c2;
  if (th < 0.1) {
    c2 = 1.0 / 12 + t2 * (1.0 / 720 + t2 * (1.0 / 30240 + t2 / 1209600));
  } else {
    const double h = 0.5 * th;
    c2 = (1.0 - h * cos(h) / sin(h)) / t2;
  }
  const double K[9] = {0, -e[2], e[1], e[2], 0, -e[0], -e[1], e[0], 0};
  const double W[9] = {0, -x[2], x[1], x[2], 0, -x[0], -x[1], x[0], 0};
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) {
      J[a * 6 + b] = (a == b ? 1.0 : 0.0) - 0.5 * K[a * 3 + b] + c2 * (e[a] * e[b] - (a == b ? t2 : 0.0));
      J[a * 6 + 3 + b] = 0.0;
      J[(3 + a) * 6 + b] = -W[a * 3 + b];
      J[(3 + a) * 6 + 3 + b] = a == b ? 1.0 : 0.0;
    }
}

struct PriorView {  // the prior set as the per-prior kernels read it
  const int *pose;      // [n] pose of every prior
  const double *hat;    // [n][12] T^
  const double *lever;  // [n][3] l
  const double *H;      // [n][36] column-major
};

// ---- per active prior k (act[k] = prior q): cost_part[k] = 1/2 rho(s_q); with FactorLoss s_q, w_q to its outputs ----
template <typename Loss>
__global__ void __launch_bounds__(PG_THREADS) prior_cost_kernel(PriorView pv, const int *act, int n_act,
                                                                const double *poses, double *cost_part, Loss loss) {
  const int k = blockIdx.x * PG_THREADS + threadIdx.x;
  if (k >= n_act) return;
  const int q = act[k];
  double e[6];
  prior_residual(poses + 12 * (size_t)pv.pose[q], pv.hat + 12 * (size_t)q, pv.lever + 3 * (size_t)q, e, nullptr);
  const double *Hq = pv.H + 36 * (size_t)q;
  double s = 0.0;
  for (int r = 0; r < 6; r++) {
    double t = 0.0;
    for (int c = 0; c < 6; c++) t += Hq[6 * c + r] * e[c];
    s += e[r] * t;
  }
  cost_part[k] = term_cost(loss, q, s);
}

// ---- per active prior k: M[k] = w J^T H J (36, column-major) and b[k] = w J^T H e; with FactorLoss w is the w_q that
// the cost pass before has written ----
template <typename Loss>
__global__ void __launch_bounds__(PG_THREADS) prior_linearise_kernel(PriorView pv, const int *act, int n_act,
                                                                     const double *poses, double *M, double *b,
                                                                     Loss loss) {
  const int k = blockIdx.x * PG_THREADS + threadIdx.x;
  if (k >= n_act) return;
  const int q = act[k];
  double e[6], J[36];
  prior_residual(poses + 12 * (size_t)pv.pose[q], pv.hat + 12 * (size_t)q, pv.lever + 3 * (size_t)q, e, J);
  double w = 1.0;
  if constexpr (std::is_same<Loss, FactorLoss>::value) w = loss.w[q];
  const double *Hq = pv.H + 36 * (size_t)q;
  double *Mk = M + 36 * (size_t)k, *bk = b + 6 * (size_t)k;
  double He[6];
  for (int r = 0; r < 6; r++) {
    double t = 0.0;
    for (int c = 0; c < 6; c++) t += Hq[6 * c + r] * e[c];
    He[r] = t;
  }
  for (int a = 0; a < 6; a++) {
    double t = 0.0;
    for (int r = 0; r < 6; r++) t += J[r * 6 + a] * He[r];
    bk[a] = w * t;
  }
  for (int d = 0; d < 6; d++) {  // column d: (H J)[:, d], then M[:, d] = J^T (H J)[:, d]
    double HJ[6];
    for (int r = 0; r < 6; r++) {
      double t = 0.0;
      for (int c = 0; c < 6; c++) t += Hq[6 * c + r] * J[c * 6 + d];
      HJ[r] = t;
    }
    for (int a = 0; a < 6; a++) {
      double t = 0.0;
      for (int r = 0; r < 6; r++) t += J[r * 6 + a] * HJ[r];
      Mk[6 * d + a] = w * t;
    }
  }
}

// Where a pose's prior sum goes: onto the dense H of a context's pose graph, or onto the pose's diagonal block of a
// BALM_PREC_BLOCKS context's pattern (the sparse pose graph's included), diag[u] its index there.
struct DenseAdd {
  double *H;
  size_t n;
  __device__ __forceinline__ void operator()(int u, int i, int a, int c6, double s) const {
    H[(6 * (size_t)i + c6) * n + 6 * (size_t)i + a] += s;
  }
};
struct DiagAdd {
  double *B;
  const int *diag;
  __device__ __forceinline__ void operator()(int u, int, int a, int c6, double s) const {
    B[36 * (size_t)diag[u] + 6 * c6 + a] += s;
  }
};

// ---- per (pose u with priors, entry): the sum of its priors' M (36 entries) or b (6 entries), in their order, added
// once onto the block and g that the factor and voxel assembly wrote. Like pg_assemble_kernel on a diagonal pair, both
// (a, c6) and (c6, a) read the lower entry, so the block stays exactly symmetric. ----
template <typename Out>
__global__ void __launch_bounds__(PG_THREADS) prior_assemble_kernel(const int *upose, const int *uptr, int n_u,
                                                                    const double *M, const double *b, Out out,
                                                                    double *g) {
  const long long t = (long long)blockIdx.x * PG_THREADS + threadIdx.x;
  if (t >= 42LL * n_u) return;
  const int u = (int)(t / 42), e = (int)(t % 42), i = upose[u];
  double s = 0.0;
  if (e < 36) {
    const int a = e % 6, c6 = e / 6, ra = max(a, c6), rc = min(a, c6);
    for (int k = uptr[u]; k < uptr[u + 1]; k++) s += M[36 * (size_t)k + 6 * rc + ra];
    out(u, i, a, c6, s);
  } else {
    const int a = e - 36;
    for (int k = uptr[u]; k < uptr[u + 1]; k++) s += b[6 * (size_t)k + a];
    g[6 * (size_t)i + a] += s;
  }
}

__global__ void prior_add_cost_kernel(const double *x, double *y) { *y += *x; }

}  // namespace

constexpr long long LOSS_BYTES_PER_FACTOR = sizeof(int) + 3 * sizeof(double);

// Launches `launch` with the loss argument of a cost pass or a linearisation: *l (robust mode, or a readout), or NoLoss
// when l is null.
template <typename Launch>
static void with_loss(const FactorLoss *l, Launch launch) {
  if (l) launch(*l);
  else launch(NoLoss{});
}

// The loss core of a term set (balm_set_factor_loss's factors, balm_set_pose_priors' priors; DESIGN.md "Robust pose
// factors"): kind, scale, s and w per term on the device, allocated only while some term's kind is non-trivial.
struct TermLoss {
  FactorLoss arr{};     // all null without arrays: every term trivial
  bool robust = false;  // an active term has a non-trivial kind
  long long bytes = 0;  // device memory the arrays hold: LOSS_BYTES_PER_FACTOR per term
  ~TermLoss() { release(); }
  void release() {
    cudaFree(arr.kind); cudaFree(arr.scale); cudaFree(arr.s); cudaFree(arr.w);
    arr = FactorLoss{};
    robust = false;
    bytes = 0;
  }
  // The loss argument of the cost pass and the linearisation: the arrays in robust mode, else null (NoLoss). With
  // arrays an evaluation runs the cost pass first, so that the linearisation can weight M and b with its w and the
  // evaluation's cost is its sum; without, the cost pass runs after the assembly.
  const FactorLoss *active() const { return robust ? &arr : nullptr; }

  // kind [n] (null: every term trivial) and scale [n] of the n terms, `act` the active ones. Every term trivial frees
  // the arrays; else they are allocated when absent (a failed allocation leaves every term trivial) and uploaded with
  // s = w = 0. Waits for the upload.
  int set(cudaStream_t st, int n, const int32_t *kind, const double *scale, const std::vector<int> &act) {
    if (!kind || std::all_of(kind, kind + n, [](int32_t k) { return k == BALM_LOSS_TRIVIAL; })) {
      release();  // no arrays: the kernels without a loss
      return BALM_OK;
    }
    if (!arr.kind) {
      if (dev_alloc(&arr.kind, n) != BALM_OK || dev_alloc(&arr.scale, n) != BALM_OK ||
          dev_alloc(&arr.s, n) != BALM_OK || dev_alloc(&arr.w, n) != BALM_OK) {
        release();
        return BALM_ERR_CUDA;
      }
      bytes = LOSS_BYTES_PER_FACTOR * n;
    }
    std::vector<double> c(n);
    bool any_active = false;
    for (int q = 0; q < n; q++) c[q] = kind[q] == BALM_LOSS_TRIVIAL ? 1.0 : scale[q];  // a trivial term's c is unused
    for (int q : act) any_active = any_active || kind[q] != BALM_LOSS_TRIVIAL;
    CUDA_TRY(cudaMemcpyAsync(arr.kind, kind, sizeof(int) * n, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(arr.scale, c.data(), sizeof(double) * n, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemsetAsync(arr.s, 0, sizeof(double) * n, st));  // inactive terms keep s = w = 0
    CUDA_TRY(cudaMemsetAsync(arr.w, 0, sizeof(double) * n, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    robust = any_active;
    return BALM_OK;
  }

  // balm_factor_residuals / balm_prior_residuals over n terms: `cost_pass` with the arrays, or with temporary s and w
  // when no loss is set (every term trivial), then s and w to the host arrays (either may be null); waits once
  template <typename Pass>
  int readout(size_t n, cudaStream_t st, double *s, double *w, Pass cost_pass) const {
    double *tmp = nullptr;
    if (!arr.kind) {
      TRY(dev_alloc(&tmp, 2 * n));
      CUDA_TRY(cudaMemsetAsync(tmp, 0, sizeof(double) * 2 * n, st));
    }
    std::unique_ptr<double, cudaError_t (*)(void *)> tmp_own(tmp, cudaFree);
    const FactorLoss loss = tmp ? FactorLoss{nullptr, nullptr, tmp, tmp + n} : arr;
    TRY(cost_pass(&loss));
    if (s) CUDA_TRY(cudaMemcpyAsync(s, loss.s, sizeof(double) * n, cudaMemcpyDeviceToHost, st));
    if (w) CUDA_TRY(cudaMemcpyAsync(w, loss.w, sizeof(double) * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return BALM_OK;
  }
};

// The registered factor set (device). Factor f owns slots [fptr[f], fptr[f+1]) and the (6N_f)^2 doubles at hoff[f] of
// H and of the staging M.
struct PoseGraph {
  int F = 0, n_act = 0, P = 0;
  long long S = 0, HS = 0, n_pairs = 0;
  long long *fptr = nullptr, *hoff = nullptr, *gp_slot = nullptr;
  int *pose = nullptr, *act = nullptr, *pair_ptr = nullptr, *gp_ptr = nullptr, *status = nullptr;
  int2 *pair = nullptr;
  int3 *term = nullptr;
  double *hat = nullptr, *H = nullptr, *M = nullptr, *b = nullptr, *cost_part = nullptr;
  TermLoss loss;             // balm_set_factor_loss
  std::vector<int2> pair_h;  // host copy of `pair`
  std::vector<int> act_h;    // host copy of `act`
  long long bytes = 0;       // device memory held, the loss arrays' aside
  ~PoseGraph() {
    cudaFree(fptr); cudaFree(hoff); cudaFree(gp_slot); cudaFree(pose); cudaFree(act); cudaFree(pair_ptr);
    cudaFree(gp_ptr); cudaFree(status); cudaFree(pair); cudaFree(term); cudaFree(hat); cudaFree(H); cudaFree(M);
    cudaFree(b); cudaFree(cost_part);
  }
  FactorView view() const { return FactorView{fptr, hoff, pose, hat, H}; }
};

void pose_graph_free(PoseGraph *p) { delete p; }

int pose_graph_setup() {
  CUDA_TRY(cudaFuncSetAttribute(pg_check_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CHECK_SMEM));
  return BALM_OK;
}

template <typename T>
static int upload(T **dst, const T *src, size_t count, cudaStream_t st) {
  TRY(dev_alloc(dst, count));
  if (count) CUDA_TRY(cudaMemcpyAsync(*dst, src, sizeof(T) * count, cudaMemcpyHostToDevice, st));
  return BALM_OK;
}

int pose_graph_build(cudaStream_t st, int P, int n_factors, const int64_t *factor_ptr, const int32_t *factor_pose,
                     const double *poses_hat12, const double *H, std::vector<int> *status_out, PoseGraph **out,
                     long long *launches) {
  std::unique_ptr<PoseGraph> p(new PoseGraph());
  const int F = n_factors;
  p->F = F;
  p->P = P;
  p->S = factor_ptr[F];
  std::vector<long long> fptr(factor_ptr, factor_ptr + F + 1), hoff(F + 1, 0);
  for (int f = 0; f < F; f++) {
    const long long N = fptr[f + 1] - fptr[f];
    hoff[f + 1] = hoff[f] + 36 * N * N;
  }
  p->HS = hoff[F];
  TRY(upload(&p->fptr, fptr.data(), F + 1, st));
  TRY(upload(&p->hoff, hoff.data(), F + 1, st));
  TRY(upload(&p->pose, factor_pose, (size_t)p->S, st));
  TRY(upload(&p->hat, poses_hat12, 12 * (size_t)p->S, st));
  TRY(upload(&p->H, H, (size_t)p->HS, st));
  TRY(dev_alloc(&p->status, F));
  pg_check_kernel<<<F, PG_THREADS, CHECK_SMEM, st>>>(p->fptr, p->hoff, p->H, p->status);
  *launches += 1;
  CUDA_TRY(cudaGetLastError());
  std::vector<int> status(F);
  CUDA_TRY(cudaMemcpyAsync(status.data(), p->status, sizeof(int) * F, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  // assembly tables: the terms of every block pair i <= j and the slots of every pose, each in factor order
  std::vector<int> act;
  struct Term { long long key; int f, k, l; };
  std::vector<Term> terms;
  std::vector<std::pair<int, long long>> slots;  // (pose, global slot)
  for (int f = 0; f < F; f++) {
    if (status[f] != BALM_OK) continue;
    act.push_back(f);
    const int N = (int)(fptr[f + 1] - fptr[f]);
    const int32_t *idx = factor_pose + fptr[f];
    for (int l = 0; l < N; l++) {
      slots.push_back({idx[l], fptr[f] + l});
      for (int k = 0; k < N; k++)
        if (idx[k] <= idx[l]) terms.push_back({(long long)idx[k] * P + idx[l], f, k, l});
    }
  }
  std::stable_sort(terms.begin(), terms.end(), [](const Term &a, const Term &b) { return a.key < b.key; });
  std::stable_sort(slots.begin(), slots.end(), [](const std::pair<int, long long> &a, const std::pair<int, long long> &b) {
    return a.first < b.first;
  });
  if (terms.size() >= ((size_t)1 << 31)) { balm_set_error("balm_set_pose_factors: too many factor terms"); return BALM_ERR_UNSUPPORTED; }
  std::vector<int2> pair;
  std::vector<int> pair_ptr;
  std::vector<int3> term(terms.size());
  for (size_t q = 0; q < terms.size(); q++) {
    if (q == 0 || terms[q].key != terms[q - 1].key) {
      pair.push_back(make_int2((int)(terms[q].key / P), (int)(terms[q].key % P)));
      pair_ptr.push_back((int)q);
    }
    term[q] = make_int3(terms[q].f, terms[q].k, terms[q].l);
  }
  pair_ptr.push_back((int)terms.size());
  std::vector<int> gp_ptr(P + 1, 0);
  std::vector<long long> gp_slot(slots.size());
  for (size_t q = 0; q < slots.size(); q++) {
    gp_ptr[slots[q].first + 1]++;
    gp_slot[q] = slots[q].second;
  }
  for (int i = 0; i < P; i++) gp_ptr[i + 1] += gp_ptr[i];
  p->n_act = (int)act.size();
  p->n_pairs = (long long)pair.size();
  TRY(upload(&p->act, act.data(), act.size(), st));
  TRY(upload(&p->pair, pair.data(), pair.size(), st));
  TRY(upload(&p->pair_ptr, pair_ptr.data(), pair_ptr.size(), st));
  TRY(upload(&p->term, term.data(), term.size(), st));
  TRY(upload(&p->gp_ptr, gp_ptr.data(), gp_ptr.size(), st));
  TRY(upload(&p->gp_slot, gp_slot.data(), gp_slot.size(), st));
  TRY(dev_alloc(&p->M, (size_t)p->HS));
  TRY(dev_alloc(&p->b, 6 * (size_t)p->S));
  TRY(dev_alloc(&p->cost_part, (size_t)std::max(1, p->n_act)));
  CUDA_TRY(cudaStreamSynchronize(st));
  p->bytes = (long long)(sizeof(long long) * (2 * (F + 1) + gp_slot.size()) +
                         sizeof(int) * (p->S + act.size() + pair_ptr.size() + gp_ptr.size() + F) +
                         sizeof(int2) * pair.size() + sizeof(int3) * term.size() +
                         sizeof(double) * (12 * p->S + 2 * p->HS + 6 * p->S + std::max(1, p->n_act)));
  p->pair_h = std::move(pair);
  p->act_h = std::move(act);
  *status_out = std::move(status);
  *out = p.release();
  return BALM_OK;
}

const std::vector<int2> &pose_graph_pairs(const PoseGraph *p) { return p->pair_h; }
long long pose_graph_bytes(const PoseGraph *p) { return p->bytes + p->loss.bytes; }
int pose_graph_n_factors(const PoseGraph *p) { return p->F; }

int pose_graph_set_loss(PoseGraph *p, cudaStream_t st, const int32_t *kind, const double *scale) {
  return p->loss.set(st, p->F, kind, scale, p->act_h);
}

// the cost pass into cost_part, and with a loss argument into its s and w
static int pg_cost_pass(const PoseGraph &p, cudaStream_t st, const double *poses, const FactorLoss *l,
                        long long *launches) {
  if (!p.n_act) return BALM_OK;
  with_loss(l, [&](auto loss) {
    pg_cost_kernel<<<p.n_act, PG_THREADS, 0, st>>>(p.view(), p.act, poses, p.cost_part, loss);
  });
  *launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

static int sum_pass(const PoseGraph &p, cudaStream_t st, double *out, long long *launches) {
  pg_sum_kernel<<<1, PG_THREADS, 0, st>>>(p.cost_part, p.n_act, out);
  *launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int pose_graph_cost(const PoseGraph *pg, cudaStream_t st, const double *poses, double *out, long long *launches) {
  TRY(pg_cost_pass(*pg, st, poses, pg->loss.active(), launches));
  return sum_pass(*pg, st, out, launches);
}

int term_residuals(const PoseGraph *p, cudaStream_t st, const double *poses, double *s, double *w,
                   long long *launches) {
  return p->loss.readout((size_t)p->F, st, s, w,
                         [&](const FactorLoss *l) { return pg_cost_pass(*p, st, poses, l, launches); });
}

// H (through `out`), g and the cost at poses, the cost pass placed by TermLoss::active
template <typename Out>
static int pose_graph_assemble(const PoseGraph &p, cudaStream_t st, const double *poses, Out out, double *g,
                               double *cost, long long *launches) {
  const FactorLoss *l = p.loss.active();
  if (l) TRY(pg_cost_pass(p, st, poses, l, launches));
  if (p.n_act)
    with_loss(l, [&](auto loss) {
      pg_linearise_kernel<<<p.n_act, PG_THREADS, 0, st>>>(p.view(), p.act, poses, p.M, p.b, loss);
    });
  const long long threads = 36 * p.n_pairs + 6 * (long long)p.P;
  pg_assemble_kernel<<<(unsigned)((threads + PG_THREADS - 1) / PG_THREADS), PG_THREADS, 0, st>>>(
      p.fptr, p.hoff, p.pair, p.pair_ptr, p.term, p.n_pairs, p.M, p.gp_ptr, p.gp_slot, p.b, p.P, out, g);
  *launches += p.n_act ? 2 : 1;
  CUDA_TRY(cudaGetLastError());
  if (!l) TRY(pg_cost_pass(p, st, poses, l, launches));
  return sum_pass(p, st, cost, launches);
}

int pose_graph_eval(balm_ctx *c, const double *poses) {
  const size_t n = c->n;
  CUDA_TRY(cudaMemsetAsync(c->H, 0, sizeof(double) * n * n, c->stream));
  TRY(pose_graph_assemble(*c->pg, c->stream, poses, DenseH{c->H}, c->g, c->scal, &c->launches));
  if (c->pr) TRY(prior_add_dense(c->pr, c->stream, poses, c->H, n, c->g, c->scal, &c->launches));
  return BALM_OK;
}

int pose_graph_eval_blocks(const PoseGraph *p, cudaStream_t st, const double *poses, double *blocks, double *g,
                           double *cost, long long *launches) {
  return pose_graph_assemble(*p, st, poses, PairBlocks{blocks}, g, cost, launches);
}

int pose_graph_add_blocks(const PoseGraph *p, cudaStream_t st, const double *poses, double *blocks, const int *map,
                          double *g, double *cost, long long *launches) {
  return pose_graph_assemble(*p, st, poses, AddBlocks{blocks, map}, g, cost, launches);
}

int pose_graph_add_dense(const PoseGraph *p, cudaStream_t st, const double *poses, double *H, double *g, double *cost,
                         long long *launches) {
  return pose_graph_assemble(*p, st, poses, AddDenseH{H}, g, cost, launches);
}

// ---------------- absolute pose priors ----------------
// The registered prior set (device). Prior q's pose, T^, l and H at index q; the active priors (status BALM_OK) in
// `act`, sorted by pose and in prior order within a pose; the poses with active priors (upose) and their ranges of `act`
// (uptr). M and b are the linearisation's staging per active prior. diag[u]: upose[u]'s diagonal block in the handle's
// block pattern (prior_set_map; absent on a dense context).
struct PriorSet {
  int n = 0, n_act = 0, n_u = 0;
  int *pose = nullptr, *act = nullptr, *upose = nullptr, *uptr = nullptr, *diag = nullptr;
  double *hat = nullptr, *lever = nullptr, *H = nullptr, *M = nullptr, *b = nullptr, *cost_part = nullptr,
         *cost = nullptr;
  TermLoss loss;  // the priors' kind and scale
  std::vector<int> upose_h;
  long long bytes = 0, diag_bytes = 0;
  ~PriorSet() {
    cudaFree(pose); cudaFree(act); cudaFree(upose); cudaFree(uptr); cudaFree(diag); cudaFree(hat); cudaFree(lever);
    cudaFree(H); cudaFree(M); cudaFree(b); cudaFree(cost_part); cudaFree(cost);
  }
  PriorView view() const { return PriorView{pose, hat, lever, H}; }
};

void prior_set_free(PriorSet *p) { delete p; }
long long prior_set_bytes(const PriorSet *p) { return p->bytes + p->diag_bytes + p->loss.bytes; }
bool prior_set_active(const PriorSet *p) { return p && p->n_act > 0; }
const std::vector<int> &prior_set_poses(const PriorSet *p) { return p->upose_h; }

// Eigenvalues of a symmetric 6 x 6 matrix (cyclic Jacobi, host)
static void sym6_eigenvalues(const double *H, double *lam) {
  double A[36];
  std::copy(H, H + 36, A);
  for (int sweep = 0; sweep < 50; sweep++) {
    double off = 0.0, tot = 0.0;
    for (int i = 0; i < 36; i++) { tot += A[i] * A[i]; if (i % 7) off += A[i] * A[i]; }
    if (off <= 1e-300 || off <= 1e-32 * tot) break;
    for (int p = 0; p < 5; p++)
      for (int q = p + 1; q < 6; q++) {
        const double apq = A[6 * q + p];
        if (apq == 0.0) continue;
        const double th = (A[6 * q + q] - A[6 * p + p]) / (2.0 * apq);
        const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 6; k++) {  // columns p, q
          const double akp = A[6 * p + k], akq = A[6 * q + k];
          A[6 * p + k] = c * akp - s * akq;
          A[6 * q + k] = s * akp + c * akq;
        }
        for (int k = 0; k < 6; k++) {  // rows p, q
          const double apk = A[6 * k + p], aqk = A[6 * k + q];
          A[6 * k + p] = c * apk - s * aqk;
          A[6 * k + q] = s * apk + c * aqk;
        }
      }
  }
  for (int i = 0; i < 6; i++) lam[i] = A[7 * i];
}

int prior_set_build(cudaStream_t st, int n, const int32_t *pose, const double *hat12, const double *lever3,
                    const double *H36, const int32_t *kind, const double *scale, std::vector<int> *status_out,
                    PriorSet **out) {
  std::unique_ptr<PriorSet> p(new PriorSet());
  p->n = n;
  std::vector<int> status(n), act;
  for (int q = 0; q < n; q++) {  // PSD and nonzero: min eigenvalue >= -1e-12 max eigenvalue > 0
    double lam[6];
    sym6_eigenvalues(H36 + 36 * (size_t)q, lam);
    const double lmin = *std::min_element(lam, lam + 6), lmax = *std::max_element(lam, lam + 6);
    status[q] = lmax > 0.0 && lmin >= -1e-12 * lmax ? BALM_OK : BALM_ERR_NOT_PD;
    if (status[q] == BALM_OK) act.push_back(q);
  }
  std::stable_sort(act.begin(), act.end(), [&](int a, int b) { return pose[a] < pose[b]; });
  std::vector<int> uptr;
  for (size_t k = 0; k < act.size(); k++)
    if (k == 0 || pose[act[k]] != pose[act[k - 1]]) { p->upose_h.push_back(pose[act[k]]); uptr.push_back((int)k); }
  uptr.push_back((int)act.size());
  p->n_act = (int)act.size();
  p->n_u = (int)p->upose_h.size();
  std::vector<double> lever(3 * (size_t)n, 0.0);
  if (lever3) std::copy(lever3, lever3 + 3 * (size_t)n, lever.begin());
  TRY(upload(&p->pose, pose, (size_t)n, st));
  TRY(upload(&p->hat, hat12, 12 * (size_t)n, st));
  TRY(upload(&p->lever, lever.data(), lever.size(), st));
  TRY(upload(&p->H, H36, 36 * (size_t)n, st));
  TRY(upload(&p->act, act.data(), act.size(), st));
  TRY(upload(&p->upose, p->upose_h.data(), p->upose_h.size(), st));
  TRY(upload(&p->uptr, uptr.data(), uptr.size(), st));
  TRY(dev_alloc(&p->M, 36 * act.size()));
  TRY(dev_alloc(&p->b, 6 * act.size()));
  TRY(dev_alloc(&p->cost_part, std::max<size_t>(1, act.size())));
  TRY(dev_alloc(&p->cost, 1));
  const auto nz = [](size_t k) { return std::max<size_t>(1, k); };
  p->bytes = (long long)(sizeof(int) * (nz(n) + nz(act.size()) + nz(p->upose_h.size()) + uptr.size()) +
                         sizeof(double) * (nz(12 * (size_t)n) + nz(3 * (size_t)n) + nz(36 * (size_t)n) +
                                           nz(36 * act.size()) + nz(6 * act.size()) + nz(act.size()) + 1));
  TRY(p->loss.set(st, n, kind, scale, act));
  CUDA_TRY(cudaStreamSynchronize(st));
  *status_out = std::move(status);
  *out = p.release();
  return BALM_OK;
}

int prior_set_map(PriorSet *p, cudaStream_t st, const std::vector<int2> &pairs) {
  std::vector<int> diag(p->upose_h.size());
  for (size_t u = 0; u < diag.size(); u++) {
    const int2 key = make_int2(p->upose_h[u], p->upose_h[u]);
    const auto it = std::lower_bound(pairs.begin(), pairs.end(), key, [](const int2 &a, const int2 &b) {
      return a.x < b.x || (a.x == b.x && a.y < b.y);
    });
    if (it == pairs.end() || it->x != key.x || it->y != key.y) {
      balm_set_error("prior_set_map: a prior's pose has no diagonal block in the pattern");
      return BALM_ERR_INVALID;
    }
    diag[u] = (int)(it - pairs.begin());
  }
  cudaFree(p->diag);
  p->diag = nullptr;
  TRY(upload(&p->diag, diag.data(), diag.size(), st));
  CUDA_TRY(cudaStreamSynchronize(st));
  p->diag_bytes = (long long)(sizeof(int) * std::max<size_t>(1, diag.size()));
  return BALM_OK;
}

// the priors' cost pass into cost_part, and with a loss argument into its s and w
static int prior_cost_pass(const PriorSet &p, cudaStream_t st, const double *poses, const FactorLoss *l,
                           long long *launches) {
  if (!p.n_act) return BALM_OK;
  const unsigned grid = (unsigned)((p.n_act + PG_THREADS - 1) / PG_THREADS);
  with_loss(l, [&](auto loss) {
    prior_cost_kernel<<<grid, PG_THREADS, 0, st>>>(p.view(), p.act, p.n_act, poses, p.cost_part, loss);
  });
  *launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

// the priors' cost summed and added onto *cost (after whatever the factors and voxels wrote there)
static int prior_sum_add(const PriorSet &p, cudaStream_t st, double *cost, long long *launches) {
  pg_sum_kernel<<<1, PG_THREADS, 0, st>>>(p.cost_part, p.n_act, p.cost);
  prior_add_cost_kernel<<<1, 1, 0, st>>>(p.cost, cost);
  *launches += 2;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int prior_add_cost(const PriorSet *p, cudaStream_t st, const double *poses, double *cost, long long *launches) {
  if (!p->n_act) return BALM_OK;
  TRY(prior_cost_pass(*p, st, poses, p->loss.active(), launches));
  return prior_sum_add(*p, st, cost, launches);
}

int term_residuals(const PriorSet *p, cudaStream_t st, const double *poses, double *s, double *w,
                   long long *launches) {
  return p->loss.readout((size_t)p->n, st, s, w,
                         [&](const FactorLoss *l) { return prior_cost_pass(*p, st, poses, l, launches); });
}

// the priors' M and b onto H (through `out`) and g, their cost onto *cost, the cost pass placed by TermLoss::active
template <typename Out>
static int prior_assemble(const PriorSet &p, cudaStream_t st, const double *poses, Out out, double *g, double *cost,
                          long long *launches) {
  if (!p.n_act) return BALM_OK;
  const FactorLoss *l = p.loss.active();
  if (l) TRY(prior_cost_pass(p, st, poses, l, launches));
  const unsigned grid = (unsigned)((p.n_act + PG_THREADS - 1) / PG_THREADS);
  with_loss(l, [&](auto loss) {
    prior_linearise_kernel<<<grid, PG_THREADS, 0, st>>>(p.view(), p.act, p.n_act, poses, p.M, p.b, loss);
  });
  const long long threads = 42LL * p.n_u;
  prior_assemble_kernel<<<(unsigned)((threads + PG_THREADS - 1) / PG_THREADS), PG_THREADS, 0, st>>>(
      p.upose, p.uptr, p.n_u, p.M, p.b, out, g);
  *launches += 2;
  CUDA_TRY(cudaGetLastError());
  if (!l) TRY(prior_cost_pass(p, st, poses, l, launches));
  return prior_sum_add(p, st, cost, launches);
}

int prior_add_dense(const PriorSet *p, cudaStream_t st, const double *poses, double *H, size_t n, double *g,
                    double *cost, long long *launches) {
  return prior_assemble(*p, st, poses, DenseAdd{H, n}, g, cost, launches);
}

int prior_add_blocks(const PriorSet *p, cudaStream_t st, const double *poses, double *blocks, double *g, double *cost,
                     long long *launches) {
  return prior_assemble(*p, st, poses, DiagAdd{blocks, p->diag}, g, cost, launches);
}

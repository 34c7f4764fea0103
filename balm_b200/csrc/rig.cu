// rig.cu -- rig calibration (DESIGN.md "Rig calibration"): the context's N scan slots driven by B base poses and L
// extrinsics, X_s = T_{base_of[s]} E_{lidar_of[s]}. The voxel evaluation runs unchanged at the composed scan poses; this
// file composes them, reduces the context's H and g to the free unknowns' system, and applies the LM step.
//
// Unknowns: free base poses ascending, then free extrinsics ascending, 6 each (phi, t), both updated by the left rule of
// pose_update_one. With T_b = (R, p) the base pose of slot s, a its base step and e its extrinsic step,
//   G(a) T_b G(e) E_l = G(delta_s) X_s,  delta_s = J_s [a; e] + delta_s^(2) + O(3),
//   J_s = [ I on base b | Ad(T_b) = [[R, 0], [p^ R, R]] on lidar l ],
//   delta_s^(2) = ( 1/2 a_phi x c ;  a_phi x (R e_t + p x c) - 1/2 c x (c x p) ),  c = R e_phi.
// So g_rig = sum_s J_s^T g_s and H_rig = sum_{s,t} J_s^T H_st J_t + sum_s d2(g_s . delta_s^(2)): the exact Hessian of
// the rig cost in these coordinates. The correction touches only the (lidar, base) and (lidar, lidar) blocks.
//
// On a BALM_PREC_BLOCKS context (balm_block_set_rig, DESIGN.md "Rig calibration on block-sparse voxel BA") nothing of
// size n_rig x 6N or n_rig^2 exists: H_rig is held as the 6x6 blocks of the rig pairs (u, v), u <= v, for which a slot
// of u and a slot of v form a pair of the context's slot pattern (plus every diagonal pair), derived from that pattern
// whenever its generation moves, and solved with the nested-dissection block LDL^T of pose_graph_sparse.cu. The
// reduction runs in two passes, the sparse form of rig_k_kernel / rig_jtk_kernel<true>:
//   rig_k_blocks_kernel    per (K block (s, v), row): K_sv = sum_{t in v, ascending} H_st J_t from the slot blocks
//   rig_jtk_blocks_kernel  per rig pair, one warp: sum_{s in u, ascending} J_s^T K_sv plus the correction of s, lane l
//                          taking the slots l, l + 32, ..., the lanes' sums meeting in warp_sum's fixed butterfly;
//                          a diagonal pair also sums g_rig(u) = sum_{s in u} J_s^T g_s the same way
#include <algorithm>
#include <memory>
#include <vector>
#include "internal.cuh"

struct Rig {
  int N = 0, B = 0, L = 0, F = 0;  // slots, bases, extrinsics, free unknowns (n_rig = 6F)
  int FB = 0;                      // free base poses (the first FB free unknowns)
  int *base_of = nullptr;          // [N]
  int *var_of = nullptr;           // [B + L] free index of every unknown, -1 when fixed
  int *var_unknown = nullptr;      // [F] the unknown of every free index (< B: a base pose, else extrinsic - B)
  int *var_ptr = nullptr;          // [F + 1] CSR: the slots of free unknown u, ascending, are
  int *var_slot = nullptr;         //   var_slot[var_ptr[u] .. var_ptr[u+1])
  int *lidar_of = nullptr;         // [N]
  double *state = nullptr, *state_trial = nullptr;  // [12 (B + L)]: base poses, then extrinsics
  double *H = nullptr;             // [n_rig^2 + n_rig] H_rig (column-major, full symmetric) | g_rig
  double *dx = nullptr, *dvec = nullptr, *A = nullptr;
  double *K = nullptr;             // [n_rig][6N] K = H J, column-major
  LdltWork lw;
  bool any_base_fixed = false;
  // block-sparse rig (balm_block_set_rig): no H, A, K or lw; g_rig in gb and the pattern derived from the slot pattern
  bool sparse = false;
  double *gb = nullptr;            // [n_rig] g_rig
  long long bytes = 0;             // device bytes of the tables, states and vectors above
  std::vector<int> h_base_of, h_lidar_of, h_var_of;  // host copies for the pattern
  std::unique_ptr<struct RigPattern> pat;
  ~Rig();
};

// The rig's block pattern (host-derived from one generation of the slot pattern) and its device tables.
struct RigPattern {
  long long gen = -1;        // the slot pattern's generation it was derived from
  std::vector<int2> pairs;   // host: rig pairs (u, v), u <= v, ascending
  long long nk = 0, bytes = 0;
  int2 *kkey = nullptr;      // [nk] (slot s, free unknown v) of every K block, s-major, v ascending
  long long *kptr = nullptr; // [nk + 1] K block k's terms kterm[kptr[k] .. kptr[k+1])
  int2 *kterm = nullptr;     // (2 x slot pair + (s > t: H_st read transposed), slot t), t ascending
  int2 *pair_dev = nullptr;  // [pairs]
  long long *jptr = nullptr; // [pairs + 1] rig pair p's terms jterm[jptr[p] .. jptr[p+1])
  int2 *jterm = nullptr;     // (slot s of u, its K block (s, v)), s ascending
  double *K = nullptr;       // [nk][36] column-major, rows of slot s
  double *blocks = nullptr;  // [pairs][36] column-major, rows of unknown u
  SparseSolver *solver = nullptr;
  ~RigPattern() {
    sparse_solver_free(solver);
    cudaFree(kkey); cudaFree(kptr); cudaFree(kterm); cudaFree(pair_dev); cudaFree(jptr); cudaFree(jterm); cudaFree(K);
    cudaFree(blocks);
  }
};

Rig::~Rig() {
  cudaFree(base_of); cudaFree(lidar_of); cudaFree(var_of); cudaFree(var_unknown); cudaFree(var_ptr);
  cudaFree(var_slot); cudaFree(state); cudaFree(state_trial); cudaFree(H); cudaFree(dx);
  cudaFree(dvec); cudaFree(A); cudaFree(K); cudaFree(gb);
  ldlt_work_free(&lw);
}

void rig_free(Rig *r) { delete r; }

namespace {

// X_s = T_b E_l for every slot: R = R_T R_E, p = R_T p_E + p_T
__global__ void rig_compose_kernel(const double *state, const int *base_of, const int *lidar_of, int N, int B,
                                   double *poses) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= N) return;
  double rt[9], pt[3], re[9], pe[3];
  load_pose(state + 12 * (size_t)base_of[s], rt, pt);
  load_pose(state + 12 * ((size_t)B + lidar_of[s]), re, pe);
  double *out = poses + 12 * (size_t)s;
#pragma unroll
  for (int a = 0; a < 3; a++) {
#pragma unroll
    for (int b = 0; b < 3; b++)  // column-major R: out[b * 3 + a] = R[a][b]
      out[b * 3 + a] = rt[a * 3] * re[b] + rt[a * 3 + 1] * re[3 + b] + rt[a * 3 + 2] * re[6 + b];
    out[9 + a] = rt[a * 3] * pe[0] + rt[a * 3 + 1] * pe[1] + rt[a * 3 + 2] * pe[2] + pt[a];
  }
}

// J_s^T x for the 6 entries x of a slot, on an extrinsic: rows k < 3 are R e_k . x_phi + (p x R e_k) . x_t, rows k >= 3
// R e_{k-3} . x_t (r row-major).
__device__ __forceinline__ double ad_column_dot(const double *r, const double *p, int k, const double *x) {
  if (k >= 3) {
    k -= 3;
    return r[k] * x[3] + r[3 + k] * x[4] + r[6 + k] * x[5];
  }
  const double c[3] = {r[k], r[3 + k], r[6 + k]};
  double pc[3];
  cross3(p, c, pc);
  return c[0] * x[0] + c[1] * x[1] + c[2] * x[2] + pc[0] * x[3] + pc[1] * x[4] + pc[2] * x[5];
}

// W[6 s + r][c] = (J Y)[6 s + r][c] for every slot s (one thread per (slot, column)): Y's rows of s's free base plus
// Ad(T_b) = [[R, 0], [p^ R, R]] times the rows of its free extrinsic (the transpose of ad_column_dot); a fixed unknown
// adds nothing. Y [6F rows in the solver's column order col[u]][ld], W [6N][ld], row-major.
__global__ void __launch_bounds__(128) rig_j_apply_kernel(const double *state, const int *base_of, const int *lidar_of,
                                                          const int *var_of, int B, const int *col, const double *Y,
                                                          int ld, int ncols, double *W) {
  const int s = blockIdx.y, c = blockIdx.x * 128 + threadIdx.x;
  if (c >= ncols) return;
  const int vb = var_of[base_of[s]], vl = var_of[B + lidar_of[s]];
  double w[6];
#pragma unroll
  for (int k = 0; k < 6; k++) w[k] = vb >= 0 ? Y[(6 * (size_t)col[vb] + k) * ld + c] : 0.0;
  if (vl >= 0) {
    double r[9], p[3], x[6];
    load_pose(state + 12 * (size_t)base_of[s], r, p);
#pragma unroll
    for (int k = 0; k < 6; k++) x[k] = Y[(6 * (size_t)col[vl] + k) * ld + c];
    double rp[3], rt[3], pc[3];
#pragma unroll
    for (int a = 0; a < 3; a++) {
      rp[a] = r[3 * a] * x[0] + r[3 * a + 1] * x[1] + r[3 * a + 2] * x[2];
      rt[a] = r[3 * a] * x[3] + r[3 * a + 1] * x[4] + r[3 * a + 2] * x[5];
    }
    cross3(p, rp, pc);
#pragma unroll
    for (int a = 0; a < 3; a++) {
      w[a] += rp[a];
      w[3 + a] += pc[a] + rt[a];
    }
  }
#pragma unroll
  for (int k = 0; k < 6; k++) W[(6 * (size_t)s + k) * ld + c] = w[k];
}

// K[:, 6u + k] = sum over the slots s of free unknown u, ascending, of H[:, 6s .. 6s+5] J_s (column block u).
// One thread per row i of H; H is symmetric, so row i of column block s is read down the columns (coalesced in i).
// The sums start at -0.0 so that a one-term sum is bitwise its term (a base with one slot copies H's columns).
__global__ void __launch_bounds__(128) rig_k_kernel(const double *__restrict__ H, int n, const double *state,
                                                    const int *base_of, const int *var_unknown, const int *var_ptr,
                                                    const int *var_slot, int B, double *__restrict__ K) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int u = blockIdx.y;
  if (i >= n) return;
  const bool lidar = var_unknown[u] >= B;
  double acc[6];
#pragma unroll
  for (int k = 0; k < 6; k++) acc[k] = -0.0;
  for (int q = var_ptr[u]; q < var_ptr[u + 1]; q++) {
    const int s = var_slot[q];
    double h[6];
#pragma unroll
    for (int m = 0; m < 6; m++) h[m] = ld_stream(H + (size_t)(6 * s + m) * n + i);
    if (!lidar) {
#pragma unroll
      for (int k = 0; k < 6; k++) acc[k] += h[k];
      continue;
    }
    double r[9], p[3];
    load_pose(state + 12 * (size_t)base_of[s], r, p);
#pragma unroll
    for (int k = 0; k < 6; k++) acc[k] += ad_column_dot(r, p, k, h);
  }
#pragma unroll
  for (int k = 0; k < 6; k++) K[(size_t)(6 * u + k) * n + i] = acc[k];
}

// Entry (row 6u + a, column ck of unknown kv) of the second-order correction of slot s on extrinsic row unknown u, base
// pose (r row-major, p) and slot gradient gs = (g_phi, g_t). Nonzero only in the (lidar, own base) block
//   [e_phi_a, a_phi_k] = (-1/2 g_phi x r_a - g_t x (p x r_a))_k,  [e_t_a, a_phi_k] = (-g_t x r_a)_k  (r_a = R e_a)
// and the (lidar, same lidar) block  [e_phi_a, e_phi_k] = (g_t . p) delta_ak - 1/2 ((r_a.g_t)(p.r_k) + (r_a.p)(g_t.r_k)).
__device__ __forceinline__ double rig_correction(const double *r, const double *p, const double *gs, int a, int k,
                                                 bool own_base) {
  const double *gp = gs, *gt = gs + 3;
  if (own_base) {
    if (k >= 3) return 0.0;
    const double ra[3] = {r[a % 3], r[3 + a % 3], r[6 + a % 3]};
    double v[3];
    if (a >= 3) {
      cross3(gt, ra, v);
      return -v[k];
    }
    double pr[3], w[3];
    cross3(gp, ra, v);
    cross3(p, ra, pr);
    cross3(gt, pr, w);
    return -0.5 * v[k] - w[k];
  }
  if (a >= 3 || k >= 3) return 0.0;
  const double ra[3] = {r[a], r[3 + a], r[6 + a]}, rk[3] = {r[k], r[3 + k], r[6 + k]};
  const double rag = ra[0] * gt[0] + ra[1] * gt[1] + ra[2] * gt[2], rkg = rk[0] * gt[0] + rk[1] * gt[1] + rk[2] * gt[2];
  const double rap = ra[0] * p[0] + ra[1] * p[1] + ra[2] * p[2], rkp = rk[0] * p[0] + rk[1] * p[1] + rk[2] * p[2];
  const double gtp = gt[0] * p[0] + gt[1] * p[1] + gt[2] * p[2];
  return (a == k ? gtp : 0.0) - 0.5 * (rag * rkp + rap * rkg);
}

// H_rig[r, c] = sum over the slots s of r's unknown u, ascending, of J_s[:, a]^T K[6s .. 6s+5, c], then (CORRECTION)
// the correction over the same slots, ascending; lower triangle only, mirrored into the upper one. Column c = n_rig is
// g: g_rig[r] = sum_s J_s[:, a]^T g_s. One thread per row r, one grid row per column c.
template <bool CORRECTION>
__global__ void __launch_bounds__(128) rig_jtk_kernel(const double *__restrict__ K, const double *__restrict__ g, int n,
                                                      int nr, const double *state, const int *base_of,
                                                      const int *var_unknown, const int *var_ptr, const int *var_slot,
                                                      int B, double *__restrict__ Hr, double *__restrict__ gr) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  const int col = blockIdx.y;
  if (row >= nr) return;
  const bool grad = col == nr;
  if (!grad && row < col) return;
  const int u = row / 6, a = row % 6;
  const int ku = var_unknown[u];
  const bool lidar = ku >= B;
  const double *x = grad ? g : K + (size_t)col * n;
  double acc = -0.0;
  for (int q = var_ptr[u]; q < var_ptr[u + 1]; q++) {
    const int s = var_slot[q];
    if (!lidar) {
      acc += x[6 * s + a];
      continue;
    }
    double r[9], p[3];
    load_pose(state + 12 * (size_t)base_of[s], r, p);
    acc += ad_column_dot(r, p, a, x + 6 * s);
  }
  if (CORRECTION && !grad && lidar) {
    const int kv = var_unknown[col / 6], k = col % 6;
    if (kv == ku || kv < B) {
      for (int q = var_ptr[u]; q < var_ptr[u + 1]; q++) {
        const int s = var_slot[q];
        if (kv != ku && base_of[s] != kv) continue;
        double r[9], p[3];
        load_pose(state + 12 * (size_t)base_of[s], r, p);
        acc += rig_correction(r, p, g + 6 * s, a, k, kv != ku);
      }
    }
  }
  if (grad) {
    gr[row] = acc;
  } else {
    Hr[(size_t)col * nr + row] = acc;
    if (row != col) Hr[(size_t)row * nr + col] = acc;
  }
}

// K block k = (s, v): K_sv[m, c] = sum over its terms (slot t of v, ascending) of J_t[:, c]^T H_st[m, :], H_st read
// from the slot blocks Hb (transposed when s > t). One thread per row m; the sums start at -0.0.
__global__ void __launch_bounds__(128) rig_k_blocks_kernel(const int2 *__restrict__ kkey, const long long *kptr,
                                                           const int2 *__restrict__ kterm, long long nk,
                                                           const double *__restrict__ Hb, const double *state,
                                                           const int *base_of, const int *var_unknown, int B,
                                                           double *__restrict__ K) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 6 * nk) return;
  const long long k = i / 6;
  const int m = (int)(i % 6);
  const bool lidar = var_unknown[kkey[k].y] >= B;
  double acc[6];
#pragma unroll
  for (int c = 0; c < 6; c++) acc[c] = -0.0;
  for (long long q = kptr[k]; q < kptr[k + 1]; q++) {
    const int2 w = kterm[q];
    const double *hb = Hb + 36 * (size_t)(w.x >> 1);
    double h[6];  // row m of H_st
#pragma unroll
    for (int n = 0; n < 6; n++) h[n] = (w.x & 1) ? hb[6 * m + n] : hb[6 * n + m];
    if (!lidar) {
#pragma unroll
      for (int c = 0; c < 6; c++) acc[c] += h[c];
      continue;
    }
    double r[9], p[3];
    load_pose(state + 12 * (size_t)base_of[w.y], r, p);
#pragma unroll
    for (int c = 0; c < 6; c++) acc[c] += ad_column_dot(r, p, c, h);
  }
#pragma unroll
  for (int c = 0; c < 6; c++) K[36 * (size_t)k + 6 * c + m] = acc[c];
}

// One warp per rig pair p = (u, v), u <= v: block[r, c] = sum over its terms (slot s of u with K block (s, v),
// ascending) of J_s[:, r]^T K_sv[:, c], each slot's correction added after its term: on a (base, lidar) pair for the
// slots of u on that lidar (rig_correction with the roles of r and c swapped: the dense kernel's (lidar, base) entry),
// on a (lidar, same lidar) pair for every slot. Lane l takes the terms l, l + 32, ... from -0.0; the lanes' sums meet
// in warp_sum. A diagonal pair keeps its lower triangle, mirrored, and sums g_rig(u) over the same terms.
__global__ void __launch_bounds__(128) rig_jtk_blocks_kernel(const int2 *__restrict__ pairs, const long long *jptr,
                                                             const int2 *__restrict__ jterm, long long np,
                                                             const double *__restrict__ K, const double *g,
                                                             const double *state, const int *base_of,
                                                             const int *lidar_of, const int *var_unknown, int B,
                                                             double *__restrict__ blocks, double *__restrict__ gr) {
  const long long p = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (p >= np) return;
  const int2 pr = pairs[p];
  const int ku = var_unknown[pr.x], kv = var_unknown[pr.y];
  const bool lidar = ku >= B, diag = pr.x == pr.y;
  const bool corr = kv >= B && (diag || !lidar);  // (lidar, same lidar) or (base, lidar)
  double acc[36], ga[6];
#pragma unroll
  for (int e = 0; e < 36; e++) acc[e] = -0.0;
#pragma unroll
  for (int a = 0; a < 6; a++) ga[a] = -0.0;
  for (long long t = jptr[p] + lane; t < jptr[p + 1]; t += 32) {
    const int2 w = jterm[t];
    const int s = w.x;
    const double *k = K + 36 * (size_t)w.y;
    double r[9], q[3];
    if (lidar || corr) load_pose(state + 12 * (size_t)base_of[s], r, q);
#pragma unroll
    for (int c = 0; c < 6; c++)
#pragma unroll
      for (int a = 0; a < 6; a++) acc[6 * c + a] += lidar ? ad_column_dot(r, q, a, k + 6 * c) : k[6 * c + a];
    if (corr && (diag || lidar_of[s] == kv - B)) {
      const double *gs = g + 6 * (size_t)s;
#pragma unroll
      for (int c = 0; c < 6; c++)
#pragma unroll
        for (int a = 0; a < 6; a++)
          acc[6 * c + a] += diag ? rig_correction(r, q, gs, a, c, false) : rig_correction(r, q, gs, c, a, true);
    }
    if (diag) {
#pragma unroll
      for (int a = 0; a < 6; a++) ga[a] += lidar ? ad_column_dot(r, q, a, g + 6 * (size_t)s) : g[6 * (size_t)s + a];
    }
  }
  double *out = blocks + 36 * (size_t)p;
#pragma unroll
  for (int e = 0; e < 36; e++) {
    const double h = warp_sum(acc[e]);
    const int a = e % 6, c = e / 6;
    if (lane == (e & 31)) {
      if (!diag) {
        out[e] = h;
      } else if (a >= c) {
        out[e] = h;
        out[6 * a + c] = h;
      }
    }
  }
  if (diag) {
#pragma unroll
    for (int a = 0; a < 6; a++) {
      const double h = warp_sum(ga[a]);
      if (lane == a) gr[6 * (size_t)pr.x + a] = h;
    }
  }
}

// Free unknowns take the left step of their slice of dx; fixed ones are copied.
__global__ void rig_update_kernel(const double *state, const double *dx, const int *var_of, int U, double *out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= U) return;
  const int v = var_of[j];
  if (v >= 0) {
    pose_update_one(state + 12 * (size_t)j, dx + 6 * (size_t)v, out + 12 * (size_t)j);
  } else {
#pragma unroll
    for (int e = 0; e < 12; e++) out[12 * (size_t)j + e] = state[12 * (size_t)j + e];
  }
}

}  // namespace

int rig_build(cudaStream_t st, int N, int B, int L, const int32_t *base_of, const int32_t *lidar_of,
              const uint8_t *base_fixed, const uint8_t *lidar_fixed, bool sparse, Rig **out) {
  std::unique_ptr<Rig> r(new Rig());
  r->N = N; r->B = B; r->L = L;
  r->sparse = sparse;
  const int U = B + L;
  std::vector<int> var_of(U, -1), var_unknown;
  for (int j = 0; j < U; j++) {
    const bool fixed = j < B ? (base_fixed && base_fixed[j]) : (lidar_fixed && lidar_fixed[j - B]);
    if (j < B && fixed) r->any_base_fixed = true;
    if (fixed) continue;
    if (j < B) r->FB++;
    var_of[j] = (int)var_unknown.size();
    var_unknown.push_back(j);
  }
  r->F = (int)var_unknown.size();
  std::vector<int> var_ptr(r->F + 1, 0), var_slot;
  for (int u = 0; u < r->F; u++) {
    const int j = var_unknown[u];
    for (int s = 0; s < N; s++)
      if ((j < B && base_of[s] == j) || (j >= B && lidar_of[s] == j - B)) var_slot.push_back(s);
    var_ptr[u + 1] = (int)var_slot.size();
  }
  const size_t nr = 6 * (size_t)r->F, n = 6 * (size_t)N;
  TRY(dev_alloc(&r->base_of, N));
  TRY(dev_alloc(&r->lidar_of, N));
  TRY(dev_alloc(&r->var_of, U));
  TRY(dev_alloc(&r->var_unknown, r->F));
  TRY(dev_alloc(&r->var_ptr, r->F + 1));
  TRY(dev_alloc(&r->var_slot, var_slot.size()));
  TRY(dev_alloc(&r->state, 12 * (size_t)U));
  TRY(dev_alloc(&r->state_trial, 12 * (size_t)U));
  TRY(dev_alloc(&r->dx, nr));
  TRY(dev_alloc(&r->dvec, nr));
  if (sparse) {
    TRY(dev_alloc(&r->gb, nr));
    r->h_base_of.assign(base_of, base_of + N);
    r->h_lidar_of.assign(lidar_of, lidar_of + N);
    r->h_var_of = var_of;
    r->bytes = (long long)(sizeof(int) * (2 * (size_t)N + U + r->F + r->F + 1 + std::max<size_t>(1, var_slot.size())) +
                           sizeof(double) * (24 * (size_t)U + 3 * nr));
  } else {
    TRY(dev_alloc(&r->H, nr * nr + nr));
    TRY(dev_alloc(&r->A, nr * nr));
    TRY(dev_alloc(&r->K, nr * n));
  }
  CUDA_TRY(cudaMemcpyAsync(r->base_of, base_of, sizeof(int) * N, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(r->lidar_of, lidar_of, sizeof(int) * N, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(r->var_of, var_of.data(), sizeof(int) * U, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(r->var_unknown, var_unknown.data(), sizeof(int) * r->F, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(r->var_ptr, var_ptr.data(), sizeof(int) * (r->F + 1), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(r->var_slot, var_slot.data(), sizeof(int) * var_slot.size(), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaStreamSynchronize(st));  // the host tables go out of scope
  *out = r.release();
  return BALM_OK;
}

int rig_blocks_sync(Rig *r, cudaStream_t st, const std::vector<int2> &slot_pairs, long long gen, double *scal,
                    int *flags, const char *who) {
  if (r->pat && r->pat->gen == gen) return BALM_OK;
  const int N = r->N, B = r->B, F = r->F;
  auto refuse = [&](const char *what) {
    balm_set_error(std::string(who) + ": " + what);
    return (int)BALM_ERR_UNSUPPORTED;
  };
  // the free unknowns of every slot, ascending (its base pose's before its extrinsic's)
  auto free_of = [&](int s, int *u) {
    int n = 0;
    const int a = r->h_var_of[r->h_base_of[s]], b = r->h_var_of[B + r->h_lidar_of[s]];
    if (a >= 0) u[n++] = a;
    if (b >= 0) u[n++] = b;
    return n;
  };
  // every slot's neighbours t in the slot pattern, ascending, with 2 x pair + (s > t)
  std::vector<long long> aptr((size_t)N + 1, 0);
  for (const int2 &q : slot_pairs) {
    aptr[q.x + 1]++;
    if (q.x != q.y) aptr[q.y + 1]++;
  }
  for (int s = 0; s < N; s++) aptr[s + 1] += aptr[s];
  std::vector<int2> adj(aptr[N]);  // (t, source); the ascending pairs fill every list in ascending t
  {
    std::vector<long long> fill(aptr.begin(), aptr.end() - 1);
    for (size_t p = 0; p < slot_pairs.size(); p++) {
      const int2 q = slot_pairs[p];
      adj[fill[q.x]++] = make_int2(q.y, (int)(2 * p));
      if (q.x != q.y) adj[fill[q.y]++] = make_int2(q.x, (int)(2 * p + 1));
    }
  }
  // K blocks (s, v) for v >= the first free unknown of s, with their terms (t ascending); every slot gets the K blocks
  // of its own free unknowns even without a diagonal slot pair
  std::vector<int2> kkey, kterm;
  std::vector<long long> kptr;
  {
    std::vector<int3> cand;  // (v, t, source); t = -1: a block without this term
    for (int s = 0; s < N; s++) {
      int us[2], ut[2];
      const int ns = free_of(s, us);
      if (!ns) continue;
      cand.clear();
      for (int a = 0; a < ns; a++) cand.push_back(make_int3(us[a], -1, -1));
      for (long long q = aptr[s]; q < aptr[s + 1]; q++) {
        const int nt = free_of(adj[q].x, ut);
        for (int b = 0; b < nt; b++)
          if (ut[b] >= us[0]) cand.push_back(make_int3(ut[b], adj[q].x, adj[q].y));
      }
      std::stable_sort(cand.begin(), cand.end(), [](const int3 &x, const int3 &y) { return x.x < y.x; });
      for (size_t q = 0; q < cand.size(); q++) {
        if (q == 0 || cand[q].x != cand[q - 1].x) {
          kptr.push_back((long long)kterm.size());
          kkey.push_back(make_int2(s, cand[q].x));
        }
        if (cand[q].y >= 0) kterm.push_back(make_int2(cand[q].z, cand[q].y));
      }
    }
    kptr.push_back((long long)kterm.size());
  }
  const long long nk = (long long)kkey.size();
  if (nk >= (1LL << 31)) return refuse("2^31 or more rig K blocks");
  // rig pairs (u, v), u <= v: one term (s, k) for every K block k = (s, v) and free unknown u <= v of s, in ascending k,
  // hence ascending s within a pair
  std::vector<unsigned long long> key;
  key.reserve(2 * nk);
  for (long long k = 0; k < nk; k++) {
    int us[2];
    const int ns = free_of(kkey[k].x, us);
    for (int a = 0; a < ns; a++)
      if (us[a] <= kkey[k].y) key.push_back((unsigned long long)us[a] * F + kkey[k].y);
  }
  std::vector<unsigned long long> ukey(key);
  std::sort(ukey.begin(), ukey.end());
  ukey.erase(std::unique(ukey.begin(), ukey.end()), ukey.end());
  if (ukey.size() >= ((size_t)1 << 30)) return refuse("2^30 or more rig block pairs");
  std::unique_ptr<RigPattern> pat(new RigPattern());
  const size_t np = ukey.size();
  pat->gen = gen;
  pat->nk = nk;
  pat->pairs.resize(np);
  for (size_t p = 0; p < np; p++) pat->pairs[p] = make_int2((int)(ukey[p] / F), (int)(ukey[p] % F));
  std::vector<long long> jptr(np + 1, 0);
  std::vector<int> jpair(key.size());
  for (size_t q = 0; q < key.size(); q++) {
    jpair[q] = (int)(std::lower_bound(ukey.begin(), ukey.end(), key[q]) - ukey.begin());
    jptr[jpair[q] + 1]++;
  }
  for (size_t p = 0; p < np; p++) jptr[p + 1] += jptr[p];
  std::vector<int2> jterm(key.size());
  {
    std::vector<long long> fill(jptr.begin(), jptr.end() - 1);
    size_t q = 0;
    for (long long k = 0; k < nk; k++) {
      int us[2];
      const int ns = free_of(kkey[k].x, us);
      for (int a = 0; a < ns; a++)
        if (us[a] <= kkey[k].y) jterm[fill[jpair[q++]]++] = make_int2(kkey[k].x, (int)k);
    }
  }
  auto put = [&](auto **d, const auto &h) -> int {  // pat frees whatever it holds when a step fails
    TRY(dev_alloc(d, h.size()));
    pat->bytes += (long long)(sizeof(**d) * std::max<size_t>(1, h.size()));
    if (!h.empty()) CUDA_TRY(cudaMemcpyAsync(*d, h.data(), sizeof(**d) * h.size(), cudaMemcpyHostToDevice, st));
    return BALM_OK;
  };
  TRY(put(&pat->kkey, kkey));
  TRY(put(&pat->kptr, kptr));
  TRY(put(&pat->kterm, kterm));
  TRY(put(&pat->pair_dev, pat->pairs));
  TRY(put(&pat->jptr, jptr));
  TRY(put(&pat->jterm, jterm));
  TRY(dev_alloc(&pat->K, 36 * (size_t)nk));
  TRY(dev_alloc(&pat->blocks, 36 * np));
  pat->bytes += (long long)(sizeof(double) * 36 * (std::max<size_t>(1, (size_t)nk) + np));
  TRY(sparse_solver_build(st, F, pat->pairs, pat->blocks, r->gb, r->dvec, r->dx, scal, flags, who, &pat->solver));
  CUDA_TRY(cudaStreamSynchronize(st));  // the host tables above are freed on return
  r->pat = std::move(pat);
  return BALM_OK;
}

int rig_reduce_blocks(const Rig *r, cudaStream_t st, const double *state, const double *Hb, const double *g,
                      long long *launches) {
  const RigPattern &u = *r->pat;
  const long long np = (long long)u.pairs.size();
  if (u.nk)
    rig_k_blocks_kernel<<<(unsigned)((6 * u.nk + 127) / 128), 128, 0, st>>>(u.kkey, u.kptr, u.kterm, u.nk, Hb, state,
                                                                            r->base_of, r->var_unknown, r->B, u.K);
  rig_jtk_blocks_kernel<<<(unsigned)((32 * np + 127) / 128), 128, 0, st>>>(u.pair_dev, u.jptr, u.jterm, np, u.K, g,
                                                                           state, r->base_of, r->lidar_of,
                                                                           r->var_unknown, r->B, u.blocks, r->gb);
  *launches += 2;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

bool rig_sparse(const Rig *r) { return r->sparse; }
const std::vector<int2> &rig_pairs(const Rig *r) { return r->pat->pairs; }
const double *rig_blocks(const Rig *r) { return r->pat->blocks; }
SparseSolver *rig_solver(const Rig *r) { return r->pat->solver; }

long long rig_blocks_bytes(const Rig *r, int64_t *l_blocks, int64_t *levels) {
  int64_t sb = 0;
  sparse_solver_stats(r->pat->solver, l_blocks, levels, &sb);
  return r->bytes + r->pat->bytes + sb;
}

int rig_n(const Rig *r) { return 6 * r->F; }
int rig_bases(const Rig *r) { return r->B; }
int rig_lidars(const Rig *r) { return r->L; }
bool rig_any_base_fixed(const Rig *r) { return r->any_base_fixed; }
int rig_free_bases(const Rig *r) { return r->FB; }
DenseSystem rig_system(Rig *r) {
  const int nr = 6 * r->F;
  if (r->sparse) return DenseSystem{nr, nullptr, r->gb, r->dx, r->dvec, nullptr, &r->lw};
  return DenseSystem{nr, r->H, r->H + (size_t)nr * nr, r->dx, r->dvec, r->A, &r->lw};
}
double *rig_state(Rig *r, bool trial) { return trial ? r->state_trial : r->state; }
void rig_swap_states(Rig *r) { std::swap(r->state, r->state_trial); }

int rig_compose(const Rig *r, cudaStream_t st, const double *state, double *poses, long long *launches) {
  rig_compose_kernel<<<(r->N + 127) / 128, 128, 0, st>>>(state, r->base_of, r->lidar_of, r->N, r->B, poses);
  *launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int rig_reduce(const Rig *r, cudaStream_t st, const double *state, const double *H, const double *g,
               long long *launches) {
  const int n = 6 * r->N, nr = 6 * r->F;
  rig_k_kernel<<<dim3((n + 127) / 128, r->F), 128, 0, st>>>(H, n, state, r->base_of, r->var_unknown, r->var_ptr,
                                                            r->var_slot, r->B, r->K);
  rig_jtk_kernel<true><<<dim3((nr + 127) / 128, nr + 1), 128, 0, st>>>(r->K, g, n, nr, state, r->base_of,
                                                                       r->var_unknown, r->var_ptr, r->var_slot, r->B,
                                                                       r->H, r->H + (size_t)nr * nr);
  *launches += 2;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int rig_reduce_raw(const Rig *r, cudaStream_t st, const double *state, const double *R, double *out,
                   long long *launches) {
  const int n = 6 * r->N, nr = 6 * r->F;
  rig_k_kernel<<<dim3((n + 127) / 128, r->F), 128, 0, st>>>(R, n, state, r->base_of, r->var_unknown, r->var_ptr,
                                                            r->var_slot, r->B, r->K);
  rig_jtk_kernel<false><<<dim3((nr + 127) / 128, nr), 128, 0, st>>>(r->K, nullptr, n, nr, state, r->base_of,
                                                                    r->var_unknown, r->var_ptr, r->var_slot, r->B,
                                                                    out, nullptr);
  *launches += 2;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int rig_update(const Rig *r, cudaStream_t st, const double *state, double *state_out, long long *launches) {
  const int U = r->B + r->L;
  rig_update_kernel<<<(U + 127) / 128, 128, 0, st>>>(state, r->dx, r->var_of, U, state_out);
  *launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int rig_apply_j(const Rig *r, cudaStream_t st, const double *state, const int *col, const double *Y, int ld, int ncols,
                double *W, long long *launches) {
  rig_j_apply_kernel<<<dim3((ncols + 127) / 128, r->N), 128, 0, st>>>(state, r->base_of, r->lidar_of, r->var_of, r->B, col,
                                                                      Y, ld, ncols, W);
  *launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

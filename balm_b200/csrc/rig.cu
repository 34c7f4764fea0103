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
};

void rig_free(Rig *r) {
  if (!r) return;
  cudaFree(r->base_of); cudaFree(r->lidar_of); cudaFree(r->var_of); cudaFree(r->var_unknown); cudaFree(r->var_ptr);
  cudaFree(r->var_slot); cudaFree(r->state); cudaFree(r->state_trial); cudaFree(r->H); cudaFree(r->dx);
  cudaFree(r->dvec); cudaFree(r->A); cudaFree(r->K);
  ldlt_work_free(&r->lw);
  delete r;
}

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
              const uint8_t *base_fixed, const uint8_t *lidar_fixed, Rig **out) {
  std::unique_ptr<Rig, void (*)(Rig *)> r(new Rig(), rig_free);
  r->N = N; r->B = B; r->L = L;
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
  TRY(dev_alloc(&r->H, nr * nr + nr));
  TRY(dev_alloc(&r->dx, nr));
  TRY(dev_alloc(&r->dvec, nr));
  TRY(dev_alloc(&r->A, nr * nr));
  TRY(dev_alloc(&r->K, nr * n));
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

int rig_n(const Rig *r) { return 6 * r->F; }
int rig_bases(const Rig *r) { return r->B; }
int rig_lidars(const Rig *r) { return r->L; }
bool rig_any_base_fixed(const Rig *r) { return r->any_base_fixed; }
int rig_free_bases(const Rig *r) { return r->FB; }
DenseSystem rig_system(Rig *r) {
  const int nr = 6 * r->F;
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

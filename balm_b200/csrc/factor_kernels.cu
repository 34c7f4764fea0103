// factor_kernels.cu -- the O(K) streaming passes of the eigen-factor evaluation (HBM-bound kernels K1-K3).
//
//   voxel_sums_kernel + voxel_eig_kernel:
//                        per voxel  C = sum_i T_i C_i T_i^T (+fix), v_bar, eig(A)  -> residual (+ stats table)
//                        = VOX_HESS::evaluate_only_residual (bavoxel.hpp:428-470) and phase 1 of
//                          left_evaluate_acc2 (bavoxel.hpp:322-360)
//   obs_pass_kernel    : per observation  g_k^i, a_i, gradient and diagonal-block terms
//                        = left_evaluate_acc2 per-observation loop (bavoxel.hpp:365-402); writes the scaled
//                          factor matrix G' (3 rows per voxel, 6N columns) consumed by the SYRK: as fp64 (OBS_FP64)
//                          or directly as int8 digit planes (OBS_INT8 / OBS_FUSED, tensor path)
//   obs_reduce_kernel  : fixed-order reduction of the per-chunk gradient / diagonal-block partials
//
// Layouts: observations SoA obs[c][s] (c<10, s in CSR order), so a warp reading 32 consecutive slots of one
// voxel issues ten fully coalesced 256-byte requests; the stats table is AoS (20 doubles per voxel) because
// the observation pass reads it warp-uniformly (one broadcast transaction per 16 bytes).
#include <type_traits>
#include "internal.cuh"

namespace {

constexpr int STATS_THREADS = 256;

struct StatsArgs {
  const double *obs;
  int64_t Kp;
  const int *pose_idx;
  const long long *row_ptr;
  const double *fix;  // SoA [10][M] or null
  int64_t M;
  const double *poses;
  int N;
  int64_t v0, v1;
};

// voxel_sums_kernel: one WARP per voxel, no block barriers. Lanes stride over the voxel's observations with two
// observations (20 independent 8-byte loads) in flight per lane.
constexpr int STATS_WARPS = STATS_THREADS / 32;

// ---- the stats / residual pass: the streaming half and the eigen half as two kernels ----
// (one kernel doing both, the eigen-solve in every lane of the voxel's warp, measured at C3: 0.916 -> 0.831 ms)
// voxel_sums_kernel: the warp only reduces the ten cluster sums and moves on -- no serial eigen-solve between two
// voxels' loads. voxel_eig_kernel: one THREAD per voxel does the eigen-solve (M independent chains instead of M x 32
// redundant ones), the residual term and the stats record.
template <bool SMEM_POSES>
__global__ void __launch_bounds__(STATS_THREADS, 3) voxel_sums_kernel(StatsArgs a, double *sums /*[v1-v0][10]*/) {
  extern __shared__ double s_poses[];
  if (SMEM_POSES) {
    for (int e = threadIdx.x; e < 12 * a.N; e += STATS_THREADS) s_poses[e] = a.poses[e];
    __syncthreads();
  }
  const double *ptab = SMEM_POSES ? s_poses : a.poses;
  const int lane = threadIdx.x & 31;
  const int64_t gw = (int64_t)blockIdx.x * STATS_WARPS + (threadIdx.x >> 5);
  const int64_t nw = (int64_t)gridDim.x * STATS_WARPS;
  for (int64_t v = a.v0 + gw; v < a.v1; v += nw) {
    const long long s0 = a.row_ptr[v];
    const int k = (int)(a.row_ptr[v + 1] - s0);
    double acc[10];
#pragma unroll
    for (int c = 0; c < 10; c++) acc[c] = 0.0;
    for (int j = lane; j < k; j += 64) {
      const long long sA = s0 + j;
      const bool hasB = j + 32 < k;
      const long long sB = hasB ? sA + 32 : sA;
      double oa[10], ob[10];
#pragma unroll
      for (int c = 0; c < 10; c++) { oa[c] = ld_stream(a.obs + c * a.Kp + sA); ob[c] = ld_stream(a.obs + c * a.Kp + sB); }
      const int pa = __ldg(a.pose_idx + sA), pb = __ldg(a.pose_idx + sB);
      double r[9], p[3];
      load_pose_any<SMEM_POSES>(ptab + 12 * pa, r, p);
      WC w = world_cluster(oa, r, p);
      acc[0] += w.p00; acc[1] += w.p01; acc[2] += w.p02; acc[3] += w.p11; acc[4] += w.p12;
      acc[5] += w.p22; acc[6] += w.v0;  acc[7] += w.v1;  acc[8] += w.v2;  acc[9] += w.n;
      if (hasB) {
        load_pose_any<SMEM_POSES>(ptab + 12 * pb, r, p);
        w = world_cluster(ob, r, p);
        acc[0] += w.p00; acc[1] += w.p01; acc[2] += w.p02; acc[3] += w.p11; acc[4] += w.p12;
        acc[5] += w.p22; acc[6] += w.v0;  acc[7] += w.v1;  acc[8] += w.v2;  acc[9] += w.n;
      }
    }
#pragma unroll
    for (int c = 0; c < 10; c++) {
      acc[c] = warp_sum(acc[c]);
      if (a.fix) acc[c] += __ldg(a.fix + c * a.M + v);
    }
    double *dst = sums + (v - a.v0) * 10;
#pragma unroll
    for (int c = 0; c < 10; c++)
      if (lane == c) dst[c] = acc[c];
  }
}

// With VoxelLoss, rho and w = rho'(lambda_0) once per voxel: the residual term is coe rho(lambda_0) and the stats row
// gets coe w in place of coe, which every Hessian, gradient and covariance term downstream is linear in.
template <bool STORE, typename Loss>
__global__ void __launch_bounds__(128) voxel_eig_kernel(const double *sums, const double *coe_all, int64_t v0, int64_t v1,
                                                        double *stats, double *res_part, Loss loss) {
  constexpr bool robust = std::is_same<Loss, VoxelLoss>::value;
  __shared__ double red[4];
  double res_acc = 0.0;
  for (int64_t v = v0 + (int64_t)blockIdx.x * 128 + threadIdx.x; v < v1; v += (int64_t)gridDim.x * 128) {
    const double2 *src = reinterpret_cast<const double2 *>(sums + (v - v0) * 10);
    double acc[10];
#pragma unroll
    for (int c = 0; c < 5; c++) {
      const double2 x = src[c];
      acc[2 * c] = x.x;
      acc[2 * c + 1] = x.y;
    }
    const double inv = 1.0 / acc[9];
    const double vb0 = acc[6] * inv, vb1 = acc[7] * inv, vb2 = acc[8] * inv;
    double lam[3], u0[3], u1[3], u2[3];
    eig3_jacobi(acc[0] * inv - vb0 * vb0, acc[1] * inv - vb0 * vb1, acc[2] * inv - vb0 * vb2,
                acc[3] * inv - vb1 * vb1, acc[4] * inv - vb1 * vb2, acc[5] * inv - vb2 * vb2, lam, u0, u1, u2);
    const double coe = __ldg(coe_all + v);
    if constexpr (robust) {
      double rho, w;
      loss_rho(loss.kind, loss.scale, lam[0], &rho, &w);
      res_acc += coe * rho;
      if (loss.lam) { loss.lam[v - v0] = lam[0]; loss.w[v - v0] = w; }
      if (STORE) store_stats_row(stats + (v - v0) * BALM_STATS_STRIDE, vb0, vb1, vb2, u0, u1, u2, inv, coe * w, lam);
    } else {
      res_acc += coe * lam[0];
      if (STORE) store_stats_row(stats + (v - v0) * BALM_STATS_STRIDE, vb0, vb1, vb2, u0, u1, u2, inv, coe, lam);
    }
  }
  res_acc = warp_sum(res_acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = res_acc;
  __syncthreads();
  if (threadIdx.x == 0) res_part[blockIdx.x] = (red[0] + red[1]) + (red[2] + red[3]);
}

// deterministic sum of the per-CTA residual partials (single warp)
__global__ void residual_reduce_kernel(const double *part, int nparts, double *out, int accumulate) {
  double s = 0.0;
  for (int i = threadIdx.x; i < nparts; i += 32) s += part[i];
  s = warp_sum(s);
  if (threadIdx.x == 0) out[0] = accumulate ? out[0] + s : s;
}

struct ObsArgs {
  const double *obs;
  int64_t Kp;
  const long long *row_ptr;
  const double *poses;
  const double *stats;  // batch-local [nv][20]
  int64_t v0, v1;       // batch voxel range
  int N, Np, ldg;
  int chunk;            // voxels per chunk (dense) or list positions per segment (csc)
  double *G;            // [3*(v1-v0)][ldg]
  double *part;         // [chunks][27][Np]
  unsigned long long *colmax;  // [ldg] or null: running max |G'[:,j]| (tensor path column scales)
  // tensor path, digit-plane output (OBS_INT8)
  const double *sc;     // [ldg] column scales 2^p
  int8_t *Gq;           // [S][rows_alloc][ldg]
  int64_t plane_stride;
  const int *S_dev;     // digit-plane count chosen on the device by tc_scale_kernel
  const int *skip;      // device flag, nonzero -> nothing to do. OBS_INT8: the speculative single sweep was accepted;
                        // OBS_FUSED: the planes and accumulators of the same poses and scales are still in place
  // csc
  const int *csc_ptr, *csc_obs, *csc_vox;
  const int *csc_lo, *csc_hi;  // [N] this batch's segment of every pose's list
};

// One lane = one pose; a warp covers 32 consecutive poses and walks a chunk of voxels, so the observation
// loads of a dense scene (slot j == pose j) are coalesced and the 27 accumulators stay in registers.
enum { OBS_FP64 = 0, OBS_MAXONLY = 1, OBS_INT8 = 2, OBS_FUSED = 3, OBS_BLOCKS = 4 };
constexpr int OBS_STAGES = 4;  // cp.async ring depth of the dense sweep (iterations in flight per warp)
// MODE: OBS_FP64    writes fp64 G' + gradient / diagonal blocks                          [fp64 SYRK path]
//       OBS_MAXONLY first sweep of the tensor path: column maxima of G' (-> power-of-two column scales) and the
//                   gradient / diagonal-block accumulators (kept here so that the second sweep is lean)
//       OBS_INT8    second sweep: writes the balanced base-256 digit planes of rint(G' * sc) directly, so the
//                   tensor path never materialises G' in fp64
//       OBS_FUSED   both sweeps in one, with the column scales of the PREVIOUS evaluation of the same voxels (an LM
//                   step moves the column maxima by far less than the factor 2 of headroom a balanced top digit
//                   has); tc_scale_kernel checks the new maxima against the scales used and, if a column overflowed
//                   or lost precision, re-arms the OBS_INT8 sweep (which otherwise returns at once)
//       OBS_BLOCKS  the three scaled G' rows of every observation into a.G[s][18] (s: the observation's CSR index) +
//                   gradient / diagonal blocks                                        [block-sparse path, blocks.cu]
template <bool DENSE, int MODE, int WPC = 4, int MINB = 2>
__global__ void __launch_bounds__(WPC * 32, MINB) obs_pass_kernel(ObsArgs a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int tile = blockIdx.y * WPC + warp;
  const int i = tile * 32 + lane;
  if (tile * 32 >= a.N) return;
  constexpr bool EMIT = (MODE == OBS_INT8 || MODE == OBS_FUSED);
  if (EMIT && a.skip && *a.skip) return;
  const bool active = i < a.N;
  double r[9], p[3];
  if (active) load_pose(a.poses + 12 * i, r, p);
  double acc[BALM_ACC];
#pragma unroll
  for (int q = 0; q < BALM_ACC; q++) acc[q] = 0.0;
  unsigned cmax[6] = {0, 0, 0, 0, 0, 0};  // high words of max|G'_j| (non-negative doubles order like their bit patterns)
  double scl[6] = {0, 0, 0, 0, 0, 0};
  const int S = EMIT ? *a.S_dev : 0;
  if (EMIT && active) {
#pragma unroll
    for (int q = 0; q < 6; q++) scl[q] = __ldg(a.sc + 6 * i + q);
  }

  long long t0, t1;
  if (DENSE) {
    t0 = a.v0 + (long long)blockIdx.x * a.chunk;
    t1 = t0 + a.chunk < a.v1 ? t0 + a.chunk : a.v1;
  } else {
    const int b = active ? a.csc_lo[i] : 0, e = active ? a.csc_hi[i] : 0;
    t0 = b + (long long)blockIdx.x * a.chunk;
    t1 = t0 + a.chunk < e ? t0 + a.chunk : e;
  }

  // Observation prefetch. Dense scenes (s = v*N + i, no index loads): the ten words of the next OBS_STAGES iterations
  // are in flight as cp.async copies into a per-warp shared-memory ring -- with 8 resident warps per SM (register
  // file) one iteration ahead kept only ~20 KB per SM in flight, which is what bounded the sweep at half the HBM rate;
  // every lane copies and later reads its own words, so no barrier is involved. Pose-major lists (sparse): the ten
  // words of iteration t+1 are requested into registers before iteration t is computed.
  __shared__ __align__(16) double s_obs[DENSE ? WPC : 1][DENSE ? OBS_STAGES : 1][10][32];
  double onext[DENSE ? 1 : 10];
  auto stage = [&](long long t, int slot) {
    if (t < t1 && active) {
      const double *src = a.obs + (t * (long long)a.N + i);
      const uint32_t dst = (uint32_t)__cvta_generic_to_shared(&s_obs[DENSE ? warp : 0][DENSE ? slot : 0][0][lane]);
#pragma unroll
      for (int c = 0; c < 10; c++)
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(dst + c * 256), "l"(src + c * a.Kp) : "memory");
    }
    asm volatile("cp.async.commit_group;\n" ::: "memory");  // one group per call, empty or not: uniform accounting
  };
  auto issue = [&](long long t, double *dst) {
    if (t < t1) {
      const long long s = a.csc_obs[t];
#pragma unroll
      for (int c = 0; c < 10; c++) dst[c] = ld_stream(a.obs + c * a.Kp + s);
    }
  };
  int slot = 0;
  if (DENSE) {
#pragma unroll
    for (int d = 0; d < OBS_STAGES; d++) stage(t0 + d, d);
  } else {
    issue(t0, onext);
  }
  // dense scenes: the voxel is warp-uniform, so its 20 stats words are fetched ONE ITERATION AHEAD by lanes 0..19
  // (one word each), parked in a per-warp shared-memory slot at the top of the iteration and read back as
  // broadcasts -- instead of ten L2-latency loads whose result is needed immediately
  __shared__ __align__(16) double s_stats[WPC][2][BALM_SWEEP_WORDS];
  double st_next = 0.0;
  if (DENSE && lane < BALM_SWEEP_WORDS && t0 < t1) st_next = __ldg(a.stats + (t0 - a.v0) * BALM_STATS_STRIDE + BALM_SWEEP_OFF + lane);
  for (long long t = t0; t < t1; t++) {
    long long v;
    double o[10];
    if (DENSE) {
      asm volatile("cp.async.wait_group %0;\n" ::"n"(OBS_STAGES - 1) : "memory");  // this iteration's group has landed
      if (active) {
#pragma unroll
        for (int c = 0; c < 10; c++) o[c] = s_obs[DENSE ? warp : 0][DENSE ? slot : 0][c][lane];
      }
      stage(t + OBS_STAGES, slot);  // refill the slot just read
      slot = (slot + 1) % OBS_STAGES;
    } else {
#pragma unroll
      for (int c = 0; c < 10; c++) o[c] = onext[c];
      issue(t + 1, onext);
    }
    double st[BALM_SWEEP_WORDS];
    if (DENSE) {
      v = t;
      double *slot = s_stats[warp][(int)(t & 1)];
      if (lane < BALM_SWEEP_WORDS) slot[lane] = st_next;
      __syncwarp();
      if (lane < BALM_SWEEP_WORDS && t + 1 < t1) st_next = __ldg(a.stats + (t + 1 - a.v0) * BALM_STATS_STRIDE + BALM_SWEEP_OFF + lane);
#pragma unroll
      for (int c = 0; c < BALM_SWEEP_WORDS / 2; c++) {
        const double2 x = reinterpret_cast<const double2 *>(slot)[c];
        st[2 * c] = x.x;
        st[2 * c + 1] = x.y;
      }
      if (!active) continue;
    } else {
      v = a.csc_vox[t];
      const double2 *st2 = reinterpret_cast<const double2 *>(a.stats + (v - a.v0) * BALM_STATS_STRIDE + BALM_SWEEP_OFF);
#pragma unroll
      for (int c = 0; c < BALM_SWEEP_WORDS / 2; c++) {
        const double2 x = __ldg(st2 + c);
        st[2 * c] = x.x;
        st[2 * c + 1] = x.y;
      }
    }
    // ---- G' rows of this observation (emitted as fp64 / digit planes / column maxima / per-observation rows), then its
    // gradient and diagonal-block terms (obs_terms) ----
    if constexpr (MODE == OBS_BLOCKS) {
      double2 *qd = reinterpret_cast<double2 *>(a.G + 18 * (size_t)(DENSE ? v * a.N + i : a.csc_obs[t]));
      obs_terms<true>(o, r, p, st, acc, [&](const double (&gv)[3][6]) {
#pragma unroll
        for (int rr = 0; rr < 3; rr++)
#pragma unroll
          for (int h = 0; h < 3; h++) qd[3 * rr + h] = make_double2(gv[rr][2 * h], gv[rr][2 * h + 1]);
      });
    } else {
    obs_terms<MODE != OBS_INT8>(o, r, p, st, acc, [&](const double (&gv)[3][6]) {
      if (MODE == OBS_FP64) {
        double *g0 = a.G + (size_t)(3 * (v - a.v0)) * a.ldg + 6 * i;
#pragma unroll
        for (int rr = 0; rr < 3; rr++) {
          double2 *qd = reinterpret_cast<double2 *>(g0 + (size_t)rr * a.ldg);
#pragma unroll
          for (int h = 0; h < 3; h++) qd[h] = make_double2(gv[rr][2 * h], gv[rr][2 * h + 1]);
        }
      }
      if (EMIT) {
        // |G' * sc| < 2^30, so X fits an int32 and ALL its balanced base-256 digits d_k in [-128,127] fall out of
        // two integer ops: the unsigned bytes of X + 0x80808080 are d_k + 128, and xor 0x80 turns them into int8.
#pragma unroll
        for (int rr = 0; rr < 3; rr++) {
          unsigned D[6];
#pragma unroll
          for (int q = 0; q < 6; q++)  // rint(G' sc) as the low word of G' sc + 1.5*2^52 (one DFMA, no conversion)
            D[q] = ((unsigned)__double2loint(fma(gv[rr][q], scl[q], 6755399441055744.0)) + 0x80808080u) ^ 0x80808080u;
          int8_t *base = a.Gq + (size_t)(3 * (v - a.v0) + rr) * a.ldg + 6 * i;
#pragma unroll
          for (int kb = 0; kb < 4; kb++) {        // byte kb = digit of weight 256^kb = plane S-1-kb
            if (kb < S) {
              unsigned short *o16 = reinterpret_cast<unsigned short *>(base + (size_t)(S - 1 - kb) * a.plane_stride);
#pragma unroll
              for (int h = 0; h < 3; h++)
                o16[h] = (unsigned short)__byte_perm(D[2 * h], D[2 * h + 1], kb | ((4 + kb) << 4));
            }
          }
        }
      }
      if (MODE != OBS_INT8) {
#pragma unroll
        for (int q = 0; q < 6; q++) {
          // column maximum on the integer pipe: compare the high words (the low word is accounted for by the +1 below)
          cmax[q] = max(max(cmax[q], (unsigned)__double2hiint(gv[0][q]) & 0x7fffffffu),
                        max((unsigned)__double2hiint(gv[1][q]) & 0x7fffffffu,
                            (unsigned)__double2hiint(gv[2][q]) & 0x7fffffffu));
          // exact diagonal of G'^T G': the split-integer SYRK drops the digit pair (S/2,S/2), which is a positive
          // bias on sums of squares only -- the n diagonal entries are therefore taken from this fp64 sum instead
          acc[27 + q] += gv[0][q] * gv[0][q] + gv[1][q] * gv[1][q] + gv[2][q] * gv[2][q];
        }
      }
    });
    }
  }
  if (MODE != OBS_INT8 && active && a.colmax) {
#pragma unroll
    for (int q = 0; q < 6; q++)  // upper bound of the maximum, tight to 2^-20: next high word, low word zero
      if (cmax[q]) atomicMax(a.colmax + 6 * i + q, (unsigned long long)(cmax[q] + 1u) << 32);
  }
  if (MODE != OBS_INT8 && active) {
    double *pp = a.part + (size_t)blockIdx.x * BALM_ACC * a.Np + i;
#pragma unroll
    for (int q = 0; q < BALM_ACC; q++) pp[(size_t)q * a.Np] = acc[q];
  }
}

__global__ void obs_reduce_kernel(const double *part, int chunks, int total, double *accum, double *accum_batch,
                                  int add, const int *skip = nullptr) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total || (skip && *skip)) return;
  double s = 0.0;
  for (int c = 0; c < chunks; c++) s += part[(size_t)c * total + e];
  accum[e] = add ? accum[e] + s : s;
  accum_batch[e] = s;  // this batch only (column concentration of the tensor path)
}

}  // namespace

int launch_voxel_stats(balm_ctx *c, const double *poses, int64_t v0, int64_t v1, double *stats_out, bool use_fix,
                       double *residual_out_dev, double *lam_out, double *w_out) {
  const bool store_stats = stats_out != nullptr;
  // residual_out_dev: accumulated (+=) when it is not the first batch -> caller zeroes it first
  const int64_t nv = v1 - v0;
  if (nv <= 0) return BALM_OK;
  const int64_t want = (nv + STATS_WARPS - 1) / STATS_WARPS;
  const int max_blocks = c->res_blocks / STATS_WARPS;
  int blocks = (int)(want < (int64_t)max_blocks ? want : max_blocks);
  StatsArgs a{c->obs, c->Kp, c->pose_idx, c->row_ptr, use_fix ? c->fix : nullptr, c->M, poses, c->N, v0, v1};
  const int psmem = 12 * c->N * (int)sizeof(double);
  const bool in_smem = psmem <= 64 * 1024;  // up to 682 poses; larger windows read the table through L1
  if (in_smem) voxel_sums_kernel<true><<<blocks, STATS_THREADS, psmem, c->stream>>>(a, c->vsums);
  else voxel_sums_kernel<false><<<blocks, STATS_THREADS, 0, c->stream>>>(a, c->vsums);
  const int64_t wantb = (nv + 127) / 128;
  const int eb = (int)(wantb < (int64_t)c->res_blocks ? wantb : c->res_blocks);
  // without a loss (and outside the readout) the NoLoss kernels, the only ones that run
  if (c->vloss_kind != BALM_LOSS_TRIVIAL || lam_out) {
    const VoxelLoss loss{c->vloss_kind, c->vloss_scale, lam_out, w_out};
    if (store_stats) voxel_eig_kernel<true><<<eb, 128, 0, c->stream>>>(c->vsums, c->coe, v0, v1, stats_out, c->res_part, loss);
    else voxel_eig_kernel<false><<<eb, 128, 0, c->stream>>>(c->vsums, c->coe, v0, v1, nullptr, c->res_part, loss);
  } else if (store_stats) {
    voxel_eig_kernel<true><<<eb, 128, 0, c->stream>>>(c->vsums, c->coe, v0, v1, stats_out, c->res_part, NoLoss{});
  } else {
    voxel_eig_kernel<false><<<eb, 128, 0, c->stream>>>(c->vsums, c->coe, v0, v1, nullptr, c->res_part, NoLoss{});
  }
  residual_reduce_kernel<<<1, 32, 0, c->stream>>>(c->res_part, eb, residual_out_dev, 1);
  c->launches += 3;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

static int obs_grid(balm_ctx *c, ObsArgs &a, int64_t nv, dim3 &grid) {
  const int tiles = (c->N + 31) / 32;
  int chunks;
  if (c->dense) {
    chunks = (int)(nv < (int64_t)c->obs_chunks ? nv : c->obs_chunks);
    a.chunk = (int)((nv + chunks - 1) / chunks);
    chunks = (int)((nv + a.chunk - 1) / a.chunk);
  } else {
    const int len = c->csc_max_len > 0 ? c->csc_max_len : 1;
    chunks = len < c->obs_chunks ? len : c->obs_chunks;
    a.chunk = (len + chunks - 1) / chunks;
    chunks = (len + a.chunk - 1) / a.chunk;
  }
  grid = dim3(chunks, (tiles + 3) / 4);
  return chunks;
}

static void obs_fill(balm_ctx *c, ObsArgs &a, const double *poses, int64_t v0, int64_t v1) {
  a = ObsArgs{};
  a.obs = c->obs; a.Kp = c->Kp; a.row_ptr = c->row_ptr; a.poses = poses; a.stats = c->stats;
  a.v0 = v0; a.v1 = v1; a.N = c->N; a.Np = c->Np; a.ldg = c->ldg; a.G = c->G; a.part = c->obs_part;
  a.csc_ptr = c->csc_ptr; a.csc_obs = c->csc_obs; a.csc_vox = c->csc_vox;
  a.csc_lo = c->csc_lo; a.csc_hi = c->csc_hi;
  a.colmax = c->colmax;
}

// fp64 SYRK path: one sweep writing fp64 G' (+ gradient / diagonal blocks); block-sparse path: the per-observation rows.
int launch_obs_pass(balm_ctx *c, const double *poses, int64_t v0, int64_t v1, bool first_batch) {
  const int64_t nv = v1 - v0;
  if (nv <= 0) return BALM_OK;
  ObsArgs a;
  obs_fill(c, a, poses, v0, v1);
  a.colmax = nullptr;
  dim3 grid;
  const int chunks = obs_grid(c, a, nv, grid);
  if (c->prec == BALM_PREC_BLOCKS) {  // per-observation rows: nothing of the dense G' to clear
    if (c->dense) obs_pass_kernel<true, OBS_BLOCKS><<<grid, 128, 0, c->stream>>>(a);
    else obs_pass_kernel<false, OBS_BLOCKS><<<grid, 128, 0, c->stream>>>(a);
  } else {
    if (!c->dense)  // sparse: G' rows of non-observing poses must be zero
      CUDA_TRY(cudaMemsetAsync(c->G, 0, sizeof(double) * (size_t)3 * nv * c->ldg, c->stream));
    if (c->dense) obs_pass_kernel<true, OBS_FP64><<<grid, 128, 0, c->stream>>>(a);
    else obs_pass_kernel<false, OBS_FP64><<<grid, 128, 0, c->stream>>>(a);
  }
  const int total = BALM_ACC * c->Np;
  obs_reduce_kernel<<<(total + 255) / 256, 256, 0, c->stream>>>(c->obs_part, chunks, total, c->accum,
                                                                c->accum_batch, first_batch ? 0 : 1);
  c->launches += 2;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

// tensor path, sweep 1: column maxima of G' + gradient / diagonal-block accumulators.
int launch_obs_colmax(balm_ctx *c, const double *poses, int64_t v0, int64_t v1, bool first_batch) {
  const int64_t nv = v1 - v0;
  if (nv <= 0) return BALM_OK;
  ObsArgs a;
  obs_fill(c, a, poses, v0, v1);
  dim3 grid;
  const int chunks = obs_grid(c, a, nv, grid);
  if (c->dense) obs_pass_kernel<true, OBS_MAXONLY><<<grid, 128, 0, c->stream>>>(a);
  else obs_pass_kernel<false, OBS_MAXONLY><<<grid, 128, 0, c->stream>>>(a);
  const int total = BALM_ACC * c->Np;
  obs_reduce_kernel<<<(total + 255) / 256, 256, 0, c->stream>>>(c->obs_part, chunks, total, c->accum,
                                                                c->accum_batch, first_batch ? 0 : 1);
  c->launches += 2;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

// tensor path, sweep 2: int8 digit planes written directly. `fused`: the single speculative sweep (column maxima,
// accumulators AND digit planes with the previous evaluation's scales); `skip`: device flag that disarms sweep 2, or
// the fused sweep and its reduction (what they would write is already in place).
int launch_obs_int8(balm_ctx *c, const double *poses, int64_t v0, int64_t v1, bool first_batch, const double *sc,
                    int8_t *Gq, int64_t plane_stride, const int *S_dev, int S_alloc, int64_t rows_padded, bool fused,
                    const int *skip) {
  const int64_t nv = v1 - v0;
  if (nv <= 0) return BALM_OK;
  ObsArgs a;
  obs_fill(c, a, poses, v0, v1);
  a.sc = sc; a.Gq = Gq; a.plane_stride = plane_stride; a.S_dev = S_dev; a.skip = skip;
  const int S = S_alloc;  // memsets cover every allocated plane
  dim3 grid;
  const int chunks = obs_grid(c, a, nv, grid);
  if (!(skip && !fused)) {  // the re-armed sweep 2 finds the padding already zeroed by the fused sweep
    if (!c->dense) {
      for (int s = 0; s < S; s++)
        CUDA_TRY(cudaMemsetAsync(Gq + (size_t)s * plane_stride, 0, (size_t)rows_padded * c->ldg, c->stream));
    } else if (rows_padded > 3 * nv) {  // zero the K-padding rows of every plane
      for (int s = 0; s < S; s++)
        CUDA_TRY(cudaMemsetAsync(Gq + (size_t)s * plane_stride + (size_t)3 * nv * c->ldg, 0,
                                 (size_t)(rows_padded - 3 * nv) * c->ldg, c->stream));
    }
  }
  if (fused) {
    if (c->dense) obs_pass_kernel<true, OBS_FUSED><<<grid, 128, 0, c->stream>>>(a);
    else obs_pass_kernel<false, OBS_FUSED><<<grid, 128, 0, c->stream>>>(a);
    const int total = BALM_ACC * c->Np;
    obs_reduce_kernel<<<(total + 255) / 256, 256, 0, c->stream>>>(c->obs_part, chunks, total, c->accum,
                                                                  c->accum_batch, first_batch ? 0 : 1, skip);
    c->launches += 2;
  } else {
    if (c->dense) obs_pass_kernel<true, OBS_INT8><<<grid, 128, 0, c->stream>>>(a);
    else obs_pass_kernel<false, OBS_INT8><<<grid, 128, 0, c->stream>>>(a);
    c->launches += 1;
  }
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

// Kernel attributes are per device: set once per context (a process may drive several GPUs).
int factor_kernels_setup() {
  CUDA_TRY(cudaFuncSetAttribute(voxel_sums_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
  return BALM_OK;
}

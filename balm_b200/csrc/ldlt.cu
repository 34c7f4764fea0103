// ldlt.cu -- dense damped solve (kernel K6) and the scalar side of the LM step (K7).
//
//   D = diag(H);  A = H + u*D;  A = L diag(d) L^T  (blocked right-looking, fp64, no pivoting);
//   dx = A^-1 (-g);  q1 = 0.5 * dx . (u*D*dx - g)
// replaces `D.diagonal() = Hess.diagonal(); dxi = (Hess + u*D).ldlt().solve(-JacT)` and the q1 line of
// BALM2::damping_iter (bavoxel.hpp:1113-1114,1127).  Eigen's LDLT pivots on the diagonal; for the damped
// normal matrix the factorisation exists without pivoting whenever the leading minors are non-singular
// (always when H + uD is positive definite, the accepted-step regime).  A zero / non-finite pivot raises the
// not_pd flag and the LM loop treats the step as rejected (u *= v), which is what happens to a bad step in
// the reference as well (the trial residual does not decrease).  The solution of a non-singular system does
// not depend on the pivot order beyond rounding.
//
// A is column-major n x n; only the lower triangle is read/written. Panel width NB = 64.
#include <stdlib.h>
#include "internal.cuh"

namespace {

constexpr int NB = BALM_NB;

__global__ void damp_copy_kernel(const double *H, double *A, double *dvec, int n, const double *u_dev) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // row (contiguous)
  const int j = blockIdx.y;
  if (i >= n) return;
  const double u = *u_dev;
  double h = H[(size_t)j * n + i];
  if (i == j) {
    dvec[i] = h;
    h += u * h;
  }
  A[(size_t)j * n + i] = h;
}

// The 64x64 diagonal block is factored in four 16-column sub-panels. The serial chain of the whole solve is n = 6N column
// steps, so the 16 x 16 diagonal block of a sub-panel is factored by ONE warp with its rows in registers and the columns
// exchanged by shuffles (no shared-memory round trip, no barrier per column), which also yields its inverse; the rows
// below follow as a 16-wide GEMM with that inverse, the rank-16 trailing update and the assembly of X = L11^-1 from the
// 16x16 inverses use all 256 threads. (Round 1 factored the whole 64-row sub-panel column by column on two warps with a
// named barrier per column: 21 us per 64 x 64 block against 12 us now.)
// In: S = the block (lower triangle), Xs = 0, all threads synchronised. Out: S = L (below the diagonal) and d (on
// it), Xs = L11^-1 (lower), all threads synchronised. Returns true if a pivot was zero / non-finite.
__device__ __forceinline__ unsigned long long gtime_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;\n" : "=l"(t));
  return t;
}
// 1/d to full double precision off the slow division path: hardware seed (rcp.approx.ftz.f64, ~2^-23) + two Newton steps.
// The reciprocal of the pivot is on the serial chain of every column, the IEEE division costs three times as much.
__device__ __forceinline__ double fast_rcp(double d) {
  double x;
  asm("rcp.approx.ftz.f64 %0, %1;\n" : "=d"(x) : "d"(d));
  double e = fma(-d, x, 1.0);
  x = fma(x, e, x);
  e = fma(-d, x, 1.0);
  return fma(x, e, x);
}
__device__ __forceinline__ bool diag_factor(double (*S)[NB + 1], double (*Xs)[NB + 1], double (*Wp)[17],
                                            double (*col16)[16], unsigned long long *stamp = nullptr) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  bool bad = false;
  double *dinv16 = &col16[0][0];  // [16] reciprocals of the current sub-panel's pivots
#pragma unroll 1
  for (int cb = 0; cb < NB; cb += 16) {
    // ---- (1) the 16 x 16 diagonal block: ONE warp, rows in registers, columns exchanged by shuffles (no barrier on the
    //      serial chain: per column one broadcast of the pivot, one shuffle per remaining column, one FMA each), then its
    //      inverse X11 = L11^-1 by forward substitution on the identity, again shuffles only ----
    if (warp == 0) {
      const int i = lane & 15;  // lanes 16..31 mirror lanes 0..15
      double a[16];
#pragma unroll
      for (int q = 0; q < 16; q++) a[q] = S[cb + i][cb + q];  // (entries above the diagonal are zero on entry and never used)
#pragma unroll
      for (int j = 0; j < 16; j++) {
        const double d = __shfl_sync(0xffffffffu, a[j], j, 16);
        if (!(fabs(d) > 1e-290 && fabs(d) < 1e300)) bad = true;
        const double dinv = fast_rcp(d);
        const double aj = a[j];
#pragma unroll
        for (int q = j + 1; q < 16; q++) {
          const double cq = __shfl_sync(0xffffffffu, aj, q, 16);  // A[q][j] before scaling
          a[q] = fma(-(aj * cq), dinv, a[q]);  // the product does not wait for the reciprocal; unmasked: what lands
        }                                      // above the diagonal is never read
        a[j] = (i > j) ? aj * dinv : aj;
        if (i == j) dinv16[j] = dinv;
      }
      double xr[16];
#pragma unroll
      for (int q = 0; q < 16; q++) xr[q] = (q == i) ? 1.0 : 0.0;
#pragma unroll
      for (int j = 0; j < 15; j++) {
        const double l = (i > j) ? a[j] : 0.0;
#pragma unroll
        for (int q = 0; q <= j; q++) {  // row j of the inverse is final and has entries q <= j only
          const double xj = __shfl_sync(0xffffffffu, xr[q], j, 16);
          xr[q] -= l * xj;
        }
      }
      __syncwarp();  // the mirror lanes 16..31 have read their copy of the block before it is overwritten
      if (lane < 16) {
#pragma unroll
        for (int q = 0; q < 16; q++) {
          if (q <= i) S[cb + i][cb + q] = a[q];  // L (q < i) and d (q == i)
          Xs[cb + i][cb + q] = xr[q];
        }
      }
    }
    __syncthreads();
    // ---- (2) the rows below: W = A21 X11^T (a 16-wide GEMM instead of a sequential triangular solve), L21 = W d^-1 ----
    {
      const int nrow = NB - cb - 16;
      double wv[3];
#pragma unroll
      for (int t = 0; t < 3; t++) {
        const int e = tid + t * 256;
        wv[t] = 0.0;
        if (e < nrow * 16) {
          const int r = cb + 16 + (e >> 4), q = e & 15;
          double sacc = 0.0;
#pragma unroll
          for (int m = 0; m < 16; m++) sacc += (m <= q) ? S[r][cb + m] * Xs[cb + q][cb + m] : 0.0;
          wv[t] = sacc;
        }
      }
      __syncthreads();  // every thread has read the unscaled panel entries it needs
#pragma unroll
      for (int t = 0; t < 3; t++) {
        const int e = tid + t * 256;
        if (e < nrow * 16) {
          const int r = cb + 16 + (e >> 4), q = e & 15;
          Wp[r][q] = wv[t];
          S[r][cb + q] = wv[t] * dinv16[q];
        }
      }
    }
    __syncthreads();
    {  // ---- (3) trailing block in 16x16 sub-blocks: thread (ri, ci) owns one element of each lower sub-block ----
      const int ri = tid >> 4, ci = tid & 15;
      for (int rb2 = cb + 16; rb2 < NB; rb2 += 16)
        for (int cb2 = cb + 16; cb2 <= rb2; cb2 += 16) {
          const int r = rb2 + ri, c = cb2 + ci;
          if (r >= c) {
            double sacc = 0.0;
#pragma unroll
            for (int q = 0; q < 16; q++) sacc += Wp[r][q] * S[c][cb + q];
            S[r][c] -= sacc;
          }
        }
    }
    __syncthreads();
    if (stamp && tid == 0) stamp[1 + (cb >> 4)] = gtime_ns();
  }
  bad = __syncthreads_or(bad ? 1 : 0) != 0;

  // ---- off-diagonal blocks by block rows: X_bc = -X_bb * sum_{m=c}^{b-1} L_bm X_mc ----
#pragma unroll 1
  for (int b = 1; b < 4; b++) {
    const int rb = 16 * b, ri = tid >> 4, ci = tid & 15;
    for (int cq = 0; cq < b; cq++) {  // T_bc = sum_{m in blocks c..b-1} L_bm X_mc, parked in the X_bc positions
      const int c = 16 * cq + ci;
      double sacc = 0.0;
      for (int m = 16 * cq; m < rb; m++) sacc += S[rb + ri][m] * Xs[m][c];
      Xs[rb + ri][c] = sacc;
    }
    __syncthreads();
    double xn[3];
#pragma unroll
    for (int cq = 0; cq < 3; cq++) {
      xn[cq] = 0.0;
      if (cq < b) {
        const int c = 16 * cq + ci;
        double sacc = 0.0;
#pragma unroll
        for (int k = 0; k < 16; k++) sacc += Xs[rb + ri][rb + k] * Xs[rb + k][c];  // X_bb (lower) times T
        xn[cq] = -sacc;
      }
    }
    __syncthreads();  // every thread has read the T values it needs
#pragma unroll
    for (int cq = 0; cq < 3; cq++)
      if (cq < b) Xs[rb + ri][16 * cq + ci] = xn[cq];
    __syncthreads();
  }
  return bad;
}


// =====================================================================================================================
// Persistent tile-DAG factorisation.  ONE cooperative launch factors the whole matrix; 64 x 64 tiles, the
// dependencies between tile tasks are counters in global memory instead of kernel boundaries:
//   chain CTA (block 0)  for k = 0 .. nt-1: D'(k) = [mini-panel L_{k,k-1} = A_{k,k-1} X_{k-1}^T d^-1, mini-update
//                        A_kk -= L W^T, both in shared memory] + the 64 x 64 factorisation (diag_factor) + y_k.
//                        The serial chain of the solve is these nt steps and nothing else.
//   worker CTAs          P(r,k): L_rk = A_rk X_k^T d_k^-1, rhs_r -= L_rk y_k        (r >= k+2; row k+1 is the chain's)
//                        U(r,c,k): A_rc -= L_rk d_k L_ck^T (fp64 tensor-core MMAs)  (r >= c > k, except (k+1,k+1))
// Tasks are enumerated step-major, row by row (the rows next to the diagonal -- what the chain needs next -- first) and
// dealt round-robin inside two groups: a few "near" CTAs take the rows within NEAR_ROWS of the diagonal, so that what
// feeds the chain never queues behind far-away trailing updates; all other CTAs take the rest. Every CTA walks its tasks
// in the global order and waits only for tasks that come earlier in that order, and all CTAs are co-resident
// (cooperative launch), so the scheme cannot deadlock. Updates of one tile are applied in step order (counter upd[r][c]),
// hence the result is bit-reproducible. W = L d is never stored: U scales its A-operand fragments by d on the fly.
// Memory model: producers  stores -> __syncthreads -> thread 0: st.release.gpu(counter);
//               consumers  thread 0: ld.acquire.gpu spin -> __syncthreads -> data through L2 (cp.async.cg / ld.global.cg).
namespace dag {

constexpr int T = 64;
constexpr int LDT = T + 4;   // smem row pitch (doubles): conflict-free DMMA fragment loads, 16-byte aligned rows
constexpr int NEAR_ROWS = 4; // rows k+2 .. k+1+NEAR_ROWS of step k go to the near group

struct Args {
  double *A;            // n x n column-major, lower triangle: in H + uD, out L (below the diagonal) and d (on it)
  int n, nt;
  double *Xinv;         // [nt][64*64] column-major inverses of the unit-lower diagonal blocks
  double *dinv, *dval;  // [n] 1/d, d
  double *sol;          // [n] running right-hand side (in: b)
  double *ysol;         // [n] y = L^-1 b
  int *flags;           // [0] bad pivot
  int *upd;             // [nt*nt] number of updates applied to tile (r,c)
  int *pdone;           // [nt*nt] L_rk final
  int *xdone;           // [nt]    X_k, d_k, y_k published
  int *rhs_cnt;         // [nt]    number of rhs updates applied to row block r
  int near_ctas;        // CTAs 1 .. near_ctas form the near group
  unsigned long long *trace;  // optional (BALM_DAG_TRACE): chain [nt][4] step timestamps, then per CTA [wait ns, busy ns, tasks]
};

__device__ __forceinline__ int ld_acquire(const int *p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release(int *p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;\n" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;\n" : "=l"(t));
  return t;
}
__device__ __forceinline__ void wait_ge(const int *p, int want) {  // called by ONE thread, followed by __syncthreads
  while (ld_acquire(p) < want) __nanosleep(20);
}
__device__ __forceinline__ double ld_cg(const double *p) { return __ldcg(p); }

// dst[kk][rr] = A[(col0+kk)*n + row0+rr], zero outside the matrix (16-byte cp.async.cg pieces: through L2)
__device__ __forceinline__ void tile_load(double *dst, const double *A, int n, int col0, int row0) {
#pragma unroll
  for (int it = 0; it < 8; it++) {
    const int e = threadIdx.x + it * 256, kk = e >> 5, rr = (e & 31) * 2;
    double *d = dst + kk * LDT + rr;
    if (col0 + kk < n && row0 + rr < n) cp_async16(d, A + (size_t)(col0 + kk) * n + row0 + rr);
    else *reinterpret_cast<double2 *>(d) = make_double2(0.0, 0.0);
  }
}
// dst[kk][c] = Xcm[kk*64 + c] = X[c][kk]   (B operand of W = A_rk X^T)
__device__ __forceinline__ void x_load(double *dst, const double *Xcm) {
#pragma unroll
  for (int it = 0; it < 8; it++) {
    const int e = threadIdx.x + it * 256, kk = e >> 5, rr = (e & 31) * 2;
    cp_async16(dst + kk * LDT + rr, Xcm + kk * T + rr);
  }
}
__device__ __forceinline__ void cp_wait_all() {
  asm volatile("cp.async.commit_group;\n" ::);
  asm volatile("cp.async.wait_group 0;\n" ::);
}

// acc (+)= sum_kk sA[kk][row] * scale[kk] * sB[kk][col]; 8 warps, warp tile 32 x 16, C fragment element (i,j,h):
// row = wm*32 + i*8 + fr, col = wn*16 + j*8 + 2*fk + h
__device__ __forceinline__ void tile_mma(double (&acc)[4][2][2], const double *sA, const double *sB, const double *scale) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int wm = warp >> 2, wn = warp & 3, fr = lane >> 2, fk = lane & 3;
#pragma unroll
  for (int kk = 0; kk < T; kk += 4) {
    const double sc = scale ? scale[kk + fk] : 1.0;
    double af[4], bf[2];
#pragma unroll
    for (int i = 0; i < 4; i++) af[i] = sA[(kk + fk) * LDT + wm * 32 + i * 8 + fr] * sc;
#pragma unroll
    for (int j = 0; j < 2; j++) bf[j] = sB[(kk + fk) * LDT + wn * 16 + j * 8 + fr];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int j = 0; j < 2; j++) dmma_8x8x4(acc[i][j][0], acc[i][j][1], af[i], bf[j]);
  }
}
__device__ __forceinline__ void acc_zero(double (&acc)[4][2][2]) {
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 2; j++) acc[i][j][0] = acc[i][j][1] = 0.0;
}

struct Prof { unsigned long long wait, load, mma, store, panel; };

// ---- worker task U(r,c,k): A_rc -= L_rk d_k L_ck^T ----
__device__ __forceinline__ void task_update(const Args &a, int r, int c, int k, double *t0, double *t1, double *vec,
                                            Prof &pf) {
  const int tid = threadIdx.x, nt = a.nt, n = a.n;
  unsigned long long q0 = a.trace ? gtime() : 0ull;
  // three counters, three threads of three different warps: the round trips overlap
  if (tid == 0) wait_ge(a.pdone + r * nt + k, 1);
  if (tid == 32) wait_ge(a.pdone + c * nt + k, 1);
  if (tid == 64) wait_ge(a.upd + r * nt + c, k);
  __syncthreads();
  if (a.trace) { const unsigned long long q = gtime(); pf.wait += q - q0; q0 = q; }
  tile_load(t0, a.A, n, k * T, r * T);
  if (r != c) tile_load(t1, a.A, n, k * T, c * T);
  if (tid < T) vec[tid] = (k * T + tid < n) ? ld_cg(a.dval + k * T + tid) : 0.0;
  asm volatile("cp.async.commit_group;\n" ::);
  // the C tile (read-modify-write) is requested while the operands are in flight
  const int lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3, fr = lane >> 2, fk = lane & 3;
  double cv[4][2][2];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 2; j++)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int row = r * T + wm * 32 + i * 8 + fr, col = c * T + wn * 16 + j * 8 + 2 * fk + h;
        cv[i][j][h] = (row < n && col < n && row >= col) ? ld_cg(a.A + (size_t)col * n + row) : 0.0;
      }
  asm volatile("cp.async.wait_group 0;\n" ::);
  __syncthreads();
  if (a.trace) { const unsigned long long q = gtime(); pf.load += q - q0; q0 = q; }
  double acc[4][2][2];
  acc_zero(acc);
  tile_mma(acc, t0, r != c ? t1 : t0, vec);
  if (a.trace) { const unsigned long long q = gtime(); pf.mma += q - q0; q0 = q; }
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 2; j++)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int row = r * T + wm * 32 + i * 8 + fr, col = c * T + wn * 16 + j * 8 + 2 * fk + h;
        if (row < n && col < n && row >= col) a.A[(size_t)col * n + row] = cv[i][j][h] - acc[i][j][h];
      }
  __syncthreads();
  if (tid == 0) { __threadfence(); st_release(a.upd + r * nt + c, k + 1); }
  if (a.trace) { const unsigned long long q = gtime(); pf.store += q - q0; }
}

// W = A_rk X_k^T into registers, then staged as  sL[c][row] = W d^-1 (= L_rk, k-major: the A-operand layout) and,
// if sW != null, sW[c][row] = W (the B-operand layout of L W^T). t0/t1: operand tiles (overwritten).
__device__ __forceinline__ void panel_tile(const Args &a, int r, int k, double *t0, double *t1, double *sL, double *sW,
                                           double *vdinv) {
  const int tid = threadIdx.x;
  tile_load(t0, a.A, a.n, k * T, r * T);
  x_load(t1, a.Xinv + (size_t)k * T * T);
  if (tid < T) vdinv[tid] = ld_cg(a.dinv + k * T + tid);  // column blocks k < nt-1 are full
  cp_wait_all();
  __syncthreads();
  double acc[4][2][2];
  acc_zero(acc);
  tile_mma(acc, t0, t1, nullptr);
  __syncthreads();  // every warp has read t0 / t1 (sL / sW may alias them)
  const int lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3, fr = lane >> 2, fk = lane & 3;
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 2; j++)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int row = wm * 32 + i * 8 + fr, col = wn * 16 + j * 8 + 2 * fk + h;
        sL[col * LDT + row] = acc[i][j][h] * vdinv[col];
        if (sW) sW[col * LDT + row] = acc[i][j][h];
      }
  __syncthreads();
}

// ---- worker task P(r,k) ----
__device__ __forceinline__ void task_panel(const Args &a, int r, int k, double *t0, double *t1, double *vec) {
  const int tid = threadIdx.x, nt = a.nt, n = a.n;
  if (tid == 0) wait_ge(a.xdone + k, 1);
  if (tid == 32) wait_ge(a.upd + r * nt + k, k);
  if (tid == 64) wait_ge(a.rhs_cnt + r, k);
  __syncthreads();
  double *vdinv = vec, *vy = vec + T;
  if (tid >= T && tid < 2 * T) vy[tid - T] = ld_cg(a.ysol + k * T + tid - T);
  panel_tile(a, r, k, t0, t1, /*sL=*/t0, nullptr, vdinv);
  // L_rk back to the matrix (coalesced along rows) and the forward-substitution update of this row block
#pragma unroll 4
  for (int e = tid; e < T * T; e += 256) {
    const int col = e >> 6, row = e & 63;
    if (r * T + row < n) a.A[(size_t)(k * T + col) * n + r * T + row] = t0[col * LDT + row];
  }
  if (tid < T && r * T + tid < n) {
    double s = 0.0;
#pragma unroll 8
    for (int cc = 0; cc < T; cc++) s += t0[cc * LDT + tid] * vy[cc];
    a.sol[r * T + tid] = ld_cg(a.sol + r * T + tid) - s;
  }
  __syncthreads();
  if (tid == 0) { __threadfence(); st_release(a.pdone + r * nt + k, 1); st_release(a.rhs_cnt + r, k + 1); }
}

// ---- the chain CTA ----
__device__ __forceinline__ void chain(const Args &a, double *smem) {
  double (*S)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(smem);
  double (*Xs)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(smem + NB * (NB + 1));
  double (*Wp)[17] = reinterpret_cast<double (*)[17]>(smem + 2 * NB * (NB + 1));
  double (*col16)[16] = reinterpret_cast<double (*)[16]>(smem + 2 * NB * (NB + 1) + NB * 17);
  double *bvec = smem + 2 * NB * (NB + 1) + NB * 17 + 32;
  double *vec = bvec + NB;                                   // [2*T] dinv_k | y_k
  double *t0 = smem + 2 * NB * (NB + 1) + NB * 17 + 32 + NB + 2 * T;  // 16-byte aligned (all terms even)
  double *t1 = t0 + T * LDT;
  double *t2 = t1 + T * LDT;
  double *t3 = t2 + T * LDT;
  const int tid = threadIdx.x, n = a.n, nt = a.nt;
  const int lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3, fr = lane >> 2, fk = lane & 3;
  for (int k = 0; k < nt; k++) {
    const int j0 = k * T;
    const int nbw = (n - j0 < T) ? n - j0 : T;
    double accu[4][2][2];
    acc_zero(accu);
    double bloc = 0.0;  // threads < 64: this block's right-hand side entry
    if (a.trace && tid == 0) a.trace[4 * k + 0] = gtime();
    if (k > 0) {
      // mini-panel of step k-1 for row block k: L_{k,k-1}, W_{k,k-1}; mini-update of A_kk and of b_k
      if (tid == 0) wait_ge(a.upd + k * nt + (k - 1), k - 1);
      if (tid == 32) wait_ge(a.rhs_cnt + k, k - 1);
      if (tid == 64) wait_ge(a.upd + k * nt + k, k - 1);  // the diagonal block has every update but the chain's own
      if (a.trace && tid == 0) a.trace[4 * k + 1] = gtime();
      __syncthreads();
    }
    // the diagonal block is requested now (lower triangle; rows/cols of a short last block act as identity): its L2
    // round trip overlaps the mini-panel
    double sld[16];
#pragma unroll
    for (int it = 0; it < 16; it++) {
      const int e = tid + it * 256, r = e & (NB - 1), c = e >> 6;
      double v = (r == c) ? 1.0 : 0.0;
      if (r < nbw && c < nbw && r >= c) v = ld_cg(a.A + (size_t)(j0 + c) * n + j0 + r);
      sld[it] = v;
    }
    if (k > 0) {
      if (tid >= T && tid < 2 * T) vec[tid] = ld_cg(a.ysol + (k - 1) * T + tid - T);
      panel_tile(a, k, k - 1, t0, t1, /*sL=*/t2, /*sW=*/t3, vec);
#pragma unroll 4
      for (int e = tid; e < T * T; e += 256) {
        const int col = e >> 6, row = e & 63;
        if (row < nbw) a.A[(size_t)((k - 1) * T + col) * n + j0 + row] = t2[col * LDT + row];
      }
      if (tid < T) {
        double s = 0.0;
#pragma unroll 8
        for (int cc = 0; cc < T; cc++) s += t2[cc * LDT + tid] * vec[T + cc];
        bloc = (tid < nbw) ? ld_cg(a.sol + j0 + tid) - s : 0.0;
      }
      tile_mma(accu, t2, t3, nullptr);  // L W^T
      __syncthreads();
      if (tid == 0) { __threadfence(); st_release(a.pdone + k * nt + (k - 1), 1); }
      if (a.trace && tid == 0) a.trace[4 * k + 2] = gtime();
    } else if (tid < T) {
      bloc = (tid < nbw) ? a.sol[j0 + tid] : 0.0;
    }
    // the diagonal block into shared memory, minus the mini-update
#pragma unroll
    for (int it = 0; it < 16; it++) {
      const int e = tid + it * 256, r = e & (NB - 1), c = e >> 6;
      S[r][c] = sld[it];
      Xs[r][c] = 0.0;
    }
    if (tid < NB) bvec[tid] = bloc;
    __syncthreads();
    if (k > 0) {
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 2; j++)
#pragma unroll
          for (int h = 0; h < 2; h++) {
            const int r = wm * 32 + i * 8 + fr, c = wn * 16 + j * 8 + 2 * fk + h;
            if (r < nbw && c < nbw && r >= c) S[r][c] -= accu[i][j][h];
          }
      __syncthreads();
    }
    unsigned long long *stamp = (a.trace && k == 20) ? a.trace + 4 * nt : nullptr;  // fine timeline of one step
    if (stamp && tid == 0) stamp[0] = gtime();
    const bool bad = diag_factor(S, Xs, Wp, col16, stamp);
    if (stamp && tid == 0) stamp[5] = gtime();
    if (bad && tid == 0) atomicOr(&a.flags[0], 1);
    double *Xcm = a.Xinv + (size_t)k * NB * NB;
#pragma unroll 4
    for (int e = tid; e < NB * NB; e += 256) {
      const int r = e & (NB - 1), c = e >> 6;
      if (r < nbw && c < nbw && r >= c) a.A[(size_t)(j0 + c) * n + j0 + r] = S[r][c];
      Xcm[c * NB + r] = (r >= c) ? Xs[r][c] : 0.0;
    }
    if (tid < nbw) { a.dinv[j0 + tid] = 1.0 / S[tid][tid]; a.dval[j0 + tid] = S[tid][tid]; }
    if (tid < NB) {
      double sacc = 0.0;
      for (int c = 0; c <= tid; c++) sacc += Xs[tid][c] * bvec[c];
      if (tid < nbw) a.ysol[j0 + tid] = sacc;
    }
    __syncthreads();
    if (stamp && tid == 0) stamp[6] = gtime();
    if (tid == 0) { __threadfence(); st_release(a.xdone + k, 1); }
    if (a.trace && tid == 0) a.trace[4 * k + 3] = gtime();
  }
}

constexpr int SMEM_DOUBLES = 2 * NB * (NB + 1) + NB * 17 + 32 + NB + 2 * T + 4 * T * LDT;

__global__ void __launch_bounds__(256, 1) ldl_dag_kernel(Args a) {
  extern __shared__ __align__(16) double dyn_smem[];
  if (blockIdx.x == 0) { chain(a, dyn_smem); return; }
  const int nt = a.nt, W = gridDim.x;
  if (nt < 2) return;
  // group of this CTA, its index and size inside the group
  const bool near = (int)blockIdx.x <= a.near_ctas;
  const int gsize = near ? a.near_ctas : W - 1 - a.near_ctas;
  const int gidx = near ? blockIdx.x - 1 : blockIdx.x - 1 - a.near_ctas;
  if (gsize <= 0) return;
  double *t0 = dyn_smem, *t1 = dyn_smem + T * LDT, *vec = dyn_smem + 2 * T * LDT;
  unsigned long long t_begin = a.trace ? gtime() : 0ull, n_tasks = 0;
  Prof pf{0, 0, 0, 0, 0};
  const bool split = a.near_ctas > 0 && W - 1 - a.near_ctas > 0;  // two groups; otherwise one group takes every row
  // `next`: position (in the group's running task count) of this CTA's next task, relative to the current list.
  // Every list below is walked with a stride of gsize from there, so a CTA touches only its own tasks (the lists of a
  // 47-step factorisation hold 18 000 tasks; enumerating all of them in every CTA cost more than executing its share).
  int next = gidx;
  for (int k = 0; k + 1 < nt; k++) {
    // Worker tasks of step k: rows r = k+2 .. nt-1 (row k+1 is the chain's): P(r,k), then U(r,c,k) for c = k+1 .. r.
    const int r_split = split ? (k + 2 + NEAR_ROWS < nt ? k + 2 + NEAR_ROWS : nt) : nt;  // rows below r_split: near group
    if (near || !split) {
      // near group: row by row (what the chain needs next first); P and the U tasks of a row are consecutive
      int base = 0;  // tasks of this list before row r
      for (int r = k + 2; r < r_split; r++) {
        const int ntask = 1 + (r - k);
        for (; next < base + ntask; next += gsize) {
          const int t = next - base;
          if (t == 0) task_panel(a, r, k, t0, t1, vec);
          else task_update(a, r, k + t, k, t0, t1, vec, pf);
          n_tasks++;
        }
        base += ntask;
      }
      next -= base;
    }
    if (!near && split) {
      // far group: ALL panel tasks of the step first, then the updates -- an update dealt in the same round as the
      // panel task it depends on would idle its CTA for the length of that task
      const int np = nt - r_split;
      for (; next < np; next += gsize) {
        const unsigned long long q0 = a.trace ? gtime() : 0ull;
        task_panel(a, r_split + next, k, t0, t1, vec);
        if (a.trace) pf.panel += gtime() - q0;
        n_tasks++;
      }
      next -= np;
      int base = 0;
      for (int r = r_split; r < nt; r++) {
        const int ntask = r - k;  // c = k+1 .. r
        for (; next < base + ntask; next += gsize) {
          task_update(a, r, k + 1 + (next - base), k, t0, t1, vec, pf);
          n_tasks++;
        }
        base += ntask;
      }
      next -= base;
    }
  }
  if (a.trace && threadIdx.x == 0) {
    unsigned long long *o = a.trace + 4 * nt + 8 * blockIdx.x;
    o[0] = t_begin; o[1] = gtime(); o[2] = n_tasks;
    o[3] = pf.wait; o[4] = pf.load; o[5] = pf.mma; o[6] = pf.store; o[7] = pf.panel;
  }
}

}  // namespace dag


// ---- backward error of the computed step, and iterative refinement -----------------------------------------------
// The factorisation does not pivot (Eigen's LDLT, bavoxel.hpp:1114, pivots on the diagonal). For the positive-definite
// systems of the accepted-step regime that is backward stable; for an INDEFINITE H + uD (strongly perturbed start, tiny
// u) element growth can cost digits. So every solve is followed by the componentwise backward error
//     omega = max_i |b - A x|_i / (|A| |x| + |b|)_i ,   A = H + u diag(H), b = -g      (Oettli-Prager)
// computed in fp64 from H itself (one warp per row). omega > tol raises flags[4]; the host then runs fp64 iterative
// refinement with the same factors (refine_solution) -- at most three rounds -- and, if omega still does not fall below
// the tolerance, reports the step as not_pd (rejected, u *= v), never a silently inaccurate dx.
__global__ void __launch_bounds__(256) solve_residual_kernel(const double *H, const double *g, const double *x, int n,
                                                             const double *u_dev, double tol, double *rres, int *flags,
                                                             double *omega_out) {
  const int lane = threadIdx.x & 31, row = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= n) return;
  const double u = *u_dev;
  double s = 0.0, sa = 0.0;
  for (int j = lane; j < n; j += 32) {  // H symmetric: row `row` = column `row`, contiguous
    double h = H[(size_t)row * n + j];
    if (j == row) h += u * h;
    const double t = h * x[j];
    s += t;
    sa += fabs(t);
  }
  s = warp_sum(s);
  sa = warp_sum(sa);
  if (lane == 0) {
    const double b = -g[row], r = b - s, den = sa + fabs(b);
    rres[row] = r;
    const double om = den > 0.0 ? fabs(r) / den : 0.0;
    if (!(om <= tol)) atomicOr(&flags[4], 1);
    atomicMax(reinterpret_cast<unsigned long long *>(omega_out), (unsigned long long)__double_as_longlong(om));
  }
}

// Forward substitution for a fresh right-hand side (refinement only; the first solve fuses it into the factorisation):
// one 64-row block per launch: y_j = X_j b_j, rows below -= L21 y_j.
__global__ void __launch_bounds__(256) ldl_fwd_block_kernel(const double *A, int n, int j0, int nbw, const double *Xcm,
                                                            double *sol, double *ysol) {
  __shared__ double b[NB], y[NB];
  const int tid = threadIdx.x;
  if (tid < NB) b[tid] = tid < nbw ? sol[j0 + tid] : 0.0;
  __syncthreads();
  if (tid < NB) {
    double sacc = 0.0;
    for (int c = 0; c <= tid; c++) sacc += Xcm[c * NB + tid] * b[c];  // X[tid][c]
    y[tid] = sacc;
    if (blockIdx.x == 0 && tid < nbw) ysol[j0 + tid] = sacc;
  }
  __syncthreads();
  const int i = j0 + nbw + blockIdx.x * 256 + tid;
  if (i < n) {
    double s = 0.0;
    for (int c = 0; c < nbw; c++) s += A[(size_t)(j0 + c) * n + i] * y[c];
    sol[i] -= s;
  }
}

__global__ void axpy_kernel(double *x, const double *d, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] += d[i];
}
__global__ void copy_kernel(double *dst, const double *src, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[i];
}

// rhs = -g (start of the forward substitution, fused into the factorisation)
__global__ void rhs_init_kernel(const double *g, double *sol, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) sol[i] = -g[i];
}

// Backward substitution L^T x = w (w = d^-1 y, scaled beforehand), block groups descending. One launch handles up to
// four 64-row blocks [g_lo, g_lo+G): every CTA first solves the group's own triangle redundantly (x_b = X_b^T w_b,
// then w_c -= L[b rows][c] x_b for the group's lower columns; a warp per column, rows contiguous -> coalesced), which
// replaces three kernel boundaries of the serial chain by block barriers, and then applies the group's G rows to its
// share of the columns left of the group (w_c -= sum_r L[g_lo+r][c] x[r], up to 2 KB contiguous per column).
constexpr int BACK_GROUP = 4;
__global__ void __launch_bounds__(256) ldl_back_kernel(const double *A, int n, int g_lo, int G, const double *Xcm,
                                                       double *sol, double *x) {
  __shared__ double w[BACK_GROUP * NB], xs[BACK_GROUP * NB];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  w[tid] = tid < G ? sol[g_lo + tid] : 0.0;
  xs[tid] = 0.0;
  __syncthreads();
  const int nblk = (G + NB - 1) / NB;
  for (int b = nblk - 1; b >= 0; b--) {
    const int j = NB * b;
    const int bw = G - j < NB ? G - j : NB;
    const double *Xb = Xcm + (size_t)b * NB * NB;  // column-major X = L_bb^-1 (identity-padded when bw < NB)
#pragma unroll
    for (int q = 0; q < 8; q++) {  // x_b[c] = sum_r X[r][c] w_b[r]
      const int c = warp * 8 + q;
      double sacc = Xb[c * NB + lane] * w[j + lane] + Xb[c * NB + lane + 32] * w[j + lane + 32];
      sacc = warp_sum(sacc);
      if (lane == 0) xs[j + c] = c < bw ? sacc : 0.0;
    }
    __syncthreads();
#pragma unroll 4
    for (int cl = warp; cl < j; cl += 8) {  // the group's columns below block b
      const double *col = A + (size_t)(g_lo + cl) * n + g_lo + j;
      double sacc = 0.0;
      if (lane < bw) sacc = col[lane] * xs[j + lane];
      if (lane + 32 < bw) sacc += col[lane + 32] * xs[j + lane + 32];
      sacc = warp_sum(sacc);
      if (lane == 0) w[cl] -= sacc;
    }
    __syncthreads();
  }
  if (blockIdx.x == 0 && tid < G) x[g_lo + tid] = xs[tid];
#pragma unroll
  for (int q = 0; q < 4; q++) {  // columns left of the group: 8 warps x 4 columns per CTA
    const int c = (blockIdx.x * 8 + warp) * 4 + q;
    if (c >= g_lo) break;
    const double *col = A + (size_t)c * n + g_lo;
    double sacc = 0.0;
#pragma unroll
    for (int r = lane; r < BACK_GROUP * NB; r += 32)
      if (r < G) sacc += col[r] * xs[r];
    sacc = warp_sum(sacc);
    if (lane == 0) sol[c] -= sacc;
  }
}

__global__ void scale_rhs_kernel(double *sol, const double *ysol, const double *dinv_all, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) sol[i] = ysol[i] * dinv_all[i];  // w = d^-1 y: start of the backward substitution
}

__global__ void __launch_bounds__(1024) q1_kernel(const double *x, const double *g, const double *dvec, int n,
                                                  const double *u_dev, double *scal) {
  __shared__ double red[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double u = *u_dev;
  double part = 0.0;
  for (int i = tid; i < n; i += 1024) {
    const double xi = x[i];
    part += xi * (u * dvec[i] * xi - g[i]);
  }
  part = warp_sum(part);
  if (lane == 0) red[warp] = part;
  __syncthreads();
  if (warp == 0) {
    double s = red[lane];
    s = warp_sum(s);
    if (lane == 0) scal[1] = 0.5 * s;  // q1 = 0.5 dx.(u D dx - g)  (bavoxel.hpp:1127)
  }
}

// R <- Exp(phi) R, p <- Exp(phi) p + dt  (bavoxel.hpp:1123-1125)
__global__ void pose_update_kernel(const double *pin, const double *dx, double *pout, int N) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  pose_update_one(pin + 12 * j, dx + 6 * j, pout + 12 * j);
}

// x_i <- T_0^-1 x_i (bavoxel.hpp:1159-1164); mode 1 also forces pose 0 to the exact identity
// (benchmark_virtual.cpp:472-479). pose 0 is read from a snapshot so the in-place update is race-free.
__global__ void gauge_kernel(double *poses, const double *pose0_snapshot, int N, int mode) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  gauge_one(poses + 12 * j, pose0_snapshot, mode == 1 && j == 0);
}

}  // namespace

// omega of the current s.dx (+ the residual vector in s.w->rres); flags[4] raised when omega > tol. scal[20] = omega.
static int enqueue_solve_check(balm_ctx *c, const DenseSystem &s) {
  const int n = s.n;
  CUDA_TRY(cudaMemsetAsync(c->scal + 20, 0, sizeof(double), c->stream));
  solve_residual_kernel<<<(n + 7) / 8, 256, 0, c->stream>>>(s.H, s.g, s.dx, n, c->scal + 3, SOLVE_OMEGA_TOL, s.w->rres,
                                                            c->flags, c->scal + 20);
  c->launches += 1;
  return BALM_OK;
}

static int enqueue_back_substitution(balm_ctx *c, const DenseSystem &s, const double *rhs_g, double *x_out, bool with_q1);

// fp64 iterative refinement of s.dx with the factors left in s.A / s.w->Xinv / s.w->dinv (host-driven, rare path: the
// backward-error check of the last solve raised flags[4]). Returns via *still_bad whether omega stayed above the tolerance.
int refine_solution(balm_ctx *c, const DenseSystem &s, int *still_bad) {
  const int n = s.n;
  LdltWork &w = *s.w;
  cudaStream_t st = c->stream;
  *still_bad = 1;
  for (int round = 0; round < 3; round++) {
    // solve A delta = r with the existing factors: forward (block by block), scale, backward
    copy_kernel<<<(n + 255) / 256, 256, 0, st>>>(w.sol, w.rres, n);
    int launches = 1;
    for (int j0 = 0, pi = 0; j0 < n; j0 += NB, pi++) {
      const int nbw = (n - j0 < NB) ? n - j0 : NB;
      const int m = n - j0 - nbw;
      ldl_fwd_block_kernel<<<m > 0 ? (m + 255) / 256 : 1, 256, 0, st>>>(s.A, n, j0, nbw, w.Xinv + (size_t)pi * NB * NB,
                                                                        w.sol, w.ysol);
      launches++;
    }
    c->launches += launches;
    TRY(enqueue_back_substitution(c, s, s.g, w.rdelta, false));
    axpy_kernel<<<(n + 255) / 256, 256, 0, st>>>(s.dx, w.rdelta, n);
    q1_kernel<<<1, 1024, 0, st>>>(s.dx, s.g, s.dvec, n, c->scal + 3, c->scal);
    c->launches += 2;
    CUDA_TRY(cudaMemsetAsync(c->flags + 4, 0, sizeof(int), st));
    TRY(enqueue_solve_check(c, s));
    CUDA_TRY(cudaMemcpyAsync(c->h_flags + 4, c->flags + 4, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(c->h_scal + 1, c->scal + 1, sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (c->h_flags[4] == 0) { *still_bad = 0; break; }
  }
  return BALM_OK;
}

// Everything of the solve that follows the factorisation: w = d^-1 y, grouped backward substitution, q1.
static int enqueue_back_substitution(balm_ctx *c, const DenseSystem &s, const double *rhs_g, double *x_out, bool with_q1) {
  const int n = s.n;
  const LdltWork &w = *s.w;
  cudaStream_t st = c->stream;
  scale_rhs_kernel<<<(n + 255) / 256, 256, 0, st>>>(w.sol, w.ysol, w.dinv, n);
  int launches = 1;
  const int npan = (n + NB - 1) / NB;
  for (int hi = npan - 1; hi >= 0; hi -= BACK_GROUP) {
    const int lo = hi - BACK_GROUP + 1 > 0 ? hi - BACK_GROUP + 1 : 0;
    const int g_lo = lo * NB;
    const int g_hi = (hi + 1) * NB < n ? (hi + 1) * NB : n;
    const int blocks = g_lo > 0 ? (g_lo + 31) / 32 : 1;
    ldl_back_kernel<<<blocks, 256, 0, st>>>(s.A, n, g_lo, g_hi - g_lo, w.Xinv + (size_t)lo * NB * NB, w.sol, x_out);
    launches++;
  }
  if (with_q1) {
    q1_kernel<<<1, 1024, 0, st>>>(x_out, rhs_g, s.dvec, n, c->scal + 3, c->scal);
    launches++;
  }
  c->launches += launches;
  return BALM_OK;
}

// The damped solve: damp/copy + rhs, ONE cooperative launch for the factorisation and forward substitution,
// then the grouped backward substitution, q1 and the backward-error check.
static int enqueue_solve_dag(balm_ctx *c, const DenseSystem &s) {
  const int n = s.n, nt = (n + NB - 1) / NB;
  const LdltWork &w = *s.w;
  cudaStream_t st = c->stream;
  dim3 g1((n + 255) / 256, n);
  damp_copy_kernel<<<g1, 256, 0, st>>>(s.H, s.A, s.dvec, n, c->scal + 3);
  rhs_init_kernel<<<(n + 255) / 256, 256, 0, st>>>(s.g, w.sol, n);
  CUDA_TRY(cudaMemsetAsync(w.dag_flags, 0, sizeof(int) * (2 * (size_t)nt * nt + 2 * nt), st));
  dag::Args a;
  a.A = s.A; a.n = n; a.nt = nt; a.Xinv = w.Xinv; a.dinv = w.dinv; a.dval = w.dval; a.sol = w.sol; a.ysol = w.ysol;
  a.flags = c->flags; a.upd = w.dag_flags; a.pdone = w.dag_flags + (size_t)nt * nt;
  a.xdone = w.dag_flags + 2 * (size_t)nt * nt; a.rhs_cnt = a.xdone + nt;
  // one CTA per SM (216 KB of shared memory each); a grid that cannot be co-resident makes the cooperative launch fail
  const int grid = nt < 2 ? 1 : c->sm_count;
  const int workers = grid - 1;
  a.near_ctas = workers >= 16 ? 8 : 0;
  a.trace = w.dag_trace;
  void *params[] = {&a};
  CUDA_TRY(cudaLaunchCooperativeKernel((const void *)dag::ldl_dag_kernel, dim3(grid), dim3(256), params,
                                       dag::SMEM_DOUBLES * sizeof(double), st));
  c->launches += 3;
  return enqueue_back_substitution(c, s, s.g, s.dx, true);
}

void ldlt_work_free(LdltWork *w) {
  cudaFree(w->Xinv); cudaFree(w->dinv); cudaFree(w->dval); cudaFree(w->sol); cudaFree(w->ysol); cudaFree(w->rres);
  cudaFree(w->rdelta); cudaFree(w->dag_flags); cudaFree(w->dag_trace);
  *w = LdltWork{};
}

int launch_ldlt_solve(balm_ctx *c, const DenseSystem &s, double u) {
  const int n = s.n;
  LdltWork &w = *s.w;
  if (!w.Xinv) {
    const int npan = (n + NB - 1) / NB;
    CUDA_TRY(cudaMalloc((void **)&w.Xinv, sizeof(double) * (size_t)npan * NB * NB));
    CUDA_TRY(cudaMalloc((void **)&w.dinv, sizeof(double) * n));
    CUDA_TRY(cudaMalloc((void **)&w.dval, sizeof(double) * n));
    CUDA_TRY(cudaMalloc((void **)&w.sol, sizeof(double) * n));
    CUDA_TRY(cudaMalloc((void **)&w.ysol, sizeof(double) * n));
    CUDA_TRY(cudaMalloc((void **)&w.rres, sizeof(double) * n));
    CUDA_TRY(cudaMalloc((void **)&w.rdelta, sizeof(double) * n));
    CUDA_TRY(cudaMalloc((void **)&w.dag_flags, sizeof(int) * (2 * (size_t)npan * npan + 2 * npan)));
    if (getenv("BALM_DAG_TRACE")) {
      CUDA_TRY(cudaMalloc((void **)&w.dag_trace, sizeof(unsigned long long) * (4 * (size_t)npan + 8 * 1024)));
      CUDA_TRY(cudaMemset(w.dag_trace, 0, sizeof(unsigned long long) * (4 * (size_t)npan + 8 * 1024)));
    }
  }
  c->h_scal[3] = u;  // pinned; the kernels read the damping factor from device memory
  CUDA_TRY(cudaMemcpyAsync(c->scal + 3, c->h_scal + 3, sizeof(double), cudaMemcpyHostToDevice, c->stream));
  CUDA_TRY(cudaMemsetAsync(c->flags, 0, sizeof(int) * 8, c->stream));
  TRY(enqueue_solve_dag(c, s));
  TRY(enqueue_solve_check(c, s));
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int launch_pose_update(balm_ctx *c, const double *poses_in, const double *dx, double *poses_out) {
  pose_update_kernel<<<(c->N + 127) / 128, 128, 0, c->stream>>>(poses_in, dx, poses_out, c->N);
  c->launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int launch_gauge(cudaStream_t st, int N, double *poses, double *snap, int mode) {
  CUDA_TRY(cudaMemcpyAsync(snap, poses, 12 * sizeof(double), cudaMemcpyDeviceToDevice, st));
  gauge_kernel<<<(N + 127) / 128, 128, 0, st>>>(poses, snap, N, mode);
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int launch_q1(cudaStream_t st, const double *x, const double *g, const double *dvec, int n, const double *u_dev,
              double *scal) {
  q1_kernel<<<1, 1024, 0, st>>>(x, g, dvec, n, u_dev, scal);
  return BALM_OK;
}

int ldlt_setup() {
  CUDA_TRY(cudaFuncSetAttribute(dag::ldl_dag_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                dag::SMEM_DOUBLES * (int)sizeof(double)));
  return BALM_OK;
}

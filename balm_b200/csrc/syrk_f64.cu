// syrk_f64.cu -- fp64 path of the rank-3M symmetric update (kernel K4) and the Hessian assembly.
//
//   S = G'^T G'  with G' (rows = 3 per voxel, cols = 6N, pose index contiguous)   [upper 128x128 tiles only]
//   H = -S + blockdiag(D_i),  g = accumulated gradient
// which restates the pair loop of left_evaluate_acc2 (bavoxel.hpp:404-418), the rank-1 parts of the diagonal
// blocks (:385,390-392) and the upper->lower mirror (:422-424) as one SYRK, because
//   H_ij += coe*(w0 a_i a_j^T + w1 g1_i g1_j^T + w2 g2_i g2_j^T),  w* < 0   <=>   H -= (G'^T G')_ij.
//
// BALM_PREC_FP64: DMMA (mma.sync.m8n8k4.f64) with cp.async double-buffered shared-memory tiles. This is the
// fp64 reference path ("fp64 accumulation", BASELINE config C2) and the on-device check of the tensor-core path.
// Work items are (tile, k-split); each item owns its slot of the partial buffer, and the assembly kernel sums
// the splits in a fixed order, so the result is run-to-run deterministic (no floating-point atomics).
#include "internal.cuh"

namespace {

constexpr int TILE = BALM_SYRK_TILE;  // 128
constexpr int KB = 16;                // G' rows per pipeline stage
constexpr int LDS = TILE + 4;         // padded smem row (doubles): conflict-free DMMA fragment loads
constexpr int SYRK_THREADS = 256;
constexpr int STAGE_DOUBLES = 2 * KB * LDS;

__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

struct SyrkArgs {
  const double *G;  // [rows][ldg]
  int64_t rows;
  int ldg;
  int nb;           // tiles per dimension
  int tiles;        // nb*(nb+1)/2
  int splits;
  double *part;     // [splits][tiles][TILE*TILE] row-major tiles
  int accumulate;   // add to existing partials (batches after the first)
  int row_xor;      // A operand taken from row (k ^ row_xor): 0 = SYRK; 4 = the partner rows of covariance.cu (Q V^T + V Q^T)
};

__device__ __forceinline__ void tile_coords(int t, int nb, int &bi, int &bj) {
  // upper-triangular enumeration: row bi, col bj >= bi
  int r = 0, rem = t;
  while (rem >= nb - r) { rem -= nb - r; r++; }
  bi = r;
  bj = r + rem;
}

__global__ void __launch_bounds__(SYRK_THREADS, 1) syrk_f64_kernel(SyrkArgs a) {
  extern __shared__ __align__(16) double smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 2, wn = warp & 3;  // 2 x 4 warps -> warp tile 64 x 32
  const int fr = lane >> 2, fk = lane & 3;

  for (int item = blockIdx.x; item < a.tiles * a.splits; item += gridDim.x) {
    const int t = item % a.tiles, sp = item / a.tiles;
    int bi, bj;
    tile_coords(t, a.nb, bi, bj);
    const int64_t per = ((a.rows + a.splits - 1) / a.splits + KB - 1) / KB * KB;
    const int64_t k_begin = (int64_t)sp * per;
    int64_t k_end = k_begin + per;
    if (k_end > a.rows) k_end = a.rows;
    const int nsteps = k_end > k_begin ? (int)((k_end - k_begin + KB - 1) / KB) : 0;

    double acc[8][4][2];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
      for (int j = 0; j < 4; j++) acc[i][j][0] = acc[i][j][1] = 0.0;

    const double *gA = a.G + (size_t)bi * TILE;
    const double *gB = a.G + (size_t)bj * TILE;

    auto load_stage = [&](int stage, int step) {
      double *sA = smem + stage * STAGE_DOUBLES;
      double *sB = sA + KB * LDS;
      const int64_t k0 = k_begin + (int64_t)step * KB;
      // KB rows x 128 doubles = KB*64 16-byte pieces per operand
      for (int e = tid; e < KB * 64; e += SYRK_THREADS) {
        const int rr = e >> 6, cc = (e & 63) * 2;
        const int64_t kr = k0 + rr;
        if (kr < k_end) {
          cp_async16(sA + rr * LDS + cc, gA + (size_t)(kr ^ a.row_xor) * a.ldg + cc);
          cp_async16(sB + rr * LDS + cc, gB + (size_t)kr * a.ldg + cc);
        } else {
          *reinterpret_cast<double2 *>(sA + rr * LDS + cc) = make_double2(0.0, 0.0);
          *reinterpret_cast<double2 *>(sB + rr * LDS + cc) = make_double2(0.0, 0.0);
        }
      }
    };

    if (nsteps > 0) {
      load_stage(0, 0);
      cp_async_commit();
    }
    for (int step = 0; step < nsteps; step++) {
      if (step + 1 < nsteps) {
        load_stage((step + 1) & 1, step + 1);
        cp_async_commit();
        cp_async_wait<1>();
      } else {
        cp_async_wait<0>();
      }
      __syncthreads();
      const double *sA = smem + (step & 1) * STAGE_DOUBLES;
      const double *sB = sA + KB * LDS;
#pragma unroll
      for (int kk = 0; kk < KB; kk += 4) {
        double af[8], bf[4];
#pragma unroll
        for (int i = 0; i < 8; i++) af[i] = sA[(kk + fk) * LDS + wm * 64 + i * 8 + fr];
#pragma unroll
        for (int j = 0; j < 4; j++) bf[j] = sB[(kk + fk) * LDS + wn * 32 + j * 8 + fr];
#pragma unroll
        for (int i = 0; i < 8; i++)
#pragma unroll
          for (int j = 0; j < 4; j++) dmma_8x8x4(acc[i][j][0], acc[i][j][1], af[i], bf[j]);
      }
      __syncthreads();
    }

    double *out = a.part + ((size_t)sp * a.tiles + t) * (TILE * TILE);
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int row = wm * 64 + i * 8 + fr;
        const int col = wn * 32 + j * 8 + 2 * fk;
        double2 *p = reinterpret_cast<double2 *>(out + row * TILE + col);
        double2 v = make_double2(acc[i][j][0], acc[i][j][1]);
        if (a.accumulate) {
          const double2 old = *p;
          v.x += old.x;
          v.y += old.y;
        }
        *p = v;
      }
  }
}

struct AsmArgs {
  const double *part;
  int splits, tiles, nb;
  const double *accum;  // [BALM_ACC][Np]: g and the exact diagonal (read only with g / exact_diag)
  int Np, n;
  const double *dblk;   // upper triangles of the 6x6 diagonal blocks, element q of pose i at dblk[q * ldd + i]
  int ldd;
  int exact_diag;       // take the diagonal of G'^T G' from the fp64 sums of squares (tensor path)
  double *H;            // n x n
  double *g;            // n, or null
  double *pack;         // multi-GPU: write the lower triangle | g straight into the all-reduce buffer instead of H (or null)
};

// H(i,j) = -sum_splits S(i,j) (NEG, the Hessian) or +sum_splits S(i,j) (the covariance's Rcov_raw), splits in ascending
// order, then + the D block on the diagonal; lower triangle mirrored from the upper tiles.
// One CTA per 32x32 block of the upper triangle: the partial tiles are read coalesced (column index fastest), the
// mirrored (lower) element is written straight away (coalesced in the same index) and the upper element goes through
// a shared-memory transpose so that its column-major store is coalesced too.
template <bool NEG>
__global__ void __launch_bounds__(1024) assemble_kernel(AsmArgs a) {
  __shared__ double tile[32][33];
  const int bx = blockIdx.x, by = blockIdx.y;  // block row bx, block column by (by >= bx)
  if (by < bx) return;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int r = bx * 32 + ty, c = by * 32 + tx;  // upper-triangle source element (r <= c except inside diagonal blocks)
  double h = 0.0;
  if (r < a.n && c < a.n) {
    const int rr = r < c ? r : c, cc = r < c ? c : r;
    const int bi = rr / TILE, bj = cc / TILE;
    const int t = bi * a.nb - bi * (bi - 1) / 2 + (bj - bi);
    const size_t off = (size_t)t * (TILE * TILE) + (size_t)(rr % TILE) * TILE + (cc % TILE);
    double s = 0.0;
    for (int sp = 0; sp < a.splits; sp++) s += a.part[(size_t)sp * a.tiles * (TILE * TILE) + off];
    h = NEG ? -s : s;
    const int pi = rr / 6, pj = cc / 6;
    if (a.exact_diag && rr == cc) h = -a.accum[(size_t)(27 + rr % 6) * a.Np + pi];
    if (pi == pj) {
      const int r6 = rr % 6, c6 = cc % 6;  // r6 <= c6
      const int q = r6 * 6 - r6 * (r6 - 1) / 2 + (c6 - r6);
      h += a.dblk[(size_t)q * a.ldd + pi];
    }
    // element (row c, col r): the mirrored (lower) one, coalesced in c -- into H, or into column r of the packed triangle
    if (a.pack) { if (c >= r) a.pack[(size_t)r * a.n - (size_t)r * (r - 1) / 2 + (c - r)] = h; }
    else a.H[(size_t)r * a.n + c] = h;
  }
  if (a.pack) {
    if (bx == 0 && ty == 0 && c < a.n) a.pack[(size_t)a.n * (a.n + 1) / 2 + c] = a.accum[(size_t)(c % 6) * a.Np + c / 6];
    return;
  }
  tile[ty][tx] = h;
  __syncthreads();
  if (by > bx) {  // element (row r', col c') of the upper block, coalesced in r'
    const int r2 = bx * 32 + tx, c2 = by * 32 + ty;
    if (r2 < a.n && c2 < a.n) a.H[(size_t)c2 * a.n + r2] = tile[tx][ty];
  }
  if (a.g && bx == 0 && ty == 0 && c < a.n) a.g[c] = a.accum[(size_t)(c % 6) * a.Np + c / 6];
}

}  // namespace

int launch_syrk_f64_on(balm_ctx *c, const double *G, int64_t rows, bool first_batch, int row_xor);
int launch_syrk_f64(balm_ctx *c, int64_t rows, bool first_batch) { return launch_syrk_f64_on(c, c->G, rows, first_batch, 0); }

int launch_syrk_f64_on(balm_ctx *c, const double *G, int64_t rows, bool first_batch, int row_xor) {
  SyrkArgs a{G, rows, c->ldg, c->syrk_nb, c->syrk_tiles, c->syrk_splits, c->syrk_part, first_batch ? 0 : 1, row_xor};
  const int smem = 2 * STAGE_DOUBLES * (int)sizeof(double);
  const int items = a.tiles * a.splits;
  const int grid = items < c->sm_count ? items : c->sm_count;
  syrk_f64_kernel<<<grid, SYRK_THREADS, smem, c->stream>>>(a);
  c->launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int launch_assemble(balm_ctx *c, const double *Dacc, double *R) {
  const int nbb = (c->n + 31) / 32;
  dim3 block(32, 32), grid(nbb, nbb);
  if (!Dacc) {
    const AsmArgs a{c->syrk_part, c->syrk_splits, c->syrk_tiles, c->syrk_nb, c->accum, c->Np, c->n, c->accum + 6 * c->Np,
                    c->Np, c->prec == BALM_PREC_TENSOR ? 1 : 0, c->H, c->g, (c->world > 1 && c->comm) ? c->Hpack : nullptr};
    assemble_kernel<true><<<grid, block, 0, c->stream>>>(a);
  } else {
    const AsmArgs a{c->syrk_part, c->syrk_splits, c->syrk_tiles, c->syrk_nb, nullptr, c->Np, c->n, Dacc, c->N, 0, R,
                    nullptr, nullptr};
    assemble_kernel<false><<<grid, block, 0, c->stream>>>(a);
  }
  c->launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int syrk_f64_setup() {
  CUDA_TRY(cudaFuncSetAttribute(syrk_f64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                2 * STAGE_DOUBLES * (int)sizeof(double)));
  return BALM_OK;
}

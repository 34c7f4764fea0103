// blocks.cu -- the block-sparse Hessian of a BALM_PREC_BLOCKS context (DESIGN.md "Block-sparse voxel BA").
// H is held as the 6x6 blocks of the pose pairs (i <= j) that share at least one voxel, plus every diagonal pair (i, i);
// the damped system is solved by the sparse pose graph's nested-dissection block LDL^T (pose_graph_sparse.cu).
// Nothing of size (6N)^2 exists.
//   Registration (block_hessian_build, every registration route ends here): every voxel emits its k(k+1)/2 observation
//   pairs keyed by their pose pair; one stable radix sort by key gives the unique pose pairs (run-length encoding) and,
//   for each, its update terms in ascending voxel order -- the fixed summation order of the evaluation.
//   Evaluation: the observation sweep (obs_pass_kernel<..., OBS_BLOCKS>) stores every observation's three scaled G' rows
//   (18 doubles) instead of the dense G'; blocks_kernel sums, per pair, the terms' outer products, one warp per pair,
//   lane l taking the terms l, l + 32, ... and the lanes' sums meeting in warp_sum's fixed butterfly. The block is minus
//   that sum, plus the observation sweep's diagonal block on a diagonal pair. fp64 throughout, no floating-point atomics.
//   Pose factors (balm_block_set_factors, DESIGN.md "Voxels and pose factors in one cost"): the pattern is the union of
//   the voxel pairs, the active factors' pairs, the diagonal pairs of the poses with an active prior and, on a context
//   of balm_create, every diagonal pair (block_pattern_build, rebuilt without re-sorting the voxel terms when only the
//   factors or the priors change); a full-range evaluation adds the factor sums of pose_graph.cu onto the voxel blocks,
//   g and residual, each entry once, in that order.
//   Absolute pose priors (balm_set_pose_priors, DESIGN.md "Absolute pose priors"): they touch only diagonal blocks; a
//   full-range evaluation adds their sums after the factors'. The sparse pose graph (balm_spg_*) is a context of this
//   kind without voxels whose pattern leaves out the other diagonal pairs.
#include <cub/cub.cuh>
#include <algorithm>
#include <memory>
#include <vector>
#include "internal.cuh"

// The union pattern: the voxel pairs, the pairs of the context's active pose factors and every diagonal pair (i, i),
// each pair's voxel terms (none for a pair no voxel gives), the blocks and their solver.
struct BlockPattern {
  std::vector<int2> pairs;           // host: (i, j), i <= j, ascending
  long long bytes = 0;
  int2 *pair_dev = nullptr;          // [pairs] (with voxel pairs only: blocks_kernel reads them)
  long long *tptr = nullptr;         // [pairs + 1] terms of pair p: term[tptr[p] .. tptr[p+1]) (same)
  double *blocks = nullptr;          // [pairs][36] column-major, rows of pose i
  // No voxel pair and every pair a factor pair (the sparse pose graph's usual pattern): the factor pass stores the
  // blocks, g and the cost, as nothing precedes it; otherwise it adds them through fmap and fgc.
  bool factors_only = false;
  int *fmap = nullptr;               // [factor pairs] index in `pairs` of each of pose_graph_pairs (with factors only)
  double *fgc = nullptr;             // [n + 1] the factors' g and cost before they are added (same)
  SparseSolver *solver = nullptr;
  long long gen = 0;                 // blocks_generation: unique to this pattern
  ~BlockPattern() {
    sparse_solver_free(solver);
    cudaFree(pair_dev); cudaFree(tptr); cudaFree(blocks); cudaFree(fmap); cudaFree(fgc);
  }
};

struct BlockHessian {
  std::vector<unsigned long long> vkey;  // host: pose pair i * N + j (i <= j) of every pair that shares a voxel, ascending
  std::vector<int> vcnt;                 // host: its number of terms
  long long nterm = 0;
  unsigned long long *term = nullptr;  // [nterm] observation of pose i (low word) | of pose j (high word), pair-major,
                                       // voxel-ascending within a pair
  std::unique_ptr<BlockPattern> pat;
  ~BlockHessian() { cudaFree(term); }
};

void block_hessian_free(BlockHessian *b) { delete b; }

namespace {

__global__ void pair_count_kernel(const long long *row_ptr, int64_t M, long long *cnt) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v > M) return;
  const long long k = v < M ? row_ptr[v + 1] - row_ptr[v] : 0;
  cnt[v] = k * (k + 1) / 2;
}

// one warp per voxel: the pairs (a, b), a <= b, of its observations, a-major, at the voxel's offset
__global__ void pair_emit_kernel(const long long *row_ptr, const int *pose_idx, int64_t M, int N, const long long *off,
                                 unsigned long long *key, unsigned long long *val) {
  const int64_t v = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (v >= M) return;
  const long long s0 = row_ptr[v];
  const int k = (int)(row_ptr[v + 1] - s0);
  long long o = off[v];
  for (int a = 0; a < k; a++) {
    const int pa = pose_idx[s0 + a];
    for (int b = a + lane; b < k; b += 32) {
      key[o + b - a] = (unsigned long long)pa * N + pose_idx[s0 + b];
      val[o + b - a] = (unsigned long long)(unsigned)(s0 + a) | ((unsigned long long)(unsigned)(s0 + b) << 32);
    }
    o += k - a;
  }
}

// One warp per pair: block = -sum_terms sum_rr Gs[s_i][rr] Gs[s_j][rr]^T (+ the diagonal block D_i on a diagonal pair),
// terms restricted to the observations [row_ptr[head], row_ptr[end]) (voxels [head, end)). Threads t < n also copy g.
__global__ void __launch_bounds__(256) blocks_kernel(const int2 *pairs, const long long *tptr,
                                                     const unsigned long long *term, long long npairs, const double *Gs,
                                                     const long long *row_ptr, int64_t head, int64_t end,
                                                     const double *accum, int Np, int n, double *blocks, double *g) {
  const long long gt = (long long)blockIdx.x * 256 + threadIdx.x;
  if (gt < n) g[gt] = accum[(size_t)(gt % 6) * Np + gt / 6];
  const long long p = gt >> 5;
  const int lane = threadIdx.x & 31;
  if (p >= npairs) return;
  const unsigned lo = (unsigned)row_ptr[head], hi = (unsigned)row_ptr[end];
  // the pair's terms are voxel-ascending, so their first observation index is too: [t0, t1) = those inside the range
  long long t0 = tptr[p], t1 = tptr[p + 1];
  {
    long long l = t0, h = t1;
    while (l < h) { const long long m = (l + h) >> 1; if ((unsigned)term[m] < lo) l = m + 1; else h = m; }
    t0 = l;
    h = t1;
    while (l < h) { const long long m = (l + h) >> 1; if ((unsigned)term[m] < hi) l = m + 1; else h = m; }
    t1 = l;
  }
  double acc[36];
#pragma unroll
  for (int e = 0; e < 36; e++) acc[e] = 0.0;
  for (long long t = t0 + lane; t < t1; t += 32) {
    const unsigned long long w = term[t];
    const double2 *gi = reinterpret_cast<const double2 *>(Gs + 18 * (size_t)(unsigned)w);
    const double2 *gj = reinterpret_cast<const double2 *>(Gs + 18 * (size_t)(unsigned)(w >> 32));
#pragma unroll
    for (int rr = 0; rr < 3; rr++) {
      double a[6], b[6];
#pragma unroll
      for (int h = 0; h < 3; h++) {
        const double2 x = __ldg(gi + 3 * rr + h), y = __ldg(gj + 3 * rr + h);
        a[2 * h] = x.x; a[2 * h + 1] = x.y;
        b[2 * h] = y.x; b[2 * h + 1] = y.y;
      }
#pragma unroll
      for (int c = 0; c < 6; c++)
#pragma unroll
        for (int r = 0; r < 6; r++) acc[6 * c + r] = fma(a[r], b[c], acc[6 * c + r]);
    }
  }
  const int2 pr = pairs[p];
  double *B = blocks + 36 * (size_t)p;
#pragma unroll
  for (int e = 0; e < 36; e++) {
    double h = -warp_sum(acc[e]);
    if (lane == (e & 31)) {
      if (pr.x == pr.y) {  // assemble_kernel's D block: upper triangle, row-major, index q of (min, max)
        const int r = e % 6, c = e / 6, r6 = r < c ? r : c, c6 = r < c ? c : r;
        const int q = r6 * 6 - r6 * (r6 - 1) / 2 + (c6 - r6);
        h += accum[(size_t)(6 + q) * Np + pr.x];
      }
      B[e] = h;
    }
  }
}

// The point-noise raw term in blocks_kernel's shape (one warp per pair, the same term ranges and butterfly): per term
// (s_i, s_j) the partner-row product sum_m rows[s_i][m] rows[s_j][m ^ 4]^T of covariance.cu's eight rows, rows of
// observation s at rows + 48 (s - row_ptr[v0]); Dacc (the diagonal blocks c2^2 D, [21][N], upper triangle) added on a
// diagonal pair when not null. A pair without voxel terms in the batch gets a zero sum.
__global__ void __launch_bounds__(256) raw_blocks_kernel(const int2 *pairs, const long long *tptr,
                                                         const unsigned long long *term, long long npairs,
                                                         const double *rows, const long long *row_ptr, int64_t v0,
                                                         int64_t v1, const double *Dacc, int N, int add, double *raw) {
  const long long p = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (p >= npairs) return;
  const unsigned lo = (unsigned)row_ptr[v0], hi = (unsigned)row_ptr[v1];
  long long t0 = tptr[p], t1 = tptr[p + 1];
  {
    long long l = t0, h = t1;
    while (l < h) { const long long m = (l + h) >> 1; if ((unsigned)term[m] < lo) l = m + 1; else h = m; }
    t0 = l;
    h = t1;
    while (l < h) { const long long m = (l + h) >> 1; if ((unsigned)term[m] < hi) l = m + 1; else h = m; }
    t1 = l;
  }
  double acc[36];
#pragma unroll
  for (int e = 0; e < 36; e++) acc[e] = 0.0;
  for (long long t = t0 + lane; t < t1; t += 32) {
    const unsigned long long w = term[t];
    const double *gi = rows + 48 * (size_t)((unsigned)w - lo), *gj = rows + 48 * (size_t)((unsigned)(w >> 32) - lo);
#pragma unroll
    for (int m = 0; m < 8; m++) {
      double a[6], b[6];
#pragma unroll
      for (int r = 0; r < 6; r++) {
        a[r] = __ldg(gi + 6 * m + r);
        b[r] = __ldg(gj + 6 * (m ^ 4) + r);
      }
#pragma unroll
      for (int c = 0; c < 6; c++)
#pragma unroll
        for (int r = 0; r < 6; r++) acc[6 * c + r] = fma(a[r], b[c], acc[6 * c + r]);
    }
  }
  const int2 pr = pairs[p];
  double *B = raw + 36 * (size_t)p;
#pragma unroll
  for (int e = 0; e < 36; e++) {
    double h = warp_sum(acc[e]);
    if (lane == (e & 31)) {
      if (add) h = B[e] + h;
      if (Dacc && pr.x == pr.y) {
        const int r = e % 6, c = e / 6, r6 = r < c ? r : c, c6 = r < c ? c : r;
        const int q = r6 * 6 - r6 * (r6 - 1) / 2 + (c6 - r6);
        h += Dacc[(size_t)q * N + pr.x];
      }
      B[e] = h;
    }
  }
}

// y[t] += x[t]: a blocks context's or a joint cost's factor g and cost added onto the voxel ones (one add per entry,
// fixed order)
__global__ void add_kernel(const double *x, int n, double *y) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) y[t] += x[t];
}

}  // namespace

// The union of bh's voxel pairs, pg's pairs (pg may be null), the diagonal pair of every pose with an active prior of pr
// (pr may be null) and, when c->every_diagonal, every diagonal pair, in ascending (i, j): a pair no voxel gives gets an
// empty term range (with every diagonal pair, a pose in no voxel and no factor gets a zero block, hence a zero pivot).
// When `same` (may be null) already has the union's pairs, *out is left empty; otherwise the blocks, the factor map and
// the symbolic factorisation -> *out.
static int block_pattern_build(balm_ctx *c, const BlockHessian &bh, const PoseGraph *pg, const PriorSet *pr,
                               const BlockPattern *same, const char *who, std::unique_ptr<BlockPattern> *out) {
  const int N = c->N;
  cudaStream_t st = c->stream;
  std::unique_ptr<BlockPattern> u(new BlockPattern());
  static const std::vector<int2> none;
  static const std::vector<int> no_pose;
  const std::vector<int2> &fp = pg ? pose_graph_pairs(pg) : none;
  const std::vector<int> &pp = prior_set_active(pr) ? prior_set_poses(pr) : no_pose;
  std::vector<long long> tptr;
  std::vector<int> fmap;
  u->pairs.reserve(bh.vkey.size() + N);
  tptr.reserve(bh.vkey.size() + N + 1);
  fmap.reserve(fp.size());
  tptr.push_back(0);
  size_t q = 0, r = 0, s = 0;  // cursors into the voxel pairs, the factor pairs and the prior poses
  const unsigned long long none_left = ~0ull;
  for (int i = 0; i < N; i++) {
    const unsigned long long row_end = (unsigned long long)(i + 1) * N;
    const bool prior = s < pp.size() && pp[s] == i;
    s += prior;
    bool diag = c->every_diagonal || prior;  // the diagonal pair is the smallest key of row i
    for (;;) {
      const unsigned long long kv = q < bh.vkey.size() && bh.vkey[q] < row_end ? bh.vkey[q] : none_left;
      const unsigned long long kf = r < fp.size() && fp[r].x == i ? (unsigned long long)i * N + fp[r].y : none_left;
      const unsigned long long k = diag ? (unsigned long long)i * N + i : std::min(kv, kf);
      if (k == none_left) break;
      diag = false;
      u->pairs.push_back(make_int2(i, (int)(k - (unsigned long long)i * N)));
      tptr.push_back(tptr.back() + (kv == k ? bh.vcnt[q++] : 0));
      if (kf == k) { fmap.push_back((int)u->pairs.size() - 1); r++; }
    }
  }
  const size_t np = u->pairs.size();
  if (same && same->pairs.size() == np &&
      std::equal(u->pairs.begin(), u->pairs.end(), same->pairs.begin(),
                 [](const int2 &a, const int2 &b) { return a.x == b.x && a.y == b.y; }))
    return BALM_OK;
  if (np >= ((size_t)1 << 30)) {
    balm_set_error(std::string(who) + ": 2^30 or more block pairs");
    return BALM_ERR_UNSUPPORTED;
  }
  TRY(dev_alloc(&u->blocks, 36 * np));
  CUDA_TRY(cudaMemsetAsync(u->blocks, 0, sizeof(double) * 36 * np, st));
  u->bytes = (long long)(np * 36 * sizeof(double));
  if (!bh.vkey.empty()) {
    TRY(dev_alloc(&u->pair_dev, np));
    TRY(dev_alloc(&u->tptr, np + 1));
    CUDA_TRY(cudaMemcpyAsync(u->pair_dev, u->pairs.data(), sizeof(int2) * np, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(u->tptr, tptr.data(), sizeof(long long) * (np + 1), cudaMemcpyHostToDevice, st));
    u->bytes += (long long)(np * (sizeof(int2) + sizeof(long long)) + sizeof(long long));
  }
  u->factors_only = pg && bh.vkey.empty() && fmap.size() == np;
  if (pg && !u->factors_only) {
    TRY(dev_alloc(&u->fmap, fmap.size()));
    TRY(dev_alloc(&u->fgc, (size_t)c->n + 1));
    if (!fmap.empty())
      CUDA_TRY(cudaMemcpyAsync(u->fmap, fmap.data(), sizeof(int) * fmap.size(), cudaMemcpyHostToDevice, st));
    u->bytes += (long long)(sizeof(int) * std::max<size_t>(1, fmap.size()) + sizeof(double) * ((size_t)c->n + 1));
  }
  TRY(sparse_solver_build(st, N, u->pairs, u->blocks, c->g, c->dvec, c->dx, c->scal, c->flags, who, &u->solver));
  CUDA_TRY(cudaStreamSynchronize(st));  // the host tables above are freed on return
  static long long generations = 0;
  u->gen = ++generations;
  *out = std::move(u);
  return BALM_OK;
}

int block_hessian_build(balm_ctx *c, const char *who) {
  const int N = c->N;
  const int64_t M = c->M;
  cudaStream_t st = c->stream;
  ScratchPool pool;
  std::unique_ptr<BlockHessian> bh(new BlockHessian());
  auto refuse = [&](const char *what) {
    balm_set_error(std::string(who) + ": " + what);
    return (int)BALM_ERR_UNSUPPORTED;
  };
  if (M > 0) {
    long long *cnt = nullptr, *off = nullptr;
    TRY(pool.get(&cnt, (size_t)M + 1));
    TRY(pool.get(&off, (size_t)M + 1));
    pair_count_kernel<<<(unsigned)((M + 1 + 255) / 256), 256, 0, st>>>(c->row_ptr, M, cnt);
    size_t tb = 0;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt, off, M + 1, st));
    char *tmp = nullptr;
    TRY(pool.get(&tmp, tb));
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tb, cnt, off, M + 1, st));
    long long nterm = 0;
    CUDA_TRY(cudaMemcpyAsync(&nterm, off + M, sizeof(long long), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    pool.drop(tmp);
    pool.drop(cnt);
    if (nterm >= (1LL << 31)) return refuse("2^31 or more observation pairs (block update terms)");
    bh->nterm = nterm;
    // key: pose pair i * N + j, value: the two observations; one stable sort by key
    unsigned long long *k0 = nullptr, *k1 = nullptr, *v0 = nullptr, *v1 = nullptr;
    TRY(pool.get(&k0, (size_t)nterm)); TRY(pool.get(&k1, (size_t)nterm));
    TRY(pool.get(&v0, (size_t)nterm)); TRY(pool.get(&v1, (size_t)nterm));
    pair_emit_kernel<<<(unsigned)((M * 32 + 255) / 256), 256, 0, st>>>(c->row_ptr, c->pose_idx, M, N, off, k0, v0);
    int bits = 1;
    while (bits < 64 && ((unsigned long long)1 << bits) < (unsigned long long)N * N) bits++;
    cub::DoubleBuffer<unsigned long long> dk(k0, k1), dv(v0, v1);
    tb = 0;
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb, dk, dv, (int)nterm, 0, bits, st));
    TRY(pool.get(&tmp, tb));
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tb, dk, dv, (int)nterm, 0, bits, st));
    pool.drop(tmp);
    // unique pose pairs and their term counts, into the sort's spare buffers
    unsigned long long *uk = dk.Alternate();
    int *uc = reinterpret_cast<int *>(dv.Alternate()), *nruns = nullptr;
    TRY(pool.get(&nruns, 1));
    tb = 0;
    CUDA_TRY(cub::DeviceRunLengthEncode::Encode(nullptr, tb, dk.Current(), uk, uc, nruns, (int)nterm, st));
    TRY(pool.get(&tmp, tb));
    CUDA_TRY(cub::DeviceRunLengthEncode::Encode(tmp, tb, dk.Current(), uk, uc, nruns, (int)nterm, st));
    int nr = 0;
    CUDA_TRY(cudaMemcpyAsync(&nr, nruns, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (nr + (long long)N >= (1LL << 30)) return refuse("2^30 or more block pairs");
    bh->vkey.resize(nr);
    bh->vcnt.resize(nr);
    CUDA_TRY(cudaMemcpyAsync(bh->vkey.data(), uk, sizeof(unsigned long long) * nr, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(bh->vcnt.data(), uc, sizeof(int) * nr, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    CUDA_TRY(cudaGetLastError());
    c->launches += 5;
    // keep the sorted terms, free everything else
    bh->term = dv.Current();
    pool.release(bh->term);
  }
  TRY(block_pattern_build(c, *bh, c->pg, c->pr, nullptr, who, &bh->pat));
  if (c->pr) TRY(prior_set_map(c->pr, st, bh->pat->pairs));
  block_hessian_free(c->bh);
  c->bh = bh.release();
  return BALM_OK;
}

int blocks_repattern(balm_ctx *c, const PoseGraph *pg, const char *who) {
  std::unique_ptr<BlockPattern> pat;
  TRY(block_pattern_build(c, *c->bh, pg, c->pr, nullptr, who, &pat));
  if (c->pr) TRY(prior_set_map(c->pr, c->stream, pat->pairs));
  c->bh->pat = std::move(pat);
  return BALM_OK;
}

int blocks_set_priors(balm_ctx *c, PriorSet *pr, const char *who) {
  std::unique_ptr<BlockPattern> pat;  // stays empty while the union keeps its pairs
  if (!c->every_diagonal) TRY(block_pattern_build(c, *c->bh, c->pg, pr, c->bh->pat.get(), who, &pat));
  if (pr) TRY(prior_set_map(pr, c->stream, (pat ? pat : c->bh->pat)->pairs));
  if (pat) c->bh->pat = std::move(pat);
  return BALM_OK;
}

int blocks_add_priors(balm_ctx *c, const double *poses) {
  return prior_add_blocks(c->pr, c->stream, poses, c->bh->pat->blocks, c->g, c->g + c->n, &c->launches);
}

int launch_blocks(balm_ctx *c, int64_t head, int64_t end) {
  const BlockHessian *b = c->bh;
  const BlockPattern &u = *b->pat;
  const long long np = (long long)u.pairs.size();
  const long long threads = std::max<long long>(32 * np, c->n);
  blocks_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, c->stream>>>(u.pair_dev, u.tptr, b->term, np, c->G,
                                                                          c->row_ptr, head, end, c->accum, c->Np, c->n,
                                                                          u.blocks, c->g);
  c->launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int blocks_add_factors(balm_ctx *c, const double *poses) {
  const BlockPattern &u = *c->bh->pat;
  if (u.factors_only) return pose_graph_eval_blocks(c->pg, c->stream, poses, u.blocks, c->g, c->g + c->n, &c->launches);
  TRY(pose_graph_add_blocks(c->pg, c->stream, poses, u.blocks, u.fmap, u.fgc, u.fgc + c->n, &c->launches));
  add_kernel<<<(unsigned)((c->n + 1 + 255) / 256), 256, 0, c->stream>>>(u.fgc, c->n + 1, c->g);  // g, then r = g[n]
  c->launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int blocks_add_factor_cost(balm_ctx *c, const double *poses, double *r) {
  const BlockPattern &u = *c->bh->pat;
  if (u.factors_only) return pose_graph_cost(c->pg, c->stream, poses, r, &c->launches);  // *r holds no voxel cost
  TRY(pose_graph_cost(c->pg, c->stream, poses, u.fgc + c->n, &c->launches));
  add_kernel<<<1, 32, 0, c->stream>>>(u.fgc + c->n, 1, r);
  c->launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int joint_add_factors(balm_ctx *c, const double *poses) {
  TRY(pose_graph_add_dense(c->pg, c->stream, poses, c->H, c->joint_fg, c->joint_fg + c->n, &c->launches));
  add_kernel<<<(unsigned)((c->n + 1 + 255) / 256), 256, 0, c->stream>>>(c->joint_fg, c->n + 1, c->g);  // g, r = g[n]
  c->launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int joint_add_factor_cost(balm_ctx *c, const double *poses, double *r) {
  TRY(pose_graph_cost(c->pg, c->stream, poses, c->joint_fg + c->n, &c->launches));
  add_kernel<<<1, 32, 0, c->stream>>>(c->joint_fg + c->n, 1, r);
  c->launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int blocks_zero(balm_ctx *c) {
  const BlockPattern &u = *c->bh->pat;
  if (u.factors_only) return BALM_OK;  // blocks_add_factors writes every block, g and r
  CUDA_TRY(cudaMemsetAsync(u.blocks, 0, sizeof(double) * 36 * u.pairs.size(), c->stream));
  CUDA_TRY(cudaMemsetAsync(c->g, 0, sizeof(double) * ((size_t)c->n + 1), c->stream));
  return BALM_OK;
}

int launch_raw_blocks(balm_ctx *c, const double *rows, int64_t v0, int64_t v1, const double *Dacc, bool add, double *raw) {
  const BlockHessian *b = c->bh;
  const BlockPattern &u = *b->pat;
  if (!u.pair_dev) { balm_set_error("raw blocks: the pattern has no voxel pairs"); return BALM_ERR_INVALID; }
  const long long np = (long long)u.pairs.size();
  raw_blocks_kernel<<<(unsigned)((32 * np + 255) / 256), 256, 0, c->stream>>>(u.pair_dev, u.tptr, b->term, np, rows,
                                                                              c->row_ptr, v0, v1, Dacc, c->N, add ? 1 : 0,
                                                                              raw);
  c->launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

const std::vector<int2> &blocks_pairs(const BlockHessian *b) { return b->pat->pairs; }
const double *blocks_device(const BlockHessian *b) { return b->pat->blocks; }
SparseSolver *blocks_solver(const BlockHessian *b) { return b->pat->solver; }
long long blocks_generation(const BlockHessian *b) { return b->pat->gen; }

long long blocks_bytes(const BlockHessian *b, int64_t *l_blocks, int64_t *levels) {
  int64_t sb = 0;
  sparse_solver_stats(b->pat->solver, l_blocks, levels, &sb);
  return (long long)sizeof(unsigned long long) * b->nterm + b->pat->bytes + sb;
}

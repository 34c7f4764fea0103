// balm_api.cu -- C ABI of libbalm_b200.so (include/balm_b200.h): context, problem registration, the
// evaluation pipeline, the damped solve and the Levenberg-Marquardt driver of BALM2::damping_iter
// (src/benchmark/bavoxel.hpp:1069-1166).  Host code is plain C++; all arithmetic of the hot
// path runs in the CUDA kernels of this directory.  There is no CPU fallback: without a CUDA device every
// entry point fails with BALM_ERR_CUDA.
#include <dlfcn.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <climits>
#include <memory>
#include <vector>
#include <time.h>
#include "internal.cuh"

void synth_host_poses(int N, uint64_t seed, double *poses_gt, double *poses_init);

static thread_local std::string g_err;
void balm_set_error(const std::string &s) { g_err = s; }
extern "C" const char *balm_last_error(void) { return g_err.c_str(); }
extern "C" int balm_version(void) { return 100; }

// ---------------- NCCL through dlopen (no link-time dependency) ----------------
struct NcclDyn {
  void *h = nullptr;
  typedef struct { char internal[128]; } uid_t;
  int (*GetUniqueId)(uid_t *) = nullptr;
  int (*CommInitRank)(void **, int, uid_t, int) = nullptr;
  int (*AllReduce)(const void *, void *, size_t, int, int, void *, cudaStream_t) = nullptr;
  int (*CommDestroy)(void *) = nullptr;
  const char *(*GetErrorString)(int) = nullptr;
  bool load() {
    if (h) return true;
    const char *names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char *nm : names) {
      h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
      if (h) break;
    }
    if (!h) return false;
    GetUniqueId = (decltype(GetUniqueId))dlsym(h, "ncclGetUniqueId");
    CommInitRank = (decltype(CommInitRank))dlsym(h, "ncclCommInitRank");
    AllReduce = (decltype(AllReduce))dlsym(h, "ncclAllReduce");
    CommDestroy = (decltype(CommDestroy))dlsym(h, "ncclCommDestroy");
    GetErrorString = (decltype(GetErrorString))dlsym(h, "ncclGetErrorString");
    return GetUniqueId && CommInitRank && AllReduce && CommDestroy;
  }
};
static NcclDyn g_nccl;

// ---------------- helpers ----------------
static void free_problem(balm_ctx *c) {
  cudaFree(c->obs); cudaFree(c->pose_idx); cudaFree(c->row_ptr); cudaFree(c->coe); cudaFree(c->fix);
  cudaFree(c->csc_ptr); cudaFree(c->csc_obs); cudaFree(c->csc_vox); cudaFree(c->csc_lo); cudaFree(c->csc_hi);
  c->csc_lo = c->csc_hi = nullptr;
  c->obs = nullptr; c->pose_idx = nullptr; c->row_ptr = nullptr; c->coe = nullptr; c->fix = nullptr;
  c->csc_ptr = c->csc_obs = c->csc_vox = nullptr;
  cudaFree(c->vsums); c->vsums = nullptr;
  cudaFree(c->stats); cudaFree(c->stats_trial); cudaFree(c->G); cudaFree(c->obs_part); cudaFree(c->syrk_part);
  c->stats = c->stats_trial = c->G = c->obs_part = c->syrk_part = nullptr;
  tensor_syrk_free(c);
  block_hessian_free(c->bh);
  c->bh = nullptr;
  c->M = c->K = c->Kp = 0;
  c->registered = false;
}
static void drop_keys(balm_ctx *c) {  // a voxel set registered from arrays carries no octree keys
  cudaFree(c->vox_key);
  cudaFree(c->vox_layer);
  c->vox_key = nullptr;
  c->vox_layer = nullptr;
  c->has_keys = false;
}

static int alloc_problem_arrays(balm_ctx *c, int64_t M, int64_t K, bool with_fix) {
  // A window of the same shape as the previous one (the common case when BA runs scan after scan, and what every
  // repetition of a benchmark does) keeps every device buffer: cudaFree/cudaMalloc of several GB cost milliseconds.
  // A blocks context rebuilds its pattern on every registration: equal M and K do not mean equal co-visibility.
  c->reuse_ws = c->prec != BALM_PREC_BLOCKS && c->obs && c->stats && c->M == M && c->K == K &&
                (c->fix != nullptr) == with_fix;
  if (c->reuse_ws) {
    cudaFree(c->csc_ptr); cudaFree(c->csc_obs); cudaFree(c->csc_vox); cudaFree(c->csc_lo); cudaFree(c->csc_hi);
    c->csc_ptr = c->csc_obs = c->csc_vox = c->csc_lo = c->csc_hi = nullptr;
    return BALM_OK;
  }
  free_problem(c);
  c->M = M; c->K = K;
  c->Kp = (K + 31) / 32 * 32;
  TRY(dev_alloc(&c->obs, (size_t)10 * c->Kp));
  TRY(dev_alloc(&c->pose_idx, (size_t)K));
  TRY(dev_alloc(&c->row_ptr, (size_t)M + 1));
  TRY(dev_alloc(&c->coe, (size_t)M));
  if (with_fix) TRY(dev_alloc(&c->fix, (size_t)10 * M));
  return BALM_OK;
}

// Workspaces that depend on the registered problem (batch size, split counts; the block pattern of a blocks context).
static int alloc_workspaces_of(balm_ctx *c) {
  if (c->reuse_ws) {  // same shape: batch size, split counts, tensor maps and digit-plane buffers are all unchanged
    c->reuse_ws = false;
    tensor_syrk_new_problem(c);
    return BALM_OK;
  }
  size_t g_budget = (size_t)16 << 30;  // bytes for the fp64 G' batch
  if (const char *e = getenv("BALM_G_BUDGET_MB")) g_budget = (size_t)atoll(e) << 20;  // tests: force batching
  const bool blocks = c->prec == BALM_PREC_BLOCKS;
  if (blocks && (size_t)18 * sizeof(double) * c->K > g_budget) {  // single batch: every observation's G' rows at once
    free_problem(c);
    balm_set_error("blocks registration: the per-observation G' rows (144 B per observation) exceed the G' budget");
    return BALM_ERR_UNSUPPORTED;
  }
  int64_t vb = blocks ? c->M : (int64_t)(g_budget / ((size_t)3 * c->ldg * sizeof(double)));
  if (vb > c->M) vb = c->M;
  if (vb < 1) vb = 1;
  c->VB = vb;
  TRY(dev_alloc(&c->stats, (size_t)vb * BALM_STATS_STRIDE));
  if (vb == c->M) TRY(dev_alloc(&c->stats_trial, (size_t)vb * BALM_STATS_STRIDE));
  TRY(dev_alloc(&c->vsums, (size_t)vb * 10));
  if (c->prec == BALM_PREC_FP64) {  // the tensor path writes int8 digit planes directly and never stores fp64 G'
    TRY(dev_alloc(&c->G, (size_t)3 * vb * c->ldg));
    CUDA_TRY(cudaMemsetAsync(c->G, 0, sizeof(double) * (size_t)3 * vb * c->ldg, c->stream));  // zero the column padding
  }
  if (blocks) TRY(dev_alloc(&c->G, (size_t)18 * c->K));
  const int tiles_p = (c->N + 31) / 32;
  c->obs_chunks = std::max(1, (c->sm_count * 16 + tiles_p - 1) / tiles_p);
  if (c->obs_chunks > 4096) c->obs_chunks = 4096;
  TRY(dev_alloc(&c->obs_part, (size_t)c->obs_chunks * BALM_ACC * c->Np));
  CUDA_TRY(cudaMemsetAsync(c->obs_part, 0, sizeof(double) * (size_t)c->obs_chunks * BALM_ACC * c->Np, c->stream));
  if (blocks) return block_hessian_build(c, "blocks registration");
  // SYRK work decomposition: (tile, k-split) items, sized so the last wave is nearly full
  c->syrk_nb = c->ldg / BALM_SYRK_TILE;
  c->syrk_tiles = c->syrk_nb * (c->syrk_nb + 1) / 2;
  const int64_t rows = 3 * vb;
  int max_splits = (int)std::max<int64_t>(1, std::min<int64_t>(rows / 512, 64));
  const size_t part_budget = (size_t)3 << 30;
  const size_t per_split = (size_t)c->syrk_tiles * BALM_SYRK_TILE * BALM_SYRK_TILE * sizeof(double);
  max_splits = (int)std::max<size_t>(1, std::min<size_t>(max_splits, part_budget / per_split));
  int best = 1;
  double best_eff = 0;
  // every split costs one fp64 partial tile per output tile (written by the SYRK epilogue, read by the assembly):
  // the tensor path (the faster SYRK, where the partial tiles weigh more) takes the SMALLEST split count that keeps the
  // last wave >= 95 % full and respects the int32 exactness bound (<= BALM_TC_MAX_ROWS_PER_ITEM = 32704 contraction
  // rows per item); the fp64 path maximises balance. As 32704 is a multiple of 64, s >= rows / 32704 splits keep every
  // item's rows, ceil(rows rounded up to 64 / s) rounded up to 64, within the bound.
  const int min_splits = c->prec == BALM_PREC_TENSOR
                             ? (int)((rows + BALM_TC_MAX_ROWS_PER_ITEM - 1) / BALM_TC_MAX_ROWS_PER_ITEM) : 1;
  const int items_per_tile = c->prec == BALM_PREC_TENSOR ? 2 : 1;  // the tensor SYRK computes a tile in two column halves
  for (int s = std::min(min_splits, max_splits); s <= max_splits; s++) {
    const int items = c->syrk_tiles * items_per_tile * s;
    const int waves = (items + c->sm_count - 1) / c->sm_count;
    const double eff = (double)items / ((double)waves * c->sm_count);
    if (c->prec == BALM_PREC_TENSOR) {
      if (eff > best_eff) { best_eff = eff; best = s; }
      if (eff >= 0.95) break;
    } else if (eff > best_eff + 0.02) {
      best_eff = eff;
      best = s;
    }
  }
  c->syrk_splits = best;
  TRY(dev_alloc(&c->syrk_part, (size_t)best * c->syrk_tiles * BALM_SYRK_TILE * BALM_SYRK_TILE));
  if (c->prec == BALM_PREC_TENSOR) TRY(tensor_syrk_init(c));
  return BALM_OK;
}

// A blocks context whose workspaces or pattern could not be built is left without a registration.
static int alloc_workspaces(balm_ctx *c) {
  const int rc = alloc_workspaces_of(c);
  if (rc != BALM_OK && c->prec == BALM_PREC_BLOCKS) free_problem(c);
  return rc;
}

// ---------------- ctx ----------------
// balm_create after its argument checks: c's streams, buffers and events (balm_destroy frees a partial c)
static int ctx_init(balm_ctx *c, int n_poses, int device, int precision);

extern "C" int balm_create(balm_ctx **out, int n_poses, int device, int precision) {
  if (!out || n_poses < 1) { balm_set_error("balm_create: bad arguments"); return BALM_ERR_INVALID; }
  if (precision != BALM_PREC_FP64 && precision != BALM_PREC_TENSOR && precision != BALM_PREC_BLOCKS) {
    balm_set_error("balm_create: unknown precision mode");
    return BALM_ERR_INVALID;
  }
  int ndev = 0;
  CUDA_TRY(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) { balm_set_error("balm_create: no such CUDA device"); return BALM_ERR_CUDA; }
  CUDA_TRY(cudaSetDevice(device));
  balm_ctx *c = new balm_ctx();
  const int rc = ctx_init(c, n_poses, device, precision);
  if (rc != BALM_OK) {
    balm_destroy(c);
    return rc;
  }
  *out = c;
  return BALM_OK;
}

static int ctx_init(balm_ctx *c, int n_poses, int device, int precision) {
  c->N = n_poses; c->n = 6 * n_poses; c->device = device; c->prec = precision;
  c->ldg = (c->n + BALM_SYRK_TILE - 1) / BALM_SYRK_TILE * BALM_SYRK_TILE;
  c->Np = (n_poses + 31) / 32 * 32;
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  c->sm_count = prop.multiProcessorCount;
  if (precision == BALM_PREC_TENSOR && getenv("BALM_TC_TRACE"))
    TRY(dev_alloc(&c->tc_trace, (size_t)c->sm_count * (BALM_TC_TRACE_WORDS + BALM_TC_COPY_TRACE_WORDS)));
  if (const char *e = getenv("BALM_TC_TILE"))  // tensor SYRK items: column halves or whole tiles (launch_syrk_tc)
    c->tc_tile = !strcmp(e, "half") ? 1 : !strcmp(e, "full") ? 2 : 0;
  int prio_least = 0, prio_greatest = 0;
  CUDA_TRY(cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest));
  CUDA_TRY(cudaStreamCreateWithPriority(&c->stream, cudaStreamNonBlocking, prio_greatest));
  TRY(factor_kernels_setup());
  TRY(syrk_f64_setup());
  TRY(ldlt_setup());
  TRY(covariance_setup());
  TRY(pose_graph_setup());
  const size_t n = c->n;
  TRY(dev_alloc(&c->poses, 12 * (size_t)c->N));
  TRY(dev_alloc(&c->poses_trial, 12 * (size_t)c->N));
  if (precision == BALM_PREC_BLOCKS) {  // nothing of size n^2
    TRY(dev_alloc(&c->g, n + 8));
  } else {
    TRY(dev_alloc(&c->H, n * n + n + 8));
    c->g = c->H + n * n;
    TRY(dev_alloc(&c->A, n * n));
  }
  TRY(dev_alloc(&c->dx, n));
  TRY(dev_alloc(&c->dvec, n));
  TRY(dev_alloc(&c->scal, 32));
  TRY(dev_alloc(&c->flags, 8));
  TRY(dev_alloc(&c->planes, 2 * (size_t)c->N));
  TRY(dev_alloc(&c->accum, (size_t)BALM_ACC * c->Np));
  TRY(dev_alloc(&c->accum_batch, (size_t)BALM_ACC * c->Np));
  // stats pass grids: voxel_sums_kernel up to 3 CTAs x 8 warps per SM, voxel_eig_kernel up to res_blocks CTAs (one
  // residual partial each)
  c->res_blocks = c->sm_count * 24;
  TRY(dev_alloc(&c->res_part, (size_t)c->res_blocks));
  CUDA_TRY(cudaMallocHost((void **)&c->h_scal, 16 * sizeof(double)));
  CUDA_TRY(cudaMallocHost((void **)&c->h_flags, 8 * sizeof(int)));
  memset(c->h_flags, 0, 8 * sizeof(int));
  for (auto &e : c->ev) CUDA_TRY(cudaEventCreate(&e));
  return BALM_OK;
}

extern "C" int balm_destroy(balm_ctx *c) {
  if (!c) return BALM_OK;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  free_problem(c);
  window_free(c->win);
  pose_graph_free(c->pg);
  prior_set_free(c->pr);
  rig_free(c->rig);
  if (c->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm);
  if (c->prec == BALM_PREC_BLOCKS) cudaFree(c->g);
  cudaFree(c->poses); cudaFree(c->poses_trial); cudaFree(c->H); cudaFree(c->A);
  cudaFree(c->dx); cudaFree(c->dvec); cudaFree(c->scal); cudaFree(c->flags); cudaFree(c->accum); cudaFree(c->accum_batch);
  cudaFree(c->vox_key); cudaFree(c->vox_layer); cudaFree(c->res_part); cudaFree(c->planes);
  ldlt_work_free(&c->lw);
  cudaFree(c->Hpack);
  cudaFree(c->joint_fg);
  cudaFree(c->tc_trace);
  cudaFreeHost(c->h_scal); cudaFreeHost(c->h_flags);
  for (auto &e : c->ev) if (e) cudaEventDestroy(e);
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;
  return BALM_OK;
}

// ---------------- problem registration ----------------
// One thread per voxel: checks the CSR invariants (pose_idx ascending, in range), finds the widest voxel and whether
// every voxel is observed by every pose; one thread per observation builds the per-pose voxel histogram
// (the ">= 20 planes per pose" precheck of bavoxel.hpp:1071-1085). Replaces a host loop over all K observations.
__global__ void csr_check_kernel(const long long *row_ptr, const int *pose_idx, int64_t M, int N, int *out /*[3]*/) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= M) return;
  const long long s0 = row_ptr[v], s1 = row_ptr[v + 1];
  const int k = (int)(s1 - s0);
  bool bad = (s1 < s0);
  int prev = -1;
  for (long long s = s0; s < s1; s++) {
    const int p = pose_idx[s];
    if (p <= prev || p >= N) bad = true;
    prev = p;
  }
  if (bad) atomicOr(&out[0], 1);
  if (k != N) atomicOr(&out[1], 1);  // not dense
  atomicMax(&out[2], k);
}
__global__ void pose_hist_kernel(const int *pose_idx, int64_t K, int N, int *planes) {
  extern __shared__ int hist[];
  for (int e = threadIdx.x; e < N; e += blockDim.x) hist[e] = 0;
  __syncthreads();
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < K; s += (int64_t)gridDim.x * blockDim.x) {
    const int p = pose_idx[s];
    if (p >= 0 && p < N) atomicAdd(&hist[p], 1);
  }
  __syncthreads();
  for (int e = threadIdx.x; e < N; e += blockDim.x)
    if (hist[e]) atomicAdd(&planes[e], hist[e]);
}
static int finish_registration(balm_ctx *c) {
  const int N = c->N;
  const int64_t M = c->M;
  int *d_out = nullptr, *d_planes = c->planes;  // c->planes [N]: per-pose voxel counts, kept for the collective guard
  TRY(dev_alloc(&d_out, 4));
  CUDA_TRY(cudaMemsetAsync(d_out, 0, sizeof(int) * 4, c->stream));
  CUDA_TRY(cudaMemsetAsync(d_planes, 0, sizeof(int) * N, c->stream));
  csr_check_kernel<<<(unsigned)((M + 127) / 128), 128, 0, c->stream>>>(c->row_ptr, c->pose_idx, M, N, d_out);
  if (sizeof(int) * N > 48 * 1024)  // a blocks context can hold more poses than the default shared-memory limit covers
    CUDA_TRY(cudaFuncSetAttribute(pose_hist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(int) * N));
  pose_hist_kernel<<<c->sm_count * 4, 256, sizeof(int) * N, c->stream>>>(c->pose_idx, c->K, N, d_planes);
  c->launches += 2;
  int h_out[4];
  std::vector<int> planes(N);
  CUDA_TRY(cudaMemcpyAsync(h_out, d_out, sizeof(int) * 4, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaMemcpyAsync(planes.data(), d_planes, sizeof(int) * N, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  cudaFree(d_out);
  if (h_out[0]) {
    free_problem(c);  // leave the context without a problem rather than with a malformed one
    balm_set_error("balm_set_voxels: pose_idx must be ascending and in [0,N) inside each voxel");
    return BALM_ERR_INVALID;
  }
  const bool dense = h_out[1] == 0;
  c->dense = dense;
  c->max_k = h_out[2];
  c->min_planes = *std::min_element(planes.begin(), planes.end());
  c->registered = true;
  if (!dense) TRY(build_pose_major_lists(c, planes.data()));  // pose-major lists for the observation sweep (device-built)
  return alloc_workspaces(c);
}

__global__ void aos_to_soa_kernel(const double *aos, double *soa, int64_t count, int64_t stride) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= count) return;
#pragma unroll
  for (int c = 0; c < 10; c++) soa[c * stride + s] = aos[s * 10 + c];
}
__global__ void soa_to_aos_kernel(const double *soa, double *aos, int64_t count, int64_t stride) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= count) return;
#pragma unroll
  for (int c = 0; c < 10; c++) aos[s * 10 + c] = soa[c * stride + s];
}

static int upload_aos(balm_ctx *c, const double *aos, bool aos_on_device, double *soa, int64_t count, int64_t stride) {
  // stage the AoS records through a device scratch buffer and transpose on the GPU
  const int64_t chunk = 1 << 22;
  double *scratch = nullptr;
  if (!aos_on_device) TRY(dev_alloc(&scratch, (size_t)std::min(chunk, count) * 10));
  for (int64_t b = 0; b < count; b += chunk) {
    const int64_t m = std::min(chunk, count - b);
    const double *src = aos + b * 10;
    if (!aos_on_device) {
      CUDA_TRY(cudaMemcpyAsync(scratch, src, sizeof(double) * m * 10, cudaMemcpyHostToDevice, c->stream));
      src = scratch;
    }
    aos_to_soa_kernel<<<(unsigned)((m + 255) / 256), 256, 0, c->stream>>>(src, soa + b, m, stride);
    c->launches++;
  }
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  cudaFree(scratch);
  return BALM_OK;
}

// An empty voxel set: evaluations give H = 0, g = 0, r = 0 (and still take part in the all-reduce).
static int register_empty(balm_ctx *c, const char *who = "blocks registration") {
  free_problem(c);
  CUDA_TRY(cudaMemsetAsync(c->planes, 0, sizeof(int) * c->N, c->stream));
  c->dense = true; c->max_k = 0; c->min_planes = 0; c->VB = 0;
  if (c->prec == BALM_PREC_BLOCKS) TRY(block_hessian_build(c, who));  // no term
  c->registered = true;
  return BALM_OK;
}

static double host_ms() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return 1e3 * ts.tv_sec + 1e-6 * ts.tv_nsec;
}

extern "C" int balm_set_voxels(balm_ctx *c, int64_t M, const int64_t *row_ptr, const int32_t *pose_idx,
                               const double *obs10, const double *fix10, const double *coe) {
  const bool trace = getenv("BALM_TRACE_REG") != nullptr;  // host-side stage times of the registration
  const double t_begin = host_ms();
  if (!c || M < 0 || !row_ptr || (M > 0 && (!pose_idx || !obs10 || !coe))) {
    balm_set_error("balm_set_voxels: bad arguments");
    return BALM_ERR_INVALID;
  }
  CUDA_TRY(cudaSetDevice(c->device));
  drop_keys(c);
  if (M == 0) return register_empty(c);  // a rank of a multi-GPU job whose shard holds no voxels still joins every collective
  const int64_t K = row_ptr[M];
  if (row_ptr[0] != 0 || K < M) { balm_set_error("balm_set_voxels: bad row_ptr"); return BALM_ERR_INVALID; }
  if (K >= ((int64_t)1 << 31)) { balm_set_error("balm_set_voxels: more than 2^31 observations per GPU"); return BALM_ERR_UNSUPPORTED; }
  TRY(alloc_problem_arrays(c, M, K, fix10 != nullptr));
  const bool reused = c->reuse_ws;
  const double t_alloc = host_ms();
  CUDA_TRY(cudaMemcpyAsync(c->row_ptr, row_ptr, sizeof(int64_t) * (M + 1), cudaMemcpyHostToDevice, c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->pose_idx, pose_idx, sizeof(int32_t) * K, cudaMemcpyHostToDevice, c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->coe, coe, sizeof(double) * M, cudaMemcpyHostToDevice, c->stream));
  if (trace) CUDA_TRY(cudaStreamSynchronize(c->stream));
  const double t_small = host_ms();
  TRY(upload_aos(c, obs10, false, c->obs, K, c->Kp));
  if (fix10) TRY(upload_aos(c, fix10, false, c->fix, M, M));
  const double t_obs = host_ms();
  const int rc = finish_registration(c);
  if (trace)
    fprintf(stderr, "[balm_set_voxels] reuse=%d alloc %.2f ms, csr+coe copies %.2f ms, observations %.2f ms, "
            "checks+workspaces %.2f ms\n", (int)reused, t_alloc - t_begin, t_small - t_alloc, t_obs - t_small,
            host_ms() - t_obs);
  return rc;
}

extern "C" int balm_set_voxels_dev(balm_ctx *c, int64_t M, const int64_t *row_ptr_dev, const int32_t *pose_idx_dev,
                                   const double *obs10_dev, const double *fix10_dev, const double *coe_dev,
                                   int64_t K) {
  if (!c || M < 1 || !row_ptr_dev || !pose_idx_dev || !obs10_dev || !coe_dev || K < M) {
    balm_set_error("balm_set_voxels_dev: bad arguments");
    return BALM_ERR_INVALID;
  }
  CUDA_TRY(cudaSetDevice(c->device));
  {  // the same checks the host path makes on row_ptr / K (the per-voxel invariants are checked by csr_check_kernel)
    int64_t ends[2] = {-1, -1};
    CUDA_TRY(cudaMemcpy(&ends[0], row_ptr_dev, sizeof(int64_t), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(&ends[1], row_ptr_dev + M, sizeof(int64_t), cudaMemcpyDeviceToHost));
    if (ends[0] != 0 || ends[1] != K) { balm_set_error("balm_set_voxels_dev: row_ptr[0] != 0 or row_ptr[M] != n_obs"); return BALM_ERR_INVALID; }
    if (K >= ((int64_t)1 << 31)) { balm_set_error("balm_set_voxels_dev: more than 2^31 observations per GPU"); return BALM_ERR_UNSUPPORTED; }
  }
  drop_keys(c);
  TRY(alloc_problem_arrays(c, M, K, fix10_dev != nullptr));
  CUDA_TRY(cudaMemcpyAsync(c->row_ptr, row_ptr_dev, sizeof(int64_t) * (M + 1), cudaMemcpyDeviceToDevice, c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->pose_idx, pose_idx_dev, sizeof(int32_t) * K, cudaMemcpyDeviceToDevice, c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->coe, coe_dev, sizeof(double) * M, cudaMemcpyDeviceToDevice, c->stream));
  TRY(upload_aos(c, obs10_dev, true, c->obs, K, c->Kp));
  if (fix10_dev) TRY(upload_aos(c, fix10_dev, true, c->fix, M, M));
  return finish_registration(c);
}

extern "C" int64_t balm_num_obs(balm_ctx *c) { return c ? c->K : 0; }

// ---------------- association on the GPU (assoc.cu) ----------------
extern "C" void balm_default_assoc_opts(balm_assoc_opts *o) {
  o->voxel_size = 1.0; o->layer_limit = 2; o->min_ps = 15;
  o->eigen_value_array[0] = o->eigen_value_array[1] = o->eigen_value_array[2] = 1.0 / 16;
}

// opts or the defaults, with the planarity thresholds rounded as the reference stores them: it keeps them in a
// `float eigen_value_array[]` (bavoxel.hpp:11) and compares the double ratio with the promoted float (bavoxel.hpp:697),
// so 1/9 is (double)(float)(1.0/9), not the double 1/9
balm_assoc_opts resolve_assoc_opts(const balm_assoc_opts *opts) {
  balm_assoc_opts o;
  if (opts) o = *opts; else balm_default_assoc_opts(&o);
  for (double &e : o.eigen_value_array) e = (double)(float)e;
  return o;
}

// BALM_ASSOC_BUDGET_MB (read at every call, default 16 GB): the association's device scratch
static size_t assoc_budget() {
  size_t budget = (size_t)16 << 30;
  if (const char *e = getenv("BALM_ASSOC_BUDGET_MB")) budget = (size_t)llround(std::max(0.0, atof(e)) * 1048576.0);
  return budget;
}

// The slab path's voxels, staged on the host, registered like the one-pass call's register step does it
static int register_slabs(balm_ctx *c, const SlabVoxels &V) {
  TRY(alloc_problem_arrays(c, V.M, V.K, false));
  drop_keys(c);
  TRY(dev_alloc(&c->vox_key, (size_t)V.M));
  TRY(dev_alloc(&c->vox_layer, (size_t)V.M));
  CUDA_TRY(cudaMemcpyAsync(c->row_ptr, V.row_ptr.data(), sizeof(long long) * (V.M + 1), cudaMemcpyHostToDevice, c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->pose_idx, V.pose_idx.data(), sizeof(int) * V.K, cudaMemcpyHostToDevice, c->stream));
  for (int col = 0; col < 10; col++)
    CUDA_TRY(cudaMemcpyAsync(c->obs + (size_t)col * c->Kp, V.obs[col].data(), sizeof(double) * V.K,
                             cudaMemcpyHostToDevice, c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->coe, V.coe.data(), sizeof(double) * V.M, cudaMemcpyHostToDevice, c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->vox_key, V.key.data(), sizeof(unsigned long long) * V.M, cudaMemcpyHostToDevice, c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->vox_layer, V.layer.data(), sizeof(int) * V.M, cudaMemcpyHostToDevice, c->stream));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  return BALM_OK;
}

extern "C" int balm_cut_voxels(balm_ctx *c, int64_t n_points, const float *xyz, const int32_t *frame,
                               const double *poses12, const balm_assoc_opts *opts, int64_t *n_voxels_out,
                               int64_t *n_obs_out) {
  if (!c || !xyz || !frame || !poses12) { balm_set_error("balm_cut_voxels: bad arguments"); return BALM_ERR_INVALID; }
  const balm_assoc_opts o = resolve_assoc_opts(opts);
  if (n_points < 1 || o.layer_limit < 0 || o.layer_limit > 2) {
    balm_set_error("balm_cut_voxels: bad arguments (n >= 1, layer_limit in 0..2)");
    return BALM_ERR_INVALID;
  }
  CUDA_TRY(cudaSetDevice(c->device));
  const double t0 = host_ms();
  const size_t budget = assoc_budget();
  const int64_t per_point = assoc_bytes_per_point(o.layer_limit), fixed = assoc_bytes_fixed(c->N);
  ScratchPool acct;  // counts the scratch of the whole call
  AssocStats ast;
  AssocInput in{"balm_cut_voxels", n_points, xyz, c->N, poses12, frame, 1, nullptr, nullptr, nullptr, n_points};
  in.outer = &acct;
  in.stats = &ast;
  int64_t st[BALM_CUT_STATS] = {1, n_points, 0, 0, 0, per_point, fixed, 0, 0, 0, 0};
  if (n_points < (1ll << 31) && (double)n_points * per_point + fixed <= (double)budget) {
    // one pass: register: allocate the problem arrays of the context and the voxel keys, which stay with it
    // (balm_append_scan / balm_marginalize need them)
    const AssocRegister reg = [c](int64_t M, int64_t K, const int64_t *, const int64_t *, AssocEmit *out) {
      if (M < 1) { balm_set_error("balm_cut_voxels: no plane voxels found"); return (int)BALM_ERR_INVALID; }
      TRY(alloc_problem_arrays(c, M, K, false));
      drop_keys(c);
      TRY(dev_alloc(&c->vox_key, (size_t)M));
      TRY(dev_alloc(&c->vox_layer, (size_t)M));
      *out = AssocEmit{c->obs, c->Kp, 1, c->pose_idx, c->row_ptr, c->coe, c->vox_key, c->vox_layer};
      return (int)BALM_OK;
    };
    TRY(assoc_cut(c->stream, in, o, reg, &c->launches));
    st[2] = ast.roots;
    st[4] = ast.h2d_bytes;
    st[9] = (int64_t)(1e3 * (host_ms() - t0));
  } else {
    // root-key slabs of at most cap points, each within the budget
    const int64_t cap = std::min<int64_t>(std::max<int64_t>(0, ((int64_t)budget - fixed) / per_point), INT_MAX);
    SlabVoxels V;
    CutSlabStats S;
    TRY(assoc_cut_slabs(c->stream, in, o, budget, cap, acct, &V, &S, &c->launches));
    if (V.M < 1) { balm_set_error("balm_cut_voxels: no plane voxels found"); return BALM_ERR_INVALID; }
    if (V.K >= ((int64_t)1 << 31)) {
      balm_set_error("balm_cut_voxels: more than 2^31 observations per GPU");
      return BALM_ERR_UNSUPPORTED;
    }
    const double t1 = host_ms();
    TRY(register_slabs(c, V));
    st[0] = S.slabs; st[1] = S.max_slab; st[2] = S.roots; st[4] = S.h2d_bytes + V.K * 84 + V.M * 28 + 8;
    st[7] = (int64_t)(1e3 * S.ms_roots); st[8] = (int64_t)(1e3 * S.ms_select); st[9] = (int64_t)(1e3 * S.ms_cut);
    st[10] = (int64_t)(1e3 * (host_ms() - t1));
  }
  c->has_keys = true;
  c->assoc = o;
  if (n_voxels_out) *n_voxels_out = c->M;
  if (n_obs_out) *n_obs_out = c->K;
  st[3] = (int64_t)acct.peak;
  const double t2 = host_ms();
  const int rc = finish_registration(c);
  st[10] += (int64_t)(1e3 * (host_ms() - t2));
  if (rc == BALM_OK) memcpy(c->cut_stats, st, sizeof(st));
  return rc;
}

extern "C" int balm_cut_voxels_stats(balm_ctx *c, int64_t *stats) {
  if (!c || !stats) { balm_set_error("balm_cut_voxels_stats: bad arguments"); return BALM_ERR_INVALID; }
  memcpy(stats, c->cut_stats, sizeof(c->cut_stats));
  return BALM_OK;
}

extern "C" int balm_download_voxel_range(balm_ctx *c, int64_t head, int64_t end, int64_t *row_ptr, int32_t *pose_idx,
                                         double *obs10, double *coe, int64_t *n_obs_out) {
  if (!c || !c->obs) { balm_set_error("balm_download_voxels: no voxels registered"); return BALM_ERR_INVALID; }
  if (head < 0 || end > c->M || head > end) { balm_set_error("balm_download_voxel_range: bad voxel range"); return BALM_ERR_INVALID; }
  CUDA_TRY(cudaSetDevice(c->device));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  int64_t s0 = 0, s1 = 0;
  CUDA_TRY(cudaMemcpy(&s0, c->row_ptr + head, sizeof(int64_t), cudaMemcpyDeviceToHost));
  CUDA_TRY(cudaMemcpy(&s1, c->row_ptr + end, sizeof(int64_t), cudaMemcpyDeviceToHost));
  const int64_t K = s1 - s0;
  if (n_obs_out) *n_obs_out = K;
  if (row_ptr) {  // re-based to 0, like a freshly registered problem of end-head voxels
    CUDA_TRY(cudaMemcpy(row_ptr, c->row_ptr + head, sizeof(int64_t) * (end - head + 1), cudaMemcpyDeviceToHost));
    for (int64_t v = 0; v <= end - head; v++) row_ptr[v] -= s0;
  }
  if (pose_idx && K) CUDA_TRY(cudaMemcpy(pose_idx, c->pose_idx + s0, sizeof(int32_t) * K, cudaMemcpyDeviceToHost));
  if (coe && end > head) CUDA_TRY(cudaMemcpy(coe, c->coe + head, sizeof(double) * (end - head), cudaMemcpyDeviceToHost));
  if (obs10 && K) {
    const int64_t chunk = 1 << 22;
    double *scratch = nullptr;
    TRY(dev_alloc(&scratch, (size_t)std::min(chunk, K) * 10));
    for (int64_t b = 0; b < K; b += chunk) {
      const int64_t m = std::min(chunk, K - b);
      soa_to_aos_kernel<<<(unsigned)((m + 255) / 256), 256, 0, c->stream>>>(c->obs + s0 + b, scratch, m, c->Kp);
      CUDA_TRY(cudaMemcpyAsync(obs10 + b * 10, scratch, sizeof(double) * m * 10, cudaMemcpyDeviceToHost, c->stream));
      CUDA_TRY(cudaStreamSynchronize(c->stream));
    }
    cudaFree(scratch);
  }
  return BALM_OK;
}

extern "C" int balm_download_voxels(balm_ctx *c, int64_t *row_ptr, int32_t *pose_idx, double *obs10, double *coe) {
  if (!c || !c->obs) { balm_set_error("balm_download_voxels: no voxels registered"); return BALM_ERR_INVALID; }
  return balm_download_voxel_range(c, 0, c->M, row_ptr, pose_idx, obs10, coe, nullptr);
}

extern "C" int balm_synth_virtual(balm_ctx *c, int64_t M, int64_t first_voxel, int pts, double noise, double range,
                                  uint64_t seed, double *poses_gt, double *poses_init) {
  if (!c || M < 1 || pts < 1) { balm_set_error("balm_synth_virtual: bad arguments"); return BALM_ERR_INVALID; }
  CUDA_TRY(cudaSetDevice(c->device));
  const int64_t K = M * c->N;
  if (K >= ((int64_t)1 << 31)) { balm_set_error("balm_synth_virtual: more than 2^31 observations per GPU"); return BALM_ERR_UNSUPPORTED; }
  std::vector<double> gt(12 * (size_t)c->N), init(12 * (size_t)c->N);
  synth_host_poses(c->N, seed, gt.data(), init.data());
  if (poses_gt) memcpy(poses_gt, gt.data(), sizeof(double) * gt.size());
  if (poses_init) memcpy(poses_init, init.data(), sizeof(double) * init.size());
  drop_keys(c);
  TRY(alloc_problem_arrays(c, M, K, false));
  CUDA_TRY(cudaMemcpyAsync(c->poses_trial, gt.data(), sizeof(double) * gt.size(), cudaMemcpyHostToDevice, c->stream));
  TRY(launch_synth(c, M, first_voxel, pts, noise, range, seed, c->poses_trial));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  c->dense = true;
  c->max_k = c->N;
  c->min_planes = (int)std::min<int64_t>(M, 1 << 30);
  {
    std::vector<int> pl((size_t)c->N, c->min_planes);
    CUDA_TRY(cudaMemcpy(c->planes, pl.data(), sizeof(int) * c->N, cudaMemcpyHostToDevice));
  }
  c->registered = true;
  return alloc_workspaces(c);
}

// ---------------- evaluation ----------------
// Multi-GPU reduction of [H | g | r]: H is symmetric, so only its lower triangle travels. With a communicator attached the
// assembly kernel writes column c of the lower triangle (n - c entries) at offset c*n - c(c-1)/2 of the send buffer,
// followed by g and r, INSTEAD of the full matrix; after the all-reduce unpack_lower_kernel writes H (both halves), g and
// r. 36 MB instead of 72 MB on the wire at N = 500, and no extra pass over the matrix.
__global__ void unpack_lower_kernel(const double *pack, double *H, int n) {
  __shared__ double tile[32][33];
  const int bc = blockIdx.y, br = blockIdx.x;  // 32 x 32 block (block row br >= block column bc)
  if (br < bc) return;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int r = br * 32 + tx, c = bc * 32 + ty;
  const size_t tri = (size_t)n * (n + 1) / 2;
  double v = 0.0;
  if (r < n && c < n && r >= c) {
    v = pack[(size_t)c * n - (size_t)c * (c - 1) / 2 + (r - c)];
    H[(size_t)c * n + r] = v;                      // lower element, coalesced in r
  }
  tile[ty][tx] = v;
  __syncthreads();
  const int r2 = br * 32 + ty, c2 = bc * 32 + tx;  // transposed read: upper element (row c2, col r2), coalesced in c2
  if (r2 < n && c2 < n && r2 > c2) H[(size_t)r2 * n + c2] = tile[tx][ty];
  if (br == 0 && bc == 0) {
    for (int e = ty * 32 + tx; e <= n; e += 1024) H[(size_t)n * n + e] = pack[tri + e];
  }
}

static int allreduce_sum(balm_ctx *c, double *buf, size_t count) {
  if (c->world <= 1 || !c->comm) return BALM_OK;
  const int rc = g_nccl.AllReduce(buf, buf, count, /*ncclFloat64*/ 8, /*ncclSum*/ 0, c->comm, c->stream);
  if (rc != 0) {
    balm_set_error(std::string("ncclAllReduce: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "?"));
    return BALM_ERR_NCCL;
  }
  return BALM_OK;
}

// The registered pose factors and priors join the full-range voxel cost: always on a blocks context, on a dense one
// while balm_set_joint_cost is on. The sum is voxels, then factors, then priors.
static bool pose_terms_in_cost(const balm_ctx *c) { return c->prec == BALM_PREC_BLOCKS || c->joint_cost; }

// H, g, r of voxels [head,end) at device poses `poses`; result in c->H | c->g | c->scal[0] (all-reduced).
// stats_cached: c->stats already holds the per-voxel eigen data of exactly these poses (left there by the residual
// pass of an accepted LM step, or by the evaluation before a rejected one) and c->scal[BALM_SCAL_RCUR] this rank's residual.
static int evaluate_dev(balm_ctx *c, const double *poses, int64_t head, int64_t end, bool include_fix,
                        bool stats_cached = false) {
  if (!c->registered) { balm_set_error("no voxels registered"); return BALM_ERR_INVALID; }
  if (head < 0 || end > c->M || head > end) { balm_set_error("evaluate: bad voxel range"); return BALM_ERR_INVALID; }
  double *r_dev = c->g + c->n;  // contiguous with H and g -> one all-reduce
  float ms;
  bool first = true;
  // defer mode (LM loop, whole problem in one batch): nothing is waited for here; collect_eval() reads the events and
  // the tensor path's flags after the iteration's single synchronisation. A blocks context without voxels (the sparse
  // pose graph) defers too: its full range is the factors and priors.
  const bool deferred = c->defer && head == 0 && end == c->M && c->VB >= c->M &&
                        (end > head || c->prec == BALM_PREC_BLOCKS);
  // the pose factors of a blocks context, or of a dense one with the joint cost, are part of every full-range evaluation
  // (sub-ranges stay voxels only)
  const bool factors = pose_terms_in_cost(c) && c->pg && head == 0 && end == c->M;
  const bool priors = pose_terms_in_cost(c) && c->pr && head == 0 && end == c->M;  // so are its pose priors
  c->pending_stats_cached = stats_cached;
  if (head == end) {  // empty range (or an empty shard): this rank contributes H = 0, g = 0, r = 0 -- and still enters
    // the all-reduce below, which the other ranks of a multi-GPU job are waiting in
    if (c->prec == BALM_PREC_BLOCKS) {
      TRY(blocks_zero(c));
    } else {
      CUDA_TRY(cudaMemsetAsync(c->H, 0, sizeof(double) * ((size_t)c->n * c->n + c->n + 1), c->stream));
    }
  } else {
    CUDA_TRY(cudaMemsetAsync(r_dev, 0, sizeof(double), c->stream));
  }
  for (int64_t v0 = head; v0 < end; v0 += c->VB) {
    const int64_t v1 = std::min(end, v0 + c->VB);
    TRY(launch_csc_batch(c, v0, v1));  // sparse problems: every pose's list restricted to this batch's voxels
    CUDA_TRY(cudaEventRecord(c->ev[0], c->stream));
    if (stats_cached) CUDA_TRY(cudaMemcpyAsync(r_dev, c->scal + BALM_SCAL_RCUR, sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    else TRY(launch_voxel_stats(c, poses, v0, v1, c->stats, include_fix, r_dev));
    CUDA_TRY(cudaEventRecord(c->ev[1], c->stream));
    if (c->prec == BALM_PREC_TENSOR) {
      TRY(tensor_obs_and_syrk(c, poses, v0, v1, first));  // records ev[2] between the sweeps and the SYRK
    } else {
      TRY(launch_obs_pass(c, poses, v0, v1, first));
      CUDA_TRY(cudaEventRecord(c->ev[2], c->stream));
      if (c->prec == BALM_PREC_BLOCKS) TRY(launch_blocks(c, v0, v1));  // single batch: the blocks and g, no assembly
      else TRY(launch_syrk_f64(c, 3 * (v1 - v0), first));
    }
    CUDA_TRY(cudaEventRecord(c->ev[3], c->stream));
    if (deferred) {
      if (c->prec == BALM_PREC_TENSOR) TRY(tensor_syrk_check_enqueue(c));
    } else {
      CUDA_TRY(cudaEventSynchronize(c->ev[3]));
      cudaEventElapsedTime(&ms, c->ev[0], c->ev[1]);
      if (!stats_cached) { c->tm.ms_stats += ms; if (first) c->tm.n_stats += 1; }
      cudaEventElapsedTime(&ms, c->ev[1], c->ev[2]); c->tm.ms_obs += ms;
      cudaEventElapsedTime(&ms, c->ev[2], c->ev[3]); c->tm.ms_syrk += ms;
      if (c->prec == BALM_PREC_TENSOR) TRY(tensor_syrk_check(c));
    }
    first = false;
  }
  if (end > head)  // local, pre all-reduce; the hand-over needs every voxel, so an empty range hands nothing over
    CUDA_TRY(cudaMemcpyAsync(c->scal + BALM_SCAL_RCUR, r_dev, sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
  CUDA_TRY(cudaEventRecord(c->ev[4], c->stream));
  if (end > head && c->prec != BALM_PREC_BLOCKS) TRY(launch_assemble(c));
  if (c->prec == BALM_PREC_BLOCKS) {  // after the RCUR copy above: the hand-over caches voxels only
    if (factors) TRY(blocks_add_factors(c, poses));
    if (priors) TRY(blocks_add_priors(c, poses));
  } else {
    if (factors) TRY(joint_add_factors(c, poses));
    if (priors) TRY(prior_add_dense(c->pr, c->stream, poses, c->H, c->n, c->g, r_dev, &c->launches));
  }
  CUDA_TRY(cudaEventRecord(c->ev[5], c->stream));
  if (c->world > 1 && c->comm) {  // the assembly wrote the lower triangle | g into c->Hpack (an empty range: zeros)
    const int n = c->n;
    const size_t tri = (size_t)n * (n + 1) / 2, cnt = tri + n + 1;
    if (end > head) CUDA_TRY(cudaMemcpyAsync(c->Hpack + tri + n, r_dev, sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    else CUDA_TRY(cudaMemsetAsync(c->Hpack, 0, sizeof(double) * cnt, c->stream));
    TRY(allreduce_sum(c, c->Hpack, cnt));
    unpack_lower_kernel<<<dim3((n + 31) / 32, (n + 31) / 32), dim3(32, 32), 0, c->stream>>>(c->Hpack, c->H, n);
    c->launches += 1;
  }
  CUDA_TRY(cudaEventRecord(c->ev[6], c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->scal, r_dev, sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
  if (deferred) {
    c->pending_eval = true;
    return BALM_OK;
  }
  CUDA_TRY(cudaEventSynchronize(c->ev[6]));
  cudaEventElapsedTime(&ms, c->ev[4], c->ev[5]);
  if (c->prec != BALM_PREC_BLOCKS || factors || priors) c->tm.ms_assemble += ms;
  cudaEventElapsedTime(&ms, c->ev[5], c->ev[6]); c->tm.ms_allreduce += ms;
  c->tm.n_eval += 1;
  return BALM_OK;
}

// defer mode: the stream has been synchronised -> account the evaluation's phases, read the tensor path's flags
static int collect_eval(balm_ctx *c) {
  if (!c->pending_eval) return BALM_OK;
  c->pending_eval = false;
  float ms;
  if (c->M > 0) {  // deferred evaluations are full-range: the voxel phases ran (a voxel-free blocks context has none)
    cudaEventElapsedTime(&ms, c->ev[0], c->ev[1]);
    if (!c->pending_stats_cached) { c->tm.ms_stats += ms; c->tm.n_stats += 1; }
    cudaEventElapsedTime(&ms, c->ev[1], c->ev[2]); c->tm.ms_obs += ms;
    cudaEventElapsedTime(&ms, c->ev[2], c->ev[3]); c->tm.ms_syrk += ms;
  }
  cudaEventElapsedTime(&ms, c->ev[4], c->ev[5]);
  if (c->prec != BALM_PREC_BLOCKS || c->pg || c->pr) c->tm.ms_assemble += ms;  // deferred: always full range
  cudaEventElapsedTime(&ms, c->ev[5], c->ev[6]); c->tm.ms_allreduce += ms;
  c->tm.n_eval += 1;
  if (c->prec == BALM_PREC_TENSOR) return tensor_syrk_check_finish(c);
  return BALM_OK;
}

static int residual_dev(balm_ctx *c, const double *poses, double *host_out, bool keep_stats = false) {
  if (!c->registered) { balm_set_error("no voxels registered"); return BALM_ERR_INVALID; }
  double *r_dev = c->scal + 2;
  CUDA_TRY(cudaEventRecord(c->ev[7], c->stream));
  CUDA_TRY(cudaMemsetAsync(r_dev, 0, sizeof(double), c->stream));
  TRY(launch_voxel_stats(c, poses, 0, c->M, keep_stats ? c->stats_trial : nullptr, true, r_dev));
  CUDA_TRY(cudaMemcpyAsync(c->scal + BALM_SCAL_RTRIAL, r_dev, sizeof(double), cudaMemcpyDeviceToDevice, c->stream));  // local, pre all-reduce
  if (pose_terms_in_cost(c) && c->pg) {  // after RTRIAL: voxels only
    if (c->prec == BALM_PREC_BLOCKS) TRY(blocks_add_factor_cost(c, poses, r_dev));
    else TRY(joint_add_factor_cost(c, poses, r_dev));
  }
  if (pose_terms_in_cost(c) && c->pr) TRY(prior_add_cost(c->pr, c->stream, poses, r_dev, &c->launches));
  TRY(allreduce_sum(c, r_dev, 1));
  CUDA_TRY(cudaEventRecord(c->ev[8], c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->h_scal + 2, r_dev, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  float ms;
  cudaEventElapsedTime(&ms, c->ev[7], c->ev[8]);
  c->tm.ms_residual += ms;
  c->tm.n_residual += 1;
  *host_out = c->h_scal[2];
  return BALM_OK;
}

// ---------------- the unknowns of a call ----------------
// What an evaluation, LM loop or covariance solves for: the context's N slot poses (rig null), or a rig's free base
// poses and extrinsics, composed to slot poses before every evaluation, with H and g reduced to H_rig and g_rig after
// it. Everything else (the dense or sparse solve, the LM rule, the undamped factor, the covariance algebra) is the same
// for both, so these functions are the only code that tells them apart. pose_terms (the dense pose-graph calls, rig
// null) costs the slot poses by the context's pose factors and priors instead of its voxels.
struct Unknowns {
  balm_ctx *c;
  Rig *rig;
  bool pose_terms = false;

  bool sparse() const { return rig ? rig_sparse(rig) : c->prec == BALM_PREC_BLOCKS; }
  DenseSystem system() const { return rig ? rig_system(rig) : ctx_system(c); }
  // the sparse solver of a blocks context or a block-sparse rig, else null (the dense solve of system())
  SparseSolver *solver() const {
    if (!sparse()) return nullptr;
    return rig ? rig_solver(rig) : blocks_solver(c->bh);
  }
  // a sparse one's block pairs and their device blocks
  const std::vector<int2> &pairs() const { return rig ? rig_pairs(rig) : blocks_pairs(c->bh); }
  const double *blocks() const { return rig ? rig_blocks(rig) : blocks_device(c->bh); }
  // the current state: the slot poses, or the base poses then the extrinsics; 12 doubles per pose
  double *state() const { return rig ? rig_state(rig, false) : c->poses; }
  int n_state() const { return rig ? rig_bases(rig) + rig_lidars(rig) : c->N; }
  // a covariance's anchor: -1, or a pose, or a free base pose (`who` prefixes the message)
  int check_anchor(const char *who, int anchor) const {
    if (anchor >= -1 && anchor < (rig ? rig_free_bases(rig) : c->N)) return BALM_OK;
    if (rig)
      balm_set_error(std::string(who) + ": anchor " + std::to_string(anchor) + " is neither -1 nor a free base index in [0, " +
                     std::to_string(rig_free_bases(rig)) + ")");
    else
      balm_set_error(std::string(who) + ": anchor outside [-1, N)");
    return BALM_ERR_INVALID;
  }

  // x12 (the slot poses, or a rig's base poses) and ext12 (a rig's extrinsics) in or out of the current state
  int upload(const double *x12, const double *ext12) const {
    const size_t nx = 12 * (size_t)(rig ? rig_bases(rig) : c->N);
    CUDA_TRY(cudaMemcpyAsync(state(), x12, sizeof(double) * nx, cudaMemcpyHostToDevice, c->stream));
    if (rig)
      CUDA_TRY(cudaMemcpyAsync(state() + nx, ext12, sizeof(double) * 12 * rig_lidars(rig), cudaMemcpyHostToDevice, c->stream));
    return BALM_OK;
  }
  int download(double *x12, double *ext12) const {
    const size_t nx = 12 * (size_t)(rig ? rig_bases(rig) : c->N);
    CUDA_TRY(cudaMemcpyAsync(x12, state(), sizeof(double) * nx, cudaMemcpyDeviceToHost, c->stream));
    if (rig)
      CUDA_TRY(cudaMemcpyAsync(ext12, state() + nx, sizeof(double) * 12 * rig_lidars(rig), cudaMemcpyDeviceToHost, c->stream));
    return BALM_OK;
  }
  // the slot poses of the current state in c->poses
  int compose() const { return rig ? rig_compose(rig, c->stream, state(), c->poses, &c->launches) : BALM_OK; }
  // evaluate_dev at the current state: H, g and the residual in c->scal[0], then a rig's H_rig and g_rig (the
  // reduction timed by ev[13] and ev[14]); with a blocks context, its slot blocks, factors and priors first. Pose terms:
  // pose_graph_eval, the factors' and priors' H, g and cost, no voxels (the other arguments are unused)
  int eval(bool include_fix, int64_t head, int64_t end, bool stats_cached = false) const {
    if (pose_terms) return pose_graph_eval(c, c->poses);
    TRY(compose());
    TRY(evaluate_dev(c, c->poses, head, end, include_fix, stats_cached));
    if (!rig) return BALM_OK;
    CUDA_TRY(cudaEventRecord(c->ev[13], c->stream));
    if (rig_sparse(rig)) TRY(rig_reduce_blocks(rig, c->stream, state(), blocks_device(c->bh), c->g, &c->launches));
    else TRY(rig_reduce(rig, c->stream, state(), c->H, c->g, &c->launches));
    CUDA_TRY(cudaEventRecord(c->ev[14], c->stream));
    return BALM_OK;
  }
  // after an eval, once the stream has been waited for: its accounting (collect_eval), a rig's reduction in ms_assemble
  int collect() const {
    TRY(collect_eval(c));
    if (rig) {
      float ms;
      CUDA_TRY(cudaEventElapsedTime(&ms, c->ev[13], c->ev[14]));
      c->tm.ms_assemble += ms;
    }
    return BALM_OK;
  }
  // the raw term R (6N x 6N, at the slot poses) in these unknowns: R itself, or a rig's J^T R J (taken from pool)
  int reduce_raw(ScratchPool &pool, double **R) const {
    if (!rig) return BALM_OK;
    double *out = nullptr;
    TRY(pool.get(&out, (size_t)rig_n(rig) * rig_n(rig)));
    TRY(rig_reduce_raw(rig, c->stream, state(), *R, out, &c->launches));
    *R = out;
    return BALM_OK;
  }
  // the LM trial state from system()'s dx, its slot poses in c->poses_trial; accept() makes it the current state
  int trial() const {
    if (!rig) return launch_pose_update(c, c->poses, c->dx, c->poses_trial);
    TRY(rig_update(rig, c->stream, state(), rig_state(rig, true), &c->launches));
    return rig_compose(rig, c->stream, rig_state(rig, true), c->poses_trial, &c->launches);
  }
  // the cost at c->poses_trial into *r2, once the stream has been waited for: residual_dev (keep_stats: its per-voxel
  // stats kept for a hand-over), or the pose factors' then the priors' cost in scal[2]
  int trial_cost(bool keep_stats, double *r2) const {
    if (!pose_terms) return residual_dev(c, c->poses_trial, r2, keep_stats);
    TRY(pose_graph_cost(c->pg, c->stream, c->poses_trial, c->scal + 2, &c->launches));
    if (c->pr) TRY(prior_add_cost(c->pr, c->stream, c->poses_trial, c->scal + 2, &c->launches));
    CUDA_TRY(cudaMemcpyAsync(c->h_scal + 2, c->scal + 2, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    *r2 = c->h_scal[2];
    return BALM_OK;
  }
  void accept() const {
    if (rig) rig_swap_states(rig);
    else std::swap(c->poses, c->poses_trial);
  }
  // gauge modes 0 and 1: the poses re-anchored to pose 0, or a rig's base poses to base 0 (extrinsics are body-frame)
  int gauge(int mode) const {
    c->launches += 1;
    return launch_gauge(c->stream, rig ? rig_bases(rig) : c->N, state(), c->scal + 4, mode);  // pose 0 into scal[4..15]
  }
};

// The n x n matrix of a block-sparse H (or H_rig), column-major, from its pairs and device blocks, zeros elsewhere, on
// the host (waits).
static int blocks_to_dense(balm_ctx *c, const std::vector<int2> &pr, const double *blocks, size_t n, double *H) {
  std::vector<double> b(36 * pr.size());
  CUDA_TRY(cudaMemcpyAsync(b.data(), blocks, sizeof(double) * b.size(), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  std::fill(H, H + n * n, 0.0);
  for (size_t p = 0; p < pr.size(); p++)
    for (int col = 0; col < 6; col++)
      for (int row = 0; row < 6; row++) {
        const double h = b[36 * p + 6 * col + row];
        const size_t r = 6 * (size_t)pr[p].x + row, cc = 6 * (size_t)pr[p].y + col;
        H[cc * n + r] = h;
        H[r * n + cc] = h;
      }
  return BALM_OK;
}

// balm_evaluate, balm_rig_evaluate and balm_pose_graph_evaluate after their checks: H (dense, expanded from blocks), g
// and the residual of voxels [head, end) (or the pose terms' cost) at x12 / ext12
static int evaluate(const Unknowns &u, const double *x12, const double *ext12, int64_t head, int64_t end,
                    bool include_fix, double *H, double *g, double *residual) {
  balm_ctx *c = u.c;
  CUDA_TRY(cudaSetDevice(c->device));
  TRY(u.upload(x12, ext12));
  TRY(u.eval(include_fix, head, end));
  const DenseSystem sys = u.system();
  const size_t n = sys.n;
  if (H && u.sparse()) TRY(blocks_to_dense(c, u.pairs(), u.blocks(), n, H));
  else if (H) CUDA_TRY(cudaMemcpyAsync(H, sys.H, sizeof(double) * n * n, cudaMemcpyDeviceToHost, c->stream));
  if (g) CUDA_TRY(cudaMemcpyAsync(g, sys.g, sizeof(double) * n, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->h_scal, c->scal, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  TRY(u.collect());
  if (residual) *residual = c->h_scal[0];
  return BALM_OK;
}

extern "C" int balm_evaluate(balm_ctx *c, const double *poses12, int64_t head, int64_t end, int include_fix,
                             double *H, double *g, double *residual) {
  if (!c || !poses12) { balm_set_error("balm_evaluate: bad arguments"); return BALM_ERR_INVALID; }
  return evaluate(Unknowns{c, nullptr}, poses12, nullptr, head, end, include_fix != 0, H, g, residual);
}

extern "C" int balm_residual(balm_ctx *c, const double *poses12, double *residual) {
  if (!c || !poses12 || !residual) { balm_set_error("balm_residual: bad arguments"); return BALM_ERR_INVALID; }
  CUDA_TRY(cudaSetDevice(c->device));
  CUDA_TRY(cudaMemcpyAsync(c->poses_trial, poses12, sizeof(double) * 12 * c->N, cudaMemcpyHostToDevice, c->stream));
  return residual_dev(c, c->poses_trial, residual);
}

extern "C" int balm_set_voxel_loss(balm_ctx *c, int kind, double scale) {
  if (!c) { balm_set_error("balm_set_voxel_loss: bad arguments"); return BALM_ERR_INVALID; }
  TRY(check_voxel_loss("balm_set_voxel_loss", kind, scale));
  c->vloss_kind = kind;
  c->vloss_scale = kind == BALM_LOSS_TRIVIAL ? 1.0 : scale;  // a trivial loss's scale is unused
  return BALM_OK;
}

extern "C" int balm_voxel_residuals(balm_ctx *c, const double *poses12, int64_t head, int64_t end, int include_fix,
                                    double *lam, double *w) {
  if (!c || !poses12) { balm_set_error("balm_voxel_residuals: bad arguments"); return BALM_ERR_INVALID; }
  if (!c->registered) { balm_set_error("no voxels registered"); return BALM_ERR_INVALID; }
  if (head < 0 || end > c->M || head > end) { balm_set_error("balm_voxel_residuals: bad voxel range"); return BALM_ERR_INVALID; }
  CUDA_TRY(cudaSetDevice(c->device));
  const int64_t nv = end - head;
  ScratchPool pool;
  double *d_out = nullptr;
  TRY(pool.get(&d_out, 2 * (size_t)nv + 1));  // lam | w | the residual the stats pass also sums
  CUDA_TRY(cudaMemcpyAsync(c->poses, poses12, sizeof(double) * 12 * c->N, cudaMemcpyHostToDevice, c->stream));
  CUDA_TRY(cudaMemsetAsync(d_out + 2 * nv, 0, sizeof(double), c->stream));
  // the evaluation's own stats instantiation (into c->stats), so that w is bitwise the weight an evaluation applies
  for (int64_t v0 = head; v0 < end; v0 += c->VB) {
    const int64_t v1 = std::min(end, v0 + c->VB);
    TRY(launch_voxel_stats(c, c->poses, v0, v1, c->stats, include_fix != 0, d_out + 2 * nv, d_out + (v0 - head),
                           d_out + nv + (v0 - head)));
  }
  if (lam && nv) CUDA_TRY(cudaMemcpyAsync(lam, d_out, sizeof(double) * nv, cudaMemcpyDeviceToHost, c->stream));
  if (w && nv) CUDA_TRY(cudaMemcpyAsync(w, d_out + nv, sizeof(double) * nv, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  return BALM_OK;
}

// The context's solve of sys (sp null) or of the sparse solver sp once its stream has been waited for: its time, then
// its outcome from the pinned mirrors of scal / flags: q1 = h_scal[1], not_pd on a bad pivot (h_flags[0]) or a
// non-finite q1. When the backward-error check failed (h_flags[4]: an indefinite H + uD factored without pivoting lost
// digits), dx is refined in fp64 with the same factors, which leaves the new q1 in h_scal[1]; if that does not bring the
// error down, the step counts as not_pd. Returns 1 in *refined when dx changed (the caller re-applies the update).
static int collect_solve(balm_ctx *c, const DenseSystem &sys, SparseSolver *sp, double *q1, int *not_pd, int *refined) {
  float ms;
  cudaEventElapsedTime(&ms, c->ev[9], c->ev[10]);
  c->tm.ms_solve += ms;
  c->tm.n_solve += 1;
  *q1 = c->h_scal[1];
  *not_pd = c->h_flags[0] != 0 || !std::isfinite(*q1);
  *refined = 0;
  if (c->h_flags[4] == 0 || *not_pd) return BALM_OK;
  int still_bad = 0;
  if (sp) TRY(sparse_refine(sp, c->stream, c->h_flags, c->h_scal, &still_bad));
  else TRY(refine_solution(c, sys, &still_bad));
  c->tm.refinements += 1;  // once per refined solve, however many rounds it took
  *q1 = c->h_scal[1];
  *refined = 1;
  if (still_bad || !std::isfinite(*q1)) *not_pd = 1;
  return BALM_OK;
}

// The damped solve of sys (the context's own system, or a rig's), or of the sparse solver sp when it is not null (a
// blocks context's blocks, or a block-sparse rig's), enqueued; collect_solve() reads it after the stream has been waited
// for
static int solve_dev(balm_ctx *c, const DenseSystem &sys, SparseSolver *sp, double u) {
  CUDA_TRY(cudaEventRecord(c->ev[9], c->stream));
  if (sp) {
    c->h_scal[3] = u;  // pinned; the kernels read the damping factor from device memory
    CUDA_TRY(cudaMemcpyAsync(c->scal + 3, c->h_scal + 3, sizeof(double), cudaMemcpyHostToDevice, c->stream));
    TRY(sparse_solve(sp, c->stream));
    c->launches += 1;
  } else {
    TRY(launch_ldlt_solve(c, sys, u));
  }
  CUDA_TRY(cudaEventRecord(c->ev[10], c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->h_scal + 1, c->scal + 1, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  if (sp) {  // no tensor-path flags in 1..3 to keep: flags 0..4 in one copy
    CUDA_TRY(cudaMemcpyAsync(c->h_flags, c->flags, sizeof(int) * 5, cudaMemcpyDeviceToHost, c->stream));
  } else {
    CUDA_TRY(cudaMemcpyAsync(c->h_flags, c->flags, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaMemcpyAsync(c->h_flags + 4, c->flags + 4, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  }
  return BALM_OK;
}

extern "C" int balm_solve(balm_ctx *c, double u, double *dx, double *q1, int *not_pd) {
  if (!c) { balm_set_error("balm_solve: bad arguments"); return BALM_ERR_INVALID; }
  CUDA_TRY(cudaSetDevice(c->device));
  const DenseSystem sys = ctx_system(c);
  SparseSolver *sp = Unknowns{c, nullptr}.solver();
  double q = 0;
  int bad = 0, refined = 0;
  TRY(solve_dev(c, sys, sp, u));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  TRY(collect_solve(c, sys, sp, &q, &bad, &refined));
  if (dx) CUDA_TRY(cudaMemcpy(dx, c->dx, sizeof(double) * c->n, cudaMemcpyDeviceToHost));
  if (q1) *q1 = q;
  if (not_pd) *not_pd = bad;
  return BALM_OK;
}

// Debug aid (include/balm_b200.h): balm_solve's path on a caller-supplied H and g, in scratch buffers of its own
extern "C" int balm_debug_ldlt(balm_ctx *c, const double *H, const double *g, double u, double *dx, double *q1,
                               int *not_pd, double *LD, double *omega) {
  if (!c || !H || !g) { balm_set_error("balm_debug_ldlt: bad arguments"); return BALM_ERR_INVALID; }
  if (c->prec == BALM_PREC_BLOCKS) {
    balm_set_error("balm_debug_ldlt: not available on a BALM_PREC_BLOCKS context (its solve is the sparse one)");
    return BALM_ERR_INVALID;
  }
  CUDA_TRY(cudaSetDevice(c->device));
  const int n = c->n;
  const size_t nn = (size_t)n * n;
  ScratchPool pool;
  struct WorkGuard {
    LdltWork w;
    ~WorkGuard() { ldlt_work_free(&w); }
  } wg;
  double *d_H, *d_g, *d_dx, *d_dvec, *d_A;
  TRY(pool.get(&d_H, nn));
  TRY(pool.get(&d_g, (size_t)n));
  TRY(pool.get(&d_dx, (size_t)n));
  TRY(pool.get(&d_dvec, (size_t)n));
  TRY(pool.get(&d_A, nn));
  const DenseSystem sys{n, d_H, d_g, d_dx, d_dvec, d_A, &wg.w};
  CUDA_TRY(cudaMemcpyAsync(d_H, H, sizeof(double) * nn, cudaMemcpyHostToDevice, c->stream));
  CUDA_TRY(cudaMemcpyAsync(d_g, g, sizeof(double) * n, cudaMemcpyHostToDevice, c->stream));
  double q = 0;
  int bad = 0, refined = 0;
  TRY(solve_dev(c, sys, nullptr, u));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  TRY(collect_solve(c, sys, nullptr, &q, &bad, &refined));
  if (dx) CUDA_TRY(cudaMemcpy(dx, d_dx, sizeof(double) * n, cudaMemcpyDeviceToHost));
  if (omega) CUDA_TRY(cudaMemcpy(omega, c->scal + 20, sizeof(double), cudaMemcpyDeviceToHost));
  if (LD) {  // the factorisation writes the lower triangle only: the upper one still holds H + u diag(H)
    CUDA_TRY(cudaMemcpy(LD, d_A, sizeof(double) * nn, cudaMemcpyDeviceToHost));
    for (int j = 1; j < n; j++) memset(LD + (size_t)j * n, 0, sizeof(double) * j);
  }
  if (q1) *q1 = q;
  if (not_pd) *not_pd = bad;
  return BALM_OK;
}

extern "C" void balm_default_lm_opts(balm_lm_opts *o) {
  o->max_iter = 10; o->u0 = 0.01; o->v0 = 2; o->rel_tol = 1e-6; o->hess_includes_fix = 0; o->gauge_mode = 0;
  o->min_planes_per_pose = 20; o->verbose = 0; o->force_hess = 0;
}

// With an active absolute pose prior the cost has no gauge freedom: re-anchoring to pose 0 would move the result off
// the priors.
static int refuse_gauge_with_priors(const char *who, const PriorSet *pr, const balm_lm_opts *o) {
  if (!prior_set_active(pr) || (o->gauge_mode != 0 && o->gauge_mode != 1)) return BALM_OK;
  balm_set_error(std::string(who) + ": gauge_mode " + std::to_string(o->gauge_mode) +
                 " re-anchors to pose 0, which moves the result off the pose priors; pass gauge_mode 2");
  return BALM_ERR_INVALID;
}

// Clears the context's LM flags (set by damping_iter) on every exit path
struct LmScope {
  balm_ctx *c;
  ~LmScope() { c->lm_active = false; c->defer = false; c->pending_eval = false; c->eval_same_poses = false; }
};

// balm_damping_iter, balm_rig_damping_iter and balm_pose_graph_iter after their checks (`who` prefixes the messages):
// LM from x12 / ext12, the result written back to them, the state after every iteration to per_iter
static int damping_iter(const Unknowns &u, const char *who, double *x12, double *ext12, const balm_lm_opts *o,
                        balm_trace *trace, int *n_iters, double *per_iter) {
  balm_ctx *c = u.c;
  // A rig's and the pose terms' evaluations stay the pure functions balm_rig_evaluate and balm_pose_graph_evaluate
  // are: no per-voxel stats handed over from the trial residual pass and no tensor scale speculation (lm_active and
  // eval_same_poses stay false). A joint cost (balm_set_joint_cost) keeps them: its terms are added after the voxel sums
  // and the RCUR / RTRIAL copies, and read no observation.
  const bool carry_over = !u.rig && !u.pose_terms;
  // Re-anchoring a rig to base pose 0 would move the result off its fixed base poses.
  const bool bases_fixed = u.rig && rig_any_base_fixed(u.rig);
  if ((o->gauge_mode == 0 || o->gauge_mode == 1) && bases_fixed) {
    balm_set_error(std::string(who) + ": gauge_mode " + std::to_string(o->gauge_mode) +
                   " re-anchors to base pose 0, which moves the result off the fixed base poses; pass gauge_mode 2");
    return BALM_ERR_INVALID;
  }
  if (pose_terms_in_cost(c)) TRY(refuse_gauge_with_priors(who, c->pr, o));
  if (o->min_planes_per_pose > 0) {  // bavoxel.hpp:1071-1085 (the shim reproduces the printf + exit(0)); per scan slot
    // The guard is on the GLOBAL count of voxels seeing each pose. With several ranks every rank all-reduces the
    // per-pose histogram of its shard first, so all ranks take the same branch (a rank returning alone would leave
    // the others waiting in the next collective).
    long long global_min = c->min_planes;
    if (c->world > 1 && c->comm) {
      int *red = c->planes + c->N;
      const int rc = g_nccl.AllReduce(c->planes, red, (size_t)c->N, /*ncclInt32*/ 2, /*ncclSum*/ 0, c->comm, c->stream);
      if (rc != 0) { balm_set_error("ncclAllReduce (plane histogram) failed"); return BALM_ERR_NCCL; }
      std::vector<int> pl((size_t)c->N);
      CUDA_TRY(cudaMemcpyAsync(pl.data(), red, sizeof(int) * c->N, cudaMemcpyDeviceToHost, c->stream));
      CUDA_TRY(cudaStreamSynchronize(c->stream));
      global_min = *std::min_element(pl.begin(), pl.end());
    }
    if (global_min < o->min_planes_per_pose) {
      balm_set_error("Initial error too large. Please loose plane determination criteria for more planes.");
      return BALM_ERR_TOO_FEW_PLANES;
    }
  }
  TRY(u.upload(x12, ext12));
  // The residual pass at the trial poses computes the same per-voxel eigen data the next evaluation starts with:
  // when the step is accepted they are handed over (same kernel, same inputs -> identical values). Needs the whole
  // problem in one batch and the same treatment of the fix cluster in both passes.
  const bool hand_over = carry_over && c->stats_trial != nullptr && (c->fix == nullptr || o->hess_includes_fix != 0);
  bool stats_cached = false;
  bool same_poses = false;  // the last step was rejected: c->poses are those of the previous evaluation
  if (carry_over) tensor_syrk_new_problem(c);  // nothing speculative is carried over from earlier calls
  LmScope lm_scope{c};
  c->lm_active = carry_over;
  // the evaluation's events and flags are read after the iteration's wait; BALM_SYNC_PHASES waits after every phase
  c->defer = !getenv("BALM_SYNC_PHASES");
  const DenseSystem sys = u.system();
  SparseSolver *sp = u.solver();
  const int ns = u.n_state();
  // BALM2::damping_iter's loop (bavoxel.hpp:1127-1155): per iteration evaluation (when H is stale), solve, trial state
  // and trial cost are enqueued back to back and the host waits once; a refined dx redoes the trial state and its cost.
  double uu = o->u0, v = o->v0, r1 = 0, r2 = 0;
  bool calc_hess = true;
  for (int it = 0; it < o->max_iter; it++) {
    if (calc_hess) {
      c->eval_same_poses = carry_over && same_poses;
      const int rc = u.eval(o->hess_includes_fix != 0, 0, c->M, stats_cached);
      c->eval_same_poses = false;
      TRY(rc);
      CUDA_TRY(cudaMemcpyAsync(c->h_scal, c->scal, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    }
    TRY(solve_dev(c, sys, sp, uu));
    if (!c->defer) CUDA_TRY(cudaStreamSynchronize(c->stream));
    TRY(u.trial());
    TRY(u.trial_cost(hand_over, &r2));
    if (calc_hess) TRY(u.collect());  // the evaluation's events, read after the trial cost's wait
    double q1 = 0;
    int not_pd = 0, refined = 0;
    TRY(collect_solve(c, sys, sp, &q1, &not_pd, &refined));
    if (refined && !not_pd) {  // dx changed: the trial state and its cost again (rare path)
      TRY(u.trial());
      TRY(u.trial_cost(hand_over, &r2));
    }
    if (calc_hess) r1 = c->h_scal[0];
    balm_trace t;
    bool stop;
    const bool accepted = lm_rule(r1, r2, q1, not_pd, calc_hess, o->rel_tol, &uu, &v, &t, &stop);
    if (o->verbose)  // the reference's trace line (bavoxel.hpp:1132)
      printf("iter%d: (%lf %lf) u: %lf v: %.1lf q: %.3lf %lf %lf\n", it, r1, r2, t.u, t.v, t.q / q1, q1, t.q);
    if (accepted) {
      u.accept();
      if (hand_over) {
        std::swap(c->stats, c->stats_trial);
        CUDA_TRY(cudaMemcpyAsync(c->scal + BALM_SCAL_RCUR, c->scal + BALM_SCAL_RTRIAL, sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
      }
      stats_cached = hand_over;
    } else {
      stats_cached = carry_over && c->stats_trial != nullptr;  // c->stats still describes c->poses (single batch)
    }
    same_poses = !accepted;
    calc_hess = accepted || o->force_hess != 0;  // after a rejection H and g of the current state are still in place
    if (trace) trace[it] = t;
    if (per_iter)
      CUDA_TRY(cudaMemcpyAsync(per_iter + (size_t)it * 12 * ns, u.state(), sizeof(double) * 12 * ns,
                               cudaMemcpyDeviceToHost, c->stream));
    if (n_iters) *n_iters = it + 1;
    if (stop) break;
  }
  if (o->gauge_mode == 0 || o->gauge_mode == 1) TRY(u.gauge(o->gauge_mode));
  TRY(u.download(x12, ext12));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  return BALM_OK;
}

extern "C" int balm_damping_iter(balm_ctx *c, double *poses12, const balm_lm_opts *o, balm_trace *trace, int *n_iters,
                                 double *poses_per_iter) {
  if (!c || !poses12 || !o) { balm_set_error("balm_damping_iter: bad arguments"); return BALM_ERR_INVALID; }
  CUDA_TRY(cudaSetDevice(c->device));
  if (n_iters) *n_iters = 0;
  if (!c->registered) { balm_set_error("no voxels registered"); return BALM_ERR_INVALID; }
  return damping_iter(Unknowns{c, nullptr}, "balm_damping_iter", poses12, nullptr, o, trace, n_iters, poses_per_iter);
}

// ---------------- pose graph (pose_graph.cu, pose_graph_sparse.cu) ----------------
// The argument checks of balm_set_pose_factors and balm_spg_set_factors over P poses; `who` prefixes the messages.
static int pose_factors_check(const char *who, int P, int n_factors, const int64_t *factor_ptr,
                              const int32_t *factor_pose, const double *poses_hat12, const double *H) {
  const std::string w = std::string(who) + ": ";
  if (n_factors < 1 || !factor_ptr || !factor_pose || !poses_hat12 || !H) {
    balm_set_error(w + "bad arguments");
    return BALM_ERR_INVALID;
  }
  if (factor_ptr[0] != 0) { balm_set_error(w + "factor_ptr[0] must be 0"); return BALM_ERR_INVALID; }
  int64_t hsize = 0;
  std::vector<char> seen((size_t)P, 0);
  for (int f = 0; f < n_factors; f++) {
    const int64_t N = factor_ptr[f + 1] - factor_ptr[f];
    if (N < 2 || N > BALM_BATCH_MAX_POSES) {
      balm_set_error(w + "factor " + std::to_string(f) + " has " + std::to_string(N) + " poses (2 .. 32 allowed)");
      return BALM_ERR_INVALID;
    }
    const int32_t *idx = factor_pose + factor_ptr[f];
    bool ok = true;
    for (int64_t k = 0; k < N && ok; k++) {
      ok = idx[k] >= 0 && idx[k] < P && !seen[idx[k]];
      if (ok) seen[idx[k]] = 1;
    }
    for (int64_t k = 0; k < N; k++)
      if (idx[k] >= 0 && idx[k] < P) seen[idx[k]] = 0;
    if (!ok) {
      balm_set_error(w + "factor " + std::to_string(f) + " needs distinct pose indices in [0, n_poses)");
      return BALM_ERR_INVALID;
    }
    hsize += 36 * N * N;
  }
  const int64_t S = factor_ptr[n_factors];
  for (int64_t e = 0; e < 12 * S; e++)
    if (!std::isfinite(poses_hat12[e])) { balm_set_error(w + "non-finite poses_hat12"); return BALM_ERR_INVALID; }
  for (int64_t e = 0; e < hsize; e++)
    if (!std::isfinite(H[e])) { balm_set_error(w + "non-finite H"); return BALM_ERR_INVALID; }
  // H_f symmetric to 1e-12 of its largest entry: the cost reads e^T H_f e, the gradient H_f's rows as given and the
  // assembly one triangle, which agree only when H_f is symmetric
  const double *Hf = H;
  for (int f = 0; f < n_factors; f++) {
    const int64_t n6 = 6 * (factor_ptr[f + 1] - factor_ptr[f]);
    double hmax = 0.0;
    for (int64_t e = 0; e < n6 * n6; e++) hmax = std::max(hmax, fabs(Hf[e]));
    for (int64_t a = 0; a < n6; a++)
      for (int64_t c = 0; c < a; c++)
        if (fabs(Hf[c * n6 + a] - Hf[a * n6 + c]) > 1e-12 * hmax) {
          balm_set_error(w + "factor " + std::to_string(f) + " has an H that is not symmetric");
          return BALM_ERR_INVALID;
        }
    Hf += n6 * n6;
  }
  return BALM_OK;
}

// balm_set_pose_factors, balm_block_set_factors and balm_spg_set_factors after their argument checks
static int block_set_factors(balm_ctx *c, const char *who, int n_factors, const int64_t *factor_ptr,
                             const int32_t *factor_pose, const double *poses_hat12, const double *H, int32_t *status_out) {
  CUDA_TRY(cudaSetDevice(c->device));
  PoseGraph *pg = nullptr;
  std::vector<int> status;
  if (n_factors != 0)  // 0 detaches the factor set
    TRY(pose_graph_build(c->stream, c->N, n_factors, factor_ptr, factor_pose, poses_hat12, H, &status, &pg, &c->launches));
  std::unique_ptr<PoseGraph, void (*)(PoseGraph *)> pg_own(pg, pose_graph_free);
  if (c->bh) TRY(blocks_repattern(c, pg, who));  // no voxels registered yet: the next registration builds the union
  if (status_out) std::copy(status.begin(), status.end(), status_out);
  pose_graph_free(c->pg);
  c->pg = pg_own.release();
  return BALM_OK;
}

extern "C" int balm_block_set_factors(balm_ctx *c, int n_factors, const int64_t *factor_ptr, const int32_t *factor_pose,
                                      const double *poses_hat12, const double *H, int32_t *status_out) {
  const char *who = "balm_block_set_factors";
  if (!c) { balm_set_error(std::string(who) + ": bad arguments"); return BALM_ERR_INVALID; }
  if (c->prec != BALM_PREC_BLOCKS) {
    balm_set_error(std::string(who) + ": BALM_PREC_BLOCKS contexts only (the dense ones take balm_set_pose_factors)");
    return BALM_ERR_INVALID;
  }
  if (n_factors != 0) TRY(pose_factors_check(who, c->N, n_factors, factor_ptr, factor_pose, poses_hat12, H));
  return block_set_factors(c, who, n_factors, factor_ptr, factor_pose, poses_hat12, H, status_out);
}

extern "C" int balm_set_pose_factors(balm_ctx *c, int n_factors, const int64_t *factor_ptr, const int32_t *factor_pose,
                                     const double *poses_hat12, const double *H, int32_t *status_out) {
  const char *who = "balm_set_pose_factors";
  if (!c) { balm_set_error(std::string(who) + ": bad arguments"); return BALM_ERR_INVALID; }
  TRY(refuse_blocks(c, who));
  TRY(pose_factors_check(who, c->N, n_factors, factor_ptr, factor_pose, poses_hat12, H));
  return block_set_factors(c, who, n_factors, factor_ptr, factor_pose, poses_hat12, H, status_out);
}

// The loss arguments of one factor or prior: kind one of balm_loss, and a finite scale > 0 unless trivial. `item`
// ("<who>: factor f" / "<who>: prior q") prefixes the messages.
static int term_loss_check(const std::string &item, int32_t kind, const double *scale) {
  if (kind != BALM_LOSS_TRIVIAL && kind != BALM_LOSS_HUBER && kind != BALM_LOSS_CAUCHY) {
    balm_set_error(item + " has loss kind " + std::to_string(kind) + " (0, 1, 2 allowed)");
    return BALM_ERR_INVALID;
  }
  if (kind != BALM_LOSS_TRIVIAL && !(scale && std::isfinite(*scale) && *scale > 0.0)) {
    balm_set_error(item + " needs a finite scale > 0");
    return BALM_ERR_INVALID;
  }
  return BALM_OK;
}

// balm_set_factor_loss / balm_spg_set_factor_loss on the factor set pg (null: none registered)
static int set_factor_loss(const char *who, PoseGraph *pg, cudaStream_t st, int n_factors, const int32_t *kind,
                           const double *scale) {
  const std::string w = std::string(who) + ": ";
  if (!pg) { balm_set_error(w + "no pose factors registered"); return BALM_ERR_INVALID; }
  if (n_factors != pose_graph_n_factors(pg)) {
    balm_set_error(w + "n_factors " + std::to_string(n_factors) + " is not the registered count " +
                   std::to_string(pose_graph_n_factors(pg)));
    return BALM_ERR_INVALID;
  }
  for (int f = 0; kind && f < n_factors; f++)
    TRY(term_loss_check(w + "factor " + std::to_string(f), kind[f], scale ? scale + f : nullptr));
  return pose_graph_set_loss(pg, st, kind, scale);
}

extern "C" int balm_set_factor_loss(balm_ctx *c, int n_factors, const int32_t *kind, const double *scale) {
  if (!c) { balm_set_error("balm_set_factor_loss: bad arguments"); return BALM_ERR_INVALID; }
  CUDA_TRY(cudaSetDevice(c->device));
  return set_factor_loss("balm_set_factor_loss", c->pg, c->stream, n_factors, kind, scale);
}

// balm_factor_residuals / balm_prior_residuals: the readout of the context's term set `set` (c->pg or c->pr), named
// `what` in the refusal when none is registered
template <typename Set>
static int set_residuals(balm_ctx *c, Set *balm_ctx::*set, const char *who, const char *what, const double *poses12,
                         double *s, double *w) {
  if (!c || !poses12) { balm_set_error(std::string(who) + ": bad arguments"); return BALM_ERR_INVALID; }
  if (!(c->*set)) { balm_set_error(std::string(who) + ": no " + what + " registered"); return BALM_ERR_INVALID; }
  CUDA_TRY(cudaSetDevice(c->device));
  CUDA_TRY(cudaMemcpyAsync(c->poses, poses12, sizeof(double) * 12 * c->N, cudaMemcpyHostToDevice, c->stream));
  return term_residuals(c->*set, c->stream, c->poses, s, w, &c->launches);
}

extern "C" int balm_factor_residuals(balm_ctx *c, const double *poses12, double *s, double *w) {
  return set_residuals(c, &balm_ctx::pg, "balm_factor_residuals", "pose factors", poses12, s, w);
}

extern "C" int balm_pose_graph_evaluate(balm_ctx *c, const double *poses12, double *H, double *g, double *cost) {
  if (!c || !poses12) { balm_set_error("balm_pose_graph_evaluate: bad arguments"); return BALM_ERR_INVALID; }
  TRY(refuse_blocks(c, "balm_pose_graph_evaluate"));
  if (!c->pg) { balm_set_error("balm_pose_graph_evaluate: no pose factors registered"); return BALM_ERR_INVALID; }
  return evaluate(Unknowns{c, nullptr, true}, poses12, nullptr, 0, 0, false, H, g, cost);
}

extern "C" int balm_pose_graph_iter(balm_ctx *c, double *poses12, const balm_lm_opts *o, balm_trace *trace, int *n_iters,
                                    double *poses_per_iter) {
  if (!c || !poses12 || !o) { balm_set_error("balm_pose_graph_iter: bad arguments"); return BALM_ERR_INVALID; }
  TRY(refuse_blocks(c, "balm_pose_graph_iter"));
  if (n_iters) *n_iters = 0;
  if (c->world > 1 || c->comm) { balm_set_error("balm_pose_graph_iter: single-GPU contexts only"); return BALM_ERR_INVALID; }
  if (!c->pg) { balm_set_error("balm_pose_graph_iter: no pose factors registered"); return BALM_ERR_INVALID; }
  TRY(refuse_gauge_with_priors("balm_pose_graph_iter", c->pr, o));
  CUDA_TRY(cudaSetDevice(c->device));
  balm_lm_opts lo = *o;
  lo.min_planes_per_pose = 0;  // no voxels
  lo.hess_includes_fix = 0;
  return damping_iter(Unknowns{c, nullptr, true}, "balm_pose_graph_iter", poses12, nullptr, &lo, trace, n_iters,
                      poses_per_iter);
}

// ---------------- covariances at a state (covariance.cu, pose_graph_sparse.cu) ----------------
// The undamped factorisation of H (or H_rig) at the unknowns' current state: `factor` runs `eval`, the evaluation
// deferred, then a factorisation that waits for the stream; the evaluation's events are read after that wait.
using FactorStep = std::function<int(const std::function<int()> &eval)>;
static int factor_at_state(const Unknowns &u, bool include_fix, const FactorStep &factor) {
  balm_ctx *c = u.c;
  const int rc = factor([&]() -> int {
    c->defer = true;
    const int e = u.eval(include_fix, 0, c->M);
    c->defer = false;
    return e;
  });
  if (rc == BALM_OK || rc == BALM_ERR_NOT_PD) TRY(u.collect());  // the stream has been synchronised
  c->pending_eval = false;
  return rc;
}

// balm_pose_covariance and balm_rig_covariance after their checks: raw = the raw term R (cov_raw_dev) at the slot
// poses of x12 / ext12 in the unknowns (J^T R J for a rig), cov = H~^-1 raw H~^-T with H (or H_rig) at the same state
// factored undamped. The anchor's rows and columns (none for -1) are deleted from both, with 1 on H~'s diagonal. Waits
// for the pivot test and at the end.
static int covariance(const Unknowns &u, const double *x12, const double *ext12, const double *c_cov81,
                      double point_noise, bool include_fix, int anchor, const char *singular_msg, double *raw,
                      double *cov) {
  balm_ctx *c = u.c;
  const DenseSystem sys = u.system();
  const int n = sys.n, a0 = anchor < 0 ? -1 : 6 * anchor;
  CUDA_TRY(cudaSetDevice(c->device));
  TRY(u.upload(x12, ext12));
  TRY(u.compose());
  ScratchPool pool;
  double *R = nullptr;
  TRY(cov_raw_dev(c, pool, c->poses, c_cov81, point_noise, include_fix, &R));
  TRY(u.reduce_raw(pool, &R));
  if (a0 >= 0) TRY(cov_delete_block(c, R, n, a0, 0.0));
  if (cov)  // H at these poses (divide_thread, BAs_left.hpp:1091)
    TRY(factor_at_state(u, include_fix, [&](const std::function<int()> &eval) -> int {
      TRY(eval());
      // the context or the rig owns H: the deletion edits it in place, and the next evaluation rewrites it
      if (a0 >= 0) TRY(cov_delete_block(c, const_cast<double *>(sys.H), n, a0, 1.0));
      return cov_factor(c, sys, a0, singular_msg);
    }));
  if (raw) CUDA_TRY(cudaMemcpyAsync(raw, R, sizeof(double) * n * n, cudaMemcpyDeviceToHost, c->stream));
  if (cov) {
    TRY(cov_sandwich(c, sys, R));
    if (a0 >= 0) TRY(cov_delete_block(c, R, n, a0, 0.0));
    CUDA_TRY(cudaMemcpyAsync(cov, R, sizeof(double) * n * n, cudaMemcpyDeviceToHost, c->stream));
  }
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  return BALM_OK;
}

// balm_block_covariance, balm_spg_covariance and balm_rig_block_covariance after their checks (`who` prefixes the
// messages): H~^-1 on the block pattern at x12 / ext12 (sparse_covariance), so the call waits twice
static int block_covariance(const Unknowns &u, const char *who, const double *x12, const double *ext12,
                            bool include_fix, int anchor, double *cov) {
  CUDA_TRY(cudaSetDevice(u.c->device));
  return factor_at_state(u, include_fix, [&](const std::function<int()> &eval) {
    return sparse_covariance(u.solver(), u.c->stream, anchor, [&]() -> int {
      TRY(u.upload(x12, ext12));
      return eval();
    }, who, cov, &u.c->launches);
  });
}

// balm_block_point_covariance and balm_rig_block_point_covariance after their checks (`who` prefixes the messages): the
// raw term on the slot pattern at x12 / ext12 into raw_blocks, and with cov or marg Sigma_sel (block_point_cov_dev)
// after the anchored undamped factorisation at the same state
static int block_point_covariance(const Unknowns &u, const char *who, const double *x12, const double *ext12,
                                  const double *c_cov81, double point_noise, bool include_fix, int anchor, int n_sel,
                                  const int32_t *sel, double *raw_blocks, double *cov, double *marg) {
  balm_ctx *c = u.c;
  const bool sigma = cov || marg;
  SparseSolver *sp = u.solver();
  CUDA_TRY(cudaSetDevice(c->device));
  TRY(u.upload(x12, ext12));
  if (sigma)  // the evaluation composes the slot poses
    TRY(factor_at_state(u, include_fix, [&](const std::function<int()> &eval) -> int {
      TRY(eval());
      return sparse_factor_undamped(sp, c->stream, anchor, who, &c->launches);
    }));
  else
    TRY(u.compose());
  ScratchPool pool;
  double *raw = nullptr;
  const size_t nraw = 36 * blocks_pairs(c->bh).size();
  TRY(pool.get(&raw, nraw));
  TRY(cov_raw_blocks_dev(c, pool, c->poses, c_cov81, point_noise, include_fix, raw));
  if (sigma) TRY(block_point_cov_dev(c, sp, u.rig, u.state(), anchor, n_sel, sel, raw, cov, marg));
  if (raw_blocks) CUDA_TRY(cudaMemcpyAsync(raw_blocks, raw, sizeof(double) * nraw, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  return BALM_OK;
}

// ---------------- rig calibration (rig.cu) ----------------
// balm_set_rig's and balm_block_set_rig's checks and attach (`who` prefixes the messages): detach on n_base 0, else the
// arguments checked and a new rig built; on a refusal the previous rig stays
static int set_rig(balm_ctx *c, const char *who, bool sparse, int n_base, int n_lidar, const int32_t *base_of,
                   const int32_t *lidar_of, const uint8_t *base_fixed, const uint8_t *lidar_fixed, int *n_rig_out) {
  const std::string w = std::string(who) + ": ";
  if (c->world > 1 || c->comm) { balm_set_error(w + "single-GPU contexts only"); return BALM_ERR_INVALID; }
  CUDA_TRY(cudaSetDevice(c->device));
  if (n_base == 0) {  // detach
    rig_free(c->rig);
    c->rig = nullptr;
    if (n_rig_out) *n_rig_out = 0;
    return BALM_OK;
  }
  if (n_base < 0 || n_lidar < 1 || !base_of || !lidar_of) { balm_set_error(w + "bad arguments"); return BALM_ERR_INVALID; }
  std::vector<char> base_used((size_t)n_base, 0), lidar_used((size_t)n_lidar, 0);
  for (int s = 0; s < c->N; s++) {
    if (base_of[s] < 0 || base_of[s] >= n_base || lidar_of[s] < 0 || lidar_of[s] >= n_lidar) {
      balm_set_error(w + "slot " + std::to_string(s) + " has base " + std::to_string(base_of[s]) + " / lidar " +
                     std::to_string(lidar_of[s]) + " outside [0, n_base) / [0, n_lidar)");
      return BALM_ERR_INVALID;
    }
    base_used[base_of[s]] = 1;
    lidar_used[lidar_of[s]] = 1;
  }
  for (int b = 0; b < n_base; b++)
    if (!base_used[b]) { balm_set_error(w + "no slot uses base " + std::to_string(b)); return BALM_ERR_INVALID; }
  for (int l = 0; l < n_lidar; l++)
    if (!lidar_used[l]) { balm_set_error(w + "no slot uses lidar " + std::to_string(l)); return BALM_ERR_INVALID; }
  int n_free = 0;
  for (int b = 0; b < n_base; b++) n_free += !(base_fixed && base_fixed[b]);
  for (int l = 0; l < n_lidar; l++) n_free += !(lidar_fixed && lidar_fixed[l]);
  if (n_free == 0) { balm_set_error(w + "every base pose and extrinsic is fixed"); return BALM_ERR_INVALID; }
  Rig *r = nullptr;
  const int rc = rig_build(c->stream, c->N, n_base, n_lidar, base_of, lidar_of, base_fixed, lidar_fixed, sparse, &r);
  if (rc != BALM_OK) {
    cudaGetLastError();  // an out-of-memory allocation must not fail the next launch check; the previous rig stays
    return rc;
  }
  rig_free(c->rig);
  c->rig = r;
  if (n_rig_out) *n_rig_out = rig_n(r);
  return BALM_OK;
}

extern "C" int balm_set_rig(balm_ctx *c, int n_base, int n_lidar, const int32_t *base_of, const int32_t *lidar_of,
                            const uint8_t *base_fixed, const uint8_t *lidar_fixed, int *n_rig_out) {
  if (!c) { balm_set_error("balm_set_rig: bad arguments"); return BALM_ERR_INVALID; }
  if (c->prec == BALM_PREC_BLOCKS) {
    balm_set_error("balm_set_rig: not available on a BALM_PREC_BLOCKS context (it holds no dense H); use "
                   "balm_block_set_rig");
    return BALM_ERR_UNSUPPORTED;
  }
  return set_rig(c, "balm_set_rig", false, n_base, n_lidar, base_of, lidar_of, base_fixed, lidar_fixed, n_rig_out);
}

extern "C" int balm_block_set_rig(balm_ctx *c, int n_base, int n_lidar, const int32_t *base_of,
                                  const int32_t *lidar_of, const uint8_t *base_fixed, const uint8_t *lidar_fixed,
                                  int *n_rig_out) {
  if (!c) { balm_set_error("balm_block_set_rig: bad arguments"); return BALM_ERR_INVALID; }
  if (c->prec != BALM_PREC_BLOCKS) {
    balm_set_error("balm_block_set_rig: BALM_PREC_BLOCKS contexts only (the dense ones take balm_set_rig)");
    return BALM_ERR_INVALID;
  }
  return set_rig(c, "balm_block_set_rig", true, n_base, n_lidar, base_of, lidar_of, base_fixed, lidar_fixed,
                 n_rig_out);
}

// A block-sparse rig's pattern follows the slot pattern: rebuilt here when that has changed (BALM_ERR_UNSUPPORTED when
// too large to index)
static int rig_check(balm_ctx *c, const char *who) {
  if (!c->rig) { balm_set_error(std::string(who) + ": no rig set (balm_set_rig)"); return BALM_ERR_INVALID; }
  // balm_comm_init may attach a communicator after balm_set_rig: the rig calls stay single-GPU
  if (c->world > 1 || c->comm) { balm_set_error(std::string(who) + ": single-GPU contexts only"); return BALM_ERR_INVALID; }
  if (!c->registered) { balm_set_error("no voxels registered"); return BALM_ERR_INVALID; }
  if (rig_sparse(c->rig)) {
    CUDA_TRY(cudaSetDevice(c->device));
    const int rc = rig_blocks_sync(c->rig, c->stream, blocks_pairs(c->bh), blocks_generation(c->bh), c->scal, c->flags,
                                   who);
    if (rc != BALM_OK) cudaGetLastError();  // as balm_set_rig: an out-of-memory build leaves no launch error behind
    TRY(rc);
  }
  return BALM_OK;
}

extern "C" int balm_rig_evaluate(balm_ctx *c, const double *base12, const double *ext12, int include_fix, double *H,
                                 double *g, double *residual) {
  if (!c || !base12 || !ext12) { balm_set_error("balm_rig_evaluate: bad arguments"); return BALM_ERR_INVALID; }
  TRY(rig_check(c, "balm_rig_evaluate"));
  return evaluate(Unknowns{c, c->rig}, base12, ext12, 0, c->M, include_fix != 0, H, g, residual);
}

extern "C" int balm_rig_covariance(balm_ctx *c, const double *base12, const double *ext12, const double *c_cov81,
                                   double point_noise, int include_fix, int anchor, double *raw, double *cov) {
  const char *who = "balm_rig_covariance";
  if (!c || !base12 || !ext12 || (!raw && !cov)) { balm_set_error(std::string(who) + ": bad arguments"); return BALM_ERR_INVALID; }
  if (c->rig && rig_sparse(c->rig)) {
    balm_set_error(std::string(who) + ": not available for a BALM_PREC_BLOCKS context's rig (it needs the dense 6N x 6N "
                   "raw term); balm_rig_block_covariance gives H_rig^-1");
    return BALM_ERR_UNSUPPORTED;
  }
  TRY(rig_check(c, who));
  if (c->M < 1) { balm_set_error(std::string(who) + ": no voxels registered"); return BALM_ERR_INVALID; }
  const Unknowns u{c, c->rig};
  TRY(u.check_anchor(who, anchor));
  return covariance(u, base12, ext12, c_cov81, point_noise, include_fix != 0, anchor,
                    "balm_rig_covariance: H_rig is singular (a gauge or an unobservable direction of the rig is not "
                    "fixed: fix clusters, fixed unknowns or an anchor)",
                    raw, cov);
}

extern "C" int balm_rig_damping_iter(balm_ctx *c, double *base12, double *ext12, const balm_lm_opts *o,
                                     balm_trace *trace, int *n_iters, double *rig_per_iter) {
  const char *who = "balm_rig_damping_iter";
  if (!c || !base12 || !ext12 || !o) { balm_set_error(std::string(who) + ": bad arguments"); return BALM_ERR_INVALID; }
  if (n_iters) *n_iters = 0;
  TRY(rig_check(c, who));
  CUDA_TRY(cudaSetDevice(c->device));
  return damping_iter(Unknowns{c, c->rig}, who, base12, ext12, o, trace, n_iters, rig_per_iter);
}

// the block-sparse rig's calls: a rig set by balm_block_set_rig, its pattern in step with the slot pattern
static int block_rig_check(balm_ctx *c, const char *who) {
  if (c->rig && !rig_sparse(c->rig)) {
    balm_set_error(std::string(who) + ": the rig was set by balm_set_rig (a dense context's)");
    return BALM_ERR_INVALID;
  }
  if (!c->rig) { balm_set_error(std::string(who) + ": no rig set (balm_block_set_rig)"); return BALM_ERR_INVALID; }
  return rig_check(c, who);
}

extern "C" int balm_rig_block_structure(balm_ctx *c, int64_t stats[4], int32_t *pairs) {
  const char *who = "balm_rig_block_structure";
  if (!c || !stats) { balm_set_error(std::string(who) + ": bad arguments"); return BALM_ERR_INVALID; }
  TRY(block_rig_check(c, who));
  const std::vector<int2> &pr = rig_pairs(c->rig);
  stats[0] = (int64_t)pr.size();
  stats[3] = rig_blocks_bytes(c->rig, &stats[1], &stats[2]);
  if (pairs)
    for (size_t p = 0; p < pr.size(); p++) { pairs[2 * p] = pr[p].x; pairs[2 * p + 1] = pr[p].y; }
  return BALM_OK;
}

extern "C" int balm_rig_block_covariance(balm_ctx *c, const double *base12, const double *ext12, int include_fix,
                                         int anchor, double *cov) {
  const char *who = "balm_rig_block_covariance";
  if (!c || !base12 || !ext12 || !cov) { balm_set_error(std::string(who) + ": bad arguments"); return BALM_ERR_INVALID; }
  TRY(block_rig_check(c, who));
  const Unknowns u{c, c->rig};
  TRY(u.check_anchor(who, anchor));
  return block_covariance(u, who, base12, ext12, include_fix != 0, anchor, cov);
}

// ---------------- point-noise covariance on blocks contexts (covariance.cu) ----------------
// sel [n_sel]: distinct indices in [0, n) (`what` names them in the message)
static int point_cov_sel_check(const char *who, int n_sel, const int32_t *sel, int n, const char *what) {
  const std::string w = std::string(who) + ": ";
  if (n_sel < 1 || !sel) { balm_set_error(w + "n_sel must be at least 1 with a selection"); return BALM_ERR_INVALID; }
  std::vector<char> seen((size_t)n, 0);
  for (int u = 0; u < n_sel; u++) {
    if (sel[u] < 0 || sel[u] >= n) {
      balm_set_error(w + "sel[" + std::to_string(u) + "] = " + std::to_string(sel[u]) + " is not a " + what + " in [0, " +
                     std::to_string(n) + ")");
      return BALM_ERR_INVALID;
    }
    if (seen[sel[u]]) {
      balm_set_error(w + "sel[" + std::to_string(u) + "] = " + std::to_string(sel[u]) + " is selected twice");
      return BALM_ERR_INVALID;
    }
    seen[sel[u]] = 1;
  }
  return BALM_OK;
}

// The budget refusal of the joint covariance (before anything is enqueued)
static int point_cov_budget_check(const char *who, int P, int N, int n_sel, bool joint) {
  if (block_point_cov_fits(P, N, n_sel, joint)) return BALM_OK;
  balm_set_error(std::string(who) + (joint ? ": the joint covariance's Y, W and Z (8 (6P + 12N) 6 n_sel bytes and its "
                                             "partial sums) exceed BALM_COV_BUDGET_MB; ask for the marginals alone"
                                           : ": one unknown's right-hand sides exceed BALM_COV_BUDGET_MB"));
  return BALM_ERR_UNSUPPORTED;
}

extern "C" int balm_rig_block_point_covariance(balm_ctx *c, const double *base12, const double *ext12,
                                               const double *c_cov81, double point_noise, int include_fix, int anchor,
                                               int n_sel, const int32_t *sel, double *cov, double *marg) {
  const char *who = "balm_rig_block_point_covariance";
  if (!c || !base12 || !ext12 || (!cov && !marg)) { balm_set_error(std::string(who) + ": bad arguments"); return BALM_ERR_INVALID; }
  if (c->prec != BALM_PREC_BLOCKS) {
    balm_set_error(std::string(who) + ": BALM_PREC_BLOCKS contexts only (the dense ones take balm_rig_covariance)");
    return BALM_ERR_INVALID;
  }
  TRY(block_rig_check(c, who));
  if (c->M < 1) { balm_set_error(std::string(who) + ": no voxels registered"); return BALM_ERR_INVALID; }
  const Unknowns u{c, c->rig};
  const int F = rig_n(u.rig) / 6;
  TRY(u.check_anchor(who, anchor));
  TRY(point_cov_sel_check(who, n_sel, sel, F, "free unknown"));
  TRY(point_cov_budget_check(who, F, c->N, n_sel, cov != nullptr));
  return block_point_covariance(u, who, base12, ext12, c_cov81, point_noise, include_fix != 0, anchor, n_sel, sel,
                                nullptr, cov, marg);
}

// ---------------- absolute pose priors (pose_graph.cu) ----------------
// The argument checks of balm_set_pose_priors and balm_spg_set_pose_priors over P poses (n_priors >= 1)
static int pose_priors_check(const char *who, int P, int n, const int32_t *pose, const double *hat12,
                             const double *lever3, const double *H36, const int32_t *kind, const double *scale) {
  const std::string w = std::string(who) + ": ";
  if (n < 0 || (n > 0 && (!pose || !hat12 || !H36))) { balm_set_error(w + "bad arguments"); return BALM_ERR_INVALID; }
  for (int q = 0; q < n; q++) {
    const std::string pq = w + "prior " + std::to_string(q);
    if (pose[q] < 0 || pose[q] >= P) { balm_set_error(pq + " names a pose outside [0, n_poses)"); return BALM_ERR_INVALID; }
    bool finite = true;
    for (int e = 0; e < 12; e++) finite = finite && std::isfinite(hat12[12 * (size_t)q + e]);
    for (int e = 0; lever3 && e < 3; e++) finite = finite && std::isfinite(lever3[3 * (size_t)q + e]);
    const double *Hq = H36 + 36 * (size_t)q;
    double hmax = 0.0;
    for (int e = 0; e < 36; e++) { finite = finite && std::isfinite(Hq[e]); hmax = std::max(hmax, fabs(Hq[e])); }
    if (!finite) { balm_set_error(pq + " has a non-finite pose_hat, lever arm or H"); return BALM_ERR_INVALID; }
    for (int a = 0; a < 6; a++)
      for (int c = 0; c < a; c++)
        if (fabs(Hq[6 * c + a] - Hq[6 * a + c]) > 1e-12 * hmax) {
          balm_set_error(pq + " has an H that is not symmetric");
          return BALM_ERR_INVALID;
        }
    if (kind) TRY(term_loss_check(pq, kind[q], scale ? scale + q : nullptr));
  }
  return BALM_OK;
}

// balm_set_pose_priors and balm_spg_set_pose_priors; `who` prefixes the messages
static int set_pose_priors(balm_ctx *c, const char *who, int n_priors, const int32_t *pose, const double *poses_hat12,
                           const double *lever3, const double *H36, const int32_t *kind, const double *scale,
                           int32_t *status_out) {
  TRY(pose_priors_check(who, c->N, n_priors, pose, poses_hat12, lever3, H36, kind, scale));
  CUDA_TRY(cudaSetDevice(c->device));
  PriorSet *pr = nullptr;
  std::vector<int> status;
  if (n_priors > 0)  // 0 detaches the prior set
    TRY(prior_set_build(c->stream, n_priors, pose, poses_hat12, lever3, H36, kind, scale, &status, &pr));
  std::unique_ptr<PriorSet, void (*)(PriorSet *)> pr_own(pr, prior_set_free);
  if (c->prec == BALM_PREC_BLOCKS && c->bh) TRY(blocks_set_priors(c, pr, who));
  if (status_out) std::copy(status.begin(), status.end(), status_out);
  prior_set_free(c->pr);
  c->pr = pr_own.release();
  return BALM_OK;
}

extern "C" int balm_set_pose_priors(balm_ctx *c, int n_priors, const int32_t *pose, const double *poses_hat12,
                                    const double *lever3, const double *H36, const int32_t *kind, const double *scale,
                                    int32_t *status_out) {
  if (!c) { balm_set_error("balm_set_pose_priors: bad arguments"); return BALM_ERR_INVALID; }
  return set_pose_priors(c, "balm_set_pose_priors", n_priors, pose, poses_hat12, lever3, H36, kind, scale, status_out);
}

extern "C" int balm_prior_residuals(balm_ctx *c, const double *poses12, double *s, double *w) {
  return set_residuals(c, &balm_ctx::pr, "balm_prior_residuals", "pose priors", poses12, s, w);
}

extern "C" int balm_set_joint_cost(balm_ctx *c, int on) {
  const char *who = "balm_set_joint_cost";
  if (!c) { balm_set_error(std::string(who) + ": bad arguments"); return BALM_ERR_INVALID; }
  if (c->prec == BALM_PREC_BLOCKS) {
    balm_set_error(std::string(who) + ": a BALM_PREC_BLOCKS context's voxel cost always holds its factors and priors");
    return BALM_ERR_INVALID;
  }
  if (c->world > 1 || c->comm) { balm_set_error(std::string(who) + ": single-GPU contexts only"); return BALM_ERR_INVALID; }
  if (on && !c->joint_fg) {
    CUDA_TRY(cudaSetDevice(c->device));
    TRY(dev_alloc(&c->joint_fg, (size_t)c->n + 1));
  }
  c->joint_cost = on != 0;
  return BALM_OK;
}

// ---------------- sliding window on the registered voxel set (assoc.cu) ----------------
// A sliding-window build of the batch (batch_marginalize_build, batch_append_build, window_push_build) run as its
// one-problem case into scratch buffers, then registered as the context's voxel set, with fix clusters when `fix` and
// octree keys when `keys`. An empty result is registered as an empty set when `empty` is null; otherwise the call is
// rejected with that message before anything is emitted, and the context keeps its registration.
static int ctx_window_step(balm_ctx *c, bool fix, bool keys, const char *empty,
                           const std::function<int(const WindowRegister &)> &build, int64_t *M_out, int64_t *K_out) {
  ScratchPool pool;
  int64_t M = 0, K = 0;
  WindowEmit dst{};
  const WindowRegister to_pool = [&](const int64_t *vp, const int64_t *op, WindowEmit *out) {
    M = vp[1];
    K = op[1];
    if (M == 0 && empty) { balm_set_error(empty); return (int)BALM_ERR_INVALID; }
    TRY(pool.get(&dst.row_ptr, (size_t)M + 1)); TRY(pool.get(&dst.pose_idx, (size_t)K));
    TRY(pool.get(&dst.obs, (size_t)K * 10)); TRY(pool.get(&dst.coe, (size_t)M));
    if (fix) TRY(pool.get(&dst.fix, (size_t)M * 10));
    if (keys) { TRY(pool.get(&dst.key, (size_t)M)); TRY(pool.get(&dst.layer, (size_t)M)); }
    *out = dst;
    return (int)BALM_OK;
  };
  TRY(build(to_pool));
  if (M == 0) {
    drop_keys(c);
    TRY(register_empty(c));
  } else {
    TRY(balm_set_voxels_dev(c, M, (const int64_t *)dst.row_ptr, dst.pose_idx, dst.obs, dst.fix, dst.coe, K));
    if (keys) {  // balm_set_voxels_dev dropped the previous ones
      TRY(dev_alloc(&c->vox_key, (size_t)M));
      TRY(dev_alloc(&c->vox_layer, (size_t)M));
      CUDA_TRY(cudaMemcpy(c->vox_key, dst.key, sizeof(unsigned long long) * M, cudaMemcpyDeviceToDevice));
      CUDA_TRY(cudaMemcpy(c->vox_layer, dst.layer, sizeof(int) * M, cudaMemcpyDeviceToDevice));
      c->has_keys = true;
    }
  }
  if (M_out) *M_out = M;
  if (K_out) *K_out = K;
  return BALM_OK;
}

// The context's registration as the sliding-window builds read it: one problem, observations SoA [10][Kp], fix SoA
// [10][M]. pose_ptr / voxel_ptr [2] receive the host tables it points into.
static BatchVoxels ctx_voxels(const balm_ctx *c, const double *poses12, int64_t *pose_ptr, int64_t *voxel_ptr) {
  pose_ptr[0] = voxel_ptr[0] = 0;
  pose_ptr[1] = c->N;
  voxel_ptr[1] = c->M;
  const bool keys = c->has_keys;
  return BatchVoxels{1, c->M, pose_ptr, voxel_ptr, nullptr, c->row_ptr, c->pose_idx, c->obs, c->Kp, 1, c->fix, c->M, 1,
                     c->coe, keys ? c->vox_key : nullptr, keys ? c->vox_layer : nullptr, poses12};
}

extern "C" int balm_marginalize(balm_ctx *c, int mg_size, const double *poses12, int min_ps, int64_t *n_voxels_out,
                                int64_t *n_obs_out) {
  if (!c || !poses12 || mg_size < 1 || mg_size >= c->N) { balm_set_error("balm_marginalize: bad arguments"); return BALM_ERR_INVALID; }
  if (!c->registered || c->M < 1) { balm_set_error("balm_marginalize: no voxels registered"); return BALM_ERR_INVALID; }
  CUDA_TRY(cudaSetDevice(c->device));
  CUDA_TRY(cudaMemcpyAsync(c->poses, poses12, sizeof(double) * 12 * c->N, cudaMemcpyHostToDevice, c->stream));
  int64_t pose_ptr[2], voxel_ptr[2];
  const BatchVoxels in = ctx_voxels(c, poses12, pose_ptr, voxel_ptr);
  return ctx_window_step(c, true, c->has_keys, "balm_marginalize: no voxel is left with two observing scans",
                         [&](const WindowRegister &reg) {
                           return batch_marginalize_build(c->stream, in, &mg_size, min_ps, reg, &c->launches);
                         },
                         n_voxels_out, n_obs_out);
}
extern "C" int balm_append_scan(balm_ctx *c, int64_t n_points, const float *xyz, const double *poses12, int slot,
                                int64_t *n_voxels_out, int64_t *n_obs_out, int64_t *n_matched_out) {
  if (!c || !xyz || !poses12 || n_points < 1 || n_points >= (1ll << 31) || slot < 0 || slot >= c->N) {
    balm_set_error("balm_append_scan: bad arguments");
    return BALM_ERR_INVALID;
  }
  if (!c->registered || c->M < 1 || !c->has_keys) {
    balm_set_error("balm_append_scan: needs a voxel set produced by balm_cut_voxels (octree keys)");
    return BALM_ERR_INVALID;
  }
  CUDA_TRY(cudaSetDevice(c->device));
  CUDA_TRY(cudaMemcpyAsync(c->poses, poses12, sizeof(double) * 12 * c->N, cudaMemcpyHostToDevice, c->stream));
  int64_t pose_ptr[2], voxel_ptr[2], matched = 0;
  const BatchVoxels in = ctx_voxels(c, poses12, pose_ptr, voxel_ptr);
  const int32_t scan = 0;
  const int64_t scan_ptr[2] = {0, n_points};
  TRY(ctx_window_step(c, c->fix != nullptr, true, "balm_append_scan: no plane voxel survives the re-judgement",
                      [&](const WindowRegister &reg) {
                        return batch_append_build(c->stream, in, c->assoc, &scan, &slot, scan_ptr, xyz, n_points, reg,
                                                  &matched, false, &c->launches);
                      },
                      n_voxels_out, n_obs_out));
  if (n_matched_out) *n_matched_out = matched;
  return BALM_OK;
}
extern "C" int balm_download_keys(balm_ctx *c, uint64_t *keys, int32_t *layers) {
  if (!c || !c->has_keys) { balm_set_error("balm_download_keys: the voxel set carries no octree keys"); return BALM_ERR_INVALID; }
  CUDA_TRY(cudaSetDevice(c->device));
  if (keys) CUDA_TRY(cudaMemcpy(keys, c->vox_key, sizeof(uint64_t) * (size_t)c->M, cudaMemcpyDeviceToHost));
  if (layers) CUDA_TRY(cudaMemcpy(layers, c->vox_layer, sizeof(int32_t) * (size_t)c->M, cudaMemcpyDeviceToHost));
  return BALM_OK;
}
extern "C" int balm_download_fix(balm_ctx *c, double *fix10) {
  if (!c || !fix10 || !c->registered) { balm_set_error("balm_download_fix: bad arguments"); return BALM_ERR_INVALID; }
  CUDA_TRY(cudaSetDevice(c->device));
  std::vector<double> soa((size_t)10 * c->M, 0.0);
  if (c->fix) CUDA_TRY(cudaMemcpy(soa.data(), c->fix, sizeof(double) * 10 * c->M, cudaMemcpyDeviceToHost));
  for (int64_t v = 0; v < c->M; v++)
    for (int q = 0; q < 10; q++) fix10[v * 10 + q] = soa[(size_t)q * c->M + v];
  return BALM_OK;
}

// ---------------- persistent sliding-window octree (assoc.cu) ----------------
// the one-problem case of the batch's window (window_*_build, internal.cuh)
static int window_check(balm_ctx *c, const char *fn, int win_count) {
  if (!c) { balm_set_error(std::string(fn) + ": bad arguments"); return BALM_ERR_INVALID; }
  if (!c->win) { balm_set_error(std::string(fn) + ": call balm_window_reset first"); return BALM_ERR_INVALID; }
  if (win_count < 1 || win_count > c->N) { balm_set_error(std::string(fn) + ": win_count must be in [1, N]"); return BALM_ERR_INVALID; }
  return BALM_OK;
}
extern "C" int balm_window_reset(balm_ctx *c, const balm_assoc_opts *opts) {
  if (!c) { balm_set_error("balm_window_reset: bad arguments"); return BALM_ERR_INVALID; }
  CUDA_TRY(cudaSetDevice(c->device));
  const balm_assoc_opts o = resolve_assoc_opts(opts);
  return window_reset_build(&c->win, "balm_window_reset", 1, &c->N, o, false);
}
extern "C" int balm_window_cut(balm_ctx *c, int64_t n_points, const float *xyz, const double *pose12, int slot) {
  TRY(window_check(c, "balm_window_cut", 1));
  if ((n_points > 0 && !xyz) || !pose12 || n_points < 0 || slot < 0 || slot >= c->N) {
    balm_set_error("balm_window_cut: bad arguments (slot must be in [0, N))");
    return BALM_ERR_INVALID;
  }
  if (n_points >= (1ll << 31)) {
    balm_set_error("balm_window_cut: bad point count (the window holds < 2^31 points)");
    return BALM_ERR_INVALID;
  }
  CUDA_TRY(cudaSetDevice(c->device));
  std::vector<double> poses((size_t)12 * c->N, 0.0);  // the scan's pose in row `slot`
  std::copy(pose12, pose12 + 12, poses.begin() + 12 * (size_t)slot);
  const int32_t scan = 0;
  const int64_t scan_ptr[2] = {0, n_points};
  return window_cut_build(c->stream, *c->win, "balm_window_cut", &scan, &slot, 1, scan_ptr, xyz, poses.data(),
                          &c->launches);
}
extern "C" int balm_window_recut(balm_ctx *c, int win_count) {
  TRY(window_check(c, "balm_window_recut", win_count));
  CUDA_TRY(cudaSetDevice(c->device));
  return window_recut_build(c->stream, *c->win, &win_count, &c->launches);
}
extern "C" int balm_window_marginalize(balm_ctx *c, int mg_size, const double *poses12, int win_count) {
  TRY(window_check(c, "balm_window_marginalize", win_count));
  if (mg_size < 1 || mg_size >= win_count) {
    balm_set_error("balm_window_marginalize: mg_size must be in [1, win_count)");
    return BALM_ERR_INVALID;
  }
  CUDA_TRY(cudaSetDevice(c->device));
  return window_marginalize_build(c->stream, *c->win, &mg_size, poses12, &win_count, &c->launches);
}
extern "C" int balm_window_push(balm_ctx *c, int win_count, int64_t *n_voxels_out, int64_t *n_obs_out) {
  TRY(window_check(c, "balm_window_push", win_count));
  CUDA_TRY(cudaSetDevice(c->device));
  return ctx_window_step(c, true, true, nullptr,
                         [&](const WindowRegister &reg) {
                           return window_push_build(c->stream, *c->win, &win_count, reg, &c->launches);
                         },
                         n_voxels_out, n_obs_out);
}

// ---------------- pose covariance (covariance.cu) ----------------
extern "C" int balm_pose_covariance(balm_ctx *c, const double *poses12, const double *c_cov81, double point_noise,
                                    int include_fix, double *Rcov_raw, double *Rcov) {
  if (!c || !poses12 || (!Rcov_raw && !Rcov)) { balm_set_error("balm_pose_covariance: bad arguments"); return BALM_ERR_INVALID; }
  TRY(refuse_blocks(c, "balm_pose_covariance"));
  if (!c->registered || c->M < 1) { balm_set_error("balm_pose_covariance: no voxels registered"); return BALM_ERR_INVALID; }
  if (c->world > 1) { balm_set_error("balm_pose_covariance: single-GPU contexts only"); return BALM_ERR_UNSUPPORTED; }
  return covariance(Unknowns{c, nullptr}, poses12, nullptr, c_cov81, point_noise, include_fix != 0, -1,
                    "balm_pose_covariance: H is singular (gauge freedom not fixed: no fix clusters in the Hessian)",
                    Rcov_raw, Rcov);
}

// ---------------- multi-GPU ----------------
extern "C" int balm_comm_unique_id(void *out128) {
  if (!out128) return BALM_ERR_INVALID;
  if (!g_nccl.load()) { balm_set_error("libnccl.so.2 not found"); return BALM_ERR_NCCL; }
  NcclDyn::uid_t id;
  const int rc = g_nccl.GetUniqueId(&id);
  if (rc != 0) { balm_set_error("ncclGetUniqueId failed"); return BALM_ERR_NCCL; }
  memcpy(out128, &id, 128);
  return BALM_OK;
}

extern "C" int balm_comm_init(balm_ctx *c, int rank, int world, const void *unique_id128) {
  if (!c || world < 1 || rank < 0 || rank >= world) { balm_set_error("balm_comm_init: bad arguments"); return BALM_ERR_INVALID; }
  TRY(refuse_blocks(c, "balm_comm_init"));
  if (world > 1 && c->joint_cost) {
    balm_set_error("balm_comm_init: the joint cost (balm_set_joint_cost) is single-GPU only; switch it off first");
    return BALM_ERR_INVALID;
  }
  c->rank = rank; c->world = world;
  if (world == 1) return BALM_OK;
  if (!unique_id128) { balm_set_error("balm_comm_init: unique id required"); return BALM_ERR_INVALID; }
  if (!g_nccl.load()) { balm_set_error("libnccl.so.2 not found"); return BALM_ERR_NCCL; }
  CUDA_TRY(cudaSetDevice(c->device));
  NcclDyn::uid_t id;
  memcpy(&id, unique_id128, 128);
  if (!c->Hpack) TRY(dev_alloc(&c->Hpack, (size_t)c->n * (c->n + 1) / 2 + c->n + 1));
  const int rc = g_nccl.CommInitRank(&c->comm, world, id, rank);
  if (rc != 0) {
    balm_set_error(std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "?"));
    return BALM_ERR_NCCL;
  }
  return BALM_OK;
}

// ---------------- instrumentation ----------------
extern "C" int balm_get_timings(balm_ctx *c, balm_timings *out) {
  if (!c || !out) return BALM_ERR_INVALID;
  *out = c->tm;
  out->launches = (int)c->launches;
  return BALM_OK;
}
extern "C" int balm_get_reused_sweeps(balm_ctx *c, int *out) {
  if (!c || !out) return BALM_ERR_INVALID;
  *out = c->reused_sweeps;
  return BALM_OK;
}
extern "C" int balm_reset_counters(balm_ctx *c) {
  if (!c) return BALM_ERR_INVALID;
  c->launches = 0;
  c->reused_sweeps = 0;
  c->tm = balm_timings{};
  return BALM_OK;
}
extern "C" int balm_sync(balm_ctx *c) {
  if (!c) return BALM_ERR_INVALID;
  CUDA_TRY(cudaSetDevice(c->device));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  return BALM_OK;
}
extern "C" int balm_timer_begin(balm_ctx *c) {
  if (!c) return BALM_ERR_INVALID;
  CUDA_TRY(cudaSetDevice(c->device));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  CUDA_TRY(cudaEventRecord(c->ev[11], c->stream));
  return BALM_OK;
}
extern "C" int balm_timer_end(balm_ctx *c, float *ms) {
  if (!c || !ms) return BALM_ERR_INVALID;
  cudaEvent_t e;
  CUDA_TRY(cudaEventCreate(&e));
  CUDA_TRY(cudaEventRecord(e, c->stream));
  CUDA_TRY(cudaEventSynchronize(e));
  CUDA_TRY(cudaEventElapsedTime(ms, c->ev[11], e));
  cudaEventDestroy(e);
  return BALM_OK;
}
// Debug aid (BALM_DAG_TRACE=1): timestamps of the last tile-DAG factorisation. out: 4*nt chain entries (step start,
// mini-panel inputs ready, diagonal block ready, step published; ns) followed by 3 per CTA (start, end, tasks).
extern "C" int balm_debug_dag_trace(balm_ctx *c, unsigned long long *out, int max_entries) {
  if (!c || !out || !c->lw.dag_trace) return BALM_ERR_INVALID;
  const int nt = (c->n + BALM_NB - 1) / BALM_NB;
  const int total = std::min(max_entries, 4 * nt + 8 * 1024);
  CUDA_TRY(cudaMemcpy(out, c->lw.dag_trace, sizeof(unsigned long long) * total, cudaMemcpyDeviceToHost));
  return BALM_OK;
}

extern "C" int balm_device_views(balm_ctx *c, double **H_dev, double **g_dev) {
  if (!c) return BALM_ERR_INVALID;
  TRY(refuse_blocks(c, "balm_device_views"));
  if (H_dev) *H_dev = c->H;
  if (g_dev) *g_dev = c->g;
  return BALM_OK;
}

// ---------------- block-sparse Hessian (blocks.cu) ----------------
extern "C" int balm_block_structure(balm_ctx *c, int64_t stats[4], int32_t *pairs) {
  if (!c || !stats) { balm_set_error("balm_block_structure: bad arguments"); return BALM_ERR_INVALID; }
  if (c->prec != BALM_PREC_BLOCKS || !c->bh) {
    balm_set_error("balm_block_structure: no voxels registered on a BALM_PREC_BLOCKS context");
    return BALM_ERR_INVALID;
  }
  const std::vector<int2> &pr = blocks_pairs(c->bh);
  stats[0] = (int64_t)pr.size();
  const size_t N = c->N, n = c->n, K = c->K, M = c->M;
  const size_t dbl = 18 * K + 10 * (size_t)c->Kp + (c->fix ? 10 * M : 0) + M + 2 * M * BALM_STATS_STRIDE + 10 * M +
                     (size_t)(c->obs_chunks + 2) * BALM_ACC * c->Np + 24 * N + 3 * n + 8 + 32 + c->res_blocks;
  const size_t ints = K + (M + 1) * 2 + 2 * N + 8 + (c->csc_ptr ? 2 * K + 3 * N + 1 : 0);
  stats[3] = blocks_bytes(c->bh, &stats[1], &stats[2]) + (int64_t)(sizeof(double) * dbl + sizeof(int) * ints) +
             (c->pg ? pose_graph_bytes(c->pg) : 0) + (c->pr ? prior_set_bytes(c->pr) : 0);
  if (pairs)
    for (size_t p = 0; p < pr.size(); p++) { pairs[2 * p] = pr[p].x; pairs[2 * p + 1] = pr[p].y; }
  return BALM_OK;
}

extern "C" int balm_download_blocks(balm_ctx *c, double *blocks) {
  if (!c || !blocks) { balm_set_error("balm_download_blocks: bad arguments"); return BALM_ERR_INVALID; }
  if (c->prec != BALM_PREC_BLOCKS || !c->bh) {
    balm_set_error("balm_download_blocks: no voxels registered on a BALM_PREC_BLOCKS context");
    return BALM_ERR_INVALID;
  }
  CUDA_TRY(cudaSetDevice(c->device));
  const size_t nbl = 36 * blocks_pairs(c->bh).size();
  CUDA_TRY(cudaMemcpyAsync(blocks, blocks_device(c->bh), sizeof(double) * nbl, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  return BALM_OK;
}

extern "C" int balm_block_covariance(balm_ctx *c, const double *poses12, int include_fix, int anchor, double *cov) {
  if (!c || !poses12 || !cov) { balm_set_error("balm_block_covariance: bad arguments"); return BALM_ERR_INVALID; }
  if (c->prec != BALM_PREC_BLOCKS || !c->bh || !c->registered) {
    balm_set_error("balm_block_covariance: no voxels registered on a BALM_PREC_BLOCKS context");
    return BALM_ERR_INVALID;
  }
  const Unknowns u{c, nullptr};
  TRY(u.check_anchor("balm_block_covariance", anchor));
  return block_covariance(u, "balm_block_covariance", poses12, nullptr, include_fix != 0, anchor, cov);
}

extern "C" int balm_block_point_covariance(balm_ctx *c, const double *poses12, const double *c_cov81, double point_noise,
                                           int include_fix, int anchor, int n_sel, const int32_t *sel,
                                           double *raw_blocks, double *cov, double *marg) {
  const char *who = "balm_block_point_covariance";
  if (!c || !poses12 || (!raw_blocks && !cov && !marg)) {
    balm_set_error(std::string(who) + ": bad arguments");
    return BALM_ERR_INVALID;
  }
  if (c->prec != BALM_PREC_BLOCKS || !c->bh || !c->registered || c->M < 1) {
    balm_set_error(std::string(who) + ": no voxels registered on a BALM_PREC_BLOCKS context");
    return BALM_ERR_INVALID;
  }
  if (c->world > 1 || c->comm) { balm_set_error(std::string(who) + ": single-GPU contexts only"); return BALM_ERR_INVALID; }
  const Unknowns u{c, nullptr};
  TRY(u.check_anchor(who, anchor));
  if (cov || marg) {
    TRY(point_cov_sel_check(who, n_sel, sel, c->N, "pose"));
    TRY(point_cov_budget_check(who, c->N, c->N, n_sel, cov != nullptr));
  }
  return block_point_covariance(u, who, poses12, nullptr, c_cov81, point_noise, include_fix != 0, anchor, n_sel, sel,
                                raw_blocks, cov, marg);
}

// ---------------- sparse pose graph (pose_graph.cu, pose_graph_sparse.cu, blocks.cu) ----------------
// A BALM_PREC_BLOCKS context without voxels whose pattern holds the factor pairs and the diagonal pair of every pose
// with an active prior, and no other diagonal pair. Each entry point makes its own checks, then runs the context's
// code.
struct balm_spg {
  balm_ctx *c = nullptr;
  ~balm_spg() { balm_destroy(c); }
};

// `who`'s refusal before the handle's first successful balm_spg_set_factors
static int spg_registered(const balm_spg *s, const char *who) {
  if (s->c->registered) return BALM_OK;
  balm_set_error(std::string(who) + ": no pose factors registered");
  return BALM_ERR_INVALID;
}

extern "C" int balm_spg_create(balm_spg **out, int n_poses, int device) {
  if (!out || n_poses < 1 || n_poses > (INT_MAX / 6 - 1)) { balm_set_error("balm_spg_create: bad arguments"); return BALM_ERR_INVALID; }
  *out = nullptr;
  std::unique_ptr<balm_spg> s(new balm_spg());
  const int rc = balm_create(&s->c, n_poses, device, BALM_PREC_BLOCKS);
  if (rc != BALM_OK) {
    balm_set_error("balm_spg_create: " + g_err);
    return rc;
  }
  s->c->every_diagonal = false;
  *out = s.release();
  return BALM_OK;
}

extern "C" void balm_spg_destroy(balm_spg *s) { delete s; }

extern "C" int balm_spg_set_factors(balm_spg *s, int n_factors, const int64_t *factor_ptr, const int32_t *factor_pose,
                                    const double *poses_hat12, const double *H, int32_t *status_out) {
  const char *who = "balm_spg_set_factors";
  if (!s) { balm_set_error(std::string(who) + ": bad arguments"); return BALM_ERR_INVALID; }
  TRY(pose_factors_check(who, s->c->N, n_factors, factor_ptr, factor_pose, poses_hat12, H));
  const bool first = !s->c->registered;  // the empty voxel set is registered after the factors: one pattern per call
  TRY(block_set_factors(s->c, who, n_factors, factor_ptr, factor_pose, poses_hat12, H, status_out));
  return first ? register_empty(s->c, who) : BALM_OK;
}

extern "C" int balm_spg_structure(balm_spg *s, int64_t stats[4], int32_t *pairs) {
  if (!s || !stats) { balm_set_error("balm_spg_structure: bad arguments"); return BALM_ERR_INVALID; }
  TRY(spg_registered(s, "balm_spg_structure"));
  return balm_block_structure(s->c, stats, pairs);
}

extern "C" int balm_spg_evaluate(balm_spg *s, const double *poses12, double *blocks, double *g, double *cost) {
  if (!s || !poses12) { balm_set_error("balm_spg_evaluate: bad arguments"); return BALM_ERR_INVALID; }
  TRY(spg_registered(s, "balm_spg_evaluate"));
  balm_ctx *c = s->c;
  CUDA_TRY(cudaSetDevice(c->device));
  CUDA_TRY(cudaMemcpyAsync(c->poses, poses12, sizeof(double) * 12 * c->N, cudaMemcpyHostToDevice, c->stream));
  c->defer = true;  // one wait: the evaluation's events are read after the copy-out's
  const int rc = evaluate_dev(c, c->poses, 0, 0, false);
  c->defer = false;
  TRY(rc);
  if (blocks) CUDA_TRY(cudaMemcpyAsync(blocks, blocks_device(c->bh), sizeof(double) * 36 * blocks_pairs(c->bh).size(),
                                       cudaMemcpyDeviceToHost, c->stream));
  if (g) CUDA_TRY(cudaMemcpyAsync(g, c->g, sizeof(double) * c->n, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->h_scal, c->scal, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  TRY(collect_eval(c));
  if (cost) *cost = c->h_scal[0];
  return BALM_OK;
}

extern "C" int balm_spg_iter(balm_spg *s, double *poses12, const balm_lm_opts *o, balm_trace *trace, int *n_iters,
                             double *poses_per_iter) {
  if (!s || !poses12 || !o) { balm_set_error("balm_spg_iter: bad arguments"); return BALM_ERR_INVALID; }
  if (n_iters) *n_iters = 0;
  TRY(spg_registered(s, "balm_spg_iter"));
  TRY(refuse_gauge_with_priors("balm_spg_iter", s->c->pr, o));
  balm_lm_opts lo = *o;
  lo.min_planes_per_pose = 0;  // no voxels
  lo.hess_includes_fix = 0;
  return balm_damping_iter(s->c, poses12, &lo, trace, n_iters, poses_per_iter);
}

extern "C" int balm_spg_covariance(balm_spg *s, const double *poses12, int anchor, double *cov) {
  if (!s || !poses12 || !cov) { balm_set_error("balm_spg_covariance: bad arguments"); return BALM_ERR_INVALID; }
  TRY(spg_registered(s, "balm_spg_covariance"));
  const Unknowns u{s->c, nullptr};
  TRY(u.check_anchor("balm_spg_covariance", anchor));
  return block_covariance(u, "balm_spg_covariance", poses12, nullptr, false, anchor, cov);
}

extern "C" int balm_spg_set_factor_loss(balm_spg *s, int n_factors, const int32_t *kind, const double *scale) {
  if (!s) { balm_set_error("balm_spg_set_factor_loss: bad arguments"); return BALM_ERR_INVALID; }
  TRY(spg_registered(s, "balm_spg_set_factor_loss"));
  CUDA_TRY(cudaSetDevice(s->c->device));
  return set_factor_loss("balm_spg_set_factor_loss", s->c->pg, s->c->stream, n_factors, kind, scale);
}

extern "C" int balm_spg_factor_residuals(balm_spg *s, const double *poses12, double *sf, double *w) {
  if (!s || !poses12) { balm_set_error("balm_spg_factor_residuals: bad arguments"); return BALM_ERR_INVALID; }
  TRY(spg_registered(s, "balm_spg_factor_residuals"));
  return balm_factor_residuals(s->c, poses12, sf, w);
}

extern "C" int balm_spg_set_pose_priors(balm_spg *s, int n_priors, const int32_t *pose, const double *poses_hat12,
                                        const double *lever3, const double *H36, const int32_t *kind,
                                        const double *scale, int32_t *status_out) {
  const char *who = "balm_spg_set_pose_priors";
  if (!s) { balm_set_error(std::string(who) + ": bad arguments"); return BALM_ERR_INVALID; }
  return set_pose_priors(s->c, who, n_priors, pose, poses_hat12, lever3, H36, kind, scale, status_out);
}

extern "C" int balm_spg_prior_residuals(balm_spg *s, const double *poses12, double *sp, double *w) {
  if (!s || !poses12) { balm_set_error("balm_spg_prior_residuals: bad arguments"); return BALM_ERR_INVALID; }
  if (!s->c->pr) { balm_set_error("balm_spg_prior_residuals: no pose priors registered"); return BALM_ERR_INVALID; }
  return balm_prior_residuals(s->c, poses12, sp, w);
}

// assoc.cu -- GPU association: point clouds + poses -> plane voxels (CSR of body-frame point clusters) directly in HBM.
//
// Restates the step that FEEDS the hot path (SURVEY.md section 8f, row N1):
//   cut_voxel                                  src/benchmark/bavoxel.hpp:1170-1223
//   OCTO_TREE_NODE::recut / judge_eigen / cut_func                     bavoxel.hpp:654-776
//   OCTO_TREE_NODE::tras_opt -> VOX_HESS::push_voxel                   bavoxel.hpp:908-929, 30-51
// The reference grows a pointer octree per root voxel on the CPU. Here every point gets a hierarchical 63-bit key
//   [root x | root y | root z | octant at layer 1 | octant at layer 2]     (19+19+19+3+3 bits, roots biased by 2^18)
// computed with the reference's own arithmetic (float32 voxel coordinate with the "-1 for negatives" rule, float
// voxel centres, child centre = centre +- quater_length), and the tree is evaluated level by level with radix sorts
// and segmented reductions: for each layer L the points are sorted by the key truncated to L digits (stable, frames
// stay ascending), (node, frame) segments are reduced to body-frame clusters (what push_voxel registers) and world-frame
// moments (what judge_eigen tests), nodes are judged planar / not planar, and a node becomes a plane voxel iff it is
// planar, has more than min_ps points and at least two observing frames, and every ancestor was large enough and NOT
// planar. All reductions run in a fixed order: the result is deterministic. Output order: ascending node key
// (digit 7 = "not split at this layer"), the order tests/assoc_ref.py uses.
//
// The same level loop serves a batch of independent problems (balm_batch_cut_voxels). Its items are the points of every
// problem in (problem, slot, point) order -- an index into the points uploaded once plus a pose row -- so a scan shared
// by two windows is read twice but stored once. Every sort is stable and ordered by (problem, key): each (problem, node,
// slot) segment is summed in the order a context holding only that problem would sum it, so each problem's voxels are
// bitwise those of balm_cut_voxels on its own points. One problem with rows = frames is balm_cut_voxels itself.
#include <cub/cub.cuh>
#include <string.h>
#include <algorithm>
#include <chrono>
#include <vector>
#include "internal.cuh"

namespace {

constexpr int ROOT_BITS = 19;
constexpr long long ROOT_BIAS = 1ll << 18;

struct AssocParams {
  double voxel_size;
  int layer_limit, min_ps;
  double eig[3];
};

__device__ __forceinline__ long long ref_voxel_index(double w, double vs) {
  float loc = (float)(w / vs);           // float loc_xyz[j] = pvec_tran[j] / voxel_size     (bavoxel.hpp:1180)
  if (loc < 0) loc -= 1.0f;              // :1181
  return (long long)loc;                 // (int64_t) cast truncates toward zero              (:1184)
}

// 63-bit key of a world point: root voxel (cut_voxel) + the octants cut_func would choose at layers 1 and 2
__device__ __forceinline__ unsigned long long world_point_key(const double *w, const AssocParams &p, int *bad);

// key of every item: its point (src) in the world frame of its pose row
__global__ void item_key_kernel(const float *xyz, const int *src, const int *row, const double *poses, int n_rows,
                                int64_t n, AssocParams p, unsigned long long *key, int *bad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int f = row[i];
  if (f < 0 || f >= n_rows) { atomicOr(bad, 2); f = 0; }
  double r[9], t[3];
  load_pose(poses + 12 * f, r, t);
  const int64_t j = src[i];
  const double b[3] = {(double)xyz[3 * j], (double)xyz[3 * j + 1], (double)xyz[3 * j + 2]};
  double w[3];
#pragma unroll
  for (int a = 0; a < 3; a++) w[a] = r[a * 3] * b[0] + r[a * 3 + 1] * b[1] + r[a * 3 + 2] * b[2] + t[a];
  key[i] = world_point_key(w, p, bad);
}

__device__ __forceinline__ unsigned long long world_point_key(const double *w, const AssocParams &p, int *bad) {
  unsigned long long k = 0;
  int oct1 = 0, oct2 = 0;
  const float quater = (float)(p.voxel_size / 4.0);  // ot->quater_length (:1216)
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const long long idx = ref_voxel_index(w[a], p.voxel_size);
    if (idx < -ROOT_BIAS || idx >= ROOT_BIAS) atomicOr(bad, 1);
    k = (k << ROOT_BITS) | (unsigned long long)((idx + ROOT_BIAS) & ((1ll << ROOT_BITS) - 1));
    const float c0 = (float)((0.5 + (double)idx) * p.voxel_size);  // float voxel_center (:1213-1215)
    const int b1 = w[a] > (double)c0 ? 1 : 0;                       // cut_func :711
    const float c1 = c0 + (float)(2 * b1 - 1) * quater;             // :717-719
    const int b2 = w[a] > (double)c1 ? 1 : 0;
    oct1 = (oct1 << 1) | b1;
    oct2 = (oct2 << 1) | b2;
  }
  return (k << 6) | (unsigned long long)(oct1 << 3) | (unsigned long long)oct2;
}

__global__ void iota_kernel(int *v, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) v[i] = (int)i;
}
__global__ void win_iota_kernel(int *v, int64_t n, int base) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) v[i] = base + (int)i;
}
// batch items: one CTA per pose row j, whose items [item_ptr[j], item_ptr[j+1]) are the points of its scan
__global__ void expand_rows_kernel(const long long *item_ptr, const long long *src_base, int *src, int *row) {
  const int j = blockIdx.x;
  const long long a = item_ptr[j], b = item_ptr[j + 1], s = src_base[j];
  for (long long e = a + threadIdx.x; e < b; e += blockDim.x) {
    src[e] = (int)(s + (e - a));
    row[e] = j;
  }
}
// digits below layer L forced to 7 ("not split")
__device__ __forceinline__ unsigned long long level_key(unsigned long long k, int L) {
  return L == 0 ? k | 63ull : (L == 1 ? k | 7ull : k);
}
__global__ void level_key_kernel(const unsigned long long *key, unsigned long long *out, int64_t n, int L) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = level_key(key[i], L);
}
__global__ void gather_prob_kernel(const int *idx, const int *row, const int *row_prob, unsigned *out, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (unsigned)row_prob[row[idx[i]]];
}
// a (problem, node, slot) segment starts where the level key or the pose row changes (rows belong to one problem)
__global__ void seg_flag_kernel(const unsigned long long *key, const int *idx, const int *row, int64_t n, int L, int *flag) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  flag[i] = (i == 0 || level_key(key[idx[i]], L) != level_key(key[idx[i - 1]], L) || row[idx[i]] != row[idx[i - 1]]) ? 1 : 0;
}
__global__ void seg_start_kernel(const int *flag, const int *scan, int64_t n, int *seg_start) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && flag[i]) seg_start[scan[i]] = (int)i;
}

// One thread per (problem, node, slot) segment: body-frame cluster (PointCluster::push, tools.hpp:311-316) and
// world-frame moments, accumulated in sorted order.
__global__ void seg_reduce_kernel(const float *xyz, const int *src, const int *row, const double *poses, const int *idx,
                                  const unsigned long long *key, int L, const int *seg_start, int nseg, int64_t n,
                                  double *segB, double *segW, int *seg_row, unsigned long long *seg_key) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nseg) return;
  const int64_t a = seg_start[s], b = (s + 1 < nseg) ? seg_start[s + 1] : n;
  const int f = row[idx[a]];
  double r[9], t[3];
  load_pose(poses + 12 * f, r, t);
  double B[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0}, W[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int64_t i = a; i < b; i++) {
    const int64_t j = src[idx[i]];
    const double x = xyz[3 * j], y = xyz[3 * j + 1], z = xyz[3 * j + 2];
    B[0] += x * x; B[1] += x * y; B[2] += x * z; B[3] += y * y; B[4] += y * z; B[5] += z * z;
    B[6] += x; B[7] += y; B[8] += z; B[9] += 1.0;
    const double wx = r[0] * x + r[1] * y + r[2] * z + t[0];
    const double wy = r[3] * x + r[4] * y + r[5] * z + t[1];
    const double wz = r[6] * x + r[7] * y + r[8] * z + t[2];
    W[0] += wx * wx; W[1] += wx * wy; W[2] += wx * wz; W[3] += wy * wy; W[4] += wy * wz; W[5] += wz * wz;
    W[6] += wx; W[7] += wy; W[8] += wz; W[9] += 1.0;
  }
#pragma unroll
  for (int c = 0; c < 10; c++) { segB[(size_t)c * nseg + s] = B[c]; segW[(size_t)c * nseg + s] = W[c]; }
  seg_row[s] = f;
  seg_key[s] = level_key(key[idx[a]], L);
}
__global__ void node_flag_kernel(const unsigned long long *seg_key, const int *seg_row, const int *row_prob, int nseg,
                                 int *flag) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < nseg)
    flag[s] = (s == 0 || seg_key[s] != seg_key[s - 1] || row_prob[seg_row[s]] != row_prob[seg_row[s - 1]]) ? 1 : 0;
}
// judge_eigen (bavoxel.hpp:654-699) on a world-frame cluster: lambda0 / lambda1 of its covariance below the layer's
// threshold (decision < eigen_value_array[layer], :665,697)
__device__ __forceinline__ bool cluster_planar(const double *W, double eig_thr) {
  const double inv = 1.0 / W[9];
  const double c0 = W[6] * inv, c1 = W[7] * inv, c2 = W[8] * inv;
  double lam[3], u0[3], u1[3], u2[3];
  eig3_jacobi(W[0] * inv - c0 * c0, W[1] * inv - c0 * c1, W[2] * inv - c0 * c2, W[3] * inv - c1 * c1,
              W[4] * inv - c1 * c2, W[5] * inv - c2 * c2, lam, u0, u1, u2);
  return lam[0] / lam[1] < eig_thr;
}
// One thread per (problem, node): total world moments over its slots -> judge_eigen (bavoxel.hpp:654-699)
__global__ void node_judge_kernel(const double *segW, const unsigned long long *seg_key, const int *seg_row,
                                  const int *row_prob, const int *node_start, int nnode, int nseg, double eig_thr,
                                  unsigned long long *node_key, int *node_prob, int *node_size, int *node_planar,
                                  int *node_nframes) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nnode) return;
  const int a = node_start[v], b = (v + 1 < nnode) ? node_start[v + 1] : nseg;
  double W[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int s = a; s < b; s++)
#pragma unroll
    for (int c = 0; c < 10; c++) W[c] += segW[(size_t)c * nseg + s];
  node_key[v] = seg_key[a];
  node_prob[v] = row_prob[seg_row[a]];
  node_size[v] = (int)(W[9] + 0.5);
  node_planar[v] = cluster_planar(W, eig_thr) ? 1 : 0;
  node_nframes[v] = b - a;
}

struct LevelTables {  // device arrays of one layer, nodes in ascending (problem, key)
  int nseg = 0, nnode = 0;
  double *segB = nullptr;          // [10][nseg] body-frame clusters
  int *seg_row = nullptr;          // [nseg] pose row
  int *node_start = nullptr;       // [nnode] first segment
  unsigned long long *node_key = nullptr;
  int *node_prob = nullptr, *node_size = nullptr, *node_planar = nullptr, *node_nframes = nullptr, *node_leaf = nullptr;
};

__device__ __forceinline__ int find_key(const unsigned long long *keys, int n, unsigned long long k) {
  int lo = 0, hi = n - 1;
  while (lo <= hi) {
    const int mid = (lo + hi) >> 1;
    const unsigned long long v = keys[mid];
    if (v == k) return mid;
    if (v < k) lo = mid + 1; else hi = mid - 1;
  }
  return -1;
}
// the same search on a table sorted by (problem, key)
__device__ __forceinline__ int find_node(const int *probs, const unsigned long long *keys, int n, int p,
                                         unsigned long long k) {
  int lo = 0, hi = n - 1;
  while (lo <= hi) {
    const int mid = (lo + hi) >> 1;
    const int q = probs[mid];
    const unsigned long long v = keys[mid];
    if (q == p && v == k) return mid;
    if (q < p || (q == p && v < k)) lo = mid + 1; else hi = mid - 1;
  }
  return -1;
}

struct AncestorTable {
  const unsigned long long *key;
  const int *prob, *size, *planar;
  int n;
};

// recut (bavoxel.hpp:737-776) evaluated per node: a node is reached iff every ancestor had more than min_ps points and
// failed the planarity test; it becomes a plane voxel iff it is planar with more than min_ps points (push_state = 1)
// and at least two frames observe it (push_voxel :37). Ancestors are looked up in the node's own problem.
__global__ void leaf_decide_kernel(int L, int nnode, const unsigned long long *key, const int *prob, const int *size,
                                   const int *planar, const int *nframes, AncestorTable t0, AncestorTable t1,
                                   int min_ps, int layer_limit, int *leaf) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nnode) return;
  bool reached = L <= layer_limit;
  if (reached && L >= 1) {
    const int r = find_node(t0.prob, t0.key, t0.n, prob[v], key[v] | 63ull);
    reached = r >= 0 && t0.size[r] > min_ps && !t0.planar[r];
  }
  if (reached && L >= 2) {
    const int r = find_node(t1.prob, t1.key, t1.n, prob[v], key[v] | 7ull);
    reached = r >= 0 && t1.size[r] > min_ps && !t1.planar[r];
  }
  leaf[v] = (reached && size[v] > min_ps && planar[v] && nframes[v] >= 2) ? 1 : 0;
}

__global__ void leaf_collect_kernel(int L, int nnode, const int *leaf, const int *leaf_scan, const unsigned long long *key,
                                    unsigned long long *out_key, int *out_ref, int base) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nnode || !leaf[v]) return;
  const int o = base + leaf_scan[v];
  out_key[o] = key[v];
  out_ref[o] = (L << 28) | v;  // layer and node id
}
// out[i] = the node table entry of leaf i (layer and node id in ref[i])
template <typename T>
__global__ void leaf_gather_kernel(const int *ref, int nleaf, const int *t0, const int *t1, const int *t2, T *out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nleaf) return;
  const int L = ref[i] >> 28, v = ref[i] & 0x0FFFFFFF;
  out[i] = (T)(L == 0 ? t0 : (L == 1 ? t1 : t2))[v];
}
// per problem b in [0, B]: its first leaf (leaves sorted by problem) and first observation
__global__ void prob_ptr_kernel(const unsigned *lprob, const int *cnt, const int *obs_start, int nleaf, int B,
                                long long *voxel_ptr, long long *obs_ptr) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > B) return;
  int lo = 0, hi = nleaf;
  while (lo < hi) { const int m = (lo + hi) >> 1; if ((int)lprob[m] < b) lo = m + 1; else hi = m; }
  voxel_ptr[b] = lo;
  obs_ptr[b] = lo < nleaf ? obs_start[lo] : (long long)obs_start[nleaf - 1] + cnt[nleaf - 1];
}
struct EmitLevel {
  const double *segB;
  const int *seg_row, *node_start, *node_size;
  const unsigned long long *node_key;
  int nseg;
};
// One CTA per plane voxel: its observations (slot = row_slot of the segment's pose row) into the registration's layout
__global__ void emit_kernel(const int *ref, const int *obs_start, int nleaf, EmitLevel e0, EmitLevel e1, EmitLevel e2,
                            const int *cnt, const int *row_slot, AssocEmit out) {
  const int i = blockIdx.x;
  if (i >= nleaf) return;
  const int L = ref[i] >> 28, v = ref[i] & 0x0FFFFFFF;
  const EmitLevel e = L == 0 ? e0 : (L == 1 ? e1 : e2);
  const int s0 = e.node_start[v], k = cnt[i], o0 = obs_start[i];
  for (int j = threadIdx.x; j < k; j += blockDim.x) {
#pragma unroll
    for (int c = 0; c < 10; c++)
      out.obs[(size_t)c * out.obs_cstride + (size_t)(o0 + j) * out.obs_ostride] = e.segB[(size_t)c * e.nseg + s0 + j];
    out.pose_idx[o0 + j] = row_slot[e.seg_row[s0 + j]];
  }
  if (threadIdx.x == 0) {
    out.row_ptr[i] = o0;
    out.coe[i] = (double)e.node_size[v];  // coe = sum of N over the window (bavoxel.hpp:42-44)
    out.key[i] = e.node_key[v];
    out.layer[i] = L;
    if (i == nleaf - 1) out.row_ptr[nleaf] = o0 + k;
  }
}

// bad: bit 2 = a frame index outside [0, n_rows), bit 1 = a point outside the root range (item_key_kernel)
int bad_points_error(const char *who, int bad) {
  balm_set_error(std::string(who) + (bad & 2 ? ": frame index outside [0, n_poses)"
                                             : ": a point lies outside the +-2^18 root-voxel range"));
  return BALM_ERR_INVALID;
}

}  // namespace

int assoc_cut(cudaStream_t st, const AssocInput &in, const balm_assoc_opts &o, const AssocRegister &reg,
              long long *launches) {
  const bool one = in.frame != nullptr;  // balm_cut_voxels: one problem, rows = frames
  const int B = one ? 1 : in.n_problems, n_rows = one ? in.n_rows : (int)in.pose_ptr[in.n_problems];
  const int64_t n = one ? in.n_points : in.n_items;
  ScratchPool pool(in.outer);
  AssocParams P{o.voxel_size, o.layer_limit, o.min_ps, {o.eigen_value_array[0], o.eigen_value_array[1], o.eigen_value_array[2]}};
  const float *xyz = in.xyz;
  float *dxyz = nullptr;
  double *poses = nullptr;
  int *src = nullptr, *row = nullptr, *row_slot = nullptr, *row_prob = nullptr, *bad = nullptr;
  if (!in.on_device) { TRY(pool.get(&dxyz, (size_t)3 * in.n_points)); xyz = dxyz; }
  TRY(pool.get(&poses, (size_t)12 * n_rows));
  TRY(pool.get(&src, (size_t)n)); TRY(pool.get(&row, (size_t)n)); TRY(pool.get(&bad, 1));
  TRY(pool.get(&row_slot, (size_t)2 * n_rows));
  row_prob = row_slot + n_rows;
  std::vector<int> hrow((size_t)2 * n_rows, 0);  // per pose row: slot in its problem, problem
  for (int p = 0; p < B; p++)
    for (int j = one ? 0 : (int)in.pose_ptr[p]; j < (one ? n_rows : (int)in.pose_ptr[p + 1]); j++) {
      hrow[j] = one ? j : j - (int)in.pose_ptr[p];
      hrow[(size_t)n_rows + j] = p;
    }
  if (in.n_points && !in.on_device)
    CUDA_TRY(cudaMemcpyAsync(dxyz, in.xyz, sizeof(float) * 3 * in.n_points, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(poses, in.poses12, sizeof(double) * 12 * n_rows, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(row_slot, hrow.data(), sizeof(int) * 2 * n_rows, cudaMemcpyHostToDevice, st));
  if (in.stats)
    in.stats->h2d_bytes += (in.on_device ? 0 : (int64_t)(sizeof(float) * 3 + (one ? sizeof(int) : 0)) * in.n_points) +
                           (int64_t)(sizeof(double) * 12 + sizeof(int) * 2) * n_rows;
  CUDA_TRY(cudaMemsetAsync(bad, 0, sizeof(int), st));
  int *flag = nullptr, *scan = nullptr, *seg_start = nullptr, *idx = nullptr, *work = nullptr, *work2 = nullptr;
  unsigned *pk = nullptr, *pk2 = nullptr;
  unsigned long long *key = nullptr, *keyL = nullptr, *keyL2 = nullptr;
  char *tmp = nullptr;
  size_t tmp_bytes = 0;
  const unsigned gb = (unsigned)((n + 255) / 256);
  int pbits = 1;
  while ((1 << pbits) < B) pbits++;
  if (n > 0) {
    TRY(pool.get(&flag, (size_t)n)); TRY(pool.get(&scan, (size_t)n)); TRY(pool.get(&seg_start, (size_t)n));
    TRY(pool.get(&idx, (size_t)n)); TRY(pool.get(&work, (size_t)n)); TRY(pool.get(&work2, (size_t)n));
    TRY(pool.get(&pk, (size_t)n)); TRY(pool.get(&pk2, (size_t)n));
    TRY(pool.get(&key, (size_t)n)); TRY(pool.get(&keyL, (size_t)n)); TRY(pool.get(&keyL2, (size_t)n));
    size_t tb1 = 0, tb2 = 0, tb3 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tb1, pk, pk2, idx, work, (int)n, 0, 32, st);
    cub::DeviceRadixSort::SortPairs(nullptr, tb2, keyL, keyL2, idx, work, (int)n, 0, 63, st);
    cub::DeviceScan::ExclusiveSum(nullptr, tb3, flag, scan, (int)n, st);
    tmp_bytes = std::max(tb1, std::max(tb2, tb3));
    TRY(pool.get(&tmp, tmp_bytes));
    if (one) {
      // items = the points in a stable order by frame, so that every later stable sort keeps the frames ascending
      // inside a node
      CUDA_TRY(cudaMemcpyAsync(pk, in.frame, sizeof(int) * n,
                               in.on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
      iota_kernel<<<gb, 256, 0, st>>>(idx, n);
      CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, pk, reinterpret_cast<unsigned *>(row), idx, src, (int)n,
                                               0, 32, st));
      *launches += 2;
    } else {
      // items in (problem, slot, point) order: frames are already ascending inside every problem
      std::vector<long long> tab((size_t)2 * n_rows + 1);  // item_ptr [n_rows + 1], then the first point of each row
      tab[0] = 0;
      for (int j = 0; j < n_rows; j++) {
        const int s = in.pose_scan[j];
        tab[j + 1] = tab[j] + (in.scan_ptr[s + 1] - in.scan_ptr[s]);
        tab[(size_t)n_rows + 1 + j] = in.scan_ptr[s];
      }
      long long *dtab = nullptr;
      TRY(pool.get(&dtab, tab.size()));
      CUDA_TRY(cudaMemcpyAsync(dtab, tab.data(), sizeof(long long) * tab.size(), cudaMemcpyHostToDevice, st));
      expand_rows_kernel<<<n_rows, 256, 0, st>>>(dtab, dtab + n_rows + 1, src, row);
      *launches += 1;
    }
    item_key_kernel<<<gb, 256, 0, st>>>(xyz, src, row, poses, n_rows, n, P, key, bad);
    *launches += 1;
  }

  LevelTables T[3];
  for (int L = 0; n > 0 && L <= o.layer_limit; L++) {
    // stable sort of the items by (problem, level key): by key, then by problem
    level_key_kernel<<<gb, 256, 0, st>>>(key, keyL, n, L);
    iota_kernel<<<gb, 256, 0, st>>>(idx, n);
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keyL, keyL2, idx, work, (int)n, 0, 63, st));
    if (B > 1) {
      gather_prob_kernel<<<gb, 256, 0, st>>>(work, row, row_prob, pk, n);
      CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, pk, pk2, work, work2, (int)n, 0, pbits, st));
      std::swap(work, work2);
      *launches += 2;
    }
    seg_flag_kernel<<<gb, 256, 0, st>>>(key, work, row, n, L, flag);
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, flag, scan, (int)n, st));
    int last_flag = 0, last_scan = 0;
    CUDA_TRY(cudaMemcpyAsync(&last_flag, flag + n - 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&last_scan, scan + n - 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    const int nseg = last_scan + last_flag;
    seg_start_kernel<<<gb, 256, 0, st>>>(flag, scan, n, seg_start);
    LevelTables &t = T[L];
    t.nseg = nseg;
    double *segW = nullptr;
    unsigned long long *seg_key = nullptr;
    int *nflag = nullptr, *nscan = nullptr;
    TRY(pool.get(&t.segB, (size_t)10 * nseg)); TRY(pool.get(&segW, (size_t)10 * nseg)); TRY(pool.get(&t.seg_row, (size_t)nseg));
    TRY(pool.get(&seg_key, (size_t)nseg)); TRY(pool.get(&nflag, (size_t)nseg)); TRY(pool.get(&nscan, (size_t)nseg));
    const unsigned gs = (unsigned)((nseg + 127) / 128);
    seg_reduce_kernel<<<gs, 128, 0, st>>>(xyz, src, row, poses, work, key, L, seg_start, nseg, n, t.segB, segW, t.seg_row,
                                          seg_key);
    node_flag_kernel<<<gs, 128, 0, st>>>(seg_key, t.seg_row, row_prob, nseg, nflag);
    size_t tb = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tb, nflag, nscan, nseg, st);
    if (tb > tmp_bytes) { pool.drop(tmp); tmp = nullptr; tmp_bytes = tb; TRY(pool.get(&tmp, tmp_bytes)); }
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, nflag, nscan, nseg, st));
    CUDA_TRY(cudaMemcpyAsync(&last_flag, nflag + nseg - 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&last_scan, nscan + nseg - 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    t.nnode = last_scan + last_flag;
    TRY(pool.get(&t.node_start, (size_t)t.nnode)); TRY(pool.get(&t.node_key, (size_t)t.nnode));
    TRY(pool.get(&t.node_prob, (size_t)t.nnode)); TRY(pool.get(&t.node_size, (size_t)t.nnode));
    TRY(pool.get(&t.node_planar, (size_t)t.nnode)); TRY(pool.get(&t.node_nframes, (size_t)t.nnode));
    TRY(pool.get(&t.node_leaf, (size_t)t.nnode));
    seg_start_kernel<<<gs, 128, 0, st>>>(nflag, nscan, nseg, t.node_start);
    node_judge_kernel<<<(unsigned)((t.nnode + 127) / 128), 128, 0, st>>>(
        segW, seg_key, t.seg_row, row_prob, t.node_start, t.nnode, nseg, P.eig[L], t.node_key, t.node_prob, t.node_size,
        t.node_planar, t.node_nframes);
    CUDA_TRY(cudaStreamSynchronize(st));
    pool.drop(segW); pool.drop(seg_key); pool.drop(nflag); pool.drop(nscan);
    *launches += 10;
  }
  int h_bad = 0;
  CUDA_TRY(cudaMemcpy(&h_bad, bad, sizeof(int), cudaMemcpyDeviceToHost));
  if (h_bad) return bad_points_error(in.who, h_bad);
  if (in.stats) in.stats->roots += T[0].nnode;  // layer-0 nodes of one problem: its root voxels

  // ---- leaves of every layer, merged in (problem, key) order ----
  int nleaf_L[3] = {0, 0, 0};
  int *lscan[3] = {nullptr, nullptr, nullptr};
  const AncestorTable a0{T[0].node_key, T[0].node_prob, T[0].node_size, T[0].node_planar, T[0].nnode};
  const AncestorTable a1{T[1].node_key, T[1].node_prob, T[1].node_size, T[1].node_planar, T[1].nnode};
  for (int L = 0; n > 0 && L <= o.layer_limit; L++) {
    LevelTables &t = T[L];
    leaf_decide_kernel<<<(unsigned)((t.nnode + 127) / 128), 128, 0, st>>>(
        L, t.nnode, t.node_key, t.node_prob, t.node_size, t.node_planar, t.node_nframes, a0, a1, o.min_ps, o.layer_limit,
        t.node_leaf);
    TRY(pool.get(&lscan[L], (size_t)t.nnode));
    size_t tb = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tb, t.node_leaf, lscan[L], t.nnode, st);
    if (tb > tmp_bytes) { pool.drop(tmp); tmp = nullptr; tmp_bytes = tb; TRY(pool.get(&tmp, tmp_bytes)); }
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, t.node_leaf, lscan[L], t.nnode, st));
    int a = 0, b = 0;
    CUDA_TRY(cudaMemcpyAsync(&a, t.node_leaf + t.nnode - 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&b, lscan[L] + t.nnode - 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    nleaf_L[L] = a + b;
  }
  const int nleaf = nleaf_L[0] + nleaf_L[1] + nleaf_L[2];
  std::vector<long long> hptr((size_t)2 * (B + 1), 0);  // voxel_ptr [B + 1], then obs_ptr [B + 1]
  int *lref = nullptr, *lcnt = nullptr, *lobs = nullptr;
  if (nleaf > 0) {
    unsigned long long *lkey = nullptr, *lkey2 = nullptr;
    int *lref2 = nullptr;
    long long *dptr = nullptr;
    TRY(pool.get(&lkey, (size_t)nleaf)); TRY(pool.get(&lkey2, (size_t)nleaf)); TRY(pool.get(&lref, (size_t)nleaf));
    TRY(pool.get(&lref2, (size_t)nleaf)); TRY(pool.get(&lcnt, (size_t)nleaf)); TRY(pool.get(&lobs, (size_t)nleaf));
    TRY(pool.get(&dptr, hptr.size()));
    int base = 0;
    for (int L = 0; L <= o.layer_limit; L++) {
      leaf_collect_kernel<<<(unsigned)((T[L].nnode + 127) / 128), 128, 0, st>>>(L, T[L].nnode, T[L].node_leaf, lscan[L],
                                                                               T[L].node_key, lkey, lref, base);
      base += nleaf_L[L];
    }
    const unsigned gl = (unsigned)((nleaf + 127) / 128);
    unsigned *lprob = pk, *lprob2 = pk2;  // the items' problem keys are free now (nleaf <= n)
    size_t tb = 0, tb2 = 0, tb3 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tb, lkey, lkey2, lref, lref2, nleaf, 0, 63, st);
    cub::DeviceRadixSort::SortPairs(nullptr, tb2, lprob, lprob2, lref, lref2, nleaf, 0, pbits, st);
    cub::DeviceScan::ExclusiveSum(nullptr, tb3, lcnt, lobs, nleaf, st);
    tb = std::max(tb, std::max(tb2, tb3));
    if (tb > tmp_bytes) { pool.drop(tmp); tmp = nullptr; tmp_bytes = tb; TRY(pool.get(&tmp, tmp_bytes)); }
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, lkey, lkey2, lref, lref2, nleaf, 0, 63, st));
    std::swap(lref, lref2);
    leaf_gather_kernel<unsigned><<<gl, 128, 0, st>>>(lref, nleaf, T[0].node_prob, T[1].node_prob, T[2].node_prob, lprob);
    if (B > 1) {
      CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, lprob, lprob2, lref, lref2, nleaf, 0, pbits, st));
      std::swap(lref, lref2);
      std::swap(lprob, lprob2);
    }
    leaf_gather_kernel<int><<<gl, 128, 0, st>>>(lref, nleaf, T[0].node_nframes, T[1].node_nframes, T[2].node_nframes, lcnt);
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, lcnt, lobs, nleaf, st));
    prob_ptr_kernel<<<(B + 128) / 128, 128, 0, st>>>(lprob, lcnt, lobs, nleaf, B, dptr, dptr + B + 1);
    CUDA_TRY(cudaMemcpyAsync(hptr.data(), dptr, sizeof(long long) * hptr.size(), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    *launches += 5 + 2 * (o.layer_limit + 1) + (B > 1 ? 1 : 0);
  }
  const int64_t K = hptr[2 * (size_t)B + 1];
  // ---- register: the caller allocates its arrays for M voxels and K observations; emit straight into them ----
  AssocEmit out{};
  TRY(reg(nleaf, K, reinterpret_cast<const int64_t *>(hptr.data()), reinterpret_cast<const int64_t *>(hptr.data() + B + 1),
           &out));
  if (nleaf > 0) {
    EmitLevel e[3];
    for (int L = 0; L < 3; L++)
      e[L] = EmitLevel{T[L].segB, T[L].seg_row, T[L].node_start, T[L].node_size, T[L].node_key, T[L].nseg};
    emit_kernel<<<nleaf, 64, 0, st>>>(lref, lobs, nleaf, e[0], e[1], e[2], lcnt, row_slot, out);
    *launches += 1;
  } else {
    CUDA_TRY(cudaMemsetAsync(out.row_ptr, 0, sizeof(long long), st));
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  CUDA_TRY(cudaGetLastError());
  // the pool's destructor frees every scratch buffer (level tables included)
  return BALM_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// balm_cut_voxels on inputs larger than BALM_ASSOC_BUDGET_MB: root-key slabs. Every decision about a plane voxel (its
// (node, frame) segment sums, the node judge, the ancestor lookups of leaf_decide_kernel, min_ps and the two-frame rule)
// depends only on the points of its root voxel, and the output is ordered by the key, whose top 57 bits are the root. So
// the points of a contiguous range of roots, kept in their input order, are cut on their own: the stable frame sort
// gives them the subsequence the full sort gives, every segment is summed over the same points in the same order, and
// the slabs' voxels, concatenated in root order, are the one-pass registration bit for bit (DESIGN.md section 7).
// A root-count pass streams the host points once and counts the points of every root; the plan closes a slab before the
// root that would take it over the cap; a selection pass per slab re-streams only the chunks whose root range overlaps
// the slab and compacts the slab's points, in input order, into device buffers that assoc_cut takes as they are.
namespace {

struct Float3 {
  float x, y, z;
};

__global__ void root_of_kernel(unsigned long long *key, int64_t n) {  // key -> its root voxel (the top 57 bits)
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) key[i] >>= 6;
}
__global__ void in_slab_kernel(const unsigned long long *key, int64_t n, unsigned long long lo, unsigned long long hi,
                               char *flag) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long r = key[i] >> 6;
  flag[i] = (r >= lo && r <= hi) ? 1 : 0;
}

// The host points in chunks of `chunk` points: stage(c, b) copies chunk c into pinned buffer b once the upload that
// read it last is done, upload(c, b) enqueues its copy into the device chunk. Two pinned buffers let the host copy of
// the next chunk run while the device works on this one.
struct PointRing {
  const AssocInput &in;
  int64_t chunk;
  float *hx[2] = {nullptr, nullptr};
  int *hf[2] = {nullptr, nullptr};
  cudaEvent_t ev[2] = {nullptr, nullptr};
  float *dx = nullptr;
  int *df = nullptr;
  PointRing(const AssocInput &i, int64_t c) : in(i), chunk(c) {}
  ~PointRing() {
    for (int b = 0; b < 2; b++) {
      if (ev[b]) cudaEventSynchronize(ev[b]);
      cudaFreeHost(hx[b]);
      cudaFreeHost(hf[b]);
      if (ev[b]) cudaEventDestroy(ev[b]);
    }
  }
  int init(ScratchPool &pool) {
    for (int b = 0; b < 2; b++) {
      CUDA_TRY(cudaHostAlloc((void **)&hx[b], sizeof(float) * 3 * chunk, cudaHostAllocDefault));
      CUDA_TRY(cudaHostAlloc((void **)&hf[b], sizeof(int) * chunk, cudaHostAllocDefault));
      CUDA_TRY(cudaEventCreateWithFlags(&ev[b], cudaEventDisableTiming));
    }
    TRY(pool.get(&dx, (size_t)3 * chunk));
    TRY(pool.get(&df, (size_t)chunk));
    return BALM_OK;
  }
  int64_t size(int64_t c) const { return std::min(chunk, in.n_points - c * chunk); }
  int stage(int64_t c, int b) {
    CUDA_TRY(cudaEventSynchronize(ev[b]));
    memcpy(hx[b], in.xyz + 3 * c * chunk, sizeof(float) * 3 * size(c));
    memcpy(hf[b], in.frame + c * chunk, sizeof(int) * size(c));
    return BALM_OK;
  }
  int upload(cudaStream_t st, int64_t c, int b, int64_t *h2d) {
    CUDA_TRY(cudaMemcpyAsync(dx, hx[b], sizeof(float) * 3 * size(c), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(df, hf[b], sizeof(int) * size(c), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaEventRecord(ev[b], st));
    *h2d += (int64_t)(sizeof(float) * 3 + sizeof(int)) * size(c);
    return BALM_OK;
  }
};

double now_ms() {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// cub scratch that grows on demand (pool-owned)
struct Tmp {
  ScratchPool &pool;
  char *p = nullptr;
  size_t bytes = 0;
  int need(size_t b) {
    if (b <= bytes) return BALM_OK;
    pool.drop(p);
    p = nullptr;
    bytes = b;
    return pool.get(&p, bytes);
  }
  void free() {
    pool.drop(p);
    p = nullptr;
    bytes = 0;
  }
};

}  // namespace

int64_t assoc_bytes_per_point(int layer_limit) {
  return 16                         // the slab's points and frames (xyz, frame)
         + 64                       // items: src row flag scan seg_start idx work work2 pk pk2 (4 B), key keyL keyL2 (8 B)
         + 16                       // radix sort scratch (alternate keys and values, digit histograms, look-back)
         + 120 * (layer_limit + 1)  // one segment per point per layer, kept to the emission: segB 80 + seg_row 4, node
                                    // tables 32 (start key prob size planar nframes leaf) + leaf scan 4
         + 96                       // one layer's transient segment tables: segW 80 + seg_key 8 + nflag 4 + nscan 4
         + 32                       // leaves: lkey lkey2 (8 B), lref lref2 lcnt lobs (4 B)
         + 112                      // the slab's emitted voxels: obs 80 + pose_idx 4 + row_ptr 8 + coe 8 + key 8 + layer 4
         + 9;                       // the slab path's chunk staging (cap / 8 points, at least 4096, at about 50 B
                                    // each) and the slab buffers' one chunk of room (16 B per chunk point)
}
int64_t assoc_bytes_fixed(int n_rows) {
  // poses twice (root pass and cut, 96 B per row each) and the row tables (8 B per row), plus 1 MiB for cub's tile
  // state, the small tables and the one-element minimum of every allocation
  return (int64_t)200 * n_rows + (1 << 20);
}

int assoc_cut_slabs(cudaStream_t st, const AssocInput &in, const balm_assoc_opts &o, size_t budget, int64_t cap,
                    ScratchPool &outer, SlabVoxels *out, CutSlabStats *stats, long long *launches) {
  const int n_rows = in.n_rows;
  const int64_t n = in.n_points;
  const AssocParams P{o.voxel_size, o.layer_limit, o.min_ps, {o.eigen_value_array[0], o.eigen_value_array[1], o.eigen_value_array[2]}};
  const int64_t chunk = std::min(n, std::max<int64_t>(4096, std::min<int64_t>(cap / 8, 1 << 23)));
  const int64_t n_chunks = (n + chunk - 1) / chunk;
  CutSlabStats S;
  const double t0 = now_ms();
  PointRing ring(in, chunk);
  TRY(ring.init(outer));
  double *poses = nullptr;
  int *iota = nullptr, *bad = nullptr, *d_num = nullptr;
  unsigned long long *key = nullptr, *key2 = nullptr;
  TRY(outer.get(&poses, (size_t)12 * n_rows)); TRY(outer.get(&iota, (size_t)ring.chunk)); TRY(outer.get(&bad, 1));
  TRY(outer.get(&d_num, 2)); TRY(outer.get(&key, (size_t)ring.chunk)); TRY(outer.get(&key2, (size_t)ring.chunk));
  CUDA_TRY(cudaMemcpyAsync(poses, in.poses12, sizeof(double) * 12 * n_rows, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemsetAsync(bad, 0, sizeof(int), st));
  S.h2d_bytes += (int64_t)sizeof(double) * 12 * n_rows;
  iota_kernel<<<(unsigned)((ring.chunk + 255) / 256), 256, 0, st>>>(iota, ring.chunk);
  *launches += 1;
  Tmp tmp{outer};

  // ---- root-count pass: (root, count) runs of every chunk merged into one table, sorted by root ----
  int64_t T = 0, tcap = 0;  // table entries and capacity (room for a chunk's runs after the table)
  unsigned long long *tk = nullptr, *sk = nullptr;
  long long *tc = nullptr, *sc = nullptr;
  std::vector<unsigned long long> cmin((size_t)n_chunks), cmax((size_t)n_chunks);
  int h_bad = 0;
  TRY(ring.stage(0, 0));
  for (int64_t c = 0; c < n_chunks; c++) {
    const int b = (int)(c & 1);
    const int64_t m = ring.size(c);
    const unsigned gm = (unsigned)((m + 255) / 256);
    TRY(ring.upload(st, c, b, &S.h2d_bytes));
    item_key_kernel<<<gm, 256, 0, st>>>(ring.dx, iota, ring.df, poses, n_rows, m, P, key, bad);
    *launches += 1;
    if (!h_bad) {  // once a point is bad the call fails: the rest of the pass only looks for a bad frame
      if (T + m > tcap) {  // grow the table (and its sort buffers) to hold this chunk's runs after it
        const int64_t ncap = std::max(2 * tcap, T + m);
        unsigned long long *nk = nullptr, *nsk = nullptr;
        long long *nc = nullptr, *nsc = nullptr;
        TRY(outer.get(&nk, (size_t)ncap)); TRY(outer.get(&nc, (size_t)ncap));
        TRY(outer.get(&nsk, (size_t)ncap)); TRY(outer.get(&nsc, (size_t)ncap));
        if (T) {
          CUDA_TRY(cudaMemcpyAsync(nk, tk, sizeof(unsigned long long) * T, cudaMemcpyDeviceToDevice, st));
          CUDA_TRY(cudaMemcpyAsync(nc, tc, sizeof(long long) * T, cudaMemcpyDeviceToDevice, st));
        }
        CUDA_TRY(cudaStreamSynchronize(st));
        outer.drop(tk); outer.drop(tc); outer.drop(sk); outer.drop(sc);
        tk = nk; tc = nc; sk = nsk; sc = nsc; tcap = ncap;
      }
      root_of_kernel<<<gm, 256, 0, st>>>(key, m);
      size_t b1 = 0, b2 = 0, b3 = 0, b4 = 0;
      cub::DeviceRadixSort::SortKeys(nullptr, b1, key, key2, (int)m, 0, 57, st);
      cub::DeviceRunLengthEncode::Encode(nullptr, b2, key2, tk + T, tc + T, d_num, (int)m, st);
      cub::DeviceRadixSort::SortPairs(nullptr, b3, tk, sk, tc, sc, (int)(T + m), 0, 57, st);
      cub::DeviceReduce::ReduceByKey(nullptr, b4, sk, tk, sc, tc, d_num + 1, cub::Sum(), (int)(T + m), st);
      TRY(tmp.need(std::max(std::max(b1, b2), std::max(b3, b4))));
      if (outer.bytes > budget) {
        balm_set_error(std::string(in.who) + ": the root table (" + std::to_string(T) +
                       " roots so far) does not fit BALM_ASSOC_BUDGET_MB (" + std::to_string(budget) + " bytes)");
        return BALM_ERR_UNSUPPORTED;
      }
      CUDA_TRY(cub::DeviceRadixSort::SortKeys(tmp.p, tmp.bytes, key, key2, (int)m, 0, 57, st));
      CUDA_TRY(cub::DeviceRunLengthEncode::Encode(tmp.p, tmp.bytes, key2, tk + T, tc + T, d_num, (int)m, st));
      int r = 0;
      CUDA_TRY(cudaMemcpyAsync(&r, d_num, sizeof(int), cudaMemcpyDeviceToHost, st));
      if (c + 1 < n_chunks) TRY(ring.stage(c + 1, b ^ 1));  // the host copy of the next chunk overlaps this one's work
      CUDA_TRY(cudaStreamSynchronize(st));
      CUDA_TRY(cudaMemcpy(&cmin[c], tk + T, sizeof(unsigned long long), cudaMemcpyDeviceToHost));
      CUDA_TRY(cudaMemcpy(&cmax[c], tk + T + r - 1, sizeof(unsigned long long), cudaMemcpyDeviceToHost));
      if (T > 0) {  // merge: sort table + runs by root, add the counts of equal roots
        CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp.p, tmp.bytes, tk, sk, tc, sc, (int)(T + r), 0, 57, st));
        CUDA_TRY(cub::DeviceReduce::ReduceByKey(tmp.p, tmp.bytes, sk, tk, sc, tc, d_num + 1, cub::Sum(), (int)(T + r), st));
        int t = 0;
        CUDA_TRY(cudaMemcpyAsync(&t, d_num + 1, sizeof(int), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        T = t;
        *launches += 2;
      } else {
        T = r;
      }
      *launches += 3;
    } else if (c + 1 < n_chunks) {
      TRY(ring.stage(c + 1, b ^ 1));
    }
    CUDA_TRY(cudaMemcpyAsync(&h_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
  }
  if (h_bad) return bad_points_error(in.who, h_bad);
  std::vector<unsigned long long> rkey((size_t)T);
  std::vector<long long> rcnt((size_t)T);
  CUDA_TRY(cudaMemcpy(rkey.data(), tk, sizeof(unsigned long long) * T, cudaMemcpyDeviceToHost));
  CUDA_TRY(cudaMemcpy(rcnt.data(), tc, sizeof(long long) * T, cudaMemcpyDeviceToHost));
  outer.drop(tk); outer.drop(tc); outer.drop(sk); outer.drop(sc);
  tmp.free();
  S.roots = T;
  S.ms_roots = now_ms() - t0;

  // ---- slab plan: roots in ascending order, a slab closed before the root that would take it over the cap ----
  std::vector<int64_t> slab_root{0};  // slab s holds the roots [slab_root[s], slab_root[s + 1])
  std::vector<int64_t> slab_pts;
  int64_t cur = 0;
  for (int64_t r = 0; r < T; r++) {
    if (rcnt[r] > cap) {
      balm_set_error(std::string(in.who) + ": a root voxel holds " + std::to_string(rcnt[r]) +
                     " points, more than the " + std::to_string(cap) + " points per slab BALM_ASSOC_BUDGET_MB allows");
      return BALM_ERR_UNSUPPORTED;
    }
    if (cur + rcnt[r] > cap) {
      slab_root.push_back(r);
      slab_pts.push_back(cur);
      cur = 0;
    }
    cur += rcnt[r];
  }
  slab_root.push_back(T);
  slab_pts.push_back(cur);
  S.slabs = (int64_t)slab_pts.size();
  S.max_slab = *std::max_element(slab_pts.begin(), slab_pts.end());

  // ---- per slab: select its points in input order, cut them, stage its voxels on the host ----
  char *flag = nullptr;
  TRY(outer.get(&flag, (size_t)ring.chunk));
  {
    size_t b1 = 0, b2 = 0;
    cub::DeviceSelect::Flagged(nullptr, b1, (const Float3 *)ring.dx, flag, (Float3 *)nullptr, d_num, (int)ring.chunk, st);
    cub::DeviceSelect::Flagged(nullptr, b2, ring.df, flag, (int *)nullptr, d_num + 1, (int)ring.chunk, st);
    TRY(tmp.need(std::max(b1, b2)));
  }
  SlabVoxels V;
  V.row_ptr.push_back(0);
  AssocStats ast;
  for (int64_t s = 0; s < S.slabs; s++) {
    const double ts = now_ms();
    const unsigned long long lo = rkey[slab_root[s]], hi = rkey[slab_root[s + 1] - 1];
    const int64_t pts = slab_pts[s];
    std::vector<int64_t> cs;
    for (int64_t c = 0; c < n_chunks; c++)
      if (cmax[c] >= lo && cmin[c] <= hi) cs.push_back(c);
    ScratchPool sp(&outer);
    float *sx = nullptr;
    int *sf = nullptr;
    // one chunk of room past the slab's count: a selection that disagreed with the root counts could not write out of
    // bounds before the check below catches it
    TRY(sp.get(&sx, (size_t)3 * (pts + ring.chunk))); TRY(sp.get(&sf, (size_t)(pts + ring.chunk)));
    int64_t filled = 0;
    TRY(ring.stage(cs[0], 0));
    for (size_t q = 0; q < cs.size(); q++) {
      const int b = (int)(q & 1);
      const int64_t m = ring.size(cs[q]);
      const unsigned gm = (unsigned)((m + 255) / 256);
      TRY(ring.upload(st, cs[q], b, &S.h2d_bytes));
      item_key_kernel<<<gm, 256, 0, st>>>(ring.dx, iota, ring.df, poses, n_rows, m, P, key, bad);
      in_slab_kernel<<<gm, 256, 0, st>>>(key, m, lo, hi, flag);
      CUDA_TRY(cub::DeviceSelect::Flagged(tmp.p, tmp.bytes, (const Float3 *)ring.dx, flag, (Float3 *)(sx + 3 * filled),
                                          d_num, (int)m, st));
      CUDA_TRY(cub::DeviceSelect::Flagged(tmp.p, tmp.bytes, ring.df, flag, sf + filled, d_num + 1, (int)m, st));
      *launches += 4;
      int got = 0;
      CUDA_TRY(cudaMemcpyAsync(&got, d_num, sizeof(int), cudaMemcpyDeviceToHost, st));
      if (q + 1 < cs.size()) TRY(ring.stage(cs[q + 1], b ^ 1));
      CUDA_TRY(cudaStreamSynchronize(st));
      filled += got;
      if (filled > pts) break;
    }
    if (filled != pts) {
      balm_set_error(std::string(in.who) + ": internal error: a slab's selection disagrees with its root counts");
      return BALM_ERR_CUDA;
    }
    const double tc0 = now_ms();
    S.ms_select += tc0 - ts;
    AssocInput sin = in;
    sin.n_points = sin.n_items = pts;
    sin.xyz = sx;
    sin.frame = sf;
    sin.on_device = true;
    sin.outer = &sp;
    sin.stats = &ast;
    // the slab's voxels land in slab-local device arrays (SoA observations, stride = the slab's K)
    double *eobs = nullptr, *ecoe = nullptr;
    int *epose = nullptr, *elayer = nullptr;
    long long *erow = nullptr;
    unsigned long long *ekey = nullptr;
    int64_t Ms = 0, Ks = 0;
    const AssocRegister reg = [&](int64_t M, int64_t K, const int64_t *, const int64_t *, AssocEmit *e) {
      Ms = M; Ks = K;
      TRY(sp.get(&eobs, (size_t)10 * K)); TRY(sp.get(&epose, (size_t)K)); TRY(sp.get(&erow, (size_t)M + 1));
      TRY(sp.get(&ecoe, (size_t)M)); TRY(sp.get(&ekey, (size_t)M)); TRY(sp.get(&elayer, (size_t)M));
      *e = AssocEmit{eobs, K, 1, epose, erow, ecoe, ekey, elayer};
      return (int)BALM_OK;
    };
    TRY(assoc_cut(st, sin, o, reg, launches));
    const int64_t M0 = V.M, K0 = V.K;
    V.M += Ms;
    V.K += Ks;
    V.row_ptr.resize((size_t)V.M + 1);
    V.pose_idx.resize((size_t)V.K);
    V.coe.resize((size_t)V.M);
    V.key.resize((size_t)V.M);
    V.layer.resize((size_t)V.M);
    for (int c = 0; c < 10; c++) V.obs[c].resize((size_t)V.K);
    CUDA_TRY(cudaMemcpy(V.row_ptr.data() + M0, erow, sizeof(long long) * (Ms + 1), cudaMemcpyDeviceToHost));
    for (int64_t v = M0; v <= V.M; v++) V.row_ptr[v] += K0;
    if (Ks) {
      CUDA_TRY(cudaMemcpy(V.pose_idx.data() + K0, epose, sizeof(int) * Ks, cudaMemcpyDeviceToHost));
      for (int c = 0; c < 10; c++)
        CUDA_TRY(cudaMemcpy(V.obs[c].data() + K0, eobs + (size_t)c * Ks, sizeof(double) * Ks, cudaMemcpyDeviceToHost));
    }
    if (Ms) {
      CUDA_TRY(cudaMemcpy(V.coe.data() + M0, ecoe, sizeof(double) * Ms, cudaMemcpyDeviceToHost));
      CUDA_TRY(cudaMemcpy(V.key.data() + M0, ekey, sizeof(unsigned long long) * Ms, cudaMemcpyDeviceToHost));
      CUDA_TRY(cudaMemcpy(V.layer.data() + M0, elayer, sizeof(int) * Ms, cudaMemcpyDeviceToHost));
    }
    S.ms_cut += now_ms() - tc0;
  }
  S.h2d_bytes += ast.h2d_bytes;
  *out = std::move(V);
  *stats = S;
  return BALM_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Keyframe merge of a batch (balm_batch_merge_scans): the items of the cut, (problem, slot, point), are moved into the
// body frame of their problem's slot 0 and reduced by down_sampling_voxel (tools.hpp:203-242) with a deterministic mean.
// Items are sorted stably by the 63-bit key [ix | iy | iz] (21 bits each, biased by 2^20), then stably by problem, so
// that a voxel's points keep their item order and every problem's voxels come out in ascending (ix, iy, iz).
namespace {

constexpr int KF_BITS = 21;
constexpr long long KF_BIAS = 1ll << 20;

// q = R_a^T (R_k b + t_k - t_a), every operation correctly rounded in this order (no contraction), rounded to float;
// with reduce, the down-sampling key of q, and the lowest problem with an index outside +-2^20 in *bad.
__global__ void merge_item_kernel(const float *xyz, const int *src, const int *row, const int *row_prob,
                                  const long long *pose_ptr, const double *poses, int64_t n, bool reduce, float vs,
                                  float *q, unsigned long long *key, int *bad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int f = row[i], p = row_prob[f];
  double r[9], t[3], ra[9], ta[3];
  load_pose(poses + 12 * (size_t)f, r, t);
  load_pose(poses + 12 * (size_t)pose_ptr[p], ra, ta);
  const int64_t j = src[i];
  const double b[3] = {(double)xyz[3 * j], (double)xyz[3 * j + 1], (double)xyz[3 * j + 2]};
  double d[3];
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const double w = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r[a * 3], b[0]), __dmul_rn(r[a * 3 + 1], b[1])),
                                         __dmul_rn(r[a * 3 + 2], b[2])), t[a]);
    d[a] = __dsub_rn(w, ta[a]);
  }
  unsigned long long k = 0;
  bool out = false;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const float qa = __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn(ra[a], d[0]), __dmul_rn(ra[3 + a], d[1])),
                                                 __dmul_rn(ra[6 + a], d[2])));
    q[3 * i + a] = qa;
    float loc = __fdiv_rn(qa, vs);  // the float32 quotient of tools.hpp:215-217, "-1 for negatives", truncated
    if (loc < 0) loc -= 1.0f;
    out |= !(loc > -(float)(KF_BIAS + 1) && loc < (float)KF_BIAS);  // catches NaN too
    const long long idx = out ? 0 : (long long)loc;
    k = (k << KF_BITS) | (unsigned long long)(idx + KF_BIAS);
  }
  if (!reduce) return;
  if (out) atomicMin(bad, p);
  key[i] = k;
}
// a (problem, voxel) segment starts where the key or the problem changes
__global__ void merge_flag_kernel(const unsigned long long *key, const int *idx, const int *row, const int *row_prob,
                                  int64_t n, int *flag) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  flag[i] = (i == 0 || key[idx[i]] != key[idx[i - 1]] || row_prob[row[idx[i]]] != row_prob[row[idx[i - 1]]]) ? 1 : 0;
}
// kf_ptr[p] = voxels of the problems below p: the voxel count before the first sorted item of a problem >= p (sorted
// problem ids in sprob; null when B = 1)
__global__ void merge_offsets_kernel(const unsigned *sprob, const int *flag, const int *scan, int64_t n, int B,
                                     long long *kf_ptr) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > B) return;
  int64_t lo = 0, hi = n;  // first position whose problem is >= p
  if (sprob) {
    while (lo < hi) {
      const int64_t m = (lo + hi) / 2;
      if ((int)sprob[m] < p) lo = m + 1; else hi = m;
    }
  } else {
    lo = p == 0 ? 0 : n;
  }
  kf_ptr[p] = lo < n ? scan[lo] : scan[n - 1] + flag[n - 1];
}
// one thread per (problem, voxel): the fp64 sum of its points in item order over the count, rounded to float
__global__ void merge_reduce_kernel(const float *q, const int *idx, const int *vstart, int nvox, int64_t n, float *out) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nvox) return;
  const int64_t a = vstart[v], b = v + 1 < nvox ? vstart[v + 1] : n;
  double s[3] = {0.0, 0.0, 0.0};
  for (int64_t e = a; e < b; e++) {
    const int64_t j = idx[e];
#pragma unroll
    for (int c = 0; c < 3; c++) s[c] = __dadd_rn(s[c], (double)q[3 * j + c]);
  }
#pragma unroll
  for (int c = 0; c < 3; c++) out[3 * (int64_t)v + c] = __double2float_rn(__ddiv_rn(s[c], (double)(b - a)));
}

}  // namespace

int merge_scans_build(cudaStream_t st, const MergeInput &in, int64_t *kf_ptr, float *kf_xyz, long long *launches) {
  const int B = in.n_problems, n_rows = (int)in.pose_ptr[B];
  const int64_t n = in.n_items;
  const bool reduce = in.voxel_size >= 0.001;
  std::vector<long long> tab((size_t)2 * n_rows + 1);  // item_ptr [n_rows + 1], then the first point of each row
  std::vector<int> hprob((size_t)n_rows);
  tab[0] = 0;
  for (int p = 0; p < B; p++)
    for (int64_t j = in.pose_ptr[p]; j < in.pose_ptr[p + 1]; j++) {
      const int s = in.pose_scan[j];
      tab[j + 1] = tab[j] + (in.scan_ptr[s + 1] - in.scan_ptr[s]);
      tab[(size_t)n_rows + 1 + j] = in.scan_ptr[s];
      hprob[j] = p;
    }
  std::vector<long long> hptr((size_t)B + 1);
  if (!reduce)  // no reduction: keyframe p is its items, in (slot, point) order
    for (int p = 0; p <= B; p++) hptr[p] = tab[in.pose_ptr[p]];
  if (n == 0) {
    if (reduce) std::fill(hptr.begin(), hptr.end(), 0ll);
    for (int p = 0; p <= B; p++) kf_ptr[p] = hptr[p];
    return BALM_OK;
  }
  ScratchPool pool;
  float *xyz = nullptr, *q = nullptr;
  double *poses = nullptr;
  long long *dtab = nullptr, *dpose_ptr = nullptr;
  int *src = nullptr, *row = nullptr, *row_prob = nullptr, *bad = nullptr;
  unsigned long long *key = nullptr;
  TRY(pool.get(&xyz, (size_t)3 * in.n_points)); TRY(pool.get(&poses, (size_t)12 * n_rows));
  TRY(pool.get(&dtab, tab.size())); TRY(pool.get(&dpose_ptr, (size_t)B + 1)); TRY(pool.get(&row_prob, (size_t)n_rows));
  TRY(pool.get(&src, (size_t)n)); TRY(pool.get(&row, (size_t)n)); TRY(pool.get(&q, (size_t)3 * n));
  TRY(pool.get(&bad, 1));
  if (reduce) TRY(pool.get(&key, (size_t)n));
  CUDA_TRY(cudaMemcpyAsync(xyz, in.xyz, sizeof(float) * 3 * in.n_points, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(poses, in.poses12, sizeof(double) * 12 * n_rows, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(dtab, tab.data(), sizeof(long long) * tab.size(), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(dpose_ptr, in.pose_ptr, sizeof(long long) * (B + 1), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(row_prob, hprob.data(), sizeof(int) * n_rows, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemsetAsync(bad, 0x7f, sizeof(int), st));  // 0x7f7f7f7f: no problem is that large
  const unsigned gb = (unsigned)((n + 255) / 256);
  expand_rows_kernel<<<n_rows, 256, 0, st>>>(dtab, dtab + n_rows + 1, src, row);
  merge_item_kernel<<<gb, 256, 0, st>>>(xyz, src, row, row_prob, dpose_ptr, poses, n, reduce, (float)in.voxel_size, q,
                                        key, bad);
  *launches += 2;
  if (!reduce) {
    CUDA_TRY(cudaMemcpyAsync(kf_xyz, q, sizeof(float) * 3 * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    CUDA_TRY(cudaGetLastError());
    for (int p = 0; p <= B; p++) kf_ptr[p] = hptr[p];
    return BALM_OK;
  }
  int *idx = nullptr, *work = nullptr, *work2 = nullptr, *flag = nullptr, *scan = nullptr;
  unsigned *pk = nullptr, *pk2 = nullptr;
  unsigned long long *key2 = nullptr;
  long long *dkf = nullptr;
  TRY(pool.get(&idx, (size_t)n)); TRY(pool.get(&work, (size_t)n)); TRY(pool.get(&work2, (size_t)n));
  TRY(pool.get(&flag, (size_t)n)); TRY(pool.get(&scan, (size_t)n)); TRY(pool.get(&key2, (size_t)n));
  TRY(pool.get(&pk, (size_t)n)); TRY(pool.get(&pk2, (size_t)n)); TRY(pool.get(&dkf, (size_t)B + 1));
  int pbits = 1;
  while ((1 << pbits) < B) pbits++;
  size_t tb1 = 0, tb2 = 0, tb3 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tb1, key, key2, idx, work, (int)n, 0, 3 * KF_BITS, st);
  cub::DeviceRadixSort::SortPairs(nullptr, tb2, pk, pk2, work, work2, (int)n, 0, pbits, st);
  cub::DeviceScan::ExclusiveSum(nullptr, tb3, flag, scan, (int)n, st);
  size_t tmp_bytes = std::max(tb1, std::max(tb2, tb3));
  char *tmp = nullptr;
  TRY(pool.get(&tmp, tmp_bytes));
  iota_kernel<<<gb, 256, 0, st>>>(idx, n);
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, key, key2, idx, work, (int)n, 0, 3 * KF_BITS, st));
  if (B > 1) {
    gather_prob_kernel<<<gb, 256, 0, st>>>(work, row, row_prob, pk, n);
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, pk, pk2, work, work2, (int)n, 0, pbits, st));
    std::swap(work, work2);
    *launches += 2;
  }
  merge_flag_kernel<<<gb, 256, 0, st>>>(key, work, row, row_prob, n, flag);
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, flag, scan, (int)n, st));
  int *vstart = work2;  // free after the sorts (n >= the voxel count)
  seg_start_kernel<<<gb, 256, 0, st>>>(flag, scan, n, vstart);
  merge_offsets_kernel<<<(B + 128) / 128, 128, 0, st>>>(B > 1 ? pk2 : nullptr, flag, scan, n, B, dkf);
  int h_bad = 0;
  CUDA_TRY(cudaMemcpyAsync(hptr.data(), dkf, sizeof(long long) * (B + 1), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(&h_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  *launches += 6;
  if (h_bad != 0x7f7f7f7f) {
    balm_set_error(std::string(in.who) + ": problem " + std::to_string(h_bad) +
                   ": a point's voxel index lies outside +-2^20 at this voxel_size");
    return BALM_ERR_INVALID;
  }
  const int nvox = (int)hptr[B];
  float *out = nullptr;
  TRY(pool.get(&out, (size_t)3 * nvox));
  merge_reduce_kernel<<<(unsigned)((nvox + 127) / 128), 128, 0, st>>>(q, work, vstart, nvox, n, out);
  *launches += 1;
  CUDA_TRY(cudaMemcpyAsync(kf_xyz, out, sizeof(float) * 3 * nvox, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  CUDA_TRY(cudaGetLastError());
  for (int p = 0; p <= B; p++) kf_ptr[p] = hptr[p];
  return BALM_OK;
}


// ---------------------------------------------------------------------------------------------------------------------
// Pose-major observation lists of a sparse co-visibility problem (the reference walks a voxel's win_size slots and
// skips the empty ones, bavoxel.hpp:332,365-366,404-408; here the observation sweep runs lane = pose and needs, per pose,
// the list of its observations in ascending voxel order). Built on the device: stable radix sort of the observation
// indices by pose (CSR order is voxel-major, so a stable sort leaves every pose's list voxel-ascending), plus the
// voxel of every observation. planes_host: per-pose counts (already on the host for the >= 20 planes guard).
namespace {
__global__ void obs_voxel_kernel(const long long *row_ptr, int64_t M, int *vox_of_obs) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= M) return;
  for (long long s = row_ptr[v]; s < row_ptr[v + 1]; s++) vox_of_obs[s] = (int)v;
}
__global__ void gather_int_kernel(const int *src, const int *idx, int *dst, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[idx[i]];
}
// one thread per pose: [lo, hi) = the part of its list whose voxels lie in [v0, v1)
__global__ void csc_batch_kernel(const int *csc_ptr, const int *csc_vox, int N, int v0, int v1, int *lo, int *hi) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int b = csc_ptr[i], e = csc_ptr[i + 1];
  int l = b, h = e;
  while (l < h) { const int m = (l + h) >> 1; if (csc_vox[m] < v0) l = m + 1; else h = m; }
  lo[i] = l;
  h = e;
  while (l < h) { const int m = (l + h) >> 1; if (csc_vox[m] < v1) l = m + 1; else h = m; }
  hi[i] = l;
}
}  // namespace

int build_pose_major_lists(balm_ctx *c, const int *planes_host) {
  const int N = c->N;
  const int64_t K = c->K, M = c->M;
  cudaStream_t st = c->stream;
  ScratchPool pool;
  std::vector<int> ptr((size_t)N + 1, 0);
  for (int i = 0; i < N; i++) ptr[i + 1] = ptr[i] + planes_host[i];
  c->csc_max_len = 0;
  for (int i = 0; i < N; i++) c->csc_max_len = std::max(c->csc_max_len, planes_host[i]);
  CUDA_TRY(cudaMalloc((void **)&c->csc_ptr, sizeof(int) * ((size_t)N + 1)));
  CUDA_TRY(cudaMalloc((void **)&c->csc_obs, sizeof(int) * (size_t)K));
  CUDA_TRY(cudaMalloc((void **)&c->csc_vox, sizeof(int) * (size_t)K));
  CUDA_TRY(cudaMalloc((void **)&c->csc_lo, sizeof(int) * (size_t)N));
  CUDA_TRY(cudaMalloc((void **)&c->csc_hi, sizeof(int) * (size_t)N));
  CUDA_TRY(cudaMemcpyAsync(c->csc_ptr, ptr.data(), sizeof(int) * ((size_t)N + 1), cudaMemcpyHostToDevice, st));
  int *vox = nullptr, *idx = nullptr, *keys = nullptr, *keys2 = nullptr;
  TRY(pool.get(&vox, (size_t)K)); TRY(pool.get(&idx, (size_t)K)); TRY(pool.get(&keys, (size_t)K)); TRY(pool.get(&keys2, (size_t)K));
  obs_voxel_kernel<<<(unsigned)((M + 127) / 128), 128, 0, st>>>(c->row_ptr, M, vox);
  iota_kernel<<<(unsigned)((K + 255) / 256), 256, 0, st>>>(idx, K);
  CUDA_TRY(cudaMemcpyAsync(keys, c->pose_idx, sizeof(int) * (size_t)K, cudaMemcpyDeviceToDevice, st));
  int bits = 1;
  while ((1 << bits) < N) bits++;
  size_t tb = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tb, keys, keys2, idx, c->csc_obs, (int)K, 0, bits, st);
  char *tmp = nullptr;
  TRY(pool.get(&tmp, tb));
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tb, keys, keys2, idx, c->csc_obs, (int)K, 0, bits, st));
  gather_int_kernel<<<(unsigned)((K + 255) / 256), 256, 0, st>>>(vox, c->csc_obs, c->csc_vox, K);
  CUDA_TRY(cudaStreamSynchronize(st));
  CUDA_TRY(cudaGetLastError());
  c->launches += 4;
  return launch_csc_batch(c, 0, M);
}

int launch_csc_batch(balm_ctx *c, int64_t v0, int64_t v1) {
  if (c->dense || !c->csc_ptr) return BALM_OK;
  csc_batch_kernel<<<(c->N + 127) / 128, 128, 0, c->stream>>>(c->csc_ptr, c->csc_vox, c->N, (int)v0, (int)v1, c->csc_lo, c->csc_hi);
  c->launches += 1;
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}


// ---------------------------------------------------------------------------------------------------------------------
// Sliding-window marginalisation on the registered voxel set (SURVEY.md 8f row N2):
//   OCTO_TREE_NODE::to_margi (bavoxel.hpp:778-816) on every plane leaf -- the clusters of the oldest mg_size scans,
//   transformed by their (optimised) poses, are folded into the leaf's fix_point when fix_point.N < 50 (:790-795), the
//   remaining scans shift down by mg_size (:797-803) -- followed by what tras_opt / push_voxel keep of the leaf
//   (bavoxel.hpp:908-929: fewer than min_ps points left -> not pushed; :32-37: fewer than 2 observing scans -> not pushed;
//   coe = number of points left, :42-44).
// The flattened voxel set has no octree any more, so a leaf that is not pushed is dropped together with its fix cluster
// (in the reference it stays in the map for later scans); documented in DESIGN.md.
//
// Both steps have one implementation, batch_marginalize_build / batch_append_build below, for the B problems of a batch
// (balm_batch_marginalize / balm_batch_append_scan, observations and fix AoS [n][10]); a context's balm_marginalize /
// balm_append_scan is its one-problem case (observations SoA [10][Kp], fix SoA [10][M]). The kernels read either layout
// through a Strided view and run the same arithmetic in the same order, so a batch problem is bitwise what a context
// holding it alone computes.
namespace {
struct Strided {  // column c of row s at p[c * cs + s * rs]; p may be null (a missing fix set reads as zeros)
  const double *p;
  int64_t cs, rs;
  __device__ __forceinline__ double operator()(int64_t s, int c) const { return p ? p[c * cs + s * rs] : 0.0; }
};
__device__ __forceinline__ void add_world(double *f, const double *ob, const double *pose12) {
  double r[9], t[3];
  load_pose(pose12, r, t);
  const WC w = world_cluster(ob, r, t);
  f[0] += w.p00; f[1] += w.p01; f[2] += w.p02; f[3] += w.p11; f[4] += w.p12; f[5] += w.p22;
  f[6] += w.v0; f[7] += w.v1; f[8] += w.v2; f[9] += w.n;
}

// keep rule of marginalisation (tras_opt / push_voxel after to_margi): the voxel's observations of slots >= mg must hold
// at least min_ps points and come from at least two scans; *k = their number
__device__ __forceinline__ int marg_keep(const long long *row_ptr, const int *pose_idx, Strided obs, int64_t v, int mg,
                                         int min_ps, int *k) {
  int n = 0;
  double pts = 0.0;
  for (long long s = row_ptr[v]; s < row_ptr[v + 1]; s++)
    if (pose_idx[s] >= mg) { n++; pts += obs(s, 9); }
  *k = n;
  return ((int)pts >= min_ps && n >= 2) ? 1 : 0;
}
// to_margi on a kept voxel: observations of slots < mg folded into the fix cluster (written to fix_out[10]) unless it
// already holds 50 points, the others moved to rows o.. with their slots shifted down by mg. Returns the points left.
__device__ __forceinline__ double marg_emit(const long long *row_ptr, const int *pose_idx, Strided obs, Strided fix,
                                            int64_t v, const double *poses, int mg, long long o, int *pose_idx_out,
                                            double *obs10_out, double *fix_out) {
  double f[10];
  for (int c = 0; c < 10; c++) f[c] = fix(v, c);
  const bool absorb = (int)f[9] < 50;  // fix_point.N < 50 (bavoxel.hpp:790; push_state == 1 for a registered plane leaf)
  double pts = 0.0;
  for (long long s = row_ptr[v]; s < row_ptr[v + 1]; s++) {
    double ob[10];
    for (int c = 0; c < 10; c++) ob[c] = obs(s, c);
    const int p = pose_idx[s];
    if (p < mg) {
      if (absorb) add_world(f, ob, poses + 12 * p);  // fix_point += sig_tran[i]  (transform: tools.hpp:333-339)
    } else {
      for (int c = 0; c < 10; c++) obs10_out[o * 10 + c] = ob[c];
      pose_idx_out[o] = p - mg;
      pts += ob[9];
      o++;
    }
  }
  for (int c = 0; c < 10; c++) fix_out[c] = f[c];
  return pts;
}
}  // namespace


// ---------------------------------------------------------------------------------------------------------------------
// Appending a scan to the voxel set in HBM (the other half of the sliding window, SURVEY.md 8f row N2).
// Reference: cut_voxel pushes the new scan's points into the root voxels (bavoxel.hpp:1170-1223), recut hands them down
// to the leaves (cut_func(win_count-1) on split nodes, :737-776) and RE-JUDGES every leaf with its fix cluster and all
// window clusters (judge_eigen, :654-699): still planar with more than min_ps window points -> pushed again with the new
// observation; otherwise the reference splits it further or freezes it. Here: every new point finds the leaf that contains
// it through the stored keys (the same arithmetic as balm_cut_voxels), its body-frame moments become a new observation
// in pose slot `slot`, and every voxel is re-judged from fix + all its clusters transformed by the current poses; a voxel
// that fails (not planar any more, too few points, fewer than two scans) is dropped. NOT done (documented): creating new
// roots / new leaves from points that fall outside the existing planes, and re-splitting a leaf that stopped being planar
// -- both appear at the next full balm_cut_voxels.
namespace {
// the registered voxel (index into keys[0 .. n), ascending) a body-frame point falls into at pose12, or -1
__device__ __forceinline__ int append_match(const float *xyz, int64_t i, const double *pose12, const AssocParams &p,
                                            const unsigned long long *vox_key, const int *vox_layer, int n) {
  double r[9], t[3];
  load_pose(pose12, r, t);
  const double b[3] = {(double)xyz[3 * i], (double)xyz[3 * i + 1], (double)xyz[3 * i + 2]};
  double w[3];
#pragma unroll
  for (int a = 0; a < 3; a++) w[a] = r[a * 3] * b[0] + r[a * 3 + 1] * b[1] + r[a * 3 + 2] * b[2] + t[a];
  int dummy = 0;
  const unsigned long long k = world_point_key(w, p, &dummy);
  // a key digit 7 means "not split" AND is octant 7, so a hit only counts when the voxel's layer agrees
  int v = find_key(vox_key, n, k | 63ull);            // a layer-0 leaf (the whole root voxel is one plane)
  if (v >= 0 && vox_layer[v] != 0) v = -1;
  if (v < 0) { v = find_key(vox_key, n, k | 7ull); if (v >= 0 && vox_layer[v] != 1) v = -1; }   // a layer-1 leaf
  if (v < 0) { v = find_key(vox_key, n, k); if (v >= 0 && vox_layer[v] != 2) v = -1; }          // a layer-2 leaf
  return v;
}
// the new scan's body-frame cluster of the voxel whose points have id `want` in vid_sorted (stable-sorted, so the
// points sum in their original order; pt_sorted: their indices into xyz)
__device__ __forceinline__ void append_cluster(const float *xyz, const unsigned *vid_sorted, const int *pt_sorted,
                                               int64_t n, unsigned want, double *out10) {
  int64_t lo = 0, hi = n;
  while (lo < hi) { const int64_t m = (lo + hi) >> 1; if (vid_sorted[m] < want) lo = m + 1; else hi = m; }
  double B[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int64_t i = lo; i < n && vid_sorted[i] == want; i++) {
    const int64_t j = pt_sorted[i];  // 3 j overflows 32 bits beyond 715 827 882 points (a batch's scan pool)
    const double x = xyz[3 * j], y = xyz[3 * j + 1], z = xyz[3 * j + 2];
    B[0] += x * x; B[1] += x * y; B[2] += x * z; B[3] += y * y; B[4] += y * z; B[5] += z * z;
    B[6] += x; B[7] += y; B[8] += z; B[9] += 1.0;
  }
#pragma unroll
  for (int q = 0; q < 10; q++) out10[q] = B[q];
}
// recut's re-judgement of a voxel: judge_eigen on fix + every window cluster (old ones and the new one nb) at the
// current poses; keep iff planar, more than min_ps window points and at least two scans (*k of them). *slot_bad: a scan
// already in the voxel does not lie below `slot`.
__device__ __forceinline__ int append_judge(const long long *row_ptr, const int *pose_idx, Strided obs, Strided fix,
                                            int64_t v, const double *poses, const double *nb, int slot, int layer,
                                            const AssocParams &p, int *k_out, bool *slot_bad) {
  double W[10];
  for (int q = 0; q < 10; q++) W[q] = fix(v, q);
  double pts = 0.0;
  int k = 0;
  bool bad = false;
  for (long long s = row_ptr[v]; s < row_ptr[v + 1]; s++) {
    double ob[10];
    for (int q = 0; q < 10; q++) ob[q] = obs(s, q);
    add_world(W, ob, poses + 12 * pose_idx[s]);
    pts += ob[9];
    k++;
    bad |= pose_idx[s] >= slot;  // the new scan must take a slot above every scan already in the voxel
  }
  if (nb[9] > 0.0) {
    add_world(W, nb, poses + 12 * slot);
    pts += nb[9];
    k++;
  }
  const double inv = 1.0 / W[9];
  const double c0 = W[6] * inv, c1 = W[7] * inv, c2 = W[8] * inv;
  double lam[3], u0[3], u1[3], u2[3];
  eig3_jacobi(W[0] * inv - c0 * c0, W[1] * inv - c0 * c1, W[2] * inv - c0 * c2, W[3] * inv - c1 * c1,
              W[4] * inv - c1 * c2, W[5] * inv - c2 * c2, lam, u0, u1, u2);
  const bool planar = lam[0] / lam[1] < p.eig[layer];                     // judge_eigen (:665,697)
  *k_out = k;
  *slot_bad = bad;
  return (planar && (int)pts > p.min_ps && k >= 2) ? 1 : 0;              // recut :755-757, push_voxel :37
}
// a kept voxel with its new observation nb (if any points) in slot `slot`, from row o on; fix row copied (unless fix_out
// is null), coe grown
__device__ __forceinline__ void append_emit(const long long *row_ptr, const int *pose_idx, Strided obs, Strided fix,
                                            const double *coe, int64_t v, const double *nb, int slot, long long o,
                                            int *pose_idx_out, double *obs10_out, double *fix_out, double *coe_out) {
  for (long long s = row_ptr[v]; s < row_ptr[v + 1]; s++, o++) {
    for (int q = 0; q < 10; q++) obs10_out[o * 10 + q] = obs(s, q);
    pose_idx_out[o] = pose_idx[s];
  }
  if (nb[9] > 0.0) {
    for (int q = 0; q < 10; q++) obs10_out[o * 10 + q] = nb[q];
    pose_idx_out[o] = slot;
  }
  if (fix_out)
    for (int q = 0; q < 10; q++) fix_out[q] = fix(v, q);
  *coe_out = coe[v] + nb[9];  // push_voxel: coe = sum of N over the window (:42-44)
}

// one thread per voxel: the new scan's body-frame cluster (points in their original order)
__global__ void append_cluster_kernel(const float *xyz, const unsigned *vid_sorted, const int *idx_sorted, int64_t n, int M,
                                      double *newobs /*[M][10]*/) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= M) return;
  append_cluster(xyz, vid_sorted, idx_sorted, n, (unsigned)(v + 1), newobs + (size_t)v * 10);
}
}  // namespace


// ---------------------------------------------------------------------------------------------------------------------
// Both steps for every problem of a batch in one call. One thread per voxel of the whole registration finds its problem
// through vox_prob (null: one problem) and runs the rule (the device functions above) on the problem's poses, mg_size or
// slot; a problem whose argument is 0 (marginalise) or -1 (append) keeps every voxel unchanged. Voxels are grouped by
// problem, so the global exclusive scans of the keep flags and of the kept observation counts give every problem a
// contiguous range of the new registration, and batch_window_ptr_kernel reads the per-problem offsets off them.
// Appending: the (problem, point) items of the new scans are expanded as the cut expands its rows, every point is looked
// up among its own problem's keys only, and a stable radix sort by global voxel id + 1 keeps the points of one voxel in
// scan order, so its new cluster sums in the order of the scan's points.
namespace {
__device__ __forceinline__ int prob_of(const int *prob, int64_t i) { return prob ? prob[i] : 0; }
__global__ void batch_marg_count_kernel(const long long *row_ptr, const int *pose_idx, Strided obs, const int *vox_prob,
                                        int64_t M, const int *mg, int min_ps, int *keep, int *cnt) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= M) return;
  const int m = mg[prob_of(vox_prob, v)];
  int k = (int)(row_ptr[v + 1] - row_ptr[v]), kp = 1;
  if (m > 0) kp = marg_keep(row_ptr, pose_idx, obs, v, m, min_ps, &k);
  keep[v] = kp;
  cnt[v] = kp ? k : 0;
}
__global__ void batch_marg_emit_kernel(const long long *row_ptr, const int *pose_idx, Strided obs, Strided fix,
                                       const double *coe, const unsigned long long *key, const int *layer,
                                       const int *vox_prob, int64_t M, const int *pose_base, const int *mg,
                                       const double *poses, const int *keep, const int *vscan, const int *oscan,
                                       WindowEmit out, int64_t Mout, int64_t Kout) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v == 0) out.row_ptr[Mout] = Kout;
  if (v >= M || !keep[v]) return;
  const int b = prob_of(vox_prob, v), m = mg[b], nv = vscan[v];
  const long long o = oscan[v];
  out.row_ptr[nv] = o;
  if (key) { out.key[nv] = key[v]; out.layer[nv] = layer[v]; }
  const double pts = marg_emit(row_ptr, pose_idx, obs, fix, v, poses + 12 * (size_t)pose_base[b], m, o, out.pose_idx,
                               out.obs, out.fix + (size_t)nv * 10);
  out.coe[nv] = m > 0 ? pts : coe[v];
}
__global__ void batch_append_match_kernel(const float *xyz, const int *src, const int *prob, int64_t n,
                                          const double *poses, const long long *vptr, const int *pose_base,
                                          const int *slot, AssocParams p, const unsigned long long *key,
                                          const int *layer, unsigned *vid1) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int b = prob_of(prob, i);
  const long long v0 = vptr[b];
  const int v = append_match(xyz, src[i], poses + 12 * (size_t)(pose_base[b] + slot[b]), p, key + v0, layer + v0,
                             (int)(vptr[b + 1] - v0));
  vid1[i] = v < 0 ? 0u : (unsigned)(v0 + v + 1);  // 0 = in no voxel of its problem
}
__global__ void batch_append_judge_kernel(const long long *row_ptr, const int *pose_idx, Strided obs, Strided fix,
                                          const int *vox_prob, int64_t M, const int *pose_base, const int *slot,
                                          const double *poses, const double *newobs, const int *layer, AssocParams p,
                                          int *keep, int *cnt, int *bad) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= M) return;
  const int b = prob_of(vox_prob, v), s = slot[b];
  int k = (int)(row_ptr[v + 1] - row_ptr[v]), kp = 1;
  if (s >= 0) {
    bool slot_bad = false;
    kp = append_judge(row_ptr, pose_idx, obs, fix, v, poses + 12 * (size_t)pose_base[b], newobs + (size_t)v * 10, s,
                      layer[v], p, &k, &slot_bad);
    if (slot_bad) atomicMin(bad, b);  // the lowest such problem is reported
  }
  keep[v] = kp;
  cnt[v] = kp ? k : 0;
}
__global__ void batch_append_emit_kernel(const long long *row_ptr, const int *pose_idx, Strided obs, Strided fix,
                                         const double *coe, const unsigned long long *key, const int *layer,
                                         const int *vox_prob, int64_t M, const int *slot, const double *newobs,
                                         const int *keep, const int *vscan, const int *oscan, WindowEmit out,
                                         int64_t Mout, int64_t Kout) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v == 0) out.row_ptr[Mout] = Kout;
  if (v >= M || !keep[v]) return;
  const int nv = vscan[v];
  const long long o = oscan[v];
  out.row_ptr[nv] = o;
  out.key[nv] = key[v];
  out.layer[nv] = layer[v];
  append_emit(row_ptr, pose_idx, obs, fix, coe, v, newobs + (size_t)v * 10, slot[prob_of(vox_prob, v)], o,
              out.pose_idx, out.obs, out.fix ? out.fix + (size_t)nv * 10 : nullptr, out.coe + nv);
}
// per problem b in [0, B]: its first voxel and first observation in the new registration ([0][B + 1], [1][B + 1]); with
// vid_sorted, for b < B the points of its new scan that fell into one of its voxels ([2][B])
__global__ void batch_window_ptr_kernel(const long long *vptr, int B, int64_t M, const int *keep, const int *vscan,
                                        const int *cnt, const int *oscan, const unsigned *vid_sorted, int64_t n,
                                        long long *out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > B) return;
  const long long v0 = vptr[b];
  out[b] = v0 < M ? vscan[v0] : (long long)vscan[M - 1] + keep[M - 1];
  out[B + 1 + b] = v0 < M ? oscan[v0] : (long long)oscan[M - 1] + cnt[M - 1];
  if (!vid_sorted || b == B) return;
  int64_t lim[2];
  for (int e = 0; e < 2; e++) {  // first point with vid >= v0 + 1, first with vid >= v1 + 1
    const unsigned want = (unsigned)(vptr[b + e] + 1);
    int64_t lo = 0, hi = n;
    while (lo < hi) { const int64_t m = (lo + hi) >> 1; if (vid_sorted[m] < want) lo = m + 1; else hi = m; }
    lim[e] = lo;
  }
  out[2 * (B + 1) + b] = lim[1] - lim[0];
}

// the poses [12 P], per-problem device table voxel_ptr [B + 1], then (pose_base, arg) [2][B]: one buffer, one copy (a
// context's call is the case B = 1, where allocations and copies dominate)
int window_tables(cudaStream_t st, ScratchPool &pool, const BatchVoxels &in, const int *arg, double **poses,
                  long long **vptr, int **pinfo) {
  const int B = in.B;
  const size_t np = (size_t)12 * in.pose_ptr[B], nw = np + (size_t)B + 1;  // 8-byte words before the int table
  std::vector<long long> h(nw + B);
  std::copy(in.poses12, in.poses12 + np, reinterpret_cast<double *>(h.data()));
  std::copy(in.voxel_ptr, in.voxel_ptr + B + 1, h.begin() + np);
  int *info = reinterpret_cast<int *>(h.data() + nw);
  for (int b = 0; b < B; b++) { info[b] = (int)in.pose_ptr[b]; info[B + b] = arg[b]; }
  long long *d = nullptr;
  TRY(pool.get(&d, h.size()));
  CUDA_TRY(cudaMemcpyAsync(d, h.data(), sizeof(long long) * h.size(), cudaMemcpyHostToDevice, st));
  *poses = reinterpret_cast<double *>(d);
  *vptr = d + np;
  *pinfo = reinterpret_cast<int *>(d + nw);
  return BALM_OK;
}
// with keep / cnt of the in.M voxels: their exclusive scans and the per-problem offsets (+ matched counts) on the host
int window_offsets(cudaStream_t st, ScratchPool &pool, const BatchVoxels &in, const long long *vptr, const int *keep,
                   const int *cnt, int *vscan, int *oscan, const unsigned *vid_sorted, int64_t n, int *bad,
                   std::vector<long long> &h, int *h_bad) {
  const int B = in.B;
  size_t tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, keep, vscan, (int)in.M, st);
  char *tmp = nullptr;
  long long *dptr = nullptr;
  TRY(pool.get(&tmp, tb)); TRY(pool.get(&dptr, h.size()));
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tb, keep, vscan, (int)in.M, st));
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tb, cnt, oscan, (int)in.M, st));
  batch_window_ptr_kernel<<<(B + 128) / 128, 128, 0, st>>>(vptr, B, in.M, keep, vscan, cnt, oscan, vid_sorted, n, dptr);
  CUDA_TRY(cudaMemcpyAsync(h.data(), dptr, sizeof(long long) * h.size(), cudaMemcpyDeviceToHost, st));
  if (bad) CUDA_TRY(cudaMemcpyAsync(h_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return BALM_OK;
}
}  // namespace

int batch_marginalize_build(cudaStream_t st, const BatchVoxels &in, const int *mg_size, int min_ps,
                            const WindowRegister &reg, long long *launches) {
  const int B = in.B;
  const int64_t M = in.M;
  const Strided obs{in.obs, in.obs_cstride, in.obs_ostride}, fix{in.fix, in.fix_cstride, in.fix_vstride};
  ScratchPool pool;
  double *poses = nullptr;
  long long *vptr = nullptr;
  int *pinfo = nullptr, *keep = nullptr, *cnt = nullptr, *vscan = nullptr, *oscan = nullptr;
  TRY(window_tables(st, pool, in, mg_size, &poses, &vptr, &pinfo));
  std::vector<long long> h((size_t)2 * (B + 1), 0);  // new voxel_ptr [B + 1], obs_ptr [B + 1]
  const unsigned gv = (unsigned)((M + 127) / 128);
  if (M > 0) {
    TRY(pool.get(&keep, (size_t)4 * M));
    cnt = keep + M; vscan = keep + 2 * M; oscan = keep + 3 * M;
    batch_marg_count_kernel<<<gv, 128, 0, st>>>(in.row_ptr, in.pose_idx, obs, in.vox_prob, M, pinfo + B, min_ps, keep, cnt);
    TRY(window_offsets(st, pool, in, vptr, keep, cnt, vscan, oscan, nullptr, 0, nullptr, h, nullptr));
    *launches += 4;
  }
  WindowEmit out{};
  TRY(reg(reinterpret_cast<const int64_t *>(h.data()), reinterpret_cast<const int64_t *>(h.data() + B + 1), &out));
  if (M > 0) {
    batch_marg_emit_kernel<<<gv, 128, 0, st>>>(in.row_ptr, in.pose_idx, obs, fix, in.coe, in.key, in.layer, in.vox_prob, M,
                                               pinfo, pinfo + B, poses, keep, vscan, oscan, out, h[B],
                                               h[2 * (size_t)B + 1]);
    *launches += 1;
  } else {
    CUDA_TRY(cudaMemsetAsync(out.row_ptr, 0, sizeof(long long), st));
  }
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaStreamSynchronize(st));
  return BALM_OK;
}

int batch_append_build(cudaStream_t st, const BatchVoxels &in, const balm_assoc_opts &o, const int32_t *scan_of,
                       const int *slot, const int64_t *scan_ptr, const float *xyz, int64_t n_points,
                       const WindowRegister &reg, int64_t *n_matched, bool batch, long long *launches) {
  const int B = in.B;
  const int64_t M = in.M;
  const Strided obs{in.obs, in.obs_cstride, in.obs_ostride}, fix{in.fix, in.fix_cstride, in.fix_vstride};
  ScratchPool pool;
  AssocParams P{o.voxel_size, o.layer_limit, o.min_ps, {o.eigen_value_array[0], o.eigen_value_array[1], o.eigen_value_array[2]}};
  std::vector<int> arg(B);
  std::vector<long long> tab((size_t)2 * B + 1, 0);  // item_ptr [B + 1], then the first point of each problem's scan
  for (int b = 0; b < B; b++) {
    const int s = scan_of[b];
    arg[b] = s >= 0 ? slot[b] : -1;
    tab[b + 1] = tab[b] + (s >= 0 ? scan_ptr[s + 1] - scan_ptr[s] : 0);
    tab[(size_t)B + 1 + b] = s >= 0 ? scan_ptr[s] : 0;
  }
  const int64_t n = tab[B];
  double *poses = nullptr, *newobs = nullptr;
  long long *vptr = nullptr, *dtab = nullptr;
  int *pinfo = nullptr, *keep = nullptr, *cnt = nullptr, *vscan = nullptr, *oscan = nullptr, *bad = nullptr;
  int *src = nullptr, *src2 = nullptr, *prob = nullptr;
  unsigned *vid = nullptr, *vid2 = nullptr;
  float *dxyz = nullptr;
  TRY(window_tables(st, pool, in, arg.data(), &poses, &vptr, &pinfo));
  std::vector<long long> h((size_t)3 * B + 2, 0);  // new voxel_ptr [B + 1], obs_ptr [B + 1], matched points [B]
  int h_bad = 0x7f7f7f7f;
  const unsigned gv = (unsigned)((M + 127) / 128);
  if (M > 0) {
    if (n > 0) {
      const unsigned gp = (unsigned)((n + 255) / 256);
      TRY(pool.get(&dxyz, (size_t)3 * n_points)); TRY(pool.get(&src, (size_t)n)); TRY(pool.get(&src2, (size_t)n));
      TRY(pool.get(&vid, (size_t)n)); TRY(pool.get(&vid2, (size_t)n));
      CUDA_TRY(cudaMemcpyAsync(dxyz, xyz, sizeof(float) * 3 * n_points, cudaMemcpyHostToDevice, st));
      if (B == 1) {  // one problem: its scan's points in order over a full grid (prob stays null: problem 0)
        win_iota_kernel<<<gp, 256, 0, st>>>(src, n, (int)tab[2]);
      } else {
        TRY(pool.get(&dtab, tab.size())); TRY(pool.get(&prob, (size_t)n));
        CUDA_TRY(cudaMemcpyAsync(dtab, tab.data(), sizeof(long long) * tab.size(), cudaMemcpyHostToDevice, st));
        expand_rows_kernel<<<B, 256, 0, st>>>(dtab, dtab + B + 1, src, prob);
      }
      batch_append_match_kernel<<<gp, 256, 0, st>>>(dxyz, src, prob, n, poses, vptr, pinfo, pinfo + B, P, in.key,
                                                    in.layer, vid);
      int bits = 1;
      while ((1ll << bits) <= M) bits++;
      size_t tb = 0;
      cub::DeviceRadixSort::SortPairs(nullptr, tb, vid, vid2, src, src2, (int)n, 0, bits, st);
      char *tmp = nullptr;
      TRY(pool.get(&tmp, tb));
      CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tb, vid, vid2, src, src2, (int)n, 0, bits, st));  // stable
      *launches += 3;
    }
    TRY(pool.get(&newobs, (size_t)M * 10));
    TRY(pool.get(&keep, (size_t)4 * M));
    cnt = keep + M; vscan = keep + 2 * M; oscan = keep + 3 * M;
    TRY(pool.get(&bad, 1));
    CUDA_TRY(cudaMemsetAsync(bad, 0x7f, sizeof(int), st));
    append_cluster_kernel<<<gv, 128, 0, st>>>(dxyz, vid2, src2, n, (int)M, newobs);
    batch_append_judge_kernel<<<gv, 128, 0, st>>>(in.row_ptr, in.pose_idx, obs, fix, in.vox_prob, M, pinfo, pinfo + B,
                                                  poses, newobs, in.layer, P, keep, cnt, bad);
    TRY(window_offsets(st, pool, in, vptr, keep, cnt, vscan, oscan, vid2, n, bad, h, &h_bad));
    *launches += 5;
  }
  if (h_bad != 0x7f7f7f7f) {
    if (batch)
      balm_set_error("balm_batch_append_scan: problem " + std::to_string(h_bad) +
                     ": `slot` must be above every scan already observing its voxels");
    else
      balm_set_error("balm_append_scan: `slot` must be above every scan already observing the voxels");
    return BALM_ERR_INVALID;
  }
  WindowEmit out{};
  TRY(reg(reinterpret_cast<const int64_t *>(h.data()), reinterpret_cast<const int64_t *>(h.data() + B + 1), &out));
  if (M > 0) {
    batch_append_emit_kernel<<<gv, 128, 0, st>>>(in.row_ptr, in.pose_idx, obs, fix, in.coe, in.key, in.layer, in.vox_prob,
                                                 M, pinfo + B, newobs, keep, vscan, oscan, out, h[B],
                                                 h[2 * (size_t)B + 1]);
    *launches += 1;
  } else {
    CUDA_TRY(cudaMemsetAsync(out.row_ptr, 0, sizeof(long long), st));
  }
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaStreamSynchronize(st));
  // a problem left without voxels (where the context call fails) matched nothing that stays registered
  for (int b = 0; b < B; b++) n_matched[b] = h[b + 1] > h[b] ? h[2 * (size_t)(B + 1) + b] : 0;
  return BALM_OK;
}


// ---------------------------------------------------------------------------------------------------------------------
// The persistent sliding-window octree in HBM (SURVEY.md 8f row N2): the reference's surf_map of OCTO_TREE_ROOTs kept
// across window shifts and driven by its four operations
//   cut_voxel                                    bavoxel.hpp:1170-1223
//   OCTO_TREE_NODE::recut / judge_eigen / cut_func                :737-776, 654-699, 700-735
//   OCTO_TREE_ROOT::marginalize -> OCTO_TREE_NODE::to_margi       :948-963, 778-816
//   OCTO_TREE_NODE::tras_opt -> VOX_HESS::push_voxel              :908-929, 30-51
// One state holds the maps of B independent problems (balm_batch_window_*); a context's balm_window_* is the case B = 1.
// State (all device arrays, grown by doubling, nothing is ever deleted from the node table):
//   node table, append-only (a node's id never changes): 63-bit key, problem, layer, split flag (octo_state),
//     push_state, fix_point [10], and per window slot the clusters sig_orig / sig_tran [N][10], N = the largest slot
//     count of the problems. A per-layer table of node ids sorted by (problem, key), with per-problem offsets, finds a
//     node inside its problem's range (a key digit 7 is both "not split" and octant 7, so keys are only unique per
//     layer and problem).
//   point store: body xyz (vec_orig, float as given), world xyz (vec_tran, fp64), slot, problem, node id and an order
//     stamp. The stamp orders the points of one (node, slot) list as the reference's vector holds them: a cut stamps
//     (op << 32 | rank of the point among the call's items), a move into a child restamps the moved points (op << 32 |
//     rank in stamp order), so they land after the child's earlier points and keep their parent's order. A cut's items
//     are the points of every problem in (problem, scan point) order, so within one problem the stamps order its points
//     as a context holding that problem alone orders them.
//   per-problem table (WinProb): slot count and first pose row, and the call's win_count / mg_size, 0 = problem left
//     alone by this call.
// Clusters are accumulated point by point in that order, exactly as PointCluster::push runs, so sums of the device
// and of the reference round alike; a (node, slot) belongs to one problem, so a problem's sums do not depend on the
// rest of the batch, and node ids never reach the output. Split nodes keep whatever points are left in them (slots
// the recut did not move); nothing reads them unless a later recut(win_count) with win_count - 1 == that slot moves
// them, as in the reference.
namespace {
struct WinProb {
  int n_slots, pose_base;
  int w, mg;  // of the current call
};
struct WinLookup {
  int n = 0;
  unsigned long long *key = nullptr;  // [n] sorted by (problem, key)
  int *id = nullptr;                  // [n]
  int *off = nullptr;                 // [B + 1] the range of each problem
};
}  // namespace

struct WindowState {
  AssocParams P;
  balm_assoc_opts opts;
  bool batch = false;              // balm_batch_window_*: errors name the problem, too many points is UNSUPPORTED
  int B = 0, N = 0;                // problems, slot stride (max n_slots)
  std::vector<WinProb> hprob;
  std::vector<int> n_slots;
  WinProb *prob = nullptr;         // device [B]
  unsigned long long op = 1;       // stamp counter
  // nodes
  int nn = 0, ncap = 0;
  unsigned long long *nkey = nullptr;
  int *nprob = nullptr, *nlayer = nullptr, *nsplit = nullptr, *npush = nullptr, *naction = nullptr;
  double *nfix = nullptr;          // [ncap][10]
  double *sig_o = nullptr, *sig_t = nullptr;  // [ncap][N][10]
  WinLookup look[3];
  // points
  int64_t np = 0, pcap = 0;
  float *pxyz = nullptr;
  double *ptran = nullptr;
  int *pslot = nullptr, *pprob = nullptr, *pnode = nullptr;
  unsigned long long *pstamp = nullptr;
  ~WindowState() {
    void *ps[] = {prob, nkey, nprob, nlayer, nsplit, npush, naction, nfix, sig_o, sig_t, pxyz, ptran, pslot, pprob, pnode,
                  pstamp};
    for (void *q : ps) cudaFree(q);
    for (WinLookup &l : look) { cudaFree(l.key); cudaFree(l.id); cudaFree(l.off); }
  }
};

namespace {
template <typename T>
int grow_array(T **p, size_t used, size_t cap) {  // new buffer of `cap` elements holding the first `used` ones
  T *q = nullptr;
  CUDA_TRY(cudaMalloc((void **)&q, sizeof(T) * (cap ? cap : 1)));
  if (used) {
    const cudaError_t e = cudaMemcpy(q, *p, sizeof(T) * used, cudaMemcpyDeviceToDevice);
    if (e != cudaSuccess) { cudaFree(q); CUDA_TRY(e); }
  }
  cudaFree(*p);
  *p = q;
  return BALM_OK;
}

int win_reserve_nodes(WindowState &w, int need) {
  if (need <= w.ncap) return BALM_OK;
  int cap = std::max(need, std::max(1024, 2 * w.ncap));
  const size_t nn = (size_t)w.nn, c = (size_t)cap, NS = (size_t)w.N * 10;
  TRY(grow_array(&w.nkey, nn, c)); TRY(grow_array(&w.nprob, nn, c)); TRY(grow_array(&w.nlayer, nn, c));
  TRY(grow_array(&w.nsplit, nn, c)); TRY(grow_array(&w.npush, nn, c)); TRY(grow_array(&w.naction, nn, c));
  TRY(grow_array(&w.nfix, nn * 10, c * 10));
  TRY(grow_array(&w.sig_o, nn * NS, c * NS)); TRY(grow_array(&w.sig_t, nn * NS, c * NS));
  w.ncap = cap;
  return BALM_OK;
}
int win_reserve_points(WindowState &w, int64_t need) {
  if (need <= w.pcap) return BALM_OK;
  int64_t cap = std::max<int64_t>(need, std::max<int64_t>(1 << 16, 2 * w.pcap));
  cap = std::min<int64_t>(cap, (1ll << 31) - 1);
  const size_t n = (size_t)w.np, c = (size_t)cap;
  TRY(grow_array(&w.pxyz, 3 * n, 3 * c)); TRY(grow_array(&w.ptran, 3 * n, 3 * c)); TRY(grow_array(&w.pslot, n, c));
  TRY(grow_array(&w.pprob, n, c)); TRY(grow_array(&w.pnode, n, c)); TRY(grow_array(&w.pstamp, n, c));
  w.pcap = cap;
  return BALM_OK;
}

// the call's win_count / mg_size per problem (null: 0) into the device table
int win_upload(WindowState &w, cudaStream_t st, const int *wc, const int *mg) {
  for (int p = 0; p < w.B; p++) {
    w.hprob[p].w = wc ? wc[p] : 0;
    w.hprob[p].mg = mg ? mg[p] : 0;
  }
  CUDA_TRY(cudaMemcpyAsync(w.prob, w.hprob.data(), sizeof(WinProb) * w.B, cudaMemcpyHostToDevice, st));
  return BALM_OK;
}

int radix_bits(unsigned long long maxval) {  // bits that hold every value in [0, maxval]
  int bits = 1;
  while (bits < 64 && (maxval >> bits)) bits++;
  return bits;
}

// cub temporary storage from the pool
struct CubTmp {
  ScratchPool &pool;
  char *p = nullptr;
  size_t bytes = 0;
  int need(size_t b) {
    if (b <= bytes) return BALM_OK;
    pool.drop(p);
    p = nullptr;
    bytes = b;
    return pool.get(&p, bytes);
  }
};

// index of key k among problem p's entries of a lookup table, or -1
__device__ __forceinline__ int look_find(const unsigned long long *key, const int *off, int p, unsigned long long k) {
  const int a = off[p];
  const int i = find_key(key + a, off[p + 1] - a, k);
  return i < 0 ? -1 : a + i;
}

__global__ void win_missing_kernel(const unsigned long long *keys, const int *probs, int m, const unsigned long long *look,
                                   const int *off, int *miss) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) miss[i] = look_find(look, off, probs[i], keys[i]) < 0 ? 1 : 0;
}
// first of every (problem, key) run of a sorted list
__global__ void win_unique_flag_kernel(const unsigned long long *keys, const int *probs, int m, int *flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) flag[i] = (i == 0 || keys[i] != keys[i - 1] || probs[i] != probs[i - 1]) ? 1 : 0;
}
__global__ void win_init_nodes_kernel(const unsigned long long *keys, const int *probs, int m, int base, int layer,
                                      unsigned long long *nkey, int *nprob, int *nlayer, int *nsplit, int *npush,
                                      double *nfix) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const int v = base + i;
  nkey[v] = keys[i]; nprob[v] = probs[i]; nlayer[v] = layer; nsplit[v] = 0; npush[v] = 0;
#pragma unroll
  for (int q = 0; q < 10; q++) nfix[(size_t)v * 10 + q] = 0.0;
}
// node id of every key (the key is in its problem's range of the layer's table)
__global__ void win_find_kernel(const unsigned long long *keys, const int *probs, const int *sel, int m,
                                const unsigned long long *look, const int *look_id, const int *off,
                                int *node_out /*indexed by sel[i] or i*/) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  node_out[sel ? sel[i] : i] = look_id[look_find(look, off, probs[i], keys[i])];
}
__global__ void win_gather_i32_kernel(const int *src, const int *idx, int m, int *dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) dst[i] = src[idx[i]];
}
__global__ void win_gather_u64_kernel(const unsigned long long *src, const int *idx, int m, unsigned long long *dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) dst[i] = src[idx[i]];
}
// off[p] = first entry of problem p (and off[B] = n) in a list of node ids sorted by problem
__global__ void win_offsets_kernel(const int *ids, int n, const int *nprob, int B, int *off) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > B) return;
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (nprob[ids[mid]] < p) lo = mid + 1; else hi = mid;
  }
  off[p] = lo;
}

// node ids in ascending (problem, key): sorted by key (64 bits), then stably by problem when there is more than one.
// ids / keys: n entries, permuted in place through the scratch buffers ids2 / keys2 (n each).
int win_sort_ids(WindowState &w, ScratchPool &pool, CubTmp &tmp, cudaStream_t st, unsigned long long *&keys, int *&ids,
                 unsigned long long *&keys2, int *&ids2, int n) {
  size_t b1 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b1, keys, keys2, ids, ids2, n, 0, 64, st);
  TRY(tmp.need(b1));
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp.p, tmp.bytes, keys, keys2, ids, ids2, n, 0, 64, st));
  std::swap(keys, keys2);
  std::swap(ids, ids2);
  if (w.B == 1) return BALM_OK;
  int *pr = nullptr, *pr2 = nullptr;
  TRY(pool.get(&pr, n)); TRY(pool.get(&pr2, n));
  const unsigned g = (unsigned)((n + 255) / 256);
  win_gather_i32_kernel<<<g, 256, 0, st>>>(w.nprob, ids, n, pr);
  const int bits = radix_bits((unsigned long long)(w.B - 1));
  size_t b2 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b2, pr, pr2, ids, ids2, n, 0, bits, st);
  TRY(tmp.need(b2));
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp.p, tmp.bytes, pr, pr2, ids, ids2, n, 0, bits, st));  // stable
  std::swap(ids, ids2);
  win_gather_u64_kernel<<<g, 256, 0, st>>>(w.nkey, ids, n, keys);
  return BALM_OK;
}

// the layer-L nodes that (keys, probs) (m entries, any order, duplicates allowed) name and that do not exist yet are
// appended to the node table in ascending (problem, key) order, and the layer's lookup table is rebuilt
int win_add_nodes(WindowState &w, ScratchPool &pool, CubTmp &tmp, cudaStream_t st, const unsigned long long *keys,
                  const int *probs, int m, int L) {
  if (m < 1) return BALM_OK;
  WinLookup &lk = w.look[L];
  int *miss = nullptr, *nsel = nullptr, *selp = nullptr, *sp = nullptr, *flag = nullptr, *up = nullptr;
  unsigned long long *sel = nullptr, *sorted = nullptr, *uniq = nullptr;
  TRY(pool.get(&miss, m)); TRY(pool.get(&nsel, 1)); TRY(pool.get(&sel, m)); TRY(pool.get(&sorted, m));
  TRY(pool.get(&uniq, m)); TRY(pool.get(&selp, m)); TRY(pool.get(&sp, m)); TRY(pool.get(&flag, m)); TRY(pool.get(&up, m));
  win_missing_kernel<<<(m + 255) / 256, 256, 0, st>>>(keys, probs, m, lk.key, lk.off, miss);
  size_t b1 = 0, b2 = 0;
  cub::DeviceSelect::Flagged(nullptr, b1, keys, miss, sel, nsel, m, st);
  cub::DeviceSelect::Flagged(nullptr, b2, probs, miss, selp, nsel, m, st);
  TRY(tmp.need(std::max(b1, b2)));
  CUDA_TRY(cub::DeviceSelect::Flagged(tmp.p, tmp.bytes, probs, miss, selp, nsel, m, st));
  CUDA_TRY(cub::DeviceSelect::Flagged(tmp.p, tmp.bytes, keys, miss, sel, nsel, m, st));
  int nmiss = 0;
  CUDA_TRY(cudaMemcpyAsync(&nmiss, nsel, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  if (nmiss == 0) return BALM_OK;
  // (problem, key) of the missing entries in ascending order: by key, then stably by problem
  size_t b3 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b3, sel, sorted, selp, sp, nmiss, 0, 64, st);
  TRY(tmp.need(b3));
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp.p, tmp.bytes, sel, sorted, selp, sp, nmiss, 0, 64, st));
  if (w.B > 1) {
    const int bits = radix_bits((unsigned long long)(w.B - 1));
    size_t b4 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, b4, sp, selp, sorted, sel, nmiss, 0, bits, st);
    TRY(tmp.need(b4));
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp.p, tmp.bytes, sp, selp, sorted, sel, nmiss, 0, bits, st));
    std::swap(sp, selp);
    std::swap(sorted, sel);
  }
  win_unique_flag_kernel<<<(nmiss + 255) / 256, 256, 0, st>>>(sorted, sp, nmiss, flag);
  size_t b5 = 0, b6 = 0;
  cub::DeviceSelect::Flagged(nullptr, b5, sorted, flag, uniq, nsel, nmiss, st);
  cub::DeviceSelect::Flagged(nullptr, b6, sp, flag, up, nsel, nmiss, st);
  TRY(tmp.need(std::max(b5, b6)));
  CUDA_TRY(cub::DeviceSelect::Flagged(tmp.p, tmp.bytes, sp, flag, up, nsel, nmiss, st));
  CUDA_TRY(cub::DeviceSelect::Flagged(tmp.p, tmp.bytes, sorted, flag, uniq, nsel, nmiss, st));
  int nnew = 0;
  CUDA_TRY(cudaMemcpyAsync(&nnew, nsel, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  if ((int64_t)w.nn + nnew >= (1ll << 31) / std::max(1, 10 * w.N)) {
    balm_set_error("balm_window: node table too large");
    return BALM_ERR_UNSUPPORTED;
  }
  TRY(win_reserve_nodes(w, w.nn + nnew));
  const int base = w.nn;
  win_init_nodes_kernel<<<(nnew + 255) / 256, 256, 0, st>>>(uniq, up, nnew, base, L, w.nkey, w.nprob, w.nlayer, w.nsplit,
                                                            w.npush, w.nfix);
  CUDA_TRY(cudaMemsetAsync(w.sig_o + (size_t)base * w.N * 10, 0, sizeof(double) * (size_t)nnew * w.N * 10, st));
  CUDA_TRY(cudaMemsetAsync(w.sig_t + (size_t)base * w.N * 10, 0, sizeof(double) * (size_t)nnew * w.N * 10, st));
  // lookup: old (key, id) pairs + the new ones, sorted by (problem, key)
  const int nl = lk.n + nnew;
  unsigned long long *k_in = nullptr, *k2 = nullptr;
  int *i_in = nullptr, *i2 = nullptr;
  TRY(pool.get(&k_in, nl)); TRY(pool.get(&i_in, nl)); TRY(pool.get(&k2, nl)); TRY(pool.get(&i2, nl));
  if (lk.n) {
    CUDA_TRY(cudaMemcpyAsync(k_in, lk.key, sizeof(unsigned long long) * lk.n, cudaMemcpyDeviceToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(i_in, lk.id, sizeof(int) * lk.n, cudaMemcpyDeviceToDevice, st));
  }
  CUDA_TRY(cudaMemcpyAsync(k_in + lk.n, uniq, sizeof(unsigned long long) * nnew, cudaMemcpyDeviceToDevice, st));
  win_iota_kernel<<<(nnew + 255) / 256, 256, 0, st>>>(i_in + lk.n, nnew, base);
  TRY(win_sort_ids(w, pool, tmp, st, k_in, i_in, k2, i2, nl));
  unsigned long long *k_out = nullptr;
  int *i_out = nullptr, *o_out = nullptr;
  if (cudaMalloc((void **)&k_out, sizeof(unsigned long long) * nl) != cudaSuccess ||
      cudaMalloc((void **)&i_out, sizeof(int) * nl) != cudaSuccess ||
      cudaMalloc((void **)&o_out, sizeof(int) * (w.B + 1)) != cudaSuccess) {
    cudaFree(k_out); cudaFree(i_out); cudaFree(o_out);
    CUDA_TRY(cudaErrorMemoryAllocation);
  }
  CUDA_TRY(cudaMemcpyAsync(k_out, k_in, sizeof(unsigned long long) * nl, cudaMemcpyDeviceToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(i_out, i_in, sizeof(int) * nl, cudaMemcpyDeviceToDevice, st));
  win_offsets_kernel<<<(w.B + 128) / 128, 128, 0, st>>>(i_out, nl, w.nprob, w.B, o_out);
  CUDA_TRY(cudaStreamSynchronize(st));
  cudaFree(lk.key);
  cudaFree(lk.id);
  cudaFree(lk.off);
  lk.key = k_out; lk.id = i_out; lk.off = o_out; lk.n = nl;
  w.nn += nnew;
  return BALM_OK;
}

// One thread per (node, slot) segment of points given in push order: sig_orig / sig_tran .push of every point, in order
// (PointCluster::push, tools.hpp:311-316), on top of what the node already holds.
__global__ void win_push_kernel(const int *order, const int *seg_start, int nseg, int m, const float *pxyz,
                                const double *ptran, const int *pnode, const int *pslot, int N, double *sig_o,
                                double *sig_t) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nseg) return;
  const int a = seg_start[s], b = (s + 1 < nseg) ? seg_start[s + 1] : m;
  const int j0 = order[a];
  double *so = sig_o + ((size_t)pnode[j0] * N + pslot[j0]) * 10;
  double *stt = sig_t + ((size_t)pnode[j0] * N + pslot[j0]) * 10;
  double B[10], W[10];
#pragma unroll
  for (int q = 0; q < 10; q++) { B[q] = so[q]; W[q] = stt[q]; }
  for (int i = a; i < b; i++) {
    const int j = order[i];
    const double x = pxyz[3 * j], y = pxyz[3 * j + 1], z = pxyz[3 * j + 2];
    B[0] += x * x; B[1] += x * y; B[2] += x * z; B[3] += y * y; B[4] += y * z; B[5] += z * z;
    B[6] += x; B[7] += y; B[8] += z; B[9] += 1.0;
    const double wx = ptran[3 * j], wy = ptran[3 * j + 1], wz = ptran[3 * j + 2];
    W[0] += wx * wx; W[1] += wx * wy; W[2] += wx * wz; W[3] += wy * wy; W[4] += wy * wz; W[5] += wz * wz;
    W[6] += wx; W[7] += wy; W[8] += wz; W[9] += 1.0;
  }
#pragma unroll
  for (int q = 0; q < 10; q++) { so[q] = B[q]; stt[q] = W[q]; }
}
__global__ void win_seg_key_kernel(const int *order, int m, const int *pnode, const int *pslot, int N,
                                   unsigned long long *ck) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) ck[i] = (unsigned long long)pnode[order[i]] * (unsigned long long)N + (unsigned long long)pslot[order[i]];
}
__global__ void win_seg_flag_kernel(const unsigned long long *ck, int m, int *flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) flag[i] = (i == 0 || ck[i] != ck[i - 1]) ? 1 : 0;
}

// pushes the m points `order` (point ids, in push order) into the clusters of their (node, slot)
int win_push_points(WindowState &w, ScratchPool &pool, CubTmp &tmp, cudaStream_t st, const int *order, int m) {
  if (m < 1) return BALM_OK;
  unsigned long long *ck = nullptr, *ck2 = nullptr;
  int *ord2 = nullptr, *flag = nullptr, *iota = nullptr, *seg = nullptr, *nsel = nullptr;
  TRY(pool.get(&ck, m)); TRY(pool.get(&ck2, m)); TRY(pool.get(&ord2, m)); TRY(pool.get(&flag, m));
  TRY(pool.get(&iota, m)); TRY(pool.get(&seg, m)); TRY(pool.get(&nsel, 1));
  const unsigned g = (unsigned)((m + 255) / 256);
  win_seg_key_kernel<<<g, 256, 0, st>>>(order, m, w.pnode, w.pslot, w.N, ck);
  const int bits = radix_bits((unsigned long long)w.nn * (unsigned long long)w.N);
  size_t b1 = 0, b2 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b1, ck, ck2, order, ord2, m, 0, bits, st);
  cub::DeviceSelect::Flagged(nullptr, b2, iota, flag, seg, nsel, m, st);
  TRY(tmp.need(std::max(b1, b2)));
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp.p, tmp.bytes, ck, ck2, order, ord2, m, 0, bits, st));  // stable
  win_seg_flag_kernel<<<g, 256, 0, st>>>(ck2, m, flag);
  win_iota_kernel<<<g, 256, 0, st>>>(iota, m, 0);
  CUDA_TRY(cub::DeviceSelect::Flagged(tmp.p, tmp.bytes, iota, flag, seg, nsel, m, st));
  int nseg = 0;
  CUDA_TRY(cudaMemcpyAsync(&nseg, nsel, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  win_push_kernel<<<(nseg + 127) / 128, 128, 0, st>>>(ord2, seg, nseg, m, w.pxyz, w.ptran, w.pnode, w.pslot, w.N, w.sig_o,
                                                      w.sig_t);
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

// cut_voxel: world coordinate R p + t (fp64) and root key of every item (point src[i] of entry row[i] = (problem,
// pose row, slot)); a point outside the root range flags its problem
__global__ void win_cut_kernel(const float *xyz, const int *src, const int *row, const int4 *ent, const double *poses,
                               int n, AssocParams p, double *tran, unsigned long long *rkey, int *iprob, int *bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int4 e = ent[row[i]];
  double r[9], t[3];
  load_pose(poses + 12 * (size_t)e.y, r, t);
  const int64_t j = src[i];
  const double b[3] = {(double)xyz[3 * j], (double)xyz[3 * j + 1], (double)xyz[3 * j + 2]};
  double wp[3];
#pragma unroll
  for (int a = 0; a < 3; a++) wp[a] = r[a * 3] * b[0] + r[a * 3 + 1] * b[1] + r[a * 3 + 2] * b[2] + t[a];
#pragma unroll
  for (int a = 0; a < 3; a++) tran[3 * i + a] = wp[a];
  rkey[i] = world_point_key(wp, p, bad + e.x) | 63ull;
  iprob[i] = e.x;
}
// the items into the point store from index 0 of the given arrays: body xyz, slot, problem, stamp (op << 32 | item)
__global__ void win_store_kernel(const float *xyz, const int *src, const int *row, const int4 *ent, int n,
                                 unsigned long long op, float *pxyz, int *pslot, int *pprob, unsigned long long *pstamp) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int4 e = ent[row[i]];
  const int64_t j = src[i];
#pragma unroll
  for (int a = 0; a < 3; a++) pxyz[3 * i + a] = xyz[3 * j + a];
  pslot[i] = e.z;
  pprob[i] = e.x;
  pstamp[i] = (op << 32) | (unsigned long long)i;
}

// recut, one layer: judge every node of layer L that is not split (recut :739-768) in a problem this call recuts
// (w = its win_count > 0); 1 = split earlier (only slot w-1 moves, :770), 2 = split now (every slot < w moves,
// :766-767), 0 = no points move
__global__ void win_judge_kernel(int nn, int L, int N, AssocParams p, const WinProb *prob, const int *nprob,
                                 const int *nlayer, int *nsplit, int *npush, const double *nfix, const double *sig_o,
                                 const double *sig_t, int *action) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nn || nlayer[v] != L) return;
  const int w = prob[nprob[v]].w;
  if (w == 0) return;
  if (nsplit[v]) { action[v] = 1; return; }
  action[v] = 0;
  npush[v] = 0;
  const double *f = nfix + (size_t)v * 10;
  double ps = f[9];
  for (int i = 0; i < w; i++) ps += sig_o[((size_t)v * N + i) * 10 + 9];
  if ((int)ps <= p.min_ps) return;                                     // point_size <= min_ps (:748)
  double W[10];
#pragma unroll
  for (int q = 0; q < 10; q++) W[q] = f[q];
  for (int i = 0; i < w; i++)                                          // covMat = fix_point + sum sig_tran (:656-658)
#pragma unroll
    for (int q = 0; q < 10; q++) W[q] += sig_t[((size_t)v * N + i) * 10 + q];
  if (cluster_planar(W, p.eig[L])) {
    npush[v] = ((int)(ps - f[9]) > p.min_ps) ? 1 : 0;                  // :752-757
    return;
  }
  if (L == p.layer_limit) return;                                      // :759-760
  nsplit[v] = 1;
  action[v] = 2;
}
// cut_func: the octant of every moving point around its node's float centre, and the child's key
__global__ void win_move_kernel(int64_t np, AssocParams p, const WinProb *prob, const int *pprob, const int *pnode,
                                const int *pslot, const double *ptran, const int *action, const unsigned long long *nkey,
                                const int *nlayer, unsigned long long *ckey, int *flag) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= np) return;
  const int v = pnode[j], a = action[v], s = pslot[j], w = prob[pprob[j]].w;
  const bool mv = (a == 2 && s < w) || (a == 1 && s == w - 1);
  flag[j] = mv ? 1 : 0;
  if (!mv) return;
  const unsigned long long k = nkey[v];
  const int L = nlayer[v];
  const float quater = (float)(p.voxel_size / 4.0);
  int oct = 0;
#pragma unroll
  for (int ax = 0; ax < 3; ax++) {
    const long long idx = (long long)((k >> (6 + ROOT_BITS * (2 - ax))) & ((1ull << ROOT_BITS) - 1)) - ROOT_BIAS;
    float c = (float)((0.5 + (double)idx) * p.voxel_size);             // root centre (:1213-1215)
    if (L == 1) c = c + (float)(2 * (int)((k >> (3 + 2 - ax)) & 1) - 1) * quater;  // child centre (:717-719)
    oct = (oct << 1) | (ptran[3 * j + ax] > (double)c ? 1 : 0);        // :709-712
  }
  ckey[j] = L == 0 ? ((k & ~63ull) | ((unsigned long long)oct << 3) | 7ull) : ((k & ~7ull) | (unsigned long long)oct);
}
__global__ void win_restamp_kernel(const int *order, int m, unsigned long long op, unsigned long long *pstamp) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) pstamp[order[i]] = (op << 32) | (unsigned long long)i;
}

// to_margi (:778-816) on every node that is not split, in a problem this call marginalises (mg > 0); poses: the
// problems' pose rows or null
__global__ void win_margi_node_kernel(int nn, int N, const WinProb *prob, const int *nprob, const double *poses,
                                      const int *nsplit, const int *npush, double *nfix, double *sig_o, double *sig_t) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nn || nsplit[v]) return;
  const WinProb pr = prob[nprob[v]];
  const int mg = pr.mg, w = pr.w;
  if (mg == 0) return;
  double *so = sig_o + (size_t)v * N * 10, *stt = sig_t + (size_t)v * N * 10;
  if (poses)
    for (int i = 0; i < w; i++) {                                      // sig_tran[i].transform(sig_orig[i], x_poses[i])
      double r[9], t[3];
      load_pose(poses + 12 * ((size_t)pr.pose_base + i), r, t);
      const WC c = world_cluster(so + i * 10, r, t);
      double *d = stt + i * 10;
      d[0] = c.p00; d[1] = c.p01; d[2] = c.p02; d[3] = c.p11; d[4] = c.p12; d[5] = c.p22;
      d[6] = c.v0; d[7] = c.v1; d[8] = c.v2; d[9] = c.n;
    }
  double *f = nfix + (size_t)v * 10;
  if (f[9] < 50 && npush[v] == 1)                                      // :790-795
    for (int i = 0; i < mg; i++)
#pragma unroll
      for (int q = 0; q < 10; q++) f[q] += stt[i * 10 + q];
  for (int i = mg; i < w; i++)                                         // :797-803
    for (int q = 0; q < 10; q++) { so[(i - mg) * 10 + q] = so[i * 10 + q]; stt[(i - mg) * 10 + q] = stt[i * 10 + q]; }
  for (int i = w - mg; i < w; i++)                                     // :805-811
    for (int q = 0; q < 10; q++) { so[i * 10 + q] = 0.0; stt[i * 10 + q] = 0.0; }
}
// ... and on their points: re-transform (plvec_trans), drop the retired slots, shift the rest
__global__ void win_margi_point_kernel(int64_t np, const WinProb *prob, const int *pprob, const double *poses,
                                       const int *nsplit, const int *pnode, int *pslot, const float *pxyz, double *ptran,
                                       int *keep) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= np) return;
  const WinProb pr = prob[pprob[j]];
  const int s = pslot[j], mg = pr.mg;
  if (mg == 0 || nsplit[pnode[j]] || s >= pr.w) { keep[j] = 1; return; }
  if (poses) {
    double r[9], t[3];
    load_pose(poses + 12 * ((size_t)pr.pose_base + s), r, t);
    const double b[3] = {(double)pxyz[3 * j], (double)pxyz[3 * j + 1], (double)pxyz[3 * j + 2]};
#pragma unroll
    for (int a = 0; a < 3; a++) ptran[3 * j + a] = r[a * 3] * b[0] + r[a * 3 + 1] * b[1] + r[a * 3 + 2] * b[2] + t[a];
  }
  keep[j] = s >= mg ? 1 : 0;
  if (s >= mg) pslot[j] = s - mg;
}
__global__ void win_compact_kernel(const int *sel, int m, const float *xyz, const double *tran, const int *slot,
                                   const int *prb, const int *node, const unsigned long long *stamp, float *xyz2,
                                   double *tran2, int *slot2, int *prb2, int *node2, unsigned long long *stamp2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const int j = sel[i];
#pragma unroll
  for (int a = 0; a < 3; a++) { xyz2[3 * i + a] = xyz[3 * j + a]; tran2[3 * i + a] = tran[3 * j + a]; }
  slot2[i] = slot[j]; prb2[i] = prb[j]; node2[i] = node[j]; stamp2[i] = stamp[j];
}

// tras_opt (:908-929) + push_voxel (:30-51), in a problem this call pushes (w > 0)
__global__ void win_push_flag_kernel(int nn, int N, int min_ps, const WinProb *prob, const int *nprob, const int *nsplit,
                                     const int *npush, const double *sig_o, int *flag) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nn) return;
  flag[v] = 0;
  const WinProb pr = prob[nprob[v]];
  if (pr.w == 0 || nsplit[v] || npush[v] != 1) return;
  double pts = 0;
  for (int i = 0; i < pr.w; i++) pts += sig_o[((size_t)v * N + i) * 10 + 9];
  if ((int)pts < min_ps) return;
  int k = 0;
  for (int i = 0; i < pr.n_slots; i++) k += sig_o[((size_t)v * N + i) * 10 + 9] != 0.0 ? 1 : 0;
  flag[v] = k >= 2 ? 1 : 0;
}
__global__ void win_obs_count_kernel(const int *ids, int M, int N, const WinProb *prob, const int *nprob,
                                     const double *sig_o, int *cnt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const int v = ids[i], ns = prob[nprob[v]].n_slots;
  int k = 0;
  for (int s = 0; s < ns; s++) k += sig_o[((size_t)v * N + s) * 10 + 9] != 0.0 ? 1 : 0;
  cnt[i] = k;
}
// per problem p: its first pushed voxel vptr[p] (vptr[B] = M) and first observation optr[p] (optr[B] = K)
__global__ void win_push_ptr_kernel(const int *ids, int M, const int *nprob, const int *cnt, const int *ostart, int B,
                                    long long *vptr, long long *optr) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > B) return;
  int lo = 0, hi = M;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (nprob[ids[mid]] < p) lo = mid + 1; else hi = mid;
  }
  vptr[p] = lo;
  optr[p] = lo < M ? (long long)ostart[lo] : (long long)ostart[M - 1] + cnt[M - 1];
}
__global__ void win_emit_kernel(const int *ids, const int *ostart, int M, int64_t K, int N, const WinProb *prob,
                                const int *nprob, const double *sig_o, const double *nfix, const unsigned long long *nkey,
                                const int *nlayer, WindowEmit out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) out.row_ptr[M] = K;
  if (i >= M) return;
  const int v = ids[i], ns = prob[nprob[v]].n_slots;
  long long o = ostart[i];
  out.row_ptr[i] = o;
  double pts = 0;
  for (int s = 0; s < ns; s++) {
    const double *c = sig_o + ((size_t)v * N + s) * 10;
    if (c[9] == 0.0) continue;
    for (int q = 0; q < 10; q++) out.obs[o * 10 + q] = c[q];
    out.pose_idx[o] = s;
    pts += c[9];
    o++;
  }
  for (int q = 0; q < 10; q++) out.fix[(size_t)i * 10 + q] = nfix[(size_t)v * 10 + q];
  out.coe[i] = pts;                                                    // coe = sum of N (:42-44)
  out.key[i] = nkey[v];
  out.layer[i] = nlayer[v];
}
}  // namespace

void window_free(WindowState *w) { delete w; }
const std::vector<int> &window_slots(const WindowState *w) { return w->n_slots; }
const balm_assoc_opts &window_opts(const WindowState *w) { return w->opts; }

int window_reset_build(WindowState **ws, const char *who, int B, const int *n_slots, const balm_assoc_opts &o, bool batch) {
  if (o.layer_limit < 0 || o.layer_limit > 2) { balm_set_error(std::string(who) + ": layer_limit must be in 0..2"); return BALM_ERR_INVALID; }
  WindowState *w = new WindowState();
  w->P = AssocParams{o.voxel_size, o.layer_limit, o.min_ps, {o.eigen_value_array[0], o.eigen_value_array[1], o.eigen_value_array[2]}};
  w->opts = o;
  w->batch = batch;
  w->B = B;
  w->n_slots.assign(n_slots, n_slots + B);
  w->hprob.resize(B);
  int base = 0;
  for (int p = 0; p < B; p++) {
    w->hprob[p] = WinProb{n_slots[p], base, 0, 0};
    base += n_slots[p];
    w->N = std::max(w->N, n_slots[p]);
  }
  cudaError_t e = cudaMalloc((void **)&w->prob, sizeof(WinProb) * B);
  for (WinLookup &l : w->look)
    if (e == cudaSuccess && (e = cudaMalloc((void **)&l.off, sizeof(int) * (B + 1))) == cudaSuccess)
      e = cudaMemset(l.off, 0, sizeof(int) * (B + 1));
  if (e != cudaSuccess) {
    delete w;
    CUDA_TRY(e);
  }
  delete *ws;
  *ws = w;
  return BALM_OK;
}

int window_cut_build(cudaStream_t st, WindowState &w, const char *who, const int32_t *scan_of, const int *slot,
                     int n_scans, const int64_t *scan_ptr, const float *xyz_h, const double *poses12_h,
                     long long *launches) {
  // entries: the problems that take a non-empty scan, in problem order; their items are that scan's points in order
  std::vector<long long> item_ptr(1, 0), src_base;
  std::vector<int4> ent;
  for (int p = 0; p < w.B; p++) {
    const int s = scan_of[p];
    if (s < 0 || scan_ptr[s + 1] == scan_ptr[s]) continue;
    ent.push_back(make_int4(p, w.hprob[p].pose_base + slot[p], slot[p], 0));
    src_base.push_back(scan_ptr[s]);
    item_ptr.push_back(item_ptr.back() + (scan_ptr[s + 1] - scan_ptr[s]));
  }
  const int64_t n = item_ptr.back();
  if (n == 0) return BALM_OK;
  if (w.np + n >= (1ll << 31)) {
    balm_set_error(std::string(who) + ": 2^31 or more points in the window");
    return w.batch ? BALM_ERR_UNSUPPORTED : BALM_ERR_INVALID;
  }
  const int E = (int)ent.size(), m = (int)n, P = w.hprob.back().pose_base + w.hprob.back().n_slots;
  const int64_t n_points = scan_ptr[n_scans];
  ScratchPool pool;
  CubTmp tmp{pool};
  float *xyz = nullptr;
  double *poses = nullptr, *tran = nullptr;
  unsigned long long *rkey = nullptr;
  long long *d_iptr = nullptr, *d_sbase = nullptr;
  int4 *d_ent = nullptr;
  int *bad = nullptr, *order = nullptr, *src = nullptr, *row = nullptr, *iprob = nullptr;
  TRY(pool.get(&xyz, 3 * (size_t)n_points)); TRY(pool.get(&poses, 12 * (size_t)P)); TRY(pool.get(&tran, 3 * (size_t)m));
  TRY(pool.get(&rkey, m)); TRY(pool.get(&bad, w.B)); TRY(pool.get(&order, m)); TRY(pool.get(&src, m));
  TRY(pool.get(&row, m)); TRY(pool.get(&iprob, m)); TRY(pool.get(&d_iptr, E + 1)); TRY(pool.get(&d_sbase, E));
  TRY(pool.get(&d_ent, E));
  CUDA_TRY(cudaMemcpyAsync(xyz, xyz_h, sizeof(float) * 3 * n_points, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(poses, poses12_h, sizeof(double) * 12 * P, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(d_iptr, item_ptr.data(), sizeof(long long) * (E + 1), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(d_sbase, src_base.data(), sizeof(long long) * E, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(d_ent, ent.data(), sizeof(int4) * E, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemsetAsync(bad, 0, sizeof(int) * w.B, st));
  const unsigned g = (unsigned)((m + 255) / 256);
  expand_rows_kernel<<<E, 256, 0, st>>>(d_iptr, d_sbase, src, row);
  win_cut_kernel<<<g, 256, 0, st>>>(xyz, src, row, d_ent, poses, m, w.P, tran, rkey, iprob, bad);
  std::vector<int> h_bad(w.B);
  CUDA_TRY(cudaMemcpyAsync(h_bad.data(), bad, sizeof(int) * w.B, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  for (int p = 0; p < w.B; p++)
    if (h_bad[p]) {
      balm_set_error(std::string(who) + (w.batch ? ": problem " + std::to_string(p) : std::string()) +
                     ": a point lies outside the +-2^18 root-voxel range");
      return BALM_ERR_INVALID;
    }
  // nothing was changed so far; from here on the scans are committed
  TRY(win_add_nodes(w, pool, tmp, st, rkey, iprob, m, 0));
  TRY(win_reserve_points(w, w.np + m));
  const int64_t b = w.np;
  CUDA_TRY(cudaMemcpyAsync(w.ptran + 3 * b, tran, sizeof(double) * 3 * m, cudaMemcpyDeviceToDevice, st));
  win_store_kernel<<<g, 256, 0, st>>>(xyz, src, row, d_ent, m, w.op++, w.pxyz + 3 * b, w.pslot + b, w.pprob + b,
                                      w.pstamp + b);
  win_find_kernel<<<g, 256, 0, st>>>(rkey, iprob, nullptr, m, w.look[0].key, w.look[0].id, w.look[0].off, w.pnode + b);
  win_iota_kernel<<<g, 256, 0, st>>>(order, m, (int)b);
  w.np += m;
  TRY(win_push_points(w, pool, tmp, st, order, m));
  CUDA_TRY(cudaStreamSynchronize(st));
  *launches += 12;
  return BALM_OK;
}

int window_recut_build(cudaStream_t st, WindowState &w, const int *win_count, long long *launches) {
  TRY(win_upload(w, st, win_count, nullptr));
  for (int L = 0; L <= w.P.layer_limit; L++) {
    ScratchPool pool;
    CubTmp tmp{pool};
    if (w.nn == 0) return BALM_OK;
    CUDA_TRY(cudaMemsetAsync(w.naction, 0, sizeof(int) * w.nn, st));
    win_judge_kernel<<<(w.nn + 127) / 128, 128, 0, st>>>(w.nn, L, w.N, w.P, w.prob, w.nprob, w.nlayer, w.nsplit, w.npush,
                                                         w.nfix, w.sig_o, w.sig_t, w.naction);
    *launches += 1;
    if (L == w.P.layer_limit || w.np == 0) break;
    const int np = (int)w.np;
    unsigned long long *ckey = nullptr, *mkey = nullptr, *stamp = nullptr, *stamp2 = nullptr;
    int *flag = nullptr, *iota = nullptr, *mv = nullptr, *mv2 = nullptr, *mprob = nullptr, *nsel = nullptr;
    TRY(pool.get(&ckey, np)); TRY(pool.get(&flag, np)); TRY(pool.get(&iota, np)); TRY(pool.get(&mv, np));
    TRY(pool.get(&nsel, 1));
    const unsigned g = (unsigned)((np + 255) / 256);
    win_move_kernel<<<g, 256, 0, st>>>(w.np, w.P, w.prob, w.pprob, w.pnode, w.pslot, w.ptran, w.naction, w.nkey, w.nlayer,
                                       ckey, flag);
    win_iota_kernel<<<g, 256, 0, st>>>(iota, np, 0);
    size_t b1 = 0;
    cub::DeviceSelect::Flagged(nullptr, b1, iota, flag, mv, nsel, np, st);
    TRY(tmp.need(b1));
    CUDA_TRY(cub::DeviceSelect::Flagged(tmp.p, tmp.bytes, iota, flag, mv, nsel, np, st));
    int m = 0;
    CUDA_TRY(cudaMemcpyAsync(&m, nsel, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    *launches += 3;
    if (m == 0) continue;
    TRY(pool.get(&mkey, m)); TRY(pool.get(&stamp, m)); TRY(pool.get(&stamp2, m)); TRY(pool.get(&mv2, m));
    TRY(pool.get(&mprob, m));
    const unsigned gm = (unsigned)((m + 255) / 256);
    win_gather_u64_kernel<<<gm, 256, 0, st>>>(ckey, mv, m, mkey);
    win_gather_i32_kernel<<<gm, 256, 0, st>>>(w.pprob, mv, m, mprob);
    TRY(win_add_nodes(w, pool, tmp, st, mkey, mprob, m, L + 1));       // children created on first use (:714-720)
    const WinLookup &lk = w.look[L + 1];
    win_find_kernel<<<gm, 256, 0, st>>>(mkey, mprob, mv, m, lk.key, lk.id, lk.off, w.pnode);
    // the moved points in the order the parents' lists hold them, appended after the children's earlier points
    win_gather_u64_kernel<<<gm, 256, 0, st>>>(w.pstamp, mv, m, stamp);
    size_t b2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, b2, stamp, stamp2, mv, mv2, m, 0, 64, st);
    TRY(tmp.need(b2));
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp.p, tmp.bytes, stamp, stamp2, mv, mv2, m, 0, 64, st));
    win_restamp_kernel<<<gm, 256, 0, st>>>(mv2, m, w.op++, w.pstamp);
    TRY(win_push_points(w, pool, tmp, st, mv2, m));
    CUDA_TRY(cudaStreamSynchronize(st));
    *launches += 10;
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int window_marginalize_build(cudaStream_t st, WindowState &w, const int *mg, const double *poses_h, const int *win_count,
                             long long *launches) {
  ScratchPool pool;
  CubTmp tmp{pool};
  TRY(win_upload(w, st, win_count, mg));
  double *poses = nullptr;
  if (poses_h) {
    const size_t P = (size_t)w.hprob.back().pose_base + w.hprob.back().n_slots;
    TRY(pool.get(&poses, 12 * P));
    CUDA_TRY(cudaMemcpyAsync(poses, poses_h, sizeof(double) * 12 * P, cudaMemcpyHostToDevice, st));
  }
  if (w.nn == 0) return BALM_OK;
  // the points first: they read the node's split flag only, and the slot before the shift
  if (w.np > 0) {
    const int np = (int)w.np;
    int *keep = nullptr, *iota = nullptr, *sel = nullptr, *nsel = nullptr;
    TRY(pool.get(&keep, np)); TRY(pool.get(&iota, np)); TRY(pool.get(&sel, np)); TRY(pool.get(&nsel, 1));
    const unsigned g = (unsigned)((np + 255) / 256);
    win_margi_point_kernel<<<g, 256, 0, st>>>(w.np, w.prob, w.pprob, poses, w.nsplit, w.pnode, w.pslot, w.pxyz, w.ptran,
                                              keep);
    win_iota_kernel<<<g, 256, 0, st>>>(iota, np, 0);
    size_t b1 = 0;
    cub::DeviceSelect::Flagged(nullptr, b1, iota, keep, sel, nsel, np, st);
    TRY(tmp.need(b1));
    CUDA_TRY(cub::DeviceSelect::Flagged(tmp.p, tmp.bytes, iota, keep, sel, nsel, np, st));
    int m = 0;
    CUDA_TRY(cudaMemcpyAsync(&m, nsel, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (m < np) {  // compact the point store (same capacity, order kept)
      float *xyz2 = nullptr;
      double *tran2 = nullptr;
      int *slot2 = nullptr, *prob2 = nullptr, *node2 = nullptr;
      unsigned long long *stamp2 = nullptr;
      const size_t cap = (size_t)w.pcap;
      if (cudaMalloc((void **)&xyz2, sizeof(float) * 3 * cap) != cudaSuccess ||
          cudaMalloc((void **)&tran2, sizeof(double) * 3 * cap) != cudaSuccess ||
          cudaMalloc((void **)&slot2, sizeof(int) * cap) != cudaSuccess ||
          cudaMalloc((void **)&prob2, sizeof(int) * cap) != cudaSuccess ||
          cudaMalloc((void **)&node2, sizeof(int) * cap) != cudaSuccess ||
          cudaMalloc((void **)&stamp2, sizeof(unsigned long long) * cap) != cudaSuccess) {
        cudaFree(xyz2); cudaFree(tran2); cudaFree(slot2); cudaFree(prob2); cudaFree(node2); cudaFree(stamp2);
        CUDA_TRY(cudaErrorMemoryAllocation);
      }
      if (m > 0)
        win_compact_kernel<<<(m + 255) / 256, 256, 0, st>>>(sel, m, w.pxyz, w.ptran, w.pslot, w.pprob, w.pnode, w.pstamp,
                                                            xyz2, tran2, slot2, prob2, node2, stamp2);
      CUDA_TRY(cudaStreamSynchronize(st));
      cudaFree(w.pxyz); cudaFree(w.ptran); cudaFree(w.pslot); cudaFree(w.pprob); cudaFree(w.pnode); cudaFree(w.pstamp);
      w.pxyz = xyz2; w.ptran = tran2; w.pslot = slot2; w.pprob = prob2; w.pnode = node2; w.pstamp = stamp2;
      w.np = m;
    }
    *launches += 3;
  }
  win_margi_node_kernel<<<(w.nn + 127) / 128, 128, 0, st>>>(w.nn, w.N, w.prob, w.nprob, poses, w.nsplit, w.npush, w.nfix,
                                                            w.sig_o, w.sig_t);
  CUDA_TRY(cudaStreamSynchronize(st));
  CUDA_TRY(cudaGetLastError());
  *launches += 1;
  return BALM_OK;
}

int window_push_build(cudaStream_t st, WindowState &w, const int *win_count, const WindowRegister &reg,
                      long long *launches) {
  ScratchPool pool;
  CubTmp tmp{pool};
  TRY(win_upload(w, st, win_count, nullptr));
  const int nn = w.nn, B = w.B;
  int M = 0;
  int *flag = nullptr, *iota = nullptr, *sel = nullptr, *nsel = nullptr;
  if (nn > 0) {
    TRY(pool.get(&flag, nn)); TRY(pool.get(&iota, nn)); TRY(pool.get(&sel, nn)); TRY(pool.get(&nsel, 1));
    const unsigned g = (unsigned)((nn + 127) / 128);
    win_push_flag_kernel<<<g, 128, 0, st>>>(nn, w.N, w.P.min_ps, w.prob, w.nprob, w.nsplit, w.npush, w.sig_o, flag);
    win_iota_kernel<<<g, 128, 0, st>>>(iota, nn, 0);
    size_t b1 = 0;
    cub::DeviceSelect::Flagged(nullptr, b1, iota, flag, sel, nsel, nn, st);
    TRY(tmp.need(b1));
    CUDA_TRY(cub::DeviceSelect::Flagged(tmp.p, tmp.bytes, iota, flag, sel, nsel, nn, st));
    CUDA_TRY(cudaMemcpyAsync(&M, nsel, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    *launches += 3;
  }
  std::vector<int64_t> h((size_t)2 * (B + 1), 0);  // voxel_ptr | obs_ptr
  WindowEmit out{};
  if (M == 0) {
    TRY(reg(h.data(), h.data() + B + 1, &out));
    CUDA_TRY(cudaMemsetAsync(out.row_ptr, 0, sizeof(long long), st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return BALM_OK;
  }
  // ascending (problem, key) (unique among one problem's pushed nodes: a pushed node is not split, so none of its
  // ancestors is pushed)
  unsigned long long *k = nullptr, *k2 = nullptr;
  int *ids = nullptr, *ids2 = nullptr, *cnt = nullptr, *ostart = nullptr;
  long long *ptrs = nullptr;
  TRY(pool.get(&k, M)); TRY(pool.get(&k2, M)); TRY(pool.get(&ids2, M)); TRY(pool.get(&cnt, M)); TRY(pool.get(&ostart, M));
  TRY(pool.get(&ptrs, 2 * ((size_t)B + 1)));
  const unsigned gm = (unsigned)((M + 127) / 128);
  ids = sel;
  win_gather_u64_kernel<<<gm, 128, 0, st>>>(w.nkey, ids, M, k);
  TRY(win_sort_ids(w, pool, tmp, st, k, ids, k2, ids2, M));
  win_obs_count_kernel<<<gm, 128, 0, st>>>(ids, M, w.N, w.prob, w.nprob, w.sig_o, cnt);
  size_t b3 = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, b3, cnt, ostart, M, st);
  TRY(tmp.need(b3));
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp.p, tmp.bytes, cnt, ostart, M, st));
  win_push_ptr_kernel<<<(B + 128) / 128, 128, 0, st>>>(ids, M, w.nprob, cnt, ostart, B, ptrs, ptrs + B + 1);
  CUDA_TRY(cudaMemcpyAsync(h.data(), ptrs, sizeof(long long) * 2 * (B + 1), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  const int64_t K = h[2 * (size_t)B + 1];
  TRY(reg(h.data(), h.data() + B + 1, &out));
  win_emit_kernel<<<gm, 128, 0, st>>>(ids, ostart, M, K, w.N, w.prob, w.nprob, w.sig_o, w.nfix, w.nkey, w.nlayer, out);
  CUDA_TRY(cudaStreamSynchronize(st));
  CUDA_TRY(cudaGetLastError());
  *launches += 8;
  return BALM_OK;
}

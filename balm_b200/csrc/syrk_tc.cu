// syrk_tc.cu -- tensor-core path of the rank-3M symmetric update S = G'^T G' (kernel K4).
//
// The tensor cores have no fp64 MMA kind at int8 rates, so the fp64 product is computed EXACTLY in integers
// (Ozaki-style split):
//   per column j of G' (= one pose DOF) a power-of-two scale sc_j = 2^p_j with |G'[c][j]| * sc_j < 2^(8S-2);
//   X[c][j] = rint(G'[c][j] * sc_j) is split into S balanced base-256 digits q_s in [-128,127] (int8 planes);
//   T_d = sum_{s+t=d} sum_c q_s[c][i] * q_t[c][j]  accumulates in int32 register accumulators with NO rounding
//   (|product| <= 2^14, at most S*rows < 2^17 terms per accumulator -> |T_d| < 2^31);
//   S_ij = (256^(S-1)/sc_i)(256^(S-1)/sc_j) * sum_{d<S} 256^-d T_d   evaluated in fp64 by the epilogue.
// The only approximation is the fixed-point rounding of G' to 8S-2 = 30 bits below each column's maximum
// (S = 4) and the dropped digit pairs s+t >= S (same order); integer accumulation is associative, so the
// result does not depend on tile order, k-splits or the number of GPUs.
//
// Kernel anatomy (syrk_tc_kernel; one CTA per SM, persistent over (tile, column half, k-split) items, 384 threads):
//   warp 8    : TMA producer -- cp.async.bulk.tensor.3d of the S int8 planes of the A block (128 columns bi, 128B
//               swizzle) and of the B half block (64 columns of bj, 64B swizzle), KS = 64 contraction rows per stage,
//               into the A and B rings (see Rings: 160-224 KB of shared memory in all, mbarrier full/empty per slot)
//   warps 9-11: B transposers -- load each landed B slot into registers, free it, and store the K-major core
//               matrices into a slot of the BT ring
//   warps 0-7 : consumers, two warpgroups of 64 output rows each -- wgmma m64n64k32 s8 x s8 -> s32 with A from
//               registers and B from the K-major copy, S(S+1)/2 digit-pair products per k32 step into S register
//               accumulators; then the epilogue: fp64 Horner combine, column scales, fp64 partial tile to global
//               (same partial layout as the fp64 path -> same assemble kernel)
// The register accumulators (S * 64 x 64 int32 per warpgroup = 128 registers per consumer thread at S = 4) are what
// bounds the output tile to 128 x 64. The digit planes are stored MN-major (pose index contiguous, as the observation
// sweep writes them coalesced) while s8 wgmma reads shared-memory operands K-major only. So A is transposed on its way
// into registers (ldmatrix.trans of 16-bit pairs, then byte permutes), once per plane and k32 step, and feeds all the
// S - s products of its plane; B is transposed once per stage by the transposer warps. Both sides assign the same
// contraction row to each k position of the MMA (the k position map below), so the integer sums are those of the plain
// product, bit for bit.
#include <cuda.h>
#include <vector>
#include <algorithm>
#include "internal.cuh"

namespace {

constexpr int TILE = BALM_SYRK_TILE;  // 128
constexpr int HALF = TILE / 2;        // output columns of one item
constexpr int SMAX = 4;               // digit planes
constexpr int KS = 64;                // contraction rows per pipeline stage
constexpr int A_PLANE_BYTES = KS * TILE;  // 8192: one plane of the A block, one stage (128-byte rows)
constexpr int B_PLANE_BYTES = KS * HALF;  // 4096: one plane of the B half block, one stage (64-byte rows)
constexpr int BT_PLANE_BYTES = KS * HALF; // 4096: the same plane K-major (wgmma core matrices, see bt_offset)
constexpr int MAX_SLOTS = 8;             // barriers per ring
constexpr int BAR_BYTES = 6 * MAX_SLOTS * 8;
constexpr int RING_BYTES = 227 * 1024 - 1024 - BAR_BYTES;  // the block's whole shared memory but alignment slack, barriers
// Three rings, one slot per 64-row stage each, all advancing by one slot per stage: A (S planes of the A block, TMA),
// B (S planes of the B half block as TMA lands them, MN-major) and BT (their K-major copies). A slot of B is free again
// as soon as the transposers have loaded it into registers, a slot of BT once the consumers' MMAs on it retired, so
// neither the in-flight loads nor the MMAs hold a copy they do not use. Depths per S (A x B x BT slots), chosen with
// the BALM_TC_TRACE per-role clocks and the benchmark at its C3 shape (S = 3): with two BT slots the transposers run
// only one stage ahead of the consumers, whose waits on BT then dominate; deeper A or B rings than below measured no
// faster:
//   S = 2: 6 x 16 KB + 4 x 8 KB + 4 x 8 KB = 160 KB; S = 3: 4 x 24 + 4 x 12 + 4 x 12 = 192 KB;
//   S = 4: 4 x 32 + 2 x 16 + 4 x 16 = 224 KB
template <int S>
struct Rings {
  static constexpr int DA = S == 2 ? 6 : 4, DB = S == 4 ? 2 : 4, DT = 4;
  static constexpr int A_SLOT = S * A_PLANE_BYTES, B_SLOT = S * B_PLANE_BYTES, T_SLOT = S * BT_PLANE_BYTES;
  static constexpr int B_OFF = DA * A_SLOT, T_OFF = B_OFF + DB * B_SLOT, BYTES = T_OFF + DT * T_SLOT;
  static_assert(BYTES <= RING_BYTES && DA <= MAX_SLOTS && DB <= MAX_SLOTS && DT <= MAX_SLOTS, "ring layout");
  static_assert(A_SLOT % 1024 == 0 && B_SLOT % 1024 == 0 && T_SLOT % 1024 == 0, "swizzle alignment");
};
// slot and phase of a ring of D slots
template <int D>
struct RingPos {
  int slot = 0;
  uint32_t ph = 0;
  __device__ __forceinline__ void next() {
    if (++slot == D) { slot = 0; ph ^= 1; }
  }
};
constexpr int CONSUMER_WARPS = 8;
constexpr int TRANSPOSE_WARPS = 3;                      // warps 9-11
constexpr int TC_THREADS = 32 * (CONSUMER_WARPS + 4);   // two consumer warpgroups + one producer warpgroup
// register split (setmaxnreg): the producer warpgroup gives registers up so the consumers can hold their accumulators
// (S * 32 + 2 * S * 4 A-fragment registers); the transposers keep a whole stage of their ldmatrix results (up to 44
// registers at S = 4). The pool is what the launch allocated, 384 threads x 168 registers, and setmaxnreg.inc waits
// until the registers are free: 2 * 128 * 216 + 128 * 72 <= 384 * 168
constexpr int CONSUMER_REGS = 216, PRODUCER_REGS = 72;
constexpr int TC_SMEM = RING_BYTES + 1024 + BAR_BYTES;  // rings + alignment slack + barriers
constexpr int MAX_ROWS_PER_ITEM = BALM_TC_MAX_ROWS_PER_ITEM;  // 32704: 4 * rows * 2^14 < 2^31 (a multiple of KS)
static_assert(MAX_ROWS_PER_ITEM % KS == 0 && 4ll * MAX_ROWS_PER_ITEM * (1 << 14) < (1ll << 31), "int32 exactness bound");

// ---------------- PTX wrappers ----------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
// Bounded spin: a pipeline bug must not hang the GPU. On timeout set the error flag and bail out.
__device__ __forceinline__ bool mbar_wait(uint64_t *bar, uint32_t parity, int *err) {
  const uint32_t a = smem_u32(bar);
  for (long long it = 0; it < (1ll << 22); it++) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(ok)
        : "r"(a), "r"(parity)
        : "memory");
    if (ok) return true;
    if ((it & 1023) == 1023 && *((volatile int *)err) != 0) return false;
  }
  atomicExch(err, 2);
  return false;
}

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;\n" : "=l"(t));
  return t;
}
// BALM_TC_TRACE (balm_debug_tc_trace): per-CTA word offsets of the stage count, the consumer warp 0 globaltimer pair and
// the clock64 sums of the consumer warps 0 and 4 (5 each), of transposer warp 9 (3) and of the producer (2)
constexpr int TR_STAGES = 0, TR_NS = 1, TR_CONS = 3, TR_XPOSE = 13, TR_PROD = 16, TR_WORDS = BALM_TC_TRACE_WORDS;
static_assert(TR_PROD + 2 == TR_WORDS, "trace layout");
// clock64 in the traced instantiation; the untraced one reads no clock
template <bool TRACE>
__device__ __forceinline__ long long tclock() {
  if constexpr (TRACE) return clock64();
  else return 0;
}

__device__ __forceinline__ void tma_load_3d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];\n"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// Four 8 x 8 matrices of 16-bit pairs, transposed: lane 8q + i gives the address of row i of matrix q; thread
// (g = lane/4, t = lane%4) receives in r[q] the pair g of row 2t (low half) and of row 2t + 1 (high half).
__device__ __forceinline__ void ldsm_x4_trans(uint32_t addr, uint32_t *r) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}

// Contraction rows and k positions. A k32 step covers 32 contraction rows: four groups of 8, one ldmatrix matrix each.
// Thread t's two rows 2t, 2t + 1 of groups q and q + 1 go to the four k positions 4t..4t+3 (q = 0) and 16+4t..16+4t+3
// (q = 2) of the MMA: k position 16 h + 4 t + j holds contraction row 16 h + 2 t + (j & 1) + 8 (j >> 1). A (in
// registers) and B (in the K-major copy) use the same map; as it is a bijection, the products are those of the plain
// contraction.
// From the ldmatrix.trans result of pairs (c, c + 1) at the rows of groups q, q + 1: the 4 k positions of column c
// (0x6420, even bytes) or c + 1 (0x7531, odd bytes).
constexpr uint32_t PERM_EVEN = 0x6420, PERM_ODD = 0x7531;

// K-major copy of one B plane, one stage: wgmma core matrices of 8 columns x 16 k bytes (128 contiguous bytes,
// no swizzle); k32 step c at c * 2048, column group n / 8 at (n / 8) * 256 (SBO), k half at 128 (LBO). The 4 k positions
// 4 kword .. 4 kword + 3 (kword in 0..7) of column n are the word at
//   bt_offset(c, n, kword) = c * BT_CHUNK + (n >> 3) * BT_SBO + (kword >> 2) * BT_LBO + (n & 7) * 16 + 4 * (kword & 3).
constexpr int BT_LBO = 128, BT_SBO = 256, BT_CHUNK = 2048;
__device__ __forceinline__ uint64_t bt_desc(uint32_t saddr) {  // wgmma matrix descriptor, no swizzle
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)(BT_LBO >> 4) << 16) | ((uint64_t)(BT_SBO >> 4) << 32);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
__device__ __forceinline__ void fence_acc(int32_t (&d)[32]) {
#pragma unroll
  for (int i = 0; i < 32; i++) asm volatile("" : "+r"(d[i])::"memory");
}

// D (64 x 64 s32, accumulated) += A (64 x 32 s8, registers) * B (32 x 64 s8, K-major shared memory)
__device__ __forceinline__ void wgmma_s8(int32_t (&d)[32], const uint32_t (&a)[4], uint64_t desc_b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, 1;\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
        "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
        "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
        "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b)
      : "memory");
}

// true iff every thread of the calling warpgroup (named barrier id, 128 threads) passes ok = true
__device__ __forceinline__ bool warpgroup_all(bool ok, int id) {
  uint32_t r;
  asm volatile(
      "{\n\t.reg .pred p, q;\n\t"
      "setp.ne.u32 p, %1, 0;\n\t"
      "bar.red.and.pred q, %2, 128, p;\n\t"
      "selp.u32 %0, 1, 0, q;\n\t}\n"
      : "=r"(r)
      : "r"((uint32_t)ok), "r"(id)
      : "memory");
  return r != 0;
}

struct TcArgs {
  int64_t rows;       // contraction rows of this batch (3 per voxel)
  int nb, tiles, splits;
  const int *S_dev;   // digit-plane count chosen by tc_scale_kernel
  const double *isc;  // [ldq]  256^(S-1) / sc_j
  double *part;       // [splits][tiles][128*128]
  int accumulate;
  int *err;
  unsigned long long *trace;  // [gridDim.x][TR_WORDS], written by the traced instantiation only
};

struct ItemInfo {
  int bi, bj, h, sp, t;
  int nsteps;
  int64_t k_begin;
};

__device__ __forceinline__ void tile_coords_tc(int t, int nb, int &bi, int &bj) {
  int r = 0, rem = t;
  while (rem >= nb - r) { rem -= nb - r; r++; }
  bi = r;
  bj = r + rem;
}

// Items are distributed round robin over the CTAs: item blockIdx.x, blockIdx.x + gridDim.x, ...
__device__ __forceinline__ int n_items(const TcArgs &a) { return a.tiles * 2 * a.splits; }
// contraction rows of a k-split item: ceil(rows / splits) rounded up to KS
__device__ __forceinline__ int64_t rows_per_item(const TcArgs &a) {
  return ((a.rows + a.splits - 1) / a.splits + KS - 1) / KS * KS;
}

// work = (sp * tiles + t) * 2 + h: the two column halves of a tile run on neighbouring CTAs and share the A block in L2
__device__ __forceinline__ ItemInfo decode_item(const TcArgs &a, int work, int64_t per) {
  ItemInfo it;
  it.h = work & 1;
  it.t = (work >> 1) % a.tiles;
  it.sp = (work >> 1) / a.tiles;
  tile_coords_tc(it.t, a.nb, it.bi, it.bj);
  it.k_begin = (int64_t)it.sp * per;
  int64_t k_end = it.k_begin + per;
  if (k_end > a.rows) k_end = a.rows;
  it.nsteps = k_end > it.k_begin ? (int)((k_end - it.k_begin + KS - 1) / KS) : 0;
  return it;
}

// Shared-memory barriers of the three rings (MAX_SLOTS each): full = the slot holds its stage, empty = it may be refilled
struct RingBars {
  uint64_t *full_a, *empty_a, *full_b, *empty_b, *full_t, *empty_t;
};

// One consumer warpgroup (wg = 0, 1): output rows 64 wg .. 64 wg + 63 of the 128 x 64 half tile, all items of this
// CTA. Warp w (0..7) holds the 16 rows of 16-byte chunk w of the A block: fragment row g is output row 16 w + 2 g,
// fragment row g + 8 is output row 16 w + 2 g + 1; fragment column n is column n of the half tile.
template <int S, bool TRACE>
__device__ __forceinline__ void consumer_loop(const TcArgs &a, uint32_t ring, const RingBars &bar) {
  using R = Rings<S>;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3, i = lane & 7, wg = warp >> 2;
  // ldmatrix row of this lane: contraction row 8 (lane / 8) + i of a k32 step, chunk `warp` under the 128B swizzle;
  // the 8 rows of each matrix sit in 8 different chunks, so the loads are free of bank conflicts
  const uint32_t lda = ring + ((lane >> 3) * 8 + i) * TILE + ((warp ^ i) << 4);
  const uint32_t bt_ring = ring + R::T_OFF;
  const double inv256 = 1.0 / 256.0;
  long long tr[4] = {0, 0, 0, 0};  // trace: wait A full, wait BT full, wgmma.wait_group, epilogue
  const long long t_start = tclock<TRACE>();
  const unsigned long long ns_start = TRACE ? globaltimer_ns() : 0;
  int k = 0;  // stages consumed so far: stage k sits in slot k % D of a ring of D slots, phase (k / D) & 1
  const int64_t per = rows_per_item(a);
  for (int item = blockIdx.x; item < n_items(a); item += gridDim.x) {
    const ItemInfo info = decode_item(a, item, per);
    int32_t acc[S][32];
#pragma unroll
    for (int d = 0; d < S; d++)
#pragma unroll
      for (int q = 0; q < 32; q++) acc[d][q] = 0;
    uint32_t af[2][S][4];  // A fragments of every plane, one set per k32 step of a stage (the other may be in flight)
    bool alive = true;
    for (int ks = 0; ks < info.nsteps; ks++, k++) {
      const int sla = k % R::DA, slt = k % R::DT;
      const long long t0 = tclock<TRACE>();
      const bool ok_a = mbar_wait(&bar.full_a[sla], (k / R::DA) & 1, a.err);
      const long long t1 = tclock<TRACE>();
      const bool ok = warpgroup_all(ok_a && mbar_wait(&bar.full_t[slt], (k / R::DT) & 1, a.err), 1 + wg);
      if constexpr (TRACE) { tr[0] += t1 - t0; tr[1] += clock64() - t1; }
      if (!ok) { alive = false; break; }  // the warpgroup leaves together (wgmma is .aligned)
      const uint32_t sa = lda + sla * R::A_SLOT;
      const uint64_t sdesc = bt_desc(bt_ring + slt * R::T_SLOT);
#pragma unroll
      for (int c = 0; c < KS / 32; c++) {
#pragma unroll
        for (int s = 0; s < S; s++) {
          uint32_t m[4];
          ldsm_x4_trans(sa + s * A_PLANE_BYTES + c * 32 * TILE, m);
          af[c][s][0] = __byte_perm(m[0], m[1], PERM_EVEN);
          af[c][s][1] = __byte_perm(m[0], m[1], PERM_ODD);
          af[c][s][2] = __byte_perm(m[2], m[3], PERM_EVEN);
          af[c][s][3] = __byte_perm(m[2], m[3], PERM_ODD);
        }
        wgmma_fence();
#pragma unroll
        for (int s = 0; s < S; s++)
#pragma unroll
          for (int tt = 0; tt + s < S; tt++)
            wgmma_s8(acc[s + tt], af[c][s], sdesc + ((tt * BT_PLANE_BYTES + c * BT_CHUNK) >> 4));
        wgmma_commit();
        // every group but this one has retired: after the first k32 step that frees the previous stage, after the
        // second the A fragments of the first
        const long long t2 = tclock<TRACE>();
        wgmma_wait<1>();
        if constexpr (TRACE) tr[2] += clock64() - t2;
        if (c == 0 && ks > 0) {  // the previous stage's MMAs have retired: free its A and BT slots
          __syncwarp();
          if (lane == 0) {
            mbar_arrive(&bar.empty_a[(k - 1) % R::DA]);
            mbar_arrive(&bar.empty_t[(k - 1) % R::DT]);
          }
        }
      }
    }
    const long long t3 = tclock<TRACE>();
    wgmma_wait<0>();
#pragma unroll
    for (int d = 0; d < S; d++) fence_acc(acc[d]);
    const long long t4 = tclock<TRACE>();
    if constexpr (TRACE) tr[2] += t4 - t3;
    if (!alive) break;
    if (info.nsteps > 0) {
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&bar.empty_a[(k - 1) % R::DA]);
        mbar_arrive(&bar.empty_t[(k - 1) % R::DT]);
      }
    }
    // ---- epilogue: Horner over the digit-pair order d = S-1 .. 0, column scales, fp64 partial tile ----
    double *tile_out = a.part + ((size_t)info.sp * a.tiles + info.t) * (TILE * TILE);
#pragma unroll
    for (int up = 0; up < 2; up++) {
      const int row = 16 * warp + 2 * g + up;
      const double isc_row = __ldg(a.isc + info.bi * TILE + row);
      double *out = tile_out + (size_t)row * TILE + info.h * HALF;
#pragma unroll
      for (int j = 0; j < HALF / 8; j++) {
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int q = 4 * j + 2 * up + e;
          const int col = 8 * j + 2 * t + e;
          double val = (double)acc[S - 1][q];
#pragma unroll
          for (int d = S - 2; d >= 0; d--) val = val * inv256 + (double)acc[d][q];
          double w = val * isc_row * __ldg(a.isc + info.bj * TILE + info.h * HALF + col);
          if (a.accumulate) w += out[col];
          out[col] = w;
        }
      }
    }
    if constexpr (TRACE) tr[3] += clock64() - t4;
  }
  if constexpr (TRACE) {
    if ((warp & 3) == 0 && lane == 0) {
      unsigned long long *o = a.trace + (size_t)blockIdx.x * TR_WORDS;
      const long long total = clock64() - t_start;
#pragma unroll
      for (int w = 0; w < 4; w++) o[TR_CONS + 5 * wg + w] = tr[w];
      o[TR_CONS + 5 * wg + 4] = total;
      if (wg == 0) {
        o[TR_STAGES] = k;
        o[TR_NS] = ns_start;
        o[TR_NS + 1] = globaltimer_ns();
      }
    }
  }
}

__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;\n" ::"r"(addr), "r"(v) : "memory");
}

// One transposer warp (TW = 0..2): the K-major copies of the B half planes of every stage this CTA consumes. Work unit
// u = (plane p, k32 step c, 16-column chunk q) = 8 p + 4 c + q of a stage; warp TW takes u = TW, TW + 3, ... One
// ldmatrix.trans of a unit's 4 x 8 contraction rows gives thread (g, t) the k positions 4t..4t+3 and 16+4t..16+4t+3 of
// columns 16 q + 2 g and 16 q + 2 g + 1. A stage: wait for its B slot, issue all of the warp's ldmatrix loads and
// release the B slot, wait for a free BT slot, permute and store, publish the BT slot.
template <int S, int TW, bool TRACE>
__device__ __forceinline__ void transpose_loop(const TcArgs &a, uint32_t ring, const RingBars &bar) {
  using R = Rings<S>;
  constexpr int J = (8 * S - TW + 2) / 3;  // units of this warp per stage, all loaded before any store (4 J <= 44
                                          // registers of the producer warpgroup's PRODUCER_REGS)
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, i = lane & 7;
  // source row of this lane: contraction row 8 (lane / 8) + i of a k32 step; 64-byte rows under the 64B swizzle
  // (chunk q of row r at q ^ ((r >> 1) & 3)), so the 8 rows of each matrix hit 8 different 16-byte bank groups. The row
  // offset is a multiple of 64, so chunk q of a unit is at (src + slot, plane and step offsets) ^ (q << 4).
  const uint32_t src = ring + R::B_OFF + ((lane >> 3) * 8 + i) * HALF + ((i >> 1) << 4);
  // lanes g >= 4 store column 2g + 1 before 2g: the 32 lanes of every store then hit 32 different banks.
  // bt_offset(c, 16 q + n, kw) for this lane's column n = 2g + flip: c * BT_CHUNK + q * 2 BT_SBO + dst0 (kw = t) or
  // + BT_LBO (kw = 4 + t); its neighbour n ^ 1 sits at dst0 ^ 16
  const int flip = g >> 2, n = 2 * g + flip;
  const uint32_t perm0 = flip ? PERM_ODD : PERM_EVEN, perm1 = flip ? PERM_EVEN : PERM_ODD;
  const uint32_t dst = ring + R::T_OFF + (n >> 3) * BT_SBO + (n & 7) * 16 + 4 * t;
  long long tr[3] = {0, 0, 0};  // trace: wait B full, wait BT empty, total
  RingPos<R::DB> pb;
  RingPos<R::DT> pt;
  bool alive = true;
  const int64_t per = rows_per_item(a);
  for (int item = blockIdx.x; alive && item < n_items(a); item += gridDim.x) {
    const ItemInfo info = decode_item(a, item, per);
    for (int ks = 0; ks < info.nsteps; ks++) {
      const long long t0 = tclock<TRACE>();
      const bool ok = __all_sync(0xffffffffu, mbar_wait(&bar.full_b[pb.slot], pb.ph, a.err));
      if constexpr (TRACE) tr[0] += clock64() - t0;
      if (!ok) { alive = false; break; }
      const uint32_t sb = src + pb.slot * R::B_SLOT, db = dst + pt.slot * R::T_SLOT;
      uint32_t m[J][4];
#pragma unroll
      for (int j = 0; j < J; j++) {
        const int u = TW + 3 * j, p = u >> 3, c = (u >> 2) & 1, q = u & 3;
        ldsm_x4_trans((sb + p * B_PLANE_BYTES + c * 32 * HALF) ^ (q << 4), m[j]);
      }
      // the slot is refilled by TMA (async proxy) once released: the proxy fence orders these generic-proxy reads
      // before that write. Without it the arrive does not wait for the ldmatrix data, and the refill can overwrite the
      // slot before it is read.
      asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
      __syncwarp();
      if (lane == 0) mbar_arrive(&bar.empty_b[pb.slot]);
      const long long t1 = tclock<TRACE>();
      const bool free_t = __all_sync(0xffffffffu, mbar_wait(&bar.empty_t[pt.slot], pt.ph ^ 1, a.err));
      if constexpr (TRACE) tr[1] += clock64() - t1;
      if (!free_t) { alive = false; break; }
#pragma unroll
      for (int j = 0; j < J; j++) {
        const int u = TW + 3 * j, p = u >> 3, c = (u >> 2) & 1, q = u & 3;
        const uint32_t d = db + p * BT_PLANE_BYTES + c * BT_CHUNK + q * 2 * BT_SBO;
        sts_u32(d, __byte_perm(m[j][0], m[j][1], perm0));
        sts_u32(d ^ 16, __byte_perm(m[j][0], m[j][1], perm1));
        sts_u32(d + BT_LBO, __byte_perm(m[j][2], m[j][3], perm0));
        sts_u32((d + BT_LBO) ^ 16, __byte_perm(m[j][2], m[j][3], perm1));
      }
      asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");  // the copy is read by wgmma (async proxy)
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&bar.full_t[pt.slot]);
      }
      pb.next();
      pt.next();
      if constexpr (TRACE) tr[2] += clock64() - t0;
    }
  }
  if constexpr (TRACE) {
    if (TW == 0 && lane == 0) {
      unsigned long long *o = a.trace + (size_t)blockIdx.x * TR_WORDS;
      o[TR_XPOSE] = tr[0];
      o[TR_XPOSE + 1] = tr[1];
      o[TR_XPOSE + 2] = tr[2] - tr[0] - tr[1];  // busy
    }
  }
}

// The TMA producer (one thread): per stage, the S planes of the B half block into the B ring first (they still have to
// be transposed), then the S planes of the A block into the A ring.
template <int S, bool TRACE>
__device__ __forceinline__ void producer_loop(const TcArgs &a, const CUtensorMap *tmap_a, const CUtensorMap *tmap_b,
                                              uint8_t *ring, const RingBars &bar) {
  using R = Rings<S>;
  asm volatile("prefetch.tensormap [%0];\n" ::"l"(tmap_a) : "memory");
  asm volatile("prefetch.tensormap [%0];\n" ::"l"(tmap_b) : "memory");
  long long tr[2] = {0, 0};  // trace: wait A empty, wait B empty
  RingPos<R::DA> pa;
  RingPos<R::DB> pb;
  bool alive = true;
  const int64_t per = rows_per_item(a);
  for (int item = blockIdx.x; alive && item < n_items(a); item += gridDim.x) {
    const ItemInfo info = decode_item(a, item, per);
    for (int ks = 0; ks < info.nsteps; ks++) {
      const int krow = (int)(info.k_begin + (int64_t)ks * KS);
      const long long t0 = tclock<TRACE>();
      if (!mbar_wait(&bar.empty_b[pb.slot], pb.ph ^ 1, a.err)) { alive = false; break; }
      const long long t1 = tclock<TRACE>();
      uint8_t *sb = ring + R::B_OFF + pb.slot * R::B_SLOT;
      mbar_expect_tx(&bar.full_b[pb.slot], S * B_PLANE_BYTES);
      for (int s = 0; s < S; s++)
        tma_load_3d(sb + s * B_PLANE_BYTES, tmap_b, &bar.full_b[pb.slot], info.bj * TILE + info.h * HALF, krow, s);
      const long long t2 = tclock<TRACE>();
      if (!mbar_wait(&bar.empty_a[pa.slot], pa.ph ^ 1, a.err)) { alive = false; break; }
      if constexpr (TRACE) { tr[0] += clock64() - t2; tr[1] += t1 - t0; }
      uint8_t *sa = ring + pa.slot * R::A_SLOT;
      mbar_expect_tx(&bar.full_a[pa.slot], S * A_PLANE_BYTES);
      for (int s = 0; s < S; s++) tma_load_3d(sa + s * A_PLANE_BYTES, tmap_a, &bar.full_a[pa.slot], info.bi * TILE, krow, s);
      pa.next();
      pb.next();
    }
  }
  if constexpr (TRACE) {
    unsigned long long *o = a.trace + (size_t)blockIdx.x * TR_WORDS;
    o[TR_PROD] = tr[0];
    o[TR_PROD + 1] = tr[1];
  }
}

template <int S, bool TRACE>
__device__ __forceinline__ void syrk_tc_cta(const CUtensorMap *tmap_a, const CUtensorMap *tmap_b, const TcArgs &a,
                                            uint8_t *ring, const RingBars &bar) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t ring_u32 = smem_u32(ring);
  if (warp >= CONSUMER_WARPS) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(PRODUCER_REGS));
    // ===================== B transposers (warps 9-11) =====================
    if (warp == CONSUMER_WARPS + 1) transpose_loop<S, 0, TRACE>(a, ring_u32, bar);
    else if (warp == CONSUMER_WARPS + 2) transpose_loop<S, 1, TRACE>(a, ring_u32, bar);
    else if (warp == CONSUMER_WARPS + 3) transpose_loop<S, 2, TRACE>(a, ring_u32, bar);
    // ===================== TMA producer (warp 8, one thread) =====================
    else if (lane == 0) producer_loop<S, TRACE>(a, tmap_a, tmap_b, ring, bar);
  } else {
    // ===================== wgmma + epilogue =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(CONSUMER_REGS));
    consumer_loop<S, TRACE>(a, ring_u32, bar);
  }
}

template <bool TRACE>
__global__ void __launch_bounds__(TC_THREADS, 1) syrk_tc_kernel(const __grid_constant__ CUtensorMap tmap_a,
                                                                const __grid_constant__ CUtensorMap tmap_b, TcArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte aligned rings (the swizzle patterns are functions of the shared-memory address), then barriers
  uint8_t *ring = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t *bars = reinterpret_cast<uint64_t *>(ring + RING_BYTES);
  const RingBars bar{bars, bars + MAX_SLOTS, bars + 2 * MAX_SLOTS, bars + 3 * MAX_SLOTS, bars + 4 * MAX_SLOTS,
                     bars + 5 * MAX_SLOTS};
  if (threadIdx.x == 0) {
    for (int i = 0; i < MAX_SLOTS; i++) {
      mbar_init(&bar.full_a[i], 1);
      mbar_init(&bar.empty_a[i], CONSUMER_WARPS);
      mbar_init(&bar.full_b[i], 1);
      mbar_init(&bar.empty_b[i], TRANSPOSE_WARPS);
      mbar_init(&bar.full_t[i], TRANSPOSE_WARPS);
      mbar_init(&bar.empty_t[i], CONSUMER_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();
  const int S = *a.S_dev;
  if (S == 4) syrk_tc_cta<4, TRACE>(&tmap_a, &tmap_b, a, ring, bar);
  else if (S == 3) syrk_tc_cta<3, TRACE>(&tmap_a, &tmap_b, a, ring, bar);
  else syrk_tc_cta<2, TRACE>(&tmap_a, &tmap_b, a, ring, bar);
}

// Column scales and digit-plane count of one batch, decided ON THE DEVICE from the column maxima and sums of squares
// of G' (one block):
//   e_j = max|G'_j| / sqrt(sum G'_j^2)  is the concentration of column j (1 = a single dominant entry, ~1/sqrt(rows)
//   for evenly spread columns); rounding G' to 2^-(8S-2) of the column maximum perturbs H_ij by about
//   2^-(8S-2) * e * sqrt(H_ii H_jj).  S = 3 is used when that stays below 5e-9 for every column, else S = 4
//   (forced_S > 0 overrides).  Then sc_j = 2^p with colmax_j * sc_j in [2^(8S-3), 2^(8S-2)), isc_j = 256^(S-1)/sc_j.
//   fresh values (scale 2^p with |G'_j| 2^p in [2^(8S-3), 2^(8S-2)), S by the concentration rule) always go to
//   sc_next/isc_next/S_next (when given): they are what the NEXT evaluation of the same voxels speculates with.
//   spec = 0: they are also the scales of this batch (sc/isc/S_dev), *spec_ok = 0 -> the OBS_INT8 sweep runs.
//   spec = 1: the digit planes were ALREADY written by the fused sweep with sc/S_dev. They stand (*spec_ok = 1)
//             iff S is still what the rule asks for and every column (a) stayed inside the balanced-digit range,
//             |G'_j| sc_j < 0.99 * 2^(8S-1), and (b) kept a rounding unit 1/sc_j <= 1e-8 sqrt(sum G'_j^2) -- the bound
//             the S rule itself guarantees. Otherwise the fresh values are adopted and sweep 2 is re-armed.
__global__ void __launch_bounds__(1024) tc_scale_kernel(const unsigned long long *colmax_bits, const double *accum_batch,
                                                        int Np, int n, double *sc, double *isc, int ldq, int forced_S,
                                                        int *S_dev, int spec, double *sc_next, double *isc_next,
                                                        int *S_next, int *spec_ok) {
  __shared__ double red[32];
  __shared__ int S_sh, bad_sh;
  if (threadIdx.x == 0) bad_sh = 0;
  double emax = 0.0;
  for (int j = threadIdx.x; j < n; j += 1024) {
    const double m = __longlong_as_double((long long)colmax_bits[j]);
    const double h = accum_batch[(size_t)(27 + j % 6) * Np + j / 6];
    if (m > 0.0 && h > 0.0) emax = fmax(emax, m / sqrt(h));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) emax = fmax(emax, __shfl_xor_sync(0xffffffffu, emax, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = emax;
  __syncthreads();
  if (threadIdx.x == 0) {
    double e = 0.0;
    for (int w = 0; w < 32; w++) e = fmax(e, red[w]);
    int S = (e * (1.0 / 4194304.0) <= 5e-9) ? 3 : 4;  // 2^-22 * e
    if (forced_S > 0) S = forced_S;
    S_sh = S;
    if (spec && *S_dev != S) bad_sh = 1;
  }
  __syncthreads();
  const int S = S_sh;
  double *fsc = sc_next ? sc_next : sc, *fisc = sc_next ? isc_next : isc;  // where the fresh values go first
  int bad = 0;
  for (int j = threadIdx.x; j < ldq; j += 1024) {
    const double m = __longlong_as_double((long long)colmax_bits[j]);
    const bool live = (m > 0.0) && (m < 1e300);
    if (spec && live && j < n) {
      const double used = sc[j];
      const double h = accum_batch[(size_t)(27 + j % 6) * Np + j / 6];
      if (!(used > 0.0) || !(m * used < 0.99 * ldexp(1.0, 8 * S - 1)) || !(1.0 <= 1e-8 * sqrt(h) * used)) bad = 1;
    }
    if (!live) {
      fsc[j] = 0.0;
      fisc[j] = 0.0;
      continue;
    }
    int e;
    frexp(m, &e);  // m = f * 2^e, f in [0.5, 1)  ->  m < 2^e
    const int p = 8 * S - 2 - e;
    fsc[j] = ldexp(1.0, p);
    fisc[j] = ldexp(1.0, 8 * (S - 1) - p);
  }
  if (bad) atomicOr(&bad_sh, 1);
  __syncthreads();
  const bool keep = spec && !bad_sh;
  if (sc_next && !keep) {
    for (int j = threadIdx.x; j < ldq; j += 1024) {
      sc[j] = sc_next[j];
      isc[j] = isc_next[j];
    }
  }
  if (threadIdx.x == 0) {
    if (!keep) *S_dev = S;
    if (S_next) *S_next = S;
    *spec_ok = keep ? 1 : 0;
  }
}

// start of a speculative evaluation: the scales found by the previous one become the ones in use
// (skew: test hook BALM_TC_SPEC_SKEW -- the adopted scales are multiplied by 2^skew so that the device-side check
//  has something to reject; 0 in production)
__global__ void tc_adopt_kernel(double *sc, double *isc, int *S_dev, const double *sc_next, const double *isc_next,
                                const int *S_next, int ldq, int skew) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < ldq) {
    sc[j] = ldexp(sc_next[j], skew);
    isc[j] = ldexp(isc_next[j], -skew);
  }
  if (j == 0) *S_dev = *S_next;
}


typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

struct TcState {
  CUtensorMap map_a;        // box {128, KS, 1}, 128-byte swizzle: the A block
  CUtensorMap map_b;        // box {64, KS, 1}, 64-byte swizzle: one column half of the B block
  double *sc = nullptr, *isc = nullptr;
  double *sc_next = nullptr, *isc_next = nullptr;  // fresh scales of the last full-range evaluation (speculation)
  int *S_next = nullptr, *spec_ok = nullptr;
  bool spec_ready = false;                         // sc_next/S_next describe the currently registered voxels
  bool spec_enabled = true;                        // BALM_NO_SPEC=1 keeps the two-sweep path
  bool last_spec = false;                          // the batch in flight used the fused sweep
  int spec_skew = 0;                               // BALM_TC_SPEC_SKEW (tests)
  unsigned long long *colmax = nullptr;
  int *err = nullptr;
  int64_t rows_alloc = 0;
  int forced_S = 0;      // BALM_TC_SLICES override (0 = decided on the device per batch)
  int *S_dev = nullptr;  // [1]
  int last_S = 0;        // read back with the error flag (instrumentation)
  int64_t last_rows_padded = 0;  // contraction rows of the last batch's SYRK (0: none since the registration)
};

// The two tensor maps of a digit-plane buffer [SMAX][rows_alloc][ldq] (int8, column index fastest): the A block
// (box {128, KS, 1}, 128-byte swizzle) and one column half of the B block (box {64, KS, 1}, 64-byte swizzle).
int encode_tc_maps(int8_t *planes, int ldq, int64_t rows_alloc, CUtensorMap *map_a, CUtensorMap *map_b) {
  EncodeTiledFn encode = nullptr;
  cudaDriverEntryPointQueryResult qres;
  CUDA_TRY(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", (void **)&encode, cudaEnableDefault, &qres));
  if (!encode || qres != cudaDriverEntryPointSuccess) {
    balm_set_error("cuTensorMapEncodeTiled not available from the driver");
    return BALM_ERR_CUDA;
  }
  const cuuint64_t dims[3] = {(cuuint64_t)ldq, (cuuint64_t)rows_alloc, (cuuint64_t)SMAX};
  const cuuint64_t strides[2] = {(cuuint64_t)ldq, (cuuint64_t)ldq * rows_alloc};
  const cuuint32_t estr[3] = {1, 1, 1};
  const cuuint32_t box_a[3] = {TILE, KS, 1};
  if (encode(map_a, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, planes, dims, strides, box_a, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
    balm_set_error("cuTensorMapEncodeTiled (A block) failed");
    return BALM_ERR_CUDA;
  }
  const cuuint32_t box_b[3] = {HALF, KS, 1};
  if (encode(map_b, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, planes, dims, strides, box_b, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
    balm_set_error("cuTensorMapEncodeTiled (B half block) failed");
    return BALM_ERR_CUDA;
  }
  return BALM_OK;
}

// One syrk_tc_kernel launch on c's stream: rows_padded (a multiple of KS) contraction rows of the planes behind the
// maps, nb x nb blocks of 128 columns, `splits` k-splits; one CTA per item up to one per SM.
// With c->tc_trace (BALM_TC_TRACE) the traced instantiation runs and records the launch.
int launch_syrk_tc(balm_ctx *c, const CUtensorMap &map_a, const CUtensorMap &map_b, int64_t rows_padded, int nb,
                   int tiles, int splits, const int *S_dev, const double *isc, double *part, bool accumulate, int *err) {
  TcArgs a{rows_padded, nb, tiles, splits, S_dev, isc, part, accumulate ? 1 : 0, err, c->tc_trace};
  const int items = a.tiles * 2 * a.splits;
  const int grid = items < c->sm_count ? items : c->sm_count;
  if (c->tc_trace) {
    CUDA_TRY(cudaMemsetAsync(c->tc_trace, 0, sizeof(unsigned long long) * c->sm_count * TR_WORDS, c->stream));
    syrk_tc_kernel<true><<<grid, TC_THREADS, TC_SMEM, c->stream>>>(map_a, map_b, a);
  } else {
    syrk_tc_kernel<false><<<grid, TC_THREADS, TC_SMEM, c->stream>>>(map_a, map_b, a);
  }
  CUDA_TRY(cudaGetLastError());
  return BALM_OK;
}

int syrk_tc_set_smem() {
  CUDA_TRY(cudaFuncSetAttribute(syrk_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
  CUDA_TRY(cudaFuncSetAttribute(syrk_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
  return BALM_OK;
}

const char *const TC_TIMEOUT_MSG = "tensor-core SYRK pipeline timed out (mbarrier wait bound exceeded)";

}  // namespace

int tensor_syrk_init(balm_ctx *c) {
  tensor_syrk_free(c);
  TcState *st = new TcState();
  c->tmap = st;
  // Digit planes (3 or 4) are chosen per batch on the device (tc_scale_kernel); BALM_TC_SLICES=2..4 forces a count.
  if (const char *e = getenv("BALM_TC_SLICES")) {
    const int v = atoi(e);
    if (v >= 2 && v <= SMAX) st->forced_S = v;
  }
  const int ldq = c->ldg;
  st->rows_alloc = (3 * c->VB + KS - 1) / KS * KS;
  CUDA_TRY(cudaMalloc((void **)&c->Gq, (size_t)SMAX * st->rows_alloc * ldq));
  CUDA_TRY(cudaMemset(c->Gq, 0, (size_t)SMAX * st->rows_alloc * ldq));  // column padding [6N, ldg) stays zero
  CUDA_TRY(cudaMalloc((void **)&st->S_dev, sizeof(int)));
  CUDA_TRY(cudaMalloc((void **)&st->sc, sizeof(double) * ldq));
  CUDA_TRY(cudaMalloc((void **)&st->isc, sizeof(double) * ldq));
  CUDA_TRY(cudaMalloc((void **)&st->sc_next, sizeof(double) * ldq));
  CUDA_TRY(cudaMalloc((void **)&st->isc_next, sizeof(double) * ldq));
  CUDA_TRY(cudaMalloc((void **)&st->S_next, sizeof(int)));
  CUDA_TRY(cudaMalloc((void **)&st->spec_ok, sizeof(int)));
  CUDA_TRY(cudaMemset(st->spec_ok, 0, sizeof(int)));
  st->spec_enabled = getenv("BALM_NO_SPEC") == nullptr;
  if (const char *e = getenv("BALM_TC_SPEC_SKEW")) st->spec_skew = atoi(e);
  CUDA_TRY(cudaMalloc((void **)&st->colmax, sizeof(unsigned long long) * ldq));
  CUDA_TRY(cudaMalloc((void **)&st->err, sizeof(int)));
  CUDA_TRY(cudaMemset(st->err, 0, sizeof(int)));
  c->colmax = st->colmax;  // the observation pass writes the column maxima here

  TRY(encode_tc_maps(c->Gq, ldq, st->rows_alloc, &st->map_a, &st->map_b));
  // int32 exactness bound: every (tile, split) item contracts at most MAX_ROWS_PER_ITEM rows
  const int64_t rows = 3 * c->VB;
  const int min_splits = (int)((rows + MAX_ROWS_PER_ITEM - 1) / MAX_ROWS_PER_ITEM);
  if (c->syrk_splits < min_splits) {
    cudaFree(c->syrk_part);
    c->syrk_splits = min_splits;
    CUDA_TRY(cudaMalloc((void **)&c->syrk_part,
                        sizeof(double) * (size_t)c->syrk_splits * c->syrk_tiles * TILE * TILE));
  }
  TRY(syrk_tc_set_smem());
  return BALM_OK;
}

void tensor_syrk_free(balm_ctx *c) {
  if (c->tmap) {
    TcState *st = static_cast<TcState *>(c->tmap);
    cudaFree(st->sc_next); cudaFree(st->isc_next); cudaFree(st->S_next); cudaFree(st->spec_ok);
    cudaFree(st->sc); cudaFree(st->isc); cudaFree(st->colmax); cudaFree(st->err); cudaFree(st->S_dev);
    delete st;
    c->tmap = nullptr;
  }
  cudaFree(c->Gq);
  c->Gq = nullptr;
  c->colmax = nullptr;
}

// One batch of the tensor path: (1) column maxima of G' -> power-of-two scales, (2) observation sweep writing the
// int8 digit planes directly, (3) tensor-core SYRK. ev[2] is recorded between the observation sweeps and the SYRK.
int tensor_obs_and_syrk(balm_ctx *c, const double *poses, int64_t v0, int64_t v1, bool first_batch) {
  TcState *st = static_cast<TcState *>(c->tmap);
  if (!st) { balm_set_error("tensor path not initialised"); return BALM_ERR_INVALID; }
  const int ldq = c->ldg;
  const int64_t rows = 3 * (v1 - v0);
  const int64_t rows_padded = (rows + KS - 1) / KS * KS;
  CUDA_TRY(cudaMemsetAsync(st->colmax, 0, sizeof(unsigned long long) * ldq, c->stream));
  // Speculation lives inside one balm_damping_iter call only: its first evaluation sweeps twice, and the public
  // balm_evaluate always does -- so every entry point stays a pure function of its arguments (same inputs, same bits,
  // whatever was evaluated before).
  const bool full = c->lm_active && v0 == 0 && v1 == c->M;
  const bool spec = full && st->spec_ready && st->spec_enabled;
  const int64_t plane_stride = (int64_t)st->rows_alloc * ldq;
  int rc;
  if (spec) {  // one sweep with the previous evaluation's scales; sweep 2 below only runs if tc_scale_kernel re-arms it
    tc_adopt_kernel<<<(ldq + 255) / 256, 256, 0, c->stream>>>(st->sc, st->isc, st->S_dev, st->sc_next, st->isc_next,
                                                              st->S_next, ldq, st->spec_skew);
    c->launches += 1;
    rc = launch_obs_int8(c, poses, v0, v1, first_batch, st->sc, c->Gq, plane_stride, st->S_dev, SMAX, rows_padded, true,
                         nullptr);
  } else {
    rc = launch_obs_colmax(c, poses, v0, v1, first_batch);
  }
  if (rc != BALM_OK) return rc;
  tc_scale_kernel<<<1, 1024, 0, c->stream>>>(st->colmax, c->accum_batch, c->Np, c->n, st->sc, st->isc, ldq,
                                             st->forced_S, st->S_dev, spec ? 1 : 0, full ? st->sc_next : nullptr,
                                             full ? st->isc_next : nullptr, full ? st->S_next : nullptr, st->spec_ok);
  rc = launch_obs_int8(c, poses, v0, v1, first_batch, st->sc, c->Gq, plane_stride, st->S_dev, SMAX, rows_padded, false,
                       spec ? st->spec_ok : nullptr);
  if (rc != BALM_OK) return rc;
  if (full) st->spec_ready = true;
  st->last_spec = spec;
  st->last_rows_padded = rows_padded;
  CUDA_TRY(cudaEventRecord(c->ev[2], c->stream));
  c->launches += 2;
  return launch_syrk_tc(c, st->map_a, st->map_b, rows_padded, c->syrk_nb, c->syrk_tiles, c->syrk_splits, st->S_dev,
                        st->isc, c->syrk_part, !first_batch, st->err);
}

// The SYRK's error flag, the digit-plane count and the speculation verdict of the batch in flight: the copies are
// enqueued (pinned host words), the host reads them after its next synchronisation of the stream.
int tensor_syrk_check_enqueue(balm_ctx *c) {
  TcState *st = static_cast<TcState *>(c->tmap);
  if (!st) return BALM_OK;
  CUDA_TRY(cudaMemcpyAsync(c->h_flags + 1, st->err, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->h_flags + 2, st->S_dev, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->h_flags + 3, st->spec_ok, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  return BALM_OK;
}

int tensor_syrk_check_finish(balm_ctx *c) {  // after the stream has been synchronised
  TcState *st = static_cast<TcState *>(c->tmap);
  if (!st) return BALM_OK;
  st->last_S = c->h_flags[2];
  c->tm.digit_planes = st->last_S;
  if (st->last_spec) (c->h_flags[3] ? c->tm.single_sweeps : c->tm.redone_sweeps) += 1;
  if (c->h_flags[1] != 0) {
    balm_set_error(TC_TIMEOUT_MSG);
    return BALM_ERR_CUDA;
  }
  return BALM_OK;
}

int tensor_syrk_check(balm_ctx *c) {
  int rc = tensor_syrk_check_enqueue(c);
  if (rc != BALM_OK) return rc;
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  return tensor_syrk_check_finish(c);
}

// same-shape re-registration: the workspaces stay; the speculation and the record of the last batch (its planes now
// describe other voxels) do not
void tensor_syrk_new_problem(balm_ctx *c) {
  TcState *st = static_cast<TcState *>(c->tmap);
  if (st) {
    st->spec_ready = false;
    st->last_rows_padded = 0;
  }
}

// ---------------- debug hooks (include/balm_b200.h): the SYRK alone, and what it consumed ----------------
extern "C" int balm_debug_syrk_tc(balm_ctx *c, const int8_t *planes, int S, int64_t rows, const double *isc, int splits,
                                  int accumulate, double *part) {
  if (!c || !planes || !isc || !part) { balm_set_error("balm_debug_syrk_tc: bad arguments"); return BALM_ERR_INVALID; }
  TRY(refuse_blocks(c, "balm_debug_syrk_tc"));
  if (S < 2 || S > SMAX || rows < 1 || rows > ((int64_t)1 << 30) || splits < 1) {
    balm_set_error("balm_debug_syrk_tc: S must be 2..4, rows 1..2^30 and splits >= 1");
    return BALM_ERR_INVALID;
  }
  const int ldq = c->ldg, nb = ldq / TILE, tiles = nb * (nb + 1) / 2;
  const int64_t rows_padded = (rows + KS - 1) / KS * KS;
  const int64_t per = ((rows_padded + splits - 1) / splits + KS - 1) / KS * KS;  // as syrk_tc_kernel splits them
  if (per > MAX_ROWS_PER_ITEM || (int64_t)tiles * 2 * splits > (1 << 30)) {
    balm_set_error("balm_debug_syrk_tc: more than 32704 contraction rows per item (int32 exactness bound)");
    return BALM_ERR_INVALID;
  }
  CUDA_TRY(cudaSetDevice(c->device));
  const size_t plane = (size_t)rows_padded * ldq, count = (size_t)splits * tiles * TILE * TILE;
  ScratchPool pool;
  int8_t *d_planes;
  double *d_isc, *d_part;
  int *d_S, *d_err;
  TRY(pool.get(&d_planes, SMAX * plane));
  TRY(pool.get(&d_isc, (size_t)ldq));
  TRY(pool.get(&d_part, count));
  TRY(pool.get(&d_S, 1));
  TRY(pool.get(&d_err, 1));
  CUDA_TRY(cudaMemsetAsync(d_planes, 0, SMAX * plane, c->stream));  // K padding rows and unused planes
  for (int s = 0; s < S; s++)
    CUDA_TRY(cudaMemcpyAsync(d_planes + s * plane, planes + (size_t)s * rows * ldq, (size_t)rows * ldq,
                             cudaMemcpyHostToDevice, c->stream));
  CUDA_TRY(cudaMemcpyAsync(d_isc, isc, sizeof(double) * ldq, cudaMemcpyHostToDevice, c->stream));
  CUDA_TRY(cudaMemcpyAsync(d_part, part, sizeof(double) * count, cudaMemcpyHostToDevice, c->stream));
  CUDA_TRY(cudaMemcpyAsync(d_S, &S, sizeof(int), cudaMemcpyHostToDevice, c->stream));
  CUDA_TRY(cudaMemsetAsync(d_err, 0, sizeof(int), c->stream));
  CUtensorMap map_a, map_b;
  TRY(encode_tc_maps(d_planes, ldq, rows_padded, &map_a, &map_b));
  TRY(syrk_tc_set_smem());
  TRY(launch_syrk_tc(c, map_a, map_b, rows_padded, nb, tiles, splits, d_S, d_isc, d_part, accumulate != 0, d_err));
  int err = 0;
  CUDA_TRY(cudaMemcpyAsync(&err, d_err, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaMemcpyAsync(part, d_part, sizeof(double) * count, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  if (err != 0) {
    balm_set_error(TC_TIMEOUT_MSG);
    return BALM_ERR_CUDA;
  }
  return BALM_OK;
}

extern "C" int balm_debug_tc_planes(balm_ctx *c, int8_t *planes, double *isc, int *S, int64_t *rows_padded,
                                    int *splits) {
  if (c) TRY(refuse_blocks(c, "balm_debug_tc_planes"));
  TcState *st = (c && c->prec == BALM_PREC_TENSOR) ? static_cast<TcState *>(c->tmap) : nullptr;
  if (!st || st->last_rows_padded == 0) {
    balm_set_error("balm_debug_tc_planes: no tensor-path evaluation of the registered voxels");
    return BALM_ERR_INVALID;
  }
  CUDA_TRY(cudaSetDevice(c->device));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  int s = 0;
  CUDA_TRY(cudaMemcpy(&s, st->S_dev, sizeof(int), cudaMemcpyDeviceToHost));
  const size_t plane = (size_t)st->last_rows_padded * c->ldg;
  if (planes)
    for (int q = 0; q < s; q++)
      CUDA_TRY(cudaMemcpy(planes + q * plane, c->Gq + (size_t)q * st->rows_alloc * c->ldg, plane, cudaMemcpyDeviceToHost));
  if (isc) CUDA_TRY(cudaMemcpy(isc, st->isc, sizeof(double) * c->ldg, cudaMemcpyDeviceToHost));
  if (S) *S = s;
  if (rows_padded) *rows_padded = st->last_rows_padded;
  if (splits) *splits = c->syrk_splits;
  return BALM_OK;
}

extern "C" int balm_debug_tc_trace(balm_ctx *c, unsigned long long *out, int max_entries) {
  if (c) TRY(refuse_blocks(c, "balm_debug_tc_trace"));
  if (!c || !out || !c->tc_trace || max_entries < 0) {
    balm_set_error("balm_debug_tc_trace: no trace (BALM_TC_TRACE=1 at the creation of a tensor-precision context)");
    return BALM_ERR_INVALID;
  }
  CUDA_TRY(cudaSetDevice(c->device));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  const size_t total = std::min<size_t>((size_t)max_entries, (size_t)c->sm_count * TR_WORDS);
  CUDA_TRY(cudaMemcpy(out, c->tc_trace, sizeof(unsigned long long) * total, cudaMemcpyDeviceToHost));
  return BALM_OK;
}

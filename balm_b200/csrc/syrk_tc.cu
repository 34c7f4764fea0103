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
// The observation sweep writes the digit planes MN-major (pose index contiguous, Gq[S][rows][ldg], coalesced), while
// s8 wgmma reads shared-memory operands K-major only. The SYRK kernel therefore transposes the planes itself, into
// GqT[S][rows / 64][ldg][64]: per 64-row band, every column's 64 contraction rows as one 64-byte row, in the order wgmma
// reads them from shared memory (64-byte swizzle, see sw64_desc). A 128- or 64-column block of one band is then one
// contiguous 8 or 4 KB run that a single bulk copy lands ready for the MMAs. The copy is HBM traffic and the SYRK is
// MMA-bound, so the copy runs in the same launch, a few bands ahead of the MMAs that need it.
//
// Kernel anatomy (syrk_tc_kernel; one CTA per SM, persistent over its items, 384 threads, a cooperative launch). An item
// is a whole 128 x 128 output tile (S <= 3 on problems with at least one (tile, k-split) pair per SM, see launch_syrk_tc)
// or one 128 x 64 column half of a tile, times one k-split:
//   warps 9-11: copiers -- copy units (64-row band b, 128-column block cb), all S planes, from Gq into GqT, band-major
//               in ascending band order, dealt round robin over the copier warps of all CTAs; each unit then stamps its
//               readiness flag with the launch's epoch (see copier_loop). A copier waits on nothing but its own loads.
//   warp 8    : producer -- acquires the flags of the A and the B blocks of 16 stages at a time, then per stage
//               cp.async.bulk of the S K-major planes of the A block (128 columns bi) and of the B block (128 columns
//               bj, or the 64 of the half), KS = 64 contraction rows per stage, into one ring of stage slots (see Ring:
//               up to 192 KB of shared memory, mbarrier full/empty per slot)
//   warps 0-7 : consumers, two warpgroups of 64 output rows each -- wgmma m64n128k32 (whole tiles) or m64n64k32 (halves)
//               s8 x s8 -> s32 with B from the landed stage and A from it too (whole tiles) or from registers
//               (ldmatrix, halves), S(S+1)/2 digit-pair
//               products per k32 step into S register accumulators; then the epilogue: fp64 Horner combine, column
//               scales, fp64 partial tile to global (same partial layout as the fp64 path -> same assemble kernel)
// The register accumulators (S * 64 x N int32 per warpgroup = S * N / 2 registers per consumer thread) are what bounds
// the output tile: 192 at S = 3 and N = 128, so S = 4 (which would need 256) keeps 128 x 64 halves.
#include <vector>
#include <algorithm>
#include "internal.cuh"

namespace {

constexpr int TILE = BALM_SYRK_TILE;  // 128
constexpr int HALF = TILE / 2;        // output columns of a half-tile item
constexpr int SMAX = 4;               // digit planes
constexpr int KS = 64;                // contraction rows per pipeline stage (= the 64-byte swizzle span of a K-major row)
constexpr int A_PLANE_BYTES = KS * TILE;  // 8192: one K-major plane of a 128-column block, one stage (64-byte rows)
constexpr int MAX_SLOTS = 8;             // barriers of the ring
constexpr int BAR_BYTES = 2 * MAX_SLOTS * 8;
constexpr int COPIER_WARPS = 3;
constexpr int STAGING_BYTES = COPIER_WARPS * KS * TILE;  // one MN-major 64 x 128 plane tile per copier warp
// the block's whole shared memory but alignment slack, the copiers' staging and the barriers
constexpr int RING_BYTES = 227 * 1024 - 1024 - STAGING_BYTES - BAR_BYTES;
// One ring of stage slots: a slot holds the S planes of the A block, then the S planes of the B block (128 or 64
// columns), all landed by bulk copies on the slot's one full barrier and freed together once the consumers' MMAs on it retired.
// As many slots as fit, at most MAX_SLOTS:
//   whole tiles: S = 2: 6 x 32 KB, S = 3: 4 x 48 KB;  halves: S = 2: 8 x 24 KB, S = 3: 5 x 36 KB, S = 4: 4 x 48 KB
template <int S, bool FULL>
struct Ring {
  static constexpr int N = FULL ? TILE : HALF;  // output columns of an item
  static constexpr int B_PLANE = KS * N;
  static constexpr int B_OFF = S * A_PLANE_BYTES, SLOT = B_OFF + S * B_PLANE;
  static constexpr int D = RING_BYTES / SLOT < MAX_SLOTS ? RING_BYTES / SLOT : MAX_SLOTS;
  static_assert(D >= 2 && SLOT % 1024 == 0, "ring layout (the 64-byte swizzle repeats every 512 bytes)");
};
constexpr int CONSUMER_WARPS = 8;
constexpr int TC_THREADS = 32 * (CONSUMER_WARPS + 4);   // two consumer warpgroups + the producer / copier warpgroup
// register split (setmaxnreg): the producer / copier warpgroup gives nearly all its registers up so the consumers
// can hold their accumulators (S * N / 2, 192 at S = 3 on whole tiles) and two k32 steps of A fragments (2 * S * 4).
// The pool is what the launch allocated, 384 threads x 168 registers, and setmaxnreg.inc waits until the registers are
// free: 2 * 128 * 232 + 128 * 40 = 384 * 168. The copiers' transposes need more than 24 registers without spilling.
constexpr int CONSUMER_REGS = 232, PRODUCER_REGS = 40;
constexpr int TC_SMEM = RING_BYTES + STAGING_BYTES + 1024 + BAR_BYTES;  // ring + staging + alignment slack + barriers
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
// BALM_TC_TRACE (balm_debug_tc_trace): per-CTA word offsets of the stage count (in 128 x 64 half-tile units: a stage of
// a whole tile counts 2), the consumer warp 0 globaltimer pair, the clock64 sums of the consumer warps 0 and 4 (5 each),
// three words that stay zero (they held a B transposer's clocks) and the producer's (2: waiting on a free slot, waiting
// on readiness flags). The copiers' words (balm_debug_tc_copy_trace) follow all CTAs' words: per CTA the clocks its
// copier warps spent on units, of those the clocks waiting on their loads, and the plane tiles copied.
constexpr int TR_STAGES = 0, TR_NS = 1, TR_CONS = 3, TR_PROD = 16, TR_WORDS = BALM_TC_TRACE_WORDS;
constexpr int TR_COPY_WORDS = BALM_TC_COPY_TRACE_WORDS;
static_assert(TR_PROD + 2 == TR_WORDS && TR_COPY_WORDS == 3, "trace layout");
// clock64 in the traced instantiation; the untraced one reads no clock
template <bool TRACE>
__device__ __forceinline__ long long tclock() {
  if constexpr (TRACE) return clock64();
  else return 0;
}

// one contiguous run of global memory into shared memory, completing on the mbarrier's transaction count
__device__ __forceinline__ void bulk_load(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// 16 bytes of global memory into shared memory, bypassing L1; cp_async_wait_all waits for all of this thread's
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];\n" : "=r"(v) : "r"(addr) : "memory");
  return v;
}

// Readiness flags of the copy units (release by the copier warp that wrote the unit, acquire by the producers that read
// it; see copier_loop and producer_loop for the ordering)
__device__ __forceinline__ void flag_release(unsigned *f, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;\n" ::"l"(f), "r"(v) : "memory");
}
// Bounded spin, as mbar_wait: true once *f == epoch; false when the error flag is set or the bound is exceeded
__device__ __forceinline__ bool flag_wait(const unsigned *f, unsigned epoch, int *err) {
  for (long long it = 0; it < (1ll << 22); it++) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(f) : "memory");
    if (v == epoch) return true;
    if ((it & 1023) == 1023 && *((volatile int *)err) != 0) return false;
  }
  atomicExch(err, 2);
  return false;
}

// Four 8 x 8 matrices of 16-bit pairs: lane 8q + i gives the address of row i of matrix q; thread (g = lane/4,
// t = lane%4) receives in r[q] the pair t of row g, i.e. bytes 4t..4t+3 of that 16-byte row.
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t *r) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}

// A K-major plane of a stage as it lands (the layout of GqT): column n of the block is the 64-byte row n (contraction rows 0..63 of the
// stage), its 16-byte chunk q at (q ^ ((n >> 1) & 3)) under the 64-byte swizzle. wgmma reads it through a descriptor of
// that swizzle mode (layout type 2): 8-row core-matrix groups SW_SBO = 512 bytes apart, the k32 step c at + 32 c bytes
// (the swizzle is a function of the address, and every plane starts on a 512-byte boundary).
constexpr int SW_SBO = 8 * KS;
__device__ __forceinline__ uint64_t sw64_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(SW_SBO >> 4) << 32) | ((uint64_t)2 << 62);
}
// Byte offset, in a K-major block of GqT, of contraction rows 4 kq .. 4 kq + 3 of column n (n counted from a multiple of
// 8, which starts the same swizzle row)
__device__ __forceinline__ int kmajor_offset(int n, int kq) {
  return n * KS + ((((kq >> 2) ^ (n >> 1)) & 3) << 4) + 4 * (kq & 3);
}
// 4 x 4 byte transpose: w[i] holds bytes (row i, columns 0..3); out[j] receives bytes (rows 0..3, column j)
__device__ __forceinline__ void transpose4x4(const uint32_t (&w)[4], uint32_t (&out)[4]) {
  const uint32_t lo01 = __byte_perm(w[0], w[1], 0x5140), hi01 = __byte_perm(w[0], w[1], 0x7362);
  const uint32_t lo23 = __byte_perm(w[2], w[3], 0x5140), hi23 = __byte_perm(w[2], w[3], 0x7362);
  out[0] = __byte_perm(lo01, lo23, 0x5410);
  out[1] = __byte_perm(lo01, lo23, 0x7632);
  out[2] = __byte_perm(hi01, hi23, 0x5410);
  out[3] = __byte_perm(hi01, hi23, 0x7632);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_acc(int32_t (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; i++) asm volatile("" : "+r"(d[i])::"memory");
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
// D (64 x 128 s32, accumulated) += A (64 x 32 s8, K-major shared memory) * B (32 x 128 s8, K-major shared memory)
__device__ __forceinline__ void wgmma_s8_ss(int32_t (&d)[64], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
      "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, 1;\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
        "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
        "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
        "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
        "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
        "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
        "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
        "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
      : "l"(desc_a), "l"(desc_b)
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
  const int8_t *planes;    // Gq [SMAX][rows][ldq], the MN-major digit planes the observation sweep wrote
  int8_t *planes_t;        // GqT [SMAX][rows / KS][ldq][KS], their K-major copy, written by the copiers
  int64_t plane;      // bytes per plane of planes and planes_t
  int ldq;
  int64_t rows;       // contraction rows of this batch (3 per voxel), padded to a multiple of KS
  unsigned *flags;    // [rows / KS][nb]: copy unit (band, 128-column block) is in planes_t once it holds epoch
  unsigned epoch;     // this launch's stamp, never 0 (flags are allocated zeroed)
  int nb, tiles, splits;
  int full;           // whole 128 x 128 tiles when S <= 3 (launch_syrk_tc decides)
  const int *S_dev;   // digit-plane count chosen by tc_scale_kernel
  const double *isc;  // [ldq]  256^(S-1) / sc_j
  double *part;       // [splits][tiles][128*128]
  int accumulate;
  int *err;
  unsigned long long *trace;       // [gridDim.x][TR_WORDS], written by the traced instantiation only
  unsigned long long *copy_trace;  // [gridDim.x][TR_COPY_WORDS], likewise
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
template <bool FULL>
__device__ __forceinline__ int n_items(const TcArgs &a) { return a.tiles * (FULL ? 1 : 2) * a.splits; }
// contraction rows of a k-split item: ceil(rows / splits) rounded up to KS
__device__ __forceinline__ int64_t rows_per_item(const TcArgs &a) {
  return ((a.rows + a.splits - 1) / a.splits + KS - 1) / KS * KS;
}

// whole tiles: work = sp * tiles + t; halves: work = (sp * tiles + t) * 2 + h, the two column halves of a tile run on
// neighbouring CTAs and share the A block in L2
template <bool FULL>
__device__ __forceinline__ ItemInfo decode_item(const TcArgs &a, int work, int64_t per) {
  ItemInfo it;
  it.h = FULL ? 0 : (work & 1);
  const int w = FULL ? work : (work >> 1);
  it.t = w % a.tiles;
  it.sp = w / a.tiles;
  tile_coords_tc(it.t, a.nb, it.bi, it.bj);
  it.k_begin = (int64_t)it.sp * per;
  int64_t k_end = it.k_begin + per;
  if (k_end > a.rows) k_end = a.rows;
  it.nsteps = k_end > it.k_begin ? (int)((k_end - it.k_begin + KS - 1) / KS) : 0;
  return it;
}

// One consumer warpgroup (wg = 0, 1): output rows 64 wg .. 64 wg + 63 of the item, all items of this CTA. Warp w (0..7)
// holds output rows 16 w .. 16 w + 15: fragment row g is output row 16 w + g, fragment row g + 8 is 16 w + g + 8;
// fragment column n is column n of the item. A stage's slot sits at slot k % D, phase (k / D) & 1, for the k-th stage
// this CTA consumes.
template <int S, bool FULL, bool TRACE>
__device__ __forceinline__ void consumer_loop(const TcArgs &a, uint32_t ring, uint64_t *full, uint64_t *empty) {
  using R = Ring<S, FULL>;
  constexpr int NACC = R::N / 2;  // accumulator registers per digit-pair sum
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3, i = lane & 7, wg = warp >> 2;
  // ldmatrix row of this lane: matrix q = lane / 8 is output rows 16 warp + 8 (q & 1) + 0..7 at 16-byte chunk 2 c + q / 2
  // of the k32 step c; under the swizzle that chunk sits at ((q / 2) ^ ((i >> 1) & 3)) ^ 2 c. The 8 rows of a matrix
  // fill the 8 distinct 16-byte positions of two 128-byte lines, free of bank conflicts.
  const int row = 16 * warp + 8 * ((lane >> 3) & 1) + i;
  const uint32_t lda = ring + row * KS + ((((lane >> 4) & 1) ^ ((i >> 1) & 3)) << 4);
  const double inv256 = 1.0 / 256.0;
  long long tr[4] = {0, 0, 0, 0};  // trace: wait stage full, warpgroup vote, wgmma.wait_group, epilogue
  // the start clock's low word (a launch spans far fewer than 2^32 clocks) and the start time written at once: at 232
  // registers, the traced whole tiles would spill more across the items
  const uint32_t t_start = (uint32_t)tclock<TRACE>();
  if (TRACE && warp == 0 && lane == 0) a.trace[(size_t)blockIdx.x * TR_WORDS + TR_NS] = globaltimer_ns();
  int k = 0;  // stages consumed so far
  const int64_t per = rows_per_item(a);
  for (int item = blockIdx.x; item < n_items<FULL>(a); item += gridDim.x) {
    const ItemInfo info = decode_item<FULL>(a, item, per);
    int32_t acc[S][NACC];
#pragma unroll
    for (int d = 0; d < S; d++)
#pragma unroll
      for (int q = 0; q < NACC; q++) acc[d][q] = 0;
    // halves: A fragments of every plane, one set per k32 step of a stage (the other may be in flight); whole tiles read
    // A from shared memory, as the 192 accumulators leave no room for them
    uint32_t af[2][FULL ? 1 : S][4];
    bool alive = true;
    for (int ks = 0; ks < info.nsteps; ks++, k++) {
      const int sl = k % R::D;
      const long long t0 = tclock<TRACE>();
      const bool ok_s = mbar_wait(&full[sl], (k / R::D) & 1, a.err);
      const long long t1 = tclock<TRACE>();
      const bool ok = warpgroup_all(ok_s, 1 + wg);
      if constexpr (TRACE) { tr[0] += t1 - t0; tr[1] += clock64() - t1; }
      if (!ok) { alive = false; break; }  // the warpgroup leaves together (wgmma is .aligned)
      const uint32_t sa = lda + sl * R::SLOT;
      const uint64_t adesc = sw64_desc(ring + sl * R::SLOT + wg * 64 * KS);  // this warpgroup's 64 rows of the A block
      const uint64_t sdesc = sw64_desc(ring + sl * R::SLOT + R::B_OFF);
#pragma unroll
      for (int c = 0; c < KS / 32; c++) {
        if constexpr (!FULL) {
#pragma unroll
          for (int s = 0; s < S; s++) ldsm_x4((sa + s * A_PLANE_BYTES) ^ (c << 5), af[c][s]);
        }
        wgmma_fence();
#pragma unroll
        for (int s = 0; s < S; s++)
#pragma unroll
          for (int tt = 0; tt + s < S; tt++) {
            const uint64_t db = sdesc + ((tt * R::B_PLANE + c * 32) >> 4);
            if constexpr (FULL) wgmma_s8_ss(acc[s + tt], adesc + ((s * A_PLANE_BYTES + c * 32) >> 4), db);
            else wgmma_s8(acc[s + tt], af[c][s], db);
          }
        wgmma_commit();
        // every group but this one has retired: after the first k32 step that frees the previous stage, after the
        // second the A fragments of the first
        const long long t2 = tclock<TRACE>();
        wgmma_wait<1>();
        if constexpr (TRACE) tr[2] += clock64() - t2;
        if (c == 0 && ks > 0) {  // the previous stage's MMAs have retired: free its slot
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[(k - 1) % R::D]);
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
      if (lane == 0) mbar_arrive(&empty[(k - 1) % R::D]);
    }
    // ---- epilogue: Horner over the digit-pair order d = S-1 .. 0, column scales, fp64 partial tile ----
    double *tile_out = a.part + ((size_t)info.sp * a.tiles + info.t) * (TILE * TILE);
#pragma unroll
    for (int up = 0; up < 2; up++) {
      const int orow = 16 * warp + g + 8 * up;
      const double isc_row = __ldg(a.isc + info.bi * TILE + orow);
      double *out = tile_out + (size_t)orow * TILE + info.h * HALF;
#pragma unroll
      for (int j = 0; j < R::N / 8; j++) {
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
      const long long total = (uint32_t)((uint32_t)clock64() - t_start);
#pragma unroll
      for (int w = 0; w < 4; w++) o[TR_CONS + 5 * wg + w] = tr[w];
      o[TR_CONS + 5 * wg + 4] = total;
      if (wg == 0) {
        o[TR_STAGES] = (FULL ? 2 : 1) * k;
        o[TR_NS + 1] = globaltimer_ns();
      }
    }
  }
}

// The producer (warp 8): per stage, lane 0 loads the S planes of the A block and the S planes of the B block (or of its
// column half) into one slot, each one contiguous run of GqT. Before stages ks .. ks + 15 of an item, the warp acquires
// their copy units' readiness flags in one round trip: lane l < 16 that of the A block of stage ks + l, lane 16 + l
// that of its B block (a B flag covers a column half too). An acquire and a proxy fence per stage would cost the
// single issuing thread about as much as the consumers spend on a stage.
constexpr int FLAG_BATCH = 16;
template <int S, bool FULL, bool TRACE>
__device__ __forceinline__ void producer_loop(const TcArgs &a, uint8_t *ring, uint64_t *full, uint64_t *empty) {
  using R = Ring<S, FULL>;
  const int lane = threadIdx.x & 31;
  long long tr = 0, trf = 0;  // trace: wait slot empty, wait readiness flags
  int sl = 0;
  uint32_t ph = 0;
  const int64_t per = rows_per_item(a);
  for (int item = blockIdx.x; item < n_items<FULL>(a); item += gridDim.x) {
    const ItemInfo info = decode_item<FULL>(a, item, per);
    for (int ks = 0; ks < info.nsteps; ks++) {
      // band (k_begin / KS + ks) of the planes, then column bi * 128 (A) or bj * 128 + h * 64 (B) within it
      const int64_t band = info.k_begin / KS + ks;
      if (ks % FLAG_BATCH == 0) {
        // Ordering of the copiers' generic-proxy stores before the bulk copies (async proxy) that read them, PTX ISA,
        // memory consistency model: a copier's st.release and this ld.acquire (flag_wait) form a release / acquire
        // pattern, so its stores happen before everything after the acquire in causality order; bar.warp.sync
        // (__syncwarp) orders every lane's acquire before lane 0's later operations; and as the bulk copies read through
        // the async proxy, "fence.proxy.async" is required between those generic-proxy writes and async-proxy reads of
        // the same memory: lane 0 issues fence.proxy.async.global after the acquires and before its cp.async.bulk.
        const long long t0 = tclock<TRACE>();
        const int st = ks + (lane & (FLAG_BATCH - 1));
        const bool ok = st >= info.nsteps ||
                        flag_wait(a.flags + (band + (lane & (FLAG_BATCH - 1))) * a.nb + (lane < FLAG_BATCH ? info.bi : info.bj),
                                  a.epoch, a.err);
        __syncwarp();
        if (!__all_sync(0xffffffffu, ok)) return;
        if (lane == 0) asm volatile("fence.proxy.async.global;\n" ::: "memory");
        if constexpr (TRACE) trf += clock64() - t0;
      }
      const long long t1 = tclock<TRACE>();
      if (!__all_sync(0xffffffffu, mbar_wait(&empty[sl], ph ^ 1, a.err))) return;
      if constexpr (TRACE) tr += clock64() - t1;
      if (lane == 0) {
        const int8_t *src = a.planes_t + band * KS * a.ldq;
        const int8_t *src_a = src + (int64_t)info.bi * TILE * KS, *src_b = src + (int64_t)(info.bj * TILE + info.h * HALF) * KS;
        uint8_t *slot = ring + sl * R::SLOT;
        mbar_expect_tx(&full[sl], R::SLOT);
        for (int s = 0; s < S; s++) bulk_load(slot + s * A_PLANE_BYTES, src_a + s * a.plane, A_PLANE_BYTES, &full[sl]);
        for (int s = 0; s < S; s++) bulk_load(slot + R::B_OFF + s * R::B_PLANE, src_b + s * a.plane, R::B_PLANE, &full[sl]);
      }
      if (++sl == R::D) { sl = 0; ph ^= 1; }
    }
  }
  if constexpr (TRACE) {
    if (lane == 0) {
      a.trace[(size_t)blockIdx.x * TR_WORDS + TR_PROD] = tr;
      a.trace[(size_t)blockIdx.x * TR_WORDS + TR_PROD + 1] = trf;
    }
  }
}

// One copier warp (cw of ncw over all CTAs): units u = cw, cw + ncw, ... of the (rows / KS) x nb units (band-major, so
// in ascending band order as the consumers of every k-split need them). Per plane s < S of a unit: the MN-major 64 x 128
// tile of Gq into this warp's staging buffer (cp.async; the 16-byte chunk ch of row r at chunk ch ^ ((r >> 2) & 7), so
// that the loads below hit 16 banks, two lanes each), then 4 x 4 byte transposes into GqT: lane (kq = lane % 16,
// h = lane / 16) takes rows 4 kq .. 4 kq + 3 and in step it the 4 columns of word m = 2 it + h; the four 4-byte stores
// of a step land, with those of the other lanes of its half-warp, whole 64-byte K-major rows. Then the unit's flag.
template <int S, bool TRACE>
__device__ __forceinline__ void copier_loop(const TcArgs &a, uint8_t *staging, int cw, int ncw) {
  const int lane = threadIdx.x & 31, kq = lane & 15, h = lane >> 4;
  const uint32_t st = smem_u32(staging), rows = st + 4 * kq * TILE;  // rows 4 kq .. 4 kq + 3 of the staged tile
  const int units = (int)(a.rows / KS) * a.nb;  // < 2^31 (launch_syrk_tc)
  for (int u = cw; u < units; u += ncw) {
    const long long t0 = tclock<TRACE>();
    const int band = u / a.nb, cb = u - band * a.nb;
    const int8_t *src = a.planes + (int64_t)band * KS * a.ldq + cb * TILE;
    int8_t *dst = a.planes_t + (int64_t)band * KS * a.ldq + cb * TILE * KS;
    for (int s = 0; s < S; s++, src += a.plane, dst += a.plane) {
#pragma unroll 1
      for (int p = 0; p < KS * TILE / 16 / 32; p++) {
        const int idx = lane + 32 * p, r = idx >> 3, ch = idx & 7;
        cp_async16(st + r * TILE + ((ch ^ ((r >> 2) & 7)) << 4), src + (int64_t)r * a.ldq + 16 * ch);
      }
      const long long t1 = tclock<TRACE>();
      cp_async_wait_all();
      __syncwarp();
      if (TRACE && lane == 0) atomicAdd(a.copy_trace + blockIdx.x * TR_COPY_WORDS + 1, (unsigned long long)(clock64() - t1));
#pragma unroll 4
      for (int it = 0; it < TILE / 8; it++) {
        const int m = 2 * it + h;
        const uint32_t wa = rows + (((m >> 2) ^ (kq & 7)) << 4) + 4 * (m & 3);  // word m of row 4 kq
        const uint32_t w[4] = {lds32(wa), lds32(wa + TILE), lds32(wa + 2 * TILE), lds32(wa + 3 * TILE)};
        uint32_t out[4];
        transpose4x4(w, out);
#pragma unroll
        for (int j = 0; j < 4; j++) *reinterpret_cast<uint32_t *>(dst + kmajor_offset(4 * m + j, kq)) = out[j];
      }
      __syncwarp();  // every lane has read the staging buffer before the next plane lands in it
    }
    // Release pattern (PTX ISA, memory consistency model): the bar.warp.sync (__syncwarp) that ends the last plane orders
    // every lane's stores before lane 0's st.release, which makes them visible to whoever acquires the flag
    // (producer_loop). No proxy fence here: these stores are generic-proxy writes, the reader fences its async proxy.
    if (lane == 0) flag_release(a.flags + u, a.epoch);
    if (TRACE && lane == 0) {  // the trace's words, added per unit: nothing stays live across units
      atomicAdd(a.copy_trace + blockIdx.x * TR_COPY_WORDS, (unsigned long long)(clock64() - t0));
      atomicAdd(a.copy_trace + blockIdx.x * TR_COPY_WORDS + 2, (unsigned long long)S);
    }
  }
}

template <int S, bool FULL, bool TRACE>
__device__ __forceinline__ void syrk_tc_cta(const TcArgs &a, uint8_t *ring, uint8_t *staging, uint64_t *full,
                                            uint64_t *empty) {
  if (threadIdx.x >= 32 * CONSUMER_WARPS) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(PRODUCER_REGS));
    const int w = (threadIdx.x >> 5) - CONSUMER_WARPS - 1;  // copier warp 0..2, or -1 for the producer's warp
    if (w < 0) {
      // ===================== producer (warp 8) =====================
      producer_loop<S, FULL, TRACE>(a, ring, full, empty);
    } else {
      // ===================== copiers (warps 9-11) =====================
      copier_loop<S, TRACE>(a, staging + w * KS * TILE, COPIER_WARPS * blockIdx.x + w, COPIER_WARPS * gridDim.x);
    }
  } else {
    // ===================== wgmma + epilogue =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(CONSUMER_REGS));
    consumer_loop<S, FULL, TRACE>(a, smem_u32(ring), full, empty);
  }
}

template <bool TRACE>
__global__ void __launch_bounds__(TC_THREADS, 1) syrk_tc_kernel(TcArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte aligned ring (the swizzle patterns are functions of the shared-memory address), then barriers
  uint8_t *ring = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t *staging = ring + RING_BYTES;  // 16-byte aligned (cp.async)
  uint64_t *full = reinterpret_cast<uint64_t *>(staging + STAGING_BYTES), *empty = full + MAX_SLOTS;
  if (threadIdx.x == 0) {
    for (int i = 0; i < MAX_SLOTS; i++) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], CONSUMER_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();
  const int S = *a.S_dev;
  if (S == 4) syrk_tc_cta<4, false, TRACE>(a, ring, staging, full, empty);
  else if (S == 3 && a.full) syrk_tc_cta<3, true, TRACE>(a, ring, staging, full, empty);
  else if (S == 3) syrk_tc_cta<3, false, TRACE>(a, ring, staging, full, empty);
  else if (a.full) syrk_tc_cta<2, true, TRACE>(a, ring, staging, full, empty);
  else syrk_tc_cta<2, false, TRACE>(a, ring, staging, full, empty);
}
static_assert(RING_BYTES % 16 == 0 && STAGING_BYTES % 16 == 0, "staging and barrier alignment");

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

// start of a speculative evaluation (one block): the scales found by the previous one become the ones in use
// (skew: test hook BALM_TC_SPEC_SKEW -- the adopted scales are multiplied by 2^skew so that the device-side check
//  has something to reject; 0 in production), and the column maxima are cleared for the fused sweep.
// same_poses: the previous evaluation was at these poses (a rejected LM step). If its planes were written by the
// fused sweep and kept (*spec_ok, still its verdict) and the adopted scales and plane count equal the ones they were
// written with, a fused sweep now would write the same planes, column maxima and accumulator partials bit for bit
// (and the check would keep them again): *reuse = 1 and the sweep, its reduction and the clearing are skipped.
__global__ void __launch_bounds__(1024) tc_adopt_kernel(double *sc, double *isc, int *S_dev, const double *sc_next,
                                                        const double *isc_next, const int *S_next, int ldq, int skew,
                                                        int same_poses, const int *spec_ok, int *reuse,
                                                        unsigned long long *colmax) {
  int differ = !same_poses || *spec_ok == 0 || *S_next != *S_dev;
  if (!differ)
    for (int j = threadIdx.x; j < ldq; j += blockDim.x)
      if (ldexp(sc_next[j], skew) != sc[j]) differ = 1;
  const bool keep = __syncthreads_or(differ) == 0;  // every read of sc / S_dev above precedes the writes below
  for (int j = threadIdx.x; j < ldq; j += blockDim.x) {
    sc[j] = ldexp(sc_next[j], skew);
    isc[j] = ldexp(isc_next[j], -skew);
    if (!keep) colmax[j] = 0ull;
  }
  if (threadIdx.x == 0) {
    *S_dev = *S_next;
    *reuse = keep ? 1 : 0;
  }
}


struct TcState {
  int8_t *GqT = nullptr;    // [SMAX][rows_alloc / KS][ldg][KS] K-major copy of c->Gq (syrk_tc_kernel's copiers)
  unsigned *flags = nullptr;  // [rows_alloc / KS][ldg / 128] readiness of its copy units, stamped with epoch
  unsigned epoch = 0;         // of the last SYRK launch
  double *sc = nullptr, *isc = nullptr;
  double *sc_next = nullptr, *isc_next = nullptr;  // fresh scales of the last full-range evaluation (speculation)
  int *S_next = nullptr, *spec_ok = nullptr;
  bool spec_ready = false;                         // sc_next/S_next describe the currently registered voxels
  bool spec_enabled = true;                        // BALM_NO_SPEC=1 keeps the two-sweep path
  bool last_spec = false;                          // the batch in flight used the fused sweep
  int spec_skew = 0;                               // BALM_TC_SPEC_SKEW (tests)
  int *reuse = nullptr;                            // tc_adopt_kernel: the fused sweep of the batch in flight is skipped
  bool reuse_enabled = true;                       // BALM_NO_SWEEP_REUSE=1 sweeps again after every rejected step
  unsigned long long *colmax = nullptr;
  int *err = nullptr;
  int64_t rows_alloc = 0;
  int forced_S = 0;      // BALM_TC_SLICES override (0 = decided on the device per batch)
  int *S_dev = nullptr;  // [1]
  int last_S = 0;        // read back with the error flag (instrumentation)
  int64_t last_rows_padded = 0;  // contraction rows of the last batch's SYRK (0: none since the registration)
};

// One syrk_tc_kernel launch on c's stream: rows_padded (a multiple of KS) contraction rows of the MN-major planes
// `planes`, copied K-major into planes_t by the launch itself (both of plane stride `plane` bytes), nb x nb blocks of 128
// columns, `splits` k-splits; one CTA per item up to one per SM. Whole 128 x 128 tiles (at S <= 3) halve the L2 traffic
// per MAC but also the item count, so they are taken only when every SM still gets an item (tiles x splits >= SMs);
// BALM_TC_TILE=half|full (c->tc_tile) overrides the rule. flags: (rows_padded / KS) x nb words, none equal to epoch.
// A CTA waits on copy units of other CTAs, so the launch is cooperative: all CTAs are resident, or it fails.
// With c->tc_trace (BALM_TC_TRACE) the traced instantiation runs and records the launch.
int launch_syrk_tc(balm_ctx *c, const int8_t *planes, int8_t *planes_t, int64_t plane, int64_t rows_padded, int nb,
                   int tiles, int splits, const int *S_dev, const double *isc, double *part, bool accumulate, int *err,
                   unsigned *flags, unsigned epoch) {
  if (rows_padded / KS * nb > INT32_MAX) {  // the copiers count units in int
    balm_set_error("tensor SYRK: more than 2^31 copy units");
    return BALM_ERR_INVALID;
  }
  const bool full = c->tc_tile == 0 ? (int64_t)tiles * splits >= c->sm_count : c->tc_tile == 2;
  unsigned long long *copy_trace = c->tc_trace ? c->tc_trace + (size_t)c->sm_count * TR_WORDS : nullptr;
  TcArgs a{planes, planes_t, plane, c->ldg, rows_padded, flags, epoch, nb, tiles, splits, full ? 1 : 0,
           S_dev, isc, part, accumulate ? 1 : 0, err, c->tc_trace, copy_trace};
  const int items = a.tiles * 2 * a.splits;  // half-tile items; the whole-tile count when S <= 3 is not known here
  const int grid = items < c->sm_count ? items : c->sm_count;
  void *params[] = {&a};
  if (c->tc_trace)
    CUDA_TRY(cudaMemsetAsync(c->tc_trace, 0, sizeof(unsigned long long) * c->sm_count * (TR_WORDS + TR_COPY_WORDS),
                             c->stream));
  const void *kernel = c->tc_trace ? (const void *)syrk_tc_kernel<true> : (const void *)syrk_tc_kernel<false>;
  CUDA_TRY(cudaLaunchCooperativeKernel(kernel, dim3(grid), dim3(TC_THREADS), params, TC_SMEM, c->stream));
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
  CUDA_TRY(cudaMalloc((void **)&st->GqT, (size_t)SMAX * st->rows_alloc * ldq));
  CUDA_TRY(cudaMemset(st->GqT, 0, (size_t)SMAX * st->rows_alloc * ldq));
  const size_t n_flags = (size_t)(st->rows_alloc / KS) * (ldq / TILE);
  CUDA_TRY(cudaMalloc((void **)&st->flags, sizeof(unsigned) * n_flags));
  CUDA_TRY(cudaMemset(st->flags, 0, sizeof(unsigned) * n_flags));
  CUDA_TRY(cudaMalloc((void **)&st->S_dev, sizeof(int)));
  CUDA_TRY(cudaMalloc((void **)&st->sc, sizeof(double) * ldq));
  CUDA_TRY(cudaMalloc((void **)&st->isc, sizeof(double) * ldq));
  CUDA_TRY(cudaMalloc((void **)&st->sc_next, sizeof(double) * ldq));
  CUDA_TRY(cudaMalloc((void **)&st->isc_next, sizeof(double) * ldq));
  CUDA_TRY(cudaMalloc((void **)&st->S_next, sizeof(int)));
  CUDA_TRY(cudaMalloc((void **)&st->spec_ok, sizeof(int)));
  CUDA_TRY(cudaMemset(st->spec_ok, 0, sizeof(int)));
  CUDA_TRY(cudaMalloc((void **)&st->reuse, sizeof(int)));
  CUDA_TRY(cudaMemset(st->reuse, 0, sizeof(int)));
  st->spec_enabled = getenv("BALM_NO_SPEC") == nullptr;
  st->reuse_enabled = getenv("BALM_NO_SWEEP_REUSE") == nullptr;
  if (const char *e = getenv("BALM_TC_SPEC_SKEW")) st->spec_skew = atoi(e);
  CUDA_TRY(cudaMalloc((void **)&st->colmax, sizeof(unsigned long long) * ldq));
  CUDA_TRY(cudaMalloc((void **)&st->err, sizeof(int)));
  CUDA_TRY(cudaMemset(st->err, 0, sizeof(int)));
  c->colmax = st->colmax;  // the observation pass writes the column maxima here

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
    cudaFree(st->sc_next); cudaFree(st->isc_next); cudaFree(st->S_next); cudaFree(st->spec_ok); cudaFree(st->reuse);
    cudaFree(st->sc); cudaFree(st->isc); cudaFree(st->colmax); cudaFree(st->err); cudaFree(st->S_dev);
    cudaFree(st->GqT); cudaFree(st->flags);
    delete st;
    c->tmap = nullptr;
  }
  cudaFree(c->Gq);
  c->Gq = nullptr;
  c->colmax = nullptr;
}

// One batch of the tensor path: (1) column maxima of G' -> power-of-two scales, (2) observation sweep writing the
// int8 digit planes directly, (3) the tensor-core SYRK, which makes their K-major copy as it goes. ev[2] is recorded
// between the observation sweeps and the SYRK.
int tensor_obs_and_syrk(balm_ctx *c, const double *poses, int64_t v0, int64_t v1, bool first_batch) {
  TcState *st = static_cast<TcState *>(c->tmap);
  if (!st) { balm_set_error("tensor path not initialised"); return BALM_ERR_INVALID; }
  const int ldq = c->ldg;
  const int64_t rows = 3 * (v1 - v0);
  const int64_t rows_padded = (rows + KS - 1) / KS * KS;
  // Speculation lives inside one balm_damping_iter call only: its first evaluation sweeps twice, and the public
  // balm_evaluate always does -- so every entry point stays a pure function of its arguments (same inputs, same bits,
  // whatever was evaluated before).
  const bool full = c->lm_active && v0 == 0 && v1 == c->M;
  const bool spec = full && st->spec_ready && st->spec_enabled;
  const int64_t plane_stride = (int64_t)st->rows_alloc * ldq;
  int rc;
  if (spec) {  // one sweep with the previous evaluation's scales; sweep 2 below only runs if tc_scale_kernel re-arms it
    // (and none at all when a rejected step left the planes of these poses and scales in place: tc_adopt_kernel).
    // Dense scenes only: a sparse batch's planes are cleared before its sweep.
    const bool may_reuse = c->eval_same_poses && st->reuse_enabled && c->dense;
    tc_adopt_kernel<<<1, 1024, 0, c->stream>>>(st->sc, st->isc, st->S_dev, st->sc_next, st->isc_next, st->S_next, ldq,
                                               st->spec_skew, may_reuse ? 1 : 0, st->spec_ok, st->reuse, st->colmax);
    c->launches += 1;
    rc = launch_obs_int8(c, poses, v0, v1, first_batch, st->sc, c->Gq, plane_stride, st->S_dev, SMAX, rows_padded, true,
                         may_reuse ? st->reuse : nullptr);
  } else {
    CUDA_TRY(cudaMemsetAsync(st->colmax, 0, sizeof(unsigned long long) * ldq, c->stream));
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
  if (++st->epoch == 0) {  // after 2^32 launches: flags of old launches could hold any stamp
    CUDA_TRY(cudaMemsetAsync(st->flags, 0, sizeof(unsigned) * (size_t)(st->rows_alloc / KS) * c->syrk_nb, c->stream));
    st->epoch = 1;
  }
  return launch_syrk_tc(c, c->Gq, st->GqT, plane_stride, rows_padded, c->syrk_nb, c->syrk_tiles, c->syrk_splits,
                        st->S_dev, st->isc, c->syrk_part, !first_batch, st->err, st->flags, st->epoch);
}

// The SYRK's error flag, the digit-plane count and the speculation verdict of the batch in flight: the copies are
// enqueued (pinned host words), the host reads them after its next synchronisation of the stream.
int tensor_syrk_check_enqueue(balm_ctx *c) {
  TcState *st = static_cast<TcState *>(c->tmap);
  if (!st) return BALM_OK;
  CUDA_TRY(cudaMemcpyAsync(c->h_flags + 1, st->err, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->h_flags + 2, st->S_dev, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->h_flags + 3, st->spec_ok, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaMemcpyAsync(c->h_flags + 5, st->reuse, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  return BALM_OK;
}

int tensor_syrk_check_finish(balm_ctx *c) {  // after the stream has been synchronised
  TcState *st = static_cast<TcState *>(c->tmap);
  if (!st) return BALM_OK;
  st->last_S = c->h_flags[2];
  c->tm.digit_planes = st->last_S;
  if (st->last_spec) {
    (c->h_flags[3] ? c->tm.single_sweeps : c->tm.redone_sweeps) += 1;
    if (c->h_flags[5]) c->reused_sweeps += 1;
  }
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
  int8_t *d_planes, *d_planes_t;
  double *d_isc, *d_part;
  int *d_S, *d_err;
  unsigned *d_flags;
  const size_t n_flags = (size_t)(rows_padded / KS) * nb;
  TRY(pool.get(&d_planes, SMAX * plane));
  TRY(pool.get(&d_planes_t, SMAX * plane));
  TRY(pool.get(&d_flags, n_flags));
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
  CUDA_TRY(cudaMemsetAsync(d_flags, 0, sizeof(unsigned) * n_flags, c->stream));
  TRY(syrk_tc_set_smem());
  TRY(launch_syrk_tc(c, d_planes, d_planes_t, (int64_t)plane, rows_padded, nb, tiles, splits, d_S, d_isc, d_part,
                     accumulate != 0, d_err, d_flags, 1));
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

extern "C" int balm_debug_tc_copy_trace(balm_ctx *c, unsigned long long *out, int max_entries) {
  if (c) TRY(refuse_blocks(c, "balm_debug_tc_copy_trace"));
  if (!c || !out || !c->tc_trace || max_entries < 0) {
    balm_set_error("balm_debug_tc_copy_trace: no trace (BALM_TC_TRACE=1 at the creation of a tensor-precision context)");
    return BALM_ERR_INVALID;
  }
  CUDA_TRY(cudaSetDevice(c->device));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  const size_t total = std::min<size_t>((size_t)max_entries, (size_t)c->sm_count * TR_COPY_WORDS);
  CUDA_TRY(cudaMemcpy(out, c->tc_trace + (size_t)c->sm_count * TR_WORDS, sizeof(unsigned long long) * total,
                      cudaMemcpyDeviceToHost));
  return BALM_OK;
}

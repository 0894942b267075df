// K1 — squared-L2 nearest-neighbour search as a wgmma distance GEMM with a fused row-wise top-2.
//
// Replaces, for one (I = database, J = query) image pair, the reference's
//   ArrayMatcher_bruteForce::SearchNeighbours  (matching/ArrayMatcher_bruteForce.hpp:98-142)
//   + feature::L2_Vectorized                   (feature/metric.hpp:48-139)
//   + partial_sort top-2                       (stl/indexedSort.hpp:40-55)
//   + the pre-filter half of NNdistanceRatio   (matching/filters.hpp:35-67)
// on integer-valued descriptors (|v| <= 1024, ||v||^2 < 2^22), where every product, partial sum and
// distance is an exact integer (or half-integer) below 2^24 in fp32.
//
//   ||a-b||^2 = ||a||^2 + 2*h,   h = ||b||^2/2 - a.b
//
// The accumulator holds -a.b (B negated by the instruction).  The database half-norm is either added in the epilogue
// (half-norm ring) or folded into the GEMM (AUG: a 9th K-step; each database row carries 16 extra fp16 columns
// [b0, l0, l1, 0...] with ||b||^2/2 = 0.5*b0 + l0 + 2048*l1, all exact in fp16, and every query row the constants
// [-0.5, -1, -2048, 0...], so the accumulator is h directly for 12.5 % more tensor work).  The epilogue reduces 16-column
// chunks to their minimum and keeps the two smallest CHUNK MINIMA plus the chunk id of the best per query row.  The
// second value is only an upper bound when best and second-best share a chunk; the exactness pass (verify.cuh) repairs
// that by re-scoring the 16 rows of the winning chunk for the few queries that pass the pre-test.
//
// CTA = 128 queries of a work item against the whole database image; a work item is 128 or 256 consecutive queries
// (`ctas_per_item` = 1 or 2 CTAs, independent of each other).  Persistent over work items, 1 CTA per SM:
//   warp 0       TMA producer: the Q tile (two 128 x 64 fp16 K-blocks, once per item), database tiles of 128 rows (two
//                K-blocks + the 128 rows' half-norms or augmentation columns) through an NS-slot ring
//   warps 2, 3   EXACTNESS PASS of the previous work item (`fused`): the epilogue queues its candidates in shared memory and
//                these warps re-score them (verify.cuh rescore_candidate) and append the final records while the next item
//                runs through the tensor cores, so the match list is complete when the kernel ends
//   warps 4-11   two consumer warpgroups of 64 query rows each: per tile 8 (AUG: 9) wgmma.m64n128k16 into 64 fp32 registers
//                per thread, then the chunk-minimum epilogue on those registers.  The two warpgroups run independently, so
//                one warpgroup's epilogue overlaps the other's MMAs.  The u8 kernel (4 wgmma.m64n128k32 per tile) pipelines each
//                warpgroup's tiles over two accumulators instead, so that its epilogue overlaps its own next MMAs.
//                The u8 norm-GEMM kernel (NG) adds a 5th K32 step that puts the database norm into the accumulator as well (below).
//   MODE_REAL adds six re-scoring warps (12-17).
//
// NG (u8 norm-GEMM kernel, template flag of the u8 body): for query views with every component <= 127, the query tile is doubled in
// shared memory (2a fits in u8) and a 5th K-step, m64n128k32 s8 x u8, multiplies constant weights [-1, -128 x 31] by the database row's 32
// norm limbs (common.cuh u8_limb), so the exact s32 accumulator is 2 a.b - ||b||^2 = -s: the epilogue is an integer max per chunk with no
// shared-memory reads and no per-element arithmetic.  Views with a component above 127 (as queries) or a norm above the limbs' capacity
// (as databases) stay on the u8 kernel (VF_U8_WIDE, VF_U8_NORMCAP).
//
// MODE (template): what the epilogue keeps per query row and what leaves the kernel
//   MODE_MATCH  integer-valued descriptors (exact accumulators): two smallest chunk minima + chunk of the best, ratio pre-test,
//               candidates re-scored exactly (in-kernel when `fused`) -> final match records.                       [the hot path]
//   MODE_KNN    the same data, ArrayMatcher surface: chunk of the second best is kept too and EVERY query leaves a candidate
//               (dense, slot = query row) for knn_finalize_kernel, which needs both neighbours' indices.
//   MODE_REAL   real-valued fp32 descriptors: the GEMM on the fp16-ROUNDED rows is only a FILTER.  The query's half-norm is folded in
//               as well (A tile of the 9th K-step = the query's own limbs, loaded per item), so the accumulator is ||a~ - b~||^2 / 2 >= 0
//               and the chunk id rides in the low mantissa bits of the chunk minimum: the FOUR smallest packed minima are kept.
//               |sqrt(d~) - sqrt(d)| <= ||a - a~|| + ||b - b~|| bounds what the rounding can do, so the rows outside the best chunks
//               are provably out of the top-2 whenever the next chunk minimum is far enough; the exact distances (the reference's
//               fp32 SSE order, from the original fp32 rows) come from re-scoring those chunks (verify.cuh rescore_real), and the
//               rare query the bound cannot decide goes to the exact_rows fallback.  Results are bit-identical to the reference
//               whatever the rounding did.
//
// Accumulator layout (ptx::wgmma_m64n128k16_f16_negb): a thread holds two query rows and, per row, 4 of the 16 columns of each
// chunk; the four threads of a quad (lanes 4k..4k+3) hold the same rows.  (The u8 kernel defines its chunks per thread instead and
// skips what follows: see its branch of the consumer loop.)  A chunk minimum is a min over the thread's 4 values
// and then over the quad: a two-step butterfly (xor 1, xor 2) that leaves each lane the full minima of chunks {q, q + 4}
// (q = lane % 4) of both rows - 12 shuffles per tile instead of 32 - and each lane keeps its own running state over its chunks.
// The four disjoint states are merged once per work item.
#pragma once
#include "common.cuh"
#include "ptx.cuh"
#include "verify.cuh"

namespace b200m {
namespace tc {

constexpr int BM = 128;                   // queries per CTA (two warpgroups x 64 rows)
constexpr int BN = 128;                   // database rows per tile (wgmma N)
constexpr int ROW_PAD = 256;              // views' fp16 / half-norm / augmentation buffers are padded to a multiple of this many rows
constexpr int CHUNK = 16;                 // columns per chunk minimum
constexpr int KB_BYTES = 128 * 64 * 2;    // 16 KB: one K-block (64 fp16) of 128 rows = one TMA box of tmap128
constexpr int Q_BYTES = 2 * KB_BYTES;     // 32 KB
constexpr int DB_BYTES = 2 * KB_BYTES;    // 32 KB
constexpr int AUG_BYTES = 128 * 16 * 2;   // 4 KB: 16 augmentation columns of 128 rows
constexpr int NB_BYTES = BN * 4;          // half-norms (u8: int32 norms) of one tile
constexpr int U8_BYTES = 128 * 128;       // 16 KB: 128 uchar rows of 128 B = one TMA box of tmap_u8 (the whole K of a u8 query or database tile)
constexpr int LIMB_BYTES = BN * 32;       // 4 KB: the 32 norm limbs of 128 database rows (NG), or the constant weight tile of 128 query rows
constexpr int EPI_WARPS = 8;
// u8 kernel: per-thread registers after set-up, warpgroup 0 (producer, exactness pass) and the two consumer warpgroups (two 64-register
// accumulators).  setmaxnreg moves them inside the launch allocation of 384 x 128: 128 * U8_REGS_WG0 + 256 * U8_REGS_CONSUMER <= 49152.
constexpr int U8_REGS_WG0 = 64;
constexpr int U8_REGS_CONSUMER = 160;
static_assert(128 * U8_REGS_WG0 + 256 * U8_REGS_CONSUMER <= 384 * 128, "the u8 kernel's register split exceeds its launch allocation");
enum : int { MODE_MATCH = 0, MODE_KNN = 1, MODE_REAL = 2 };

template <bool AUG, bool REAL = false, bool U8 = false, bool NG = false> struct Lay {
  // database ring slots (AUG: leaves shared memory to L1 for the re-scoring warps; U8: half-size stages, twice as many in about the same bytes)
  static constexpr int NS = U8 ? 8 : AUG ? 3 : 4;
  static constexpr int QT = U8 ? U8_BYTES : Q_BYTES;                 // one query tile buffer
  // + augmentation columns, the (half-)norms (padded: tiles stay 1024-B aligned) or (NG) the norm limbs
  static constexpr int STAGE = U8 ? U8_BYTES + (NG ? LIMB_BYTES : 1024) : DB_BYTES + (AUG ? AUG_BYTES : 1024);
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_DB = OFF_Q + 2 * QT;
  // AUG: the constant A tile of the 9th K-step; REAL: the query's own limb tile, 2 buffers; NG: the constant weight tile of the 5th K-step
  static constexpr int OFF_A = OFF_DB + NS * STAGE;
  static constexpr int OFF_MRG = OFF_A + (AUG ? (REAL ? 2 : 1) * AUG_BYTES : NG ? LIMB_BYTES : 0);   // per-row merged state, 2 buffers x 128 x 16 B
  static constexpr int OFF_VQ = OFF_MRG + 2 * BM * 16;               // candidate queue: 2 buffers x 128 Cand (32 slots per row quadrant)
  static constexpr int OFF_VQX = OFF_VQ + 2 * BM * 16;               // REAL: 5th word of the queued candidates (p4), 2 x 128 x 4 B
  static constexpr int OFF_VQN = OFF_VQX + (REAL ? 2 * BM * 4 : 0);  // 2 x (4 per-quadrant counts + pair index), 32 B each
  static constexpr int OFF_BAR = OFF_VQN + 2 * 32;
  static constexpr int NUM_BARS = 2 + 2 + NS + NS + 2 + 2;
  static constexpr int SMEM_BYTES = OFF_BAR + NUM_BARS * 8;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory of one CTA");
};

struct Top2 { float m1, m2; uint32_t g1; };
// MODE_KNN: the chunk of the second smallest minimum too
struct Top2g { float m1, m2; uint32_t g1, g2; };
// Packed four-smallest list of the real-valued filter (non-negative float bit patterns order like unsigned integers).
struct Top4 { uint32_t p1, p2, p3, p4; };

// Folds see the chunks of one lane in ascending chunk order; strict comparisons keep the lowest chunk id among equal minima.
__device__ __forceinline__ void fold_chunk(float cm, uint32_t gid, Top2& s) {
  s.m2 = fminf(s.m2, fmaxf(s.m1, cm));
  s.g1 = (cm < s.m1) ? gid : s.g1;
  s.m1 = fminf(s.m1, cm);
}
__device__ __forceinline__ void fold_chunk_knn(float cm, uint32_t gid, Top2g& s) {
  const bool lt1 = cm < s.m1, lt2 = cm < s.m2;
  s.g2 = lt1 ? s.g1 : (lt2 ? gid : s.g2);
  s.m2 = fminf(s.m2, fmaxf(s.m1, cm));
  s.g1 = lt1 ? gid : s.g1;
  s.m1 = fminf(s.m1, cm);
}
__device__ __forceinline__ void top4_insert(Top4& s, uint32_t pk) {
  s.p4 = min(s.p4, max(s.p3, pk));
  s.p3 = min(s.p3, max(s.p2, pk));
  s.p2 = min(s.p2, max(s.p1, pk));
  s.p1 = min(s.p1, pk);
}
__device__ __forceinline__ void fold_chunk_real(float cm, uint32_t gid, Top4& s) {
  top4_insert(s, (__float_as_uint(fmaxf(cm, 0.f)) & ~REAL_IDMASK) | gid);   // d~/2 >= 0 up to accumulation rounding
}

// Merges of two lanes' states over disjoint chunk sets: the result is what one sequential fold over all chunks would give
// (order (value, chunk id)).
__device__ __forceinline__ void merge_xor(Top2& s, int m) {
  const float om1 = __shfl_xor_sync(0xffffffffu, s.m1, m), om2 = __shfl_xor_sync(0xffffffffu, s.m2, m);
  const uint32_t og1 = __shfl_xor_sync(0xffffffffu, s.g1, m);
  s.m2 = fminf(fmaxf(s.m1, om1), fminf(s.m2, om2));
  s.g1 = (om1 < s.m1 || (om1 == s.m1 && og1 < s.g1)) ? og1 : s.g1;
  s.m1 = fminf(s.m1, om1);
}
__device__ __forceinline__ bool lex_less(float a, uint32_t ga, float b, uint32_t gb) { return a < b || (a == b && ga < gb); }
__device__ __forceinline__ void merge_xor(Top2g& s, int m) {
  const float om1 = __shfl_xor_sync(0xffffffffu, s.m1, m), om2 = __shfl_xor_sync(0xffffffffu, s.m2, m);
  const uint32_t og1 = __shfl_xor_sync(0xffffffffu, s.g1, m), og2 = __shfl_xor_sync(0xffffffffu, s.g2, m);
  if (lex_less(om1, og1, s.m1, s.g1)) {
    if (!lex_less(s.m1, s.g1, om2, og2)) { s.m2 = om2; s.g2 = og2; } else { s.m2 = s.m1; s.g2 = s.g1; }
    s.m1 = om1; s.g1 = og1;
  } else if (lex_less(om1, og1, s.m2, s.g2)) {
    s.m2 = om1; s.g2 = og1;
  }
}
__device__ __forceinline__ void merge_xor(Top4& s, int m) {
  const uint32_t o1 = __shfl_xor_sync(0xffffffffu, s.p1, m), o2 = __shfl_xor_sync(0xffffffffu, s.p2, m);
  const uint32_t o3 = __shfl_xor_sync(0xffffffffu, s.p3, m), o4 = __shfl_xor_sync(0xffffffffu, s.p4, m);
  top4_insert(s, o1); top4_insert(s, o2); top4_insert(s, o3); top4_insert(s, o4);
}

__device__ __forceinline__ float vmin(float a, float b) { return fminf(a, b); }
// Per row, the thread's minima of the 8 chunks (over its 4 columns of each) -> the full minima of chunks qlane and qlane + 4 (over the quad),
// v2[row][h] = chunk 4h + qlane: a two-step butterfly, 12 shuffles
template <typename T>
__device__ __forceinline__ void quad_chunk_minima(const T (&pm)[2][8], int qlane, T (&v2)[2][2]) {
  const bool b0 = qlane & 1, b1 = (qlane >> 1) & 1;
  T v1[2][4];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {        // keep chunks 2i + b0, hand the other to lane ^ 1
      const T keep = b0 ? pm[r][2 * i + 1] : pm[r][2 * i], send = b0 ? pm[r][2 * i] : pm[r][2 * i + 1];
      v1[r][i] = vmin(keep, __shfl_xor_sync(0xffffffffu, send, 1));
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {        // keep chunks 4h + 2 b1 + b0 = 4h + qlane
      const T keep = b1 ? v1[r][2 * h + 1] : v1[r][2 * h], send = b1 ? v1[r][2 * h] : v1[r][2 * h + 1];
      v2[r][h] = vmin(keep, __shfl_xor_sync(0xffffffffu, send, 2));
    }
  }
}

// u8 kernel, per element: s + U8_NORM_BIAS = (||b||^2 + U8_NORM_BIAS) - 2 a.b on the fp32 pipe.  Both operands are integers in [0, 2^24]; read as
// floats their bit patterns are the (sub)normal numbers x * 2^-149, the product and the sum are exact, and the result (positive: the bias
// exceeds ||a||^2) read back as an integer is the integer result: one full-rate FFMA where an IMAD issues at half rate.  This needs
// denormals kept: the library is built without -ftz / fast-math.  A pad row (a.b = 0) gives back its norm word unchanged.
__device__ __forceinline__ int32_t u8_elem(int32_t nb, int32_t ab) { return __float_as_int(fmaf(-2.f, __int_as_float(ab), __int_as_float(nb))); }
// ... and of a chunk minimum, h = s / 2: what the fp16 kernel's accumulator holds (exact, |s| <= 2^24)
__device__ __forceinline__ float u8_half_dist(int32_t biased) { return fmaf(0.5f, (float)biased, -0.5f * (float)U8_NORM_BIAS); }
__device__ __forceinline__ int32_t min16(const int32_t (&x)[16]) {
  const int32_t a = __vimin3_s32(x[0], x[1], x[2]), b = __vimin3_s32(x[3], x[4], x[5]), c = __vimin3_s32(x[6], x[7], x[8]);
  const int32_t d = __vimin3_s32(x[9], x[10], x[11]), e = __vimin3_s32(x[12], x[13], x[14]);
  return min(__vimin3_s32(a, b, c), __vimin3_s32(d, e, x[15]));
}
__device__ __forceinline__ int32_t max16(const int32_t (&x)[16]) {
  const int32_t a = __vimax3_s32(x[0], x[1], x[2]), b = __vimax3_s32(x[3], x[4], x[5]), c = __vimax3_s32(x[6], x[7], x[8]);
  const int32_t d = __vimax3_s32(x[9], x[10], x[11]), e = __vimax3_s32(x[12], x[13], x[14]);
  return max(__vimax3_s32(a, b, c), __vimax3_s32(d, e, x[15]));
}

// The u8 epilogue of one tile, from the s32 accumulator acc = a.b (exact).  Per element s = ||b||^2 - 2 a.b = ||a - b||^2 - ||a||^2
// (u8_elem), chunk minima in integers, and only the four minima per thread become h = s / 2: exactly the fp16 kernel's accumulator value
// (|s| < 2^24), so everything from the folds on is shared.  Pad rows: a.b = 0 (TMA zero fill), ||b||^2 = 2^24 (prep.cuh) -> h = 2^23, as
// in the fp16 kernel.  A chunk is the 16 columns THIS thread holds of a query row in one 64-column half of the tile (common.cuh chunk_row),
// so its minimum needs no shuffle; pad rows of a partial last tile share chunks with real rows and lose to them.
// Column 8j + 2 qlane + e of the tile (j = 0..15, e = 0, 1) is acc[4j + e] (row r0), acc[4j + 2 + e] (row r0 + 8); its norm is nb2[4j].
// v2[r][h] = minimum h of chunk 4h + qlane of row r0 + 8r.
__device__ __forceinline__ void u8_tile_minima(const int32_t (&acc)[64], const int2* nb2, float (&v2)[2][2]) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    int32_t x[2][16];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int2 n = nb2[4 * (8 * h + j)];
      const int a = 32 * h + 4 * j;
      x[0][2 * j] = u8_elem(n.x, acc[a + 0]); x[0][2 * j + 1] = u8_elem(n.y, acc[a + 1]);
      x[1][2 * j] = u8_elem(n.x, acc[a + 2]); x[1][2 * j + 1] = u8_elem(n.y, acc[a + 3]);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) v2[r][h] = u8_half_dist(min16(x[r]));
  }
}

// The norm-GEMM (NG) epilogue of one tile: the accumulator already holds acc = 2 a.b - ||b||^2 = -s (exact s32), so a chunk minimum of s is
// minus the chunk maximum of acc, and h = s / 2 is exactly what u8_tile_minima computes.  Same chunks and v2 layout as there.  Pad rows:
// a.b = 0 (TMA zero fill) and all limbs 255 -> s = U8_LIMB_PAD, above every real row's s <= ||b||^2 <= U8_LIMB_CAP.
__device__ __forceinline__ void u8ng_tile_minima(const int32_t (&acc)[64], float (&v2)[2][2]) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    int32_t x[2][16];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int a = 32 * h + 4 * j;
      x[0][2 * j] = acc[a + 0]; x[0][2 * j + 1] = acc[a + 1];
      x[1][2 * j] = acc[a + 2]; x[1][2 * j + 1] = acc[a + 3];
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) v2[r][h] = 0.5f * (float)(-max16(x[r]));   // |s| < 2^24: exact, and +0 for s = 0 as in u8_half_dist
  }
}

// The real-valued re-scoring reads 32 fp32 rows per candidate (16 KB, mostly from HBM) and is latency-bound: two warps cannot keep up with
// the tensor cores, so MODE_REAL adds six re-scoring warps behind the epilogue warps.
constexpr int REAL_EXTRA_VERIFY_WARPS = 6;
template <int MODE> constexpr int block_threads() { return 128 + EPI_WARPS * 32 + (MODE == MODE_REAL ? REAL_EXTRA_VERIFY_WARPS * 32 : 0); }

// The kernel body (entry points at the end of the file).  U8: the operands are the views' uchar rows (tmap_u8) on the 8-bit tensor cores,
// MODE_MATCH only; see the consumer loop.  NG (with U8): the norm-GEMM kernel (header comment).
template <bool AUG, int MODE, bool U8, bool NG = false>
__device__ __forceinline__ void
l2_top2_tc(const ViewDev* __restrict__ views, const PairDev* __restrict__ pairs, const WorkItem* __restrict__ items, int n_items,
           int ctas_per_item, Cand* __restrict__ cands, int* __restrict__ cand_count, float ratio_sq, long long* __restrict__ trace_buf,
           unsigned int* __restrict__ err_count, int fused, uint32_t* __restrict__ candx, FbSink fb) {
  long long* trace = (blockIdx.x == 0) ? trace_buf : nullptr;
  constexpr bool REAL = MODE == MODE_REAL, KNN = MODE == MODE_KNN;
  constexpr int VERIFY_WARPS_K = REAL ? 2 + REAL_EXTRA_VERIFY_WARPS : 2;   // warps 2, 3 (+ the warps behind the epilogue warps)
  static_assert(!(REAL || KNN) || AUG, "MODE_REAL / MODE_KNN exist for the AUG layout only");
  static_assert(!U8 || (MODE == MODE_MATCH && !AUG), "the u8 kernel is MODE_MATCH with its norms in the database ring");
  static_assert(!NG || U8, "the norm-GEMM kernel is a form of the u8 kernel");
  using L = Lay<AUG, REAL, U8, NG>;
  constexpr int NS = L::NS, STAGE = L::STAGE, QT = L::QT;
  extern __shared__ __align__(1024) uint8_t smem[];   // SWIZZLE_128B operand tiles need 1024-B alignment
  if ((ptx::smem_u32(smem) & 1023u) != 0) { asm volatile("trap;"); }
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::OFF_BAR);
  uint64_t* q_full = bars;                  // [2]  producer + TMA bytes
  uint64_t* q_empty = q_full + 2;           // [2]  8 consumer warps
  uint64_t* db_full = q_empty + 2;          // [NS] producer + TMA bytes
  uint64_t* db_empty = db_full + NS;        // [NS] 8 consumer warps
  uint64_t* vq_full = db_empty + NS;        // [2]  4 arrivals (the epilogue quadrants that emit candidates)
  uint64_t* vq_empty = vq_full + 2;         // [2]  the exactness-pass warps

  // U8: the role branches hold setmaxnreg and the wgmma pipeline, which ptxas only keeps on a path it can prove warp-uniform
  const int warp = U8 ? __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0) : (int)(threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  // the roles take these as arguments: the u8 kernel computes them in each role (see the dispatch at the end)
  const int rank = (int)blockIdx.x % ctas_per_item;   // which 128 queries of the work item
  const int cl = (int)blockIdx.x / ctas_per_item;
  const int n_cl = (int)gridDim.x / ctas_per_item;

  if (warp == 1 && lane == 0) {
    for (int i = 0; i < 2; ++i) {
      ptx::mbar_init(&q_full[i], 1); ptx::mbar_init(&q_empty[i], EPI_WARPS);
      ptx::mbar_init(&vq_full[i], 4); ptx::mbar_init(&vq_empty[i], VERIFY_WARPS_K);
    }
    for (int i = 0; i < NS; ++i) { ptx::mbar_init(&db_full[i], 1); ptx::mbar_init(&db_empty[i], EPI_WARPS); }
    ptx::fence_mbar_init();
  }
  if (AUG && !REAL && warp >= 4 && warp < 8) {
    // the constant augmentation tile of the A operand: 128 rows x 16 fp16 in the 32-byte-swizzled K-major layout
    // (16-byte chunk index XOR ((row >> 2) & 1)); logical chunk 0 = [-0.5, -1, -2048, 0, 0, 0, 0, 0], chunk 1 = zeros
    const int r = (warp - 4) * 32 + lane;
    uint4* rowp = reinterpret_cast<uint4*>(smem + L::OFF_A + r * 32);
    const uint32_t c01 = (uint32_t)__half_as_ushort(__float2half_rn(-0.5f)) | ((uint32_t)__half_as_ushort(__float2half_rn(-1.f)) << 16);
    const uint32_t c23 = (uint32_t)__half_as_ushort(__float2half_rn(-2048.f));
    const int sw = (r >> 2) & 1;
    rowp[sw] = make_uint4(c01, c23, 0u, 0u);
    rowp[sw ^ 1] = make_uint4(0u, 0u, 0u, 0u);
    ptx::fence_proxy_async();          // generic-proxy stores -> visible to the tensor core (async proxy)
  }
  if (NG && warp >= 4 && warp < 8) {
    // the constant s8 weight tile of the 5th K-step: 128 rows x 32 B in the 32-byte-swizzled K-major layout (16-byte chunk index XOR
    // ((row >> 2) & 1)); logical chunk 0 = [-1, -128 x 15], chunk 1 = [-128 x 16] (U8_LIMB_W0, U8_LIMB_W)
    static_assert(U8_LIMB_W0 == -1 && U8_LIMB_W == -128, "the weight bytes below");
    const int r = (warp - 4) * 32 + lane;
    uint4* rowp = reinterpret_cast<uint4*>(smem + L::OFF_A + r * 32);
    const int sw = (r >> 2) & 1;
    rowp[sw] = make_uint4(0x808080FFu, 0x80808080u, 0x80808080u, 0x80808080u);
    rowp[sw ^ 1] = make_uint4(0x80808080u, 0x80808080u, 0x80808080u, 0x80808080u);
    ptx::fence_proxy_async();
  }
  __syncthreads();

  auto producer = [&](int rank, int cl) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      uint32_t qb = 0, qph = 0, st = 0, sph = 0, tt = 0;
      for (int it = cl; it < n_items; it += n_cl) {
        const WorkItem w = items[it];
        const PairDev p = pairs[w.pair];
        const ViewDev* vi = views + p.view_i;
        const ViewDev* vj = views + p.view_j;
        const int qrow = ((int)w.qtile * ctas_per_item + rank) * BM;
        ptx::mbar_wait(&q_empty[qb], qph ^ 1);
        ptx::mbar_arrive_expect_tx(&q_full[qb], QT + (REAL ? AUG_BYTES : 0));
        uint8_t* qs = smem + L::OFF_Q + qb * QT;
        if (U8) {
          ptx::tma_load_2d(qs, &vj->tmap_u8, &q_full[qb], 0, qrow);
        } else {
          ptx::tma_load_2d(qs, &vj->tmap128, &q_full[qb], 0, qrow);
          ptx::tma_load_2d(qs + KB_BYTES, &vj->tmap128, &q_full[qb], 64, qrow);
        }
        if (REAL) ptx::tma_load_2d(smem + L::OFF_A + qb * AUG_BYTES, &vj->tmap_augq, &q_full[qb], 0, qrow);   // the query rows' own half-norm limbs
        qb ^= 1; if (qb == 0) qph ^= 1;
        const int ntiles = ((int)p.m_i + BN - 1) / BN;
        for (int t = 0; t < ntiles; ++t) {
          ptx::mbar_wait(&db_empty[st], sph ^ 1);
          ptx::trace_stamp(trace, 0, tt, 0);
          uint8_t* ds = smem + L::OFF_DB + st * STAGE;
          if (NG) {
            ptx::mbar_arrive_expect_tx(&db_full[st], U8_BYTES + LIMB_BYTES);
            ptx::tma_load_2d(ds, &vi->tmap_u8, &db_full[st], 0, t * BN);
            ptx::tma_load_2d(ds + U8_BYTES, &vi->tmap_limb, &db_full[st], 0, t * BN);
          } else if (U8) {
            ptx::mbar_arrive_expect_tx(&db_full[st], U8_BYTES + NB_BYTES);
            ptx::tma_load_2d(ds, &vi->tmap_u8, &db_full[st], 0, t * BN);
            ptx::bulk_load_1d(ds + U8_BYTES, vi->nb32 + (size_t)t * BN, NB_BYTES, &db_full[st]);
          } else {
            ptx::mbar_arrive_expect_tx(&db_full[st], DB_BYTES + (AUG ? AUG_BYTES : NB_BYTES));
            ptx::tma_load_2d(ds, &vi->tmap128, &db_full[st], 0, t * BN);
            ptx::tma_load_2d(ds + KB_BYTES, &vi->tmap128, &db_full[st], 64, t * BN);
            if (AUG) ptx::tma_load_2d(ds + DB_BYTES, &vi->tmap_aug, &db_full[st], 0, t * BN);
            else ptx::bulk_load_1d(ds + DB_BYTES, vi->nbh + (size_t)t * BN, NB_BYTES, &db_full[st]);
          }
          ptx::trace_stamp(trace, 0, tt, 1); ++tt;
          if (++st == NS) { st = 0; sph ^= 1; }
        }
      }
    }
  };
  auto exactness_pass = [&](int cl) {
    // ------------------------------------------------------------------ exactness pass of the previous item
    // fused == 0 (short database images: an item lasts only a few tiles, two warps cannot hide the re-scoring latency):
    // the epilogue writes its candidates to global memory and the stand-alone exactness kernel handles them.
    uint32_t par = 0, vph = 0;
    for (int it = cl; fused && it < n_items; it += n_cl) {
      ptx::mbar_wait(&vq_full[par], vph);
      const uint32_t* hdr = reinterpret_cast<const uint32_t*>(smem + L::OFF_VQN + par * 32);
      const PairDev p = pairs[hdr[4]];
      const __half* db16 = views[p.view_i].h16;
      const __half* q16 = views[p.view_j].h16;
      const Cand* queue = reinterpret_cast<const Cand*>(smem + L::OFF_VQ) + par * BM;
      const uint32_t* queuex = reinterpret_cast<const uint32_t*>(smem + L::OFF_VQX) + par * BM;
      // MATCH: warp 2 serves quadrants 0-1, warp 3 quadrants 2-3.  REAL (8 warps): two warps per quadrant, alternate entries.
      const int vw = warp < 4 ? warp - 2 : warp - (4 + EPI_WARPS) + 2;
      const int quad_lo = REAL ? (vw & 3) : vw * 2, quad_hi = REAL ? quad_lo + 1 : quad_lo + 2;
      const int e_first = REAL ? (vw >> 2) : 0, e_step = REAL ? 2 : 1;
      for (int quad = quad_lo; quad < quad_hi; ++quad) {
        const int n = (int)hdr[quad];
        for (int e = e_first; e < n; e += e_step) {
          const Cand k = queue[quad * 32 + e];
          Rec rec;
          int verdict;                                                          // 0 drop, 1 keep, 2 undecided -> exact_rows fallback
          if (REAL) verdict = rescore_real(views[p.view_i], views[p.view_j], p.m_i, k, queuex[quad * 32 + e], ratio_sq, lane, err_count, rec);
          else verdict = rescore_candidate(db16, q16, p.m_i, k, U8, ratio_sq, lane, err_count, rec) ? 1 : 0;
          if (verdict == 1 && lane == 0) {
            const int slot = atomicAdd(&cand_count[hdr[4]], 1);
            cands[p.cand_base + slot] = Cand{rec.j, rec.i, rec.d1, rec.d2};     // final record, (query, database row) order like the exact kernels
          }
          if (REAL && verdict == 2 && lane == 0) fb_push(fb, hdr[4], k.q, 0u, 0u, err_count);   // no slot of its own: the fallback appends
        }
      }
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&vq_empty[par]);
      par ^= 1; if (par == 0) vph ^= 1;
    }
  };
  auto consumers = [&](int rank, int cl) {
    // ------------------------------------------------------------------ consumers: MMA + epilogue (two warpgroups of 64 rows)
    const int wg = (warp - 4) >> 2;
    const int qlane = lane & 3;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);    // first of this thread's two rows (the second is r0 + 8)
    const uint32_t q_addr = ptx::smem_u32(smem + L::OFF_Q) + wg * 64 * 128;
    const uint32_t db_addr = ptx::smem_u32(smem + L::OFF_DB);
    const uint32_t a_aug = ptx::smem_u32(smem + L::OFF_A) + wg * 64 * 32;
    long long* etrace = (lane == 0 && (warp & 3) == 0) ? trace : nullptr;
    uint32_t qb = 0, qph = 0, st = 0, sph = 0, par = 0, vqph = 0, tt = 0;
    for (int it = cl; it < n_items; it += n_cl) {
      const WorkItem w = items[it];
      const PairDev p = pairs[w.pair];
      const int ntiles = ((int)p.m_i + BN - 1) / BN;
      Top2 s[2] = {{INFINITY, INFINITY, 0u}, {INFINITY, INFINITY, 0u}};
      Top2g sk[2] = {{INFINITY, INFINITY, 0xFFFFu, 0xFFFFu}, {INFINITY, INFINITY, 0xFFFFu, 0xFFFFu}};   // MODE_KNN
      constexpr uint32_t NONE = 0x7F800000u | REAL_IDMASK;                                               // MODE_REAL: +inf, id = none
      Top4 s4[2] = {{NONE, NONE, NONE, NONE}, {NONE, NONE, NONE, NONE}};
      ptx::mbar_wait(&q_full[qb], qph);
      auto release_slot = [&] {
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&db_empty[st]);               // this warp is done with the slot (operands and (half-)norms)
        if (++st == NS) { st = 0; sph ^= 1; }
      };
      // v2[r][h]: chunk minima h of chunks 4h + qlane of tile t, rows r0, r0 + 8
      auto fold_tile = [&](int t, const float (&v2)[2][2]) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t gid = (uint32_t)t * (BN / CHUNK) + 4 * h + qlane;
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            if (REAL) fold_chunk_real(v2[r][h], gid, s4[r]);
            else if (KNN) fold_chunk_knn(v2[r][h], gid, sk[r]);
            else fold_chunk(v2[r][h], gid, s[r]);
          }
        }
      };
      if constexpr (U8) {
        // Software pipeline over the item's tiles: the MMAs of tile t + 1 are issued into the other accumulator before the epilogue of
        // tile t, and wgmma.wait_group 1 waits for tile t's group only, so each warpgroup's epilogue runs under its own next MMAs.  The
        // pipeline fills and drains inside the work item: the item boundary (q_empty, the merge, the candidate hand-off) is unchanged.
        // Slot t is released after its epilogue (its norms are read there), one MMA group later than without the pipeline; NG reads nothing
        // from the slot in its epilogue and releases it as soon as tile t's MMAs have completed.
        const int nt = __shfl_sync(0xffffffffu, ntiles, 0);           // warp-uniform bounds keep the wgmma pipeline out of divergent paths
        const uint32_t a_base = q_addr + qb * QT;
        if constexpr (NG) {
          // 2a in place: this warpgroup's 64 query rows (8 KB, contiguous whatever the swizzle).  Every byte is <= 127 (VF_U8_WIDE), so a
          // left shift of each 32-bit word doubles its four bytes without carries.  The exactness pass reads the queries from global memory.
          uint4* qw = reinterpret_cast<uint4*>(smem + L::OFF_Q + qb * QT + wg * 64 * 128);
          const int tid = (warp & 3) * 32 + lane;
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            uint4 x = qw[tid + 128 * k];
            x.x <<= 1; x.y <<= 1; x.z <<= 1; x.w <<= 1;
            qw[tid + 128 * k] = x;
          }
          ptx::fence_proxy_async();                                    // generic-proxy stores -> visible to this warpgroup's wgmma
          if (wg == 0) ptx::named_bar_sync(2, 128); else ptx::named_bar_sync(3, 128);   // immediate ids: ptxas reserves all 16 for a register id
        }
        uint32_t ist = st, isph = sph;                                 // ring slot of the next tile to issue
        auto issue = [&](int32_t (&acc)[64]) {
          const uint32_t b_base = db_addr + ist * STAGE;
          ptx::wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)
            ptx::wgmma_m64n128k32_u8(acc, ptx::wgmma_desc_k_sw128(a_base + k * 32), ptx::wgmma_desc_k_sw128(b_base + k * 32), k > 0 ? 1u : 0u);
          if (NG) ptx::wgmma_m64n128k32_s8u8(acc, ptx::wgmma_desc_k_sw32(a_aug), ptx::wgmma_desc_k_sw32(b_base + U8_BYTES), 1u);   // - ||b||^2
          ptx::wgmma_commit();
          if (++ist == NS) { ist = 0; isph ^= 1; }
        };
        // trace per tile: 0 start, 1 tile t + 1 landed (db_full), 2 tile t's MMAs complete (the wait_group 1), 3 tile t folded
        // `last` is a constant after inlining: the wgmma sequence of each copy is branch-free, which ptxas needs to keep the pipeline
        auto tile = [&](int t, const int32_t (&acc)[64], int32_t (&acc_next)[64], bool last) {
          ptx::trace_stamp(etrace, 1 + wg, tt, 0);
          if (!last) {
            ptx::mbar_wait(&db_full[ist], isph);
            ptx::trace_stamp(etrace, 1 + wg, tt, 1);
            issue(acc_next);
            ptx::wgmma_wait<1>();                                      // tile t's group has completed, tile t + 1's runs on
          } else {
            ptx::trace_stamp(etrace, 1 + wg, tt, 1);
            ptx::wgmma_wait<0>();
          }
          ptx::trace_stamp(etrace, 1 + wg, tt, 2);
          float v2[2][2];
          if (NG) {
            release_slot();
            u8ng_tile_minima(acc, v2);
          } else {
            u8_tile_minima(acc, reinterpret_cast<const int2*>(smem + L::OFF_DB + st * STAGE + U8_BYTES) + qlane, v2);
            release_slot();
          }
          fold_tile(t, v2);
          ptx::trace_stamp(etrace, 1 + wg, tt, 3); ++tt;
        };
        int32_t acc0[64], acc1[64];
        if (nt > 0) {
          ptx::mbar_wait(&db_full[ist], isph);
          issue(acc0);
          for (int t = 0;; t += 2) {                                   // unrolled by two: even tiles in acc0, odd tiles in acc1; the only
            if (t + 1 == nt) { tile(t, acc0, acc1, true); break; }     // exits follow a drained last tile
            tile(t, acc0, acc1, false);
            if (t + 2 == nt) { tile(t + 1, acc1, acc0, true); break; }
            tile(t + 1, acc1, acc0, false);
          }
        }
      } else {
        for (int t = 0; t < ntiles; ++t) {
          ptx::trace_stamp(etrace, 1 + wg, tt, 0);
          ptx::mbar_wait(&db_full[st], sph);
          ptx::trace_stamp(etrace, 1 + wg, tt, 1);
          const uint32_t b_base = db_addr + st * STAGE;
          float acc[64];
          ptx::wgmma_fence();
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const uint64_t da = ptx::wgmma_desc_k_sw128(q_addr + qb * Q_BYTES + (k >> 2) * KB_BYTES + (k & 3) * 32);
            const uint64_t db = ptx::wgmma_desc_k_sw128(b_base + (k >> 2) * KB_BYTES + (k & 3) * 32);
            ptx::wgmma_m64n128k16_f16_negb(acc, da, db, k > 0 ? 1u : 0u);
          }
          if (AUG) {  // 9th K-step: constants (or the query's limbs) x the database rows' half-norm limbs
            const uint64_t da = ptx::wgmma_desc_k_sw32(a_aug + (REAL ? qb * AUG_BYTES : 0));
            const uint64_t db = ptx::wgmma_desc_k_sw32(b_base + DB_BYTES);
            ptx::wgmma_m64n128k16_f16_negb(acc, da, db, 1u);
          }
          ptx::wgmma_commit();
          ptx::wgmma_wait_all();
          ptx::trace_stamp(etrace, 1 + wg, tt, 2);
          if (!AUG) {
            const float2* nb2 = reinterpret_cast<const float2*>(smem + L::OFF_DB + st * STAGE + DB_BYTES) + qlane;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              const float2 nb = nb2[4 * j];
              acc[4 * j + 0] += nb.x; acc[4 * j + 1] += nb.y; acc[4 * j + 2] += nb.x; acc[4 * j + 3] += nb.y;
            }
          }
          release_slot();
          // chunk c of row r0: acc[8c + {0, 1, 4, 5}]; of row r0 + 8: acc[8c + {2, 3, 6, 7}]
          float pm[2][8];
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            pm[0][c] = fminf(fminf(acc[8 * c + 0], acc[8 * c + 1]), fminf(acc[8 * c + 4], acc[8 * c + 5]));
            pm[1][c] = fminf(fminf(acc[8 * c + 2], acc[8 * c + 3]), fminf(acc[8 * c + 6], acc[8 * c + 7]));
          }
          float v2[2][2];
          quad_chunk_minima(pm, qlane, v2);
          fold_tile(t, v2);
          ptx::trace_stamp(etrace, 1 + wg, tt, 3); ++tt;
        }
      }
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&q_empty[qb]);                 // every MMA of this item has completed
      qb ^= 1; if (qb == 0) qph ^= 1;
      // merge the four lanes' chunk sets, hand each row's state to the emitting warps through shared memory
      float4* mrg = reinterpret_cast<float4*>(smem + L::OFF_MRG) + par * BM;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        for (int m = 1; m <= 2; m <<= 1) {
          if (REAL) merge_xor(s4[r], m); else if (KNN) merge_xor(sk[r], m); else merge_xor(s[r], m);
        }
        if (qlane == 0) {
          const int row = r0 + 8 * r;
          if (REAL) mrg[row] = make_float4(__uint_as_float(s4[r].p1), __uint_as_float(s4[r].p2), __uint_as_float(s4[r].p3), __uint_as_float(s4[r].p4));
          else if (KNN) mrg[row] = make_float4(sk[r].m1, sk[r].m2, __uint_as_float(sk[r].g1), __uint_as_float(sk[r].g2));
          else mrg[row] = make_float4(s[r].m1, s[r].m2, __uint_as_float(s[r].g1), 0.f);
        }
      }
      ptx::named_bar_sync(1, EPI_WARPS * 32);
      if (wg == 0) {
        // pre-test and emit: warp 4 + quad handles rows 32 quad .. 32 quad + 31
        const int quad = warp & 3;
        const int row = quad * 32 + lane;
        const float4 o = mrg[row];
        const uint32_t q = ((uint32_t)w.qtile * ctas_per_item + rank) * BM + row;
        if (REAL) {
          const Top4 r4{__float_as_uint(o.x), __float_as_uint(o.y), __float_as_uint(o.z), __float_as_uint(o.w)};
          bool keep = false;
          if (q < p.m_j) {
            // superset pre-test on bounds of the TRUE (reference) distances: lower(best) < r^2 * upper(second smallest chunk minimum)
            const RealBound rb = real_bound(views[p.view_i], views[p.view_j], q);
            const float d1t = 2.f * __uint_as_float(r4.p1 & ~REAL_IDMASK), d2t = 2.f * __uint_as_float(r4.p2 & ~REAL_IDMASK);
            keep = rb.lower(d1t) < __fmul_rn(ratio_sq, rb.upper(d2t));
          }
          const uint32_t mask = __ballot_sync(0xffffffffu, keep);
          const int pos = __popc(mask & ((1u << lane) - 1));
          if (fused) {
            ptx::mbar_wait(&vq_empty[par], vqph ^ 1);
            Cand* queue = reinterpret_cast<Cand*>(smem + L::OFF_VQ) + par * BM + quad * 32;
            uint32_t* queuex = reinterpret_cast<uint32_t*>(smem + L::OFF_VQX) + par * BM + quad * 32;
            if (keep) { queue[pos] = Cand{q, r4.p1, __uint_as_float(r4.p2), __uint_as_float(r4.p3)}; queuex[pos] = r4.p4; }
            uint32_t* hdr = reinterpret_cast<uint32_t*>(smem + L::OFF_VQN + par * 32);
            if (lane == 0) { hdr[quad] = (uint32_t)__popc(mask); if (quad == 0) hdr[4] = w.pair; }
            __syncwarp();
            if (lane == 0) ptx::mbar_arrive(&vq_full[par]);
          } else if (mask) {
            int base = 0;
            if (lane == 0) base = atomicAdd(&cand_count[w.pair], __popc(mask));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (keep) { cands[p.cand_base + base + pos] = Cand{q, r4.p1, __uint_as_float(r4.p2), __uint_as_float(r4.p3)}; candx[p.cand_base + base + pos] = r4.p4; }
          }
        } else if (KNN) {
          if (q < p.m_j) {                                   // dense: every query leaves its two chunks for knn_finalize_kernel
            const float na = views[p.view_j].nrm[q];
            const uint32_t g1 = __float_as_uint(o.z), g2 = __float_as_uint(o.w);
            cands[p.cand_base + q] = Cand{q, (g1 & 0xFFFFu) | (g2 << 16), fmaf(2.f, o.x, na), fmaf(2.f, o.y, na)};
          }
        } else {
          const uint32_t g1 = __float_as_uint(o.z);
          bool keep = false;
          float d1 = 0.f, d2 = 0.f;
          if (q < p.m_j) {
            const float na = views[p.view_j].nrm[q];
            d1 = fmaf(2.f, o.x, na);
            d2 = fmaf(2.f, o.y, na);
            keep = d1 < __fmul_rn(ratio_sq, d2);
          }
          const uint32_t mask = __ballot_sync(0xffffffffu, keep);
          if (fused) {
            // hand the survivors of the pre-test to the exactness-pass warps through shared memory (32 slots per quadrant)
            ptx::mbar_wait(&vq_empty[par], vqph ^ 1);        // they finished the item that used this buffer two items ago
            Cand* queue = reinterpret_cast<Cand*>(smem + L::OFF_VQ) + par * BM + quad * 32;
            if (keep) queue[__popc(mask & ((1u << lane) - 1))] = Cand{q, g1, d1, d2};
            uint32_t* hdr = reinterpret_cast<uint32_t*>(smem + L::OFF_VQN + par * 32);
            if (lane == 0) { hdr[quad] = (uint32_t)__popc(mask); if (quad == 0) hdr[4] = w.pair; }
            __syncwarp();
            if (lane == 0) ptx::mbar_arrive(&vq_full[par]);
          } else if (mask) {
            int base = 0;
            if (lane == 0) base = atomicAdd(&cand_count[w.pair], __popc(mask));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (keep) cands[p.cand_base + base + __popc(mask & ((1u << lane) - 1))] = Cand{q, g1, d1, d2};
          }
        }
      }
      par ^= 1; if (par == 0) vqph ^= 1;
    }
  };
  if constexpr (U8) {
    // Registers move from warpgroup 0 (producer, exactness pass: little state) to the consumers (two accumulators each).  One
    // setmaxnreg per warpgroup, at the head of a branch that holds all of its code: ptxas compiles each region to its count, and code
    // that both counts reach would have to fit the smaller one.  It spills a value that lives across setmaxnreg, so each role reads
    // the block index itself.
    if (warp < 4) {
      ptx::setmaxnreg_dec<U8_REGS_WG0>();
      const int b = ptx::block_index();
      if (warp == 0) producer(b % ctas_per_item, b / ctas_per_item);
      else if (warp >= 2) exactness_pass(b / ctas_per_item);
    } else {
      ptx::setmaxnreg_inc<U8_REGS_CONSUMER>();
      const int b = ptx::block_index();
      consumers(b % ctas_per_item, b / ctas_per_item);
    }
  } else {
    if (warp == 0) producer(rank, cl);
    else if (warp == 2 || warp == 3 || warp >= 4 + EPI_WARPS) exactness_pass(cl);
    else if (warp >= 4) consumers(rank, cl);
  }
}

#define B200M_TC_PARAMS const ViewDev* __restrict__ views, const PairDev* __restrict__ pairs, const WorkItem* __restrict__ items, int n_items, \
    int ctas_per_item, Cand* __restrict__ cands, int* __restrict__ cand_count, float ratio_sq, long long* __restrict__ trace_buf, \
    unsigned int* __restrict__ err_count, int fused, uint32_t* __restrict__ candx, FbSink fb
#define B200M_TC_ARGS views, pairs, items, n_items, ctas_per_item, cands, cand_count, ratio_sq, trace_buf, err_count, fused, candx, fb

template <bool AUG, int MODE = MODE_MATCH>
__global__ void __launch_bounds__(block_threads<MODE>(), 1) l2_top2_tc_kernel(B200M_TC_PARAMS) { l2_top2_tc<AUG, MODE, false>(B200M_TC_ARGS); }

// The u8 kernel is launched with 128 registers per thread: the 512-thread, 32-register device finishing kernel (finish.cuh) of the previous
// batch then still fits beside the persistent CTA of each SM, as it does beside the fp16 kernel.  At 130 registers it waited for the search
// kernel to end, and consecutive batches' search kernels no longer ran back to back.  Inside that allocation setmaxnreg gives the consumers
// 160 (U8_REGS_CONSUMER) for their two accumulators.
__global__ void __maxnreg__(128) l2_top2_tc_u8_kernel(B200M_TC_PARAMS) {
  l2_top2_tc<false, MODE_MATCH, true>(B200M_TC_ARGS);
}
// The u8 norm-GEMM kernel: the same launch shape and register split.
__global__ void __maxnreg__(128) l2_top2_tc_u8ng_kernel(B200M_TC_PARAMS) {
  l2_top2_tc<false, MODE_MATCH, true, true>(B200M_TC_ARGS);
}

#undef B200M_TC_PARAMS
#undef B200M_TC_ARGS

}  // namespace tc
}  // namespace b200m

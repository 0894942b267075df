// Device-side data model shared by the kernels of the descriptor-matching engine.
// Names follow the reference's domain: views (images), regions/descriptors, pairs (I = database image,
// J = query image; matching/RegionsMatcher.hpp:126-176), putative matches.
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace b200m {

enum : int { DT_F32 = 0, DT_U8 = 1, DT_BIN = 2 };

// Per-view flag bits written by the prep kernel.
enum : uint32_t {
  VF_NONINTEGER = 1u,   // some component is not an integer
  VF_RANGE = 2u,        // some |component| > 1024 (2v would not be exact in fp16)
  VF_NORM = 4u,         // some squared norm >= 2^22 (distances would leave the exact-fp32 range)
  VF_EXACT_MASK = 7u,   // the bits above: any of them set -> the view cannot take the (integer) tensor-core path
  VF_POS_NONGENERIC = 8u,   // feature positions: two features share an x or a y (or a NaN): coordinate de-duplication stays on the host
  // uchar-stored views only (prep.cuh), outside VF_EXACT_MASK: which side of the u8 norm-GEMM kernel (l2_tc.cuh NG) a view may take
  VF_U8_WIDE = 16u,     // some component > 127: 2a would not fit in u8, so the view is no QUERY of the norm-GEMM kernel
  VF_U8_NORMCAP = 32u,  // some squared norm > U8_LIMB_CAP: its limbs cannot hold it, so the view is no DATABASE of the norm-GEMM kernel
};

// One uploaded view (image) resident in HBM.
struct alignas(128) ViewDev {
  CUtensorMap tmap128;  // fp16 [m x 128], box {64 x 128 rows}, SWIZZLE_128B: one K-block of a query or database tile (only when dim == 128 scalar)
  CUtensorMap tmap_aug; // fp16 [m_pad x 16] half-norm limbs, box {16 x 128 rows}, SWIZZLE_32B (9th K-step of the AUG kernel)
  CUtensorMap tmap_augq; // the same for augq16 (the view as QUERY of the real-valued kernel: its own half-norm limbs as A columns)
  CUtensorMap tmap_u8;  // uchar-stored views only: `raw` as u8 [m x 128], box {128 B x 128 rows}, SWIZZLE_128B (the u8 kernel's operand tile)
  CUtensorMap tmap_limb; // uchar-stored views only: limb8 as u8 [m_pad x 32], box {32 B x 128 rows}, SWIZZLE_32B (the norm-GEMM kernel's 5th K-step)
  const int32_t* nb32;  // uchar-stored views only: ||row||^2 + U8_NORM_BIAS as int32, padded to a multiple of 256 rows with 2^24 + U8_NORM_BIAS (prep.cuh), else nullptr
  const void* raw;      // descriptors as STORED, row-major m x dim: f32 / u8 / 64-byte binary; `dtype` is the storage type (integer-valued
                        // fp32 descriptors are staged and stored as u8: same values, a quarter of the bytes)
  const __half* h16;    // fp16 copy (scalar, dim == 128) or nullptr
  const float* nbh;     // ||row||^2 / 2, padded to a multiple of 256 rows with 1e30f
  const float* nrm;     // ||row||^2
  const __half* aug16;  // m_pad x 16: [b0, l0, l1, -0.5, -1, -2048, 0...] with ||row||^2/2 = 0.5*b0 + l0 + 2048*l1; pad rows [0, 0, 4096, ...] (prep.cuh)
  const __half* augq16; // m_pad x 16: [-0.5, -1, -2048, b0, l0, l1, 0...] (prep.cuh)
  const float* err;     // m_pad: upper bound of ||row - fp16(row)||_2 (0 for integer-valued rows)
  const uint32_t* stats; // float bits: [0] max err over the view, [1] max ||fp16(row)||^2
  int32_t m;            // number of regions
  int32_t dim;          // components (scalar) or bytes (binary)
  int32_t dtype;        // storage type of `raw` (DT_*)
  int32_t pad_;
  const uint32_t* yrank;  // per feature: rank of its y among the view's features (finish.cuh), or nullptr without positions
};
static_assert(sizeof(ViewDev) % 128 == 0, "ViewDev must keep CUtensorMap 64-byte aligned in arrays");

// One image pair of the current batch.
struct PairDev {
  uint32_t view_i, view_j;   // slots into the view table (I = database, J = query)
  uint32_t m_i, m_j;
  uint32_t cand_base;        // first candidate slot of this pair (prefix sum of m_j over the batch)
  uint32_t mode;             // PM_*
  uint32_t slot_base;        // prefix sum of m_i over the batch: this pair's scratch range of the device finishing stage (finish.cuh)
  uint32_t thread_chunks;    // PM_TC: 1 when the pair's candidates come from the u8 kernel (chunk ids in its per-thread layout, chunk_row)
};
enum : uint32_t { PM_TC = 0, PM_EXACT_F32 = 1, PM_EXACT_U8 = 2, PM_HAMMING = 3, PM_SKIP = 4,
                  PM_TC_FUSED = 5 /* tensor-core pair whose kernel also ran the exactness pass: candidates are final */,
                  PM_GENERIC_F32 = 6, PM_GENERIC_U8 = 7 /* scalar descriptors whose length is not 128 (AKAZE float 64, LIOP 144): one warp per query */,
                  PM_TC_REAL = 8 /* real-valued fp32 pair on the tensor-core FILTER kernel (l2_tc.cuh MODE_REAL): its candidates are made final by
                                    the exact re-scoring (in-kernel or rescore_real_kernel) and the exact_rows fallback before they are packed */ };

// Work item of the tensor-core kernel: 128 or 256 (per launch) consecutive queries of pair `pair` against the whole database image.
struct WorkItem { uint32_t pair, qtile; };

// Candidate produced by a search kernel, one per query that passed the (pre-)ratio test.
//   PM_TC:   a = query row, b = 16-row chunk id of the best database row (chunk_row), d1 exact, d2 = upper bound (exactness pass needed)
//   others:  a = query row, b = database row of the nearest neighbour, d1/d2 exact (float bits, or uint32 bits for Hamming)
//   PM_TC_REAL (before re-scoring): q = query row, b / d1 / d2 = bit patterns p1 / p2 / p3 of the three smallest packed chunk minima
//            (value with the chunk id in the low REAL_IDBITS bits), p4 in the parallel `candx` word
struct Cand { uint32_t q, b; float d1, d2; };

// ViewDev::nb32 holds ||row||^2 + U8_NORM_BIAS: with it the u8 kernel's per-element value ||b||^2 - 2 a.b > -||a||^2 > -2^22 is positive, and
// positive values order the same as integers and as float bit patterns (l2_tc.cuh u8_elem)
constexpr int32_t U8_NORM_BIAS = 1 << 22;

// The u8 norm-GEMM kernel (l2_tc.cuh NG) folds the database norm into its s32 accumulator with one extra K32 step: per database row 32 u8
// limbs l_k with ||b||^2 = l_0 + 128 * (l_1 + ... + l_31), l_0 < 128, each limb <= 255, against the constant s8 weights
// w_0 = -1, w_1..31 = -128 (U8_LIMB_W0, U8_LIMB_W).  Capacity: 127 + 128 * 31 * 255.  Pad rows carry all limbs 255, whose norm
// U8_LIMB_PAD exceeds every real row's.
constexpr int32_t U8_LIMB_W0 = -1, U8_LIMB_W = -128;
constexpr int32_t U8_LIMB_CAP = 127 + 128 * 31 * 255;          // 1,011,967
constexpr int32_t U8_LIMB_PAD = 255 + 128 * 31 * 255;          // 1,012,095
__host__ __device__ __forceinline__ uint32_t u8_limb(int32_t nrm2, int k) {
  if (k == 0) return (uint32_t)(nrm2 & 127);
  const int32_t q = (nrm2 >> 7) - 255 * (k - 1);                // limbs 1..31 fill up to 255 each, in order
  return (uint32_t)(q < 0 ? 0 : q > 255 ? 255 : q);
}

// Database row r (0..15, ascending) of 16-row chunk g of a tensor-core candidate.  The fp16 kernels' chunks are contiguous rows.  The u8
// kernel's chunk g = 8t + 4h + q is what ONE thread (lane % 4 = q) holds of a query row in the 64-column half h of tile t:
// rows 128t + 64h + 8j + 2q + e (j = 0..7, e = 0, 1), so that a chunk minimum needs no exchange between threads.
__device__ __forceinline__ uint32_t chunk_row(uint32_t g, int r, bool thread_chunks) {
  return thread_chunks ? (g >> 2) * 64 + (uint32_t)(r >> 1) * 8 + (g & 3) * 2 + (uint32_t)(r & 1) : g * 16 + (uint32_t)r;
}

// Real-valued filter: chunk ids ride in the low mantissa bits of the (non-negative) chunk minima
constexpr int REAL_IDBITS = 13;                       // 8191 chunks of 16 rows = 131056 database rows at most
constexpr uint32_t REAL_IDMASK = (1u << REAL_IDBITS) - 1u;
constexpr int REAL_MAX_ROWS = 16 * (int)REAL_IDMASK;   // the all-ones id means "no chunk"

// Raw match record handed to the host: i = database (I) feature, j = query (J) feature, the two smallest distances.
// i == 0xFFFFFFFF marks a candidate dropped by the exactness pass.  For Hamming d1/d2 hold uint32 bit patterns.
struct Rec { uint32_t i, j; float d1, d2; };

// Element k of a view's descriptors as float, whatever the storage type (block-uniform branch).
__device__ __forceinline__ float view_elem(const ViewDev& v, size_t k) {
  return v.dtype == DT_F32 ? reinterpret_cast<const float*>(v.raw)[k] : (float)reinterpret_cast<const uint8_t*>(v.raw)[k];
}

}  // namespace b200m

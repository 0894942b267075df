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
};

// One uploaded view (image) resident in HBM.
struct alignas(128) ViewDev {
  CUtensorMap tmap128;  // fp16 [m x 128], box {64 x 128 rows}, SWIZZLE_128B: one K-block of a query or database tile (only when dim == 128 scalar)
  CUtensorMap tmap_aug; // fp16 [m_pad x 16] half-norm limbs, box {16 x 128 rows}, SWIZZLE_32B (9th K-step of the AUG kernel)
  CUtensorMap tmap_augq; // the same for augq16 (the view as QUERY of the real-valued kernel: its own half-norm limbs as A columns)
  const void* raw;      // descriptors as STORED, row-major m x dim: f32 / u8 / 64-byte binary; `dtype` is the storage type (integer-valued
                        // fp32 descriptors are staged and stored as u8: same values, a quarter of the bytes)
  const __half* h16;    // fp16 copy (scalar, dim == 128) or nullptr
  const float* nbh;     // ||row||^2 / 2, padded to a multiple of 256 rows with 1e30f
  const float* nrm;     // ||row||^2
  const __half* aug16;  // m_pad x 16: [b0, l0, l1, -0.5, -1, -2048, 0...] with ||row||^2/2 = 0.5*b0 + l0 + 2048*l1; pad rows [0, 0, 2047, ...]
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
};
enum : uint32_t { PM_TC = 0, PM_EXACT_F32 = 1, PM_EXACT_U8 = 2, PM_HAMMING = 3, PM_SKIP = 4,
                  PM_TC_FUSED = 5 /* tensor-core pair whose kernel also ran the exactness pass: candidates are final */,
                  PM_GENERIC_F32 = 6, PM_GENERIC_U8 = 7 /* scalar descriptors whose length is not 128 (AKAZE float 64, LIOP 144): one warp per query */,
                  PM_TC_REAL = 8 /* real-valued fp32 pair on the tensor-core FILTER kernel (l2_tc.cuh MODE_REAL): its candidates are made final by
                                    the exact re-scoring (in-kernel or rescore_real_kernel) and the exact_rows fallback before they are packed */ };

// Work item of the tensor-core kernel: 128 or 256 (per launch) consecutive queries of pair `pair` against the whole database image.
struct WorkItem { uint32_t pair, qtile; };

// Candidate produced by a search kernel, one per query that passed the (pre-)ratio test.
//   PM_TC:   a = query row, b = 16-row chunk id of the best database row, d1 exact, d2 = upper bound (exactness pass needed)
//   others:  a = query row, b = database row of the nearest neighbour, d1/d2 exact (float bits, or uint32 bits for Hamming)
//   PM_TC_REAL (before re-scoring): q = query row, b / d1 / d2 = bit patterns p1 / p2 / p3 of the three smallest packed chunk minima
//            (value with the chunk id in the low REAL_IDBITS bits), p4 in the parallel `candx` word
struct Cand { uint32_t q, b; float d1, d2; };

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

// K2 — per-view preparation at upload time (runs once per image, not on the pair hot path):
// fp16 copy of the 128-D descriptors for the tensor-core kernels, squared row norms, the half-norm limbs that fold the
// norms into the distance GEMM, the per-row / per-view rounding-error bounds of the real-valued path, and the exactness
// flags that decide which tensor-core path (if any) a view may take (see common.cuh VF_*).
#pragma once
#include "common.cuh"

namespace b200m {

// Limbs of x = ||row||^2 / 2 as three fp16 numbers with  x = 0.5*b0 + l0 + 2048*l1:
//  * integer-valued rows (||row||^2 an integer < 2^22): b0 = parity bit, l0 < 2048 integer, l1 < 2048 -> EXACT;
//  * real-valued rows (norms computed from the fp16-ROUNDED components): l1 = floor(x/2048) exact, l0 = fp16(rest) (error <= 0.5),
//    b0 = fp16(2*(rest - l0)) -> residual <= 2^-12: far below the accumulation slack the real-valued path budgets for.
__device__ __forceinline__ void halfnorm_limbs(float s, bool integer_valued, float& b0, float& l0, float& l1) {
  if (integer_valued) {
    b0 = fmodf(s, 2.f);
    const float rest = (s - b0) * 0.5f;
    l1 = floorf(rest * (1.f / 2048.f));
    l0 = rest - 2048.f * l1;
  } else {
    const float x = 0.5f * s;
    l1 = floorf(x * (1.f / 2048.f));
    const float rest = x - 2048.f * l1;                  // exact: x < 2^22, a multiple of 2^-? well inside fp32 after the subtraction
    l0 = __half2float(__float2half_rn(rest));
    b0 = 2.f * (rest - l0);
  }
  l1 = fminf(l1, 2047.f);
}

// One warp per row; lane handles components lane, lane+32, lane+64, lane+96.
//   h16   m x 128 fp16 (rounded to nearest)
//   nrm   ||fp16(row)||^2 (== ||row||^2 for integer-valued rows), nbh = half of it (pad rows 1e30)
//   aug16 m_pad x 16, the row as DATABASE (B operand):  [b0, l0, l1, -0.5, -1, -2048, 0...]   pad rows [0, 0, 4096, ...]
//   augq16 m_pad x 16, the row as QUERY (A operand):    [-0.5, -1, -2048, b0, l0, l1, 0...]
//         With B negated by the instruction descriptor the 9th K-step adds  +nb/2 (cols 0-2)  and, in the real-valued kernel whose
//         A tile is augq16,  +na/2 (cols 3-5): the accumulator is ||a-b||^2 / 2.  The integer kernel's constant A tile has zeros in
//         cols 3-5, so the extra database columns cost it nothing.
//   err   ||row - fp16(row)||_2 inflated by 2^-9 (upper bound of the rounding error norm), 0 for integer-valued rows
//   stats [0] = max err over the view, [1] = max nrm  (float bits, atomicMax on the non-negative patterns)
//   nb32  (uchar-stored views, else nullptr) m_pad x int32 ||row||^2 + U8_NORM_BIAS for the u8 kernel; pad rows 2^24 + U8_NORM_BIAS (see below)
//   limb8 (uchar-stored views, else nullptr) m_pad x 32 u8 norm limbs of the norm-GEMM kernel (common.cuh u8_limb); pad rows all 255, and the
//         flags VF_U8_WIDE / VF_U8_NORMCAP that gate it
template <typename T>
__global__ void __launch_bounds__(256)
prep_view_kernel(const T* __restrict__ raw, int m, __half* __restrict__ h16, float* __restrict__ nbh, float* __restrict__ nrm,
                 int m_pad, uint32_t* __restrict__ flags, __half* __restrict__ aug16, __half* __restrict__ augq16,
                 float* __restrict__ err, uint32_t* __restrict__ stats, int32_t* __restrict__ nb32,
                 uint8_t* __restrict__ limb8) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= m_pad) return;
  const float cst = lane == 0 ? -0.5f : lane == 1 ? -1.f : lane == 2 ? -2048.f : 0.f;     // the constant limb multipliers
  if (row >= m) {
    // pad rows (zero in h16): their AUG accumulator is 2048 * 4096 = 2^23 (+ ||a||^2/2 in MODE_REAL), exact in fp16 and fp32 and above
    // every real row's: h = ||b||^2/2 - a.b < 2^21 + 2^22 for signed rows inside the domain, and ||a - b||^2/2 < 2^21 + 2^22 + ||a||^2/2.
    // So a chunk of padding never wins and never ties with another; it is the second chunk minimum only when m <= 16, and then the
    // exactness pass re-scores the one real chunk.  (A pad half-norm below 2^21 + 2^22 lost to anti-correlated queries.)
    // The u8 kernel's pad rows (zero-filled by TMA, a.b = 0) get s = ||b||^2 - 2 a.b = 2^24 and h = s/2 = 2^23: the same value as here.
    if (lane == 0) { nbh[row] = 1e30f; err[row] = 0.f; if (nb32) nb32[row] = (1 << 24) + U8_NORM_BIAS; }
    if (limb8) limb8[(size_t)row * 32 + lane] = 255;     // U8_LIMB_PAD: above every real row's norm, so s = U8_LIMB_PAD - 0 never wins
    if (lane < 16) {
      aug16[(size_t)row * 16 + lane] = __float2half_rn(lane == 2 ? 4096.f : (lane >= 3 && lane < 6) ? (lane == 3 ? -0.5f : lane == 4 ? -1.f : -2048.f) : 0.f);
      augq16[(size_t)row * 16 + lane] = __float2half_rn(cst);
    }
    return;
  }
  float s = 0.f, e2 = 0.f; uint32_t f = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float v = (float)raw[(size_t)row * 128 + lane + 32 * k];
    if (v != rintf(v)) f |= VF_NONINTEGER;
    if (!(fabsf(v) <= 1024.f)) f |= VF_RANGE;
    if (limb8 && v > 127.f) f |= VF_U8_WIDE;
    const __half hv = __float2half_rn(v);
    h16[(size_t)row * 128 + lane + 32 * k] = hv;
    const float r = __half2float(hv);
    s = fmaf(r, r, s);                      // norm of the ROUNDED row: what the GEMM sees (identical to the row itself when integer-valued)
    const float d = v - r;
    e2 = fmaf(d, d, e2);
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o); e2 += __shfl_xor_sync(0xffffffffu, e2, o); f |= __shfl_xor_sync(0xffffffffu, f, o);
  }
  if (!(s < 4194304.f)) f |= VF_NORM;
  if (limb8) {
    if (s > (float)U8_LIMB_CAP) f |= VF_U8_NORMCAP;     // s is an exact integer here (uchar rows)
    limb8[(size_t)row * 32 + lane] = (uint8_t)u8_limb((int32_t)s, lane);
  }
  const float er = (f & VF_NONINTEGER) ? sqrtf(e2) * (1.f + 1.f / 512.f) + 1e-30f : 0.f;
  if (lane == 0) {
    nrm[row] = s;
    nbh[row] = 0.5f * s;
    err[row] = er;
    if (nb32) nb32[row] = (int32_t)s + U8_NORM_BIAS;       // exact: at most 128 * 255^2 < 2^24
    if (f) atomicOr(flags, f);
    atomicMax(&stats[0], __float_as_uint(er));
    atomicMax(&stats[1], __float_as_uint(s));
  }
  float b0, l0, l1;
  halfnorm_limbs(s, (f & VF_NONINTEGER) == 0, b0, l0, l1);
  if (lane < 16) {
    const float limb = lane == 0 ? b0 : lane == 1 ? l0 : lane == 2 ? l1 : 0.f;
    const float limbq = lane == 3 ? b0 : lane == 4 ? l0 : lane == 5 ? l1 : 0.f;
    aug16[(size_t)row * 16 + lane] = __float2half_rn(lane < 3 ? limb : (lane == 3 ? -0.5f : lane == 4 ? -1.f : lane == 5 ? -2048.f : 0.f));
    augq16[(size_t)row * 16 + lane] = __float2half_rn(lane < 3 ? cst : limbq);
  }
}

}  // namespace b200m

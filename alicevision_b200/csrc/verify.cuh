// Exactness pass + packing of the per-pair candidate lists into one contiguous record array.
//
// For tensor-core pairs (PM_TC) a candidate carries the exact best distance d1, the 16-row chunk of the
// database image that contains the best row, and an UPPER BOUND of the second-best distance (second
// smallest chunk minimum).  One warp re-scores the 16 rows of that chunk against the query with exact
// arithmetic (integer-valued fp16 data, fp32 accumulation of integers < 2^24), which yields
//   * the index of the nearest neighbour (first minimum inside the chunk),
//   * the true second-best distance min(bound, second minimum inside the chunk),
// and re-applies the reference's ratio test  d1 < ratio^2 * d2  (matching/filters.hpp:60,
// matching/RegionsMatcher.hpp:150) in float.  A mismatch between the re-scored and the tensor-core d1
// increments `err_count` (it would mean the tensor-core accumulation was not exact).
// For the other modes candidates are already exact and are only moved to their packed position.
#pragma once
#include "common.cuh"

namespace b200m {

constexpr int VERIFY_WARPS_REAL = 8;

// Where the real-valued path parks the queries its error bound could not decide (x = pair of the batch, y = query row, z = the candidate
// slot to write the answer to when w != 0): FB_PER_PAIR slots per pair, which the per-pair fallback kernel consumes with the database image
// read once per group of queries, and a global overflow list for the (pathological) pair that flags more.
constexpr int FB_PER_PAIR = 64;
struct FbSink { uint4* pair_list; int* pair_cnt; uint4* list; int* count; int cap; int* total; };
__device__ __forceinline__ void fb_push(const FbSink& s, uint32_t pair, uint32_t q, uint32_t slot, uint32_t has_slot, unsigned int* err_count) {
  atomicAdd(s.total, 1);
  const int k = atomicAdd(&s.pair_cnt[pair], 1);
  if (k < FB_PER_PAIR) { s.pair_list[(size_t)pair * FB_PER_PAIR + k] = make_uint4(pair, q, slot, has_slot); return; }
  const int g = atomicAdd(s.count, 1);
  if (g < s.cap) s.list[g] = make_uint4(pair, q, slot, has_slot); else atomicAdd(err_count, 1u);
}

// offsets[p] = exclusive prefix sum of cand_count[0..n); offsets[n] = total. Single block.
__global__ void scan_counts_kernel(const int* __restrict__ cand_count, int n, int* __restrict__ offsets) {
  __shared__ int carry;
  __shared__ int wsum[32];
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int base = 0; base < n; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const int v = i < n ? cand_count[i] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int s = lane < nw ? wsum[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
      wsum[lane] = s;
    }
    __syncthreads();
    const int before = carry + (warp ? wsum[warp - 1] : 0) + x - v;
    if (i < n) offsets[i] = before;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry = before + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) offsets[n] = carry;
}

// Warp-level exact re-scoring of one tensor-core candidate (see the header comment). All 32 lanes call it with the same
// candidate; lane l handles row (l & 15) of chunk k.b (chunk_row: ascending in l, so ties go to the smallest database row in either
// layout), components 64*(l >> 4)..+63. Returns (on every lane)
// whether the match survives the ratio test; `rec` is the final record (i = database row, j = query row, d1, d2).
__device__ __forceinline__ bool rescore_candidate(const __half* __restrict__ db16, const __half* __restrict__ q16, uint32_t m_i, const Cand& k,
                                                  bool thread_chunks, float ratio_sq, int lane, unsigned int* __restrict__ err_count, Rec& rec) {
  const int r = lane & 15, hv = lane >> 4;
  const uint32_t row = chunk_row(k.b, r, thread_chunks);
  float acc = INFINITY;
  if (row < m_i) {
    const uint4* a = reinterpret_cast<const uint4*>(q16 + (size_t)k.q * 128 + hv * 64);
    const uint4* b = reinterpret_cast<const uint4*>(db16 + (size_t)row * 128 + hv * 64);
    acc = 0.f;
#pragma unroll
    for (int v = 0; v < 8; ++v) {
      const uint4 x = a[v], y = b[v];
      const __half2* xh = reinterpret_cast<const __half2*>(&x);
      const __half2* yh = reinterpret_cast<const __half2*>(&y);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 fx = __half22float2(xh[e]), fy = __half22float2(yh[e]);
        const float d0 = fx.x - fy.x, d1 = fx.y - fy.y;
        acc = fmaf(d0, d0, acc);
        acc = fmaf(d1, d1, acc);
      }
    }
  }
  const float dist = acc + __shfl_xor_sync(0xffffffffu, acc, 16);      // INF for rows past the end
  float best = dist; int arg = r;                                        // argmin over the 16 rows (ties -> smallest row)
#pragma unroll
  for (int o = 8; o >= 1; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
    if (ob < best || (ob == best && oa < arg)) { best = ob; arg = oa; }
  }
  float second = (r == arg) ? INFINITY : dist;
#pragma unroll
  for (int o = 8; o >= 1; o >>= 1) second = fminf(second, __shfl_xor_sync(0xffffffffu, second, o));
  if (lane == 0 && best != k.d1) atomicAdd(err_count, 1u);             // tensor-core accumulation was not exact
  const float d2 = fminf(k.d2, second);
  rec = Rec{chunk_row(k.b, arg, thread_chunks), k.q, best, d2};
  return best < __fmul_rn(ratio_sq, d2);                                // matching/filters.hpp:60
}

// ------------------------------------------------------------------------------------------------ real-valued fp32 path
// The reference's L2_Vectorized<float> (feature/metric.hpp:94-123): four SSE lanes, lane l accumulates s_l += (a-b)*(a-b) over
// components l, l+4, ... with a separate multiply and add, result ((s0+s1)+s2)+s3.  One thread, one (query, database row) pair.
// Rows are read in their storage type (integer-valued fp32 views are stored as uchar: same values).
__device__ __forceinline__ float ref_l2_sse(const ViewDev& vq, uint32_t q, const ViewDev& vd, uint32_t row) {
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  if (vq.dtype == DT_F32 && vd.dtype == DT_F32) {
    const float4* a = reinterpret_cast<const float4*>(vq.raw) + (size_t)q * 32;      // same address on every lane of a warp re-scoring one query
    const float4* b = reinterpret_cast<const float4*>(vd.raw) + (size_t)row * 32;
#pragma unroll 8
    for (int t = 0; t < 32; ++t) {
      const float4 x = __ldg(a + t), y = __ldg(b + t);
      float d;
      d = __fsub_rn(x.x, y.x); s0 = __fadd_rn(s0, __fmul_rn(d, d));
      d = __fsub_rn(x.y, y.y); s1 = __fadd_rn(s1, __fmul_rn(d, d));
      d = __fsub_rn(x.z, y.z); s2 = __fadd_rn(s2, __fmul_rn(d, d));
      d = __fsub_rn(x.w, y.w); s3 = __fadd_rn(s3, __fmul_rn(d, d));
    }
  } else {
#pragma unroll 4
    for (int t = 0; t < 32; ++t) {
      float d;
      d = __fsub_rn(view_elem(vq, (size_t)q * 128 + 4 * t + 0), view_elem(vd, (size_t)row * 128 + 4 * t + 0)); s0 = __fadd_rn(s0, __fmul_rn(d, d));
      d = __fsub_rn(view_elem(vq, (size_t)q * 128 + 4 * t + 1), view_elem(vd, (size_t)row * 128 + 4 * t + 1)); s1 = __fadd_rn(s1, __fmul_rn(d, d));
      d = __fsub_rn(view_elem(vq, (size_t)q * 128 + 4 * t + 2), view_elem(vd, (size_t)row * 128 + 4 * t + 2)); s2 = __fadd_rn(s2, __fmul_rn(d, d));
      d = __fsub_rn(view_elem(vq, (size_t)q * 128 + 4 * t + 3), view_elem(vd, (size_t)row * 128 + 4 * t + 3)); s3 = __fadd_rn(s3, __fmul_rn(d, d));
    }
  }
  return __fadd_rn(__fadd_rn(__fadd_rn(s0, s1), s2), s3);
}

// What the fp16 rounding and the fp32 tensor-core accumulation can do to a distance, per (query row, database view):
//   d~ = ||a~ - b~||^2 as the filter kernel sees it, d = the reference's float distance of the original rows.
//   * rounding:      | sqrt(d_exact) - ||a~ - b~|| | <= ||a - a~|| + ||b - b~|| <= eta = err[q] + max err of the database view
//   * accumulation:  | d~ - ||a~ - b~||^2 | <= sigma: 144 products + limb terms summed in fp32 by the tensor core (each partial result within a
//                    few ulp of the running magnitude <= S = (||a~||^2 + max||b~||^2)/2 + ||a~|| max||b~||) and the limb residuals (<= 2^-22
//                    relative per half-norm); budgeted generously as 2^-14 * S on d~ - scale-invariant, like everything else here  (checked on
//                    the device: every re-scored best row must land inside [lower(p1), upper(p1)], `err_count` otherwise)
//   * the reference's own float summation: relative 2^-17 (33 roundings of 2^-24 on positive terms)
//   * the chunk id in the low REAL_IDBITS mantissa bits: the packed value is <= the true one and at most 2^-(23-REAL_IDBITS) below it
struct RealBound {
  float eta, sigma;
  __device__ __forceinline__ float lower(float dt) const {          // every reference distance whose filter value is >= dt is >= lower(dt)
    const float r = fmaxf(sqrtf(fmaxf(dt - sigma, 0.f)) - eta, 0.f);
    return r * r * (1.f - 1.f / 65536.f);
  }
  __device__ __forceinline__ float upper(float dt) const {          // ... whose (packed) filter value is dt is <= upper(dt)
    const float r = sqrtf(dt * (1.f + 1.f / 512.f) + sigma) + eta;
    return r * r * (1.f + 1.f / 65536.f);
  }
};
__device__ __forceinline__ RealBound real_bound(const ViewDev& vi, const ViewDev& vj, uint32_t q) {
  const float emax = __uint_as_float(vi.stats[0]), nmax = __uint_as_float(vi.stats[1]);
  const float na = vj.nrm[q];
  RealBound b;
  b.eta = (vj.err[q] + emax) * (1.f + 1.f / 1024.f);
  const float S = 0.5f * (na + nmax) + sqrtf(na * nmax);
  b.sigma = S * (1.f / 16384.f);
  return b;
}

// Warp-level exact re-scoring of one real-valued candidate: k.q = query row, k.b / k.d1 / k.d2 / p4 = the four smallest packed chunk minima
// (ids in the low bits).  Lane l re-scores row 16*id1 + l (l < 16) or 16*id2 + (l - 16) in the reference's arithmetic; if the third
// chunk minimum cannot be excluded its 16 rows follow; if the fourth cannot either the query is left to the exact_rows fallback.
// Returns (on every lane) 0 = fails the ratio test, 1 = final match in `rec`, 2 = undecided.
__device__ __forceinline__ int rescore_real(const ViewDev& vi, const ViewDev& vj, uint32_t m_i, const Cand& k, uint32_t p4, float ratio_sq, int lane,
                                            unsigned int* __restrict__ err_count, Rec& rec) {
  const uint32_t p1 = k.b, p2 = __float_as_uint(k.d1), p3 = __float_as_uint(k.d2);
  const RealBound rb = real_bound(vi, vj, k.q);
  const int r = lane & 15;
  uint32_t row = ((lane < 16 ? p1 : p2) & REAL_IDMASK) * 16 + r;
  float dist = row < m_i ? ref_l2_sse(vj, k.q, vi, row) : INFINITY;
  // bound self-check: the best row of the best chunk must lie inside the interval its packed minimum promises
  {
    float c1 = lane < 16 ? dist : INFINITY;
#pragma unroll
    for (int o = 8; o >= 1; o >>= 1) c1 = fminf(c1, __shfl_xor_sync(0xffffffffu, c1, o));
    const float d1t = 2.f * __uint_as_float(p1 & ~REAL_IDMASK);
    if (lane == 0 && !(rb.lower(d1t) <= c1 && c1 <= rb.upper(d1t))) atomicAdd(err_count, 1u);
  }
  float best = dist; uint32_t arg = row;
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const uint32_t oa = __shfl_xor_sync(0xffffffffu, arg, o);
    if (ob < best || (ob == best && oa < arg)) { best = ob; arg = oa; }
  }
  float second = (row == arg) ? INFINITY : dist;
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) second = fminf(second, __shfl_xor_sync(0xffffffffu, second, o));
  if (!(rb.lower(2.f * __uint_as_float(p3 & ~REAL_IDMASK)) >= second)) {
    // the third chunk may hold a row closer than the second best so far: re-score it as well
    row = (p3 & REAL_IDMASK) * 16 + r;
    dist = (lane < 16 && row < m_i) ? ref_l2_sse(vj, k.q, vi, row) : INFINITY;
    float b3 = dist; uint32_t a3 = row;
#pragma unroll
    for (int o = 8; o >= 1; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, b3, o);
      const uint32_t oa = __shfl_xor_sync(0xffffffffu, a3, o);
      if (ob < b3 || (ob == b3 && oa < a3)) { b3 = ob; a3 = oa; }
    }
    float s3 = (row == a3) ? INFINITY : dist;
#pragma unroll
    for (int o = 8; o >= 1; o >>= 1) s3 = fminf(s3, __shfl_xor_sync(0xffffffffu, s3, o));
    b3 = __shfl_sync(0xffffffffu, b3, 0); a3 = __shfl_sync(0xffffffffu, a3, 0); s3 = __shfl_sync(0xffffffffu, s3, 0);
    if (b3 < best || (b3 == best && a3 < arg)) { second = fminf(best, s3); best = b3; arg = a3; }
    else second = fminf(second, b3);
    if (!(rb.lower(2.f * __uint_as_float(p4 & ~REAL_IDMASK)) >= second)) return 2;
  }
  rec = Rec{arg, k.q, best, second};
  return best < __fmul_rn(ratio_sq, second) ? 1 : 0;                     // matching/filters.hpp:60
}

// Un-fused real-valued pairs (short database images): the filter kernel left its candidates in global memory; re-score them IN PLACE
// (a final candidate {q, row, d1, d2}, or b = 0xFFFFFFFF = dropped, which the packing kernel turns into the dropped-record marker).
__global__ void __launch_bounds__(VERIFY_WARPS_REAL * 32)
rescore_real_kernel(const ViewDev* __restrict__ views, const PairDev* __restrict__ pairs, Cand* __restrict__ cands, const uint32_t* __restrict__ candx,
                    const int* __restrict__ cand_count, float ratio_sq, unsigned int* __restrict__ err_count, FbSink fb) {
  const PairDev p = pairs[blockIdx.x];
  if (p.mode != PM_TC_REAL) return;
  const int n = cand_count[blockIdx.x];
  const int lane = threadIdx.x & 31;
  const int wid = blockIdx.y * VERIFY_WARPS_REAL + (threadIdx.x >> 5);
  const int nwarps = gridDim.y * VERIFY_WARPS_REAL;
  Cand* src = cands + p.cand_base;
  for (int c = wid; c < n; c += nwarps) {
    const Cand k = src[c];
    Rec rec;
    const int verdict = rescore_real(views[p.view_i], views[p.view_j], p.m_i, k, candx[p.cand_base + c], ratio_sq, lane, err_count, rec);
    if (lane == 0) {
      src[c] = verdict == 1 ? Cand{rec.j, rec.i, rec.d1, rec.d2} : Cand{k.q, 0xFFFFFFFFu, 0.f, 0.f};
      // the fallback writes its answer into THIS slot (the pair's candidate region has no room to append: a self pair fills every slot)
      if (verdict == 2) fb_push(fb, blockIdx.x, k.q, (uint32_t)c, 1u, err_count);
    }
  }
}

// Fallback of the real-valued path, per pair: the flagged queries of one pair (a few; FB_PER_PAIR at most here) against the whole database
// image in the reference's arithmetic.  One block per (pair, group of XP_MAXQ queries); the database rows stream through shared memory in coalesced 64-row tiles
// (read once per group); thread (r, l) owns SSE lane l of tile row r: s_l += (q - row)^2 over components l, l+4, ...
// in order, the four lanes of a row combined as ((s0+s1)+s2)+s3 (feature/metric.hpp:100-116).
constexpr int XP_THREADS = 256, XP_ROWS = 64, XP_LD = 132, XP_MAXQ = 4;   // 4 queries per block: their components live in REGISTERS (with 8
// queries in shared memory the inner loop was LDS-bound; with 2 the database image was re-read too often: 26.8 % of the device time of the
// real-valued bench).  The tiles are double-buffered with cp.async so that a block streams its 4 MB image without stalling on every tile.
constexpr int XP_TILE_BYTES = XP_ROWS * XP_LD * 4;
constexpr int XP_SMEM = 2 * XP_TILE_BYTES;
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
  const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
  const int n = valid ? 16 : 0;                                   // src-size 0: the 16 bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__global__ void __launch_bounds__(XP_THREADS)
exact_rows_pairs_kernel(const ViewDev* __restrict__ views, const PairDev* __restrict__ pairs, const uint4* __restrict__ pair_list, const int* __restrict__ pair_cnt,
                        Cand* __restrict__ cands, int* __restrict__ cand_count, float ratio_sq) {
  const PairDev p = pairs[blockIdx.x];
  if (p.mode != PM_TC_REAL) return;
  const int n_all = min(pair_cnt[blockIdx.x], FB_PER_PAIR);
  const int e0 = blockIdx.y * XP_MAXQ;                      // grid.y = FB_PER_PAIR / XP_MAXQ: one block per group of XP_MAXQ flagged queries of the pair
  if (e0 >= n_all) return;
  const int ne = min(XP_MAXQ, n_all - e0);
  extern __shared__ __align__(16) float xp_tiles[];         // 2 x [XP_ROWS][XP_LD]
  __shared__ float qs[XP_MAXQ * 128];
  __shared__ float rm1[XP_MAXQ][XP_THREADS / 32], rm2[XP_MAXQ][XP_THREADS / 32];
  __shared__ uint32_t ri1[XP_MAXQ][XP_THREADS / 32];
  const ViewDev& vi = views[p.view_i]; const ViewDev& vj = views[p.view_j];
  const int tid = threadIdx.x, r = tid >> 2, l = tid & 3, lane = tid & 31, warp = tid >> 5;
  const unsigned gmask = 0xFu << (lane & ~3);
  for (int k = tid; k < XP_MAXQ * 128; k += XP_THREADS)
    qs[k] = (k >> 7) < ne ? view_elem(vj, (size_t)pair_list[(size_t)blockIdx.x * FB_PER_PAIR + e0 + (k >> 7)].y * 128 + (k & 127)) : 0.f;
  __syncthreads();
  float qr[XP_MAXQ][32];                                    // this thread's SSE lane of every query: components l, l + 4, ...
#pragma unroll
  for (int e = 0; e < XP_MAXQ; ++e)
#pragma unroll
    for (int t = 0; t < 32; ++t) qr[e][t] = qs[e * 128 + 4 * t + l];
  float m1[XP_MAXQ], m2[XP_MAXQ]; uint32_t i1[XP_MAXQ];
#pragma unroll
  for (int e = 0; e < XP_MAXQ; ++e) { m1[e] = INFINITY; m2[e] = INFINITY; i1[e] = 0xFFFFFFFFu; }

  const bool f32 = vi.dtype == DT_F32;                      // fp32 rows: asynchronous 16-byte copies; uchar-stored rows (integer-valued view of a
  const int ntile = ((int)p.m_i + XP_ROWS - 1) / XP_ROWS;   // mixed pair): converted on a synchronous load
  auto load_tile = [&](int t, int buf) {
    float* tile = xp_tiles + buf * (XP_ROWS * XP_LD);
    const uint32_t row0 = (uint32_t)t * XP_ROWS;
    for (int k = tid; k < XP_ROWS * 32; k += XP_THREADS) {  // 64 rows x 32 chunks of 16 B, coalesced
      const int rr = k >> 5, c4 = k & 31;
      const bool valid = row0 + rr < p.m_i;
      if (f32) {
        cp_async16(&tile[rr * XP_LD + c4 * 4], reinterpret_cast<const float4*>(vi.raw) + (valid ? ((size_t)(row0 + rr) * 32 + c4) : 0), valid);
      } else {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (valid) { const size_t base = (size_t)(row0 + rr) * 128 + c4 * 4; v = make_float4(view_elem(vi, base), view_elem(vi, base + 1), view_elem(vi, base + 2), view_elem(vi, base + 3)); }
        *reinterpret_cast<float4*>(&tile[rr * XP_LD + c4 * 4]) = v;
      }
    }
    cp_async_commit();
  };
  load_tile(0, 0);
  for (int t = 0; t < ntile; ++t) {
    if (t + 1 < ntile) { load_tile(t + 1, (t + 1) & 1); cp_async_wait<1>(); } else cp_async_wait<0>();
    __syncthreads();                                        // tile t is complete for every thread
    const float* tile = xp_tiles + (t & 1) * (XP_ROWS * XP_LD);
    float s[XP_MAXQ];
#pragma unroll
    for (int e = 0; e < XP_MAXQ; ++e) s[e] = 0.f;
#pragma unroll
    for (int tt = 0; tt < 32; ++tt) {
      const float tv = tile[r * XP_LD + 4 * tt + l];
#pragma unroll
      for (int e = 0; e < XP_MAXQ; ++e) { const float d = __fsub_rn(qr[e][tt], tv); s[e] = __fadd_rn(s[e], __fmul_rn(d, d)); }   // an unused query slot holds zeros
    }
    const uint32_t row = (uint32_t)t * XP_ROWS + r;
#pragma unroll
    for (int e = 0; e < XP_MAXQ; ++e) {
      const float s1 = __shfl_xor_sync(gmask, s[e], 1);
      const float pr = (l & 1) ? __fadd_rn(s1, s[e]) : __fadd_rn(s[e], s1);          // s0+s1 on lanes 0,1 ; s2+s3 on lanes 2,3
      const float s01 = __shfl_sync(gmask, pr, 0, 4);
      const float s2 = __shfl_sync(gmask, s[e], 2, 4), s3 = __shfl_sync(gmask, s[e], 3, 4);
      const float d = __fadd_rn(__fadd_rn(s01, s2), s3);
      if (l == 0 && row < p.m_i) {
        if (d < m1[e] || (d == m1[e] && row < i1[e])) { m2[e] = m1[e]; m1[e] = d; i1[e] = row; } else m2[e] = fminf(m2[e], d);
      }
    }
    __syncthreads();                                        // everyone is done with buffer t & 1 before tile t + 2 lands in it
  }
  // reduce the per-thread top-2 (held by the l == 0 threads) over the block
#pragma unroll
  for (int e = 0; e < XP_MAXQ; ++e) {
    float a1 = m1[e], a2 = m2[e]; uint32_t ai = i1[e];
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
      const float o1 = __shfl_xor_sync(0xffffffffu, a1, o), o2 = __shfl_xor_sync(0xffffffffu, a2, o);
      const uint32_t oi = __shfl_xor_sync(0xffffffffu, ai, o);
      if (o1 < a1 || (o1 == a1 && oi < ai)) { a2 = fminf(a1, o2); a1 = o1; ai = oi; } else a2 = fminf(a2, o1);
    }
    if (lane == 0) { rm1[e][warp] = a1; rm2[e][warp] = a2; ri1[e][warp] = ai; }
  }
  __syncthreads();
  if (tid < ne) {
    float a1 = rm1[tid][0], a2 = rm2[tid][0]; uint32_t ai = ri1[tid][0];
    for (int w2 = 1; w2 < XP_THREADS / 32; ++w2) {
      const float o1 = rm1[tid][w2], o2 = rm2[tid][w2]; const uint32_t oi = ri1[tid][w2];
      if (o1 < a1 || (o1 == a1 && oi < ai)) { a2 = fminf(a1, o2); a1 = o1; ai = oi; } else a2 = fminf(a2, o1);
    }
    const uint4 ent = pair_list[(size_t)blockIdx.x * FB_PER_PAIR + e0 + tid];
    if (a1 < __fmul_rn(ratio_sq, a2)) {                                // matching/filters.hpp:60
      const int slot = ent.w ? (int)ent.z : atomicAdd(&cand_count[blockIdx.x], 1);
      cands[p.cand_base + slot] = Cand{ent.y, ai, a1, a2};
    }
  }
}

// The same for the overflow list (a pair that flagged more than FB_PER_PAIR queries): the queries whose top-2 the bound could not decide get the exact search over the WHOLE
// database image in the reference's arithmetic.  One block per list entry (grid-stride), thread t scans rows t, t + 256, ...;
// the survivor of the ratio test goes to the entry's own candidate slot (stand-alone re-scoring: ent.w = 1, slot ent.z holds the
// "dropped" marker until then) or is appended to the pair's final candidates (in-kernel re-scoring: only final candidates were emitted).
constexpr int XR_THREADS = 256;
__global__ void __launch_bounds__(XR_THREADS)
exact_rows_kernel(const ViewDev* __restrict__ views, const PairDev* __restrict__ pairs, const uint4* __restrict__ fb_list, const int* __restrict__ fb_count,
                  int fb_cap, Cand* __restrict__ cands, int* __restrict__ cand_count, float ratio_sq) {
  __shared__ float sv[XR_THREADS / 32][2]; __shared__ uint32_t si[XR_THREADS / 32];
  const int n = min(*fb_count, fb_cap);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int e = blockIdx.x; e < n; e += gridDim.x) {
    const uint4 ent = fb_list[e];
    const PairDev p = pairs[ent.x];
    const ViewDev& vi = views[p.view_i]; const ViewDev& vj = views[p.view_j];
    float m1 = INFINITY, m2 = INFINITY; uint32_t i1 = 0xFFFFFFFFu;
    for (uint32_t row = threadIdx.x; row < p.m_i; row += XR_THREADS) {
      const float d = ref_l2_sse(vj, ent.y, vi, row);
      if (d < m1 || (d == m1 && row < i1)) { m2 = m1; m1 = d; i1 = row; } else m2 = fminf(m2, d);
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
      const float o1 = __shfl_xor_sync(0xffffffffu, m1, o), o2 = __shfl_xor_sync(0xffffffffu, m2, o);
      const uint32_t oi = __shfl_xor_sync(0xffffffffu, i1, o);
      if (o1 < m1 || (o1 == m1 && oi < i1)) { m2 = fminf(m1, o2); m1 = o1; i1 = oi; } else m2 = fminf(m2, o1);
    }
    __syncthreads();                                   // previous entry's shared values consumed
    if (lane == 0) { sv[warp][0] = m1; sv[warp][1] = m2; si[warp] = i1; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w2 = 1; w2 < XR_THREADS / 32; ++w2) {
        const float o1 = sv[w2][0], o2 = sv[w2][1]; const uint32_t oi = si[w2];
        if (o1 < m1 || (o1 == m1 && oi < i1)) { m2 = fminf(m1, o2); m1 = o1; i1 = oi; } else m2 = fminf(m2, o1);
      }
      if (m1 < __fmul_rn(ratio_sq, m2)) {                               // matching/filters.hpp:60
        const int slot = ent.w ? (int)ent.z : atomicAdd(&cand_count[ent.x], 1);
        cands[p.cand_base + slot] = Cand{ent.y, i1, m1, m2};
      }
    }
  }
}

// ArrayMatcher surface (MODE_KNN of the tensor-core kernel): one warp per query turns its two chunks into the two nearest rows.
// Lanes 0-15 re-score the rows of the best chunk, lanes 16-31 those of the chunk with the second smallest minimum (integer-valued
// fp16 data, exact fp32 sums); the two smallest (distance, row) of the 32 are the query's neighbours, ascending.
__global__ void __launch_bounds__(256)
knn_finalize_kernel(const ViewDev* __restrict__ views, const PairDev* __restrict__ pairs, const Cand* __restrict__ cands, int32_t* __restrict__ idx,
                    float* __restrict__ dist, unsigned int* __restrict__ err_count) {
  const PairDev p = pairs[0];
  const int q = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= (int)p.m_j) return;
  const Cand k = cands[p.cand_base + q];
  const uint32_t chunk = lane < 16 ? (k.b & 0xFFFFu) : (k.b >> 16);
  const uint32_t row = chunk * 16 + (lane & 15);
  float acc = INFINITY;
  if (chunk != 0xFFFFu && row < p.m_i) {
    const uint4* a = reinterpret_cast<const uint4*>(views[p.view_j].h16 + (size_t)q * 128);
    const uint4* b = reinterpret_cast<const uint4*>(views[p.view_i].h16 + (size_t)row * 128);
    acc = 0.f;
#pragma unroll 4
    for (int v = 0; v < 16; ++v) {
      const uint4 x = a[v], y = b[v];
      const __half2* xh = reinterpret_cast<const __half2*>(&x);
      const __half2* yh = reinterpret_cast<const __half2*>(&y);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 fx = __half22float2(xh[e]), fy = __half22float2(yh[e]);
        const float d0 = fx.x - fy.x, d1 = fx.y - fy.y;
        acc = fmaf(d0, d0, acc);
        acc = fmaf(d1, d1, acc);
      }
    }
  }
  float b1 = acc; uint32_t a1 = row;
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, b1, o); const uint32_t oa = __shfl_xor_sync(0xffffffffu, a1, o);
    if (ob < b1 || (ob == b1 && oa < a1)) { b1 = ob; a1 = oa; }
  }
  float b2 = (row == a1) ? INFINITY : acc; uint32_t a2 = row;
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, b2, o); const uint32_t oa = __shfl_xor_sync(0xffffffffu, a2, o);
    if (ob < b2 || (ob == b2 && oa < a2)) { b2 = ob; a2 = oa; }
  }
  if (lane == 0) {
    if (b1 != k.d1 || b2 > k.d2) atomicAdd(err_count, 1u);            // the tensor-core values are exact on this path (k.d2: second smallest CHUNK minimum)
    idx[2 * q] = (int32_t)a1; idx[2 * q + 1] = (int32_t)a2;
    dist[2 * q] = b1; dist[2 * q + 1] = b2;
  }
}

constexpr int VERIFY_BLOCKS_PER_PAIR = 4;
constexpr int VERIFY_WARPS = 8;

__global__ void __launch_bounds__(VERIFY_WARPS * 32)
verify_pack_kernel(const ViewDev* __restrict__ views, const PairDev* __restrict__ pairs, const Cand* __restrict__ cands,
                   const int* __restrict__ cand_count, const int* __restrict__ offsets, Rec* __restrict__ out, float ratio_sq,
                   unsigned int* __restrict__ err_count) {
  const PairDev p = pairs[blockIdx.x];
  const int n = cand_count[blockIdx.x];
  const int lane = threadIdx.x & 31;
  const int wid = blockIdx.y * VERIFY_WARPS + (threadIdx.x >> 5);
  const int nwarps = gridDim.y * VERIFY_WARPS;
  const Cand* src = cands + p.cand_base;
  Rec* dst = out + offsets[blockIdx.x];
  if (p.mode != PM_TC) {      // exact / Hamming pairs, and tensor-core pairs whose candidates were already re-scored in-kernel
    for (int c = wid * 32 + lane; c < n; c += nwarps * 32) {
      const Cand k = src[c];
      dst[c] = Rec{k.b, k.q, k.d1, k.d2};
    }
    return;
  }
  const ViewDev& vi = views[p.view_i];
  const ViewDev& vj = views[p.view_j];
  for (int c = wid; c < n; c += nwarps) {
    const Cand k = src[c];
    Rec rec;
    const bool keep = rescore_candidate(vi.h16, vj.h16, p.m_i, k, p.thread_chunks != 0, ratio_sq, lane, err_count, rec);
    if (lane == 0) dst[c] = keep ? rec : Rec{0xFFFFFFFFu, k.q, rec.d1, rec.d2};
  }
}

}  // namespace b200m

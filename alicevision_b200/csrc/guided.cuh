// K7 — guided matching: descriptor top-2 + ratio test restricted to the correspondences that agree with a fundamental
// matrix (SURVEY 8f rank 4).  Replaces matching::guidedMatching<Mat3Model, FundamentalEpipolarDistanceError>(model, camL,
// lRegions, camR, rRegions, errorTh, distRatio, matches) for cameras without distortion (matching/guidedMatching.hpp:206-268)
// with the error of multiview/relativePose/FundamentalError.hpp:52-64 and the accumulator matching/guidedMatching.hpp:77-118.
//
// The geometric predicate passes ~0.1-1 % of the (left, right) pairs (a band of +-sqrt(errorTh) pixels around the epipolar
// line), so this is not tensor-core work: the O(M_l x M_r) part is ~12 double-precision operations per pair (done exactly as
// the reference does them: separate multiply / add / divide, no contraction), and only the survivors pay for a 128-D
// descriptor distance, computed with the reference's own summation order so that distances, hence the ratio test, are
// bit-identical (float: feature/metric.hpp:94-123 four sequential lanes, ((s0+s1)+s2)+s3; uchar: exact integers;
// binary: feature/Hamming.hpp:174-185 squared popcount).
//
// One warp per left feature; the right positions stream through shared memory; survivors are queued per warp and their
// distances evaluated eight at a time (4 lanes per candidate = the 4 SSE lanes).
//
// A whole list of pairs runs per launch (b200m_guided_match_pairs; the one-pair calls are lists of one): the work items are
// (pair, block of GM_WARPS left features), the items of one pair adjacent; per-pair parameters sit in a device table.  Each
// (pair, left i) writes its best j or -1 to a flat slot array, and an exclusive scan of the keep flags places each pair's list in
// ascending i.  There is one record per left feature, so IndMatch::getDeduplicated (guidedMatching.hpp:267) changes nothing.
#pragma once
#include "common.cuh"

#include <cfloat>

namespace b200m {

constexpr int GM_WARPS = 8;          // left features per block
constexpr int GM_TILE = 1024;        // right positions per shared-memory tile
constexpr int GM_QUEUE = 40;         // >= 8 + 32: survivors of one 32-wide step appended to at most 7 waiting ones

enum : int { GM_FUNDAMENTAL = 0, GM_HOMOGRAPHY = 1 };

struct GuidedPair {
  const void* rawl; const void* rawr;           // descriptors (kernel dtype: a uchar-stored view of a mixed pair points at its fp32 expansion)
  const double2* gl; const double2* gr;         // geometry positions, or nullptr: the float upload positions below, widened
  const float2* fl; const float2* fr;
  double M[9];          // row-major model matrix: fundamental (x_right^T F x_left = 0) or homography (x_right ~ H x_left)
  double errorTh;       // Square(precision), guidedMatching.hpp:211 / GeometricFilterMatrix_F_AC.hpp:387
  int model;            // GM_FUNDAMENTAL: FundamentalEpipolarDistanceError; GM_HOMOGRAPHY: HomographyAsymmetricError (HomographyError.hpp:23-31)
  int ml, mr;
  int block_base;       // first block of this pair in the launch (blocks of one pair are adjacent: the right view is reused out of L2)
  int left_base;        // first slot of this pair in the flat per-batch arrays
};

__device__ __forceinline__ double2 guided_pos(const double2* g, const float2* f, int k) {
  if (g) return g[k];
  const float2 v = f[k];
  return make_double2((double)v.x, (double)v.y);
}

// The model applied to left point x, once per left feature.  F_x = F * (x, y, 1), row r = (F(r,0)*x + F(r,1)*y) + F(r,2)*1, and
// nrm = F_x.head<2>().squaredNorm(); for a homography (fx0, fx1) = x2_est = x2h_est.head<2>() / x2h_est[2] (HomographyError.hpp:27-28).
__device__ __forceinline__ void guided_left(const double* M, int model, double2 x, double& fx0, double& fx1, double& fx2, double& nrm) {
  fx0 = __dadd_rn(__dadd_rn(__dmul_rn(M[0], x.x), __dmul_rn(M[1], x.y)), M[2]);
  fx1 = __dadd_rn(__dadd_rn(__dmul_rn(M[3], x.x), __dmul_rn(M[4], x.y)), M[5]);
  fx2 = __dadd_rn(__dadd_rn(__dmul_rn(M[6], x.x), __dmul_rn(M[7], x.y)), M[8]);
  nrm = __dadd_rn(__dmul_rn(fx0, fx0), __dmul_rn(fx1, fx1));
  if (model == GM_HOMOGRAPHY) { fx0 = __ddiv_rn(fx0, fx2); fx1 = __ddiv_rn(fx1, fx2); }
}

// ErrorT::error of right point y against the left point's guided_left values: HomographyAsymmetricError (x2 - x2_est).squaredNorm()
// or FundamentalEpipolarDistanceError Square(F_x.dot((y, 1))) / squaredNorm, separate multiply / add as the reference evaluates them
__device__ __forceinline__ double guided_error(int model, double fx0, double fx1, double fx2, double nrm, double2 y) {
  if (model == GM_HOMOGRAPHY) {
    const double d0 = __dsub_rn(y.x, fx0), d1 = __dsub_rn(y.y, fx1);
    return __dadd_rn(__dmul_rn(d0, d0), __dmul_rn(d1, d1));
  }
  const double dot = __dadd_rn(__dadd_rn(__dmul_rn(fx0, y.x), __dmul_rn(fx1, y.y)), fx2);
  return __ddiv_rn(__dmul_rn(dot, dot), nrm);
}

// distance of candidate descriptors a (left) and b (right) evaluated by the 4 lanes of a group; returns the value on every lane of the group
template <int DTYPE>
__device__ __forceinline__ double guided_distance(const void* __restrict__ left, const void* __restrict__ right, int i, int j, int sub, unsigned gmask) {
  if (DTYPE == DT_BIN) {
    const uint32_t* a = reinterpret_cast<const uint32_t*>(left) + (size_t)i * 16;
    const uint32_t* b = reinterpret_cast<const uint32_t*>(right) + (size_t)j * 16;
    unsigned h = 0;
#pragma unroll
    for (int w = 0; w < 4; ++w) h += __popc(a[sub * 4 + w] ^ b[sub * 4 + w]);
    h += __shfl_xor_sync(gmask, h, 1);
    h += __shfl_xor_sync(gmask, h, 2);
    return (double)(h * h);                                           // SquaredHamming: h * h in unsigned, then double
  }
  float s = 0.f;
  if (DTYPE == DT_F32) {
    const float* a = reinterpret_cast<const float*>(left) + (size_t)i * 128;
    const float* b = reinterpret_cast<const float*>(right) + (size_t)j * 128;
    for (int t = 0; t < 32; ++t) {                                    // SSE lane `sub`: s += (a-b)*(a-b), t ascending (metric.hpp:100-110)
      const float d = __fsub_rn(a[4 * t + sub], b[4 * t + sub]);
      s = __fadd_rn(s, __fmul_rn(d, d));
    }
  } else {
    const uint8_t* a = reinterpret_cast<const uint8_t*>(left) + (size_t)i * 128;
    const uint8_t* b = reinterpret_cast<const uint8_t*>(right) + (size_t)j * 128;
    int acc = 0;
    for (int t = 0; t < 32; ++t) { const int d = (int)a[4 * t + sub] - (int)b[4 * t + sub]; acc += d * d; }
    s = (float)acc;                                                   // exact integers < 2^24: any order gives the reference's float
  }
  const float s1 = __shfl_xor_sync(gmask, s, 1);                      // lanes (0,1) and (2,3)
  const float p = (sub & 1) ? __fadd_rn(s1, s) : __fadd_rn(s, s1);    // s0+s1 on lanes 0,1 ; s2+s3 on lanes 2,3
  const float s0123 = __shfl_sync(gmask, p, 0, 4);                    // (s0+s1)
  const float s2 = __shfl_sync(gmask, s, 2, 4), s3 = __shfl_sync(gmask, s, 3, 4);
  return (double)__fadd_rn(__fadd_rn(s0123, s2), s3);                 // ((s0+s1)+s2)+s3, metric.hpp:112-116
}

// The K7 body for left feature i of pair P, one warp per left feature; every thread of the block calls it for the same pair (the
// right positions stream through the block's shared tile).  The geometric gate, the survivor queue, the descriptor distances and
// the distanceRatio fold; returns the kept right feature, or -1, on every lane.
template <int DTYPE>
__device__ __forceinline__ int guided_row(const GuidedPair& P, int i, double distRatio, double2* tile, int* queue) {
  const int lane = threadIdx.x & 31;
  const bool live = i < P.ml;
  const int model = P.model, m_r = P.mr;
  const double errorTh = P.errorTh;
  // epipolar line of the left point in the right image, or its homography transfer
  double fx0 = 0, fx1 = 0, fx2 = 0, nrm = 1;
  if (live) guided_left(P.M, model, guided_pos(P.gl, P.fl, i), fx0, fx1, fx2, nrm);
  double bd = DBL_MAX, sbd = DBL_MAX; int idx = 0;                   // distanceRatio<double>, guidedMatching.hpp:77-90
  int nq = 0;
  const int sub = lane & 3, grp = lane >> 2;
  const unsigned gmask = 0xFu << (grp * 4);

  auto drain = [&](int count) {                                       // evaluate `count` (<= 8) queued candidates, oldest first
    const int j = grp < count ? queue[grp] : -1;
    double d = 0;
    if (j >= 0) d = guided_distance<DTYPE>(P.rawl, P.rawr, i, j, sub, gmask);
    for (int g = 0; g < count; ++g) {                                 // distanceRatio::update in ascending j (:95-110)
      const double dist = __shfl_sync(0xffffffffu, d, g * 4);
      const int jj = __shfl_sync(0xffffffffu, j, g * 4);
      if (dist < bd) { idx = jj; sbd = bd; bd = dist; }
      else if (dist < sbd) sbd = dist;
    }
  };

  for (int t0 = 0; t0 < m_r; t0 += GM_TILE) {
    __syncthreads();
    for (int e = threadIdx.x; e < GM_TILE && t0 + e < m_r; e += GM_WARPS * 32) tile[e] = guided_pos(P.gr, P.fr, t0 + e);
    __syncthreads();
    if (!live) continue;
    const int n = min(GM_TILE, m_r - t0);
    for (int b = 0; b < n; b += 32) {
      const int e = b + lane;
      bool pass = false;
      if (e < n) pass = guided_error(model, fx0, fx1, fx2, nrm, tile[e]) < errorTh;                 // guidedMatching.hpp:252
      const unsigned m = __ballot_sync(0xffffffffu, pass);
      if (m) {
        if (pass) queue[nq + __popc(m & ((1u << lane) - 1))] = t0 + e;
        nq += __popc(m);
        __syncwarp();
        while (nq >= 8) {
          drain(8);
          __syncwarp();
          const int rest = nq - 8;                                    // shift the remaining entries to the front
          const int v = lane < rest ? queue[8 + lane] : 0;
          __syncwarp();
          if (lane < rest) queue[lane] = v;
          nq = rest;
          __syncwarp();
        }
      }
    }
  }
  if (!live) return -1;
  if (nq > 0) drain(nq);
  // distanceRatio::isValid (:115-118) and the emitted pair (:259-263)
  return sbd != DBL_MAX && bd < __dmul_rn(distRatio, sbd) ? idx : -1;
}

// One launch per kernel class and batch: block b runs GM_WARPS left features of the pair whose blocks contain b.  Every (pair, left i)
// writes its kept right feature or -1 to best_j and the keep flag of the ordered compaction to keep.
template <int DTYPE>
__global__ void __launch_bounds__(GM_WARPS * 32)
guided_pairs_kernel(const GuidedPair* __restrict__ pairs, int n_pairs, double distRatio, int* __restrict__ best_j, int* __restrict__ keep) {
  __shared__ double2 tile[GM_TILE];
  __shared__ int queue[GM_WARPS][GM_QUEUE];
  int lo = 0, hi = n_pairs;                                           // last pair with block_base <= blockIdx.x
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (pairs[mid].block_base <= (int)blockIdx.x) lo = mid; else hi = mid; }
  const GuidedPair& P = pairs[lo];
  const int warp = threadIdx.x >> 5;
  const int i = ((int)blockIdx.x - P.block_base) * GM_WARPS + warp;
  const int j = guided_row<DTYPE>(P, i, distRatio, tile, queue[warp]);
  if (i < P.ml && (threadIdx.x & 31) == 0) { best_j[P.left_base + i] = j; keep[P.left_base + i] = j >= 0; }
}

// ordered compaction: kept (i, j) at kpos[g] (ascending i per pair, pairs in batch order); pstart[p] = first output of pair p
__global__ void guided_pairs_emit_kernel(const GuidedPair* __restrict__ pairs, int n_pairs, int n_left, const int* __restrict__ best_j,
                                         const int* __restrict__ keep, const int* __restrict__ kpos, uint2* __restrict__ out, int* __restrict__ pstart) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g <= n_pairs) pstart[g] = kpos[g < n_pairs ? pairs[g].left_base : n_left];
  if (g >= n_left || !keep[g]) return;
  int lo = 0, hi = n_pairs;                                           // last pair with left_base <= g
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (pairs[mid].left_base <= g) lo = mid; else hi = mid; }
  out[kpos[g]] = make_uint2((unsigned)(g - pairs[lo].left_base), (unsigned)best_j[g]);
}

// ---- position-only guided matching (b200m_guided_match_positions_pairs) -------------------------------------------------------------
// matching::guidedMatching<Mat3Model, ErrorT>(model, xLeft, xRight, errorTh, matches) (guidedMatching.hpp:37-70): for every left
// feature, the right feature of smallest error among those with err < errorTh, the first j on ties; no descriptors.  What
// GeometricFilterMatrix_H_AC::Geometry_guided_matching runs with distanceRatio < 0 (featureMatching's guided H filter).
//
// One thread per left feature: the block reads each right position of the shared tile by broadcast, so every thread scans j in
// ascending order and the reference's strict `err < errorTh && err < min` keeps the first j of a tie with no reduction.  Both tests
// are one compare against bound = min(errorTh, min) (errorTh NaN: bound NaN, nothing passes).  ~5 FP64 instructions per candidate
// for a homography.  The pair table and the work-item layout are K7's, with GP_THREADS left features per block.
//
// The reference's `match` is a default IndMatch() = (0, 0), pushed whenever min < errorTh: with errorTh = +inf a left feature whose
// errors are all inf / NaN / >= DBL_MAX contributes (0, 0), not (i, -).  Such a row writes -1 and raises the pair's `phantom`
// flag; the host (or guided_positions_deco_kernel) puts (0, 0) where IndMatch::getDeduplicated's sort puts it.
constexpr int GP_THREADS = 256;

template <int MODEL>
__device__ __forceinline__ void guided_positions_scan(const double2* tile, int n, int t0, double fx0, double fx1, double fx2, double nrm,
                                                      double& bound, int& bj) {
#pragma unroll 4
  for (int e = 0; e < n; ++e) {
    const double err = guided_error(MODEL, fx0, fx1, fx2, nrm, tile[e]);
    if (err < bound) { bound = err; bj = t0 + e; }
  }
}

__global__ void __launch_bounds__(GP_THREADS)
guided_positions_pairs_kernel(const GuidedPair* __restrict__ pairs, int n_pairs, int* __restrict__ best_j, int* __restrict__ keep,
                              int* __restrict__ phantom) {
  __shared__ double2 tile[GM_TILE];
  int lo = 0, hi = n_pairs;                                           // last pair with block_base <= blockIdx.x
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (pairs[mid].block_base <= (int)blockIdx.x) lo = mid; else hi = mid; }
  const GuidedPair& P = pairs[lo];
  const int i = ((int)blockIdx.x - P.block_base) * GP_THREADS + (int)threadIdx.x;
  const bool live = i < P.ml;
  const int model = P.model, m_r = P.mr;
  const double errorTh = P.errorTh;
  double fx0 = 0, fx1 = 0, fx2 = 0, nrm = 1;
  if (live) guided_left(P.M, model, guided_pos(P.gl, P.fl, i), fx0, fx1, fx2, nrm);
  double bound = errorTh > DBL_MAX ? DBL_MAX : errorTh;               // min(errorTh, min = DBL_MAX)
  int bj = -1;
  for (int t0 = 0; t0 < m_r; t0 += GM_TILE) {
    __syncthreads();
    for (int e = threadIdx.x; e < GM_TILE && t0 + e < m_r; e += GP_THREADS) tile[e] = guided_pos(P.gr, P.fr, t0 + e);
    __syncthreads();
    if (!live) continue;
    const int n = min(GM_TILE, m_r - t0);
    if (model == GM_HOMOGRAPHY) guided_positions_scan<GM_HOMOGRAPHY>(tile, n, t0, fx0, fx1, fx2, nrm, bound, bj);
    else guided_positions_scan<GM_FUNDAMENTAL>(tile, n, t0, fx0, fx1, fx2, nrm, bound, bj);
  }
  if (!live) return;
  if (bj < 0 && errorTh > DBL_MAX) phantom[lo] = 1;                  // min = DBL_MAX < errorTh = +inf: IndMatch() is pushed
  best_j[P.left_base + i] = bj;
  keep[P.left_base + i] = bj >= 0;
}

// IndMatchDecorator::getDeduplicated on the device (see finish.cuh): for a pair whose left view is in general position (yrank[p] set)
// the decorated list is the kept matches by ascending left y, so row i goes to slot left_base + yrank[i].  IndMatch::getDeduplicated
// puts a phantom (0, 0) first, and the decorator keeps the first match of left feature 0, so the phantom replaces row 0's match.
// Other pairs are copied in ascending i and finished on the host.  rec / keep2 are then compacted like K7's slots.
__global__ void guided_positions_deco_kernel(const GuidedPair* __restrict__ pairs, const uint32_t* const* __restrict__ yrank, int n_pairs, int n_left,
                                             const int* __restrict__ best_j, const int* __restrict__ phantom, uint2* __restrict__ rec,
                                             int* __restrict__ keep2) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_left) return;
  int lo = 0, hi = n_pairs;                                           // last pair with left_base <= g
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (pairs[mid].left_base <= g) lo = mid; else hi = mid; }
  const int base = pairs[lo].left_base, i = g - base;
  const uint32_t* yr = yrank[lo];
  int j = best_j[g];
  if (yr && i == 0 && phantom[lo]) j = 0;
  const int slot = yr ? base + (int)yr[i] : g;
  rec[slot] = make_uint2((unsigned)i, (unsigned)j);
  keep2[slot] = j >= 0;
}

// ordered compaction of guided_positions_deco_kernel's slots, as guided_pairs_emit_kernel does for K7's
__global__ void guided_positions_emit_kernel(const GuidedPair* __restrict__ pairs, int n_pairs, int n_left, const uint2* __restrict__ rec,
                                             const int* __restrict__ keep, const int* __restrict__ kpos, uint2* __restrict__ out, int* __restrict__ pstart) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g <= n_pairs) pstart[g] = kpos[g < n_pairs ? pairs[g].left_base : n_left];
  if (g >= n_left || !keep[g]) return;
  out[kpos[g]] = rec[g];
}
}  // namespace b200m

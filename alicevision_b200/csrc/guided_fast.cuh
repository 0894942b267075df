// K9 — bucketed guided matching from known poses: matching::guidedMatchingFundamentalFast<FundamentalEpipolarDistanceError>
// (matching/guidedMatching.hpp:353-460, helpers pixToBucket / lineToEndPoints in guidedMatching.cpp:13-70), the matcher of
// StructureEstimationFromKnownPoses::match (sfm/pipeline/structureFromKnownPoses/StructureEstimationFromKnownPoses.cpp:72-163),
// for a whole list of pairs of resident views per launch.
//
// The reference puts every left feature into the bucket (a pixel of the right image's border) where its epipolar line ends, and
// gives every right feature the range of buckets that the lines through the epipole at +-sqrt(errorTh) pixels reach; every left
// feature of that range is a candidate (no geometric-error test).  Here, per batch of pairs:
//   guided_fast_left_kernel   one thread per (pair, left i): bucket of i (or none), count per (pair, bucket)
//   exclusive scan            CSR offsets over all (pair, bucket)
//   guided_fast_scatter_kernel   left features into their bucket's CSR slice
//   guided_fast_right_kernel  one thread per (pair, right j): candidate range = CSR slice [off[start], off[stop]), O(1)
//   exclusive scan            a flat, load-balanced candidate space over all (pair, j)
//   guided_fast_cand_kernel   one 4-lane group per candidate: guided_distance (guided.cuh), then the distanceRatio fold
//   guided_fast_keep_kernel / exclusive scan / guided_fast_emit_kernel   ordered compaction: (i, idx) in ascending i per pair
//
// The fold.  distanceRatio::update over ascending j (guidedMatching.hpp:93-109) ends with bd = the minimum, idx = the smallest j
// reaching it and sbd = the second smallest value of the multiset of distances; each (i, j) is visited at most once (i lies in one
// bucket, a range is contiguous), so this does not depend on the visit order.  Every distance is a float widened to double
// (L2_Vectorized: float; squared Hamming <= 2^18), so key = (float bits << 32) | j is totally ordered and two atomicMin per
// candidate - best = min(key), second = min over k of max(key, best before k) - give exactly (bd, idx, sbd), ties included.
// A NaN distance never passes `dist < bd` nor `dist < sbd` in the reference: it is skipped.
//
// Arithmetic.  All double arithmetic that decides a bucket is uncontracted (__dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn /
// __dsqrt_rn): when neither end point is clamped, r1 and r2 are rounding noise and the choice of x0 depends on the exact operations.
// Each row of F x is summed as (F(r,0) x + F(r,1) y) + F(r,2); Eigen's own association for that product is not compiled here, and
// DESIGN.md (K9) gives the reading of it, why this order is kept and what the difference changes.  r1 and r2 are floats, as in
// lineToEndPoints.
//
// Divergence (documented in include/b200match.h and DESIGN.md): where the reference is undefined - an epipole at infinity
// (ep2(2) == 0: division by 0) or a right feature exactly at the epipole (n = 0 * inf = NaN) - it casts NaN to int and indexes
// `buckets` out of range.  Here a line with a non-finite coefficient has no end points: no bucket for that left feature, no
// candidates for that right feature.
#pragma once
#include "guided.cuh"

namespace b200m {

constexpr int GF_THREADS = 256;       // per-feature kernels
constexpr int GF_CAND_CHUNK = 8;      // consecutive candidates per 4-lane group and step (one range search per chunk)

struct FastPair {
  const void* rawl; const void* rawr;           // descriptors (kernel dtype: a uchar-stored view of a mixed pair points at its fp32 expansion)
  const double2* gl; const double2* gr;         // geometry positions, or nullptr: the float upload positions below, widened
  const float2* fl; const float2* fr;
  double F[9];                                  // row-major, already negated when ep2(2) > 0
  double e0, e1, e2;                            // ep2 / ep2(2) (e2 == 1, or NaN for an epipole at infinity)
  int ml, mr, W, H, nb;                         // nb = 2 (W + H - 2)
  int left_base, right_base, bucket_base;       // offsets of this pair in the flat per-batch arrays (buckets: nb + 1 slots)
};

__device__ __forceinline__ bool gf_finite(double v) { return isfinite(v); }

// pixToBucket (guidedMatching.cpp:13-22) on x0.cast<int>()
__device__ __forceinline__ int gf_pix_to_bucket(int x, int y, int W, int H) {
  if (y == 0) return x;                          // top border
  if (x == W - 1) return W - 1 + y;              // right border
  if (y == H - 1) return 2 * W + H - 3 - x;      // bottom border
  return 2 * (W + H - 2) - y;                    // left border
}

// lineToEndPoints (guidedMatching.cpp:24-70) followed by pixToBucket(x0.cast<int>()); -1 = no end points
__device__ __forceinline__ int gf_line_bucket(double a, double b, double c, int W, int H) {
  if (!gf_finite(a) || !gf_finite(b) || !gf_finite(c)) return -1;      // the documented divergence (see the header comment)
  if (b == 0) return -1;
  const double xa = b < 0 ? 0.0 : (double)(W - 1);
  double ya = __ddiv_rn(-__dadd_rn(__dmul_rn(a, xa), c), b);         // y = -(a * x + c) / b
  if (ya < 0) ya = 0.0;
  else if (ya >= H) ya = (double)(H - 1);
  const float r1 = (float)fabs(__dadd_rn(__dadd_rn(__dmul_rn(a, xa), __dmul_rn(b, ya)), c));
  if (a == 0) return -1;
  const double yb = a < 0 ? (double)(H - 1) : 0.0;
  double xb = __ddiv_rn(-__dadd_rn(__dmul_rn(b, yb), c), a);         // x = -(b * y + c) / a
  if (xb < 0) xb = 0.0;
  else if (xb >= W) xb = (double)(W - 1);
  const float r2 = (float)fabs(__dadd_rn(__dadd_rn(__dmul_rn(a, xb), __dmul_rn(b, yb)), c));
  const double x0 = r1 > r2 ? xb : xa, y0 = r1 > r2 ? yb : ya;         // if (r1 > r2) std::swap(x0, x1)
  return gf_pix_to_bucket((int)x0, (int)y0, W, H);
}

// ep2.cross(Vec3(x, y, 1)) (Eigen's order: (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0))
__device__ __forceinline__ void gf_cross(const FastPair& P, double x, double y, double& l0, double& l1, double& l2) {
  l0 = __dsub_rn(__dmul_rn(P.e1, 1.0), __dmul_rn(P.e2, y));
  l1 = __dsub_rn(__dmul_rn(P.e2, x), __dmul_rn(P.e0, 1.0));
  l2 = __dsub_rn(__dmul_rn(P.e0, y), __dmul_rn(P.e1, x));
}

// grid (features / GF_THREADS, pairs): bucket of every left feature, counts per (pair, bucket); keys reset to the sentinel
__global__ void __launch_bounds__(GF_THREADS)
guided_fast_left_kernel(const FastPair* __restrict__ pairs, int* __restrict__ lbucket, int* __restrict__ bcount,
                        unsigned long long* __restrict__ best, unsigned long long* __restrict__ second) {
  const FastPair& P = pairs[blockIdx.y];
  const int i = blockIdx.x * GF_THREADS + threadIdx.x;
  if (i >= P.ml) return;
  const double2 x = guided_pos(P.gl, P.fl, i);
  // line = F * (x, y, 1), row r = (F(r,0) x + F(r,1) y) + F(r,2)
  const double a = __dadd_rn(__dadd_rn(__dmul_rn(P.F[0], x.x), __dmul_rn(P.F[1], x.y)), P.F[2]);
  const double b = __dadd_rn(__dadd_rn(__dmul_rn(P.F[3], x.x), __dmul_rn(P.F[4], x.y)), P.F[5]);
  const double c = __dadd_rn(__dadd_rn(__dmul_rn(P.F[6], x.x), __dmul_rn(P.F[7], x.y)), P.F[8]);
  const int bk = gf_line_bucket(a, b, c, P.W, P.H);
  const int g = P.left_base + i;
  lbucket[g] = bk;
  best[g] = ~0ull; second[g] = ~0ull;
  if (bk >= 0) atomicAdd(&bcount[P.bucket_base + bk], 1);
}

// left feature i -> its bucket's slice of the CSR (order inside a bucket is irrelevant: the fold does not depend on it)
__global__ void __launch_bounds__(GF_THREADS)
guided_fast_scatter_kernel(const FastPair* __restrict__ pairs, const int* __restrict__ lbucket, int* __restrict__ cursor, int* __restrict__ csr) {
  const FastPair& P = pairs[blockIdx.y];
  const int i = blockIdx.x * GF_THREADS + threadIdx.x;
  if (i >= P.ml) return;
  const int bk = lbucket[P.left_base + i];
  if (bk >= 0) csr[atomicAdd(&cursor[P.bucket_base + bk], 1)] = i;
}

// one thread per (pair, right j): the candidate slice of j in the CSR (guidedMatching.hpp:410-441)
__global__ void __launch_bounds__(GF_THREADS)
guided_fast_right_kernel(const FastPair* __restrict__ pairs, double sqrt_th, const int* __restrict__ boff, int* __restrict__ rstart,
                         unsigned long long* __restrict__ rcount, int* __restrict__ rpair) {
  const FastPair& P = pairs[blockIdx.y];
  const int j = blockIdx.x * GF_THREADS + threadIdx.x;
  if (j >= P.mr) return;
  const int r = P.right_base + j;
  const double2 x = guided_pos(P.gr, P.fr, j);
  double l0, l1, l2;
  gf_cross(P, x.x, x.y, l0, l1, l2);
  const double s = __ddiv_rn(sqrt_th, __dsqrt_rn(__dadd_rn(__dmul_rn(l0, l0), __dmul_rn(l1, l1))));   // sqrt(errorTh) / l2.head<2>().norm()
  const double n0 = __dmul_rn(l0, s), n1 = __dmul_rn(l1, s);
  double a, b, c;
  gf_cross(P, __dsub_rn(x.x, n0), __dsub_rn(x.y, n1), a, b, c);                                          // l2min
  const int start = gf_line_bucket(a, b, c, P.W, P.H);
  gf_cross(P, __dadd_rn(x.x, n0), __dadd_rn(x.y, n1), a, b, c);                                          // l2max
  const int stop = start < 0 ? -1 : gf_line_bucket(a, b, c, P.W, P.H);
  int s0 = 0, cnt = 0;
  if (start >= 0 && stop > start) {
    s0 = boff[P.bucket_base + start];
    cnt = boff[P.bucket_base + stop] - s0;
  }
  rstart[r] = s0; rcount[r] = (unsigned long long)cnt; rpair[r] = blockIdx.y;
}

// The candidate space [0, total): candidate c belongs to the right feature r with coff[r] <= c < coff[r + 1].  One 4-lane group per
// candidate, GF_CAND_CHUNK consecutive candidates per group and step; groups stride over the space.
template <int DTYPE>
__global__ void __launch_bounds__(GF_THREADS)
guided_fast_cand_kernel(const FastPair* __restrict__ pairs, int n_right, const unsigned long long* __restrict__ coff, const int* __restrict__ rstart,
                        const int* __restrict__ rpair, const int* __restrict__ csr, unsigned long long* __restrict__ best,
                        unsigned long long* __restrict__ second) {
  const unsigned long long total = coff[n_right];
  const int lane = threadIdx.x & 31, sub = lane & 3, grp = lane >> 2;
  const unsigned gmask = 0xFu << (grp * 4);
  const unsigned long long ngroups = (unsigned long long)gridDim.x * (GF_THREADS / 4);
  for (unsigned long long q = (unsigned long long)blockIdx.x * (GF_THREADS / 4) + (threadIdx.x >> 2); q * GF_CAND_CHUNK < total; q += ngroups) {
    const unsigned long long c0 = q * GF_CAND_CHUNK, c1 = min(c0 + GF_CAND_CHUNK, total);
    int lo = 0, hi = n_right;                     // last r with coff[r] <= c0
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (coff[mid] <= c0) lo = mid; else hi = mid; }
    int r = lo;
    for (unsigned long long c = c0; c < c1; ++c) {
      while (coff[r + 1] <= c) ++r;               // right features without candidates are skipped here
      const FastPair& P = pairs[rpair[r]];
      const int j = r - P.right_base;
      const int i = csr[rstart[r] + (int)(c - coff[r])];
      const double d = guided_distance<DTYPE>(P.rawl, P.rawr, i, j, sub, gmask);
      if (sub == 0 && d == d) {                  // SquaredDescriptorDistance: a float widened to double; NaN never updates (:95-110)
        const unsigned long long k = ((unsigned long long)__float_as_uint((float)d) << 32) | (unsigned)j;
        const int g = P.left_base + i;
        const unsigned long long old = atomicMin(&best[g], k);
        atomicMin(&second[g], old > k ? old : k);
      }
    }
  }
}

// distanceRatio::isValid (:114-120): two distances seen and bd < distRatio * sbd (double product)
__global__ void __launch_bounds__(GF_THREADS)
guided_fast_keep_kernel(const FastPair* __restrict__ pairs, double dist_ratio, const unsigned long long* __restrict__ best,
                        const unsigned long long* __restrict__ second, int* __restrict__ keep) {
  const FastPair& P = pairs[blockIdx.y];
  const int i = blockIdx.x * GF_THREADS + threadIdx.x;
  if (i >= P.ml) return;
  const int g = P.left_base + i;
  const unsigned long long s = second[g];
  int k = 0;
  if (s != ~0ull) {
    const double bd = (double)__uint_as_float((unsigned)(best[g] >> 32)), sbd = (double)__uint_as_float((unsigned)(s >> 32));
    k = bd < __dmul_rn(dist_ratio, sbd);
  }
  keep[g] = k;
}

// ordered compaction: kept (i, idx) at kpos[g] (ascending i per pair, pairs in batch order); pstart[p] = first output of pair p
__global__ void __launch_bounds__(GF_THREADS)
guided_fast_emit_kernel(const FastPair* __restrict__ pairs, int n_pairs, int n_left, const int* __restrict__ keep, const int* __restrict__ kpos,
                        const unsigned long long* __restrict__ best, uint2* __restrict__ out, int* __restrict__ pstart) {
  const FastPair& P = pairs[blockIdx.y];
  const int i = blockIdx.x * GF_THREADS + threadIdx.x;
  if (i == 0) {
    pstart[blockIdx.y] = kpos[P.left_base];
    if (blockIdx.y == n_pairs - 1) pstart[n_pairs] = kpos[n_left];
  }
  if (i >= P.ml) return;
  const int g = P.left_base + i;
  if (keep[g]) out[kpos[g]] = make_uint2((unsigned)i, (unsigned)(best[g] & 0xffffffffull));
}

}  // namespace b200m

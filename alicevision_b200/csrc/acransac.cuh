// K10: a-contrario RANSAC estimation for a list of pairs, sm_90a: the fundamental matrix (b200m_acransac_fundamental_pairs,
// FPolicy), the homography (b200m_acransac_homography_pairs, HPolicy) and the fundamental matrix of two equidistant cameras on
// lifted unit vectors (b200m_acransac_fundamental_spherical_pairs, SPolicy) and the essential matrix of two pinhole cameras
// (b200m_acransac_essential_pairs, EPolicy) and the fundamental matrix with two radial distortion coefficients
// (b200m_acransac_fundamental_distortion_pairs, F10Policy).  The kernel is one template over the model policy.
//
// One CTA runs one pair's robustEstimation::ACRANSAC loop (robustEstimation/ACRansac.hpp:186-272) iteration by iteration, with the
// reference's control flow (10 % reserve, strict `<` on minNFA, the switch to sampling among the inliers, the "no model at all"
// extension, the precision mode and its early exit).  Per iteration thread 0 draws the sample from the pair's own copy of the
// caller's std::mt19937 (shared memory) and fits the models (7-point F, 4-point H, 5-point E or 10-point F10, acransac_math.h); then the whole CTA scores
// each model:
//   * n residuals (F: point-to-line error, H: point-to-point transfer error, on normalised points; S: (F x_I . x_J)^2 on bearings);
//   * certified skip: a shared-memory histogram of the residuals over quarter-binade bins gives, for every k, a lower bound of the
//     k-th smallest residual (the low edge of its bin), hence of NFA(k), which increases with that residual.  When the least bound
//     over k is not below the current minNFA (less a 1e-9 relative margin that covers the device log10), the model cannot be
//     `better` and is not scored exactly.  The loop is sequential, so the bound is compared with the true running minNFA;
//   * exact score: (residual bits, index) keys sorted by a bitonic network, in shared memory up to kSmemSort keys and in a
//     per-pair global scratch beyond; every k's NFA; the (NFA, k)-lexicographic argmin (bestNFA keeps the first k reaching the
//     minimum).  NaN residuals sort after +inf, where std::sort is unspecified.
// The winner's sorted indices are its inlier list in the reference's order.  When asked, the generator's state after the pair's
// last draw is written back (HPolicy, SPolicy: the reference passes its std::mt19937 by reference from pair to pair).
#pragma once
#include "acransac_math.h"

#include <cfloat>
#include <cstdint>

namespace acrk {

constexpr int kThreads = 128;
constexpr int kSmemSort = 1024;    // keys sorted in shared memory; larger pairs sort in global scratch
constexpr int kBinLo = 1023 - 100; // biased exponent of the first quarter-binade bin (2^-100); bin 0 holds [0, 2^-100)
constexpr int kBins = 2 + 4 * 128; // ... up to 2^28; the last bin holds everything above, +inf and NaN
constexpr int kTraceCap = 256;      // `better` events (iteration, new minNFA) kept per pair (b200m_acransac_last_trace)

struct Pair { long long off, sort_off; int n, w1, h1, w2, h2; };
struct PairE { Pair q; double kinv[18]; };   // EPolicy's pair: K_I^-1 then K_J^-1, row-major
struct Out {
  double model[9]; double error_max, min_nfa;
  long long evaluated, skipped, exact;
  int valid, n_inl, iterations, n_trace;
};
struct OutL { Out o; double L[2]; };   // F10Policy's result: the winner's radial distortion (l1, l2) beside it

__device__ __forceinline__ int bin_of(double r) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(r);
  const int e = (int)(b >> 52);
  if (e < kBinLo) return 0;
  const int q = 1 + (e - kBinLo) * 4 + (int)((b >> 50) & 3);
  return q < kBins - 1 ? q : kBins - 1;
}
__device__ __forceinline__ double bin_low(int b) {
  if (b == 0) return 0.0;
  const int q = b - 1;
  return __longlong_as_double((long long)(((unsigned long long)(kBinLo + q / 4) << 52) | ((unsigned long long)(q & 3) << 50)));
}

// Model policies: sample size, maximum number of models, fit, residual, logalpha0, errorVectorDimension, unnormaliser, and the
// correspondence layout: kPlanar = pixel pairs (xI, yI, xJ, yJ) preconditioned by the image sizes; kCalibrated = pixel pairs
// followed by their K^-1-normalised copies (xI, yI, xJ, yJ, uI, vI, uJ, vJ), fitted on the copies, scored on the pixels; else
// lifted unit vectors (xI, yI, zI, xJ, yJ, zJ) used as given; kWidth doubles per correspondence.  kDistortion: the model carries
// (l1, l2) beside its matrix, the fit runs in a per-CTA shared-memory workspace and the result is an OutL.
struct FPolicy {   // RelativePoseKernel<Fundamental7PSolver, FundamentalEpipolarDistanceError, UnnormalizerT>
  static constexpr int kSample = acr::kSample, kMaxModels = acr::kMaxModels, kErrDim = 1, kWidth = 4;
  static constexpr bool kPlanar = true, kCalibrated = false, kDistortion = false;
  __device__ static int fit(const double* a, const double* b, const double* c, const double* d, double* m) {
    return acr::fit7_solve<false>(a, b, c, d, m);   // = acr::fit7, one inlining level shallower
  }
  __device__ static double error(const double* m, double x1, double y1, double x2, double y2) { return acr::epipolar_error(m, x1, y1, x2, y2); }
  __device__ static double logalpha0(int w2, int h2, const acr::Norm& n2) {
    return log10(2.0 * sqrt(acr::add(acr::mul((double)w2, (double)w2), acr::mul((double)h2, (double)h2))) / acr::mul((double)w2, (double)h2) / n2.s);
  }
  __device__ static void unnormalize(const acr::Norm& n1, const acr::Norm& n2, double* m) { acr::unnormalize(n1, n2, m); }
};
struct HPolicy {   // RelativePoseKernel<Homography4PSolver, HomographyAsymmetricError, UnnormalizerI>, point to point
  static constexpr int kSample = acr::kSampleH, kMaxModels = acr::kMaxModelsH, kErrDim = 2, kWidth = 4;
  static constexpr bool kPlanar = true, kCalibrated = false, kDistortion = false;
  __device__ static int fit(const double* a, const double* b, const double* c, const double* d, double* m) { return acr::fit4(a, b, c, d, m); }
  __device__ static double error(const double* m, double x1, double y1, double x2, double y2) { return acr::homography_error(m, x1, y1, x2, y2); }
  __device__ static double logalpha0(int w2, int h2, const acr::Norm& n2) { return acr::logalpha0_h(w2, h2, n2); }
  __device__ static void unnormalize(const acr::Norm& n1, const acr::Norm& n2, double* m) { acr::unnormalize_h(n1, n2, m); }
};
struct SPolicy {   // RelativePoseSphericalKernel<Fundamental7PSphericalSolver, EpipolarSphericalDistanceError>
  static constexpr int kSample = acr::kSample, kMaxModels = acr::kMaxModels, kErrDim = 2, kWidth = 6;
  static constexpr bool kPlanar = false, kCalibrated = false, kDistortion = false;
  __device__ static int fit(const double* x1, const double* x2, double* m) { return acr::fit7s(x1, x2, m); }
  __device__ static double error(const double* m, const double* x1, const double* x2) { return acr::spherical_error(m, x1, x2); }
  __device__ static double logalpha0(int, int, const acr::Norm&) { return M_PI; }   // the value itself, not its log10
  __device__ static void unnormalize(const acr::Norm&, const acr::Norm&, double*) {}
};
struct EPolicy {   // RelativePoseKernel_K<Essential5PSolver, FundamentalEpipolarDistanceError, Mat3Model>
  // models[] holds F = K_J^-T E K_I^-1 of each model for the residuals, then the Es.  errorVectorDimension is 0.5, which the int
  // kErrDim of the other policies cannot hold: nfa_of applies it under `if constexpr (P::kCalibrated)`, and kErrDim = 0 is unused.
  static constexpr int kSample = acr::kSampleE, kMaxModels = acr::kMaxModelsE, kErrDim = 0, kWidth = 8;
  static constexpr bool kPlanar = false, kCalibrated = true, kDistortion = false;
  __device__ static int fit(const double* a, const double* b, const double* c, const double* d, const double* kinv, double* m) {
    double* E = m + 9 * kMaxModels;
    const int nb = acr::fit5(a, b, c, d, E);
    for (int k = 0; k < nb; ++k) acr::fundamental_from_essential(E + 9 * k, kinv, kinv + 9, m + 9 * k);
    return nb;
  }
  __device__ static double error(const double* m, double x1, double y1, double x2, double y2) { return acr::epipolar_error(m, x1, y1, x2, y2); }
  __device__ static double logalpha0(int w2, int h2, const acr::Norm&) { return acr::logalpha0_e(w2, h2); }
  __device__ static void unnormalize(const acr::Norm&, const acr::Norm&, double*) {}
};
struct F10Policy {   // RelativePoseKernel<Fundamental10PSolver, FundamentalEpipolarDistanceError, UnnormalizerT, Fundamental10PModel>
  // FPolicy's preconditioning, error, logalpha0 and unnormaliser (on the matrix only); models[] holds the 10 matrices, then their
  // (l1, l2).  The error scores the matrix alone, transposed against the solver's constraint, as the reference does.
  static constexpr int kSample = acr::kSampleF10, kMaxModels = acr::kMaxModelsF10, kErrDim = 1, kWidth = 4;
  static constexpr bool kPlanar = true, kCalibrated = false, kDistortion = true;
  __device__ static int fit(const double* a, const double* b, const double* c, const double* d, double* m, acr::F10Work& w) {
    return acr::fit10(a, b, c, d, m, m + 9 * kMaxModels, w);
  }
  __device__ static double error(const double* m, double x1, double y1, double x2, double y2) { return acr::epipolar_error(m, x1, y1, x2, y2); }
  __device__ static double logalpha0(int w2, int h2, const acr::Norm& n2) { return FPolicy::logalpha0(w2, h2, n2); }
  __device__ static void unnormalize(const acr::Norm& n1, const acr::Norm& n2, double* m) { acr::unnormalize(n1, n2, m); }
};

// NFA(k) of bestNFA for the squared residual e of rank k: loge0 + (la0 + d log10(sqrt(e) + FLT_EPSILON)) (k - kSample) + logc_n[k]
// + logc_k[k], d = errorVectorDimension (1: F, 2: H and S, 0.5: E; the products are exact)
template <class P>
__device__ __forceinline__ double nfa_of(double e, int k, double la0, double loge0, const float* lcn, const float* lck) {
  const double l = log10(acr::add(sqrt(e), (double)FLT_EPSILON));
  double la;
  if constexpr (P::kCalibrated) la = acr::add(la0, acr::mul(0.5, l));
  else la = acr::add(la0, P::kErrDim == 1 ? l : acr::mul((double)P::kErrDim, l));
  return acr::add(acr::add(acr::add(loge0, acr::mul(la, (double)(k - P::kSample))), (double)lcn[k]), (double)lck[k]);
}

__device__ __forceinline__ bool lex_less(double v, int k, double v2, int k2) { return v2 < v || (v2 == v && k2 < k); }

// (value, k) lexicographic minimum over the CTA; every thread gets the result
__device__ void block_min(double& v, int& k, double* sv, int* sk) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 16; o; o >>= 1) {
    const double v2 = __shfl_down_sync(0xffffffffu, v, o);
    const int k2 = __shfl_down_sync(0xffffffffu, k, o);
    if (lex_less(v, k, v2, k2)) { v = v2; k = k2; }
  }
  if (lane == 0) { sv[warp] = v; sk[warp] = k; }
  __syncthreads();
  v = sv[0]; k = sk[0];
  for (int w = 1; w < kThreads / 32; ++w)
    if (lex_less(v, k, sv[w], sk[w])) { v = sv[w]; k = sk[w]; }
  __syncthreads();
}

__device__ int block_sum(int x, int* si) {
  for (int o = 16; o; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
  if ((threadIdx.x & 31) == 0) si[threadIdx.x >> 5] = x;
  __syncthreads();
  int s = 0;
  for (int w = 0; w < kThreads / 32; ++w) s += si[w];
  __syncthreads();
  return s;
}

__device__ void bitonic(unsigned long long* K, uint32_t* V, int N2) {
  for (int size = 2; size <= N2; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = threadIdx.x; t < N2 / 2; t += kThreads) {
        const int i = 2 * t - (t & (stride - 1)), j = i + stride;
        const unsigned long long ki = K[i], kj = K[j];
        const uint32_t vi = V[i], vj = V[j];
        const bool gt = ki > kj || (ki == kj && vi > vj);
        if (gt == ((i & size) == 0)) { K[i] = kj; K[j] = ki; V[i] = vj; V[j] = vi; }
      }
      __syncthreads();
    }
}

template <class P>
__device__ __forceinline__ double residual(const double* M, const double* pts, int i) {
  if constexpr (P::kPlanar) {
    const double2 a = reinterpret_cast<const double2*>(pts)[2 * i], b = reinterpret_cast<const double2*>(pts)[2 * i + 1];
    return P::error(M, a.x, a.y, b.x, b.y);
  } else if constexpr (P::kCalibrated) {   // the pixel half of the correspondence
    const double2 a = reinterpret_cast<const double2*>(pts)[4 * i], b = reinterpret_cast<const double2*>(pts)[4 * i + 1];
    return P::error(M, a.x, a.y, b.x, b.y);
  } else {   // 48 bytes a correspondence: three aligned 16-byte loads
    const double2* q = reinterpret_cast<const double2*>(pts) + 3 * i;
    const double2 a = q[0], b = q[1], c = q[2];
    const double x1[3] = {a.x, a.y, b.x}, x2[3] = {b.y, c.x, c.y};
    return P::error(M, x1, x2);
  }
}

// corr: per correspondence P::kWidth doubles at the pair's offset, (xI, yI, xJ, yJ) or (xI, yI, zI, xJ, yJ, zJ); 4 doubles
// (xI, yI, xJ, yJ) for EPolicy, whose pairs are PairE; l10[k] = (float)log10((double)k) for k <= the largest n.
// Scratch at the pair's offset: pts (P::kWidth doubles), idx (the sampling list), logc (n + 1 floats each of logc_n and logc_k, at
// 2 * (off + pair)), gkeys / gvals (pow2(n) at sort_off, pairs above kSmemSort only).  inliers: the result list at the offset.
// mt_state: 625 words at p * mt_stride (mt_stride 0: one state for every pair); mt_out: NULL, or 625 words per pair receiving the
// generator state after the pair's last draw.  out_all: Out per pair, OutL for kDistortion.
template <class P>
__global__ void __launch_bounds__(kThreads, 4) acransac_kernel(const Pair* __restrict__ pairs, const double* __restrict__ corr,
                                                             const float* __restrict__ l10, const uint32_t* __restrict__ mt_state,
                                                             int mt_stride, long long max_iter, double precision, int skip_on, double* pts_all,
                                                             uint32_t* idx_all, float* logc_all, unsigned long long* gkeys,
                                                             uint32_t* gvals, uint32_t* inliers_all, int* trace_all, double* trace_nfa_all,
                                                             Out* out_all, uint32_t* mt_out) {
  __shared__ acr::Mt19937 g;
  __shared__ double models[9 * P::kMaxModels * (P::kCalibrated ? 2 : 1) + (P::kDistortion ? 2 * P::kMaxModels : 0)];
  __shared__ double bestF[9 + (P::kDistortion ? 2 : 0)];   // F10: the winner's (l1, l2) at 9, 10
  __shared__ int hist[kBins];
  __shared__ unsigned long long skeys[kSmemSort];
  __shared__ uint32_t svals[kSmemSort];
  __shared__ double red_v[kThreads / 32];
  __shared__ int red_k[kThreads / 32];
  __shared__ long long nIter, nReserve, iter, evaluated, skipped, exact;
  __shared__ int nb, mode, better, n_inl, n_idx, stop, copy_idx, n_trace;
  __shared__ double minNFA, errorMax;

  const int p = blockIdx.x, tid = threadIdx.x;
  const Pair Q = P::kCalibrated ? reinterpret_cast<const PairE*>(pairs)[p].q : pairs[p];
  const int n = Q.n;
  Out* out = P::kDistortion ? &reinterpret_cast<OutL*>(out_all)[p].o : out_all + p;
  const double inf = __longlong_as_double(0x7ff0000000000000ll);
  const uint32_t* st_in = mt_state + (long long)p * mt_stride;
  if (n <= P::kSample) {   // ACRANSAC returns (0, 0) at once, without a draw
    if (tid == 0) {
      for (int t = 0; t < 9; ++t) out->model[t] = 0;
      out->error_max = 0; out->min_nfa = 0; out->evaluated = out->skipped = out->exact = 0;
      out->valid = 0; out->n_inl = 0; out->iterations = 0; out->n_trace = 0;
      if constexpr (P::kDistortion) reinterpret_cast<OutL*>(out)->L[0] = reinterpret_cast<OutL*>(out)->L[1] = 0;
    }
    if (mt_out)
      for (int i = tid; i <= acr::kMtN; i += kThreads) mt_out[(long long)p * (acr::kMtN + 1) + i] = st_in[i];
    return;
  }
  acr::Norm n1{1.0, 0.0, 0.0}, n2{1.0, 0.0, 0.0};   // identity for bearings (no image size)
  if constexpr (P::kPlanar) { n1 = acr::precondition(Q.w1, Q.h1); n2 = acr::precondition(Q.w2, Q.h2); }
  double* pts = pts_all + P::kWidth * Q.off;
  uint32_t* idx = idx_all + Q.off;
  uint32_t* inl = inliers_all + Q.off;
  float* lcn = logc_all + 2 * (Q.off + p);
  float* lck = lcn + n + 1;
  const double* c = corr + (P::kCalibrated ? 4 : P::kWidth) * Q.off;
  const double* kinv = P::kCalibrated ? reinterpret_cast<const PairE*>(pairs)[p].kinv : nullptr;
  for (int i = tid; i < n; i += kThreads) {
    if constexpr (P::kCalibrated) {   // RelativePoseKernel_K's constructor: the pixels, and K^-1 applied to them
      for (int t = 0; t < 4; ++t) pts[8 * i + t] = c[4 * i + t];
      acr::transform_point(kinv, c[4 * i], c[4 * i + 1], pts[8 * i + 4], pts[8 * i + 5]);
      acr::transform_point(kinv + 9, c[4 * i + 2], c[4 * i + 3], pts[8 * i + 6], pts[8 * i + 7]);
    } else if constexpr (P::kPlanar) {
      pts[4 * i] = acr::norm_x(n1, c[4 * i]); pts[4 * i + 1] = acr::norm_y(n1, c[4 * i + 1]);
      pts[4 * i + 2] = acr::norm_x(n2, c[4 * i + 2]); pts[4 * i + 3] = acr::norm_y(n2, c[4 * i + 3]);
    } else {
      for (int t = 0; t < P::kWidth; ++t) pts[P::kWidth * i + t] = c[P::kWidth * i + t];
    }
    idx[i] = i;
  }
  // makelogcombi: logcombi(k, n) is the float sum of the first min(k, n - k) terms l10[n - i + 1] - l10[i] in ascending i, so one
  // running sum over k <= n / 2 gives every entry with the reference's bits (k >= n and k <= 0 give 0)
  if (tid == 0) {
    float r = 0.0f;
    lcn[0] = 0.0f;
    for (int k = 1; k <= n / 2; ++k) {
      r = __fadd_rn(r, __fsub_rn(l10[n - k + 1], l10[k]));
      lcn[k] = r;
    }
  }
  __syncthreads();
  for (int k = n / 2 + 1 + tid; k <= n; k += kThreads) lcn[k] = k >= n ? 0.0f : lcn[n - k];
  for (int k = tid; k <= n; k += kThreads) {   // logcombi(kSample, k): at most kSample terms
    float s = 0.0f;
    if (!(P::kSample >= k)) {
      int kk = P::kSample;
      if (k - kk < kk) kk = k - kk;
      for (int i = 1; i <= kk; ++i) s = __fadd_rn(s, __fsub_rn(l10[k - i + 1], l10[i]));
    }
    lck[k] = s;
  }
  for (int i = tid; i < acr::kMtN; i += kThreads) g.x[i] = st_in[i];
  const double la0 = P::logalpha0(Q.w2, Q.h2, n2);
  const double loge0 = log10(acr::mul((double)P::kMaxModels, (double)(n - P::kSample)));
  double maxThr;   // precision^2 thresholdNormalizer()^2; thresholdNormalizer() = 1 for bearings
  if constexpr (P::kPlanar) maxThr = precision == inf ? inf : acr::mul(acr::mul(acr::mul(precision, precision), n2.s), n2.s);
  else maxThr = precision == inf ? inf : acr::mul(precision, precision);
  if (tid == 0) {
    g.p = (int)st_in[acr::kMtN];
    nReserve = max_iter / 10; nIter = max_iter - nReserve; iter = 0;
    evaluated = skipped = exact = 0;
    mode = precision == inf; minNFA = inf; errorMax = inf; n_inl = 0; n_idx = n; stop = 0; n_trace = 0;
    for (int t = 0; t < 9 + (P::kDistortion ? 2 : 0); ++t) bestF[t] = 0;
  }
  __syncthreads();

  while (true) {
    if (tid == 0) {
      if (iter >= nIter) {
        stop = 1;
      } else {
        uint32_t s[P::kSample];
        acr::rand_sample<P::kSample>(g, (uint32_t)(mode ? n_idx : n), s);
        if constexpr (P::kPlanar) {
          double a[P::kSample], b[P::kSample], cc[P::kSample], d[P::kSample];
          for (int i = 0; i < P::kSample; ++i) {
            const uint32_t j = mode ? idx[s[i]] : s[i];
            a[i] = pts[4 * j]; b[i] = pts[4 * j + 1]; cc[i] = pts[4 * j + 2]; d[i] = pts[4 * j + 3];
          }
          if constexpr (P::kDistortion) {   // the 10-point solver's working arrays: thread 0's, in shared memory
            __shared__ acr::F10Work work;
            nb = P::fit(a, b, cc, d, models, work);
          } else {
            nb = P::fit(a, b, cc, d, models);
          }
        } else if constexpr (P::kCalibrated) {
          double a[P::kSample], b[P::kSample], cc[P::kSample], d[P::kSample];
          for (int i = 0; i < P::kSample; ++i) {
            const uint32_t j = mode ? idx[s[i]] : s[i];
            a[i] = pts[8 * j + 4]; b[i] = pts[8 * j + 5]; cc[i] = pts[8 * j + 6]; d[i] = pts[8 * j + 7];
          }
          nb = P::fit(a, b, cc, d, kinv, models);
        } else {
          double x1[3 * P::kSample], x2[3 * P::kSample];
          for (int i = 0; i < P::kSample; ++i) {
            const uint32_t j = mode ? idx[s[i]] : s[i];
            for (int t = 0; t < 3; ++t) { x1[3 * i + t] = pts[6 * j + t]; x2[3 * i + t] = pts[6 * j + 3 + t]; }
          }
          nb = P::fit(x1, x2, models);
        }
        better = 0; copy_idx = 0;
      }
    }
    __syncthreads();
    if (stop) break;
    for (int m = 0; m < nb; ++m) {
      const double* F = models + 9 * m;
      if (!mode) {   // precision mode: a model with more than 2.5 * kSample inliers switches to the a-contrario mode
        int cnt = 0;
        for (int i = tid; i < n; i += kThreads) cnt += residual<P>(F, pts, i) <= maxThr;
        cnt = block_sum(cnt, red_k);
        if (tid == 0 && cnt > 2.5 * P::kSample) mode = 1;
        __syncthreads();
        if (!mode) continue;
      }
      if (tid == 0) ++evaluated;
      if (skip_on && minNFA < inf) {
        for (int b = tid; b < kBins; b += kThreads) hist[b] = 0;
        __syncthreads();
        for (int i = tid; i < n; i += kThreads) atomicAdd(&hist[bin_of(residual<P>(F, pts, i))], 1);
        __syncthreads();
        if (tid < 32) {   // inclusive prefix counts, 17 bins per lane
          constexpr int per = (kBins + 31) / 32;
          int s = 0;
          for (int b = tid * per; b < min(kBins, (tid + 1) * per); ++b) s += hist[b];
          int incl = s;
          for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (tid >= o) incl += t; }
          int run = incl - s;
          for (int b = tid * per; b < min(kBins, (tid + 1) * per); ++b) { run += hist[b]; hist[b] = run; }
        }
        __syncthreads();
        double lb = inf; int lk = 0;
        for (int k = P::kSample + 1 + tid; k <= n; k += kThreads) {
          int lo = 0, hi = kBins - 1;   // first bin whose prefix count reaches k
          while (lo < hi) { const int mid = (lo + hi) >> 1; if (hist[mid] >= k) hi = mid; else lo = mid + 1; }
          const double v = nfa_of<P>(bin_low(lo), k, la0, loge0, lcn, lck);
          if (v < lb) { lb = v; lk = k; }
        }
        block_min(lb, lk, red_v, red_k);
        if (acr::sub(lb, 1e-9 * fmax(1.0, fabs(lb))) >= minNFA) {
          if (tid == 0) ++skipped;
          continue;
        }
      }
      if (tid == 0) ++exact;
      int N2 = 1;
      while (N2 < n) N2 <<= 1;
      unsigned long long* K = N2 <= kSmemSort ? skeys : gkeys + Q.sort_off;
      uint32_t* V = N2 <= kSmemSort ? svals : gvals + Q.sort_off;
      for (int i = tid; i < N2; i += kThreads) {
        K[i] = i < n ? (unsigned long long)__double_as_longlong(residual<P>(F, pts, i)) : ~0ull;
        V[i] = i < n ? (uint32_t)i : ~0u;
      }
      __syncthreads();
      bitonic(K, V, N2);
      double bv = inf; int bk = P::kSample;
      for (int k = P::kSample + 1 + tid; k <= n; k += kThreads) {
        const double e = __longlong_as_double((long long)K[k - 1]);
        if (!(e <= maxThr)) continue;   // sorted: the ranks with e <= maxThreshold are a prefix
        const double v = nfa_of<P>(e, k, la0, loge0, lcn, lck);
        if (lex_less(bv, bk, v, k)) { bv = v; bk = k; }
      }
      block_min(bv, bk, red_v, red_k);
      if (bv < minNFA) {   // every thread holds the same (bv, bk) and minNFA
        for (int i = tid; i < bk; i += kThreads) inl[i] = V[i];
        __syncthreads();
        if (tid == 0) {
          better = 1; minNFA = bv; n_inl = bk;
          errorMax = __longlong_as_double((long long)K[bk - 1]);
          const double* Mo = P::kCalibrated ? models + 9 * (P::kMaxModels + m) : F;   // E: the fitted model, not its F
          for (int t = 0; t < 9; ++t) bestF[t] = Mo[t];
          if constexpr (P::kDistortion) { bestF[9] = models[9 * P::kMaxModels + 2 * m]; bestF[10] = models[9 * P::kMaxModels + 2 * m + 1]; }
          if (n_trace < kTraceCap) {
            trace_all[(long long)p * kTraceCap + n_trace] = (int)iter;
            trace_nfa_all[(long long)p * kTraceCap + n_trace] = bv;
          }
          ++n_trace;
        }
      }
      __syncthreads();
    }
    if (tid == 0) {
      if (!mode && iter > nReserve * 2) stop = 1;
      else if (mode && ((better && minNFA < 0) || (iter + 1 == nIter && nReserve))) {
        if (n_inl == 0) { ++nIter; --nReserve; }
        else {
          copy_idx = 1; n_idx = n_inl;
          if (nReserve) { nIter = iter + 1 + nReserve; nReserve = 0; }
        }
      }
      ++iter;
    }
    __syncthreads();
    const bool done = stop, copy = copy_idx;
    if (done) break;
    if (copy)
      for (int i = tid; i < n_idx; i += kThreads) idx[i] = inl[i];
    __syncthreads();   // every thread has read stop / copy_idx, and the sampling list is complete, before thread 0 draws again
  }
  if (tid == 0) {
    const bool valid = minNFA < 0 && n_inl > 0;
    double Fo[9];
    for (int t = 0; t < 9; ++t) Fo[t] = bestF[t];
    double em = errorMax;
    if (valid) {   // unormalizeError: sqrt(e) / s2 (planar), sqrt(e) (bearings, calibrated)
      P::unnormalize(n1, n2, Fo);
      if constexpr (P::kPlanar) em = sqrt(em) / n2.s;
      else em = sqrt(em);
    }
    for (int t = 0; t < 9; ++t) out->model[t] = Fo[t];
    out->error_max = em; out->min_nfa = minNFA;
    out->evaluated = evaluated; out->skipped = skipped; out->exact = exact;
    out->valid = valid; out->n_inl = valid ? n_inl : 0; out->iterations = (int)iter; out->n_trace = n_trace;
    if constexpr (P::kDistortion) { reinterpret_cast<OutL*>(out)->L[0] = bestF[9]; reinterpret_cast<OutL*>(out)->L[1] = bestF[10]; }
  }
  if (mt_out) {   // thread 0's last draw is ordered before the loop's final __syncthreads
    uint32_t* so = mt_out + (long long)p * (acr::kMtN + 1);
    for (int i = tid; i < acr::kMtN; i += kThreads) so[i] = g.x[i];
    if (tid == 0) so[acr::kMtN] = (uint32_t)g.p;
  }
}

// One launch of acransac_kernel<P> over n_pairs CTAs on `st`, the kernel's arguments in order.
template <class P>
void launch(int n_pairs, cudaStream_t st, const Pair* pairs, const double* corr, const float* l10, const uint32_t* mt_state, int mt_stride,
            long long max_iter, double precision, int skip_on, double* pts_all, uint32_t* idx_all, float* logc_all,
            unsigned long long* gkeys, uint32_t* gvals, uint32_t* inliers_all, int* trace_all, double* trace_nfa_all, Out* out_all,
            uint32_t* mt_out) {
  acransac_kernel<P><<<n_pairs, kThreads, 0, st>>>(pairs, corr, l10, mt_state, mt_stride, max_iter, precision, skip_on, pts_all, idx_all,
                                                   logc_all, gkeys, gvals, inliers_all, trace_all, trace_nfa_all, out_all, mt_out);
}
// F10Policy's kernel is compiled in its own translation unit (acransac_f10.cu), so that engine.cu's module, the other policies'
// kernels among it, compiles exactly as it did before this policy.
template <>
void launch<F10Policy>(int n_pairs, cudaStream_t st, const Pair* pairs, const double* corr, const float* l10, const uint32_t* mt_state,
                       int mt_stride, long long max_iter, double precision, int skip_on, double* pts_all, uint32_t* idx_all, float* logc_all,
                       unsigned long long* gkeys, uint32_t* gvals, uint32_t* inliers_all, int* trace_all, double* trace_nfa_all, Out* out_all,
                       uint32_t* mt_out);

}  // namespace acrk

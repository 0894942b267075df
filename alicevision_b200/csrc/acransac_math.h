// Host + device building blocks of the a-contrario fundamental-matrix (planar and spherical) and homography estimations
// (acransac.cuh):
//   * std::mt19937 (libstdc++), std::uniform_int_distribution<int>(0, d) on it (GCC 13: Lemire's nearly-divisionless reduction
//     of one 32-bit draw), and the sample of robustEstimation::randSample(g, 0, range, K) as ACRANSAC draws it: Floyd's algorithm
//     with the iteration order of the std::unordered_set<std::size_t> it fills, or std::shuffle with its two-swaps-per-draw path
//     when K * 1.5 > range (range 8..10 for K = 7, range 5 for K = 4);
//   * the F kernel of RelativePoseKernel<Fundamental7PSolver, FundamentalEpipolarDistanceError, UnnormalizerT>: image-size
//     preconditioning, the 7-point solver (the 2-D null space of the epipolar rows, the cubic det(F1 + a F2) = 0 as written,
//     SolveCubicPolynomial branch for branch), the point-to-line error and the unnormalisation N2^T F N1;
//   * the spherical F kernel of RelativePoseSphericalKernel<Fundamental7PSphericalSolver, EpipolarSphericalDistanceError> for two
//     equidistant cameras: the same 7-point null space and cubic on the rows of lifted unit vectors, the error (F x1 . x2)^2;
//   * the H kernel of RelativePoseKernel<Homography4PSolver, HomographyAsymmetricError, UnnormalizerI> (point-to-point): the same
//     preconditioning, the 4-point DLT and its 1-D null space, the asymmetric transfer error and the unnormalisation N2^-1 H N1.
// The same code runs in the engine (device) and in the oracle's restated kernels (host, -ffp-contract=off), so the two differ
// only through acos / cos / pow / log10.  Device double arithmetic goes through __dmul_rn / __dadd_rn / __dsub_rn so that no
// product is contracted into an FMA.
// The null spaces are the one piece that cannot match the reference bit for bit (they come from Eigen's JacobiSVD there): here
// they are the last columns of the Householder QR of A^T.  Any basis of the same null space gives the same models up to scale
// (F: the same rank-2 matrices; H: the same matrix up to scale and sign) and the errors are scale-invariant, so models agree up to
// rounding.
#pragma once
#include <cmath>
#include <cstdint>

#ifdef __CUDACC__
#define ACR_HD __host__ __device__ __forceinline__
#else
#define ACR_HD inline
#endif

namespace acr {

constexpr int kSample = 7;      // Fundamental7PSolver::getMinimumNbRequiredSamples
constexpr int kMaxModels = 3;   // Fundamental7PSolver::getMaximumNbModels
constexpr int kMtN = 624, kMtM = 397;

ACR_HD double mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
ACR_HD double add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
ACR_HD double sub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}

// ---------------------------------------------------------------------------------------------------------------- std::mt19937
struct Mt19937 {
  uint32_t x[kMtN];
  int p;   // next word; kMtN = twist before the next draw (std::mt19937's _M_p)
};

ACR_HD void mt_seed(Mt19937& g, uint32_t seed) {
  g.x[0] = seed;
  for (int i = 1; i < kMtN; ++i) g.x[i] = 1812433253u * (g.x[i - 1] ^ (g.x[i - 1] >> 30)) + (uint32_t)i;
  g.p = kMtN;
}

ACR_HD void mt_twist(Mt19937& g) {
  const uint32_t up = 0x80000000u, lo = 0x7fffffffu, a = 0x9908b0dfu;
  for (int k = 0; k < kMtN - kMtM; ++k) {
    const uint32_t y = (g.x[k] & up) | (g.x[k + 1] & lo);
    g.x[k] = g.x[k + kMtM] ^ (y >> 1) ^ ((y & 1u) ? a : 0u);
  }
  for (int k = kMtN - kMtM; k < kMtN - 1; ++k) {
    const uint32_t y = (g.x[k] & up) | (g.x[k + 1] & lo);
    g.x[k] = g.x[k + (kMtM - kMtN)] ^ (y >> 1) ^ ((y & 1u) ? a : 0u);
  }
  const uint32_t y = (g.x[kMtN - 1] & up) | (g.x[0] & lo);
  g.x[kMtN - 1] = g.x[kMtM - 1] ^ (y >> 1) ^ ((y & 1u) ? a : 0u);
  g.p = 0;
}

ACR_HD uint32_t mt_next(Mt19937& g) {
  if (g.p >= kMtN) mt_twist(g);
  uint32_t z = g.x[g.p++];
  z ^= z >> 11;
  z ^= (z << 7) & 0x9d2c5680u;
  z ^= (z << 15) & 0xefc60000u;
  z ^= z >> 18;
  return z;
}

// uniform integer in [0, range) for 1 <= range < 2^32: uniform_int_distribution<>(0, range - 1) on a 32-bit engine
ACR_HD uint32_t uniform_below(Mt19937& g, uint32_t range) {
  uint64_t prod = (uint64_t)mt_next(g) * range;
  uint32_t low = (uint32_t)prod;
  if (low < range) {
    const uint32_t th = (0u - range) % range;
    while (low < th) {
      prod = (uint64_t)mt_next(g) * range;
      low = (uint32_t)prod;
    }
  }
  return (uint32_t)(prod >> 32);
}

// The K positions in [0, range) that randSample(g, 0, range, K) returns, in its order; range > K.
template <int K>
ACR_HD void rand_sample(Mt19937& g, uint32_t range, uint32_t out[K]) {
  if (K * 1.5 > range) {
    // std::shuffle of iota(range) (range 8..10 for K = 7, 5 for K = 4): a leading single swap when range is even, then two swap
    // positions per draw
    uint32_t a[K * 3 / 2];
    for (uint32_t i = 0; i < range; ++i) a[i] = i;
    uint32_t i = 1;
    if (range % 2 == 0) {
      const uint32_t j = uniform_below(g, 2);
      const uint32_t t = a[i]; a[i] = a[j]; a[j] = t; ++i;
    }
    while (i != range) {
      const uint32_t sr = i + 1;
      const uint32_t x = uniform_below(g, sr * (sr + 1));
      uint32_t j = x / (sr + 1), t = a[i]; a[i] = a[j]; a[j] = t; ++i;
      j = x % (sr + 1); t = a[i]; a[i] = a[j]; a[j] = t; ++i;
    }
    for (int k = 0; k < K; ++k) out[k] = a[k];
    return;
  }
  // Floyd's algorithm into a std::unordered_set<std::size_t>: identity hash, 13 buckets from the first insertion on (libstdc++'s
  // prime rehash policy; no rehash below 14 elements).  Its iteration order is the node list: a key goes in front of the first
  // node of its bucket, or at the front of the list when its bucket is empty.
  uint32_t list[K];
  int cnt = 0;
  for (uint32_t d = range - K; d < range; ++d) {
    const uint32_t t = uniform_below(g, d + 1);
    bool seen = false;
    for (int q = 0; q < cnt; ++q) seen |= (list[q] == t);
    const uint32_t key = seen ? d : t;
    int pos = 0;
    for (int q = 0; q < cnt; ++q)
      if (list[q] % 13u == key % 13u) { pos = q; break; }
    for (int q = cnt; q > pos; --q) list[q] = list[q - 1];
    list[pos] = key;
    ++cnt;
  }
  for (int k = 0; k < K; ++k) out[k] = list[k];
}

// randSample(g, 0, range, 7), the Fundamental7PSolver sample; range >= 8
ACR_HD void rand_sample7(Mt19937& g, uint32_t range, uint32_t out[kSample]) { rand_sample<kSample>(g, range, out); }

// ---------------------------------------------------------------------------------------------------------------- F kernel
// preconditionerFromImageSize: N = [s 0 -w/2 s; 0 s -h/2 s; 0 0 1], s = 1 / sqrt(w h) (w h an int product; -.5f * w in float)
struct Norm { double s, tx, ty; };
ACR_HD Norm precondition(int w, int h) {
  Norm n;
  n.s = 1.0 / sqrt((double)(w * h));
  n.tx = mul((double)(-.5f * w), n.s);
  n.ty = mul(mul(-.5, (double)h), n.s);
  return n;
}
ACR_HD double norm_x(const Norm& n, double x) { return add(mul(n.s, x), n.tx); }
ACR_HD double norm_y(const Norm& n, double y) { return add(mul(n.s, y), n.ty); }

// FundamentalEpipolarDistanceError on normalised points: (F x . y)^2 / ((F x)_0^2 + (F x)_1^2)
ACR_HD double epipolar_error(const double* F, double x1, double y1, double x2, double y2) {
  const double l0 = add(add(mul(F[0], x1), mul(F[1], y1)), F[2]);
  const double l1 = add(add(mul(F[3], x1), mul(F[4], y1)), F[5]);
  const double l2 = add(add(mul(F[6], x1), mul(F[7], y1)), F[8]);
  const double d = add(add(mul(l0, x2), mul(l1, y2)), l2);
  return mul(d, d) / add(mul(l0, l0), mul(l1, l1));
}

// SolveCubicPolynomial(coeffs, roots) of numeric/polynomial.hpp, restated branch for branch
ACR_HD int solve_cubic(const double P[4], double x[3]) {
  if (P[0] == 0.0) return 0;
  const double a = P[2] / P[3], b = P[1] / P[3], c = P[0] / P[3];
  const double q = sub(mul(a, a), mul(3.0, b));
  const double r = add(sub(mul(mul(mul(2.0, a), a), a), mul(mul(9.0, a), b)), mul(27.0, c));
  const double Q = q / 9, R = r / 54;
  const double Q3 = mul(mul(Q, Q), Q), R2 = mul(R, R);
  const double CR2 = mul(mul(729.0, r), r), CQ3 = mul(mul(mul(2916.0, q), q), q);
  const double a3 = a / 3;
  if (R == 0 && Q == 0) {
    x[0] = x[1] = x[2] = -a / 3;
    return 3;
  } else if (CR2 == CQ3) {
    const double sq = sqrt(Q);
    if (R > 0) {
      x[0] = sub(mul(-2.0, sq), a3); x[1] = sub(sq, a3); x[2] = sub(sq, a3);
    } else {
      x[0] = sub(-sq, a3); x[1] = sub(-sq, a3); x[2] = sub(mul(2.0, sq), a3);
    }
    return 3;
  } else if (CR2 < CQ3) {
    const double sq = sqrt(Q);
    const double sq3 = mul(mul(sq, sq), sq);
    const double theta = acos(R / sq3);
    const double nrm = mul(-2.0, sq);
    const double pi2 = mul(2.0, M_PI);
    x[0] = sub(mul(nrm, cos(theta / 3)), a3);
    x[1] = sub(mul(nrm, cos(add(theta, pi2) / 3)), a3);
    x[2] = sub(mul(nrm, cos(sub(theta, pi2) / 3)), a3);
    double t;
    if (x[0] > x[1]) { t = x[0]; x[0] = x[1]; x[1] = t; }
    if (x[1] > x[2]) {
      t = x[1]; x[1] = x[2]; x[2] = t;
      if (x[0] > x[1]) { t = x[0]; x[0] = x[1]; x[1] = t; }
    }
    return 3;
  }
  const double sgnR = (R >= 0 ? 1 : -1);
  const double A = mul(-sgnR, pow(add(fabs(R), sqrt(sub(R2, Q3))), 1.0 / 3.0));
  const double B = Q / A;
  x[0] = sub(add(A, B), a3);
  return 1;
}

// The null space of an R x 9 system (R = 7: the epipolar rows, R = 8: the homography DLT rows): the last 9 - R columns of Q in
// A^T = Q R (Householder, no pivoting; a column that is already zero below the diagonal gets no reflection).  N[0] = Q e8,
// N[1] = Q e7, unit norm.  A rank-deficient system has a larger null space; the columns returned then lie in it as rounding sets.
template <int R>
ACR_HD void nullspace(const double A[R][9], double N[9 - R][9]) {
  double M[9][R];   // A^T
  for (int r = 0; r < 9; ++r)
    for (int c = 0; c < R; ++c) M[r][c] = A[c][r];
  double V[R][9];   // Householder vectors (zero above their diagonal)
  double vn[R];     // their squared norms (0: no reflection)
  for (int j = 0; j < R; ++j) {
    double s = 0;
    for (int r = j; r < 9; ++r) s = add(s, mul(M[r][j], M[r][j]));
    const double nrm = sqrt(s);
    const double alpha = M[j][j] >= 0 ? -nrm : nrm;
    for (int r = 0; r < 9; ++r) V[j][r] = r < j ? 0.0 : M[r][j];
    V[j][j] = sub(V[j][j], alpha);
    double v2 = 0;
    for (int r = j; r < 9; ++r) v2 = add(v2, mul(V[j][r], V[j][r]));
    vn[j] = v2;
    if (v2 == 0) continue;
    for (int c = j; c < R; ++c) {
      double d = 0;
      for (int r = j; r < 9; ++r) d = add(d, mul(V[j][r], M[r][c]));
      const double f = mul(2.0, d) / v2;
      for (int r = j; r < 9; ++r) M[r][c] = sub(M[r][c], mul(f, V[j][r]));
    }
  }
  for (int q = 0; q < 9 - R; ++q)
    for (int r = 0; r < 9; ++r) N[q][r] = r == 8 - q ? 1.0 : 0.0;
  for (int j = R - 1; j >= 0; --j) {
    if (vn[j] == 0) continue;
    for (int q = 0; q < 9 - R; ++q) {
      double d = 0;
      for (int r = j; r < 9; ++r) d = add(d, mul(V[j][r], N[q][r]));
      const double g = mul(2.0, d) / vn[j];
      for (int r = j; r < 9; ++r) N[q][r] = sub(N[q][r], mul(g, V[j][r]));
    }
  }
}

// The 7-point solver of Fundamental7PSolver (kSpherical = false) and Fundamental7PSphericalSolver (true); returns the number of
// models (0..3) written row-major to F[m * 9].  Only the epipolar rows differ:
//   planar     encodeEpipolarEquation on 7 normalised correspondences (p0[i], p1[i]) <-> (p2[i], p3[i]);
//   spherical  encodeEpipolarSphericalEquation on 7 bearing pairs x1 = p0[3 i + a] <-> x2 = p2[3 i + a], A(i, 3 a + b) = x2_a x1_b
//              (p1, p3 unused);
// then both take the 2-D null space F1, F2 of the rows, the cubic det(F1 + a F2) = 0 and its real roots.  One function rather than
// a shared tail: the F kernel calls it at the depth fit7 had, which keeps its device code what it was before the spherical solver.
template <bool kSpherical>
ACR_HD int fit7_solve(const double* p0, const double* p1, const double* p2, const double* p3, double* F) {
  double A[kSample][9];
  if constexpr (!kSpherical) {
    const double *x1 = p0, *y1 = p1, *x2 = p2, *y2 = p3;
    for (int i = 0; i < kSample; ++i) {   // encodeEpipolarEquation
      A[i][0] = mul(x2[i], x1[i]); A[i][1] = mul(x2[i], y1[i]); A[i][2] = x2[i];
      A[i][3] = mul(y2[i], x1[i]); A[i][4] = mul(y2[i], y1[i]); A[i][5] = y2[i];
      A[i][6] = x1[i]; A[i][7] = y1[i]; A[i][8] = 1.0;
    }
  } else {
    for (int i = 0; i < kSample; ++i)     // encodeEpipolarSphericalEquation
      for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) A[i][3 * a + b] = mul(p2[3 * i + a], p0[3 * i + b]);
  }
  double f12[2][9];
  nullspace<kSample>(A, f12);
  const double* f1 = f12[0];
  const double* f2 = f12[1];
  const double a = f1[0], j = f2[0], b = f1[1], k = f2[1], c = f1[2], l = f2[2], d = f1[3], m = f2[3], e = f1[4], n = f2[4],
               f = f1[5], o = f2[5], g = f1[6], p = f2[6], h = f1[7], q = f2[7], i = f1[8], r = f2[8];
#define ACR_T(u, v, w) mul(mul(u, v), w)
  double P[4];
  P[0] = sub(sub(sub(add(add(ACR_T(a, e, i), ACR_T(b, f, g)), ACR_T(c, d, h)), ACR_T(a, f, h)), ACR_T(b, d, i)), ACR_T(c, e, g));
  {
    double s = ACR_T(a, e, r);
    s = add(s, ACR_T(a, i, n)); s = add(s, ACR_T(b, f, p)); s = add(s, ACR_T(b, g, o)); s = add(s, ACR_T(c, d, q));
    s = add(s, ACR_T(c, h, m)); s = add(s, ACR_T(d, h, l)); s = add(s, ACR_T(e, i, j)); s = add(s, ACR_T(f, g, k));
    s = sub(s, ACR_T(a, f, q)); s = sub(s, ACR_T(a, h, o)); s = sub(s, ACR_T(b, d, r)); s = sub(s, ACR_T(b, i, m));
    s = sub(s, ACR_T(c, e, p)); s = sub(s, ACR_T(c, g, n)); s = sub(s, ACR_T(d, i, k)); s = sub(s, ACR_T(e, g, l));
    s = sub(s, ACR_T(f, h, j));
    P[1] = s;
  }
  {
    double s = ACR_T(a, n, r);
    s = add(s, ACR_T(b, o, p)); s = add(s, ACR_T(c, m, q)); s = add(s, ACR_T(d, l, q)); s = add(s, ACR_T(e, j, r));
    s = add(s, ACR_T(f, k, p)); s = add(s, ACR_T(g, k, o)); s = add(s, ACR_T(h, l, m)); s = add(s, ACR_T(i, j, n));
    s = sub(s, ACR_T(a, o, q)); s = sub(s, ACR_T(b, m, r)); s = sub(s, ACR_T(c, n, p)); s = sub(s, ACR_T(d, k, r));
    s = sub(s, ACR_T(e, l, p)); s = sub(s, ACR_T(f, j, q)); s = sub(s, ACR_T(g, l, n)); s = sub(s, ACR_T(h, j, o));
    s = sub(s, ACR_T(i, k, m));
    P[2] = s;
  }
  P[3] = sub(sub(sub(add(add(ACR_T(j, n, r), ACR_T(k, o, p)), ACR_T(l, m, q)), ACR_T(j, o, q)), ACR_T(k, m, r)), ACR_T(l, n, p));
#undef ACR_T
  double roots[3];
#ifdef ACR_REFERENCE_CUBIC
  const int nb = ACR_REFERENCE_CUBIC(P, roots);
#else
  const int nb = solve_cubic(P, roots);
#endif
  for (int kk = 0; kk < nb; ++kk)
    for (int t = 0; t < 9; ++t) F[kk * 9 + t] = add(f1[t], mul(roots[kk], f2[t]));
  return nb;
}

// Fundamental7PSolver::solve on 7 normalised correspondences (x1[i], y1[i]) <-> (x2[i], y2[i])
ACR_HD int fit7(const double* x1, const double* y1, const double* x2, const double* y2, double* F) {
  return fit7_solve<false>(x1, y1, x2, y2, F);
}

// ---------------------------------------------------------------------------------------------------------------- spherical F kernel
// RelativePoseSphericalKernel<Fundamental7PSphericalSolver, EpipolarSphericalDistanceError>: correspondences are the lifted unit
// vectors x1, x2 of two equidistant cameras (third component anywhere in [-1, 1]); no normalisation, logalpha0 = pi,
// errorVectorDimension = 2, thresholdNormalizer = 1, unormalizeError = sqrt.

// Fundamental7PSphericalSolver::solve on 7 bearing pairs x1[3 i + a] <-> x2[3 i + a]; returns the number of models (0..3)
ACR_HD int fit7s(const double* x1, const double* x2, double* F) { return fit7_solve<true>(x1, nullptr, x2, nullptr, F); }

// EpipolarSphericalDistanceError: (F x1 . x2)^2
ACR_HD double spherical_error(const double* F, const double* x1, const double* x2) {
  const double l0 = add(add(mul(F[0], x1[0]), mul(F[1], x1[1])), mul(F[2], x1[2]));
  const double l1 = add(add(mul(F[3], x1[0]), mul(F[4], x1[1])), mul(F[5], x1[2]));
  const double l2 = add(add(mul(F[6], x1[0]), mul(F[7], x1[1])), mul(F[8], x1[2]));
  const double d = add(add(mul(l0, x2[0]), mul(l1, x2[1])), mul(l2, x2[2]));
  return mul(d, d);
}

// UnnormalizerT: F <- N2^T F N1
ACR_HD void unnormalize(const Norm& n1, const Norm& n2, double F[9]) {
  const double N1[9] = {n1.s, 0, n1.tx, 0, n1.s, n1.ty, 0, 0, 1};
  const double N2t[9] = {n2.s, 0, 0, 0, n2.s, 0, n2.tx, n2.ty, 1};
  double T[9], O[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) T[r * 3 + c] = add(add(mul(F[r * 3], N1[c]), mul(F[r * 3 + 1], N1[3 + c])), mul(F[r * 3 + 2], N1[6 + c]));
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) O[r * 3 + c] = add(add(mul(N2t[r * 3], T[c]), mul(N2t[r * 3 + 1], T[3 + c])), mul(N2t[r * 3 + 2], T[6 + c]));
  for (int t = 0; t < 9; ++t) F[t] = O[t];
}

// ---------------------------------------------------------------------------------------------------------------- H kernel
// RelativePoseKernel<Homography4PSolver, HomographyAsymmetricError, UnnormalizerI> (point-to-point): the same preconditioning, the
// 4-point DLT, the asymmetric transfer error and the unnormalisation N2^-1 H N1.
constexpr int kSampleH = 4;      // Homography4PSolver::getMinimumNbRequiredSamples
constexpr int kMaxModelsH = 1;   // Homography4PSolver::getMaximumNbModels

// Homography4PSolver::solve on 4 normalised correspondences: the 8 DLT rows of buildActionMatrix (the non-zero rows of the
// reference's Mat16_9), their null space, mapped row-major to H[9] (x2 ~ H x1).  Always one model: a degenerate sample
// (duplicated or collinear points) has a null space of dimension 2 or more, and the vector taken from it is set by rounding.
ACR_HD int fit4(const double* x1, const double* y1, const double* x2, const double* y2, double* H) {
  double L[2 * kSampleH][9];
  for (int i = 0; i < kSampleH; ++i) {
    double* a = L[2 * i];
    double* b = L[2 * i + 1];
    a[0] = x1[i]; a[1] = y1[i]; a[2] = 1.0; a[3] = 0.0; a[4] = 0.0; a[5] = 0.0;
    a[6] = mul(-x2[i], x1[i]); a[7] = mul(-x2[i], y1[i]); a[8] = -x2[i];
    b[0] = 0.0; b[1] = 0.0; b[2] = 0.0; b[3] = x1[i]; b[4] = y1[i]; b[5] = 1.0;
    b[6] = mul(-y2[i], x1[i]); b[7] = mul(-y2[i], y1[i]); b[8] = -y2[i];
  }
  double h[1][9];
  nullspace<2 * kSampleH>(L, h);
  for (int t = 0; t < 9; ++t) H[t] = h[0][t];
  return 1;
}

// HomographyAsymmetricError on normalised points: |x2 - dehomogenised(H (x1, 1))|^2.  A zero third component gives inf or NaN.
ACR_HD double homography_error(const double* H, double x1, double y1, double x2, double y2) {
  const double u = add(add(mul(H[0], x1), mul(H[1], y1)), H[2]);
  const double v = add(add(mul(H[3], x1), mul(H[4], y1)), H[5]);
  const double w = add(add(mul(H[6], x1), mul(H[7], y1)), H[8]);
  const double dx = sub(x2, u / w), dy = sub(y2, v / w);
  return add(mul(dx, dx), mul(dy, dy));
}

// M^-1 of a 3 x 3 row-major matrix by cofactors: R(i, j) = C(j, i) / det, det expanded along the first column
ACR_HD void inverse3(const double M[9], double R[9]) {
  double C[9];   // cofactors C(i, j) = M(i1, j1) M(i2, j2) - M(i1, j2) M(i2, j1), i1 = i + 1, i2 = i + 2 (mod 3)
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
      C[i * 3 + j] = sub(mul(M[i1 * 3 + j1], M[i2 * 3 + j2]), mul(M[i1 * 3 + j2], M[i2 * 3 + j1]));
    }
  const double det = add(add(mul(C[0], M[0]), mul(C[3], M[3])), mul(C[6], M[6]));
  const double inv = 1.0 / det;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) R[i * 3 + j] = mul(C[j * 3 + i], inv);
}

// UnnormalizerI: H <- N2^-1 H N1
ACR_HD void unnormalize_h(const Norm& n1, const Norm& n2, double H[9]) {
  const double N1[9] = {n1.s, 0, n1.tx, 0, n1.s, n1.ty, 0, 0, 1};
  const double N2[9] = {n2.s, 0, n2.tx, 0, n2.s, n2.ty, 0, 0, 1};
  double N2i[9], T[9];
  inverse3(N2, N2i);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) T[r * 3 + c] = add(add(mul(N2i[r * 3], H[c]), mul(N2i[r * 3 + 1], H[3 + c])), mul(N2i[r * 3 + 2], H[6 + c]));
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) H[r * 3 + c] = add(add(mul(T[r * 3], N1[c]), mul(T[r * 3 + 1], N1[3 + c])), mul(T[r * 3 + 2], N1[6 + c]));
}

// logalpha0 of the point-to-point error: log10(pi / (w2 h2) / s2^2), the unit circle over the image area in normalised units
ACR_HD double logalpha0_h(int w2, int h2, const Norm& n2) { return log10(M_PI / mul((double)w2, (double)h2) / mul(n2.s, n2.s)); }

}  // namespace acr

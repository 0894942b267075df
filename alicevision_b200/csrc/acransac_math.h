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
//     preconditioning, the 4-point DLT and its 1-D null space, the asymmetric transfer error and the unnormalisation N2^-1 H N1;
//   * the E kernel of RelativePoseKernel_K<Essential5PSolver, FundamentalEpipolarDistanceError> for two pinhole cameras: the 5-point
//     solver (null space, constraint matrix, full-pivot LU, action matrix, and Eigen's RealSchur / EigenSolver restated for it)
//     on K^-1 x, and F = K_J^-T E K_I^-1 for the point-to-line error on pixels.
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

// ---------------------------------------------------------------------------------------------------------------- E kernel
// RelativePoseKernel_K<Essential5PSolver, FundamentalEpipolarDistanceError, Mat3Model> of two pinhole cameras: the fit runs on
// K^-1 x (applyTransformationToPoints, once per pair), the residual is the point-to-line error of F = K_J^-T E K_I^-1 on the pixel
// points; no normaliser (thresholdNormalizer = 1, unormalizeError = sqrt), errorVectorDimension = 0.5,
// logalpha0 = log10(2 D / A * .5) of the raw w_J, h_J.
constexpr int kSampleE = 5;       // Essential5PSolver::getMinimumNbRequiredSamples
constexpr int kMaxModelsE = 10;   // Essential5PSolver::getMaximumNbModels

ACR_HD double logalpha0_e(int w2, int h2) {
  const double D = sqrt(add(mul((double)w2, (double)w2), mul((double)h2, (double)h2)));
  const double A = mul((double)w2, (double)h2);
  return log10(mul(mul(2.0, D) / A, .5));
}

// applyTransformationToPoints(x, T): (T (x, y, 1))_{0,1} / (T (x, y, 1))_2
ACR_HD void transform_point(const double T[9], double x, double y, double& u, double& v) {
  const double a = add(add(mul(T[0], x), mul(T[1], y)), T[2]);
  const double b = add(add(mul(T[3], x), mul(T[4], y)), T[5]);
  const double c = add(add(mul(T[6], x), mul(T[7], y)), T[8]);
  u = a / c;
  v = b / c;
}

// fundamentalFromEssential: F = K_J^-T E K_I^-1, formed as (K_J^-T E) K_I^-1; all three row-major
ACR_HD void fundamental_from_essential(const double E[9], const double KIinv[9], const double KJinv[9], double F[9]) {
  double T[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) T[r * 3 + c] = add(add(mul(KJinv[r], E[c]), mul(KJinv[3 + r], E[3 + c])), mul(KJinv[6 + r], E[6 + c]));
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) F[r * 3 + c] = add(add(mul(T[r * 3], KIinv[c]), mul(T[r * 3 + 1], KIinv[3 + c])), mul(T[r * 3 + 2], KIinv[6 + c]));
}

namespace e5 {
constexpr int N = 10;   // the action matrix is 10 x 10
constexpr double kEps = 2.220446049250313e-16;       // NumTraits<double>::epsilon()
constexpr double kMin = 2.2250738585072014e-308;     // std::numeric_limits<double>::min()

// Essential5PSolver's monomials (Pc::coef_*): cubic 0..9, then xx xy yy xz yz zz x y z 1 (10..19).  Degree-1 polynomials (the
// entries of E) are kept as their (x, y, z, 1) coefficients and degree-2 ones as their coefficients 10..19: o1 and o2 read nothing
// else, so this is the reference's arithmetic on its non-zero entries.
enum { XXX, XXY, XYY, YYY, XXZ, XYZ, YYZ, XZZ, YZZ, ZZZ };
enum { XX, XY, YY, XZ, YZ, ZZ, X1, Y1, Z1, ONE };   // degree 2, offset 10
enum { X, Y, Z, W };                                 // degree 1

// o1: degree 1 x degree 1
ACR_HD void o1(const double* a, const double* b, double* r) {
  r[XX] = mul(a[X], b[X]);
  r[XY] = add(mul(a[X], b[Y]), mul(a[Y], b[X]));
  r[XZ] = add(mul(a[X], b[Z]), mul(a[Z], b[X]));
  r[YY] = mul(a[Y], b[Y]);
  r[YZ] = add(mul(a[Y], b[Z]), mul(a[Z], b[Y]));
  r[ZZ] = mul(a[Z], b[Z]);
  r[X1] = add(mul(a[X], b[W]), mul(a[W], b[X]));
  r[Y1] = add(mul(a[Y], b[W]), mul(a[W], b[Y]));
  r[Z1] = add(mul(a[Z], b[W]), mul(a[W], b[Z]));
  r[ONE] = mul(a[W], b[W]);
}

// o2: degree 2 x degree 1, all 20 coefficients
ACR_HD void o2(const double* a, const double* b, double* r) {
  r[XXX] = mul(a[XX], b[X]);
  r[XXY] = add(mul(a[XX], b[Y]), mul(a[XY], b[X]));
  r[XXZ] = add(mul(a[XX], b[Z]), mul(a[XZ], b[X]));
  r[XYY] = add(mul(a[XY], b[Y]), mul(a[YY], b[X]));
  r[XYZ] = add(add(mul(a[XY], b[Z]), mul(a[YZ], b[X])), mul(a[XZ], b[Y]));
  r[XZZ] = add(mul(a[XZ], b[Z]), mul(a[ZZ], b[X]));
  r[YYY] = mul(a[YY], b[Y]);
  r[YYZ] = add(mul(a[YY], b[Z]), mul(a[YZ], b[Y]));
  r[YZZ] = add(mul(a[YZ], b[Z]), mul(a[ZZ], b[Y]));
  r[ZZZ] = mul(a[ZZ], b[Z]);
  r[10 + XX] = add(mul(a[XX], b[W]), mul(a[X1], b[X]));
  r[10 + XY] = add(add(mul(a[XY], b[W]), mul(a[X1], b[Y])), mul(a[Y1], b[X]));
  r[10 + XZ] = add(add(mul(a[XZ], b[W]), mul(a[X1], b[Z])), mul(a[Z1], b[X]));
  r[10 + YY] = add(mul(a[YY], b[W]), mul(a[Y1], b[Y]));
  r[10 + YZ] = add(add(mul(a[YZ], b[W]), mul(a[Y1], b[Z])), mul(a[Z1], b[Y]));
  r[10 + ZZ] = add(mul(a[ZZ], b[W]), mul(a[Z1], b[Z]));
  r[10 + X1] = add(mul(a[X1], b[W]), mul(a[ONE], b[X]));
  r[10 + Y1] = add(mul(a[Y1], b[W]), mul(a[ONE], b[Y]));
  r[10 + Z1] = add(mul(a[Z1], b[W]), mul(a[ONE], b[Z]));
  r[10 + ONE] = mul(a[ONE], b[W]);
}

// fivePointsPolynomialConstraints: the 10 x 20 matrix of det(E) = 0 (row 0) and 2 E E^T E - tr(E E^T) E = 0 (rows 1..9, (i, j)
// row-major), E = x B0 + y B1 + z B2 + B3 with B_c the basis columns (Eb[t][c], t = 3 i + j)
ACR_HD void constraints(const double Eb[9][4], double M[N][20]) {
  double a[10], b[10], r0[20], r1[20], r2[20];
  const int det[3][5] = {{1, 5, 2, 4, 6}, {2, 3, 0, 5, 7}, {0, 4, 1, 3, 8}};   // o2(o1(E_p, E_q) - o1(E_r, E_s), E_t)
  double* r[3] = {r0, r1, r2};
  for (int u = 0; u < 3; ++u) {
    o1(Eb[det[u][0]], Eb[det[u][1]], a);
    o1(Eb[det[u][2]], Eb[det[u][3]], b);
    for (int t = 0; t < 10; ++t) a[t] = sub(a[t], b[t]);
    o2(a, Eb[det[u][4]], r[u]);
  }
  for (int t = 0; t < 20; ++t) M[0][t] = add(add(r0[t], r1[t]), r2[t]);
  double L[3][3][10];   // E E^T (upper triangle computed, mirrored), then its diagonal less half its trace
  for (int i = 0; i < 3; ++i)
    for (int j = i; j < 3; ++j) {
      o1(Eb[3 * i], Eb[3 * j], L[i][j]);
      o1(Eb[3 * i + 1], Eb[3 * j + 1], a);
      o1(Eb[3 * i + 2], Eb[3 * j + 2], b);
      for (int t = 0; t < 10; ++t) L[i][j][t] = add(add(L[i][j][t], a[t]), b[t]);
    }
  for (int i = 1; i < 3; ++i)
    for (int j = 0; j < i; ++j)
      for (int t = 0; t < 10; ++t) L[i][j][t] = L[j][i][t];
  for (int t = 0; t < 10; ++t) {
    const double tr = mul(0.5, add(add(L[0][0][t], L[1][1][t]), L[2][2][t]));
    for (int i = 0; i < 3; ++i) L[i][i][t] = sub(L[i][i][t], tr);
  }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      o2(L[i][0], Eb[j], r0);
      o2(L[i][1], Eb[3 + j], r1);
      o2(L[i][2], Eb[6 + j], r2);
      for (int t = 0; t < 20; ++t) M[1 + 3 * i + j][t] = add(add(r0[t], r1[t]), r2[t]);
    }
}

// FullPivLU<Mat10>(M[:, 0:10]).solve(M[:, 10:20]) into X: complete pivoting on the largest |entry| of the remaining corner (the first
// in column-major order on a tie), a zero corner ends the factorisation, the rank counts the pivots above |max pivot| * 10 eps, and
// the unknowns of the columns past the rank are 0.  The substitutions accumulate in index order.
ACR_HD void lu_solve(double M[N][20], double X[N][N]) {
  int colT[N], nz = N;
  double maxpivot = 0;
  for (int k = 0; k < N; ++k) {
    int br = k, bc = k;
    double big = fabs(M[k][k]);
    for (int c = k; c < N; ++c)
      for (int r = k; r < N; ++r)
        if (fabs(M[r][c]) > big) { big = fabs(M[r][c]); br = r; bc = c; }
    if (big == 0) {
      nz = k;
      for (int i = k; i < N; ++i) colT[i] = i;
      break;
    }
    if (big > maxpivot) maxpivot = big;
    colT[k] = bc;
    if (br != k)
      for (int c = 0; c < 20; ++c) { const double t = M[k][c]; M[k][c] = M[br][c]; M[br][c] = t; }   // the right side moves with P
    if (bc != k)
      for (int r = 0; r < N; ++r) { const double t = M[r][k]; M[r][k] = M[r][bc]; M[r][bc] = t; }
    for (int r = k + 1; r < N; ++r) M[r][k] = M[r][k] / M[k][k];
    for (int r = k + 1; r < N; ++r)
      for (int c = k + 1; c < N; ++c) M[r][c] = sub(M[r][c], mul(M[r][k], M[k][c]));
  }
  const double thr = mul(maxpivot, mul((double)N, kEps));
  int rank = 0;
  for (int i = 0; i < nz; ++i) rank += fabs(M[i][i]) > thr;
  int q[N];   // permutationQ().indices()
  for (int i = 0; i < N; ++i) q[i] = i;
  for (int k = 0; k < N; ++k) { const int t = q[k]; q[k] = q[colT[k]]; q[colT[k]] = t; }
  for (int j = 0; j < N; ++j) {
    double c[N];
    for (int i = 0; i < N; ++i) c[i] = M[i][10 + j];
    for (int i = 1; i < N; ++i)   // unit lower
      for (int k = 0; k < i; ++k) c[i] = sub(c[i], mul(M[i][k], c[k]));
    for (int i = rank - 1; i >= 0; --i) {   // upper, on the leading rank x rank block
      for (int k = i + 1; k < rank; ++k) c[i] = sub(c[i], mul(M[i][k], c[k]));
      c[i] = c[i] / M[i][i];
    }
    for (int i = 0; i < N; ++i) X[q[i]][j] = i < rank ? c[i] : 0.0;
  }
}

// Householder::makeHouseholder of the real n-vector v: essential part ess[n - 1], tau, beta
ACR_HD void make_householder(const double* v, int n, double* ess, double& tau, double& beta) {
  double tail = 0;
  for (int i = 1; i < n; ++i) tail = add(tail, mul(v[i], v[i]));
  const double c0 = v[0];
  if (tail <= kMin) {
    tau = 0; beta = c0;
    for (int i = 1; i < n; ++i) ess[i - 1] = 0;
  } else {
    beta = sqrt(add(mul(c0, c0), tail));
    if (c0 >= 0) beta = -beta;
    for (int i = 1; i < n; ++i) ess[i - 1] = v[i] / sub(c0, beta);
    tau = sub(beta, c0) / beta;
  }
}

// applyHouseholderOnTheLeft / OnTheRight of (ess (length m - 1), tau) to the rows r0..r0+m-1, columns c0..c1 (left) or the columns
// c0..c0+m-1, rows r0..r1 (right) of A
ACR_HD void house_left(double A[N][N], int r0, int m, int c0, int c1, const double* ess, double tau) {
  if (m == 1) {
    for (int c = c0; c <= c1; ++c) A[r0][c] = mul(A[r0][c], sub(1.0, tau));
    return;
  }
  if (tau == 0) return;
  for (int c = c0; c <= c1; ++c) {
    double t = mul(ess[0], A[r0 + 1][c]);
    for (int i = 1; i < m - 1; ++i) t = add(t, mul(ess[i], A[r0 + 1 + i][c]));
    t = add(t, A[r0][c]);
    A[r0][c] = sub(A[r0][c], mul(tau, t));
    for (int i = 0; i < m - 1; ++i) A[r0 + 1 + i][c] = sub(A[r0 + 1 + i][c], mul(mul(tau, ess[i]), t));
  }
}
ACR_HD void house_right(double A[N][N], int c0, int m, int r0, int r1, const double* ess, double tau) {
  if (m == 1) {
    for (int r = r0; r <= r1; ++r) A[r][c0] = mul(A[r][c0], sub(1.0, tau));
    return;
  }
  if (tau == 0) return;
  for (int r = r0; r <= r1; ++r) {
    double t = mul(A[r][c0 + 1], ess[0]);
    for (int j = 1; j < m - 1; ++j) t = add(t, mul(A[r][c0 + 1 + j], ess[j]));
    t = add(t, A[r][c0]);
    A[r][c0] = sub(A[r][c0], mul(tau, t));
    const double tt = mul(tau, t);
    for (int j = 0; j < m - 1; ++j) A[r][c0 + 1 + j] = sub(A[r][c0 + 1 + j], mul(tt, ess[j]));
  }
}

// JacobiRotation::makeGivens(p, q) (real, no r)
ACR_HD void make_givens(double p, double q, double& c, double& s) {
  if (q == 0) {
    c = p < 0 ? -1.0 : 1.0; s = 0;
  } else if (p == 0) {
    c = 0; s = q < 0 ? 1.0 : -1.0;
  } else if (fabs(p) > fabs(q)) {
    const double t = q / p;
    double u = sqrt(add(1.0, mul(t, t)));
    if (p < 0) u = -u;
    c = 1.0 / u; s = mul(-t, c);
  } else {
    const double t = p / q;
    double u = sqrt(add(1.0, mul(t, t)));
    if (q < 0) u = -u;
    s = -1.0 / u; c = mul(-t, s);
  }
}

// apply_rotation_in_the_plane(x, y, (c, s')) with s' = -s, as applyOnTheLeft(rot.adjoint()) and applyOnTheRight(rot) both reduce to
// for a real rotation: x <- c x - s y, y <- s x + c y
ACR_HD void rotate(double& x, double& y, double c, double s) {
  const double xi = x, yi = y;
  x = add(mul(c, xi), mul(-s, yi));
  y = add(mul(s, xi), mul(c, yi));
}

// RealSchur<Mat10>::compute(A, computeU = true) on the action matrix: scale by max |A|, Householder Hessenberg reduction (and its Q
// accumulated as HouseholderSequence::evalTo does), then computeFromHessenberg: Francis double-shift QR steps with Eigen's deflation
// test (findSmallSubdiagEntry), exceptional shifts at iterations 10 and 30 (computeShift), splitOffTwoRows for converged 2 x 2 blocks
// and at most 40 N iterations in all.  T is quasi-triangular on return; false when the iteration limit was reached (NoConvergence).
ACR_HD bool real_schur(const double A[N][N], double T[N][N], double U[N][N]) {
  double scale = 0;
  for (int r = 0; r < N; ++r)
    for (int c = 0; c < N; ++c) scale = fmax(scale, fabs(A[r][c]));
  for (int r = 0; r < N; ++r)
    for (int c = 0; c < N; ++c) { T[r][c] = scale < kMin ? 0.0 : A[r][c] / scale; U[r][c] = r == c ? 1.0 : 0.0; }
  if (scale < kMin) return true;
  // HessenbergDecomposition::_compute: the essential parts stay below the subdiagonal of T
  double h[N - 1];
  for (int i = 0; i < N - 1; ++i) {
    const int rem = N - i - 1;
    double v[N], ess[N], beta;
    for (int t = 0; t < rem; ++t) v[t] = T[i + 1 + t][i];
    make_householder(v, rem, ess, h[i], beta);
    for (int t = 0; t < rem - 1; ++t) T[i + 2 + t][i] = ess[t];
    T[i + 1][i] = beta;
    house_left(T, i + 1, rem, i + 1, N - 1, ess, h[i]);
    house_right(T, i + 1, rem, 0, N - 1, ess, h[i]);
  }
  for (int k = N - 2; k >= 0; --k) {   // Q = H_0 ... H_{N-2}, applied from the last
    const int m = N - k - 1;
    double ess[N];
    for (int t = 0; t < m - 1; ++t) ess[t] = T[k + 2 + t][k];
    house_left(U, k + 1, m, k + 1, N - 1, ess, h[k]);
  }
  for (int r = 2; r < N; ++r)
    for (int c = 0; c < r - 1; ++c) T[r][c] = 0;

  int iu = N - 1, iter = 0, total = 0;
  double exshift = 0, norm = 0;
  for (int j = 0; j < N; ++j)
    for (int r = 0; r < (j + 2 < N ? j + 2 : N); ++r) norm = add(norm, fabs(T[r][j]));
  const double zero = fmax(mul(norm, mul(kEps, kEps)), kMin);
  if (norm != 0) {
    while (iu >= 0) {
      int il = iu;   // findSmallSubdiagEntry
      while (il > 0) {
        double s = add(fabs(T[il - 1][il - 1]), fabs(T[il][il]));
        s = fmax(mul(s, kEps), zero);
        if (fabs(T[il][il - 1]) <= s) break;
        --il;
      }
      if (il == iu) {   // one root
        T[iu][iu] = add(T[iu][iu], exshift);
        if (iu > 0) T[iu][iu - 1] = 0;
        --iu; iter = 0;
      } else if (il == iu - 1) {   // two roots: splitOffTwoRows
        const double p = mul(0.5, sub(T[iu - 1][iu - 1], T[iu][iu]));
        const double q = add(mul(p, p), mul(T[iu][iu - 1], T[iu - 1][iu]));
        T[iu][iu] = add(T[iu][iu], exshift);
        T[iu - 1][iu - 1] = add(T[iu - 1][iu - 1], exshift);
        if (q >= 0) {
          const double z = sqrt(fabs(q));
          double c, s;
          make_givens(p >= 0 ? add(p, z) : sub(p, z), T[iu][iu - 1], c, s);
          for (int k = iu - 1; k < N; ++k) rotate(T[iu - 1][k], T[iu][k], c, s);
          for (int k = 0; k <= iu; ++k) rotate(T[k][iu - 1], T[k][iu], c, s);
          T[iu][iu - 1] = 0;
          for (int k = 0; k < N; ++k) rotate(U[k][iu - 1], U[k][iu], c, s);
        }
        if (iu > 1) T[iu - 1][iu - 2] = 0;
        iu -= 2; iter = 0;
      } else {
        double sh[3] = {T[iu][iu], T[iu - 1][iu - 1], mul(T[iu][iu - 1], T[iu - 1][iu])};   // computeShift
        if (iter == 10) {   // Wilkinson's original ad hoc shift
          exshift = add(exshift, sh[0]);
          for (int i = 0; i <= iu; ++i) T[i][i] = sub(T[i][i], sh[0]);
          const double s = add(fabs(T[iu][iu - 1]), fabs(T[iu - 1][iu - 2]));
          sh[0] = mul(0.75, s); sh[1] = mul(0.75, s); sh[2] = mul(mul(-0.4375, s), s);
        }
        if (iter == 30) {   // MATLAB's ad hoc shift
          double s = sub(sh[1], sh[0]) / 2.0;
          s = add(mul(s, s), sh[2]);
          if (s > 0) {
            s = sqrt(s);
            if (sh[1] < sh[0]) s = -s;
            s = add(s, sub(sh[1], sh[0]) / 2.0);
            s = sub(sh[0], sh[2] / s);
            exshift = add(exshift, s);
            for (int i = 0; i <= iu; ++i) T[i][i] = sub(T[i][i], s);
            sh[0] = sh[1] = sh[2] = 0.964;
          }
        }
        ++iter; ++total;
        if (total > 40 * N) return false;
        double v[3] = {0, 0, 0};   // initFrancisQRStep
        int im;
        for (im = iu - 2; im >= il; --im) {
          const double Tmm = T[im][im], r = sub(sh[0], Tmm), s = sub(sh[1], Tmm);
          v[0] = add(sub(mul(r, s), sh[2]) / T[im + 1][im], T[im][im + 1]);
          v[1] = sub(sub(sub(T[im + 1][im + 1], Tmm), r), s);
          v[2] = T[im + 2][im + 1];
          if (im == il) break;
          const double lhs = mul(T[im][im - 1], add(fabs(v[1]), fabs(v[2])));
          const double rhs = mul(v[0], add(add(fabs(T[im - 1][im - 1]), fabs(Tmm)), fabs(T[im + 1][im + 1])));
          if (fabs(lhs) < mul(kEps, rhs)) break;
        }
        for (int k = im; k <= iu - 2; ++k) {   // performFrancisQRStep
          const bool first = k == im;
          double w[3], ess[2], tau, beta;
          for (int t = 0; t < 3; ++t) w[t] = first ? v[t] : T[k + t][k - 1];
          make_householder(w, 3, ess, tau, beta);
          if (beta != 0) {
            if (first && k > il) T[k][k - 1] = -T[k][k - 1];
            else if (!first) T[k][k - 1] = beta;
            house_left(T, k, 3, k, N - 1, ess, tau);
            house_right(T, k, 3, 0, (iu < k + 3 ? iu : k + 3), ess, tau);
            house_right(U, k, 3, 0, N - 1, ess, tau);
          }
        }
        {
          double w[2] = {T[iu - 1][iu - 2], T[iu][iu - 2]}, ess[1], tau, beta;
          make_householder(w, 2, ess, tau, beta);
          if (beta != 0) {
            T[iu - 1][iu - 2] = beta;
            house_left(T, iu - 1, 2, iu - 1, N - 1, ess, tau);
            house_right(T, iu - 1, 2, 0, iu, ess, tau);
            house_right(U, iu - 1, 2, 0, N - 1, ess, tau);
          }
        }
        for (int i = im + 2; i <= iu; ++i) {   // clean up pollution due to round-off errors
          T[i][i - 2] = 0;
          if (i > im + 2) T[i][i - 3] = 0;
        }
      }
    }
  }
  for (int r = 0; r < N; ++r)
    for (int c = 0; c < N; ++c) T[r][c] = mul(T[r][c], scale);
  return true;
}

// std::complex<double> division as GCC compiles it (libgcc's __divdc3): Smith's algorithm on the larger of |c|, |d|, with its
// rescaling of extreme operands and its recovery of a zero divisor; (a + b i) / (c + d i) -> (x, y).  The recovery of infinite
// operands is not restated (every operand here is finite or NaN).
ACR_HD void cdiv(double a, double b, double c, double d, double& x, double& y) {
  constexpr double kRbig = 1.7976931348623157e308 / 2, kRmin = kMin, kRmin2 = kEps, kRminscal = 1.0 / kEps, kRmax2 = kRbig * kRmin2;
  double ratio, denom;
  if (fabs(c) < fabs(d)) {
    if (fabs(d) >= kRbig) { a = a / 2; b = b / 2; c = c / 2; d = d / 2; }
    if (fabs(d) < kRmin2 || (fabs(a) < kRmin && fabs(b) < kRmax2 && fabs(d) < kRmax2) ||
        (fabs(b) < kRmin && fabs(a) < kRmax2 && fabs(d) < kRmax2)) {
      a = mul(a, kRminscal); b = mul(b, kRminscal); c = mul(c, kRminscal); d = mul(d, kRminscal);
    }
    ratio = c / d;
    denom = add(mul(c, ratio), d);
    if (fabs(ratio) > kRmin) {
      x = add(mul(a, ratio), b) / denom;
      y = sub(mul(b, ratio), a) / denom;
    } else {
      x = add(mul(c, a / d), b) / denom;
      y = sub(mul(c, b / d), a) / denom;
    }
  } else {
    if (fabs(c) >= kRbig) { a = a / 2; b = b / 2; c = c / 2; d = d / 2; }
    if (fabs(c) < kRmin2 || (fabs(a) < kRmin && fabs(b) < kRmax2 && fabs(c) < kRmax2) ||
        (fabs(b) < kRmin && fabs(a) < kRmax2 && fabs(c) < kRmax2)) {
      a = mul(a, kRminscal); b = mul(b, kRminscal); c = mul(c, kRminscal); d = mul(d, kRminscal);
    }
    ratio = d / c;
    denom = add(mul(d, ratio), c);
    if (fabs(ratio) > kRmin) {
      x = add(mul(b, ratio), a) / denom;
      y = sub(b, mul(a, ratio)) / denom;
    } else {
      x = add(a, mul(d, b / c)) / denom;
      y = sub(b, mul(d, a / c)) / denom;
    }
  }
  if (x != x && y != y && c == 0 && d == 0 && (a == a || b == b)) {   // NaN + NaN i from a zero divisor: signed infinities
    const double inf = copysign((double)INFINITY, c);
    x = mul(inf, a); y = mul(inf, b);
  }
}

// EigenSolver<Mat10>(A): the real Schur form, its eigenvalues (a 2 x 2 block gives (T(i+1, i+1) + p) +- z i, z computed without
// overflow), and the normalised eigenvectors of the real ones (imag() exactly 0), by doComputeEigenvectors' back-substitution
// and back-transformation.  re[i], im[i]: the eigenvalues in Schur order; V[i][*]: the eigenvector of eigenvalue i when im[i] == 0.
// Returns false where Eigen reports NoConvergence or NumericalIssue (no eigenvector computed).
ACR_HD bool eigen_solve(const double A[N][N], double re[N], double im[N], double V[N][N]) {
  double T[N][N], U[N][N];
  if (!real_schur(A, T, U)) return false;
  for (int i = 0; i < N;) {
    if (i == N - 1 || T[i + 1][i] == 0) {
      re[i] = T[i][i]; im[i] = 0;
      if (!(fabs(re[i]) <= 1.7976931348623157e308)) return false;   // not finite
      ++i;
    } else {
      const double p = mul(0.5, sub(T[i][i], T[i + 1][i + 1]));
      double t0 = T[i + 1][i], t1 = T[i][i + 1];
      const double mx = fmax(fabs(p), fmax(fabs(t0), fabs(t1)));
      t0 = t0 / mx; t1 = t1 / mx;
      const double p0 = p / mx;
      const double z = mul(mx, sqrt(fabs(add(mul(p0, p0), mul(t0, t1)))));
      re[i] = re[i + 1] = add(T[i + 1][i + 1], p);
      im[i] = z; im[i + 1] = -z;
      i += 2;
    }
  }
  double norm = 0;
  for (int j = 0; j < N; ++j)
    for (int c = (j > 0 ? j - 1 : 0); c < N; ++c) norm = add(norm, fabs(T[j][c]));
  if (norm != 0) {
    for (int n = N - 1; n >= 0; --n) {   // back-substitution, real eigenvalues only (the complex ones touch no column used here)
      if (im[n] != 0) continue;
      const double p = re[n];
      double lastr = 0, lastw = 0;
      int l = n;
      T[n][n] = 1.0;
      for (int i = n - 1; i >= 0; --i) {
        const double w = sub(T[i][i], p);
        double r = 0;
        for (int k = l; k <= n; ++k) r = add(r, mul(T[i][k], T[k][n]));
        if (im[i] < 0) {
          lastw = w; lastr = r;
        } else {
          l = i;
          if (im[i] == 0) {
            T[i][n] = w != 0 ? -r / w : -r / mul(kEps, norm);
          } else {   // a complex pair above: solve the real 2 x 2 equations
            const double x = T[i][i + 1], y = T[i + 1][i];
            const double dr = sub(re[i], p);
            const double denom = add(mul(dr, dr), mul(im[i], im[i]));
            const double t = sub(mul(x, lastr), mul(lastw, r)) / denom;
            T[i][n] = t;
            T[i + 1][n] = fabs(x) > fabs(lastw) ? sub(-r, mul(w, t)) / x : sub(-lastr, mul(y, t)) / lastw;
          }
          const double t = fabs(T[i][n]);   // overflow control
          if (mul(mul(kEps, t), t) > 1)
            for (int k = i; k < N; ++k) T[k][n] = T[k][n] / t;
        }
      }
    }
    for (int j = N - 1; j >= 0; --j) {   // back-transformation: column j <- U[:, 0..j] T[0..j, j]
      if (im[j] != 0) continue;
      double col[N];
      for (int r = 0; r < N; ++r) {
        double s = mul(U[r][0], T[0][j]);
        for (int k = 1; k <= j; ++k) s = add(s, mul(U[r][k], T[k][j]));
        col[r] = s;
      }
      for (int r = 0; r < N; ++r) U[r][j] = col[r];
    }
  }
  for (int j = 0; j < N; ++j) {
    if (im[j] != 0) continue;
    double s = 0;
    for (int r = 0; r < N; ++r) s = add(s, mul(U[r][j], U[r][j]));
    const double nr = sqrt(s);
    for (int r = 0; r < N; ++r) V[j][r] = s > 0 ? U[r][j] / nr : U[r][j];
  }
  return true;
}
// EigenSolver<Mat10>(A) as the F10 solver reads it: eigen_solve's Schur form, eigenvalues and real back-substitution, with in
// addition doComputeEigenvectors' complex branch (the pair (j, j + 1), im[j] > 0, leaves its vector's real part in m_eivec's column j
// and its imaginary part in column j + 1), every column back-transformed, and eigenvectors()' assembly: column j is real when
// |im[j]| <= |re[j]| 2 eps or j + 1 == N, else the pair is (col j) +- i (col j + 1); each column normalised (squared norm summed in
// index order, divided by its square root when positive).  V[j][*] + i Vi[j][*] is eigenvectors().col(j).  A function of its own:
// E's eigen_solve, which it restates in part, keeps the code it compiles to.
ACR_HD bool eigen_solve_complex(const double A[N][N], double re[N], double im[N], double V[N][N], double Vi[N][N]) {
  double T[N][N], U[N][N];
  if (!real_schur(A, T, U)) return false;
  for (int i = 0; i < N;) {
    if (i == N - 1 || T[i + 1][i] == 0) {
      re[i] = T[i][i]; im[i] = 0;
      if (!(fabs(re[i]) <= 1.7976931348623157e308)) return false;   // not finite
      ++i;
    } else {
      const double p = mul(0.5, sub(T[i][i], T[i + 1][i + 1]));
      double t0 = T[i + 1][i], t1 = T[i][i + 1];
      const double mx = fmax(fabs(p), fmax(fabs(t0), fabs(t1)));
      t0 = t0 / mx; t1 = t1 / mx;
      const double p0 = p / mx;
      const double z = mul(mx, sqrt(fabs(add(mul(p0, p0), mul(t0, t1)))));
      re[i] = re[i + 1] = add(T[i + 1][i + 1], p);
      im[i] = z; im[i + 1] = -z;
      i += 2;
    }
  }
  double norm = 0;
  for (int j = 0; j < N; ++j)
    for (int c = (j > 0 ? j - 1 : 0); c < N; ++c) norm = add(norm, fabs(T[j][c]));
  if (norm != 0) {
    for (int n = N - 1; n >= 0; --n) {   // back-substitution
      {
        if (im[n] < 0 && n > 0) {   // the complex branch: columns n - 1 (real part) and n (imaginary part)
          const double p = re[n], q = im[n];
          double lastra = 0, lastsa = 0, lastw = 0;
          int l = n - 1;
          if (fabs(T[n][n - 1]) > fabs(T[n - 1][n])) {   // last vector component imaginary: the matrix is triangular
            T[n - 1][n - 1] = q / T[n][n - 1];
            T[n - 1][n] = -sub(T[n][n], p) / T[n][n - 1];
          } else {
            cdiv(0.0, -T[n - 1][n], sub(T[n - 1][n - 1], p), q, T[n - 1][n - 1], T[n - 1][n]);
          }
          T[n][n - 1] = 0;
          T[n][n] = 1.0;
          for (int i = n - 2; i >= 0; --i) {
            double ra = 0, sa = 0;
            for (int k = l; k <= n; ++k) { ra = add(ra, mul(T[i][k], T[k][n - 1])); sa = add(sa, mul(T[i][k], T[k][n])); }
            const double w = sub(T[i][i], p);
            if (im[i] < 0) {
              lastw = w; lastra = ra; lastsa = sa;
            } else {
              l = i;
              if (im[i] == 0) {
                cdiv(-ra, -sa, w, q, T[i][n - 1], T[i][n]);
              } else {   // solve the complex equations
                const double x = T[i][i + 1], y = T[i + 1][i];
                const double dr = sub(re[i], p);
                double vr = sub(add(mul(dr, dr), mul(im[i], im[i])), mul(q, q));
                const double vi = mul(mul(dr, 2.0), q);
                if (vr == 0 && vi == 0)
                  vr = mul(mul(kEps, norm), add(add(add(add(fabs(w), fabs(q)), fabs(x)), fabs(y)), fabs(lastw)));
                cdiv(add(sub(mul(x, lastra), mul(lastw, ra)), mul(q, sa)), sub(sub(mul(x, lastsa), mul(lastw, sa)), mul(q, ra)), vr, vi,
                     T[i][n - 1], T[i][n]);
                if (fabs(x) > add(fabs(lastw), fabs(q))) {
                  T[i + 1][n - 1] = add(sub(-ra, mul(w, T[i][n - 1])), mul(q, T[i][n])) / x;
                  T[i + 1][n] = sub(sub(-sa, mul(w, T[i][n])), mul(q, T[i][n - 1])) / x;
                } else {
                  cdiv(sub(-lastra, mul(y, T[i][n - 1])), sub(-lastsa, mul(y, T[i][n])), lastw, q, T[i + 1][n - 1], T[i + 1][n]);
                }
              }
              const double t = fmax(fabs(T[i][n - 1]), fabs(T[i][n]));   // overflow control
              if (mul(mul(kEps, t), t) > 1)
                for (int k = i; k < N; ++k) { T[k][n - 1] = T[k][n - 1] / t; T[k][n] = T[k][n] / t; }
            }
          }
          --n;   // the pair is done
          continue;
        }
      }
      if (im[n] != 0) continue;
      const double p = re[n];
      double lastr = 0, lastw = 0;
      int l = n;
      T[n][n] = 1.0;
      for (int i = n - 1; i >= 0; --i) {
        const double w = sub(T[i][i], p);
        double r = 0;
        for (int k = l; k <= n; ++k) r = add(r, mul(T[i][k], T[k][n]));
        if (im[i] < 0) {
          lastw = w; lastr = r;
        } else {
          l = i;
          if (im[i] == 0) {
            T[i][n] = w != 0 ? -r / w : -r / mul(kEps, norm);
          } else {   // a complex pair above: solve the real 2 x 2 equations
            const double x = T[i][i + 1], y = T[i + 1][i];
            const double dr = sub(re[i], p);
            const double denom = add(mul(dr, dr), mul(im[i], im[i]));
            const double t = sub(mul(x, lastr), mul(lastw, r)) / denom;
            T[i][n] = t;
            T[i + 1][n] = fabs(x) > fabs(lastw) ? sub(-r, mul(w, t)) / x : sub(-lastr, mul(y, t)) / lastw;
          }
          const double t = fabs(T[i][n]);   // overflow control
          if (mul(mul(kEps, t), t) > 1)
            for (int k = i; k < N; ++k) T[k][n] = T[k][n] / t;
        }
      }
    }
    for (int j = N - 1; j >= 0; --j) {   // back-transformation: column j <- U[:, 0..j] T[0..j, j]
      double col[N];
      for (int r = 0; r < N; ++r) {
        double s = mul(U[r][0], T[0][j]);
        for (int k = 1; k <= j; ++k) s = add(s, mul(U[r][k], T[k][j]));
        col[r] = s;
      }
      for (int r = 0; r < N; ++r) U[r][j] = col[r];
    }
  }
  {   // eigenvectors()
    for (int j = 0; j < N; ++j) {
      const bool real = fabs(im[j]) <= mul(fabs(re[j]), 2 * kEps) || j + 1 == N;
      double s = 0;
      for (int r = 0; r < N; ++r) s = real ? add(s, mul(U[r][j], U[r][j])) : add(s, add(mul(U[r][j], U[r][j]), mul(U[r][j + 1], U[r][j + 1])));
      const double nr = sqrt(s);
      for (int r = 0; r < N; ++r) {
        V[j][r] = s > 0 ? U[r][j] / nr : U[r][j];
        Vi[j][r] = real ? 0.0 : (s > 0 ? U[r][j + 1] / nr : U[r][j + 1]);
        if (!real) { V[j + 1][r] = V[j][r]; Vi[j + 1][r] = -Vi[j][r]; }
      }
      if (!real) ++j;
    }
  }
  return true;
}
// Steps 1-4 of Essential5PSolver::solve on the 5 epipolar rows A: the null-space basis Eb (column c = N[c] of nullspace<5>), the
// constraint matrix, its full-pivot LU solve and the action matrix At
ACR_HD void action_matrix(const double A[5][9], double Eb[9][4], double At[N][N]) {
  double Nb[4][9];
  nullspace<5>(A, Nb);
  for (int t = 0; t < 9; ++t)
    for (int c = 0; c < 4; ++c) Eb[t][c] = Nb[c][t];
  double M[N][20], X[N][N];
  constraints(Eb, M);
  lu_solve(M, X);
  for (int r = 0; r < N; ++r)
    for (int c = 0; c < N; ++c) At[r][c] = 0;
  const int from[6] = {0, 1, 2, 4, 5, 7};
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < N; ++c) At[r][c] = X[from[r]][c];
  At[6][0] = At[7][1] = At[8][3] = At[9][6] = -1;
}
}  // namespace e5

// Essential5PSolver::solve on 5 K^-1-normalised correspondences (x1[i], y1[i]) <-> (x2[i], y2[i]): the 4-D null space of the
// epipolar rows (nullspace<5>; basis column c = N[c]), the 10 x 20 constraint matrix, its full-pivot LU solve, the action matrix,
// and E = (EBasis v.tail<4>())^T in Eigen's column-major map for every eigenvalue whose imaginary part is exactly 0, in Schur
// order.  Returns the number of models (0..10) written row-major to E[m * 9] (x_J^T E x_I = 0 on normalised points).
ACR_HD int fit5(const double* x1, const double* y1, const double* x2, const double* y2, double* E) {
  double A[kSampleE][9];
  for (int i = 0; i < kSampleE; ++i) {   // encodeEpipolarEquation
    A[i][0] = mul(x2[i], x1[i]); A[i][1] = mul(x2[i], y1[i]); A[i][2] = x2[i];
    A[i][3] = mul(y2[i], x1[i]); A[i][4] = mul(y2[i], y1[i]); A[i][5] = y2[i];
    A[i][6] = x1[i]; A[i][7] = y1[i]; A[i][8] = 1.0;
  }
  double Eb[9][4], At[e5::N][e5::N];
  e5::action_matrix(A, Eb, At);
  double re[e5::N], im[e5::N], V[e5::N][e5::N];
  if (!e5::eigen_solve(At, re, im, V)) return 0;
  int nb = 0;
  for (int s = 0; s < e5::N; ++s) {
    if (im[s] != 0) continue;
    const double* v = V[s] + 6;
    for (int t = 0; t < 9; ++t)
      E[nb * 9 + t] = add(add(add(mul(Eb[t][0], v[0]), mul(Eb[t][1], v[1])), mul(Eb[t][2], v[2])), mul(Eb[t][3], v[3]));
    ++nb;
  }
  return nb;
}

// ---------------------------------------------------------------------------------------------------------------- F10 kernel
// RelativePoseKernel<Fundamental10PSolver, FundamentalEpipolarDistanceError, UnnormalizerT, Fundamental10PModel>: F's image-size
// preconditioning, point-to-line error (on model.getMatrix() alone: the distortion L plays no part in the score), logalpha0,
// errorVectorDimension 1 and N2^T F N1 (L stays in preconditioned units); only the sample size, the model count and the fit
// differ.  F10RelativePose's F satisfies [x_I, y_I, 1 + l1 r_I^2] F [x_J, y_J, 1 + l2 r_J^2]^T = 0: the error reads it as
// x_J^T F x_I, the transpose, as the reference does.
//
// Eigen 3.4 rules restated for it (the E solver's RealSchur / EigenSolver code is shared):
//   * PartialPivLU<Mat10>: unblocked at this size; per column the first largest |entry| at or below the diagonal is the pivot
//     (strict >), the rows swap (the right-hand side with them, as P b), the column below divides by the pivot unless it is
//     exactly 0 (not caught: inf / NaN flow on), and the rank-1 update follows.  The solve is the TRSM of triangular_solve_matrix
//     with its 4-wide panels: inside a panel x_i = b_i * (1 / u_ii) (unit lower: b_i) and the panel's rows update sequentially;
//     the rows past a panel take the panel's products summed in index order (the GEBP accumulator) in one subtraction.
//   * colEchelonForm(M, 1e-16) as written: p starts at DBL_MIN, `tp > p` (the first column wins a tie, a NaN never), a row below
//     the tolerance is zeroed, column swap, scaling (division), elimination of every other column.
//   * EigenSolver: eigen_solve_complex (doComputeEigenvectors with its complex branch, the complex divisions as cdiv, and
//     eigenvectors()' assembly and normalisation).
//   * esols = row(2) / row(0) and row(1) / row(0) of eigenvectors(): the rows are strided, so Eigen takes the scalar path, std::complex
//     division, i.e. cdiv; a solution is kept when both imaginary parts are at most 100 eps in magnitude.
//   * the dot products of the model step in Eigen's unrolled redux order: b(4:10) . m2 and b(0:4) . m1 on SSE2 packets of 2,
//     m3 . mr.row(k) (a strided row) as the scalar unroller's halving tree.
// Divergences (rounding level): every other summation runs in index order where Eigen's packet code may pair terms differently,
// and where the Schur iteration does not converge or an eigenvalue is not finite the fit returns no model (Eigen then leaves
// eigenvectors() unspecified).
constexpr int kSampleF10 = 10;      // Fundamental10PSolver::getMinimumNbRequiredSamples
constexpr int kMaxModelsF10 = 10;   // Fundamental10PSolver::getMaximumNbModels

// fit10's working arrays (5960 bytes): the device keeps them in a per-CTA shared-memory workspace, the host on its stack (the Schur
// form and its vectors, 1.6 KB, stay eigen_solve_complex's locals)
struct F10Work {
  double A[10][16];   // the monomial matrix; after the solve its last 6 columns hold mr
  double M[20][10];   // f10e_gb's M, then its column echelon form
  double At[10][10];  // the action matrix
  double V[10][10], Vi[10][10];   // eigenvectors(): V[j] + i Vi[j] is column j
  double P[29], c[36];
  double re[10], im[10];
};

// A(:, 0:10) x = A(:, 10:16) by PartialPivLU, in place: x lands in A(:, 10:16)
ACR_HD void partial_lu_solve(double A[10][16]) {
  constexpr int n = 10, kPanel = 4;
  for (int k = 0; k < n; ++k) {
    int br = k;
    double big = fabs(A[k][k]);
    for (int r = k + 1; r < n; ++r)
      if (fabs(A[r][k]) > big) { big = fabs(A[r][k]); br = r; }
    if (big != 0) {
      if (br != k)
        for (int c = 0; c < 16; ++c) { const double t = A[k][c]; A[k][c] = A[br][c]; A[br][c] = t; }
      for (int r = k + 1; r < n; ++r) A[r][k] = A[r][k] / A[k][k];
    }
    for (int c = k + 1; c < n; ++c)
      for (int r = k + 1; r < n; ++r) A[r][c] = sub(A[r][c], mul(A[r][k], A[k][c]));
  }
  for (int j = 10; j < 16; ++j) {
    for (int k1 = 0; k1 < n; k1 += kPanel) {   // unit lower, panels from the top
      const int w = k1 + kPanel < n ? kPanel : n - k1;
      for (int i = k1; i < k1 + w; ++i)
        for (int r = i + 1; r < k1 + w; ++r) A[r][j] = sub(A[r][j], mul(A[i][j], A[r][i]));
      for (int r = k1 + w; r < n; ++r) {
        double acc = 0;
        for (int i = k1; i < k1 + w; ++i) acc = add(acc, mul(A[r][i], A[i][j]));
        A[r][j] = sub(A[r][j], acc);
      }
    }
    for (int k1 = 0; k1 < n; k1 += kPanel) {   // upper, panels from the bottom
      const int w = k1 + kPanel < n ? kPanel : n - k1, top = n - k1 - w;
      for (int i = n - k1 - 1; i >= top; --i) {
        A[i][j] = mul(A[i][j], 1.0 / A[i][i]);
        for (int r = top; r < i; ++r) A[r][j] = sub(A[r][j], mul(A[i][j], A[r][i]));
      }
      for (int r = 0; r < top; ++r) {
        double acc = 0;
        for (int i = top; i < top + w; ++i) acc = add(acc, mul(A[r][i], A[i][j]));
        A[r][j] = sub(A[r][j], acc);
      }
    }
  }
}

// colEchelonForm(M, pivtol) on the 20 x 10 M
ACR_HD void col_echelon(double M[20][10], double pivtol) {
  constexpr int n = 20, m = 10;
  int i = 0, j = 0;
  while (i < m && j < n) {
    double p = e5::kMin;
    int col = i;
    for (int k = i; k < m; ++k) {
      const double tp = fabs(M[j][k]);
      if (tp > p) { p = tp; col = k; }
    }
    if (p < pivtol) {
      for (int k = i; k < m; ++k) M[j][k] = 0;
      ++j;
    } else {
      if (col != i)
        for (int r = j; r < n; ++r) { const double t = M[r][i]; M[r][i] = M[r][col]; M[r][col] = t; }
      for (int r = j + 1; r < n; ++r) M[r][i] = M[r][i] / M[j][i];
      M[j][i] = 1.0;
      for (int k = 0; k < m; ++k) {
        if (k == i) continue;
        const double s = M[j][k];
        for (int r = j; r < n; ++r) M[r][k] = sub(M[r][k], mul(s, M[r][i]));
      }
      ++i; ++j;
    }
  }
}

// Fundamental10PSolver::solve (F10RelativePose, f10e_gb) on 10 preconditioned correspondences (x1[i], y1[i]) <-> (x2[i], y2[i]):
// returns the number of models (0..10), F row-major at F[9 m] (F(2, 2) = 1) and (l1, l2) at L[2 m].
ACR_HD int fit10(const double* x1, const double* y1, const double* x2, const double* y2, double* F, double* L, F10Work& w) {
  double(&A)[10][16] = w.A;
  for (int i = 0; i < 10; ++i) {   // X = the I points, U = the J points
    const double x = x1[i], y = y1[i], u = x2[i], v = y2[i];
    const double z1 = add(mul(x, x), mul(y, y)), z2 = add(mul(u, u), mul(v, v));
    double* a = A[i];
    a[0] = mul(x, u); a[1] = mul(x, v); a[2] = mul(y, u); a[3] = mul(y, v); a[4] = mul(u, z1); a[5] = u; a[6] = mul(v, z1); a[7] = v;
    a[8] = mul(x, z2); a[9] = x; a[10] = mul(y, z2); a[11] = y; a[12] = mul(z1, z2); a[13] = z1; a[14] = z2; a[15] = 1.0;
  }
  partial_lu_solve(A);
#define MR(r, c) A[r][10 + (c)]
  double* P = w.P;
  {
    const double p[29] = {MR(5, 0), MR(5, 1), -MR(4, 0), -MR(4, 1), MR(5, 2), MR(5, 3), sub(MR(5, 4), MR(4, 2)), sub(MR(5, 5), MR(4, 3)),
                          -MR(4, 4), -MR(4, 5), MR(7, 0), MR(7, 1), -MR(6, 0), -MR(6, 1), MR(7, 2), MR(7, 3), sub(MR(7, 4), MR(6, 2)),
                          sub(MR(7, 5), MR(6, 3)), -MR(6, 4), -MR(6, 5), MR(9, 0), sub(MR(9, 1), MR(8, 0)), -MR(8, 1), MR(9, 2), MR(9, 4),
                          sub(MR(9, 3), MR(8, 2)), -MR(8, 3), sub(MR(9, 5), MR(8, 4)), -MR(8, 5)};
    for (int t = 0; t < 29; ++t) P[t] = p[t];
  }
  double* c = w.c;
  c[0] = sub(mul(P[0], P[14]), mul(P[4], P[10]));
  c[1] = sub(sub(add(mul(P[0], P[16]), mul(P[2], P[14])), mul(P[4], P[12])), mul(P[6], P[10]));
  c[2] = sub(mul(P[2], P[18]), mul(P[8], P[12]));
  c[3] = sub(mul(P[1], P[15]), mul(P[5], P[11]));
  c[4] = sub(sub(add(mul(P[1], P[17]), mul(P[3], P[15])), mul(P[5], P[13])), mul(P[7], P[11]));
  c[5] = sub(sub(add(mul(P[0], P[15]), mul(P[1], P[14])), mul(P[4], P[11])), mul(P[5], P[10]));
  c[6] = sub(sub(sub(sub(add(add(add(mul(P[0], P[17]), mul(P[1], P[16])), mul(P[2], P[15])), mul(P[3], P[14])), mul(P[4], P[13])), mul(P[5], P[12])), mul(P[6], P[11])), mul(P[7], P[10]));
  c[7] = sub(sub(add(mul(P[0], P[18]), mul(P[2], P[16])), mul(P[6], P[12])), mul(P[8], P[10]));
  c[8] = sub(sub(sub(sub(add(add(add(mul(P[0], P[19]), mul(P[1], P[18])), mul(P[2], P[17])), mul(P[3], P[16])), mul(P[6], P[13])), mul(P[7], P[12])), mul(P[8], P[11])), mul(P[9], P[10]));
  c[9] = sub(sub(add(mul(P[2], P[19]), mul(P[3], P[18])), mul(P[8], P[13])), mul(P[9], P[12]));
  c[10] = sub(sub(add(mul(P[1], P[19]), mul(P[3], P[17])), mul(P[7], P[13])), mul(P[9], P[11]));
  c[11] = sub(mul(P[3], P[19]), mul(P[9], P[13]));
  c[12] = sub(mul(P[0], P[23]), mul(P[4], P[20]));
  c[13] = sub(sub(add(mul(P[1], P[23]), mul(P[0], P[25])), mul(P[4], P[21])), mul(P[5], P[20]));
  c[14] = sub(mul(P[2], P[24]), mul(P[8], P[20]));
  c[15] = sub(sub(add(mul(P[3], P[24]), mul(P[2], P[27])), mul(P[8], P[21])), mul(P[9], P[20]));
  c[16] = sub(mul(P[1], P[26]), mul(P[5], P[22]));
  c[17] = sub(add(mul(P[0], P[24]), mul(P[2], P[23])), mul(P[6], P[20]));
  c[18] = sub(sub(add(mul(P[0], P[26]), mul(P[1], P[25])), mul(P[4], P[22])), mul(P[5], P[21]));
  c[19] = sub(sub(add(add(add(mul(P[1], P[24]), mul(P[3], P[23])), mul(P[0], P[27])), mul(P[2], P[25])), mul(P[6], P[21])), mul(P[7], P[20]));
  c[20] = sub(sub(add(add(add(mul(P[0], P[28]), mul(P[1], P[27])), mul(P[2], P[26])), mul(P[3], P[25])), mul(P[6], P[22])), mul(P[7], P[21]));
  c[21] = sub(sub(add(mul(P[2], P[28]), mul(P[3], P[27])), mul(P[8], P[22])), mul(P[9], P[21]));
  c[22] = sub(add(mul(P[1], P[28]), mul(P[3], P[26])), mul(P[7], P[22]));
  c[23] = sub(mul(P[3], P[28]), mul(P[9], P[22]));
  c[24] = sub(mul(P[10], P[23]), mul(P[14], P[20]));
  c[25] = sub(sub(add(mul(P[11], P[23]), mul(P[10], P[25])), mul(P[14], P[21])), mul(P[15], P[20]));
  c[26] = sub(mul(P[12], P[24]), mul(P[18], P[20]));
  c[27] = sub(sub(add(mul(P[13], P[24]), mul(P[12], P[27])), mul(P[18], P[21])), mul(P[19], P[20]));
  c[28] = sub(mul(P[11], P[26]), mul(P[15], P[22]));
  c[29] = sub(add(mul(P[10], P[24]), mul(P[12], P[23])), mul(P[16], P[20]));
  c[30] = sub(sub(add(mul(P[10], P[26]), mul(P[11], P[25])), mul(P[14], P[22])), mul(P[15], P[21]));
  c[31] = sub(sub(add(add(add(mul(P[11], P[24]), mul(P[13], P[23])), mul(P[10], P[27])), mul(P[12], P[25])), mul(P[16], P[21])), mul(P[17], P[20]));
  c[32] = sub(sub(add(add(add(mul(P[10], P[28]), mul(P[11], P[27])), mul(P[12], P[26])), mul(P[13], P[25])), mul(P[16], P[22])), mul(P[17], P[21]));
  c[33] = sub(sub(add(mul(P[12], P[28]), mul(P[13], P[27])), mul(P[18], P[22])), mul(P[19], P[21]));
  c[34] = sub(add(mul(P[11], P[28]), mul(P[13], P[26])), mul(P[17], P[22]));
  c[35] = sub(mul(P[13], P[28]), mul(P[19], P[22]));
  double(&M)[20][10] = w.M;   // M(k) of the column-major 20 x 10 matrix is M[k % 20][k / 20]
  for (int r = 0; r < 20; ++r)
    for (int q = 0; q < 10; ++q) M[r][q] = 0;
#define ACR_F10_M3(k, i0, i1, i2) (M[(i0) % 20][(i0) / 20] = M[(i1) % 20][(i1) / 20] = M[(i2) % 20][(i2) / 20] = c[k])
#define ACR_F10_M(k, i0, i1, i2, i3) (ACR_F10_M3(k, i0, i1, i2), M[(i3) % 20][(i3) / 20] = c[k])
  ACR_F10_M(0, 0, 61, 82, 144); ACR_F10_M(1, 2, 64, 85, 148); ACR_F10_M(2, 9, 72, 93, 156); ACR_F10_M(3, 3, 66, 87, 150); ACR_F10_M(4, 7, 70, 91, 154); ACR_F10_M(5, 1, 63, 84, 147);
  ACR_F10_M(6, 4, 67, 88, 151); ACR_F10_M(7, 5, 68, 89, 152); ACR_F10_M(8, 8, 71, 92, 155); ACR_F10_M(9, 12, 75, 96, 158); ACR_F10_M(10, 11, 74, 95, 157); ACR_F10_M(11, 15, 77, 98, 159);
  ACR_F10_M3(12, 20, 102, 165); ACR_F10_M3(13, 21, 104, 168); ACR_F10_M3(14, 25, 109, 173); ACR_F10_M3(15, 28, 112, 176); ACR_F10_M3(16, 26, 110, 174); ACR_F10_M3(17, 22, 105, 169);
  ACR_F10_M3(18, 23, 107, 171); ACR_F10_M3(19, 24, 108, 172); ACR_F10_M3(20, 27, 111, 175); ACR_F10_M3(21, 31, 115, 178); ACR_F10_M3(22, 30, 114, 177); ACR_F10_M3(23, 34, 117, 179);
  ACR_F10_M3(24, 40, 122, 185); ACR_F10_M3(25, 41, 124, 188); ACR_F10_M3(26, 45, 129, 193); ACR_F10_M3(27, 48, 132, 196); ACR_F10_M3(28, 46, 130, 194); ACR_F10_M3(29, 42, 125, 189);
  ACR_F10_M3(30, 43, 127, 191); ACR_F10_M3(31, 44, 128, 192); ACR_F10_M3(32, 47, 131, 195); ACR_F10_M3(33, 51, 135, 198); ACR_F10_M3(34, 50, 134, 197); ACR_F10_M3(35, 54, 137, 199);
#undef ACR_F10_M
#undef ACR_F10_M3
  col_echelon(M, 1e-16);
  double(&At)[10][10] = w.At;
  for (int r = 0; r < 10; ++r)
    for (int q = 0; q < 10; ++q) At[r][q] = 0;
  At[0][2] = At[1][4] = At[2][5] = At[3][7] = At[4][8] = At[5][9] = 1.0;
  for (int r = 6; r < 10; ++r)
    for (int q = 0; q < 10; ++q) At[r][q] = -M[19 - q][15 - r];
  if (!e5::eigen_solve_complex(At, w.re, w.im, w.V, w.Vi)) return 0;
  int nb = 0;
  for (int j = 0; j < 10; ++j) {   // esols = (row 2 / row 0, row 1 / row 0), kept when both imaginary parts are within 100 eps
    const double *v = w.V[j], *vi = w.Vi[j];
    double l1r, l1i, l2r, l2i;
    e5::cdiv(v[2], vi[2], v[0], vi[0], l1r, l1i);
    e5::cdiv(v[1], vi[1], v[0], vi[0], l2r, l2i);
    if (fabs(l1i) <= 100 * e5::kEps && fabs(l2i) <= 100 * e5::kEps) { L[2 * nb] = l1r; L[2 * nb + 1] = l2r; ++nb; }
  }
  if (nb == 0) return 0;
  for (int m = 0; m < nb; ++m) {
    const double l1 = L[2 * m], l2 = L[2 * m + 1], l1l1 = mul(l1, l1), l1l2 = mul(l1, l2);
    // b = P[0..9]; f23 = -b(4:10) . m2 / b(0:4) . m1, both in SSE2 packet order
    const double m1[4] = {l1l2, l1, l2, 1.0}, m2[6] = {mul(l1l2, l1), l1l1, l1l2, l1, l2, 1.0};
    double t2[6], t1[4];
    for (int k = 0; k < 6; ++k) t2[k] = mul(P[4 + k], m2[k]);
    for (int k = 0; k < 4; ++k) t1[k] = mul(P[k], m1[k]);
    const double d2 = add(add(t2[0], add(t2[2], t2[4])), add(t2[1], add(t2[3], t2[5])));
    const double d1 = add(add(t1[0], t1[2]), add(t1[1], t1[3]));
    const double f23 = -d2 / d1;
    const double m3[6] = {mul(l2, f23), f23, l1l2, l1, l2, 1.0};
    auto dot = [&](int row) {   // m3 . -mr.row(row), the scalar unroller's (0 + (1 + 2)) + (3 + (4 + 5))
      double t[6];
      for (int k = 0; k < 6; ++k) t[k] = mul(m3[k], -MR(row, k));
      return add(add(t[0], add(t[1], t[2])), add(t[3], add(t[4], t[5])));
    };
    double* f = F + 9 * m;
    f[0] = dot(0); f[1] = dot(1); f[2] = dot(9);
    f[3] = dot(2); f[4] = dot(3); f[5] = f23;
    f[6] = dot(5); f[7] = dot(7); f[8] = 1.0;
  }
#undef MR
  return nb;
}

}  // namespace acr

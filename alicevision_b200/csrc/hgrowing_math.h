// Host + device building blocks of the homography-growing filter (hgrowing.cuh, K12), after
// matchingImageCollection/GeometricFilterMatrix_HGrowing.cpp and geometricFilterUtils.cpp:
//   * computeSimilarity (A2 A1^-1 from the seed's position, scale and orientation), the transfer error of findTransformationInliers,
//     Eigen's isIdentity(1e-12) and the centring of centerMatrix (float mean, float sample deviation, clamped at 0.1), restated;
//   * estimateAffinity and estimateHomography: the fits are restated, not transcribed.  The reference solves them with Eigen's
//     JacobiSVD; here the rows are reduced by a tall-skinny QR (Givens rotations) to a small triangular R, and R goes through a
//     one-sided Jacobi SVD: the minimum-norm least-squares solution with JacobiSVD's rank threshold for the affinity, the right singular
//     vector of the smallest singular value for the homography DLT (never the normal equations);
//   * refineHomography: a restatement of Ceres' trust-region Levenberg-Marquardt at the Solver::Options defaults the reference leaves in
//     place (max_num_iterations = 10), on the residual of RefineHRobustCostFunctor with its analytic Jacobian.
// There is no bit-parity target for any of this: JacobiSVD and Ceres cannot be compiled without Eigen and Ceres, so results agree with
// the reference up to rounding (and a match whose error lies at a tolerance can fall on either side).
//
// The same code runs in the engine (device, one warp per seed or item) and in the oracle's port (host, -ffp-contract=off), and the
// engine and the port agree bit for bit.  For that, every reduction has one fixed order, which the port replays:
//   * lane l of a warp takes the remaining-list positions j = l, l + 32, l + 64, ... in ascending order;
//   * the 32 lane partials are folded as a tree: for off = 16, 8, 4, 2, 1, lane l < off absorbs lane l + off; lane 0 holds the result.
// Double arithmetic goes through acr::mul / add / sub (no contraction); the float centring through fmul / fadd / fsub below.
#pragma once
#include "acransac_math.h"

#include <cfloat>

namespace hg {

using acr::add;
using acr::mul;
using acr::sub;

constexpr int kLanes = 32;
constexpr int kMaxSweeps = 40;        // one-sided Jacobi sweeps (convergence takes far fewer on these sizes)
constexpr double kIdentityPrec = 1e-12;
constexpr double kRobustT = 0.25;     // RefineHRobustCostFunctor::robustify

ACR_HD float fmul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
ACR_HD float fadd(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
ACR_HD float fsub(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}

// exp and log of the refine, written out so that the engine and the port evaluate them identically (CUDA's and glibc's libm can
// differ in the last bit, and these values feed every bit of the refined homography): Cody-Waite reduction by ln 2, then a Taylor
// polynomial (exp) or the atanh series of log m = 2 atanh((m - 1) / (m + 1)), m in [sqrt(1/2), sqrt(2)) (log).  Both are within a few
// ulp of the correctly rounded values on the ranges used here.
// true for a finite value (x - x is NaN for inf and NaN)
ACR_HD bool finite_(double x) { return sub(x, x) == 0; }

constexpr double kLn2Hi = 6.93147180369123816490e-01, kLn2Lo = 1.90821492927058770002e-10;

ACR_HD double exp_(double x) {
  if (x != x) return x;
  if (x > 709.0) return INFINITY;
  if (x < -745.0) return 0.0;
  const double k = rint(x / 0.69314718055994530942);
  const double r = sub(sub(x, mul(k, kLn2Hi)), mul(k, kLn2Lo));
  double p = 1.0 / 6227020800.0;   // 1/13!
  const double inv[13] = {1.0 / 479001600.0, 1.0 / 39916800.0, 1.0 / 3628800.0, 1.0 / 362880.0, 1.0 / 40320.0, 1.0 / 5040.0,
                          1.0 / 720.0, 1.0 / 120.0, 1.0 / 24.0, 1.0 / 6.0, 0.5, 1.0, 1.0};
  for (int q = 0; q < 13; ++q) p = add(mul(p, r), inv[q]);
  return ldexp(p, (int)k);
}

ACR_HD double log_(double y) {
  if (y != y || y < 0) return NAN;
  if (y == 0) return -INFINITY;
  if (y > DBL_MAX) return y;
  int e;
  double m = frexp(y, &e);   // y = m 2^e, m in [0.5, 1)
  if (m < 0.70710678118654752440) { m = mul(m, 2.0); --e; }
  const double s = sub(m, 1.0) / add(m, 1.0), s2 = mul(s, s);
  double p = 1.0 / 25.0;
  for (int n = 11; n >= 0; --n) p = add(mul(p, s2), 1.0 / (2 * n + 1));
  const double lm = mul(mul(2.0, s), p);
  return add(add(mul((double)e, kLn2Lo), lm), mul((double)e, kLn2Hi));
}

// GrowParameters + HGrowingFilteringParam (GeometricFilterMatrix_HGrowing.hpp); _maxFractionPlanarMatches is unused by the reference
struct Param {
  double tol_similarity = 20, tol_affinity = 10, tol_homography = 5;
  int min_inliers_to_refine = 6, nb_refining_iterations = 8;
  int max_nb_homographies = 10, min_nb_matches_per_h = 20;
};

// One putative: xI, yI, scaleI, orientationI, xJ, yJ, scaleJ, orientationJ (the PointFeatures of its two features)
constexpr int kFeat = 8;

// The tolerance of growHomography's step s: similarity, affinity (s <= 4), homography
ACR_HD double step_tolerance(const Param& p, int s) { return s == 0 ? p.tol_similarity : (s <= 4 ? p.tol_affinity : p.tol_homography); }

// 3 x 3 row-major product C = A B, each entry (a0 b0 + a1 b1) + a2 b2
ACR_HD void mat3_mul(const double* A, const double* B, double* C) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) C[r * 3 + c] = add(add(mul(A[r * 3], B[c]), mul(A[r * 3 + 1], B[3 + c])), mul(A[r * 3 + 2], B[6 + c]));
}

// computeSimilarity: S = A2 A1^-1, A = [s cos(o), -s sin(o), x; s sin(o), s cos(o), y; 0, 0, 1] (float features widened to double)
ACR_HD void similarity(const float* f, double S[9]) {
  double A[2][9];
  for (int k = 0; k < 2; ++k) {
    const double x = f[4 * k], y = f[4 * k + 1], s = f[4 * k + 2], o = f[4 * k + 3];
    const double c = cos(o), sn = sin(o);
    A[k][0] = mul(s, c); A[k][1] = mul(s, -sn); A[k][2] = x;
    A[k][3] = mul(s, sn); A[k][4] = mul(s, c); A[k][5] = y;
    A[k][6] = 0; A[k][7] = 0; A[k][8] = 1;
  }
  double A1i[9];
  acr::inverse3(A[0], A1i);
  mat3_mul(A[1], A1i, S);
}

// findTransformationInliers' error (ptJ - (T (ptI, 1)).hnormalized()).squaredNorm(), in the operation order of K11's homography error
// (guided.cuh guided_left + guided_error).  A zero third component gives inf or NaN, and NaN is never below a tolerance.
ACR_HD double transfer_error(const double* T, const float* f) {
  const double x = f[0], y = f[1];
  double u = add(add(mul(T[0], x), mul(T[1], y)), T[2]);
  double v = add(add(mul(T[3], x), mul(T[4], y)), T[5]);
  const double w = add(add(mul(T[6], x), mul(T[7], y)), T[8]);
  u = u / w; v = v / w;
  const double d0 = sub((double)f[4], u), d1 = sub((double)f[5], v);
  return add(mul(d0, d0), mul(d1, d1));
}

// Eigen's isIdentity(1e-12): |T(i,i) - 1| <= min(|T(i,i)|, 1) prec on the diagonal, |T(i,j)| <= prec elsewhere
ACR_HD bool is_identity(const double* T) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const double a = T[i * 3 + j];
      if (i == j) {
        if (!(fabs(sub(a, 1.0)) <= mul(fmin(fabs(a), 1.0), kIdentityPrec))) return false;
      } else if (!(fabs(a) <= kIdentityPrec)) {
        return false;
      }
    }
  return true;
}

// ------------------------------------------------------------------------------------------------ tall-skinny QR
// An M x W upper-trapezoidal R, rows packed: row i holds columns i..W-1.
template <int M, int W>
struct Tri {
  static constexpr int kSize = M * W - M * (M - 1) / 2;
  double r[kSize];
  static constexpr ACR_HD int at(int i, int k) { return i * W - i * (i - 1) / 2 + (k - i); }
};

template <int M, int W>
ACR_HD void tri_zero(Tri<M, W>& t) {
  for (int q = 0; q < Tri<M, W>::kSize; ++q) t.r[q] = 0;
}

// Absorb row v (zero in columns < i0) into R by Givens rotations: for each column i, (R(i,i), v(i)) -> (sqrt(a^2 + b^2), 0)
template <int M, int W>
ACR_HD void tri_absorb(Tri<M, W>& t, double* v, int i0) {
  for (int i = i0; i < M; ++i) {
    const double b = v[i];
    if (b == 0) continue;
    const double a = t.r[Tri<M, W>::at(i, i)];
    const double rr = sqrt(add(mul(a, a), mul(b, b)));
    const double c = a / rr, s = b / rr;
    t.r[Tri<M, W>::at(i, i)] = rr;
    for (int k = i + 1; k < W; ++k) {
      const double x = t.r[Tri<M, W>::at(i, k)], y = v[k];
      t.r[Tri<M, W>::at(i, k)] = add(mul(c, x), mul(s, y));
      v[k] = sub(mul(c, y), mul(s, x));
    }
  }
}

// The fold step "lane l absorbs lane l + off": R_lo absorbs the rows of R_hi, row 0 first
template <int M, int W>
ACR_HD void tri_merge(Tri<M, W>& lo, const Tri<M, W>& hi) {
  for (int i = 0; i < M; ++i) {
    double v[W];
    for (int k = 0; k < W; ++k) v[k] = k < i ? 0.0 : hi.r[Tri<M, W>::at(i, k)];
    tri_absorb(lo, v, i);
  }
}

// One-sided (Hestenes) Jacobi SVD of the M x M matrix whose columns are a[c][.]: rotates column pairs until every pair is orthogonal
// to working precision; on return the column norms are the singular values and v[c][.] the right singular vectors (columns).
template <int M>
ACR_HD void jacobi_svd(double a[M][M], double v[M][M]) {
  for (int c = 0; c < M; ++c)
    for (int r = 0; r < M; ++r) v[c][r] = c == r ? 1.0 : 0.0;
  for (int sweep = 0; sweep < kMaxSweeps; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < M - 1; ++p)
      for (int q = p + 1; q < M; ++q) {
        double al = 0, be = 0, ga = 0;
        for (int r = 0; r < M; ++r) {
          al = add(al, mul(a[p][r], a[p][r]));
          be = add(be, mul(a[q][r], a[q][r]));
          ga = add(ga, mul(a[p][r], a[q][r]));
        }
        if (!(fabs(ga) > mul(DBL_EPSILON, sqrt(mul(al, be))))) continue;
        const double zeta = sub(be, al) / mul(2.0, ga);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / add(fabs(zeta), sqrt(add(1.0, mul(zeta, zeta))));
        const double c = 1.0 / sqrt(add(1.0, mul(t, t))), s = mul(c, t);
        if (s == 0) continue;
        rotated = true;
        for (int r = 0; r < M; ++r) {
          const double x = a[p][r], y = a[q][r];
          a[p][r] = sub(mul(c, x), mul(s, y));
          a[q][r] = add(mul(s, x), mul(c, y));
          const double vx = v[p][r], vy = v[q][r];
          v[p][r] = sub(mul(c, vx), mul(s, vy));
          v[q][r] = add(mul(s, vx), mul(c, vy));
        }
      }
    if (!rotated) break;
  }
}

template <int M>
ACR_HD double col_norm(const double a[M][M], int c) {
  double s = 0;
  for (int r = 0; r < M; ++r) s = add(s, mul(a[c][r], a[c][r]));
  return sqrt(s);
}

// ------------------------------------------------------------------------------------------------ estimateAffinity
// Rows [x y 1 | xJ yJ] of the inliers: R (3 x 3) and Q^T b for both right-hand sides
using AffAcc = Tri<3, 5>;

ACR_HD void aff_add(AffAcc& acc, const float* f) {
  double v[5] = {(double)f[0], (double)f[1], 1.0, (double)f[4], (double)f[5]};
  tri_absorb(acc, v, 0);
}

// The minimum-norm least-squares solution: by back-substitution in R when every singular value is kept, otherwise
// a = sum over kept sigma_i of v_i (u_i . c) / sigma_i, where a singular value is kept when
// sigma_i >= max(6 eps sigma_max, DBL_MIN): JacobiSVD's rank() on the 2k x 6 block system, whose singular values are those of [x y 1]
// each twice.  The result is [a0 a1 a2; a3 a4 a5; 0 0 1].
ACR_HD void aff_solve(const AffAcc& acc, double T[9]) {
  double a[3][3], v[3][3];
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r) a[c][r] = r <= c ? acc.r[AffAcc::at(r, c)] : 0.0;
  jacobi_svd<3>(a, v);
  double sig[3], smax = 0;
  for (int c = 0; c < 3; ++c) { sig[c] = col_norm<3>(a, c); smax = fmax(smax, sig[c]); }
  const double th = fmax(mul(mul(6.0, DBL_EPSILON), smax), DBL_MIN);
  double sol[2][3] = {{0, 0, 0}, {0, 0, 0}};
  if (sig[0] >= th && sig[1] >= th && sig[2] >= th) {
    // full rank: the least-squares solution is unique, R a = Q^T b by back-substitution (exact when b is a column of [x y 1])
    for (int h = 0; h < 2; ++h)
      for (int r = 2; r >= 0; --r) {
        double s = acc.r[AffAcc::at(r, 3 + h)];
        for (int q = r + 1; q < 3; ++q) s = sub(s, mul(acc.r[AffAcc::at(r, q)], sol[h][q]));
        sol[h][r] = s / acc.r[AffAcc::at(r, r)];
      }
    for (int r = 0; r < 3; ++r) { T[r] = sol[0][r]; T[3 + r] = sol[1][r]; }
    T[6] = 0; T[7] = 0; T[8] = 1;
    return;
  }
  for (int c = 0; c < 3; ++c) {
    if (!(sig[c] >= th)) continue;
    const double s2 = mul(sig[c], sig[c]);
    for (int h = 0; h < 2; ++h) {
      double d = 0;
      for (int r = 0; r < 3; ++r) d = add(d, mul(a[c][r], acc.r[AffAcc::at(r, 3 + h)]));
      const double g = d / s2;
      for (int r = 0; r < 3; ++r) sol[h][r] = add(sol[h][r], mul(v[c][r], g));
    }
  }
  for (int r = 0; r < 3; ++r) { T[r] = sol[0][r]; T[3 + r] = sol[1][r]; }
  T[6] = 0; T[7] = 0; T[8] = 1;
}

// ------------------------------------------------------------------------------------------------ estimateHomography
// centerMatrix in float: pass 1 sums the coordinates, pass 2 the squared deviations from the float mean
struct CenAcc { float s[4]; };   // xI, yI, xJ, yJ
ACR_HD void cen_zero(CenAcc& c) { for (int q = 0; q < 4; ++q) c.s[q] = 0.f; }
ACR_HD void cen_add_sum(CenAcc& c, const float* f) {
  c.s[0] = fadd(c.s[0], f[0]); c.s[1] = fadd(c.s[1], f[1]); c.s[2] = fadd(c.s[2], f[4]); c.s[3] = fadd(c.s[3], f[5]);
}
ACR_HD void cen_add_dev(CenAcc& c, const float* mean, const float* f) {
  const float p[4] = {f[0], f[1], f[4], f[5]};
  for (int q = 0; q < 4; ++q) {
    const float d = fsub(p[q], mean[q]);
    c.s[q] = fadd(c.s[q], fmul(d, d));
  }
}
ACR_HD void cen_merge(CenAcc& lo, const CenAcc& hi) { for (int q = 0; q < 4; ++q) lo.s[q] = fadd(lo.s[q], hi.s[q]); }
ACR_HD void cen_mean(const CenAcc& sum, int k, float mean[4]) { for (int q = 0; q < 4; ++q) mean[q] = sum.s[q] / (float)k; }

// t = [1/sd_x, 0, -mean_x/sd_x; 0, 1/sd_y, -mean_y/sd_y; 0, 0, 1] with sd = sqrt(dev / (k - 1)) clamped below at 0.1, for I (q0 = 0)
// and J (q0 = 2); 1. / sd in double, -mean / sd in float
ACR_HD void cen_matrix(const float mean[4], const CenAcc& dev, int k, int q0, double t[9]) {
  float sd[2];
  for (int d = 0; d < 2; ++d) {
    sd[d] = sqrtf(dev.s[q0 + d] / (float)(k - 1));
    if (sd[d] < 0.1f) sd[d] = 0.1f;
  }
  t[0] = 1.0 / (double)sd[0]; t[1] = 0; t[2] = (double)(-mean[q0] / sd[0]);
  t[3] = 0; t[4] = 1.0 / (double)sd[1]; t[5] = (double)(-mean[q0 + 1] / sd[1]);
  t[6] = 0; t[7] = 0; t[8] = 1;
}

using DltAcc = Tri<9, 9>;

ACR_HD void mat3_vec(const double* M, double x, double y, double o[3]) {
  for (int r = 0; r < 3; ++r) o[r] = add(add(mul(M[r * 3], x), mul(M[r * 3 + 1], y)), M[r * 3 + 2]);
}

// The two DLT rows of one inlier on the centred points pI = CI (x, 1), pJ = CJ (y, 1):
//   [pI, 0, -pJ0 pI] and [0, pI, -pJ1 pI]
ACR_HD void dlt_add(DltAcc& acc, const double* CI, const double* CJ, const float* f) {
  double pI[3], pJ[3];
  mat3_vec(CI, (double)f[0], (double)f[1], pI);
  mat3_vec(CJ, (double)f[4], (double)f[5], pJ);
  double a[9], b[9];
  for (int k = 0; k < 3; ++k) {
    a[k] = pI[k]; a[3 + k] = 0; a[6 + k] = mul(-pJ[0], pI[k]);
    b[k] = 0; b[3 + k] = pI[k]; b[6 + k] = mul(-pJ[1], pI[k]);
  }
  tri_absorb(acc, a, 0);
  tri_absorb(acc, b, 0);
}

// H0 = the right singular vector of R's smallest singular value (the first of equal ones), H = CJ^-1 H0 CI, then H /= H(2,2) when
// |H(2,2)| > DBL_EPSILON
ACR_HD void dlt_solve(const DltAcc& acc, const double* CI, const double* CJ, double H[9]) {
  double a[9][9], v[9][9];
  for (int c = 0; c < 9; ++c)
    for (int r = 0; r < 9; ++r) a[c][r] = r <= c ? acc.r[DltAcc::at(r, c)] : 0.0;
  jacobi_svd<9>(a, v);
  int best = 0;
  double bs = col_norm<9>(a, 0);
  for (int c = 1; c < 9; ++c) {
    const double s = col_norm<9>(a, c);
    if (s < bs) { bs = s; best = c; }
  }
  double CJi[9], T[9];
  acr::inverse3(CJ, CJi);
  mat3_mul(CJi, v[best], T);
  mat3_mul(T, CI, H);
  const double h22 = H[8];
  if (fabs(h22) > DBL_EPSILON)
    for (int q = 0; q < 9; ++q) H[q] = H[q] / h22;
}

// ------------------------------------------------------------------------------------------------ refineHomography
// Parameters p are Ceres' view of the Eigen matrix: column-major, p[3 c + r] = H(r, c).
// RefineHRobustCostFunctor: e2 = |y - (H (x, 1)).hnormalized()|^2, e = e2 == 0 ? e2 : sqrt(e2),
// r = -log(exp(-e^2 / (2 sigma^2)) + t) + log(1 + t), sigma = tol / sqrt(-log(t^2)), t = 0.25.
// Its Jacobian: dr/dp = 2 E / (2 sigma^2 (E + t)) (ex dex/dp + ey dey/dp), E = exp(-e^2 / (2 sigma^2)); zero in the e2 == 0 branch
// (where the functor's Jet derivative is 0 too).
struct LmAcc {
  double jtj[45];   // J^T J, upper triangle packed by rows (Tri<9, 9> order)
  double jtr[9];    // J^T r, the gradient of the cost
  double rr;        // sum of r^2
};
constexpr int kLmDoubles = 55;

ACR_HD double two_sigma2(double tol) {
  const double sigma = tol / sqrt(-log_(mul(kRobustT, kRobustT)));
  return mul(mul(2.0, sigma), sigma);
}

// The residual of one match at p; J (9 entries) when non-null
ACR_HD double lm_residual(const double* p, double ts2, const float* f, double* J) {
  const double x = f[0], y = f[1];
  const double u = add(add(mul(p[0], x), mul(p[3], y)), p[6]);
  const double v = add(add(mul(p[1], x), mul(p[4], y)), p[7]);
  const double w = add(add(mul(p[2], x), mul(p[5], y)), p[8]);
  const double uw = u / w, vw = v / w;
  const double ex = sub((double)f[4], uw), ey = sub((double)f[5], vw);
  const double e2 = add(mul(ex, ex), mul(ey, ey));
  const double e = e2 == 0 ? e2 : sqrt(e2);
  const double E = exp_(-mul(e, e) / ts2);
  const double r = add(-log_(add(E, kRobustT)), log_(1.0 + kRobustT));
  if (J) {
    if (e2 == 0) {
      for (int q = 0; q < 9; ++q) J[q] = 0;
    } else {
      const double k = mul(2.0, E) / mul(ts2, add(E, kRobustT));
      const double X[3] = {x, y, 1.0};
      const double gx = mul(k, ex), gy = mul(k, ey);
      const double g2 = add(mul(gx, uw), mul(gy, vw));
      for (int c = 0; c < 3; ++c) {
        const double xw = X[c] / w;
        J[3 * c] = -mul(gx, xw);
        J[3 * c + 1] = -mul(gy, xw);
        J[3 * c + 2] = mul(g2, xw);
      }
    }
  }
  return r;
}

ACR_HD void lm_zero(LmAcc& a) {
  for (int q = 0; q < 45; ++q) a.jtj[q] = 0;
  for (int q = 0; q < 9; ++q) a.jtr[q] = 0;
  a.rr = 0;
}

ACR_HD void lm_add(LmAcc& a, const double* p, double ts2, const float* f, bool jac) {
  double J[9];
  const double r = lm_residual(p, ts2, f, jac ? J : nullptr);
  a.rr = add(a.rr, mul(r, r));
  if (!jac) return;
  for (int i = 0; i < 9; ++i) {
    a.jtr[i] = add(a.jtr[i], mul(J[i], r));
    for (int k = i; k < 9; ++k) a.jtj[DltAcc::at(i, k)] = add(a.jtj[DltAcc::at(i, k)], mul(J[i], J[k]));
  }
}

ACR_HD void lm_merge(LmAcc& lo, const LmAcc& hi) {
  for (int q = 0; q < 45; ++q) lo.jtj[q] = add(lo.jtj[q], hi.jtj[q]);
  for (int q = 0; q < 9; ++q) lo.jtr[q] = add(lo.jtr[q], hi.jtr[q]);
  lo.rr = add(lo.rr, hi.rr);
}

ACR_HD bool lm_finite(const LmAcc& a, bool jac) {
  if (!finite_(a.rr)) return false;
  if (jac)
    for (int i = 0; i < 9; ++i)
      if (!finite_(a.jtj[DltAcc::at(i, i)]) || !finite_(a.jtr[i])) return false;
  return true;
}

// Solve (A + diag(d)) y = b for the 9 x 9 symmetric A (packed upper) by Cholesky; false when a pivot is not positive and finite
ACR_HD bool lm_solve(const double* A, const double* d, const double* b, double* y) {
  double L[45];   // packed lower triangle by rows: L(i, k), k <= i at i (i + 1) / 2 + k
  for (int i = 0; i < 9; ++i)
    for (int k = 0; k <= i; ++k) {
      double s = k == i ? add(A[DltAcc::at(k, i)], d[i]) : A[DltAcc::at(k, i)];
      for (int m = 0; m < k; ++m) s = sub(s, mul(L[i * (i + 1) / 2 + m], L[k * (k + 1) / 2 + m]));
      if (k == i) {
        if (!(s > 0) || !finite_(s)) return false;
        L[i * (i + 1) / 2 + i] = sqrt(s);
      } else {
        L[i * (i + 1) / 2 + k] = s / L[k * (k + 1) / 2 + k];
      }
    }
  double z[9];
  for (int i = 0; i < 9; ++i) {
    double s = b[i];
    for (int m = 0; m < i; ++m) s = sub(s, mul(L[i * (i + 1) / 2 + m], z[m]));
    z[i] = s / L[i * (i + 1) / 2 + i];
  }
  for (int i = 8; i >= 0; --i) {
    double s = z[i];
    for (int m = i + 1; m < 9; ++m) s = sub(s, mul(L[m * (m + 1) / 2 + i], y[m]));
    y[i] = s / L[i * (i + 1) / 2 + i];
  }
  return true;
}

// Ceres' TrustRegionMinimizer with the LEVENBERG_MARQUARDT strategy at the Solver::Options defaults, max_num_iterations = 10:
// Jacobi column scaling s_i = 1 / (1 + |J_i|) from the first Jacobian; LM diagonal |J_i s_i|^2 clamped to [1e-6, 1e32], recomputed
// after an accepted step only; step = -(Js^T Js + D / radius)^-1 Js^T r in the scaled space, delta = step * s; initial radius 1e4,
// maximum 1e16; a step is accepted when (cost - cost') / model decrease > 1e-3, then radius /= max(1/3, 1 - (2 rho - 1)^3) and the
// decrease factor resets to 2; otherwise radius /= factor and the factor doubles; a non-positive model decrease is an invalid step
// (treated as a rejection; five in a row fail the solve).  Termination: gradient max norm <= 1e-10 (also before the first step),
// |cost - cost'| <= 1e-6 cost, |delta| <= (|x| + 1e-8) 1e-8, radius < 1e-32, or 10 iterations.
// eval(p, jac, acc) fills acc over the residual blocks.  Returns whether the solution is usable (Summary::IsSolutionUsable): false when
// an evaluation at an accepted point (the initial one included) is not finite, or after five invalid steps in a row.  p holds the
// solution (the last accepted point).
template <class Eval>
ACR_HD bool lm_refine(double p[9], Eval& eval) {
  LmAcc A;
  eval(p, true, A);
  if (!lm_finite(A, true)) return false;
  double cost = mul(0.5, A.rr);
  double scale[9];
  for (int i = 0; i < 9; ++i) scale[i] = 1.0 / add(1.0, sqrt(A.jtj[DltAcc::at(i, i)]));
  auto gmax_of = [](const LmAcc& a) {
    double g = 0;
    for (int i = 0; i < 9; ++i) g = fmax(g, fabs(a.jtr[i]));
    return g;
  };
  if (gmax_of(A) <= 1e-10) return true;
  double radius = 1e4, factor = 2.0, diag[9];
  bool reuse = false;
  int invalid = 0;
  for (int iter = 1; iter <= 10; ++iter) {
    double S[45], g[9];   // Js^T Js and Js^T r
    for (int i = 0; i < 9; ++i) {
      g[i] = mul(A.jtr[i], scale[i]);
      for (int k = i; k < 9; ++k) S[DltAcc::at(i, k)] = mul(mul(A.jtj[DltAcc::at(i, k)], scale[i]), scale[k]);
    }
    if (!reuse)
      for (int i = 0; i < 9; ++i) diag[i] = fmin(fmax(S[DltAcc::at(i, i)], 1e-6), 1e32);
    reuse = true;
    double d[9], y[9];
    for (int i = 0; i < 9; ++i) d[i] = diag[i] / radius;
    bool valid = lm_solve(S, d, g, y);
    double model = 0;
    if (valid) {
      double sg = 0, sSs = 0;   // -(step^T g + step^T S step / 2), step = -y
      for (int i = 0; i < 9; ++i) {
        sg = add(sg, mul(-y[i], g[i]));
        double Sy = 0;
        for (int k = 0; k < 9; ++k) Sy = add(Sy, mul(S[i <= k ? DltAcc::at(i, k) : DltAcc::at(k, i)], -y[k]));
        sSs = add(sSs, mul(-y[i], Sy));
      }
      model = -add(sg, mul(0.5, sSs));
      valid = model > 0;
    }
    if (!valid) {
      if (++invalid >= 5) return false;
      radius = radius / factor; factor = mul(factor, 2.0);
      if (radius < 1e-32) return true;
      continue;
    }
    invalid = 0;
    double xn[9], xnorm = 0, snorm = 0;
    for (int i = 0; i < 9; ++i) {
      xn[i] = add(p[i], mul(-y[i], scale[i]));
      xnorm = add(xnorm, mul(p[i], p[i]));
      const double dd = sub(p[i], xn[i]);
      snorm = add(snorm, mul(dd, dd));
    }
    LmAcc C;
    eval(xn, false, C);
    const double cand = lm_finite(C, false) ? mul(0.5, C.rr) : DBL_MAX;
    if (sqrt(snorm) <= mul(add(sqrt(xnorm), 1e-8), 1e-8)) return true;
    const double change = sub(cost, cand);
    if (fabs(change) <= mul(1e-6, cost)) return true;
    const double rho = change / model;
    if (rho > 1e-3) {
      for (int i = 0; i < 9; ++i) p[i] = xn[i];
      eval(p, true, A);
      if (!lm_finite(A, true)) return false;
      cost = mul(0.5, A.rr);
      const double q = sub(mul(2.0, rho), 1.0);
      radius = fmin(radius / fmax(1.0 / 3.0, sub(1.0, mul(mul(q, q), q))), 1e16);
      factor = 2.0;
      reuse = false;
      if (gmax_of(A) <= 1e-10) return true;
    } else {
      radius = radius / factor; factor = mul(factor, 2.0);
    }
    if (radius < 1e-32) return true;
  }
  return true;
}

// H (row-major) <-> Ceres' column-major parameters; after a usable solve H /= H(2,2) when |H(2,2)| > DBL_EPSILON
ACR_HD void to_params(const double* H, double* p) { for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) p[3 * c + r] = H[3 * r + c]; }
ACR_HD void from_params(const double* p, double* H) {
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) H[3 * r + c] = p[3 * c + r];
  const double h22 = H[8];
  if (fabs(h22) > DBL_EPSILON)
    for (int q = 0; q < 9; ++q) H[q] = H[q] / h22;
}

}  // namespace hg

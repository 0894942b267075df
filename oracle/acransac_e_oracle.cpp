// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product; nothing under alicevision_b200/ may include, link or call this file.
//
// A-contrario RANSAC essential-matrix estimation of one pair of pinhole cameras, as GeometricFilterMatrix_E_AC::geometricEstimation
// runs it (matchingImageCollection/GeometricFilterMatrix_E_AC.hpp): ACRANSAC over RelativePoseKernel_K<Essential5PSolver,
// FundamentalEpipolarDistanceError, Mat3Model>, the std::mt19937 passed by reference.  Built twice by oracle/Makefile (`all`, `ref`)
// around the loop, sampling and estimate driver of oracle/acransac_loop.h; the port takes the sampling and the kernel from the
// engine's alicevision_b200/csrc/acransac_math.h.
// The kernel (K^-1 applied once to the pixels, the 5-point solver on them, F = K_J^-T E K_I^-1 and the point-to-line error on the
// pixels; thresholdNormalizer = 1, unormalizeError = sqrt, errorVectorDimension = 0.5, logalpha0 = log10(2 D / A * .5)) is restated
// in both builds: the reference's Essential5PSolver needs Eigen.  Everything else in "ref" is compiled reference code, so "ref" ==
// "port" bit for bit pins the control flow, the 5-sample draws, the NFA with d = 0.5 and the generator's end state.
#include "acransac_loop.h"

namespace {

struct Model : TracedModel {
  double F[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
};

// RelativePoseKernel_K<Essential5PSolver, FundamentalEpipolarDistanceError, Mat3Model>, restated
struct EKernel {
  using ModelT = Model;
  std::vector<double> px, nx;   // 4 per correspondence: the pixels (xI, yI, xJ, yJ) and K^-1 applied to them
  double kinv[18];
  int w2, h2;

  EKernel(const double* corr, int n, const double* K, int w2_, int h2_) : w2(w2_), h2(h2_) {
    acr::inverse3(K, kinv);
    acr::inverse3(K + 9, kinv + 9);
    for (int i = 0; i < n; ++i) {
      double u[4];
      acr::transform_point(kinv, corr[4 * i], corr[4 * i + 1], u[0], u[1]);
      acr::transform_point(kinv + 9, corr[4 * i + 2], corr[4 * i + 3], u[2], u[3]);
      for (int t = 0; t < 4; ++t) { px.push_back(corr[4 * i + t]); nx.push_back(u[t]); }
    }
  }
  static constexpr int kSampleSize = acr::kSampleE;
  std::size_t getMinimumNbRequiredSamples() const { return kSampleSize; }
  std::size_t getMaximumNbModels() const { return acr::kMaxModelsE; }
  std::size_t nbSamples() const { return px.size() / 4; }
  double logalpha0() const { return acr::logalpha0_e(w2, h2); }
  double errorVectorDimension() const { return 0.5; }
  double thresholdNormalizer() const { return 1; }
  double unormalizeError(double v) const { return sqrt(v); }
  void unnormalize(Model&) const {}
  void fit(const std::vector<std::size_t>& s, std::vector<Model>& models) const {
    trace_fit();
    double a[5], b[5], c[5], d[5], E[90];
    for (int i = 0; i < 5; ++i) { a[i] = nx[4 * s[i]]; b[i] = nx[4 * s[i] + 1]; c[i] = nx[4 * s[i] + 2]; d[i] = nx[4 * s[i] + 3]; }
    const int nb = acr::fit5(a, b, c, d, E);
    for (int m = 0; m < nb; ++m) {
      Model M;
      std::memcpy(M.F, E + 9 * m, sizeof M.F);
      models.push_back(M);
    }
  }
  void errors(const Model& m, std::vector<double>& e) const {
    double F[9];
    acr::fundamental_from_essential(m.F, kinv, kinv + 9, F);
    for (std::size_t i = 0; i < nbSamples(); ++i) e[i] = acr::epipolar_error(F, px[4 * i], px[4 * i + 1], px[4 * i + 2], px[4 * i + 3]);
  }
};

}  // namespace

extern "C" {

// 1 = "ref" (compiled reference loop, sampling and NFA), 0 = "port"
int acre_is_reference(void) { return is_reference(); }

// std::mt19937(seed) as 624 words + position (the library's operator<< order)
void acre_mt_seed(uint32_t seed, uint32_t* state) { mt_seed(seed, state); }

// The E kernel's primitives, for the tests that check them against an independent high-precision reference.
// the 5-point solver on 5 normalised correspondences (5 x (xI, yI, xJ, yJ)): models row-major in E[90]; returns their number
int acre_fit5(const double* c, double* E) {
  double a[5], b[5], cc[5], d[5];
  for (int i = 0; i < 5; ++i) { a[i] = c[4 * i]; b[i] = c[4 * i + 1]; cc[i] = c[4 * i + 2]; d[i] = c[4 * i + 3]; }
  return acr::fit5(a, b, cc, d, E);
}

// the action matrix the solver builds from 5 normalised correspondences (as acre_fit5 takes them), row-major in At[100]
void acre_action(const double* c, double* At) {
  double A[5][9], Eb[9][4], M[10][10];
  for (int i = 0; i < 5; ++i) {   // encodeEpipolarEquation, as acr::fit5 writes it
    const double x1 = c[4 * i], y1 = c[4 * i + 1], x2 = c[4 * i + 2], y2 = c[4 * i + 3];
    const double row[9] = {x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, 1.0};
    for (int t = 0; t < 9; ++t) A[i][t] = row[t];
  }
  acr::e5::action_matrix(A, Eb, M);
  for (int r = 0; r < 10; ++r)
    for (int q = 0; q < 10; ++q) At[10 * r + q] = M[r][q];
}

// the action matrix's eigenvalues as the solver sees them (re, im in Schur order); returns 0 where the solver gives no model
int acre_eigen(const double* A, double* re, double* im) {
  double M[10][10], V[10][10];
  for (int r = 0; r < 10; ++r)
    for (int c = 0; c < 10; ++c) M[r][c] = A[10 * r + c];
  return acr::e5::eigen_solve(M, re, im, V) ? 1 : 0;
}

// geometricEstimation's ACRANSAC of one pair.  corr: n x (xI, yI, xJ, yJ) pixels; K: K_I then K_J, row-major; w2, h2: view J's size.
// precision: ACRANSAC's argument (the filter's Square(m_dPrecision)).  inliers: capacity n.
// state: the generator on entry; state_out: the generator after the estimation (the reference's std::mt19937& afterwards).
// trace: the iterations at which a better model was found (first trace_cap of *n_trace); trace_nfa: the new minNFA of each (NaN in
// the "ref" build).  Returns the iterations executed.
long acre_estimate(int n, const double* corr, const double* K, int w2, int h2, const uint32_t* state, long max_iter, double precision, int* valid, int* n_inliers,
                   uint32_t* inliers, double* F, double* error_max, double* min_nfa, int* trace, double* trace_nfa, int trace_cap,
                   int* n_trace, uint32_t* state_out) {
  Model model;
  const long fits = estimate(EKernel(corr, n, K, w2, h2), state, state_out, max_iter, precision, model, valid, n_inliers, inliers,
                             error_max, min_nfa, trace, trace_nfa, trace_cap, n_trace);
  std::memcpy(F, model.F, sizeof model.F);
  return fits;
}

}  // extern "C"

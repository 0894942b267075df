// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product; nothing under alicevision_b200/ may include, link or call this file.
//
// A-contrario RANSAC fundamental-matrix estimation of one pair, as GeometricFilterMatrix_F_AC::geometricEstimation_Mat_ACRANSAC
// <Fundamental7PSolver, Mat3Model> runs it (matchingImageCollection/GeometricFilterMatrix_F_AC.hpp:266-299).
// Built twice by oracle/Makefile (`all`, `ref`) around the loop, sampling and estimate driver of oracle/acransac_loop.h; the "ref"
// build also compiles SolveCubicPolynomial (numeric/polynomial.hpp) verbatim, and the port takes the sampling and the F kernel from
// the engine's alicevision_b200/csrc/acransac_math.h.
// The F kernel (normalisation, 7-point fit with its Householder null space, error, unnormalisation) is restated in both builds:
// the reference takes its null space from Eigen's JacobiSVD, which is not available here.  Everything else in "ref" is compiled
// reference code, so "ref" == "port" bit for bit pins the control flow, the sampling, the NFA and the cubic solver.
#ifdef ACR_USE_REFERENCE
#include <aliceVision/numeric/polynomial.hpp>
#define ACR_REFERENCE_CUBIC aliceVision::SolveCubicPolynomial<double>
#endif
#include "acransac_loop.h"

namespace {

struct Model : TracedModel {
  double F[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
};

// RelativePoseKernel<Fundamental7PSolver, FundamentalEpipolarDistanceError, UnnormalizerT, Mat3Model>, restated
struct FKernel {
  using ModelT = Model;
  std::vector<double> x1, y1, x2, y2;   // normalised
  acr::Norm n1, n2;
  double la0;

  FKernel(const double* corr, int n, int w1, int h1, int w2, int h2) {
    n1 = acr::precondition(w1, h1);
    n2 = acr::precondition(w2, h2);
    for (int i = 0; i < n; ++i) {
      x1.push_back(acr::norm_x(n1, corr[4 * i])); y1.push_back(acr::norm_y(n1, corr[4 * i + 1]));
      x2.push_back(acr::norm_x(n2, corr[4 * i + 2])); y2.push_back(acr::norm_y(n2, corr[4 * i + 3]));
    }
    const double D = sqrt(w2 * (double)w2 + h2 * (double)h2);
    const double A = w2 * (double)h2;
    la0 = log10(2.0 * D / A / n2.s);
  }
  static constexpr int kSampleSize = acr::kSample;
  std::size_t getMinimumNbRequiredSamples() const { return kSampleSize; }
  std::size_t getMaximumNbModels() const { return acr::kMaxModels; }
  std::size_t nbSamples() const { return x1.size(); }
  double logalpha0() const { return la0; }
  double errorVectorDimension() const { return 1.0; }
  double thresholdNormalizer() const { return n2.s; }
  double unormalizeError(double v) const { return sqrt(v) / n2.s; }
  void unnormalize(Model& m) const { acr::unnormalize(n1, n2, m.F); }
  void fit(const std::vector<std::size_t>& s, std::vector<Model>& models) const {
    trace_fit();
    double a[7], b[7], c[7], d[7], F[27];
    for (int i = 0; i < 7; ++i) { a[i] = x1[s[i]]; b[i] = y1[s[i]]; c[i] = x2[s[i]]; d[i] = y2[s[i]]; }
    const int nb = acr::fit7(a, b, c, d, F);
    for (int m = 0; m < nb; ++m) {
      Model M;
      std::memcpy(M.F, F + 9 * m, sizeof M.F);
      models.push_back(M);
    }
  }
  void errors(const Model& m, std::vector<double>& e) const {
    for (std::size_t i = 0; i < x1.size(); ++i) e[i] = acr::epipolar_error(m.F, x1[i], y1[i], x2[i], y2[i]);
  }
};

}  // namespace

extern "C" {

// 1 = "ref" (compiled reference loop, sampling, NFA and cubic), 0 = "port"
int acr_is_reference(void) { return is_reference(); }

// std::mt19937(seed) as 624 words + position (the library's operator<< order)
void acr_mt_seed(uint32_t seed, uint32_t* state) { mt_seed(seed, state); }

// `draws` consecutive randSample(g, 0, range, 7) from `state`: the samples in their order (draws x 7), and the generator state
// after each draw (draws x 625) when states != nullptr
void acr_rand_sample(const uint32_t* state, int range, int draws, uint32_t* out, uint32_t* states) {
  rand_sample_draws(state, 7, range, draws, out, states);
}

// the float tables logc_n[0..n], logc_k[0..n] of ACRANSAC for sizeSample 7
void acr_logc(int n, float* logc_n, float* logc_k) { logc(7, n, logc_n, logc_k); }

// the 7-point solver alone on 7 raw correspondences (no normalisation): models row-major in F[27]; returns their number
int acr_fit7(const double* corr, double* F) {
  double a[7], b[7], c[7], d[7];
  for (int i = 0; i < 7; ++i) { a[i] = corr[4 * i]; b[i] = corr[4 * i + 1]; c[i] = corr[4 * i + 2]; d[i] = corr[4 * i + 3]; }
  return acr::fit7(a, b, c, d, F);
}

// The F kernel's primitives one by one, for the tests that check them against an independent high-precision reference.
// SolveCubicPolynomial(P, x): the compiled reference's own in the "ref" build, the restated one in "port"; returns the root count.
int acr_solve_cubic(const double* P, double* x) {
#ifdef ACR_USE_REFERENCE
  return aliceVision::SolveCubicPolynomial<double>(P, x);
#else
  return acr::solve_cubic(P, x);
#endif
}

// the null space of a 7 x 9 row-major system: N[2 x 9], rows N[0] = Q e8 and N[1] = Q e7
void acr_nullspace7(const double* A, double* N) {
  double a[7][9], n[2][9];
  std::memcpy(a, A, sizeof a);
  acr::nullspace<7>(a, n);
  std::memcpy(N, n, sizeof n);
}

// FundamentalEpipolarDistanceError of F on n correspondences as given (no normalisation): e[i]
void acr_epipolar_error(const double* F, int n, const double* corr, double* e) {
  for (int i = 0; i < n; ++i) e[i] = acr::epipolar_error(F, corr[4 * i], corr[4 * i + 1], corr[4 * i + 2], corr[4 * i + 3]);
}

// preconditionerFromImageSize(w, h): (s, tx, ty), and the n coordinates x[i], y[i] mapped through it in place
void acr_precondition(int w, int h, double* sxy, int n, double* x, double* y) {
  const acr::Norm nm = acr::precondition(w, h);
  sxy[0] = nm.s; sxy[1] = nm.tx; sxy[2] = nm.ty;
  for (int i = 0; i < n; ++i) { x[i] = acr::norm_x(nm, x[i]); y[i] = acr::norm_y(nm, y[i]); }
}

// UnnormalizerT in place (F <- N2^T F N1), with the kernel's preconditioners of (w1, h1) and (w2, h2)
void acr_unnormalize(int w1, int h1, int w2, int h2, double* F) {
  const FKernel k(nullptr, 0, w1, h1, w2, h2);
  Model m;
  std::memcpy(m.F, F, sizeof m.F);
  k.unnormalize(m);
  std::memcpy(F, m.F, sizeof m.F);
}

// the kernel's logalpha0() and unormalizeError(v) for image J = (w2, h2)
double acr_logalpha0(int w1, int h1, int w2, int h2) { return FKernel(nullptr, 0, w1, h1, w2, h2).logalpha0(); }
double acr_unnormalize_error(int w1, int h1, int w2, int h2, double v) { return FKernel(nullptr, 0, w1, h1, w2, h2).unormalizeError(v); }

// geometricEstimation_Mat_ACRANSAC<Fundamental7PSolver, Mat3Model> of one pair.  corr: n x (xI, yI, xJ, yJ).  inliers: capacity n.
// trace: the iterations at which a better model was found (first trace_cap of *n_trace); trace_nfa: the new minNFA of each
// (NaN in the "ref" build).  Returns the iterations executed.
long acr_estimate(int n, const double* corr, int wI, int hI, int wJ, int hJ, const uint32_t* state, long max_iter, double precision,
                  int* valid, int* n_inliers, uint32_t* inliers, double* F, double* error_max, double* min_nfa, int* trace, double* trace_nfa,
                  int trace_cap, int* n_trace) {
  Model model;
  const long fits = estimate(FKernel(corr, n, wI, hI, wJ, hJ), state, nullptr, max_iter, precision, model, valid, n_inliers, inliers,
                             error_max, min_nfa, trace, trace_nfa, trace_cap, n_trace);
  std::memcpy(F, model.F, sizeof model.F);
  return fits;
}

}  // extern "C"

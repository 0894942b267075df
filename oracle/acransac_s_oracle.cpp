// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product; nothing under alicevision_b200/ may include, link or call this file.
//
// A-contrario RANSAC fundamental-matrix estimation of one pair of equidistant cameras, as
// GeometricFilterMatrix_F_AC::geometricEstimation_Spherical_Mat runs it (matchingImageCollection/GeometricFilterMatrix_F_AC.hpp:186-253):
// ACRANSAC over RelativePoseSphericalKernel<Fundamental7PSphericalSolver, EpipolarSphericalDistanceError, Mat3Model> on the lifted
// unit vectors, the std::mt19937 passed by reference.  Built twice by oracle/Makefile (`all`, `ref`) around the loop, sampling and
// estimate driver of oracle/acransac_loop.h; the "ref" build also compiles SolveCubicPolynomial (numeric/polynomial.hpp) verbatim,
// and the port takes the sampling and the kernel from the engine's alicevision_b200/csrc/acransac_math.h.
// The kernel (the spherical 7-point rows with the Householder null space, the error; no normalisation, logalpha0 = pi,
// errorVectorDimension = 2, thresholdNormalizer = 1, unormalizeError = sqrt) is restated in both builds.  Everything else in "ref" is
// compiled reference code, so "ref" == "port" bit for bit pins the control flow, the sampling, the NFA, the cubic solver and the
// generator's end state.
#ifdef ACR_USE_REFERENCE
#include <aliceVision/numeric/polynomial.hpp>
#define ACR_REFERENCE_CUBIC aliceVision::SolveCubicPolynomial<double>
#endif
#include "acransac_loop.h"

namespace {

struct Model : TracedModel {
  double F[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
};

// RelativePoseSphericalKernel<Fundamental7PSphericalSolver, EpipolarSphericalDistanceError, Mat3Model>, restated
struct SKernel {
  using ModelT = Model;
  std::vector<double> x1, x2;   // 3 per correspondence, as given

  SKernel(const double* b, int n) {
    for (int i = 0; i < n; ++i)
      for (int t = 0; t < 3; ++t) { x1.push_back(b[6 * i + t]); x2.push_back(b[6 * i + 3 + t]); }
  }
  static constexpr int kSampleSize = acr::kSample;
  std::size_t getMinimumNbRequiredSamples() const { return kSampleSize; }
  std::size_t getMaximumNbModels() const { return acr::kMaxModels; }
  std::size_t nbSamples() const { return x1.size() / 3; }
  double logalpha0() const { return M_PI; }
  double errorVectorDimension() const { return 2.0; }
  double thresholdNormalizer() const { return 1; }
  double unormalizeError(double v) const { return sqrt(v); }
  void unnormalize(Model&) const {}
  void fit(const std::vector<std::size_t>& s, std::vector<Model>& models) const {
    trace_fit();
    double a[21], b[21], F[27];
    for (int i = 0; i < 7; ++i)
      for (int t = 0; t < 3; ++t) { a[3 * i + t] = x1[3 * s[i] + t]; b[3 * i + t] = x2[3 * s[i] + t]; }
    const int nb = acr::fit7s(a, b, F);
    for (int m = 0; m < nb; ++m) {
      Model M;
      std::memcpy(M.F, F + 9 * m, sizeof M.F);
      models.push_back(M);
    }
  }
  void errors(const Model& m, std::vector<double>& e) const {
    for (std::size_t i = 0; i < nbSamples(); ++i) e[i] = acr::spherical_error(m.F, &x1[3 * i], &x2[3 * i]);
  }
};

}  // namespace

extern "C" {

// 1 = "ref" (compiled reference loop, sampling, NFA and cubic), 0 = "port"
int acrs_is_reference(void) { return is_reference(); }

// std::mt19937(seed) as 624 words + position (the library's operator<< order)
void acrs_mt_seed(uint32_t seed, uint32_t* state) { mt_seed(seed, state); }

// The spherical kernel's primitives, for the tests that check them against an independent high-precision reference.
// the 7-point solver on 7 bearing pairs (7 x (xI, yI, zI, xJ, yJ, zJ)): models row-major in F[27]; returns their number
int acrs_fit7s(const double* b, double* F) {
  double x1[21], x2[21];
  for (int i = 0; i < 7; ++i)
    for (int t = 0; t < 3; ++t) { x1[3 * i + t] = b[6 * i + t]; x2[3 * i + t] = b[6 * i + 3 + t]; }
  return acr::fit7s(x1, x2, F);
}

// EpipolarSphericalDistanceError of F on n bearing pairs: e[i] = (F x_I . x_J)^2
void acrs_spherical_error(const double* F, int n, const double* b, double* e) {
  for (int i = 0; i < n; ++i) e[i] = acr::spherical_error(F, b + 6 * i, b + 6 * i + 3);
}

// geometricEstimation_Spherical_Mat's ACRANSAC of one pair.  bearings: n x (xI, yI, zI, xJ, yJ, zJ).  inliers: capacity n.
// state: the generator on entry; state_out: the generator after the estimation (the reference's std::mt19937& afterwards).
// trace: the iterations at which a better model was found (first trace_cap of *n_trace); trace_nfa: the new minNFA of each (NaN in
// the "ref" build).  Returns the iterations executed.
long acrs_estimate(int n, const double* bearings, const uint32_t* state, long max_iter, double precision, int* valid, int* n_inliers,
                   uint32_t* inliers, double* F, double* error_max, double* min_nfa, int* trace, double* trace_nfa, int trace_cap,
                   int* n_trace, uint32_t* state_out) {
  Model model;
  const long fits = estimate(SKernel(bearings, n), state, state_out, max_iter, precision, model, valid, n_inliers, inliers, error_max,
                             min_nfa, trace, trace_nfa, trace_cap, n_trace);
  std::memcpy(F, model.F, sizeof model.F);
  return fits;
}

}  // extern "C"

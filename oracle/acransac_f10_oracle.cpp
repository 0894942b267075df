// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product; nothing under alicevision_b200/ may include, link or call this file.
//
// A-contrario RANSAC fundamental-matrix estimation with radial distortion of one planar pair, as
// GeometricFilterMatrix_F_AC::geometricEstimation_Mat_ACRANSAC<Fundamental10PSolver, Fundamental10PModel> runs it (the
// `fundamental_with_distortion` filter): ACRANSAC over RelativePoseKernel<Fundamental10PSolver, FundamentalEpipolarDistanceError,
// UnnormalizerT, Fundamental10PModel>, the std::mt19937 taken by value.  Built twice by oracle/Makefile (`all`, `ref`) around the
// loop, sampling and estimate driver of oracle/acransac_loop.h; the port takes the sampling and the kernel from the engine's
// alicevision_b200/csrc/acransac_math.h.
// The kernel (image-size preconditioning, the 10-point solver acr::fit10, the point-to-line error of model.getMatrix() on the
// preconditioned points, thresholdNormalizer = s_J, unormalizeError = sqrt(e) / s_J, errorVectorDimension = 1, logalpha0 of F,
// N2^T F N1 on the matrix only) is restated in both builds: the reference's Fundamental10PSolver needs Eigen.  "ref" == "port"
// bit for bit pins the control flow, the 10-sample draws (std::shuffle for ranges 11..14, Floyd from 15 on), the NFA with 10 models
// and the generator's end state.
#include "acransac_loop.h"

namespace {

struct Model : TracedModel {   // Fundamental10PModel: getMatrix() and getRadialDistortion()
  double F[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  double L[2] = {0, 0};
};

// RelativePoseKernel<Fundamental10PSolver, FundamentalEpipolarDistanceError, UnnormalizerT, Fundamental10PModel>, restated
struct F10Kernel {
  using ModelT = Model;
  std::vector<double> x1, y1, x2, y2;   // preconditioned
  acr::Norm n1, n2;
  double la0;

  F10Kernel(const double* corr, int n, int w1, int h1, int w2, int h2) {
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
  static constexpr int kSampleSize = acr::kSampleF10;
  std::size_t getMinimumNbRequiredSamples() const { return kSampleSize; }
  std::size_t getMaximumNbModels() const { return acr::kMaxModelsF10; }
  std::size_t nbSamples() const { return x1.size(); }
  double logalpha0() const { return la0; }
  double errorVectorDimension() const { return 1.0; }
  double thresholdNormalizer() const { return n2.s; }
  double unormalizeError(double v) const { return sqrt(v) / n2.s; }
  void unnormalize(Model& m) const { acr::unnormalize(n1, n2, m.F); }
  void fit(const std::vector<std::size_t>& s, std::vector<Model>& models) const {
    trace_fit();
    double a[10], b[10], c[10], d[10], F[90], L[20];
    for (int i = 0; i < 10; ++i) { a[i] = x1[s[i]]; b[i] = y1[s[i]]; c[i] = x2[s[i]]; d[i] = y2[s[i]]; }
    acr::F10Work w;
    const int nb = acr::fit10(a, b, c, d, F, L, w);
    for (int m = 0; m < nb; ++m) {
      Model M;
      std::memcpy(M.F, F + 9 * m, sizeof M.F);
      std::memcpy(M.L, L + 2 * m, sizeof M.L);
      models.push_back(M);
    }
  }
  void errors(const Model& m, std::vector<double>& e) const {
    for (std::size_t i = 0; i < x1.size(); ++i) e[i] = acr::epipolar_error(m.F, x1[i], y1[i], x2[i], y2[i]);
  }
};

}  // namespace

extern "C" {

// 1 = "ref" (compiled reference loop, sampling and NFA), 0 = "port"
int acrf10_is_reference(void) { return is_reference(); }

// std::mt19937(seed) as 624 words + position (the library's operator<< order)
void acrf10_mt_seed(uint32_t seed, uint32_t* state) { mt_seed(seed, state); }

// The F10 kernel's primitives, for the tests that check them against an independent high-precision reference.
// the 10-point solver on 10 correspondences (10 x (xI, yI, xJ, yJ)): models row-major in F[90], (l1, l2) in L[20]; the action
// matrix it built, row-major, in At[100] (At may be NULL); returns the number of models
int acrf10_fit10(const double* c, double* F, double* L, double* At) {
  double a[10], b[10], cc[10], d[10];
  for (int i = 0; i < 10; ++i) { a[i] = c[4 * i]; b[i] = c[4 * i + 1]; cc[i] = c[4 * i + 2]; d[i] = c[4 * i + 3]; }
  acr::F10Work w;
  const int nb = acr::fit10(a, b, cc, d, F, L, w);
  if (At)
    for (int r = 0; r < 10; ++r)
      for (int q = 0; q < 10; ++q) At[10 * r + q] = w.At[r][q];
  return nb;
}

// geometricEstimation_Mat_ACRANSAC<Fundamental10PSolver> of one pair.  corr: n x (xI, yI, xJ, yJ) pixels; wh: (wI, hI, wJ, hJ).
// precision: ACRANSAC's argument.  inliers: capacity n.  F, L: the model (F unnormalised, L in preconditioned units).
// state: the generator on entry; state_out: the generator after the estimation (the filter itself takes it by value).
// trace: the iterations at which a better model was found (first trace_cap of *n_trace); trace_nfa: the new minNFA of each (NaN in
// the "ref" build).  Returns the iterations executed.
long acrf10_estimate(int n, const double* corr, const int* wh, const uint32_t* state, long max_iter, double precision, int* valid,
                     int* n_inliers, uint32_t* inliers, double* F, double* L, double* error_max, double* min_nfa, int* trace,
                     double* trace_nfa, int trace_cap, int* n_trace, uint32_t* state_out) {
  Model model;
  const long fits = estimate(F10Kernel(corr, n, wh[0], wh[1], wh[2], wh[3]), state, state_out, max_iter, precision, model, valid,
                             n_inliers, inliers, error_max, min_nfa, trace, trace_nfa, trace_cap, n_trace);
  std::memcpy(F, model.F, sizeof model.F);
  std::memcpy(L, model.L, sizeof model.L);
  return fits;
}

}  // extern "C"

// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product; nothing under alicevision_b200/ may include, link or call this file.
//
// A-contrario RANSAC homography estimation of one pair, as GeometricFilterMatrix_H_AC::geometricEstimation runs it
// (matchingImageCollection/GeometricFilterMatrix_H_AC.hpp:40-100): ACRANSAC over RelativePoseKernel<Homography4PSolver,
// HomographyAsymmetricError, UnnormalizerI, Mat3Model> with the point-to-point error, the std::mt19937 passed by reference.
// Built twice by oracle/Makefile (`all`, `ref`) around the loop, sampling and estimate driver of oracle/acransac_loop.h; the port
// takes the sampling and the H kernel from the engine's alicevision_b200/csrc/acransac_math.h.
// The H kernel (normalisation, 4-point DLT with its Householder null space, error, unnormalisation with a restated 3 x 3 inverse)
// is restated in both builds: the reference takes its null space from Eigen's JacobiSVD and its inverse from Eigen, neither of
// which is available here.  Everything else in "ref" is compiled reference code, so "ref" == "port" bit for bit pins the control
// flow, the sampling, the NFA and the generator's end state.
#include "acransac_loop.h"

namespace {

struct Model : TracedModel {
  double M[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
};

// RelativePoseKernel<Homography4PSolver, HomographyAsymmetricError, UnnormalizerI, Mat3Model> with pointToLine = false, restated
struct HKernel {
  using ModelT = Model;
  std::vector<double> x1, y1, x2, y2;   // normalised
  acr::Norm n1, n2;
  double la0;

  HKernel(const double* corr, int n, int w1, int h1, int w2, int h2) {
    n1 = acr::precondition(w1, h1);
    n2 = acr::precondition(w2, h2);
    for (int i = 0; i < n; ++i) {
      x1.push_back(acr::norm_x(n1, corr[4 * i])); y1.push_back(acr::norm_y(n1, corr[4 * i + 1]));
      x2.push_back(acr::norm_x(n2, corr[4 * i + 2])); y2.push_back(acr::norm_y(n2, corr[4 * i + 3]));
    }
    la0 = acr::logalpha0_h(w2, h2, n2);
  }
  static constexpr int kSampleSize = acr::kSampleH;
  std::size_t getMinimumNbRequiredSamples() const { return kSampleSize; }
  std::size_t getMaximumNbModels() const { return acr::kMaxModelsH; }
  std::size_t nbSamples() const { return x1.size(); }
  double logalpha0() const { return la0; }
  double errorVectorDimension() const { return 2.0; }
  double thresholdNormalizer() const { return n2.s; }
  double unormalizeError(double v) const { return sqrt(v) / n2.s; }
  void unnormalize(Model& m) const { acr::unnormalize_h(n1, n2, m.M); }
  void fit(const std::vector<std::size_t>& s, std::vector<Model>& models) const {
    trace_fit();
    double a[4], b[4], c[4], d[4];
    for (int i = 0; i < 4; ++i) { a[i] = x1[s[i]]; b[i] = y1[s[i]]; c[i] = x2[s[i]]; d[i] = y2[s[i]]; }
    Model M;
    acr::fit4(a, b, c, d, M.M);
    models.push_back(M);
  }
  void errors(const Model& m, std::vector<double>& e) const {
    for (std::size_t i = 0; i < x1.size(); ++i) e[i] = acr::homography_error(m.M, x1[i], y1[i], x2[i], y2[i]);
  }
};

}  // namespace

extern "C" {

// 1 = "ref" (compiled reference loop, sampling and NFA), 0 = "port"
int acrh_is_reference(void) { return is_reference(); }

// std::mt19937(seed) as 624 words + position (the library's operator<< order)
void acrh_mt_seed(uint32_t seed, uint32_t* state) { mt_seed(seed, state); }

// `draws` consecutive randSample(g, 0, range, k) from `state`, k = 4 or 7: the samples in their order (draws x k), and the
// generator state after each draw (draws x 625) when states != nullptr
void acr_rand_sample_k(const uint32_t* state, int k, int range, int draws, uint32_t* out, uint32_t* states) {
  rand_sample_draws(state, k, range, draws, out, states);
}

// the float tables logc_n[0..n], logc_k[0..n] of ACRANSAC for sizeSample k
void acr_logc_k(int k, int n, float* logc_n, float* logc_k) { logc(k, n, logc_n, logc_k); }

// the 4-point solver alone on 4 raw correspondences (no normalisation): H row-major (x2 ~ H x1); returns the number of models (1)
int acr_fit4(const double* corr, double* H) {
  double a[4], b[4], c[4], d[4];
  for (int i = 0; i < 4; ++i) { a[i] = corr[4 * i]; b[i] = corr[4 * i + 1]; c[i] = corr[4 * i + 2]; d[i] = corr[4 * i + 3]; }
  return acr::fit4(a, b, c, d, H);
}

// HomographyAsymmetricError of H on raw correspondences: e[i] = |x2 - H(x1)|^2
void acr_homography_error(const double* H, int n, const double* corr, double* e) {
  for (int i = 0; i < n; ++i) e[i] = acr::homography_error(H, corr[4 * i], corr[4 * i + 1], corr[4 * i + 2], corr[4 * i + 3]);
}

// The H kernel's primitives one by one, for the tests that check them against an independent high-precision reference.
// the null space of an 8 x 9 row-major system: N[9] = Q e8
void acr_nullspace8(const double* A, double* N) {
  double a[8][9], n[1][9];
  std::memcpy(a, A, sizeof a);
  acr::nullspace<8>(a, n);
  std::memcpy(N, n, sizeof n);
}

// the restated 3 x 3 inverse (cofactors over the first-column determinant), row-major
void acr_inverse3(const double* M, double* R) { acr::inverse3(M, R); }

// UnnormalizerI in place (H <- N2^-1 H N1), with the kernel's preconditioners of (w1, h1) and (w2, h2)
void acr_unnormalize_h(int w1, int h1, int w2, int h2, double* H) {
  const HKernel k(nullptr, 0, w1, h1, w2, h2);
  Model m;
  std::memcpy(m.M, H, sizeof m.M);
  k.unnormalize(m);
  std::memcpy(H, m.M, sizeof m.M);
}

// the kernel's logalpha0() and unormalizeError(v) for image J = (w2, h2)
double acr_logalpha0_h(int w1, int h1, int w2, int h2) { return HKernel(nullptr, 0, w1, h1, w2, h2).logalpha0(); }
double acr_unnormalize_error_h(int w1, int h1, int w2, int h2, double v) { return HKernel(nullptr, 0, w1, h1, w2, h2).unormalizeError(v); }

// GeometricFilterMatrix_H_AC::geometricEstimation's ACRANSAC of one pair.  corr: n x (xI, yI, xJ, yJ).  inliers: capacity n.
// state: the generator on entry; state_out: the generator after the estimation (the reference's std::mt19937& afterwards).
// trace: the iterations at which a better model was found (first trace_cap of *n_trace); trace_nfa: the new minNFA of each (NaN in
// the "ref" build).  Returns the iterations executed.
long acr_estimate_h(int n, const double* corr, int wI, int hI, int wJ, int hJ, const uint32_t* state, long max_iter, double precision,
                    int* valid, int* n_inliers, uint32_t* inliers, double* H, double* error_max, double* min_nfa, int* trace,
                    double* trace_nfa, int trace_cap, int* n_trace, uint32_t* state_out) {
  Model model;
  const long fits = estimate(HKernel(corr, n, wI, hI, wJ, hJ), state, state_out, max_iter, precision, model, valid, n_inliers,
                             inliers, error_max, min_nfa, trace, trace_nfa, trace_cap, n_trace);
  std::memcpy(H, model.M, sizeof model.M);
  return fits;
}

}  // extern "C"

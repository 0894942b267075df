// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product; nothing under alicevision_b200/ may include, link or call this file.
//
// A-contrario RANSAC homography estimation of one pair, as GeometricFilterMatrix_H_AC::geometricEstimation runs it
// (matchingImageCollection/GeometricFilterMatrix_H_AC.hpp:40-100): ACRANSAC over RelativePoseKernel<Homography4PSolver,
// HomographyAsymmetricError, UnnormalizerI, Mat3Model> with the point-to-point error, the std::mt19937 passed by reference.
// Built twice by oracle/Makefile (`all`, `ref`), like oracle/acransac_oracle.cpp (the fundamental-matrix oracle, a separate library):
//   -DACR_USE_REFERENCE -> _ref/libref_acransac_h.so: robustEstimation::ACRANSAC, makelogcombi (robustEstimation/ACRansac.hpp) and
//                          randSample (robustEstimation/randSampling.hpp) compiled verbatim from an AliceVision source tree through
//                          oracle/shim, around the restated H kernel below; the generator is the library's own std::mt19937.
//   (none)              -> libport_acransac_h.so: the loop, the NFA tables and the sampling restated (the sampling and the H kernel
//                          are the engine's alicevision_b200/csrc/acransac_math.h, so the port pins the engine's sampler).
// The H kernel (normalisation, 4-point DLT with its Householder null space, error, unnormalisation with a restated 3 x 3 inverse)
// is restated in both builds: the reference takes its null space from Eigen's JacobiSVD and its inverse from Eigen, neither of
// which is available here.  Everything else in "ref" is compiled reference code, so "ref" == "port" bit for bit pins the control
// flow, the sampling, the NFA and the generator's end state.
#ifdef ACR_USE_REFERENCE
#include <aliceVision/robustEstimation/ACRansac.hpp>
#endif
#include "../alicevision_b200/csrc/acransac_math.h"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <numeric>
#include <random>
#include <sstream>
#include <unordered_set>
#include <utility>
#include <vector>

namespace {

struct Trace {
  std::vector<int> better;
  std::vector<double> nfa;   // the new minNFA of each `better` event (the restated loop only; the verbatim loop does not expose it)
  long fits = 0;
};
Trace* g_trace = nullptr;

struct Model {
  double M[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  Model() = default;
  Model(const Model& o) { std::memcpy(M, o.M, sizeof M); }
  Model& operator=(const Model& o) {   // ACRANSAC: `*model = vec_models[k]` when a better model is found
    std::memcpy(M, o.M, sizeof M);
    if (g_trace) g_trace->better.push_back((int)(g_trace->fits - 1));
    return *this;
  }
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
  std::size_t getMinimumNbRequiredSamples() const { return acr::kSampleH; }
  std::size_t getMaximumNbModels() const { return acr::kMaxModelsH; }
  std::size_t nbSamples() const { return x1.size(); }
  double logalpha0() const { return la0; }
  double errorVectorDimension() const { return 2.0; }
  double thresholdNormalizer() const { return n2.s; }
  double unormalizeError(double v) const { return sqrt(v) / n2.s; }
  void unnormalize(Model& m) const { acr::unnormalize_h(n1, n2, m.M); }
  void fit(const std::vector<std::size_t>& s, std::vector<Model>& models) const {
    if (g_trace) ++g_trace->fits;
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

#ifndef ACR_USE_REFERENCE
// ---- the restated loop (robustEstimation/ACRansac.hpp:145-285) and tables, for any sample size
void logc_tables(std::size_t k_sample, std::size_t n, std::vector<float>& logc_n, std::vector<float>& logc_k) {
  std::vector<float> l10(n + 1);
  for (std::size_t k = 0; k <= n; ++k) l10[k] = (float)log10((double)k);
  auto logcombi = [&](std::size_t k, std::size_t nn) {
    if (k >= nn || k <= 0) return 0.0f;
    if (nn - k < k) k = nn - k;
    float r = 0.0f;
    for (std::size_t i = 1; i <= k; ++i) r += l10[nn - i + 1] - l10[i];
    return r;
  };
  logc_n.resize(n + 1); logc_k.resize(n + 1);
  for (std::size_t k = 0; k <= n; ++k) logc_n[k] = logcombi(k, n);
  for (std::size_t m = 0; m <= n; ++m) logc_k[m] = logcombi(k_sample, m);
}

void sample(acr::Mt19937& g, const std::vector<std::size_t>& elements, std::vector<std::size_t>& out) {
  uint32_t s[acr::kSampleH];
  acr::rand_sample<acr::kSampleH>(g, (uint32_t)elements.size(), s);
  out.resize(acr::kSampleH);
  for (int i = 0; i < acr::kSampleH; ++i) out[i] = elements[s[i]];
}

template <class Kernel>
std::pair<double, double> acransac_port(const Kernel& kernel, acr::Mt19937& g, std::vector<std::size_t>& vec_inliers, std::size_t nIter,
                                        Model* model, double precision) {
  const double inf = std::numeric_limits<double>::infinity();
  vec_inliers.clear();
  const std::size_t sizeSample = kernel.getMinimumNbRequiredSamples(), nData = kernel.nbSamples();
  if (nData <= sizeSample) return {0.0, 0.0};
  const double maxThreshold = precision == inf ? inf : precision * precision * kernel.thresholdNormalizer() * kernel.thresholdNormalizer();
  std::vector<std::pair<double, std::size_t>> res(nData);
  std::vector<double> res_(nData);
  std::vector<std::size_t> vec_index(nData), all(nData);
  std::iota(vec_index.begin(), vec_index.end(), 0);
  std::iota(all.begin(), all.end(), 0);
  const double loge0 = log10((double)kernel.getMaximumNbModels() * (nData - sizeSample));
  std::vector<float> logc_n, logc_k;
  logc_tables(sizeSample, nData, logc_n, logc_k);
  double minNFA = inf, errorMax = inf;
  std::size_t nIterReserve = nIter / 10;
  nIter -= nIterReserve;
  bool mode = precision == inf;
  for (std::size_t iter = 0; iter < nIter; ++iter) {
    std::vector<std::size_t> s;
    sample(g, mode ? vec_index : all, s);
    std::vector<Model> models;
    kernel.fit(s, models);
    bool better = false;
    for (std::size_t k = 0; k < models.size(); ++k) {
      kernel.errors(models[k], res_);
      if (!mode) {
        unsigned nin = 0;
        for (std::size_t i = 0; i < nData; ++i) nin += res_[i] <= maxThreshold;
        if (nin > 2.5 * sizeSample) mode = true;
      }
      if (!mode) continue;
      for (std::size_t i = 0; i < nData; ++i) res[i] = {res_[i], i};
      std::sort(res.begin(), res.end());
      std::pair<double, std::size_t> best(inf, sizeSample);
      for (std::size_t kk = sizeSample + 1; kk <= nData && res[kk - 1].first <= maxThreshold; ++kk) {
        const double r = sqrt(res[kk - 1].first) + std::numeric_limits<float>::epsilon();
        const double la = kernel.logalpha0() + kernel.errorVectorDimension() * log10(r);
        const double nfa = loge0 + la * (double)(kk - sizeSample) + logc_n[kk] + logc_k[kk];
        if (nfa < best.first) best = {nfa, kk};
      }
      if (best.first < minNFA) {
        better = true;
        minNFA = best.first;
        vec_inliers.resize(best.second);
        for (std::size_t i = 0; i < best.second; ++i) vec_inliers[i] = res[i].second;
        errorMax = res[best.second - 1].first;
        *model = models[k];
        if (g_trace) g_trace->nfa.push_back(minNFA);
      }
    }
    if (!mode && iter > nIterReserve * 2) break;
    if (mode && ((better && minNFA < 0) || (iter + 1 == nIter && nIterReserve))) {
      if (vec_inliers.empty()) {
        ++nIter;
        --nIterReserve;
      } else {
        vec_index = vec_inliers;
        if (nIterReserve) {
          nIter = iter + 1 + nIterReserve;
          nIterReserve = 0;
        }
      }
    }
  }
  if (minNFA >= 0) vec_inliers.clear();
  if (!vec_inliers.empty()) {
    kernel.unnormalize(*model);
    errorMax = kernel.unormalizeError(errorMax);
  }
  return {errorMax, minNFA};
}

void load(acr::Mt19937& g, const uint32_t* st) {
  std::memcpy(g.x, st, sizeof g.x);
  g.p = (int)st[624];
}
void store(const acr::Mt19937& g, uint32_t* st) {
  std::memcpy(st, g.x, sizeof g.x);
  st[624] = (uint32_t)g.p;
}
#else
std::mt19937 to_std(const uint32_t* st) {
  std::stringstream ss;
  for (int i = 0; i < 625; ++i) ss << st[i] << ' ';
  std::mt19937 g;
  ss >> g;
  return g;
}
void from_std(const std::mt19937& g, uint32_t* st) {
  std::stringstream ss;
  ss << g;
  for (int i = 0; i < 625; ++i) ss >> st[i];
}
#endif

}  // namespace

extern "C" {

// 1 = "ref" (compiled reference loop, sampling and NFA), 0 = "port"
int acrh_is_reference(void) {
#ifdef ACR_USE_REFERENCE
  return 1;
#else
  return 0;
#endif
}

// std::mt19937(seed) as 624 words + position (the library's operator<< order)
void acrh_mt_seed(uint32_t seed, uint32_t* state) {
#ifdef ACR_USE_REFERENCE
  from_std(std::mt19937(seed), state);
#else
  acr::Mt19937 g;
  acr::mt_seed(g, seed);
  store(g, state);
#endif
}

// `draws` consecutive randSample(g, 0, range, k) from `state`, k = 4 or 7: the samples in their order (draws x k), and the
// generator state after each draw (draws x 625) when states != nullptr
void acr_rand_sample_k(const uint32_t* state, int k, int range, int draws, uint32_t* out, uint32_t* states) {
#ifdef ACR_USE_REFERENCE
  std::mt19937 g = to_std(state);
  for (int d = 0; d < draws; ++d) {
    const auto s = aliceVision::robustEstimation::randSample<std::size_t>(g, 0, (std::size_t)range, (std::size_t)k);
    for (int i = 0; i < k; ++i) out[(size_t)k * d + i] = (uint32_t)s[i];
    if (states) from_std(g, states + 625 * (size_t)d);
  }
#else
  acr::Mt19937 g;
  load(g, state);
  for (int d = 0; d < draws; ++d) {
    if (k == 4) acr::rand_sample<4>(g, (uint32_t)range, out + 4 * (size_t)d);
    else acr::rand_sample<7>(g, (uint32_t)range, out + 7 * (size_t)d);
    if (states) store(g, states + 625 * (size_t)d);
  }
#endif
}

// the float tables logc_n[0..n], logc_k[0..n] of ACRANSAC for sizeSample k
void acr_logc_k(int k, int n, float* logc_n, float* logc_k) {
  std::vector<float> a, b;
#ifdef ACR_USE_REFERENCE
  aliceVision::robustEstimation::makelogcombi<float>((std::size_t)k, (std::size_t)n, b, a);
#else
  logc_tables((std::size_t)k, (std::size_t)n, a, b);
#endif
  std::memcpy(logc_n, a.data(), (n + 1) * sizeof(float));
  std::memcpy(logc_k, b.data(), (n + 1) * sizeof(float));
}

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
  HKernel kernel(corr, n, wI, hI, wJ, hJ);
  Trace tr;
  g_trace = &tr;
  std::vector<std::size_t> inl;
  Model model;
  std::pair<double, double> out;
#ifdef ACR_USE_REFERENCE
  std::mt19937 g = to_std(state);
  out = aliceVision::robustEstimation::ACRANSAC(kernel, g, inl, (std::size_t)max_iter, &model, precision);
  from_std(g, state_out);
#else
  acr::Mt19937 g;
  load(g, state);
  out = acransac_port(kernel, g, inl, (std::size_t)max_iter, &model, precision);
  store(g, state_out);
#endif
  g_trace = nullptr;
  *valid = !inl.empty();
  *n_inliers = (int)inl.size();
  for (std::size_t i = 0; i < inl.size(); ++i) inliers[i] = (uint32_t)inl[i];
  std::memcpy(H, model.M, sizeof model.M);
  *error_max = out.first;
  *min_nfa = out.second;
  *n_trace = (int)tr.better.size();
  for (int i = 0; i < std::min(trace_cap, (int)tr.better.size()); ++i) {
    trace[i] = tr.better[i];
    trace_nfa[i] = i < (int)tr.nfa.size() ? tr.nfa[i] : std::numeric_limits<double>::quiet_NaN();
  }
  return tr.fits;
}

}  // extern "C"

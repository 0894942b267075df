// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product; nothing under alicevision_b200/ may include, link or call this file.
//
// A-contrario RANSAC fundamental-matrix estimation of one pair of equidistant cameras, as
// GeometricFilterMatrix_F_AC::geometricEstimation_Spherical_Mat runs it (matchingImageCollection/GeometricFilterMatrix_F_AC.hpp:186-253):
// ACRANSAC over RelativePoseSphericalKernel<Fundamental7PSphericalSolver, EpipolarSphericalDistanceError, Mat3Model> on the lifted
// unit vectors, the std::mt19937 passed by reference.  Built twice by oracle/acransac_s.mk, like oracle/acransac_oracle.cpp:
//   -DACR_USE_REFERENCE -> _ref/libref_acransac_s.so: robustEstimation::ACRANSAC, makelogcombi (robustEstimation/ACRansac.hpp),
//                          randSample (robustEstimation/randSampling.hpp) and SolveCubicPolynomial (numeric/polynomial.hpp) compiled
//                          verbatim from an AliceVision source tree through oracle/shim, around the restated spherical kernel below;
//                          the generator is the library's own std::mt19937.
//   (none)              -> libport_acransac_s.so: the loop, the NFA tables and the sampling restated (the sampling and the kernel are
//                          the engine's alicevision_b200/csrc/acransac_math.h, so the port pins the engine's sampler).
// The kernel (the spherical 7-point rows with the Householder null space, the error; no normalisation, logalpha0 = pi,
// errorVectorDimension = 2, thresholdNormalizer = 1, unormalizeError = sqrt) is restated in both builds.  Everything else in "ref" is
// compiled reference code, so "ref" == "port" bit for bit pins the control flow, the sampling, the NFA, the cubic solver and the
// generator's end state.
#ifdef ACR_USE_REFERENCE
#include <aliceVision/numeric/polynomial.hpp>
#include <aliceVision/robustEstimation/ACRansac.hpp>
#define ACR_REFERENCE_CUBIC aliceVision::SolveCubicPolynomial<double>
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
  double F[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  Model() = default;
  Model(const Model& o) { std::memcpy(F, o.F, sizeof F); }
  Model& operator=(const Model& o) {   // ACRANSAC: `*model = vec_models[k]` when a better model is found
    std::memcpy(F, o.F, sizeof F);
    if (g_trace) g_trace->better.push_back((int)(g_trace->fits - 1));
    return *this;
  }
};

// RelativePoseSphericalKernel<Fundamental7PSphericalSolver, EpipolarSphericalDistanceError, Mat3Model>, restated
struct SKernel {
  using ModelT = Model;
  std::vector<double> x1, x2;   // 3 per correspondence, as given

  SKernel(const double* b, int n) {
    for (int i = 0; i < n; ++i)
      for (int t = 0; t < 3; ++t) { x1.push_back(b[6 * i + t]); x2.push_back(b[6 * i + 3 + t]); }
  }
  std::size_t getMinimumNbRequiredSamples() const { return acr::kSample; }
  std::size_t getMaximumNbModels() const { return acr::kMaxModels; }
  std::size_t nbSamples() const { return x1.size() / 3; }
  double logalpha0() const { return M_PI; }
  double errorVectorDimension() const { return 2.0; }
  double thresholdNormalizer() const { return 1; }
  double unormalizeError(double v) const { return sqrt(v); }
  void unnormalize(Model&) const {}
  void fit(const std::vector<std::size_t>& s, std::vector<Model>& models) const {
    if (g_trace) ++g_trace->fits;
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

#ifndef ACR_USE_REFERENCE
// ---- the restated loop (robustEstimation/ACRansac.hpp:145-285) and tables
void logc_tables(std::size_t n, std::vector<float>& logc_n, std::vector<float>& logc_k) {
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
  for (std::size_t m = 0; m <= n; ++m) logc_k[m] = logcombi(acr::kSample, m);
}

void sample(acr::Mt19937& g, const std::vector<std::size_t>& elements, std::vector<std::size_t>& out) {
  uint32_t s[7];
  acr::rand_sample7(g, (uint32_t)elements.size(), s);
  out.resize(7);
  for (int i = 0; i < 7; ++i) out[i] = elements[s[i]];
}

std::pair<double, double> acransac_port(const SKernel& kernel, acr::Mt19937& g, std::vector<std::size_t>& vec_inliers, std::size_t nIter,
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
  logc_tables(nData, logc_n, logc_k);
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

// 1 = "ref" (compiled reference loop, sampling, NFA and cubic), 0 = "port"
int acrs_is_reference(void) {
#ifdef ACR_USE_REFERENCE
  return 1;
#else
  return 0;
#endif
}

// std::mt19937(seed) as 624 words + position (the library's operator<< order)
void acrs_mt_seed(uint32_t seed, uint32_t* state) {
#ifdef ACR_USE_REFERENCE
  from_std(std::mt19937(seed), state);
#else
  acr::Mt19937 g;
  acr::mt_seed(g, seed);
  store(g, state);
#endif
}

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
  SKernel kernel(bearings, n);
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
  std::memcpy(F, model.F, sizeof model.F);
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

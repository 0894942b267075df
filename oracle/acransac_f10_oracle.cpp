// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product; nothing under alicevision_b200/ may include, link or call this file.
//
// A-contrario RANSAC fundamental-matrix estimation with radial distortion of one planar pair, as
// GeometricFilterMatrix_F_AC::geometricEstimation_Mat_ACRANSAC<Fundamental10PSolver, Fundamental10PModel> runs it (the
// `fundamental_with_distortion` filter): ACRANSAC over RelativePoseKernel<Fundamental10PSolver, FundamentalEpipolarDistanceError,
// UnnormalizerT, Fundamental10PModel>, the std::mt19937 taken by value.  Built twice by oracle/Makefile (`all`, `ref`), like
// oracle/acransac_e_oracle.cpp:
//   -DACR_USE_REFERENCE -> _ref/libref_acransac_f10.so: robustEstimation::ACRANSAC, makelogcombi (robustEstimation/ACRansac.hpp)
//                          and randSample (robustEstimation/randSampling.hpp) compiled verbatim from an AliceVision source tree
//                          through oracle/shim, around the restated F10 kernel below; the generator is the library's std::mt19937.
//   (none)              -> libport_acransac_f10.so: the loop, the NFA tables and the sampling restated (the sampling and the kernel
//                          are the engine's alicevision_b200/csrc/acransac_math.h, so the port pins the engine's sampler).
// The kernel (image-size preconditioning, the 10-point solver acr::fit10, the point-to-line error of model.getMatrix() on the
// preconditioned points, thresholdNormalizer = s_J, unormalizeError = sqrt(e) / s_J, errorVectorDimension = 1, logalpha0 of F,
// N2^T F N1 on the matrix only) is restated in both builds: the reference's Fundamental10PSolver needs Eigen.  "ref" == "port"
// bit for bit pins the control flow, the 10-sample draws (std::shuffle for ranges 11..14, Floyd from 15 on), the NFA with 10 models
// and the generator's end state.
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

struct Model {   // Fundamental10PModel: getMatrix() and getRadialDistortion()
  double F[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  double L[2] = {0, 0};
  Model() = default;
  Model(const Model& o) { std::memcpy(F, o.F, sizeof F); std::memcpy(L, o.L, sizeof L); }
  Model& operator=(const Model& o) {   // ACRANSAC: `*model = vec_models[k]` when a better model is found
    std::memcpy(F, o.F, sizeof F);
    std::memcpy(L, o.L, sizeof L);
    if (g_trace) g_trace->better.push_back((int)(g_trace->fits - 1));
    return *this;
  }
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
  std::size_t getMinimumNbRequiredSamples() const { return acr::kSampleF10; }
  std::size_t getMaximumNbModels() const { return acr::kMaxModelsF10; }
  std::size_t nbSamples() const { return x1.size(); }
  double logalpha0() const { return la0; }
  double errorVectorDimension() const { return 1.0; }
  double thresholdNormalizer() const { return n2.s; }
  double unormalizeError(double v) const { return sqrt(v) / n2.s; }
  void unnormalize(Model& m) const { acr::unnormalize(n1, n2, m.F); }
  void fit(const std::vector<std::size_t>& s, std::vector<Model>& models) const {
    if (g_trace) ++g_trace->fits;
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
  for (std::size_t m = 0; m <= n; ++m) logc_k[m] = logcombi(acr::kSampleF10, m);
}

void sample(acr::Mt19937& g, const std::vector<std::size_t>& elements, std::vector<std::size_t>& out) {
  uint32_t s[acr::kSampleF10];
  acr::rand_sample<acr::kSampleF10>(g, (uint32_t)elements.size(), s);
  out.resize(acr::kSampleF10);
  for (int i = 0; i < acr::kSampleF10; ++i) out[i] = elements[s[i]];
}

std::pair<double, double> acransac_port(const F10Kernel& kernel, acr::Mt19937& g, std::vector<std::size_t>& vec_inliers, std::size_t nIter,
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

// 1 = "ref" (compiled reference loop, sampling and NFA), 0 = "port"
int acrf10_is_reference(void) {
#ifdef ACR_USE_REFERENCE
  return 1;
#else
  return 0;
#endif
}

// std::mt19937(seed) as 624 words + position (the library's operator<< order)
void acrf10_mt_seed(uint32_t seed, uint32_t* state) {
#ifdef ACR_USE_REFERENCE
  from_std(std::mt19937(seed), state);
#else
  acr::Mt19937 g;
  acr::mt_seed(g, seed);
  store(g, state);
#endif
}

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
  F10Kernel kernel(corr, n, wh[0], wh[1], wh[2], wh[3]);
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
  std::memcpy(L, model.L, sizeof model.L);
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

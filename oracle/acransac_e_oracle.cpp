// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product; nothing under alicevision_b200/ may include, link or call this file.
//
// A-contrario RANSAC essential-matrix estimation of one pair of pinhole cameras, as GeometricFilterMatrix_E_AC::geometricEstimation
// runs it (matchingImageCollection/GeometricFilterMatrix_E_AC.hpp): ACRANSAC over RelativePoseKernel_K<Essential5PSolver,
// FundamentalEpipolarDistanceError, Mat3Model>, the std::mt19937 passed by reference.  Built twice by oracle/Makefile (`all`, `ref`), like
// oracle/acransac_s_oracle.cpp:
//   -DACR_USE_REFERENCE -> _ref/libref_acransac_e.so: robustEstimation::ACRANSAC, makelogcombi (robustEstimation/ACRansac.hpp) and
//                          randSample (robustEstimation/randSampling.hpp) compiled verbatim from an AliceVision source tree through
//                          oracle/shim, around the restated E kernel below; the generator is the library's own std::mt19937.
//   (none)              -> libport_acransac_e.so: the loop, the NFA tables and the sampling restated (the sampling and the kernel are
//                          the engine's alicevision_b200/csrc/acransac_math.h, so the port pins the engine's sampler).
// The kernel (K^-1 applied once to the pixels, the 5-point solver on them, F = K_J^-T E K_I^-1 and the point-to-line error on the
// pixels; thresholdNormalizer = 1, unormalizeError = sqrt, errorVectorDimension = 0.5, logalpha0 = log10(2 D / A * .5)) is restated
// in both builds: the reference's Essential5PSolver needs Eigen.  Everything else in "ref" is compiled reference code, so "ref" ==
// "port" bit for bit pins the control flow, the 5-sample draws, the NFA with d = 0.5 and the generator's end state.
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
  double F[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  Model() = default;
  Model(const Model& o) { std::memcpy(F, o.F, sizeof F); }
  Model& operator=(const Model& o) {   // ACRANSAC: `*model = vec_models[k]` when a better model is found
    std::memcpy(F, o.F, sizeof F);
    if (g_trace) g_trace->better.push_back((int)(g_trace->fits - 1));
    return *this;
  }
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
  std::size_t getMinimumNbRequiredSamples() const { return acr::kSampleE; }
  std::size_t getMaximumNbModels() const { return acr::kMaxModelsE; }
  std::size_t nbSamples() const { return px.size() / 4; }
  double logalpha0() const { return acr::logalpha0_e(w2, h2); }
  double errorVectorDimension() const { return 0.5; }
  double thresholdNormalizer() const { return 1; }
  double unormalizeError(double v) const { return sqrt(v); }
  void unnormalize(Model&) const {}
  void fit(const std::vector<std::size_t>& s, std::vector<Model>& models) const {
    if (g_trace) ++g_trace->fits;
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
  for (std::size_t m = 0; m <= n; ++m) logc_k[m] = logcombi(acr::kSampleE, m);
}

void sample(acr::Mt19937& g, const std::vector<std::size_t>& elements, std::vector<std::size_t>& out) {
  uint32_t s[acr::kSampleE];
  acr::rand_sample<acr::kSampleE>(g, (uint32_t)elements.size(), s);
  out.resize(acr::kSampleE);
  for (int i = 0; i < acr::kSampleE; ++i) out[i] = elements[s[i]];
}

std::pair<double, double> acransac_port(const EKernel& kernel, acr::Mt19937& g, std::vector<std::size_t>& vec_inliers, std::size_t nIter,
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
int acre_is_reference(void) {
#ifdef ACR_USE_REFERENCE
  return 1;
#else
  return 0;
#endif
}

// std::mt19937(seed) as 624 words + position (the library's operator<< order)
void acre_mt_seed(uint32_t seed, uint32_t* state) {
#ifdef ACR_USE_REFERENCE
  from_std(std::mt19937(seed), state);
#else
  acr::Mt19937 g;
  acr::mt_seed(g, seed);
  store(g, state);
#endif
}

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
  EKernel kernel(corr, n, K, w2, h2);
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

// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product; nothing under alicevision_b200/ may include, link or call this file.
//
// What the five a-contrario RANSAC checkers (acransac{,_h,_s,_e,_f10}_oracle.cpp) share: each defines its model and its restated
// kernel, includes this header and runs `estimate` on the kernel.  Each is built twice by oracle/Makefile (`all`, `ref`):
//   -DACR_USE_REFERENCE -> _ref/libref_<checker>.so: robustEstimation::ACRANSAC, makelogcombi (robustEstimation/ACRansac.hpp) and
//                          randSample (robustEstimation/randSampling.hpp) compiled verbatim from an AliceVision source tree through
//                          oracle/shim, around the checker's restated kernel; the generator is the library's own std::mt19937.
//   (none)              -> libport_<checker>.so: the loop, the NFA tables and the sampling restated below (the sampling is the
//                          engine's alicevision_b200/csrc/acransac_math.h, so the port pins the engine's sampler).
// The trace (iterations at which a better model was found) comes from the model's copy assignment, which ACRANSAC performs exactly
// when `better` fires, and from the number of fit calls (one per iteration).
// Everything here is in an anonymous namespace, so each checker library keeps its own copy, g_trace included.
#pragma once

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

// The base of each checker's Model: ACRANSAC's `*model = vec_models[k]` when a better model is found records the iteration.  Copy
// construction (the models ACRANSAC collects) records nothing.
struct TracedModel {
  TracedModel() = default;
  TracedModel(const TracedModel&) = default;
  TracedModel& operator=(const TracedModel&) {
    if (g_trace) g_trace->better.push_back((int)(g_trace->fits - 1));
    return *this;
  }
};

// each kernel's fit() counts its call
void trace_fit() {
  if (g_trace) ++g_trace->fits;
}

#ifndef ACR_USE_REFERENCE
// ---- the restated loop (robustEstimation/ACRansac.hpp:145-285) and tables, for any kernel
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

template <int K>
void sample(acr::Mt19937& g, const std::vector<std::size_t>& elements, std::vector<std::size_t>& out) {
  uint32_t s[K];
  acr::rand_sample<K>(g, (uint32_t)elements.size(), s);
  out.resize(K);
  for (int i = 0; i < K; ++i) out[i] = elements[s[i]];
}

template <class Kernel>
std::pair<double, double> acransac_port(const Kernel& kernel, acr::Mt19937& g, std::vector<std::size_t>& vec_inliers, std::size_t nIter,
                                        typename Kernel::ModelT* model, double precision) {
  using Model = typename Kernel::ModelT;
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
    sample<Kernel::kSampleSize>(g, mode ? vec_index : all, s);
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

// 1 = "ref" (compiled reference loop, sampling and NFA), 0 = "port"
int is_reference() {
#ifdef ACR_USE_REFERENCE
  return 1;
#else
  return 0;
#endif
}

// std::mt19937(seed) as 624 words + position (the library's operator<< order)
void mt_seed(uint32_t seed, uint32_t* state) {
#ifdef ACR_USE_REFERENCE
  from_std(std::mt19937(seed), state);
#else
  acr::Mt19937 g;
  acr::mt_seed(g, seed);
  store(g, state);
#endif
}

// `draws` consecutive randSample(g, 0, range, k) from `state`: the samples in their order (draws x k), and the generator state after
// each draw (draws x 625) when states != nullptr.  The port samples k = 4 or 7.
void rand_sample_draws(const uint32_t* state, int k, int range, int draws, uint32_t* out, uint32_t* states) {
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
void logc(int k, int n, float* logc_n, float* logc_k) {
  std::vector<float> a, b;
#ifdef ACR_USE_REFERENCE
  aliceVision::robustEstimation::makelogcombi<float>((std::size_t)k, (std::size_t)n, b, a);
#else
  logc_tables((std::size_t)k, (std::size_t)n, a, b);
#endif
  std::memcpy(logc_n, a.data(), (n + 1) * sizeof(float));
  std::memcpy(logc_k, b.data(), (n + 1) * sizeof(float));
}

// ACRANSAC of one pair on a constructed kernel: the compiled reference's in "ref", acransac_port in "port".  state: the generator on
// entry; state_out: the generator after the estimation (nullptr: not wanted).  inliers: capacity kernel.nbSamples().  trace: the
// iterations at which a better model was found (first trace_cap of *n_trace); trace_nfa: the new minNFA of each (NaN in the "ref"
// build).  The caller copies its model out of `model`.  Returns the iterations executed.
template <class Kernel>
long estimate(const Kernel& kernel, const uint32_t* state, uint32_t* state_out, long max_iter, double precision,
              typename Kernel::ModelT& model, int* valid, int* n_inliers, uint32_t* inliers, double* error_max, double* min_nfa,
              int* trace, double* trace_nfa, int trace_cap, int* n_trace) {
  Trace tr;
  g_trace = &tr;
  std::vector<std::size_t> inl;
  std::pair<double, double> out;
#ifdef ACR_USE_REFERENCE
  std::mt19937 g = to_std(state);
  out = aliceVision::robustEstimation::ACRANSAC(kernel, g, inl, (std::size_t)max_iter, &model, precision);
  if (state_out) from_std(g, state_out);
#else
  acr::Mt19937 g;
  load(g, state);
  out = acransac_port(kernel, g, inl, (std::size_t)max_iter, &model, precision);
  if (state_out) store(g, state_out);
#endif
  g_trace = nullptr;
  *valid = !inl.empty();
  *n_inliers = (int)inl.size();
  for (std::size_t i = 0; i < inl.size(); ++i) inliers[i] = (uint32_t)inl[i];
  *error_max = out.first;
  *min_nfa = out.second;
  *n_trace = (int)tr.better.size();
  for (int i = 0; i < std::min(trace_cap, (int)tr.better.size()); ++i) {
    trace[i] = tr.better[i];
    trace_nfa[i] = i < (int)tr.nfa.size() ? tr.nfa[i] : std::numeric_limits<double>::quiet_NaN();
  }
  return tr.fits;
}

}  // namespace

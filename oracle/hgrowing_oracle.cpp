// ORACLE (test infrastructure): the single-threaded port of filterMatchesByHGrowing (GeometricFilterMatrix_HGrowing.cpp:59-194) on
// the shared math of alicevision_b200/csrc/hgrowing_math.h.
//
// The loops are the reference's: each round walks the seeds of the remaining list in order, skips a seed its round has already used,
// grows the others (growHomography: similarity, 4 affinities, 3 homographies, each followed by the inlier scan), unions every grown set
// into the used set and keeps the first seed of maximal size; then refineHomography, the minNbMatchesPerH stops, the store and the
// stable removal.  A round in which no seed grows ends the filter (the reference would refine an uninitialised homography on an empty
// problem there).  The fits and the refine fold their 32 lane partials in the order the engine's warps use (see the header), so the
// engine reproduces this port bit for bit.  No reference build exists: the reference's fits need Eigen's JacobiSVD and Ceres.
#include "../alicevision_b200/csrc/hgrowing_math.h"

#include <cstdint>
#include <vector>

using namespace hg;

namespace {

template <class Acc, class Merge>
void fold(Acc* a, Merge merge) {
  for (int off = kLanes / 2; off >= 1; off /= 2)
    for (int l = 0; l < off; ++l) merge(a[l], a[l + off]);
}

struct Item {
  const float* feat;
  std::vector<int> rem;   // remaining putatives (indices into feat), in order
  const float* f(int j) const { return feat + (size_t)kFeat * rem[j]; }
  int n() const { return (int)rem.size(); }
};

int scan(const Item& it, const double* T, double tol, std::vector<char>& in) {
  const double t2 = mul(tol, tol);
  in.assign(it.n(), 0);
  int cnt = 0;
  for (int j = 0; j < it.n(); ++j) cnt += (in[j] = transfer_error(T, it.f(j)) < t2);
  return cnt;
}

void fit_affinity(const Item& it, const std::vector<char>& in, double T[9]) {
  AffAcc a[kLanes];
  for (auto& x : a) tri_zero(x);
  for (int j = 0; j < it.n(); ++j)
    if (in[j]) aff_add(a[j % kLanes], it.f(j));
  fold(a, [](AffAcc& lo, const AffAcc& hi) { tri_merge(lo, hi); });
  aff_solve(a[0], T);
}

void fit_homography(const Item& it, const std::vector<char>& in, int k, double H[9]) {
  CenAcc c[kLanes];
  for (auto& x : c) cen_zero(x);
  for (int j = 0; j < it.n(); ++j)
    if (in[j]) cen_add_sum(c[j % kLanes], it.f(j));
  fold(c, [](CenAcc& lo, const CenAcc& hi) { cen_merge(lo, hi); });
  float mean[4];
  cen_mean(c[0], k, mean);
  for (auto& x : c) cen_zero(x);
  for (int j = 0; j < it.n(); ++j)
    if (in[j]) cen_add_dev(c[j % kLanes], mean, it.f(j));
  fold(c, [](CenAcc& lo, const CenAcc& hi) { cen_merge(lo, hi); });
  double CI[9], CJ[9];
  cen_matrix(mean, c[0], k, 0, CI);
  cen_matrix(mean, c[0], k, 2, CJ);
  std::vector<DltAcc> d(kLanes);
  for (auto& x : d) tri_zero(x);
  for (int j = 0; j < it.n(); ++j)
    if (in[j]) dlt_add(d[j % kLanes], CI, CJ, it.f(j));
  fold(d.data(), [](DltAcc& lo, const DltAcc& hi) { tri_merge(lo, hi); });
  dlt_solve(d[0], CI, CJ, H);
}

// growHomography: returns whether the seed grows; T and in hold the last transformation and its inlier set
bool grow(const Item& it, int seed, const Param& p, double T[9], std::vector<char>& in, int& cnt) {
  cnt = 0;
  for (int q = 0; q < 9; ++q) T[q] = q % 4 == 0 ? 1.0 : 0.0;
  for (int s = 0; s < p.nb_refining_iterations; ++s) {
    if (s == 0) similarity(it.f(seed), T);
    else if (s <= 4) fit_affinity(it, in, T);
    else fit_homography(it, in, cnt, T);
    cnt = scan(it, T, step_tolerance(p, s), in);
    if (cnt < p.min_inliers_to_refine) return false;
  }
  return !is_identity(T);
}

struct RefineEval {
  const Item& it;
  const std::vector<char>& in;
  double ts2;
  void operator()(const double* x, bool jac, LmAcc& out) const {
    LmAcc a[kLanes];
    for (auto& v : a) lm_zero(v);
    for (int j = 0; j < it.n(); ++j)
      if (in[j]) lm_add(a[j % kLanes], x, ts2, it.f(j), jac);
    fold(a, [](LmAcc& lo, const LmAcc& hi) { lm_merge(lo, hi); });
    out = a[0];
  }
};

}  // namespace

extern "C" {

// filterMatchesByHGrowing on n putatives feat[8 n].  tols: similarity, affinity, homography; ints: minInliersToRefine,
// nbRefiningIterations, maxNbHomographies, minNbMatchesPerH.  Outputs: n_h; H[max_h x 9] (row-major, x_J ~ H x_I); counts[max_h];
// inliers[<= n] (putative indices, outGeometricInliers order); trace[max_h x 3] per round (chosen seed's remaining-list position or -1,
// best-set size before and after the refine); rounds; stats[2] += seeds grown, seeds skipped.
int hg_filter(int n, const float* feat, const double* tols, const int32_t* ints, int32_t* n_h, double* H, int32_t* counts, int32_t* inliers,
              int32_t* trace, int32_t* rounds, int64_t* stats) {
  Param p;
  p.tol_similarity = tols[0]; p.tol_affinity = tols[1]; p.tol_homography = tols[2];
  p.min_inliers_to_refine = ints[0]; p.nb_refining_iterations = ints[1]; p.max_nb_homographies = ints[2]; p.min_nb_matches_per_h = ints[3];
  Item it{feat, {}};
  for (int j = 0; j < n; ++j) it.rem.push_back(j);
  *n_h = 0; *rounds = 0;
  int n_out = 0;
  std::vector<char> used, in, best_in;
  for (int iH = 0; iH < p.max_nb_homographies; ++iH) {
    ++*rounds;
    int32_t* tr = trace + 3 * iH;
    used.assign(it.n(), 0);
    int best_seed = -1, best_cnt = 0;
    double best_H[9];
    for (int seed = 0; seed < it.n(); ++seed) {
      if (used[seed]) { ++stats[1]; continue; }
      ++stats[0];
      double T[9];
      int cnt;
      if (!grow(it, seed, p, T, in, cnt)) continue;
      for (int j = 0; j < it.n(); ++j) used[j] |= in[j];
      if (cnt > best_cnt) {
        best_cnt = cnt; best_seed = seed; best_in = in;
        for (int q = 0; q < 9; ++q) best_H[q] = T[q];
      }
    }
    tr[0] = best_seed; tr[1] = best_cnt; tr[2] = 0;
    if (best_seed < 0) break;
    // refineHomography on the best seed's planar set
    int cnt = best_cnt;
    double x[9];
    to_params(best_H, x);
    RefineEval ev{it, best_in, two_sigma2(p.tol_homography)};
    if (lm_refine(x, ev)) {
      from_params(x, best_H);
      cnt = scan(it, best_H, p.tol_homography, best_in);
    }
    tr[2] = cnt;
    if (cnt < p.min_nb_matches_per_h) break;
    for (int q = 0; q < 9; ++q) H[9 * *n_h + q] = best_H[q];
    counts[*n_h] = cnt;
    ++*n_h;
    std::vector<int> keep;
    for (int j = 0; j < it.n(); ++j) {
      if (best_in[j]) inliers[n_out++] = it.rem[j];
      else keep.push_back(it.rem[j]);
    }
    it.rem.swap(keep);
    if (it.n() < p.min_nb_matches_per_h) break;
  }
  return n_out;
}

// the transformation of every growHomography step of one seed (steps x 9) and the inlier count after it; returns the steps run
int hg_grow_steps(int n, const float* feat, const double* tols, const int32_t* ints, int seed, double* T_out, int32_t* cnt_out) {
  Param p;
  p.tol_similarity = tols[0]; p.tol_affinity = tols[1]; p.tol_homography = tols[2];
  p.min_inliers_to_refine = ints[0]; p.nb_refining_iterations = ints[1];
  Item it{feat, {}};
  for (int j = 0; j < n; ++j) it.rem.push_back(j);
  std::vector<char> in;
  double T[9];
  int cnt = 0;
  for (int s = 0; s < p.nb_refining_iterations; ++s) {
    if (s == 0) similarity(it.f(seed), T);
    else if (s <= 4) fit_affinity(it, in, T);
    else fit_homography(it, in, cnt, T);
    cnt = scan(it, T, step_tolerance(p, s), in);
    for (int q = 0; q < 9; ++q) T_out[9 * s + q] = T[q];
    cnt_out[s] = cnt;
    if (cnt < p.min_inliers_to_refine) return s + 1;
  }
  return p.nb_refining_iterations;
}

// refineHomography of H (row-major, in place) on the n matches feat; returns whether the solution is usable
int hg_refine(int n, const float* feat, double tol, double* H) {
  Item it{feat, {}};
  for (int j = 0; j < n; ++j) it.rem.push_back(j);
  std::vector<char> in(n, 1);
  double x[9];
  to_params(H, x);
  RefineEval ev{it, in, two_sigma2(tol)};
  if (!lm_refine(x, ev)) return 0;
  from_params(x, H);
  return 1;
}

double hg_exp(double x) { return exp_(x); }
double hg_log(double x) { return log_(x); }

}  // extern "C"

// K12: the homography-growing filter (filterMatchesByHGrowing, GeometricFilterMatrix_HGrowing.cpp:108-194) for a list of work items.
// A work item is one (pair, describer type) with its n putatives, 8 floats each (hgrowing_math.h).  Every round of the reference runs
// over all live items of a batch at once:
//   * grow (hg_grow_kernel), in windows of W seeds per item: every seed of the window that no earlier window of the round has used is
//     grown by one warp (growHomography: 8 fit-and-scan steps over the remaining list; each scan writes a bitset, counted by popcount);
//     the seed's last transformation and set size go to its slot;
//   * replay (hg_replay_kernel), one warp per item: walks the window's seeds in order with the reference's rules (skip a used seed,
//     union a grown seed's set into the used bitset, a strictly larger set becomes the best), so seeds grown speculatively and then
//     covered by an earlier seed of the same window are discarded;
//   * finish (hg_finish_kernel), one warp per item: refineHomography, the minNbMatchesPerH stops, the store of H, its count and its
//     inliers, and the stable removal of the stored set from the remaining list.
// A grown seed's set is the inlier set of its last transformation at the last step's tolerance, so the replay and the finish rescan
// it instead of keeping one bitset per seed.  Growth does not depend on the used set, so the result is the same for every window size;
// W = 1 is the reference's loop.
#pragma once
#include "hgrowing_math.h"

#include <cstdint>

namespace hgk {

constexpr int kWarps = 4;                 // warps per block of every K12 kernel
constexpr int kMaxItem = 1 << 18;         // putatives per work item
constexpr int kMaxH = 64;                 // maxNbHomographies bound (the trace holds one row per round)
constexpr unsigned kFull = 0xffffffffu;

struct Item {
  long long off;        // first putative of the item in the call's feature array; also its first inlier slot in the output
  long long rem_off;    // first slot of its remaining list in the batch
  long long used_off;   // first word of its used bitset in the batch
  int n, n_r;           // putatives, remaining putatives
  int done, round, n_h, n_out;
  int best_seed, best_cnt;
  int row;              // item index in the call (output row)
  double best_H[9];
};

struct Seed { double T[9]; int cnt, ok; };

struct Ctl {
  const float* feat;    // the call's putatives, 8 floats each
  Item* items; int n_items;
  int* rem; uint32_t* used;
  Seed* seeds;          // n_items x window
  int window;
  uint32_t* scratch; int scratch_words;   // per grow warp: the bitset of its current step
  hg::Param p;
  // outputs (rows = call item indices)
  double* H; int* counts; int* trace; int* inl; int* n_h; int* rounds;
  unsigned long long* stats;   // seeds grown, seeds skipped
};

__device__ __forceinline__ bool bit(const uint32_t* b, int j) { return (b[j >> 5] >> (j & 31)) & 1u; }

__device__ __forceinline__ double bcast(double v) { return __shfl_sync(kFull, v, 0); }

template <int M, int W>
__device__ __forceinline__ void fold_tri(hg::Tri<M, W>& t, int lane) {
  for (int off = 16; off >= 1; off >>= 1) {
    hg::Tri<M, W> h;
#pragma unroll
    for (int q = 0; q < hg::Tri<M, W>::kSize; ++q) h.r[q] = __shfl_down_sync(kFull, t.r[q], off);
    if (lane < off) hg::tri_merge(t, h);
  }
}

__device__ __forceinline__ void fold_cen(hg::CenAcc& c, int lane) {
  for (int off = 16; off >= 1; off >>= 1) {
    hg::CenAcc h;
#pragma unroll
    for (int q = 0; q < 4; ++q) h.s[q] = __shfl_down_sync(kFull, c.s[q], off);
    if (lane < off) hg::cen_merge(c, h);
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) c.s[q] = __shfl_sync(kFull, c.s[q], 0);
}

// the inliers of T at tolerance tol over the remaining list, as a bitset (one word per 32 positions); returns the count on every lane
__device__ __forceinline__ int scan(const float* F, const int* rem, int n_r, const double* T, double tol, uint32_t* bits, int lane) {
  const double t2 = hg::mul(tol, tol);
  int cnt = 0;
  for (int j0 = 0; j0 < n_r; j0 += 32) {
    const int j = j0 + lane;
    const bool in = j < n_r && hg::transfer_error(T, F + (size_t)hg::kFeat * rem[j]) < t2;
    const unsigned b = __ballot_sync(kFull, in);
    if (lane == 0) bits[j0 >> 5] = b;
    cnt += __popc(b);
  }
  __syncwarp();
  return cnt;
}

__device__ void fit_affinity(const float* F, const int* rem, int n_r, const uint32_t* bits, double T[9], int lane) {
  hg::AffAcc a;
  hg::tri_zero(a);
  for (int j = lane; j < n_r; j += 32)
    if (bit(bits, j)) hg::aff_add(a, F + (size_t)hg::kFeat * rem[j]);
  fold_tri(a, lane);
  if (lane == 0) hg::aff_solve(a, T);
#pragma unroll
  for (int q = 0; q < 9; ++q) T[q] = bcast(T[q]);
}

__device__ void fit_homography(const float* F, const int* rem, int n_r, const uint32_t* bits, int k, double H[9], int lane) {
  hg::CenAcc c;
  hg::cen_zero(c);
  for (int j = lane; j < n_r; j += 32)
    if (bit(bits, j)) hg::cen_add_sum(c, F + (size_t)hg::kFeat * rem[j]);
  fold_cen(c, lane);
  float mean[4];
  hg::cen_mean(c, k, mean);
  hg::cen_zero(c);
  for (int j = lane; j < n_r; j += 32)
    if (bit(bits, j)) hg::cen_add_dev(c, mean, F + (size_t)hg::kFeat * rem[j]);
  fold_cen(c, lane);
  double CI[9], CJ[9];
  hg::cen_matrix(mean, c, k, 0, CI);
  hg::cen_matrix(mean, c, k, 2, CJ);
  hg::DltAcc d;
  hg::tri_zero(d);
  for (int j = lane; j < n_r; j += 32)
    if (bit(bits, j)) hg::dlt_add(d, CI, CJ, F + (size_t)hg::kFeat * rem[j]);
  fold_tri(d, lane);
  if (lane == 0) hg::dlt_solve(d, CI, CJ, H);
#pragma unroll
  for (int q = 0; q < 9; ++q) H[q] = bcast(H[q]);
}

// growHomography of the seed at remaining-list position `seed`
__device__ bool grow(const Ctl& c, const Item& it, int seed, uint32_t* bits, double T[9], int& cnt, int lane) {
  const float* F = c.feat + (size_t)hg::kFeat * it.off;
  const int* rem = c.rem + it.rem_off;
  cnt = 0;
  for (int s = 0; s < c.p.nb_refining_iterations; ++s) {
    if (s == 0) hg::similarity(F + (size_t)hg::kFeat * rem[seed], T);
    else if (s <= 4) fit_affinity(F, rem, it.n_r, bits, T, lane);
    else fit_homography(F, rem, it.n_r, bits, cnt, T, lane);
    cnt = scan(F, rem, it.n_r, T, hg::step_tolerance(c.p, s), bits, lane);
    if (cnt < c.p.min_inliers_to_refine) return false;
  }
  return c.p.nb_refining_iterations > 0 && !hg::is_identity(T);
}

__global__ void __launch_bounds__(32 * kWarps) hg_grow_kernel(Ctl c, int win) {
  const int lane = threadIdx.x & 31;
  const long long gw = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5), nw = (long long)gridDim.x * kWarps;
  uint32_t* bits = c.scratch + (size_t)gw * c.scratch_words;
  const long long tasks = (long long)c.n_items * c.window;
  for (long long t = gw; t < tasks; t += nw) {
    const int k = (int)(t / c.window), seed = win * c.window + (int)(t % c.window);
    const Item& it = c.items[k];
    if (it.done || seed >= it.n_r || bit(c.used + it.used_off, seed)) continue;
    double T[9];
    int cnt;
    const bool ok = grow(c, it, seed, bits, T, cnt, lane);
    if (lane == 0) {
      Seed& s = c.seeds[t];
      for (int q = 0; q < 9; ++q) s.T[q] = T[q];
      s.cnt = cnt; s.ok = ok;
      atomicAdd(&c.stats[0], 1ull);
    }
  }
}

__global__ void __launch_bounds__(32 * kWarps) hg_replay_kernel(Ctl c, int win) {
  const int lane = threadIdx.x & 31;
  const int k = blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (k >= c.n_items) return;
  Item& it = c.items[k];
  const int base = win * c.window;
  if (it.done || base >= it.n_r) return;
  const float* F = c.feat + (size_t)hg::kFeat * it.off;
  const int* rem = c.rem + it.rem_off;
  uint32_t* used = c.used + it.used_off;
  const double tol = hg::step_tolerance(c.p, c.p.nb_refining_iterations - 1);
  const double t2 = hg::mul(tol, tol);
  int best_seed = it.best_seed, best_cnt = it.best_cnt, skipped = 0;
  for (int slot = 0; slot < c.window && base + slot < it.n_r; ++slot) {
    const int seed = base + slot;
    if (bit(used, seed)) { ++skipped; continue; }
    const Seed& s = c.seeds[(size_t)k * c.window + slot];
    if (!s.ok) continue;
    for (int j0 = 0; j0 < it.n_r; j0 += 32) {
      const int j = j0 + lane;
      const bool in = j < it.n_r && hg::transfer_error(s.T, F + (size_t)hg::kFeat * rem[j]) < t2;
      const unsigned b = __ballot_sync(kFull, in);
      if (lane == 0 && b) used[j0 >> 5] |= b;
    }
    __syncwarp();
    if (s.cnt > best_cnt) {
      best_cnt = s.cnt; best_seed = seed;
      if (lane < 9) it.best_H[lane] = s.T[lane];
    }
  }
  if (lane == 0) {
    it.best_seed = best_seed; it.best_cnt = best_cnt;
    if (skipped) atomicAdd(&c.stats[1], (unsigned long long)skipped);
  }
}

// refineHomography's residual blocks: the set bits of `bits`, folded in lane order and broadcast
struct RefineEval {
  const float* F; const int* rem; const uint32_t* bits; int n_r; double ts2; int lane;
  __device__ void operator()(const double* x, bool jac, hg::LmAcc& out) const {
    hg::LmAcc a;
    hg::lm_zero(a);
    for (int j = lane; j < n_r; j += 32)
      if (bit(bits, j)) hg::lm_add(a, x, ts2, F + (size_t)hg::kFeat * rem[j], jac);
    for (int off = 16; off >= 1; off >>= 1) {
      hg::LmAcc h;
#pragma unroll
      for (int q = 0; q < 45; ++q) h.jtj[q] = __shfl_down_sync(kFull, a.jtj[q], off);
#pragma unroll
      for (int q = 0; q < 9; ++q) h.jtr[q] = __shfl_down_sync(kFull, a.jtr[q], off);
      h.rr = __shfl_down_sync(kFull, a.rr, off);
      if (lane < off) hg::lm_merge(a, h);
    }
#pragma unroll
    for (int q = 0; q < 45; ++q) out.jtj[q] = bcast(a.jtj[q]);
#pragma unroll
    for (int q = 0; q < 9; ++q) out.jtr[q] = bcast(a.jtr[q]);
    out.rr = bcast(a.rr);
  }
};

__global__ void __launch_bounds__(32 * kWarps) hg_finish_kernel(Ctl c) {
  const int lane = threadIdx.x & 31;
  const int k = blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (k >= c.n_items) return;
  Item& it = c.items[k];
  if (it.done) return;
  const int mh = c.p.max_nb_homographies;
  const float* F = c.feat + (size_t)hg::kFeat * it.off;
  int* rem = c.rem + it.rem_off;
  uint32_t* used = c.used + it.used_off;
  int* tr = c.trace + ((size_t)it.row * mh + it.round) * 3;
  const int n_r0 = it.n_r;
  bool done = false;
  if (it.best_seed < 0) {
    if (lane == 0) { tr[0] = -1; tr[1] = 0; tr[2] = 0; }
    done = true;
  } else {
    // the best seed's set, then refineHomography on it
    double H[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) H[q] = it.best_H[q];
    int cnt = scan(F, rem, n_r0, H, hg::step_tolerance(c.p, c.p.nb_refining_iterations - 1), used, lane);
    double x[9];
    hg::to_params(H, x);
    RefineEval ev{F, rem, used, n_r0, hg::two_sigma2(c.p.tol_homography), lane};
    if (hg::lm_refine(x, ev)) {
      hg::from_params(x, H);
      cnt = scan(F, rem, n_r0, H, c.p.tol_homography, used, lane);
    }
    if (lane == 0) { tr[0] = it.best_seed; tr[1] = it.best_cnt; tr[2] = cnt; }
    if (cnt < c.p.min_nb_matches_per_h) {
      done = true;
    } else {
      if (lane < 9) c.H[((size_t)it.row * mh + it.n_h) * 9 + lane] = H[lane];
      if (lane == 0) c.counts[(size_t)it.row * mh + it.n_h] = cnt;
      // store the set's putatives in order and remove them from the remaining list, keeping the order
      int* out = c.inl + it.off + it.n_out;
      int n_in = 0, n_keep = 0;
      const unsigned lt = (1u << lane) - 1;
      for (int j0 = 0; j0 < n_r0; j0 += 32) {
        const int j = j0 + lane;
        const bool live = j < n_r0;
        const int v = live ? rem[j] : 0;
        const bool in = live && bit(used, j);
        const unsigned bi = __ballot_sync(kFull, in), bk = __ballot_sync(kFull, live && !in);
        __syncwarp();
        if (in) out[n_in + __popc(bi & lt)] = v;
        else if (live) rem[n_keep + __popc(bk & lt)] = v;
        n_in += __popc(bi); n_keep += __popc(bk);
      }
      __syncwarp();
      if (lane == 0) { it.n_out += n_in; it.n_r = n_keep; it.n_h += 1; }
      done = n_keep < c.p.min_nb_matches_per_h;
    }
  }
  for (int w = lane; w < (n_r0 + 31) / 32; w += 32) used[w] = 0;
  __syncwarp();
  if (lane == 0) {
    it.round += 1;
    it.best_seed = -1; it.best_cnt = 0;
    it.done = done || it.round >= mh;
    c.n_h[it.row] = it.n_h;
    c.rounds[it.row] = it.round;
  }
}

}  // namespace hgk

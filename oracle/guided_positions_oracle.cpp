// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product; nothing under alicevision_b200/ may include, link or call this file.
//
// Position-only guided matching on DOUBLE positions:
//   gf_guided_match_positions  matching::guidedMatching<Mat3Model, FundamentalEpipolarDistanceError | HomographyAsymmetricError>
//                              (model, xLeft, xRight, errorTh, matches) (matching/guidedMatching.hpp:37-70), then
//                              IndMatch::getDeduplicated (IndMatch.hpp:52-58)
// No descriptor is read, so there is nothing of the reference to compile in: the "ref" and "port" builds of the other guided oracles
// would be the same code, and oracle/Makefile (target `all`) builds this file once.  The geometry is RESTATED, as in
// guided_fast_oracle.cpp: the association a coefficient-wise Eigen evaluation gives (H x)(r) = (H(r,0)*x + H(r,1)*y) + H(r,2)*1,
// separate multiply / add (-ffp-contract=off).  Eigen is not in this image, so this part of the parity is not pinned by compiled
// reference code.  The decorator that follows in GeometricFilterMatrix_H_AC is the compiled reference's own (ref_decorator_dedup,
// oracle/ref_oracle.cpp).
#include <cstdint>
#include <limits>
#include <set>
#include <utility>

extern "C" {

// model 0 = FundamentalEpipolarDistanceError (FundamentalError.hpp:52-64), 1 = HomographyAsymmetricError (HomographyError.hpp:23-31).
// xy_l: n_l x 2, xy_r: n_r x 2, M row-major; out_ij: capacity max(n_l, 1) matches (i, j), sorted by (i, j).  Returns the count.
int gf_guided_match_positions(int model, const double* xy_l, int n_l, const double* xy_r, int n_r, const double* M, double errorTh, uint32_t* out_ij) {
  std::set<std::pair<uint32_t, uint32_t>> out;                                 // IndMatch::getDeduplicated
  for (int i = 0; i < n_l; ++i) {
    const double x0 = xy_l[2 * i], x1 = xy_l[2 * i + 1];
    const double Fx0 = (M[0] * x0 + M[1] * x1) + M[2] * 1.0, Fx1 = (M[3] * x0 + M[4] * x1) + M[5] * 1.0, Fx2 = (M[6] * x0 + M[7] * x1) + M[8] * 1.0;
    double min = std::numeric_limits<double>::max();
    std::pair<uint32_t, uint32_t> match(0, 0);                                 // matching::IndMatch match; = IndMatch(0, 0)
    for (int j = 0; j < n_r; ++j) {
      const double y0 = xy_r[2 * j], y1 = xy_r[2 * j + 1];
      double err;
      if (model == 1) {
        const double e0 = Fx0 / Fx2, e1 = Fx1 / Fx2;                           // x2h_est.head<2>() / x2h_est[2]
        const double d0 = y0 - e0, d1 = y1 - e1;
        err = d0 * d0 + d1 * d1;
      } else {
        const double dot = (Fx0 * y0 + Fx1 * y1) + Fx2 * 1.0;
        err = (dot * dot) / (Fx0 * Fx0 + Fx1 * Fx1);
      }
      if (err < errorTh && err < min) {
        min = err;
        match = {(uint32_t)i, (uint32_t)j};
      }
    }
    if (min < errorTh) out.insert(match);
  }
  int n = 0;
  for (const auto& m : out) { out_ij[2 * n] = m.first; out_ij[2 * n + 1] = m.second; ++n; }
  return n;
}

}  // extern "C"

// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product; nothing under alicevision_b200/ may include, link or call this file.
//
// Guided matching on DOUBLE positions (the undistorted positions a caller computes with the reference's camera code):
//   gf_guided_fast   matching::guidedMatchingFundamentalFast<FundamentalEpipolarDistanceError> (matching/guidedMatching.hpp:353-460)
//                    with pixToBucket / lineToEndPoints (matching/guidedMatching.cpp:13-70)
//   gf_guided_match  matching::guidedMatching<Mat3Model, FundamentalEpipolarDistanceError | HomographyAsymmetricError>
//                    (matching/guidedMatching.hpp:206-268), the loop of ref_oracle.cpp / port_oracle.cpp on double positions
// Built twice by oracle/guided_fast.mk:
//   -DGF_USE_REFERENCE  -> _ref/libref_guided_fast.so: descriptor distances from the reference's own Regions::SquaredDescriptorDistance
//                          (feature/Regions.hpp:198-207 -> SquaredMetric), compiled from an AliceVision source tree through oracle/shim
//   (none)              -> libport_guided_fast.so: the restated metrics (L2_Vectorized, squared Hamming)
// The geometry (the 3x3 products, the cross products, lineToEndPoints, pixToBucket) is RESTATED in both builds, with the association
// a coefficient-wise evaluation gives and separate multiply / add (-ffp-contract=off): Eigen is not in this image and
// guidedMatching.cpp cannot be compiled here, so this part of the parity is not pinned by compiled reference code.
// Inputs where the reference is undefined (a non-finite epipolar line: an epipole at infinity, a right feature at the epipole) are
// given "no end points" here, as in the engine; the tests do not compare those with the oracle.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <memory>
#include <utility>
#include <vector>

#ifdef GF_USE_REFERENCE
#include <aliceVision/feature/regionsFactory.hpp>
using namespace aliceVision;
using namespace aliceVision::feature;
#endif

namespace {

enum { DT_F32 = 0, DT_U8 = 1, DT_BIN = 2 };

#ifdef GF_USE_REFERENCE
template <class RegionsT>
std::unique_ptr<Regions> make_regions(const void* desc, int n) {
  std::unique_ptr<RegionsT> r(new RegionsT());
  r->Features().reserve(n);
  r->Descriptors().resize(n);
  for (int i = 0; i < n; ++i) r->Features().emplace_back(0.f, 0.f, 1.0f, 0.0f);     // positions are passed separately (double)
  if (n) std::memcpy((void*)r->DescriptorRawData(), desc, (size_t)n * sizeof(typename RegionsT::DescriptorT));
  return std::unique_ptr<Regions>(r.release());
}
std::unique_ptr<Regions> make_any_regions(int dtype, const void* desc, int n) {
  switch (dtype) {
    case DT_F32: return make_regions<SIFT_Float_Regions>(desc, n);
    case DT_U8: return make_regions<SIFT_Regions>(desc, n);
    default: return make_regions<AKAZE_BinaryRegions>(desc, n);
  }
}
#else
// feature/metric.hpp:94-123 L2_Vectorized<float> (four lanes, ((s0+s1)+s2)+s3) and :128-139 <uchar> (exact integers)
float l2_vec_f32(const float* a, const float* b, int n) {
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  for (int i = 0; i < n; i += 4) {
    float t0 = a[i] - b[i], t1 = a[i + 1] - b[i + 1], t2 = a[i + 2] - b[i + 2], t3 = a[i + 3] - b[i + 3];
    t0 = t0 * t0; t1 = t1 * t1; t2 = t2 * t2; t3 = t3 * t3;
    s0 = s0 + t0; s1 = s1 + t1; s2 = s2 + t2; s3 = s3 + t3;
  }
  return ((s0 + s1) + s2) + s3;
}
float l2_vec_u8(const uint8_t* a, const uint8_t* b, int n) {
  int r = 0;
  for (int i = 0; i < n; ++i) { const int d = (int)a[i] - (int)b[i]; r += d * d; }
  return (float)r;
}
// feature/Hamming.hpp:174-185 SquaredHamming: h * h in unsigned, returned as double
double sq_hamming(const uint8_t* a, const uint8_t* b, int n) {
  uint32_t h = 0;
  for (int i = 0; i < n; i += 8) { uint64_t x, y; std::memcpy(&x, a + i, 8); std::memcpy(&y, b + i, 8); h += (uint32_t)__builtin_popcountll(x ^ y); }
  return (double)(h * h);
}
#endif

// Regions::SquaredDescriptorDistance(i, &rRegions, j) of the build
struct Dist {
  int dtype; const void* l; const void* r;
#ifdef GF_USE_REFERENCE
  std::unique_ptr<Regions> rl, rr;
  Dist(int dt, const void* dl, int nl, const void* dr, int nr) : dtype(dt), l(dl), r(dr), rl(make_any_regions(dt, dl, nl)), rr(make_any_regions(dt, dr, nr)) {}
  double operator()(int i, int j) const { return rl->SquaredDescriptorDistance((size_t)i, rr.get(), (size_t)j); }
#else
  Dist(int dt, const void* dl, int, const void* dr, int) : dtype(dt), l(dl), r(dr) {}
  double operator()(int i, int j) const {
    if (dtype == DT_F32) return (double)l2_vec_f32((const float*)l + (size_t)i * 128, (const float*)r + (size_t)j * 128, 128);
    if (dtype == DT_U8) return (double)l2_vec_u8((const uint8_t*)l + (size_t)i * 128, (const uint8_t*)r + (size_t)j * 128, 128);
    return sq_hamming((const uint8_t*)l + (size_t)i * 64, (const uint8_t*)r + (size_t)j * 64, 64);
  }
#endif
};

// distanceRatio<double> (guidedMatching.hpp:77-121)
struct DistanceRatio {
  double bd = std::numeric_limits<double>::max(), sbd = std::numeric_limits<double>::max(); std::size_t idx = 0;
  void update(std::size_t index, double dist) {
    if (dist < bd) { idx = index; sbd = dist; std::swap(bd, sbd); }
    else if (dist < sbd) sbd = dist;
  }
  bool isValid(double distRatio) const { return sbd != std::numeric_limits<double>::max() && bd < distRatio * sbd; }
};

// guidedMatching.cpp:13-22
unsigned int pixToBucket(int x, int y, int W, int H) {
  if (y == 0) return x;
  if (x == W - 1) return W - 1 + y;
  if (y == H - 1) return 2 * W + H - 3 - x;
  return 2 * (W + H - 2) - y;
}

// guidedMatching.cpp:24-70; a non-finite line has no end points (see the header comment)
bool lineToEndPoints(const double line[3], int W, int H, double x0[2], double x1[2]) {
  const double a = line[0], b = line[1], c = line[2];
  if (!std::isfinite(a) || !std::isfinite(b) || !std::isfinite(c)) return false;
  float r1, r2;
  if (b != 0) {
    const double x = (b < 0) ? 0 : W - 1;
    double y = -(a * x + c) / b;
    if (y < 0) y = 0.;
    else if (y >= H) y = H - 1;
    r1 = std::fabs(a * x + b * y + c);
    x0[0] = x; x0[1] = y;
  } else {
    return false;
  }
  if (a != 0) {
    const double y = (a < 0) ? H - 1 : 0;
    double x = -(b * y + c) / a;
    if (x < 0) x = 0.;
    else if (x >= W) x = W - 1;
    r2 = std::fabs(a * x + b * y + c);
    x1[0] = x; x1[1] = y;
  } else {
    return false;
  }
  if (r1 > r2) { std::swap(x0[0], x1[0]); std::swap(x0[1], x1[1]); }
  return true;
}

// Eigen's Vector3::cross: (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0)
void cross(const double a[3], double x, double y, double out[3]) {
  const double b[3] = {x, y, 1.};
  out[0] = a[1] * b[2] - a[2] * b[1];
  out[1] = a[2] * b[0] - a[0] * b[2];
  out[2] = a[0] * b[1] - a[1] * b[0];
}

}  // namespace

extern "C" {

// guidedMatchingFundamentalFast: matches (i, j) in ascending i (the reference emits them so and does not de-duplicate)
int gf_guided_fast(int dtype, const void* desc_l, const double* xy_l, int n_l, const void* desc_r, const double* xy_r, int n_r, const double* FMat,
                   const double* epipole2, int widthR, int heightR, double errorTh, double distRatio, uint32_t* out_ij) {
  const Dist DIST(dtype, desc_l, n_l, desc_r, n_r);
  double F[9], ep2[3];
  for (int k = 0; k < 9; ++k) F[k] = FMat[k];
  for (int k = 0; k < 3; ++k) ep2[k] = epipole2[k];
  if (ep2[2] > 0.0) {                                                       // :378-383
    for (double& f : F) f = -f;
    for (double& e : ep2) e = -e;
  }
  const double e2 = ep2[2];
  for (double& e : ep2) e = e / e2;                                         // :384
  const int nb_buckets = 2 * (widthR + heightR - 2);
  std::vector<std::vector<uint32_t>> buckets(nb_buckets);
  for (int i = 0; i < n_l; ++i) {                                           // :394-406
    const double x = xy_l[2 * i], y = xy_l[2 * i + 1];
    const double line[3] = {(F[0] * x + F[1] * y) + F[2] * 1., (F[3] * x + F[4] * y) + F[5] * 1., (F[6] * x + F[7] * y) + F[8] * 1.};
    double x0[2], x1[2];
    if (lineToEndPoints(line, widthR, heightR, x0, x1)) buckets[pixToBucket((int)x0[0], (int)x0[1], widthR, heightR)].push_back((uint32_t)i);
  }
  std::vector<DistanceRatio> dR(n_l);
  for (int j = 0; j < n_r; ++j) {                                           // :409-442
    const double xr = xy_r[2 * j], yr = xy_r[2 * j + 1];
    double l2[3];
    cross(ep2, xr, yr, l2);
    const double s = std::sqrt(errorTh) / std::sqrt(l2[0] * l2[0] + l2[1] * l2[1]);
    const double n0 = l2[0] * s, n1 = l2[1] * s;
    double l2min[3], l2max[3], x0[2], x1[2];
    cross(ep2, xr - n0, yr - n1, l2min);
    cross(ep2, xr + n0, yr + n1, l2max);
    if (!lineToEndPoints(l2min, widthR, heightR, x0, x1)) continue;
    const unsigned bucketStart = pixToBucket((int)x0[0], (int)x0[1], widthR, heightR);
    if (!lineToEndPoints(l2max, widthR, heightR, x0, x1)) continue;
    const unsigned bucketStop = pixToBucket((int)x0[0], (int)x0[1], widthR, heightR);
    if (bucketStop > bucketStart)
      for (unsigned b = bucketStart; b < bucketStop; ++b)
        for (uint32_t i : buckets[b]) dR[i].update((std::size_t)j, DIST((int)i, j));
  }
  int n = 0;
  for (int i = 0; i < n_l; ++i)                                             // :444-451
    if (dR[i].isValid(distRatio)) { out_ij[2 * n] = (uint32_t)i; out_ij[2 * n + 1] = (uint32_t)dR[i].idx; ++n; }
  return n;
}

// guidedMatching on double positions: model 0 = FundamentalEpipolarDistanceError (FundamentalError.hpp:52-64),
// 1 = HomographyAsymmetricError (HomographyError.hpp:23-31); sorted and de-duplicated (:267)
int gf_guided_match(int dtype, int model, const void* desc_l, const double* xy_l, int n_l, const void* desc_r, const double* xy_r, int n_r,
                    const double* F, double errorTh, double distRatio, uint32_t* out_ij) {
  const Dist DIST(dtype, desc_l, n_l, desc_r, n_r);
  std::vector<std::pair<uint32_t, uint32_t>> out;
  for (int i = 0; i < n_l; ++i) {
    const double x0 = xy_l[2 * i], x1 = xy_l[2 * i + 1];
    const double Fx0 = (F[0] * x0 + F[1] * x1) + F[2] * 1.0, Fx1 = (F[3] * x0 + F[4] * x1) + F[5] * 1.0, Fx2 = (F[6] * x0 + F[7] * x1) + F[8] * 1.0;
    const double nrm = Fx0 * Fx0 + Fx1 * Fx1;
    DistanceRatio dR;
    for (int j = 0; j < n_r; ++j) {
      const double y0 = xy_r[2 * j], y1 = xy_r[2 * j + 1];
      double geomErr;
      if (model == 1) {
        const double e0 = Fx0 / Fx2, e1 = Fx1 / Fx2;
        const double d0 = y0 - e0, d1 = y1 - e1;
        geomErr = d0 * d0 + d1 * d1;
      } else {
        const double dot = (Fx0 * y0 + Fx1 * y1) + Fx2 * 1.0;
        geomErr = (dot * dot) / nrm;
      }
      if (geomErr < errorTh) dR.update((std::size_t)j, DIST(i, j));
    }
    if (dR.isValid(distRatio)) out.push_back({(uint32_t)i, (uint32_t)dR.idx});
  }
  std::sort(out.begin(), out.end());
  out.erase(std::unique(out.begin(), out.end()), out.end());
  for (size_t k = 0; k < out.size(); ++k) { out_ij[2 * k] = out[k].first; out_ij[2 * k + 1] = out[k].second; }
  return (int)out.size();
}

}  // extern "C"

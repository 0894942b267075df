// Compiles alicevision_b200/adaptor/GeometricFilter_b200.hpp against the REFERENCE's own interface headers (through oracle/shim) and
// checks, on a GPU, GeometricFilterMatrix_F_AC_Batch_b200 on a list that mixes planar pairs (addPair) and pairs of two equidistant
// cameras (addPairSpherical) against the "ref" oracles: the reference's ACRANSAC loop around the restated planar (acr_estimate) or
// spherical (acrs_estimate) kernel from the same generator state, the inlier copy and support rules, and guidedMatching on the
// reference's Regions distances (gf_guided_match) with the adaptor's own F and errorMax^2.  Every pair's estimate is also checked bit
// for bit against a one-pair engine call of its own kind from the same state, which pins how run() splits the list into its planar and
// spherical calls and merges them back in addPair order.
// Built by oracle/spherical_filter.mk into oracle/_ref/spherical_filter_test.
#include <aliceVision/feature/regionsFactory.hpp>

#include <GeometricFilter_b200.hpp>

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <random>
#include <vector>

extern "C" long acr_estimate(int n, const double* corr, int wI, int hI, int wJ, int hJ, const uint32_t* state, long max_iter, double precision,
                             int* valid, int* n_inliers, uint32_t* inliers, double* F, double* error_max, double* min_nfa, int* trace,
                             double* trace_nfa, int trace_cap, int* n_trace);
extern "C" long acrs_estimate(int n, const double* bearings, const uint32_t* state, long max_iter, double precision, int* valid,
                              int* n_inliers, uint32_t* inliers, double* F, double* error_max, double* min_nfa, int* trace, double* trace_nfa,
                              int trace_cap, int* n_trace, uint32_t* state_out);
extern "C" int gf_guided_match(int dtype, int model, const void* desc_l, const double* xy_l, int n_l, const void* desc_r, const double* xy_r,
                               int n_r, const double* F, double errorTh, double distRatio, uint32_t* out_ij);

using namespace aliceVision;
using namespace aliceVision::matching;
using namespace aliceVision::matchingImageCollection;
using namespace aliceVision::feature;

static int g_fail = 0;
#define CHECK(c)                                                              \
    do                                                                        \
    {                                                                         \
        if (!(c))                                                             \
        {                                                                     \
            std::printf("CHECK FAILED %s:%d  %s\n", __FILE__, __LINE__, #c);  \
            ++g_fail;                                                         \
        }                                                                     \
    } while (0)

// 2 x n matrix of the positions of the putatives (what fillMatricesWithUndistortFeaturesMatches gathers for cameras without distortion)
struct Mat2N
{
    std::vector<double> v;
    int cols() const { return (int)v.size() / 2; }
    double operator()(int r, int c) const { return v[2 * c + r]; }
};
// 3 x n matrix of unit vectors
struct Mat3N
{
    std::vector<double> v;
    int cols() const { return (int)v.size() / 3; }
    double operator()(int r, int c) const { return v[3 * c + r]; }
};

static const int W = 1920, Hh = 1080;
static const double f = 1500, cx = 960, cy = 540;

int main()
{
    std::mt19937 g(3);
    std::uniform_real_distribution<double> ux(-3, 3), uy(-2, 2), uz(8, 12), un(-0.5, 0.5);
    const int NP = 1500, NV = 4;
    std::vector<std::array<double, 3>> X(NP);
    std::vector<std::array<unsigned char, 128>> base(NP);
    for (int p = 0; p < NP; ++p)
    {
        X[p] = {ux(g), uy(g), uz(g)};
        for (auto& b : base[p])
            b = (unsigned char)(g() % 64);
    }
    const double C[NV][3] = {{0, 0, 0}, {1.0, 0.1, 0.3}, {-0.8, -0.15, -0.4}, {0.4, 0.3, 0.1}};
    std::vector<std::unique_ptr<SIFT_Regions>> regs(NV);
    std::vector<std::vector<int>> idx(NV, std::vector<int>(NP, -1));     // feature of point p in view v
    std::vector<std::vector<double>> pos(NV);
    for (int v = 0; v < NV; ++v)
    {
        regs[v].reset(new SIFT_Regions());
        for (int p = 0; p < NP; ++p)
        {
            const double x = f * (X[p][0] - C[v][0]) / (X[p][2] - C[v][2]) + cx + un(g), y = f * (X[p][1] - C[v][1]) / (X[p][2] - C[v][2]) + cy + un(g);
            if (x < 0 || y < 0 || x >= W - 1 || y >= Hh - 1 || (g() % 4) == 0)
                continue;
            idx[v][p] = (int)regs[v]->RegionCount();
            regs[v]->Features().emplace_back((float)x, (float)y, 1.f, 0.f);
            SIFT_Regions::DescriptorT d;
            for (int k = 0; k < 128; ++k)
                d[k] = (unsigned char)std::min(255, (int)base[p][k] + (int)(g() % 5));
            regs[v]->Descriptors().push_back(d);
        }
        for (const auto& ft : regs[v]->Features())
        {
            pos[v].push_back((double)ft.x());
            pos[v].push_back((double)ft.y());
        }
    }
    // putatives: true correspondences and 30 % wrong ones; pair (0, 3) gets only 40 true ones (50 inliers or fewer: no strong support)
    const std::vector<Pair> pairs = {{0, 1}, {1, 2}, {0, 2}, {0, 3}, {2, 3}};
    const std::vector<bool> spherical = {true, false, true, false, true};   // views 0, 2 and 3 stand for equidistant cameras
    std::map<Pair, MatchesPerDescType> put;
    for (const Pair& pr : pairs)
    {
        IndMatches& m = put[pr][EImageDescriberType::SIFT];
        for (int p = 0; p < NP; ++p)
            if (idx[pr.first][p] >= 0 && idx[pr.second][p] >= 0)
            {
                if (pr == Pair(0, 3) && m.size() >= 40)
                    break;
                const bool wrong = g() % 10 < 3;
                m.emplace_back(idx[pr.first][p], wrong ? (IndexT)(g() % regs[pr.second]->RegionCount()) : (IndexT)idx[pr.second][p], 0.5f, 100.f + p);
            }
    }
    const std::vector<EImageDescriberType> types = {EImageDescriberType::SIFT};
    const std::size_t maxIt = 400;
    const std::mt19937 rng(42);
    std::stringstream ss;
    ss << rng;
    uint32_t state[625];
    for (auto& s : state)
        ss >> s;
    long kept = 0, guidedTotal = 0, compared = 0, oneCall = 0;
    const double inf = std::numeric_limits<double>::infinity();
    for (const bool guided : {false, true})
    {
        long comparedKind[2] = {0, 0};   // oracle comparisons of planar, spherical pairs in this run
        GeometricFilterMatrix_F_AC_Batch_b200 batch;
        CHECK(batch.available());
        for (int v = 0; v < NV; ++v)
            CHECK(batch.addView(v, EImageDescriberType::SIFT, *regs[v]));
        std::vector<Mat2N> xI(pairs.size()), xJ(pairs.size());
        std::vector<Mat3N> bI(pairs.size()), bJ(pairs.size());
        const auto lift = [](Mat3N& b, double x, double y) {   // a stand-in for toUnitSphere(removeDistortion(ima2cam(x)))
            const double u = (x - cx) / f, w = (y - cy) / f, s = std::sqrt(u * u + w * w + 1);
            b.v.insert(b.v.end(), {u / s, w / s, 1 / s});
        };
        for (std::size_t k = 0; k < pairs.size(); ++k)
        {
            for (const IndMatch& m : put[pairs[k]][EImageDescriberType::SIFT])
            {
                xI[k].v.insert(xI[k].v.end(), {pos[pairs[k].first][2 * m._i], pos[pairs[k].first][2 * m._i + 1]});
                xJ[k].v.insert(xJ[k].v.end(), {pos[pairs[k].second][2 * m._j], pos[pairs[k].second][2 * m._j + 1]});
                lift(bI[k], pos[pairs[k].first][2 * m._i], pos[pairs[k].first][2 * m._i + 1]);
                lift(bJ[k], pos[pairs[k].second][2 * m._j], pos[pairs[k].second][2 * m._j + 1]);
            }
            if (spherical[k])
                batch.addPairSpherical(pairs[k], put[pairs[k]], types, bI[k], bJ[k]);
            else
                batch.addPair(pairs[k], put[pairs[k]], types, xI[k], xJ[k], {W, Hh}, {W, Hh});
        }
        PairwiseMatches out;
        CHECK(batch.run(rng, maxIt, std::numeric_limits<double>::infinity(), guided, 0.6, out));
        for (std::size_t k = 0; k < pairs.size(); ++k)
        {
            const Pair& pr = pairs[k];
            const auto& e = batch.estimate(k);
            const IndMatches& pm = put[pr][EImageDescriberType::SIFT];
            const int n = (int)pm.size();
            std::vector<double> corr;
            for (int c = 0; c < n; ++c)
                if (spherical[k])
                    corr.insert(corr.end(), {bI[k](0, c), bI[k](1, c), bI[k](2, c), bJ[k](0, c), bJ[k](1, c), bJ[k](2, c)});
                else
                    corr.insert(corr.end(), {xI[k](0, c), xI[k](1, c), xJ[k](0, c), xJ[k](1, c)});
            int valid = 0, nInl = 0, nTr = 0;
            std::vector<uint32_t> inl(n + 1), stOut(625);
            std::vector<int> tr(4096);
            std::vector<double> trn(4096);
            double F[9], em = 0, nfa = 0;
            if (spherical[k])
                acrs_estimate(n, corr.data(), state, (long)maxIt, std::numeric_limits<double>::infinity(), &valid, &nInl, inl.data(), F, &em, &nfa,
                              tr.data(), trn.data(), 4096, &nTr, stOut.data());
            else
                acr_estimate(n, corr.data(), W, Hh, W, Hh, state, (long)maxIt, std::numeric_limits<double>::infinity(), &valid, &nInl, inl.data(), F,
                             &em, &nfa, tr.data(), trn.data(), 4096, &nTr);
            CHECK(e.valid == (valid != 0));
            // the same pair alone through the engine entry point of its kind, from the same state: the adaptor's estimate is that call's
            // bit for bit, and its support decision and kept list follow from that call's inliers
            {
                const int64_t offs[2] = {0, n};
                const int32_t wh[4] = {W, Hh, W, Hh};
                uint8_t v1 = 0;
                int32_t ni1 = 0, it1 = 0;
                std::vector<uint32_t> in1(n + 1);
                double F1[9], em1 = 0, nfa1 = 0;
                b200m_ctx* ctx = matching::b200detail::sharedContext();
                const int rc = spherical[k]
                                 ? b200m_acransac_fundamental_spherical_pairs(ctx, 1, offs, corr.data(), state, 0, (int64_t)maxIt, inf, &v1, &ni1, in1.data(),
                                                                              F1, &em1, &nfa1, &it1, nullptr)
                                 : b200m_acransac_fundamental_pairs(ctx, 1, offs, corr.data(), wh, state, (int64_t)maxIt, inf, &v1, &ni1, in1.data(), F1,
                                                                    &em1, &nfa1, &it1);
                CHECK(rc == B200M_OK);
                CHECK(e.valid == (v1 != 0) && std::memcmp(e.F, F1, sizeof F1) == 0);
                if (v1)
                {
                    ++oneCall;
                    CHECK(e.errorMax == em1);
                    MatchesPerDescType want1;
                    matchingImageCollection::b200detail::copyInlierMatches(std::vector<std::size_t>(in1.begin(), in1.begin() + ni1), put[pr], types, want1);
                    const bool strong1 = matchingImageCollection::b200detail::hasStrongSupport(want1, 7);
                    CHECK(e.strongSupport == strong1 && (out.count(pr) > 0) == strong1);
                    if (strong1 && !guided)
                        CHECK(out[pr][EImageDescriberType::SIFT] == want1[EImageDescriberType::SIFT]);
                }
            }
            // where the engine's model is the oracle's up to rounding (K10's parity protocol: F and errorMax within 1e-9), the decision
            // and the inliers are the oracle's
            double fmax = 0, fdiff = 0;
            for (int q = 0; q < 9; ++q)
            {
                fmax = std::max(fmax, std::fabs(F[q]));
                fdiff = std::max(fdiff, std::fabs(F[q] - e.F[q]));
            }
            if (valid && fdiff <= 1e-9 * fmax && std::fabs(em - e.errorMax) <= 1e-9 * em)
            {
                ++compared;
                ++comparedKind[spherical[k] ? 1 : 0];
                MatchesPerDescType want;
                matchingImageCollection::b200detail::copyInlierMatches(std::vector<std::size_t>(inl.begin(), inl.begin() + nInl), put[pr], types, want);
                const bool strong = matchingImageCollection::b200detail::hasStrongSupport(want, 7);
                CHECK(e.strongSupport == strong);
                CHECK((out.count(pr) > 0) == strong);
                if (strong && !guided)
                {
                    const IndMatches& a = out[pr][EImageDescriberType::SIFT];
                    const IndMatches& b = want[EImageDescriberType::SIFT];
                    CHECK(a.size() == b.size());
                    for (std::size_t q = 0; q < a.size() && q < b.size(); ++q)
                        CHECK(a[q] == b[q] && a[q]._distance == b[q]._distance && a[q]._distanceRatio == b[q]._distanceRatio);
                }
            }
            if (pr == Pair(0, 3))
                CHECK(out.count(pr) == 0);
            if (!out.count(pr))
                continue;
            kept += !guided;
            if (guided)
            {
                // the guided lists on the adaptor's own model and threshold
                const SIFT_Regions& L = *regs[pr.first];
                const SIFT_Regions& R = *regs[pr.second];
                std::vector<uint32_t> want(2 * L.RegionCount() + 2);
                const int nw = gf_guided_match(1, 0, L.DescriptorRawData(), pos[pr.first].data(), (int)L.RegionCount(), R.DescriptorRawData(),
                                               pos[pr.second].data(), (int)R.RegionCount(), e.F, e.errorMax * e.errorMax, 0.36, want.data());
                const IndMatches& m = out[pr][EImageDescriberType::SIFT];
                CHECK((int)m.size() == nw);
                for (int q = 0; q < nw && q < (int)m.size(); ++q)
                    CHECK(m[q]._i == want[2 * q] && m[q]._j == want[2 * q + 1]);
                guidedTotal += nw;
            }
        }
        // every run compares pairs of both kinds with the oracle (3 spherical and 2 planar pairs are added)
        CHECK(comparedKind[0] >= 1 && comparedKind[1] >= 2);
        std::printf("run (guided %d): %ld planar and %ld spherical estimates equal to the oracle's\n", (int)guided, comparedKind[0], comparedKind[1]);
    }
    CHECK(kept >= 3 && guidedTotal > 500 && compared >= 4 && oneCall >= 8);
    std::printf("%s: %ld kept pairs, %ld guided matches, %ld estimates equal to the oracle's, %ld valid estimates equal to one-pair calls\n",
                g_fail ? "FAILED" : "spherical_filter adaptor ok", kept, guidedTotal, compared, oneCall);
    return g_fail ? 1 : 0;
}

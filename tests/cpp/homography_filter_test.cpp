// Compiles alicevision_b200/adaptor/GeometricFilter_b200.hpp against the REFERENCE's own interface headers (through oracle/shim) and
// checks, on a GPU, GeometricFilterMatrix_H_AC_Batch_b200 against the "ref" oracles: the reference's ACRANSAC loop around the restated
// homography kernel (acr_estimate_h) from the same generator state, the inlier copy and hasStrongSupport(.., 4), and with
// distanceRatio = -1 the position-only guidedMatching loop (gf_guided_match_positions) followed by the reference's own
// IndMatchDecorator, on the adaptor's own H and errorMax^2.
// Built by oracle/homography_filter.mk into oracle/_ref/homography_filter_test.
#include <aliceVision/feature/regionsFactory.hpp>
#include <aliceVision/matching/IndMatchDecorator.hpp>

#include <GeometricFilter_b200.hpp>

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <map>
#include <memory>
#include <random>
#include <vector>

extern "C" long acr_estimate_h(int n, const double* corr, int wI, int hI, int wJ, int hJ, const uint32_t* state, long max_iter, double precision,
                               int* valid, int* n_inliers, uint32_t* inliers, double* H, double* error_max, double* min_nfa, int* trace,
                               double* trace_nfa, int trace_cap, int* n_trace, uint32_t* state_out);
extern "C" int gf_guided_match_positions(int model, const double* xy_l, int n_l, const double* xy_r, int n_r, const double* M, double errorTh,
                                         uint32_t* out_ij);

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

struct Mat2N
{
    std::vector<double> v;
    int cols() const { return (int)v.size() / 2; }
    double operator()(int r, int c) const { return v[2 * c + r]; }
};

static const int W = 1920, Hh = 1080;
static const double f = 1500, cx = 960, cy = 540;

int main()
{
    // a camera turning about its centre: every pair of views is related by a homography
    std::mt19937 g(5);
    std::uniform_real_distribution<double> ux(-0.9, 0.9), uy(-0.4, 0.4), un(-0.5, 0.5);
    const int NP = 1500, NV = 4;
    std::vector<std::array<double, 3>> X(NP);
    std::vector<std::array<unsigned char, 128>> base(NP);
    for (int p = 0; p < NP; ++p)
    {
        X[p] = {ux(g), uy(g), 1.0};
        for (auto& b : base[p])
            b = (unsigned char)(g() % 64);
    }
    const double yaw[NV] = {0.0, 0.08, -0.1, 0.15};
    std::vector<std::unique_ptr<SIFT_Regions>> regs(NV);
    std::vector<std::vector<int>> idx(NV, std::vector<int>(NP, -1));
    std::vector<std::vector<double>> pos(NV);
    for (int v = 0; v < NV; ++v)
    {
        regs[v].reset(new SIFT_Regions());
        const double c = std::cos(yaw[v]), s = std::sin(yaw[v]);
        for (int p = 0; p < NP; ++p)
        {
            const double x0 = c * X[p][0] + s * X[p][2], z = -s * X[p][0] + c * X[p][2];
            const double x = f * x0 / z + cx + un(g), y = f * X[p][1] / z + cy + un(g);
            if (z <= 0 || x < 0 || y < 0 || x >= W - 1 || y >= Hh - 1 || (g() % 4) == 0)
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
    // putatives: true correspondences and 30 % wrong ones; pair (0, 3) gets only 20 true ones (no strong support)
    const std::vector<Pair> pairs = {{0, 1}, {1, 2}, {0, 2}, {0, 3}, {2, 3}};
    std::map<Pair, MatchesPerDescType> put;
    for (const Pair& pr : pairs)
    {
        IndMatches& m = put[pr][EImageDescriberType::SIFT];
        for (int p = 0; p < NP; ++p)
            if (idx[pr.first][p] >= 0 && idx[pr.second][p] >= 0)
            {
                if (pr == Pair(0, 3) && m.size() >= 20)
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
    long kept = 0, guidedTotal = 0, compared = 0;
    for (const bool guided : {false, true})
    {
        GeometricFilterMatrix_H_AC_Batch_b200 batch;
        CHECK(batch.available());
        for (int v = 0; v < NV; ++v)
            CHECK(batch.addView(v, EImageDescriberType::SIFT, *regs[v]));
        std::vector<Mat2N> xI(pairs.size()), xJ(pairs.size());
        for (std::size_t k = 0; k < pairs.size(); ++k)
        {
            for (const IndMatch& m : put[pairs[k]][EImageDescriberType::SIFT])
            {
                xI[k].v.insert(xI[k].v.end(), {pos[pairs[k].first][2 * m._i], pos[pairs[k].first][2 * m._i + 1]});
                xJ[k].v.insert(xJ[k].v.end(), {pos[pairs[k].second][2 * m._j], pos[pairs[k].second][2 * m._j + 1]});
            }
            batch.addPair(pairs[k], put[pairs[k]], types, xI[k], xJ[k], {W, Hh}, {W, Hh});
        }
        PairwiseMatches out;
        CHECK(batch.run(rng, maxIt, std::numeric_limits<double>::infinity(), guided, -1.0, out));
        for (std::size_t k = 0; k < pairs.size(); ++k)
        {
            const Pair& pr = pairs[k];
            const auto& e = batch.estimate(k);
            const int n = (int)put[pr][EImageDescriberType::SIFT].size();
            std::vector<double> corr;
            for (int c = 0; c < n; ++c)
                corr.insert(corr.end(), {xI[k](0, c), xI[k](1, c), xJ[k](0, c), xJ[k](1, c)});
            int valid = 0, nInl = 0, nTr = 0;
            std::vector<uint32_t> inl(n + 1), sto(625);
            std::vector<int> tr(4096);
            std::vector<double> trn(4096);
            double Hm[9], em = 0, nfa = 0;
            acr_estimate_h(n, corr.data(), W, Hh, W, Hh, state, (long)maxIt, std::numeric_limits<double>::infinity(), &valid, &nInl, inl.data(), Hm,
                           &em, &nfa, tr.data(), trn.data(), 4096, &nTr, sto.data());
            CHECK(e.valid == (valid != 0));
            // where the engine's model is the oracle's up to rounding (H up to scale and errorMax within 1e-9), the decision and the
            // inliers are the oracle's
            double na = 0, nb = 0, dot = 0;
            for (int q = 0; q < 9; ++q)
            {
                na += Hm[q] * Hm[q];
                nb += e.H[q] * e.H[q];
                dot += Hm[q] * e.H[q];
            }
            if (valid && na > 0 && nb > 0 && 1 - std::fabs(dot) / std::sqrt(na * nb) <= 1e-12 && std::fabs(em - e.errorMax) <= 1e-9 * em)
            {
                ++compared;
                MatchesPerDescType want;
                matchingImageCollection::b200detail::copyInlierMatches(std::vector<std::size_t>(inl.begin(), inl.begin() + nInl), put[pr], types, want);
                const bool strong = matchingImageCollection::b200detail::hasStrongSupport(want, 4);
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
                // position-only guided matching and the reference's decorator, on the adaptor's own model and threshold
                const SIFT_Regions& L = *regs[pr.first];
                const SIFT_Regions& R = *regs[pr.second];
                std::vector<uint32_t> ij(2 * L.RegionCount() + 2);
                const int nw = gf_guided_match_positions(1, pos[pr.first].data(), (int)L.RegionCount(), pos[pr.second].data(), (int)R.RegionCount(), e.H,
                                                         e.errorMax * e.errorMax, ij.data());
                IndMatches want;
                for (int q = 0; q < nw; ++q)
                    want.emplace_back(ij[2 * q], ij[2 * q + 1]);
                IndMatchDecorator<float> deco(want, L.GetRegionsPositions(), R.GetRegionsPositions());
                deco.getDeduplicated(want);
                const IndMatches& m = out[pr][EImageDescriberType::SIFT];
                CHECK(m.size() == want.size());
                for (std::size_t q = 0; q < m.size() && q < want.size(); ++q)
                    CHECK(m[q]._i == want[q]._i && m[q]._j == want[q]._j);
                guidedTotal += (long)m.size();
            }
        }
    }
    CHECK(kept >= 3 && guidedTotal > 500 && compared >= 3);
    std::printf("%s: %ld kept pairs, %ld guided matches, %ld estimates equal to the oracle's\n", g_fail ? "FAILED" : "homography_filter adaptor ok",
                kept, guidedTotal, compared);
    return g_fail ? 1 : 0;
}

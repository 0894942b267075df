// Compiles alicevision_b200/adaptor/GeometricFilter_b200.hpp against the REFERENCE's own interface headers (through oracle/shim) and
// checks, on a GPU, GeometricFilterMatrix_F_AC_Batch_b200 with estimateDistortion (the fundamental_with_distortion filter) against
// the "ref" oracles: the reference's ACRANSAC loop around the restated F10 kernel (acrf10_estimate) from the same generator state,
// the inlier copy and hasStrongSupport(.., 10), and with guided matching the reference's guidedMatching loop (gf_guided_match,
// fundamental model) on the adaptor's own F and errorMax^2.
// Built by oracle/Makefile target `adaptors` into oracle/_ref/distortion_filter_test.
#include <aliceVision/feature/regionsFactory.hpp>

#include <GeometricFilter_b200.hpp>

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <map>
#include <memory>
#include <random>
#include <vector>

extern "C" long acrf10_estimate(int n, const double* corr, const int* wh, const uint32_t* state, long max_iter, double precision, int* valid,
                                int* n_inliers, uint32_t* inliers, double* F, double* L, double* error_max, double* min_nfa, int* trace,
                                double* trace_nfa, int trace_cap, int* n_trace, uint32_t* state_out);
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

struct Mat2N
{
    std::vector<double> v;
    int cols() const { return (int)v.size() / 2; }
    double operator()(int r, int c) const { return v[2 * c + r]; }
};

static const int W = 1920, Hh = 1080;
static const double K[9] = {1500, 0, 960, 0, 1500, 540, 0, 0, 1};

// division-model distortion about the image centre in preconditioned units s = 1 / sqrt(W H): u - c = (d - c) / (1 + lam |s (d - c)|^2)
static void distort(double& x, double& y, double lam)
{
    const double s = 1.0 / std::sqrt((double)W * Hh), ux = (x - W / 2.0) * s, uy = (y - Hh / 2.0) * s;
    double dx = ux, dy = uy;
    for (int it = 0; it < 100; ++it)
    {
        const double f = 1 + lam * (dx * dx + dy * dy);
        dx = ux * f;
        dy = uy * f;
    }
    x = dx / s + W / 2.0;
    y = dy / s + Hh / 2.0;
}

int main()
{
    // a camera sliding sideways past a cloud of points: every pair is calibrated with the same K and a real baseline
    std::mt19937 g(5);
    std::uniform_real_distribution<double> ux(-2.0, 2.0), uz(6.0, 10.0), un(-0.5, 0.5);
    const int NP = 1500, NV = 4;
    std::vector<std::array<double, 3>> X(NP);
    std::vector<std::array<unsigned char, 128>> base(NP);
    for (int p = 0; p < NP; ++p)
    {
        X[p] = {ux(g), 0.5 * ux(g), uz(g)};
        for (auto& b : base[p])
            b = (unsigned char)(g() % 64);
    }
    const double tx[NV] = {0.0, 0.3, 0.7, 1.2}, yaw[NV] = {0.0, 0.03, -0.04, 0.06};
    std::vector<std::unique_ptr<SIFT_Regions>> regs(NV);
    std::vector<std::vector<int>> idx(NV, std::vector<int>(NP, -1));
    std::vector<std::vector<double>> pos(NV);
    for (int v = 0; v < NV; ++v)
    {
        regs[v].reset(new SIFT_Regions());
        const double c = std::cos(yaw[v]), s = std::sin(yaw[v]);
        for (int p = 0; p < NP; ++p)
        {
            const double x0 = X[p][0] - tx[v], z0 = X[p][2];
            const double xr = c * x0 + s * z0, z = -s * x0 + c * z0;
            double x = K[0] * xr / z + K[2], y = K[4] * X[p][1] / z + K[5];
            distort(x, y, -0.2);
            x += un(g);
            y += un(g);
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
    // putatives: true correspondences and 30 % wrong ones; pair (0, 3) gets only 70 (0.14 x 70 = 9.8: below the 10-point threshold,
    // above the 7-point one)
    const std::vector<Pair> pairs = {{0, 1}, {1, 2}, {0, 2}, {0, 3}, {2, 3}};
    std::map<Pair, MatchesPerDescType> put;
    for (const Pair& pr : pairs)
    {
        IndMatches& m = put[pr][EImageDescriberType::SIFT];
        for (int p = 0; p < NP; ++p)
            if (idx[pr.first][p] >= 0 && idx[pr.second][p] >= 0)
            {
                if (pr == Pair(0, 3) && m.size() >= 70)
                    break;
                const bool wrong = g() % 10 < 3;
                m.emplace_back(idx[pr.first][p], wrong ? (IndexT)(g() % regs[pr.second]->RegionCount()) : (IndexT)idx[pr.second][p], 0.5f, 100.f + p);
            }
    }
    const std::vector<EImageDescriberType> types = {EImageDescriberType::SIFT};
    const std::size_t maxIt = 400;
    const double precision = std::numeric_limits<double>::infinity();   // featureMatching's default geometricErrorMax
    const std::mt19937 rng(42);
    std::stringstream ss;
    ss << rng;
    uint32_t state[625];
    for (auto& s : state)
        ss >> s;
    long kept = 0, guidedTotal = 0, compared = 0;
    for (const bool guided : {false, true})
    {
        GeometricFilterMatrix_F_AC_Batch_b200 batch(matching::b200detail::sharedContext(), true);
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
            batch.addPair(pairs[k], put[pairs[k]], types, xI[k], xJ[k], std::make_pair<std::size_t, std::size_t>(W, Hh),
                          std::make_pair<std::size_t, std::size_t>(W, Hh));
        }
        PairwiseMatches out;
        CHECK(batch.run(rng, maxIt, precision, guided, 0.6, out));
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
            double Fm[9], Lm[2], em = 0, nfa = 0;
            const int wh[4] = {W, Hh, W, Hh};
            acrf10_estimate(n, corr.data(), wh, state, (long)maxIt, precision, &valid, &nInl, inl.data(), Fm, Lm, &em, &nfa, tr.data(), trn.data(),
                            4096, &nTr, sto.data());
            // the engine is the port bit for bit, and the port the compiled reference loop: F, L, errorMax and the inliers are the oracle's
            CHECK(e.valid == (valid != 0));
            if (valid)
            {
                ++compared;
                CHECK(std::equal(Fm, Fm + 9, e.F) && std::equal(Lm, Lm + 2, e.L) && em == e.errorMax);
                MatchesPerDescType want;
                matchingImageCollection::b200detail::copyInlierMatches(std::vector<std::size_t>(inl.begin(), inl.begin() + nInl), put[pr], types, want);
                const bool strong = matchingImageCollection::b200detail::hasStrongSupport(want, 10);
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
                CHECK(e.valid && !e.strongSupport && out.count(pr) == 0);
            if (!out.count(pr))
                continue;
            kept += !guided;
            if (guided)
            {
                const double* F = e.F;   // the model matrix, read as x_J^T F x_I as the reference's guided step reads it
                const SIFT_Regions& L = *regs[pr.first];
                const SIFT_Regions& R = *regs[pr.second];
                std::vector<uint32_t> ij(2 * L.RegionCount() + 2);
                const int nw = gf_guided_match(1, 0, L.DescriptorRawData(), pos[pr.first].data(), (int)L.RegionCount(), R.DescriptorRawData(),
                                               pos[pr.second].data(), (int)R.RegionCount(), F, e.errorMax * e.errorMax, 0.36, ij.data());
                const IndMatches& m = out[pr][EImageDescriberType::SIFT];
                CHECK((int)m.size() == nw);
                for (int q = 0; q < nw && q < (int)m.size(); ++q)
                    CHECK(m[q]._i == ij[2 * q] && m[q]._j == ij[2 * q + 1]);
                guidedTotal += (long)m.size();
            }
        }
    }
    CHECK(kept >= 3 && guidedTotal > 500 && compared >= 4);
    std::printf("%s: %ld kept pairs, %ld guided matches, %ld estimates equal to the oracle's\n", g_fail ? "FAILED" : "distortion_filter adaptor ok",
                kept, guidedTotal, compared);
    return g_fail ? 1 : 0;
}

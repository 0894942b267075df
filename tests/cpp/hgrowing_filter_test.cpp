// Compiles alicevision_b200/adaptor/GeometricFilter_b200.hpp against the REFERENCE's own interface headers (through oracle/shim) and
// checks, on a GPU, GeometricFilterMatrix_HGrowing_Batch_b200 against the single-threaded port of filterMatchesByHGrowing
// (oracle/libport_hgrowing.so, hg_filter) on the same putatives: every (pair, type)'s homographies bit for bit, their matches, the
// kept lists, and the stage rules (an empty filtered list is kept, a type without putatives is skipped, a pair without a common type
// gets nothing, guidedMatching gives an empty map).
// Built by oracle/Makefile target `adaptors` into oracle/_ref/hgrowing_filter_test.
#include <aliceVision/feature/regionsFactory.hpp>

#include <GeometricFilter_b200.hpp>

#include <array>
#include <cmath>
#include <cstdio>
#include <map>
#include <random>
#include <vector>

extern "C" int hg_filter(int n, const float* feat, const double* tols, const int32_t* ints, int32_t* n_h, double* H, int32_t* counts,
                         int32_t* inliers, int32_t* trace, int32_t* rounds, int64_t* stats);

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

using M3 = std::array<double, 9>;

static void apply(const M3& H, double x, double y, double& u, double& v, double A[4])
{
    const double w = H[6] * x + H[7] * y + H[8];
    const double a = H[0] * x + H[1] * y + H[2], b = H[3] * x + H[4] * y + H[5];
    u = a / w;
    v = b / w;
    A[0] = (H[0] * w - a * H[6]) / (w * w); A[1] = (H[1] * w - a * H[7]) / (w * w);
    A[2] = (H[3] * w - b * H[6]) / (w * w); A[3] = (H[4] * w - b * H[7]) / (w * w);
}

int main()
{
    // three views of a scene with two planes: view 0 holds the points, views 1 and 2 map each plane by its own homography; every
    // feature's scale and orientation follow the plane's local affinity; 30 % of the features of views 1 and 2 are outliers
    std::mt19937 g(7);
    std::uniform_real_distribution<double> ux(0, 2000), us(1.5, 8), uo(-M_PI, M_PI), u01(0, 1);
    const int NP = 600, NV = 3;
    const M3 Hp[2][NV] = {{{1, 0, 0, 0, 1, 0, 0, 0, 1}, {0.98, -0.12, 40, 0.11, 0.97, -30, 2e-5, -1e-5, 1}, {1.05, 0.2, -80, -0.18, 1.02, 60, -3e-5, 2e-5, 1}},
                          {{1, 0, 0, 0, 1, 0, 0, 0, 1}, {0.9, 0.05, 150, -0.06, 0.93, 20, 4e-5, 3e-5, 1}, {1.1, -0.1, -20, 0.12, 1.08, -90, -2e-5, -4e-5, 1}}};
    std::vector<std::vector<PointFeature>> feats(NV, std::vector<PointFeature>(NP));
    for (int p = 0; p < NP; ++p)
    {
        const int plane = p % 2;
        const double x = ux(g), y = ux(g), s = us(g), o = uo(g);
        feats[0][p] = PointFeature((float)x, (float)y, (float)s, (float)o);
        for (int v = 1; v < NV; ++v)
        {
            if (u01(g) < 0.3)
            {
                feats[v][p] = PointFeature((float)ux(g), (float)ux(g), (float)us(g), (float)uo(g));
                continue;
            }
            double u, w, A[4];
            apply(Hp[plane][v], x, y, u, w, A);
            const double c = s * std::cos(o), sn = s * std::sin(o);
            const double F[4] = {A[0] * c + A[1] * sn, -A[0] * sn + A[1] * c, A[2] * c + A[3] * sn, -A[2] * sn + A[3] * c};
            feats[v][p] = PointFeature((float)u, (float)w, (float)std::sqrt(std::fabs(F[0] * F[3] - F[1] * F[2])),
                                       (float)std::atan2(F[2] - F[1], F[0] + F[3]));
        }
    }
    const EImageDescriberType SIFT = EImageDescriberType::SIFT, AKAZE = EImageDescriberType::AKAZE;
    std::vector<PointFeature> few(10, PointFeature(1, 2, 3, 0.5f));
    auto featuresOf = [&](IndexT view, EImageDescriberType t) -> const std::vector<PointFeature>& { return t == AKAZE ? few : feats[view]; };

    // putatives i <-> i in a shuffled order, per pair
    std::map<Pair, MatchesPerDescType> putatives;
    for (int a = 0; a < NV; ++a)
        for (int b = a + 1; b < NV; ++b)
        {
            IndMatches m;
            for (int p = 0; p < NP; ++p)
                m.emplace_back(p, p);
            std::shuffle(m.begin(), m.end(), g);
            putatives[Pair(a, b)][SIFT] = m;
        }
    putatives[Pair(0, 1)][AKAZE] = IndMatches{IndMatch(0, 1), IndMatch(2, 3)};   // too few: filtered, empty, kept
    const std::vector<EImageDescriberType> both = {SIFT, AKAZE}, siftOnly = {SIFT};

    const double tols[3] = {20, 10, 5};
    const int32_t ints[4] = {6, 8, 10, 20};
    auto port = [&](const IndMatches& m, IndexT i, IndexT j, EImageDescriberType t, std::vector<M3>& Hs, std::vector<IndMatches>& sets) {
        std::vector<float> f;
        for (const IndMatch& x : m)
        {
            const PointFeature &a = featuresOf(i, t).at(x._i), &b = featuresOf(j, t).at(x._j);
            for (float v : {a.x(), a.y(), a.scale(), a.orientation(), b.x(), b.y(), b.scale(), b.orientation()})
                f.push_back(v);
        }
        int32_t nh = 0, rounds = 0, counts[10], trace[30];
        double H[90];
        std::vector<int32_t> inl(m.size() + 1);
        int64_t stats[2] = {0, 0};
        hg_filter((int)m.size(), f.data(), tols, ints, &nh, H, counts, inl.data(), trace, &rounds, stats);
        int at = 0;
        for (int h = 0; h < nh; ++h)
        {
            M3 M;
            std::copy(H + 9 * h, H + 9 * h + 9, M.begin());
            Hs.push_back(M);
            IndMatches s;
            for (int q = 0; q < counts[h]; ++q)
                s.push_back(m[inl[at++]]);
            sets.push_back(s);
        }
    };

    for (const bool guided : {false, true})
    {
        GeometricFilterMatrix_HGrowing_Batch_b200 batch;
        CHECK(batch.available());
        for (const auto& p : putatives)
            batch.addPair(p.first, p.second, p.first == Pair(0, 1) ? both : siftOnly, featuresOf);
        batch.addPair(Pair(5, 6), MatchesPerDescType(), {}, featuresOf);   // no common type: no estimation
        PairwiseMatches out;
        CHECK(batch.run(guided, out));
        CHECK(out.size() == 3 && !out.count(Pair(5, 6)));
        int stored = 0;
        for (const auto& p : putatives)
            for (const auto& t : p.second)
            {
                std::vector<M3> Hs;
                std::vector<IndMatches> sets;
                port(t.second, p.first.first, p.first.second, t.first, Hs, sets);
                const auto& hs = batch.homographies(p.first, t.first);
                CHECK(hs.size() == Hs.size());
                IndMatches all;
                for (std::size_t h = 0; h < std::min(hs.size(), Hs.size()); ++h)
                {
                    CHECK(hs[h].first == Hs[h]);
                    CHECK(hs[h].second == sets[h]);
                    all.insert(all.end(), sets[h].begin(), sets[h].end());
                }
                stored += (int)Hs.size();
                if (guided)
                    CHECK(out.at(p.first).empty());
                else
                    CHECK(out.at(p.first).count(t.first) && out.at(p.first).at(t.first) == all);
            }
        CHECK(out.at(Pair(0, 1)).count(AKAZE) == (guided ? 0u : 1u));
        CHECK(stored >= 3);   // at least one plane in each of the three pairs
        std::printf("guided=%d: %d homographies\n", (int)guided, stored);
    }
    if (g_fail)
    {
        std::printf("%d checks failed\n", g_fail);
        return 1;
    }
    std::printf("hgrowing_filter adaptor ok\n");
    return 0;
}

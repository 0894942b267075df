// Compiles the C++ adaptors against the REFERENCE's own interface headers (through oracle/shim) and checks, on a GPU,
// that ArrayMatcher_b200 / ImageCollectionMatcher_b200 return exactly what the reference classes return on the same
// Regions.  Built by oracle/Makefile target `adaptors` into oracle/_ref/adaptor_test (needs an AliceVision source tree at build time).
#include <aliceVision/matching/ArrayMatcher_bruteForce.hpp>
#include <aliceVision/matching/RegionsMatcher.hpp>
#include <aliceVision/feature/regionsFactory.hpp>

#include <ArrayMatcher_b200.hpp>
#include <ImageCollectionMatcher_b200.hpp>
#include <RegionsMatcher_b200.hpp>
#include <guidedMatching_b200.hpp>

// oracle/_ref/libref_oracle.so: guided-matching loop restated around the reference's Regions::SquaredDescriptorDistance
extern "C" int ref_guided_match(int dtype, int model, const void* desc_l, const float* xy_l, int n_l, const void* desc_r, const float* xy_r, int n_r, const double* F,
                                double errorTh, double distRatio, uint32_t* out_ij);
struct Mat3Lite { double v[9]; double operator()(int r, int c) const { return v[3 * r + c]; } };

#include <cstdio>
#include <memory>
#include <random>

using namespace aliceVision;
using namespace aliceVision::matching;
using namespace aliceVision::feature;

static int g_fail = 0;
#define CHECK(c)                                                     \
    do                                                               \
    {                                                                \
        if (!(c))                                                    \
        {                                                            \
            std::printf("CHECK FAILED %s:%d  %s\n", __FILE__, __LINE__, #c); \
            ++g_fail;                                                \
        }                                                            \
    } while (0)

template<class RegionsT, class T>
RegionsT* makeRegions(int n, unsigned seed, int lo, int hi, const RegionsT* plantFrom)
{
    std::mt19937 g(seed);
    auto* r = new RegionsT();
    std::vector<int> px(n), py(n);
    for (int i = 0; i < n; ++i) { px[i] = i; py[i] = i; }
    std::shuffle(px.begin(), px.end(), g);
    std::shuffle(py.begin(), py.end(), g);
    for (int i = 0; i < n; ++i)
    {
        r->Features().emplace_back(px[i] + 0.25f, py[i] + 0.5f, 1.f, 0.f);
        typename RegionsT::DescriptorT d;
        for (int k = 0; k < (int)RegionsT::DescriptorT::static_size; ++k)
        {
            int v = lo + int(g() % unsigned(hi - lo + 1));
            if (plantFrom && i < n / 3)
                v = std::min(hi, std::max(lo, int((*plantFrom).Descriptors()[i * 2 % n][k]) + int(g() % 5) - 2));
            d[k] = T(v);
        }
        r->Descriptors().push_back(d);
    }
    return r;
}

// Stand-in for the reference's ImageCollectionMatcher_generic (its .cpp needs FLANN / Boost, absent here) as the FALLBACK of the
// collection adaptor: the same pair loop around the reference's own RegionsMatcher<ArrayMatcher_bruteForce> (forward pairs only).
class RefLoopMatcher : public matchingImageCollection::IImageCollectionMatcher
{
  public:
    mutable int calls = 0;
    void Match(std::mt19937& rng, const RegionsPerView& rpv, const PairSet& pairs, EImageDescriberType descType, PairwiseMatches& out) const override
    {
        ++calls;
        for (const Pair& p : pairs)
        {
            const Regions& ri = rpv.getRegions(p.first, descType);
            const Regions& rj = rpv.getRegions(p.second, descType);
            if (ri.RegionCount() == 0 || rj.RegionCount() == 0) continue;
            RegionsMatcher<ArrayMatcher_bruteForce<unsigned char, L2_Vectorized<unsigned char>>> fw(rng, ri, true);
            IndMatches v; fw.Match(0.8f, rj, v);
            if (!v.empty()) out[p].emplace(descType, v);
        }
    }
};

int main()
{
    if (b200m_device_count() < 1)
    {
        std::printf("SKIP: no CUDA device\n");
        return 0;
    }
    std::mt19937 rng;
    // --- matching_test.cpp:40-71 on the adaptor (default metric L2_Simple)
    {
        const float array[] = {0, 1, 2, 5, 6};
        ArrayMatcher_b200<float> m;
        CHECK(m.Build(rng, array, 5, 1));
        const float query[] = {2};
        IndMatches idx; std::vector<float> d;
        CHECK(m.SearchNeighbours(query, 1, &idx, &d, 5));
        CHECK(idx.size() == 5 && d.size() == 5);
        const float wantD[] = {0, 1, 4, 9, 16}; const unsigned wantI[] = {2, 1, 0, 3, 4};
        for (int k = 0; k < 5; ++k) CHECK(d[k] == wantD[k] && idx[k]._i == 0 && idx[k]._j == wantI[k]);
        int ni = -1; float fd = -1;
        CHECK(m.SearchNeighbour(query, &ni, &fd) && ni == 2 && fd == 0.f);
        ArrayMatcher_b200<float> e;
        CHECK(!e.Build(rng, array, 0, 4));
        CHECK(!e.SearchNeighbour(query, &ni, &fd));
    }
    // --- raw top-2: adaptor vs ArrayMatcher_bruteForce on SIFT-like uchar and float
    SIFT_Regions* a = makeRegions<SIFT_Regions, unsigned char>(1500, 1, 0, 90, nullptr);
    SIFT_Regions* b = makeRegions<SIFT_Regions, unsigned char>(1300, 2, 0, 90, a);
    {
        typedef L2_Vectorized<unsigned char> M;
        ArrayMatcher_bruteForce<unsigned char, M> ref; ArrayMatcher_b200<unsigned char, M> gpu;
        const unsigned char* A = reinterpret_cast<const unsigned char*>(a->DescriptorRawData());
        const unsigned char* B = reinterpret_cast<const unsigned char*>(b->DescriptorRawData());
        CHECK(ref.Build(rng, A, 1500, 128) && gpu.Build(rng, A, 1500, 128));
        IndMatches ir, ig; std::vector<float> dr, dg;
        CHECK(ref.SearchNeighbours(B, 1300, &ir, &dr, 2) && gpu.SearchNeighbours(B, 1300, &ig, &dg, 2));
        CHECK(dr == dg);
        for (size_t q = 0; q < 1300; ++q)
            if (dr[2 * q] < dr[2 * q + 1]) CHECK(ir[2 * q]._j == ig[2 * q]._j);
    }
    // --- the reference's own RegionsMatcher template instantiated on the adaptor (what createRegionsMatcher would build,
    //     matching/RegionsMatcher.cpp:74-79) must give the same IndMatches as on ArrayMatcher_bruteForce
    {
        typedef L2_Vectorized<unsigned char> M;
        RegionsMatcher<ArrayMatcher_bruteForce<unsigned char, M>> ref(rng, *a, true);
        RegionsMatcher<ArrayMatcher_b200<unsigned char, M>> gpu(rng, *a, true);
        IndMatches vr, vg;
        const bool okr = ref.Match(0.8f, *b, vr), okg = gpu.Match(0.8f, *b, vg);
        CHECK(okr == okg && vr.size() == vg.size() && !vr.empty());
        for (size_t k = 0; k < std::min(vr.size(), vg.size()); ++k)
            CHECK(vr[k]._i == vg[k]._i && vr[k]._j == vg[k]._j && vr[k]._distanceRatio == vg[k]._distanceRatio && vr[k]._distance == vg[k]._distance);
        std::printf("RegionsMatcher<ArrayMatcher_b200>: %zu matches compared\n", vr.size());
    }
    // --- full collection Match: adaptor vs RegionsMatcher (reference) incl. cross matching
    SIFT_Regions* c = makeRegions<SIFT_Regions, unsigned char>(900, 3, 0, 90, a);
    RegionsPerView rpv;
    rpv.addRegions(10, EImageDescriberType::SIFT, a);
    rpv.addRegions(11, EImageDescriberType::SIFT, b);
    rpv.addRegions(12, EImageDescriberType::SIFT, c);
    rpv.addRegions(13, EImageDescriberType::SIFT, new SIFT_Regions());
    PairSet pairs = {{10, 11}, {10, 12}, {11, 12}, {10, 13}};
    for (int cross = 0; cross < 2; ++cross)
    {
        matchingImageCollection::ImageCollectionMatcher_b200 gpu(0.8f, cross != 0);
        PairwiseMatches got;
        gpu.Match(rng, rpv, pairs, EImageDescriberType::SIFT, got);
        PairwiseMatches want;
        for (const Pair& p : pairs)
        {
            const Regions& ri = rpv.getRegions(p.first, EImageDescriberType::SIFT);
            const Regions& rj = rpv.getRegions(p.second, EImageDescriberType::SIFT);
            if (ri.RegionCount() == 0 || rj.RegionCount() == 0) continue;
            typedef ArrayMatcher_bruteForce<unsigned char, L2_Vectorized<unsigned char>> MatcherT;
            RegionsMatcher<MatcherT> fw(rng, ri, true);
            IndMatches v; fw.Match(0.8f, rj, v);
            if (cross)
            {
                RegionsMatcher<MatcherT> bw(rng, rj, true);
                IndMatches vc; bw.Match(0.8f, ri, vc);
                std::set<std::pair<IndexT, IndexT>> chk;
                for (auto& m : vc) chk.insert({m._i, m._j});
                IndMatches kept;
                for (auto& m : v) if (chk.count({m._j, m._i})) kept.push_back(m);
                v.swap(kept);
            }
            if (!v.empty()) want[p].emplace(EImageDescriberType::SIFT, v);
        }
        CHECK(got.size() == want.size());
        for (auto& kv : want)
        {
            auto it = got.find(kv.first);
            CHECK(it != got.end());
            if (it == got.end()) continue;
            const IndMatches& w = kv.second.at(EImageDescriberType::SIFT);
            const IndMatches& g = it->second.at(EImageDescriberType::SIFT);
            CHECK(w.size() == g.size());
            for (size_t k = 0; k < std::min(w.size(), g.size()); ++k)
                CHECK(w[k]._i == g[k]._i && w[k]._j == g[k]._j && w[k]._distanceRatio == g[k]._distanceRatio && w[k]._distance == g[k]._distance);
        }
        std::printf("collection cross=%d: %zu pairs compared\n", cross, want.size());
        // the same call sharded over two engine contexts inside this process (b200m_multi_match; both on device 0 here)
        matchingImageCollection::ImageCollectionMatcher_b200 multi(0.8f, cross != 0, false, std::vector<int>{0, 0});
        PairwiseMatches got2;
        multi.Match(rng, rpv, pairs, EImageDescriberType::SIFT, got2);
        CHECK(got2.size() == got.size());
        for (auto& kv : got)
        {
            auto it = got2.find(kv.first);
            CHECK(it != got2.end());
            if (it == got2.end()) continue;
            const IndMatches& w = kv.second.at(EImageDescriberType::SIFT);
            const IndMatches& g = it->second.at(EImageDescriberType::SIFT);
            CHECK(w.size() == g.size());
            for (size_t k = 0; k < std::min(w.size(), g.size()); ++k)
                CHECK(w[k]._i == g[k]._i && w[k]._j == g[k]._j && w[k]._distanceRatio == g[k]._distanceRatio && w[k]._distance == g[k]._distance);
        }
    }
    // --- error convention (SURVEY 8b): an engine that cannot be created, or that fails in Match, delegates to the fallback matcher
    //     (the integration passes ImageCollectionMatcher_generic) instead of aborting featureMatching; without a fallback it throws
    {
        auto fb = std::make_shared<RefLoopMatcher>();
        matchingImageCollection::ImageCollectionMatcher_b200 broken(0.8f, false, false, /*device=*/99, fb);   // no such device
        CHECK(broken.usesFallbackOnly());
        PairwiseMatches got, want;
        broken.Match(rng, rpv, pairs, EImageDescriberType::SIFT, got);
        RefLoopMatcher().Match(rng, rpv, pairs, EImageDescriberType::SIFT, want);
        CHECK(fb->calls == 1 && got.size() == want.size() && !want.empty());
        for (auto& kv : want)
        {
            auto it = got.find(kv.first);
            CHECK(it != got.end());
            if (it == got.end()) continue;
            const IndMatches& w = kv.second.at(EImageDescriberType::SIFT);
            const IndMatches& g = it->second.at(EImageDescriberType::SIFT);
            CHECK(w.size() == g.size());
            for (size_t k = 0; k < std::min(w.size(), g.size()); ++k) CHECK(w[k]._i == g[k]._i && w[k]._j == g[k]._j);
        }
        bool threw = false;
        try { matchingImageCollection::ImageCollectionMatcher_b200 nofb(0.8f, false, false, /*device=*/99); } catch (const std::runtime_error&) { threw = true; }
        CHECK(threw);
        // a working engine never touches the fallback, and gives the same lists
        auto fb2 = std::make_shared<RefLoopMatcher>();
        matchingImageCollection::ImageCollectionMatcher_b200 ok(0.8f, false, false, 0, fb2);
        PairwiseMatches got2;
        ok.Match(rng, rpv, pairs, EImageDescriberType::SIFT, got2);
        CHECK(!ok.usesFallbackOnly() && fb2->calls == 0 && got2.size() == want.size());
        std::printf("fallback matcher: %zu pairs through the fallback, engine path untouched by it\n", want.size());
    }
    // --- IRegionsMatcher adaptor (what createRegionsMatcher returns for the new enum values) vs the reference's
    //     RegionsMatcher<ArrayMatcher_bruteForce<...>>: one database, several queries, uchar / float / binary, factory rules
    {
        typedef ArrayMatcher_bruteForce<unsigned char, L2_Vectorized<unsigned char>> MatcherT;
        RegionsMatcher<MatcherT> ref(rng, *a, true);
        std::unique_ptr<IRegionsMatcher> gpu = createRegionsMatcher_b200(rng, *a, false);
        CHECK(gpu != nullptr);
        CHECK(createRegionsMatcher_b200(rng, *a, true) == nullptr);   // scalar regions + Hamming matcher: RegionsMatcher.cpp:61-62
        size_t compared = 0;
        for (const SIFT_Regions* q : {b, c})
        {
            IndMatches vr, vg;
            const bool okr = ref.Match(0.8f, *q, vr), okg = gpu && gpu->Match(0.8f, *q, vg);
            CHECK(okr == okg && vr.size() == vg.size() && !vr.empty());
            for (size_t k = 0; k < std::min(vr.size(), vg.size()); ++k)
                CHECK(vr[k]._i == vg[k]._i && vr[k]._j == vg[k]._j && vr[k]._distanceRatio == vg[k]._distanceRatio && vr[k]._distance == vg[k]._distance);
            compared += vr.size();
        }
        SIFT_Regions empty;
        IndMatches ve;
        CHECK(gpu && !gpu->Match(0.8f, empty, ve) && ve.empty());
        std::unique_ptr<IRegionsMatcher> gpuEmptyDb = createRegionsMatcher_b200(rng, empty, false);
        CHECK(gpuEmptyDb && !gpuEmptyDb->Match(0.8f, *b, ve) && ve.empty());
        CHECK(gpu && &gpu->getDatabaseRegions() == static_cast<const Regions*>(a));
        // float descriptors (integer-valued: tensor-core path)
        SIFT_Float_Regions* fa = makeRegions<SIFT_Float_Regions, float>(1100, 5, 0, 120, nullptr);
        SIFT_Float_Regions* fb = makeRegions<SIFT_Float_Regions, float>(1000, 6, 0, 120, fa);
        {
            RegionsMatcher<ArrayMatcher_bruteForce<float, L2_Vectorized<float>>> rf(rng, *fa, true);
            RegionsMatcher_b200 gf(rng, *fa);
            IndMatches vr, vg;
            CHECK(rf.Match(0.8f, *fb, vr) == gf.Match(0.8f, *fb, vg) && vr.size() == vg.size() && !vr.empty());
            for (size_t k = 0; k < std::min(vr.size(), vg.size()); ++k)
                CHECK(vr[k]._i == vg[k]._i && vr[k]._j == vg[k]._j && vr[k]._distanceRatio == vg[k]._distanceRatio && vr[k]._distance == vg[k]._distance);
            compared += vr.size();
            IndMatches vm;
            CHECK(!gf.Match(0.8f, *b, vm) && vm.empty());              // element type differs from the database's
        }
        // binary descriptors (Hamming, ratio not squared)
        AKAZE_BinaryRegions* ba = makeRegions<AKAZE_BinaryRegions, unsigned char>(900, 7, 0, 255, nullptr);
        AKAZE_BinaryRegions* bb = makeRegions<AKAZE_BinaryRegions, unsigned char>(800, 8, 0, 255, ba);
        {
            RegionsMatcher<ArrayMatcher_bruteForce<unsigned char, Hamming<unsigned char>>> rh(rng, *ba, false);
            std::unique_ptr<IRegionsMatcher> gh = createRegionsMatcher_b200(rng, *ba, true);
            CHECK(gh != nullptr && createRegionsMatcher_b200(rng, *ba, false) == nullptr);
            IndMatches vr, vg;
            const bool okr = rh.Match(0.8f, *bb, vr), okg = gh && gh->Match(0.8f, *bb, vg);
            CHECK(okr == okg && vr.size() == vg.size());
            for (size_t k = 0; k < std::min(vr.size(), vg.size()); ++k)
                CHECK(vr[k]._i == vg[k]._i && vr[k]._j == vg[k]._j && vr[k]._distanceRatio == vg[k]._distanceRatio && vr[k]._distance == vg[k]._distance);
            compared += vr.size();
        }
        delete fa; delete fb; delete ba; delete bb;
        std::printf("RegionsMatcher_b200 (IRegionsMatcher): %zu matches compared\n", compared);
    }
    // --- guided matching adaptor (step after the path) vs the oracle loop on the same Regions
    {
        const Mat3Lite F{{0, 0, 0, 0, 0, -1, 0, 1, 0}};                  // rectified pair: the epipolar error is (y_r - y_l)^2
        std::vector<float> xl, xr;
        for (const auto& f : a->Features()) { xl.push_back(f.x()); xl.push_back(f.y()); }
        for (const auto& f : b->Features()) { xr.push_back(f.x()); xr.push_back(f.y()); }
        std::vector<uint32_t> want(2 * a->RegionCount());
        const int nw = ref_guided_match(1, 0, a->DescriptorRawData(), xl.data(), (int)a->RegionCount(), b->DescriptorRawData(), xr.data(), (int)b->RegionCount(), F.v,
                                        400.0, 0.81, want.data());
        IndMatches got;
        CHECK(guidedMatchingFundamental_b200(F, *a, *b, 400.0, 0.81, got));
        CHECK(nw > 0 && (int)got.size() == nw);
        for (int k = 0; k < std::min(nw, (int)got.size()); ++k) CHECK(got[k]._i == want[2 * k] && got[k]._j == want[2 * k + 1]);
        std::printf("guidedMatchingFundamental_b200: %d matches compared\n", nw);
    }
    std::printf(g_fail ? "ADAPTOR TEST FAILED (%d)\n" : "ADAPTOR TEST PASSED\n", g_fail);
    return g_fail ? 1 : 0;
}

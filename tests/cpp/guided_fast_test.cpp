// Compiles alicevision_b200/adaptor/guidedMatchingFast_b200.hpp against the REFERENCE's own interface headers (through oracle/shim)
// and checks, on a GPU, that GuidedMatchingFastBatch_b200 and guidedMatchingFundamentalFast_b200 return exactly what the "ref"
// oracle (guidedMatchingFundamentalFast restated around the reference's Regions::SquaredDescriptorDistance) returns.
// Built by oracle/guided_fast.mk target `adaptor` into oracle/_ref/guided_fast_adaptor_test.
#include <aliceVision/feature/regionsFactory.hpp>

#include <guidedMatchingFast_b200.hpp>

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <map>
#include <memory>
#include <random>
#include <vector>

extern "C" int gf_guided_fast(int dtype, const void* desc_l, const double* xy_l, int n_l, const void* desc_r, const double* xy_r, int n_r,
                              const double* FMat, const double* epipole2, int widthR, int heightR, double errorTh, double distRatio, uint32_t* out_ij);

using namespace aliceVision;
using namespace aliceVision::matching;
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

struct M3 { double v[9]; double operator()(int r, int c) const { return v[3 * r + c]; } };
struct V3 { double v[3]; double operator()(int k) const { return v[k]; } };

static const int W = 4000, H = 3000;
static const double f = 3600, cx = 2000, cy = 1500;

static double det4(const double m[4][4])
{
    double d = 0;
    for (int c = 0; c < 4; ++c)
    {
        double s[3][3];
        for (int r = 1; r < 4; ++r)
            for (int k = 0, kk = 0; k < 4; ++k)
                if (k != c)
                    s[r - 1][kk++] = m[r][k];
        const double minor = s[0][0] * (s[1][1] * s[2][2] - s[1][2] * s[2][1]) - s[0][1] * (s[1][0] * s[2][2] - s[1][2] * s[2][0]) +
                             s[0][2] * (s[1][0] * s[2][1] - s[1][1] * s[2][0]);
        d += (c % 2 ? -1 : 1) * m[0][c] * minor;
    }
    return d;
}

// camera k: P_k = K [I | -C_k]; F = F_from_P(P_L, P_R) (numeric/projection.cpp:115-143: determinants of stacked row pairs, which
// fix the sign of F relative to the epipole), epipole2 = P_R (C_L, 1) (epipole_from_P)
static void geometry(const double CL[3], const double CR[3], M3& F, V3& e)
{
    double PL[3][4], PR[3][4];
    const double K[3][3] = {{f, 0, cx}, {0, f, cy}, {0, 0, 1}};
    for (int r = 0; r < 3; ++r)
    {
        for (int c = 0; c < 3; ++c)
            PL[r][c] = PR[r][c] = K[r][c];
        PL[r][3] = -(K[r][0] * CL[0] + K[r][1] * CL[1] + K[r][2] * CL[2]);
        PR[r][3] = -(K[r][0] * CR[0] + K[r][1] * CR[1] + K[r][2] * CR[2]);
    }
    const int rows[3][2] = {{1, 2}, {2, 0}, {0, 1}};
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c)
        {
            double m[4][4];
            for (int k = 0; k < 4; ++k)
            {
                m[0][k] = PL[rows[c][0]][k];
                m[1][k] = PL[rows[c][1]][k];
                m[2][k] = PR[rows[r][0]][k];
                m[3][k] = PR[rows[r][1]][k];
            }
            F.v[3 * r + c] = det4(m);
        }
    for (int r = 0; r < 3; ++r)
        e.v[r] = PR[r][0] * CL[0] + PR[r][1] * CL[1] + PR[r][2] * CL[2] + PR[r][3];
}

int main()
{
    std::mt19937 g(7);
    std::uniform_real_distribution<double> ux(-3, 3), uy(-2, 2), uz(8, 12), un(-0.6, 0.6);
    const int NP = 3000, NV = 3;
    std::vector<std::array<double, 3>> X(NP);
    std::vector<std::array<unsigned char, 128>> base(NP);
    for (int p = 0; p < NP; ++p)
    {
        X[p] = {ux(g), uy(g), uz(g)};
        for (auto& b : base[p])
            b = (unsigned char)(g() % 64);
    }
    const double C[NV][3] = {{0, 0, 0}, {1.2, 0.1, 0.3}, {-0.8, -0.15, -0.4}};
    std::vector<std::unique_ptr<SIFT_Regions>> regs(NV);
    std::vector<std::vector<double>> pos(NV);     // what the oracle sees: geometry positions where given, else the float positions
    std::vector<std::vector<double>> geo(NV);
    for (int v = 0; v < NV; ++v)
    {
        regs[v].reset(new SIFT_Regions());
        for (int p = 0; p < NP; ++p)
        {
            const double x = f * (X[p][0] - C[v][0]) / (X[p][2] - C[v][2]) + cx + un(g), y = f * (X[p][1] - C[v][1]) / (X[p][2] - C[v][2]) + cy + un(g);
            if (x < 0 || y < 0 || x >= W - 1 || y >= H - 1 || (g() % 3) == 0)
                continue;
            regs[v]->Features().emplace_back((float)x, (float)y, 1.f, 0.f);
            SIFT_Regions::DescriptorT d;
            for (int k = 0; k < 128; ++k)
                d[k] = (unsigned char)std::min(255, (int)base[p][k] + (int)(g() % 5));
            regs[v]->Descriptors().push_back(d);
            geo[v].push_back(x);
            geo[v].push_back(y);
        }
        for (const auto& ft : regs[v]->Features())
        {
            pos[v].push_back((double)ft.x());
            pos[v].push_back((double)ft.y());
        }
    }
    // view 1 gets geometry positions (the unrounded doubles)
    pos[1] = geo[1];
    const std::pair<IndexT, IndexT> pairs[] = {{0, 1}, {1, 2}, {0, 2}, {2, 0}, {1, 0}};
    const double errorTh = 16.0, distRatio = 0.64;
    std::map<std::pair<IndexT, IndexT>, IndMatches> got;
    {
        GuidedMatchingFastBatch_b200 batch;
        CHECK(batch.available());
        for (int v = 0; v < NV; ++v)
            CHECK(batch.addView(v, *regs[v], v == 1 ? geo[1].data() : nullptr));
        for (const auto& p : pairs)
        {
            M3 F; V3 e;
            geometry(C[p.first], C[p.second], F, e);
            batch.addPair(p.first, p.second, F, e, W, H);
        }
        CHECK(batch.run(errorTh, distRatio, got));
    }
    CHECK(got.size() == 5);
    long total = 0;
    for (const auto& p : pairs)
    {
        M3 F; V3 e;
        geometry(C[p.first], C[p.second], F, e);
        const SIFT_Regions& L = *regs[p.first];
        const SIFT_Regions& R = *regs[p.second];
        std::vector<uint32_t> want(2 * L.RegionCount() + 2);
        const int n = gf_guided_fast(1, L.DescriptorRawData(), pos[p.first].data(), (int)L.RegionCount(), R.DescriptorRawData(), pos[p.second].data(),
                                     (int)R.RegionCount(), F.v, e.v, W, H, errorTh, distRatio, want.data());
        const IndMatches& m = got[p];
        CHECK((int)m.size() == n);
        for (int k = 0; k < n && k < (int)m.size(); ++k)
            CHECK(m[k]._i == want[2 * k] && m[k]._j == want[2 * k + 1]);
        total += n;
        // the one-pair form, with the same positions
        IndMatches one;
        CHECK(guidedMatchingFundamentalFast_b200(F, e, L, R, W, H, errorTh, distRatio, one, p.first == 1 ? geo[1].data() : nullptr,
                                                 p.second == 1 ? geo[1].data() : nullptr));
        CHECK(one.size() == m.size());
        for (std::size_t k = 0; k < one.size() && k < m.size(); ++k)
            CHECK(one[k]._i == m[k]._i && one[k]._j == m[k]._j);
    }
    CHECK(total > 500);
    std::printf("%s: %ld matches over 5 pairs\n", g_fail ? "FAILED" : "guided_fast adaptor ok", total);
    return g_fail ? 1 : 0;
}

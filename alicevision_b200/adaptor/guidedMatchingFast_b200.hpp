// Reference-side adaptor for guided matching from known poses: matching::guidedMatchingFundamentalFast<FundamentalEpipolarDistanceError>
// (matching/guidedMatching.hpp:353-460), the matcher StructureEstimationFromKnownPoses::match runs for every pair of its list
// (sfm/pipeline/structureFromKnownPoses/StructureEstimationFromKnownPoses.cpp:72-163), on the b200match engine (H100).
// Header-only; compiled inside an AliceVision build and linked against libb200match.so.  Uses only Regions and IndMatch: the
// caller computes the undistorted positions with its camera code (camera::IntrinsicBase::getUndistortedPixel) and passes them
// as n x 2 doubles; nullptr = the regions' own positions (a camera without distortion).
#pragma once

#include <aliceVision/matching/IndMatch.hpp>
#include <aliceVision/feature/Regions.hpp>

#include <b200match.h>

#include "RegionsMatcher_b200.hpp"   // b200detail::sharedContext / nextViewId / regionsDtype / uploadRegions (same directory: matching/)

#include <cstdint>
#include <map>
#include <utility>
#include <vector>

namespace aliceVision {
namespace matching {

namespace b200detail {
/// Appends the matches of result pair k to out.
inline void appendResultPair(const b200m_result* res, int k, IndMatches& out)
{
    const int64_t* off = nullptr;
    const b200m_match* m = nullptr;
    b200m_result_get(res, nullptr, &off, &m);
    for (int64_t e = off[k]; e < off[k + 1]; ++e)
        out.emplace_back(m[e].i, m[e].j);
}
}  // namespace b200detail

/// One pair.  F: any 3x3 matrix type with operator()(row, col); ep2: the epipole in the right image, not normalised, with
/// operator()(k).  errorTh / distRatio already squared as the reference's caller passes them.  Appends to out like the reference
/// (ascending left index, not de-duplicated).  lPos / rPos: optional n x 2 undistorted positions.  Returns false when the engine
/// is unavailable or fails (the caller then runs the reference's own function).
template<class Mat3T, class Vec3T>
bool guidedMatchingFundamentalFast_b200(const Mat3T& F,
                                        const Vec3T& ep2,
                                        const feature::Regions& lRegions,
                                        const feature::Regions& rRegions,
                                        int widthR,
                                        int heightR,
                                        double errorTh,
                                        double distRatio,
                                        IndMatches& out,
                                        const double* lPos = nullptr,
                                        const double* rPos = nullptr)
{
    b200m_ctx* ctx = b200detail::sharedContext();
    const int dtype = b200detail::regionsDtype(lRegions);
    if (ctx == nullptr || dtype < 0)
        return false;
    if (b200detail::regionsDtype(rRegions) != dtype || lRegions.DescriptorLength() != rRegions.DescriptorLength())
        return true;   // no common descriptor type: nothing to add
    const uint32_t ids[2] = {b200detail::nextViewId(), b200detail::nextViewId()};
    bool upL = b200detail::uploadRegions(ctx, ids[0], lRegions, dtype);
    bool upR = upL && b200detail::uploadRegions(ctx, ids[1], rRegions, dtype);
    bool ok = upR && (lPos == nullptr || b200m_set_view_geometry(ctx, ids[0], lPos, (int)lRegions.RegionCount()) == B200M_OK) &&
              (rPos == nullptr || b200m_set_view_geometry(ctx, ids[1], rPos, (int)rRegions.RegionCount()) == B200M_OK);
    if (ok)
    {
        const double f[9] = {F(0, 0), F(0, 1), F(0, 2), F(1, 0), F(1, 1), F(1, 2), F(2, 0), F(2, 1), F(2, 2)};
        const double e[3] = {ep2(0), ep2(1), ep2(2)};
        const int32_t wh[2] = {widthR, heightR};
        b200m_result* res = nullptr;
        ok = b200m_guided_match_fast_pairs(ctx, ids, 1, f, e, wh, errorTh, distRatio, &res) == B200M_OK;
        if (ok)
            b200detail::appendResultPair(res, 0, out);
        b200m_result_free(res);
    }
    if (upL)
        b200m_remove_view(ctx, ids[0]);
    if (upR)
        b200m_remove_view(ctx, ids[1]);
    return ok;
}

/// A pair list over views that are uploaded ONCE each: addView every view (with its undistorted positions, if any), addPair every
/// pair, then run().  One descriptor type per batch (StructureEstimationFromKnownPoses::match loops over the types).  The views
/// are removed from the engine when the batch is destroyed.
class GuidedMatchingFastBatch_b200
{
public:
    explicit GuidedMatchingFastBatch_b200(b200m_ctx* ctx = b200detail::sharedContext())
      : _ctx(ctx)
    {}
    ~GuidedMatchingFastBatch_b200()
    {
        if (_ctx)
            for (const auto& v : _views)
                b200m_remove_view(_ctx, v.second);
    }
    GuidedMatchingFastBatch_b200(const GuidedMatchingFastBatch_b200&) = delete;
    GuidedMatchingFastBatch_b200& operator=(const GuidedMatchingFastBatch_b200&) = delete;

    bool available() const { return _ctx != nullptr && _ok; }

    /// Uploads a view once (later calls for the same id are ignored).  pos: n x 2 undistorted positions or nullptr.
    bool addView(IndexT viewId, const feature::Regions& regions, const double* pos = nullptr)
    {
        if (!available())
            return false;
        if (_views.count(viewId))
            return true;
        const int dtype = b200detail::regionsDtype(regions);
        if (dtype < 0)
            return _ok = false;
        const uint32_t id = b200detail::nextViewId();
        if (!b200detail::uploadRegions(_ctx, id, regions, dtype))
            return _ok = false;
        _views[viewId] = id;
        if (pos != nullptr && b200m_set_view_geometry(_ctx, id, pos, (int)regions.RegionCount()) != B200M_OK)
            return _ok = false;
        return true;
    }

    /// F: x_R^T F x_L = 0; ep2: the epipole in image R, not normalised; (widthR, heightR): the size of image R.
    template<class Mat3T, class Vec3T>
    void addPair(IndexT left, IndexT right, const Mat3T& F, const Vec3T& ep2, int widthR, int heightR)
    {
        _pairs.emplace_back(left, right);
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c)
                _F.push_back(F(r, c));
        for (int k = 0; k < 3; ++k)
            _ep2.push_back(ep2(k));
        _wh.push_back(widthR);
        _wh.push_back(heightR);
    }

    /// Runs every pair added so far; out[pair] gets the pair's matches appended (an entry for every pair, empty lists included).
    /// Returns false (out untouched) when the engine is unavailable or fails.
    template<class PairMapT>
    bool run(double errorTh, double distRatio, PairMapT& out)
    {
        if (!available())
            return false;
        std::vector<uint32_t> ids;
        ids.reserve(2 * _pairs.size());
        for (const auto& p : _pairs)
        {
            const auto l = _views.find(p.first), r = _views.find(p.second);
            if (l == _views.end() || r == _views.end())
                return false;
            ids.push_back(l->second);
            ids.push_back(r->second);
        }
        b200m_result* res = nullptr;
        if (b200m_guided_match_fast_pairs(_ctx, ids.data(), (int)_pairs.size(), _F.data(), _ep2.data(), _wh.data(), errorTh, distRatio, &res) != B200M_OK)
        {
            b200m_result_free(res);
            return false;
        }
        for (std::size_t k = 0; k < _pairs.size(); ++k)
            b200detail::appendResultPair(res, (int)k, out[_pairs[k]]);
        b200m_result_free(res);
        return true;
    }

private:
    b200m_ctx* _ctx;
    bool _ok = true;
    std::map<IndexT, uint32_t> _views;
    std::vector<std::pair<IndexT, IndexT>> _pairs;
    std::vector<double> _F, _ep2;
    std::vector<int32_t> _wh;
};

}  // namespace matching
}  // namespace aliceVision

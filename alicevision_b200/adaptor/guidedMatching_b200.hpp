// Reference-side adaptor for the step after the path: matching::guidedMatching<Mat3Model, FundamentalEpipolarDistanceError>
// (matching/guidedMatching.hpp:206-268, called by GeometricFilterMatrix_F_AC.hpp:381-389 / GeometricFilterMatrix_E_AC.hpp:163)
// on the b200match engine (H100).  Header-only; compiled inside an AliceVision build and linked against libb200match.so.
// Cameras with distortion are not handled here (the reference un-distorts the positions first, :220-243): pass
// camL == camR == nullptr semantics, i.e. call it when the intrinsics have no distortion or the positions are already undistorted.
#pragma once

#include <aliceVision/matching/IndMatch.hpp>
#include <aliceVision/feature/Regions.hpp>

#include <b200match.h>

#include "RegionsMatcher_b200.hpp"   // b200detail::sharedContext / nextViewId / regionsDtype / uploadRegions (same directory: matching/)

namespace aliceVision {
namespace matching {

/// F: any 3x3 matrix type with operator()(row, col) (aliceVision::Mat3 / robustEstimation::Mat3Model::getMatrix()).
/// errorTh and distRatio are the already squared values the reference passes (Square(precision), Square(distanceRatio)).
/// Appends to out_matches and de-duplicates it like the reference (:267).  Returns false when the engine is unavailable.
template<class Mat3T>
bool guidedMatchingFundamental_b200(const Mat3T& F,
                                    const feature::Regions& lRegions,
                                    const feature::Regions& rRegions,
                                    double errorTh,
                                    double distRatio,
                                    matching::IndMatches& out_matches)
{
    b200m_ctx* ctx = b200detail::sharedContext();
    const int dtype = b200detail::regionsDtype(lRegions);
    if (ctx == nullptr || dtype < 0)
        return false;
    if (b200detail::regionsDtype(rRegions) != dtype || lRegions.DescriptorLength() != rRegions.DescriptorLength())
        return true;   // no common descriptor type: nothing to add (guidedMatching.hpp:300-306)
    const uint32_t idL = b200detail::nextViewId(), idR = b200detail::nextViewId();
    bool ok = b200detail::uploadRegions(ctx, idL, lRegions, dtype);
    const bool upR = ok && b200detail::uploadRegions(ctx, idR, rRegions, dtype);
    ok = upR;
    if (ok)
    {
        const double f[9] = {F(0, 0), F(0, 1), F(0, 2), F(1, 0), F(1, 1), F(1, 2), F(2, 0), F(2, 1), F(2, 2)};
        b200m_result* res = nullptr;
        ok = b200m_guided_match(ctx, idL, idR, f, errorTh, distRatio, &res) == B200M_OK;
        if (ok)
        {
            const int64_t* off = nullptr;
            const b200m_match* m = nullptr;
            b200m_result_get(res, nullptr, &off, &m);
            for (int64_t e = off[0]; e < off[1]; ++e)
                out_matches.emplace_back(m[e].i, m[e].j);
            b200m_result_free(res);
            matching::IndMatch::getDeduplicated(out_matches);
        }
    }
    b200m_remove_view(ctx, idL);
    if (upR)
        b200m_remove_view(ctx, idR);
    return ok;
}

}  // namespace matching
}  // namespace aliceVision

// Reference-side adaptors for the `fundamental_matrix` and `homography_matrix` geometric filters: matchingImageCollection::
// robustModelEstimation with GeometricFilterMatrix_F_AC (ACRANSAC, Fundamental7PSolver; GeometricFilter.hpp:40-88,
// GeometricFilterMatrix_F_AC.hpp:90-174, :266-299, :357-392) or GeometricFilterMatrix_H_AC (Homography4PSolver;
// GeometricFilterMatrix_H_AC.hpp:43-103, :160-212) for a whole putative list on the b200match engine (H100): one a-contrario RANSAC
// call (b200m_acransac_fundamental_pairs / b200m_acransac_homography_pairs; for F a second one, b200m_acransac_fundamental_spherical_pairs,
// over the pairs whose two cameras are camera::Equidistant, GeometricFilterMatrix_F_AC.hpp:186-253), the reference's inlier copy and
// support rules, then one
// guided-matching call for every kept pair and common descriptor type (b200m_guided_match_pairs, or for H with distanceRatio < 0
// b200m_guided_match_positions_pairs).
// GeometricFilterMatrix_E_AC_Batch_b200 does the same for the `essential_matrix` filter (GeometricFilterMatrix_E_AC.hpp, pinhole pairs):
// one b200m_acransac_essential_pairs call, then guided matching with F = K_J^-T E K_I^-1.
// GeometricFilterMatrix_F_AC_Batch_b200 with estimateDistortion is the `fundamental_with_distortion` filter: its planar pairs go
// through one b200m_acransac_fundamental_distortion_pairs call (Fundamental10PSolver, hasStrongSupport(.., 10)).
// GeometricFilterMatrix_HGrowing_Batch_b200 does the same for the `homography_growing` filter (GeometricFilterMatrix_HGrowing.hpp:176-266,
// filterMatchesByHGrowing): one b200m_hgrowing_pairs call for every (pair, common describer type) of the list.
// Header-only; compiled inside an AliceVision build and linked against libb200match.so.  The caller gathers xI / xJ with the
// reference's fillMatricesWithUndistortFeaturesMatches and the guided positions with camera::IntrinsicBase::getUndistortedPixel.
// Inside the AliceVision build (ALICEVISION_B200_REFERENCE_FILTER_UTILS defined) the library's own copyInlierMatches and
// hasStrongSupport run; elsewhere their restatement below.
#pragma once

#include <aliceVision/matching/IndMatch.hpp>
#include <aliceVision/feature/Regions.hpp>
#include <aliceVision/feature/imageDescriberCommon.hpp>
#ifdef ALICEVISION_B200_REFERENCE_FILTER_UTILS
#include <aliceVision/matchingImageCollection/geometricFilterUtils.hpp>
#include <aliceVision/matching/supportEstimation.hpp>
#endif

#include <b200match.h>

// matching::b200detail: sharedContext / nextViewId / regionsDtype / uploadRegions (matching/ in an AliceVision tree, alongside here otherwise)
#if __has_include(<aliceVision/matching/RegionsMatcher_b200.hpp>)
#include <aliceVision/matching/RegionsMatcher_b200.hpp>
#else
#include "RegionsMatcher_b200.hpp"
#endif

#include <algorithm>
#include <array>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <limits>
#include <map>
#include <numeric>
#include <random>
#include <sstream>
#include <type_traits>
#include <utility>
#include <vector>

namespace aliceVision {
namespace matchingImageCollection {

namespace b200detail {
/// copyInlierMatches (geometricFilterUtils.cpp:13-37)
inline void copyInlierMatches(const std::vector<std::size_t>& inliers,
                              const matching::MatchesPerDescType& putatives,
                              const std::vector<feature::EImageDescriberType>& descTypes,
                              matching::MatchesPerDescType& out)
{
#ifdef ALICEVISION_B200_REFERENCE_FILTER_UTILS
    matchingImageCollection::copyInlierMatches(inliers, putatives, descTypes, out);
#else
    std::vector<std::size_t> ordered = inliers;
    std::sort(ordered.begin(), ordered.end());
    std::size_t type = 0, start = 0, end = putatives.getNbMatches(descTypes[0]);
    for (const std::size_t g : ordered)
    {
        while (g >= end)
        {
            ++type;
            start = end;
            end += putatives.getNbMatches(descTypes[type]);
        }
        out[descTypes[type]].push_back(putatives.at(descTypes[type])[g - start]);
    }
#endif
}

/// matching::hasStrongSupport(MatchesPerDescType, minimumSamples) (supportEstimation.cpp:48-59)
inline bool hasStrongSupport(const matching::MatchesPerDescType& matches, std::size_t minimumSamples)
{
#ifdef ALICEVISION_B200_REFERENCE_FILTER_UTILS
    return matching::hasStrongSupport(matches, minimumSamples);
#else
    float score = 0;
    for (const auto& m : matches)
        score += feature::getStrongSupportCoeff(m.first) * m.second.size();
    return score > minimumSamples;
#endif
}

/// The generator as its operator<< writes it: 624 words, then the position.
inline void mtState(const std::mt19937& g, uint32_t state[625])
{
    std::stringstream ss;
    ss << g;
    for (int k = 0; k < 625; ++k)
        ss >> state[k];
}
}  // namespace b200detail

/// The bookkeeping the a-contrario batch adaptors share: a putative list over views that are uploaded ONCE per descriptor type.
/// addView every (view, type) with its guided positions, addPair every pair, then the derived class's run(), which makes its engine
/// call(s) and hands them to finish().  The views are removed from the engine when the batch is destroyed.
class GeometricFilterBatchBase_b200
{
public:
    explicit GeometricFilterBatchBase_b200(b200m_ctx* ctx)
      : _ctx(ctx)
    {}
    ~GeometricFilterBatchBase_b200()
    {
        if (_ctx)
            for (const auto& v : _views)
                b200m_remove_view(_ctx, v.second);
    }
    GeometricFilterBatchBase_b200(const GeometricFilterBatchBase_b200&) = delete;
    GeometricFilterBatchBase_b200& operator=(const GeometricFilterBatchBase_b200&) = delete;

    bool available() const { return _ctx != nullptr && _ok; }

    /// Uploads one (view, type) once, with the regions' own positions; guidedPos: n x 2 positions guided matching uses
    /// (getUndistortedPixel when the camera isValid()), or nullptr for the regions' own positions.
    bool addView(IndexT viewId, feature::EImageDescriberType type, const feature::Regions& regions, const double* guidedPos = nullptr)
    {
        if (!available())
            return false;
        const auto key = std::make_pair(viewId, type);
        if (_views.count(key))
            return true;
        const int dtype = matching::b200detail::regionsDtype(regions);
        if (dtype < 0)
            return _ok = false;
        const uint32_t id = matching::b200detail::nextViewId();
        if (!matching::b200detail::uploadRegions(_ctx, id, regions, dtype))
            return _ok = false;
        _views[key] = id;
        if (guidedPos != nullptr && b200m_set_view_geometry(_ctx, id, guidedPos, (int)regions.RegionCount()) != B200M_OK)
            return _ok = false;
        return true;
    }

    /// descTypes: getCommonDescTypes of the pair (an empty list: the pair is not estimated, as the reference returns
    /// EstimationStatus(false, false)); xI / xJ: 2 x n (fillMatricesWithUndistortFeaturesMatches); sizes: (width, height).
    template<class MatT>
    void addPair(const Pair& pair,
                 const matching::MatchesPerDescType& putatives,
                 const std::vector<feature::EImageDescriberType>& descTypes,
                 const MatT& xI,
                 const MatT& xJ,
                 const std::pair<std::size_t, std::size_t>& sizeI,
                 const std::pair<std::size_t, std::size_t>& sizeJ)
    {
        PairIn p{pair, putatives, descTypes, _corr.size() / 4};
        if (!descTypes.empty())
            for (int c = 0; c < (int)xI.cols(); ++c)
            {
                _corr.push_back(xI(0, c));
                _corr.push_back(xI(1, c));
                _corr.push_back(xJ(0, c));
                _corr.push_back(xJ(1, c));
            }
        _wh.insert(_wh.end(), {(int32_t)sizeI.first, (int32_t)sizeI.second, (int32_t)sizeJ.first, (int32_t)sizeJ.second});
        _pairs.push_back(std::move(p));
    }

protected:
    struct PairIn
    {
        Pair pair;
        matching::MatchesPerDescType putatives;
        std::vector<feature::EImageDescriberType> descTypes;
        std::size_t offset;
    };

    /// What one K10 call returned for its pairs (indices in addPair order, ascending), entry q for pairs[q], and the minimum sample
    /// count of its solver (getMinimumNbRequiredSamples, the pairs' hasStrongSupport threshold).
    struct K10Out
    {
        std::vector<int> pairs;
        std::size_t minimumSamples;
        std::vector<int64_t> offsets;
        std::vector<uint8_t> valid;
        std::vector<int32_t> nInl, iters;
        std::vector<uint32_t> inl;
        std::vector<double> M, L, errMax, nfa;
        /// nCorr: the size, in correspondences, of the buffer the pairs' offsets index
        K10Out(const std::vector<PairIn>& added, std::vector<int> ks, std::size_t nCorr, std::size_t minSamples)
          : pairs(std::move(ks)), minimumSamples(minSamples)
        {
            const int n = (int)pairs.size();
            for (const int k : pairs)
                offsets.push_back((int64_t)added[k].offset);
            offsets.push_back((int64_t)nCorr);
            valid.resize(std::max(n, 1));
            nInl.resize(std::max(n, 1));
            iters.resize(std::max(n, 1));
            inl.resize(std::max<std::size_t>(nCorr, 1));
            M.resize(9 * std::max(n, 1));
            L.resize(2 * std::max(n, 1));
            errMax.resize(std::max(n, 1));
            nfa.resize(std::max(n, 1));
        }
    };

    /// 0 .. n-1: every pair added
    std::vector<int> allPairs() const
    {
        std::vector<int> ks(_pairs.size());
        std::iota(ks.begin(), ks.end(), 0);
        return ks;
    }

    const double* corrData() const
    {
        static const double dummy[4] = {0, 0, 0, 0};
        return _corr.empty() ? dummy : _corr.data();
    }

    /// What every stage does after its engine call(s), each call's entries given with their pairs: fills estimates (the model into
    /// the field `model`; errorMax and support only for a pair ACRANSAC found valid), keeps the pairs whose copied inliers pass
    /// hasStrongSupport(.., minimumSamples), minimumSamples the minimum sample count of the pair's call, and with guidedMatching
    /// replaces their lists by the guided ones (see guided) over pair k's model, or over modelOf(k) when the guided step needs
    /// another matrix.  Then moves the kept lists into out.
    template<class Estimate, class Call, class ModelOf = std::nullptr_t>
    bool finish(std::initializer_list<const K10Out*> calls, std::vector<Estimate>& estimates, double (Estimate::*model)[9],
                bool guidedMatching, double distanceRatio, Call call, matching::PairwiseMatches& out,
                ModelOf modelOf = nullptr) const
    {
        estimates.assign(_pairs.size(), Estimate());
        std::map<Pair, matching::MatchesPerDescType> result;
        std::vector<int> kept;
        for (const K10Out* r : calls)
            for (int q = 0; q < (int)r->pairs.size(); ++q)
            {
                const int k = r->pairs[q];
                Estimate& e = estimates[k];
                e.valid = r->valid[q] != 0;
                std::copy(r->M.begin() + 9 * q, r->M.begin() + 9 * q + 9, e.*model);
                if (!e.valid)
                    continue;
                e.errorMax = r->errMax[q];
                const std::vector<std::size_t> inliers(r->inl.begin() + r->offsets[q], r->inl.begin() + r->offsets[q] + r->nInl[q]);
                matching::MatchesPerDescType perType;
                b200detail::copyInlierMatches(inliers, _pairs[k].putatives, _pairs[k].descTypes, perType);
                e.strongSupport = b200detail::hasStrongSupport(perType, r->minimumSamples);
                if (e.strongSupport)
                {
                    result[_pairs[k].pair] = std::move(perType);
                    kept.push_back(k);
                }
            }
        std::sort(kept.begin(), kept.end());
        const auto guidedModel = [&](int k) -> const double* {
            if constexpr (std::is_null_pointer_v<ModelOf>)
                return estimates[k].*model;
            else
                return modelOf(k);
        };
        if (guidedMatching && !guided(kept, estimates, guidedModel, call, distanceRatio * distanceRatio, result))
            return false;
        for (auto& x : result)
            out[x.first] = std::move(x.second);
        return true;
    }

    /// The guided step of the kept pairs: their lists are replaced by one entry per common type (empty ones included) when errorMax
    /// is finite, else by nothing.  M(k) is pair k's 9 model coefficients; call(ids, n, M, errorTh, distRatio, &res) makes the one
    /// batched call, with errorTh = errorMax^2 per item and distRatio = distanceRatio^2.
    template<class Estimate, class ModelOf, class Call>
    bool guided(const std::vector<int>& kept, const std::vector<Estimate>& estimates, ModelOf M_of, Call call, double distRatio,
                std::map<Pair, matching::MatchesPerDescType>& result) const
    {
        std::vector<uint32_t> ids;
        std::vector<double> M, th;
        std::vector<std::pair<Pair, feature::EImageDescriberType>> items;
        for (const int k : kept)
        {
            result[_pairs[k].pair] = matching::MatchesPerDescType();       // the guided result replaces the inliers, even when empty
            const double errorMax = estimates[k].errorMax;
            if (errorMax == std::numeric_limits<double>::infinity())
                continue;                                                  // Geometry_guided_matching: m_dPrecision_robust infinite
            const double* m = M_of(k);
            for (const feature::EImageDescriberType t : _pairs[k].descTypes)
            {
                const auto l = _views.find(std::make_pair(_pairs[k].pair.first, t)), r = _views.find(std::make_pair(_pairs[k].pair.second, t));
                if (l == _views.end() || r == _views.end())
                    return false;
                ids.push_back(l->second);
                ids.push_back(r->second);
                M.insert(M.end(), m, m + 9);
                th.push_back(errorMax * errorMax);
                items.emplace_back(_pairs[k].pair, t);
            }
        }
        if (items.empty())
            return true;
        b200m_result* res = nullptr;
        if (call(ids.data(), (int)items.size(), M.data(), th.data(), distRatio, &res) != B200M_OK)
        {
            b200m_result_free(res);
            return false;
        }
        const int64_t* off = nullptr;
        const b200m_match* m = nullptr;
        b200m_result_get(res, nullptr, &off, &m);
        for (std::size_t q = 0; q < items.size(); ++q)
        {
            matching::IndMatches& dst = result[items[q].first][items[q].second];
            for (int64_t e = off[q]; e < off[q + 1]; ++e)
                dst.emplace_back(m[e].i, m[e].j);
        }
        b200m_result_free(res);
        return true;
    }

    b200m_ctx* _ctx;
    bool _ok = true;
    std::map<std::pair<IndexT, feature::EImageDescriberType>, uint32_t> _views;
    std::vector<PairIn> _pairs;
    std::vector<double> _corr;
    std::vector<int32_t> _wh;
};

/// robustModelEstimation with GeometricFilterMatrix_F_AC for the pairs added (addView / addPair of the base, addPairSpherical for
/// pairs of two equidistant cameras), then run().
class GeometricFilterMatrix_F_AC_Batch_b200 : public GeometricFilterBatchBase_b200
{
public:
    /// What the estimation of one pair gave (in addPair order): ACRANSAC's validity, F (row-major, x_J^T F x_I = 0; with
    /// estimateDistortion a planar pair's F is Fundamental10PModel::getMatrix(), read the same way by the error and guided matching
    /// while its solver's constraint is [x_I, y_I, 1 + l1 r_I^2] F [x_J, y_J, 1 + l2 r_J^2]^T = 0), L (that model's
    /// getRadialDistortion(), in preconditioned units; 0 otherwise), errorMax (m_dPrecision_robust; infinite when not valid) and
    /// the support decision.
    struct Estimate
    {
        bool valid = false, strongSupport = false;
        double F[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        double L[2] = {0, 0};
        double errorMax = std::numeric_limits<double>::infinity();
    };

    /// estimateDistortion: GeometricFilterMatrix_F_AC's m_estimateDistortion (the `fundamental_with_distortion` filter): the planar
    /// pairs are estimated by geometricEstimation_Mat_ACRANSAC<Fundamental10PSolver, Fundamental10PModel>.
    explicit GeometricFilterMatrix_F_AC_Batch_b200(b200m_ctx* ctx = matching::b200detail::sharedContext(), bool estimateDistortion = false)
      : GeometricFilterBatchBase_b200(ctx),
        _estimateDistortion(estimateDistortion)
    {}

    /// addPair for a pair whose two cameras are camera::Equidistant (geometricEstimation_Spherical_Mat): bI / bJ are 3 x n, column c
    /// the unit vector toUnitSphere(removeDistortion(ima2cam(x))) of column c of the xI / xJ addPair would take.  No image size.
    template<class MatT>
    void addPairSpherical(const Pair& pair,
                          const matching::MatchesPerDescType& putatives,
                          const std::vector<feature::EImageDescriberType>& descTypes,
                          const MatT& bI,
                          const MatT& bJ)
    {
        _spherical.resize(_pairs.size() + 1, 0);
        _spherical.back() = 1;
        PairIn p{pair, putatives, descTypes, _bear.size() / 6};
        if (!descTypes.empty())
            for (int c = 0; c < (int)bI.cols(); ++c)
            {
                for (int a = 0; a < 3; ++a)
                    _bear.push_back(bI(a, c));
                for (int a = 0; a < 3; ++a)
                    _bear.push_back(bJ(a, c));
            }
        _wh.insert(_wh.end(), {0, 0, 0, 0});
        _pairs.push_back(std::move(p));
    }

    /// robustModelEstimation over every pair added so far: each pair starts from `rng`.  geometricEstimation_Mat_ACRANSAC takes the
    /// generator by value; geometricEstimation_Spherical_Mat takes it by reference, so a single-threaded reference run hands it on
    /// from a spherical pair to the next pair, which no batch reproduces.  The planar pairs go through one K10 call (the 10-point
    /// call with estimateDistortion), the spherical ones through another.  Pairs with strong support (hasStrongSupport(.., 10) for
    /// the 10-point call, (.., 7) for the 7-point ones) enter out; with guidedMatching their lists are the guided ones (errorTh =
    /// errorMax^2, distRatio = distanceRatio^2, every common type, empty lists included; nothing when errorMax is infinite; a
    /// spherical F is applied to the guided positions, as the reference does).  Returns false (out untouched) when the engine is
    /// unavailable or fails.
    bool run(const std::mt19937& rng, std::size_t maxIteration, double precision, bool guidedMatching, double distanceRatio,
             matching::PairwiseMatches& out)
    {
        if (!available())
            return false;
        const int n = (int)_pairs.size();
        _spherical.resize(n, 0);
        uint32_t state[625];
        b200detail::mtState(rng, state);
        std::vector<int> sub[2];                                        // in addPair order: the planar pairs, the spherical pairs
        for (int k = 0; k < n; ++k)
            sub[(int)_spherical[k]].push_back(k);
        std::vector<int32_t> wh;
        for (const int k : sub[0])
            wh.insert(wh.end(), _wh.begin() + 4 * k, _wh.begin() + 4 * k + 4);
        // minimum sample counts: Fundamental10PSolver 10, Fundamental7PSolver and Fundamental7PSphericalSolver 7
        K10Out r0(_pairs, sub[0], _corr.size() / 4, _estimateDistortion ? 10 : 7), r1(_pairs, sub[1], _bear.size() / 6, 7);
        const int n0 = (int)sub[0].size(), n1 = (int)sub[1].size();
        if (n0 > 0 && !_estimateDistortion &&
            b200m_acransac_fundamental_pairs(_ctx, n0, r0.offsets.data(), corrData(), wh.data(), state, (int64_t)maxIteration,
                                             precision, r0.valid.data(), r0.nInl.data(), r0.inl.data(), r0.M.data(),
                                             r0.errMax.data(), r0.nfa.data(), r0.iters.data()) != B200M_OK)
            return false;
        if (n0 > 0 && _estimateDistortion &&
            b200m_acransac_fundamental_distortion_pairs(_ctx, n0, r0.offsets.data(), corrData(), wh.data(), state, (int64_t)maxIteration,
                                                        precision, r0.valid.data(), r0.nInl.data(), r0.inl.data(), r0.M.data(),
                                                        r0.L.data(), r0.errMax.data(), r0.nfa.data(), r0.iters.data()) != B200M_OK)
            return false;
        if (n1 > 0 && b200m_acransac_fundamental_spherical_pairs(_ctx, n1, r1.offsets.data(), _bear.data(), state, 0, (int64_t)maxIteration,
                                                                 precision, r1.valid.data(), r1.nInl.data(), r1.inl.data(), r1.M.data(),
                                                                 r1.errMax.data(), r1.nfa.data(), r1.iters.data(), nullptr) != B200M_OK)
            return false;
        const bool ok = finish({&r0, &r1}, _estimates, &Estimate::F, guidedMatching, distanceRatio,
                               [&](const uint32_t* ids, int np, const double* M, const double* th, double distRatio, b200m_result** res) {
                                   return b200m_guided_match_pairs(_ctx, ids, np, B200M_MODEL_FUNDAMENTAL, M, th, distRatio, res);
                               },
                               out);
        if (_estimateDistortion)
            for (int q = 0; q < n0; ++q)
                std::copy(r0.L.begin() + 2 * q, r0.L.begin() + 2 * q + 2, _estimates[sub[0][q]].L);
        return ok;
    }

    /// The estimation of the k-th pair added, after run().
    const Estimate& estimate(std::size_t k) const { return _estimates.at(k); }

private:
    std::vector<Estimate> _estimates;
    bool _estimateDistortion;
    std::vector<char> _spherical;   // per pair added: 1 = addPairSpherical (its offset indexes _bear)
    std::vector<double> _bear;      // 6 doubles per correspondence (xI, yI, zI, xJ, yJ, zJ)
};

/// robustModelEstimation with GeometricFilterMatrix_H_AC (ACRANSAC, Homography4PSolver, point-to-point error;
/// GeometricFilterMatrix_H_AC.hpp:43-103, :160-212) for the pairs added (addView / addPair of the base), then run().
class GeometricFilterMatrix_H_AC_Batch_b200 : public GeometricFilterBatchBase_b200
{
public:
    /// What the estimation of one pair gave (in addPair order): ACRANSAC's validity, H (row-major, x_J ~ H x_I), errorMax
    /// (m_dPrecision_robust; infinite when not valid) and the support decision.
    struct Estimate
    {
        bool valid = false, strongSupport = false;
        double H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        double errorMax = std::numeric_limits<double>::infinity();
    };

    explicit GeometricFilterMatrix_H_AC_Batch_b200(b200m_ctx* ctx = matching::b200detail::sharedContext())
      : GeometricFilterBatchBase_b200(ctx)
    {}

    /// robustModelEstimation over every pair added so far.  Every pair starts from `rng`: the reference hands one generator from pair
    /// to pair by reference, which featureMatching's OpenMP loop shares between threads without order, so no run of it is
    /// reproducible; starting every pair from the same state is deterministic and independent of the thread count.  Pairs with strong
    /// support (hasStrongSupport(.., 4)) enter out; with guidedMatching their lists are the guided ones, errorTh = errorMax^2, every
    /// common type, empty lists included, nothing when errorMax is infinite:
    ///   distanceRatio < 0   position-only guidedMatching and IndMatchDecorator on the regions' positions (featureMatching's case)
    ///   distanceRatio >= 0  guidedMatching with descriptors, distRatio = distanceRatio^2
    /// Returns false (out untouched) when the engine is unavailable or fails.
    bool run(const std::mt19937& rng, std::size_t maxIteration, double precision, bool guidedMatching, double distanceRatio,
             matching::PairwiseMatches& out)
    {
        if (!available())
            return false;
        const int n = (int)_pairs.size();
        uint32_t state[625];
        b200detail::mtState(rng, state);
        K10Out r(_pairs, allPairs(), _corr.size() / 4, 4);   // 4: Homography4PSolver
        if (n > 0 && b200m_acransac_homography_pairs(_ctx, n, r.offsets.data(), corrData(), _wh.data(), state, 0, (int64_t)maxIteration, precision,
                                                     r.valid.data(), r.nInl.data(), r.inl.data(), r.M.data(), r.errMax.data(), r.nfa.data(),
                                                     r.iters.data(), nullptr) != B200M_OK)
            return false;
        return finish({&r}, _estimates, &Estimate::H, guidedMatching, distanceRatio,
                      [&](const uint32_t* ids, int np, const double* M, const double* th, double distRatio, b200m_result** res) {
                          if (distanceRatio < 0)
                              return b200m_guided_match_positions_pairs(_ctx, ids, np, B200M_MODEL_HOMOGRAPHY, M, th, 1, res);
                          return b200m_guided_match_pairs(_ctx, ids, np, B200M_MODEL_HOMOGRAPHY, M, th, distRatio, res);
                      },
                      out);
    }

    /// The estimation of the k-th pair added, after run().
    const Estimate& estimate(std::size_t k) const { return _estimates.at(k); }

private:
    std::vector<Estimate> _estimates;
};

/// robustModelEstimation with GeometricFilterMatrix_E_AC (ACRANSAC, Essential5PSolver on K^-1 x, FundamentalEpipolarDistanceError of
/// F = K_J^-T E K_I^-1 on the pixels; GeometricFilterMatrix_E_AC.hpp) for the pairs added (addView of the base, addPairCalibrated),
/// then run().
class GeometricFilterMatrix_E_AC_Batch_b200 : public GeometricFilterBatchBase_b200
{
public:
    /// What the estimation of one pair gave (in addPairCalibrated order): ACRANSAC's validity, E (row-major), errorMax
    /// (m_dPrecision_robust, in pixels; infinite when not valid) and the support decision.
    struct Estimate
    {
        bool valid = false, strongSupport = false;
        double E[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        double errorMax = std::numeric_limits<double>::infinity();
    };

    explicit GeometricFilterMatrix_E_AC_Batch_b200(b200m_ctx* ctx = matching::b200detail::sharedContext())
      : GeometricFilterBatchBase_b200(ctx)
    {}

    /// addPair with the pair's two camera::Pinhole::K() (row-major, 9 doubles each).  A pair the reference does not estimate (no
    /// common describer type, a missing or non-pinhole intrinsic) is simply not added.
    template<class MatT>
    void addPairCalibrated(const Pair& pair,
                           const matching::MatchesPerDescType& putatives,
                           const std::vector<feature::EImageDescriberType>& descTypes,
                           const MatT& xI,
                           const MatT& xJ,
                           const std::pair<std::size_t, std::size_t>& sizeI,
                           const std::pair<std::size_t, std::size_t>& sizeJ,
                           const double KI[9],
                           const double KJ[9])
    {
        addPair(pair, putatives, descTypes, xI, xJ, sizeI, sizeJ);
        _K.insert(_K.end(), KI, KI + 9);
        _K.insert(_K.end(), KJ, KJ + 9);
    }

    /// robustModelEstimation over every pair added so far.  ACRANSAC's precision is Square(precision), as the filter passes
    /// upperBoundPrecision = Square(m_dPrecision) (the residual threshold is then precision^4).  Every pair starts from `rng`: the
    /// reference hands one generator from pair to pair by reference, shared by featureMatching's OpenMP threads in no fixed order, so
    /// no run of it is reproducible.  Pairs with strong support (hasStrongSupport(.., 5)) enter out; with guidedMatching their lists
    /// are guidedMatching's with F = K_J^-T E K_I^-1, errorTh = errorMax^2 and distRatio = distanceRatio^2 (every common type, empty
    /// lists included; nothing when errorMax is infinite).  Returns false (out untouched) when the engine is unavailable or fails.
    bool run(const std::mt19937& rng, std::size_t maxIteration, double precision, bool guidedMatching, double distanceRatio,
             matching::PairwiseMatches& out)
    {
        if (!available())
            return false;
        const int n = (int)_pairs.size();
        uint32_t state[625];
        b200detail::mtState(rng, state);
        K10Out r(_pairs, allPairs(), _corr.size() / 4, 5);   // 5: Essential5PSolver
        if (n > 0 && b200m_acransac_essential_pairs(_ctx, n, r.offsets.data(), corrData(), _wh.data(), _K.data(), state, 0, (int64_t)maxIteration,
                                                    precision * precision, r.valid.data(), r.nInl.data(), r.inl.data(), r.M.data(),
                                                    r.errMax.data(), r.nfa.data(), r.iters.data(), nullptr) != B200M_OK)
            return false;
        std::vector<double> F(9 * n);   // the guided step's F of each kept pair
        return finish({&r}, _estimates, &Estimate::E, guidedMatching, distanceRatio,
                      [&](const uint32_t* ids, int np, const double* M, const double* th, double distRatio, b200m_result** res) {
                          return b200m_guided_match_pairs(_ctx, ids, np, B200M_MODEL_FUNDAMENTAL, M, th, distRatio, res);
                      },
                      out,
                      [&](int k) {
                          fundamentalFromEssential(_estimates[k].E, &_K[18 * k], &_K[18 * k + 9], &F[9 * k]);
                          return &F[9 * k];
                      });
    }

    /// The estimation of the k-th pair added, after run().
    const Estimate& estimate(std::size_t k) const { return _estimates.at(k); }

    /// fundamentalFromEssential (multiview/essential.cpp): F = K_J^-T E K_I^-1, formed as (K_J^-T E) K_I^-1 with the engine's cofactor
    /// inverse; all row-major.
    static void fundamentalFromEssential(const double E[9], const double KI[9], const double KJ[9], double F[9])
    {
        double iI[9], iJ[9], T[9];
        inverse3(KI, iI);
        inverse3(KJ, iJ);
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c)
                T[3 * r + c] = (iJ[r] * E[c] + iJ[3 + r] * E[3 + c]) + iJ[6 + r] * E[6 + c];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c)
                F[3 * r + c] = (T[3 * r] * iI[c] + T[3 * r + 1] * iI[3 + c]) + T[3 * r + 2] * iI[6 + c];
    }

private:
    /// M^-1 by cofactors over the determinant expanded along the first column
    static void inverse3(const double M[9], double R[9])
    {
        double C[9];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j)
            {
                const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
                C[3 * i + j] = M[3 * i1 + j1] * M[3 * i2 + j2] - M[3 * i1 + j2] * M[3 * i2 + j1];
            }
        const double inv = 1.0 / ((C[0] * M[0] + C[3] * M[3]) + C[6] * M[6]);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j)
                R[3 * i + j] = C[3 * j + i] * inv;
    }

    std::vector<Estimate> _estimates;
    std::vector<double> _K;   // 18 per pair: K_I, K_J
};

/// robustModelEstimation with GeometricFilterMatrix_HGrowing (the `homography_growing` filter: filterMatchesByHGrowing on the
/// regions' raw PointFeatures, GeometricFilterMatrix_HGrowing.hpp:176-266, GeometricFilterMatrix_HGrowing.cpp:108-194) for the pairs
/// added, then run().  No view is uploaded: each (pair, type) goes to the engine as its putatives' feature pairs.  The result is the
/// reference's single-threaded seed loop, which is what featureMatching runs (its seed loop sits inside robustModelEstimation's OpenMP
/// loop).
class GeometricFilterMatrix_HGrowing_Batch_b200
{
public:
    /// GrowParameters and HGrowingFilteringParam at the reference's defaults (GeometricFilterMatrix_HGrowing.hpp:23-106), which
    /// featureMatching never changes
    struct Param
    {
        double similarityTolerance = 20, affinityTolerance = 10, homographyTolerance = 5;
        int minInliersToRefine = 6, nbRefiningIterations = 8, maxNbHomographies = 10, minNbMatchesPerH = 20;
    };
    /// per (pair, type): each homography (row-major, x_J ~ H x_I) with its matches, like the reference's _HsAndMatchesPerDesc
    using HsAndMatches = std::vector<std::pair<std::array<double, 9>, matching::IndMatches>>;

    explicit GeometricFilterMatrix_HGrowing_Batch_b200(b200m_ctx* ctx = matching::b200detail::sharedContext())
      : _ctx(ctx)
    {}
    GeometricFilterMatrix_HGrowing_Batch_b200(b200m_ctx* ctx, const Param& param)
      : _ctx(ctx),
        _param(param)
    {}

    bool available() const { return _ctx != nullptr; }

    /// One pair of the putative list: its common describer types (RegionsPerView::getCommonDescTypes), its putatives, and
    /// featuresOf(view, type) -> const std::vector<feature::PointFeature>& (Regions::Features()).  A pair without a common type, or with
    /// a CCTag or AprilTag type among them in builds that have those describers, gets no estimation; a type without a putative entry is
    /// skipped.  The putatives are walked in their given order (featureMatching sorts them by Lowe ratio first).
    template <class FeaturesOf>
    void addPair(const Pair& pair, const matching::MatchesPerDescType& putatives, const std::vector<feature::EImageDescriberType>& descTypes,
                 FeaturesOf featuresOf)
    {
        if (descTypes.empty())
            return;
        auto has = [&](feature::EImageDescriberType t) { return std::find(descTypes.begin(), descTypes.end(), t) != descTypes.end(); };
        (void)has;
#if ALICEVISION_IS_DEFINED(ALICEVISION_HAVE_CCTAG)
        if (has(feature::EImageDescriberType::CCTAG3) || has(feature::EImageDescriberType::CCTAG4))
            return;
#endif
#if ALICEVISION_IS_DEFINED(ALICEVISION_HAVE_APRILTAG)
        if (has(feature::EImageDescriberType::APRILTAG16H5))
            return;
#endif
        for (const feature::EImageDescriberType t : descTypes)
        {
            const auto it = putatives.find(t);
            if (it == putatives.end())
                continue;
            const std::vector<feature::PointFeature>& fI = featuresOf(pair.first, t);
            const std::vector<feature::PointFeature>& fJ = featuresOf(pair.second, t);
            for (const matching::IndMatch& m : it->second)
            {
                const feature::PointFeature& a = fI.at(m._i);
                const feature::PointFeature& b = fJ.at(m._j);
                const float v[8] = {a.x(), a.y(), a.scale(), a.orientation(), b.x(), b.y(), b.scale(), b.orientation()};
                _feat.insert(_feat.end(), v, v + 8);
            }
            _items.push_back(Item{pair, t, it->second});
            _offsets.push_back(_offsets.back() + (int64_t)it->second.size());
        }
    }

    /// filterMatchesByHGrowing for every (pair, type) added, in one engine call.  Every pair with at least one filtered type enters
    /// out, with an entry per filtered type even when it is empty; with guidedMatching its lists are an empty map (the reference's
    /// Geometry_guided_matching is an empty stub).  Returns false (out untouched) when the engine is unavailable or fails.
    bool run(bool guidedMatching, matching::PairwiseMatches& out)
    {
        if (!available())
            return false;
        const int n = (int)_items.size();
        const int mh = _param.maxNbHomographies;
        std::vector<int32_t> nH(n), counts((std::size_t)n * std::max(mh, 1)), inl(std::max<int64_t>(_offsets.back(), 1));
        std::vector<double> H((std::size_t)n * std::max(mh, 1) * 9);
        if (n > 0 && b200m_hgrowing_pairs(_ctx, n, _offsets.data(), _feat.data(), _param.similarityTolerance, _param.affinityTolerance,
                                          _param.homographyTolerance, _param.minInliersToRefine, _param.nbRefiningIterations, mh,
                                          _param.minNbMatchesPerH, nH.data(), H.data(), counts.data(), inl.data(), nullptr, nullptr) != B200M_OK)
            return false;
        _hs.clear();
        std::map<Pair, matching::MatchesPerDescType> result;
        for (int k = 0; k < n; ++k)
        {
            const Item& item = _items[k];
            HsAndMatches& hs = _hs[item.pair][item.type];
            matching::IndMatches all;
            int64_t at = _offsets[k];
            for (int h = 0; h < nH[k]; ++h)
            {
                std::array<double, 9> M;
                std::copy(H.begin() + ((std::size_t)k * mh + h) * 9, H.begin() + ((std::size_t)k * mh + h) * 9 + 9, M.begin());
                matching::IndMatches ms;
                for (int q = 0; q < counts[(std::size_t)k * mh + h]; ++q)
                    ms.push_back(item.putatives[inl[at++]]);
                all.insert(all.end(), ms.begin(), ms.end());
                hs.emplace_back(M, std::move(ms));
            }
            matching::MatchesPerDescType& r = result[item.pair];
            if (!guidedMatching)
                r.emplace(item.type, std::move(all));
        }
        for (auto& x : result)
            out[x.first] = std::move(x.second);
        return true;
    }

    /// The homographies of one (pair, type) after run(); empty when it was not filtered.
    const HsAndMatches& homographies(const Pair& pair, feature::EImageDescriberType type) const
    {
        static const HsAndMatches none;
        const auto p = _hs.find(pair);
        if (p == _hs.end())
            return none;
        const auto t = p->second.find(type);
        return t == p->second.end() ? none : t->second;
    }

private:
    struct Item
    {
        Pair pair;
        feature::EImageDescriberType type;
        matching::IndMatches putatives;
    };
    b200m_ctx* _ctx;
    Param _param{};
    std::vector<Item> _items;
    std::vector<int64_t> _offsets{0};
    std::vector<float> _feat;
    std::map<Pair, std::map<feature::EImageDescriberType, HsAndMatches>> _hs;
};

}  // namespace matchingImageCollection
}  // namespace aliceVision

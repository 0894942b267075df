// Reference-side adaptor, Surface 2: an IImageCollectionMatcher that hands the whole pair list to the b200match engine (H100).
// Header-only; compiled inside an AliceVision build, derives from the reference's own interface
// (src/aliceVision/matchingImageCollection/IImageCollectionMatcher.hpp:28-42) and is the drop-in for
// ImageCollectionMatcher_generic with BRUTE_FORCE_L2 / BRUTE_FORCE_HAMMING (ImageCollectionMatcher_generic.cpp:30-123).
#pragma once

#include <aliceVision/matchingImageCollection/IImageCollectionMatcher.hpp>
#include <aliceVision/feature/RegionsPerView.hpp>
#include <aliceVision/system/Logger.hpp>

#include <b200match.h>

#include <memory>
#include <set>
#include <stdexcept>
#include <string>
#include <typeinfo>
#include <vector>

namespace aliceVision {
namespace matchingImageCollection {

/// Error convention (SURVEY 8b): the reference's ImageCollectionMatcher_generic::Match cannot fail, so an engine failure (no
/// usable GPU, CUDA error, out of device memory ...) must not abort featureMatching.  Give the adaptor a `fallback` matcher - the
/// integration passes the reference's own ImageCollectionMatcher_generic(BRUTE_FORCE_L2 | BRUTE_FORCE_HAMMING), see
/// integration/patches - and every failure is logged and the call is delegated to it, output map untouched by the failed attempt.
/// This is reference-side adaptor code: libb200match itself keeps no CPU path.  Without a fallback the failure is thrown.
class ImageCollectionMatcher_b200 : public IImageCollectionMatcher
{
  public:
    ImageCollectionMatcher_b200(float distRatio, bool crossMatching, bool hamming = false, int device = 0,
                                std::shared_ptr<const IImageCollectionMatcher> fallback = nullptr)
      : _f_dist_ratio(distRatio),
        _useCrossMatching(crossMatching),
        _hamming(hamming),
        _fallback(std::move(fallback))
    {
        if (b200m_ctx_create(device, nullptr, &_ctx) != B200M_OK)
            engineUnavailable(b200m_last_error());
    }
    /// Several GPUs behind one Match call: the pair list is sharded (2-D blocks, b200m_shard_pairs_2d) over one engine context
    /// per device (b200m_multi_match; no collective, pairs are independent).  An empty list means "every visible device".
    ImageCollectionMatcher_b200(float distRatio, bool crossMatching, bool hamming, std::vector<int> devices,
                                std::shared_ptr<const IImageCollectionMatcher> fallback = nullptr)
      : _f_dist_ratio(distRatio),
        _useCrossMatching(crossMatching),
        _hamming(hamming),
        _fallback(std::move(fallback))
    {
        if (devices.empty())
            for (int d = 0; d < b200m_device_count(); ++d)
                devices.push_back(d);
        if (devices.empty())
            engineUnavailable("no CUDA device");
        else if (devices.size() == 1)
        {
            if (b200m_ctx_create(devices[0], nullptr, &_ctx) != B200M_OK)
                engineUnavailable(b200m_last_error());
        }
        else if (b200m_multi_create(devices.data(), static_cast<int>(devices.size()), &_multi) != B200M_OK)
            engineUnavailable(b200m_last_error());
    }
    /// true when the engine could not be created and every Match goes to the fallback matcher
    bool usesFallbackOnly() const { return _ctx == nullptr && _multi == nullptr; }
    ~ImageCollectionMatcher_b200() override
    {
        if (_ctx != nullptr)
            b200m_ctx_destroy(_ctx);
        if (_multi != nullptr)
            b200m_multi_destroy(_multi);
    }

    /// Same contract as ImageCollectionMatcher_generic::Match: appends to map_PutativesMatches, never inserts empty lists,
    /// silently skips empty / type-mismatched views (:59-63,:74-78), unknown view ids throw std::out_of_range (RegionsPerView.hpp:85).
    void Match(std::mt19937& randomNumberGenerator,
               const feature::RegionsPerView& regionsPerView,
               const PairSet& pairs,
               feature::EImageDescriberType descType,
               matching::PairwiseMatches& map_PutativesMatches) const override
    {
        std::string error;
        if (!usesFallbackOnly() && engineMatch(regionsPerView, pairs, descType, map_PutativesMatches, error))
            return;
        if (_fallback == nullptr)
            throw std::runtime_error("b200match: " + error);
        if (!usesFallbackOnly())
            ALICEVISION_LOG_WARNING("b200match: " << error << " - matching this pair list with the fallback matcher");
        _fallback->Match(randomNumberGenerator, regionsPerView, pairs, descType, map_PutativesMatches);
    }

  private:
    void engineUnavailable(const std::string& why)
    {
        if (_fallback == nullptr)
            throw std::runtime_error("b200match: " + why);
        ALICEVISION_LOG_WARNING("b200match: engine unavailable (" << why << ") - using the fallback matcher");
    }

    /// One Match on the engine.  Returns false with `error` set on an engine failure; the output map is only written on success.
    /// Unknown view ids throw std::out_of_range exactly like the reference (RegionsPerView.hpp:85): that is the caller's error.
    bool engineMatch(const feature::RegionsPerView& regionsPerView,
                     const PairSet& pairs,
                     feature::EImageDescriberType descType,
                     matching::PairwiseMatches& map_PutativesMatches,
                     std::string& error) const
    {
        std::set<IndexT> used;
        for (const Pair& p : pairs)
        {
            used.insert(p.first);
            used.insert(p.second);
        }
        // one bulk upload per element type; asynchronous: the copies overlap the search of the first pairs, and the Regions
        // (owned by regionsPerView) outlive b200m_match_pairs, which returns after the last copy has left host memory
        struct Group { std::vector<uint32_t> ids; std::vector<const void*> descs; std::vector<int> counts; std::vector<std::vector<float>> xy; int dim = 0; };
        Group groups[3];
        for (IndexT viewId : used)
        {
            const feature::Regions& r = regionsPerView.getRegions(viewId, descType);   // throws like the reference on unknown ids
            const int n = static_cast<int>(r.RegionCount());
            int dtype;
            if (r.IsBinary())
                dtype = B200M_BIN;
            else if (r.Type_id() == typeid(float).name())
                dtype = B200M_F32;
            else if (r.Type_id() == typeid(unsigned char).name())
                dtype = B200M_U8;
            else
                continue;   // createRegionsMatcher has no brute-force case for other scalar types on this engine
            Group& g = groups[dtype];
            g.dim = static_cast<int>(r.DescriptorLength());
            g.ids.push_back(viewId);
            g.descs.push_back(n ? r.DescriptorRawData() : nullptr);
            g.counts.push_back(n);
            g.xy.emplace_back(2 * static_cast<size_t>(n));
            const auto& feats = r.Features();
            for (int k = 0; k < n; ++k)
            {
                g.xy.back()[2 * k] = feats[k].x();
                g.xy.back()[2 * k + 1] = feats[k].y();
            }
        }
        std::vector<uint32_t> flat;
        flat.reserve(2 * pairs.size());
        for (const Pair& p : pairs)
        {
            flat.push_back(p.first);
            flat.push_back(p.second);
        }
        b200m_result* res = nullptr;
        if (_multi != nullptr)
        {
            // all views of one descriptor type share one element type (the Regions class of descType); views of another
            // type would be skipped by the reference as well (:74-78)
            int dtype = 0;
            for (int t = 1; t < 3; ++t)
                if (groups[t].ids.size() > groups[dtype].ids.size())
                    dtype = t;
            Group& g = groups[dtype];
            std::vector<const float*> xyp;
            for (auto& v : g.xy)
                xyp.push_back(v.data());
            std::set<uint32_t> have(g.ids.begin(), g.ids.end());
            std::vector<uint32_t> usable;
            for (size_t k = 0; k + 1 < flat.size(); k += 2)
                if (have.count(flat[k]) && have.count(flat[k + 1]))
                {
                    usable.push_back(flat[k]);
                    usable.push_back(flat[k + 1]);
                }
            if (b200m_multi_match(_multi, static_cast<int>(g.ids.size()), g.ids.data(), g.descs.data(), g.counts.data(), g.dim, dtype, xyp.data(),
                                  usable.data(), static_cast<int>(usable.size() / 2), _f_dist_ratio, _useCrossMatching ? 1 : 0, &res) != B200M_OK)
            {
                error = b200m_last_error();
                return false;
            }
        }
        for (int dtype = 0; dtype < 3 && _multi == nullptr; ++dtype)
        {
            Group& g = groups[dtype];
            if (g.ids.empty())
                continue;
            std::vector<const float*> xyp;
            for (auto& v : g.xy)
                xyp.push_back(v.data());
            if (b200m_upload_views_async(_ctx, static_cast<int>(g.ids.size()), g.ids.data(), g.descs.data(), g.counts.data(), g.dim, dtype, xyp.data()) != B200M_OK)
            {
                error = b200m_last_error();
                b200m_wait_uploads(_ctx);   // earlier groups may still be reading the Regions
                return false;
            }
        }
        if (_multi == nullptr &&
            b200m_match_pairs(_ctx, flat.data(), static_cast<int>(pairs.size()), _f_dist_ratio, _useCrossMatching ? 1 : 0, B200M_STAGE_FULL, &res) != B200M_OK)
        {
            error = b200m_last_error();
            return false;
        }
        const uint32_t* ids = nullptr;
        const int64_t* off = nullptr;
        const b200m_match* m = nullptr;
        b200m_result_get(res, &ids, &off, &m);
        const int n = b200m_result_num_pairs(res);
        for (int k = 0; k < n; ++k)
        {
            if (off[k + 1] == off[k])
                continue;   // :116-119: empty results are not inserted
            matching::IndMatches v;
            v.reserve(static_cast<size_t>(off[k + 1] - off[k]));
            for (int64_t e = off[k]; e < off[k + 1]; ++e)
                v.emplace_back(m[e].i, m[e].j, m[e].distance_ratio, m[e].distance);
            map_PutativesMatches[std::make_pair(ids[2 * k], ids[2 * k + 1])].emplace(descType, std::move(v));
        }
        b200m_result_free(res);
        return true;
    }

    float _f_dist_ratio;
    bool _useCrossMatching;
    bool _hamming;
    b200m_ctx* _ctx = nullptr;
    b200m_multi* _multi = nullptr;
    std::shared_ptr<const IImageCollectionMatcher> _fallback;
};

}  // namespace matchingImageCollection
}  // namespace aliceVision

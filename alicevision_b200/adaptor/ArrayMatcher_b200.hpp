// Reference-side adaptor, Surface 1: a matching::ArrayMatcher whose search runs on the b200match engine (H100) through the C ABI.
// Header-only; compiled INSIDE an AliceVision build (it derives from the reference's own interface,
// src/aliceVision/matching/ArrayMatcher.hpp:19-66) and linked against libb200match.so.  Drop-in for
// ArrayMatcher_bruteForce<Scalar,Metric> (matching/ArrayMatcher_bruteForce.hpp:24-151): same template parameters,
// same bool-return error behaviour, results per query in ascending distance order.
#pragma once

#include <map>
#include <mutex>
#include <aliceVision/matching/ArrayMatcher.hpp>
#include <aliceVision/feature/metric.hpp>

#include <b200match.h>

#include <type_traits>
#include <vector>

namespace aliceVision {
namespace matching {

namespace b200detail {
template <class Metric> struct MetricId;
template <class T> struct MetricId<feature::L2_Simple<T>> { static constexpr int value = B200M_L2_SIMPLE; };
template <class T> struct MetricId<feature::L2_Vectorized<T>> { static constexpr int value = B200M_L2_VECTORIZED; };
template <class T> struct MetricId<feature::Hamming<T>> { static constexpr int value = B200M_HAMMING; };

template <class Scalar, class Metric> constexpr int dtypeOf()
{
    static_assert(std::is_same<Scalar, float>::value || std::is_same<Scalar, unsigned char>::value,
                  "ArrayMatcher_b200 supports float and unsigned char descriptors");
    return std::is_same<Scalar, float>::value ? B200M_F32 : (MetricId<Metric>::value == B200M_HAMMING ? B200M_BIN : B200M_U8);
}

/// One engine context per process and device, created on first use.  Thread-safe (IRegionsMatcher adaptors are created from
/// OpenMP regions): the per-device table is guarded by a mutex, a context is created at most once per device, and a failed
/// creation is retried by the next caller instead of being cached.
inline b200m_ctx* sharedContext(int device = 0)
{
    static std::mutex mu;
    static std::map<int, b200m_ctx*> table;
    std::lock_guard<std::mutex> lock(mu);
    auto it = table.find(device);
    if (it != table.end())
        return it->second;
    b200m_ctx* ctx = nullptr;
    if (b200m_ctx_create(device, nullptr, &ctx) != B200M_OK)
        return nullptr;
    table[device] = ctx;
    return ctx;
}
}  // namespace b200detail

template<typename Scalar = float, typename Metric = feature::L2_Simple<Scalar>>
class ArrayMatcher_b200 : public ArrayMatcher<Scalar, Metric>
{
  public:
    typedef typename Metric::ResultType DistanceType;

    ArrayMatcher_b200() = default;
    ~ArrayMatcher_b200() override { release(); }
    ArrayMatcher_b200(const ArrayMatcher_b200&) = delete;
    ArrayMatcher_b200& operator=(const ArrayMatcher_b200&) = delete;

    /// Copies the dataset to the GPU (the reference borrows the pointer, ArrayMatcher_bruteForce.hpp:49).
    bool Build(std::mt19937& /*randomNumberGenerator*/, const Scalar* dataset, int nbRows, int dimension) override
    {
        release();
        if (nbRows < 1)
            return false;
        b200m_ctx* ctx = b200detail::sharedContext();
        if (ctx == nullptr)
            return false;
        _dim = dimension;
        return b200m_db_create(ctx, dataset, nbRows, dimension, b200detail::dtypeOf<Scalar, Metric>(), b200detail::MetricId<Metric>::value, &_db) ==
               B200M_OK;
    }

    bool SearchNeighbour(const Scalar* query, int* indice, DistanceType* distance) override
    {
        if (_db == nullptr)
            return false;
        int32_t idx = -1;
        DistanceType d = DistanceType();
        static_assert(sizeof(DistanceType) == 4, "float (L2) or unsigned int (Hamming) distances");
        if (b200m_knn(b200detail::sharedContext(), _db, query, 1, 1, &idx, &d) != B200M_OK)
            return false;
        *indice = idx;
        *distance = d;
        return true;
    }

    bool SearchNeighbours(const Scalar* query, int nbQuery, IndMatches* pvec_indices, std::vector<DistanceType>* pvec_distances, size_t NN) override
    {
        if (_db == nullptr || nbQuery < 1)
            return false;
        std::vector<int32_t> idx(static_cast<size_t>(nbQuery) * NN);
        pvec_distances->resize(static_cast<size_t>(nbQuery) * NN);
        if (b200m_knn(b200detail::sharedContext(), _db, query, nbQuery, static_cast<int>(NN), idx.data(), pvec_distances->data()) != B200M_OK)
        {
            pvec_distances->clear();
            return false;
        }
        pvec_indices->resize(static_cast<size_t>(nbQuery) * NN);
        for (int q = 0; q < nbQuery; ++q)
            for (size_t k = 0; k < NN; ++k)
                (*pvec_indices)[q * NN + k] = IndMatch(q, idx[q * NN + k]);   // (query, database) as ArrayMatcher_bruteForce.hpp:138
        return true;
    }

  private:
    void release()
    {
        if (_db != nullptr)
            b200m_db_destroy(_db);
        _db = nullptr;
    }
    b200m_db* _db = nullptr;
    int _dim = 0;
};

}  // namespace matching
}  // namespace aliceVision

// diskann_b200.hpp — C++ host-side mirror of the reference's operator interface for the distance
// hot path, layered on the C ABI in diskann_b200.h (header-only; link libdiskann_b200.so).
//
// The reference is compiled Rust and this image has no Rust toolchain, so the host layer above
// the C ABI is C++ with the reference's names, argument meaning and error behaviour:
//
//   Metric                         diskann-vector/src/distance/metric.rs:8-20
//   Distance<T,U>::call            diskann-vector/src/distance/distance_provider.rs:62-100
//   distance_comparer<T,U>         DistanceProvider::distance_comparer, distance_provider.rs:44-46
//   Provider                       diskann_inmem::Provider (diskann-inmem/src/provider.rs:71-131):
//                                  set_element / set_neighbors / search accessor creation
//   QueryDistance / expand_beam    layers::QueryDistance::evaluate + SearchAccessor::expand_beam
//                                  (diskann-inmem/src/layers/mod.rs:59-77; provider.rs:436-479),
//                                  batched over queries
//   GpuKNN::search                 benchmark_core::search::graph::KNN::search
//                                  (diskann-benchmark-core/src/search/graph/knn.rs:208-238) for a
//                                  whole query batch (the 3' boundary of SURVEY.md §8b)
//   SearchStats                    diskann/src/graph/index.rs:90 (cmps, hops, result_count)
//   Transform                      Transform::{PaddingHadamard, DoubleHadamard} (diskann-quantization/src/algorithms/
//                                  transforms): try_from_parts + transform_into
//   MinMaxQuantizer                diskann-quantization/src/minmax/quantizer.rs:69-228 (Transform::Null or one of the
//                                  above) + the MinMax distance functors over compressed rows (vectors.rs:231-455)
//
// Errors: every non-zero status becomes ANNError (the inmem layer returns Err on length / type
// mismatch, layers/full.rs:203-213, 306-314; it never panics across the boundary).
#pragma once

#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "diskann_b200.h"

namespace diskann_b200 {

enum class Metric : int { Cosine = DAB_COSINE, InnerProduct = DAB_INNER_PRODUCT, L2 = DAB_L2, CosineNormalized = DAB_COSINE_NORMALIZED };

// IEEE binary16 storage type (the reference uses half::f16)
struct f16 {
    uint16_t bits;
};

class ANNError : public std::runtime_error {
   public:
    ANNError(int code, const std::string& msg) : std::runtime_error(msg), code_(code) {}
    int code() const { return code_; }

   private:
    int code_;
};

inline void check(int status) {
    if (status != DAB_OK) throw ANNError(status, dab_last_error());
}

template <class T>
struct ElementType;
template <>
struct ElementType<float> {
    static constexpr int value = DAB_F32;
};
template <>
struct ElementType<f16> {
    static constexpr int value = DAB_F16;
};
template <>
struct ElementType<int8_t> {
    static constexpr int value = DAB_I8;
};
template <>
struct ElementType<uint8_t> {
    static constexpr int value = DAB_U8;
};

// Distance<T, U>: what T::distance_comparer(metric, Some(dim)) returns.
template <class T, class U = T>
class Distance {
   public:
    Distance(Metric metric, size_t dim, int device = 0) : metric_(metric), dim_(dim), device_(device) {}
    // distance_comparer.call(x, y): both slices must have the comparer's dimension
    float call(const T* x, size_t xlen, const U* y, size_t ylen) const {
        if (xlen != dim_ || ylen != dim_)
            throw ANNError(DAB_ERR_INVALID_ARGUMENT, "expected slices of length " + std::to_string(dim_) + " - instead got " +
                                                         std::to_string(xlen) + " and " + std::to_string(ylen));
        float out = 0.0f;
        check(dab_pair_distances(ElementType<T>::value, ElementType<U>::value, (int)metric_, (uint32_t)dim_, x, y, 1, &out, device_));
        return out;
    }
    // n pairs at once (rows dense, dim elements each)
    std::vector<float> call_batch(const T* x, const U* y, size_t n) const {
        std::vector<float> out(n);
        check(dab_pair_distances(ElementType<T>::value, ElementType<U>::value, (int)metric_, (uint32_t)dim_, x, y, n, out.data(), device_));
        return out;
    }

   private:
    Metric metric_;
    size_t dim_;
    int device_;
};

template <class T, class U = T>
Distance<T, U> distance_comparer(Metric metric, size_t dim, int device = 0) {
    return Distance<T, U>(metric, dim, device);
}

struct SearchStats {
    uint32_t cmps, hops, result_count;
};

struct KnnResults {
    uint32_t nq, k;
    std::vector<uint32_t> ids;     // [nq][k], padded UINT32_MAX
    std::vector<float> distances;  // [nq][k], padded +inf
    std::vector<SearchStats> stats;
};

// Device-resident snapshot of an in-memory provider for element type T.
template <class T>
class Provider {
   public:
    Provider(Metric metric, uint32_t dim, uint64_t n_points, uint32_t n_start, uint32_t max_degree, int device = 0)
        : dim_(dim), n_points_(n_points), n_start_(n_start), max_degree_(max_degree) {
        check(dab_create(&h_, ElementType<T>::value, (int)metric, dim, n_points, n_start, max_degree, device));
    }
    ~Provider() { dab_destroy(h_); }
    Provider(const Provider&) = delete;
    Provider& operator=(const Provider&) = delete;

    uint32_t dim() const { return dim_; }
    uint64_t n_points() const { return n_points_; }
    uint32_t n_start() const { return n_start_; }
    dab_index* raw() { return h_; }

    // SetElement: rows [first, first + count)
    void set_elements(const T* rows, uint64_t first, uint64_t count) { check(dab_upload_vectors(h_, rows, first, count)); }
    // neighbors().set_neighbors for rows [first, first + count): row = [len, ids...]
    void set_neighbors(const uint32_t* adj, uint32_t stride, uint64_t first, uint64_t count) {
        check(dab_upload_graph(h_, adj, stride, first, count));
    }
    std::vector<uint32_t> get_neighbors(uint64_t first, uint64_t count) {
        std::vector<uint32_t> adj(count * (size_t)(max_degree_ + 1));
        check(dab_download_graph(h_, adj.data(), max_degree_ + 1, first, count));
        return adj;
    }

    // QueryDistance::evaluate for every (query q, id ids[q][j]): expand_beam's distance stage
    std::vector<float> query_distances(const T* queries, uint32_t nq, const uint32_t* ids, uint32_t c) {
        std::vector<float> out((size_t)nq * c);
        check(dab_distances(h_, queries, nq, ids, c, out.data()));
        return out;
    }
    // Distance<T,T> between stored rows (prune closure)
    std::vector<float> row_distances(const uint32_t* a, const uint32_t* b, uint64_t n) {
        std::vector<float> out(n);
        check(dab_row_pair_distances(h_, a, b, n, out.data()));
        return out;
    }

    // AttributeValueProvider for diverse search: ids [first, first + count) take values[i]; present[i] == 0 (present
    // NULL: none) marks an id without an attribute
    void set_attributes(const uint32_t* values, const uint8_t* present, uint64_t first, uint64_t count) {
        check(dab_upload_attributes(h_, values, present, first, count));
    }

    // the 64-bit label sets of ids [first, first + count) for filtered search
    void set_labels(const uint64_t* labels, uint64_t first, uint64_t count) { check(dab_upload_labels(h_, labels, first, count)); }

    // index construction on the device (multi_insert semantics)
    void build(uint32_t pruned_degree, uint32_t l_build, float alpha = 1.2f, uint32_t batch = 0) {
        check(dab_build(h_, pruned_degree, l_build, alpha, batch));
    }
    // DiskANNIndex::insert / multi_insert into the graph as it stands: rows [ids.size()][dim] become points ids
    void insert(const std::vector<uint32_t>& ids, const T* rows, uint32_t pruned_degree, uint32_t l_build, float alpha = 1.2f,
                uint32_t batch = 0) {
        check(dab_insert(h_, ids.data(), rows, ids.size(), pruned_degree, l_build, alpha, batch));
    }

    // deletion: Delete::delete / release / status_by_internal_id, and consolidate_vector for every node
    void remove(const std::vector<uint32_t>& ids) { check(dab_delete(h_, ids.data(), ids.size())); }
    void release(const std::vector<uint32_t>& ids) { check(dab_release(h_, ids.data(), ids.size())); }
    std::vector<uint8_t> delete_status(const std::vector<uint32_t>& ids) {
        std::vector<uint8_t> out(ids.size());
        check(dab_delete_status(h_, ids.data(), ids.size(), out.data()));
        return out;
    }
    uint64_t consolidate(uint32_t pruned_degree, float alpha = 1.2f) {
        uint64_t rewritten = 0;
        check(dab_consolidate(h_, pruned_degree, alpha, &rewritten));
        return rewritten;
    }
    // DiskANNIndex::multi_inplace_delete in chunks of batch_size (1: inplace_delete id by id, 0: one chunk);
    // method: DAB_INPLACE_VISITED_AND_TOPK (k_value, l_value), DAB_INPLACE_TWO_HOP_AND_ONE_HOP or DAB_INPLACE_ONE_HOP
    void inplace_delete(const std::vector<uint32_t>& ids, uint32_t num_to_replace, int method, uint32_t pruned_degree, float alpha = 1.2f,
                        uint32_t k_value = 20, uint32_t l_value = 50, uint32_t batch_size = 1) {
        check(dab_inplace_delete(h_, ids.data(), ids.size(), method, num_to_replace, k_value, l_value, pruned_degree, alpha, batch_size));
    }
    // drop_deleted_neighbors for every node; returns the lists rewritten
    uint64_t drop_deleted_neighbors(uint32_t pruned_degree, bool only_orphans = false) {
        uint64_t rewritten = 0;
        check(dab_drop_deleted_neighbors(h_, pruned_degree, only_orphans ? 1 : 0, &rewritten));
        return rewritten;
    }

    // DiskANNIndex::count_reachable_nodes from the start points, or from explicit start ids
    uint64_t count_reachable() {
        uint64_t count = 0;
        check(dab_count_reachable(h_, nullptr, 0, &count));
        return count;
    }
    uint64_t count_reachable(const std::vector<uint32_t>& start_ids) {
        uint64_t count = 0;
        const uint32_t none = 0;  // an empty list still passes a pointer: NULL would mean the start points
        check(dab_count_reachable(h_, start_ids.empty() ? &none : start_ids.data(), (uint32_t)start_ids.size(), &count));
        return count;
    }
    // DiskANNIndex::get_degree_stats over every id, or over explicit ids (an empty list gives all zeros)
    struct DegreeStats {
        uint32_t max_degree = 0;
        float avg_degree = 0.0f;
        uint32_t min_degree = 0;
        uint64_t cnt_less_than_two = 0;
    };
    DegreeStats degree_stats() { return degree_stats_of(nullptr, 0); }
    DegreeStats degree_stats(const std::vector<uint32_t>& ids) {
        const uint32_t none = 0;
        return degree_stats_of(ids.empty() ? &none : ids.data(), ids.size());
    }
    // DiskANNIndex::prune_range over every id, or over explicit ids; returns the lists rewritten
    uint64_t prune_range(uint32_t pruned_degree, float alpha = 1.2f) {
        uint64_t rewritten = 0;
        check(dab_prune_range(h_, nullptr, 0, pruned_degree, alpha, &rewritten));
        return rewritten;
    }
    uint64_t prune_range(const std::vector<uint32_t>& ids, uint32_t pruned_degree, float alpha = 1.2f) {
        uint64_t rewritten = 0;
        const uint32_t none = 0;
        check(dab_prune_range(h_, ids.empty() ? &none : ids.data(), ids.size(), pruned_degree, alpha, &rewritten));
        return rewritten;
    }

   private:
    DegreeStats degree_stats_of(const uint32_t* ids, uint64_t n) {
        DegreeStats s;
        check(dab_degree_stats(h_, ids, n, &s.max_degree, &s.avg_degree, &s.min_degree, &s.cnt_less_than_two));
        return s;
    }

    dab_index* h_ = nullptr;
    uint32_t dim_;
    uint64_t n_points_;
    uint32_t n_start_, max_degree_;
};

// Range::search for a whole batch (range_search.rs:255-469): query q's results are ids / distances
// [offsets[q], offsets[q + 1]) in the reference's output order
struct RangeResults {
    uint32_t nq = 0;
    std::vector<uint64_t> offsets;  // [nq + 1]
    std::vector<uint32_t> ids;
    std::vector<float> distances;
    std::vector<uint32_t> cmps, hops;
    std::vector<uint8_t> second_round;  // range_search_second_round
};

// Range::builder(starting_l, radius) with its optional fields; max_returned 0: None
template <class T>
class GpuRange {
   public:
    GpuRange(Provider<T>& provider, uint32_t starting_l, float radius, uint32_t beam_width = 1, bool has_inner_radius = false,
             float inner_radius = 0.0f, float initial_slack = 1.0f, float range_slack = 1.0f, uint64_t max_returned = 0)
        : p_(provider), l_(starting_l), beam_(beam_width), radius_(radius), has_inner_(has_inner_radius), inner_(inner_radius),
          initial_slack_(initial_slack), range_slack_(range_slack), max_returned_(max_returned) {}
    RangeResults search(const T* queries, uint32_t nq) {
        dab_range* set = nullptr;
        check(dab_range_search(p_.raw(), queries, nq, l_, beam_, radius_, has_inner_ ? 1 : 0, inner_, initial_slack_, range_slack_,
                               max_returned_, &set));
        return take(set, nq);
    }
    // Range::search over the provider's PQ, SQ or MinMax store: every distance of both phases the store's; `rerank`: the
    // in_range ids by full-precision distance, those within (inner_radius, radius] of it, sorted by it, with it
    RangeResults search_pq(const T* queries, uint32_t nq, bool rerank = false) { return search_store(dab_range_search_pq, queries, nq, rerank); }
    RangeResults search_sq(const T* queries, uint32_t nq, bool rerank = false) { return search_store(dab_range_search_sq, queries, nq, rerank); }
    RangeResults search_minmax(const T* queries, uint32_t nq, bool rerank = false) {
        return search_store(dab_range_search_minmax, queries, nq, rerank);
    }
    // FilteredRange::search over the provider's label table: every point within the radius that masks[q] accepts (one
    // mask per query; match_all: ALL, else ANY, as GpuFiltered)
    RangeResults search_filtered(const T* queries, uint32_t nq, const uint64_t* masks, bool match_all = false) {
        dab_range* set = nullptr;
        check(dab_range_search_filtered(p_.raw(), queries, nq, l_, beam_, radius_, has_inner_ ? 1 : 0, inner_, initial_slack_, range_slack_,
                                        max_returned_, masks, match_all ? 1 : 0, &set));
        return take(set, nq);
    }
    // FilteredRange::search over the provider's PQ, SQ or MinMax store: every distance of both phases the store's;
    // `rerank`: the returned matches by full-precision distance, sorted by it (NaN last), those above inner_radius, with
    // it (no outer-radius filter, as in FilteredRange::search)
    RangeResults search_filtered_pq(const T* queries, uint32_t nq, const uint64_t* masks, bool match_all = false, bool rerank = false) {
        return search_filtered_store(dab_range_search_filtered_pq, queries, nq, masks, match_all, rerank);
    }
    RangeResults search_filtered_sq(const T* queries, uint32_t nq, const uint64_t* masks, bool match_all = false, bool rerank = false) {
        return search_filtered_store(dab_range_search_filtered_sq, queries, nq, masks, match_all, rerank);
    }
    RangeResults search_filtered_minmax(const T* queries, uint32_t nq, const uint64_t* masks, bool match_all = false, bool rerank = false) {
        return search_filtered_store(dab_range_search_filtered_minmax, queries, nq, masks, match_all, rerank);
    }

   private:
    using StoreSearch = int (*)(dab_index*, const void*, uint32_t, uint32_t, uint32_t, float, int, float, float, float, uint64_t, int, dab_range**);
    RangeResults search_store(StoreSearch f, const T* queries, uint32_t nq, bool rerank) {
        dab_range* set = nullptr;
        check(f(p_.raw(), queries, nq, l_, beam_, radius_, has_inner_ ? 1 : 0, inner_, initial_slack_, range_slack_, max_returned_, rerank ? 1 : 0,
                &set));
        return take(set, nq);
    }
    using FilteredStoreSearch = int (*)(dab_index*, const void*, uint32_t, uint32_t, uint32_t, float, int, float, float, float, uint64_t,
                                        const uint64_t*, uint32_t, int, dab_range**);
    RangeResults search_filtered_store(FilteredStoreSearch f, const T* queries, uint32_t nq, const uint64_t* masks, bool match_all, bool rerank) {
        dab_range* set = nullptr;
        check(f(p_.raw(), queries, nq, l_, beam_, radius_, has_inner_ ? 1 : 0, inner_, initial_slack_, range_slack_, max_returned_, masks,
                match_all ? 1 : 0, rerank ? 1 : 0, &set));
        return take(set, nq);
    }
    // the offsets, stats and results of a result set, which is freed
    static RangeResults take(dab_range* set, uint32_t nq) {
        std::unique_ptr<dab_range, void (*)(dab_range*)> owned(set, dab_range_free);
        RangeResults r;
        r.nq = nq;
        r.offsets.resize((size_t)nq + 1);
        r.cmps.resize(nq);
        r.hops.resize(nq);
        r.second_round.resize(nq);
        check(dab_range_offsets(set, r.offsets.data(), r.cmps.data(), r.hops.data(), r.second_round.data()));
        r.ids.resize(r.offsets[nq]);
        r.distances.resize(r.offsets[nq]);
        check(dab_range_results(set, r.ids.data(), r.distances.data()));
        return r;
    }

    Provider<T>& p_;
    uint32_t l_, beam_;
    float radius_;
    bool has_inner_;
    float inner_, initial_slack_, range_slack_;
    uint64_t max_returned_;
};

// Diverse::search for a whole batch (diverse_search.rs:114-234): Diverse::new(Knn::new(l_value, beam_width),
// DiverseSearchParams::new(_, diverse_k, k, provider's attributes)); at most diverse_k results per attribute value.
template <class T>
class GpuDiverse {
   public:
    GpuDiverse(Provider<T>& provider, uint32_t l_value, uint32_t diverse_k, uint32_t beam_width = 1)
        : p_(provider), l_(l_value), diverse_k_(diverse_k), beam_(beam_width) {}
    KnnResults search(const T* queries, uint32_t nq, uint32_t k) {
        KnnResults r;
        r.nq = nq;
        r.k = k;
        r.ids.resize((size_t)nq * k);
        r.distances.resize((size_t)nq * k);
        std::vector<uint32_t> counts(nq), cmps(nq), hops(nq);
        check(dab_search_batch_diverse(p_.raw(), queries, nq, k, l_, beam_, diverse_k_, r.ids.data(), r.distances.data(), counts.data(),
                                       cmps.data(), hops.data()));
        r.stats.resize(nq);
        for (uint32_t i = 0; i < nq; ++i) r.stats[i] = SearchStats{cmps[i], hops[i], counts[i]};
        return r;
    }
    // The same over the quantized stores (the store must be resident): the traversal distances of
    // dab_search_batch_pq / _sq / _minmax; `rerank`: Pipeline<FilterStartPoints, Rerank> over the post-processed list
    KnnResults search_pq(const T* queries, uint32_t nq, uint32_t k, bool rerank) {
        return search_quantized(dab_search_batch_diverse_pq, queries, nq, k, rerank);
    }
    KnnResults search_sq(const T* queries, uint32_t nq, uint32_t k, bool rerank) {
        return search_quantized(dab_search_batch_diverse_sq, queries, nq, k, rerank);
    }
    KnnResults search_minmax(const T* queries, uint32_t nq, uint32_t k, bool rerank) {
        return search_quantized(dab_search_batch_diverse_minmax, queries, nq, k, rerank);
    }

   private:
    using Quantized = int (*)(dab_index*, const void*, uint32_t, uint32_t, uint32_t, uint32_t, uint32_t, int, uint32_t*, float*, uint32_t*,
                              uint32_t*, uint32_t*);
    KnnResults search_quantized(Quantized fn, const T* queries, uint32_t nq, uint32_t k, bool rerank) {
        KnnResults r;
        r.nq = nq;
        r.k = k;
        r.ids.resize((size_t)nq * k);
        r.distances.resize((size_t)nq * k);
        std::vector<uint32_t> counts(nq), cmps(nq), hops(nq);
        check(fn(p_.raw(), queries, nq, k, l_, beam_, diverse_k_, rerank ? 1 : 0, r.ids.data(), r.distances.data(), counts.data(), cmps.data(),
                 hops.data()));
        r.stats.resize(nq);
        for (uint32_t i = 0; i < nq; ++i) r.stats[i] = SearchStats{cmps[i], hops[i], counts[i]};
        return r;
    }

    Provider<T>& p_;
    uint32_t l_, diverse_k_, beam_;
};

// InlineFilterSearch::search for a whole batch (inline_filter_search.rs:89-160): InlineFilterSearch::new(Knn::new(l_value,
// beam_width), adaptive L), over the provider's labels (set_labels).  Query q accepts id i when labels[i] & masks[q] != 0
// (match_all false) or == masks[q] (match_all true).  adaptive_samples == 0: no AdaptiveL.
template <class T>
class GpuFiltered {
   public:
    GpuFiltered(Provider<T>& provider, uint32_t l_value, uint32_t beam_width = 1, uint32_t adaptive_samples = 0, double adaptive_scale = 1.0)
        : p_(provider), l_(l_value), beam_(beam_width), samples_(adaptive_samples), scale_(adaptive_scale) {}
    KnnResults search(const T* queries, const uint64_t* masks, uint32_t nq, uint32_t k, bool match_all = false) {
        KnnResults r;
        r.nq = nq;
        r.k = k;
        r.ids.resize((size_t)nq * k);
        r.distances.resize((size_t)nq * k);
        std::vector<uint32_t> counts(nq), cmps(nq), hops(nq);
        check(dab_search_batch_filtered(p_.raw(), queries, nq, k, l_, beam_, masks, match_all ? 1 : 0, samples_, scale_, r.ids.data(),
                                        r.distances.data(), counts.data(), cmps.data(), hops.data()));
        r.stats.resize(nq);
        for (uint32_t i = 0; i < nq; ++i) r.stats[i] = SearchStats{cmps[i], hops[i], counts[i]};
        return r;
    }
    // The same over the quantized stores (the store must be resident): the traversal distances of
    // dab_search_batch_pq / _sq / _minmax; `rerank`: Pipeline<FilterStartPoints, Rerank> over the first L matches
    KnnResults search_pq(const T* queries, const uint64_t* masks, uint32_t nq, uint32_t k, bool rerank, bool match_all = false) {
        return search_quantized(dab_search_batch_filtered_pq, queries, masks, nq, k, rerank, match_all);
    }
    KnnResults search_sq(const T* queries, const uint64_t* masks, uint32_t nq, uint32_t k, bool rerank, bool match_all = false) {
        return search_quantized(dab_search_batch_filtered_sq, queries, masks, nq, k, rerank, match_all);
    }
    KnnResults search_minmax(const T* queries, const uint64_t* masks, uint32_t nq, uint32_t k, bool rerank, bool match_all = false) {
        return search_quantized(dab_search_batch_filtered_minmax, queries, masks, nq, k, rerank, match_all);
    }

   private:
    using Quantized = int (*)(dab_index*, const void*, uint32_t, uint32_t, uint32_t, uint32_t, const uint64_t*, uint32_t, uint32_t, double,
                              int, uint32_t*, float*, uint32_t*, uint32_t*, uint32_t*);
    KnnResults search_quantized(Quantized fn, const T* queries, const uint64_t* masks, uint32_t nq, uint32_t k, bool rerank, bool match_all) {
        KnnResults r;
        r.nq = nq;
        r.k = k;
        r.ids.resize((size_t)nq * k);
        r.distances.resize((size_t)nq * k);
        std::vector<uint32_t> counts(nq), cmps(nq), hops(nq);
        check(fn(p_.raw(), queries, nq, k, l_, beam_, masks, match_all ? 1 : 0, samples_, scale_, rerank ? 1 : 0, r.ids.data(),
                 r.distances.data(), counts.data(), cmps.data(), hops.data()));
        r.stats.resize(nq);
        for (uint32_t i = 0; i < nq; ++i) r.stats[i] = SearchStats{cmps[i], hops[i], counts[i]};
        return r;
    }

    Provider<T>& p_;
    uint32_t l_, beam_, samples_;
    double scale_;
};

// KNN::search for a whole batch: Knn::new(l_value, beam_width) + k results per query.
template <class T>
class GpuKNN {
   public:
    GpuKNN(Provider<T>& provider, uint32_t l_value, uint32_t beam_width = 1) : p_(provider), l_(l_value), beam_(beam_width) {
        if (l_value == 0) throw ANNError(DAB_ERR_INVALID_ARGUMENT, "l_value cannot be zero");       // KnnSearchError::LZero
        if (beam_width == 0) throw ANNError(DAB_ERR_INVALID_ARGUMENT, "beam_width cannot be zero");  // BeamWidthZero
    }
    KnnResults search(const T* queries, uint32_t nq, uint32_t k) {
        KnnResults r;
        r.nq = nq;
        r.k = k;
        r.ids.resize((size_t)nq * k);
        r.distances.resize((size_t)nq * k);
        std::vector<uint32_t> counts(nq), cmps(nq), hops(nq);
        check(dab_search_batch(p_.raw(), queries, nq, k, l_, beam_, r.ids.data(), r.distances.data(), counts.data(), cmps.data(),
                               hops.data()));
        r.stats.resize(nq);
        for (uint32_t i = 0; i < nq; ++i) r.stats[i] = SearchStats{cmps[i], hops[i], counts[i]};
        return r;
    }

    // Batches in flight (search_all's one task per query partition, api.rs:410-419, as slots of the device):
    // `search_async` queues a batch on `slot` and returns at once, `wait` joins it and returns its results.
    // `queries` must stay valid until then.
    void search_async(uint32_t slot, const T* queries, uint32_t nq, uint32_t k) {
        if (slot >= DAB_MAX_SLOTS) throw ANNError(DAB_ERR_INVALID_ARGUMENT, "slot out of range");
        Pending& s = pending_[slot];
        s.r.nq = nq;
        s.r.k = k;
        s.r.ids.resize((size_t)nq * k);
        s.r.distances.resize((size_t)nq * k);
        s.counts.resize(nq), s.cmps.resize(nq), s.hops.resize(nq);
        check(dab_search_batch_async(p_.raw(), slot, queries, nq, k, l_, beam_, s.r.ids.data(), s.r.distances.data(), s.counts.data(),
                                     s.cmps.data(), s.hops.data()));
    }
    // The same over the quantized stores (the store must be resident; `rerank`: the full-precision Rerank): PQ, SQ and
    // MinMax batches share the slots with search_async, and `wait` joins a batch of any kind.  Results equal those of
    // dab_search_batch_pq[_rerank] / dab_search_batch_sq / dab_search_batch_minmax.
    void search_pq_async(uint32_t slot, const T* queries, uint32_t nq, uint32_t k, bool rerank) {
        queue_quantized(dab_search_batch_pq_async, slot, queries, nq, k, rerank);
    }
    void search_sq_async(uint32_t slot, const T* queries, uint32_t nq, uint32_t k, bool rerank) {
        queue_quantized(dab_search_batch_sq_async, slot, queries, nq, k, rerank);
    }
    void search_minmax_async(uint32_t slot, const T* queries, uint32_t nq, uint32_t k, bool rerank) {
        queue_quantized(dab_search_batch_minmax_async, slot, queries, nq, k, rerank);
    }
    KnnResults wait(uint32_t slot) {
        check(dab_wait(p_.raw(), slot));
        Pending& s = pending_[slot];
        s.r.stats.resize(s.r.nq);
        for (uint32_t i = 0; i < s.r.nq; ++i) s.r.stats[i] = SearchStats{s.cmps[i], s.hops[i], s.counts[i]};
        return std::move(s.r);
    }

   private:
    struct Pending {
        KnnResults r;
        std::vector<uint32_t> counts, cmps, hops;
    };
    using QuantizedAsync = int (*)(dab_index*, uint32_t, const void*, uint32_t, uint32_t, uint32_t, uint32_t, int, uint32_t*, float*,
                                   uint32_t*, uint32_t*, uint32_t*);
    void queue_quantized(QuantizedAsync fn, uint32_t slot, const T* queries, uint32_t nq, uint32_t k, bool rerank) {
        if (slot >= DAB_MAX_SLOTS) throw ANNError(DAB_ERR_INVALID_ARGUMENT, "slot out of range");
        Pending s;  // the slot's buffers are replaced only once the batch is queued
        s.r.nq = nq;
        s.r.k = k;
        s.r.ids.resize((size_t)nq * k);
        s.r.distances.resize((size_t)nq * k);
        s.counts.resize(nq), s.cmps.resize(nq), s.hops.resize(nq);
        check(fn(p_.raw(), slot, queries, nq, k, l_, beam_, rerank ? 1 : 0, s.r.ids.data(), s.r.distances.data(), s.counts.data(),
                 s.cmps.data(), s.hops.data()));
        pending_[slot] = std::move(s);  // moving a std::vector keeps its buffer
    }
    Provider<T>& p_;
    uint32_t l_, beam_;
    Pending pending_[DAB_MAX_SLOTS];
};

// DiskANNIndex::paged_search + PagedSearch::next_page (diskann/src/graph/search/paged.rs) for a whole query batch: every
// next_page(k) returns the next k results of each query's one resumable search, whose list and visited set stay on the
// device.  Results across pages do not overlap; stats are the session's cumulative cmps / hops.  The provider must
// outlive the session and stay unchanged (a changed index fails the next page); `queries` are copied at construction.
template <class T>
class PagedSearch {
   public:
    // the traversal store of a session: full precision, or one of the quantized stores (no rerank: pages return the
    // store's distances)
    enum class Store { FullPrecision, PQ, SQ, MinMax };

    PagedSearch(Provider<T>& provider, const T* queries, uint32_t nq, uint32_t l_value) : nq_(nq) {
        check(dab_paged_search_begin(provider.raw(), queries, nq, l_value, &h_));
    }
    PagedSearch(Provider<T>& provider, Store store, const T* queries, uint32_t nq, uint32_t l_value) : nq_(nq) {
        auto begin = store == Store::PQ ? dab_paged_search_begin_pq : store == Store::SQ ? dab_paged_search_begin_sq
                     : store == Store::MinMax ? dab_paged_search_begin_minmax : dab_paged_search_begin;
        check(begin(provider.raw(), queries, nq, l_value, &h_));
    }
    ~PagedSearch() { dab_paged_search_end(h_); }
    PagedSearch(const PagedSearch&) = delete;
    PagedSearch& operator=(const PagedSearch&) = delete;

    // 0 < k <= l_value; stats[q].result_count == 0 once query q is exhausted
    KnnResults next_page(uint32_t k) {
        KnnResults r;
        r.nq = nq_;
        r.k = k;
        r.ids.resize((size_t)nq_ * k);
        r.distances.resize((size_t)nq_ * k);
        std::vector<uint32_t> counts(nq_), cmps(nq_), hops(nq_);
        check(dab_paged_search_next(h_, k, r.ids.data(), r.distances.data(), counts.data(), cmps.data(), hops.data()));
        r.stats.resize(nq_);
        for (uint32_t i = 0; i < nq_; ++i) r.stats[i] = SearchStats{cmps[i], hops[i], counts[i]};
        return r;
    }

   private:
    dab_paged* h_ = nullptr;
    uint32_t nq_;
};

// Transform::PaddingHadamard / Transform::DoubleHadamard from the parts the reference serializes (try_from_parts:
// padding_hadamard.rs:137-173, double_hadamard.rs:146-206); signs are 0 / 1 bytes.  A host-side object; apply() runs
// transform_into on the device.
class Transform {
   public:
    static Transform padding_hadamard(const std::vector<uint8_t>& signs, uint32_t padded_dim, const std::vector<uint32_t>* subsample = nullptr) {
        return Transform(DAB_TRANSFORM_PADDING_HADAMARD, signs, padded_dim, nullptr, subsample);
    }
    static Transform double_hadamard(const std::vector<uint8_t>& signs0, const std::vector<uint8_t>& signs1,
                                     const std::vector<uint32_t>* subsample = nullptr) {
        return Transform(DAB_TRANSFORM_DOUBLE_HADAMARD, signs0, static_cast<uint32_t>(signs1.size()), &signs1, subsample);
    }
    Transform(Transform&& o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
    Transform& operator=(Transform&& o) noexcept {
        std::swap(h_, o.h_);
        return *this;
    }
    Transform(const Transform&) = delete;
    Transform& operator=(const Transform&) = delete;
    ~Transform() { dab_transform_destroy(h_); }

    uint32_t input_dim() const { return dab_transform_input_dim(h_); }
    uint32_t output_dim() const { return dab_transform_output_dim(h_); }
    // transform_into for n rows: [n][input_dim] -> [n][output_dim]
    std::vector<float> apply(const float* src, uint64_t n, int device = 0) const {
        std::vector<float> out(n * output_dim());
        check(dab_transform_apply(h_, device, src, n, out.data()));
        return out;
    }
    const dab_transform* handle() const { return h_; }

   private:
    Transform(int kind, const std::vector<uint8_t>& signs0, uint32_t inner_dim, const std::vector<uint8_t>* signs1,
              const std::vector<uint32_t>* subsample) {
        check(dab_transform_create(&h_, kind, static_cast<uint32_t>(signs0.size()), inner_dim, signs0.data(), signs1 ? signs1->data() : nullptr,
                                   subsample ? subsample->data() : nullptr, subsample ? static_cast<uint32_t>(subsample->size()) : 0u));
    }
    dab_transform* h_ = nullptr;
};

// MinMaxQuantizer (diskann-quantization/src/minmax/quantizer.rs:69-110) with Transform::Null, or behind a Transform, and
// the MinMax distance functors over compressed rows (vectors.rs:231-455).  Rows are the reference's canonical-front
// Data<NBITS> bytes at output_dim().
class MinMaxQuantizer {
   public:
    MinMaxQuantizer(uint32_t dim, float grid_scale, int device = 0) : dim_(dim), out_dim_(dim), grid_scale_(grid_scale), device_(device) {}
    MinMaxQuantizer(std::shared_ptr<const Transform> transform, float grid_scale, int device = 0)
        : dim_(transform->input_dim()), out_dim_(transform->output_dim()), grid_scale_(grid_scale), device_(device), transform_(std::move(transform)) {}
    uint32_t dim() const { return dim_; }
    uint32_t output_dim() const { return out_dim_; }
    // Data::<NBITS>::canonical_bytes(output_dim)
    size_t canonical_bytes(int nbits) const { return dab_minmax_row_bytes(out_dim_, nbits); }
    // CompressInto<&[f32], DataMutRef<NBITS>> for n vectors of dim() values; throws ANNError when a (transformed) vector
    // holds NaN (InputContainsNaN)
    std::vector<uint8_t> compress(const float* vectors, uint64_t n, int nbits, std::vector<float>* loss = nullptr) const {
        std::vector<uint8_t> rows(n * canonical_bytes(nbits));
        if (loss) loss->resize(n);
        if (transform_)
            check(dab_minmax_compress_transformed(transform_->handle(), device_, grid_scale_, nbits, vectors, n, rows.data(),
                                                  loss ? loss->data() : nullptr));
        else
            check(dab_minmax_compress(device_, grid_scale_, dim_, nbits, vectors, n, rows.data(), loss ? loss->data() : nullptr));
        return rows;
    }
    // MinMax{L2Squared, IP, Cosine, CosineNormalized}::evaluate(DataRef<N>, DataRef<M>) row by row (N x N, 8 x N)
    std::vector<float> distances(Metric metric, int nbits_x, int nbits_y, const uint8_t* x_rows, const uint8_t* y_rows, uint64_t n) const {
        std::vector<float> out(n);
        check(dab_minmax_distances(device_, static_cast<int>(metric), nbits_x, nbits_y, out_dim_, x_rows, y_rows, n, out.data()));
        return out;
    }

    // CompressInto<&[f32], FullQueryMut> + MinMax*::evaluate(FullQueryRef, DataRef<NBITS>) for every (query, row): [nq][n]
    std::vector<float> query_distances(Metric metric, int nbits, const float* queries, uint32_t nq, const uint8_t* rows, uint64_t n) const {
        std::vector<float> out(static_cast<size_t>(nq) * n);
        if (transform_)
            check(dab_minmax_query_distances_transformed(transform_->handle(), device_, static_cast<int>(metric), nbits, queries, nq, rows, n,
                                                         out.data()));
        else
            check(dab_minmax_query_distances(device_, static_cast<int>(metric), nbits, dim_, queries, nq, rows, n, out.data()));
        return out;
    }

   private:
    uint32_t dim_, out_dim_;
    float grid_scale_;
    int device_;
    std::shared_ptr<const Transform> transform_;
};

}  // namespace diskann_b200

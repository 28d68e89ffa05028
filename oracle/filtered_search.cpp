// filtered_search.cpp — CPU restatement of the reference's inline label-filtered search (test infrastructure only).
//
// InlineFilterSearch::search (diskann/src/graph/search/inline_filter_search.rs:89-160): inline_filter_search_internal
// (:166-282) — search_internal's traversal, every evaluated neighbour into scratch.best, the accepted start points and
// neighbours also into matched_results — with the optional AdaptiveL: once the evaluated neighbours of the hops reach
// sample_count, compute_adaptive_l (:294-310) runs once and, when the new L is above L, scratch.resize(new_l), i.e.
// NeighborPriorityQueue::reconfigure (neighbor/queue.rs:339-353), which sets the capacity and cuts a longer queue.  Then
// matched_results sorted by distance, the first L through the default post-processing: start points and deleted ids
// dropped, the first k kept.  The reference's sort_unstable_by(fast_distance) leaves the order of exactly equal
// distances open; here the sort is stable (an earlier match first) with NaN after every number.
//
// Built on its own into liboracle_filtered_search.so (oracle/filtered_search.mk), linked against liboracle.so for the
// distances.  C ABI (declared here, bound by tests/filtered_oracle.py):
//   uint64_t orc_compute_adaptive_l(uint64_t base_l, uint64_t visited, uint64_t matched, double max_multiplier);
//   void orc_search_batch_filtered(const orc_index* idx, const void* queries, uint64_t query_stride, uint32_t nq, uint32_t k,
//                                  uint32_t l_search, uint32_t beam_width, const uint64_t* labels, const uint64_t* masks,
//                                  int match_all, uint32_t adaptive_samples, double adaptive_scale, const uint32_t* deleted,
//                                  int flavour, uint32_t* out_ids, float* out_dists, uint32_t* out_counts, uint32_t* out_cmps,
//                                  uint32_t* out_hops);
//     labels: one u64 per id of the index (n_points + n_start); masks: one per query; match_all 0: ANY (labels & mask != 0),
//     else ALL (labels & mask == mask); adaptive_samples 0: no AdaptiveL; deleted: NULL or a bitmap of (n_total + 31) / 32
//     words, bit i of word i / 32 for id i.
#include "oracle.h"

#include <algorithm>
#include <cmath>
#include <limits>
#include <unordered_set>
#include <vector>

namespace {

// NeighborPriorityQueue with the capacity reconfigure sets (queue.rs:66-353)
struct Npq {
    size_t size = 0, capacity = 0, cursor = 0;
    std::vector<uint32_t> ids;
    std::vector<uint8_t> visited;
    std::vector<float> dists;

    explicit Npq(size_t cap) : capacity(cap) {}

    // queue.rs:130-171
    void insert(uint32_t id, float d) {
        if (std::isnan(d)) return;
        if (size == capacity && dists[size - 1] < d) return;
        size_t at = 0;
        while (at < size && dists[at] < d) ++at;
        if (size == capacity) {
            ids.pop_back(), visited.pop_back(), dists.pop_back();
            --size;
        }
        ids.insert(ids.begin() + at, id);
        visited.insert(visited.begin() + at, 0);
        dists.insert(dists.begin() + at, d);
        ++size;
        if (at < cursor) cursor = at;
    }

    // queue.rs:316-318
    bool has_notvisited() const { return cursor < std::min(capacity, size); }

    // queue.rs:297-313
    bool closest_notvisited(uint32_t* id) {
        if (!has_notvisited()) return false;
        const size_t cur = cursor;
        visited[cur] = 1;
        ++cursor;
        while (cursor < size && visited[cursor]) ++cursor;
        *id = ids[cur];
        return true;
    }

    // queue.rs:339-353
    void reconfigure(size_t l) {
        if (l < size) {
            ids.resize(l), visited.resize(l), dists.resize(l);
            size = l;
            cursor = std::min(cursor, l);
        }
        capacity = l;
    }
};

// inline_filter_search.rs:294-310
uint64_t compute_adaptive_l(uint64_t base_l, uint64_t visited, uint64_t matched, double max_multiplier) {
    if (matched == 0 || visited == 0) return (uint64_t)((double)base_l * max_multiplier);
    const double specificity = (double)matched / (double)visited;
    double multiplier;
    if (specificity >= 0.5) {
        multiplier = 1.0;
    } else if (specificity >= 0.1) {
        multiplier = 2.0;
    } else {
        const double neg_log10 = -std::log10(specificity);
        multiplier = std::pow(2.0, neg_log10);
    }
    // f64::clamp
    if (multiplier < 1.0) multiplier = 1.0;
    if (multiplier > max_multiplier) multiplier = max_multiplier;
    return (uint64_t)((double)base_l * multiplier);
}

struct QueryDist {
    const orc_index* idx;
    int flavour, dq;
    const void* q;
    std::vector<float> widened;
    QueryDist(const orc_index* i, const void* query, int fl) : idx(i), flavour(fl), dq(i->dtype), q(query) {
        if (idx->dtype == ORC_F16) {  // layers/full.rs:421-423
            widened.resize(idx->dim);
            const uint16_t* h = (const uint16_t*)query;
            for (uint32_t k = 0; k < idx->dim; ++k) widened[k] = orc_f16_to_f32(h[k]);
            dq = ORC_F32;
            q = widened.data();
        }
    }
    float operator()(uint32_t id) const {
        return orc_distance(flavour, dq, idx->dtype, idx->metric, q, (const char*)idx->vectors + (size_t)id * idx->row_stride, idx->dim, nullptr);
    }
};

struct Match {
    uint32_t id;
    float dist;
};

// fast_distance as a strict weak order made total: NaN after every number (-0.0 == +0.0 as floats compare)
bool before(const Match& a, const Match& b) {
    if (std::isnan(a.dist)) return false;
    if (std::isnan(b.dist)) return true;
    return a.dist < b.dist;
}

uint32_t search_one(const orc_index* idx, const void* query, uint32_t k, uint32_t l_search, uint32_t beam_width, const uint64_t* labels,
                    uint64_t mask, int match_all, uint32_t samples, double scale, const uint32_t* deleted, int flavour, uint32_t* out_ids,
                    float* out_dists, uint32_t* out_cmps, uint32_t* out_hops) {
    const QueryDist dist(idx, query, flavour);
    const uint64_t total = idx->n_points + idx->n_start;
    auto accept = [&](uint32_t id) { return match_all ? (labels[id] & mask) == mask : (labels[id] & mask) != 0; };
    // search/scratch.rs:195-208: capacity L + #start
    Npq best((size_t)l_search + idx->n_start);
    std::unordered_set<uint32_t> visited;
    std::vector<Match> matched;
    uint32_t cmps = 0, hops = 0;
    // start_point_distances: the start points count in neither cmps nor the sample
    for (uint32_t s = 0; s < idx->n_start; ++s) {
        const uint32_t id = (uint32_t)(idx->n_points + s);
        const float d = dist(id);
        visited.insert(id);
        best.insert(id, d);
        if (accept(id)) matched.push_back(Match{id, d});
    }
    if (beam_width == 0) beam_width = 1;
    uint64_t sample_visited = 0, sample_matched = 0;
    bool adjusted = false;
    std::vector<uint32_t> beam, list;
    for (;;) {
        beam.clear();
        uint32_t id;
        while (beam.size() < beam_width && best.closest_notvisited(&id)) beam.push_back(id);
        if (beam.empty()) break;
        // expand_beam (provider.rs:436-479): unvisited, in-bounds neighbours in adjacency order
        list.clear();
        for (uint32_t node : beam) {
            const uint32_t* row = idx->adj + (size_t)node * idx->adj_stride;
            for (uint32_t j = 0; j < row[0]; ++j) {
                const uint32_t n = row[1 + j];
                if (!visited.insert(n).second) continue;
                if (n >= total) continue;
                list.push_back(n);
            }
        }
        for (uint32_t n : list) {
            const float d = dist(n);
            if (accept(n)) {
                matched.push_back(Match{n, d});
                ++sample_matched;
            }
            best.insert(n, d);
            ++sample_visited;
        }
        cmps += (uint32_t)list.size();
        hops += (uint32_t)beam.size();
        if (samples && !adjusted && sample_visited >= samples) {
            adjusted = true;
            const uint64_t new_l = compute_adaptive_l(l_search, sample_visited, sample_matched, scale);
            if (new_l > l_search) best.reconfigure(new_l);
        }
    }
    std::stable_sort(matched.begin(), matched.end(), before);
    const size_t n = std::min<size_t>(matched.size(), l_search);
    uint32_t count = 0;
    for (size_t i = 0; i < n && count < k; ++i) {
        const uint32_t id = matched[i].id;
        if (id >= idx->n_points) continue;
        if (deleted && (deleted[id >> 5] >> (id & 31) & 1u)) continue;
        out_ids[count] = id;
        out_dists[count] = matched[i].dist;
        ++count;
    }
    for (uint32_t i = count; i < k; ++i) {
        out_ids[i] = 0xFFFFFFFFu;
        out_dists[i] = std::numeric_limits<float>::infinity();
    }
    *out_cmps = cmps;
    *out_hops = hops;
    return count;
}

}  // namespace

extern "C" {

uint64_t orc_compute_adaptive_l(uint64_t base_l, uint64_t visited, uint64_t matched, double max_multiplier) {
    return compute_adaptive_l(base_l, visited, matched, max_multiplier);
}

void orc_search_batch_filtered(const orc_index* idx, const void* queries, uint64_t query_stride, uint32_t nq, uint32_t k, uint32_t l_search,
                               uint32_t beam_width, const uint64_t* labels, const uint64_t* masks, int match_all, uint32_t adaptive_samples,
                               double adaptive_scale, const uint32_t* deleted, int flavour, uint32_t* out_ids, float* out_dists,
                               uint32_t* out_counts, uint32_t* out_cmps, uint32_t* out_hops) {
    for (uint32_t q = 0; q < nq; ++q) {
        out_counts[q] = search_one(idx, (const char*)queries + (size_t)q * query_stride, k, l_search, beam_width, labels, masks[q], match_all,
                                   adaptive_samples, adaptive_scale, deleted, flavour, out_ids + (size_t)q * k, out_dists + (size_t)q * k,
                                   out_cmps + q, out_hops + q);
    }
}

}  // extern "C"

// filtered_range_search.cpp — CPU restatement of the reference's filtered range search (test infrastructure only).
//
// FilteredRange::search (diskann/src/graph/search/filtered_range_search.rs:119-248) and
// filtered_range_search_internal (:259-322):
//   phase 1   inline_filter_search_internal without AdaptiveL: search_internal's traversal with a list of L + #start
//             entries, every evaluated neighbour into the list; matched: every accepted start point and neighbour, sorted
//             by distance (stable: an earlier match first among exactly equal distances, the order the device fixes;
//             the reference's sort_unstable_by leaves it open).  Not cut to L.
//   in_range  the list's first L entries and matched, those with d <= radius, sorted by (distance, id) (fast_distance_total:
//             -0.0 equal to +0.0) with adjacent equal ids removed;
//   matched   the matches with d <= radius, in their sorted order;
//   round 2   iff |in_range| >= (f32(L) * initial_slack) as usize and |matched| < max_returned: the visited set is
//             cleared and seeded with the in_range ids, which are also a FIFO frontier.  While it is not empty and
//             |matched| < max_returned: up to beam_width ids are popped and expanded (expand_beam order, accepted or
//             not); each neighbour with d <= radius * range_slack (an f32 product) is pushed onto the frontier, and
//             appended to matched if also d <= radius, accepted and |matched| < max_returned.  cmps += #neighbours,
//             hops += #beam, on the counters of phase 1.
//   output    matched.take(max_returned) in order without ids with d <= inner_radius (when given), start points and
//             deleted ids.
// Stats: cmps (start points not counted) and hops of both phases when the second round ran, else phase 1's.
//
// Built on its own into liboracle_filtered_range_search.so (oracle/filtered_range_search.mk), linked against
// liboracle.so for its distances and its NeighborPriorityQueue.  C ABI (bound by tests/filtered_range_oracle.py):
//   uint64_t orc_filtered_range_search(const orc_index* idx, const void* query, uint32_t l_search, uint32_t beam_width,
//                                      float radius, int has_inner, float inner_radius, float initial_slack,
//                                      float range_slack, uint64_t max_returned, const uint64_t* labels, uint64_t mask,
//                                      int match_all, const uint32_t* deleted, int flavour, uint32_t* out_ids,
//                                      float* out_dists, uint32_t* out_cmps, uint32_t* out_hops,
//                                      uint8_t* out_second_round);
//     One query of the index dtype; returns how many results it wrote (at most n_points).  labels: one u64 per id;
//     match_all 0: ANY (labels & mask != 0), else ALL (labels & mask == mask); max_returned 0: None; deleted: NULL or a
//     bitmap of (n_total + 31) / 32 words.  The argument checks are orc_range_check's (range_search.cpp).
#include "oracle.h"

#include <algorithm>
#include <cmath>
#include <deque>
#include <limits>
#include <unordered_set>
#include <vector>

namespace {

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

// expand_beam (provider.rs:436-479): the unvisited, in-bounds neighbours of `beam` in adjacency order; every neighbour
// enters the visited set before the bounds check
void expand(const orc_index* idx, const std::vector<uint32_t>& beam, std::unordered_set<uint32_t>& visited, std::vector<uint32_t>& out) {
    const uint64_t total = idx->n_points + idx->n_start;
    out.clear();
    for (uint32_t node : beam) {
        const uint32_t* row = idx->adj + (size_t)node * idx->adj_stride;
        for (uint32_t j = 0; j < row[0]; ++j) {
            const uint32_t n = row[1 + j];
            if (!visited.insert(n).second) continue;
            if (n >= total) continue;
            out.push_back(n);
        }
    }
}

struct Match {
    uint32_t id;
    float dist;
};

// fast_distance made total: NaN after every number (-0.0 == +0.0 as floats compare)
bool by_distance(const Match& a, const Match& b) {
    if (std::isnan(a.dist)) return false;
    if (std::isnan(b.dist)) return true;
    return a.dist < b.dist;
}

// fast_distance_total: distance, then id (no NaN reaches it)
bool by_distance_id(const Match& a, const Match& b) { return a.dist < b.dist || (!(b.dist < a.dist) && a.id < b.id); }

}  // namespace

extern "C" {

uint64_t orc_filtered_range_search(const orc_index* idx, const void* query, uint32_t l_search, uint32_t beam_width, float radius, int has_inner,
                                   float inner_radius, float initial_slack, float range_slack, uint64_t max_returned, const uint64_t* labels,
                                   uint64_t mask, int match_all, const uint32_t* deleted, int flavour, uint32_t* out_ids, float* out_dists,
                                   uint32_t* out_cmps, uint32_t* out_hops, uint8_t* out_second_round) {
    const QueryDist dist(idx, query, flavour);
    const uint64_t limit = max_returned ? max_returned : std::numeric_limits<uint64_t>::max();
    auto accept = [&](uint32_t id) { return match_all ? (labels[id] & mask) == mask : (labels[id] & mask) != 0; };

    // ---- phase 1: inline_filter_search_internal, no AdaptiveL
    orc_queue* best = orc_queue_new(l_search + idx->n_start);
    std::unordered_set<uint32_t> visited;
    std::vector<Match> matched;
    uint32_t cmps = 0, hops = 0;
    for (uint32_t s = 0; s < idx->n_start; ++s) {
        const uint32_t id = (uint32_t)(idx->n_points + s);
        const float d = dist(id);
        visited.insert(id);
        orc_queue_insert(best, id, d);
        if (accept(id)) matched.push_back(Match{id, d});
    }
    std::vector<uint32_t> beam, list;
    for (;;) {
        beam.clear();
        uint32_t id;
        float d;
        while (beam.size() < beam_width && orc_queue_closest_notvisited(best, &id, &d)) beam.push_back(id);
        if (beam.empty()) break;
        expand(idx, beam, visited, list);
        for (uint32_t n : list) {
            const float dn = dist(n);
            if (accept(n)) matched.push_back(Match{n, dn});
            orc_queue_insert(best, n, dn);
        }
        cmps += (uint32_t)list.size();
        hops += (uint32_t)beam.size();
    }
    std::stable_sort(matched.begin(), matched.end(), by_distance);

    // ---- in_range and the matches within the radius
    std::vector<Match> in_range;
    const uint32_t n_list = std::min<uint32_t>(orc_queue_size(best), l_search);
    for (uint32_t i = 0; i < n_list; ++i) {
        uint32_t id;
        float d;
        int v;
        orc_queue_get(best, i, &id, &d, &v);
        if (d <= radius) in_range.push_back(Match{id, d});
    }
    orc_queue_free(best);
    std::vector<Match> within;
    for (const Match& m : matched)
        if (m.dist <= radius) in_range.push_back(m), within.push_back(m);
    std::sort(in_range.begin(), in_range.end(), by_distance_id);
    in_range.erase(std::unique(in_range.begin(), in_range.end(), [](const Match& a, const Match& b) { return a.id == b.id; }), in_range.end());

    // ---- the second round
    const bool second = in_range.size() >= (uint64_t)((float)l_search * initial_slack) && within.size() < limit;
    if (second) {
        visited.clear();
        std::deque<uint32_t> frontier;
        for (const Match& m : in_range) visited.insert(m.id), frontier.push_back(m.id);
        const float bound = radius * range_slack;
        while (!frontier.empty() && within.size() < limit) {
            beam.clear();
            while (!frontier.empty() && beam.size() < beam_width) beam.push_back(frontier.front()), frontier.pop_front();
            expand(idx, beam, visited, list);
            for (uint32_t n : list) {
                const float d = dist(n);
                if (!(d <= bound)) continue;
                frontier.push_back(n);
                if (d <= radius && accept(n) && within.size() < limit) within.push_back(Match{n, d});
            }
            cmps += (uint32_t)list.size();
            hops += (uint32_t)beam.size();
        }
    }

    // ---- output: matched.take(max_returned) without the inner radius, start points and deleted ids
    uint64_t count = 0;
    const size_t n_out = (size_t)std::min<uint64_t>(within.size(), limit);
    for (size_t i = 0; i < n_out; ++i) {
        const uint32_t id = within[i].id;
        const float d = within[i].dist;
        if (has_inner && d <= inner_radius) continue;
        if (id >= idx->n_points) continue;
        if (deleted && (deleted[id >> 5] >> (id & 31) & 1u)) continue;
        out_ids[count] = id;
        out_dists[count] = d;
        ++count;
    }
    *out_cmps = cmps;
    *out_hops = hops;
    *out_second_round = second ? 1 : 0;
    return count;
}

}  // extern "C"

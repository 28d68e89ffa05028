// range_table.cpp — the reference's Range::search over any traversal distance (test infrastructure only).
//
// Range::search (diskann/src/graph/search/range_search.rs:255-469) is generic over the search strategy: both phases
// read the strategy's accessor, so every distance — the phase-1 traversal, the `d <= radius` test that builds
// in_range and the second round's `d <= radius * range_slack` test — is the accessor's.  Here those distances come
// from a table the caller fills (a quantized store's distances to every id).  The output is the strategy's
// post-processor behind a DistanceFiltered buffer (inner_radius < d <= radius):
//   rerank == 0  Pipeline<FilterStartPoints, RemoveDeletedIdsAndCopy>: in_range in insertion order without start points
//                and deleted ids, filtered on the table's distances (orc_range_search's output rule);
//   rerank != 0  Pipeline<FilterStartPoints, Rerank> (providers inmem/product.rs:391-401, full_precision.rs:356-399):
//                start points and deleted ids dropped, every other id's full-precision Distance<T, T> to the query,
//                the entries outside (inner_radius, radius] of it dropped, the rest sorted by it stably (the
//                reference's sort_unstable_by leaves ties unspecified and has no order with NaN: filtering first and
//                sorting stably gives its result wherever that is defined).
// The phase-1 list is liboracle's NeighborPriorityQueue through its C ABI, as in orc_range_search.
//
// Built on its own into liboracle_range_table.so (oracle/range_table.mk), linked against liboracle.so.  C ABI (bound
// by tests/range_table_oracle.py):
//   uint64_t orc_range_search_table(const orc_index* idx, const float* dists, const void* query, uint32_t l_search,
//                                   uint32_t beam_width, float radius, int has_inner, float inner_radius,
//                                   float initial_slack, float range_slack, uint64_t max_returned,
//                                   const uint32_t* deleted, int rerank, int flavour, uint32_t* out_ids,
//                                   float* out_dists, uint32_t* out_cmps, uint32_t* out_hops, uint8_t* out_second_round);
//     One query: the traversal distance to id i is dists[i] (n_points + n_start entries); query (index dtype) is read
//     only with rerank.  Arguments, deleted, outputs and the returned count as orc_range_search.
#include "oracle.h"

#include <algorithm>
#include <limits>
#include <unordered_set>
#include <utility>
#include <vector>

namespace {

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

bool in_band(float d, float radius, int has_inner, float inner_radius) { return !(has_inner && d <= inner_radius) && d <= radius; }

}  // namespace

extern "C" {

uint64_t orc_range_search_table(const orc_index* idx, const float* dist, const void* query, uint32_t l_search, uint32_t beam_width, float radius,
                                int has_inner, float inner_radius, float initial_slack, float range_slack, uint64_t max_returned,
                                const uint32_t* deleted, int rerank, int flavour, uint32_t* out_ids, float* out_dists, uint32_t* out_cmps,
                                uint32_t* out_hops, uint8_t* out_second_round) {
    const uint64_t limit = max_returned ? max_returned : std::numeric_limits<uint64_t>::max();

    // ---- phase 1: search_internal over L + #start entries
    orc_queue* best = orc_queue_new(l_search + idx->n_start);
    std::unordered_set<uint32_t> visited;
    uint32_t cmps = 0, hops = 0;
    for (uint32_t s = 0; s < idx->n_start; ++s) {
        const uint32_t id = (uint32_t)(idx->n_points + s);
        visited.insert(id);
        orc_queue_insert(best, id, dist[id]);
        ++cmps;
    }
    std::vector<uint32_t> beam, list;
    while (orc_queue_has_notvisited(best)) {
        beam.clear();
        uint32_t id;
        float d;
        while (beam.size() < beam_width && orc_queue_closest_notvisited(best, &id, &d)) beam.push_back(id);
        expand(idx, beam, visited, list);
        for (uint32_t n : list) orc_queue_insert(best, n, dist[n]);
        cmps += (uint32_t)list.size();
        hops += (uint32_t)beam.size();
    }

    // ---- in_range: the list's first L entries within the radius
    std::vector<uint32_t> in_ids;
    std::vector<float> in_d;
    const uint32_t n_list = std::min<uint32_t>(orc_queue_size(best), l_search);
    for (uint32_t i = 0; i < n_list; ++i) {
        uint32_t id;
        float d;
        int v;
        orc_queue_get(best, i, &id, &d, &v);
        if (d <= radius) in_ids.push_back(id), in_d.push_back(d);
    }
    orc_queue_free(best);

    // ---- the second round
    const uint32_t phase1_hops = hops;
    const bool second = in_ids.size() >= (uint64_t)((float)l_search * initial_slack) && in_ids.size() < limit;
    if (second) {
        visited.clear();
        for (uint32_t id : in_ids) visited.insert(id);
        const float bound = radius * range_slack;
        size_t front = 0;
        while (front < in_ids.size() && in_ids.size() < limit) {
            beam.clear();
            while (beam.size() < beam_width && front < in_ids.size()) beam.push_back(in_ids[front++]);
            expand(idx, beam, visited, list);
            for (uint32_t n : list) {
                if (dist[n] <= bound && in_ids.size() < limit) in_ids.push_back(n), in_d.push_back(dist[n]);
            }
            hops += (uint32_t)beam.size();
        }
        hops += phase1_hops;  // scratch.hops (phase 1 + phase 2) added to phase 1's hops
    }

    // ---- the post-processor: start points and deleted ids dropped, then the distance filter (after the rerank's
    // distances, and before its stable sort)
    std::vector<std::pair<float, uint32_t>> out;
    for (size_t i = 0; i < in_ids.size(); ++i) {
        const uint32_t id = in_ids[i];
        if (id >= idx->n_points) continue;
        if (deleted && (deleted[id >> 5] >> (id & 31) & 1u)) continue;
        float d = in_d[i];
        if (rerank) d = orc_distance(flavour, idx->dtype, idx->dtype, idx->metric, query, (const char*)idx->vectors + (size_t)id * idx->row_stride,
                                     idx->dim, nullptr);
        if (in_band(d, radius, has_inner, inner_radius)) out.emplace_back(d, id);
    }
    if (rerank) std::stable_sort(out.begin(), out.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
    for (size_t i = 0; i < out.size(); ++i) out_ids[i] = out[i].second, out_dists[i] = out[i].first;
    *out_cmps = cmps;
    *out_hops = hops;
    *out_second_round = second ? 1 : 0;
    return out.size();
}

}  // extern "C"

// range_search.cpp — CPU restatement of the reference's range search (test infrastructure only).
//
// Range::search and range_search_internal (diskann/src/graph/search/range_search.rs:255-469):
//   phase 1   search_internal (diskann/src/graph/index.rs:1933-2000) with a list of L + #start entries;
//   in_range  the first L entries of the list with distance <= radius, in list order (start points and deleted ids kept);
//   round 2   iff |in_range| >= (f32(L) * initial_slack) as usize and |in_range| < max_returned: the visited set is
//             cleared and re-seeded with the in_range ids, and a FIFO frontier (the unconsumed suffix of in_range) is
//             expanded up to beam_width ids at a time in expand_beam order; each new neighbour with
//             d <= radius * range_slack (an f32 product) is appended while |in_range| < max_returned;
//   output    in_range in insertion order without start points, deleted ids, ids with d <= inner_radius (when given)
//             and ids with d > radius.
// Stats: cmps are phase 1's; hops are phase1 + (phase1 + phase2) when the second round ran (scratch.hops is cumulative
// and the reference adds it to phase 1's again), else phase 1's.
//
// Built on its own into liboracle_range_search.so (oracle/range_search.mk), linked against liboracle.so for its
// distances and its NeighborPriorityQueue.  C ABI (bound by tests/range_oracle.py):
//   int orc_range_check(uint32_t l_search, uint32_t beam_width, uint64_t max_returned, float radius, int has_inner,
//                       float inner_radius, float initial_slack, float range_slack);
//     Range::validate_and_create's checks in its order: 0 valid, else 1 BeamWidthZero, 2 LZero,
//     3 MaxReturnedLessThanInitialL, 4 StartingListSlackValueError, 5 RangeSearchSlackValueError, 6 InnerRadiusValueError.
//     max_returned 0 stands for None.
//   uint64_t orc_range_search(const orc_index* idx, const void* query, uint32_t l_search, uint32_t beam_width, float radius,
//                             int has_inner, float inner_radius, float initial_slack, float range_slack,
//                             uint64_t max_returned, const uint32_t* deleted, int flavour, uint32_t* out_ids,
//                             float* out_dists, uint32_t* out_cmps, uint32_t* out_hops, uint8_t* out_second_round);
//     One query of the index dtype; returns how many results it wrote (at most n_points: out_* hold that many).
//     deleted: NULL or a bitmap of (n_total + 31) / 32 words, bit i of word i / 32 for id i.
#include "oracle.h"

#include <cmath>
#include <cstring>
#include <limits>
#include <unordered_set>
#include <vector>

namespace {

// the full-precision query distance (f16 queries widened once, layers/full.rs:421-423)
struct QueryDist {
    const orc_index* idx;
    int flavour, dq;
    const void* q;
    std::vector<float> widened;
    QueryDist(const orc_index* i, const void* query, int fl) : idx(i), flavour(fl), dq(i->dtype), q(query) {
        if (idx->dtype == ORC_F16) {
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

}  // namespace

extern "C" {

int orc_range_check(uint32_t l_search, uint32_t beam_width, uint64_t max_returned, float radius, int has_inner, float inner_radius,
                    float initial_slack, float range_slack) {
    if (beam_width == 0) return 1;
    if (l_search == 0) return 2;
    if (max_returned != 0 && max_returned < l_search) return 3;
    if (!(initial_slack >= 0.0f && initial_slack <= 1.0f)) return 4;  // !(0.0..=1.0).contains(): NaN fails
    if (range_slack < 1.0f) return 5;                                  // NaN passes
    if (has_inner && inner_radius > radius) return 6;                  // NaN passes
    return 0;
}

uint64_t orc_range_search(const orc_index* idx, const void* query, uint32_t l_search, uint32_t beam_width, float radius, int has_inner,
                          float inner_radius, float initial_slack, float range_slack, uint64_t max_returned, const uint32_t* deleted,
                          int flavour, uint32_t* out_ids, float* out_dists, uint32_t* out_cmps, uint32_t* out_hops,
                          uint8_t* out_second_round) {
    const QueryDist dist(idx, query, flavour);
    const uint64_t limit = max_returned ? max_returned : std::numeric_limits<uint64_t>::max();

    // ---- phase 1: search_internal over L + #start entries
    orc_queue* best = orc_queue_new(l_search + idx->n_start);
    std::unordered_set<uint32_t> visited;
    uint32_t cmps = 0, hops = 0;
    for (uint32_t s = 0; s < idx->n_start; ++s) {
        const uint32_t id = (uint32_t)(idx->n_points + s);
        visited.insert(id);
        orc_queue_insert(best, id, dist(id));
        ++cmps;
    }
    std::vector<uint32_t> beam, list;
    while (orc_queue_has_notvisited(best)) {
        beam.clear();
        uint32_t id;
        float d;
        while (beam.size() < beam_width && orc_queue_closest_notvisited(best, &id, &d)) beam.push_back(id);
        expand(idx, beam, visited, list);
        std::vector<float> ds;
        for (uint32_t n : list) ds.push_back(dist(n));
        for (size_t i = 0; i < list.size(); ++i) orc_queue_insert(best, list[i], ds[i]);
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
                const float d = dist(n);
                if (d <= bound && in_ids.size() < limit) in_ids.push_back(n), in_d.push_back(d);
            }
            hops += (uint32_t)beam.size();
        }
        hops += phase1_hops;  // scratch.hops (phase 1 + phase 2) added to phase 1's hops
    }

    // ---- output: start points, deleted ids, the inner radius and the radius filtered out, in insertion order
    uint64_t count = 0;
    for (size_t i = 0; i < in_ids.size(); ++i) {
        const uint32_t id = in_ids[i];
        const float d = in_d[i];
        if (id >= idx->n_points) continue;
        if (deleted && (deleted[id >> 5] >> (id & 31) & 1u)) continue;
        if (has_inner && d <= inner_radius) continue;
        if (!(d <= radius)) continue;
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
